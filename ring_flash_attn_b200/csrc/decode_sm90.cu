// Split-KV ("flash-decoding") attention for sm_90a: a few new query tokens against a long K/V cache.
//
// One CTA = (split of the key range) x (64-row tile of packed query rows) x (sequence, kv head).  The query rows of
// one kv head are packed into the wgmma M dimension as (token t, head-in-group g) -> row t * G + g, so that a GQA
// group reads each K/V tile once instead of once per query head.  The CTA streams the 128-key tiles of its split
// with TMA through an mbarrier ring and runs the forward kernel's online softmax; it writes a normalised fp32
// partial out and its lse.  decode_combine_kernel merges partials (over the splits of one rank, and again over the
// gathered partials of all ranks): lse = logsumexp(lse_p), out = sum_p exp(lse_p - lse) out_p, in partial order.
//
// Roles (160 threads): warpgroup 0 computes (S = Q K^T, mask, softmax, O += P V, epilogue); warp 4 is the TMA
// producer (one thread).
//
// e4m3 caches (288 threads): the producer (warp 8) TMA-loads e4m3 tiles into a ring of fp8 slots, and a converter
// warpgroup (warps 4-7) widens each one, exactly, into the bf16 / fp16 slot layout TMA fills for a bf16 / fp16 cache,
// then arrives on that slot's kv_full barrier.  The compute warpgroup is the same code; k_descale[b, kv head]
// multiplies its scale_log2 once and v_descale[b, kv head] its 1 / l.  So with power-of-two descales 2^a, 2^c the
// result is bitwise the bf16 / fp16 kernel's on the widened cache with softmax_scale * 2^a, out scaled by 2^c.
//
// e4m3 queries (kQ8, over e4m3 caches only; 288 threads): wgmma takes 8-bit operands K-major, and the e4m3 K tile TMA
// writes is already K-major for Q K^T, so S = Q K^T is an m64n128k32 e4m3 wgmma with A = the e4m3 Q tile (kD-byte
// rows in the swizzle of the K tile: 128-byte at kD = 128, 64-byte at 64) and B = the fp8 K slot as TMA filled it.
// Only V (MN-major in P V) is widened.  The fp8 ring still alternates K, V, K, V (the producer is unchanged); with
// an even slot count K always lands in even slots, which the compute warps release once the S wgmma has completed,
// and V in odd ones, which the converter widens into a bf16 ring of V slots only and releases.  Both kinds keep four
// arrivals per f8_empty.  q_descale[b, kv head] joins k_descale in t2 = scale_log2 * q_descale * k_descale; P and
// V are bf16 and the rest of the softmax is unchanged.  Shared memory at kD = 128: Q 8 KB + 6 fp8 slots of 16 KB
// + 3 bf16 V slots of 32 KB + barriers = 206848 bytes with the slack (half of each at kD = 64: 104448).
//
// Varlen queries (cu_seqlens_q): sequence b brings n_b = cu[b + 1] - cu[b] tokens.  The grid is (split, tile slot,
// kv head) instead, with decode_tile_slots() slots, a bound from shapes on sum_b ceil(n_b * G / 64); each CTA finds
// its (sequence, row tile) by a warp-wide prefix sum over cu, and slots past the last real tile exit at once.
// Everything after that mapping is the uniform code with the sequence's own row base and count.
//
// Rotary embeddings (rotary_cos set): the compute warpgroup rotates the 16-byte chunks of each Q row below rotary_dim
// as it loads the Q tile, before the key loop, and the append kernels rotate K before they store it.  The key loop,
// the producer, the converter and the combine do not see it.
//
// Visibility: key j of the shard is visible to query token t iff j < seqlens[b] + n_vis(t), where n_vis(t) counts
// the keys this call appended to this shard that t may see (0 on every rank but the append rank; t + 1 when causal,
// the sequence's token count otherwise).  Cache rows at or past that limit are never read into a result: their K
// columns are masked to -inf and their V rows are zeroed in shared memory before P V (the cache may hold anything
// there, NaN included).
//
// Tree masks (kTree, launched when tree_mask is set; causal): n_vis(t) is the sequence's token count for every row, so
// kmax, the split ranges and the V-row zeroing are those of a non-causal call, and the tiles holding appended keys
// (key0 + kTile > seqlen, at most two per sequence) then set S = -inf where the row's mask byte for key
// u = key0 + c - seqlen is 0.  Rotary positions of new tokens come from one helper (new_token_pos), the mask row's
// depth with a mask.  The prefix pass masks nothing (its keys are visible to every row); its kTree instantiation,
// launched with a mask and rotary, differs only in the rotary positions.  Without a mask the kernels are the ones
// compiled before tree masks existed.
//
// Cache slots and left padding (contiguous caches): sequence b's keys live in slot cache_batch_idx[b] and start at
// row lp = cache_leftpad[b].  Each CTA resolves both once and then runs on keys relative to lp: seqlens[b] - lp valid
// rows under a capacity of S_cap - lp, so the key loop, masks and split ranges are those of a plain call on the
// slot shifted down by lp rows.  Only the producer's row coordinate (slot * S_cap + lp + key) and the append's target
// row see the slot and the pad.  Tile rows past the last visible key may reach into the next slot or past the tensor
// (TMA fills those with zeros); they are discarded like any row at or past the limit.
//
// Shared prefixes (kPrefix, decode_prefix_launch): the n = B / P consecutive sequences of group i share prefix i, a
// (P, P_cap, Hkv, D) cache read by a second pass.  Its grid is (prefix split, row-tile slot, P x Hkv): a CTA takes 64
// consecutive packed rows of the group's (sequence, token, head-in-group) rows, which are rows [b0 * sq, (b0 + n) *
// sq) of a uniform q or [cu[b0], cu[b0 + n]) of a varlen one, so the group's samples share each prefix K / V tile.
// Everything runs as a call with cache slot i, seqlens[i] valid rows, no append (every prefix key is visible to every
// row) and descales [i, kv head]; only the rotary position and the lse address need a row's own sequence and token.
// Its partials go to slabs after the suffix pass's, and the one combine merges both.  A paged prefix (page_size set)
// is a pool of pages named by a (P, max_prefix_blocks) block table, P_cap = max_prefix_blocks * page_size: with b the
// prefix, the paged producer indexes the table by prefix exactly as the suffix pass indexes it by sequence, so the pool
// may be the suffix pass's own pool, with the prompt's pages in one table and each sample's pages in the other.
#include <limits.h>
#include <math_constants.h>

#include <type_traits>

#include "decode.h"
#include "sm90_ptx.cuh"

namespace rfa {

namespace dec {

constexpr int kTile = 128;    // keys per K / V tile
constexpr int kRows = 64;     // packed query rows per CTA (one wgmma M)
constexpr int kStages = 6;    // K/V ring slots (one key tile takes two: K, then V)
constexpr int kStagesFp8 = 4;  // the same with an e4m3 cache, whose kF8Stages fp8 slots take the rest of the memory
constexpr int kF8Stages = 4;
constexpr int kF8StagesQ8 = 6;  // e4m3 queries: fp8 K / V slots (even: K in the even slots, V in the odd ones)
constexpr int kVStagesQ8 = 3;   // e4m3 queries: bf16 slots, V only
static_assert(kF8StagesQ8 % 2 == 0, "K and V must keep their slot parity");
constexpr int kThreads = 160;  // one compute warpgroup + one producer warp
constexpr int kThreadsFp8 = 288;  // + one converter warpgroup
constexpr int kKHalfBytes = kTile * 128;  // one 64-element-wide (128-byte) swizzled K / V sub-tile
constexpr int kQHalfBytes = kRows * 128;  // the same for the query tile
constexpr int kBarBytes = 1024;           // the ring's mbarriers
// Tree masks: one 32-bit word per (tile w, row half h, compute thread), the thread's hidden columns of the two key
// tiles that can hold appended keys, so the key loop reads one word instead of 32 mask bytes per row
constexpr int kTreeHideBytes = 2 * 2 * 128 * 4;

template <int kD, bool kFp8, bool kQ8, bool kTree = false>
constexpr int smem_bytes() {
  constexpr int tree = kTree ? kTreeHideBytes : 0;
  if constexpr (kQ8)
    return kRows * kD + kF8StagesQ8 * kTile * kD + kVStagesQ8 * kTile * kD * 2 + kBarBytes + tree +
           1024 /*align slack*/;
  return kRows * kD * 2 + (kFp8 ? kStagesFp8 * kTile * kD * 3 : kStages * kTile * kD * 2) + kBarBytes + tree +
         1024 /*align slack*/;
}

template <int kWide, int kLoad>
struct RingBarriers {
  uint64_t kv_full[kWide];  // the bf16 / fp16 slots the compute warpgroup reads (V only with e4m3 queries)
  uint64_t kv_empty[kWide];
  uint64_t f8_full[kLoad];  // e4m3 caches: the fp8 slots
  uint64_t f8_empty[kLoad];
};
template <bool kQ8>
using Barriers = std::conditional_t<kQ8, RingBarriers<kVStagesQ8, kF8StagesQ8>, RingBarriers<kStages, kF8Stages>>;

// The ring the TMA producer fills: bf16 / fp16 slots of kD / 64 128-byte-swizzled sub-tiles of 128-byte rows, or
// e4m3 slots of one sub-tile of kD-byte rows (128-byte swizzle at kD = 128, 64-byte at kD = 64).
template <int kD, bool kFp8, bool kQ8>
struct LoadRing {
  static constexpr int kSlots = kQ8 ? kF8StagesQ8 : (kFp8 ? kF8Stages : kStages);
  static constexpr int kSubTiles = kFp8 ? 1 : kD / 64;
  static constexpr int kRowBytes = kFp8 ? kD : 128;  // bytes per row of one sub-tile
  static constexpr int kSlotBytes = kTile * kSubTiles * kRowBytes;
};

// Keys of the shard visible to token t of a sequence with n_q new tokens (see the file comment), at most cap, all
// counted from the sequence's first key row.  With a tree mask (kTree) every row gets all n_q appended keys here, and
// the mask step of the key loop hides the ones its row may not see.
template <bool kTree>
__device__ __forceinline__ int key_limit(const DecodeParams& p, int seqlen, int cap, int n_q, int t) {
  const int n_vis = p.n_new == 0 ? 0 : (p.causal && !kTree ? t + 1 : n_q);
  const int lim = seqlen + n_vis;
  return lim < cap ? lim : cap;
}

__device__ __forceinline__ int clamp_to(int x, int lo, int hi) { return x < lo ? lo : (x > hi ? hi : x); }

// Sequence b's new tokens: first packed row (x) and count (y).  Varlen offsets are clamped to [0, total_q] and counts
// to [0, sq], so rows [x, x + y) always lie inside q, k_new / v_new and the partial buffer.
__device__ __forceinline__ int2 q_rows(const DecodeParams& p, int b) {
  if (p.cu_seqlens_q == nullptr) return make_int2(b * p.sq, p.sq);
  const int lo = clamp_to(__ldg(p.cu_seqlens_q + b), 0, p.total_q);
  const int hi = clamp_to(__ldg(p.cu_seqlens_q + b + 1), 0, p.total_q);
  return make_int2(lo, clamp_to(hi - lo, 0, p.sq));
}

// Rotary position of new token t of sequence b (t = 0 for every query token of a non-causal call), clamped to the
// tables: a bad rotary_seqlens gives a wrong rotation, never a read outside them.
__device__ __forceinline__ int rotary_pos(const DecodeParams& p, int b, int t) {
  const long long x = static_cast<long long>(__ldg(p.rotary_seqlens + b)) + t;
  return x < 0 ? 0 : (x >= p.seqlen_ro ? p.seqlen_ro - 1 : static_cast<int>(x));
}

// Offset from rotary_seqlens[b] of new token t of sequence b: with a tree mask, its depth (the nonzero bytes among
// the first n_b of its mask row, minus one; 0 for an empty row), for its query and its key alike; otherwise t for a
// key or a causal query token, and 0 for a query token of a non-causal call.  kMaybeTree = false: no mask.
template <bool kMaybeTree>
__device__ __forceinline__ int new_token_pos(const DecodeParams& p, int b, int t, bool key) {
  if (!kMaybeTree || p.tree_mask == nullptr) return key || p.causal ? t : 0;
  const int2 r = q_rows(p, b);
  const uint8_t* row = p.tree_mask + static_cast<long long>(r.x + t) * p.sq;
  int n = 0;
  for (int u = 0; u < r.y; ++u) n += __ldg(row + u) != 0;
  return n > 0 ? n - 1 : 0;
}

template <typename T>
__device__ __forceinline__ T round_to(float x) {
  if constexpr (std::is_same_v<T, __half>) return __float2half_rn(x);
  else return __float2bfloat16_rn(x);
}

// The rotated 16-byte chunk c (elements 8c .. 8c + 7, all below rotary_dim) of a q / k row `row` whose chunk c holds
// `val`, at table row pos: y = x * cos -+ x_pair * sin, every operand widened to fp32, each product and the sum rounded
// to fp32 (no FMA), the result rounded to nearest even into T.  Interleaved, the pairs (2i, 2i + 1) lie inside the
// chunk; otherwise chunk c pairs with the chunk rotary_half / 8 away, 16-byte aligned since rotary_half % 8 == 0.
template <typename T>
__device__ __forceinline__ uint4 rotate_chunk(uint4 val, const T* row, int c, int pos, const DecodeParams& p) {
  const int h = p.rotary_half;
  const T* cos_row = static_cast<const T*>(p.rotary_cos) + static_cast<long long>(pos) * h;
  const T* sin_row = static_cast<const T*>(p.rotary_sin) + static_cast<long long>(pos) * h;
  const T* x = reinterpret_cast<const T*>(&val);
  uint4 res;
  T* y = reinterpret_cast<T*>(&res);
  if (p.rotary_interleaved) {
    const uint2 cr = __ldg(reinterpret_cast<const uint2*>(cos_row + 4 * c));
    const uint2 sr = __ldg(reinterpret_cast<const uint2*>(sin_row + 4 * c));
    const T* cv = reinterpret_cast<const T*>(&cr);
    const T* sv = reinterpret_cast<const T*>(&sr);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float x0 = static_cast<float>(x[2 * i]), x1 = static_cast<float>(x[2 * i + 1]);
      const float co = static_cast<float>(cv[i]), si = static_cast<float>(sv[i]);
      y[2 * i] = round_to<T>(__fsub_rn(__fmul_rn(x0, co), __fmul_rn(x1, si)));
      y[2 * i + 1] = round_to<T>(__fadd_rn(__fmul_rn(x1, co), __fmul_rn(x0, si)));
    }
  } else {
    const int half_chunks = h / 8;
    const bool first = c < half_chunks;  // y[i] = x[i] c - x[i + h] s, else y[i + h] = x[i + h] c + x[i] s
    const int tc = first ? c : c - half_chunks;  // chunk of the tables
    const uint4 pr = *reinterpret_cast<const uint4*>(row + 8 * (first ? c + half_chunks : tc));
    const uint4 cr = __ldg(reinterpret_cast<const uint4*>(cos_row + 8 * tc));
    const uint4 sr = __ldg(reinterpret_cast<const uint4*>(sin_row + 8 * tc));
    const T* xp = reinterpret_cast<const T*>(&pr);
    const T* cv = reinterpret_cast<const T*>(&cr);
    const T* sv = reinterpret_cast<const T*>(&sr);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float a = __fmul_rn(static_cast<float>(x[i]), static_cast<float>(cv[i]));
      const float b = __fmul_rn(static_cast<float>(xp[i]), static_cast<float>(sv[i]));
      y[i] = round_to<T>(first ? __fsub_rn(a, b) : __fadd_rn(a, b));
    }
  }
  return res;
}

// Varlen schedule: tile slot -> (sequence b, row tile), by a prefix sum over the sequences' row-tile counts
// ceil(n_b * G / 64), 32 sequences per step (one per lane).  Run by each warp on its own; every lane gets the same
// answer.  False for a slot past the last real tile.
__device__ __forceinline__ bool varlen_tile(const DecodeParams& p, int slot, int group, int& b, int& tile,
                                            int2& rows) {
  const int lane = threadIdx.x & 31;
  int base = 0;  // tiles of the sequences before this step's 32
  for (int c = 0; c < p.batch; c += 32) {
    const int i = c + lane;
    const int2 r = i < p.batch ? q_rows(p, i) : make_int2(0, 0);
    const int tiles = (r.y * group + kRows - 1) / kRows;
    int incl = tiles;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int x = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += x;
    }
    const int excl = base + incl - tiles;
    const unsigned hit = __ballot_sync(0xffffffffu, slot >= excl && slot < base + incl);
    if (hit != 0u) {
      const int src = __ffs(hit) - 1;
      b = c + src;
      tile = slot - __shfl_sync(0xffffffffu, excl, src);
      rows = make_int2(__shfl_sync(0xffffffffu, r.x, src), __shfl_sync(0xffffffffu, r.y, src));
      return true;
    }
    base += __shfl_sync(0xffffffffu, incl, 31);
  }
  return false;
}

// Shared-prefix pass: the group of sequences [b0, b0 + prefix_n): its first packed query row (x) and row count (y),
// clamped like q_rows, so rows [x, x + y) always lie inside q and the partial buffer.
__device__ __forceinline__ int2 prefix_rows(const DecodeParams& p, int b0) {
  if (p.cu_seqlens_q == nullptr) return make_int2(b0 * p.sq, p.prefix_n * p.sq);
  const int lo = clamp_to(__ldg(p.cu_seqlens_q + b0), 0, p.total_q);
  const int hi = clamp_to(__ldg(p.cu_seqlens_q + b0 + p.prefix_n), 0, p.total_q);
  return make_int2(lo, hi > lo ? hi - lo : 0);
}

// The sequence b and token t of packed query row `row` of the group starting at sequence b0: the last sequence of the
// group whose first row is at or before `row` (a binary search over cu when varlen).
__device__ __forceinline__ void prefix_token(const DecodeParams& p, int b0, int row, int& b, int& t) {
  if (p.cu_seqlens_q == nullptr) {
    b = row / p.sq;
    t = row - b * p.sq;
    return;
  }
  int lo = b0, hi = b0 + p.prefix_n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (clamp_to(__ldg(p.cu_seqlens_q + mid), 0, p.total_q) <= row) lo = mid;
    else hi = mid - 1;
  }
  b = lo;
  t = row - clamp_to(__ldg(p.cu_seqlens_q + lo), 0, p.total_q);
}

// TMA producer over a paged cache, run by the whole producer warp.  A 128-key tile is one page (page_size >= 128,
// the tile starts at row key0 % page_size of it) or 128 / page_size pages, each loaded as its own box of page_size
// rows into the matching rows of the slot: an offset of i * page_size * 128 bytes stays 1024-byte aligned, so the
// 128-byte swizzle is the one a single 128-row box writes.  Pages past the last visible key (kmax) are neither
// looked up nor loaded, and neither are pages whose id lies outside the pool (a caller error); the slot's expected
// byte count covers only the boxes issued.  The rows left unwritten hold an older tile, and the compute warpgroup
// already discards every row at or past kmax (K columns masked, V rows zeroed), exactly as for a contiguous cache.
// Table entries are read 32 at a time, one per lane, a window ahead of use, and broadcast with shuffles.  The e4m3
// ring works the same way: a box of page_size < 128 rows is page_size * kD bytes, a multiple of 1024, so every box
// starts on a swizzle period of the fp8 layout too.
template <int kD, bool kFp8, bool kQ8>
__device__ __forceinline__ void produce_paged(const CUtensorMap* tm_k, const CUtensorMap* tm_v, uint64_t* full,
                                              uint64_t* empty, uint8_t* smem_kv, const DecodeParams& p, int b,
                                              int kv_head, int j0, int n_tiles, int kmax) {
  using L = LoadRing<kD, kFp8, kQ8>;
  constexpr int kSubTiles = L::kSubTiles;
  constexpr int kSlotBytes = L::kSlotBytes;
  const int lane = threadIdx.x & 31;
  const int ps = p.page_size;
  const int box = ps < kTile ? ps : kTile;  // rows per TMA box, as in the tensor maps
  const int n_sub = kTile / box;            // pages per tile: 8, 4, 2 or 1
  const int* table = p.block_table + b * p.bt_stride;
  const int last = (kmax - 1) / ps;  // last page holding a visible key; later entries are never read
  auto entry = [&](int i) { return i <= last ? __ldg(table + i) : -1; };
  int win = j0 * kTile / ps;  // first page of the split; cur holds table entries [win, win + 32), nxt the next 32
  int cur = entry(win + lane), nxt = entry(win + 32 + lane);
  uint32_t slot = 0, phase = 0;
  for (int jj = 0; jj < n_tiles; ++jj) {
    const int key0 = (j0 + jj) * kTile;
    const int pg0 = key0 / ps;  // first page of the tile
    if (pg0 - win >= 32) {      // n_sub divides 32 and win starts at a tile's first page: a tile never straddles
      win += 32;
      cur = nxt;
      nxt = entry(win + 32 + lane);
    }
    // lane i < n_sub: sub-tile i, i.e. keys [key0 + i * box, key0 + (i + 1) * box)
    const int page = __shfl_sync(0xffffffffu, cur, (pg0 - win + lane) & 31);
    const bool live = lane < n_sub && key0 + lane * box < kmax && page >= 0 && page < p.num_pages;
    const int row = live ? page * ps + (key0 - pg0 * ps) : 0;
    const unsigned loads = __ballot_sync(0xffffffffu, live);
    const uint32_t tx = __popc(loads) * box * L::kRowBytes * kSubTiles;
    for (int kv = 0; kv < 2; ++kv) {
      uint8_t* dst = smem_kv + slot * kSlotBytes;
      if (lane == 0) {
        mbar_wait(&empty[slot], phase ^ 1);
        mbar_arrive_expect_tx(&full[slot], tx);
      }
      for (int i = 0; i < n_sub; ++i) {
        const int r = __shfl_sync(0xffffffffu, row, i);
        if (lane == 0 && (loads >> i & 1u)) {
#pragma unroll
          for (int h = 0; h < kSubTiles; ++h)
            tma_load_3d(dst + h * kKHalfBytes + i * box * L::kRowBytes, kv == 0 ? tm_k : tm_v, &full[slot], 64 * h,
                        kv_head, r);
        }
      }
      if (++slot == L::kSlots) {
        slot = 0;
        phase ^= 1;
      }
    }
  }
}

// two e4m3 (low 16 bits of x) -> two T in one word, exactly
template <typename T>
__device__ __forceinline__ uint32_t widen2(uint32_t x) {
  if constexpr (std::is_same_v<T, __half>) return e4m3x2_to_f16x2(x);
  else return e4m3x2_to_bf16x2(x);
}

// One e4m3 K / V tile as TMA wrote it (kTile rows of kD bytes; 128-byte swizzle at kD = 128, 64-byte at kD = 64)
// -> the T tile TMA writes for a bf16 / fp16 cache (kD / 64 sub-tiles of 128-byte swizzled rows), by the 128 threads
// of the converter warpgroup.  16 e4m3 values (one 16-byte chunk) per thread and step; the 8 threads of one 128-byte
// store phase take chunks 0-3 of two adjacent rows, whose swizzled 16-byte positions are then all distinct.
template <typename T, int kD>
__device__ __forceinline__ void widen_tile(const uint8_t* src, uint8_t* dst, int ctid) {
  constexpr int kChunks = kD / 16;  // e4m3 chunks per row
#pragma unroll
  for (int i = 0; i < kTile * kChunks / 128; ++i) {
    const int idx = ctid + 128 * i;
    const int r = kD == 128 ? ((idx >> 4) << 1) | ((idx >> 2) & 1) : idx >> 2;
    const int c = kD == 128 ? (idx & 3) | ((idx >> 1) & 4) : idx & 3;
    const int phys = kD == 128 ? c ^ (r & 7) : c ^ ((r >> 1) & 3);
    const uint4 x = *reinterpret_cast<const uint4*>(src + r * kD + (phys << 4));
    uint4 lo, hi;
    lo.x = widen2<T>(x.x);
    lo.y = widen2<T>(x.x >> 16);
    lo.z = widen2<T>(x.y);
    lo.w = widen2<T>(x.y >> 16);
    hi.x = widen2<T>(x.z);
    hi.y = widen2<T>(x.z >> 16);
    hi.z = widen2<T>(x.w);
    hi.w = widen2<T>(x.w >> 16);
    uint8_t* row = dst + (c >> 2) * kKHalfBytes + r * 128;
    const int c0 = 2 * (c & 3);
    *reinterpret_cast<uint4*>(row + ((c0 ^ (r & 7)) << 4)) = lo;
    *reinterpret_cast<uint4*>(row + (((c0 + 1) ^ (r & 7)) << 4)) = hi;
  }
}

// wgmma descriptor of an e4m3 K-major tile of kD-byte rows as TMA writes it (128-byte swizzle at kD = 128, 64-byte
// at kD = 64); a K step of 32 elements advances the start by 32 bytes.
template <int kD>
__device__ __forceinline__ uint64_t f8_desc(const uint8_t* tile) {
  return kD == 128 ? gmma_desc(smem_u32(tile), 0) : gmma_desc_sw64(smem_u32(tile));
}

// kQ8: e4m3 queries (T = bf16, kFp8 set); kPrefix: the shared-prefix pass; kTree: p.tree_mask is set.  See the file
// comment.
template <typename T, int kD, bool kFp8, bool kQ8, bool kPrefix = false, bool kTree = false>
__global__ void __launch_bounds__(kFp8 ? kThreadsFp8 : kThreads, 1)
decode_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
              const __grid_constant__ DecodeParams p) {
  static_assert(kD == 64 || kD == 128, "head dim 64 or 128");
  static_assert(!kQ8 || (kFp8 && std::is_same_v<T, __nv_bfloat16>), "e4m3 queries: e4m3 cache, bf16 P V");
  static_assert(!(kPrefix && kQ8), "a shared prefix takes a bf16 / fp16 q");
  using L = LoadRing<kD, kFp8, kQ8>;
  constexpr int kSubTiles = kD / 64;
  // T slots the compute warpgroup reads
  constexpr int kSlots = kQ8 ? kVStagesQ8 : (kFp8 ? kStagesFp8 : kStages);
  constexpr int kSlotBytes = kTile * kD * 2;
  constexpr int kQBytes = kRows * kD * (kQ8 ? 1 : 2);
  constexpr int kProducer = kFp8 ? 256 : 128;  // first thread of the producer warp
  const int split = blockIdx.x;
  const int group = p.hq / p.hkv;
  int b, kv_head, row0;
  int2 qr;  // the sequence's first packed query row and token count (kPrefix: the group's)
  if constexpr (kPrefix) {  // b is the prefix: it indexes seqlens, the cache slot or block table, and the descales
    b = blockIdx.z / p.hkv;
    kv_head = blockIdx.z % p.hkv;
    qr = prefix_rows(p, b * p.prefix_n);
    row0 = blockIdx.y * kRows;
    if (row0 >= qr.y * group) return;  // an idle slot, in every role: nothing to write
  } else if (p.cu_seqlens_q == nullptr) {
    b = blockIdx.z / p.hkv;
    kv_head = blockIdx.z % p.hkv;
    row0 = blockIdx.y * kRows;
    qr = make_int2(b * p.sq, p.sq);
  } else {
    int tile;
    kv_head = blockIdx.z;
    if (!varlen_tile(p, blockIdx.y, group, b, tile, qr)) return;  // an idle slot, in every role: nothing to write
    row0 = tile * kRows;
  }
  const int n_rows = qr.y * group;  // packed query rows of this kv head
  const int rows_here = n_rows - row0 < kRows ? n_rows - row0 : kRows;
  int seqlen = p.seqlens[b];
  seqlen = seqlen < 0 ? 0 : (seqlen > p.s_cap ? p.s_cap : seqlen);
  // the sequence's cache slot and first key row; keys below are counted from lp (see the file comment)
  int cache_slot = b, cap = p.s_cap;
  if (p.cache_batch_idx != nullptr) {
    cache_slot = __ldg(p.cache_batch_idx + b);
    if (cache_slot < 0 || cache_slot >= p.cache_batch) seqlen = cap = 0;  // no slot: no key, nor any appended one
  }
  const int lp = p.cache_leftpad != nullptr ? clamp_to(__ldg(p.cache_leftpad + b), 0, seqlen) : 0;
  seqlen -= lp;
  cap -= lp;
  // the last row of the tile sees the most keys (the limit never decreases with t)
  const int kmax = key_limit<kTree>(p, seqlen, cap, qr.y, (row0 + rows_here - 1) / group);
  const int j0 = split * p.tiles_per_split;
  int j1 = (kmax + kTile - 1) / kTile;
  if (j1 > j0 + p.tiles_per_split) j1 = j0 + p.tiles_per_split;
  const int n_tiles = j1 - j0;  // <= 0: this split starts past the visible keys

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_q = smem;
  uint8_t* smem_kv = smem + kQBytes;
  uint8_t* smem_f8 = smem_kv + kSlots * kSlotBytes;  // e4m3 caches only
  auto* bars = reinterpret_cast<Barriers<kQ8>*>(smem_f8 + (kFp8 ? L::kSlots * L::kSlotBytes : 0));
  static_assert(sizeof(Barriers<kQ8>) <= kBarBytes, "the barriers outgrew their space");
  // the ring TMA fills
  uint8_t* smem_load = kFp8 ? smem_f8 : smem_kv;
  uint64_t* load_full = kFp8 ? bars->f8_full : bars->kv_full;
  uint64_t* load_empty = kFp8 ? bars->f8_empty : bars->kv_empty;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    for (int i = 0; i < kSlots; ++i) {
      mbar_init(&bars->kv_full[i], kFp8 ? 4 : 1);  // TMA, or one arrival per converter warp
      mbar_init(&bars->kv_empty[i], 4);  // one arrival per compute warp
    }
    if constexpr (kFp8) {
      for (int i = 0; i < L::kSlots; ++i) {
        mbar_init(&bars->f8_full[i], 1);
        mbar_init(&bars->f8_empty[i], 4);  // one arrival per converter warp
      }
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (threadIdx.x >= kProducer) {
    // ------------------------------------------------------------------ TMA producer
    if (p.page_size != 0) {
      if (n_tiles > 0)
        produce_paged<kD, kFp8, kQ8>(&tm_k, &tm_v, load_full, load_empty, smem_load, p, b, kv_head, j0, n_tiles,
                                     kmax);
    } else if (threadIdx.x == kProducer) {
      uint32_t slot = 0, phase = 0;
      for (int jj = 0; jj < n_tiles; ++jj) {
        const int row = cache_slot * p.s_cap + lp + (j0 + jj) * kTile;  // rows past the tensor's end arrive as zeros
        for (int kv = 0; kv < 2; ++kv) {
          mbar_wait(&load_empty[slot], phase ^ 1);
          uint8_t* dst = smem_load + slot * L::kSlotBytes;
          mbar_arrive_expect_tx(&load_full[slot], L::kSlotBytes);
#pragma unroll
          for (int h = 0; h < L::kSubTiles; ++h)
            tma_load_3d(dst + h * kKHalfBytes, kv == 0 ? &tm_k : &tm_v, &load_full[slot], 64 * h, kv_head, row);
          if (++slot == L::kSlots) {
            slot = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }

  if constexpr (kQ8) {
    if (threadIdx.x >= 128) {
      // ---------------------------------------------------------------- converter: fp8 V slot -> bf16 V slot
      uint32_t slot = 0, phase = 0, fslot = 1, fphase = 0;  // V of tile jj is fp8 item 2 jj + 1
      for (int jj = 0; jj < n_tiles; ++jj) {
        mbar_wait(&bars->f8_full[fslot], fphase);
        mbar_wait(&bars->kv_empty[slot], phase ^ 1);
        widen_tile<T, kD>(smem_f8 + fslot * L::kSlotBytes, smem_kv + slot * kSlotBytes, threadIdx.x - 128);
        fence_proxy_async_smem();  // the generic-proxy writes, before wgmma reads them
        __syncwarp();
        if ((threadIdx.x & 31) == 0) {
          mbar_arrive(&bars->kv_full[slot]);
          mbar_arrive(&bars->f8_empty[fslot]);
        }
        if (++slot == kSlots) {
          slot = 0;
          phase ^= 1;
        }
        fslot += 2;
        if (fslot >= L::kSlots) {
          fslot -= L::kSlots;
          fphase ^= 1;
        }
      }
      return;
    }
  } else if constexpr (kFp8) {
    if (threadIdx.x >= 128) {
      // ---------------------------------------------------------------- converter: fp8 slot -> T slot
      uint32_t slot = 0, phase = 0, fslot = 0, fphase = 0;
      for (int i = 0; i < 2 * n_tiles; ++i) {  // K, V, K, V, ...
        mbar_wait(&bars->f8_full[fslot], fphase);
        mbar_wait(&bars->kv_empty[slot], phase ^ 1);
        widen_tile<T, kD>(smem_f8 + fslot * L::kSlotBytes, smem_kv + slot * kSlotBytes, threadIdx.x - 128);
        fence_proxy_async_smem();  // the generic-proxy writes, before wgmma reads them
        __syncwarp();
        if ((threadIdx.x & 31) == 0) {
          mbar_arrive(&bars->kv_full[slot]);
          mbar_arrive(&bars->f8_empty[fslot]);
        }
        if (++slot == kSlots) {
          slot = 0;
          phase ^= 1;
        }
        if (++fslot == kF8Stages) {
          fslot = 0;
          fphase ^= 1;
        }
      }
      return;
    }
  }

  // -------------------------------------------------------------------- compute warpgroup
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const bool warp_leader = lane == 0;
  const int r_base = 16 * (tid >> 5) + (lane >> 2);  // this thread's rows: r_base, r_base + 8
  const int quad_col = 2 * (lane & 3);                // its columns: 8 j + quad_col + {0, 1}
  const T* q = reinterpret_cast<const T*>(p.q);

  // Q tile: packed rows in the 128-byte swizzled K-major layout TMA would write; rows past the group are zero.  With
  // rotary, chunks below rotary_dim are rotated on the way (at new_token_pos).
  if constexpr (kQ8) {
    // e4m3 Q tile: kD-byte rows in the swizzle TMA writes for the e4m3 K tile (no rotary: the caller quantised q)
    const uint8_t* q8 = static_cast<const uint8_t*>(p.q);
    constexpr int kChunks = kD / 16;
#pragma unroll 4
    for (int idx = tid; idx < kRows * kChunks; idx += 128) {
      const int r = idx / kChunks, c = idx % kChunks;
      uint4 val = make_uint4(0u, 0u, 0u, 0u);
      if (r < rows_here) {
        const int pr = row0 + r;
        const int t = pr / group, head = kv_head * group + pr % group;
        val = *reinterpret_cast<const uint4*>(q8 + static_cast<long long>(qr.x + t) * p.q_row_stride +
                                              head * p.q_head_stride + 16 * c);
      }
      const int phys = kD == 128 ? c ^ (r & 7) : c ^ ((r >> 1) & 3);
      *reinterpret_cast<uint4*>(smem_q + r * kD + (phys << 4)) = val;
    }
  } else {
    constexpr int kChunks = kD / 8;  // 16-byte chunks per row
#pragma unroll 4
    for (int idx = tid; idx < kRows * kChunks; idx += 128) {
      const int r = idx / kChunks, c = idx % kChunks;
      uint4 val = make_uint4(0u, 0u, 0u, 0u);
      if (r < rows_here) {
        const int pr = row0 + r;
        const int t = pr / group, head = kv_head * group + pr % group;
        const T* q_row = q + static_cast<long long>(qr.x + t) * p.q_row_stride + head * p.q_head_stride;
        val = *reinterpret_cast<const uint4*>(q_row + 8 * c);
        if (p.rotary_cos != nullptr && c < p.rotary_half / 4) {
          int rb = b, rt = t;  // the row's own sequence and token
          if constexpr (kPrefix) prefix_token(p, b * p.prefix_n, qr.x + t, rb, rt);
          val = rotate_chunk<T>(val, q_row, c, rotary_pos(p, rb, new_token_pos<kTree>(p, rb, rt, false)), p);
        }
      }
      *reinterpret_cast<uint4*>(smem_q + (c >> 3) * kQHalfBytes + r * 128 + (((c & 7) ^ (r & 7)) << 4)) = val;
    }
  }
  fence_proxy_async_smem();
  named_bar_sync(1, 128);

  // Tree mask: the tiles holding appended keys start at key tile0 (seqlen < tile0 + kTile) and, for a sequence with
  // more than tile0 + kTile - seqlen new tokens, at tile0 + kTile (n_q <= kTile).  Bit 2 j + e of word (w, h) hides
  // this thread's column 8 j + quad_col + e of row r_base + 8 h in tile w.  Each thread reads back only its own words.
  // tile0 stays INT_MAX in splits that end before it: the key loop keeps one register for all of this, and only the
  // CTAs that reach the appended keys read the mask.
  [[maybe_unused]] int tile0 = INT_MAX;
  [[maybe_unused]] uint32_t* tree_hide = nullptr;  // after the barriers (smem_bytes<..., kTree>)
  if constexpr (kTree && !kPrefix) {
    tree_hide = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(bars) + kBarBytes);
    if (p.n_new > 0 && (j0 + n_tiles) * kTile > seqlen) {
      tile0 = seqlen / kTile * kTile;
#pragma unroll 1
      for (int wh = 0; wh < 4; ++wh) {
        const int r = r_base + 8 * (wh & 1);
        uint32_t hide = 0u;
        if (r < rows_here) {  // then qr.y >= 1
          const uint8_t* mrow = p.tree_mask + static_cast<long long>(qr.x + (row0 + r) / group) * p.sq;
          const int u0 = tile0 + (wh >> 1) * kTile + quad_col - seqlen;  // appended key of column quad_col
          // every load is issued, at a column clamped into the row, so that the 32 are in flight together (a load
          // under a branch would wait for the one before it)
          uint8_t m[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) m[i] = __ldg(mrow + clamp_to(u0 + 8 * (i >> 1) + (i & 1), 0, qr.y - 1));
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const int u = u0 + 8 * (i >> 1) + (i & 1);
            if (u >= 0 && u < qr.y && m[i] == 0) hide |= 1u << i;
          }
        }
        tree_hide[wh * 128 + tid] = hide;
      }
    }
  }

  int lim[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r_base + 8 * h;
    lim[h] = r < rows_here ? key_limit<kTree>(p, seqlen, cap, qr.y, (row0 + r) / group) : 0;
  }
  float o[kD / 2];
#pragma unroll
  for (int i = 0; i < kD / 2; ++i) o[i] = 0.f;
  float m2[2] = {-CUDART_INF_F, -CUDART_INF_F};
  float l[2] = {0.f, 0.f};
  float t2 = p.scale_log2;
  if constexpr (kQ8) t2 = t2 * p.q_descale[b * p.hkv + kv_head] * p.k_descale[b * p.hkv + kv_head];
  else if constexpr (kFp8) t2 *= p.k_descale[b * p.hkv + kv_head];

  // K-major A; e4m3 queries: the e4m3 Q tile, and the fp8 K slots (K-major B) instead of the T ones
  const uint64_t q_desc = kQ8 ? f8_desc<kD>(smem_q) : gmma_desc(smem_u32(smem_q), 0);
  const uint64_t k_desc0 = kQ8 ? f8_desc<kD>(smem_f8) : gmma_desc(smem_u32(smem_kv), 0);  // K tile, K-major B
  const uint64_t v_desc0 = gmma_desc(smem_u32(smem_kv), kKHalfBytes);  // V tile, MN-major B

  uint32_t slot = 0, phase = 0;
  [[maybe_unused]] uint32_t kf_slot = 0, kf_phase = 0;  // e4m3 queries: K of tile jj is fp8 item 2 jj
  for (int jj = 0; jj < n_tiles; ++jj) {
    uint32_t k_slot, k_phase, v_slot, v_phase;
    if constexpr (kQ8) {
      k_slot = kf_slot;
      k_phase = kf_phase;
      kf_slot += 2;
      if (kf_slot >= L::kSlots) {
        kf_slot -= L::kSlots;
        kf_phase ^= 1;
      }
      v_slot = slot;
      v_phase = phase;
      if (++slot == kSlots) {
        slot = 0;
        phase ^= 1;
      }
    } else {
      k_slot = slot;
      k_phase = phase;
      if (++slot == kSlots) {
        slot = 0;
        phase ^= 1;
      }
      v_slot = slot;
      v_phase = phase;
      if (++slot == kSlots) {
        slot = 0;
        phase ^= 1;
      }
    }
    const int key0 = (j0 + jj) * kTile;

    // ---- S = Q K^T
    float s[64];
    if constexpr (kQ8) {
      mbar_wait(&bars->f8_full[k_slot], k_phase);
      const uint64_t k_desc = gmma_desc_add(k_desc0, k_slot * L::kSlotBytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kD / 32; ++k)
        wgmma_ss_m64n128k32_e4m3(s, gmma_desc_add(q_desc, 32 * k), gmma_desc_add(k_desc, 32 * k), k > 0);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);
      __syncwarp();
      if (warp_leader) mbar_arrive(&bars->f8_empty[k_slot]);  // the fp8 K slot goes straight back to TMA
    } else {
      mbar_wait(&bars->kv_full[k_slot], k_phase);
      const uint64_t k_desc = gmma_desc_add(k_desc0, k_slot * kSlotBytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kD / 16; ++k)
        Gmma<T>::template ss128<0, 0>(s, gmma_desc_add(q_desc, (k >> 2) * kQHalfBytes + (k & 3) * 32),
                                      gmma_desc_add(k_desc, (k >> 2) * kKHalfBytes + (k & 3) * 32), k > 0);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);
      __syncwarp();
      if (warp_leader) mbar_arrive(&bars->kv_empty[k_slot]);
    }

    // ---- mask keys at or past each row's limit
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (key0 + kTile > lim[h]) {
        const int c_lim = lim[h] - key0;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (8 * j + quad_col + e >= c_lim) s[4 * j + 2 * h + e] = -CUDART_INF_F;
          }
        }
      }
    }
    // ---- tree mask: appended key u = key0 + c - seqlen stays visible only where the row's mask byte is set
    if constexpr (kTree) {
      if (key0 >= tile0) {
        const uint32_t* hide = tree_hide + (key0 - tile0) / kTile * 256 + tid;  // words (w, 0), (w, 1)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t bits = hide[128 * h];
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            if (bits >> i & 1u) s[4 * (i >> 1) + 2 * h + (i & 1)] = -CUDART_INF_F;
          }
        }
      }
    }

    // ---- online softmax (two rows per thread; a row lives in the 4 threads of a quad)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -CUDART_INF_F;
#pragma unroll
      for (int j = 0; j < 16; ++j) mx = fmaxf(mx, fmaxf(s[4 * j + 2 * h], s[4 * j + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m2[h], mx * t2);
      const float f = m_new == -CUDART_INF_F ? 1.f : fast_exp2(m2[h] - m_new);
      m2[h] = m_new;
      l[h] *= f;
#pragma unroll
      for (int j = 0; j < kD / 8; ++j) {
        o[4 * j + 2 * h] *= f;
        o[4 * j + 2 * h + 1] *= f;
      }
      const float mc = m_new == -CUDART_INF_F ? 0.f : m_new;
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float x = fast_exp2(fmaf(s[4 * j + 2 * h + e], t2, -mc));
          s[4 * j + 2 * h + e] = x;
          sum += x;
        }
      }
      l[h] += sum;
    }
    uint32_t pa[kTile / 16][4];
#pragma unroll
    for (int kk = 0; kk < kTile / 16; ++kk) pack_a<T>(pa[kk], s, kk);

    // ---- O += P V
    mbar_wait(&bars->kv_full[v_slot], v_phase);
    uint8_t* v_tile = smem_kv + v_slot * kSlotBytes;
    if (key0 + kTile > kmax) {
      // V rows no query row may see: zero them (P is 0 there, but 0 * NaN is not)
      const int z0 = kmax - key0;
      for (int idx = tid; idx < kSubTiles * (kTile - z0) * 8; idx += 128) {
        const int h = idx / ((kTile - z0) * 8), rem = idx % ((kTile - z0) * 8);
        *reinterpret_cast<uint4*>(v_tile + h * kKHalfBytes + (z0 + rem / 8) * 128 + (rem % 8) * 16) =
            make_uint4(0u, 0u, 0u, 0u);
      }
      fence_proxy_async_smem();
      named_bar_sync(1, 128);
    }
    const uint64_t v_desc = gmma_desc_add(v_desc0, v_slot * kSlotBytes);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kTile / 16; ++kk) gmma_rs<T, kD>(o, pa[kk], gmma_desc_add(v_desc, kk * 2048), 1);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    __syncwarp();
    if (warp_leader) mbar_arrive(&bars->kv_empty[v_slot]);
  }

  // ------------------------------------------------------------------ epilogue: O / l -> partial out, lse
  const long long n_out = static_cast<long long>(p.total_q) * p.hq;  // rows of out
  float* part = p.part + split * p.part_stride;
  // lse of (head, t) at lse_row + head * lse_stride + t: (b, head, t) uniform, (head, cu[b] + t) varlen
  const bool varlen = p.cu_seqlens_q != nullptr;
  float* lse_row =
      part + n_out * kD + (varlen ? static_cast<long long>(qr.x) : static_cast<long long>(b) * p.hq * p.sq);
  const int lse_stride = varlen ? p.total_q : p.sq;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float lt = l[h];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    const int r = r_base + 8 * h;
    if (r >= rows_here) continue;
    const int pr = row0 + r;
    const int t = pr / group, head = kv_head * group + pr % group;
    float inv = lt > 0.f ? 1.0f / lt : 0.f;
    if constexpr (kFp8) inv *= p.v_descale[b * p.hkv + kv_head];
    float* out_row = part + (static_cast<long long>(qr.x + t) * p.hq + head) * kD;
#pragma unroll
    for (int j = 0; j < kD / 8; ++j)
      *reinterpret_cast<float2*>(out_row + 8 * j + quad_col) =
          make_float2(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv);
    if ((lane & 3) == 0) {
      const float lse = lt > 0.f ? (m2[h] + __log2f(lt)) * 0.6931471805599453f : -CUDART_INF_F;
      if constexpr (kPrefix) {
        // packed row qr.x + t: lse at (head, row) varlen, at (b, head, t) of row = b * sq + t uniform
        const int row = qr.x + t;
        const long long li = varlen ? static_cast<long long>(head) * p.total_q + row
                                    : (static_cast<long long>(row / p.sq) * p.hq + head) * p.sq + row % p.sq;
        part[n_out * kD + li] = lse;
      } else {
        lse_row[static_cast<long long>(head) * lse_stride + t] = lse;
      }
    }
  }
}

// Cache row of new key t of sequence b (the pool row with a block table, a row of slot cache_batch_idx[b] with one),
// or -1 when the row is dropped: past the capacity, with a page id outside the pool, or with a slot outside the cache.
__device__ __forceinline__ long long append_row(const DecodeParams& p, int b, int t) {
  const int row = p.seqlens[b] + t;
  if (row < 0 || row >= p.s_cap) return -1;
  if (p.page_size == 0) {
    const int slot = p.cache_batch_idx != nullptr ? __ldg(p.cache_batch_idx + b) : b;
    if (slot < 0 || (p.cache_batch_idx != nullptr && slot >= p.cache_batch)) return -1;
    return static_cast<long long>(slot) * p.s_cap + row;
  }
  const int page = p.block_table[b * p.bt_stride + row / p.page_size];
  if (page < 0 || page >= p.num_pages) return -1;
  return static_cast<long long>(page) * p.page_size + row % p.page_size;
}

// Packed row of new key t of sequence b (in k_new / v_new), or -1 past the sequence's count (varlen: one block per
// (b, t < max_seqlen_q), and those past n_b exit).
__device__ __forceinline__ long long new_row(const DecodeParams& p, int b, int t) {
  const int2 r = q_rows(p, b);
  return t < r.y ? r.x + t : -1;
}

// One block per (b, t) row of the new keys, blockIdx.y selects K or V.  16-byte chunks; rows past the capacity
// are dropped, and so are rows whose page id lies outside the pool.  With rotary, the K chunks below rotary_dim are
// rotated as elements of T (at rotary_seqlens[b] + new_token_pos) before they are stored; everything else is a byte
// copy.
template <typename T>
__global__ void decode_append_kernel(uint8_t* k_cache, uint8_t* v_cache, long long row_stride_bytes,
                                     long long head_stride_bytes, const uint8_t* k_new, const uint8_t* v_new,
                                     const DecodeParams p, int row_bytes) {
  const int sq = p.sq, hkv = p.hkv;
  const int b = blockIdx.x / sq, t = blockIdx.x % sq;
  const long long in_row = new_row(p, b, t);
  if (in_row < 0) return;
  const long long cache_row = append_row(p, b, t);
  if (cache_row < 0) return;
  uint8_t* dst = (blockIdx.y == 0 ? k_cache : v_cache) + cache_row * row_stride_bytes;
  const uint8_t* src = (blockIdx.y == 0 ? k_new : v_new) + in_row * hkv * row_bytes;
  const bool rotate = blockIdx.y == 0 && p.rotary_cos != nullptr;
  const int pos = rotate ? rotary_pos(p, b, new_token_pos<true>(p, b, t, true)) : 0;
  const int chunks = row_bytes / 16;
  for (int idx = threadIdx.x; idx < hkv * chunks; idx += blockDim.x) {
    const int head = idx / chunks, c = idx % chunks;
    const uint8_t* in = src + static_cast<long long>(head) * row_bytes;
    uint4 val = *reinterpret_cast<const uint4*>(in + 16 * c);
    if (rotate && c < p.rotary_half / 4) val = rotate_chunk<T>(val, reinterpret_cast<const T*>(in), c, pos, p);
    *reinterpret_cast<uint4*>(dst + head * head_stride_bytes + 16 * c) = val;
  }
}

// The same into e4m3 caches: x / descale[b, head] (IEEE division), saturated to +-448 and rounded to nearest even
// (NaN stays NaN), 8 values per step.  With rotary, K is first rotated and rounded to T, as in decode_append_kernel.
template <typename T>
__global__ void decode_append_e4m3_kernel(uint8_t* k_cache, uint8_t* v_cache, long long row_stride,
                                          long long head_stride, const T* k_new, const T* v_new,
                                          const DecodeParams p, int head_dim) {
  const int sq = p.sq, hkv = p.hkv;
  const int b = blockIdx.x / sq, t = blockIdx.x % sq;
  const long long in_row = new_row(p, b, t);
  if (in_row < 0) return;
  const long long cache_row = append_row(p, b, t);
  if (cache_row < 0) return;
  uint8_t* dst = (blockIdx.y == 0 ? k_cache : v_cache) + cache_row * row_stride;
  const T* src = (blockIdx.y == 0 ? k_new : v_new) + in_row * hkv * head_dim;
  const float* descale = (blockIdx.y == 0 ? p.k_descale : p.v_descale) + b * hkv;
  const bool rotate = blockIdx.y == 0 && p.rotary_cos != nullptr;
  const int pos = rotate ? rotary_pos(p, b, new_token_pos<true>(p, b, t, true)) : 0;
  const int chunks = head_dim / 8;
  for (int idx = threadIdx.x; idx < hkv * chunks; idx += blockDim.x) {
    const int head = idx / chunks, c = idx % chunks;
    const float ds = descale[head];
    const T* in = src + static_cast<long long>(head) * head_dim;
    uint4 raw = *reinterpret_cast<const uint4*>(in + 8 * c);
    if (rotate && c < p.rotary_half / 4) raw = rotate_chunk<T>(raw, in, c, pos, p);
    const T* x = reinterpret_cast<const T*>(&raw);
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = __fdiv_rn(static_cast<float>(x[j]), ds);
    *reinterpret_cast<uint2*>(dst + head * head_stride + 8 * c) =
        make_uint2(pack4_e4m3(f[0], f[1], f[2], f[3]), pack4_e4m3(f[4], f[5], f[6], f[7]));
  }
}

template <typename OutT>
__device__ __forceinline__ void store_out(OutT* p, float x) {
  if constexpr (std::is_same_v<OutT, float>) *p = x;
  else if constexpr (std::is_same_v<OutT, __nv_bfloat16>) *p = __float2bfloat16_rn(x);
  else *p = __float2half_rn(x);
}

// One warp per (b, t, h) row.  Partials with lse = -inf (no visible key) are skipped, so their out is never read.
template <typename OutT>
__global__ void decode_combine_kernel(const float* parts, long long part_stride, int n_parts, int sq, int hq,
                                      int head_dim, long long n_rows, OutT* out, float* lse_out) {
  const long long n = static_cast<long long>(blockIdx.x) * (blockDim.x / 32) + threadIdx.x / 32;
  if (n >= n_rows) return;
  const int lane = threadIdx.x & 31;
  const long long b = n / (static_cast<long long>(sq) * hq);
  const int t = static_cast<int>((n / hq) % sq), h = static_cast<int>(n % hq);
  const long long li = (b * hq + h) * sq + t;
  const float* lse_in = parts + n_rows * head_dim + li;
  float mx = -CUDART_INF_F;
  for (int i = 0; i < n_parts; ++i) mx = fmaxf(mx, lse_in[i * part_stride]);
  float lse = -CUDART_INF_F;
  if (mx != -CUDART_INF_F) {
    float sum = 0.f;
    for (int i = 0; i < n_parts; ++i) {
      const float x = lse_in[i * part_stride];
      if (x != -CUDART_INF_F) sum += expf(x - mx);
    }
    lse = mx + logf(sum);
  }
  for (int d = lane; d < head_dim; d += 32) {
    float acc = 0.f;
    if (lse != -CUDART_INF_F) {
      for (int i = 0; i < n_parts; ++i) {
        const float x = lse_in[i * part_stride];
        if (x != -CUDART_INF_F) acc += expf(x - lse) * parts[i * part_stride + n * head_dim + d];
      }
    }
    store_out(out + n * head_dim + d, acc);
  }
  if (lane == 0) lse_out[li] = lse;
}

// Rows per TMA box of a cache's tensor maps, or an error for a bad page size: a paged cache's maps cover the whole
// pool and a box is at most one page; a contiguous cache takes one 128-key tile per box.
const char* box_rows_of(const DecodeParams& p, int& box_rows) {
  box_rows = kTile;
  if (p.page_size == 0) return nullptr;
  const bool size_ok = p.page_size == 16 || p.page_size == 32 || p.page_size == 64 ||
                       (p.page_size > 0 && p.page_size % kTile == 0);
  if (!size_ok) return "page_size must be 16, 32, 64 or a positive multiple of 128";
  if (p.block_table == nullptr) return "a paged cache needs a block table";
  if (p.page_size < kTile) box_rows = p.page_size;
  return nullptr;
}

}  // namespace dec

const char* decode_fwd_launch(int dtype, int cache_dtype, const TensorView& k_cache, const TensorView& v_cache,
                              const void* k_new, const void* v_new, int new_dtype, const DecodeParams& p,
                              int n_splits, int head_dim, cudaStream_t stream) {
  if (head_dim != 64 && head_dim != 128) return "the sm_90a decode kernel is instantiated for head_dim 64 and 128";
  if (dtype != kDtypeBF16 && dtype != kDtypeFP16 && dtype != kDtypeE4M3)
    return "the sm_90a decode kernel takes a bf16 / fp16 / e4m3 q";
  const bool fp8 = cache_dtype == kDtypeE4M3;
  const bool q8 = dtype == kDtypeE4M3;
  if (!fp8 && cache_dtype != dtype) return "the caches must have q's dtype or be e4m3";
  if (fp8 != (p.k_descale != nullptr && p.v_descale != nullptr))
    return "e4m3 caches need k / v descales, and only e4m3 caches take them";
  if (q8 != (p.q_descale != nullptr)) return "e4m3 queries need q_descale, and only they take it";
  if (q8 && p.rotary_cos != nullptr) return "rotary needs a bf16 / fp16 q: rotate before quantising";
  if (k_new != nullptr) {
    const bool new_ok = new_dtype == dtype || (fp8 && new_dtype == kDtypeE4M3) ||
                        (q8 && (new_dtype == kDtypeBF16 || new_dtype == kDtypeFP16));
    if (!new_ok) return "k_new / v_new must have q's dtype, be e4m3 over an e4m3 cache, or bf16 / fp16 with an e4m3 q";
    if (new_dtype == kDtypeE4M3 && p.rotary_cos != nullptr) return "rotary needs a bf16 / fp16 k_new";
  }
  if (p.hkv <= 0 || p.hq % p.hkv != 0) return "query heads must be a multiple of kv heads";
  if (p.tree_mask != nullptr && !p.causal) return "a tree mask replaces the causal rule: it needs causal";
  if (k_cache.row_stride != v_cache.row_stride || k_cache.head_stride != v_cache.head_stride)
    return "k_cache and v_cache must have the same strides";
  int box_rows;
  if (const char* e = dec::box_rows_of(p, box_rows)) return e;
  if (p.rotary_cos != nullptr) {
    if (p.rotary_sin == nullptr || p.rotary_seqlens == nullptr) return "rotary needs cos, sin and rotary_seqlens";
    if (p.rotary_half <= 0 || p.rotary_half % 8 != 0 || 2 * p.rotary_half > head_dim)
      return "rotary_dim must be a positive multiple of 16, at most head_dim";
    if (p.seqlen_ro < 1) return "the rotary tables must have at least one row";
  }
  // e4m3 rows are head_dim bytes: one 128-byte swizzle span at head_dim 128, one 64-byte span at 64
  const int elem_bytes = fp8 ? 1 : 2;
  const int swizzle = fp8 ? head_dim : 128;
  CUtensorMap tk, tv;
  if (const char* e = make_tensor_map(&tk, k_cache, elem_bytes, box_rows, head_dim, swizzle)) return e;
  if (const char* e = make_tensor_map(&tv, v_cache, elem_bytes, box_rows, head_dim, swizzle)) return e;
  if (k_new != nullptr && p.n_new > 0) {
    const dim3 agrid(p.batch * p.sq, 2);
    uint8_t* kc = static_cast<uint8_t*>(k_cache.ptr);
    uint8_t* vc = static_cast<uint8_t*>(v_cache.ptr);
    const uint8_t* kn = static_cast<const uint8_t*>(k_new);
    const uint8_t* vn = static_cast<const uint8_t*>(v_new);
    if (!fp8 && dtype == kDtypeBF16)
      dec::decode_append_kernel<__nv_bfloat16><<<agrid, 128, 0, stream>>>(
          kc, vc, k_cache.row_stride * 2, k_cache.head_stride * 2, kn, vn, p, head_dim * 2);
    else if (!fp8)
      dec::decode_append_kernel<__half><<<agrid, 128, 0, stream>>>(kc, vc, k_cache.row_stride * 2,
                                                                   k_cache.head_stride * 2, kn, vn, p, head_dim * 2);
    else if (new_dtype == kDtypeE4M3)  // pre-quantised k / v: their bytes, as they are (never rotated)
      dec::decode_append_kernel<__nv_bfloat16><<<agrid, 128, 0, stream>>>(kc, vc, k_cache.row_stride,
                                                                          k_cache.head_stride, kn, vn, p, head_dim);
    else if (new_dtype == kDtypeBF16)
      dec::decode_append_e4m3_kernel<<<agrid, 128, 0, stream>>>(
          kc, vc, k_cache.row_stride, k_cache.head_stride, static_cast<const __nv_bfloat16*>(k_new),
          static_cast<const __nv_bfloat16*>(v_new), p, head_dim);
    else
      dec::decode_append_e4m3_kernel<<<agrid, 128, 0, stream>>>(kc, vc, k_cache.row_stride, k_cache.head_stride,
                                                                static_cast<const __half*>(k_new),
                                                                static_cast<const __half*>(v_new), p, head_dim);
  }
  const int row_tiles = (p.sq * (p.hq / p.hkv) + dec::kRows - 1) / dec::kRows;
  dim3 grid(n_splits, row_tiles, p.batch * p.hkv);
  if (p.cu_seqlens_q != nullptr) {  // varlen: tile slots x kv heads, mapped to (sequence, row tile) on the device
    const long long slots = decode_tile_slots(p);
    if (slots > 65535) return "varlen decode: more than 65535 row tiles (total_q * Hq / Hkv too large)";
    if (slots == 0) return nullptr;  // no query rows
    grid = dim3(n_splits, static_cast<unsigned>(slots), p.hkv);
  }
  cudaError_t err = cudaSuccess;
  auto launch = [&](auto kern, int smem, int threads) {
    err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (err == cudaSuccess) kern<<<grid, threads, smem, stream>>>(tk, tv, p);
  };
  auto pick = [&](auto t, auto f8, auto tree) {
    using T = decltype(t);
    constexpr bool kFp8 = decltype(f8)::value, kTree = decltype(tree)::value;
    const int threads = kFp8 ? dec::kThreadsFp8 : dec::kThreads;
    if (head_dim == 128)
      launch(dec::decode_kernel<T, 128, kFp8, false, false, kTree>, dec::smem_bytes<128, kFp8, false, kTree>(),
             threads);
    else
      launch(dec::decode_kernel<T, 64, kFp8, false, false, kTree>, dec::smem_bytes<64, kFp8, false, kTree>(),
             threads);
  };
  auto pick_q8 = [&](auto tree) {  // e4m3 queries over an e4m3 cache: bf16 P V
    constexpr bool kTree = decltype(tree)::value;
    if (head_dim == 128)
      launch(dec::decode_kernel<__nv_bfloat16, 128, true, true, false, kTree>,
             dec::smem_bytes<128, true, true, kTree>(), dec::kThreadsFp8);
    else
      launch(dec::decode_kernel<__nv_bfloat16, 64, true, true, false, kTree>, dec::smem_bytes<64, true, true, kTree>(),
             dec::kThreadsFp8);
  };
  auto pick_cache = [&](auto tree) {
    if (q8) pick_q8(tree);
    else if (dtype == kDtypeBF16 && fp8) pick(__nv_bfloat16{}, std::true_type{}, tree);
    else if (dtype == kDtypeBF16) pick(__nv_bfloat16{}, std::false_type{}, tree);
    else if (fp8) pick(__half{}, std::true_type{}, tree);
    else pick(__half{}, std::false_type{}, tree);
  };
  if (p.tree_mask != nullptr) pick_cache(std::true_type{});
  else pick_cache(std::false_type{});
  if (err != cudaSuccess) return cudaGetErrorString(err);
  err = cudaGetLastError();
  return err == cudaSuccess ? nullptr : cudaGetErrorString(err);
}

const char* decode_prefix_launch(int dtype, int cache_dtype, const TensorView& k_prefix, const TensorView& v_prefix,
                                 const DecodeParams& p, int n_prefix, int n_splits, int head_dim,
                                 cudaStream_t stream) {
  if (head_dim != 64 && head_dim != 128) return "the sm_90a decode kernel is instantiated for head_dim 64 and 128";
  if (dtype != kDtypeBF16 && dtype != kDtypeFP16) return "a shared prefix takes a bf16 / fp16 q";
  const bool fp8 = cache_dtype == kDtypeE4M3;
  if (!fp8 && cache_dtype != dtype) return "the prefix caches must have q's dtype or be e4m3";
  if (fp8 != (p.k_descale != nullptr && p.v_descale != nullptr))
    return "e4m3 prefix caches need k / v descales, and only e4m3 caches take them";
  if (p.q_descale != nullptr || p.n_new != 0 || p.cache_batch_idx != nullptr || p.cache_leftpad != nullptr)
    return "the shared-prefix pass takes no q_descale, append, cache slots or left pads";
  int box_rows;
  if (const char* e = dec::box_rows_of(p, box_rows)) return e;
  if (p.hkv <= 0 || p.hq % p.hkv != 0) return "query heads must be a multiple of kv heads";
  if (p.tree_mask != nullptr && !p.causal) return "a tree mask replaces the causal rule: it needs causal";
  if (n_prefix < 1 || p.batch % n_prefix != 0 || p.prefix_n != p.batch / n_prefix)
    return "the batch must be prefix_n sequences per prefix";
  if (k_prefix.row_stride != v_prefix.row_stride || k_prefix.head_stride != v_prefix.head_stride)
    return "the prefix caches must have the same strides";
  if (p.rotary_cos != nullptr) {
    if (p.rotary_sin == nullptr || p.rotary_seqlens == nullptr) return "rotary needs cos, sin and rotary_seqlens";
    if (p.rotary_half <= 0 || p.rotary_half % 8 != 0 || 2 * p.rotary_half > head_dim)
      return "rotary_dim must be a positive multiple of 16, at most head_dim";
    if (p.seqlen_ro < 1) return "the rotary tables must have at least one row";
  }
  const long long slots = decode_prefix_slots(p);
  if (slots > 65535) return "shared prefix: more than 65535 row tiles per group";
  if (static_cast<long long>(n_prefix) * p.hkv > 65535) return "shared prefix: more than 65535 (prefix, kv head) pairs";
  if (slots == 0) return nullptr;  // no query rows
  const int elem_bytes = fp8 ? 1 : 2;
  const int swizzle = fp8 ? head_dim : 128;
  CUtensorMap tk, tv;
  if (const char* e = make_tensor_map(&tk, k_prefix, elem_bytes, box_rows, head_dim, swizzle)) return e;
  if (const char* e = make_tensor_map(&tv, v_prefix, elem_bytes, box_rows, head_dim, swizzle)) return e;
  const dim3 grid(n_splits, static_cast<unsigned>(slots), n_prefix * p.hkv);
  cudaError_t err = cudaSuccess;
  auto launch = [&](auto kern, int smem, int threads) {
    err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (err == cudaSuccess) kern<<<grid, threads, smem, stream>>>(tk, tv, p);
  };
  // the prefix pass masks nothing: a tree mask only moves its rotary positions
  auto pick = [&](auto t, auto f8, auto tree) {
    using T = decltype(t);
    constexpr bool kFp8 = decltype(f8)::value, kTree = decltype(tree)::value;
    const int threads = kFp8 ? dec::kThreadsFp8 : dec::kThreads;
    if (head_dim == 128)
      launch(dec::decode_kernel<T, 128, kFp8, false, true, kTree>, dec::smem_bytes<128, kFp8, false>(), threads);
    else launch(dec::decode_kernel<T, 64, kFp8, false, true, kTree>, dec::smem_bytes<64, kFp8, false>(), threads);
  };
  auto pick_cache = [&](auto tree) {
    if (dtype == kDtypeBF16 && fp8) pick(__nv_bfloat16{}, std::true_type{}, tree);
    else if (dtype == kDtypeBF16) pick(__nv_bfloat16{}, std::false_type{}, tree);
    else if (fp8) pick(__half{}, std::true_type{}, tree);
    else pick(__half{}, std::false_type{}, tree);
  };
  if (p.tree_mask != nullptr && p.rotary_cos != nullptr) pick_cache(std::true_type{});
  else pick_cache(std::false_type{});
  if (err != cudaSuccess) return cudaGetErrorString(err);
  err = cudaGetLastError();
  return err == cudaSuccess ? nullptr : cudaGetErrorString(err);
}

long long decode_prefix_slots(const DecodeParams& p) {
  const long long group = p.hq / p.hkv;
  long long rows = static_cast<long long>(p.prefix_n) * p.sq;
  if (p.cu_seqlens_q != nullptr && p.total_q < rows) rows = p.total_q;
  return (rows * group + dec::kRows - 1) / dec::kRows;
}

long long decode_tile_slots(const DecodeParams& p) {
  const long long group = p.hq / p.hkv;
  const long long per_seq = (p.sq * group + dec::kRows - 1) / dec::kRows;
  const long long bound = (p.total_q * group + (dec::kRows - 1) * static_cast<long long>(p.batch)) / dec::kRows;
  return p.batch * per_seq < bound ? p.batch * per_seq : bound;
}

const char* decode_combine_launch(const float* parts, long long part_stride, int n_parts, int batch, int sq, int hq,
                                  int head_dim, void* out, int out_dtype, float* lse, cudaStream_t stream) {
  const long long n_rows = static_cast<long long>(batch) * sq * hq;
  if (n_rows == 0) return nullptr;
  constexpr int kWarps = 8;
  const unsigned blocks = static_cast<unsigned>((n_rows + kWarps - 1) / kWarps);
  if (out_dtype == kDtypeBF16)
    dec::decode_combine_kernel<<<blocks, 32 * kWarps, 0, stream>>>(parts, part_stride, n_parts, sq, hq, head_dim,
                                                                   n_rows, static_cast<__nv_bfloat16*>(out), lse);
  else if (out_dtype == kDtypeFP16)
    dec::decode_combine_kernel<<<blocks, 32 * kWarps, 0, stream>>>(parts, part_stride, n_parts, sq, hq, head_dim,
                                                                   n_rows, static_cast<__half*>(out), lse);
  else
    dec::decode_combine_kernel<<<blocks, 32 * kWarps, 0, stream>>>(parts, part_stride, n_parts, sq, hq, head_dim,
                                                                   n_rows, static_cast<float*>(out), lse);
  const cudaError_t err = cudaGetLastError();
  return err == cudaSuccess ? nullptr : cudaGetErrorString(err);
}

}  // namespace rfa
