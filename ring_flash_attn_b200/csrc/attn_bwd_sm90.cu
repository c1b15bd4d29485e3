// Blockwise flash-attention backward for sm_90a (head_dim 64 / 128, bf16 / fp16).
//
// One CTA = one 128-key tile of one kv head.  dK and dV of that tile stay in registers while the CTA sweeps every
// query tile (64 rows) of every query head of the GQA group and every query segment that can see the keys; dQ
// tiles are staged through shared memory and added into an fp32 accumulator with TMA reduce-add.  This replaces
// flash_attn's backward + the reference's fp32 dq/dk/dv bookkeeping per ring step
// (/root/reference/ring_flash_attn/ring_flash_attn.py:97-152).
//
// Two warpgroups (256 threads); warpgroup w owns keys [64 w, 64 w + 64) of the tile.  Per query tile i (wgmma,
// fp32 accumulators in registers):
//   S^T  = K_w Q_i^T         (64 keys x 64 queries)   both operands K-major in shared memory
//   dP^T = V_w dO_i^T                                 likewise
//   P^T  = exp2(S^T * c - lse_i),  dS^T = P^T o (dP^T - delta_i) * scale      (registers)
//   dV_w += P^T dO_i         (A = P^T from registers, B = dO MN-major)
//   dK_w += dS^T Q_i         (A = dS^T from registers, B = Q MN-major)
//   dQ_i[:, 64 w : 64 w + 64] = dS_i K[:, 64 w : 64 w + 64]   (A = dS^T of both groups in shared memory,
//                            read MN-major; B = K MN-major) -> fp32 shared memory (128-byte swizzled boxes of
//                            32 dims) -> TMA reduce-add of the group's own two boxes, issued by its thread 0
// Both warpgroups meet at two named barriers per query tile (previous tile retired, dS^T complete), so the Q / dO
// ring needs no "empty" barriers: thread 0 refills the stage of tile i - 1 while tile i runs.  At head dim 128,
// between the dQ GEMM and the next tile's S^T each group only meets its own 128 threads, around its dQ staging (at
// head dim 64 group 0 stages all of dQ and both groups meet there).  The loader's tile iterator lives in shared
// memory.
// Each stage also holds the 64 lse and delta values of its rows and a description of its tile.  Threads 0-63 copy
// lse / delta for tile i + 2 (one row each, coalesced, cp.async: no register held in flight) at the top of tile i
// and wait for the copies before its first barrier, so the softmax reads shared memory and no global load sits
// between a GEMM's completion and the exp2 that needs it.  S^T and dP^T are separate commit groups: P^T is
// computed while dP^T still runs.  S^T of tile i + 1 is issued right after the dQ GEMM of tile i, before the wait
// for dQ, so the tensor pipe works on it while dQ of tile i is staged and its reduce-add issued.
#include <math_constants.h>
#include <stdio.h>

#include "attn_common.h"
#include "comm_device.cuh"
#include "sm90_ptx.cuh"

namespace rfa {
namespace bwd {

#ifdef RFA_TRACE
// per-tile stamps of CTA 0 (16 slots), thread 0: 0 S^T complete, 1 dP^T complete, 2 dS^T staged, 3 dQ issued,
// 4 dQ complete, 5 dQ reduce-add issued, 6 S^T issued, 7 dV / dK issued (benchmark/trace_bwd.py)
#define RFA_STAMP(cond, iter, slot)                                                              \
  do {                                                                                            \
    if ((cond) && cta == 0 && p.trace != nullptr && (iter) < 64) p.trace[(iter)*16 + (slot)] = clock64(); \
  } while (0)
#else
#define RFA_STAMP(cond, iter, slot) \
  do {                              \
  } while (0)
#endif

constexpr int kTileK = 128;  // keys per CTA
constexpr int kTileQ = 64;   // queries per inner iteration
constexpr int kStages = 3;   // Q/dO ring
constexpr int kThreads = 256;
constexpr int kQHalf = kTileQ * 128;               // 64-wide swizzled sub-tile of a 64-row tile (8 KB)
constexpr int kKVHalf = kTileK * 128;              // 64-wide swizzled sub-tile of a 128-row tile (16 KB)
constexpr int kDSBytes = kTileK * kTileQ * 2;      // 16 KB
// Head dim kD (64 or 128) is a template parameter: tiles are kD / 64 sub-tiles wide.
template <int kD>
struct Geo {
  static constexpr int kKVBytes = kTileK * kD * 2;  // K, V tile: 32 KB at kD = 128
  static constexpr int kQBytes = kTileQ * kD * 2;   // Q, dO tile: 16 KB
  static constexpr int kDQBytes = kTileQ * kD * 4;  // fp32 dQ staging: 32 KB
  static constexpr int kSmemBytes = 2 * kKVBytes + kStages * 2 * kQBytes + kDSBytes + kDQBytes +
                                    kStages * 2 * kTileQ * 4 /*lse2, delta*/ + 1024 /*barriers*/ + 1024 /*slack*/;
};

struct Barriers {
  uint64_t kv_full;
  uint64_t qdo_full[kStages];
};
// The query tile in a Q/dO stage, as the consumers need it (written by the loader with the stage; the consumers keep
// no tile iterator of their own in registers)
struct alignas(16) StageTile {
  int ti, diag, lo;
  int head, row;  // of the tile's dQ rows (first row)
};

// Query tiles of one segment that can see this key tile.
struct QGeom {
  int q_row0, q_len, diag, lo;
  int t_begin, t_end;  // 64-row tile range
};
__device__ __forceinline__ QGeom q_geom(const BwdQSegment& s) {
  QGeom g;
  g.q_row0 = s.q_row0;
  g.q_len = s.q_len;
  g.diag = s.diag;
  g.lo = s.lo;
  const int first = s.diag >= 0 ? 0 : -s.diag;  // first chunk row that sees key 0 of the tile
  g.t_begin = first / kTileQ;
  g.t_end = (s.q_len + kTileQ - 1) / kTileQ;
  if (g.t_begin > g.t_end) g.t_begin = g.t_end;
  return g;
}

// Walks the query tiles of a CTA in sweep order: query heads of the group, segments, 64-row tiles.
struct TileIter {
  const BwdQSegment* segs;
  int seg_begin, seg_count, group;
  int gq, si, ti;
  QGeom g;
  __device__ __forceinline__ void init(const BwdQSegment* s, int begin, int count, int grp) {
    segs = s;
    seg_begin = begin;
    seg_count = count;
    group = grp;
    gq = 0;
    si = 0;
    if (seg_count > 0) {
      g = q_geom(segs[seg_begin]);
      ti = g.t_begin;
      settle();
    }
  }
  __device__ __forceinline__ void settle() {  // skip segments without tiles
    while (gq < group && ti >= g.t_end) {
      if (++si == seg_count) {
        si = 0;
        ++gq;
      }
      if (gq < group) {
        g = q_geom(segs[seg_begin + si]);
        ti = g.t_begin;
      }
    }
  }
  __device__ __forceinline__ void next() {
    ++ti;
    settle();
  }
};

static_assert(sizeof(Barriers) + kStages * sizeof(StageTile) + sizeof(TileIter) <= 1024, "barrier area");

template <typename T, bool kWindow, int kD>
__global__ void __launch_bounds__(kThreads, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_do,
                const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                const __grid_constant__ CUtensorMap tm_ks, const __grid_constant__ CUtensorMap tm_vs,
                const __grid_constant__ CUtensorMap tm_dq, const __grid_constant__ BwdParams p) {
  // communication CTAs first (see comm_device.cuh): they re-publish this rank's K/V rows to the peers
  if (static_cast<int>(blockIdx.x) < p.push.n_ctas) {
    if (p.push.use_tma) {
      extern __shared__ uint8_t push_smem_raw[];
      push_role_tma(p.push, reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(push_smem_raw) + 1023) & ~uintptr_t(1023)));
    } else {
      push_role(p.push);
    }
    return;
  }
  static_assert(kD == 64 || kD == 128, "head dim 64 or 128");
  constexpr int kKVBytes = Geo<kD>::kKVBytes, kQBytes = Geo<kD>::kQBytes, kDQBytes = Geo<kD>::kDQBytes;
  constexpr int kSubTiles = kD / 64;
  const int cta = static_cast<int>(blockIdx.x) - p.push.n_ctas;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_k = smem;
  uint8_t* smem_v = smem_k + kKVBytes;
  uint8_t* smem_qdo = smem_v + kKVBytes;                 // kStages x (Q 16 KB, dO 16 KB)
  uint8_t* smem_ds = smem_qdo + kStages * 2 * kQBytes;   // 16 KB, [128 keys][64 queries] swizzled
  float* smem_dq = reinterpret_cast<float*>(smem_ds + kDSBytes);   // [64 queries][kD dims] fp32
  // [kStages][64] lse (natural log, as the forward wrote it), then [kStages][64] delta; 32-bit shared addresses
  constexpr uint32_t kLseBytes = kStages * kTileQ * 4;
  const uint32_t lse_base = smem_u32(smem_dq) + kDQBytes;
  Barriers* bars = reinterpret_cast<Barriers*>(reinterpret_cast<uint8_t*>(smem_dq) + kDQBytes + 2 * kLseBytes);
  StageTile* tiles = reinterpret_cast<StageTile*>(bars + 1);  // [kStages]

  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int w = tid >> 7;          // warpgroup: keys [64 w, 64 w + 64)
  const int wtid = tid & 127;
  // CTA -> (key tile, kv head).  One GPU: head-major, so that concurrently running CTAs re-read the Q / dO of ONE
  // head out of L2 (at S = 32K all heads together do not fit).  Fused multi-GPU launches: tile-major - the table
  // is sorted by ring step (local keys first, then the sources in the order their K/V arrives), and with head-major
  // numbering the tiles of the LAST source of head 0 would be scheduled, and sit waiting for their data, before any
  // tile of head 1 that could already run.
  const int kv_head = p.item_major ? cta % p.hkv : cta / p.n_items;
  const int group = p.hq / p.hkv;
  BwdItem it = p.items[p.item_major ? cta / p.hkv : cta % p.n_items];
  if (p.flags & 4) it.seg_count = 0;  // timing experiment: K/V push + dK/dV return only

  // total number of query tiles this CTA sweeps
  int tiles_per_head = 0;
  for (int si = 0; si < it.seg_count; ++si) {
    const QGeom g = q_geom(p.qsegs[it.seg_begin + si]);
    tiles_per_head += g.t_end - g.t_begin;
  }
  const int total_tiles = tiles_per_head * group;

  // ---------------------------------------------------------------- loads (threads 0-63; TMA: thread 0)
  // (a tile no local query reaches only sends zero rows: nothing is loaded, and in particular no TMA write can
  // land in the K | V area after the epilogue has started to stage those rows there)
  // The loader's iterator: threads 0-63 walk it in registers over the first kStages - 1 tiles; from then on it
  // lives in shared memory and thread 0 advances it after each refill, so it holds no register across the loop.
  TileIter* ld_smem = reinterpret_cast<TileIter*>(tiles + kStages);
  // Q / dO of tile n (at `ld`) -> stage n % kStages; thread 0
  auto load_tile = [&](const TileIter& ld, int n) {
    const int stage = n % kStages;
    const int head = kv_head * group + ld.gq;
    const int row = ld.g.q_row0 + ld.ti * kTileQ;
    uint8_t* dq_ = smem_qdo + stage * 2 * kQBytes;
    uint8_t* ddo = dq_ + kQBytes;
    mbar_arrive_expect_tx(&bars->qdo_full[stage], 2 * kQBytes);
#pragma unroll
    for (int h = 0; h < kSubTiles; ++h) {
      tma_load_3d(dq_ + h * kQHalf, &tm_q, &bars->qdo_full[stage], 64 * h, head, row);
      tma_load_3d(ddo + h * kQHalf, &tm_do, &bars->qdo_full[stage], 64 * h, head, row);
    }
    // (its slot was last read by tile n - kStages: by every thread before barrier 1 of that tile, and by the
    // threads that issue its dQ reduce-add before barrier 1 of the next tile, which precedes this refill)
    tiles[stage] = StageTile{ld.ti, ld.g.diag, ld.g.lo, head, row};
  };
  // lse and delta of row `tid` of tile n (at `ld`) -> the stage's slots, with cp.async (no register is held while
  // the copy is in flight; complete after cp_async_wait_all).  Rows that do not exist: lse -inf, delta 0.
  auto lse_stage = [&](const TileIter& ld, int n) {
    const uint32_t sl = lse_base + ((n % kStages) * kTileQ + tid) * 4;
    const int qi = ld.ti * kTileQ + tid;
    if (qi < ld.g.q_len) {
      const int row = ld.g.q_row0 + qi;
      const size_t b = row / p.lse_S, sidx = row % p.lse_S;
      const size_t idx = (b * p.hq + kv_head * group + ld.gq) * static_cast<size_t>(p.lse_S) + sidx;
      cp_async_4(sl, p.lse + idx);
      cp_async_4(sl + kLseBytes, p.delta + idx);
    } else {
      st_shared_f32(sl, -CUDART_INF_F);
      st_shared_f32(sl + kLseBytes, 0.f);
    }
  };
  if (tid == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_do);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    tma_prefetch_desc(&tm_dq);
    tma_prefetch_desc(&tm_ks);
    tma_prefetch_desc(&tm_vs);
    mbar_init(&bars->kv_full, 1);
    for (int i = 0; i < kStages; ++i) mbar_init(&bars->qdo_full[i], 1);
    fence_mbar_init();
    if (total_tiles > 0) {
      const bool staged = it.flag >= 0 && p.ready_flags != nullptr;
      if (staged && !(p.flags & 2)) {
        wait_epoch(p.ready_flags + it.flag, p.ready_epoch);
        fence_proxy_async_all();
      }
      const CUtensorMap* mk = staged ? &tm_ks : &tm_k;
      const CUtensorMap* mv = staged ? &tm_vs : &tm_v;
      mbar_arrive_expect_tx(&bars->kv_full, 2 * kKVBytes);
#pragma unroll
      for (int h = 0; h < kSubTiles; ++h) {
        tma_load_3d(smem_k + h * kKVHalf, mk, &bars->kv_full, 64 * h, kv_head, it.kv_row0);
        tma_load_3d(smem_v + h * kKVHalf, mv, &bars->kv_full, 64 * h, kv_head, it.kv_row0);
      }
    }
  }
  if (tid < kTileQ) {
    TileIter ld;
    ld.init(p.qsegs, it.seg_begin, it.seg_count, group);
    for (int n = 0; n < kStages - 1 && n < total_tiles; ++n) {
      lse_stage(ld, n);
      if (tid == 0) load_tile(ld, n);
      ld.next();
    }
    if (tid == 0) *ld_smem = ld;
    cp_async_wait_all();
  }
  __syncthreads();

  // ---------------------------------------------------------------- compute (both warpgroups)
  const int k_lo = 16 * (wtid >> 5) + (lane >> 2);  // this thread's keys in the group's 64: k_lo, k_lo + 8
  const int quad_col = 2 * (lane & 3);              // its columns: 8 j + quad_col + {0, 1}
  float dv[kD / 2], dk[kD / 2];
#pragma unroll
  for (int i = 0; i < kD / 2; ++i) dv[i] = dk[i] = 0.f;

  const uint32_t k_base = smem_u32(smem_k), v_base = smem_u32(smem_v), qdo_base = smem_u32(smem_qdo);
  const uint64_t k_km = gmma_desc(k_base + w * 64 * 128, 0);          // K_w, K-major A (S^T)
  const uint64_t v_km = gmma_desc(v_base + w * 64 * 128, 0);          // V_w, K-major A (dP^T)
  const uint64_t q_km0 = gmma_desc(qdo_base, 0);                      // stage 0 Q, K-major B
  const uint64_t q_mn0 = gmma_desc(qdo_base, kQHalf);                 // stage 0 Q, MN-major B
  const uint64_t ds_mn = gmma_desc(smem_u32(smem_ds), kDSBytes);      // dS (64 queries x 128 keys), MN-major A
  const uint64_t k_mn = gmma_desc(k_base + w * kKVHalf, kKVHalf);     // K[:, 64 w : 64 w + 64], MN-major B

  const bool do_dq = kD == 128 || w == 0;  // head dim 64: group 0 computes all of dQ
  float st[32];
  // ---- top of tile n: lse / delta copies of tile n + 2, the stage wait, S^T issued (one commit group).  Called
  // for n = total_tiles too (after the last tile): that S^T reads whatever stage n % kStages holds and is never
  // used, but the issue stays unconditional (a conditional wgmma issue makes ptxas serialise every wgmma).
  auto issue_st = [&](int n) {
    // lse / delta of tile n + 2 go into the slot of tile n - 1, whose softmax every thread finished before the
    // barriers of tile n - 1; they are copied under tile n's GEMMs and softmax and complete before its barrier 1
    if (tid < kTileQ && n + kStages - 1 < total_tiles) lse_stage(*ld_smem, n + kStages - 1);
    if (n < total_tiles) mbar_wait(&bars->qdo_full[n % kStages], (n / kStages) & 1);
    const uint32_t st_off = (n % kStages) * 2 * kQBytes;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kD / 16; ++k) {
      const uint32_t oa = (k >> 2) * kKVHalf + (k & 3) * 32;
      const uint32_t ob = st_off + (k >> 2) * kQHalf + (k & 3) * 32;
      Gmma<T>::template ss64<0, 0>(st, gmma_desc_add(k_km, oa), gmma_desc_add(q_km0, ob), k > 0);
    }
    wgmma_commit();
    RFA_STAMP(tid == 0, n, 6);
  };
  if (total_tiles > 0) {
    mbar_wait(&bars->kv_full, 0);
    issue_st(0);
  }
  for (int i = 0; i < total_tiles; ++i) {
    const int stage = i % kStages;
    const StageTile g = tiles[stage];
    const int ti = g.ti;
    const uint32_t st_off = stage * 2 * kQBytes;

    // ---- dP^T (S^T of this tile was issued at the end of the previous one; two commit groups)
    float dpt[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kD / 16; ++k) {
      const uint32_t oa = (k >> 2) * kKVHalf + (k & 3) * 32;
      const uint32_t ob = st_off + kQBytes + (k >> 2) * kQHalf + (k & 3) * 32;
      Gmma<T>::template ss64<0, 0>(dpt, gmma_desc_add(v_km, oa), gmma_desc_add(q_km0, ob), k > 0);
    }
    wgmma_commit();
    // causal boundary per key: key visible to query qi iff key <= qi + diag  <=>  qi >= key - diag; sliding window:
    // ... and iff key >= qi + lo  <=>  qi <= key - lo (the host already dropped the query tiles past the last such row)
    int q_lo[2], q_hi[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int key = 64 * w + k_lo + 8 * h;  // row in the key tile
      const long long first_q = static_cast<long long>(key) - g.diag - static_cast<long long>(ti) * kTileQ;
      q_lo[h] = key >= it.kv_rows ? kTileQ
                                  : (first_q < 0 ? 0 : (first_q > kTileQ ? kTileQ : static_cast<int>(first_q)));
      q_hi[h] = kTileQ;
      if constexpr (kWindow) {
        const long long last_q = static_cast<long long>(key) - g.lo - static_cast<long long>(ti) * kTileQ;
        q_hi[h] = last_q < 0 ? 0 : (last_q >= kTileQ ? kTileQ : static_cast<int>(last_q) + 1);
      }
    }
    wgmma_wait<1>();
    fence_regs(st);
    RFA_STAMP(tid == 0, i, 0);

    // ---- P^T (into st) while dP^T runs.  lse in log2 units: +inf for rows that do not exist or saw no key => P = 0
    const uint32_t lse = lse_base + stage * kTileQ * 4;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = 8 * j + quad_col + e;
        const float x = ld_shared_f32(lse + c * 4);
        const float l = x == -CUDART_INF_F ? CUDART_INF_F : x * 1.4426950408889634f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = 4 * j + 2 * h + e;
          const float pe = fast_exp2(fmaf(st[r], p.scale_log2, -l));
          st[r] = (c >= q_lo[h] && c < q_hi[h]) ? pe : 0.f;
        }
      }
    }
    wgmma_wait<0>();
    fence_regs(dpt);
    RFA_STAMP(tid == 0, i, 1);

    // ---- dS^T (into dpt)
    const uint32_t delta = lse_base + kLseBytes + stage * kTileQ * 4;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = 8 * j + quad_col + e;
        const float dl = ld_shared_f32(delta + c * 4);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = 4 * j + 2 * h + e;
          dpt[r] = st[r] * (dpt[r] - dl) * p.scale;
        }
      }
    }
    uint32_t pa[4][4], da[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      pack_a<T>(pa[kk], st, kk);
      pack_a<T>(da[kk], dpt, kk);
    }

    // ---- dV += P^T dO, dK += dS^T Q
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      gmma_rs<T, kD>(dv, pa[kk], gmma_desc_add(q_mn0, st_off + kQBytes + kk * 2048), 1);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) gmma_rs<T, kD>(dk, da[kk], gmma_desc_add(q_mn0, st_off + kk * 2048), 1);
    wgmma_commit();
    RFA_STAMP(tid == 0, i, 7);

    // tile i - 1 has retired everywhere past this barrier: the dQ GEMMs no longer read smem_ds, and its Q / dO
    // stage may be refilled
    if (tid < kTileQ) cp_async_wait_all();
    named_bar_sync(1, kThreads);
    // (thread 0 advances the loader's iterator; the other loader threads read it at the top of tile i + 1, after
    // barrier 2)
    if (tid == 0 && i + kStages - 1 < total_tiles) {
      TileIter ld = *ld_smem;
      load_tile(ld, i + kStages - 1);
      ld.next();
      *ld_smem = ld;
    }

    // ---- dS^T -> shared memory: [128 keys][64 queries] bf16, 128-byte swizzled rows
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int key = 64 * w + k_lo + 8 * h;
      uint8_t* ds_row = smem_ds + key * 128;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        *reinterpret_cast<uint32_t*>(ds_row + ((j ^ (key & 7)) << 4) + quad_col * 2) =
            Pack2<T>::pack(dpt[4 * j + 2 * h], dpt[4 * j + 2 * h + 1]);
    }
    fence_proxy_async_smem();
    // this group's dQ boxes of tile i - 1 have been read out by its reduce-add before the group stages tile i's
    if (wtid == 0) tma_store_wait_read<0>();
    named_bar_sync(2, kThreads);
    RFA_STAMP(tid == 0, i, 2);

    // ---- dQ[:, 64 w : 64 w + 64] = dS K[:, 64 w : 64 w + 64]
    float dq[32];
    if (do_dq) {
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kTileK / 16; ++k)
        Gmma<T>::template ss64<1, 1>(dq, gmma_desc_add(ds_mn, k * 2048), gmma_desc_add(k_mn, k * 2048), k > 0);
      wgmma_commit();
    }
    RFA_STAMP(tid == 0, i, 3);
    // ---- S^T of tile i + 1, so that the tensor pipe has it queued behind dQ while this tile's dQ is staged
    issue_st(i + 1);
    // commit groups in flight: dV / dK (i), dQ (i, groups that compute dQ), S^T (i + 1).  Groups complete in
    // order: this retires those of tile i and leaves S^T (i + 1) running.  Past barrier 1 of tile i + 1 no GEMM of
    // tile i runs anywhere: smem_ds may be rewritten and the stage of tile i refilled.
    wgmma_wait<1>();
    fence_regs(dv);
    fence_regs(dk);
    RFA_STAMP(tid == 0, i, 4);
    if (do_dq) {
      fence_regs(dq);
      // smem_dq holds the tile as kD / 32 boxes of [64 queries][32 dims] fp32, 128-byte rows with the TMA 128-byte
      // swizzle (16-byte unit u of row q at u ^ (q & 7)), so that the eight rows one store instruction writes fall
      // into distinct banks: 2 shared-memory wavefronts per warp store instead of 8 with 512-byte unswizzled rows.
      // Warpgroup w owns boxes 2 w and 2 w + 1 (dims [64 w, 64 w + 64)) and adds them itself: its 128 threads
      // meet at their own barrier and its thread 0 issues the two reduce-adds, so the groups do not wait for each
      // other between the dQ GEMM and the next tile's S^T.
      const int q0 = 16 * (wtid >> 5) + (lane >> 2);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int q = q0 + 8 * h;
        uint8_t* row = reinterpret_cast<uint8_t*>(smem_dq) + q * 128 + (quad_col & 3) * 4;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int box = 2 * w + (j >> 2), unit = 2 * (j & 3) + (quad_col >> 2);
          *reinterpret_cast<float2*>(row + box * (kTileQ * 128) + ((unit ^ (q & 7)) << 4)) =
              make_float2(dq[4 * j + 2 * h], dq[4 * j + 2 * h + 1]);
        }
      }
      fence_proxy_async_smem();
    }
    // head dim 64: group 0 computes all of dQ, and both groups still meet here (letting group 1 run ahead into the
    // next tile made the head-dim-64 backward slower on an H100)
    if constexpr (kD == 128) named_bar_sync(6 + w, 128);
    else named_bar_sync(3, kThreads);
    if (do_dq && wtid == 0) {
#pragma unroll
      for (int b = 2 * w; b < 2 * w + 2; ++b)
        tma_reduce_add_3d(&tm_dq, reinterpret_cast<uint8_t*>(smem_dq) + b * (kTileQ * 128), 32 * b, tiles[stage].head,
                          tiles[stage].row);
      tma_store_commit();
    }
    RFA_STAMP(tid == 0, i, 5);
  }
  // the unused S^T issued after the last tile has retired, and every reduce-add of this group has been read out
  // and written, before the epilogue reuses shared memory
  wgmma_wait<0>();
  if (wtid == 0) tma_store_wait<0>();

  // ---------------------------------------------------------------- epilogue: dK / dV -> global
  const bool remote = p.dkv.world > 0;
  if (remote && wtid == 0) {
    // the owner must have drained what we stored into its inbox during the previous backward call
    wait_epoch(p.dkv.my_pad + kPadInboxFree + it.owner, p.dkv.wait_epoch);
  }
  // every GEMM of this CTA has retired and every TMA load has landed: K | V | the Q/dO ring are free
  named_bar_sync(1, kThreads);
  // Every thread parks its fragments of dK (rows [0, 128) of the staging area) and dV (rows [128, 256)) in shared
  // memory; then each of the 128 threads of a warpgroup ships ONE row of its 64 keys (dK for threads 0-63, dV
  // for 64-127) with one bulk copy.  Rows are pitched 16 bytes past their length so that the 16-byte stores
  // fall into distinct bank groups.  The row is written in the model dtype (fused multi-GPU launches and world
  // size 1: half the NVLink / HBM bytes of fp32 rows, and no cast pass afterwards; the owner-side reduction
  // accumulates the partials of different ranks in fp32) or in fp32 (torch.distributed fallback transports,
  // which add the partials of successive ring steps).
  auto store_rows = [&](auto tag) {
    using O = decltype(tag);
    constexpr int kRowBytes = kD * static_cast<int>(sizeof(O));
    constexpr int kPitch = kRowBytes + 16;
    static_assert(2 * kTileK * kPitch <= 2 * kKVBytes + kStages * 2 * kQBytes, "staging must fit in K|V|Q/dO");
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int key = 64 * w + k_lo + 8 * h;
      uint8_t* rk = smem_k + key * kPitch;
      uint8_t* rv = smem_k + (kTileK + key) * kPitch;
#pragma unroll
      for (int j = 0; j < kD / 8; ++j) {
        const int c = 8 * j + quad_col;
        if constexpr (sizeof(O) == 4) {
          *reinterpret_cast<float2*>(rk + c * 4) = make_float2(dk[4 * j + 2 * h], dk[4 * j + 2 * h + 1]);
          *reinterpret_cast<float2*>(rv + c * 4) = make_float2(dv[4 * j + 2 * h], dv[4 * j + 2 * h + 1]);
        } else {
          *reinterpret_cast<uint32_t*>(rk + c * 2) = Pack2<T>::pack(dk[4 * j + 2 * h], dk[4 * j + 2 * h + 1]);
          *reinterpret_cast<uint32_t*>(rv + c * 2) = Pack2<T>::pack(dv[4 * j + 2 * h], dv[4 * j + 2 * h + 1]);
        }
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(4 + w, 128);
    const int key = 64 * w + (wtid & 63);
    const bool is_dv = wtid >= 64;
    if (key < it.kv_rows) {
      const int row = (remote ? it.out_row0 : it.kv_row0) + key;
      uint8_t* base = static_cast<uint8_t*>(remote ? (is_dv ? p.dkv.dv_ptrs[it.owner] : p.dkv.dk_ptrs[it.owner])
                                                   : (is_dv ? p.dv : p.dk));
      bulk_store(base + (static_cast<size_t>(row) * p.hkv + kv_head) * kRowBytes,
                 smem_k + ((is_dv ? kTileK : 0) + key) * kPitch, kRowBytes);
      tma_store_commit();
      tma_store_wait<0>();  // written, not just read: the flag below must not overtake the data
      fence_proxy_async_all();
    }
  };
  if (p.dkv_fp32) store_rows(float{});
  else store_rows(T{});
  if (remote) {
    // publish: the last tile destined for an owner raises that owner's "gradients landed" flag
    __threadfence_system();
    named_bar_sync(1, kThreads);  // both groups have stored and fenced their rows
    if (tid == 0) {
      const uint32_t old = atomicAdd(p.dkv.sent_count + it.owner, 1u);
      if (old + 1u == p.dkv.sent_target[it.owner]) {
        __threadfence_system();
        st_release_sys(p.dkv.peer_pads[it.owner] + kPadDkvReady + p.dkv.my_rank, p.dkv.epoch);
      }
    }
  }

  __syncthreads();
  if (tid == 0 && p.sig.world > 0) consumer_done(p.sig);
}

// delta[h, t] = sum_d out[t,h,d] * dout[t,h,d]; one warp per (row, head).
template <typename T>
__global__ void bwd_delta_kernel(const T* __restrict__ out, const T* __restrict__ dout, float* __restrict__ delta,
                                 int rows, int hq, int lse_S, int64_t o_rs, int64_t o_hs, int64_t do_rs,
                                 int64_t do_hs, int head_dim) {
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= rows * hq) return;
  const int row = gw / hq, head = gw % hq;
  float s = 0.f;
  if (lane * 4 < head_dim) {  // 4 elements per lane: 32 lanes cover head_dim 128, 16 lanes head_dim 64
    const uint2 a = *reinterpret_cast<const uint2*>(out + row * o_rs + head * o_hs + lane * 4);
    const uint2 b = *reinterpret_cast<const uint2*>(dout + row * do_rs + head * do_hs + lane * 4);
    const T* pa = reinterpret_cast<const T*>(&a);
    const T* pb = reinterpret_cast<const T*>(&b);
#pragma unroll
    for (int i = 0; i < 4; ++i) s += static_cast<float>(pa[i]) * static_cast<float>(pb[i]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    const size_t b_ = row / lse_S, sidx = row % lse_S;
    delta[(b_ * hq + head) * static_cast<size_t>(lse_S) + sidx] = s;
  }
}

}  // namespace bwd

const char* attn_bwd_delta_launch(int dtype, const TensorView& out, const TensorView& dout, float* delta, int lse_S,
                                  int head_dim, cudaStream_t stream) {
  const int rows = static_cast<int>(out.rows), hq = out.heads;
  const long long warps = static_cast<long long>(rows) * hq;
  if (warps == 0) return nullptr;
  const int threads = 256;
  const int blocks = static_cast<int>((warps * 32 + threads - 1) / threads);
  if (dtype == kDtypeBF16) {
    bwd::bwd_delta_kernel<__nv_bfloat16><<<blocks, threads, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(out.ptr), static_cast<const __nv_bfloat16*>(dout.ptr), delta, rows, hq, lse_S,
        out.row_stride, out.head_stride, dout.row_stride, dout.head_stride, head_dim);
  } else {
    bwd::bwd_delta_kernel<__half><<<blocks, threads, 0, stream>>>(
        static_cast<const __half*>(out.ptr), static_cast<const __half*>(dout.ptr), delta, rows, hq, lse_S,
        out.row_stride, out.head_stride, dout.row_stride, dout.head_stride, head_dim);
  }
  cudaError_t err = cudaGetLastError();
  return err == cudaSuccess ? nullptr : cudaGetErrorString(err);
}

const char* attn_bwd_launch(int dtype, const TensorView& q, const TensorView& dout, const TensorView& k,
                            const TensorView& v, const TensorView& k_stage, const TensorView& v_stage,
                            const TensorView& dq_accum, const BwdParams& p, cudaStream_t stream) {
  const int n_blocks = p.push.n_ctas + p.n_items * p.hkv;
  if (n_blocks <= 0) return nullptr;
  if (p.sig.world > 0) set_peer_timeout_from_env();
  CUtensorMap tq, tdo, tk, tv, tks, tvs, tdq;
  const int d = p.head_dim;
  if (d != 64 && d != 128) return "the sm_90a backward is instantiated for head_dim 64 and 128";
  if (const char* e = make_tensor_map(&tq, q, 2, bwd::kTileQ, d)) return e;
  if (const char* e = make_tensor_map(&tdo, dout, 2, bwd::kTileQ, d)) return e;
  if (const char* e = make_tensor_map(&tk, k, 2, bwd::kTileK, d)) return e;
  if (const char* e = make_tensor_map(&tv, v, 2, bwd::kTileK, d)) return e;
  if (const char* e = make_tensor_map(&tks, k_stage, 2, bwd::kTileK, d)) return e;
  if (const char* e = make_tensor_map(&tvs, v_stage, 2, bwd::kTileK, d)) return e;
  if (const char* e = make_tensor_map(&tdq, dq_accum, 4, bwd::kTileQ, d)) return e;  // 32-float swizzled boxes
  dim3 grid(n_blocks, 1, 1), block(bwd::kThreads, 1, 1);
  cudaError_t err;
  err = cudaSuccess;
  auto launch = [&](auto kern, int smem) {
    if (p.push.n_ctas > 0 && smem < kPushSmemBytes) smem = kPushSmemBytes;  // (head dim 64: the push ring is larger)
    err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (err == cudaSuccess) kern<<<grid, block, smem, stream>>>(tq, tdo, tk, tv, tks, tvs, tdq, p);
  };
  auto pick = [&](auto tag) {
    using T = decltype(tag);
    if (d == 128) {
      if (p.window) launch(bwd::attn_bwd_kernel<T, true, 128>, bwd::Geo<128>::kSmemBytes);
      else launch(bwd::attn_bwd_kernel<T, false, 128>, bwd::Geo<128>::kSmemBytes);
    } else {
      if (p.window) launch(bwd::attn_bwd_kernel<T, true, 64>, bwd::Geo<64>::kSmemBytes);
      else launch(bwd::attn_bwd_kernel<T, false, 64>, bwd::Geo<64>::kSmemBytes);
    }
  };
  if (dtype == kDtypeBF16) pick(__nv_bfloat16{});
  else pick(__half{});
  if (err != cudaSuccess) return cudaGetErrorString(err);
  err = cudaGetLastError();
  return err == cudaSuccess ? nullptr : cudaGetErrorString(err);
}

}  // namespace rfa
