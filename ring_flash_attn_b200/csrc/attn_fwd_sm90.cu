// Blockwise flash-attention forward for sm_90a (head_dim 64 / 128, bf16 / fp16, and e4m3 with block descales).
//
// One CTA = one work item (<= 128 query rows of one chunk) x one query head.  The CTA walks a *segment list*:
// runs of keys - possibly from several source ranks - each with its own causal diagonal.  The output
// accumulator never leaves registers between segments, so a whole ring / zigzag / stripe / llama3 forward is
// ordinary online softmax over the concatenated segments (this replaces the reference's flash_attn call + fp32
// out/lse merge per ring step, /root/reference/ring_flash_attn/ring_flash_attn.py:26-63 and utils.py:32-73).
//
// Roles (288 threads):
//   warpgroup 0   query rows [0, 64) of the item, warpgroup 1 rows [64, 128): S = Q K^T (wgmma, both operands
//                 in shared memory), mask, online softmax in registers, O += P V (wgmma, P from registers, V
//                 MN-major from shared memory), final normalisation + store of out / lse
//   warp 8        TMA producer (one thread): the Q tile once, then K / V tiles through a ring of kStages slots
// A warpgroup whose rows cannot see a key tile (causal diagonal) skips its GEMMs and only releases the slots.
#include <math_constants.h>
#include <stdio.h>

#include <cstdlib>
#include <type_traits>

#include "attn_common.h"
#include "comm_device.cuh"
#include "sm90_ptx.cuh"

namespace rfa {

namespace fwd {

#ifdef RFA_TRACE
// slot layout per key-tile iteration (16 stamps), thread 0 of each compute warpgroup w: 8w + 0 S complete,
// 8w + 1 P ready, 8w + 2 P V complete
#define RFA_STAMP(cond, iter, slot)                                                              \
  do {                                                                                            \
    if ((cond) && cta == 0 && p.trace != nullptr && (iter) < 64) p.trace[(iter)*16 + (slot)] = clock64(); \
  } while (0)
#else
#define RFA_STAMP(cond, iter, slot) \
  do {                              \
  } while (0)
#endif

constexpr int kTile = 128;               // query rows per CTA and keys per K / V tile
constexpr int kRowsWG = 64;              // query rows per compute warpgroup (wgmma M)
constexpr int kStages = 4;               // K/V ring slots (one key tile takes two: K, then V)
constexpr int kHalfBytes = kTile * 128;  // one 64-element-wide (128-byte) swizzled sub-tile of 16-bit elements
constexpr int kThreads = 288;  // two compute warpgroups + one producer warp

// Element traits.  Fp8E4M3 is the tag of the fp8 forward: q / k / v are e4m3 bytes, a tile is ONE 128-byte
// swizzle span per row; S = Q K^T runs as an e4m3 wgmma (K = 32 per instruction).  wgmma takes 8-bit operands
// only K-major, and V is MN-major for P V, so every compute warpgroup widens the V tile to bf16 in its own shared
// buffer and P V runs in bf16.  Block descales (q: per token block x head, k / v: per 128-token block x kv head,
// or coarser) come in through FwdParams::q_scale / k_scale / v_scale; they are applied to the fp32 scores and
// folded into P, at no extra tensor-core or memory cost.  The output is bf16.
struct Fp8E4M3 {};
template <typename T>
struct Elem {
  static constexpr bool kFp8 = false;
  static constexpr uint32_t kBytes = 2;
  using Out = T;
  using Pv = T;  // element type of the P V GEMM
};
template <>
struct Elem<Fp8E4M3> {
  static constexpr bool kFp8 = true;
  static constexpr uint32_t kBytes = 1;
  using Out = __nv_bfloat16;
  using Pv = __nv_bfloat16;
};

template <typename T, int kD>
constexpr int slot_bytes() {
  return kTile * kD * static_cast<int>(Elem<T>::kBytes);
}
template <typename T, int kD>
constexpr int smem_bytes() {
  return slot_bytes<T, kD>() /*Q*/ + kStages * slot_bytes<T, kD>() +
         (Elem<T>::kFp8 ? 2 * kTile * kD * 2 : 0) /*bf16 V, one per compute warpgroup*/ + 1024 /*barriers*/ +
         1024 /*align slack*/;
}

struct Barriers {
  uint64_t q_full;
  uint64_t kv_full[kStages];
  uint64_t kv_empty[kStages];
};

// Per-(item, segment) geometry shared by all roles so that they agree on the iteration space.
struct SegGeom {
  int kv_row0, kv_len, diag;
  int n_tiles;  // key tiles to visit
};

__device__ __forceinline__ SegGeom seg_geom(const KVSegment& s, const WorkItem& it) {
  SegGeom g;
  g.kv_row0 = s.kv_row0;
  g.kv_len = s.kv_len;
  g.diag = s.diag;
  const int last_row = it.q_off + it.q_rows - 1;
  long long lim = static_cast<long long>(last_row) + s.diag + 1;  // keys [0, lim) reachable by the last row
  int reach = lim < 0 ? 0 : (lim > s.kv_len ? s.kv_len : static_cast<int>(lim));
  g.n_tiles = (reach + kTile - 1) / kTile;
  return g;
}
// Do the rows of warpgroup w (item rows [64 w, 64 w + 64)) touch key tile jj at all?
__device__ __forceinline__ bool wg_active(const SegGeom& g, const WorkItem& it, int w, int jj) {
  const int n_w = it.q_rows - w * kRowsWG;
  if (n_w <= 0) return false;
  const int last_row = it.q_off + w * kRowsWG + (n_w < kRowsWG ? n_w : kRowsWG) - 1;
  return static_cast<long long>(jj) * kTile <= static_cast<long long>(last_row) + g.diag;
}
__device__ __forceinline__ bool wg_needs_mask(const SegGeom& g, const WorkItem& it, int w, int jj) {
  const int first_row = it.q_off + w * kRowsWG;
  const bool ragged = (jj + 1) * kTile > g.kv_len;
  const bool diagonal = static_cast<long long>(jj) * kTile + (kTile - 1) > static_cast<long long>(first_row) + g.diag;
  return ragged || diagonal;
}
// Sliding window (kWindow kernels): key j of the segment is visible to chunk row i only if j >= i + lo.  The host
// trims every segment per work item so that the loop still starts at key tile 0 (ops/attn_cuda.py); what remains
// for the kernel is the slanted lower edge of the band.
__device__ __forceinline__ bool wg_needs_lower_mask(int lo, const WorkItem& it, int w, int jj) {
  const long long last_row = static_cast<long long>(it.q_off) + w * kRowsWG + (kRowsWG - 1);
  return last_row + lo > static_cast<long long>(jj) * kTile;
}

// e4m3 V tile (one 128-byte swizzled span per key) -> bf16 V tile in the 16-bit layout (two 64-dim sub-tiles of
// 128-byte swizzled rows), by the 128 threads of one warpgroup.
__device__ __forceinline__ void widen_v_tile(const uint8_t* src, uint8_t* dst, int wtid) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int idx = wtid + 128 * i;
    const int r = idx >> 3, cc = idx & 7;  // key row, 16-dim chunk
    const uint4 x = *reinterpret_cast<const uint4*>(src + r * 128 + ((cc ^ (r & 7)) << 4));
    uint4 lo, hi;
    lo.x = e4m3x2_to_bf16x2(x.x);
    lo.y = e4m3x2_to_bf16x2(x.x >> 16);
    lo.z = e4m3x2_to_bf16x2(x.y);
    lo.w = e4m3x2_to_bf16x2(x.y >> 16);
    hi.x = e4m3x2_to_bf16x2(x.z);
    hi.y = e4m3x2_to_bf16x2(x.z >> 16);
    hi.z = e4m3x2_to_bf16x2(x.w);
    hi.w = e4m3x2_to_bf16x2(x.w >> 16);
    uint8_t* row = dst + (cc >> 2) * kHalfBytes + r * 128;
    const int c0 = 2 * (cc & 3);
    *reinterpret_cast<uint4*>(row + ((c0 ^ (r & 7)) << 4)) = lo;
    *reinterpret_cast<uint4*>(row + (((c0 + 1) ^ (r & 7)) << 4)) = hi;
  }
}

template <typename T, bool kWindow, int kD>
__global__ void __launch_bounds__(kThreads, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                const __grid_constant__ CUtensorMap tm_v, const __grid_constant__ CUtensorMap tm_ks,
                const __grid_constant__ CUtensorMap tm_vs, const __grid_constant__ FwdParams p) {
  // The first blocks of the grid are communication CTAs: they push this rank's K/V rows to the peers that
  // need them while the remaining (compute) CTAs already work on the local shard.
  if (static_cast<int>(blockIdx.x) < p.push.n_ctas) {
    if (p.push.use_tma) {
      extern __shared__ uint8_t push_smem_raw[];
      push_role_tma(p.push, reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(push_smem_raw) + 1023) & ~uintptr_t(1023)));
    } else {
      push_role(p.push);
    }
    return;
  }
  using E = Elem<T>;
  using Pv = typename E::Pv;
  static_assert(kD == 64 || kD == 128, "head dim 64 or 128");
  static_assert(!E::kFp8 || kD == 128, "the fp8 forward is instantiated for head dim 128 only");
  constexpr int kSlotBytes = slot_bytes<T, kD>();
  constexpr int kSubTiles = E::kFp8 ? 1 : kD / 64;  // 128-byte spans per row
  constexpr uint32_t kTxBytes = kTile * kD * E::kBytes;
  const int cta = static_cast<int>(blockIdx.x) - p.push.n_ctas;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_q = smem;
  uint8_t* smem_kv = smem + kSlotBytes;                  // kStages slots
  uint8_t* smem_vb = smem_kv + kStages * kSlotBytes;     // fp8 only: 2 x bf16 V tile
  Barriers* bars = reinterpret_cast<Barriers*>(smem_vb + (E::kFp8 ? 2 * kTile * kD * 2 : 0));

  const int head = cta / p.n_items;  // consecutive CTAs share a head => K/V tiles are reused out of L2
  const int kv_head = head / (p.hq / p.hkv);
  WorkItem it = p.items[cta % p.n_items];
  if (p.flags & 4) it.seg_count = 0;  // timing experiment: communication only (compute CTAs have nothing to do)

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    tma_prefetch_desc(&tm_ks);
    tma_prefetch_desc(&tm_vs);
    mbar_init(&bars->q_full, 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&bars->kv_full[i], 1);
      mbar_init(&bars->kv_empty[i], 8);  // one arrival per compute warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x >= 256) {
    // ------------------------------------------------------------------ TMA producer
    if (threadIdx.x == 256) {
      mbar_arrive_expect_tx(&bars->q_full, kTxBytes);
#pragma unroll
      for (int h = 0; h < kSubTiles; ++h)
        tma_load_3d(smem_q + h * kHalfBytes, &tm_q, &bars->q_full, 64 * h, head, it.q_row0);
      uint32_t slot = 0, phase = 0;
      for (int si = 0; si < it.seg_count; ++si) {
        const KVSegment sg = p.segs[it.seg_begin + si];
        const SegGeom g = seg_geom(sg, it);
        const bool staged = sg.flag >= 0 && p.ready_flags != nullptr;
        if (g.n_tiles > 0 && staged && !(p.flags & 2)) {  // (flags bit 1: timing experiment, compute only)
          wait_epoch(p.ready_flags + sg.flag, p.ready_epoch);
          fence_proxy_async_all();
        }
        for (int jj = 0; jj < g.n_tiles; ++jj) {
          const int row = g.kv_row0 + jj * kTile;
          for (int kv = 0; kv < 2; ++kv) {
            mbar_wait(&bars->kv_empty[slot], phase ^ 1);
            uint8_t* dst = smem_kv + slot * kSlotBytes;
            const CUtensorMap* tm = staged ? (kv == 0 ? &tm_ks : &tm_vs) : (kv == 0 ? &tm_k : &tm_v);
            mbar_arrive_expect_tx(&bars->kv_full[slot], kTxBytes);
#pragma unroll
            for (int h = 0; h < kSubTiles; ++h)
              tma_load_3d(dst + h * kHalfBytes, tm, &bars->kv_full[slot], 64 * h, kv_head, row);
            if (++slot == kStages) {
              slot = 0;
              phase ^= 1;
            }
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ compute warpgroups
    const int w = threadIdx.x >> 7;
    const int wtid = threadIdx.x & 127;
    const int lane = threadIdx.x & 31;
    const bool warp_leader = lane == 0;
    const int r_in_item = w * kRowsWG + 16 * (wtid >> 5) + (lane >> 2);  // this thread's rows: r_in_item, + 8
    const int quad_col = 2 * (lane & 3);                                  // its columns: 8 j + quad_col + {0, 1}
    const bool stamper = wtid == 0;
    (void)stamper;

    // Scores in log2 units are s * t2 with t2 = softmax_scale * log2(e); the running max m2 is kept in those
    // units.  fp8 (block-scaled inputs): the descale of the query row (per token block x head) rides on t2 for the
    // whole row, the descale of the key block (128-token blocks x kv head, or per head) is multiplied in per key
    // tile, and the V descale of the key block enters P as a ratio to the head's largest V descale (so that P
    // keeps the range of an ordinary softmax) with the reference value applied once in the epilogue.
    float base_l2[2] = {p.scale_log2, p.scale_log2};
    [[maybe_unused]] float inv_vref = 1.f;
    if constexpr (E::kFp8) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r_in_item + 8 * h;
        const int qrow = it.q_row0 + (r < it.q_rows ? r : 0);
        base_l2[h] *= p.q_scale[static_cast<size_t>(qrow / p.q_scale_block) * p.hq + head];
      }
      inv_vref = 1.0f / p.v_ref[kv_head];
    }
    float o[kD / 2];
#pragma unroll
    for (int i = 0; i < kD / 2; ++i) o[i] = 0.f;
    float m2[2] = {-CUDART_INF_F, -CUDART_INF_F};
    float l[2] = {0.f, 0.f};

    const uint64_t q_desc = gmma_desc(smem_u32(smem_q) + w * kRowsWG * 128, 0);  // K-major A, this group's rows
    const uint64_t k_desc0 = gmma_desc(smem_u32(smem_kv), 0);                    // K tile, K-major B
    uint8_t* my_vb = smem_vb + w * (kTile * kD * 2);
    const uint64_t v_desc0 = E::kFp8 ? gmma_desc(smem_u32(my_vb), kHalfBytes)    // V tile, MN-major B
                                     : gmma_desc(smem_u32(smem_kv), kHalfBytes);

    mbar_wait(&bars->q_full, 0);
    uint32_t slot = 0, phase = 0;
    int xi = 0;
    for (int si = 0; si < it.seg_count; ++si) {
      const KVSegment sg = p.segs[it.seg_begin + si];
      const SegGeom g = seg_geom(sg, it);
      int seg_lo = 0;
      if constexpr (kWindow) seg_lo = p.seg_lo[it.seg_begin + si];
      // fp8: row of the key tile in the scale tables (staged rows are indexed like the staging buffer, local rows
      // are offset to this rank's slot)
      [[maybe_unused]] const long long scale_row0 =
          g.kv_row0 + ((sg.flag >= 0 && p.ready_flags != nullptr) ? 0ll : static_cast<long long>(p.kv_scale_row0));
      for (int jj = 0; jj < g.n_tiles; ++jj, ++xi) {
        const uint32_t k_slot = slot, k_phase = phase;
        if (++slot == kStages) {
          slot = 0;
          phase ^= 1;
        }
        const uint32_t v_slot = slot, v_phase = phase;
        if (++slot == kStages) {
          slot = 0;
          phase ^= 1;
        }
        if (!wg_active(g, it, w, jj)) {
          // nothing of this tile is visible to our rows; the slots are released only after they were filled, so
          // that the arrivals always count towards the fill they belong to
          mbar_wait(&bars->kv_full[k_slot], k_phase);
          mbar_wait(&bars->kv_full[v_slot], v_phase);
          __syncwarp();
          if (warp_leader) {
            mbar_arrive(&bars->kv_empty[k_slot]);
            mbar_arrive(&bars->kv_empty[v_slot]);
          }
          continue;
        }

        // ---- S = Q K^T
        mbar_wait(&bars->kv_full[k_slot], k_phase);
        float s[64];
        const uint64_t k_desc = gmma_desc_add(k_desc0, k_slot * kSlotBytes);
        wgmma_fence();
        if constexpr (E::kFp8) {
#pragma unroll
          for (int k = 0; k < kD / 32; ++k)
            wgmma_ss_m64n128k32_e4m3(s, gmma_desc_add(q_desc, 32 * k), gmma_desc_add(k_desc, 32 * k), k > 0);
        } else {
#pragma unroll
          for (int k = 0; k < kD / 16; ++k) {
            const uint32_t off = (k >> 2) * kHalfBytes + (k & 3) * 32;
            Gmma<T>::template ss128<0, 0>(s, gmma_desc_add(q_desc, off), gmma_desc_add(k_desc, off), k > 0);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(s);
        __syncwarp();
        if (warp_leader) mbar_arrive(&bars->kv_empty[k_slot]);
        RFA_STAMP(stamper, xi, 8 * w + 0);

        bool masked = wg_needs_mask(g, it, w, jj);
        if constexpr (kWindow) masked = masked || wg_needs_lower_mask(seg_lo, it, w, jj);
        if (masked) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const long long chunk_row = static_cast<long long>(it.q_off) + r_in_item + 8 * h;
            long long lim_ll = chunk_row + g.diag;
            if (lim_ll > g.kv_len - 1) lim_ll = g.kv_len - 1;
            lim_ll -= static_cast<long long>(jj) * kTile;
            const int lim = lim_ll < -1 ? -1 : (lim_ll > 127 ? 127 : static_cast<int>(lim_ll));
            int lo_lim = 0;
            if constexpr (kWindow) {
              const long long lo_ll = chunk_row + seg_lo - static_cast<long long>(jj) * kTile;
              lo_lim = lo_ll < 0 ? 0 : (lo_ll > 128 ? 128 : static_cast<int>(lo_ll));
            }
#pragma unroll
            for (int j = 0; j < 16; ++j) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int c = 8 * j + quad_col + e;
                if (c > lim || c < lo_lim) s[4 * j + 2 * h + e] = -CUDART_INF_F;
              }
            }
          }
        }

        float t2[2] = {base_l2[0], base_l2[1]};
        [[maybe_unused]] float log2_ratio = 0.f, inv_ratio = 1.f;
        if constexpr (E::kFp8) {
          const size_t sb = static_cast<size_t>((scale_row0 + static_cast<long long>(jj) * kTile) / p.kv_scale_block) *
                                p.hkv + kv_head;
          t2[0] *= p.k_scale[sb];
          t2[1] *= p.k_scale[sb];
          const float ratio = p.v_scale[sb] * inv_vref;
          log2_ratio = __log2f(ratio);
          inv_ratio = 1.0f / ratio;
        }
        // ---- online softmax (two rows per thread; a row lives in the 4 threads of a quad)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float mx = -CUDART_INF_F;
#pragma unroll
          for (int j = 0; j < 16; ++j) mx = fmaxf(mx, fmaxf(s[4 * j + 2 * h], s[4 * j + 2 * h + 1]));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          const float m_new = fmaxf(m2[h], mx * t2[h]);
          const float f = m_new == -CUDART_INF_F ? 1.f : fast_exp2(m2[h] - m_new);
          m2[h] = m_new;
          l[h] *= f;
#pragma unroll
          for (int j = 0; j < kD / 8; ++j) {
            o[4 * j + 2 * h] *= f;
            o[4 * j + 2 * h + 1] *= f;
          }
          const float mc = (m_new == -CUDART_INF_F ? 0.f : m_new) - log2_ratio;
          float sum = 0.f;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float x = fast_exp2(fmaf(s[4 * j + 2 * h + e], t2[h], -mc));
              s[4 * j + 2 * h + e] = x;
              sum += x;
            }
          }
          l[h] += sum * inv_ratio;
        }
        uint32_t pa[kTile / 16][4];
#pragma unroll
        for (int kk = 0; kk < kTile / 16; ++kk) pack_a<Pv>(pa[kk], s, kk);
        RFA_STAMP(stamper, xi, 8 * w + 1);

        // ---- O += P V
        mbar_wait(&bars->kv_full[v_slot], v_phase);
        uint64_t v_desc = v_desc0;
        if constexpr (E::kFp8) {
          named_bar_sync(1 + w, 128);  // the previous P V of this warpgroup has finished reading my_vb
          widen_v_tile(smem_kv + v_slot * kSlotBytes, my_vb, wtid);
          fence_proxy_async_smem();
          named_bar_sync(1 + w, 128);
          __syncwarp();
          if (warp_leader) mbar_arrive(&bars->kv_empty[v_slot]);
        } else {
          v_desc = gmma_desc_add(v_desc0, v_slot * kSlotBytes);
        }
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kTile / 16; ++kk) gmma_rs<Pv, kD>(o, pa[kk], gmma_desc_add(v_desc, kk * 2048), 1);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(o);
        if constexpr (!E::kFp8) {
          __syncwarp();
          if (warp_leader) mbar_arrive(&bars->kv_empty[v_slot]);
        }
        RFA_STAMP(stamper, xi, 8 * w + 2);
      }
    }

    // ---------------------------------------------------------------- epilogue: O / l -> out, lse
    using OutT = typename E::Out;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float lt = l[h];
      lt += __shfl_xor_sync(0xffffffffu, lt, 1);
      lt += __shfl_xor_sync(0xffffffffu, lt, 2);
      const int r = r_in_item + 8 * h;
      if (r >= it.q_rows) continue;
      const int row = it.q_row0 + r;
      float inv = lt > 0.f ? 1.0f / lt : 0.f;
      if constexpr (E::kFp8) inv *= p.v_ref[kv_head];
      OutT* out_row = reinterpret_cast<OutT*>(p.out) + (static_cast<size_t>(row) * p.hq + head) * kD;
#pragma unroll
      for (int j = 0; j < kD / 8; ++j)
        *reinterpret_cast<uint32_t*>(out_row + 8 * j + quad_col) =
            Pack2<OutT>::pack(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv);
      if ((lane & 3) == 0) {
        const float lse = lt > 0.f ? (m2[h] + __log2f(lt)) * 0.6931471805599453f : -CUDART_INF_F;
        const size_t b = row / p.lse_S, sidx = row % p.lse_S;
        p.lse[(b * p.hq + head) * static_cast<size_t>(p.lse_S) + sidx] = lse;
      }
    }
  }

  __syncthreads();
  if (threadIdx.x == 0 && p.sig.world > 0) consumer_done(p.sig);
}

}  // namespace fwd

const char* attn_fwd_launch(int dtype, const TensorView& q, const TensorView& k, const TensorView& v,
                            const TensorView& k_stage, const TensorView& v_stage, const FwdParams& p,
                            cudaStream_t stream) {
  const int n_blocks = p.push.n_ctas + p.n_items * p.hq;
  if (n_blocks <= 0) return nullptr;
  if (p.sig.world > 0) set_peer_timeout_from_env();
  CUtensorMap tq, tk, tv, tks, tvs;
  const int eb = dtype == kDtypeE4M3 ? 1 : 2;
  const int d = p.head_dim;
  if (d != 64 && d != 128) return "the sm_90a forward is instantiated for head_dim 64 and 128";
  if (dtype == kDtypeE4M3 && (p.q_scale == nullptr || p.k_scale == nullptr || p.v_scale == nullptr ||
                              p.v_ref == nullptr || p.q_scale_block < 1 || p.kv_scale_block < 1 ||
                              p.seg_lo != nullptr || d != 128))
    return "fp8 forward needs q / k / v descale tables and head_dim 128, and does not support sliding windows yet";
  if (const char* e = make_tensor_map(&tq, q, eb, fwd::kTile, d)) return e;
  if (const char* e = make_tensor_map(&tk, k, eb, fwd::kTile, d)) return e;
  if (const char* e = make_tensor_map(&tv, v, eb, fwd::kTile, d)) return e;
  if (const char* e = make_tensor_map(&tks, k_stage, eb, fwd::kTile, d)) return e;
  if (const char* e = make_tensor_map(&tvs, v_stage, eb, fwd::kTile, d)) return e;
  dim3 grid(n_blocks, 1, 1), block(fwd::kThreads, 1, 1);
  cudaError_t err = cudaSuccess;
  auto launch = [&](auto kern, int smem) {
    if (p.push.n_ctas > 0 && smem < kPushSmemBytes) smem = kPushSmemBytes;  // (head dim 64: the push ring is larger)
    err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (err == cudaSuccess) kern<<<grid, block, smem, stream>>>(tq, tk, tv, tks, tvs, p);
  };
  auto pick = [&](auto tag, auto window) {
    using T = decltype(tag);
    constexpr bool kW = decltype(window)::value;
    if (d == 128) launch(fwd::attn_fwd_kernel<T, kW, 128>, fwd::smem_bytes<T, 128>());
    else launch(fwd::attn_fwd_kernel<T, kW, 64>, fwd::smem_bytes<T, 64>());
  };
  if (dtype == kDtypeE4M3) {  // fp8 forward (e4m3 in, bf16 out)
    launch(fwd::attn_fwd_kernel<fwd::Fp8E4M3, false, 128>, fwd::smem_bytes<fwd::Fp8E4M3, 128>());
  } else if (p.seg_lo != nullptr) {  // sliding-window tables: the lower band edge is masked in-kernel
    if (dtype == kDtypeBF16) pick(__nv_bfloat16{}, std::true_type{});
    else pick(__half{}, std::true_type{});
  } else {
    if (dtype == kDtypeBF16) pick(__nv_bfloat16{}, std::false_type{});
    else pick(__half{}, std::false_type{});
  }
  if (err != cudaSuccess) return cudaGetErrorString(err);
  err = cudaGetLastError();
  return err == cudaSuccess ? nullptr : cudaGetErrorString(err);
}

}  // namespace rfa
