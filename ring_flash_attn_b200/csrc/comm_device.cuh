// Device-side NVLink communication roles that live INSIDE the attention kernels.
//
// The reference rotates K/V (and fp32 dK/dV) around the ring with NCCL isend/irecv between flash_attn calls
// (/root/reference/ring_flash_attn/utils.py:98-151).  Here every GPU is one NVSwitch hop from every other, so:
//
//  * "push" CTAs (the first blocks of the attention grid) stream the rows of the local K/V shard that each
//    peer will need straight into that peer's staging buffer with posted stores over NVLink, in ring order
//    (next neighbour first), and raise a per-source "landed" flag in the peer's signal pad;
//  * compute CTAs wait on those flags only when they reach a remote segment, so the transfer of shard s+1
//    overlaps the tensor-core work on shard s inside one kernel launch;
//  * when the last compute CTA retires it tells every source that its staging buffer may be overwritten;
//  * backward compute CTAs store their dK/dV tiles directly into the owner's fp32 inbox and the last tile for
//    an owner raises that owner's "gradients landed" flag.
//
// All cross-GPU flags are monotonically increasing epochs (one per collective call), so nothing is reset.
#pragma once
#include <cstdlib>

#include "attn_common.h"
#include "sm90_ptx.cuh"

namespace rfa {

// Copy RFA_B200_PEER_TIMEOUT_S into this translation unit's g_peer_timeout_ns (once per process and unit).
inline void set_peer_timeout_from_env() {
  static const bool done = [] {
    if (const char* e = std::getenv("RFA_B200_PEER_TIMEOUT_S")) {
      const double s = std::atof(e);
      const unsigned long long ns = s <= 0 ? 0ull : static_cast<unsigned long long>(s * 1e9);
      cudaMemcpyToSymbol(g_peer_timeout_ns, &ns, sizeof(ns));
    }
    return true;
  }();
  (void)done;
}

// Epochs are compared with wrap-around safe signed distance.
__device__ __forceinline__ bool epoch_reached(uint32_t have, uint32_t want) {
  return static_cast<int32_t>(have - want) >= 0;
}
// Traps (without a message, see RFA_WATCHDOG_NS in sm90_ptx.cuh) after RFA_B200_PEER_TIMEOUT_S; 0 disables the limit.
__device__ __forceinline__ void wait_epoch(const uint32_t* flag, uint32_t want) {
  if (epoch_reached(ld_acquire_sys(flag), want)) return;
  const uint64_t t0 = global_timer_ns();
  const unsigned long long limit = g_peer_timeout_ns;
  while (!epoch_reached(ld_acquire_sys(flag), want)) {
    if (limit != 0 && global_timer_ns() - t0 > limit) __trap();
    __nanosleep(64);  // the peer is microseconds to seconds away: do not hammer the memory system while spinning
  }
}

__device__ __forceinline__ uint4 ld_nc_v4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void st_v4(uint4* p, const uint4& v) {
  asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// Task ti of this launch.  Static mode: a row of the host-built table.  Dynamic mode: tasks are enumerated as
// (ring step, K|V, range, chunk) and cut out of the destination's all-gathered needs; rows == 0 means "nothing to
// copy" (the task still counts towards the destination's "everything is out" target).
__device__ __forceinline__ PushTask push_task_at(const PushParams& pp, int ti) {
  if (pp.tasks != nullptr) return pp.tasks[ti];
  PushTask t;
  const int per_dst = 2 * kNeedRanges * pp.dyn_chunks;
  const int step = ti / per_dst + 1;
  int rem = ti - (step - 1) * per_dst;
  t.dst = (pp.my_rank + step) % pp.world;
  t.which = rem / (kNeedRanges * pp.dyn_chunks);
  rem -= t.which * (kNeedRanges * pp.dyn_chunks);
  const int range = rem / pp.dyn_chunks, c = rem - range * pp.dyn_chunks;
  const int* nd = pp.dyn_needs + ((t.dst * pp.world + pp.my_rank) * kNeedRanges + range) * 2;
  const int lo = nd[0], hi = nd[1];
  const long long r0 = static_cast<long long>(lo) + static_cast<long long>(c) * pp.dyn_chunk_rows;
  const long long n = r0 < hi ? (hi - r0 < pp.dyn_chunk_rows ? hi - r0 : pp.dyn_chunk_rows) : 0;
  t.rows = static_cast<int>(n);
  t.src_row = r0;
  t.dst_off = t.which * pp.region_bytes + (static_cast<long long>(pp.my_rank) * pp.rows_cap + r0) * pp.row_bytes;
  t.pad = 0;
  return t;
}

// Body of a push CTA.  Tasks are sorted by destination in ring order; CTA b takes tasks b, b + n, ...
__device__ __forceinline__ void push_role(const PushParams& pp) {
  const int tid = threadIdx.x, nthr = blockDim.x;
  __shared__ int s_last;
  for (int ti = blockIdx.x; ti < pp.n_tasks; ti += pp.n_ctas) {
    const PushTask t = push_task_at(pp, ti);
    if (tid == 0 && pp.epoch > 2 && t.rows > 0) {
      // the destination must have finished reading what we pushed into this staging parity two calls ago
      wait_epoch(pp.my_pad + kPadConsumed + t.dst, pp.epoch - 2);
    }
    __syncthreads();
    const int vec_per_row = pp.row_bytes >> 4;
    const long long total = static_cast<long long>(t.rows) * vec_per_row;
    const long long src_pitch = pp.src_row_bytes[t.which];
    const char* src = pp.src_base[t.which] + t.src_row * src_pitch;
    char* dst = pp.stage_ptrs[t.dst] + pp.parity_off + t.dst_off;
    constexpr int U = 8;
    for (long long base = static_cast<long long>(tid); base < total; base += static_cast<long long>(nthr) * U) {
      uint4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long e = base + static_cast<long long>(u) * nthr;
        if (e < total) {
          const long long r = e / vec_per_row, c = e - r * vec_per_row;
          v[u] = ld_nc_v4(reinterpret_cast<const uint4*>(src + r * src_pitch + c * 16));
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long e = base + static_cast<long long>(u) * nthr;
        if (e < total) st_v4(reinterpret_cast<uint4*>(dst + e * 16), v[u]);
      }
    }
    __threadfence_system();
    __syncthreads();
    if (tid == 0) {
      const uint32_t old = atomicAdd(pp.sent_count + t.dst, 1u);
      s_last = (old + 1u == pp.sent_target[t.dst]) ? 1 : 0;
      if (s_last) {
        __threadfence_system();
        st_release_sys(pp.peer_pads[t.dst] + kPadKvReady + pp.my_rank, pp.epoch);
      }
    }
    __syncthreads();
  }
}

// ---- TMA variant of the push role -----------------------------------------------------------------------
// One thread drives bulk copies local HBM -> shared memory -> peer HBM through a ring of 32 KB buffers, so a
// single CTA keeps ~100 KB of loads and ~100 KB of NVLink stores in flight (the LSU loop above is limited to
// the 48 KB its threads can hold in registers and measured only ~16 GB/s per CTA).
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_store(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)),
               "r"(bytes)
               : "memory");
}

constexpr int kPushBufBytes = 32768;
constexpr int kPushBufs = 6;
constexpr int kPushDepth = 3;  // loads in flight; with 6 buffers at most 2 store groups may still be reading
// dynamic shared memory a launch with push CTAs must provide (buffers + mbarriers + 1 KB alignment slack)
constexpr int kPushSmemBytes = kPushBufs * kPushBufBytes + 1024 + 1024;

__device__ __forceinline__ void push_role_tma(const PushParams& pp, uint8_t* smem) {
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kPushBufs * kPushBufBytes);
  if (threadIdx.x == 0) {
    for (int i = 0; i < kPushBufs; ++i) mbar_init(&bars[i], 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const int rows_per_piece = pp.row_bytes >= kPushBufBytes ? 1 : kPushBufBytes / pp.row_bytes;
  uint32_t n_loaded = 0, n_stored = 0;  // global piece counters (ring position / parity)
  // Completion is published per DESTINATION, not per task: the tasks of a CTA are sorted by destination, so the
  // copy pipeline keeps running across task boundaries and is drained (all bytes written, system-scope fence)
  // only when the destination changes: draining after every task would cost a load-latency fill plus an NVLink
  // write-completion wait per task.
  int cur_dst = -1;
  uint32_t pending = 0;  // finished tasks for cur_dst that are not yet counted
  auto publish = [&]() {
    if (pending == 0) return;
    tma_store_wait<0>();  // every byte for this destination has been written
    fence_proxy_async_all();
    __threadfence_system();
    const uint32_t old = atomicAdd(pp.sent_count + cur_dst, pending);
    if (old + pending == pp.sent_target[cur_dst]) {
      __threadfence_system();
      st_release_sys(pp.peer_pads[cur_dst] + kPadKvReady + pp.my_rank, pp.epoch);
    }
    pending = 0;
  };
  for (int ti = blockIdx.x; ti < pp.n_tasks; ti += pp.n_ctas) {
    const PushTask t = push_task_at(pp, ti);
    if (t.dst != cur_dst) {
      publish();
      cur_dst = t.dst;
    }
    if (pp.epoch > 2 && t.rows > 0)
      wait_epoch(pp.my_pad + kPadConsumed + t.dst, pp.epoch - 2);
    const long long pitch = pp.src_row_bytes[t.which];
    const char* src = pp.src_base[t.which] + t.src_row * pitch;
    char* dst = pp.stage_ptrs[t.dst] + pp.parity_off + t.dst_off;
    const int pieces = (t.rows + rows_per_piece - 1) / rows_per_piece;
    int ld = 0, stv = 0;
    while (stv < pieces) {
      while (ld < pieces && ld - stv < kPushDepth) {
        const uint32_t slot = n_loaded % kPushBufs;
        if (n_loaded >= kPushBufs) tma_store_wait_read<2>();  // the store that last used this buffer is done reading
        const int r0 = ld * rows_per_piece;
        const int nr = min(rows_per_piece, t.rows - r0);
        uint8_t* buf = smem + slot * kPushBufBytes;
        mbar_arrive_expect_tx(&bars[slot], static_cast<uint32_t>(nr) * pp.row_bytes);
        if (pitch == pp.row_bytes) {
          bulk_load(buf, src + static_cast<long long>(r0) * pitch, static_cast<uint32_t>(nr) * pp.row_bytes, &bars[slot]);
        } else {
          for (int r = 0; r < nr; ++r)
            bulk_load(buf + r * pp.row_bytes, src + static_cast<long long>(r0 + r) * pitch, pp.row_bytes, &bars[slot]);
        }
        ++n_loaded;
        ++ld;
      }
      const uint32_t slot = n_stored % kPushBufs;
      mbar_wait(&bars[slot], (n_stored / kPushBufs) & 1);
      const int r0 = stv * rows_per_piece;
      const int nr = min(rows_per_piece, t.rows - r0);
      bulk_store(dst + static_cast<long long>(r0) * pp.row_bytes, smem + slot * kPushBufBytes,
                 static_cast<uint32_t>(nr) * pp.row_bytes);
      tma_store_commit();
      ++n_stored;
      ++stv;
    }
    ++pending;
  }
  publish();
}

// Called by one thread of every compute CTA after the CTA has finished reading staged K/V.
__device__ __forceinline__ void consumer_done(const SignalParams& sp) {
  if (sp.peer_pads == nullptr) return;
  __threadfence();
  const uint32_t old = atomicAdd(sp.done_count, 1u);
  if (old + 1u == sp.done_target) {
    __threadfence_system();
    for (int r = 0; r < sp.world; ++r) {
      if (r == sp.my_rank) continue;
      st_release_sys(sp.peer_pads[r] + kPadConsumed + sp.my_rank, sp.epoch);
    }
  }
}

}  // namespace rfa
