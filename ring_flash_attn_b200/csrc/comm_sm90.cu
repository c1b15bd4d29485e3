// Owner-side reduction of the backward "inbox".
//
// During the fused backward every rank stores its dK/dV partials for a shard (rounded once to the model dtype)
// directly into the shard owner's inbox slot over NVLink (attn_bwd_sm90.cu epilogue).  This kernel runs on the owner afterwards:
// it waits until every contributing rank has raised its "gradients landed" epoch, sums the slots that hold a
// partial for each row range in a fixed order (so the result is deterministic), writes dK/dV in the model
// dtype and finally tells every peer that the inbox may be reused.  It replaces the reference's W-hop fp32
// dK/dV ring (/root/reference/ring_flash_attn/ring_flash_attn.py:139-152) and llama3's blocking
// reduce_scatter (llama3_flash_attn_varlen.py:292-293).
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "attn_common.h"
#include "comm_device.cuh"

namespace rfa {
namespace comm {

template <typename T>
__device__ __forceinline__ uint2 pack4(const float4& a);
template <>
__device__ __forceinline__ uint2 pack4<__nv_bfloat16>(const float4& a) {
  return make_uint2(Pack2<__nv_bfloat16>::pack(a.x, a.y), Pack2<__nv_bfloat16>::pack(a.z, a.w));
}
template <>
__device__ __forceinline__ uint2 pack4<__half>(const float4& a) {
  return make_uint2(Pack2<__half>::pack(a.x, a.y), Pack2<__half>::pack(a.z, a.w));
}

template <typename T>
__device__ __forceinline__ float4 unpack4(const uint2& a);
template <>
__device__ __forceinline__ float4 unpack4<__nv_bfloat16>(const uint2& a) {
  // bf16 -> fp32 is a 16-bit shift
  return make_float4(__uint_as_float(a.x << 16), __uint_as_float(a.x & 0xffff0000u), __uint_as_float(a.y << 16),
                     __uint_as_float(a.y & 0xffff0000u));
}
template <>
__device__ __forceinline__ float4 unpack4<__half>(const uint2& a) {
  const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&a.x));
  const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&a.y));
  return make_float4(lo.x, lo.y, hi.x, hi.y);
}
__device__ __forceinline__ uint4 ldcv_u4(const uint4* p) {
  uint4 r;
  // written by a peer over NVLink: always read from L2, never from a stale L1 line
  asm volatile("ld.global.cv.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

// grid: (blocks_per_task, n_tasks).  The partials arrive in the model dtype (the backward epilogue rounds each
// rank's fp32 tile once - what flash-attn does for every block in the reference, ring_flash_attn.py:131-141) and
// are summed here in fp32 in fixed rank order.
template <typename T>
__global__ void __launch_bounds__(256) reduce_dkv_kernel(const __grid_constant__ ReduceParams p) {
  const ReduceTask t = p.tasks[blockIdx.y];
  // dynamic mode: which rows of my shard rank s returns = the rows it read = needs[s][me] (all-gathered table)
  __shared__ int s_need[kMaxRanks][kNeedRanges][2];
  const bool dyn = p.dyn_needs != nullptr;
  if (dyn) {
    for (int i = threadIdx.x; i < p.world * kNeedRanges * 2; i += blockDim.x) {
      const int s = i / (kNeedRanges * 2), j = i - s * (kNeedRanges * 2);
      (&s_need[s][0][0])[j] = p.dyn_needs[(s * p.world + p.my_rank) * kNeedRanges * 2 + j];
    }
    __syncthreads();
  }
  auto dyn_mask = [&](int row) {
    unsigned m = 0;
    for (int s = 0; s < p.world; ++s)
#pragma unroll
      for (int j = 0; j < kNeedRanges; ++j)
        if (row >= s_need[s][j][0] && row < s_need[s][j][1]) m |= 1u << s;
    return m;
  };
  if (threadIdx.x == 0) {
    for (int r = 0; r < p.world; ++r) {
      bool contributes = (t.src_mask >> r) & 1u;
      if (dyn) {
        contributes = false;
        for (int j = 0; j < kNeedRanges; ++j) contributes |= s_need[r][j][1] > s_need[r][j][0];
      }
      if (contributes && r != p.my_rank) wait_epoch(p.my_pad + kPadDkvReady + r, p.epoch);
    }
  }
  __syncthreads();
  // 8 elements (16 bytes) per access; rows are multiples of 128 elements, so a vector never straddles a row
  const long long n8 = static_cast<long long>(t.rows) * p.row_elems / 8;
  const long long off8 = static_cast<long long>(t.row0) * p.row_elems / 8;
  const long long slot8 = p.slot_stride / 8;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  constexpr int U = 4;
  for (int which = 0; which < 2; ++which) {
    const uint4* in = reinterpret_cast<const uint4*>(static_cast<const T*>(p.inbox) + which * p.kv_stride) + off8;
    uint4* out = reinterpret_cast<uint4*>(which == 0 ? p.dk : p.dv) + off8;
    for (long long i0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i0 < n8; i0 += stride * U) {
      float4 acc[U][2];
      unsigned mask[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        acc[u][0] = acc[u][1] = make_float4(0.f, 0.f, 0.f, 0.f);
        mask[u] = t.src_mask;
        if (dyn) mask[u] = dyn_mask(t.row0 + static_cast<int>((i0 + u * stride) * 8 / p.row_elems));
      }
      for (int r = 0; r < p.world; ++r) {
        if (!dyn && !((t.src_mask >> r) & 1u)) continue;
        uint4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const long long i = i0 + u * stride;
          v[u] = make_uint4(0u, 0u, 0u, 0u);
          if (i < n8 && ((mask[u] >> r) & 1u)) v[u] = ldcv_u4(in + r * slot8 + i);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const float4 lo = unpack4<T>(make_uint2(v[u].x, v[u].y)), hi = unpack4<T>(make_uint2(v[u].z, v[u].w));
          acc[u][0].x += lo.x; acc[u][0].y += lo.y; acc[u][0].z += lo.z; acc[u][0].w += lo.w;
          acc[u][1].x += hi.x; acc[u][1].y += hi.y; acc[u][1].z += hi.z; acc[u][1].w += hi.w;
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long i = i0 + u * stride;
        if (i < n8) {
          const uint2 lo = pack4<T>(acc[u][0]), hi = pack4<T>(acc[u][1]);
          out[i] = make_uint4(lo.x, lo.y, hi.x, hi.y);
        }
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const uint32_t old = atomicAdd(p.ticket, 1u);
    if (old + 1u == p.ticket_target) {
      __threadfence_system();
      for (int r = 0; r < p.world; ++r) st_release_sys(p.peer_pads[r] + kPadInboxFree + p.my_rank, p.epoch);
    }
  }
}

// dQ leaves the backward kernel as an fp32 accumulator (key-tile CTAs add their partial tiles with TMA
// reduce-add).  This kernel turns it into the model dtype AND zeroes the accumulator again, so the workspace is
// ready for the next backward: one pass of our own instead of a memset before and a cast after every call.
template <typename T>
__global__ void __launch_bounds__(256) dq_finalize_kernel(float4* __restrict__ acc, uint2* __restrict__ out,
                                                          long long n4) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = __ldcs(acc + i);
    out[i] = pack4<T>(v);
    acc[i] = zero;
  }
}

}  // namespace comm

const char* reduce_dkv_launch(int dtype, const ReduceParams& p, cudaStream_t stream) {
  if (p.n_tasks <= 0) return nullptr;
  set_peer_timeout_from_env();
  dim3 grid(kReduceBlocksPerTask, p.n_tasks, 1);
  if (dtype == kDtypeBF16) {
    comm::reduce_dkv_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(p);
  } else {
    comm::reduce_dkv_kernel<__half><<<grid, 256, 0, stream>>>(p);
  }
  cudaError_t err = cudaGetLastError();
  return err == cudaSuccess ? nullptr : cudaGetErrorString(err);
}

const char* dq_finalize_launch(int dtype, float* acc, void* out, long long numel, cudaStream_t stream) {
  if (numel <= 0) return nullptr;
  if (numel % 4) return "dq_finalize: element count must be a multiple of 4";
  const long long n4 = numel / 4;
  const long long want = (n4 + 255) / 256;
  // grid-stride loop: 8 blocks per SM of the device are enough to saturate HBM
  static const int max_blocks = [] {
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return 8 * (sms > 0 ? sms : 1);
  }();
  const int blocks = static_cast<int>(want < max_blocks ? want : max_blocks);
  if (dtype == kDtypeBF16) {
    comm::dq_finalize_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(reinterpret_cast<float4*>(acc),
                                                                        static_cast<uint2*>(out), n4);
  } else {
    comm::dq_finalize_kernel<__half><<<blocks, 256, 0, stream>>>(reinterpret_cast<float4*>(acc),
                                                                 static_cast<uint2*>(out), n4);
  }
  cudaError_t err = cudaGetLastError();
  return err == cudaSuccess ? nullptr : cudaGetErrorString(err);
}

}  // namespace rfa
