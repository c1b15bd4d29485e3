// TMA tensor-map construction without linking libcuda: the driver entry point is resolved at run time.
#include <cudaTypedefs.h>

#include <mutex>

#include "attn_common.h"

namespace rfa {

static PFN_cuTensorMapEncodeTiled_v12000 resolve_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    }
  });
  return fn;
}

const char* make_tensor_map(CUtensorMap* out, const TensorView& t, int elem_bytes, int box_rows, int dim_inner,
                            int swizzle_bytes) {
  auto encode = resolve_encode();
  if (!encode) return "cuTensorMapEncodeTiled is not available from this driver";
  if (swizzle_bytes != 128 && swizzle_bytes != 64) return "tensor maps use a 64- or 128-byte swizzle";
  if (reinterpret_cast<uintptr_t>(t.ptr) % 16) return "tensor base must be 16-byte aligned for TMA";
  if ((t.row_stride * elem_bytes) % 16 || (t.head_stride * elem_bytes) % 16)
    return "tensor strides must be multiples of 16 bytes for TMA";
  const int box_inner = swizzle_bytes / elem_bytes;  // one swizzle span
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(dim_inner), static_cast<cuuint64_t>(t.heads),
                        static_cast<cuuint64_t>(t.rows)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(t.head_stride) * elem_bytes,
                           static_cast<cuuint64_t>(t.row_stride) * elem_bytes};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(box_inner), 1u, static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[3] = {1u, 1u, 1u};
  CUtensorMapDataType dt = elem_bytes == 4   ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                           : elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8  // fp8: 128 one-byte elements per span
                                             : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUresult r = encode(out, dt, 3, t.ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return "cuTensorMapEncodeTiled failed";
  return nullptr;
}

const char* make_plain_tensor_map(CUtensorMap* out, const TensorView& t, int elem_bytes, int box_rows, int dim_inner) {
  auto encode = resolve_encode();
  if (!encode) return "cuTensorMapEncodeTiled is not available from this driver";
  if (reinterpret_cast<uintptr_t>(t.ptr) % 16) return "tensor base must be 16-byte aligned for TMA";
  if ((t.row_stride * elem_bytes) % 16 || (t.head_stride * elem_bytes) % 16)
    return "tensor strides must be multiples of 16 bytes for TMA";
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(dim_inner), static_cast<cuuint64_t>(t.heads),
                        static_cast<cuuint64_t>(t.rows)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(t.head_stride) * elem_bytes,
                           static_cast<cuuint64_t>(t.row_stride) * elem_bytes};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(dim_inner), 1u, static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[3] = {1u, 1u, 1u};
  CUtensorMapDataType dt = elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUresult r = encode(out, dt, 3, t.ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return "cuTensorMapEncodeTiled (plain) failed";
  return nullptr;
}

}  // namespace rfa
