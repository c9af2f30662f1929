// Host-side TMA tensor-map encoders.  cuTensorMapEncodeTiled is resolved at run time through the
// runtime's driver-entry-point query so that libd4d.so carries no DT_NEEDED on libcuda.so.1 and can
// be dlopen'ed (symbol check) on a box without a driver.
#include "common.cuh"

#include <mutex>

namespace d4d {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
    else (void)cudaGetLastError();
  });
  return fn;
}

static CUtensorMapSwizzle swz(int bytes) {
  switch (bytes) {
    case 128: return CU_TENSOR_MAP_SWIZZLE_128B;
    case 64: return CU_TENSOR_MAP_SWIZZLE_64B;
    case 32: return CU_TENSOR_MAP_SWIZZLE_32B;
    default: return CU_TENSOR_MAP_SWIZZLE_NONE;
  }
}

int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_cols,
                 uint32_t box_rows, int swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return 2;
  }
  D4D_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base must be 16-byte aligned");
  D4D_REQUIRE((ld * 2) % 16 == 0, "TMA row pitch must be a multiple of 16 bytes");
  D4D_REQUIRE(box_cols <= 256 && box_rows <= 256 && box_cols >= 1 && box_rows >= 1, "TMA box dims must be in [1,256]");
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstr[1] = {ld * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz(swizzle_bytes), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(2d) failed, CUresult=" + std::to_string(static_cast<int>(r)) +
              " rows=" + std::to_string(rows) + " cols=" + std::to_string(cols) + " ld=" + std::to_string(ld) +
              " box=" + std::to_string(box_cols) + "x" + std::to_string(box_rows));
    return 2;
  }
  return 0;
}

int make_tmap_nhwc(CUtensorMap* out, const void* base, uint64_t n, uint64_t h, uint64_t w, uint64_t c, uint32_t box_c,
                   uint32_t box_w, uint32_t box_h, uint32_t box_n, int swizzle_bytes, int stride) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return 2;
  }
  D4D_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base must be 16-byte aligned");
  D4D_REQUIRE((c * 2) % 16 == 0, "NHWC channel count must be a multiple of 8");
  cuuint64_t gdim[4] = {c, w, h, n};
  cuuint64_t gstr[3] = {c * 2, w * c * 2, h * w * c * 2};
  D4D_REQUIRE(stride >= 1 && stride <= 8 && box_w * stride <= 256 && box_h * stride <= 256, "TMA traversal stride");
  // with elementStrides the box is given in tensor pixels and every stride-th one is loaded: ceil(box / stride) elements
  const cuuint32_t s = static_cast<cuuint32_t>(stride);
  cuuint32_t box[4] = {box_c, box_w * s, box_h * s, box_n};
  cuuint32_t estr[4] = {1, s, s, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz(swizzle_bytes), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(4d) failed, CUresult=" + std::to_string(static_cast<int>(r)));
    return 2;
  }
  return 0;
}

}  // namespace d4d
