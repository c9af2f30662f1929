// Shared device/host helpers for the sm_90a kernels: PTX wrappers for mbarrier, TMA (cp.async.bulk.tensor), register
// reallocation, and host-side error plumbing.  The warpgroup MMA wrappers are in wgmma.cuh.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>

namespace d4d {

typedef __nv_bfloat16 bf16;

// ------------------------------------------------------------------------------------------
// host-side error handling: every entry point returns a status and records a message
// ------------------------------------------------------------------------------------------
void set_error(const std::string& msg);          // thread-local last error (d4d_api.cu)
#define D4D_CUDA_OK(expr)                                                                        \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      d4d::set_error(std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " @" + __FILE__ + \
                     ":" + std::to_string(__LINE__));                                            \
      return 2;                                                                                  \
    }                                                                                            \
  } while (0)
#define D4D_REQUIRE(cond, msg)                                                                   \
  do {                                                                                           \
    if (!(cond)) {                                                                               \
      d4d::set_error(std::string("invalid argument: ") + msg + " (" #cond ") @" + __FILE__ + ":" + \
                     std::to_string(__LINE__));                                                  \
      return 1;                                                                                  \
    }                                                                                            \
  } while (0)

// TMA tensor-map encoders (host).  Implemented in tmap.cu through cudaGetDriverEntryPoint so the
// library has no link-time dependency on libcuda (it must dlopen on a CPU-only box).
// 2-D row-major bf16 matrix [rows, cols] with leading dimension ld (elements); box = {box_cols, box_rows}.
int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                 uint32_t box_cols, uint32_t box_rows, int swizzle_bytes);
// NHWC bf16 tensor [n, h, w, c] as the DESTINATION of 32-row x 32-channel epilogue boxes {32, box_w, box_h, box_n}
int make_tmap_nhwc_store(CUtensorMap* out, void* base, uint64_t n, uint64_t h, uint64_t w, uint64_t c, uint32_t box_w,
                         uint32_t box_h, uint32_t box_n);
// 4-D NHWC bf16 tensor [n, h, w, c]; box = {box_c, box_w, box_h, box_n} ELEMENTS LOADED; `stride` > 1 loads every
// stride-th pixel along w and h (elementStrides: the box then spans stride * box_w x stride * box_h pixels).
int make_tmap_nhwc(CUtensorMap* out, const void* base, uint64_t n, uint64_t h, uint64_t w, uint64_t c,
                   uint32_t box_c, uint32_t box_w, uint32_t box_h, uint32_t box_n, int swizzle_bytes, int stride = 1);

#ifdef __CUDACC__
// ------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
      "elect.sync rx|px, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, px;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier ----------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must trap (-> cudaErrorLaunchFailure) instead of hanging the GPU box.
#ifndef D4D_SPIN_LIMIT
#define D4D_SPIN_LIMIT (1u << 26)
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > D4D_SPIN_LIMIT) {
      printf("d4d: mbarrier timeout block=(%d,%d) thread=%d bar=%u parity=%u\n", blockIdx.x, blockIdx.y,
             threadIdx.x, smem_u32(bar), parity);
      __trap();
    }
  }
}

// ---- proxies / fences ----------------------------------------------------------------------
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// programmatic dependent launch (see launch_pdl in kernels.h): wait for the predecessor grid's memory, then let the successor
// grid become resident
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// warpgroup-wide register reallocation: producer warpgroups give registers back, MMA warpgroups take them
template <int R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// ---- TMA -----------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* t) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(t)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* t, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(t)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* t, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(t)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3)
      : "memory");
}

// TMA stores (shared -> global), bulk-group completion.  The writing threads must make their st.shared visible to the
// async proxy first (fence_proxy_async_smem) and synchronise with the issuing thread.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* t, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(t)), "r"(smem_u32(src)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* t, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(t)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_group_read() {  // <= N groups still READING shared memory
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N> __device__ __forceinline__ void bulk_wait_group() {  // <= N groups not yet complete
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ---- misc math ---------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
// exact-erf GELU with ONE MUFU:  gelu(g) = relu(g) - 0.5 |g| erfc(|g| / sqrt 2), and -log2 erfc(u / sqrt 2) is so close to a
// polynomial that  erfc(u / sqrt 2) = 2^-(d1 u + d2 u^2 + ... + d5 u^5)  holds to 7e-7 absolute in the GELU (least-squares
// fit; the polynomial is increasing, so large |g| underflow to 0 cleanly).
__device__ __forceinline__ float gelu_erf_f(float g) {
  const float u = fabsf(g);
  float q = fmaf(-4.8811754095e-04f, u, 7.1988063864e-03f);  // negated: p = -(d1 u + ... + d5 u^5)
  q = fmaf(q, u, -5.2146803588e-02f);
  q = fmaf(q, u, -4.5959571004e-01f);
  q = fmaf(q, u, -1.1510006189e+00f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(q * u));
  return fmaf(-0.5f * u, e, fmaxf(g, 0.f));
}
#endif  // __CUDACC__

}  // namespace d4d
