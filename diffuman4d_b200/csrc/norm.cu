// HBM-bound normalisation kernels (128-bit loads/stores, fp32 arithmetic).
//
// GroupNorm(+SiLU) over NHWC activations, with an optional *virtual channel concat* of two sources
// (the up-block `torch.cat([hidden, skip], dim=1)` of unet_multiview_blocks.py:669 is never materialised
// un-normalised: the normalised/activated concat is written once, as the next conv's input).
// Replaces F.group_norm + F.silu of diffusers ResnetBlock2D (norm1/norm2), Transformer2DModel.norm
// (eps 1e-6, transformer_multiview.py:43) and conv_norm_out (unet_multiview_condition.py:590-592).
// LayerNorm replaces norm1/norm2/norm3 of BasicTransformerBlock (attention.py:50,108,127).
//
// GroupNorm statistics have one format: per-(image, channel) {sum, sum of squares} in 64-bit fixed point (kGnSumScale,
// kGnSqScale, kernels.h).  The GEMM / conv epilogue that produces a normalised tensor accumulates them (gemm_wgmma.cu);
// gn_stats_kernel computes the same sums from the stored tensor where that epilogue cannot.  Both sum at most 16 pixels
// in fp32 before rounding to fixed point, and integer adds commute, so the totals do not depend on the order in which
// CTAs finish.  gn_apply_kernel reduces them to group (mean, rstd) in its prologue and normalises.
#include <algorithm>

#include "kernels.h"

namespace d4d {

namespace {

constexpr int GN_MAX_THREADS = 512;
constexpr int GN_STATS_THREADS = 256;
constexpr int GN_STATS_PIXELS = 16;  // pixels per fp32 partial: the 16 rows of one epilogue warp (gemm_wgmma.cu)

struct GnArgs {
  const bf16* x1;
  const bf16* x2;
  int C1, C2, C, n_oct, rows_per_iter;
  int hw, pps, groups, cpg;
  float eps;
  const float* gamma;
  const float* beta;
  int silu;
  bf16* out;
  // per-(image, channel) {sum, sum of squares} of each source, fixed point (kGnSumScale, kGnSqScale)
  const long long* ch_stats1;
  const long long* ch_stats2;
};

__device__ __forceinline__ uint4 gn_load(const GnArgs& a, int img, int pixel, int oct) {
  const int c = oct * 8;
  const size_t tok = static_cast<size_t>(img) * a.hw + pixel;
  if (c < a.C1) return __ldg(reinterpret_cast<const uint4*>(a.x1 + tok * a.C1 + c));
  return __ldg(reinterpret_cast<const uint4*>(a.x2 + tok * a.C2 + (c - a.C1)));
}

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  float2 p;
  p = unpack_bf16x2(u.x); f[0] = p.x; f[1] = p.y;
  p = unpack_bf16x2(u.y); f[2] = p.x; f[3] = p.y;
  p = unpack_bf16x2(u.z); f[4] = p.x; f[5] = p.y;
  p = unpack_bf16x2(u.w); f[6] = p.x; f[7] = p.y;
}

// one thread: one channel octet of GN_STATS_PIXELS consecutive pixels of one image; adds its 8 {sum, sum of squares}
// pairs to stats [n_img][C][2] in fixed point, like the epilogue adds one warp's 16 rows
__global__ void __launch_bounds__(GN_STATS_THREADS) gn_stats_kernel(const bf16* __restrict__ x, int n_oct, int hw,
                                                                      long long* __restrict__ stats) {
  const int img = blockIdx.y;
  const int t = blockIdx.x * GN_STATS_THREADS + threadIdx.x;
  const int oct = t % n_oct;
  const int p0 = (t / n_oct) * GN_STATS_PIXELS;
  pdl_wait();
  pdl_launch_dependents();
  if (p0 >= hw) return;
  const int npix = min(GN_STATS_PIXELS, hw - p0);
  const size_t C = static_cast<size_t>(n_oct) * 8;
  const bf16* src = x + (static_cast<size_t>(img) * hw + p0) * C + oct * 8;
  uint4 u[GN_STATS_PIXELS];  // all loads in flight before the first use
#pragma unroll
  for (int k = 0; k < GN_STATS_PIXELS; ++k)
    u[k] = k < npix ? __ldg(reinterpret_cast<const uint4*>(src + k * C)) : make_uint4(0u, 0u, 0u, 0u);
  float s[8], q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s[i] = 0.f; q[i] = 0.f; }
#pragma unroll
  for (int k = 0; k < GN_STATS_PIXELS; ++k) {
    float f[8];
    unpack8(u[k], f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s[i] += f[i];
      q[i] = fmaf(f[i], f[i], q[i]);
    }
  }
  unsigned long long* st = reinterpret_cast<unsigned long long*>(stats) + (img * C + oct * 8) * 2;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    atomicAdd(st + 2 * i + 0, static_cast<unsigned long long>(__float2ll_rn(s[i] * kGnSumScale)));
    atomicAdd(st + 2 * i + 1, static_cast<unsigned long long>(__float2ll_rn(q[i] * kGnSqScale)));
  }
}

// smem: g_mean[groups], g_rstd[groups]
__global__ void __launch_bounds__(GN_MAX_THREADS, 2) gn_apply_kernel(const GnArgs a) {
  extern __shared__ float sm[];
  const int split = blockIdx.x, img = blockIdx.y;
  pdl_wait();
  pdl_launch_dependents();
  // one warp per group, up to 4 groups per warp side by side (their load / shuffle chains are independent, so the
  // latencies overlap); the channel totals are summed as integers (exact), the butterfly runs on doubles in a fixed order
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  if (warp < nwarps) {  // (a trailing partial warp sits out)
    for (int g0 = warp; g0 < a.groups; g0 += 4 * nwarps) {
      double ds[4], dq[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int g = g0 + u * nwarps;
        long long s = 0, q = 0;
        if (g < a.groups) {
          for (int i = lane; i < a.cpg; i += 32) {  // (the virtual concat may straddle the two sources)
            const int c = g * a.cpg + i;
            const longlong2 v = c < a.C1 ? __ldcg(reinterpret_cast<const longlong2*>(a.ch_stats1) + static_cast<size_t>(img) * a.C1 + c)
                                         : __ldcg(reinterpret_cast<const longlong2*>(a.ch_stats2) + static_cast<size_t>(img) * a.C2 + (c - a.C1));
            s += v.x;
            q += v.y;
          }
        }
        ds[u] = static_cast<double>(s);
        dq[u] = static_cast<double>(q);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          ds[u] += __shfl_xor_sync(0xffffffffu, ds[u], o);
          dq[u] += __shfl_xor_sync(0xffffffffu, dq[u], o);
        }
      }
      if (lane < 4) {
        const int g = g0 + lane * nwarps;
        if (g < a.groups) {
          const double s = lane == 0 ? ds[0] : (lane == 1 ? ds[1] : (lane == 2 ? ds[2] : ds[3]));
          const double q = lane == 0 ? dq[0] : (lane == 1 ? dq[1] : (lane == 2 ? dq[2] : dq[3]));
          // double precision keeps E[x^2] - mean^2 exact up to the fixed-point resolution
          const double inv_n = 1.0 / (static_cast<double>(a.cpg) * static_cast<double>(a.hw));
          const double mean = s * (1.0 / static_cast<double>(kGnSumScale)) * inv_n;
          const double var = fmax(q * (1.0 / static_cast<double>(kGnSqScale)) * inv_n - mean * mean, 0.0);
          sm[g] = static_cast<float>(mean);
          sm[a.groups + g] = rsqrtf(static_cast<float>(var) + a.eps);
        }
      }
    }
  }
  __syncthreads();
  const int oct = threadIdx.x % a.n_oct;
  const int prow = threadIdx.x / a.n_oct;
  float sc[8], sh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = oct * 8 + i;
    const int g = c / a.cpg;
    const float w = a.gamma[c] * sm[a.groups + g];
    sc[i] = w;
    sh[i] = a.beta[c] - sm[g] * w;
  }
  const int p0 = split * a.pps;
  const int p1 = min(a.hw, p0 + a.pps);
  auto apply_one = [&](const uint4& u, int p) {
    float f[8];
    unpack8(u, f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float y = fmaf(f[i], sc[i], sh[i]);
      f[i] = a.silu ? silu_f(y) : y;
    }
    uint4 o;
    o.x = pack_bf16x2(f[0], f[1]);
    o.y = pack_bf16x2(f[2], f[3]);
    o.z = pack_bf16x2(f[4], f[5]);
    o.w = pack_bf16x2(f[6], f[7]);
    const size_t tok = static_cast<size_t>(img) * a.hw + p;
    *reinterpret_cast<uint4*>(a.out + tok * a.C + oct * 8) = o;
  };
  const int stride = a.rows_per_iter;
  int p = p0 + prow;
  for (; p + 3 * stride < p1; p += 4 * stride) {
    uint4 u[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) u[k] = gn_load(a, img, p + k * stride, oct);
#pragma unroll
    for (int k = 0; k < 4; ++k) apply_one(u[k], p + k * stride);
  }
  for (; p < p1; p += stride) apply_one(gn_load(a, img, p, oct), p);
}

// one warp per row; the row lives in registers (<= 8 x 16-byte chunks per lane => C <= 2048)
template <int CHUNKS>
__global__ void layernorm_kernel(const bf16* __restrict__ x, int rows, int C, float eps, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, bf16* __restrict__ out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  pdl_wait();
  pdl_launch_dependents();
  if (warp >= rows) return;
  const int n_oct = C / 8;
  const bf16* xr = x + static_cast<size_t>(warp) * C;
  float f[CHUNKS][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < CHUNKS; ++i) {
    const int o = lane + 32 * i;
    if (o < n_oct) {
      uint4 u = __ldg(reinterpret_cast<const uint4*>(xr + o * 8));
      unpack8(u, f[i]);
#pragma unroll
      for (int k = 0; k < 8; ++k) sum += f[i][k];
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) f[i][k] = 0.f;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / C;
  float var = 0.f;
#pragma unroll
  for (int i = 0; i < CHUNKS; ++i) {
    const int o = lane + 32 * i;
    if (o < n_oct) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float d = f[i][k] - mean;
        var = fmaf(d, d, var);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
  const float rstd = rsqrtf(var / C + eps);
  bf16* orow = out + static_cast<size_t>(warp) * C;
#pragma unroll
  for (int i = 0; i < CHUNKS; ++i) {
    const int o = lane + 32 * i;
    if (o < n_oct) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + o * 8));
      const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + o * 8 + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + o * 8));
      const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + o * 8 + 4));
      float y[8];
      y[0] = (f[i][0] - mean) * rstd * g0.x + b0.x;
      y[1] = (f[i][1] - mean) * rstd * g0.y + b0.y;
      y[2] = (f[i][2] - mean) * rstd * g0.z + b0.z;
      y[3] = (f[i][3] - mean) * rstd * g0.w + b0.w;
      y[4] = (f[i][4] - mean) * rstd * g1.x + b1.x;
      y[5] = (f[i][5] - mean) * rstd * g1.y + b1.y;
      y[6] = (f[i][6] - mean) * rstd * g1.z + b1.z;
      y[7] = (f[i][7] - mean) * rstd * g1.w + b1.w;
      uint4 u;
      u.x = pack_bf16x2(y[0], y[1]);
      u.y = pack_bf16x2(y[2], y[3]);
      u.z = pack_bf16x2(y[4], y[5]);
      u.w = pack_bf16x2(y[6], y[7]);
      *reinterpret_cast<uint4*>(orow + o * 8) = u;
    }
  }
}

}  // namespace

int groupnorm_stats_run(const bf16* x, int C, int n_img, int hw, long long* stats, cudaStream_t stream) {
  D4D_REQUIRE(C > 0 && C % 8 == 0, "GroupNorm statistics: channels must be a positive multiple of 8");
  D4D_REQUIRE(n_img > 0 && hw > 0 && n_img <= 65535, "GroupNorm batch");
  D4D_REQUIRE(x != nullptr && stats != nullptr, "GroupNorm statistics: null tensor");
  const long long threads = static_cast<long long>(C / 8) * ((hw + GN_STATS_PIXELS - 1) / GN_STATS_PIXELS);
  D4D_REQUIRE(threads < (1LL << 31) - GN_STATS_THREADS, "GroupNorm statistics: image too large");
  const dim3 grid(static_cast<unsigned>((threads + GN_STATS_THREADS - 1) / GN_STATS_THREADS), n_img);
  D4D_CUDA_OK(launch_pdl(gn_stats_kernel, grid, dim3(GN_STATS_THREADS), 0, stream, x, C / 8, hw, stats));
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int groupnorm_apply_run(const bf16* x1, int C1, const long long* stats1, const bf16* x2, int C2, const long long* stats2, int n_img,
                        int hw, int groups, float eps, const float* gamma, const float* beta, int silu, bf16* out,
                        cudaStream_t stream) {
  if (x2 == nullptr) C2 = 0;
  const int C = C1 + C2;
  D4D_REQUIRE(C1 % 8 == 0 && C2 % 8 == 0 && C % groups == 0, "GroupNorm channel counts");
  D4D_REQUIRE(C / 8 <= GN_MAX_THREADS, "GroupNorm supports at most 4096 channels");
  D4D_REQUIRE(n_img > 0 && hw > 0 && n_img <= 65535, "GroupNorm batch");
  D4D_REQUIRE(stats1 != nullptr && (C2 == 0 || stats2 != nullptr), "GroupNorm statistics arrays");
  GnArgs a;
  memset(&a, 0, sizeof(a));
  a.x1 = x1; a.x2 = x2; a.C1 = C1; a.C2 = C2; a.C = C;
  a.n_oct = C / 8;
  a.rows_per_iter = GN_MAX_THREADS / a.n_oct;
  if (a.rows_per_iter < 1) a.rows_per_iter = 1;
  if (a.rows_per_iter > 8) a.rows_per_iter = 8;
  a.hw = hw;
  // one wave of CTAs (2 per SM), at most 32 per image and at least 16 pixels each: every CTA pays the group-statistics
  // prologue once, so few long CTAs
  int splits;
  {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int sp = (2 * sms) / n_img;
    const int cap = std::min(32, std::max(1, hw / 16));
    splits = sp < 1 ? 1 : (sp > cap ? cap : sp);
  }

  a.pps = (hw + splits - 1) / splits;
  a.groups = groups;
  a.cpg = C / groups;
  a.eps = eps;
  a.gamma = gamma; a.beta = beta; a.silu = silu; a.out = out;
  a.ch_stats1 = stats1; a.ch_stats2 = stats2;
  const int threads = a.n_oct * a.rows_per_iter;
  D4D_REQUIRE(threads >= 32, "GroupNorm needs at least 32 threads");
  dim3 grid(splits, n_img);
  D4D_CUDA_OK(launch_pdl(gn_apply_kernel, grid, dim3(threads), sizeof(float) * 2 * groups, stream, a));
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int layernorm_run(const bf16* x, int rows, int C, float eps, const float* gamma, const float* beta, bf16* out,
                  cudaStream_t stream) {
  D4D_REQUIRE(C % 8 == 0 && C <= 2048 && C > 0, "LayerNorm width must be a multiple of 8, <= 2048");
  if (rows <= 0) return 0;
  const int threads = 256;
  const int wpb = threads / 32;
  const int blocks = (rows + wpb - 1) / wpb;
  const int chunks = (C / 8 + 31) / 32;
  if (chunks <= 2) D4D_CUDA_OK(launch_pdl(layernorm_kernel<2>, dim3(blocks), dim3(threads), 0, stream, x, rows, C, eps, gamma, beta, out));
  else if (chunks <= 4) D4D_CUDA_OK(launch_pdl(layernorm_kernel<4>, dim3(blocks), dim3(threads), 0, stream, x, rows, C, eps, gamma, beta, out));
  else if (chunks <= 5) D4D_CUDA_OK(launch_pdl(layernorm_kernel<5>, dim3(blocks), dim3(threads), 0, stream, x, rows, C, eps, gamma, beta, out));
  else D4D_CUDA_OK(launch_pdl(layernorm_kernel<8>, dim3(blocks), dim3(threads), 0, stream, x, rows, C, eps, gamma, beta, out));
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace d4d
