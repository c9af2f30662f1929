// HBM-bound normalisation kernels (128-bit loads/stores, fp32 statistics).
//
// GroupNorm(+SiLU) over NHWC activations, with an optional *virtual channel concat* of two sources
// (the up-block `torch.cat([hidden, skip], dim=1)` of unet_multiview_blocks.py:669 is never materialised
// un-normalised: the normalised/activated concat is written once, as the next conv's input).
// Replaces F.group_norm + F.silu of diffusers ResnetBlock2D (norm1/norm2), Transformer2DModel.norm
// (eps 1e-6, transformer_multiview.py:43) and conv_norm_out (unet_multiview_condition.py:590-592).
// LayerNorm replaces norm1/norm2/norm3 of BasicTransformerBlock (attention.py:50,108,127).
//
// Statistics: each CTA reduces a slab of pixels with per-channel *shifted* sums (pivot = first pixel of
// the slab) to avoid E[x^2]-E[x]^2 cancellation, converts to (mean, M2) and merges groups / slabs with
// Chan's parallel-variance update.
#include "kernels.h"

namespace d4d {

namespace {

constexpr int GN_MAX_THREADS = 512;

struct GnArgs {
  const bf16* x1;
  const bf16* x2;
  int C1, C2, C, n_oct, rows_per_iter;
  int hw, pps, splits, groups, cpg;
  float eps;
  const float* gamma;
  const float* beta;
  int silu;
  bf16* out;
  float* partials;  // [n_img][splits][groups][2] = (mean, M2)
  float* final_stats;   // [n_img][groups][2] = (mean, rstd), written by the last stats CTA of each image
  unsigned int* counters;  // [n_img] arrival counters (self-resetting)
  // fused-statistics mode (groupnorm_apply_run): per-(image, channel) {sum, sum of squares} of each source, accumulated by
  // the epilogue of the GEMM / conv that produced it (gemm_wgmma.cu); the apply kernel derives (mean, rstd) itself
  const long long* ch_stats1;  // fixed point (kGnSumScale, kGnSqScale)
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

// smem: ch_mean[C], ch_m2[C] then scratch [rows_per_iter][C][2]
__global__ void __launch_bounds__(GN_MAX_THREADS, 2) gn_stats_kernel(const GnArgs a) {
  extern __shared__ float sm[];
  const int split = blockIdx.x, img = blockIdx.y;
  const int oct = threadIdx.x % a.n_oct;
  const int prow = threadIdx.x / a.n_oct;
  const int p0 = split * a.pps;
  const int p1 = min(a.hw, p0 + a.pps);
  const int npix = p1 - p0;
  float* scratch = sm + 2 * a.C;  // [rows_per_iter][C][2]
  pdl_wait();
  pdl_launch_dependents();

  float s[8], ss[8], piv[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s[i] = 0.f; ss[i] = 0.f; }
  if (npix > 0) {
    uint4 u0 = gn_load(a, img, p0, oct);
    unpack8(u0, piv);
    // 4 independent 16-byte loads in flight per thread (memory-level parallelism), then accumulate
    const int stride = a.rows_per_iter;
    int p = p0 + prow;
    for (; p + 3 * stride < p1; p += 4 * stride) {
      uint4 u[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) u[k] = gn_load(a, img, p + k * stride, oct);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float f[8];
        unpack8(u[k], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = f[i] - piv[i];
          s[i] += d;
          ss[i] = fmaf(d, d, ss[i]);
        }
      }
    }
    for (; p < p1; p += stride) {
      uint4 u = gn_load(a, img, p, oct);
      float f[8];
      unpack8(u, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float d = f[i] - piv[i];
        s[i] += d;
        ss[i] = fmaf(d, d, ss[i]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    scratch[(prow * a.C + oct * 8 + i) * 2 + 0] = s[i];
    scratch[(prow * a.C + oct * 8 + i) * 2 + 1] = ss[i];
  }
  __syncthreads();
  // per-channel totals over the slab -> (mean, M2)
  for (int c = threadIdx.x; c < a.C; c += blockDim.x) {
    float ts = 0.f, tss = 0.f;
    for (int r = 0; r < a.rows_per_iter; ++r) {
      ts += scratch[(r * a.C + c) * 2 + 0];
      tss += scratch[(r * a.C + c) * 2 + 1];
    }
    // pivot of channel c (same value every thread of that octet used)
    float pv = 0.f;
    if (npix > 0) {
      const size_t tok = static_cast<size_t>(img) * a.hw + p0;
      pv = __bfloat162float(c < a.C1 ? a.x1[tok * a.C1 + c] : a.x2[tok * a.C2 + (c - a.C1)]);
    }
    const float n = static_cast<float>(npix);
    const float dm = npix > 0 ? ts / n : 0.f;
    sm[c] = pv + dm;                              // mean
    sm[a.C + c] = npix > 0 ? tss - ts * dm : 0.f; // M2
  }
  __syncthreads();
  // merge the cpg channels of each group (equal counts npix each)
  for (int g = threadIdx.x; g < a.groups; g += blockDim.x) {
    float mean = 0.f, m2 = 0.f, cnt = 0.f;
    const float nb = static_cast<float>(npix);
    if (npix > 0) {
      for (int i = 0; i < a.cpg; ++i) {
        const int c = g * a.cpg + i;
        const float mb = sm[c], m2b = sm[a.C + c];
        const float tot = cnt + nb;
        const float delta = mb - mean;
        mean += delta * (nb / tot);
        m2 += m2b + delta * delta * (cnt * nb / tot);
        cnt = tot;
      }
    }
    float* dst = a.partials + ((static_cast<size_t>(img) * a.splits + split) * a.groups + g) * 2;
    dst[0] = mean;
    dst[1] = m2;
  }
  // ---- the last CTA of this image merges the slabs once (instead of every apply-CTA re-merging them) ----
  __shared__ unsigned int s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(&a.counters[img], 1u);
    s_last = (prev == static_cast<unsigned int>(a.splits - 1)) ? 1u : 0u;
    if (s_last) a.counters[img] = 0u;  // reset for the next GroupNorm on this stream
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int g = threadIdx.x; g < a.groups; g += blockDim.x) {
    float mean = 0.f, m2 = 0.f, cnt = 0.f;
    for (int sp = 0; sp < a.splits; ++sp) {
      const int q0 = sp * a.pps;
      const int q1 = min(a.hw, q0 + a.pps);
      const float nb = static_cast<float>(max(0, q1 - q0)) * a.cpg;
      if (nb <= 0.f) continue;
      const float* src = a.partials + ((static_cast<size_t>(img) * a.splits + sp) * a.groups + g) * 2;
      const float mb = __ldcg(src), m2b = __ldcg(src + 1);
      const float tot = cnt + nb;
      const float delta = mb - mean;
      mean += delta * (nb / tot);
      m2 += m2b + delta * delta * (cnt * nb / tot);
      cnt = tot;
    }
    float* dst = a.final_stats + (static_cast<size_t>(img) * a.groups + g) * 2;
    dst[0] = mean;
    dst[1] = rsqrtf(m2 / cnt + a.eps);
  }
}

// smem: g_mean[groups], g_rstd[groups]
__global__ void __launch_bounds__(GN_MAX_THREADS, 2) gn_apply_kernel(const GnArgs a) {
  extern __shared__ float sm[];
  const int split = blockIdx.x, img = blockIdx.y;
  pdl_wait();
  pdl_launch_dependents();
  if (a.ch_stats1 == nullptr) {
    for (int g = threadIdx.x; g < 2 * a.groups; g += blockDim.x)
      sm[(g & 1) * a.groups + (g >> 1)] = a.final_stats[static_cast<size_t>(img) * a.groups * 2 + g];
  } else {
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

int groupnorm_splits(int hw) {
  int s = hw / 16;
  if (s < 1) s = 1;
  if (s > 32) s = 32;
  return s;
}

int groupnorm_run(const bf16* x1, int C1, const bf16* x2, int C2, int n_img, int hw, int groups, float eps,
                  const float* gamma, const float* beta, int silu, bf16* out, float* partials, cudaStream_t stream) {
  if (x2 == nullptr) C2 = 0;
  const int C = C1 + C2;
  D4D_REQUIRE(C1 % 8 == 0 && C2 % 8 == 0 && C % groups == 0, "GroupNorm channel counts");
  D4D_REQUIRE(C / 8 <= GN_MAX_THREADS, "GroupNorm supports at most 4096 channels");
  D4D_REQUIRE(n_img > 0 && hw > 0 && n_img <= 65535, "GroupNorm batch");
  GnArgs a;
  a.x1 = x1; a.x2 = x2; a.C1 = C1; a.C2 = C2; a.C = C;
  a.n_oct = C / 8;
  a.rows_per_iter = GN_MAX_THREADS / a.n_oct;
  if (a.rows_per_iter < 1) a.rows_per_iter = 1;
  if (a.rows_per_iter > 8) a.rows_per_iter = 8;
  a.hw = hw;
  a.splits = groupnorm_splits(hw);
  a.pps = (hw + a.splits - 1) / a.splits;
  a.groups = groups;
  a.cpg = C / groups;
  a.eps = eps;
  a.gamma = gamma; a.beta = beta; a.silu = silu; a.out = out; a.partials = partials;
  a.ch_stats1 = a.ch_stats2 = nullptr;
  // scratch layout: partials | final stats | counters (counters must be zero before first use; they self-reset)
  a.final_stats = partials + static_cast<size_t>(n_img) * 32 * groups * 2;
  a.counters = reinterpret_cast<unsigned int*>(a.final_stats + static_cast<size_t>(n_img) * groups * 2);
  const int threads = a.n_oct * a.rows_per_iter;
  dim3 grid(a.splits, n_img);
  const size_t smem_stats = sizeof(float) * (2 * C + 2 * static_cast<size_t>(a.rows_per_iter) * C);
  D4D_REQUIRE(smem_stats <= 48 * 1024, "GroupNorm stats smem");
  D4D_CUDA_OK(launch_pdl(gn_stats_kernel, grid, dim3(threads), smem_stats, stream, a));
  D4D_CUDA_OK(cudaGetLastError());
  D4D_CUDA_OK(launch_pdl(gn_apply_kernel, grid, dim3(threads), sizeof(float) * 2 * groups, stream, a));
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
  // one wave of CTAs (2 per SM): every CTA pays the group-statistics prologue once, so fewer and longer CTAs than the
  // stand-alone path (which sizes its slabs for the partials it has to merge)
  {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int sp = (2 * sms) / n_img;
    const int cap = groupnorm_splits(hw);
    a.splits = sp < 1 ? 1 : (sp > cap ? cap : sp);
  }

  a.pps = (hw + a.splits - 1) / a.splits;
  a.groups = groups;
  a.cpg = C / groups;
  a.eps = eps;
  a.gamma = gamma; a.beta = beta; a.silu = silu; a.out = out;
  a.ch_stats1 = stats1; a.ch_stats2 = stats2;
  const int threads = a.n_oct * a.rows_per_iter;
  D4D_REQUIRE(threads >= 32, "GroupNorm needs at least 32 threads");
  dim3 grid(a.splits, n_img);
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
