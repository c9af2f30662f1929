// HBM-/latency-bound helper kernels of the denoise step: embeddings, layout changes feeding the
// tensor-core kernels, the pose-encoder's small-channel convolutions, and the fused pipeline pieces
// (input assembly, CFG combine + per-frame scheduler step).  All global traffic is 128-bit where the
// layout allows it.
#include "ddpm_noise.cuh"
#include "kernels.h"

namespace d4d {

namespace {

__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// ---------------------------------------------------------------------------------------------
// sinusoidal position embedding (upstream get_timestep_embedding; unet_multiview_condition.py:464,255)
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void sinusoid_kernel(const T* __restrict__ pos, int n, int dim, int flip, float freq_shift,
                                bf16* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int half = dim / 2;
  if (idx >= n * half) return;
  const int r = idx / half, i = idx % half;
  const float exponent = -logf(10000.0f) * static_cast<float>(i) / (static_cast<float>(half) - freq_shift);
  const float arg = static_cast<float>(pos[r]) * expf(exponent);
  const float s = sinf(arg), c = cosf(arg);
  bf16* o = out + static_cast<size_t>(r) * dim;
  if (flip) { o[i] = __float2bfloat16_rn(c); o[half + i] = __float2bfloat16_rn(s); }
  else { o[i] = __float2bfloat16_rn(s); o[half + i] = __float2bfloat16_rn(c); }
}

__global__ void silu_kernel(const bf16* __restrict__ x, long long n, bf16* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __float2bfloat16_rn(silu_f(__bfloat162float(x[i])));
}

// ---------------------------------------------------------------------------------------------
// im2col of an NCHW input for the 3x3 pad-1 conv_in:  out[pixel, tap*cin_pad + c], zero padded to KP
// ---------------------------------------------------------------------------------------------
__global__ void im2col_nchw_kernel(const bf16* __restrict__ x, int n, int Cin, int H, int W, int cin_pad, int KP,
                                   bf16* __restrict__ out) {
  // one thread per (pixel, tap): writes cin_pad contiguous values
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int taps_total = KP / cin_pad;  // >= 9; taps >= 9 are zero padding
  const long long total = static_cast<long long>(n) * H * W * taps_total;
  if (idx >= total) return;
  const int tap = static_cast<int>(idx % taps_total);
  const long long pix = idx / taps_total;
  const int xw = static_cast<int>(pix % W);
  const int yh = static_cast<int>((pix / W) % H);
  const int img = static_cast<int>(pix / (static_cast<long long>(W) * H));
  bf16* o = out + pix * KP + tap * cin_pad;
  const int ky = tap / 3, kx = tap % 3;
  const int yy = yh + ky - 1, xx = xw + kx - 1;
  const bool in = tap < 9 && yy >= 0 && yy < H && xx >= 0 && xx < W;
  const bf16 zero = __float2bfloat16_rn(0.f);
  for (int c = 0; c < cin_pad; ++c) {
    bf16 v = zero;
    if (in && c < Cin) v = x[((static_cast<size_t>(img) * Cin + c) * H + yy) * W + xx];
    o[c] = v;
  }
}

// generic NHWC im2col (pad 1): out[opix, (ky*k+kx)*C + c]; used by the stride-2 downsample convs
// (Downsample2D, unet_multiview_blocks.py:460) and the pose encoder's 4x4 stride-2 conv
__global__ void im2col_nhwc_kernel(const bf16* __restrict__ x, int n, int H, int W, int C, int ksize, int stride,
                                   bf16* __restrict__ out) {
  const int Ho = (H + 2 - ksize) / stride + 1, Wo = (W + 2 - ksize) / stride + 1, oct = C / 8;
  const int kk = ksize * ksize;
  const long long total = static_cast<long long>(n) * Ho * Wo * kk * oct;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int o8 = static_cast<int>(idx % oct);
  long long r = idx / oct;
  const int tap = static_cast<int>(r % kk);
  r /= kk;
  const int xo = static_cast<int>(r % Wo);
  const int yo = static_cast<int>((r / Wo) % Ho);
  const int img = static_cast<int>(r / (static_cast<long long>(Wo) * Ho));
  const int yy = yo * stride + tap / ksize - 1, xx = xo * stride + tap % ksize - 1;
  uint4 v = make_uint4(0, 0, 0, 0);
  if (yy >= 0 && yy < H && xx >= 0 && xx < W)
    v = __ldg(reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(img) * H + yy) * W + xx) * C + o8 * 8));
  *reinterpret_cast<uint4*>(out + (r * kk + tap) * C + o8 * 8) = v;
}

// [n*H*W, ld] (first C columns) -> NCHW [n, C, H, W] in destination out.p[blockIdx.y]
// (__grid_constant__: the destination is indexed in parameter space, not from a local copy of the array)
__global__ void nhwc_to_nchw_kernel(const bf16* __restrict__ x, int ld, int n, int C, int hw, const __grid_constant__ NchwDst out) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(n) * C * hw;
  if (idx >= total) return;
  const int p = static_cast<int>(idx % hw);
  const int c = static_cast<int>((idx / hw) % C);
  const int img = static_cast<int>(idx / (static_cast<long long>(hw) * C));
  out.p[blockIdx.y][idx] = x[(static_cast<size_t>(img) * hw + p) * ld + c];
}

// ---------------------------------------------------------------------------------------------
// pose encoder, first layer (pose_encoder.py:14-31, conv_layers.0): 3 -> 3 channels, 3x3, stride 1, pad 1, SiLU, on the
// full-resolution NCHW skeleton images.  One thread per kPix0 horizontally adjacent output pixels (every weight read from
// shared memory - a warp-wide broadcast - feeds kPix0 FMAs); the output is NHWC with the 3 channels padded to 4 (8-byte
// pixels, channel 3 = 0), the layout the tensor-core layers below read.
// ---------------------------------------------------------------------------------------------
constexpr int kPix0 = 4;
__global__ void pose_conv0_kernel(const bf16* __restrict__ x, int n, int H, int W, const bf16* __restrict__ w /*[9][3][3]*/,
                                  const float* __restrict__ bias, bf16* __restrict__ out /*[n,H,W,4]*/) {
  __shared__ float sw[81];
  if (threadIdx.x < 81) sw[threadIdx.x] = __bfloat162float(w[threadIdx.x]);
  __syncthreads();
  const int Wg = (W + kPix0 - 1) / kPix0;
  const long long total = static_cast<long long>(n) * H * Wg;
  const long long grp = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (grp >= total) return;
  const int xo0 = static_cast<int>(grp % Wg) * kPix0;
  const int yo = static_cast<int>((grp / Wg) % H);
  const int img = static_cast<int>(grp / (static_cast<long long>(Wg) * H));
  float acc[kPix0][3];
#pragma unroll
  for (int p = 0; p < kPix0; ++p)
#pragma unroll
    for (int i = 0; i < 3; ++i) acc[p][i] = bias[i];
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int yy = yo + ky - 1;
    if (yy < 0 || yy >= H) continue;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const bf16* row = x + ((static_cast<size_t>(img) * 3 + c) * H + yy) * W;
      float v[kPix0 + 2];  // input columns xo0-1 .. xo0+kPix0
#pragma unroll
      for (int j = 0; j < kPix0 + 2; ++j) {
        const int xx = xo0 + j - 1;
        v[j] = (xx >= 0 && xx < W) ? __bfloat162float(row[xx]) : 0.f;
      }
#pragma unroll
      for (int kx = 0; kx < 3; ++kx)
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const float wv = sw[((ky * 3 + kx) * 3 + c) * 3 + i];
#pragma unroll
          for (int p = 0; p < kPix0; ++p) acc[p][i] = fmaf(v[p + kx], wv, acc[p][i]);
        }
    }
  }
#pragma unroll
  for (int p = 0; p < kPix0; ++p) {
    if (xo0 + p >= W) break;
    uint2 o;
    o.x = pack_bf16x2(silu_f(acc[p][0]), silu_f(acc[p][1]));
    o.y = pack_bf16x2(silu_f(acc[p][2]), 0.f);
    *reinterpret_cast<uint2*>(out + ((static_cast<size_t>(img) * H + yo) * W + xo0 + p) * 4) = o;
  }
}

// ---------------------------------------------------------------------------------------------
// pose encoder, layers 1-4 (conv_layers.2/4/6/8: 3->16 k4 s2, 16->16 k3, 16->32 k4 s2, 32->32 k3; pad 1, SiLU): implicit
// GEMM on the warp-level tensor-core path (mma.sync m16n8k16, bf16 x bf16 -> fp32).  These layers are 1-3 GMAC each on
// 16/32 output channels - far too narrow for a wgmma tile (the UNet's convs use csrc/gemm_wgmma.cu) but, one thread per
// pixel on the FMA pipe, they cost more than a whole 3x3 conv of the UNet.  Here a warp owns 32 output pixels (2 M tiles)
// x all COUT channels; K = taps x CIN runs in chunks of 16.  The A fragment of m16n8k16 is, per lane, two adjacent
// channels of one pixel at one tap = one 4-byte load straight from the NHWC activation (L1 keeps the 9-16x tap reuse);
// the B fragments come from the [COUT][K+8] weights staged once per CTA in shared memory (the +8 skews the rows over the banks).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mma_bf16_m16n8k16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int COUT, int CIN, int KS, int STRIDE>
__global__ void __launch_bounds__(256, 2) pose_conv_mma_kernel(const bf16* __restrict__ x, int n, int H, int W,
                                                               const bf16* __restrict__ w /*[COUT][KS*KS*CIN + 8]*/,
                                                               const float* __restrict__ bias, bf16* __restrict__ out) {
  constexpr int K = KS * KS * CIN, KP = K + 8, NT = COUT / 8;
  static_assert(K % 16 == 0 && CIN % 4 == 0 && COUT % 8 == 0 && (COUT * KP * 2) % 16 == 0, "pose conv tile shape");
  extern __shared__ __align__(16) unsigned char pose_smem[];
  {
    const uint4* src = reinterpret_cast<const uint4*>(w);
    uint4* dst = reinterpret_cast<uint4*>(pose_smem);
    for (int i = threadIdx.x; i < COUT * KP * 2 / 16; i += blockDim.x) dst[i] = __ldg(src + i);
  }
  __syncthreads();
  const uint32_t* sw = reinterpret_cast<const uint32_t*>(pose_smem);  // bf16 pairs, row stride KP / 2 words
  const int Ho = (H + 2 - KS) / STRIDE + 1, Wo = (W + 2 - KS) / STRIDE + 1;
  const int total = n * Ho * Wo;
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int warps = gridDim.x * (blockDim.x >> 5);
  float bs[NT][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    bs[nt][0] = bias[nt * 8 + 2 * t];
    bs[nt][1] = bias[nt * 8 + 2 * t + 1];
  }
  for (int tile = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); tile * 32 < total; tile += warps) {
    // this lane's four pixel rows: q = 2 * m_tile + half, fragment row g + 8 * half
    int y0[4], x0[4], ib[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int p = tile * 32 + (q >> 1) * 16 + (q & 1) * 8 + g;
      const int pc = p < total ? p : 0;
      const int xo = pc % Wo, yo = (pc / Wo) % Ho, img = pc / (Wo * Ho);
      y0[q] = p < total ? yo * STRIDE - 1 : -(1 << 20);  // a row past the end fails every bounds check below: zeros
      x0[q] = xo * STRIDE - 1;
      ib[q] = img * H * W * CIN;
    }
    float acc[2][NT][4];
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[m][nt][i] = 0.f;
#pragma unroll
    for (int ch = 0; ch < K / 16; ++ch) {
      uint32_t a[2][4];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = ch * 16 + h * 8 + 2 * t;  // this lane's channel pair: columns k, k+1 of the im2col row
        const int tap = k / CIN, c = k % CIN, ky = tap / KS, kx = tap % KS;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int yy = y0[q] + ky, xx = x0[q] + kx;
          uint32_t v = 0u;
          if (static_cast<unsigned>(yy) < static_cast<unsigned>(H) && static_cast<unsigned>(xx) < static_cast<unsigned>(W))
            v = __ldg(reinterpret_cast<const uint32_t*>(x + ib[q] + (yy * W + xx) * CIN + c));
          a[q >> 1][(q & 1) + 2 * h] = v;
        }
      }
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const uint32_t b0 = sw[((nt * 8 + g) * KP + ch * 16 + 2 * t) >> 1];
        const uint32_t b1 = sw[((nt * 8 + g) * KP + ch * 16 + 8 + 2 * t) >> 1];
        mma_bf16_m16n8k16(acc[0][nt], a[0], b0, b1);
        mma_bf16_m16n8k16(acc[1][nt], a[1], b0, b1);
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int p = tile * 32 + (q >> 1) * 16 + (q & 1) * 8 + g;
      if (p >= total) continue;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const float v0 = silu_f(acc[q >> 1][nt][2 * (q & 1)] + bs[nt][0]);
        const float v1 = silu_f(acc[q >> 1][nt][2 * (q & 1) + 1] + bs[nt][1]);
        *reinterpret_cast<uint32_t*>(out + static_cast<size_t>(p) * COUT + nt * 8 + 2 * t) = pack_bf16x2(v0, v1);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// a-1 input assembly (pipeline_diffuman4d.py:373-395)
// ---------------------------------------------------------------------------------------------
__global__ void assemble_kernel(const AssembleArgs a, int Cin) {
  const int f = blockIdx.y;
  const int hw = a.h * a.w;
  const bool is_cond = __bfloat162float(a.mask[static_cast<size_t>(f) * hw]) == 0.f;
  // the rows of frame f's positive and negative images (-1: not written); the positive half is the LAST half when cfg
  // (torch.cat([negative, positive]))
  const bool whole = a.half < 0;
  const bool shard = !whole && a.n_f > 0;
  const bool rows = !shard || (f >= a.f0 && f < a.f0 + a.n_f);  // frame f has sample rows
  if (!rows && !is_cond) return;                                // nothing to write for frame f
  const int fr = shard ? f - a.f0 : f;
  const int pos_img = !rows ? -1 : whole ? (a.cfg ? a.F + f : f) : (a.half == 1 ? fr : -1);
  const int neg_img = !rows ? -1 : whole ? (a.cfg ? f : -1) : (a.half == 0 ? fr : -1);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    long long t = 0;
    if (!is_cond) {
      long long idx = a.timestep_indices[f];
      idx = idx < 0 ? 0 : (idx >= a.n_steps ? a.n_steps - 1 : idx);
      t = a.timesteps_table[idx];
    }
    if (pos_img >= 0) a.timestep_out[pos_img] = t;
    if (neg_img >= 0) a.timestep_out[neg_img] = t;
  }
  const bf16 one = __float2bfloat16_rn(1.f), zero = __float2bfloat16_rn(0.f), mone = __float2bfloat16_rn(-1.f);
  bf16* const pos = pos_img >= 0 ? a.sample + static_cast<size_t>(pos_img) * Cin * hw : nullptr;
  bf16* const neg = neg_img >= 0 ? a.sample + static_cast<size_t>(neg_img) * Cin * hw : nullptr;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += gridDim.x * blockDim.x) {
    const bf16 m = a.mask[static_cast<size_t>(f) * hw + p];
    for (int c = 0; c < 4; ++c) {
      const size_t li = (static_cast<size_t>(f) * 4 + c) * hw + p;
      bf16 lat = a.latents[li];
      if (is_cond) {
        lat = a.pixel[li];
        a.latents[li] = lat;  // reference aliasing quirk: latents <- image latents at cond frames (PIPE:375-379)
      }
      if (pos) pos[static_cast<size_t>(c) * hw + p] = lat;
      if (neg) neg[static_cast<size_t>(c) * hw + p] = is_cond ? one : lat;
    }
    int ch = 4;
    for (int c = 0; c < 6; ++c, ++ch) {
      if (pos) pos[static_cast<size_t>(ch) * hw + p] = a.plucker[(static_cast<size_t>(f) * 6 + c) * hw + p];
      if (neg) neg[static_cast<size_t>(ch) * hw + p] = zero;
    }
    if (a.skel_latents) {
      for (int c = 0; c < 4; ++c, ++ch) {
        if (pos) pos[static_cast<size_t>(ch) * hw + p] = a.skel_latents[(static_cast<size_t>(f) * 4 + c) * hw + p];
        if (neg) neg[static_cast<size_t>(ch) * hw + p] = mone;
      }
    }
    if (pos) pos[static_cast<size_t>(ch) * hw + p] = m;
    if (neg) neg[static_cast<size_t>(ch) * hw + p] = m;
  }
}

// images 0..n_neg-1 <- small image 0 ; images n_neg..n_neg+n_pos-1 <- small images 1..n_pos   (per_img elements each,
// multiple of 8)
__global__ void broadcast_neg_images_kernel(const bf16* __restrict__ small, long long per_img8, int n_neg, int n_pos,
                                            bf16* __restrict__ full) {
  const long long total = per_img8 * (n_neg + n_pos);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long img = i / per_img8, off = i - img * per_img8;
    const long long src = img < n_neg ? 0 : img - n_neg + 1;
    reinterpret_cast<uint4*>(full)[i] = __ldg(reinterpret_cast<const uint4*>(small) + src * per_img8 + off);
  }
}
__global__ void fill_bf16_kernel(bf16* __restrict__ p, long long n, float v) {
  const bf16 b = __float2bfloat16_rn(v);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    p[i] = b;
}

// ---------------------------------------------------------------------------------------------
// a-13 + a-14: CFG combine + per-frame scheduler step (pipeline_diffuman4d.py:408-423).  One kernel per scheduler, one CTA
// row per frame (blockIdx.y); a frame's step index is its timestep index.  The helpers below are the part they all share.
// ---------------------------------------------------------------------------------------------
template <bool EMU>
__device__ __forceinline__ float rnd(float x) { return EMU ? bf16_round(x) : x; }
// fp32 a - b without contraction into an FMA with a preceding product (the reference evaluates each op separately)
template <bool EMU>
__device__ __forceinline__ float sub_nc(float a, float b) { return EMU ? __fsub_rn(a, b) : a - b; }
template <bool EMU>
__device__ __forceinline__ float mul_nc(float a, float b) { return EMU ? __fmul_rn(a, b) : a * b; }

// The frame prologue: writes the frame's advanced timestep index and, for a multistep solver (lon_in != null), its
// advanced order count.  A conditioning frame is never stepped: its latents pass through and its history stays untouched;
// the function returns false for it.  Otherwise idx receives the step index clamped to the table, lon the order count.
__device__ __forceinline__ bool step_frame(const StepArgs& a, int n_steps, const int* lon_in, int* lon_out,
                                           int solver_order, long long& idx, int& lon) {
  const int f = blockIdx.y;
  const bool is_cond = __bfloat162float(a.mask[static_cast<size_t>(f) * a.hw]) == 0.f;
  idx = a.timestep_indices[f];
  lon = lon_in ? lon_in[f] : 0;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.ts_out[f] = is_cond ? 0 : idx + 1;
    if (lon_out) lon_out[f] = is_cond ? lon : min(lon + 1, solver_order);
  }
  if (is_cond) {
    const size_t base = static_cast<size_t>(f) * a.chw;
    if (a.out != a.latents)
      for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.chw; i += gridDim.x * blockDim.x)
        a.out[base + i] = a.latents[base + i];
    return false;
  }
  idx = idx < 0 ? 0 : (idx >= n_steps ? n_steps - 1 : idx);
  return true;
}

// The CFG combine u + g * (c - u) of the two halves' predictions u (negative) and c (positive).
template <bool EMU>
__device__ __forceinline__ float cfg_combine(const StepArgs& a, float u, float c) {
  return rnd<EMU>(u + rnd<EMU>(a.guidance * rnd<EMU>(c - u)));
}

// The model output at element j of the frames: the CFG combine of the two halves, or the one prediction.
template <bool EMU>
__device__ __forceinline__ float model_output(const StepArgs& a, size_t j) {
  if (!a.cfg) return __bfloat162float(a.noise[j]);
  return cfg_combine<EMU>(a, __bfloat162float(a.noise[j]),
                          __bfloat162float(a.noise[static_cast<size_t>(a.F) * a.chw + j]));
}

// four consecutive bf16 as fp32 (one 8-byte load; p 8-byte aligned), and the reverse, rounding to nearest
__device__ __forceinline__ void load_bf16x4(const bf16* p, float v[4]) {
  const uint2 r = *reinterpret_cast<const uint2*>(p);
  v[0] = __uint_as_float(r.x << 16); v[1] = __uint_as_float(r.x & 0xFFFF0000u);
  v[2] = __uint_as_float(r.y << 16); v[3] = __uint_as_float(r.y & 0xFFFF0000u);
}
__device__ __forceinline__ void store_bf16x4(bf16* p, const float v[4]) {
  const __nv_bfloat162 lo = __floats2bfloat162_rn(v[0], v[1]), hi = __floats2bfloat162_rn(v[2], v[3]);
  uint2 r;
  r.x = *reinterpret_cast<const unsigned int*>(&lo);
  r.y = *reinterpret_cast<const unsigned int*>(&hi);
  *reinterpret_cast<uint2*>(p) = r;
}

// convert_model_output: the data prediction of model output m at sample x (alpha_t, sigma_t of the step), computed in
// the model output's dtype.
template <bool EMU>
__device__ __forceinline__ float data_prediction(int prediction_type, float x, float m, float alpha, float sigma) {
  if (prediction_type == 0) return rnd<EMU>(rnd<EMU>(x - rnd<EMU>(sigma * m)) / alpha);   // epsilon
  if (prediction_type == 1) return rnd<EMU>(rnd<EMU>(alpha * x) - rnd<EMU>(sigma * m));   // v_prediction
  return m;                                                                             // sample
}

// upstream DDIMScheduler.step
template <bool EMU>
__global__ void cfg_ddim_kernel(const StepArgs a, const d4d_sched s) {
  long long idx;
  int lon;
  if (!step_frame(a, s.n_steps, nullptr, nullptr, 0, idx, lon)) return;
  const size_t base = static_cast<size_t>(blockIdx.y) * a.chw;
  const long long t = s.timesteps_table[idx];
  const long long prev_t = t - s.num_train_timesteps / s.n_steps;
  const float a_t = s.alphas_cumprod[t];
  const float a_prev = prev_t >= 0 ? s.alphas_cumprod[prev_t] : s.final_alpha_cumprod;
  const float b_t = 1.0f - a_t;
  const float sa = sqrtf(a_t), sb = sqrtf(b_t);
  const float sa_prev = sqrtf(a_prev), sdir = sqrtf(1.0f - a_prev);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.chw; i += gridDim.x * blockDim.x) {
    const float eps_in = model_output<EMU>(a, base + i);
    const float x = __bfloat162float(a.latents[base + i]);
    float x0 = data_prediction<EMU>(s.prediction_type, x, eps_in, sa, sb);
    float eps = eps_in;
    if (s.prediction_type == 1) eps = rnd<EMU>(rnd<EMU>(sa * eps_in) + rnd<EMU>(sb * x));
    else if (s.prediction_type == 2) eps = rnd<EMU>(rnd<EMU>(x - rnd<EMU>(sa * x0)) / sb);
    if (s.clip_sample) x0 = fminf(fmaxf(x0, -s.clip_sample_range), s.clip_sample_range);
    const float dir = rnd<EMU>(sdir * eps);
    const float prev = rnd<EMU>(rnd<EMU>(sa_prev * x0) + dir);
    a.out[base + i] = __float2bfloat16_rn(prev);
  }
}

// upstream DDPMScheduler.step (fixed variances): x0 by prediction type, the clip, the posterior mean c0 * x0 + c1 * x and,
// on rows with t > 0, std * z with z of ddpm_noise.cuh keyed by the frame's task index st.frame_ids[f] and its row.  A
// thread steps four consecutive elements, the four draws of one Philox call, with 8-byte loads and stores.
template <bool EMU>
__global__ void cfg_ddpm_kernel(const StepArgs a, const d4d_ddpm_sched s, const SolverState st) {
  long long idx;
  int lon;
  if (!step_frame(a, s.n_steps, nullptr, nullptr, 0, idx, lon)) return;
  const size_t base = static_cast<size_t>(blockIdx.y) * a.chw;
  const float* k = s.coefs + idx * kDdpmCoefs;
  const float sa = k[0], sb = k[1], c0 = k[2], c1 = k[3], std = k[4];
  const bool noisy = k[5] != 0.f;
  const uint32_t frame = static_cast<uint32_t>(st.frame_ids[blockIdx.y]);
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < a.chw / 4; q += gridDim.x * blockDim.x) {
    double z[4] = {0.0, 0.0, 0.0, 0.0};
    if (noisy) ddpm_normal4(s.seed, static_cast<uint32_t>(q), frame, static_cast<uint32_t>(idx), z);
    const size_t e = base + 4 * static_cast<size_t>(q);
    float x[4], m[4], prev[4];
    load_bf16x4(a.latents + e, x);
    load_bf16x4(a.noise + e, m);
    if (a.cfg) {
      float c[4];
      load_bf16x4(a.noise + static_cast<size_t>(a.F) * a.chw + e, c);
#pragma unroll
      for (int j = 0; j < 4; ++j) m[j] = cfg_combine<EMU>(a, m[j], c[j]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float x0 = data_prediction<EMU>(s.prediction_type, x[j], m[j], sa, sb);
      if (s.clip_sample) x0 = fminf(fmaxf(x0, -s.clip_sample_range), s.clip_sample_range);
      prev[j] = rnd<EMU>(rnd<EMU>(c0 * x0) + rnd<EMU>(c1 * x[j]));
      if (noisy) prev[j] = rnd<EMU>(prev[j] + rnd<EMU>(std * round_noise<EMU>(z[j])));
    }
    store_bf16x4(a.out + e, prev);
  }
}

__global__ void ddpm_noise_kernel(unsigned long long seed, const long long* __restrict__ frame_ids,
                                  const long long* __restrict__ ts_idx, int quads, float* __restrict__ out) {
  const int f = blockIdx.y;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < quads; q += gridDim.x * blockDim.x) {
    double z[4];
    ddpm_normal4(seed, static_cast<uint32_t>(q), static_cast<uint32_t>(frame_ids[f]), static_cast<uint32_t>(ts_idx[f]), z);
    for (int j = 0; j < 4; ++j) out[(static_cast<size_t>(f) * quads + q) * 4 + j] = round_noise<false>(z[j]);
  }
}

// upstream DPMSolverMultistepScheduler.step (dpmsolver++ / midpoint, order <= 2); history x0_prev, lower_order_nums
template <bool EMU>
__global__ void cfg_dpm_kernel(const StepArgs a, const d4d_dpm_sched s, const SolverState st) {
  long long idx;
  int lon;
  if (!step_frame(a, s.n_steps, st.lower_order_nums, st.lower_order_nums_out, s.solver_order, idx, lon)) return;
  const size_t base = static_cast<size_t>(blockIdx.y) * a.chw;
  const float* k = s.coefs + idx * kDpmCoefs;
  const float alpha_s = k[0], sigma_s = k[1], ratio = k[2], c = k[3], half_c = k[4], inv_r0 = k[5];
  const bool first = s.solver_order == 1 || lon < 1 || (s.final_first_order && idx == s.n_steps - 1);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.chw; i += gridDim.x * blockDim.x) {
    const float m = model_output<EMU>(a, base + i);
    const float x = __bfloat162float(a.latents[base + i]);
    const float x0 = data_prediction<EMU>(s.prediction_type, x, m, alpha_s, sigma_s);
    const float m1 = __bfloat162float(st.x0_prev[base + i]);
    st.x0_prev[base + i] = __float2bfloat16_rn(x0);
    // sample is upcast to fp32: (sigma_t / sigma_s) * sample stays fp32, each coef * (bf16 tensor) rounds to bf16
    float prev = sub_nc<EMU>(mul_nc<EMU>(ratio, x), rnd<EMU>(c * x0));
    if (!first) {
      const float d1 = rnd<EMU>(inv_r0 * rnd<EMU>(x0 - m1));
      prev = sub_nc<EMU>(prev, rnd<EMU>(half_c * d1));
    }
    a.out[base + i] = __float2bfloat16_rn(prev);
  }
}

// upstream UniPCMultistepScheduler.step (predict_x0, bh1 / bh2, order <= 2); history x0_prev, x0_prev2, last_sample,
// lower_order_nums.  Unlike DPM-Solver++, upstream does not upcast the sample: every product and difference rounds to
// bf16 in EMU mode.
template <bool EMU>
__global__ void cfg_unipc_kernel(const StepArgs a, const d4d_unipc_sched s, const SolverState st) {
  long long idx;
  int lon;
  if (!step_frame(a, s.n_steps, st.lower_order_nums, st.lower_order_nums_out, s.solver_order, idx, lon)) return;
  const size_t base = static_cast<size_t>(blockIdx.y) * a.chw;
  const float* k = s.coefs + idx * kUniPCCoefs;
  const float alpha_s = k[0], sigma_s = k[1];
  const float p_ratio = k[2], p_cphi = k[3], p_cB = k[4], p_rk = k[5];
  const float c_ratio = k[6], c_cphi = k[7], c_cB = k[8], c_rk = k[9];
  const float rho0 = rnd<EMU>(k[10]), rho1 = rnd<EMU>(k[11]);   // upstream casts the solved rhos to the sample dtype
  // the corrector runs at the previous step's order, which is lon; the predictor's order is capped by the row
  const bool correct = lon >= 1 && k[12] != 0.f;
  const int c_order = min(lon, s.solver_order);
  const int p_order = min(static_cast<int>(k[13]), lon + 1);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.chw; i += gridDim.x * blockDim.x) {
    const float m = model_output<EMU>(a, base + i);
    float x = __bfloat162float(a.latents[base + i]);
    const float x0 = data_prediction<EMU>(s.prediction_type, x, m, alpha_s, sigma_s);
    const float m0 = __bfloat162float(st.x0_prev[base + i]);
    const float m1 = st.x0_prev2 ? __bfloat162float(st.x0_prev2[base + i]) : 0.f;
    if (correct) {  // UniC: recompute the sample from last_sample with this step's data prediction
      const float last = __bfloat162float(st.last_sample[base + i]);
      const float xt = rnd<EMU>(sub_nc<EMU>(rnd<EMU>(c_ratio * last), rnd<EMU>(c_cphi * m0)));
      const float d1t = rnd<EMU>(x0 - m0);
      float inner;
      if (c_order == 1) {
        inner = rnd<EMU>(0.f + rnd<EMU>(0.5f * d1t));   // upstream: 0 + rhos_c[-1] * D1_t
      } else {
        const float d1 = rnd<EMU>(rnd<EMU>(m1 - m0) / c_rk);
        inner = rnd<EMU>(rnd<EMU>(rho0 * d1) + rnd<EMU>(rho1 * d1t));
      }
      x = rnd<EMU>(sub_nc<EMU>(xt, rnd<EMU>(c_cB * inner)));
    }
    if (st.x0_prev2) st.x0_prev2[base + i] = __float2bfloat16_rn(m0);
    st.x0_prev[base + i] = __float2bfloat16_rn(x0);
    st.last_sample[base + i] = __float2bfloat16_rn(x);
    // UniP from the (corrected) sample
    const float xt = rnd<EMU>(sub_nc<EMU>(rnd<EMU>(p_ratio * x), rnd<EMU>(p_cphi * x0)));
    float prev;
    if (p_order == 1) {
      prev = sub_nc<EMU>(xt, mul_nc<EMU>(p_cB, 0.f));   // upstream: x_t_ - alpha_t * B_h * 0 (a signed zero)
    } else {
      const float d1 = rnd<EMU>(rnd<EMU>(m0 - x0) / p_rk);
      prev = rnd<EMU>(sub_nc<EMU>(xt, rnd<EMU>(p_cB * rnd<EMU>(0.5f * d1))));
    }
    a.out[base + i] = __float2bfloat16_rn(prev);
  }
}

// upstream PNDMScheduler.step_plms (skip_prk_steps) and _get_prev_sample; history ets[4] (a ring of the last model
// outputs), cur_sample and the frame's counter (lower_order_nums, uncapped).  Upstream does not upcast: in EMU mode every
// product, sum and quotient rounds to bf16, the Adams-Bashforth sums one operation at a time as upstream writes them.
constexpr int kPndmNoCap = 0x7fffffff;
template <bool EMU>
__global__ void cfg_pndm_kernel(const StepArgs a, const d4d_pndm_sched s, const SolverState st) {
  long long idx;
  int counter;
  if (!step_frame(a, s.n_steps, st.lower_order_nums, st.lower_order_nums_out, kPndmNoCap, idx, counter)) return;
  const size_t base = static_cast<size_t>(blockIdx.y) * a.chw;
  const float* k = s.coefs + idx * kPndmCoefs + (counter == 1 ? 5 : 0);   // counter 1 steps from t + T/n to t
  const float sqrt_a = k[0], sqrt_b = k[1], sample_coef = k[2], alpha_diff = k[3], denom = k[4];
  // the output of counter c (c != 1) goes to ring slot (c == 0 ? 0 : c - 1) % 4; after it, the last min(c, 4) outputs
  // are kept (1 at counters 0 and 1: counter 1's output is not kept)
  const int slot = counter == 0 ? 0 : counter - 1;
  const int kept = counter < 2 ? 1 : min(counter, 4);
  bf16* const e1p = st.ets[slot & 3];
  const bf16* const e2p = st.ets[(slot + 3) & 3];
  const bf16* const e3p = st.ets[(slot + 2) & 3];
  const bf16* const e4p = st.ets[(slot + 1) & 3];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.chw; i += gridDim.x * blockDim.x) {
    const float m = model_output<EMU>(a, base + i);
    float x = __bfloat162float(a.latents[base + i]);
    float eps;
    if (counter == 0) {
      eps = m;
      e1p[base + i] = __float2bfloat16_rn(m);
      st.cur_sample[base + i] = a.latents[base + i];
    } else if (counter == 1) {  // (model_output + ets[-1]) / 2, from the sample counter 0 started from
      eps = rnd<EMU>(rnd<EMU>(m + __bfloat162float(st.ets[0][base + i])) / 2.f);
      x = __bfloat162float(st.cur_sample[base + i]);
    } else {
      e1p[base + i] = __float2bfloat16_rn(m);
      const float e2 = __bfloat162float(e2p[base + i]);
      if (kept == 2) {
        eps = rnd<EMU>(rnd<EMU>(rnd<EMU>(3.f * m) - e2) / 2.f);
      } else {
        const float e3 = __bfloat162float(e3p[base + i]);
        const float s3 = rnd<EMU>(rnd<EMU>(rnd<EMU>(kept == 3 ? 23.f * m : 55.f * m) -
                                           rnd<EMU>(kept == 3 ? 16.f * e2 : 59.f * e2)) +
                                  rnd<EMU>(kept == 3 ? 5.f * e3 : 37.f * e3));
        if (kept == 3) {
          eps = rnd<EMU>(s3 / 12.f);
        } else {
          const float e4 = __bfloat162float(e4p[base + i]);
          eps = rnd<EMU>(static_cast<float>(1.0 / 24.0) * rnd<EMU>(s3 - rnd<EMU>(9.f * e4)));
        }
      }
    }
    if (s.prediction_type == 1) eps = rnd<EMU>(rnd<EMU>(sqrt_a * eps) + rnd<EMU>(sqrt_b * x));   // v -> epsilon
    const float prev = rnd<EMU>(rnd<EMU>(sample_coef * x) - rnd<EMU>(rnd<EMU>(alpha_diff * eps) / denom));
    a.out[base + i] = __float2bfloat16_rn(prev);
  }
}

// upstream DEISMultistepScheduler.step (deis / logrho, order <= 3); history m_prev, m_prev2 (the last model outputs in
// their epsilon form), lower_order_nums.  Upstream does not upcast the sample: in EMU mode every product, sum and
// quotient rounds to bf16, the higher-order sums one term at a time as upstream writes them.
template <bool EMU>
__global__ void cfg_deis_kernel(const StepArgs a, const d4d_deis_sched s, const SolverState st) {
  long long idx;
  int lon;
  if (!step_frame(a, s.n_steps, st.lower_order_nums, st.lower_order_nums_out, s.solver_order, idx, lon)) return;
  const size_t base = static_cast<size_t>(blockIdx.y) * a.chw;
  const float* k = s.coefs + idx * kDeisCoefs;
  const float alpha_s = k[0], sigma_s = k[1], ratio = k[2], c_first = k[3], alpha_t = k[4];
  const int order = min(min(s.solver_order, lon + 1), static_cast<int>(k[10]));
  const float c0 = order == 3 ? k[7] : k[5], c1 = order == 3 ? k[8] : k[6], c2 = k[9];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.chw; i += gridDim.x * blockDim.x) {
    const float m = model_output<EMU>(a, base + i);
    const float x = __bfloat162float(a.latents[base + i]);
    // convert_model_output: the data prediction, then back to its epsilon form (in the model output's dtype)
    const float x0 = data_prediction<EMU>(s.prediction_type, x, m, alpha_s, sigma_s);
    const float m0 = rnd<EMU>(rnd<EMU>(x - rnd<EMU>(alpha_s * x0)) / sigma_s);
    const bf16 m1b = st.m_prev[base + i];
    const float m1 = __bfloat162float(m1b);
    const float m2 = st.m_prev2 ? __bfloat162float(st.m_prev2[base + i]) : 0.f;
    if (st.m_prev2) st.m_prev2[base + i] = m1b;
    st.m_prev[base + i] = __float2bfloat16_rn(m0);
    float prev;
    if (order == 1) {
      prev = rnd<EMU>(rnd<EMU>(ratio * x) - rnd<EMU>(c_first * m0));
    } else {
      float acc = rnd<EMU>(rnd<EMU>(x / alpha_s) + rnd<EMU>(c0 * m0));
      acc = rnd<EMU>(acc + rnd<EMU>(c1 * m1));
      if (order == 3) acc = rnd<EMU>(acc + rnd<EMU>(c2 * m2));
      prev = rnd<EMU>(alpha_t * acc);
    }
    a.out[base + i] = __float2bfloat16_rn(prev);
  }
}

// upstream DPMSolverSinglestepScheduler.step (dpmsolver++ / midpoint, order <= 3); history x0_prev, x0_prev2 (the last
// data predictions), cur_sample (the sample the frame's current block started from), lower_order_nums.  A step at order
// 1 starts a block and saves its sample; a step at order 2 or 3 updates from that sample with the block start's data
// prediction (x0_prev at order 2, x0_prev2 at order 3).  Upstream does not upcast the sample: in EMU mode every product
// and difference rounds to bf16, the sums one term at a time as upstream writes them.
template <bool EMU>
__global__ void cfg_dpm_single_kernel(const StepArgs a, const d4d_dpm_single_sched s, const SolverState st) {
  long long idx;
  int lon;
  if (!step_frame(a, s.n_steps, st.lower_order_nums, st.lower_order_nums_out, s.solver_order, idx, lon)) return;
  const size_t base = static_cast<size_t>(blockIdx.y) * a.chw;
  const float* k = s.coefs + idx * kDpmSingleCoefs;
  const float alpha_s = k[0], sigma_s = k[1];
  // upstream lowers the row's order while the history it needs is missing
  const int order = min(static_cast<int>(k[12]), lon + 1);
  const float* u = k + (order == 1 ? 2 : order == 2 ? 4 : 8);
  const float ratio = u[0], c = u[1], c_d1 = u[2], inv_r0 = u[3];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.chw; i += gridDim.x * blockDim.x) {
    const float m = model_output<EMU>(a, base + i);
    const bf16 xb = a.latents[base + i];
    const float x = __bfloat162float(xb);
    const float x0 = data_prediction<EMU>(s.prediction_type, x, m, alpha_s, sigma_s);
    const bf16 m1b = st.x0_prev[base + i];
    const float m1 = __bfloat162float(m1b);
    const float m2 = st.x0_prev2 ? __bfloat162float(st.x0_prev2[base + i]) : 0.f;
    if (st.x0_prev2) st.x0_prev2[base + i] = m1b;
    st.x0_prev[base + i] = __float2bfloat16_rn(x0);
    float prev;
    if (order == 1) {
      st.cur_sample[base + i] = xb;
      prev = rnd<EMU>(rnd<EMU>(ratio * x) - rnd<EMU>(c * x0));
    } else {
      const float xs = __bfloat162float(st.cur_sample[base + i]);
      const float d0 = order == 2 ? m1 : m2;     // the block start's data prediction
      const float d1 = rnd<EMU>(inv_r0 * rnd<EMU>(x0 - d0));
      prev = rnd<EMU>(rnd<EMU>(ratio * xs) - rnd<EMU>(c * d0));
      prev = order == 2 ? rnd<EMU>(prev - rnd<EMU>(c_d1 * d1)) : rnd<EMU>(prev + rnd<EMU>(c_d1 * d1));
    }
    a.out[base + i] = __float2bfloat16_rn(prev);
  }
}

// ---------------------------------------------------------------------------------------------
// frame-sharded window: K/V arrival flags in peer memory
// ---------------------------------------------------------------------------------------------
__global__ void kv_signal_kernel(const KvFlagArgs a) {
  const int r = threadIdx.x;
  if (r >= a.world) return;
  __threadfence_system();  // order the K/V stores of the preceding kernels (this stream) before the flag
  unsigned int* f = a.flags[r] + a.slot * 8 + a.rank;
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(f), "r"(a.epoch) : "memory");
}
__global__ void kv_wait_kernel(const KvFlagArgs a) {
  const int r = threadIdx.x;
  if (r >= a.world) return;
  const unsigned int* f = a.flags[a.rank] + a.slot * 8 + r;
  unsigned int v = 0;
  unsigned long long spins = 0;
  do {
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
    if (++spins > (1ull << 31)) {  // ~ seconds: a lost peer must trap, not hang the box
      printf("d4d: K/V flag timeout rank=%d waiting for rank=%d epoch=%u have=%u\n", a.rank, r, a.epoch, v);
      __trap();
    }
  } while (static_cast<int>(v - a.epoch) < 0);
  __threadfence_system();
}

// frame-sharded sliding loop: this rank's updated frames into every rank's gathered window (blockIdx.y = destination),
// plain 16-byte stores through the peer pointers like the K/V scatter epilogue; the flag round follows in the stream
__global__ void window_scatter_kernel(const WindowScatterArgs a, const WindowResultLayout L) {
  char* d = static_cast<char*>(a.dst[blockIdx.y]);
  const long long row0 = static_cast<long long>(a.rank) * a.F_local;
  const long long n = a.F_local * a.chw / 8;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const uint4* lat = reinterpret_cast<const uint4*>(a.latents);
  uint4* lat_d = reinterpret_cast<uint4*>(d) + row0 * a.chw / 8;
  for (long long i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) lat_d[i] = lat[i];
  if (a.x0_prev) {
    const uint4* x0 = reinterpret_cast<const uint4*>(a.x0_prev);
    uint4* x0_d = reinterpret_cast<uint4*>(d + L.x0) + row0 * a.chw / 8;
    for (long long i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) x0_d[i] = x0[i];
  }
  if (blockIdx.x == 0) {
    long long* ts_d = reinterpret_cast<long long*>(d + L.ts) + row0;
    int* lon_d = reinterpret_cast<int*>(d + L.lon) + row0;
    for (int f = threadIdx.x; f < a.F_local; f += blockDim.x) {
      ts_d[f] = a.ts[f];
      if (a.lower_order_nums) lon_d[f] = a.lower_order_nums[f];
    }
  }
}

inline int blocks_for(long long total, int threads) { return static_cast<int>((total + threads - 1) / threads); }

}  // namespace

int sinusoid_run(const float* pos, int n, int dim, int flip, float freq_shift, bf16* out, cudaStream_t stream) {
  D4D_REQUIRE(dim % 2 == 0 && n > 0, "sinusoid dims");
  const int total = n * (dim / 2);
  sinusoid_kernel<float><<<blocks_for(total, 256), 256, 0, stream>>>(pos, n, dim, flip, freq_shift, out);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int sinusoid_i64_run(const long long* pos, int n, int dim, int flip, float freq_shift, bf16* out, cudaStream_t stream) {
  D4D_REQUIRE(dim % 2 == 0 && n > 0, "sinusoid dims");
  const int total = n * (dim / 2);
  sinusoid_kernel<long long><<<blocks_for(total, 256), 256, 0, stream>>>(pos, n, dim, flip, freq_shift, out);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int silu_run(const bf16* x, long long n, bf16* out, cudaStream_t stream) {
  if (n <= 0) return 0;
  silu_kernel<<<blocks_for(n, 256), 256, 0, stream>>>(x, n, out);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int im2col_nchw_run(const bf16* x, int n, int Cin, int H, int W, int cin_pad, int KP, bf16* out, cudaStream_t stream) {
  D4D_REQUIRE(cin_pad >= Cin && KP % cin_pad == 0 && KP >= 9 * cin_pad, "im2col padding");
  const long long total = static_cast<long long>(n) * H * W * (KP / cin_pad);
  im2col_nchw_kernel<<<blocks_for(total, 256), 256, 0, stream>>>(x, n, Cin, H, W, cin_pad, KP, out);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int im2col_nhwc_run(const bf16* x, int n, int H, int W, int C, int ksize, int stride, bf16* out, cudaStream_t stream) {
  D4D_REQUIRE(C % 8 == 0 && (ksize == 3 || ksize == 4) && (stride == 1 || stride == 2), "im2col_nhwc dims");
  const int Ho = (H + 2 - ksize) / stride + 1, Wo = (W + 2 - ksize) / stride + 1;
  const long long total = static_cast<long long>(n) * Ho * Wo * ksize * ksize * (C / 8);
  im2col_nhwc_kernel<<<blocks_for(total, 256), 256, 0, stream>>>(x, n, H, W, C, ksize, stride, out);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int nhwc_to_nchw_run(const bf16* x, int ld, int n, int C, int hw, bf16* out, cudaStream_t stream) {
  NchwDst d = {};
  d.p[0] = out;
  d.n = 1;
  return nhwc_to_nchw_run(x, ld, n, C, hw, d, stream);
}
int nhwc_to_nchw_run(const bf16* x, int ld, int n, int C, int hw, const NchwDst& out, cudaStream_t stream) {
  D4D_REQUIRE(out.n >= 1 && out.n <= 8, "nhwc_to_nchw: 1 to 8 destinations");
  for (int i = 0; i < out.n; ++i) D4D_REQUIRE(out.p[i] != nullptr, "nhwc_to_nchw: null destination");
  const long long total = static_cast<long long>(n) * C * hw;
  nhwc_to_nchw_kernel<<<dim3(blocks_for(total, 256), out.n), 256, 0, stream>>>(x, ld, n, C, hw, out);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int pose_conv0_run(const bf16* x_nchw, int n, int H, int W, const bf16* w, const float* bias, bf16* out_nhwc4,
                   cudaStream_t stream) {
  const long long groups = static_cast<long long>(n) * H * ((W + kPix0 - 1) / kPix0);
  pose_conv0_kernel<<<blocks_for(groups, 128), 128, 0, stream>>>(x_nchw, n, H, W, w, bias, out_nhwc4);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int pose_conv_run(const bf16* x, int n, int Cin, int H, int W, const bf16* w, const float* bias, int Cout, int ksize,
                  int stride, bf16* out_nhwc, cudaStream_t stream) {
  // pad 1 on each side: a kernel larger than the padded input has no output pixel (C's truncating division below
  // would still count one)
  D4D_REQUIRE(H + 2 >= ksize && W + 2 >= ksize, "pose conv: kernel larger than the padded input");
  const int Ho = (H + 2 - ksize) / stride + 1, Wo = (W + 2 - ksize) / stride + 1;
  const long long total = static_cast<long long>(n) * Ho * Wo;
  D4D_REQUIRE(static_cast<long long>(n) * H * W * Cin < (1ll << 31) && total * Cout < (1ll << 31), "pose conv: 32-bit offsets");
  D4D_REQUIRE(reinterpret_cast<uintptr_t>(w) % 16 == 0, "pose conv weights must be 16-byte aligned");
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int threads = 256;
  const long long tiles = (total + 31) / 32;
  const int blocks = static_cast<int>(std::min<long long>((tiles + threads / 32 - 1) / (threads / 32), 2ll * sms));
#define D4D_PC(CO, CI, KS, ST)                                                                                          \
  if (Cout == CO && Cin == CI && ksize == KS && stride == ST) {                                                          \
    const size_t smem = static_cast<size_t>(CO) * (KS * KS * CI + 8) * 2;                                                 \
    pose_conv_mma_kernel<CO, CI, KS, ST><<<blocks, threads, smem, stream>>>(x, n, H, W, w, bias, out_nhwc);               \
    D4D_CUDA_OK(cudaGetLastError());                                                                                     \
    return 0;                                                                                                            \
  }
  D4D_PC(16, 4, 4, 2)
  D4D_PC(16, 16, 3, 1)
  D4D_PC(32, 16, 4, 2)
  D4D_PC(32, 32, 3, 1)
#undef D4D_PC
  set_error("pose conv: unsupported layer " + std::to_string(Cin) + "->" + std::to_string(Cout) + " k" + std::to_string(ksize) +
            " s" + std::to_string(stride));
  return 1;
}

int kv_signal_run(const KvFlagArgs& a, cudaStream_t stream) {
  kv_signal_kernel<<<1, 32, 0, stream>>>(a);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}
int kv_wait_run(const KvFlagArgs& a, cudaStream_t stream) {
  kv_wait_kernel<<<1, 32, 0, stream>>>(a);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int window_scatter_run(const WindowScatterArgs& a, size_t dst_bytes, cudaStream_t stream) {
  D4D_REQUIRE(a.world >= 1 && a.world <= 8, "window scatter: world must be in [1, 8]");
  D4D_REQUIRE(a.rank >= 0 && a.rank < a.world, "window scatter: rank must be in [0, world)");
  D4D_REQUIRE(a.F_local >= 1 && static_cast<long long>(a.F_local) * a.world == a.F_total,
              "window scatter: F_total must equal world * local frames");
  D4D_REQUIRE(a.chw > 0 && a.chw % 8 == 0, "window scatter: 4*h*w must be a positive multiple of 8");
  D4D_REQUIRE(a.latents != nullptr && a.ts != nullptr, "window scatter: null source");
  D4D_REQUIRE((a.x0_prev == nullptr) == (a.lower_order_nums == nullptr),
              "window scatter: x0_prev and lower_order_nums are given together or not at all");
  for (int r = 0; r < a.world; ++r) {
    D4D_REQUIRE(a.dst[r] != nullptr, "window scatter: null destination buffer");
    D4D_REQUIRE(reinterpret_cast<uintptr_t>(a.dst[r]) % 16 == 0, "window scatter: destinations must be 16-byte aligned");
  }
  D4D_REQUIRE(reinterpret_cast<uintptr_t>(a.latents) % 16 == 0 && reinterpret_cast<uintptr_t>(a.x0_prev) % 16 == 0,
              "window scatter: latents and x0_prev must be 16-byte aligned");
  const WindowResultLayout L = window_result_layout(a.F_total, a.chw, a.x0_prev != nullptr);
  if (L.bytes > dst_bytes) {
    set_error("window scatter: the window result (" + std::to_string(L.bytes) + " bytes) does not fit the " +
              std::to_string(dst_bytes) + "-byte exchange buffer (d4d_exchange_alloc)");
    return 1;
  }
  const long long n = a.F_local * a.chw / 8;
  dim3 grid(static_cast<unsigned>(std::min<long long>(132, blocks_for(n, 256))), a.world);
  window_scatter_kernel<<<grid, 256, 0, stream>>>(a, L);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int assemble_input_run(const AssembleArgs& a, cudaStream_t stream) {
  const int Cin = 4 + 6 + (a.skel_latents ? 4 : 0) + 1;
  const int hw = a.h * a.w;
  dim3 grid(min(64, blocks_for(hw, 256)), a.F);
  assemble_kernel<<<grid, 256, 0, stream>>>(a, Cin);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int broadcast_neg_images_run(const bf16* small, long long per_img, int n_neg, int n_pos, bf16* full, cudaStream_t stream) {
  D4D_REQUIRE(per_img % 8 == 0 && n_neg > 0 && n_pos >= 0, "broadcast_neg_images arguments");
  broadcast_neg_images_kernel<<<132 * 8, 256, 0, stream>>>(small, per_img / 8, n_neg, n_pos, full);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}
int fill_bf16_run(bf16* p, long long n, float v, cudaStream_t stream) {
  fill_bf16_kernel<<<132 * 4, 256, 0, stream>>>(p, n, v);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

// The checks every scheduler step shares.  coefs: the table the kernel reads besides the timesteps (alphas_cumprod for
// DDIM); st: the solver state of a multistep solver, null for DDIM.  A block advancing a frame's counters must not change
// what the frame's other blocks still read, hence no aliasing of the counter outputs.
static int check_step(const StepArgs& a, const int64_t* timesteps_table, const float* coefs, int n_steps,
                      int prediction_type, const SolverState* st) {
  D4D_REQUIRE(a.noise && a.latents && a.mask && a.timestep_indices && a.out && a.ts_out && timesteps_table && coefs,
              "null argument");
  D4D_REQUIRE(a.F > 0 && n_steps > 0, "the frame and step counts must be positive");
  D4D_REQUIRE(prediction_type >= 0 && prediction_type <= 2, "prediction_type");
  D4D_REQUIRE(a.ts_out != a.timestep_indices, "timestep_indices_out must not alias timestep_indices");
  if (st) {
    D4D_REQUIRE(st->lower_order_nums && st->lower_order_nums_out, "null argument");
    D4D_REQUIRE(st->lower_order_nums != st->lower_order_nums_out,
                "the timestep index and order count outputs may not alias their inputs");
  }
  return 0;
}

// grid (blocks per frame, F) and the fp32 / bf16-emulating instantiation of a step kernel
template <typename... Rest>
static int launch_step(void (*emu)(StepArgs, Rest...), void (*fp32)(StepArgs, Rest...), bool emulate_bf16,
                       cudaStream_t stream, const StepArgs& a, const Rest&... rest) {
  dim3 grid(min(64, blocks_for(a.chw, 256)), a.F);
  (emulate_bf16 ? emu : fp32)<<<grid, 256, 0, stream>>>(a, rest...);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int cfg_step_run(const StepArgs& a, const d4d_sched& s, const SolverState&, cudaStream_t stream, bool launch) {
  if (int rc = check_step(a, s.timesteps_table, s.alphas_cumprod, s.n_steps, s.prediction_type, nullptr)) return rc;
  D4D_REQUIRE(s.num_train_timesteps > 0, "ddim args");
  if (!launch) return 0;
  return launch_step(cfg_ddim_kernel<true>, cfg_ddim_kernel<false>, s.emulate_bf16, stream, a, s);
}

int cfg_step_run(const StepArgs& a, const d4d_dpm_sched& s, const SolverState& st, cudaStream_t stream, bool launch) {
  if (int rc = check_step(a, s.timesteps_table, s.coefs, s.n_steps, s.prediction_type, &st)) return rc;
  D4D_REQUIRE(st.x0_prev != nullptr, "null argument");
  D4D_REQUIRE(s.solver_order == 1 || s.solver_order == 2, "solver_order must be 1 or 2");
  if (!launch) return 0;
  return launch_step(cfg_dpm_kernel<true>, cfg_dpm_kernel<false>, s.emulate_bf16, stream, a, s, st);
}

int cfg_step_run(const StepArgs& a, const d4d_unipc_sched& s, const SolverState& st, cudaStream_t stream, bool launch) {
  if (int rc = check_step(a, s.timesteps_table, s.coefs, s.n_steps, s.prediction_type, &st)) return rc;
  D4D_REQUIRE(s.solver_order == 1 || s.solver_order == 2, "solver_order must be 1 or 2");
  D4D_REQUIRE(st.x0_prev != nullptr && st.last_sample != nullptr, "null argument");
  D4D_REQUIRE((st.x0_prev2 != nullptr) == (s.solver_order == 2), "x0_prev2 is given exactly when solver_order is 2");
  if (!launch) return 0;
  return launch_step(cfg_unipc_kernel<true>, cfg_unipc_kernel<false>, s.emulate_bf16, stream, a, s, st);
}

int cfg_step_run(const StepArgs& a, const d4d_pndm_sched& s, const SolverState& st, cudaStream_t stream, bool launch) {
  if (int rc = check_step(a, s.timesteps_table, s.coefs, s.n_steps, s.prediction_type, &st)) return rc;
  D4D_REQUIRE(st.ets[0] && st.ets[1] && st.ets[2] && st.ets[3] && st.cur_sample, "null argument");
  D4D_REQUIRE(s.prediction_type <= 1, "PNDM's prediction_type must be 0 (epsilon) or 1 (v_prediction)");
  if (!launch) return 0;
  return launch_step(cfg_pndm_kernel<true>, cfg_pndm_kernel<false>, s.emulate_bf16, stream, a, s, st);
}

int cfg_step_run(const StepArgs& a, const d4d_deis_sched& s, const SolverState& st, cudaStream_t stream, bool launch) {
  if (int rc = check_step(a, s.timesteps_table, s.coefs, s.n_steps, s.prediction_type, &st)) return rc;
  D4D_REQUIRE(s.solver_order >= 1 && s.solver_order <= 3, "solver_order must be 1, 2 or 3");
  D4D_REQUIRE(st.m_prev != nullptr, "null argument");
  D4D_REQUIRE((st.m_prev2 != nullptr) == (s.solver_order == 3), "m_prev2 is given exactly when solver_order is 3");
  if (!launch) return 0;
  return launch_step(cfg_deis_kernel<true>, cfg_deis_kernel<false>, s.emulate_bf16, stream, a, s, st);
}

int cfg_step_run(const StepArgs& a, const d4d_dpm_single_sched& s, const SolverState& st, cudaStream_t stream,
                 bool launch) {
  if (int rc = check_step(a, s.timesteps_table, s.coefs, s.n_steps, s.prediction_type, &st)) return rc;
  D4D_REQUIRE(s.solver_order >= 1 && s.solver_order <= 3, "solver_order must be 1, 2 or 3");
  D4D_REQUIRE(st.x0_prev != nullptr && st.cur_sample != nullptr, "null argument");
  D4D_REQUIRE((st.x0_prev2 != nullptr) == (s.solver_order == 3), "x0_prev2 is given exactly when solver_order is 3");
  if (!launch) return 0;
  return launch_step(cfg_dpm_single_kernel<true>, cfg_dpm_single_kernel<false>, s.emulate_bf16, stream, a, s, st);
}

int cfg_step_run(const StepArgs& a, const d4d_ddpm_sched& s, const SolverState& st, cudaStream_t stream, bool launch) {
  if (int rc = check_step(a, s.timesteps_table, s.coefs, s.n_steps, s.prediction_type, nullptr)) return rc;
  D4D_REQUIRE(st.frame_ids != nullptr, "null argument");
  const auto aligned8 = [](const void* p) { return reinterpret_cast<uintptr_t>(p) % 8 == 0; };
  D4D_REQUIRE(aligned8(a.noise) && aligned8(a.latents) && aligned8(a.out),
              "the DDPM step needs 8-byte aligned noise, latents and output");
  if (!launch) return 0;
  // a thread steps four elements: a grid sized by the quads of a frame, not its elements
  dim3 grid(min(64, blocks_for(a.chw / 4, 256)), a.F);
  (s.emulate_bf16 ? cfg_ddpm_kernel<true> : cfg_ddpm_kernel<false>)<<<grid, 256, 0, stream>>>(a, s, st);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int ddpm_noise_run(unsigned long long seed, const long long* frame_ids, const long long* ts_idx, int F, int hw, float* out,
                   cudaStream_t stream) {
  D4D_REQUIRE(frame_ids && ts_idx && out, "null argument");
  D4D_REQUIRE(F > 0 && hw > 0, "the frame count and latent size must be positive");
  dim3 grid(min(64, blocks_for(hw, 256)), F);
  ddpm_noise_kernel<<<grid, 256, 0, stream>>>(seed, frame_ids, ts_idx, hw, out);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace d4d
