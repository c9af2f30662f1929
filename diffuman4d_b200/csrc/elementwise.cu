// HBM-/latency-bound helper kernels of the denoise step: embeddings, layout changes feeding the
// tensor-core kernels, the pose-encoder's small-channel convolutions, and the fused pipeline pieces
// (input assembly, CFG combine + per-frame DDIM update).  All global traffic is 128-bit where the
// layout allows it.
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

// [n*H*W, ld] (first C columns) -> NCHW [n, C, H, W]
__global__ void nhwc_to_nchw_kernel(const bf16* __restrict__ x, int ld, int n, int C, int hw, bf16* __restrict__ out) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(n) * C * hw;
  if (idx >= total) return;
  const int p = static_cast<int>(idx % hw);
  const int c = static_cast<int>((idx / hw) % C);
  const int img = static_cast<int>(idx / (static_cast<long long>(hw) * C));
  out[idx] = x[(static_cast<size_t>(img) * hw + p) * ld + c];
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
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    long long t = 0;
    if (!is_cond) {
      long long idx = a.timestep_indices[f];
      idx = idx < 0 ? 0 : (idx >= a.n_steps ? a.n_steps - 1 : idx);
      t = a.timesteps_table[idx];
    }
    a.timestep_out[f] = t;
    if (a.cfg) a.timestep_out[a.F + f] = t;
  }
  const bf16 one = __float2bfloat16_rn(1.f), zero = __float2bfloat16_rn(0.f), mone = __float2bfloat16_rn(-1.f);
  const int halves = a.cfg ? 2 : 1;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += gridDim.x * blockDim.x) {
    const bf16 m = a.mask[static_cast<size_t>(f) * hw + p];
    for (int c = 0; c < 4; ++c) {
      const size_t li = (static_cast<size_t>(f) * 4 + c) * hw + p;
      bf16 lat = a.latents[li];
      if (is_cond) {
        lat = a.pixel[li];
        a.latents[li] = lat;  // reference aliasing quirk: latents <- image latents at cond frames (PIPE:375-379)
      }
      // positive half is the LAST half when cfg (torch.cat([negative, positive]))
      const int pos_img = a.cfg ? a.F + f : f;
      a.sample[(static_cast<size_t>(pos_img) * Cin + c) * hw + p] = lat;
      if (a.cfg) a.sample[(static_cast<size_t>(f) * Cin + c) * hw + p] = is_cond ? one : lat;
    }
    int ch = 4;
    for (int c = 0; c < 6; ++c, ++ch) {
      const bf16 v = a.plucker[(static_cast<size_t>(f) * 6 + c) * hw + p];
      const int pos_img = a.cfg ? a.F + f : f;
      a.sample[(static_cast<size_t>(pos_img) * Cin + ch) * hw + p] = v;
      if (a.cfg) a.sample[(static_cast<size_t>(f) * Cin + ch) * hw + p] = zero;
    }
    if (a.skel_latents) {
      for (int c = 0; c < 4; ++c, ++ch) {
        const bf16 v = a.skel_latents[(static_cast<size_t>(f) * 4 + c) * hw + p];
        const int pos_img = a.cfg ? a.F + f : f;
        a.sample[(static_cast<size_t>(pos_img) * Cin + ch) * hw + p] = v;
        if (a.cfg) a.sample[(static_cast<size_t>(f) * Cin + ch) * hw + p] = mone;
      }
    }
    for (int hf = 0; hf < halves; ++hf)
      a.sample[(static_cast<size_t>(hf * a.F + f) * Cin + ch) * hw + p] = m;
  }
}

// images 0..F-1 <- small image 0 ; images F..2F-1 <- small images 1..F   (per_img elements each, multiple of 8)
__global__ void broadcast_neg_images_kernel(const bf16* __restrict__ small, long long per_img8, int F, bf16* __restrict__ full) {
  const long long total = per_img8 * 2 * F;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long img = i / per_img8, off = i - img * per_img8;
    const long long src = img < F ? 0 : img - F + 1;
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
// a-13 + a-14: CFG combine + per-frame DDIM step (pipeline_diffuman4d.py:408-423, upstream DDIMScheduler.step)
// ---------------------------------------------------------------------------------------------
template <bool EMU>
__device__ __forceinline__ float rnd(float x) { return EMU ? bf16_round(x) : x; }

template <bool EMU>
__global__ void cfg_ddim_kernel(const DdimArgs a, long long* ts_out) {
  const int f = blockIdx.y;
  const bool is_cond = __bfloat162float(a.mask[static_cast<size_t>(f) * a.hw]) == 0.f;
  long long idx = a.timestep_indices[f];
  if (blockIdx.x == 0 && threadIdx.x == 0) ts_out[f] = is_cond ? 0 : idx + 1;
  const size_t base = static_cast<size_t>(f) * a.chw;
  if (is_cond) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.chw; i += gridDim.x * blockDim.x)
      a.out[base + i] = a.latents[base + i];
    return;
  }
  idx = idx < 0 ? 0 : (idx >= a.n_steps ? a.n_steps - 1 : idx);
  const long long t = a.timesteps_table[idx];
  const long long prev_t = t - a.T / a.n_steps;
  const float a_t = a.alphas_cumprod[t];
  const float a_prev = prev_t >= 0 ? a.alphas_cumprod[prev_t] : a.final_alpha_cumprod;
  const float b_t = 1.0f - a_t;
  const float sa = sqrtf(a_t), sb = sqrtf(b_t);
  const float sa_prev = sqrtf(a_prev), sdir = sqrtf(1.0f - a_prev);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.chw; i += gridDim.x * blockDim.x) {
    float eps_in;
    if (a.cfg) {
      const float u = __bfloat162float(a.noise[base + i]);
      const float c = __bfloat162float(a.noise[static_cast<size_t>(a.F) * a.chw + base + i]);
      // u + g * (c - u)
      eps_in = rnd<EMU>(u + rnd<EMU>(a.guidance * rnd<EMU>(c - u)));
    } else {
      eps_in = __bfloat162float(a.noise[base + i]);
    }
    const float x = __bfloat162float(a.latents[base + i]);
    float x0, eps;
    if (a.prediction_type == 0) {        // epsilon
      x0 = rnd<EMU>(rnd<EMU>(x - rnd<EMU>(sb * eps_in)) / sa);
      eps = eps_in;
    } else if (a.prediction_type == 1) { // v_prediction
      x0 = rnd<EMU>(rnd<EMU>(sa * x) - rnd<EMU>(sb * eps_in));
      eps = rnd<EMU>(rnd<EMU>(sa * eps_in) + rnd<EMU>(sb * x));
    } else {                             // sample
      x0 = eps_in;
      eps = rnd<EMU>(rnd<EMU>(x - rnd<EMU>(sa * x0)) / sb);
    }
    if (a.clip_sample) x0 = fminf(fmaxf(x0, -a.clip_range), a.clip_range);
    const float dir = rnd<EMU>(sdir * eps);
    const float prev = rnd<EMU>(rnd<EMU>(sa_prev * x0) + dir);
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
  const long long total = static_cast<long long>(n) * C * hw;
  nhwc_to_nchw_kernel<<<blocks_for(total, 256), 256, 0, stream>>>(x, ld, n, C, hw, out);
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

int assemble_input_run(const AssembleArgs& a, cudaStream_t stream) {
  const int Cin = 4 + 6 + (a.skel_latents ? 4 : 0) + 1;
  const int hw = a.h * a.w;
  dim3 grid(min(64, blocks_for(hw, 256)), a.F);
  assemble_kernel<<<grid, 256, 0, stream>>>(a, Cin);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int broadcast_neg_images_run(const bf16* small, long long per_img, int F, bf16* full, cudaStream_t stream) {
  D4D_REQUIRE(per_img % 8 == 0 && F > 0, "broadcast_neg_images arguments");
  broadcast_neg_images_kernel<<<132 * 8, 256, 0, stream>>>(small, per_img / 8, F, full);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}
int fill_bf16_run(bf16* p, long long n, float v, cudaStream_t stream) {
  fill_bf16_kernel<<<132 * 4, 256, 0, stream>>>(p, n, v);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

int cfg_ddim_step_run(const DdimArgs& a, long long* ts_out, cudaStream_t stream) {
  D4D_REQUIRE(a.n_steps > 0 && a.T > 0 && a.F > 0, "ddim args");
  dim3 grid(min(64, blocks_for(a.chw, 256)), a.F);
  if (a.emulate_bf16) cfg_ddim_kernel<true><<<grid, 256, 0, stream>>>(a, ts_out);
  else cfg_ddim_kernel<false><<<grid, 256, 0, stream>>>(a, ts_out);
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace d4d
