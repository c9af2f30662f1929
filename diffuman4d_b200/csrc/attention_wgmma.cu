// Warpgroup-MMA (wgmma) flash-attention forward for sm_90a (no mask, non-causal; the only attention on the path).
//
//   O[b, i, h, :] = softmax_j(scale * Q[b,i,h,:] . K[b,j,h,:]) V[b,j,h,:]
//
// Replaces F.scaled_dot_product_attention as called by diffusers' AttnProcessor2_0 for attn1 (3-D: the tokens of all F
// frames of one CFG half form ONE sequence, reference src/diffusers/models/attention.py:68-83) and attn2 (per-image).
// Q/K/V are read in place from the fused QKV-GEMM output [tokens, 3C] through strided TMA boxes, so
// "(b t) hw c -> b (t hw) c" and the head split are address arithmetic only.
//
// One CTA = 128 query rows of one (batch, head); head_dim D = 64 NB (64, 128 or 192), K/V tiles of 64 keys.
//   warps 0-7  two MMA warpgroups, 64 query rows each:  S = Q K^T (wgmma, both operands K-major in shared memory),
//              online softmax in registers (exp2, running max and sum per row), O += P V (wgmma with P as the register
//              A operand - the S accumulator layout is the A fragment layout - and V MN-major in shared memory)
//   warp  8    TMA producer: Q once, then K_j | V_j into a ring of stages
// The two warpgroups run out of step, so one's softmax overlaps the other's MMAs; at head_dim 64 two CTAs share an SM.
#include <math.h>

#include "kernels.h"
#include "wgmma.cuh"

namespace d4d {

namespace {

constexpr int BLOCK_Q = 128;
constexpr int BLOCK_KV = 64;
constexpr int ATT_THREADS = 288;
constexpr int QBOX_BYTES = BLOCK_Q * 64 * 2;   // one [128 rows][64 ch] swizzled box
constexpr int KVBOX_BYTES = BLOCK_KV * 64 * 2;  // one [64 keys][64 ch] swizzled box

template <int NB>
struct AttCfg {
  static constexpr int D = 64 * NB;
  static constexpr int STAGES = NB == 3 ? 3 : 4;
  static constexpr int Q_BYTES = QBOX_BYTES * NB;
  static constexpr int STAGE_BYTES = 2 * KVBOX_BYTES * NB;  // K boxes, then V boxes
  static constexpr int SMEM_BYTES = 1024 + Q_BYTES + STAGES * STAGE_BYTES + 256;
  static constexpr int MIN_BLOCKS = NB == 1 ? 2 : 1;
};

struct AttKernelArgs {
  int seq_q, seq_kv, heads, n_kv_tiles;
  float scale_log2;
  bf16* out;
  int ld_out;
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int NB>
__global__ void __launch_bounds__(ATT_THREADS, AttCfg<NB>::MIN_BLOCKS)
attn_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                  const __grid_constant__ CUtensorMap tmap_v, const AttKernelArgs a) {
  using C = AttCfg<NB>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* ring = smem + C::Q_BYTES;
  uint64_t* kv_full = reinterpret_cast<uint64_t*>(ring + C::STAGES * C::STAGE_BYTES);  // [STAGES]
  uint64_t* kv_empty = kv_full + C::STAGES;                                              // [STAGES]
  uint64_t* q_full = kv_empty + C::STAGES;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);  // role branches are warp-uniform
  const int lane = threadIdx.x & 31;
  const int q_tile = blockIdx.x;
  const int bh = blockIdx.y;
  const int b = bh / a.heads;
  const int hd = bh - b * a.heads;
  const int q_row0 = b * a.seq_q;    // first query-token row of this batch
  const int kv_row0 = b * a.seq_kv;  // first key/value-token row of this batch
  const int col0 = hd * C::D;        // first column of this head inside the q/k/v slice
  const int n_tiles = a.n_kv_tiles;

  if (threadIdx.x == 0) {
    for (int i = 0; i < C::STAGES; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 2);  // one arrival per MMA warpgroup
    }
    mbar_init(q_full, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      tma_prefetch_desc(&tmap_q);
      tma_prefetch_desc(&tmap_k);
      tma_prefetch_desc(&tmap_v);
      mbar_expect_tx(q_full, C::Q_BYTES);
#pragma unroll
      for (int nb = 0; nb < NB; ++nb)
        tma_load_2d(sQ + nb * QBOX_BYTES, &tmap_q, q_full, col0 + nb * 64, q_row0 + q_tile * BLOCK_Q);
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < n_tiles; ++j) {
        mbar_wait(&kv_empty[stage], phase ^ 1);
        uint8_t* dst = ring + stage * C::STAGE_BYTES;
        mbar_expect_tx(&kv_full[stage], C::STAGE_BYTES);
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) {
          tma_load_2d(dst + nb * KVBOX_BYTES, &tmap_k, &kv_full[stage], col0 + nb * 64, kv_row0 + j * BLOCK_KV);
          tma_load_2d(dst + (NB + nb) * KVBOX_BYTES, &tmap_v, &kv_full[stage], col0 + nb * 64, kv_row0 + j * BLOCK_KV);
        }
        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ===================== MMA warpgroups =====================
  const int wg = warp >> 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const int c_base = 2 * (lane & 3);
  const uint32_t q_addr = smem_u32(sQ) + wg * 64 * 128;  // this warpgroup's 64 rows of each Q box
  const uint32_t ring_u32 = smem_u32(ring);

  float o[NB][32];
#pragma unroll
  for (int nb = 0; nb < NB; ++nb)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[nb][i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};  // running row max of scale * log2(e) * S
  float l_run[2] = {0.f, 0.f};              // this thread's share of the row sums
  mbar_wait(q_full, 0);

  int stage = 0;
  uint32_t phase = 0;
  for (int j = 0; j < n_tiles; ++j) {
    mbar_wait(&kv_full[stage], phase);
    const uint32_t kv = ring_u32 + stage * C::STAGE_BYTES;
    float s[32];
    wgmma_fence();
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) {
      const uint64_t qd = make_wgmma_desc(q_addr + nb * QBOX_BYTES, 16, 1024);
      const uint64_t kd = make_wgmma_desc(kv + nb * KVBOX_BYTES, 16, 1024);
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_ss_n64(s, qd + 2 * k, kd + 2 * k, (nb | k) != 0 ? 1 : 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);

    // keys past the end of this batch entry's sequence (last tile) do not take part
    const int valid = a.seq_kv - j * BLOCK_KV;
    if (valid < BLOCK_KV) {
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (8 * (i >> 2) + c_base + (i & 1) >= valid) s[i] = -INFINITY;
    }
    float corr[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx * a.scale_log2);
      corr[h] = ex2_approx(m_run[h] - m_new);  // 0 on the first tile (m_run = -inf)
      m_run[h] = m_new;
      float sum = 0.f;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float p = ex2_approx(fmaf(s[4 * jj + 2 * h + e], a.scale_log2, -m_new));
          s[4 * jj + 2 * h + e] = p;
          sum += p;
        }
      }
      l_run[h] = l_run[h] * corr[h] + sum;
    }
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[nb][i] *= corr[(i >> 1) & 1];

    // P (bf16) as the A operand: k-chunk kk = S fragments 2kk, 2kk+1
    uint32_t pf[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      pf[kk][0] = pack_bf16x2(s[8 * kk + 0], s[8 * kk + 1]);
      pf[kk][1] = pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]);
      pf[kk][2] = pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]);
      pf[kk][3] = pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7]);
    }
    wgmma_fence();
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) {
      // V box nb: [64 keys][64 channels], channels contiguous = MN-major B; 8-key groups 1024 B apart, 16 keys = 2048 B
      const uint64_t vd = make_wgmma_desc(kv + (NB + nb) * KVBOX_BYTES, KVBOX_BYTES, 1024);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_rs_n64_bmn(o[nb], pf[kk], vd + (2048 >> 4) * kk);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) wgmma_fence_regs(o[nb]);
    if (wg_leader) mbar_arrive(&kv_empty[stage]);
    if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
  }

  // ---- O / l -> bf16
  const int r_base = q_tile * BLOCK_Q + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv_l = 1.f / l;
    const int qrow = r_base + 8 * h;
    if (qrow >= a.seq_q) continue;
    bf16* orow = a.out + static_cast<size_t>(q_row0 + qrow) * a.ld_out + col0;
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(orow + nb * 64 + 8 * jj + c_base) =
            pack_bf16x2(o[nb][4 * jj + 2 * h] * inv_l, o[nb][4 * jj + 2 * h + 1] * inv_l);
  }
}

template <int NB>
int launch_attn(const AttnLaunch& L, cudaStream_t stream) {
  using C = AttCfg<NB>;
  static PerDeviceOnce attr_once;
  if (int rc = ensure_dyn_smem(attn_wgmma_kernel<NB>, C::SMEM_BYTES, attr_once)) return rc;
  AttKernelArgs a;
  a.seq_q = L.d.seq;
  a.seq_kv = L.d.seq_kv > 0 ? L.d.seq_kv : L.d.seq;
  a.heads = L.d.heads;
  a.n_kv_tiles = (a.seq_kv + BLOCK_KV - 1) / BLOCK_KV;
  a.scale_log2 = L.d.scale * 1.4426950408889634f;
  a.out = L.d.out;
  a.ld_out = L.d.ld_out;
  dim3 grid(L.grid_x, L.grid_y);
  D4D_CUDA_OK(launch_pdl(attn_wgmma_kernel<NB>, grid, dim3(ATT_THREADS), C::SMEM_BYTES, stream, L.tmap_q, L.tmap_k, L.tmap_v, a));
  D4D_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace

int attn_prepare(const AttnDesc& d, AttnLaunch* L) {
  D4D_REQUIRE(d.head_dim == 64 || d.head_dim == 128 || d.head_dim == 192,
              "attention head_dim (after padding) must be 64, 128 or 192");
  D4D_REQUIRE(d.batch > 0 && d.seq > 0 && d.heads > 0 && d.seq_kv >= 0, "empty attention problem");
  D4D_REQUIRE(d.ld_qkv % 8 == 0 && d.ld_out % 8 == 0 && d.ld_kv % 8 == 0, "leading dimensions must be multiples of 8");
  D4D_REQUIRE(d.scale > 0.f, "softmax scale must be positive");
  L->d = d;
  L->variant = d.head_dim / 64;
  const int seq_kv = d.seq_kv > 0 ? d.seq_kv : d.seq;
  const int ld_kv = d.ld_kv > 0 ? d.ld_kv : d.ld_qkv;
  const uint64_t q_tokens = static_cast<uint64_t>(d.batch) * d.seq;
  const uint64_t kv_tokens = static_cast<uint64_t>(d.batch) * seq_kv;
  const uint64_t width = static_cast<uint64_t>(d.heads) * d.head_dim;
  if (int rc = make_tmap_2d(&L->tmap_q, d.q, q_tokens, width, d.ld_qkv, 64, BLOCK_Q, 128)) return rc;
  if (int rc = make_tmap_2d(&L->tmap_k, d.k, kv_tokens, width, ld_kv, 64, BLOCK_KV, 128)) return rc;
  if (int rc = make_tmap_2d(&L->tmap_v, d.v, kv_tokens, width, ld_kv, 64, BLOCK_KV, 128)) return rc;
  L->grid_x = (d.seq + BLOCK_Q - 1) / BLOCK_Q;
  L->grid_y = d.batch * d.heads;
  D4D_REQUIRE(L->grid_y <= 65535, "batch*heads exceeds grid.y limit");
  return 0;
}

int attn_run(const AttnLaunch& L, cudaStream_t stream) {
  switch (L.variant) {
    case 1: return launch_attn<1>(L, stream);
    case 2: return launch_attn<2>(L, stream);
    case 3: return launch_attn<3>(L, stream);
  }
  set_error("attention: unsupported head_dim variant");
  return 1;
}

double attn_flops(const AttnDesc& d) {
  const double skv = d.seq_kv > 0 ? d.seq_kv : d.seq;
  return 4.0 * d.batch * d.heads * static_cast<double>(d.seq) * skv * d.head_dim;
}

}  // namespace d4d
