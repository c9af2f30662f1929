// Internal kernel-launcher interface shared by the op-level C-ABI (d4d_api.cu) and the UNet
// executor (unet.cu).  Every launcher returns 0 on success, non-zero after d4d::set_error().
#pragma once
#include <cstdlib>
#include <mutex>
#include <utility>
#include <string.h>

#include "common.cuh"

namespace d4d {

// --------------------------------------------------------------------------------------------
// wgmma GEMM / implicit-GEMM conv3x3  (gemm_wgmma.cu)
// --------------------------------------------------------------------------------------------
// fixed-point scales of the fused GroupNorm statistics: |sum| < 2^35 (|x| <= 2e6 over 16384 pixels), sum of squares < 2^39
// (rms |x| <= 5800 over 16384 pixels); resolutions 3.7e-9 / 6e-8 per 16-row partial
constexpr float kGnSumScale = 268435456.f;  // 2^28
constexpr float kGnSqScale = 16777216.f;    // 2^24

struct GemmKernelArgs {
  int M, N, k_blocks, block_n, n_tiles, m_tiles;
  int mode;      // 0 plain, 1 implicit-GEMM convolution over NHWC (tap table below; TMA zero fill = padding)
  int kb_split;  // plain: k-blocks served by A (rest by A2)
  int H, W, n_img, Cin, cin_blocks, BW, BH, BN, tiles_x, tiles_y;  // H, W: the grid of output positions the tiles walk
  // conv: tap t reads input pixel (y * in_stride + tap_dy[t], x * in_stride + tap_dx[t]) for output position (y, x); the
  // result goes to output pixel (y * out_sy + out_oy, x * out_sx + out_ox) of an [n_img, out_H, out_W, ldo] tensor.
  //   3x3 / pad 1:            9 taps (-1..1), strides 1
  //   3x3 / stride 2 / pad 1: 9 taps (-1..1), in_stride 2 (the tensor map skips every other pixel)   [Downsample2D]
  //   nearest x2 + 3x3:       four 2x2 sub-pixel phases on the LOW-resolution input, out stride 2     [Upsample2D]
  int n_taps, in_stride, out_sy, out_sx, out_oy, out_ox, out_H, out_W;
  int n_phases, tiles_per_phase;  // 4: all sub-pixel phases in ONE launch (phase = m_tile / tiles_per_phase; weights [4][N][4][Cin])
  signed char tap_dy[9], tap_dx[9];
  const float* bias;  // [N] fp32 or null
  const bf16* rowvec; // [images, ld_rowvec] bf16 or null (added to every row of image row/rows_per_image)
  int ld_rowvec, rows_per_image;
  const bf16* residual;
  int ld_res;
  bf16* out;
  int ldo;
  int geglu;
  int act;          // 0 none, 1 SiLU applied to (acc + bias + rowvec) before scale/residual
  float out_scale;  // multiplies (acc + bias + rowvec) after the activation
  // fused GroupNorm statistics of the OUTPUT tensor: per (image, column) sum and sum of squares in 64-bit FIXED POINT
  // (kGnSumScale / kGnSqScale), accumulated with red.global.add.u64 into stats[(image * N + column) * 2 + {0, 1}] (zeroed by
  // the caller); image = row / stats_rows.  Integer adds commute, so the result does not depend on the order in which the
  // tiles finish: repeated forwards and the frame-sharded window stay bit-identical (float atomics would not).
  long long* stats;
  int stats_rows;
  // fused K/V all-gather (frame-sharded window): columns >= kv_col0 are stored into every rank's gathered buffer
  int kv_world, kv_col0, kv_ld;
  long long kv_rows_local, kv_rows_global, kv_row_offset;
  bf16* kv_dst[8];
};

struct GemmDesc {
  // plain: A [M, K1] (lda), optional second source A2 [M, K2] (lda2) concatenated along K
  const bf16* A = nullptr;
  int lda = 0, K1 = 0;
  const bf16* A2 = nullptr;
  int lda2 = 0, K2 = 0;
  const bf16* Wt = nullptr;  // [N, K] row-major (K contiguous); conv: [N][9][Cin]
  int M = 0, N = 0;
  const float* bias = nullptr;
  const bf16* rowvec = nullptr;
  int ld_rowvec = 0, rows_per_image = 0;
  const bf16* residual = nullptr;
  int ld_res = 0;
  bf16* out = nullptr;
  int ldo = 0;
  int geglu = 0;
  int act = 0;
  float out_scale = 1.0f;
  int block_n = 0;  // 0 = auto (64, 128 or 256; the last N tile may overhang)
  // GroupNorm statistics of the output (see GemmKernelArgs::stats); plain GEMM: stats_rows = rows per image
  long long* stats = nullptr;
  int stats_rows = 0;
  // fused K/V all-gather: rows of CFG half h (local row / kv_rows_local) land at global row
  // h*kv_rows_global + kv_row_offset + (local row % kv_rows_local) of every kv_dst[r] (leading dim kv_ld)
  int kv_world = 0, kv_col0 = 0, kv_ld = 0;
  long long kv_rows_local = 0, kv_rows_global = 0, kv_row_offset = 0;
  bf16* kv_dst[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  // conv: A is NHWC [n_img, H, W, Cin]; Wt [N][taps][Cin]
  int conv = 0, n_img = 0, H = 0, W = 0, Cin = 0;
  // conv_kind: 0 = 3x3 stride 1 pad 1 (output H x W);  1 = 3x3 stride 2 pad 1 (output H/2 x W/2);
  //            2 = one sub-pixel phase (up_a, up_b) of "nearest x2 upsample, then 3x3 pad 1": 4 taps on the H x W input with
  //                pre-summed weights (Wt [N][4][Cin]), written to pixels (2y + up_a, 2x + up_b) of the 2H x 2W output
  //            3 = all four phases in one launch (Wt [4 phases = a*2+b][N][4][Cin]): 4x the tiles, no wave quantisation per phase
  int conv_kind = 0, up_a = 0, up_b = 0;
};

struct GemmLaunch {
  CUtensorMap tmap_a, tmap_a2, tmap_b;
  GemmKernelArgs args;
  int grid;
};

int gemm_prepare(const GemmDesc& d, GemmLaunch* L);
int gemm_run(const GemmLaunch& L, cudaStream_t stream);
double gemm_flops(const GemmLaunch& L);

// --------------------------------------------------------------------------------------------
// wgmma flash attention forward (attention_wgmma.cu)
//   q/k/v are column slices of one row-major [tokens, ld] bf16 matrix (the fused QKV GEMM output);
//   head hd of batch b covers rows [b*S, (b+1)*S) and columns [hd*D, (hd+1)*D) of each slice.
// --------------------------------------------------------------------------------------------
struct AttnDesc {
  const bf16* q = nullptr;
  const bf16* k = nullptr;
  const bf16* v = nullptr;
  int ld_qkv = 0;
  bf16* out = nullptr;  // [tokens, ld_out]
  int ld_out = 0;
  int batch = 0, seq = 0, heads = 0, head_dim = 0;
  int seq_kv = 0;     // keys/values per batch entry (0 = seq); k/v rows of batch b start at b*seq_kv
  int ld_kv = 0;      // leading dimension of the k/v matrix (0 = ld_qkv)
  float scale = 0.f;  // softmax scale (head_dim^-0.5)
};
struct AttnLaunch {
  CUtensorMap tmap_q, tmap_k, tmap_v;
  AttnDesc d;
  int grid_x, grid_y;
  int variant;
};
int attn_prepare(const AttnDesc& d, AttnLaunch* L);
int attn_run(const AttnLaunch& L, cudaStream_t stream);
double attn_flops(const AttnDesc& d);

// --------------------------------------------------------------------------------------------
// HBM-bound kernels (norm.cu, elementwise.cu)
// --------------------------------------------------------------------------------------------
// GroupNorm over NHWC tokens [n_img, hw, C1 (+C2)] (optional virtual channel concat of two sources),
// fused affine + optional SiLU; writes bf16 [n_img*hw, C1+C2].  scratch: groupnorm_scratch_floats(n_img, groups) floats,
// zero-initialised once (slab partials | final mean/rstd | self-resetting arrival counters).
int groupnorm_splits(int hw);
inline size_t groupnorm_scratch_floats(int n_img, int groups) {
  return static_cast<size_t>(n_img) * 32 * groups * 2 + static_cast<size_t>(n_img) * groups * 2 + n_img + 16;
}
int groupnorm_run(const bf16* x1, int C1, const bf16* x2, int C2, int n_img, int hw, int groups, float eps,
                  const float* gamma, const float* beta, int silu, bf16* out, float* partials, cudaStream_t stream);
// Same normalisation with the statistics taken from the per-(image, channel) {sum, sum of squares} arrays that the
// producing GEMM / conv epilogue accumulated (GemmDesc::stats): one launch, one read of x, no statistics pass.
// stats1: [n_img][C1][2], stats2: [n_img][C2][2] (null when C2 == 0), fixed point (kGnSumScale, kGnSqScale).
int groupnorm_apply_run(const bf16* x1, int C1, const long long* stats1, const bf16* x2, int C2, const long long* stats2, int n_img,
                        int hw, int groups, float eps, const float* gamma, const float* beta, int silu, bf16* out,
                        cudaStream_t stream);
// LayerNorm over rows of width C (C % 8 == 0, C <= 2048)
int layernorm_run(const bf16* x, int rows, int C, float eps, const float* gamma, const float* beta, bf16* out,
                  cudaStream_t stream);

// sinusoidal embedding (flip_sin_to_cos / freq_shift) of integer/real positions -> bf16 [n, dim]
int sinusoid_run(const float* pos, int n, int dim, int flip, float freq_shift, bf16* out, cudaStream_t stream);
int sinusoid_i64_run(const long long* pos, int n, int dim, int flip, float freq_shift, bf16* out, cudaStream_t stream);
int silu_run(const bf16* x, long long n, bf16* out, cudaStream_t stream);
// im2col of an NCHW tensor for a 3x3 pad-1 conv: out[pixel, tap*cin_pad + c] zero-padded to KP columns
int im2col_nchw_run(const bf16* x, int n, int Cin, int H, int W, int cin_pad, int KP, bf16* out, cudaStream_t stream);
// [n*hw, ld] (first C columns) -> NCHW [n, C, hw]
int nhwc_to_nchw_run(const bf16* x, int ld, int n, int C, int hw, bf16* out, cudaStream_t stream);
// pose encoder layer 0: NCHW [n,3,H,W] -> NHWC [n,H,W,4] (channel 3 = 0), 3x3 pad 1 + SiLU; w [9][3][3] (tap, cin, cout)
int pose_conv0_run(const bf16* x_nchw, int n, int H, int W, const bf16* w, const float* bias, bf16* out_nhwc4,
                   cudaStream_t stream);
// pose encoder layers 1-4 on mma.sync: NHWC in / out, pad 1 + SiLU; w [Cout][k*k*Cin + 8] (K index = tap*Cin + c, zero pad)
int pose_conv_run(const bf16* x, int n, int Cin, int H, int W, const bf16* w, const float* bias, int Cout, int ksize,
                  int stride, bf16* out_nhwc, cudaStream_t stream);
// generic NHWC im2col, pad 1: [n,H,W,C] -> [n*Ho*Wo, k*k*C]
int im2col_nhwc_run(const bf16* x, int n, int H, int W, int C, int ksize, int stride, bf16* out, cudaStream_t stream);

// a-1 input assembly (pipeline_diffuman4d.py:373-395), writes NCHW [2F or F, Cin, h, w] + timesteps
struct AssembleArgs {
  bf16* latents;            // [F,4,h,w]  (cond frames are overwritten in place like the reference)
  const bf16* pixel;        // [F,4,h,w]
  const bf16* plucker;      // [F,6,h,w]
  const bf16* skel_latents; // [F,4,h,w] or null (only when the pose encoder is disabled)
  const bf16* mask;         // [F,1,h,w]
  const long long* timestep_indices;  // [F] (device)
  const long long* timesteps_table;   // [n_steps] (device)
  int n_steps;
  int F, h, w, cfg;
  bf16* sample;             // out [(cfg?2:1)*F, Cin, h, w]
  long long* timestep_out;  // out [(cfg?2:1)*F]
};
int assemble_input_run(const AssembleArgs& a, cudaStream_t stream);

// a-13 + a-14: CFG combine + per-frame DDIM step (pipeline_diffuman4d.py:408-423)
struct DdimArgs {
  const bf16* noise;        // [(cfg?2:1)*F,4,h,w]
  const bf16* latents;      // [F,4,h,w]
  const bf16* mask;         // [F,1,h,w]  (cond frame <=> mask[f,0,0,0]==0)
  const long long* timestep_indices;  // [F]
  const long long* timesteps_table;   // [n_steps]
  const float* alphas_cumprod;        // [T]
  int n_steps, T;
  float final_alpha_cumprod;
  int F, chw, hw, cfg;
  float guidance;
  int prediction_type;      // 0 epsilon, 1 v_prediction, 2 sample
  int clip_sample;
  float clip_range;
  int emulate_bf16;         // 1: round after every op like the reference's bf16 eager arithmetic
  bf16* out;                // [F,4,h,w]
};
// ts_out[F]: updated timestep indices (targets +1, cond 0); may not alias a.timestep_indices
int cfg_ddim_step_run(const DdimArgs& a, long long* ts_out, cudaStream_t stream);

// cross-rank K/V arrival flags (frame-sharded window): signal = system-scope release of `epoch` into slot `my_rank` of
// every rank's flag array; wait = acquire-spin until all `world` slots of the local array reach `epoch`
struct KvFlagArgs {
  unsigned int* flags[8];  // flags[r] = rank r's array (peer mapped); flags[my_rank] is local
  int rank, world;
  unsigned int epoch;
  int slot;                // parity slot: arrays are [2][8]
};
int kv_signal_run(const KvFlagArgs& a, cudaStream_t stream);
int kv_wait_run(const KvFlagArgs& a, cudaStream_t stream);

// per-device "opt in to large dynamic smem" helper.  `once` holds one flag per device ordinal; the reference drives one
// pipeline per GPU from its own thread (sampling_runner.py:36-43), so the first launches may race: std::call_once.
struct PerDeviceOnce {
  std::once_flag flag[64];
};
template <typename F>
inline int ensure_dyn_smem(F func, int bytes, PerDeviceOnce& once) {
  int dev = 0;
  D4D_CUDA_OK(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return 0;
  cudaError_t err = cudaSuccess;
  std::call_once(once.flag[dev], [&] { err = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes); });
  D4D_CUDA_OK(err);
  return 0;
}

// Programmatic dependent launch: the kernel may become resident while its predecessor in the stream drains; it must
// execute pdl_wait() (common.cuh) before touching anything a predecessor wrote.  The attribute is left off (serialised
// launches): the kernels of a forward are long enough that launch gaps do not show.
inline bool pdl_enabled() { return false; }
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

}  // namespace d4d
