// Internal kernel-launcher interface shared by the op-level C-ABI (d4d_api.cu) and the UNet
// executor (unet.cu).  Every launcher returns 0 on success, non-zero after d4d::set_error().
#pragma once
#include <cstdlib>
#include <mutex>
#include <utility>
#include <string.h>

#include "../../include/d4d.h"
#include "common.cuh"

namespace d4d {

// --------------------------------------------------------------------------------------------
// wgmma GEMM / implicit-GEMM conv3x3  (gemm_wgmma.cu)
// --------------------------------------------------------------------------------------------
// fixed-point scales of the GroupNorm statistics (GEMM / conv epilogue, groupnorm_stats_run): |sum| < 2^35 (|x| <= 2e6
// over 16384 pixels), sum of squares < 2^39 (rms |x| <= 5800 over 16384 pixels); resolutions 3.7e-9 / 6e-8 per 16-row partial
constexpr float kGnSumScale = 268435456.f;  // 2^28
constexpr float kGnSqScale = 16777216.f;    // 2^24

struct GemmKernelArgs {
  int M, N, k_blocks, block_n, n_tiles, m_tiles;
  int block_m;   // tile rows: 128, or 256 (conv; each MMA warpgroup owns two 64-row blocks)
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
  // plain GEMM: the MMA warpgroups stage the output tile in shared memory and TMA stores it (tmap_c); the residual tile
  // arrives by TMA into the same buffer (tmap_r).  0: stores from registers (conv, K/V scatter, narrow block_n)
  int staged;
  int pingpong;  // staged plain GEMM on the ping-pong schedule: each MMA warpgroup owns every other 128-row tile
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
  int block_n = 0;  // 0 = auto (64, 128, 160, 192 or 256; the last N tile may overhang)
  int block_m = 0;  // 0 = auto, 128, or 256 (conv at block_n 128 / 160 only)
  // plain GEMM: 0 = auto, kSchedCooperative, or kSchedPingPong (block_n 64 or 128; GEGLU 128; staged epilogue only)
  int schedule = 0;
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
  CUtensorMap tmap_a, tmap_a2, tmap_b, tmap_c, tmap_r;  // tmap_c / tmap_r: output / residual of a staged epilogue
  GemmKernelArgs args;
  int grid;
};

constexpr int kSchedCooperative = 1, kSchedPingPong = 2;
// the tile rows, width and schedule gemm_prepare runs d at on a device of `sms` SMs (shape fields and block_m / block_n /
// schedule only; `schedule` may be null).  Ping-pong is chosen on shape alone: gemm_prepare runs a launch that cannot
// stage its epilogue cooperatively.
int gemm_choose_tile(const GemmDesc& d, int sms, int* block_m, int* block_n, int* schedule = nullptr);
// whether the epilogue of d can accumulate the GroupNorm statistics of its output (GemmDesc::stats) on a device of `sms`
// SMs: every 32-row warp of the tile gemm_choose_tile picks stays inside one image (plain GEMM: stats_rows % 32 == 0 and
// M % stats_rows == 0).  Shape fields only; `why` (may be null) gets the reason when not.  gemm_prepare refuses stats
// otherwise.
bool gemm_stats_fusable(const GemmDesc& d, int sms, const char** why = nullptr);
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
// GroupNorm statistics of an NHWC tensor [n_img, hw, C] in the format the GEMM / conv epilogue writes (GemmDesc::stats):
// per-(image, channel) {sum, sum of squares}, fixed point (kGnSumScale, kGnSqScale), added into stats [n_img][C][2],
// which the caller zeroes.  For tensors whose producer cannot accumulate them in its epilogue.
int groupnorm_stats_run(const bf16* x, int C, int n_img, int hw, long long* stats, cudaStream_t stream);
// GroupNorm over NHWC tokens [n_img, hw, C1 (+C2)] (optional virtual channel concat of two sources), fused affine +
// optional SiLU; writes bf16 [n_img*hw, C1+C2].  The group (mean, rstd) come from the statistics of each source
// (stats1: [n_img][C1][2], stats2: [n_img][C2][2], null when C2 == 0): one launch, one read of x.  32 <= C1 + C2 <= 4096.
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
// the same permute storing the same NCHW tensor into every p[i], i < n (the CFG-split window stores its half of the noise
// into every rank's exchange buffer, peer memory mapped with cudaIpc, like the K/V scatter epilogue)
struct NchwDst {
  bf16* p[8];
  int n;
};
int nhwc_to_nchw_run(const bf16* x, int ld, int n, int C, int hw, const NchwDst& out, cudaStream_t stream);
// pose encoder layer 0: NCHW [n,3,H,W] -> NHWC [n,H,W,4] (channel 3 = 0), 3x3 pad 1 + SiLU; w [9][3][3] (tap, cin, cout)
int pose_conv0_run(const bf16* x_nchw, int n, int H, int W, const bf16* w, const float* bias, bf16* out_nhwc4,
                   cudaStream_t stream);
// pose encoder layers 1-4 on mma.sync: NHWC in / out, pad 1 + SiLU; w [Cout][k*k*Cin + 8] (K index = tap*Cin + c, zero pad)
int pose_conv_run(const bf16* x, int n, int Cin, int H, int W, const bf16* w, const float* bias, int Cout, int ksize,
                  int stride, bf16* out_nhwc, cudaStream_t stream);
// generic NHWC im2col, pad 1: [n,H,W,C] -> [n*Ho*Wo, k*k*C]
int im2col_nhwc_run(const bf16* x, int n, int H, int W, int C, int ksize, int stride, bf16* out, cudaStream_t stream);
// [1 + n_pos images of per_img elements] -> [n_neg + n_pos images]: images 0..n_neg-1 <- small image 0, images
// n_neg..n_neg+n_pos-1 <- small images 1..n_pos (per_img % 8 == 0)
int broadcast_neg_images_run(const bf16* small, long long per_img, int n_neg, int n_pos, bf16* full, cudaStream_t stream);
// p[0 .. n) = v
int fill_bf16_run(bf16* p, long long n, float v, cudaStream_t stream);

// a-1 input assembly (pipeline_diffuman4d.py:373-395), writes NCHW [2F or F, Cin, h, w] + timesteps
struct AssembleArgs {
  // -1: the whole batch, (cfg ? 2 : 1) * F images; 0 / 1: only CFG half k's F images (0 negative, 1 positive) at rows
  // [0, F), the rows the whole batch has at [k*F, (k+1)*F) (cfg is then not read).  Every mode overwrites the cond frames'
  // latents in place alike.
  int half = -1;
  // with a half and n_f > 0: only frames [f0, f0 + n_f) get sample rows, at rows [0, n_f) (a frame shard of the CFG
  // grid); the cond frames of all F frames are still overwritten in place
  int f0 = 0, n_f = 0;
  bf16* latents;            // [F,4,h,w]  (cond frames are overwritten in place like the reference)
  const bf16* pixel;        // [F,4,h,w]
  const bf16* plucker;      // [F,6,h,w]
  const bf16* skel_latents; // [F,4,h,w] or null (only when the pose encoder is disabled)
  const bf16* mask;         // [F,1,h,w]
  const long long* timestep_indices;  // [F] (device)
  const long long* timesteps_table;   // [n_steps] (device)
  int n_steps;
  int F, h, w, cfg;
  bf16* sample;             // out [(cfg?2:1)*F, Cin, h, w]; [F, Cin, h, w] for one half
  long long* timestep_out;  // out [(cfg?2:1)*F]; [F] for one half
};
int assemble_input_run(const AssembleArgs& a, cudaStream_t stream);

// a-13 + a-14: CFG combine + per-frame scheduler step (pipeline_diffuman4d.py:408-423): DDIM, DPM-Solver++ (dpmsolver++ /
// midpoint, order <= 2), UniPC (predict_x0, bh1 / bh2, order <= 2; the UniC corrector of the frame's previous step,
// then the UniP predictor), PNDM (skip_prk_steps: the PLMS steps), DEIS (deis / logrho, order <= 3), DPM-Solver++
// singlestep (dpmsolver++ / midpoint, order <= 3) or DDPM (ancestral sampling with the counter-based noise of
// ddpm_noise.cuh).  The scheduler's constants, step count, prediction type and bf16 emulation come from its table struct
// in include/d4d.h, passed as it is; the coefficient rows of the schedulers that have them are laid out there too.
constexpr int kDpmCoefs = 6;
constexpr int kUniPCCoefs = 14;
constexpr int kPndmCoefs = 10;
constexpr int kDeisCoefs = 11;
constexpr int kDpmSingleCoefs = 13;
constexpr int kDdpmCoefs = 6;
struct StepArgs {
  const bf16* noise;        // [(cfg?2:1)*F,4,h,w]
  const bf16* latents;      // [F,4,h,w]
  const bf16* mask;         // [F,1,h,w]  (cond frame <=> mask[f,0,0,0]==0; never stepped, solver state untouched)
  const long long* timestep_indices;  // [F] = the step index of each frame
  int F, chw, hw, cfg;
  float guidance;
  bf16* out;                // [F,4,h,w] (may alias latents)
  long long* ts_out;        // [F] updated timestep indices (targets +1, cond 0); may not alias timestep_indices
};
// The multistep solvers' per-frame history, read and updated in place; members a scheduler does not keep are null (all
// of them for DDIM).
struct SolverState {
  bf16* x0_prev = nullptr;      // [F,4,h,w]: each frame's previous data prediction
  // [F,4,h,w]: the one before (UniPC at solver_order 2, DPM-Solver++ singlestep at solver_order 3)
  bf16* x0_prev2 = nullptr;
  bf16* last_sample = nullptr;  // [F,4,h,w]: the sample each frame's last predictor started from (UniPC)
  bf16* ets[4] = {};            // [F,4,h,w] each: the ring of PNDM's last model outputs (d4d_denoise_window_pndm)
  // [F,4,h,w]: the sample the frame's first step started from: PNDM's counter-0 step, or the order-1 step that started
  // the frame's current DPM-Solver++ singlestep block
  bf16* cur_sample = nullptr;
  bf16* m_prev = nullptr;       // [F,4,h,w]: each frame's previous DEIS model output, in its epsilon form
  bf16* m_prev2 = nullptr;      // [F,4,h,w]: the one before (DEIS at solver_order 3)
  const long long* frame_ids = nullptr;  // [F]: each frame's index in its task, DDPM's noise counter (no history)
  // [F]: steps each frame has taken, capped at solver_order (PNDM: uncapped, its `counter`)
  const int* lower_order_nums = nullptr;
  int* lower_order_nums_out = nullptr;    // [F]: the advanced counts (may not alias lower_order_nums)
};
// Each checks its arguments, then launches one kernel (launch = false: only the checks, so that a caller can refuse bad
// arguments before it enqueues the work that precedes the step).
int cfg_step_run(const StepArgs& a, const d4d_sched& s, const SolverState& st, cudaStream_t stream, bool launch = true);
int cfg_step_run(const StepArgs& a, const d4d_dpm_sched& s, const SolverState& st, cudaStream_t stream, bool launch = true);
int cfg_step_run(const StepArgs& a, const d4d_unipc_sched& s, const SolverState& st, cudaStream_t stream,
                 bool launch = true);
int cfg_step_run(const StepArgs& a, const d4d_pndm_sched& s, const SolverState& st, cudaStream_t stream,
                 bool launch = true);
int cfg_step_run(const StepArgs& a, const d4d_deis_sched& s, const SolverState& st, cudaStream_t stream,
                 bool launch = true);
int cfg_step_run(const StepArgs& a, const d4d_dpm_single_sched& s, const SolverState& st, cudaStream_t stream,
                 bool launch = true);
int cfg_step_run(const StepArgs& a, const d4d_ddpm_sched& s, const SolverState& st, cudaStream_t stream,
                 bool launch = true);
// The DDPM step's noise alone, in fp32: out [F,4,h,w] for frames frame_ids [F] at timestep indices ts_idx [F]
int ddpm_noise_run(unsigned long long seed, const long long* frame_ids, const long long* ts_idx, int F, int hw, float* out,
                   cudaStream_t stream);

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

// frame-sharded sliding loop: the updated frames of a window, gathered in every rank's exchange buffer.  Layout of the
// gathered window (F_total frames in window order, chw = 4*h*w): latents [F_total][chw] bf16 | x0_prev [F_total][chw] bf16
// (DPM-Solver++ only) | timestep indices [F_total] int64 | lower_order_nums [F_total] int32 (DPM-Solver++ only).
struct WindowResultLayout {
  size_t x0, ts, lon, bytes;  // byte offsets of the regions after the latents (at 0), and the total size
};
inline WindowResultLayout window_result_layout(long long F_total, long long chw, bool dpm) {
  WindowResultLayout L;
  const size_t rows = static_cast<size_t>(F_total) * static_cast<size_t>(chw) * 2;
  L.x0 = rows;
  L.ts = dpm ? 2 * rows : rows;
  L.lon = L.ts + static_cast<size_t>(F_total) * 8;
  L.bytes = L.lon + (dpm ? static_cast<size_t>(F_total) * 4 : 0);
  return L;
}
struct WindowScatterArgs {
  void* dst[8];              // dst[r] = rank r's gathered window (peer mapped); r < world
  int world, rank, F_local, F_total;
  long long chw;
  const bf16* latents;       // [F_local][chw], 16-byte aligned
  const long long* ts;       // [F_local]
  const bf16* x0_prev;       // [F_local][chw] or nullptr (DDIM), 16-byte aligned
  const int* lower_order_nums;  // [F_local] or nullptr, with x0_prev
};
// Stores this rank's F_local frames at rows [rank*F_local, (rank+1)*F_local) of every dst[r].  Returns 1 before any launch
// for arguments that would store outside a dst_bytes destination.
int window_scatter_run(const WindowScatterArgs& a, size_t dst_bytes, cudaStream_t stream);

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
