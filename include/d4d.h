/* d4d.h -- C ABI of libd4d.so: the H100-native (sm_90a) replacement of the Diffuman4D denoise-step hot path.
 *
 * The reference is pure Python and has no FFI; the seams this ABI stands behind are (SURVEY.md section 8b):
 *   B-2  `pipeline.unet(sample, timestep, skeletons, domains, num_frames)`
 *        src/diffusers/pipelines/diffuman4d/pipeline_diffuman4d.py:398-405
 *        src/diffusers/models/unets/unet_multiview_condition.py:501-598      -> d4d_unet_forward
 *   B-3  one window denoise step (input assembly + UNet + CFG + per-frame scheduler step)
 *        src/diffusers/pipelines/diffuman4d/pipeline_diffuman4d.py:369-425   -> d4d_denoise_window
 *   weights: diffusers-layout state_dict keys of `unet/diffusion_pytorch_model.safetensors`
 *        (loaded by SUTIL load_pipelines, src/samplers/utils/sampling_utils.py:45-50)          -> d4d_load_weight
 * INTEGRATION.md shows the ctypes stub a maintainer of the reference would add.
 *
 * Conventions: every function returns 0 on success, 1 for invalid arguments, 2 for CUDA/driver failures,
 * 3 for "weights not finalized / missing"; d4d_last_error() returns a thread-local message.  No function
 * aborts.  All device pointers are borrowed for the duration of the call; work is enqueued on `stream`
 * (a cudaStream_t passed as void*) and NOT synchronised.  One handle per device; a handle must not be
 * entered by two threads at once (the reference drives one pipeline per GPU from its own thread,
 * src/samplers/sampling_runner.py:26-43); different handles are independent.  bf16 everywhere unless noted.
 */
#ifndef D4D_H_
#define D4D_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct d4d_handle d4d_handle;

/* Constructor knobs of UNetMultiviewConditionModel that change arithmetic on this path
 * (unet_multiview_condition.py:149-212).  Everything else is fixed to the reference defaults. */
typedef struct d4d_config {
  int32_t in_channels;            /* 11 (pose encoder) or 15 (skeleton latents concatenated) */
  int32_t out_channels;           /* 4 */
  int32_t block_out_channels[4];  /* 320, 640, 1280, 1280 */
  int32_t layers_per_block;       /* 2 */
  int32_t num_heads[4];           /* the reference's `attention_head_dim` (= number of heads) per level */
  int32_t has_attn2[4];           /* cross_attention_dim[level] is not None */
  int32_t use_linear_projection;
  int32_t norm_num_groups;        /* 32 */
  float norm_eps;                 /* 1e-5 (transformer GroupNorm is fixed at 1e-6) */
  int32_t flip_sin_to_cos;
  float freq_shift;
  int32_t num_3d_attn_blocks;     /* 3 */
  int32_t enable_tem_embeds;
  int32_t enable_pose_encoder;
  int32_t center_input_sample;
} d4d_config;

/* DDIM scheduler constants for the fused step (upstream diffusers DDIMScheduler, deep-copied per frame at
 * pipeline_diffuman4d.py:265-271). */
typedef struct d4d_sched {
  const int64_t* timesteps_table;   /* device, [n_steps]  (scheduler.timesteps after set_timesteps) */
  const float* alphas_cumprod;      /* device, [num_train_timesteps] */
  int32_t n_steps;
  int32_t num_train_timesteps;
  float final_alpha_cumprod;
  int32_t prediction_type;          /* 0 epsilon, 1 v_prediction, 2 sample */
  int32_t clip_sample;
  float clip_sample_range;
  int32_t emulate_bf16;             /* 1: round after every arithmetic op like the reference's bf16 eager maths */
} d4d_sched;

const char* d4d_last_error(void);
int d4d_version(void);

/* ---- lifecycle --------------------------------------------------------------------------------- */
int d4d_create(const d4d_config* cfg, int device, d4d_handle** out);
void d4d_destroy(d4d_handle* h);

/* Stage one parameter by its diffusers key.  `data` is a HOST pointer to a contiguous tensor of `dtype`
 * (0 = float32, 1 = bfloat16, 2 = float16) with `ndim` dims `shape`.  Unknown keys are an error. */
int d4d_load_weight(d4d_handle* h, const char* key, const void* data, const int64_t* shape, int ndim, int dtype);
/* Check completeness, re-lay-out (OIHW -> [Cout][tap][Cin], fused QKV, GEGLU interleave, ...) and upload. */
int d4d_finalize_weights(d4d_handle* h);
/* Number of expected parameter tensors and the i-th expected key (for loaders / error messages). */
int d4d_num_weights(d4d_handle* h);
const char* d4d_weight_key(d4d_handle* h, int i);

/* ---- B-2: UNet forward ---------------------------------------------------------------------------
 * sample     device bf16 NCHW [B, in_channels, h, w]
 * timestep   device int64 [B]
 * skeletons  device bf16 NCHW [B, 3, 8h, 8w] when enable_pose_encoder, else NULL
 * domain_ids HOST int32 [n_domains] with n_domains * F == B; 0 = "spatial", 1 = "temporal"
 * out        device bf16 NCHW [B, out_channels, h, w] (caller-allocated, fresh tensor)
 * h, w must be divisible by 8 (three 2x down/up-samplings; upsample_size is always None in the reference). */
int d4d_unet_forward(d4d_handle* h, const void* sample, const int64_t* timestep, const void* skeletons,
                     const int32_t* domain_ids, int n_domains, int B, int F, int height, int width, void* out,
                     void* stream);
/* Same call, but with a CUDA event around every launch; synchronises, then reports the device time (ms), launch
 * count and executed tensor-core FLOPs per kernel kind: 0 GEMM, 1 conv3x3, 2 attention, 3 GroupNorm, 4 LayerNorm,
 * 5 other.  Used by bench.py for the live roofline figures. */
int d4d_profile_forward(d4d_handle* h, const void* sample, const int64_t* timestep, const void* skeletons,
                        const int32_t* domain_ids, int n_domains, int B, int F, int height, int width, void* out,
                        void* stream, float* ms_by_kind /*[6]*/, int32_t* launches_by_kind /*[6]*/,
                        double* flops_by_kind /*[6]*/);
/* Bytes of activation workspace the plan for this shape owns (allocated lazily, kept in the handle). */
int d4d_workspace_bytes(d4d_handle* h, int n_domains, int B, int F, int height, int width, size_t* bytes);
/* Kernel launches one forward of this shape enqueues (0 if the plan does not exist yet). */
int d4d_forward_launches(d4d_handle* h, int n_domains, int B, int F, int height, int width, int* launches);

/* ---- B-3: one window denoise step (a-1 + UNet + a-13 + a-14), `num_steps` times ---------------------
 * latents [F,4,h,w] in/out (cond frames receive the image latents, reference aliasing quirk PIPE:375-379),
 * pixel_latents [F,4,h,w], plucker [F,6,h,w], skeletons [F,3,8h,8w] (pose encoder) or [F,4,h,w] (latents),
 * cond_mask [F,1,h,w] (0 = conditioning frame), timestep_indices device int64 [F] in/out.
 * guidance_scale > 1 enables classifier-free guidance (batch 2F).  domain: 0 spatial, 1 temporal. */
int d4d_denoise_window(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                       const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                       const d4d_sched* sched, float guidance_scale, int domain, int F, int height, int width,
                       int num_steps, void* stream);

/* ---- building blocks of B-3, exported for parity tests ------------------------------------------------ */
int d4d_assemble_input(void* latents, const void* pixel_latents, const void* plucker, const void* skel_latents,
                       const void* cond_mask, const int64_t* timestep_indices, const int64_t* timesteps_table,
                       int n_steps, int F, int height, int width, int cfg, void* sample_out, int64_t* timestep_out,
                       void* stream);
int d4d_cfg_ddim_step(const void* noise, const void* latents, const void* cond_mask, const int64_t* timestep_indices,
                      int64_t* timestep_indices_out, const d4d_sched* sched, float guidance_scale, int cfg, int F,
                      int height, int width, void* latents_out, void* stream);

/* ---- op-level entry points (each is one hot-path kernel; used by tests/ and bench.py) ------------------
 * d4d_op_gemm:   out[M,N] = act((A|A2)[M,K1+K2] . W[N,K]^T + bias + rowvec[row/rows_per_image]) * scale + residual
 *                geglu: W rows / bias interleaved in groups of 8 (a rows, then g rows), out is [M, N/2].
 * d4d_op_conv3x3: NHWC x [n,H,W,Cin], W [Cout][9][Cin] (tap = ky*3+kx), stride 1, pad 1.  */
int d4d_op_gemm(const void* A, int lda, int K1, const void* A2, int lda2, int K2, const void* W, int M, int N,
                const float* bias, const void* rowvec, int ld_rowvec, int rows_per_image, const void* residual,
                int ld_res, void* out, int ldo, int geglu, int act, float out_scale, int block_n, void* stream);
int d4d_op_conv3x3(const void* x_nhwc, int n_img, int H, int W, int Cin, const void* Wt, int Cout, const float* bias,
                   const void* rowvec, int ld_rowvec, const void* residual, int act, void* out, int block_n,
                   void* stream);
/* q, k, v: column slices of one row-major [batch*seq, ld_qkv] matrix; head hd = columns [hd*D, (hd+1)*D). */
int d4d_op_attention(const void* q, const void* k, const void* v, int ld_qkv, void* out, int ld_out, int batch,
                     int seq, int heads, int head_dim, float scale, void* stream);
int d4d_op_groupnorm(const void* x1, int C1, const void* x2, int C2, int n_img, int hw, int groups, float eps,
                     const float* gamma, const float* beta, int silu, void* out, void* stream);
/* The two resampling convolutions of the UNet, read / written in place (no im2col, no materialised upsampled tensor):
 *   kind 1: 3x3 stride-2 pad-1 conv (diffusers Downsample2D): x [n,H,W,Cin] -> out [n,H/2,W/2,Cout], Wt [Cout][9][Cin];
 *   kind 2: one sub-pixel phase (up_a, up_b in {0,1}) of "nearest x2 upsample, then 3x3 pad-1 conv" (Upsample2D): a 2x2 conv on
 *           the low-resolution x with pre-summed weights Wt [Cout][4][Cin] (tap = ty*2+tx; rows {-1,0} for up_a = 0, {0,+1} for
 *           up_a = 1, same for columns), written to pixels (2y+up_a, 2x+up_b) of out [n,2H,2W,Cout].  Four calls fill out;
 *   kind 3: all four phases in one launch, Wt [4 (= up_a*2+up_b)][Cout][4][Cin] (what the UNet plan uses). */
int d4d_op_conv_resample(const void* x_nhwc, int n_img, int H, int W, int Cin, const void* Wt, int Cout, const float* bias,
                         int kind, int up_a, int up_b, void* out, void* stream);
/* conv3x3 (+bias, +residual) whose epilogue accumulates the per-(image, channel) sums of its output, followed by the
 * GroupNorm(+SiLU) that reads those sums instead of running a statistics pass: the pair every ResnetBlock2D of the UNet
 * executes (needs H*W % 32 == 0).  conv_out [n,H,W,Cout] and gn_out [n,H,W,Cout] are both written. */
int d4d_op_conv3x3_groupnorm(const void* x_nhwc, int n_img, int H, int W, int Cin, const void* Wt, int Cout,
                             const float* bias, const void* residual, int groups, float eps, const float* gamma,
                             const float* beta, int silu, void* conv_out, void* gn_out, void* stream);
int d4d_op_layernorm(const void* x, int rows, int C, float eps, const float* gamma, const float* beta, void* out,
                     void* stream);
/* Debug tap (per-level drift reports in tests/): runs the forward of d4d_unet_forward up to intermediate activation
 * `tap` (0 = conv_in(+pose), then down_blocks.0-3, mid_block, up_blocks.0-3) and copies it out as NCHW bf16
 * [B, C, H, W].  name64 (64 bytes) / dims3 (C, H, W) are filled when non-NULL; out == NULL only queries them.
 * Returns 1 when `tap` is out of range. */
int d4d_debug_tap(d4d_handle* h, const void* sample, const int64_t* timestep, const void* skeletons,
                  const int32_t* domain_ids, int n_domains, int B, int F, int height, int width, int tap, void* out,
                  char* name64, int32_t* dims3, void* stream);

/* ---- multi-GPU: frame-sharded window with fused K/V exchange over peer memory (SURVEY.md section 8e.2) ------------
 * One process per GPU.  Rank r of `world` owns frames [r*F_local, (r+1)*F_local) of each CFG half (F_total = world *
 * F_local); everything except the 3-D attention is per image.  At each 3-D block the fused-QKV GEMM epilogue stores
 * its K|V columns directly into EVERY rank's gathered K/V buffer (peer pointers mapped with cudaIpc, NVLink stores),
 * a system-scope flag round publishes them, and the local attention reads all F_total frames.  Two buffer parities
 * alternate per layer so a rank may run one layer ahead of its peers.
 *   d4d_exchange_alloc  allocates this rank's two K/V buffers (kv_bytes each) + flag array and returns three 64-byte
 *                       cudaIpcMemHandle_t blobs (kv0, kv1, flags) to be all-gathered by the host (torch.distributed);
 *   d4d_exchange_open   maps the peers' buffers: all_handles = [world][3][64] bytes in rank order.
 * kv_bytes must cover 2 (CFG halves) * F_total * (h/2)*(w/2) tokens * 2*C_level1' bf16 (the largest 3-D layer). */
int d4d_exchange_alloc(d4d_handle* h, size_t kv_bytes, unsigned char* handles_out /* [3][64] */);
int d4d_exchange_open(d4d_handle* h, int rank, int world, const unsigned char* all_handles /* [world][3][64] */);
/* B-2 / B-3 on a frame shard: same contracts as d4d_unet_forward / d4d_denoise_window on the LOCAL frames; every rank
 * must call them in the same order (SPMD).  Results are bit-identical to the single-GPU call on the gathered window. */
int d4d_unet_forward_sharded(d4d_handle* h, const void* sample, const int64_t* timestep, const void* skeletons,
                             const int32_t* domain_ids, int n_domains, int B_local, int F_local, int F_total, int height,
                             int width, void* out, void* stream);
int d4d_denoise_window_sharded(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                               const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                               const d4d_sched* sched, float guidance_scale, int domain, int F_local, int F_total,
                               int height, int width, int num_steps, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* D4D_H_ */
