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

/* DPM-Solver++ constants for the fused step (upstream diffusers DPMSolverMultistepScheduler with algorithm_type
 * "dpmsolver++", solver_type "midpoint", solver_order 1 or 2).  The solver's history is per frame and lives on the device
 * (x0_prev / lower_order_nums of d4d_denoise_window_dpm); a frame's step index is its timestep index, so schedules with
 * duplicate timesteps are not accepted by the host tables.
 * coefs row i (fp32), computed on the host from the sigma table in the upstream scheduler's own fp32 order of operations
 * (so the device evaluates no log / exp and the bf16-emulating step is bit-exact against a CPU evaluation):
 *   [0] alpha_s = 1 / sqrt(sigma_i^2 + 1)   [1] sigma_s = sigma_i * alpha_s   [2] sigma_t(i+1) / sigma_s
 *   [3] c = alpha_t(i+1) * (exp(-h) - 1), h = lambda_(i+1) - lambda_i        [4] 0.5 * c
 *   [5] 1 / r0, r0 = (lambda_i - lambda_(i-1)) / h   (0 in row 0) */
typedef struct d4d_dpm_sched {
  const int64_t* timesteps_table;   /* device, [n_steps]  (scheduler.timesteps after set_timesteps) */
  const float* coefs;               /* device, [n_steps][6], see above */
  int32_t n_steps;
  int32_t prediction_type;          /* 0 epsilon, 1 v_prediction, 2 sample */
  int32_t solver_order;             /* 1 or 2 */
  int32_t final_first_order;        /* 1: the last step is first order (euler_at_final, lower_order_final with fewer
                                       than 15 steps, or final_sigmas_type "zero") */
  int32_t emulate_bf16;             /* 1: round like the reference's bf16 eager maths (history and x0 in bf16) */
} d4d_dpm_sched;

/* UniPC constants for the fused step (upstream diffusers UniPCMultistepScheduler with predict_x0, solver_type "bh1" or
 * "bh2", solver_order 1 or 2, no solver_p; d4d_version() 107 and later).  The solver's history is per frame and lives on
 * the device (x0_prev / x0_prev2 / last_sample / lower_order_nums of d4d_denoise_window_unipc); a frame's step index is
 * its timestep index.  Step i runs the corrector (UniC) of the frame's previous step when lower_order_nums >= 1 and row
 * i enables it, at order lower_order_nums, then the predictor (UniP) at order min(row i's cap, lower_order_nums + 1).
 * coefs row i (fp32), computed on the host in the upstream scheduler's fp32 order of operations (the device evaluates no
 * log / exp / solve), with alpha_j = 1 / sqrt(sigma_j^2 + 1), sigma'_j = sigma_j * alpha_j, lambda_j = log alpha_j -
 * log sigma'_j, h_j = lambda_(j+1) - lambda_j, hphi1(h) = expm1(-h), B(h) = -h ("bh1") or expm1(-h) ("bh2"):
 *   [0] alpha_i   [1] sigma'_i                                               (convert_model_output)
 *   [2] sigma'_(i+1) / sigma'_i   [3] alpha_(i+1) * hphi1(h_i)   [4] alpha_(i+1) * B(h_i)
 *   [5] rk = (lambda_(i-1) - lambda_i) / h_i (0 in row 0)                    (predictor)
 *   [6] sigma'_i / sigma'_(i-1)   [7] alpha_i * hphi1(h_(i-1))   [8] alpha_i * B(h_(i-1))
 *   [9] rk' = (lambda_(i-2) - lambda_(i-1)) / h_(i-1) (0 in rows 0, 1)       (corrector; all 0 in row 0)
 *   [10] rho0  [11] rho1: solve(R, b) of the order-2 corrector in fp32 (0 in rows 0, 1; the bf16-emulating step rounds
 *        them to bf16 like upstream's cast to the sample dtype)
 *   [12] 1 if the corrector runs at step i (i > 0 and i - 1 not in disable_corrector), else 0
 *   [13] the predictor's order cap: min(solver_order, n_steps - i) with lower_order_final, else solver_order */
typedef struct d4d_unipc_sched {
  const int64_t* timesteps_table;   /* device, [n_steps]  (scheduler.timesteps after set_timesteps) */
  const float* coefs;               /* device, [n_steps][14], see above */
  int32_t n_steps;
  int32_t prediction_type;          /* 0 epsilon, 1 v_prediction, 2 sample */
  int32_t solver_order;             /* 1 or 2 */
  int32_t emulate_bf16;             /* 1: round like the reference's bf16 eager maths (history, x0 and every op in bf16) */
} d4d_unipc_sched;

/* PNDM constants for the fused step (upstream diffusers PNDMScheduler with skip_prk_steps, i.e. the PLMS linear
 * multistep steps only; d4d_version() 110 and later).  The solver's history is per frame and lives on the device (ets0..3 /
 * cur_sample / counter of d4d_denoise_window_pndm); a frame's counter is the number of steps it has taken (upstream's
 * `counter`), and its row of the table is its timestep index.  Counter 0 steps with the model output as it is and saves
 * the sample; counter 1 re-steps from that saved sample with the mean of the two outputs, from t + T/n to t; counters
 * 2, 3 and >= 4 use the Adams-Bashforth combinations of the last 2, 3 and 4 outputs (counter 1's output is not kept).
 * The table has one row per entry of upstream's timesteps (num_inference_steps + 1 of them from 2 steps on).
 * coefs row i (fp32), computed on the host in the upstream scheduler's fp32 order of operations (the device evaluates no
 * pow), for t = timesteps[i], prev = t - T/n (T/n = num_train_timesteps // num_inference_steps), a_j = alphas_cumprod[j]
 * (final_alpha_cumprod for j < 0):
 *   [0] a_t^0.5  [1] (1 - a_t)^0.5                                          (v_prediction -> epsilon)
 *   [2] (a_prev / a_t)^0.5  [3] a_prev - a_t  [4] a_t * (1 - a_prev)^0.5 + (a_t * (1 - a_t) * a_prev)^0.5
 *   [5..9] the same for the counter-1 step, with (prev, t) = (t, t + T/n); NaN where t + T/n >= T, where upstream's
 *          lookup fails */
typedef struct d4d_pndm_sched {
  const int64_t* timesteps_table;   /* device, [n_steps]  (scheduler.timesteps after set_timesteps) */
  const float* coefs;               /* device, [n_steps][10], see above */
  int32_t n_steps;                  /* rows of the table */
  int32_t prediction_type;          /* 0 epsilon, 1 v_prediction */
  int32_t emulate_bf16;             /* 1: round like the reference's bf16 eager maths (history and every op in bf16) */
} d4d_pndm_sched;

/* DEIS constants for the fused step (upstream diffusers DEISMultistepScheduler with algorithm_type "deis", solver_type
 * "logrho", solver_order 1, 2 or 3; d4d_version() 111 and later).  The solver's history is per frame and lives on the
 * device (m_prev / m_prev2 / lower_order_nums of d4d_denoise_window_deis); a frame's step index is its timestep index.
 * The history holds model outputs converted to their epsilon form, m = (x - alpha_i * x0) / sigma'_i with x0 the data
 * prediction.  Step i runs at order min(solver_order, lower_order_nums + 1, row i's cap).  Every sigma is nonzero: the
 * table ends on the sigma of the first training timestep.
 * coefs row i (fp32), computed on the host in the upstream scheduler's fp32 order of operations (the device evaluates no
 * log / exp), with alpha_j = 1 / sqrt(sigma_j^2 + 1), sigma'_j = sigma_j * alpha_j, lambda_j = log alpha_j - log sigma'_j,
 * rho_j = sigma'_j / alpha_j, and upstream's ind_fn integrals of the Lagrange basis in log rho (np.log in fp32):
 *   [0] alpha_i   [1] sigma'_i                                               (convert_model_output)
 *   [2] alpha_(i+1) / alpha_i   [3] sigma'_(i+1) * (exp(lambda_(i+1) - lambda_i) - 1)
 *                                                     (first order: x' = [2] * x - [3] * m0)
 *   [4] alpha_(i+1)                                   (higher orders: x' = [4] * (x / alpha_i + sum_k c_k * m_k))
 *   [5] c_0  [6] c_1 of the second-order update from rho_i, rho_(i-1) to rho_(i+1)         (0 in row 0)
 *   [7] c_0  [8] c_1  [9] c_2 of the third-order update from rho_i, rho_(i-1), rho_(i-2)    (0 in rows 0, 1)
 *   [10] the order cap: min(solver_order, i + 1), and with lower_order_final below 15 steps 1 in the last row and 2 in
 *        the row before it */
typedef struct d4d_deis_sched {
  const int64_t* timesteps_table;   /* device, [n_steps]  (scheduler.timesteps after set_timesteps) */
  const float* coefs;               /* device, [n_steps][11], see above */
  int32_t n_steps;
  int32_t prediction_type;          /* 0 epsilon, 1 v_prediction, 2 sample */
  int32_t solver_order;             /* 1, 2 or 3 */
  int32_t emulate_bf16;             /* 1: round like the reference's bf16 eager maths (history and every op in bf16) */
} d4d_deis_sched;

/* DPM-Solver++ singlestep constants for the fused step (upstream diffusers DPMSolverSinglestepScheduler with
 * algorithm_type "dpmsolver++", solver_type "midpoint", solver_order 1, 2 or 3; d4d_version() 112 and later).  The
 * solver's history is per frame and lives on the device (x0_prev / x0_prev2 / cur_sample / lower_order_nums of
 * d4d_denoise_window_dpm_single); a frame's step index is its timestep index.  Upstream's order list splits the steps
 * into blocks 1, 2, .., k; step i runs at order min(row i's order, lower_order_nums + 1).  A step at order 1 starts a
 * block and saves its sample in cur_sample; a step at order k > 1 updates from that sample, k - 1 rows back, with the
 * data predictions x0 (this step), x0_prev and, at order 3, x0_prev2 (the block start's).
 * coefs row i (fp32), computed on the host in the upstream scheduler's fp32 order of operations (the device evaluates no
 * log / exp), with alpha_j = 1 / sqrt(sigma_j^2 + 1), sigma'_j = sigma_j * alpha_j, lambda_j = log alpha_j - log sigma'_j
 * and, for the update of order k, b = i - k + 1 (the block start), h = lambda_(i+1) - lambda_b,
 * r0 = (lambda_i - lambda_b) / h, c = alpha_(i+1) * (exp(-h) - 1):
 *   [0] alpha_i   [1] sigma'_i                                               (convert_model_output)
 *   [2] sigma'_(i+1) / sigma'_i   [3] c                 (order 1: x' = [2] * x - [3] * x0; [2], [3] as d4d_dpm_sched's)
 *   [4] sigma'_(i+1) / sigma'_(i-1)   [5] c   [6] 0.5 * c   [7] 1 / r0
 *        (order 2: x' = [4] * s - [5] * x0_prev - [6] * ([7] * (x0 - x0_prev)), s = cur_sample)
 *   [8] sigma'_(i+1) / sigma'_(i-2)   [9] c   [10] alpha_(i+1) * ((exp(-h) - 1) / h + 1)   [11] 1 / r0
 *        (order 3: x' = [8] * s - [9] * x0_prev2 + [10] * ([11] * (x0 - x0_prev2)))
 *   [12] the row's order from upstream's order list
 * [4..7] are 0 in rows of order 1 and [8..11] in rows of order 1 or 2 (those rows never run the update; with
 * final_sigmas_type "zero" the last row has order 1 and an infinite h). */
typedef struct d4d_dpm_single_sched {
  const int64_t* timesteps_table;   /* device, [n_steps]  (scheduler.timesteps after set_timesteps) */
  const float* coefs;               /* device, [n_steps][13], see above */
  int32_t n_steps;
  int32_t prediction_type;          /* 0 epsilon, 1 v_prediction, 2 sample */
  int32_t solver_order;             /* 1, 2 or 3 */
  int32_t emulate_bf16;             /* 1: round like the reference's bf16 eager maths (history and every op in bf16) */
} d4d_dpm_single_sched;

/* DDPM constants for the fused step (upstream diffusers DDPMScheduler with variance_type "fixed_small",
 * "fixed_small_log" or "fixed_large", no thresholding; d4d_version() 115 and later).  Ancestral sampling: the step adds
 * std * z on rows with t > 0, so it is the first stochastic step.  z is a pure function of the task's 64-bit `seed`, the
 * frame's index in its task (the `frame_ids` argument), the frame's timestep index before the step and the element:
 * Philox4x32-10 with key = seed (low word first) and counter (e / 4, frame id, timestep index, 0) for element e of the
 * frame's [4,h,w] latent, which takes word e % 4; a word x maps to u = (x + 0.5) * 2^-32, Box-Muller turns (u0, u1) into
 * z0, z1 and (u2, u3) into z2, z3 in fp64, and the result is rounded once (to bf16 with emulate_bf16, as upstream draws
 * the noise in the model output's dtype; to fp32 otherwise).  No rank, window position or launch order enters it, so
 * every multi-GPU mode draws the single-GPU bits.  DDPM keeps no history; a frame's step index is its timestep index.
 * coefs row i (fp32), computed on the host in the upstream scheduler's fp32 order of operations (the device evaluates no
 * pow / log / exp), with t = timesteps[i], a_t = alphas_cumprod[t], a_prev = alphas_cumprod[timesteps[i + 1]] (1 after
 * the last row), beta = 1 - a_t / a_prev:
 *   [0] a_t^0.5   [1] (1 - a_t)^0.5                        (x0 by prediction type; epsilon divides by [0] like upstream)
 *   [2] a_prev^0.5 * beta / (1 - a_t)   [3] (a_t / a_prev)^0.5 * (1 - a_prev) / (1 - a_t)   (x' = [2] * x0 + [3] * x)
 *   [4] the noise std: fixed_small (max((1 - a_prev) / (1 - a_t) * beta, 1e-20))^0.5, fixed_small_log
 *       exp(0.5 * log(that)), fixed_large beta^0.5
 *   [5] 1 if t > 0 (the row adds std * z), else 0 */
typedef struct d4d_ddpm_sched {
  const int64_t* timesteps_table;   /* device, [n_steps]  (scheduler.timesteps after set_timesteps) */
  const float* coefs;               /* device, [n_steps][6], see above */
  int32_t n_steps;
  int32_t prediction_type;          /* 0 epsilon, 1 v_prediction, 2 sample */
  int32_t clip_sample;
  float clip_sample_range;
  int32_t emulate_bf16;             /* 1: round like the reference's bf16 eager maths (every op and the noise in bf16) */
  uint64_t seed;                    /* the task's noise seed */
} d4d_ddpm_sched;

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
/* The same window step with a DPM-Solver++ scheduler.  Arguments as d4d_denoise_window, plus the window frames' solver
 * state, read and updated in place (conditioning frames keep theirs):
 *   x0_prev           device bf16 [F,4,h,w]: each frame's data prediction of its previous step (zeros for a new task)
 *   lower_order_nums  device int32 [F]: steps each frame has taken, capped at solver_order (zeros for a new task)
 * A caller carries both across the windows of one task, gathered and scattered with the frames like the latents. */
int d4d_denoise_window_dpm(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                           const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                           const d4d_dpm_sched* sched, float guidance_scale, int domain, int F, int height, int width,
                           int num_steps, void* x0_prev, int32_t* lower_order_nums, void* stream);

/* The same window step with a UniPC scheduler (d4d_version() 107 and later).  Arguments as d4d_denoise_window, plus the
 * window frames' solver state, read and updated in place (conditioning frames keep theirs; zeros for a new task):
 *   x0_prev           device bf16 [F,4,h,w]: each frame's data prediction of its previous step
 *   x0_prev2          device bf16 [F,4,h,w]: the one before (solver_order 2; NULL exactly when solver_order is 1)
 *   last_sample       device bf16 [F,4,h,w]: the sample each frame's last predictor started from, after correction
 *   lower_order_nums  device int32 [F]: steps each frame has taken, capped at solver_order
 * A caller carries them across the windows of one task, gathered and scattered with the frames like the latents. */
int d4d_denoise_window_unipc(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                             const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                             const d4d_unipc_sched* sched, float guidance_scale, int domain, int F, int height, int width,
                             int num_steps, void* x0_prev, void* x0_prev2, void* last_sample, int32_t* lower_order_nums,
                             void* stream);

/* The same window step with a PNDM scheduler (d4d_version() 110 and later).  Arguments as d4d_denoise_window, plus the
 * window frames' solver state, read and updated in place (conditioning frames keep theirs; zeros for a new task):
 *   ets0, ets1, ets2, ets3  device bf16 [F,4,h,w]: each frame's last model outputs, in a ring: the output of counter c
 *                           (c != 1) is stored in ets((c == 0 ? 0 : c - 1) % 4)
 *   cur_sample              device bf16 [F,4,h,w]: the sample each frame's counter-0 step started from
 *   counter                 device int32 [F]: steps each frame has taken
 * A caller carries them across the windows of one task, gathered and scattered with the frames like the latents. */
int d4d_denoise_window_pndm(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                            const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                            const d4d_pndm_sched* sched, float guidance_scale, int domain, int F, int height, int width,
                            int num_steps, void* ets0, void* ets1, void* ets2, void* ets3, void* cur_sample,
                            int32_t* counter, void* stream);

/* The same window step with a DEIS scheduler (d4d_version() 111 and later).  Arguments as d4d_denoise_window, plus the
 * window frames' solver state, read and updated in place (conditioning frames keep theirs; zeros for a new task):
 *   m_prev            device bf16 [F,4,h,w]: each frame's previous model output in its epsilon form
 *   m_prev2           device bf16 [F,4,h,w]: the one before (solver_order 3; NULL exactly when solver_order is 1 or 2)
 *   lower_order_nums  device int32 [F]: steps each frame has taken, capped at solver_order
 * A caller carries them across the windows of one task, gathered and scattered with the frames like the latents. */
int d4d_denoise_window_deis(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                            const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                            const d4d_deis_sched* sched, float guidance_scale, int domain, int F, int height, int width,
                            int num_steps, void* m_prev, void* m_prev2, int32_t* lower_order_nums, void* stream);

/* The same window step with a DPM-Solver++ singlestep scheduler (d4d_version() 112 and later).  Arguments as
 * d4d_denoise_window, plus the window frames' solver state, read and updated in place (conditioning frames keep theirs;
 * zeros for a new task):
 *   x0_prev           device bf16 [F,4,h,w]: each frame's data prediction of its previous step
 *   x0_prev2          device bf16 [F,4,h,w]: the one before (solver_order 3; NULL exactly when solver_order is 1 or 2)
 *   cur_sample        device bf16 [F,4,h,w]: the sample each frame's current block started from
 *   lower_order_nums  device int32 [F]: steps each frame has taken, capped at solver_order
 * A caller carries them across the windows of one task, gathered and scattered with the frames like the latents. */
int d4d_denoise_window_dpm_single(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                  const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                  const d4d_dpm_single_sched* sched, float guidance_scale, int domain, int F, int height,
                                  int width, int num_steps, void* x0_prev, void* x0_prev2, void* cur_sample,
                                  int32_t* lower_order_nums, void* stream);

/* The same window step with a DDPM scheduler (d4d_version() 115 and later).  Arguments as d4d_denoise_window, plus
 *   frame_ids  device int64 [F]: each window frame's index in its task, which keys its noise (see d4d_ddpm_sched)
 * DDPM keeps no history: nothing but the latents and timestep indices is updated.  The step reads and writes four
 * elements at a time: latents must be 8-byte aligned (a call with unaligned latents returns 1 before any launch). */
int d4d_denoise_window_ddpm(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                            const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                            const d4d_ddpm_sched* sched, float guidance_scale, int domain, int F, int height, int width,
                            int num_steps, const int64_t* frame_ids, void* stream);

/* ---- building blocks of B-3, exported for parity tests ------------------------------------------------ */
int d4d_assemble_input(void* latents, const void* pixel_latents, const void* plucker, const void* skel_latents,
                       const void* cond_mask, const int64_t* timestep_indices, const int64_t* timesteps_table,
                       int n_steps, int F, int height, int width, int cfg, void* sample_out, int64_t* timestep_out,
                       void* stream);
int d4d_cfg_ddim_step(const void* noise, const void* latents, const void* cond_mask, const int64_t* timestep_indices,
                      int64_t* timestep_indices_out, const d4d_sched* sched, float guidance_scale, int cfg, int F,
                      int height, int width, void* latents_out, void* stream);
/* One CFG + DPM-Solver++ step of the frames (cfg: noise holds [uncond F | cond F]).  x0_prev [F,4,h,w] is updated in
 * place; lower_order_nums_out and timestep_indices_out receive the advanced counters (they may not alias the inputs);
 * latents_out may alias latents. */
int d4d_cfg_dpm_step(const void* noise, const void* latents, const void* cond_mask, const int64_t* timestep_indices,
                     int64_t* timestep_indices_out, void* x0_prev, const int32_t* lower_order_nums,
                     int32_t* lower_order_nums_out, const d4d_dpm_sched* sched, float guidance_scale, int cfg, int F,
                     int height, int width, void* latents_out, void* stream);
/* One CFG + UniPC step of the frames (d4d_version() 107 and later; state as d4d_denoise_window_unipc).  x0_prev, x0_prev2
 * and last_sample are updated in place; lower_order_nums_out and timestep_indices_out receive the advanced counters (they
 * may not alias the inputs); latents_out may alias latents. */
int d4d_cfg_unipc_step(const void* noise, const void* latents, const void* cond_mask, const int64_t* timestep_indices,
                       int64_t* timestep_indices_out, void* x0_prev, void* x0_prev2, void* last_sample,
                       const int32_t* lower_order_nums, int32_t* lower_order_nums_out, const d4d_unipc_sched* sched,
                       float guidance_scale, int cfg, int F, int height, int width, void* latents_out, void* stream);
/* One CFG + PNDM step of the frames (d4d_version() 110 and later; state as d4d_denoise_window_pndm).  ets0..3 and
 * cur_sample are updated in place; counter_out and timestep_indices_out receive the advanced counters (they may not alias
 * the inputs); latents_out may alias latents. */
int d4d_cfg_pndm_step(const void* noise, const void* latents, const void* cond_mask, const int64_t* timestep_indices,
                      int64_t* timestep_indices_out, void* ets0, void* ets1, void* ets2, void* ets3, void* cur_sample,
                      const int32_t* counter, int32_t* counter_out, const d4d_pndm_sched* sched, float guidance_scale,
                      int cfg, int F, int height, int width, void* latents_out, void* stream);
/* One CFG + DEIS step of the frames (d4d_version() 111 and later; state as d4d_denoise_window_deis).  m_prev and m_prev2
 * are updated in place; lower_order_nums_out and timestep_indices_out receive the advanced counters (they may not alias
 * the inputs); latents_out may alias latents. */
int d4d_cfg_deis_step(const void* noise, const void* latents, const void* cond_mask, const int64_t* timestep_indices,
                      int64_t* timestep_indices_out, void* m_prev, void* m_prev2, const int32_t* lower_order_nums,
                      int32_t* lower_order_nums_out, const d4d_deis_sched* sched, float guidance_scale, int cfg, int F,
                      int height, int width, void* latents_out, void* stream);
/* One CFG + DPM-Solver++ singlestep step of the frames (d4d_version() 112 and later; state as
 * d4d_denoise_window_dpm_single).  x0_prev, x0_prev2 and cur_sample are updated in place; lower_order_nums_out and
 * timestep_indices_out receive the advanced counters (they may not alias the inputs); latents_out may alias latents. */
int d4d_cfg_dpm_single_step(const void* noise, const void* latents, const void* cond_mask,
                            const int64_t* timestep_indices, int64_t* timestep_indices_out, void* x0_prev,
                            void* x0_prev2, void* cur_sample, const int32_t* lower_order_nums,
                            int32_t* lower_order_nums_out, const d4d_dpm_single_sched* sched, float guidance_scale,
                            int cfg, int F, int height, int width, void* latents_out, void* stream);

/* One CFG + DDPM step of the frames (d4d_version() 115 and later); frame_ids [F] as d4d_denoise_window_ddpm.
 * timestep_indices_out receives the advanced indices (it may not alias the input); latents_out may alias latents.
 * noise, latents and latents_out must be 8-byte aligned. */
int d4d_cfg_ddpm_step(const void* noise, const void* latents, const void* cond_mask, const int64_t* timestep_indices,
                      int64_t* timestep_indices_out, const int64_t* frame_ids, const d4d_ddpm_sched* sched,
                      float guidance_scale, int cfg, int F, int height, int width, void* latents_out, void* stream);
/* The DDPM step's noise alone (d4d_version() 115 and later): out fp32 [F,4,h,w] receives z of frames frame_ids [F]
 * (device int64) at timestep indices timestep_indices [F] (device int64) for `seed`, rounded once to fp32. */
int d4d_op_ddpm_noise(uint64_t seed, const int64_t* frame_ids, const int64_t* timestep_indices, int F, int height,
                      int width, float* out, void* stream);

/* ---- op-level entry points (each is one hot-path kernel; used by tests/ and bench.py) ------------------
 * d4d_op_gemm:   out[M,N] = act((A|A2)[M,K1+K2] . W[N,K]^T + bias + rowvec[row/rows_per_image]) * scale + residual
 *                geglu: W rows / bias interleaved in groups of 8 (a rows, then g rows), out is [M, N/2].
 * d4d_op_conv3x3: NHWC x [n,H,W,Cin], W [Cout][9][Cin] (tap = ky*3+kx), stride 1, pad 1.
 * stats (gemm, conv3x3, conv_resample): NULL, or a caller-allocated, ZEROED int64 workspace that receives the GroupNorm
 *   statistics of the stored output in d4d_op_groupnorm's format: per-(image, column) fixed-point {sum * 2^28, sum of
 *   squares * 2^24}.  Conv: [n_img][Cout][2], needs tiles whose 32-row warps stay inside one image.  GEMM: [M /
 *   stats_rows][N][2], image = row / stats_rows; needs stats_rows % 32 == 0 and M % stats_rows == 0, and no GEGLU.  */
int d4d_op_gemm(const void* A, int lda, int K1, const void* A2, int lda2, int K2, const void* W, int M, int N,
                const float* bias, const void* rowvec, int ld_rowvec, int rows_per_image, const void* residual,
                int ld_res, void* out, int ldo, int geglu, int act, float out_scale, int block_n, int64_t* stats,
                int stats_rows, void* stream);
/* The QKV projection of a frame-sharded 3-D attention layer (d4d_version() 105 and later): out = A[M,K] . W[N,K]^T, but
 * only columns < kv_col0 (Q) are written to out [M, ldo]; columns >= kv_col0 (K|V) are NOT written to out and go instead to
 * every kv_dst[r], r < world, a [halves * rows_global, kv_ld] matrix: local row m of CFG half h = m / rows_local lands at
 * row h * rows_global + row_offset + m % rows_local, column - kv_col0.  Needs 1 <= world <= 8, kv_col0 % 16 == 0,
 * kv_ld % 8 == 0, M % rows_local == 0 and row_offset + rows_local <= rows_global; returns 1 otherwise, before any launch. */
int d4d_op_gemm_kv_scatter(const void* A, int lda, int K, const void* W, int M, int N, void* out, int ldo, int kv_col0,
                           int kv_ld, int64_t rows_local, int64_t rows_global, int64_t row_offset, int world,
                           void* const* kv_dst, int block_n, void* stream);
int d4d_op_conv3x3(const void* x_nhwc, int n_img, int H, int W, int Cin, const void* Wt, int Cout, const float* bias,
                   const void* rowvec, int ld_rowvec, const void* residual, int act, void* out, int block_n,
                   int64_t* stats, void* stream);
/* The three convolutions of the UNet at an explicit tile (d4d_version() 108 and later).  kind 0: d4d_op_conv3x3; kind 1 / 3:
 * d4d_op_conv_resample's stride-2 conv / four-phase upsampling conv (residual then has the output's shape).
 * block_m: 0 (automatic), 128 or 256 output positions per tile; 256 needs block_n 0, 128 or 160.  The output and the
 * statistics do not depend on the tile: every sum runs in the same order.  Anything else returns 1, before any launch. */
int d4d_op_conv_tiled(const void* x_nhwc, int n_img, int H, int W, int Cin, const void* Wt, int Cout, const float* bias,
                      const void* rowvec, int ld_rowvec, const void* residual, int act, void* out, int kind, int block_m,
                      int block_n, int64_t* stats, void* stream);
/* The tile (rows, width) an automatic conv launch of this shape (kind as d4d_op_conv_tiled) takes on a device with `sms`
 * SMs; needs no device. */
int d4d_conv_tile_choice(int n_img, int H, int W, int Cin, int Cout, int kind, int sms, int* block_m, int* block_n);
/* d4d_op_gemm at an explicit schedule (d4d_version() 109 and later): 0 automatic, 1 cooperative (both MMA warpgroups
 * share each 128-row tile), 2 ping-pong (each MMA warpgroup owns every other tile, so one tile's epilogue runs under the
 * other's MMAs; block_n 0, 64 or 128, GEGLU 0 or 128, 16-byte aligned out and residual).  The output and the
 * statistics do not depend on the schedule: every sum runs in the same order.  Anything else returns 1, before any launch. */
int d4d_op_gemm_tiled(const void* A, int lda, int K1, const void* A2, int lda2, int K2, const void* W, int M, int N,
                      const float* bias, const void* rowvec, int ld_rowvec, int rows_per_image, const void* residual,
                      int ld_res, void* out, int ldo, int geglu, int act, float out_scale, int block_n, int schedule,
                      int64_t* stats, int stats_rows, void* stream);
/* The width and schedule (1 cooperative, 2 ping-pong) an automatic plain GEMM launch of this shape takes on a device with
 * `sms` SMs (K2: columns of the second source, 0 for none); needs no device. */
int d4d_gemm_tile_choice(int M, int N, int K1, int K2, int geglu, int sms, int* block_n, int* schedule);
/* q: column slice of a row-major [batch*seq, ld_qkv] matrix; head hd = columns [hd*D, (hd+1)*D).  k, v: column slices of a
 * row-major [batch*seq_kv, ld_kv] matrix, the keys of batch entry b in rows [b*seq_kv, (b+1)*seq_kv).  seq_kv = 0 means
 * seq and ld_kv = 0 means ld_qkv (k and v in the QKV matrix). */
int d4d_op_attention(const void* q, const void* k, const void* v, int ld_qkv, void* out, int ld_out, int batch,
                     int seq, int heads, int head_dim, float scale, int seq_kv, int ld_kv, void* stream);
/* GroupNorm(+SiLU) of NHWC x1 [n_img, hw, C1], virtually concatenated on channels with x2 [n_img, hw, C2] when x2 is not
 * NULL, into out [n_img, hw, C1+C2]; 32 <= C1 + C2 <= 4096, C1 and C2 multiples of 8.  One statistics launch per source
 * fills `stats`, then one launch normalises.  stats: caller-allocated, ZEROED int64 workspace [n_img][C1+C2][2] (x1's
 * channels, then x2's) that receives the per-(image, channel) fixed-point {sum, sum of squares}. */
int d4d_op_groupnorm(const void* x1, int C1, const void* x2, int C2, int n_img, int hw, int groups, float eps,
                     const float* gamma, const float* beta, int silu, void* out, int64_t* stats, void* stream);
/* The two resampling convolutions of the UNet, read / written in place (no im2col, no materialised upsampled tensor):
 *   kind 1: 3x3 stride-2 pad-1 conv (diffusers Downsample2D): x [n,H,W,Cin] -> out [n,H/2,W/2,Cout], Wt [Cout][9][Cin];
 *   kind 2: one sub-pixel phase (up_a, up_b in {0,1}) of "nearest x2 upsample, then 3x3 pad-1 conv" (Upsample2D): a 2x2 conv on
 *           the low-resolution x with pre-summed weights Wt [Cout][4][Cin] (tap = ty*2+tx; rows {-1,0} for up_a = 0, {0,+1} for
 *           up_a = 1, same for columns), written to pixels (2y+up_a, 2x+up_b) of out [n,2H,2W,Cout].  Four calls fill out;
 *   kind 3: all four phases in one launch, Wt [4 (= up_a*2+up_b)][Cout][4][Cin] (what the UNet plan uses). */
int d4d_op_conv_resample(const void* x_nhwc, int n_img, int H, int W, int Cin, const void* Wt, int Cout, const float* bias,
                         int kind, int up_a, int up_b, void* out, int64_t* stats, void* stream);
/* conv3x3 (+bias, +residual) whose epilogue accumulates the per-(image, channel) sums of its output, followed by the
 * GroupNorm(+SiLU) that reads those sums instead of running a statistics pass: the pair every ResnetBlock2D of the UNet
 * executes (needs H*W % 32 == 0).  conv_out [n,H,W,Cout] and gn_out [n,H,W,Cout] are both written.  stats:
 * caller-allocated, ZEROED int64 workspace [n][Cout][2] for the sums (same format as d4d_op_groupnorm's). */
int d4d_op_conv3x3_groupnorm(const void* x_nhwc, int n_img, int H, int W, int Cin, const void* Wt, int Cout,
                             const float* bias, const void* residual, int groups, float eps, const float* gamma,
                             const float* beta, int silu, void* conv_out, void* gn_out, int64_t* stats, void* stream);
int d4d_op_layernorm(const void* x, int rows, int C, float eps, const float* gamma, const float* beta, void* out,
                     void* stream);
/* Pose encoder, conv_layers.0: 3 -> 3 channels, 3x3, stride 1, pad 1, + bias, SiLU.  x_nchw [n,3,H,W] (the skeleton
 * images), Wt [9][3][3] = [tap = ky*3+kx][Cin][Cout], bias fp32 [3], out_nhwc4 [n,H,W,4] with channel 3 written as 0. */
int d4d_op_pose_conv0(const void* x_nchw, int n, int H, int W, const void* Wt, const float* bias, void* out_nhwc4,
                      void* stream);
/* Pose encoder, conv_layers.2/4/6/8: pad 1, + bias, SiLU, NHWC x [n,H,W,Cin] -> out [n,Ho,Wo,Cout],
 * Ho = (H + 2 - ksize) / stride + 1 (Wo alike).  (Cin, Cout, ksize, stride) is one of (4,16,4,2) (conv_layers.2 reading
 * conv_layers.0's 4-channel pixels), (16,16,3,1), (16,32,4,2), (32,32,3,1); anything else returns 1.  Wt: 16-byte aligned
 * [Cout][ksize*ksize*Cin + 8], column tap*Cin + ci with tap = ky*ksize+kx; the 8 trailing columns of each row are not read
 * for arithmetic, and for Cin 4 the weights of channel 3 must be 0.  bias fp32 [Cout]. */
int d4d_op_pose_conv(const void* x_nhwc, int n, int Cin, int H, int W, const void* Wt, const float* bias, int Cout,
                     int ksize, int stride, void* out, void* stream);
/* Debug tap (per-level drift reports and per-module checks in tests/): runs the forward of d4d_unet_forward up to
 * intermediate activation `tap` and copies it out as NCHW bf16 [B, C, H, W].  name64 (64 bytes) / dims3 (C, H, W) are
 * filled when non-NULL; out == NULL only queries them.  Returns 1 when `tap` is out of range.
 *   0-9   block outputs: conv_in (+ pose encoder), down_blocks.0-3, mid_block, up_blocks.0-3
 *   10-   module outputs, named after the diffusers module paths (d4d_version() 104 and later), in forward order:
 *         time_embedding (time embedding + frame-index embedding, before the SiLU; C = 4 * block_out_channels[0],
 *         H = W = 1), down_blocks.i.resnets.j, down_blocks.i.attentions.j and down_blocks.i.downsamplers.0 (i < 3),
 *         mid_block.resnets.0, mid_block.attentions.0, mid_block.resnets.1, up_blocks.i.resnets.j,
 *         up_blocks.i.attentions.j (i > 0) and up_blocks.i.upsamplers.0 (i < 3).
 * Taps add no launch: a forward enqueues the same kernels whether or not they are read. */
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
 *   d4d_exchange_open   maps the peers' buffers: all_handles = [world][3][64] bytes in rank order.  world = 1 (rank 0 on
 *                       its own buffers) runs the sharded plan on one GPU.
 * kv_bytes must cover the largest 3-D attention layer: 2 (CFG halves) * F_total * (h >> L)*(w >> L) tokens * 2*C'_L bf16
 * (C'_L = heads * padded head_dim) over the levels L that run 3-D attention: the mid block's (L = 3) always, and level
 * L < 3 when 3 - L < num_3d_attn_blocks (level 0 with num_3d_attn_blocks = 4).  sharded.exchange_bytes computes it. */
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
/* d4d_denoise_window_ddpm on a frame shard (d4d_version() 115 and later): frame_ids [F_local] holds the LOCAL frames'
 * indices in their task. */
int d4d_denoise_window_ddpm_sharded(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                    const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                    const d4d_ddpm_sched* sched, float guidance_scale, int domain, int F_local,
                                    int F_total, int height, int width, int num_steps, const int64_t* frame_ids,
                                    void* stream);
/* d4d_denoise_window_dpm on a frame shard (d4d_version() 106 and later): x0_prev [F_local,4,h,w] and lower_order_nums
 * [F_local] hold the LOCAL frames' solver state. */
int d4d_denoise_window_dpm_sharded(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                   const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                   const d4d_dpm_sched* sched, float guidance_scale, int domain, int F_local, int F_total,
                                   int height, int width, int num_steps, void* x0_prev, int32_t* lower_order_nums,
                                   void* stream);
/* Window-result exchange of the frame-sharded sliding loop (d4d_version() 106 and later): after a window step every rank
 * passes its F_local updated frames -- latents [F_local,4,h,w], timestep indices int64 [F_local] and, with DPM-Solver++,
 * x0_prev [F_local,4,h,w] and lower_order_nums int32 [F_local] (both NULL for DDIM and DDPM) -- and receives the whole window,
 * F_total = world * F_local frames in window order, in latents_out / timestep_indices_out / x0_prev_out /
 * lower_order_nums_out (NULL exactly when the inputs are).  The frames are stored into every rank's exchange buffer at
 * row rank * F_local (d4d_op_window_scatter), one flag round publishes them, and each rank copies the gathered window out.
 * It is one exchange of the same epoch sequence as the 3-D attention layers, so every rank must call it in the same
 * order as its sharded window steps (SPMD).  The gathered window needs F_total * (4*h*w * 2 * (1 + dpm) + 8 + 4 * dpm)
 * bytes of the exchange buffer; a larger window returns 1 before any launch.  Latent pointers must be 16-byte aligned. */
int d4d_window_exchange(d4d_handle* h, const void* latents_local, const int64_t* timestep_indices_local,
                        const void* x0_prev_local, const int32_t* lower_order_nums_local, int F_local, int F_total,
                        int height, int width, void* latents_out, int64_t* timestep_indices_out, void* x0_prev_out,
                        int32_t* lower_order_nums_out, void* stream);
/* The store kernel of d4d_window_exchange alone, with explicit destinations (d4d_version() 106 and later): writes this
 * rank's frames into every dst[r], r < world, each a gathered window of dst_bytes bytes laid out as
 *   latents [F_total][4*h*w] bf16 | x0_prev [F_total][4*h*w] bf16 (DPM only) | timestep indices [F_total] int64 |
 *   lower_order_nums [F_total] int32 (DPM only),
 * at frame rows [rank * F_local, (rank + 1) * F_local); nothing else of dst is written.  Returns 1 before any launch for a
 * null destination, world outside [1, 8], rank outside [0, world), F_local * world != F_total, x0_prev without
 * lower_order_nums (or the reverse), unaligned pointers, or a window larger than dst_bytes. */
int d4d_op_window_scatter(const void* latents, const int64_t* timestep_indices, const void* x0_prev,
                          const int32_t* lower_order_nums, int F_local, int F_total, int height, int width, int world,
                          int rank, void* const* dst, size_t dst_bytes, void* stream);

/* ---- multi-GPU: CFG-split window (d4d_version() 113 and later) ------------------------------------------------------
 * With classifier-free guidance on, the two halves of a window's UNet batch (F negative images, then F positive ones)
 * never read each other; they meet in the CFG combine.  One process per GPU, world = 2: rank k runs the UNet on CFG half
 * k only (rank 0 the negative half, rank 1 the positive half) and its output permute stores the half's noise
 * [F,out_channels,h,w] at rows [k*F, (k+1)*F) of BOTH ranks' exchange buffers (d4d_exchange_alloc / d4d_exchange_open,
 * the same peer buffers and epoch sequence as the frame-sharded window).  One flag round publishes them; then every rank
 * runs the unchanged CFG + scheduler step of d4d_denoise_window on the whole window, reading the gathered [2F] noise
 * in place.  The ranks compute the step from the same bits, so they end with identical latents, timestep indices and
 * solver state, and nothing else is exchanged.
 *   - Arguments are those of the single-GPU counterpart (d4d_denoise_window, _dpm, _unipc, _pndm, _deis, _dpm_single):
 *     EVERY rank passes the whole window and the whole window's solver state, and all of it is updated in place alike
 *     on every rank.  Results are bit-identical to the single-GPU call.
 *   - SPMD: both ranks make the same calls in the same order, with the same guidance_scale.  guidance_scale <= 1 has no
 *     halves: the call runs the single-GPU step on every rank and exchanges nothing.
 *   - Each exchange buffer (kv_bytes of d4d_exchange_alloc) must hold 2 * F * out_channels * h * w bf16; a larger window,
 *     or a handle opened with world > 2, returns 1 before any launch.
 *   - world = 1 (rank 0 on its own buffers) is a loopback on one GPU: the rank runs half 0, then half 1, into its own
 *     buffer, followed by the flag round. */
int d4d_denoise_window_cfg_split(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                 const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                 const d4d_sched* sched, float guidance_scale, int domain, int F, int height, int width,
                                 int num_steps, void* stream);
int d4d_denoise_window_dpm_cfg_split(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                     const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                     const d4d_dpm_sched* sched, float guidance_scale, int domain, int F, int height,
                                     int width, int num_steps, void* x0_prev, int32_t* lower_order_nums, void* stream);
int d4d_denoise_window_unipc_cfg_split(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                       const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                       const d4d_unipc_sched* sched, float guidance_scale, int domain, int F, int height,
                                       int width, int num_steps, void* x0_prev, void* x0_prev2, void* last_sample,
                                       int32_t* lower_order_nums, void* stream);
int d4d_denoise_window_pndm_cfg_split(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                      const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                      const d4d_pndm_sched* sched, float guidance_scale, int domain, int F, int height,
                                      int width, int num_steps, void* ets0, void* ets1, void* ets2, void* ets3,
                                      void* cur_sample, int32_t* counter, void* stream);
int d4d_denoise_window_deis_cfg_split(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                      const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                      const d4d_deis_sched* sched, float guidance_scale, int domain, int F, int height,
                                      int width, int num_steps, void* m_prev, void* m_prev2, int32_t* lower_order_nums,
                                      void* stream);
int d4d_denoise_window_dpm_single_cfg_split(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                            const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                            const d4d_dpm_single_sched* sched, float guidance_scale, int domain, int F,
                                            int height, int width, int num_steps, void* x0_prev, void* x0_prev2,
                                            void* cur_sample, int32_t* lower_order_nums, void* stream);
/* (d4d_version() 115 and later) frame_ids [F]: the whole window's, as d4d_denoise_window_ddpm */
int d4d_denoise_window_ddpm_cfg_split(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                      const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                      const d4d_ddpm_sched* sched, float guidance_scale, int domain, int F, int height,
                                      int width, int num_steps, const int64_t* frame_ids, void* stream);

/* ---- multi-GPU: CFG grid, the CFG-split window on 2 x R ranks (d4d_version() 114 and later) -------------------------
 * The CFG-split window with each CFG half frame-sharded over R ranks.  One process per GPU, world = 2R with R in
 * {1, 2, 3, 4}: global rank g runs CFG half k = g / R (ranks 0 .. R-1 the negative half) on frame shard r = g % R, frames
 * [r*F/R, (r+1)*F/R) of the window.  At each 3-D attention layer the rank's fused-QKV GEMM epilogue stores its K|V rows
 * into the gathered K/V buffers of the R ranks of its half only (the frame-sharded window's scatter, within the half); the
 * output permute stores the rank's noise [F/R,out_channels,h,w] at rows [k*F + r*F/R, k*F + (r+1)*F/R) of EVERY rank's
 * exchange buffer.  One flag round publishes the noise; then every rank runs the unchanged CFG + scheduler step of
 * d4d_denoise_window on the whole window, reading the gathered [2F] noise in place, as in the CFG split.  Every flag round,
 * those of the K/V layers included, waits for all 2R ranks.
 *   - Arguments, SPMD rules, guidance_scale <= 1 and the whole-window state are those of the *_cfg_split counterpart;
 *     results are bit-identical to the single-GPU call on every rank.
 *   - With R = 1 (world 1 or 2) the call is the CFG-split window, the same code and the same bits.
 *   - Returns 1 before any launch for a world other than 1, 2, 4, 6 or 8; with guidance_scale > 1, for F not divisible by
 *     R, or an exchange buffer (kv_bytes of d4d_exchange_alloc) smaller than the larger of 2 * F * out_channels * h * w
 *     bf16 and, for R > 1, one CFG half's largest 3-D K|V layer at F frames (sharded.exchange_bytes with one half). */
int d4d_denoise_window_cfg_grid(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                const d4d_sched* sched, float guidance_scale, int domain, int F, int height, int width,
                                int num_steps, void* stream);
int d4d_denoise_window_dpm_cfg_grid(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                    const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                    const d4d_dpm_sched* sched, float guidance_scale, int domain, int F, int height,
                                    int width, int num_steps, void* x0_prev, int32_t* lower_order_nums, void* stream);
int d4d_denoise_window_unipc_cfg_grid(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                      const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                      const d4d_unipc_sched* sched, float guidance_scale, int domain, int F, int height,
                                      int width, int num_steps, void* x0_prev, void* x0_prev2, void* last_sample,
                                      int32_t* lower_order_nums, void* stream);
int d4d_denoise_window_pndm_cfg_grid(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                     const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                     const d4d_pndm_sched* sched, float guidance_scale, int domain, int F, int height,
                                     int width, int num_steps, void* ets0, void* ets1, void* ets2, void* ets3,
                                     void* cur_sample, int32_t* counter, void* stream);
int d4d_denoise_window_deis_cfg_grid(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                     const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                     const d4d_deis_sched* sched, float guidance_scale, int domain, int F, int height,
                                     int width, int num_steps, void* m_prev, void* m_prev2, int32_t* lower_order_nums,
                                     void* stream);
int d4d_denoise_window_dpm_single_cfg_grid(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                           const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                           const d4d_dpm_single_sched* sched, float guidance_scale, int domain, int F,
                                           int height, int width, int num_steps, void* x0_prev, void* x0_prev2,
                                           void* cur_sample, int32_t* lower_order_nums, void* stream);
/* (d4d_version() 115 and later) frame_ids [F]: the whole window's, as d4d_denoise_window_ddpm */
int d4d_denoise_window_ddpm_cfg_grid(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                     const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                     const d4d_ddpm_sched* sched, float guidance_scale, int domain, int F, int height,
                                     int width, int num_steps, const int64_t* frame_ids, void* stream);

/* ---- multi-GPU: the UNet alone on the CFG split and the CFG grid (d4d_version() 116 and later) ------------------------
 * B-2 (a drop-in pipeline.unet) on the ranks of the CFG split or grid, for callers that run their own scheduler loop.  The
 * arguments are d4d_unet_forward's, and so is the result: every rank gets the whole noise out [B, out_channels, h, w].
 *   - n_domains == 2: the reference's CFG batch, [F negative | F positive] images, half k of domain domain_ids[k].  Rank g
 *     forwards rows [k*F + r*F/R, k*F + (r+1)*F/R) of sample, timestep and skeletons (k, r and R as for the CFG grid; the
 *     split is R = 1; a loopback, world 1, forwards all 2F rows) and stores their noise into every rank's exchange buffer;
 *     one flag round publishes it, and the gathered noise is copied into out.  The negative half's skeletons are the
 *     caller's rows, not assumed constant.  Needs d4d_exchange_open first.
 *   - n_domains == 1: no CFG halves; every rank runs d4d_unet_forward on the whole batch and exchanges nothing.
 *   - SPMD: every rank makes the same calls with the same (whole-batch) arguments; the result is bit-identical to
 *     d4d_unet_forward on one GPU on every rank.
 *   - Returns 1 before any launch for n_domains other than 1 or 2, B != n_domains * F, a world the mode does not run
 *     (split: 1 or 2; grid: 1, 2, 4, 6 or 8), and with n_domains == 2 for F not divisible by R or noise
 *     (2 * F * out_channels * h * w bf16) larger than the exchange buffer. */
int d4d_unet_forward_cfg_split(d4d_handle* h, const void* sample, const int64_t* timestep, const void* skeletons,
                               const int32_t* domain_ids, int n_domains, int B, int F, int height, int width, void* out,
                               void* stream);
int d4d_unet_forward_cfg_grid(d4d_handle* h, const void* sample, const int64_t* timestep, const void* skeletons,
                              const int32_t* domain_ids, int n_domains, int B, int F, int height, int width, void* out,
                              void* stream);

#ifdef __cplusplus
}
#endif
#endif /* D4D_H_ */
