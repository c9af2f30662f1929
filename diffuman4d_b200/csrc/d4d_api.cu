// C ABI of libd4d.so (see include/d4d.h).  Thin, exception-safe wrappers: no torch types, plain pointers.
#include <new>
#include <stdexcept>

#include "unet.h"

namespace d4d {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
}  // namespace d4d

struct d4d_handle {
  d4d::Model* model;
};

using d4d::bf16;

#define D4D_API_BEGIN try {
#define D4D_API_END                                        \
  }                                                        \
  catch (const std::bad_alloc&) {                          \
    d4d::set_error("out of host memory");                  \
    return 2;                                              \
  }                                                        \
  catch (const std::exception& e) {                        \
    d4d::set_error(std::string("internal error: ") + e.what()); \
    return 2;                                              \
  }

namespace {
struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; prev = -1; }
    if (ok && prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

// d4d_unet_forward and d4d_unet_forward_sharded; F_total = 0 runs the single-GPU plan
int unet_forward(d4d_handle* h, const void* sample, const int64_t* timestep, const void* skeletons,
                 const int32_t* domain_ids, int n_domains, int B, int F, int F_total, int height, int width, void* out,
                 void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(h != nullptr, "null handle");
  DeviceGuard g(h->model->device());
  return h->model->forward(static_cast<const bf16*>(sample), reinterpret_cast<const long long*>(timestep),
                           static_cast<const bf16*>(skeletons), domain_ids, n_domains, B, F, height, width,
                           static_cast<bf16*>(out), static_cast<cudaStream_t>(stream), F_total);
  D4D_API_END
}

// every d4d_denoise_window* entry point: `step` names the scheduler table and the frames' solver state; F_total = 0 runs
// the single-GPU plan; mode kSplit runs this rank's CFG half (the *_cfg_split entry points), kGrid its frame shard of
// its CFG half (the *_cfg_grid entry points)
int denoise_window(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker, const void* skeletons,
                   const void* cond_mask, int64_t* timestep_indices, const d4d::WindowStep& step, float guidance_scale,
                   int domain, int F, int F_total, int height, int width, int num_steps, void* stream,
                   d4d::CfgMode mode = d4d::CfgMode::kWhole) {
  D4D_API_BEGIN
  D4D_REQUIRE(h != nullptr && step.tables() > 0, "null argument");
  DeviceGuard g(h->model->device());
  return h->model->denoise_window(static_cast<bf16*>(latents), static_cast<const bf16*>(pixel_latents),
                                  static_cast<const bf16*>(plucker), static_cast<const bf16*>(skeletons),
                                  static_cast<const bf16*>(cond_mask), reinterpret_cast<long long*>(timestep_indices),
                                  step, guidance_scale, domain, F, height, width, num_steps,
                                  static_cast<cudaStream_t>(stream), F_total, mode);
  D4D_API_END
}

d4d::WindowStep ddim_step(const d4d_sched* sched) {
  d4d::WindowStep s;
  s.ddim = sched;
  return s;
}

d4d::WindowStep dpm_step(const d4d_dpm_sched* sched, void* x0_prev, int32_t* lower_order_nums) {
  d4d::WindowStep s;
  s.dpm = sched;
  s.state.x0_prev = static_cast<bf16*>(x0_prev);
  s.state.lower_order_nums = s.state.lower_order_nums_out = lower_order_nums;
  return s;
}

d4d::WindowStep unipc_step(const d4d_unipc_sched* sched, void* x0_prev, void* x0_prev2, void* last_sample,
                           int32_t* lower_order_nums) {
  d4d::WindowStep s;
  s.unipc = sched;
  s.state.x0_prev = static_cast<bf16*>(x0_prev); s.state.x0_prev2 = static_cast<bf16*>(x0_prev2);
  s.state.last_sample = static_cast<bf16*>(last_sample);
  s.state.lower_order_nums = s.state.lower_order_nums_out = lower_order_nums;
  return s;
}

// the PNDM state of d4d_denoise_window_pndm / d4d_cfg_pndm_step (the counter arrays are set by the caller)
d4d::SolverState pndm_state(void* ets0, void* ets1, void* ets2, void* ets3, void* cur_sample) {
  d4d::SolverState st;
  void* const ets[4] = {ets0, ets1, ets2, ets3};
  for (int i = 0; i < 4; ++i) st.ets[i] = static_cast<bf16*>(ets[i]);
  st.cur_sample = static_cast<bf16*>(cur_sample);
  return st;
}

d4d::WindowStep pndm_step(const d4d_pndm_sched* sched, void* ets0, void* ets1, void* ets2, void* ets3, void* cur_sample,
                          int32_t* counter) {
  d4d::WindowStep s;
  s.pndm = sched;
  s.state = pndm_state(ets0, ets1, ets2, ets3, cur_sample);
  s.state.lower_order_nums = s.state.lower_order_nums_out = counter;
  return s;
}

d4d::WindowStep deis_step(const d4d_deis_sched* sched, void* m_prev, void* m_prev2, int32_t* lower_order_nums) {
  d4d::WindowStep s;
  s.deis = sched;
  s.state.m_prev = static_cast<bf16*>(m_prev); s.state.m_prev2 = static_cast<bf16*>(m_prev2);
  s.state.lower_order_nums = s.state.lower_order_nums_out = lower_order_nums;
  return s;
}

d4d::WindowStep dpm_single_step(const d4d_dpm_single_sched* sched, void* x0_prev, void* x0_prev2, void* cur_sample,
                                int32_t* lower_order_nums) {
  d4d::WindowStep s;
  s.dpm_single = sched;
  s.state.x0_prev = static_cast<bf16*>(x0_prev); s.state.x0_prev2 = static_cast<bf16*>(x0_prev2);
  s.state.cur_sample = static_cast<bf16*>(cur_sample);
  s.state.lower_order_nums = s.state.lower_order_nums_out = lower_order_nums;
  return s;
}

// the step arguments of every d4d_cfg_*_step entry point
d4d::StepArgs step_args(const void* noise, const void* latents, const void* cond_mask, const int64_t* timestep_indices,
                        int64_t* timestep_indices_out, float guidance_scale, int cfg, int F, int height, int width,
                        void* latents_out) {
  d4d::StepArgs a;
  const int hw = height * width;
  a.noise = static_cast<const bf16*>(noise); a.latents = static_cast<const bf16*>(latents);
  a.mask = static_cast<const bf16*>(cond_mask);
  a.timestep_indices = reinterpret_cast<const long long*>(timestep_indices);
  a.F = F; a.chw = 4 * hw; a.hw = hw; a.cfg = cfg; a.guidance = guidance_scale;
  a.out = static_cast<bf16*>(latents_out);
  a.ts_out = reinterpret_cast<long long*>(timestep_indices_out);
  return a;
}
}  // namespace

extern "C" {

const char* d4d_last_error(void) { return d4d::g_last_error.c_str(); }
int d4d_version(void) { return 114; }

int d4d_create(const d4d_config* cfg, int device, d4d_handle** out) {
  D4D_API_BEGIN
  D4D_REQUIRE(cfg != nullptr && out != nullptr, "null argument");
  *out = nullptr;
  D4D_REQUIRE(cfg->layers_per_block >= 1 && cfg->layers_per_block <= 4, "layers_per_block");
  D4D_REQUIRE(cfg->out_channels >= 1 && cfg->out_channels <= 16, "out_channels must be in [1,16]");
  D4D_REQUIRE(cfg->in_channels >= 1 && cfg->in_channels <= 16, "in_channels must be in [1,16]");
  D4D_REQUIRE(cfg->norm_num_groups >= 1 && cfg->norm_num_groups <= 64, "norm_num_groups");
  for (int i = 0; i < 4; ++i) {
    const int c = cfg->block_out_channels[i], hds = cfg->num_heads[i];
    D4D_REQUIRE(c > 0 && c % 64 == 0, "block_out_channels must be positive multiples of 64");
    D4D_REQUIRE(c % cfg->norm_num_groups == 0, "channels must be divisible by norm_num_groups");
    D4D_REQUIRE(hds > 0 && c % hds == 0, "channels must be divisible by the number of heads");
    D4D_REQUIRE(c / hds <= 192 && (c / hds) % 8 == 0, "head_dim must be a multiple of 8 and <= 192");
  }
  int ndev = 0;
  D4D_CUDA_OK(cudaGetDeviceCount(&ndev));
  D4D_REQUIRE(device >= 0 && device < ndev, "device index out of range");
  cudaDeviceProp prop;
  D4D_CUDA_OK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    d4d::set_error("libd4d requires an sm_90a (Hopper H100) device; found compute capability " +
                   std::to_string(prop.major) + "." + std::to_string(prop.minor));
    return 2;
  }
  d4d_handle* h = new d4d_handle();
  h->model = new d4d::Model(*cfg, device);
  *out = h;
  return 0;
  D4D_API_END
}

void d4d_destroy(d4d_handle* h) {
  if (!h) return;
  try {
    delete h->model;
  } catch (...) {
  }
  delete h;
}

int d4d_load_weight(d4d_handle* h, const char* key, const void* data, const int64_t* shape, int ndim, int dtype) {
  D4D_API_BEGIN
  D4D_REQUIRE(h != nullptr, "null handle");
  return h->model->load_weight(key, data, shape, ndim, dtype);
  D4D_API_END
}

int d4d_finalize_weights(d4d_handle* h) {
  D4D_API_BEGIN
  D4D_REQUIRE(h != nullptr, "null handle");
  DeviceGuard g(h->model->device());
  return h->model->finalize();
  D4D_API_END
}

int d4d_num_weights(d4d_handle* h) { return h ? static_cast<int>(h->model->keys().size()) : 0; }
const char* d4d_weight_key(d4d_handle* h, int i) {
  if (!h || i < 0 || i >= static_cast<int>(h->model->keys().size())) return nullptr;
  return h->model->keys()[i].c_str();
}

int d4d_unet_forward(d4d_handle* h, const void* sample, const int64_t* timestep, const void* skeletons,
                     const int32_t* domain_ids, int n_domains, int B, int F, int height, int width, void* out,
                     void* stream) {
  return unet_forward(h, sample, timestep, skeletons, domain_ids, n_domains, B, F, 0, height, width, out, stream);
}

int d4d_profile_forward(d4d_handle* h, const void* sample, const int64_t* timestep, const void* skeletons,
                        const int32_t* domain_ids, int n_domains, int B, int F, int height, int width, void* out,
                        void* stream, float* ms_by_kind, int32_t* launches_by_kind, double* flops_by_kind) {
  D4D_API_BEGIN
  D4D_REQUIRE(h != nullptr, "null handle");
  DeviceGuard g(h->model->device());
  return h->model->profile(static_cast<const bf16*>(sample), reinterpret_cast<const long long*>(timestep),
                           static_cast<const bf16*>(skeletons), domain_ids, n_domains, B, F, height, width,
                           static_cast<bf16*>(out), static_cast<cudaStream_t>(stream), ms_by_kind, launches_by_kind,
                           flops_by_kind);
  D4D_API_END
}

int d4d_workspace_bytes(d4d_handle* h, int n_domains, int B, int F, int height, int width, size_t* bytes) {
  D4D_API_BEGIN
  D4D_REQUIRE(h != nullptr && bytes != nullptr, "null argument");
  d4d::Plan* p = h->model->find_plan(n_domains, B, F, height, width);
  *bytes = p ? p->arena_bytes : 0;
  return 0;
  D4D_API_END
}

int d4d_forward_launches(d4d_handle* h, int n_domains, int B, int F, int height, int width, int* launches) {
  D4D_API_BEGIN
  D4D_REQUIRE(h != nullptr && launches != nullptr, "null argument");
  d4d::Plan* p = h->model->find_plan(n_domains, B, F, height, width);
  *launches = p ? p->launches : 0;
  return 0;
  D4D_API_END
}

int d4d_denoise_window(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                       const void* skeletons, const void* cond_mask, int64_t* timestep_indices, const d4d_sched* sched,
                       float guidance_scale, int domain, int F, int height, int width, int num_steps, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices, ddim_step(sched),
                        guidance_scale, domain, F, 0, height, width, num_steps, stream);
}

int d4d_denoise_window_dpm(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                           const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                           const d4d_dpm_sched* sched, float guidance_scale, int domain, int F, int height, int width,
                           int num_steps, void* x0_prev, int32_t* lower_order_nums, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        dpm_step(sched, x0_prev, lower_order_nums), guidance_scale, domain, F, 0, height, width, num_steps,
                        stream);
}

int d4d_denoise_window_unipc(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                             const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                             const d4d_unipc_sched* sched, float guidance_scale, int domain, int F, int height, int width,
                             int num_steps, void* x0_prev, void* x0_prev2, void* last_sample, int32_t* lower_order_nums,
                             void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        unipc_step(sched, x0_prev, x0_prev2, last_sample, lower_order_nums), guidance_scale, domain, F, 0,
                        height, width, num_steps, stream);
}

int d4d_denoise_window_pndm(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                            const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                            const d4d_pndm_sched* sched, float guidance_scale, int domain, int F, int height, int width,
                            int num_steps, void* ets0, void* ets1, void* ets2, void* ets3, void* cur_sample,
                            int32_t* counter, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        pndm_step(sched, ets0, ets1, ets2, ets3, cur_sample, counter), guidance_scale, domain, F, 0, height,
                        width, num_steps, stream);
}

int d4d_denoise_window_deis(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                            const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                            const d4d_deis_sched* sched, float guidance_scale, int domain, int F, int height, int width,
                            int num_steps, void* m_prev, void* m_prev2, int32_t* lower_order_nums, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        deis_step(sched, m_prev, m_prev2, lower_order_nums), guidance_scale, domain, F, 0, height, width,
                        num_steps, stream);
}

int d4d_denoise_window_dpm_single(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                  const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                  const d4d_dpm_single_sched* sched, float guidance_scale, int domain, int F, int height,
                                  int width, int num_steps, void* x0_prev, void* x0_prev2, void* cur_sample,
                                  int32_t* lower_order_nums, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        dpm_single_step(sched, x0_prev, x0_prev2, cur_sample, lower_order_nums), guidance_scale, domain, F,
                        0, height, width, num_steps, stream);
}

int d4d_assemble_input(void* latents, const void* pixel_latents, const void* plucker, const void* skel_latents,
                       const void* cond_mask, const int64_t* timestep_indices, const int64_t* timesteps_table,
                       int n_steps, int F, int height, int width, int cfg, void* sample_out, int64_t* timestep_out,
                       void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(latents && pixel_latents && plucker && cond_mask && timestep_indices && timesteps_table && sample_out &&
                  timestep_out, "null argument");
  d4d::AssembleArgs a;
  a.latents = static_cast<bf16*>(latents);
  a.pixel = static_cast<const bf16*>(pixel_latents);
  a.plucker = static_cast<const bf16*>(plucker);
  a.skel_latents = static_cast<const bf16*>(skel_latents);
  a.mask = static_cast<const bf16*>(cond_mask);
  a.timestep_indices = reinterpret_cast<const long long*>(timestep_indices);
  a.timesteps_table = reinterpret_cast<const long long*>(timesteps_table);
  a.n_steps = n_steps; a.F = F; a.h = height; a.w = width; a.cfg = cfg;
  a.sample = static_cast<bf16*>(sample_out);
  a.timestep_out = reinterpret_cast<long long*>(timestep_out);
  return d4d::assemble_input_run(a, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_cfg_ddim_step(const void* noise, const void* latents, const void* cond_mask, const int64_t* timestep_indices,
                      int64_t* timestep_indices_out, const d4d_sched* sched, float guidance_scale, int cfg, int F,
                      int height, int width, void* latents_out, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(sched != nullptr, "null argument");
  return d4d::cfg_step_run(step_args(noise, latents, cond_mask, timestep_indices, timestep_indices_out, guidance_scale, cfg,
                                     F, height, width, latents_out),
                           *sched, d4d::SolverState(), static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_cfg_dpm_step(const void* noise, const void* latents, const void* cond_mask, const int64_t* timestep_indices,
                     int64_t* timestep_indices_out, void* x0_prev, const int32_t* lower_order_nums,
                     int32_t* lower_order_nums_out, const d4d_dpm_sched* sched, float guidance_scale, int cfg, int F,
                     int height, int width, void* latents_out, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(sched != nullptr, "null argument");
  d4d::SolverState st;
  st.x0_prev = static_cast<bf16*>(x0_prev);
  st.lower_order_nums = lower_order_nums; st.lower_order_nums_out = lower_order_nums_out;
  return d4d::cfg_step_run(step_args(noise, latents, cond_mask, timestep_indices, timestep_indices_out, guidance_scale, cfg,
                                     F, height, width, latents_out),
                           *sched, st, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_cfg_unipc_step(const void* noise, const void* latents, const void* cond_mask, const int64_t* timestep_indices,
                       int64_t* timestep_indices_out, void* x0_prev, void* x0_prev2, void* last_sample,
                       const int32_t* lower_order_nums, int32_t* lower_order_nums_out, const d4d_unipc_sched* sched,
                       float guidance_scale, int cfg, int F, int height, int width, void* latents_out, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(sched != nullptr, "null argument");
  d4d::SolverState st;
  st.x0_prev = static_cast<bf16*>(x0_prev); st.x0_prev2 = static_cast<bf16*>(x0_prev2);
  st.last_sample = static_cast<bf16*>(last_sample);
  st.lower_order_nums = lower_order_nums; st.lower_order_nums_out = lower_order_nums_out;
  return d4d::cfg_step_run(step_args(noise, latents, cond_mask, timestep_indices, timestep_indices_out, guidance_scale, cfg,
                                     F, height, width, latents_out),
                           *sched, st, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_cfg_pndm_step(const void* noise, const void* latents, const void* cond_mask, const int64_t* timestep_indices,
                      int64_t* timestep_indices_out, void* ets0, void* ets1, void* ets2, void* ets3, void* cur_sample,
                      const int32_t* counter, int32_t* counter_out, const d4d_pndm_sched* sched, float guidance_scale,
                      int cfg, int F, int height, int width, void* latents_out, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(sched != nullptr, "null argument");
  d4d::SolverState st = pndm_state(ets0, ets1, ets2, ets3, cur_sample);
  st.lower_order_nums = counter; st.lower_order_nums_out = counter_out;
  return d4d::cfg_step_run(step_args(noise, latents, cond_mask, timestep_indices, timestep_indices_out, guidance_scale, cfg,
                                     F, height, width, latents_out),
                           *sched, st, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_cfg_deis_step(const void* noise, const void* latents, const void* cond_mask, const int64_t* timestep_indices,
                      int64_t* timestep_indices_out, void* m_prev, void* m_prev2, const int32_t* lower_order_nums,
                      int32_t* lower_order_nums_out, const d4d_deis_sched* sched, float guidance_scale, int cfg, int F,
                      int height, int width, void* latents_out, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(sched != nullptr, "null argument");
  d4d::SolverState st;
  st.m_prev = static_cast<bf16*>(m_prev); st.m_prev2 = static_cast<bf16*>(m_prev2);
  st.lower_order_nums = lower_order_nums; st.lower_order_nums_out = lower_order_nums_out;
  return d4d::cfg_step_run(step_args(noise, latents, cond_mask, timestep_indices, timestep_indices_out, guidance_scale, cfg,
                                     F, height, width, latents_out),
                           *sched, st, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_cfg_dpm_single_step(const void* noise, const void* latents, const void* cond_mask,
                            const int64_t* timestep_indices, int64_t* timestep_indices_out, void* x0_prev,
                            void* x0_prev2, void* cur_sample, const int32_t* lower_order_nums,
                            int32_t* lower_order_nums_out, const d4d_dpm_single_sched* sched, float guidance_scale,
                            int cfg, int F, int height, int width, void* latents_out, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(sched != nullptr, "null argument");
  d4d::SolverState st;
  st.x0_prev = static_cast<bf16*>(x0_prev); st.x0_prev2 = static_cast<bf16*>(x0_prev2);
  st.cur_sample = static_cast<bf16*>(cur_sample);
  st.lower_order_nums = lower_order_nums; st.lower_order_nums_out = lower_order_nums_out;
  return d4d::cfg_step_run(step_args(noise, latents, cond_mask, timestep_indices, timestep_indices_out, guidance_scale, cfg,
                                     F, height, width, latents_out),
                           *sched, st, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_op_gemm(const void* A, int lda, int K1, const void* A2, int lda2, int K2, const void* W, int M, int N,
                const float* bias, const void* rowvec, int ld_rowvec, int rows_per_image, const void* residual,
                int ld_res, void* out, int ldo, int geglu, int act, float out_scale, int block_n, int64_t* stats,
                int stats_rows, void* stream) {
  return d4d_op_gemm_tiled(A, lda, K1, A2, lda2, K2, W, M, N, bias, rowvec, ld_rowvec, rows_per_image, residual, ld_res, out,
                           ldo, geglu, act, out_scale, block_n, 0, stats, stats_rows, stream);
}

int d4d_op_gemm_tiled(const void* A, int lda, int K1, const void* A2, int lda2, int K2, const void* W, int M, int N,
                      const float* bias, const void* rowvec, int ld_rowvec, int rows_per_image, const void* residual,
                      int ld_res, void* out, int ldo, int geglu, int act, float out_scale, int block_n, int schedule,
                      int64_t* stats, int stats_rows, void* stream) {
  D4D_API_BEGIN
  d4d::GemmDesc d;
  d.A = static_cast<const bf16*>(A); d.lda = lda; d.K1 = K1;
  d.A2 = static_cast<const bf16*>(A2); d.lda2 = lda2; d.K2 = K2;
  d.Wt = static_cast<const bf16*>(W); d.M = M; d.N = N; d.bias = bias;
  d.rowvec = static_cast<const bf16*>(rowvec); d.ld_rowvec = ld_rowvec; d.rows_per_image = rows_per_image;
  d.residual = static_cast<const bf16*>(residual); d.ld_res = ld_res;
  d.out = static_cast<bf16*>(out); d.ldo = ldo; d.geglu = geglu; d.act = act; d.out_scale = out_scale; d.block_n = block_n;
  d.schedule = schedule;
  d.stats = reinterpret_cast<long long*>(stats); d.stats_rows = stats_rows;
  D4D_REQUIRE(M > 0, "empty GEMM");
  d4d::GemmLaunch L;
  if (int rc = d4d::gemm_prepare(d, &L)) return rc;
  return d4d::gemm_run(L, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_gemm_tile_choice(int M, int N, int K1, int K2, int geglu, int sms, int* block_n, int* schedule) {
  D4D_API_BEGIN
  D4D_REQUIRE(M > 0 && N > 0 && K1 > 0 && K2 >= 0 && sms > 0 && block_n && schedule, "gemm_tile_choice arguments");
  d4d::GemmDesc d;
  D4D_REQUIRE(K2 == 0 || K1 % 64 == 0, "two-source GEMM needs K1 % 64 == 0");
  d.M = M; d.N = N; d.K1 = K1 + K2; d.geglu = geglu;  // K1 % 64 == 0: the k-blocks of A | A2 are those of one source
  int block_m = 0;
  return d4d::gemm_choose_tile(d, sms, &block_m, block_n, schedule);
  D4D_API_END
}

int d4d_op_gemm_kv_scatter(const void* A, int lda, int K, const void* W, int M, int N, void* out, int ldo, int kv_col0,
                           int kv_ld, int64_t rows_local, int64_t rows_global, int64_t row_offset, int world,
                           void* const* kv_dst, int block_n, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(M > 0, "empty GEMM");
  D4D_REQUIRE(world >= 1 && world <= 8, "K/V scatter: world must be in [1, 8]");
  D4D_REQUIRE(kv_dst != nullptr, "K/V scatter: null destination buffer");
  // the descriptor of the frame-sharded QKV projection (PlanBuilder::sharded_qkv_attention, csrc/unet.cu)
  d4d::GemmDesc d;
  d.A = static_cast<const bf16*>(A); d.lda = lda; d.K1 = K; d.Wt = static_cast<const bf16*>(W); d.M = M; d.N = N;
  d.out = static_cast<bf16*>(out); d.ldo = ldo; d.block_n = block_n;
  d.kv_world = world; d.kv_col0 = kv_col0; d.kv_ld = kv_ld;
  d.kv_rows_local = rows_local; d.kv_rows_global = rows_global; d.kv_row_offset = row_offset;
  for (int r = 0; r < world; ++r) d.kv_dst[r] = static_cast<bf16*>(kv_dst[r]);
  d4d::GemmLaunch L;
  if (int rc = d4d::gemm_prepare(d, &L)) return rc;
  return d4d::gemm_run(L, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_op_conv3x3(const void* x_nhwc, int n_img, int H, int W, int Cin, const void* Wt, int Cout, const float* bias,
                   const void* rowvec, int ld_rowvec, const void* residual, int act, void* out, int block_n,
                   int64_t* stats, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(n_img > 0 && H > 0 && W > 0, "empty conv");
  d4d::GemmDesc d;
  d.conv = 1; d.A = static_cast<const bf16*>(x_nhwc); d.n_img = n_img; d.H = H; d.W = W; d.Cin = Cin;
  d.Wt = static_cast<const bf16*>(Wt); d.N = Cout; d.bias = bias;
  d.rowvec = static_cast<const bf16*>(rowvec); d.ld_rowvec = ld_rowvec;
  d.residual = static_cast<const bf16*>(residual); d.ld_res = Cout;
  d.out = static_cast<bf16*>(out); d.ldo = Cout; d.act = act; d.block_n = block_n;
  d.stats = reinterpret_cast<long long*>(stats);
  d4d::GemmLaunch L;
  if (int rc = d4d::gemm_prepare(d, &L)) return rc;
  return d4d::gemm_run(L, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_op_conv_tiled(const void* x_nhwc, int n_img, int H, int W, int Cin, const void* Wt, int Cout, const float* bias,
                      const void* rowvec, int ld_rowvec, const void* residual, int act, void* out, int kind, int block_m,
                      int block_n, int64_t* stats, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(n_img > 0 && H > 0 && W > 0 && (kind == 0 || kind == 1 || kind == 3), "conv_tiled arguments");
  d4d::GemmDesc d;
  d.conv = 1; d.conv_kind = kind; d.A = static_cast<const bf16*>(x_nhwc); d.n_img = n_img; d.H = H; d.W = W; d.Cin = Cin;
  d.Wt = static_cast<const bf16*>(Wt); d.N = Cout; d.bias = bias;
  d.rowvec = static_cast<const bf16*>(rowvec); d.ld_rowvec = ld_rowvec;
  d.residual = static_cast<const bf16*>(residual); d.ld_res = Cout;
  d.out = static_cast<bf16*>(out); d.ldo = Cout; d.act = act; d.block_m = block_m; d.block_n = block_n;
  d.stats = reinterpret_cast<long long*>(stats);
  d4d::GemmLaunch L;
  if (int rc = d4d::gemm_prepare(d, &L)) return rc;
  return d4d::gemm_run(L, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_conv_tile_choice(int n_img, int H, int W, int Cin, int Cout, int kind, int sms, int* block_m, int* block_n) {
  D4D_API_BEGIN
  D4D_REQUIRE(n_img > 0 && H > 0 && W > 0 && Cin > 0 && kind >= 0 && kind <= 3 && sms > 0 && block_m && block_n,
              "conv_tile_choice arguments");
  d4d::GemmDesc d;
  d.conv = 1; d.conv_kind = kind; d.n_img = n_img; d.H = H; d.W = W; d.Cin = Cin; d.N = Cout;
  return d4d::gemm_choose_tile(d, sms, block_m, block_n);
  D4D_API_END
}

int d4d_op_attention(const void* q, const void* k, const void* v, int ld_qkv, void* out, int ld_out, int batch, int seq,
                     int heads, int head_dim, float scale, int seq_kv, int ld_kv, void* stream) {
  D4D_API_BEGIN
  d4d::AttnDesc d;
  d.q = static_cast<const bf16*>(q); d.k = static_cast<const bf16*>(k); d.v = static_cast<const bf16*>(v);
  d.ld_qkv = ld_qkv; d.out = static_cast<bf16*>(out); d.ld_out = ld_out;
  d.batch = batch; d.seq = seq; d.heads = heads; d.head_dim = head_dim; d.scale = scale;
  d.seq_kv = seq_kv; d.ld_kv = ld_kv;
  d4d::AttnLaunch L;
  if (int rc = d4d::attn_prepare(d, &L)) return rc;
  return d4d::attn_run(L, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_op_groupnorm(const void* x1, int C1, const void* x2, int C2, int n_img, int hw, int groups, float eps,
                     const float* gamma, const float* beta, int silu, void* out, int64_t* stats, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(n_img > 0 && hw > 0 && groups > 0, "empty GroupNorm");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (x2 == nullptr) C2 = 0;
  long long* s1 = reinterpret_cast<long long*>(stats);
  long long* s2 = C2 > 0 ? s1 + static_cast<size_t>(n_img) * C1 * 2 : nullptr;
  if (int rc = d4d::groupnorm_stats_run(static_cast<const bf16*>(x1), C1, n_img, hw, s1, st)) return rc;
  if (C2 > 0) {
    if (int rc = d4d::groupnorm_stats_run(static_cast<const bf16*>(x2), C2, n_img, hw, s2, st)) return rc;
  }
  return d4d::groupnorm_apply_run(static_cast<const bf16*>(x1), C1, s1, static_cast<const bf16*>(x2), C2, s2, n_img, hw, groups,
                                  eps, gamma, beta, silu, static_cast<bf16*>(out), st);
  D4D_API_END
}

int d4d_op_conv_resample(const void* x_nhwc, int n_img, int H, int W, int Cin, const void* Wt, int Cout, const float* bias,
                         int kind, int up_a, int up_b, void* out, int64_t* stats, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(n_img > 0 && H > 0 && W > 0 && kind >= 1 && kind <= 3, "conv_resample arguments");
  d4d::GemmDesc d;
  d.conv = 1; d.conv_kind = kind; d.up_a = up_a; d.up_b = up_b;
  d.A = static_cast<const bf16*>(x_nhwc); d.n_img = n_img; d.H = H; d.W = W; d.Cin = Cin;
  d.Wt = static_cast<const bf16*>(Wt); d.N = Cout; d.bias = bias;
  d.out = static_cast<bf16*>(out); d.ldo = Cout;
  d.stats = reinterpret_cast<long long*>(stats);
  d4d::GemmLaunch L;
  if (int rc = d4d::gemm_prepare(d, &L)) return rc;
  return d4d::gemm_run(L, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_op_conv3x3_groupnorm(const void* x_nhwc, int n_img, int H, int W, int Cin, const void* Wt, int Cout, const float* bias,
                             const void* residual, int groups, float eps, const float* gamma, const float* beta, int silu,
                             void* conv_out, void* gn_out, int64_t* stats, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(n_img > 0 && H > 0 && W > 0 && groups > 0, "empty conv");
  D4D_REQUIRE(stats != nullptr, "null statistics workspace");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  d4d::GemmDesc d;
  d.conv = 1; d.A = static_cast<const bf16*>(x_nhwc); d.n_img = n_img; d.H = H; d.W = W; d.Cin = Cin;
  d.Wt = static_cast<const bf16*>(Wt); d.N = Cout; d.bias = bias;
  d.residual = static_cast<const bf16*>(residual); d.ld_res = Cout;
  d.out = static_cast<bf16*>(conv_out); d.ldo = Cout;
  d.stats = reinterpret_cast<long long*>(stats);
  d4d::GemmLaunch L;
  if (int rc = d4d::gemm_prepare(d, &L)) return rc;
  if (int rc = d4d::gemm_run(L, st)) return rc;
  return d4d::groupnorm_apply_run(static_cast<const bf16*>(conv_out), Cout, d.stats, nullptr, 0, nullptr, n_img, H * W, groups, eps,
                                  gamma, beta, silu, static_cast<bf16*>(gn_out), st);
  D4D_API_END
}

int d4d_op_layernorm(const void* x, int rows, int C, float eps, const float* gamma, const float* beta, void* out,
                     void* stream) {
  D4D_API_BEGIN
  return d4d::layernorm_run(static_cast<const bf16*>(x), rows, C, eps, gamma, beta, static_cast<bf16*>(out),
                            static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_op_pose_conv0(const void* x_nchw, int n, int H, int W, const void* Wt, const float* bias, void* out_nhwc4,
                      void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(n > 0 && H > 0 && W > 0, "empty pose conv");
  return d4d::pose_conv0_run(static_cast<const bf16*>(x_nchw), n, H, W, static_cast<const bf16*>(Wt), bias,
                             static_cast<bf16*>(out_nhwc4), static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_op_pose_conv(const void* x_nhwc, int n, int Cin, int H, int W, const void* Wt, const float* bias, int Cout,
                     int ksize, int stride, void* out, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(n > 0 && H > 0 && W > 0, "empty pose conv");
  return d4d::pose_conv_run(static_cast<const bf16*>(x_nhwc), n, Cin, H, W, static_cast<const bf16*>(Wt), bias, Cout,
                            ksize, stride, static_cast<bf16*>(out), static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_debug_tap(d4d_handle* h, const void* sample, const int64_t* timestep, const void* skeletons,
                  const int32_t* domain_ids, int n_domains, int B, int F, int height, int width, int tap, void* out,
                  char* name64, int32_t* dims3, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(h != nullptr, "null handle");
  DeviceGuard g(h->model->device());
  return h->model->debug_tap(static_cast<const bf16*>(sample), reinterpret_cast<const long long*>(timestep),
                             static_cast<const bf16*>(skeletons), domain_ids, n_domains, B, F, height, width, tap,
                             static_cast<bf16*>(out), name64, dims3, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_unet_forward_sharded(d4d_handle* h, const void* sample, const int64_t* timestep, const void* skeletons,
                             const int32_t* domain_ids, int n_domains, int B_local, int F_local, int F_total, int height,
                             int width, void* out, void* stream) {
  return unet_forward(h, sample, timestep, skeletons, domain_ids, n_domains, B_local, F_local, F_total, height, width,
                      out, stream);
}

int d4d_denoise_window_sharded(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                               const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                               const d4d_sched* sched, float guidance_scale, int domain, int F_local, int F_total,
                               int height, int width, int num_steps, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices, ddim_step(sched),
                        guidance_scale, domain, F_local, F_total, height, width, num_steps, stream);
}

int d4d_denoise_window_dpm_sharded(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                   const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                   const d4d_dpm_sched* sched, float guidance_scale, int domain, int F_local, int F_total,
                                   int height, int width, int num_steps, void* x0_prev, int32_t* lower_order_nums,
                                   void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        dpm_step(sched, x0_prev, lower_order_nums), guidance_scale, domain, F_local, F_total, height,
                        width, num_steps, stream);
}

int d4d_window_exchange(d4d_handle* h, const void* latents_local, const int64_t* timestep_indices_local,
                        const void* x0_prev_local, const int32_t* lower_order_nums_local, int F_local, int F_total,
                        int height, int width, void* latents_out, int64_t* timestep_indices_out, void* x0_prev_out,
                        int32_t* lower_order_nums_out, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(h != nullptr, "null handle");
  DeviceGuard g(h->model->device());
  return h->model->window_exchange(static_cast<const bf16*>(latents_local),
                                   reinterpret_cast<const long long*>(timestep_indices_local),
                                   static_cast<const bf16*>(x0_prev_local), lower_order_nums_local, F_local, F_total, height,
                                   width, static_cast<bf16*>(latents_out), reinterpret_cast<long long*>(timestep_indices_out),
                                   static_cast<bf16*>(x0_prev_out), lower_order_nums_out, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_op_window_scatter(const void* latents, const int64_t* timestep_indices, const void* x0_prev,
                          const int32_t* lower_order_nums, int F_local, int F_total, int height, int width, int world,
                          int rank, void* const* dst, size_t dst_bytes, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(world >= 1 && world <= 8, "window scatter: world must be in [1, 8]");
  D4D_REQUIRE(dst != nullptr, "window scatter: null destination buffer");
  D4D_REQUIRE(height > 0 && width > 0, "window scatter: latent height/width");
  d4d::WindowScatterArgs a;
  for (int r = 0; r < 8; ++r) a.dst[r] = r < world ? dst[r] : nullptr;
  a.world = world; a.rank = rank; a.F_local = F_local; a.F_total = F_total;
  a.chw = 4ll * height * width;
  a.latents = static_cast<const bf16*>(latents); a.ts = reinterpret_cast<const long long*>(timestep_indices);
  a.x0_prev = static_cast<const bf16*>(x0_prev); a.lower_order_nums = lower_order_nums;
  return d4d::window_scatter_run(a, dst_bytes, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_denoise_window_cfg_split(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                 const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                 const d4d_sched* sched, float guidance_scale, int domain, int F, int height, int width,
                                 int num_steps, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices, ddim_step(sched),
                        guidance_scale, domain, F, 0, height, width, num_steps, stream, d4d::CfgMode::kSplit);
}

int d4d_denoise_window_dpm_cfg_split(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                     const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                     const d4d_dpm_sched* sched, float guidance_scale, int domain, int F, int height,
                                     int width, int num_steps, void* x0_prev, int32_t* lower_order_nums, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        dpm_step(sched, x0_prev, lower_order_nums), guidance_scale, domain, F, 0, height, width, num_steps,
                        stream, d4d::CfgMode::kSplit);
}

int d4d_denoise_window_unipc_cfg_split(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                       const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                       const d4d_unipc_sched* sched, float guidance_scale, int domain, int F, int height,
                                       int width, int num_steps, void* x0_prev, void* x0_prev2, void* last_sample,
                                       int32_t* lower_order_nums, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        unipc_step(sched, x0_prev, x0_prev2, last_sample, lower_order_nums), guidance_scale, domain, F, 0,
                        height, width, num_steps, stream, d4d::CfgMode::kSplit);
}

int d4d_denoise_window_pndm_cfg_split(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                      const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                      const d4d_pndm_sched* sched, float guidance_scale, int domain, int F, int height,
                                      int width, int num_steps, void* ets0, void* ets1, void* ets2, void* ets3,
                                      void* cur_sample, int32_t* counter, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        pndm_step(sched, ets0, ets1, ets2, ets3, cur_sample, counter), guidance_scale, domain, F, 0, height,
                        width, num_steps, stream, d4d::CfgMode::kSplit);
}

int d4d_denoise_window_deis_cfg_split(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                      const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                      const d4d_deis_sched* sched, float guidance_scale, int domain, int F, int height,
                                      int width, int num_steps, void* m_prev, void* m_prev2, int32_t* lower_order_nums,
                                      void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        deis_step(sched, m_prev, m_prev2, lower_order_nums), guidance_scale, domain, F, 0, height, width,
                        num_steps, stream, d4d::CfgMode::kSplit);
}

int d4d_denoise_window_dpm_single_cfg_split(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                            const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                            const d4d_dpm_single_sched* sched, float guidance_scale, int domain, int F,
                                            int height, int width, int num_steps, void* x0_prev, void* x0_prev2,
                                            void* cur_sample, int32_t* lower_order_nums, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        dpm_single_step(sched, x0_prev, x0_prev2, cur_sample, lower_order_nums), guidance_scale, domain, F,
                        0, height, width, num_steps, stream, d4d::CfgMode::kSplit);
}

int d4d_denoise_window_cfg_grid(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                const d4d_sched* sched, float guidance_scale, int domain, int F, int height, int width,
                                int num_steps, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices, ddim_step(sched),
                        guidance_scale, domain, F, 0, height, width, num_steps, stream, d4d::CfgMode::kGrid);
}

int d4d_denoise_window_dpm_cfg_grid(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                    const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                    const d4d_dpm_sched* sched, float guidance_scale, int domain, int F, int height,
                                    int width, int num_steps, void* x0_prev, int32_t* lower_order_nums, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        dpm_step(sched, x0_prev, lower_order_nums), guidance_scale, domain, F, 0, height, width, num_steps,
                        stream, d4d::CfgMode::kGrid);
}

int d4d_denoise_window_unipc_cfg_grid(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                      const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                      const d4d_unipc_sched* sched, float guidance_scale, int domain, int F, int height,
                                      int width, int num_steps, void* x0_prev, void* x0_prev2, void* last_sample,
                                      int32_t* lower_order_nums, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        unipc_step(sched, x0_prev, x0_prev2, last_sample, lower_order_nums), guidance_scale, domain, F, 0,
                        height, width, num_steps, stream, d4d::CfgMode::kGrid);
}

int d4d_denoise_window_pndm_cfg_grid(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                     const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                     const d4d_pndm_sched* sched, float guidance_scale, int domain, int F, int height,
                                     int width, int num_steps, void* ets0, void* ets1, void* ets2, void* ets3,
                                     void* cur_sample, int32_t* counter, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        pndm_step(sched, ets0, ets1, ets2, ets3, cur_sample, counter), guidance_scale, domain, F, 0, height,
                        width, num_steps, stream, d4d::CfgMode::kGrid);
}

int d4d_denoise_window_deis_cfg_grid(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                     const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                     const d4d_deis_sched* sched, float guidance_scale, int domain, int F, int height,
                                     int width, int num_steps, void* m_prev, void* m_prev2, int32_t* lower_order_nums,
                                     void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        deis_step(sched, m_prev, m_prev2, lower_order_nums), guidance_scale, domain, F, 0, height, width,
                        num_steps, stream, d4d::CfgMode::kGrid);
}

int d4d_denoise_window_dpm_single_cfg_grid(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                                           const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                                           const d4d_dpm_single_sched* sched, float guidance_scale, int domain, int F,
                                           int height, int width, int num_steps, void* x0_prev, void* x0_prev2,
                                           void* cur_sample, int32_t* lower_order_nums, void* stream) {
  return denoise_window(h, latents, pixel_latents, plucker, skeletons, cond_mask, timestep_indices,
                        dpm_single_step(sched, x0_prev, x0_prev2, cur_sample, lower_order_nums), guidance_scale, domain, F,
                        0, height, width, num_steps, stream, d4d::CfgMode::kGrid);
}

int d4d_exchange_alloc(d4d_handle* h, size_t kv_bytes, unsigned char* handles_out) {
  D4D_API_BEGIN
  D4D_REQUIRE(h != nullptr, "null handle");
  DeviceGuard g(h->model->device());
  return h->model->exchange_alloc(kv_bytes, handles_out);
  D4D_API_END
}

int d4d_exchange_open(d4d_handle* h, int rank, int world, const unsigned char* all_handles) {
  D4D_API_BEGIN
  D4D_REQUIRE(h != nullptr, "null handle");
  DeviceGuard g(h->model->device());
  return h->model->exchange_open(rank, world, all_handles);
  D4D_API_END
}

}  // extern "C"
