// C ABI of libd4d.so (see include/d4d.h).  Thin, exception-safe wrappers: no torch types, plain pointers.
#include <new>
#include <stdexcept>

#include "unet.h"

namespace d4d {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
int nhwc_to_nchw_run(const bf16* x, int ld, int n, int C, int hw, bf16* out, cudaStream_t stream);
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
// scratch for the op-level GroupNorm entry point (per thread, grown on demand)
float* gn_scratch(size_t floats) {
  static thread_local float* p = nullptr;
  static thread_local size_t cap = 0;
  if (floats > cap) {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    if (cudaMalloc(&p, floats * sizeof(float)) != cudaSuccess) return nullptr;
    if (cudaMemset(p, 0, floats * sizeof(float)) != cudaSuccess) return nullptr;
    cap = floats;
  }
  return p;
}
}  // namespace

extern "C" {

const char* d4d_last_error(void) { return d4d::g_last_error.c_str(); }
int d4d_version(void) { return 100; }

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
  D4D_API_BEGIN
  D4D_REQUIRE(h != nullptr, "null handle");
  DeviceGuard g(h->model->device());
  return h->model->forward(static_cast<const bf16*>(sample), reinterpret_cast<const long long*>(timestep),
                           static_cast<const bf16*>(skeletons), domain_ids, n_domains, B, F, height, width,
                           static_cast<bf16*>(out), static_cast<cudaStream_t>(stream));
  D4D_API_END
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
  D4D_API_BEGIN
  D4D_REQUIRE(h != nullptr && sched != nullptr, "null argument");
  DeviceGuard g(h->model->device());
  return h->model->denoise_window(static_cast<bf16*>(latents), static_cast<const bf16*>(pixel_latents),
                                  static_cast<const bf16*>(plucker), static_cast<const bf16*>(skeletons),
                                  static_cast<const bf16*>(cond_mask), reinterpret_cast<long long*>(timestep_indices),
                                  *sched, guidance_scale, domain, F, height, width, num_steps,
                                  static_cast<cudaStream_t>(stream));
  D4D_API_END
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
  D4D_REQUIRE(noise && latents && cond_mask && timestep_indices && timestep_indices_out && sched && latents_out,
              "null argument");
  D4D_REQUIRE(timestep_indices != timestep_indices_out, "timestep_indices_out must not alias timestep_indices");
  d4d::DdimArgs d;
  const int hw = height * width;
  d.noise = static_cast<const bf16*>(noise); d.latents = static_cast<const bf16*>(latents);
  d.mask = static_cast<const bf16*>(cond_mask);
  d.timestep_indices = reinterpret_cast<const long long*>(timestep_indices);
  d.timesteps_table = reinterpret_cast<const long long*>(sched->timesteps_table);
  d.alphas_cumprod = sched->alphas_cumprod;
  d.n_steps = sched->n_steps; d.T = sched->num_train_timesteps; d.final_alpha_cumprod = sched->final_alpha_cumprod;
  d.F = F; d.chw = 4 * hw; d.hw = hw; d.cfg = cfg; d.guidance = guidance_scale;
  d.prediction_type = sched->prediction_type; d.clip_sample = sched->clip_sample; d.clip_range = sched->clip_sample_range;
  d.emulate_bf16 = sched->emulate_bf16; d.out = static_cast<bf16*>(latents_out);
  return d4d::cfg_ddim_step_run(d, reinterpret_cast<long long*>(timestep_indices_out), static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_op_gemm(const void* A, int lda, int K1, const void* A2, int lda2, int K2, const void* W, int M, int N,
                const float* bias, const void* rowvec, int ld_rowvec, int rows_per_image, const void* residual,
                int ld_res, void* out, int ldo, int geglu, int act, float out_scale, int block_n, void* stream) {
  D4D_API_BEGIN
  d4d::GemmDesc d;
  d.A = static_cast<const bf16*>(A); d.lda = lda; d.K1 = K1;
  d.A2 = static_cast<const bf16*>(A2); d.lda2 = lda2; d.K2 = K2;
  d.Wt = static_cast<const bf16*>(W); d.M = M; d.N = N; d.bias = bias;
  d.rowvec = static_cast<const bf16*>(rowvec); d.ld_rowvec = ld_rowvec; d.rows_per_image = rows_per_image;
  d.residual = static_cast<const bf16*>(residual); d.ld_res = ld_res;
  d.out = static_cast<bf16*>(out); d.ldo = ldo; d.geglu = geglu; d.act = act; d.out_scale = out_scale; d.block_n = block_n;
  D4D_REQUIRE(M > 0, "empty GEMM");
  d4d::GemmLaunch L;
  if (int rc = d4d::gemm_prepare(d, &L)) return rc;
  return d4d::gemm_run(L, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_op_conv3x3(const void* x_nhwc, int n_img, int H, int W, int Cin, const void* Wt, int Cout, const float* bias,
                   const void* rowvec, int ld_rowvec, const void* residual, int act, void* out, int block_n,
                   void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(n_img > 0 && H > 0 && W > 0, "empty conv");
  d4d::GemmDesc d;
  d.conv = 1; d.A = static_cast<const bf16*>(x_nhwc); d.n_img = n_img; d.H = H; d.W = W; d.Cin = Cin;
  d.Wt = static_cast<const bf16*>(Wt); d.N = Cout; d.bias = bias;
  d.rowvec = static_cast<const bf16*>(rowvec); d.ld_rowvec = ld_rowvec;
  d.residual = static_cast<const bf16*>(residual); d.ld_res = Cout;
  d.out = static_cast<bf16*>(out); d.ldo = Cout; d.act = act; d.block_n = block_n;
  d4d::GemmLaunch L;
  if (int rc = d4d::gemm_prepare(d, &L)) return rc;
  return d4d::gemm_run(L, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_op_attention(const void* q, const void* k, const void* v, int ld_qkv, void* out, int ld_out, int batch, int seq,
                     int heads, int head_dim, float scale, void* stream) {
  D4D_API_BEGIN
  d4d::AttnDesc d;
  d.q = static_cast<const bf16*>(q); d.k = static_cast<const bf16*>(k); d.v = static_cast<const bf16*>(v);
  d.ld_qkv = ld_qkv; d.out = static_cast<bf16*>(out); d.ld_out = ld_out;
  d.batch = batch; d.seq = seq; d.heads = heads; d.head_dim = head_dim; d.scale = scale;
  d4d::AttnLaunch L;
  if (int rc = d4d::attn_prepare(d, &L)) return rc;
  return d4d::attn_run(L, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_op_groupnorm(const void* x1, int C1, const void* x2, int C2, int n_img, int hw, int groups, float eps,
                     const float* gamma, const float* beta, int silu, void* out, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(n_img > 0 && hw > 0 && groups > 0, "empty GroupNorm");
  float* part = gn_scratch(d4d::groupnorm_scratch_floats(n_img, groups));
  if (!part) {
    d4d::set_error("GroupNorm scratch allocation failed");
    return 2;
  }
  // the arrival counters live behind the (n_img-dependent) partial/final regions: zero them for this shape
  const size_t ctr_off = static_cast<size_t>(n_img) * 32 * groups * 2 + static_cast<size_t>(n_img) * groups * 2;
  D4D_CUDA_OK(cudaMemsetAsync(part + ctr_off, 0, sizeof(unsigned int) * n_img, static_cast<cudaStream_t>(stream)));
  return d4d::groupnorm_run(static_cast<const bf16*>(x1), C1, static_cast<const bf16*>(x2), C2, n_img, hw, groups, eps,
                            gamma, beta, silu, static_cast<bf16*>(out), part, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_op_conv_resample(const void* x_nhwc, int n_img, int H, int W, int Cin, const void* Wt, int Cout, const float* bias,
                         int kind, int up_a, int up_b, void* out, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(n_img > 0 && H > 0 && W > 0 && kind >= 1 && kind <= 3, "conv_resample arguments");
  d4d::GemmDesc d;
  d.conv = 1; d.conv_kind = kind; d.up_a = up_a; d.up_b = up_b;
  d.A = static_cast<const bf16*>(x_nhwc); d.n_img = n_img; d.H = H; d.W = W; d.Cin = Cin;
  d.Wt = static_cast<const bf16*>(Wt); d.N = Cout; d.bias = bias;
  d.out = static_cast<bf16*>(out); d.ldo = Cout;
  d4d::GemmLaunch L;
  if (int rc = d4d::gemm_prepare(d, &L)) return rc;
  return d4d::gemm_run(L, static_cast<cudaStream_t>(stream));
  D4D_API_END
}

int d4d_op_conv3x3_groupnorm(const void* x_nhwc, int n_img, int H, int W, int Cin, const void* Wt, int Cout, const float* bias,
                             const void* residual, int groups, float eps, const float* gamma, const float* beta, int silu,
                             void* conv_out, void* gn_out, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(n_img > 0 && H > 0 && W > 0 && groups > 0, "empty conv");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t floats = static_cast<size_t>(n_img) * Cout * 2 * 2;  // [n_img][Cout][2] 64-bit {sum, sumsq}
  // accumulated by the conv epilogue; lives behind the stand-alone kernel's scratch (16-byte aligned for the 128-bit loads)
  const size_t off = (d4d::groupnorm_scratch_floats(n_img, groups) + 3) & ~size_t(3);
  float* base = gn_scratch(off + floats);
  if (!base) {
    d4d::set_error("GroupNorm scratch allocation failed");
    return 2;
  }
  long long* stats = reinterpret_cast<long long*>(base + off);
  D4D_CUDA_OK(cudaMemsetAsync(stats, 0, floats * sizeof(float), st));
  d4d::GemmDesc d;
  d.conv = 1; d.A = static_cast<const bf16*>(x_nhwc); d.n_img = n_img; d.H = H; d.W = W; d.Cin = Cin;
  d.Wt = static_cast<const bf16*>(Wt); d.N = Cout; d.bias = bias;
  d.residual = static_cast<const bf16*>(residual); d.ld_res = Cout;
  d.out = static_cast<bf16*>(conv_out); d.ldo = Cout;
  d.stats = stats;
  d4d::GemmLaunch L;
  if (int rc = d4d::gemm_prepare(d, &L)) return rc;
  if (int rc = d4d::gemm_run(L, st)) return rc;
  return d4d::groupnorm_apply_run(static_cast<const bf16*>(conv_out), Cout, stats, nullptr, 0, nullptr, n_img, H * W, groups, eps,
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
  D4D_API_BEGIN
  D4D_REQUIRE(h != nullptr, "null handle");
  DeviceGuard g(h->model->device());
  return h->model->forward(static_cast<const bf16*>(sample), reinterpret_cast<const long long*>(timestep),
                           static_cast<const bf16*>(skeletons), domain_ids, n_domains, B_local, F_local, height, width,
                           static_cast<bf16*>(out), static_cast<cudaStream_t>(stream), F_total);
  D4D_API_END
}

int d4d_denoise_window_sharded(d4d_handle* h, void* latents, const void* pixel_latents, const void* plucker,
                               const void* skeletons, const void* cond_mask, int64_t* timestep_indices,
                               const d4d_sched* sched, float guidance_scale, int domain, int F_local, int F_total,
                               int height, int width, int num_steps, void* stream) {
  D4D_API_BEGIN
  D4D_REQUIRE(h != nullptr && sched != nullptr, "null argument");
  DeviceGuard g(h->model->device());
  return h->model->denoise_window(static_cast<bf16*>(latents), static_cast<const bf16*>(pixel_latents),
                                  static_cast<const bf16*>(plucker), static_cast<const bf16*>(skeletons),
                                  static_cast<const bf16*>(cond_mask), reinterpret_cast<long long*>(timestep_indices),
                                  *sched, guidance_scale, domain, F_local, height, width, num_steps,
                                  static_cast<cudaStream_t>(stream), F_total);
  D4D_API_END
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
