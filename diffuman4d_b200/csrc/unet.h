// UNet executor: weights (diffusers key contract), per-shape launch plans, window denoise step.
#pragma once
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/d4d.h"
#include "kernels.h"

namespace d4d {

struct HostTensor {
  std::vector<float> v;
  std::vector<int64_t> shape;
};

struct NormW { float* g = nullptr; float* b = nullptr; int c = 0; };
struct LinW { bf16* w = nullptr; float* b = nullptr; int in = 0, out = 0; };
struct ResnetW {
  NormW n1, n2;
  LinW c1, c2;   // conv3x3 weights [Cout][9][Cin]; in = Cin, out = Cout
  LinW sc;       // 1x1 shortcut (w == nullptr when Cin == Cout)
  int temb_off = 0;
  int cin = 0, cout = 0;
};
struct AttnW { LinW qkv, out; };
struct XfW {
  NormW gn, ln1, ln2, ln3;
  LinW pin, pout, ff1, ff2;
  AttnW a1, a2;
  bool has2 = false;
  int C = 0, heads = 0, d = 0, dpad = 0;
};
struct PoseW {
  LinW conv[8];   // layers 0..5 direct layout [k*k][Cin][Cout]; 5 -> GEMM layout [Cout][16*Cin]; 6,7 conv3x3 layout
  LinW proj;      // [C0][128]
  float scale = 1.f;
};

struct Plan {
  int n_domains = 0, B = 0, F = 0, h = 0, w = 0;
  std::vector<int> domains;
  void* arena = nullptr;
  size_t arena_bytes = 0;
  int launches = 0;
  // frame-sharded window (DESIGN.md section 7): this rank owns F of F_total frames per CFG half
  int F_total = 0, rank = 0, world = 1;
  bool pose_shared_neg = false;  // skeleton batch = [1 CFG-negative image | F positive images] (window step)
  size_t stats_words = 0;      // GroupNorm statistics pool: 64-bit fixed-point per-(image, channel) sums written by the producers' epilogues
  int n3d = 0;                 // number of 3-D attention layers (K/V exchanges) per forward
  unsigned int run_index = 0;  // forwards executed on this plan
  unsigned int epoch0 = 0;     // exchange counter at the start of the current forward (epoch / buffer parity per layer)
  std::vector<std::function<int(cudaStream_t)>> ops;
  std::vector<int> op_kind;       // 0 gemm, 1 conv3x3, 2 attention, 3 groupnorm, 4 layernorm, 5 other
  std::vector<double> op_flops;   // executed FLOPs (incl. tile/head padding) of tensor-core ops
  std::vector<cudaEvent_t> events; // lazily created by profile()
  // debug taps (per-level drift report, tests/test_gpu_fullsize.py): a named intermediate activation [B*H*W, C] (NHWC) that is
  // complete once ops[0 .. n_ops) have run; the arena may reuse its storage afterwards
  struct Tap { std::string name; const bf16* p; int C, H, W; size_t n_ops; };
  std::vector<Tap> taps;
  // per-call externals, set by Model::forward before running the ops
  const bf16* sample = nullptr;
  const long long* timestep = nullptr;
  const bf16* skeletons = nullptr;
  bf16* out = nullptr;
  ~Plan();
};

struct WindowBufs {  // scratch of d4d_denoise_window for one (F, h, w, cfg)
  bf16* sample = nullptr;
  long long* timestep = nullptr;
  bf16* skel = nullptr;
  bf16* noise = nullptr;
  bf16* latents_tmp = nullptr;
  long long* ts_tmp = nullptr;
  ~WindowBufs();
};

struct Exchange {  // K/V exchange buffers in peer memory (cudaIpc), two parities
  bool ready = false;
  int rank = 0, world = 1;
  size_t kv_bytes = 0;
  void* kv[2] = {nullptr, nullptr};
  unsigned int* flags = nullptr;  // [2][8]
  void* peer_kv[2][8] = {};
  unsigned int* peer_flags[8] = {};
  unsigned int epoch_base = 0;    // monotonic across plans
};

class Model {
 public:
  Model(const d4d_config& cfg, int device);
  ~Model();
  int load_weight(const char* key, const void* data, const int64_t* shape, int ndim, int dtype);
  int finalize();
  // F_total > F: frame-sharded window (needs exchange_open); B, F are the LOCAL batch / frames
  int forward(const bf16* sample, const long long* timestep, const bf16* skeletons, const int* domain_ids,
              int n_domains, int B, int F, int h, int w, bf16* out, cudaStream_t stream, int F_total = 0,
              bool pose_shared_neg = false);
  int exchange_alloc(size_t kv_bytes, unsigned char* handles_out /* 3 x 64 bytes */);
  int exchange_open(int rank, int world, const unsigned char* all_handles /* world x 3 x 64 bytes */);
  int denoise_window(bf16* latents, const bf16* pixel, const bf16* plucker, const bf16* skeletons, const bf16* mask,
                     long long* ts_idx, const d4d_sched& sched, float guidance, int domain, int F, int h, int w,
                     int num_steps, cudaStream_t stream, int F_total = 0);
  // per-kind device time (ms) of one forward, measured with CUDA events around every op
  int profile(const bf16* sample, const long long* timestep, const bf16* skeletons, const int* domain_ids, int n_domains,
              int B, int F, int h, int w, bf16* out, cudaStream_t stream, float* ms_by_kind, int* launches_by_kind,
              double* flops_by_kind);
  int get_plan(const int* domain_ids, int n_domains, int B, int F, int h, int w, Plan** out, int F_total = 0,
               bool pose_shared_neg = false);
  // debug: run the forward up to tap `tap` and copy that activation out as NCHW bf16 [B, C, H, W]; out == nullptr only
  // reports name / dims.  Returns 1 when tap is out of range.
  int debug_tap(const bf16* sample, const long long* timestep, const bf16* skeletons, const int* domain_ids, int n_domains,
                int B, int F, int h, int w, int tap, bf16* out, char* name64, int* dims3, cudaStream_t stream);
  Plan* find_plan(int n_domains, int B, int F, int h, int w);
  const std::vector<std::string>& keys() const { return key_order_; }
  int device() const { return device_; }

 private:
  friend class PlanBuilder;
  d4d_config cfg_;
  int device_;
  bool finalized_ = false;
  std::map<std::string, std::vector<int64_t>> expected_;  // key -> diffusers shape (trailing 1s dropped)
  std::vector<std::string> key_order_;
  std::map<std::string, HostTensor> staged_;
  std::vector<void*> dev_allocs_;

  // device weights
  LinW conv_in_;          // [C0][KP_IN]
  LinW time1_, time2_, tem1_, tem2_;
  LinW temb_all_;         // concatenated time_emb_proj [sum Cout][1280]
  PoseW pose_;
  std::vector<ResnetW> down_res_[4], up_res_[4];
  std::vector<XfW> down_xf_[4], up_xf_[4];
  LinW down_ds_[4];
  LinW up_us_[4];         // Upsample2D convs as four sub-pixel phase kernels: [phase = a*2+b][Cout][4][Cin] (unet.cu)
  ResnetW mid_res_[2];
  XfW mid_xf_;
  NormW norm_out_;
  LinW conv_out_;         // [16][9][C0]
  int temb_total_ = 0;

  std::map<std::string, std::unique_ptr<Plan>> plans_;
  std::map<std::string, std::unique_ptr<WindowBufs>> wbufs_;
  Exchange xch_;

  void need(const std::string& key, std::vector<int64_t> shape);
  void declare_keys();
  int cin_pad() const { return 16; }
  int kp_in() const { return 192; }
};

}  // namespace d4d
