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

// Module structs: the Model constructor sets the diffusers module path (also the module's debug tap name) and the shapes;
// finalize() uploads the weights of the keys path + ".conv1.weight" etc.
struct NormW { float* g = nullptr; float* b = nullptr; };
struct LinW { bf16* w = nullptr; float* b = nullptr; int in = 0, out = 0; };
struct ResnetW {
  std::string path;
  NormW n1, n2;
  LinW c1, c2;   // conv3x3 weights [Cout][9][Cin]; in = Cin, out = Cout
  LinW sc;       // 1x1 shortcut (w == nullptr when Cin == Cout)
  int temb_off = 0;  // first row of this block's time_emb_proj in the concatenated projection
  int cin = 0, cout = 0;
};
struct AttnW { LinW qkv, out; };
struct XfW {
  std::string path;
  NormW gn, ln1, ln2, ln3;
  LinW pin, pout, ff1, ff2;
  AttnW a1, a2;
  bool has2 = false;
  bool is3d = false;  // attn1 attends over all frames of a sequence (num_3d_attn_blocks deepest levels, mid block)
  int C = 0, heads = 0, d = 0, dpad = 0;
};
struct LevelW {  // down_blocks.i / up_blocks.i
  std::string path;
  std::vector<ResnetW> res;
  std::vector<XfW> xf;   // empty where the level has no transformers
  std::string sampler;   // module path of the Downsample2D / Upsample2D (empty on the last level)
  int C = 0;             // output channels (also the sampler's)
  LinW conv;             // Downsample2D [C][9][C]; Upsample2D as four sub-pixel phase kernels [phase = a*2+b][C][4][C] (unet.cu)
};
struct PoseW {
  LinW conv[8];   // layers 0..5 direct layout [k*k][Cin][Cout]; 5 -> GEMM layout [Cout][16*Cin], in = 16*Cin; 6,7 conv3x3 layout
  LinW proj;      // [C0][128]
  float scale = 1.f;
};

// Kernel kinds of d4d_profile_forward (include/d4d.h), in its order.
enum OpKind { kOpGemm, kOpConv, kOpAttention, kOpGroupNorm, kOpLayerNorm, kOpOther, kNumOpKinds };
static_assert(kNumOpKinds == 6, "d4d_profile_forward reports [6] arrays per kind");

// one op of a plan: what it enqueues, its kernel launches and executed FLOPs (tensor-core ops, incl. tile / head padding)
struct PlanOp { std::function<int(cudaStream_t)> run; OpKind kind; int launches; double flops; };

// What a plan is built for, and so what it allocates.
struct PlanShape {
  int n_domains = 0, B = 0, F = 0, h = 0, w = 0;
  std::vector<int> domains;
  // frame-sharded plan (DESIGN.md section 7): this rank owns frames [shard * F, (shard + 1) * F) of F_total per CFG half,
  // and the 3-D layers store their K|V rows into the kv_world ranks kv_rank0 .. kv_rank0 + kv_world - 1: every rank for
  // the frame-sharded window (shard = rank), the R ranks of this rank's CFG half for the CFG grid (shard = rank % R)
  int F_total = 0, shard = 0, kv_rank0 = 0, kv_world = 1;
  // the first pose_neg images of the batch are CFG-negative, whose skeletons are all one constant image: the skeleton
  // batch is [1 negative image | B - pose_neg positive images], encoded once and broadcast (window step: F of 2F, or
  // the whole batch on the negative rank of the CFG-split window)
  int pose_neg = 0;
};

struct Plan {
  PlanShape shape;
  void* arena = nullptr;
  size_t arena_bytes = 0;
  int launches = 0;            // sum of ops[i].launches
  size_t stats_words = 0;      // GroupNorm statistics pool: 64-bit fixed-point per-(image, channel) sums of every tensor a GroupNorm reads
  int n3d = 0;                 // number of 3-D attention layers (K/V exchanges) per forward
  unsigned int epoch0 = 0;     // exchange counter at the start of the current forward (epoch / buffer parity per layer)
  std::vector<PlanOp> ops;
  std::vector<cudaEvent_t> events; // lazily created by a timed Model::run_ops (profile)
  // debug taps (per-level drift report, tests/test_gpu_fullsize.py; per-module checks, tests/test_gpu_unet_modules.py): a
  // named intermediate activation [B*H*W, C] (NHWC) that is complete once ops[0 .. n_ops) have run; the arena may reuse its
  // storage afterwards.  The ten block taps come first, then the module taps in forward order (include/d4d.h).
  struct Tap { std::string name; const bf16* p; int C, H, W; size_t n_ops; };
  std::vector<Tap> taps;
  // per-call externals, set by Model::run_ops before running the ops
  const bf16* sample = nullptr;
  const long long* timestep = nullptr;
  const bf16* skeletons = nullptr;
  NchwDst out = {};
  ~Plan();
};

struct WindowBufs {  // scratch of d4d_denoise_window for one (F, h, w, cfg)
  bf16* sample = nullptr;
  long long* timestep = nullptr;
  bf16* skel = nullptr;
  bf16* noise = nullptr;
  long long* ts_tmp = nullptr;
  int* order_tmp = nullptr;  // multistep schedulers only (allocated on first use)
  ~WindowBufs();
};

// The scheduler of a window step: exactly one of the tables is set.  The stateful schedulers (DPM-Solver++, UniPC,
// PNDM, DEIS, DPM-Solver++ singlestep) also get the window frames' solver state, read and updated in place: the order
// counts are read from state.lower_order_nums and the advanced ones end up in state.lower_order_nums_out, both the
// caller's array.  DDPM gets the frames' task indices in state.frame_ids.
struct WindowStep {
  const d4d_sched* ddim = nullptr;
  const d4d_dpm_sched* dpm = nullptr;
  const d4d_unipc_sched* unipc = nullptr;
  const d4d_pndm_sched* pndm = nullptr;
  const d4d_deis_sched* deis = nullptr;
  const d4d_dpm_single_sched* dpm_single = nullptr;
  const d4d_ddpm_sched* ddpm = nullptr;
  SolverState state;
  // the number of tables set (a valid step has one)
  int tables() const {
    return (ddim != nullptr) + (dpm != nullptr) + (unipc != nullptr) + (pndm != nullptr) + (deis != nullptr) +
           (dpm_single != nullptr) + (ddpm != nullptr);
  }
  // fn(table) with whichever table is set
  template <typename Fn>
  int with_table(Fn&& fn) const {
    return ddim ? fn(*ddim) : dpm ? fn(*dpm) : unipc ? fn(*unipc) : pndm ? fn(*pndm) : deis ? fn(*deis)
           : dpm_single ? fn(*dpm_single) : fn(*ddpm);
  }
};

// Where a window step runs its two CFG halves (DESIGN.md section 7): both on this rank (kWhole); one per rank of a world
// of 2, or both on a loopback world of 1 (kSplit, the CFG-split window); or each half frame-sharded over the R = world / 2
// ranks k*R .. k*R + R - 1 of half k (kGrid, the CFG grid; with R = 1 it is the CFG split).
enum class CfgMode { kWhole, kSplit, kGrid };

// The rows of one CFG half that a rank of the CFG split / grid forwards: sample [n, Cin, h, w], timestep [n] and, with the
// pose encoder, skeletons [n, 3, 8h, 8w], n = F / R (its frame shard of the half's F frames).
struct CfgHalfRows {
  const bf16* sample = nullptr;
  const long long* timestep = nullptr;
  const bf16* skeletons = nullptr;
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
              int pose_neg = 0);
  // the same forward, its output stored into every out.p[i]; kv_world > 0 (with F_total): the 3-D layers exchange K|V
  // within this rank's group of kv_world consecutive ranks only (the CFG grid), 0: with every rank
  int forward(const bf16* sample, const long long* timestep, const bf16* skeletons, const int* domain_ids,
              int n_domains, int B, int F, int h, int w, const NchwDst& out, cudaStream_t stream, int F_total,
              int pose_neg, int kv_world = 0);
  int exchange_alloc(size_t kv_bytes, unsigned char* handles_out /* 3 x 64 bytes */);
  int exchange_open(int rank, int world, const unsigned char* all_handles /* world x 3 x 64 bytes */);
  // num_steps x (assemble -> UNet -> CFG + scheduler step) on the window's F frames; latents, ts_idx and the solver state
  // of `step` are updated in place.  mode kSplit (guidance > 1, needs exchange_open with world 1 or 2): this rank runs the
  // UNet on its CFG half only and the halves meet in the exchange buffers; kGrid (world 1, 2, 4, 6 or 8): this rank runs
  // it on its frame shard of its CFG half (DESIGN.md section 7).
  int denoise_window(bf16* latents, const bf16* pixel, const bf16* plucker, const bf16* skeletons, const bf16* mask,
                     long long* ts_idx, const WindowStep& step, float guidance, int domain, int F, int h, int w,
                     int num_steps, cudaStream_t stream, int F_total, CfgMode mode = CfgMode::kWhole);
  // B-2 on the CFG split (kSplit) or grid (kGrid): sample [B, Cin, h, w] is the reference's batch, and every rank gets the
  // whole noise [B, out_channels, h, w] in `out`.  n_domains 2: [F negative | F positive]; this rank forwards its rows
  // (cfg_split_forward) and the gathered noise is copied out.  n_domains 1: the plain forward, nothing exchanged.
  int unet_forward_cfg(const bf16* sample, const long long* timestep, const bf16* skeletons, const int* domain_ids,
                       int n_domains, int B, int F, int h, int w, bf16* out, cudaStream_t stream, CfgMode mode);
  // frame-sharded sliding loop: this rank's F updated frames (+ DPM-Solver++ state when x0_prev != nullptr) to every rank,
  // one flag round (one more exchange of the epoch sequence), then the gathered F_total frames to the *_out buffers
  int window_exchange(const bf16* latents, const long long* ts_idx, const bf16* x0_prev, const int* lower_order_nums, int F,
                      int F_total, int h, int w, bf16* latents_out, long long* ts_out, bf16* x0_out, int* lon_out,
                      cudaStream_t stream);
  // per-kind device time (ms) of one forward, measured with CUDA events around every op
  int profile(const bf16* sample, const long long* timestep, const bf16* skeletons, const int* domain_ids, int n_domains,
              int B, int F, int h, int w, bf16* out, cudaStream_t stream, float* ms_by_kind, int* launches_by_kind,
              double* flops_by_kind);
  int get_plan(const int* domain_ids, int n_domains, int B, int F, int h, int w, Plan** out, int F_total = 0,
               int pose_neg = 0, int kv_world = 0);
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
  LinW temb_all_;         // every resnet's time_emb_proj, concatenated: [sum Cout][TE] (in / out set by the constructor)
  PoseW pose_;
  LevelW down_[4], up_[4];
  ResnetW mid_res_[2];
  XfW mid_xf_;
  NormW norm_out_;
  LinW conv_out_;         // [16][9][C0]

  std::map<std::string, std::unique_ptr<Plan>> plans_;
  std::map<std::string, std::unique_ptr<WindowBufs>> wbufs_;
  Exchange xch_;

  void need(const std::string& key, std::vector<int64_t> shape);
  // checks and binds the per-call externals of p, then enqueues ops[0 .. n); timed: events[i] is recorded before op i and
  // events[n] after the last
  int run_ops(Plan& p, const bf16* sample, const long long* timestep, const bf16* skeletons, const NchwDst& out, size_t n,
              cudaStream_t stream, bool timed = false);
  // closes exchange epoch_base: signal it to every rank, count it, wait for every rank's signal
  int flag_round(cudaStream_t stream);
  // The CFG split / grid forward of F frames per CFG half (domain_ids[k]: half k's domain), before any launch: the
  // mode's world, F divisible by R, the noise within the exchange buffer, and this rank's plans built (a grid plan
  // refuses a K/V buffer too small for one half's 3-D layers).  *R: the frame shards per half.  neg_const: the negative
  // half's skeletons are one constant image, encoded once (the window step); otherwise the caller's rows.
  int cfg_split_prepare(CfgMode mode, const int* domain_ids, int F, int h, int w, bool neg_const, int* R);
  // the worlds a mode runs: the split 1 (loopback) or 2 ranks, the grid 1, 2, 4, 6 or 8
  int cfg_world_check(CfgMode mode) const;
  // the CFG halves [k0, k1) this rank forwards (both on a loopback) and its frame shard r of R per half
  void cfg_cell(int R, int* k0, int* k1, int* r) const;
  // The UNet on rows[k] for each half k this rank runs, each half's noise stored at rows [k*F + r*F/R, k*F + (r+1)*F/R)
  // of every rank's exchange buffer, then one flag round.  *noise: this rank's buffer that holds the gathered
  // [2F, out_channels, h, w] noise; reads of it enqueued before this rank's next exchange signal are safe (DESIGN.md
  // section 7).
  int cfg_split_forward(const CfgHalfRows* rows, const int* domain_ids, int F, int h, int w, int R, bool neg_const,
                        cudaStream_t stream, const bf16** noise);
  int cin_pad() const { return 16; }
  int kp_in() const { return 192; }
};

}  // namespace d4d
