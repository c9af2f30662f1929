// UNet executor for the Diffuman4D denoise step.
//
// Mirrors UNetMultiviewConditionModel.forward (reference unet_multiview_condition.py:501-598) and the block
// wiring of unet_multiview_blocks.py:233-712 / transformer_multiview.py:79-232 / attention.py:22-153 as a
// static launch plan per (domains, B, F, h, w): NHWC bf16 activations end to end, one arena, every FLOP in the
// wgmma GEMM / conv / attention kernels, norms and layout glue in 128-bit HBM kernels.  The channel concat
// of the up path, the (b t) hw c <-> b (t hw) c rearranges and the NCHW<->token permutes of the reference are
// address arithmetic here.
#include "unet.h"

#include <math.h>

#include <algorithm>
#include <stdexcept>

namespace d4d {

namespace {

inline uint16_t f2bf(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return static_cast<uint16_t>((u >> 16) | 0x40);  // NaN
  const uint32_t lsb = (u >> 16) & 1u;
  u += 0x7fffu + lsb;
  return static_cast<uint16_t>(u >> 16);
}
inline float bf2f(uint16_t h) {
  uint32_t u = static_cast<uint32_t>(h) << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
inline float h2f(uint16_t h) {  // IEEE half -> float
  const uint32_t s = (h >> 15) & 1, e = (h >> 10) & 0x1f, m = h & 0x3ff;
  uint32_t u;
  if (e == 0) {
    if (m == 0) u = s << 31;
    else {
      int ee = -1;
      uint32_t mm = m;
      do { ++ee; mm <<= 1; } while (!(mm & 0x400));
      u = (s << 31) | ((127 - 15 - ee) << 23) | ((mm & 0x3ff) << 13);
    }
  } else if (e == 31) u = (s << 31) | 0x7f800000u | (m << 13);
  else u = (s << 31) | ((e - 15 + 127) << 23) | (m << 13);
  float f;
  memcpy(&f, &u, 4);
  return f;
}

inline int pad_head_dim(int d) { return d <= 64 ? 64 : (d <= 128 ? 128 : (d <= 192 ? 192 : 0)); }

// the pose encoder's convolutions: module path, Cin, Cout, kernel
const struct { const char* path; int cin, cout, k; } kPoseLayers[8] = {
    {"pose_encoder.conv_layers.0", 3, 3, 3},    {"pose_encoder.conv_layers.2", 3, 16, 4},
    {"pose_encoder.conv_layers.4", 16, 16, 3},  {"pose_encoder.conv_layers.6", 16, 32, 4},
    {"pose_encoder.conv_layers.8", 32, 32, 3},  {"pose_encoder.conv_layers.10", 32, 64, 4},
    {"pose_encoder.conv_layers.12", 64, 64, 3}, {"pose_encoder.conv_layers.14", 64, 128, 3}};

std::string plan_key(const PlanShape& s) {
  std::string k = std::to_string(s.B) + "_" + std::to_string(s.F) + "_" + std::to_string(s.h) + "_" + std::to_string(s.w) + "_";
  for (int d : s.domains) k += d ? 't' : 's';
  if (s.F_total > 0) k += "_sh" + std::to_string(s.F_total) + "_g" + std::to_string(s.kv_rank0) + "x" + std::to_string(s.kv_world);
  return s.pose_neg > 0 ? k + "_pn" + std::to_string(s.pose_neg) : k;
}

NchwDst one_dst(bf16* out) {
  NchwDst d = {};
  d.p[0] = out;
  d.n = out ? 1 : 0;
  return d;
}

}  // namespace

Plan::~Plan() {
  if (arena) cudaFree(arena);
  for (cudaEvent_t e : events) cudaEventDestroy(e);
}
WindowBufs::~WindowBufs() {
  cudaFree(sample);
  cudaFree(timestep);
  cudaFree(skel);
  cudaFree(noise);
  cudaFree(ts_tmp);
  cudaFree(order_tmp);
}

// =================================================================================================
// weights
// =================================================================================================
// The module tree: every module's path and shapes, and its weight keys in state_dict order (weights.state_dict_spec).
Model::Model(const d4d_config& cfg, int device) : cfg_(cfg), device_(device) {
  const int* ch = cfg_.block_out_channels;
  const int C0 = ch[0], TE = 4 * C0, L = cfg_.layers_per_block;
  temb_all_.in = TE;
  auto lin = [&](const std::string& p, int out, int in, bool bias = true) {
    need(p + ".weight", {out, in});
    if (bias) need(p + ".bias", {out});
  };
  auto conv = [&](const std::string& p, int out, int in, int k) {
    need(p + ".weight", {out, in, k, k});
    need(p + ".bias", {out});
  };
  auto norm = [&](const std::string& p, int c) {
    need(p + ".weight", {c});
    need(p + ".bias", {c});
  };
  auto resnet = [&](const std::string& p, int cin, int cout) {
    ResnetW r;
    r.path = p;
    r.cin = cin;
    r.cout = cout;
    r.temb_off = temb_all_.out;
    temb_all_.out += cout;
    norm(p + ".norm1", cin);
    conv(p + ".conv1", cout, cin, 3);
    lin(p + ".time_emb_proj", cout, TE);
    norm(p + ".norm2", cout);
    conv(p + ".conv2", cout, cout, 3);
    if (cin != cout) conv(p + ".conv_shortcut", cout, cin, 1);
    return r;
  };
  // transformer at channel level c; attn1 is 3-D at the num_3d_attn_blocks deepest levels and in the mid block
  auto xf = [&](const std::string& p, int c, bool mid = false) {
    XfW x;
    x.path = p;
    x.C = ch[c];
    x.heads = cfg_.num_heads[c];
    x.d = x.C / x.heads;
    x.dpad = pad_head_dim(x.d);
    x.has2 = cfg_.has_attn2[c] != 0;
    x.is3d = mid || 3 - c < cfg_.num_3d_attn_blocks;
    const int C = x.C;
    norm(p + ".norm", C);
    lin(p + ".proj_in", C, C);
    const std::string b = p + ".transformer_blocks.0";
    norm(b + ".norm1", C);
    lin(b + ".attn1.to_q", C, C, false);
    lin(b + ".attn1.to_k", C, C, false);
    lin(b + ".attn1.to_v", C, C, false);
    lin(b + ".attn1.to_out.0", C, C);
    if (x.has2) {
      norm(b + ".norm2", C);
      lin(b + ".attn2.to_q", C, C, false);
      lin(b + ".attn2.to_k", C, C, false);
      lin(b + ".attn2.to_v", C, C, false);
      lin(b + ".attn2.to_out.0", C, C);
    }
    norm(b + ".norm3", C);
    lin(b + ".ff.net.0.proj", 8 * C, C);
    lin(b + ".ff.net.2", C, 4 * C);
    lin(p + ".proj_out", C, C);
    return x;
  };
  auto sampler = [&](LevelW& lv, const char* name) {
    lv.sampler = lv.path + name;
    conv(lv.sampler + ".conv", lv.C, lv.C, 3);
  };
  conv("conv_in", C0, cfg_.in_channels, 3);
  lin("time_embedding.linear_1", TE, C0);
  lin("time_embedding.linear_2", TE, TE);
  if (cfg_.enable_tem_embeds) {
    lin("temporal_pos_embed.linear_1", TE, C0);
    lin("temporal_pos_embed.linear_2", TE, TE);
  }
  if (cfg_.enable_pose_encoder) {
    for (const auto& l : kPoseLayers) conv(l.path, l.cout, l.cin, l.k);
    conv("pose_encoder.final_proj", C0, 128, 1);
    need("pose_encoder.scale", {1});
  }
  int cout = C0;
  for (int i = 0; i < 4; ++i) {
    const int cin = cout;
    cout = ch[i];
    LevelW& lv = down_[i];
    lv.path = "down_blocks." + std::to_string(i);
    lv.C = cout;
    for (int j = 0; j < L; ++j) {
      lv.res.push_back(resnet(lv.path + ".resnets." + std::to_string(j), j == 0 ? cin : cout, cout));
      if (i < 3) lv.xf.push_back(xf(lv.path + ".attentions." + std::to_string(j), i));
    }
    if (i < 3) sampler(lv, ".downsamplers.0");
  }
  mid_res_[0] = resnet("mid_block.resnets.0", ch[3], ch[3]);
  mid_xf_ = xf("mid_block.attentions.0", 3, true);
  mid_res_[1] = resnet("mid_block.resnets.1", ch[3], ch[3]);
  cout = ch[3];
  for (int i = 0; i < 4; ++i) {
    const int cprev = cout;
    cout = ch[3 - i];
    const int cin = ch[3 - std::min(i + 1, 3)];
    LevelW& lv = up_[i];
    lv.path = "up_blocks." + std::to_string(i);
    lv.C = cout;
    for (int j = 0; j <= L; ++j) {
      const int skip = j == L ? cin : cout;
      const int rin = j == 0 ? cprev : cout;
      lv.res.push_back(resnet(lv.path + ".resnets." + std::to_string(j), rin + skip, cout));
      if (i > 0) lv.xf.push_back(xf(lv.path + ".attentions." + std::to_string(j), 3 - i));
    }
    if (i < 3) sampler(lv, ".upsamplers.0");
  }
  norm("conv_norm_out", C0);
  conv("conv_out", cfg_.out_channels, C0, 3);
}

Model::~Model() {
  cudaSetDevice(device_);
  plans_.clear();
  wbufs_.clear();
  for (void* p : dev_allocs_) cudaFree(p);
}

void Model::need(const std::string& key, std::vector<int64_t> shape) {
  expected_[key] = std::move(shape);
  key_order_.push_back(key);
}

int Model::load_weight(const char* key, const void* data, const int64_t* shape, int ndim, int dtype) {
  D4D_REQUIRE(key != nullptr && data != nullptr && shape != nullptr, "null argument");
  D4D_REQUIRE(!finalized_, "weights already finalized");
  auto it = expected_.find(key);
  if (it == expected_.end()) {
    set_error(std::string("unknown weight key: ") + key);
    return 1;
  }
  // full shape check (a transposed / mis-shaped tensor with the right element count must not load silently); trailing
  // dims of size 1 are ignored so that 1x1-conv [C, C, 1, 1] and Linear [C, C] projections are interchangeable
  auto squeeze = [](std::vector<int64_t> v) {
    while (v.size() > 1 && v.back() == 1) v.pop_back();
    return v;
  };
  const std::vector<int64_t> got = squeeze(std::vector<int64_t>(shape, shape + ndim)), want = squeeze(it->second);
  auto fmt = [](const std::vector<int64_t>& v) {
    std::string o = "[";
    for (size_t i = 0; i < v.size(); ++i) o += (i ? ", " : "") + std::to_string(v[i]);
    return o + "]";
  };
  if (got != want) {
    set_error(std::string("shape mismatch for ") + key + ": got " + fmt(got) + ", expected " + fmt(want));
    return 1;
  }
  int64_t numel = 1;
  for (int i = 0; i < ndim; ++i) numel *= shape[i];
  HostTensor& t = staged_[key];
  t.shape.assign(shape, shape + ndim);
  t.v.resize(static_cast<size_t>(numel));
  if (dtype == 0) memcpy(t.v.data(), data, sizeof(float) * numel);
  else if (dtype == 1) {
    const uint16_t* s = static_cast<const uint16_t*>(data);
    for (int64_t i = 0; i < numel; ++i) t.v[i] = bf2f(s[i]);
  } else if (dtype == 2) {
    const uint16_t* s = static_cast<const uint16_t*>(data);
    for (int64_t i = 0; i < numel; ++i) t.v[i] = h2f(s[i]);
  } else {
    set_error("unsupported dtype code (0 f32, 1 bf16, 2 f16)");
    return 1;
  }
  return 0;
}

int Model::finalize() {
  if (finalized_) return 0;
  for (const auto& k : key_order_) {
    if (!staged_.count(k)) {
      set_error("missing weight: " + k);
      return 3;
    }
  }
  D4D_CUDA_OK(cudaSetDevice(device_));
  bool failed = false;
  auto dev_alloc = [&](size_t bytes) -> void* {
    void* p = nullptr;
    if (cudaMalloc(&p, bytes ? bytes : 16) != cudaSuccess) {
      failed = true;
      return nullptr;
    }
    dev_allocs_.push_back(p);
    return p;
  };
  auto up_bf16 = [&](const std::vector<float>& v) -> bf16* {
    std::vector<uint16_t> h(v.size());
    for (size_t i = 0; i < v.size(); ++i) h[i] = f2bf(v[i]);
    void* p = dev_alloc(h.size() * 2);
    if (p && cudaMemcpy(p, h.data(), h.size() * 2, cudaMemcpyHostToDevice) != cudaSuccess) failed = true;
    return static_cast<bf16*>(p);
  };
  auto up_f32 = [&](const std::vector<float>& v) -> float* {
    void* p = dev_alloc(v.size() * 4);
    if (p && cudaMemcpy(p, v.data(), v.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess) failed = true;
    return static_cast<float*>(p);
  };
  auto T = [&](const std::string& k) -> const std::vector<float>& { return staged_.at(k).v; };
  auto normw = [&](const std::string& p) { return NormW{up_f32(T(p + ".weight")), up_f32(T(p + ".bias"))}; };
  auto linw = [&](const std::string& p) {  // Linear / 1x1 conv [out][in]
    const std::vector<int64_t>& s = expected_.at(p + ".weight");
    return LinW{up_bf16(T(p + ".weight")), up_f32(T(p + ".bias")), static_cast<int>(s[1]), static_cast<int>(s[0])};
  };
  // OIHW [Cout,Cin,k,k] -> [Cout][tap][Cin]
  auto conv_gemm_layout = [&](const std::vector<float>& w, int cout, int cin, int k, int cout_pad = 0) {
    const int co_total = cout_pad > cout ? cout_pad : cout;
    std::vector<float> o(static_cast<size_t>(co_total) * k * k * cin, 0.f);
    for (int co = 0; co < cout; ++co)
      for (int ci = 0; ci < cin; ++ci)
        for (int t = 0; t < k * k; ++t)
          o[(static_cast<size_t>(co) * k * k + t) * cin + ci] = w[(static_cast<size_t>(co) * cin + ci) * k * k + t];
    return o;
  };
  auto convw = [&](const std::string& p) {  // conv3x3
    const std::vector<int64_t>& s = expected_.at(p + ".weight");
    const int cout = static_cast<int>(s[0]), cin = static_cast<int>(s[1]);
    return LinW{up_bf16(conv_gemm_layout(T(p + ".weight"), cout, cin, 3)), up_f32(T(p + ".bias")), cin, cout};
  };
  const int C0 = cfg_.block_out_channels[0], TE = temb_all_.in;

  // every time_emb_proj at its block's rows of one [sum Cout][TE] projection
  std::vector<float> temb_w(static_cast<size_t>(temb_all_.out) * TE), temb_b(temb_all_.out);
  auto resnetw = [&](ResnetW& r) {
    r.n1 = normw(r.path + ".norm1");
    r.c1 = convw(r.path + ".conv1");
    r.n2 = normw(r.path + ".norm2");
    r.c2 = convw(r.path + ".conv2");
    if (r.cin != r.cout) r.sc = linw(r.path + ".conv_shortcut");
    const auto& tw = T(r.path + ".time_emb_proj.weight");
    const auto& tb = T(r.path + ".time_emb_proj.bias");
    std::copy(tw.begin(), tw.end(), temb_w.begin() + static_cast<size_t>(r.temb_off) * TE);
    std::copy(tb.begin(), tb.end(), temb_b.begin() + r.temb_off);
  };
  auto attnw = [&](const std::string& p, const XfW& x) {
    const int C = x.C, heads = x.heads, d = x.d, dpad = x.dpad, Cp = heads * dpad;
    std::vector<float> qkv(static_cast<size_t>(3) * Cp * C, 0.f);
    const char* names[3] = {".to_q.weight", ".to_k.weight", ".to_v.weight"};
    for (int s = 0; s < 3; ++s) {
      const auto& w = T(p + names[s]);
      for (int hh = 0; hh < heads; ++hh)
        for (int j = 0; j < d; ++j)
          memcpy(&qkv[(static_cast<size_t>(s) * Cp + hh * dpad + j) * C], &w[static_cast<size_t>(hh * d + j) * C],
                 sizeof(float) * C);
    }
    const auto& wo = T(p + ".to_out.0.weight");
    std::vector<float> o(static_cast<size_t>(C) * Cp, 0.f);
    for (int r = 0; r < C; ++r)
      for (int hh = 0; hh < heads; ++hh)
        for (int j = 0; j < d; ++j) o[static_cast<size_t>(r) * Cp + hh * dpad + j] = wo[static_cast<size_t>(r) * C + hh * d + j];
    return AttnW{LinW{up_bf16(qkv), nullptr, C, 3 * Cp}, LinW{up_bf16(o), up_f32(T(p + ".to_out.0.bias")), Cp, C}};
  };
  auto xfw = [&](XfW& x) {
    const int C = x.C;
    const std::string b = x.path + ".transformer_blocks.0";
    x.gn = normw(x.path + ".norm");
    x.pin = linw(x.path + ".proj_in");
    x.pout = linw(x.path + ".proj_out");
    x.ln1 = normw(b + ".norm1");
    x.a1 = attnw(b + ".attn1", x);
    if (x.has2) {
      x.ln2 = normw(b + ".norm2");
      x.a2 = attnw(b + ".attn2", x);
    }
    x.ln3 = normw(b + ".norm3");
    // GEGLU interleave in groups of 8 rows: rows 16p .. 16p+7 = a[8p .. 8p+7], rows 16p+8 .. 16p+15 = g[8p .. 8p+7]
    const int N = 8 * C;
    const auto& w = T(b + ".ff.net.0.proj.weight");
    const auto& bb = T(b + ".ff.net.0.proj.bias");
    std::vector<float> wi(w.size()), bi(bb.size());
    for (int r = 0; r < N; ++r) {
      const int p = r / 16, i = r % 16;
      const int src = (i < 8 ? 0 : 4 * C) + 8 * p + (i & 7);
      memcpy(&wi[static_cast<size_t>(r) * C], &w[static_cast<size_t>(src) * C], sizeof(float) * C);
      bi[r] = bb[src];
    }
    x.ff1 = LinW{up_bf16(wi), up_f32(bi), C, N};
    x.ff2 = linw(b + ".ff.net.2");
  };
  // Upsample2D = nearest x2 followed by a 3x3 conv: every output pixel (2y + a, 2x + b) only ever sees a 2x2 patch of
  // the LOW-resolution input, so the layer is computed as four sub-pixel phases with pre-summed weights
  // (rows {-1, 0} weigh {w0, w1 + w2} for a = 0 and rows {0, +1} weigh {w0 + w1, w2} for a = 1; same for columns):
  // 4/9 of the multiply-adds and no materialised upsampled tensor.  Layout per phase: [Cout][ty*2 + tx][Cin].
  auto upsamplew = [&](const std::string& p, int C) {
    const auto& w = T(p + ".weight");
    std::vector<float> o(static_cast<size_t>(4) * C * 4 * C, 0.f);  // [phase = a*2+b][Cout][ty*2+tx][Cin]
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b)
        for (int co = 0; co < C; ++co)
          for (int ci = 0; ci < C; ++ci)
            for (int ky = 0; ky < 3; ++ky)
              for (int kx = 0; kx < 3; ++kx) {
                const int ty = a == 0 ? (ky == 0 ? 0 : 1) : (ky == 2 ? 1 : 0);
                const int tx = b == 0 ? (kx == 0 ? 0 : 1) : (kx == 2 ? 1 : 0);
                o[((static_cast<size_t>(a * 2 + b) * C + co) * 4 + ty * 2 + tx) * C + ci] +=
                    w[(static_cast<size_t>(co) * C + ci) * 9 + ky * 3 + kx];
              }
    return LinW{up_bf16(o), up_f32(T(p + ".bias")), C, C};
  };

  {  // conv_in -> [C0][KP] with k = tap*16 + c
    const int Cin = cfg_.in_channels, KP = kp_in(), cp = cin_pad();
    const auto& w = T("conv_in.weight");
    std::vector<float> o(static_cast<size_t>(C0) * KP, 0.f);
    for (int co = 0; co < C0; ++co)
      for (int ci = 0; ci < Cin; ++ci)
        for (int t = 0; t < 9; ++t) o[static_cast<size_t>(co) * KP + t * cp + ci] = w[(static_cast<size_t>(co) * Cin + ci) * 9 + t];
    conv_in_ = LinW{up_bf16(o), up_f32(T("conv_in.bias")), KP, C0};
  }
  time1_ = linw("time_embedding.linear_1");
  time2_ = linw("time_embedding.linear_2");
  if (cfg_.enable_tem_embeds) {
    tem1_ = linw("temporal_pos_embed.linear_1");
    tem2_ = linw("temporal_pos_embed.linear_2");
  }
  if (cfg_.enable_pose_encoder) {
    for (int i = 0; i < 8; ++i) {
      const std::string p = kPoseLayers[i].path;
      const int cin = kPoseLayers[i].cin, cout = kPoseLayers[i].cout, k = kPoseLayers[i].k;
      const auto& w = T(p + ".weight");
      LinW l{nullptr, up_f32(T(p + ".bias")), cin, cout};
      if (i == 0) {  // FMA kernel: [k*k][Cin][Cout]
        std::vector<float> o(w.size());
        for (int co = 0; co < cout; ++co)
          for (int ci = 0; ci < cin; ++ci)
            for (int t = 0; t < k * k; ++t) o[(static_cast<size_t>(t) * cin + ci) * cout + co] = w[(static_cast<size_t>(co) * cin + ci) * k * k + t];
        l.w = up_bf16(o);
      } else if (i < 5) {  // mma.sync kernel: [Cout][k*k*cin_pad + 8], K index = tap*cin_pad + ci (layer 1 reads 4-channel pixels)
        const int cp = cin < 4 ? 4 : cin, KP = k * k * cp + 8;
        std::vector<float> o(static_cast<size_t>(cout) * KP, 0.f);
        for (int co = 0; co < cout; ++co)
          for (int ci = 0; ci < cin; ++ci)
            for (int t = 0; t < k * k; ++t) o[static_cast<size_t>(co) * KP + t * cp + ci] = w[(static_cast<size_t>(co) * cin + ci) * k * k + t];
        l.w = up_bf16(o);
        l.in = cp;
      } else {
        l.w = up_bf16(conv_gemm_layout(w, cout, cin, k));
        if (i == 5) l.in = k * k * cin;  // GEMM over the im2col columns
      }
      pose_.conv[i] = l;
    }
    pose_.proj = linw("pose_encoder.final_proj");
    pose_.scale = T("pose_encoder.scale")[0];
  }
  for (LevelW& lv : down_) {
    for (ResnetW& r : lv.res) resnetw(r);
    for (XfW& x : lv.xf) xfw(x);
    if (!lv.sampler.empty()) lv.conv = convw(lv.sampler + ".conv");
  }
  resnetw(mid_res_[0]);
  xfw(mid_xf_);
  resnetw(mid_res_[1]);
  for (LevelW& lv : up_) {
    for (ResnetW& r : lv.res) resnetw(r);
    for (XfW& x : lv.xf) xfw(x);
    if (!lv.sampler.empty()) lv.conv = upsamplew(lv.sampler + ".conv", lv.C);
  }
  norm_out_ = normw("conv_norm_out");
  {  // conv_out, zero-padded to 16 output channels
    std::vector<float> b(16, 0.f);
    const auto& bo = T("conv_out.bias");
    std::copy(bo.begin(), bo.end(), b.begin());
    conv_out_ = LinW{up_bf16(conv_gemm_layout(T("conv_out.weight"), cfg_.out_channels, C0, 3, 16)), up_f32(b), C0, 16};
  }
  temb_all_.w = up_bf16(temb_w);
  temb_all_.b = up_f32(temb_b);
  if (failed) {
    set_error(std::string("device allocation/upload failed while finalizing weights: ") + cudaGetErrorString(cudaGetLastError()));
    return 2;
  }
  staged_.clear();
  finalized_ = true;
  return 0;
}

// =================================================================================================
// plan builder
// =================================================================================================
class PlanBuilder {
 public:
  PlanBuilder(Model& m, Plan& p, bool dry, char* base) : m_(m), p_(p), dry_(dry), base_(base) {}

  struct Act { bf16* p; int C, H, W; long long* stats = nullptr; };  // stats: [B][C][2] {sum, sumsq} when a GroupNorm reads p

  size_t peak() const { return peak_; }
  size_t stats_words() const { return stats_used_; }
  // per-(image, channel) statistics of a GEMM / conv output that a GroupNorm will read: a slice of one pool that a single
  // memset at the head of the plan zeroes
  long long* stats_alloc(int n_img, int C) {
    long long* p = stats_pool_ ? stats_pool_ + stats_used_ : nullptr;  // (the dry run only counts)
    stats_used_ += static_cast<size_t>(n_img) * C * 2;
    return p;
  }
  // Runs the producer of `out` (d writes out.p) so that out.stats holds its statistics.  The epilogue accumulates them
  // where it can (gemm_stats_fusable) and the grid its tiles walk, H x W per image, has H > 1 and a multiple of 32
  // positions: every level of the 64x64 and 128x128 latents.  Otherwise a statistics launch follows the producer.  Eager, not
  // at the norm: a down-path output is read by two GroupNorms (the next block's and the up-path concat's), summed once.
  void gemm_stats(GemmDesc d, const Act& out, int n_img, int H, int W) {
    if (H > 1 && (H * W) % 32 == 0 && gemm_stats_fusable(d, sms_)) {
      d.stats = out.stats;
      gemm(d);
      return;
    }
    gemm(d);
    const bf16* x = out.p;
    long long* st = out.stats;
    const int C = out.C, hw = out.H * out.W;
    op([=](cudaStream_t s) { return groupnorm_stats_run(x, C, n_img, hw, st, s); }, kOpGroupNorm);
  }
  int rc() const { return rc_; }

  bf16* alloc(size_t elems) {
    size_t bytes = (elems * 2 + 255) & ~size_t(255);
    // best-fit from the free list
    int best = -1;
    for (size_t i = 0; i < free_.size(); ++i)
      if (free_[i].second >= bytes && (best < 0 || free_[i].second < free_[best].second)) best = static_cast<int>(i);
    size_t off;
    if (best >= 0) {
      off = free_[best].first;
      const size_t sz = free_[best].second;
      free_.erase(free_.begin() + best);
      if (sz > bytes) free_.push_back({off + bytes, sz - bytes});
    } else {
      off = bump_;
      bump_ += bytes;
      peak_ = std::max(peak_, bump_);
    }
    live_[off] = bytes;
    return reinterpret_cast<bf16*>(base_ + off);
  }
  void release(const void* ptr) {
    const size_t off = static_cast<size_t>(reinterpret_cast<const char*>(ptr) - base_);
    auto it = live_.find(off);
    if (it == live_.end()) return;
    size_t o = off, sz = it->second;
    live_.erase(it);
    // coalesce with neighbours
    bool merged = true;
    while (merged) {
      merged = false;
      for (size_t i = 0; i < free_.size(); ++i) {
        if (free_[i].first + free_[i].second == o) { o = free_[i].first; sz += free_[i].second; free_.erase(free_.begin() + i); merged = true; break; }
        if (o + sz == free_[i].first) { sz += free_[i].second; free_.erase(free_.begin() + i); merged = true; break; }
      }
    }
    if (o + sz == bump_) bump_ = o;
    else free_.push_back({o, sz});
  }

  // the one place a plan's ops and launch count are recorded (the dry run counts launches only)
  void op(std::function<int(cudaStream_t)> f, OpKind kind = kOpOther, int launches = 1, double flops = 0.0) {
    p_.launches += launches;
    if (!dry_) p_.ops.push_back({std::move(f), kind, launches, flops});
  }
  void tap(const std::string& name, const Act& a) {
    if (!dry_) p_.taps.push_back({name, a.p, a.C, a.H, a.W, p_.ops.size()});
  }
  // module taps, named after the diffusers module path whose output `a` is; numbered after the block taps (end of build)
  void module_tap(const std::string& name, const Act& a) {
    if (!dry_) module_taps_.push_back({name, a.p, a.C, a.H, a.W, p_.ops.size()});
  }
  void gemm(const GemmDesc& d) {
    const OpKind kind = d.conv ? kOpConv : kOpGemm;
    if (dry_) { op(nullptr, kind); return; }
    GemmLaunch L;
    if (int rc = gemm_prepare(d, &L)) { if (!rc_) rc_ = rc; return; }
    op([L](cudaStream_t s) { return gemm_run(L, s); }, kind, 1, gemm_flops(L));
  }
  void attention(const AttnDesc& d) {
    if (dry_) { op(nullptr, kOpAttention); return; }
    AttnLaunch L;
    if (int rc = attn_prepare(d, &L)) { if (!rc_) rc_ = rc; return; }
    op([L](cudaStream_t s) { return attn_run(L, s); }, kOpAttention, 1, attn_flops(d));
  }
  // GroupNorm(+SiLU) of (a | b) from their statistics (Act::stats, see gemm_stats): one apply launch
  void groupnorm(const Act& xa, const Act* xb, int n_img, float eps, const NormW& n, int silu, bf16* out) {
    const int groups = m_.cfg_.norm_num_groups, hw = xa.H * xa.W;
    const bf16 *x1 = xa.p, *x2 = xb ? xb->p : nullptr;
    const int C1 = xa.C, C2 = xb ? xb->C : 0;
    const long long *s1 = xa.stats, *s2 = xb ? xb->stats : nullptr;
    op([=](cudaStream_t s) { return groupnorm_apply_run(x1, C1, s1, x2, C2, s2, n_img, hw, groups, eps, n.g, n.b, silu, out, s); },
       kOpGroupNorm);
  }
  void layernorm(const bf16* x, int rows, int C, const NormW& n, bf16* out) {
    op([=](cudaStream_t s) { return layernorm_run(x, rows, C, 1e-5f, n.g, n.b, out, s); }, kOpLayerNorm);
  }
  // GEMM descriptors of a weight: out[M, w.out] = A[M, w.in] * w^T + bias, and the conv (conv_kind `kind`) of n_img NHWC
  // images [H, W, w.in]; call sites set what differs
  static GemmDesc linear(const LinW& w, const bf16* A, int M, bf16* out) {
    GemmDesc d;
    d.A = A; d.lda = w.in; d.K1 = w.in; d.Wt = w.w; d.M = M; d.N = w.out; d.bias = w.b; d.out = out; d.ldo = w.out;
    return d;
  }
  static GemmDesc conv(const LinW& w, const bf16* A, int n_img, int H, int W, bf16* out, int kind = 0) {
    GemmDesc d;
    d.conv = 1; d.conv_kind = kind; d.A = A; d.n_img = n_img; d.H = H; d.W = W; d.Cin = w.in;
    d.Wt = w.w; d.N = w.out; d.bias = w.b; d.out = out; d.ldo = w.out;
    return d;
  }

  // ResnetBlock2D on (xa | xb) -> new buffer   (reference semantics: SURVEY R-1)
  Act resnet(const ResnetW& r, Act xa, const Act* xb, const bf16* temb_all, int ld_temb) {
    const int B = p_.shape.B, hw = xa.H * xa.W, M = B * hw;
    const int Cb = xb ? xb->C : 0;
    const int Cin = xa.C + Cb;
    bf16* h0 = alloc(static_cast<size_t>(M) * Cin);
    groupnorm(xa, xb, B, m_.cfg_.norm_eps, r.n1, 1, h0);
    Act h1{alloc(static_cast<size_t>(M) * r.cout), r.cout, xa.H, xa.W, stats_alloc(B, r.cout)};
    {
      GemmDesc d = conv(r.c1, h0, B, xa.H, xa.W, h1.p);
      d.rowvec = temb_all + r.temb_off; d.ld_rowvec = ld_temb;
      gemm_stats(d, h1, B, xa.H, xa.W);
    }
    release(h0);
    bf16* h2 = alloc(static_cast<size_t>(M) * r.cout);
    groupnorm(h1, nullptr, B, m_.cfg_.norm_eps, r.n2, 1, h2);
    release(h1.p);
    const bf16* res = xa.p;
    bf16* sc = nullptr;
    if (r.sc.w) {
      sc = alloc(static_cast<size_t>(M) * r.cout);
      GemmDesc d = linear(r.sc, xa.p, M, sc);
      d.lda = xa.C; d.K1 = xa.C;
      if (xb) { d.A2 = xb->p; d.lda2 = Cb; d.K2 = Cb; }
      gemm(d);
      res = sc;
    }
    Act out{alloc(static_cast<size_t>(M) * r.cout), r.cout, xa.H, xa.W, stats_alloc(B, r.cout)};
    {
      GemmDesc d = conv(r.c2, h2, B, xa.H, xa.W, out.p);
      d.residual = res; d.ld_res = r.cout;
      gemm_stats(d, out, B, xa.H, xa.W);
    }
    release(h2);
    if (sc) release(sc);
    return out;
  }

  // Frame-sharded 3-D attention: the QKV GEMM epilogue stores its K|V columns straight into the gathered K/V buffer of
  // every rank of the plan's K/V group (peer memory), a flag round of every rank makes them visible, attention reads all
  // F_total frames locally.
  void sharded_qkv_attention(const AttnW& a, const XfW& x, const bf16* normed, bf16* qkv, bf16* o, int M, int batch, int seq) {
    const int Cp = x.heads * x.dpad;
    const Exchange& X = m_.xch_;
    const PlanShape& sh = p_.shape;
    const int idx = p_.n3d++;
    const long long rows_local = seq;                                   // F_loc * hw tokens per CFG half
    const long long rows_global = static_cast<long long>(seq) / sh.F * sh.F_total;
    if (static_cast<size_t>(batch) * rows_global * 2 * Cp * sizeof(bf16) > X.kv_bytes) {
      set_error("K/V exchange buffer too small for this window (d4d_exchange_alloc)");
      if (!rc_) rc_ = 1;
      return;
    }
    // two ops: QKV GEMM + flag signal + flag wait, then the attention
    if (dry_) { op(nullptr, kOpGemm, 3); op(nullptr, kOpAttention); return; }
    GemmLaunch G[2];
    AttnLaunch A[2];
    for (int par = 0; par < 2; ++par) {
      GemmDesc d = linear(a.qkv, normed, M, qkv);
      d.kv_world = sh.kv_world; d.kv_col0 = Cp; d.kv_ld = 2 * Cp;
      d.kv_rows_local = rows_local; d.kv_rows_global = rows_global; d.kv_row_offset = static_cast<long long>(sh.shard) * rows_local;
      for (int r = 0; r < sh.kv_world; ++r) d.kv_dst[r] = static_cast<bf16*>(X.peer_kv[par][sh.kv_rank0 + r]);
      if (int rc = gemm_prepare(d, &G[par])) { if (!rc_) rc_ = rc; return; }
      AttnDesc t;
      t.q = qkv; t.ld_qkv = 3 * Cp;
      t.k = static_cast<const bf16*>(X.kv[par]); t.v = t.k + Cp; t.ld_kv = 2 * Cp;
      t.out = o; t.ld_out = Cp; t.batch = batch; t.seq = seq; t.seq_kv = static_cast<int>(rows_global);
      t.heads = x.heads; t.head_dim = x.dpad; t.scale = 1.0f / sqrtf(static_cast<float>(x.d));
      if (int rc = attn_prepare(t, &A[par])) { if (!rc_) rc_ = rc; return; }
    }
    // the flag round spans every rank, also those outside the K/V group: the CFG grid's noise store crosses groups, and
    // the write-after-read argument of DESIGN.md section 7 needs every exchange to wait for every rank
    KvFlagArgs fa;
    for (int r = 0; r < 8; ++r) fa.flags[r] = r < X.world ? X.peer_flags[r] : nullptr;
    fa.rank = X.rank; fa.world = X.world; fa.epoch = 0; fa.slot = 0;
    Plan* pl = &p_;
    const GemmLaunch G0 = G[0], G1 = G[1];
    const AttnLaunch A0 = A[0], A1 = A[1];
    op([=](cudaStream_t s) {
      const unsigned int counter = pl->epoch0 + idx;
      const int par = counter & 1;
      if (int rc = gemm_run(par ? G1 : G0, s)) return rc;
      KvFlagArgs f = fa;
      f.epoch = counter + 1;
      f.slot = par;
      if (int rc = kv_signal_run(f, s)) return rc;
      return kv_wait_run(f, s);
    }, kOpGemm, 3, gemm_flops(G0));
    op([=](cudaStream_t s) {
      const unsigned int counter = pl->epoch0 + idx;
      return attn_run((counter & 1) ? A1 : A0, s);
    }, kOpAttention, 1, attn_flops(A0.d));
  }

  void self_attention(const AttnW& a, const XfW& x, const bf16* normed, const bf16* resid, bf16* out, int M, int batch, int seq,
                      bool is3d = false) {
    const int Cp = x.heads * x.dpad;
    bf16* qkv = alloc(static_cast<size_t>(M) * 3 * Cp);
    bf16* o = nullptr;
    if (is3d && p_.shape.F_total > 0) {
      o = alloc(static_cast<size_t>(M) * Cp);
      sharded_qkv_attention(a, x, normed, qkv, o, M, batch, seq);
    } else {
      gemm(linear(a.qkv, normed, M, qkv));
      o = alloc(static_cast<size_t>(M) * Cp);
      AttnDesc d;
      d.q = qkv; d.k = qkv + Cp; d.v = qkv + 2 * Cp; d.ld_qkv = 3 * Cp;
      d.out = o; d.ld_out = Cp; d.batch = batch; d.seq = seq; d.heads = x.heads; d.head_dim = x.dpad;
      d.scale = 1.0f / sqrtf(static_cast<float>(x.d));
      attention(d);
    }
    release(qkv);
    {
      GemmDesc d = linear(a.out, o, M, out);
      d.residual = resid; d.ld_res = x.C;
      gemm(d);
    }
    release(o);
  }

  // TransformerMultiviewModel (+ its single MultiviewTransformerBlock): x -> new buffer
  Act transformer(const XfW& x, Act in) {
    const int B = p_.shape.B, hw = in.H * in.W, M = B * hw, C = x.C, num_frames = x.is3d ? p_.shape.F : 1;
    bf16* n = alloc(static_cast<size_t>(M) * C);
    groupnorm(in, nullptr, B, 1e-6f, x.gn, 0, n);
    bf16* t = alloc(static_cast<size_t>(M) * C);
    gemm(linear(x.pin, n, M, t));
    // attn1 (3-D when the window has more than one frame: batch = B / num_frames sequences of num_frames*hw local
    // tokens; a frame-sharded rank may hold a single frame of a larger window, and still attends over all F_total)
    const int window_frames = p_.shape.F_total > 0 ? p_.shape.F_total : p_.shape.F;
    layernorm(t, M, C, x.ln1, n);
    bf16* t1 = alloc(static_cast<size_t>(M) * C);
    self_attention(x.a1, x, n, t, t1, M, B / num_frames, num_frames * hw, x.is3d && window_frames > 1);
    release(t);
    if (x.has2) {  // attn2 with encoder_hidden_states=None: per-image self-attention
      layernorm(t1, M, C, x.ln2, n);
      bf16* t2 = alloc(static_cast<size_t>(M) * C);
      self_attention(x.a2, x, n, t1, t2, M, B, hw);
      release(t1);
      t1 = t2;
    }
    layernorm(t1, M, C, x.ln3, n);
    bf16* g = alloc(static_cast<size_t>(M) * 4 * C);
    {
      GemmDesc d = linear(x.ff1, n, M, g);
      d.geglu = 1; d.ldo = 4 * C;
      gemm(d);
    }
    release(n);
    bf16* t3 = alloc(static_cast<size_t>(M) * C);
    {
      GemmDesc d = linear(x.ff2, g, M, t3);
      d.residual = t1; d.ld_res = C;
      gemm(d);
    }
    release(g);
    release(t1);
    Act out{alloc(static_cast<size_t>(M) * C), C, in.H, in.W, stats_alloc(B, C)};
    {
      GemmDesc d = linear(x.pout, t3, M, out.p);
      d.residual = in.p; d.ld_res = C; d.stats_rows = hw;
      gemm_stats(d, out, B, in.H, in.W);
    }
    release(t3);
    return out;
  }

  Act conv3x3(const LinW& w, Act in, int act = 0, int n_img = 0) {
    if (n_img <= 0) n_img = p_.shape.B;
    const int M = n_img * in.H * in.W;
    Act out{alloc(static_cast<size_t>(M) * w.out), w.out, in.H, in.W};
    GemmDesc d = conv(w, in.p, n_img, in.H, in.W, out.p);
    d.act = act;
    gemm(d);
    return out;
  }

  int build() {
    Model& m = m_;
    const d4d_config& cfg = m.cfg_;
    Plan* pl = &p_;
    const PlanShape& sh = p_.shape;
    const int B = sh.B, F = sh.F, h = sh.h, w = sh.w;
    const int* ch = cfg.block_out_channels;
    const int C0 = ch[0], TE = 4 * C0, L = cfg.layers_per_block;
    const int M0 = B * h * w;
    D4D_CUDA_OK(cudaDeviceGetAttribute(&sms_, cudaDevAttrMultiProcessorCount, m.device_));  // (gemm_stats)

    if (!dry_ && p_.stats_words > 0) {  // GroupNorm statistics pool (size from the dry run): zeroed once per forward
      stats_pool_ = reinterpret_cast<long long*>(alloc(p_.stats_words * 4));
      long long* pool = stats_pool_;
      const size_t bytes = p_.stats_words * sizeof(long long);
      op([=](cudaStream_t s) {
        D4D_CUDA_OK(cudaMemsetAsync(pool, 0, bytes, s));
        return 0;
      });
    }

    // ---- 1. time (+ frame-index) embedding: UNET:519-546 ----
    bf16* tsin = alloc(static_cast<size_t>(B) * C0);
    op([=](cudaStream_t s) { return sinusoid_i64_run(pl->timestep, B, C0, cfg.flip_sin_to_cos, cfg.freq_shift, tsin, s); });
    bf16* e1 = alloc(static_cast<size_t>(B) * TE);
    {
      GemmDesc d = linear(m.time1_, tsin, B, e1);
      d.act = 1;
      gemm(d);
    }
    bf16* emb = alloc(static_cast<size_t>(B) * TE);
    gemm(linear(m.time2_, e1, B, emb));
    if (cfg.enable_tem_embeds) {
      float* pos = reinterpret_cast<float*>(alloc(static_cast<size_t>(B) * 2));
      if (!dry_) {
        std::vector<float> hp(B);
        for (int dmn = 0; dmn < sh.n_domains; ++dmn)
          for (int f = 0; f < F; ++f) hp[dmn * F + f] = sh.domains[dmn] == 0 ? 0.f : static_cast<float>((sh.shard * F + f) % std::max(1, (sh.F_total > 0 ? sh.F_total : F) / 2));
        if (cudaMemcpy(pos, hp.data(), sizeof(float) * B, cudaMemcpyHostToDevice) != cudaSuccess) rc_ = 2;
      }
      op([=](cudaStream_t s) { return sinusoid_run(pos, B, C0, 1, 0.f, tsin, s); });
      {
        GemmDesc d = linear(m.tem1_, tsin, B, e1);
        d.act = 1;
        gemm(d);
      }
      bf16* emb2 = alloc(static_cast<size_t>(B) * TE);
      {
        GemmDesc d = linear(m.tem2_, e1, B, emb2);
        d.residual = emb; d.ld_res = TE;
        gemm(d);
      }
      // pos stays allocated for the lifetime of the plan (it is read on every forward)
      release(emb);
      emb = emb2;
    }
    module_tap("time_embedding", Act{emb, TE, 1, 1});
    op([=](cudaStream_t s) { return silu_run(emb, static_cast<long long>(B) * TE, e1, s); });
    const int ldt = m.temb_all_.out;
    bf16* temb_all = alloc(static_cast<size_t>(B) * ldt);
    gemm(linear(m.temb_all_, e1, B, temb_all));
    release(tsin);
    release(e1);
    release(emb);

    // ---- 2. conv_in (+ pose encoder): UNET:549-554 ----
    bf16* pose_emb = nullptr;
    if (cfg.enable_pose_encoder) {
      const int Hs = 8 * h, Ws = 8 * w;
      // pose_neg: the skeleton batch is [1 constant CFG-negative image | B - pose_neg positive images] instead of B images
      // (pipeline_diffuman4d.py:349-356 makes every negative skeleton the same all(-1) image); its embedding is computed
      // once per forward and broadcast to the pose_neg negative images below
      const int PB = sh.pose_neg > 0 ? B - sh.pose_neg + 1 : B;
      const int PM0 = PB * h * w;
      const PoseW& pw = m.pose_;
      bf16* a0 = alloc(static_cast<size_t>(PB) * Hs * Ws * 4);  // 3 channels padded to 4
      op([=](cudaStream_t s) { return pose_conv0_run(pl->skeletons, PB, Hs, Ws, pw.conv[0].w, pw.conv[0].b, a0, s); });
      bf16* a1 = alloc(static_cast<size_t>(PB) * (Hs / 2) * (Ws / 2) * 16);
      op([=](cudaStream_t s) { return pose_conv_run(a0, PB, 4, Hs, Ws, pw.conv[1].w, pw.conv[1].b, 16, 4, 2, a1, s); });
      release(a0);
      bf16* a2 = alloc(static_cast<size_t>(PB) * (Hs / 2) * (Ws / 2) * 16);
      op([=](cudaStream_t s) { return pose_conv_run(a1, PB, 16, Hs / 2, Ws / 2, pw.conv[2].w, pw.conv[2].b, 16, 3, 1, a2, s); });
      release(a1);
      bf16* a3 = alloc(static_cast<size_t>(PB) * (Hs / 4) * (Ws / 4) * 32);
      op([=](cudaStream_t s) { return pose_conv_run(a2, PB, 16, Hs / 2, Ws / 2, pw.conv[3].w, pw.conv[3].b, 32, 4, 2, a3, s); });
      release(a2);
      bf16* a4 = alloc(static_cast<size_t>(PB) * (Hs / 4) * (Ws / 4) * 32);
      op([=](cudaStream_t s) { return pose_conv_run(a3, PB, 32, Hs / 4, Ws / 4, pw.conv[4].w, pw.conv[4].b, 32, 3, 1, a4, s); });
      release(a3);
      bf16* col = alloc(static_cast<size_t>(PM0) * 512);
      op([=](cudaStream_t s) { return im2col_nhwc_run(a4, PB, Hs / 4, Ws / 4, 32, 4, 2, col, s); });
      release(a4);
      bf16* a5 = alloc(static_cast<size_t>(PM0) * 64);
      {
        GemmDesc d = linear(pw.conv[5], col, PM0, a5);
        d.act = 1;
        gemm(d);
      }
      release(col);
      Act x5{a5, 64, h, w};
      Act x6 = conv3x3(pw.conv[6], x5, 1, PB);
      release(a5);
      Act x7 = conv3x3(pw.conv[7], x6, 1, PB);
      release(x6.p);
      pose_emb = alloc(static_cast<size_t>(PM0) * C0);
      {
        GemmDesc d = linear(pw.proj, x7.p, PM0, pose_emb);
        d.out_scale = pw.scale;
        gemm(d);
      }
      release(x7.p);
      if (sh.pose_neg > 0) {  // broadcast: images 0..pose_neg-1 <- embedding 0, the rest <- embeddings 1..B-pose_neg
        bf16* full = alloc(static_cast<size_t>(M0) * C0);
        bf16* small = pose_emb;
        const long long per_img = static_cast<long long>(h) * w * C0;
        const int n_neg = sh.pose_neg, n_pos = B - sh.pose_neg;
        op([=](cudaStream_t s) { return broadcast_neg_images_run(small, per_img, n_neg, n_pos, full, s); });
        release(small);
        pose_emb = full;
      }
    }
    Act x;
    {
      const int KP = m.kp_in(), cp = m.cin_pad(), Cin = cfg.in_channels;
      bf16* col = alloc(static_cast<size_t>(M0) * KP);
      op([=](cudaStream_t s) { return im2col_nchw_run(pl->sample, B, Cin, h, w, cp, KP, col, s); });
      x = {alloc(static_cast<size_t>(M0) * C0), C0, h, w, stats_alloc(B, C0)};
      GemmDesc d = linear(m.conv_in_, col, M0, x.p);
      if (pose_emb) { d.residual = pose_emb; d.ld_res = C0; }
      d.stats_rows = h * w;
      gemm_stats(d, x, B, h, w);
      release(col);
      if (pose_emb) release(pose_emb);
    }
    tap("conv_in", x);

    // ---- 3. down: UNET:557-565 ----
    std::vector<Act> skips;
    skips.push_back(x);
    for (int i = 0; i < 4; ++i) {
      const LevelW& lv = m.down_[i];
      for (int j = 0; j < L; ++j) {
        Act y = resnet(lv.res[j], x, nullptr, temb_all, ldt);
        module_tap(lv.res[j].path, y);
        if (i < 3) {
          Act z = transformer(lv.xf[j], y);
          module_tap(lv.xf[j].path, z);
          release(y.p);
          y = z;
        }
        x = y;
        skips.push_back(x);
      }
      if (i < 3) {  // Downsample2D: 3x3 stride-2 pad-1 conv, read in place through a strided tensor map
        const int Ho = x.H / 2, Wo = x.W / 2, Mo = B * Ho * Wo;
        const Act y{alloc(static_cast<size_t>(Mo) * x.C), x.C, Ho, Wo, stats_alloc(B, x.C)};
        gemm_stats(conv(lv.conv, x.p, B, x.H, x.W, y.p, 1), y, B, Ho, Wo);
        module_tap(lv.sampler, y);
        x = y;
        skips.push_back(x);
      }
      tap(lv.path, x);
    }
    // ---- 4. mid: UNET:568-572 ----
    {
      Act y = resnet(m.mid_res_[0], x, nullptr, temb_all, ldt);  // x is a skip: keep it
      module_tap(m.mid_res_[0].path, y);
      Act z = transformer(m.mid_xf_, y);
      module_tap(m.mid_xf_.path, z);
      release(y.p);
      Act u = resnet(m.mid_res_[1], z, nullptr, temb_all, ldt);
      module_tap(m.mid_res_[1].path, u);
      release(z.p);
      x = u;
    }
    tap("mid_block", x);
    // ---- 5. up: UNET:575-587 ----
    for (int i = 0; i < 4; ++i) {
      const LevelW& lv = m.up_[i];
      for (int j = 0; j <= L; ++j) {
        const Act sk = skips.back();
        skips.pop_back();
        Act y = resnet(lv.res[j], x, &sk, temb_all, ldt);
        module_tap(lv.res[j].path, y);
        release(x.p);
        release(sk.p);
        if (i > 0) {
          Act z = transformer(lv.xf[j], y);
          module_tap(lv.xf[j].path, z);
          release(y.p);
          y = z;
        }
        x = y;
      }
      if (i < 3) {  // Upsample2D (nearest x2, then 3x3 conv) as four sub-pixel phases on the low-resolution tensor
        const int H2 = 2 * x.H, W2 = 2 * x.W;
        Act y{alloc(static_cast<size_t>(B) * H2 * W2 * x.C), x.C, H2, W2, stats_alloc(B, x.C)};
        gemm_stats(conv(lv.conv, x.p, B, x.H, x.W, y.p, 3), y, B, x.H, x.W);  // (tiles walk the low-resolution grid)
        module_tap(lv.sampler, y);
        release(x.p);
        x = y;
      }
      tap(lv.path, x);
    }
    // ---- 6. out: UNET:590-593 ----
    {
      bf16* n = alloc(static_cast<size_t>(M0) * C0);
      groupnorm(x, nullptr, B, cfg.norm_eps, m.norm_out_, 1, n);
      release(x.p);
      Act na{n, C0, h, w};
      Act y = conv3x3(m.conv_out_, na);
      release(n);
      const int Co = cfg.out_channels;
      bf16* yp = y.p;
      op([=](cudaStream_t s) { return nhwc_to_nchw_run(yp, 16, B, Co, h * w, pl->out, s); });
      release(y.p);
    }
    release(temb_all);
    p_.taps.insert(p_.taps.end(), module_taps_.begin(), module_taps_.end());
    return rc_;
  }

 private:
  Model& m_;
  Plan& p_;
  bool dry_;
  char* base_;
  size_t bump_ = 0, peak_ = 0;
  std::vector<std::pair<size_t, size_t>> free_;
  std::map<size_t, size_t> live_;
  long long* stats_pool_ = nullptr;
  size_t stats_used_ = 0;
  int sms_ = 0;
  int rc_ = 0;
  std::vector<Plan::Tap> module_taps_;
};

Plan* Model::find_plan(int n_domains, int B, int F, int h, int w) {
  for (auto& kv : plans_) {
    const PlanShape& s = kv.second->shape;
    if (s.n_domains == n_domains && s.B == B && s.F == F && s.h == h && s.w == w) return kv.second.get();
  }
  return nullptr;
}

int Model::get_plan(const int* domain_ids, int n_domains, int B, int F, int h, int w, Plan** out, int F_total, int pose_neg,
                    int kv_world) {
  if (!finalized_) {
    set_error("weights not finalized (call d4d_finalize_weights)");
    return 3;
  }
  D4D_REQUIRE(domain_ids != nullptr, "null argument");
  D4D_REQUIRE(B > 0 && F > 0 && n_domains > 0, "empty batch");
  if (n_domains * F != B) {
    // same message as the reference's ValueError (unet_multiview_condition.py:524-525)
    set_error("num_frames: " + std::to_string(F) + " * len(domains): " + std::to_string(n_domains) + " != len(emb): " + std::to_string(B));
    return 1;
  }
  D4D_REQUIRE(h % 8 == 0 && w % 8 == 0 && h > 0 && w > 0, "latent height/width must be divisible by 8");
  for (int i = 0; i < n_domains; ++i) D4D_REQUIRE(domain_ids[i] == 0 || domain_ids[i] == 1, "Invalid domain for temporal embedding");
  // every *_sharded call runs the sharded plan, also with world = 1 (rank 0 exchanging with itself)
  const bool sharded = F_total > 0;
  PlanShape s;
  s.n_domains = n_domains; s.B = B; s.F = F; s.h = h; s.w = w;
  s.domains.assign(domain_ids, domain_ids + n_domains);
  if (sharded) {
    D4D_REQUIRE(xch_.ready && xch_.world >= 1, "frame-sharded forward needs d4d_exchange_open first");
    // the K/V group: kv_world consecutive ranks, this rank's frame shard its place in them (0: every rank)
    if (kv_world == 0) kv_world = xch_.world;
    D4D_REQUIRE(kv_world >= 1 && xch_.world % kv_world == 0, "the K/V group size must divide the world");
    D4D_REQUIRE(F * kv_world == F_total, "F_total must equal the K/V group size * local frames");
    s.F_total = F_total;
    s.kv_world = kv_world;
    s.kv_rank0 = xch_.rank / kv_world * kv_world;
    s.shard = xch_.rank - s.kv_rank0;
  }
  D4D_REQUIRE(pose_neg >= 0 && pose_neg <= B, "pose_neg must be in [0, B]");
  s.pose_neg = cfg_.enable_pose_encoder ? pose_neg : 0;
  const std::string key = plan_key(s);
  auto it = plans_.find(key);
  if (it != plans_.end()) {
    *out = it->second.get();
    return 0;
  }
  D4D_CUDA_OK(cudaSetDevice(device_));
  std::unique_ptr<Plan> p(new Plan());
  p->shape = s;
  size_t peak = 0;
  {
    Plan scratch;
    scratch.shape = s;
    PlanBuilder dry(*this, scratch, true, nullptr);
    if (int rc = dry.build()) return rc;
    peak = dry.peak();
    p->stats_words = dry.stats_words();
    peak += (p->stats_words * sizeof(long long) + 255) & ~size_t(255);
  }
  D4D_CUDA_OK(cudaMalloc(&p->arena, peak + 1024));
  p->arena_bytes = peak;
  PlanBuilder real(*this, *p, false, static_cast<char*>(p->arena));
  if (int rc = real.build()) return rc;
  *out = p.get();
  plans_[key] = std::move(p);
  return 0;
}

int Model::run_ops(Plan& p, const bf16* sample, const long long* timestep, const bf16* skeletons, const NchwDst& out, size_t n,
                   cudaStream_t stream, bool timed) {
  D4D_REQUIRE(sample && timestep && (out.n > 0 || n < p.ops.size()), "null argument");
  D4D_REQUIRE(!cfg_.enable_pose_encoder || skeletons != nullptr, "skeletons are required when enable_pose_encoder");
  D4D_REQUIRE(!cfg_.center_input_sample, "center_input_sample is not supported");
  D4D_CUDA_OK(cudaSetDevice(device_));
  p.sample = sample; p.timestep = timestep; p.skeletons = skeletons; p.out = out;
  p.epoch0 = xch_.epoch_base;  // global, monotonic exchange counter: every rank runs the same forwards in the same order
  while (timed && p.events.size() < n + 1) {
    cudaEvent_t e;
    D4D_CUDA_OK(cudaEventCreate(&e));
    p.events.push_back(e);
  }
  for (size_t i = 0; i < n; ++i) {
    if (timed) D4D_CUDA_OK(cudaEventRecord(p.events[i], stream));
    if (int rc = p.ops[i].run(stream)) return rc;
  }
  if (timed) D4D_CUDA_OK(cudaEventRecord(p.events[n], stream));
  return 0;
}

int Model::forward(const bf16* sample, const long long* timestep, const bf16* skeletons, const int* domain_ids,
                   int n_domains, int B, int F, int h, int w, bf16* out, cudaStream_t stream, int F_total, int pose_neg) {
  return forward(sample, timestep, skeletons, domain_ids, n_domains, B, F, h, w, one_dst(out), stream, F_total, pose_neg);
}

int Model::forward(const bf16* sample, const long long* timestep, const bf16* skeletons, const int* domain_ids,
                   int n_domains, int B, int F, int h, int w, const NchwDst& out, cudaStream_t stream, int F_total,
                   int pose_neg, int kv_world) {
  Plan* p = nullptr;
  if (int rc = get_plan(domain_ids, n_domains, B, F, h, w, &p, F_total, pose_neg, kv_world)) return rc;
  if (int rc = run_ops(*p, sample, timestep, skeletons, out, p->ops.size(), stream)) return rc;
  xch_.epoch_base += static_cast<unsigned int>(p->n3d);
  return 0;
}

int Model::debug_tap(const bf16* sample, const long long* timestep, const bf16* skeletons, const int* domain_ids, int n_domains,
                     int B, int F, int h, int w, int tap, bf16* out, char* name64, int* dims3, cudaStream_t stream) {
  Plan* p = nullptr;
  if (int rc = get_plan(domain_ids, n_domains, B, F, h, w, &p)) return rc;
  if (tap < 0 || tap >= static_cast<int>(p->taps.size())) {
    set_error("tap index out of range");
    return 1;
  }
  const Plan::Tap& t = p->taps[tap];
  if (name64) {
    strncpy(name64, t.name.c_str(), 63);
    name64[63] = 0;
  }
  if (dims3) { dims3[0] = t.C; dims3[1] = t.H; dims3[2] = t.W; }
  if (!out) return 0;
  if (int rc = run_ops(*p, sample, timestep, skeletons, one_dst(nullptr), t.n_ops, stream)) return rc;
  return nhwc_to_nchw_run(t.p, t.C, B, t.C, t.H * t.W, out, stream);
}

int Model::exchange_alloc(size_t kv_bytes, unsigned char* handles_out) {
  D4D_REQUIRE(handles_out != nullptr && kv_bytes > 0, "exchange_alloc arguments");
  D4D_REQUIRE(xch_.kv[0] == nullptr, "exchange buffers already allocated");
  D4D_CUDA_OK(cudaSetDevice(device_));
  for (int i = 0; i < 2; ++i) {
    D4D_CUDA_OK(cudaMalloc(&xch_.kv[i], kv_bytes));
    dev_allocs_.push_back(xch_.kv[i]);
  }
  void* fl = nullptr;
  D4D_CUDA_OK(cudaMalloc(&fl, 64 * sizeof(unsigned int)));
  D4D_CUDA_OK(cudaMemset(fl, 0, 64 * sizeof(unsigned int)));
  dev_allocs_.push_back(fl);
  xch_.flags = static_cast<unsigned int*>(fl);
  xch_.kv_bytes = kv_bytes;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t hnd;
  void* ptrs[3] = {xch_.kv[0], xch_.kv[1], fl};
  for (int i = 0; i < 3; ++i) {
    D4D_CUDA_OK(cudaIpcGetMemHandle(&hnd, ptrs[i]));
    memcpy(handles_out + 64 * i, &hnd, 64);
  }
  return 0;
}

int Model::exchange_open(int rank, int world, const unsigned char* all_handles) {
  D4D_REQUIRE(all_handles != nullptr && world >= 1 && world <= 8 && rank >= 0 && rank < world, "exchange_open arguments");
  D4D_REQUIRE(xch_.kv[0] != nullptr, "call d4d_exchange_alloc first");
  D4D_REQUIRE(!xch_.ready, "exchange already opened");
  D4D_CUDA_OK(cudaSetDevice(device_));
  for (int r = 0; r < world; ++r) {
    if (r == rank) {
      xch_.peer_kv[0][r] = xch_.kv[0];
      xch_.peer_kv[1][r] = xch_.kv[1];
      xch_.peer_flags[r] = xch_.flags;
      continue;
    }
    void* ptrs[3];
    for (int i = 0; i < 3; ++i) {
      cudaIpcMemHandle_t hnd;
      memcpy(&hnd, all_handles + (static_cast<size_t>(r) * 3 + i) * 64, 64);
      D4D_CUDA_OK(cudaIpcOpenMemHandle(&ptrs[i], hnd, cudaIpcMemLazyEnablePeerAccess));
    }
    xch_.peer_kv[0][r] = ptrs[0];
    xch_.peer_kv[1][r] = ptrs[1];
    xch_.peer_flags[r] = static_cast<unsigned int*>(ptrs[2]);
  }
  xch_.rank = rank;
  xch_.world = world;
  xch_.ready = true;
  return 0;
}

int Model::profile(const bf16* sample, const long long* timestep, const bf16* skeletons, const int* domain_ids, int n_domains,
                   int B, int F, int h, int w, bf16* out, cudaStream_t stream, float* ms_by_kind, int* launches_by_kind,
                   double* flops_by_kind) {
  D4D_REQUIRE(ms_by_kind && launches_by_kind && flops_by_kind, "null argument");
  Plan* p = nullptr;
  if (int rc = get_plan(domain_ids, n_domains, B, F, h, w, &p)) return rc;
  const size_t n = p->ops.size();
  if (int rc = run_ops(*p, sample, timestep, skeletons, one_dst(out), n, stream, true)) return rc;
  D4D_CUDA_OK(cudaEventSynchronize(p->events[n]));
  for (int k = 0; k < kNumOpKinds; ++k) { ms_by_kind[k] = 0.f; launches_by_kind[k] = 0; flops_by_kind[k] = 0.0; }
  for (size_t i = 0; i < n; ++i) {
    float ms = 0.f;
    D4D_CUDA_OK(cudaEventElapsedTime(&ms, p->events[i], p->events[i + 1]));
    const PlanOp& op = p->ops[i];
    ms_by_kind[op.kind] += ms;
    launches_by_kind[op.kind] += op.launches;
    flops_by_kind[op.kind] += op.flops;
  }
  return 0;
}

int Model::denoise_window(bf16* latents, const bf16* pixel, const bf16* plucker, const bf16* skeletons, const bf16* mask,
                          long long* ts_idx, const WindowStep& step, float guidance, int domain, int F, int h, int w,
                          int num_steps, cudaStream_t stream, int F_total, CfgMode mode) {
  D4D_REQUIRE(latents && pixel && plucker && mask && ts_idx && step.tables() == 1, "null argument");
  D4D_REQUIRE(domain == 0 || domain == 1, "Invalid domain");
  const bool cfg_on = guidance > 1.0f;
  // guidance <= 1 has no halves: the plain step runs and nothing is exchanged
  const bool split = mode != CfgMode::kWhole && cfg_on;
  const int B = cfg_on ? 2 * F : F;
  const bool pose = cfg_.enable_pose_encoder != 0;
  const int Cin = 4 + 6 + (pose ? 0 : 4) + 1;
  const int Co = cfg_.out_channels;
  D4D_REQUIRE(Cin == cfg_.in_channels, "in_channels does not match the latent/plucker/skeleton/mask channel layout");
  D4D_REQUIRE(skeletons != nullptr, "skeletons required");
  const int world = xch_.world;
  if (mode == CfgMode::kGrid)
    D4D_REQUIRE(world == 1 || world == 2 || world == 4 || world == 6 || world == 8,
                "the CFG grid runs on 2 * R ranks with R in {1, 2, 3, 4} (or 1 as a loopback)");
  // frame shards per CFG half: R > 1 only on a grid of 4, 6 or 8 ranks
  const int R = mode == CfgMode::kGrid && world > 1 ? world / 2 : 1;
  Plan* grid_plan = nullptr;  // R > 1: this rank's plan, built before any launch (it refuses a too small K/V buffer)
  if (split) {
    D4D_REQUIRE(xch_.ready, "the CFG-split window needs d4d_exchange_open first");
    D4D_REQUIRE(mode == CfgMode::kGrid || world <= 2, "the CFG-split window runs on 1 (loopback) or 2 ranks");
    D4D_REQUIRE(F > 0 && h > 0 && w > 0, "empty window");
    D4D_REQUIRE(F % R == 0, "the window's frames (" + std::to_string(F) + ") must be divisible by the frame shards per CFG "
                "half (" + std::to_string(R) + ")");
    D4D_REQUIRE(2ull * F * Co * h * w * sizeof(bf16) <= xch_.kv_bytes,
                "the window's noise (2 * F * out_channels * h * w bf16) does not fit the exchange buffer (d4d_exchange_alloc)");
    if (R > 1) {
      const int doms1[1] = {domain};
      const int k = xch_.rank / R;
      if (int rc = get_plan(doms1, 1, F / R, F / R, h, w, &grid_plan, F, pose && k == 0 ? F / R : 0, R)) return rc;
    }
  }
  D4D_CUDA_OK(cudaSetDevice(device_));
  const std::string key = std::to_string(B) + "_" + std::to_string(F) + "_" + std::to_string(h) + "_" + std::to_string(w);
  auto it = wbufs_.find(key);
  if (it == wbufs_.end()) {
    std::unique_ptr<WindowBufs> wb(new WindowBufs());
    const size_t hw = static_cast<size_t>(h) * w;
    D4D_CUDA_OK(cudaMalloc(&wb->sample, sizeof(bf16) * B * Cin * hw));
    D4D_CUDA_OK(cudaMalloc(&wb->timestep, sizeof(long long) * B));
    if (pose) {
      D4D_CUDA_OK(cudaMalloc(&wb->skel, sizeof(bf16) * (F + 1) * 3 * 64 * hw));
      if (int rc = fill_bf16_run(wb->skel, static_cast<long long>(3) * 64 * hw, -1.0f, stream)) return rc;  // constant negative image
    }
    D4D_CUDA_OK(cudaMalloc(&wb->noise, sizeof(bf16) * B * Co * hw));
    D4D_CUDA_OK(cudaMalloc(&wb->ts_tmp, sizeof(long long) * F));
    it = wbufs_.emplace(key, std::move(wb)).first;
  }
  WindowBufs& wb = *it->second;
  const bool multistep = step.state.lower_order_nums != nullptr;
  if (multistep && !wb.order_tmp) D4D_CUDA_OK(cudaMalloc(&wb.order_tmp, sizeof(int) * F));
  const int doms[2] = {domain, domain};
  const int hw = h * w;
  // The scheduler step runs in place (each element is read and written by the same thread); the counters go through
  // ts_tmp / order_tmp, since a kernel may not overwrite the counters its other blocks still read.
  StepArgs sa;
  sa.noise = wb.noise; sa.latents = latents; sa.mask = mask; sa.timestep_indices = ts_idx;
  sa.F = F; sa.chw = 4 * hw; sa.hw = hw; sa.cfg = cfg_on ? 1 : 0; sa.guidance = guidance;
  sa.out = latents; sa.ts_out = wb.ts_tmp;
  SolverState state = step.state;
  state.lower_order_nums_out = wb.order_tmp;
  // the scheduler's checks, before the window's work is enqueued; the input assembly reads its timestep table
  const int64_t* timesteps_table = nullptr;
  int n_steps = 0;
  if (int rc = step.with_table([&](const auto& s) {
        timesteps_table = s.timesteps_table;
        n_steps = s.n_steps;
        return cfg_step_run(sa, s, state, stream, false);
      }))
    return rc;
  for (int s = 0; s < num_steps; ++s) {
    AssembleArgs a;
    a.latents = latents; a.pixel = pixel; a.plucker = plucker; a.skel_latents = pose ? nullptr : skeletons; a.mask = mask;
    a.timestep_indices = ts_idx; a.timesteps_table = reinterpret_cast<const long long*>(timesteps_table);
    a.n_steps = n_steps; a.F = F; a.h = h; a.w = w; a.cfg = cfg_on ? 1 : 0;
    a.sample = wb.sample; a.timestep_out = wb.timestep;
    if (split) {
      // CFG split / grid (DESIGN.md section 7): the UNet on this rank's half k (a loopback runs both) of its frame shard r
      // (Fr = F / R frames), its noise stored at rows [k*F + r*Fr, k*F + (r+1)*Fr) of the exchange buffer parity that
      // follows the forward's n3d K/V exchanges, on every rank; one flag round; the step reads the gathered [2F] noise in
      // place.  Every rank then computes the step from the same bits.
      const int Fr = F / R, r = xch_.rank % R;
      const int k0 = world == 1 ? 0 : xch_.rank / R, k1 = world == 1 ? 2 : k0 + 1;
      const unsigned int n3d = grid_plan ? static_cast<unsigned int>(grid_plan->n3d) : 0u;
      for (int k = k0; k < k1; ++k) {
        a.half = k;
        // a grid rank writes sample rows for its frame shard only, but overwrites every cond frame's latents, so that
        // every rank's whole-window latents stay those of the single-GPU step
        if (R > 1) { a.f0 = r * Fr; a.n_f = Fr; }
        if (int rc = assemble_input_run(a, stream)) return rc;
        const unsigned int e = xch_.epoch_base + n3d;
        NchwDst dst = {};
        dst.n = world;
        for (int g = 0; g < world; ++g)
          dst.p[g] = static_cast<bf16*>(xch_.peer_kv[e & 1][g]) + (static_cast<size_t>(k) * F + r * Fr) * Co * hw;
        // every negative skeleton is the constant image wb.skel[0]: the negative half encodes it once (pose_neg = Fr)
        const bf16* skel_in = pose ? (k == 0 ? wb.skel : skeletons + static_cast<size_t>(r) * Fr * 3 * 64 * hw) : nullptr;
        if (int rc = forward(wb.sample, wb.timestep, skel_in, doms, 1, Fr, Fr, h, w, dst, stream, R > 1 ? F : 0,
                             pose && k == 0 ? Fr : 0, R > 1 ? R : 0))
          return rc;
      }
      const unsigned int e = xch_.epoch_base;  // the exchange the flag round closes: the noise's buffer parity
      if (int rc = flag_round(stream)) return rc;
      sa.noise = static_cast<const bf16*>(xch_.kv[e & 1]);
    } else {
      if (int rc = assemble_input_run(a, stream)) return rc;
      const bf16* skel_in = nullptr;
      if (pose) {
        if (cfg_on) {  // [negative (filled once) | F positive images]
          D4D_CUDA_OK(cudaMemcpyAsync(wb.skel + static_cast<size_t>(3) * 64 * hw, skeletons, sizeof(bf16) * F * 3 * 64 * hw,
                                      cudaMemcpyDeviceToDevice, stream));
          skel_in = wb.skel;
        } else {
          skel_in = skeletons;
        }
      }
      if (int rc = forward(wb.sample, wb.timestep, skel_in, doms, cfg_on ? 2 : 1, B, F, h, w, wb.noise, stream, F_total,
                           pose && cfg_on ? F : 0))
        return rc;
    }
    if (int rc = step.with_table([&](const auto& s) { return cfg_step_run(sa, s, state, stream); })) return rc;
    D4D_CUDA_OK(cudaMemcpyAsync(ts_idx, wb.ts_tmp, sizeof(long long) * F, cudaMemcpyDeviceToDevice, stream));
    if (multistep)
      D4D_CUDA_OK(cudaMemcpyAsync(step.state.lower_order_nums_out, wb.order_tmp, sizeof(int) * F, cudaMemcpyDeviceToDevice,
                                  stream));
  }
  return 0;
}

// One flag round, closing exchange e = epoch_base (the caller enqueued its stores into buffer parity e & 1 before it):
// every rank's flag slot e & 1 receives epoch e + 1, the exchange is counted, and the stream waits for every rank's signal.
int Model::flag_round(cudaStream_t stream) {
  const unsigned int counter = xch_.epoch_base;
  KvFlagArgs f;
  for (int r = 0; r < 8; ++r) f.flags[r] = r < xch_.world ? xch_.peer_flags[r] : nullptr;
  f.rank = xch_.rank; f.world = xch_.world; f.epoch = counter + 1; f.slot = counter & 1;
  xch_.epoch_base += 1;  // the stores are enqueued: every rank counts this exchange, whatever happens below
  if (int rc = kv_signal_run(f, stream)) return rc;
  return kv_wait_run(f, stream);
}

// One more exchange of the global epoch sequence (DESIGN.md section 7): counter e = epoch_base stores into parity e & 1 of
// every rank's K/V buffers, signals epoch e + 1 in flag slot e & 1, and reads the gathered window back after the wait.  The
// next write to parity e & 1 by any rank is exchange e + 2, which needs this rank's signal of exchange e + 1, enqueued after
// the copies below: a rank one exchange ahead cannot overwrite the rows a peer is still reading.
int Model::window_exchange(const bf16* latents, const long long* ts_idx, const bf16* x0_prev, const int* lower_order_nums,
                           int F, int F_total, int h, int w, bf16* latents_out, long long* ts_out, bf16* x0_out,
                           int* lon_out, cudaStream_t stream) {
  D4D_REQUIRE(xch_.ready, "window exchange needs d4d_exchange_open first");
  D4D_REQUIRE(h > 0 && w > 0, "latent height/width");
  D4D_REQUIRE(latents_out && ts_out, "null argument");
  const bool dpm = x0_prev != nullptr;
  D4D_REQUIRE((x0_out != nullptr) == dpm && (lon_out != nullptr) == dpm,
              "x0_prev, lower_order_nums and their outputs are given together or not at all");
  D4D_CUDA_OK(cudaSetDevice(device_));
  const unsigned int counter = xch_.epoch_base;
  const int par = counter & 1;
  WindowScatterArgs a;
  for (int r = 0; r < 8; ++r) a.dst[r] = r < xch_.world ? xch_.peer_kv[par][r] : nullptr;
  a.world = xch_.world; a.rank = xch_.rank; a.F_local = F; a.F_total = F_total;
  a.chw = 4ll * h * w;
  a.latents = latents; a.ts = ts_idx; a.x0_prev = x0_prev; a.lower_order_nums = lower_order_nums;
  if (int rc = window_scatter_run(a, xch_.kv_bytes, stream)) return rc;
  if (int rc = flag_round(stream)) return rc;
  const char* g = static_cast<const char*>(xch_.kv[par]);
  const WindowResultLayout L = window_result_layout(F_total, a.chw, dpm);
  D4D_CUDA_OK(cudaMemcpyAsync(latents_out, g, L.x0, cudaMemcpyDeviceToDevice, stream));
  D4D_CUDA_OK(cudaMemcpyAsync(ts_out, g + L.ts, sizeof(long long) * F_total, cudaMemcpyDeviceToDevice, stream));
  if (dpm) {
    D4D_CUDA_OK(cudaMemcpyAsync(x0_out, g + L.x0, L.x0, cudaMemcpyDeviceToDevice, stream));
    D4D_CUDA_OK(cudaMemcpyAsync(lon_out, g + L.lon, sizeof(int) * F_total, cudaMemcpyDeviceToDevice, stream));
  }
  return 0;
}

}  // namespace d4d
