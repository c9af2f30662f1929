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

int silu_run(const bf16* x, long long n, bf16* out, cudaStream_t stream);
int broadcast_neg_images_run(const bf16* small, long long per_img, int F, bf16* full, cudaStream_t stream);
int fill_bf16_run(bf16* p, long long n, float v, cudaStream_t stream);

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

std::string plan_key(const int* dom, int nd, int B, int F, int h, int w) {
  std::string k = std::to_string(B) + "_" + std::to_string(F) + "_" + std::to_string(h) + "_" + std::to_string(w) + "_";
  for (int i = 0; i < nd; ++i) k += dom[i] ? 't' : 's';
  return k;
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
  cudaFree(latents_tmp);
  cudaFree(ts_tmp);
}

// =================================================================================================
// weights
// =================================================================================================
Model::Model(const d4d_config& cfg, int device) : cfg_(cfg), device_(device) { declare_keys(); }

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

void Model::declare_keys() {
  const int* ch = cfg_.block_out_channels;
  const int C0 = ch[0], TE = 4 * C0, L = cfg_.layers_per_block;
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
    norm(p + ".norm1", cin);
    conv(p + ".conv1", cout, cin, 3);
    lin(p + ".time_emb_proj", cout, TE);
    norm(p + ".norm2", cout);
    conv(p + ".conv2", cout, cout, 3);
    if (cin != cout) conv(p + ".conv_shortcut", cout, cin, 1);
  };
  auto xf = [&](const std::string& p, int C, bool attn2) {
    norm(p + ".norm", C);
    lin(p + ".proj_in", C, C);
    const std::string b = p + ".transformer_blocks.0";
    norm(b + ".norm1", C);
    lin(b + ".attn1.to_q", C, C, false);
    lin(b + ".attn1.to_k", C, C, false);
    lin(b + ".attn1.to_v", C, C, false);
    lin(b + ".attn1.to_out.0", C, C);
    if (attn2) {
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
  };
  conv("conv_in", C0, cfg_.in_channels, 3);
  lin("time_embedding.linear_1", TE, C0);
  lin("time_embedding.linear_2", TE, TE);
  if (cfg_.enable_tem_embeds) {
    lin("temporal_pos_embed.linear_1", TE, C0);
    lin("temporal_pos_embed.linear_2", TE, TE);
  }
  if (cfg_.enable_pose_encoder) {
    static const int spec[8][3] = {{3, 3, 3}, {3, 16, 4}, {16, 16, 3}, {16, 32, 4}, {32, 32, 3}, {32, 64, 4}, {64, 64, 3}, {64, 128, 3}};
    for (int i = 0; i < 8; ++i) conv("pose_encoder.conv_layers." + std::to_string(2 * i), spec[i][1], spec[i][0], spec[i][2]);
    conv("pose_encoder.final_proj", C0, 128, 1);
    need("pose_encoder.scale", {1});
  }
  int cout = C0;
  for (int i = 0; i < 4; ++i) {
    const int cin = cout;
    cout = ch[i];
    const std::string p = "down_blocks." + std::to_string(i);
    for (int j = 0; j < L; ++j) {
      resnet(p + ".resnets." + std::to_string(j), j == 0 ? cin : cout, cout);
      if (i < 3) xf(p + ".attentions." + std::to_string(j), cout, cfg_.has_attn2[i] != 0);
    }
    if (i < 3) conv(p + ".downsamplers.0.conv", cout, cout, 3);
  }
  resnet("mid_block.resnets.0", ch[3], ch[3]);
  xf("mid_block.attentions.0", ch[3], cfg_.has_attn2[3] != 0);
  resnet("mid_block.resnets.1", ch[3], ch[3]);
  cout = ch[3];
  for (int i = 0; i < 4; ++i) {
    const int cprev = cout;
    cout = ch[3 - i];
    const int cin = ch[3 - std::min(i + 1, 3)];
    const std::string p = "up_blocks." + std::to_string(i);
    for (int j = 0; j <= L; ++j) {
      const int skip = j == L ? cin : cout;
      const int rin = j == 0 ? cprev : cout;
      resnet(p + ".resnets." + std::to_string(j), rin + skip, cout);
      if (i > 0) xf(p + ".attentions." + std::to_string(j), cout, cfg_.has_attn2[3 - i] != 0);
    }
    if (i < 3) conv(p + ".upsamplers.0.conv", cout, cout, 3);
  }
  norm("conv_norm_out", C0);
  conv("conv_out", cfg_.out_channels, C0, 3);
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
  auto normw = [&](const std::string& p, int c) {
    NormW n;
    n.g = up_f32(T(p + ".weight"));
    n.b = up_f32(T(p + ".bias"));
    n.c = c;
    return n;
  };
  auto linw = [&](const std::string& p, int out, int in, bool bias = true) {
    LinW l;
    l.w = up_bf16(T(p + ".weight"));
    l.b = bias ? up_f32(T(p + ".bias")) : nullptr;
    l.in = in;
    l.out = out;
    return l;
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
  auto convw = [&](const std::string& p, int cout, int cin) {
    LinW l;
    l.w = up_bf16(conv_gemm_layout(T(p + ".weight"), cout, cin, 3));
    l.b = up_f32(T(p + ".bias"));
    l.in = cin;
    l.out = cout;
    return l;
  };
  const int* ch = cfg_.block_out_channels;
  const int C0 = ch[0], TE = 4 * C0, L = cfg_.layers_per_block;

  std::vector<float> temb_w, temb_b;
  auto resnetw = [&](const std::string& p, int cin, int cout) {
    ResnetW r;
    r.cin = cin;
    r.cout = cout;
    r.n1 = normw(p + ".norm1", cin);
    r.c1 = convw(p + ".conv1", cout, cin);
    r.n2 = normw(p + ".norm2", cout);
    r.c2 = convw(p + ".conv2", cout, cout);
    if (cin != cout) r.sc = linw(p + ".conv_shortcut", cout, cin);
    r.temb_off = static_cast<int>(temb_b.size());
    const auto& tw = T(p + ".time_emb_proj.weight");
    const auto& tb = T(p + ".time_emb_proj.bias");
    temb_w.insert(temb_w.end(), tw.begin(), tw.end());
    temb_b.insert(temb_b.end(), tb.begin(), tb.end());
    return r;
  };
  auto attnw = [&](const std::string& p, int C, int heads, int d, int dpad) {
    AttnW a;
    const int Cp = heads * dpad;
    std::vector<float> qkv(static_cast<size_t>(3) * Cp * C, 0.f);
    const char* names[3] = {".to_q.weight", ".to_k.weight", ".to_v.weight"};
    for (int s = 0; s < 3; ++s) {
      const auto& w = T(p + names[s]);
      for (int hh = 0; hh < heads; ++hh)
        for (int j = 0; j < d; ++j)
          memcpy(&qkv[(static_cast<size_t>(s) * Cp + hh * dpad + j) * C], &w[static_cast<size_t>(hh * d + j) * C],
                 sizeof(float) * C);
    }
    a.qkv.w = up_bf16(qkv);
    a.qkv.b = nullptr;
    a.qkv.in = C;
    a.qkv.out = 3 * Cp;
    const auto& wo = T(p + ".to_out.0.weight");
    std::vector<float> o(static_cast<size_t>(C) * Cp, 0.f);
    for (int r = 0; r < C; ++r)
      for (int hh = 0; hh < heads; ++hh)
        for (int j = 0; j < d; ++j) o[static_cast<size_t>(r) * Cp + hh * dpad + j] = wo[static_cast<size_t>(r) * C + hh * d + j];
    a.out.w = up_bf16(o);
    a.out.b = up_f32(T(p + ".to_out.0.bias"));
    a.out.in = Cp;
    a.out.out = C;
    return a;
  };
  auto xfw = [&](const std::string& p, int C, int heads, bool attn2) {
    XfW x;
    x.C = C;
    x.heads = heads;
    x.d = C / heads;
    x.dpad = pad_head_dim(x.d);
    x.has2 = attn2;
    x.gn = normw(p + ".norm", C);
    x.pin = linw(p + ".proj_in", C, C);
    x.pout = linw(p + ".proj_out", C, C);
    const std::string b = p + ".transformer_blocks.0";
    x.ln1 = normw(b + ".norm1", C);
    x.a1 = attnw(b + ".attn1", C, heads, x.d, x.dpad);
    if (attn2) {
      x.ln2 = normw(b + ".norm2", C);
      x.a2 = attnw(b + ".attn2", C, heads, x.d, x.dpad);
    }
    x.ln3 = normw(b + ".norm3", C);
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
    x.ff1.w = up_bf16(wi);
    x.ff1.b = up_f32(bi);
    x.ff1.in = C;
    x.ff1.out = N;
    x.ff2 = linw(b + ".ff.net.2", C, 4 * C);
    return x;
  };

  {  // conv_in -> [C0][KP] with k = tap*16 + c
    const int Cin = cfg_.in_channels, KP = kp_in(), cp = cin_pad();
    const auto& w = T("conv_in.weight");
    std::vector<float> o(static_cast<size_t>(C0) * KP, 0.f);
    for (int co = 0; co < C0; ++co)
      for (int ci = 0; ci < Cin; ++ci)
        for (int t = 0; t < 9; ++t) o[static_cast<size_t>(co) * KP + t * cp + ci] = w[(static_cast<size_t>(co) * Cin + ci) * 9 + t];
    conv_in_.w = up_bf16(o);
    conv_in_.b = up_f32(T("conv_in.bias"));
    conv_in_.in = KP;
    conv_in_.out = C0;
  }
  time1_ = linw("time_embedding.linear_1", TE, C0);
  time2_ = linw("time_embedding.linear_2", TE, TE);
  if (cfg_.enable_tem_embeds) {
    tem1_ = linw("temporal_pos_embed.linear_1", TE, C0);
    tem2_ = linw("temporal_pos_embed.linear_2", TE, TE);
  }
  if (cfg_.enable_pose_encoder) {
    static const int spec[8][3] = {{3, 3, 3}, {3, 16, 4}, {16, 16, 3}, {16, 32, 4}, {32, 32, 3}, {32, 64, 4}, {64, 64, 3}, {64, 128, 3}};
    for (int i = 0; i < 8; ++i) {
      const std::string p = "pose_encoder.conv_layers." + std::to_string(2 * i);
      const int cin = spec[i][0], cout = spec[i][1], k = spec[i][2];
      const auto& w = T(p + ".weight");
      LinW l;
      l.in = cin;
      l.out = cout;
      l.b = up_f32(T(p + ".bias"));
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
      }
      pose_.conv[i] = l;
    }
    pose_.proj = linw("pose_encoder.final_proj", C0, 128);
    pose_.scale = T("pose_encoder.scale")[0];
  }
  int cout = C0;
  for (int i = 0; i < 4; ++i) {
    const int cin = cout;
    cout = ch[i];
    const std::string p = "down_blocks." + std::to_string(i);
    for (int j = 0; j < L; ++j) {
      down_res_[i].push_back(resnetw(p + ".resnets." + std::to_string(j), j == 0 ? cin : cout, cout));
      if (i < 3) down_xf_[i].push_back(xfw(p + ".attentions." + std::to_string(j), cout, cfg_.num_heads[i], cfg_.has_attn2[i] != 0));
    }
    if (i < 3) down_ds_[i] = convw(p + ".downsamplers.0.conv", cout, cout);
  }
  mid_res_[0] = resnetw("mid_block.resnets.0", ch[3], ch[3]);
  mid_xf_ = xfw("mid_block.attentions.0", ch[3], cfg_.num_heads[3], cfg_.has_attn2[3] != 0);
  mid_res_[1] = resnetw("mid_block.resnets.1", ch[3], ch[3]);
  cout = ch[3];
  for (int i = 0; i < 4; ++i) {
    const int cprev = cout;
    cout = ch[3 - i];
    const int cin = ch[3 - std::min(i + 1, 3)];
    const std::string p = "up_blocks." + std::to_string(i);
    for (int j = 0; j <= L; ++j) {
      const int skip = j == L ? cin : cout;
      const int rin = j == 0 ? cprev : cout;
      up_res_[i].push_back(resnetw(p + ".resnets." + std::to_string(j), rin + skip, cout));
      if (i > 0) up_xf_[i].push_back(xfw(p + ".attentions." + std::to_string(j), cout, cfg_.num_heads[3 - i], cfg_.has_attn2[3 - i] != 0));
    }
    if (i < 3) {
      // Upsample2D = nearest x2 followed by a 3x3 conv: every output pixel (2y + a, 2x + b) only ever sees a 2x2 patch of
      // the LOW-resolution input, so the layer is computed as four sub-pixel phases with pre-summed weights
      // (rows {-1, 0} weigh {w0, w1 + w2} for a = 0 and rows {0, +1} weigh {w0 + w1, w2} for a = 1; same for columns):
      // 4/9 of the multiply-adds and no materialised upsampled tensor.  Layout per phase: [Cout][ty*2 + tx][Cin].
      const auto& w = T(p + ".upsamplers.0.conv.weight");
      std::vector<float> o(static_cast<size_t>(4) * cout * 4 * cout, 0.f);  // [phase = a*2+b][Cout][ty*2+tx][Cin]
      for (int a = 0; a < 2; ++a)
        for (int b = 0; b < 2; ++b)
          for (int co = 0; co < cout; ++co)
            for (int ci = 0; ci < cout; ++ci)
              for (int ky = 0; ky < 3; ++ky)
                for (int kx = 0; kx < 3; ++kx) {
                  const int ty = a == 0 ? (ky == 0 ? 0 : 1) : (ky == 2 ? 1 : 0);
                  const int tx = b == 0 ? (kx == 0 ? 0 : 1) : (kx == 2 ? 1 : 0);
                  o[((static_cast<size_t>(a * 2 + b) * cout + co) * 4 + ty * 2 + tx) * cout + ci] +=
                      w[(static_cast<size_t>(co) * cout + ci) * 9 + ky * 3 + kx];
                }
      up_us_[i].w = up_bf16(o);
      up_us_[i].b = up_f32(T(p + ".upsamplers.0.conv.bias"));
      up_us_[i].in = cout;
      up_us_[i].out = cout;
    }
  }
  norm_out_ = normw("conv_norm_out", C0);
  {
    conv_out_.w = up_bf16(conv_gemm_layout(T("conv_out.weight"), cfg_.out_channels, C0, 3, 16));
    std::vector<float> b(16, 0.f);
    const auto& bo = T("conv_out.bias");
    for (int i = 0; i < cfg_.out_channels; ++i) b[i] = bo[i];
    conv_out_.b = up_f32(b);
    conv_out_.in = C0;
    conv_out_.out = 16;
  }
  temb_total_ = static_cast<int>(temb_b.size());
  temb_all_.w = up_bf16(temb_w);
  temb_all_.b = up_f32(temb_b);
  temb_all_.in = TE;
  temb_all_.out = temb_total_;
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
  static long long* dry_stats_marker() {  // dry run: "has statistics" marker, never dereferenced
    static long long marker;
    return &marker;
  }
 public:
  PlanBuilder(Model& m, Plan& p, bool dry, char* base) : m_(m), p_(p), dry_(dry), base_(base) {}

  struct Act { bf16* p; int C, H, W; long long* stats = nullptr; };  // stats: [B][C][2] {sum, sumsq} filled by the producer's epilogue

  size_t peak() const { return peak_; }
  size_t stats_words() const { return stats_used_; }
  // per-(image, channel) statistics of a GEMM / conv output that a GroupNorm will read: a slice of one pool that a single
  // memset at the head of the plan zeroes
  // (only when every 32-row warp of the producer's tiles stays inside one image: true for every level of a >= 32x32
  //  latent; smaller test shapes fall back to the stand-alone statistics kernel)
  long long* stats_alloc(int n_img, int C, int H, int W) {
    int bw = 16;
    while (bw > W) bw >>= 1;
    int bh = 128 / bw;
    while (bh > H && bh > 1) bh >>= 1;
    if ((bw * bh) % 32 != 0 || (H * W) % 32 != 0) return nullptr;
    const size_t n = static_cast<size_t>(n_img) * C * 2;
    long long* p = stats_pool_ ? stats_pool_ + stats_used_ : dry_stats_marker();
    stats_used_ += n;
    return p;
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

  void op(std::function<int(cudaStream_t)> f, int launches = 1, int kind = 5, double flops = 0.0) {
    p_.launches += launches;
    if (!dry_) {
      p_.ops.push_back(std::move(f));
      p_.op_kind.push_back(kind);
      p_.op_flops.push_back(flops);
    }
  }
  void tap(const std::string& name, const Act& a) {
    if (!dry_) p_.taps.push_back({name, a.p, a.C, a.H, a.W, p_.ops.size()});
  }
  void gemm(const GemmDesc& d) {
    if (dry_) { p_.launches += 1; return; }
    GemmLaunch L;
    if (int rc = gemm_prepare(d, &L)) { if (!rc_) rc_ = rc; return; }
    op([L](cudaStream_t s) { return gemm_run(L, s); }, 1, d.conv ? 1 : 0, gemm_flops(L));
  }
  void attention(const AttnDesc& d) {
    if (dry_) { p_.launches += 1; return; }
    AttnLaunch L;
    if (int rc = attn_prepare(d, &L)) { if (!rc_) rc_ = rc; return; }
    op([L](cudaStream_t s) { return attn_run(L, s); }, 1, 2, attn_flops(d));
  }
  // GroupNorm(+SiLU) of (a | b): statistics come from the producers' epilogues (Act::stats), one apply launch
  void groupnorm(const Act& xa, const Act* xb, int n_img, float eps, const NormW& n, int silu, bf16* out) {
    const int groups = m_.cfg_.norm_num_groups, hw = xa.H * xa.W;
    const bf16 *x1 = xa.p, *x2 = xb ? xb->p : nullptr;
    const int C1 = xa.C, C2 = xb ? xb->C : 0;
    const long long *s1 = xa.stats, *s2 = xb ? xb->stats : nullptr;
    if (s1 == nullptr || (xb && s2 == nullptr)) {  // small shapes: stand-alone statistics pass
      float* part = gn_partials_;
      op([=](cudaStream_t s) { return groupnorm_run(x1, C1, x2, C2, n_img, hw, groups, eps, n.g, n.b, silu, out, part, s); }, 2, 3);
      return;
    }
    op([=](cudaStream_t s) { return groupnorm_apply_run(x1, C1, s1, x2, C2, s2, n_img, hw, groups, eps, n.g, n.b, silu, out, s); }, 1, 3);
  }
  void layernorm(const bf16* x, int rows, int C, const NormW& n, bf16* out) {
    op([=](cudaStream_t s) { return layernorm_run(x, rows, C, 1e-5f, n.g, n.b, out, s); }, 1, 4);
  }

  // ResnetBlock2D on (xa | xb) -> new buffer   (reference semantics: SURVEY R-1)
  Act resnet(const ResnetW& r, Act xa, const Act* xb, const bf16* temb_all, int ld_temb) {
    const int B = p_.B, hw = xa.H * xa.W, M = B * hw;
    const int Cb = xb ? xb->C : 0;
    const int Cin = xa.C + Cb;
    bf16* h0 = alloc(static_cast<size_t>(M) * Cin);
    groupnorm(xa, xb, B, m_.cfg_.norm_eps, r.n1, 1, h0);
    Act h1{alloc(static_cast<size_t>(M) * r.cout), r.cout, xa.H, xa.W, stats_alloc(B, r.cout, xa.H, xa.W)};
    {
      GemmDesc d;
      d.conv = 1; d.A = h0; d.n_img = B; d.H = xa.H; d.W = xa.W; d.Cin = Cin;
      d.Wt = r.c1.w; d.N = r.cout; d.bias = r.c1.b;
      d.rowvec = temb_all + r.temb_off; d.ld_rowvec = ld_temb;
      d.out = h1.p; d.ldo = r.cout;
      d.stats = h1.stats;
      gemm(d);
    }
    release(h0);
    bf16* h2 = alloc(static_cast<size_t>(M) * r.cout);
    groupnorm(h1, nullptr, B, m_.cfg_.norm_eps, r.n2, 1, h2);
    release(h1.p);
    const bf16* res = xa.p;
    bf16* sc = nullptr;
    if (r.sc.w) {
      sc = alloc(static_cast<size_t>(M) * r.cout);
      GemmDesc d;
      d.A = xa.p; d.lda = xa.C; d.K1 = xa.C;
      if (xb) { d.A2 = xb->p; d.lda2 = Cb; d.K2 = Cb; }
      d.Wt = r.sc.w; d.M = M; d.N = r.cout; d.bias = r.sc.b; d.out = sc; d.ldo = r.cout;
      gemm(d);
      res = sc;
    }
    Act out{alloc(static_cast<size_t>(M) * r.cout), r.cout, xa.H, xa.W, stats_alloc(B, r.cout, xa.H, xa.W)};
    {
      GemmDesc d;
      d.conv = 1; d.A = h2; d.n_img = B; d.H = xa.H; d.W = xa.W; d.Cin = r.cout;
      d.Wt = r.c2.w; d.N = r.cout; d.bias = r.c2.b;
      d.residual = res; d.ld_res = r.cout;
      d.out = out.p; d.ldo = r.cout;
      d.stats = out.stats;
      gemm(d);
    }
    release(h2);
    if (sc) release(sc);
    return out;
  }

  // Frame-sharded 3-D attention: the QKV GEMM epilogue stores its K|V columns straight into every rank's gathered
  // K/V buffer (peer memory), a flag round makes them visible, attention reads all F_total frames locally.
  void sharded_qkv_attention(const AttnW& a, const XfW& x, const bf16* normed, bf16* qkv, bf16* o, int M, int batch, int seq) {
    const int Cp = x.heads * x.dpad;
    const Exchange& X = m_.xch_;
    const int idx = p_.n3d++;
    p_.launches += 4;
    const long long rows_local = seq;                                   // F_loc * hw tokens per CFG half
    const long long rows_global = static_cast<long long>(seq) / p_.F * p_.F_total;
    if (static_cast<size_t>(batch) * rows_global * 2 * Cp * sizeof(bf16) > X.kv_bytes) {
      set_error("K/V exchange buffer too small for this window (d4d_exchange_alloc)");
      if (!rc_) rc_ = 1;
      return;
    }
    if (dry_) return;
    GemmLaunch G[2];
    AttnLaunch A[2];
    for (int par = 0; par < 2; ++par) {
      GemmDesc d;
      d.A = normed; d.lda = x.C; d.K1 = x.C; d.Wt = a.qkv.w; d.M = M; d.N = 3 * Cp; d.out = qkv; d.ldo = 3 * Cp;
      d.kv_world = X.world; d.kv_col0 = Cp; d.kv_ld = 2 * Cp;
      d.kv_rows_local = rows_local; d.kv_rows_global = rows_global; d.kv_row_offset = static_cast<long long>(X.rank) * rows_local;
      for (int r = 0; r < X.world; ++r) d.kv_dst[r] = static_cast<bf16*>(X.peer_kv[par][r]);
      if (int rc = gemm_prepare(d, &G[par])) { if (!rc_) rc_ = rc; return; }
      AttnDesc t;
      t.q = qkv; t.ld_qkv = 3 * Cp;
      t.k = static_cast<const bf16*>(X.kv[par]); t.v = t.k + Cp; t.ld_kv = 2 * Cp;
      t.out = o; t.ld_out = Cp; t.batch = batch; t.seq = seq; t.seq_kv = static_cast<int>(rows_global);
      t.heads = x.heads; t.head_dim = x.dpad; t.scale = 1.0f / sqrtf(static_cast<float>(x.d));
      if (int rc = attn_prepare(t, &A[par])) { if (!rc_) rc_ = rc; return; }
    }
    KvFlagArgs fa;
    for (int r = 0; r < 8; ++r) fa.flags[r] = r < X.world ? X.peer_flags[r] : nullptr;
    fa.rank = X.rank; fa.world = X.world; fa.epoch = 0; fa.slot = 0;
    Plan* pl = &p_;
    const GemmLaunch G0 = G[0], G1 = G[1];
    const AttnLaunch A0 = A[0], A1 = A[1];
    const double fl_g = gemm_flops(G0), fl_a = attn_flops(A0.d);
    p_.ops.push_back([=](cudaStream_t s) {
      const unsigned int counter = pl->epoch0 + idx;
      const int par = counter & 1;
      if (int rc = gemm_run(par ? G1 : G0, s)) return rc;
      KvFlagArgs f = fa;
      f.epoch = counter + 1;
      f.slot = par;
      if (int rc = kv_signal_run(f, s)) return rc;
      return kv_wait_run(f, s);
    });
    p_.op_kind.push_back(0);
    p_.op_flops.push_back(fl_g);
    p_.ops.push_back([=](cudaStream_t s) {
      const unsigned int counter = pl->epoch0 + idx;
      return attn_run((counter & 1) ? A1 : A0, s);
    });
    p_.op_kind.push_back(2);
    p_.op_flops.push_back(fl_a);
  }

  void self_attention(const AttnW& a, const XfW& x, const bf16* normed, const bf16* resid, bf16* out, int M, int batch, int seq,
                      bool is3d = false) {
    const int Cp = x.heads * x.dpad;
    bf16* qkv = alloc(static_cast<size_t>(M) * 3 * Cp);
    bf16* o = nullptr;
    if (is3d && p_.world > 1) {
      o = alloc(static_cast<size_t>(M) * Cp);
      sharded_qkv_attention(a, x, normed, qkv, o, M, batch, seq);
    } else {
      {
        GemmDesc d;
        d.A = normed; d.lda = x.C; d.K1 = x.C; d.Wt = a.qkv.w; d.M = M; d.N = 3 * Cp; d.out = qkv; d.ldo = 3 * Cp;
        gemm(d);
      }
      o = alloc(static_cast<size_t>(M) * Cp);
      AttnDesc d;
      d.q = qkv; d.k = qkv + Cp; d.v = qkv + 2 * Cp; d.ld_qkv = 3 * Cp;
      d.out = o; d.ld_out = Cp; d.batch = batch; d.seq = seq; d.heads = x.heads; d.head_dim = x.dpad;
      d.scale = 1.0f / sqrtf(static_cast<float>(x.d));
      attention(d);
    }
    release(qkv);
    {
      GemmDesc d;
      d.A = o; d.lda = Cp; d.K1 = Cp; d.Wt = a.out.w; d.M = M; d.N = x.C; d.bias = a.out.b;
      d.residual = resid; d.ld_res = x.C; d.out = out; d.ldo = x.C;
      gemm(d);
    }
    release(o);
  }

  // TransformerMultiviewModel (+ its single MultiviewTransformerBlock): x -> new buffer
  Act transformer(const XfW& x, Act in, int num_frames) {
    const int B = p_.B, hw = in.H * in.W, M = B * hw, C = x.C;
    bf16* n = alloc(static_cast<size_t>(M) * C);
    groupnorm(in, nullptr, B, 1e-6f, x.gn, 0, n);
    bf16* t = alloc(static_cast<size_t>(M) * C);
    {
      GemmDesc d;
      d.A = n; d.lda = C; d.K1 = C; d.Wt = x.pin.w; d.M = M; d.N = C; d.bias = x.pin.b; d.out = t; d.ldo = C;
      gemm(d);
    }
    // attn1 (3-D when num_frames > 1: batch = B / num_frames sequences of num_frames*hw tokens)
    layernorm(t, M, C, x.ln1, n);
    bf16* t1 = alloc(static_cast<size_t>(M) * C);
    self_attention(x.a1, x, n, t, t1, M, B / num_frames, num_frames * hw, num_frames > 1);
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
      GemmDesc d;
      d.A = n; d.lda = C; d.K1 = C; d.Wt = x.ff1.w; d.M = M; d.N = 8 * C; d.bias = x.ff1.b; d.out = g; d.ldo = 4 * C;
      d.geglu = 1;
      gemm(d);
    }
    release(n);
    bf16* t3 = alloc(static_cast<size_t>(M) * C);
    {
      GemmDesc d;
      d.A = g; d.lda = 4 * C; d.K1 = 4 * C; d.Wt = x.ff2.w; d.M = M; d.N = C; d.bias = x.ff2.b;
      d.residual = t1; d.ld_res = C; d.out = t3; d.ldo = C;
      gemm(d);
    }
    release(g);
    release(t1);
    Act out{alloc(static_cast<size_t>(M) * C), C, in.H, in.W, stats_alloc(B, C, in.H, in.W)};
    {
      GemmDesc d;
      d.A = t3; d.lda = C; d.K1 = C; d.Wt = x.pout.w; d.M = M; d.N = C; d.bias = x.pout.b;
      d.residual = in.p; d.ld_res = C; d.out = out.p; d.ldo = C;
      d.stats = out.stats; d.stats_rows = hw;
      gemm(d);
    }
    release(t3);
    return out;
  }

  Act conv3x3(const LinW& w, Act in, int act = 0, int n_img = 0, bool want_stats = false) {
    if (n_img <= 0) n_img = p_.B;
    const int M = n_img * in.H * in.W;
    Act out{alloc(static_cast<size_t>(M) * w.out), w.out, in.H, in.W, want_stats ? stats_alloc(n_img, w.out, in.H, in.W) : nullptr};
    GemmDesc d;
    d.conv = 1; d.A = in.p; d.n_img = n_img; d.H = in.H; d.W = in.W; d.Cin = in.C;
    d.Wt = w.w; d.N = w.out; d.bias = w.b; d.out = out.p; d.ldo = w.out; d.act = act;
    d.stats = out.stats;
    gemm(d);
    return out;
  }

  int build() {
    Model& m = m_;
    const d4d_config& cfg = m.cfg_;
    Plan* pl = &p_;
    const int B = p_.B, F = p_.F, h = p_.h, w = p_.w;
    const int* ch = cfg.block_out_channels;
    const int C0 = ch[0], TE = 4 * C0, L = cfg.layers_per_block;
    const int M0 = B * h * w;

    {  // scratch of the stand-alone GroupNorm statistics kernel (small shapes only)
      const size_t fl = groupnorm_scratch_floats(B, cfg.norm_num_groups);
      gn_partials_ = reinterpret_cast<float*>(alloc(fl * 2));
      if (!dry_ && cudaMemset(gn_partials_, 0, fl * sizeof(float)) != cudaSuccess) rc_ = 2;
    }
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
      GemmDesc d;
      d.A = tsin; d.lda = C0; d.K1 = C0; d.Wt = m.time1_.w; d.M = B; d.N = TE; d.bias = m.time1_.b; d.act = 1; d.out = e1; d.ldo = TE;
      gemm(d);
    }
    bf16* emb = alloc(static_cast<size_t>(B) * TE);
    {
      GemmDesc d;
      d.A = e1; d.lda = TE; d.K1 = TE; d.Wt = m.time2_.w; d.M = B; d.N = TE; d.bias = m.time2_.b; d.out = emb; d.ldo = TE;
      gemm(d);
    }
    if (cfg.enable_tem_embeds) {
      float* pos = reinterpret_cast<float*>(alloc(static_cast<size_t>(B) * 2));
      if (!dry_) {
        std::vector<float> hp(B);
        for (int dmn = 0; dmn < p_.n_domains; ++dmn)
          for (int f = 0; f < F; ++f) hp[dmn * F + f] = p_.domains[dmn] == 0 ? 0.f : static_cast<float>((p_.rank * F + f) % std::max(1, (p_.world > 1 ? p_.F_total : F) / 2));
        if (cudaMemcpy(pos, hp.data(), sizeof(float) * B, cudaMemcpyHostToDevice) != cudaSuccess) rc_ = 2;
      }
      op([=](cudaStream_t s) { return sinusoid_run(pos, B, C0, 1, 0.f, tsin, s); });
      {
        GemmDesc d;
        d.A = tsin; d.lda = C0; d.K1 = C0; d.Wt = m.tem1_.w; d.M = B; d.N = TE; d.bias = m.tem1_.b; d.act = 1; d.out = e1; d.ldo = TE;
        gemm(d);
      }
      bf16* emb2 = alloc(static_cast<size_t>(B) * TE);
      {
        GemmDesc d;
        d.A = e1; d.lda = TE; d.K1 = TE; d.Wt = m.tem2_.w; d.M = B; d.N = TE; d.bias = m.tem2_.b;
        d.residual = emb; d.ld_res = TE; d.out = emb2; d.ldo = TE;
        gemm(d);
      }
      // pos stays allocated for the lifetime of the plan (it is read on every forward)
      release(emb);
      emb = emb2;
    }
    op([=](cudaStream_t s) { return silu_run(emb, static_cast<long long>(B) * TE, e1, s); });
    const int ldt = m.temb_total_;
    bf16* temb_all = alloc(static_cast<size_t>(B) * ldt);
    {
      GemmDesc d;
      d.A = e1; d.lda = TE; d.K1 = TE; d.Wt = m.temb_all_.w; d.M = B; d.N = ldt; d.bias = m.temb_all_.b; d.out = temb_all; d.ldo = ldt;
      gemm(d);
    }
    release(tsin);
    release(e1);
    release(emb);

    // ---- 2. conv_in (+ pose encoder): UNET:549-554 ----
    bf16* pose_emb = nullptr;
    if (cfg.enable_pose_encoder) {
      const int Hs = 8 * h, Ws = 8 * w;
      // pose_shared_neg: the skeleton batch is [1 constant CFG-negative image | F positive images] instead of 2F images
      // (pipeline_diffuman4d.py:349-356 makes every negative skeleton the same all(-1) image); its embedding is computed
      // once per forward and broadcast to the F negative images below
      const int PB = p_.pose_shared_neg ? F + 1 : B;
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
        GemmDesc d;
        d.A = col; d.lda = 512; d.K1 = 512; d.Wt = pw.conv[5].w; d.M = PM0; d.N = 64; d.bias = pw.conv[5].b; d.act = 1; d.out = a5; d.ldo = 64;
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
        GemmDesc d;
        d.A = x7.p; d.lda = 128; d.K1 = 128; d.Wt = pw.proj.w; d.M = PM0; d.N = C0; d.bias = pw.proj.b; d.out_scale = pw.scale;
        d.out = pose_emb; d.ldo = C0;
        gemm(d);
      }
      release(x7.p);
      if (p_.pose_shared_neg) {  // broadcast: images 0..F-1 <- embedding 0, images F..2F-1 <- embeddings 1..F
        bf16* full = alloc(static_cast<size_t>(M0) * C0);
        bf16* small = pose_emb;
        const long long per_img = static_cast<long long>(h) * w * C0;
        op([=](cudaStream_t s) { return broadcast_neg_images_run(small, per_img, F, full, s); });
        release(small);
        pose_emb = full;
      }
    }
    Act x;
    {
      const int KP = m.kp_in(), cp = m.cin_pad(), Cin = cfg.in_channels;
      bf16* col = alloc(static_cast<size_t>(M0) * KP);
      op([=](cudaStream_t s) { return im2col_nchw_run(pl->sample, B, Cin, h, w, cp, KP, col, s); });
      bf16* x0 = alloc(static_cast<size_t>(M0) * C0);
      long long* st0 = stats_alloc(B, C0, h, w);
      GemmDesc d;
      d.A = col; d.lda = KP; d.K1 = KP; d.Wt = m.conv_in_.w; d.M = M0; d.N = C0; d.bias = m.conv_in_.b;
      if (pose_emb) { d.residual = pose_emb; d.ld_res = C0; }
      d.out = x0; d.ldo = C0;
      d.stats = st0; d.stats_rows = h * w;
      gemm(d);
      release(col);
      if (pose_emb) release(pose_emb);
      x = {x0, C0, h, w, st0};
    }
    tap("conv_in", x);

    // ---- 3. down: UNET:557-565 ----
    std::vector<Act> skips;
    skips.push_back(x);
    for (int i = 0; i < 4; ++i) {
      const int nf = (4 - i - 1) < cfg.num_3d_attn_blocks ? F : 1;
      for (int j = 0; j < L; ++j) {
        Act y = resnet(m.down_res_[i][j], x, nullptr, temb_all, ldt);
        if (i < 3) {
          Act z = transformer(m.down_xf_[i][j], y, nf);
          release(y.p);
          y = z;
        }
        x = y;
        skips.push_back(x);
      }
      if (i < 3) {  // Downsample2D: 3x3 stride-2 pad-1 conv, read in place through a strided tensor map
        const int Ho = x.H / 2, Wo = x.W / 2, Mo = B * Ho * Wo;
        bf16* y = alloc(static_cast<size_t>(Mo) * x.C);
        long long* sty = stats_alloc(B, x.C, Ho, Wo);
        GemmDesc d;
        d.conv = 1; d.conv_kind = 1; d.A = x.p; d.n_img = B; d.H = x.H; d.W = x.W; d.Cin = x.C;
        d.Wt = m.down_ds_[i].w; d.N = x.C; d.bias = m.down_ds_[i].b; d.out = y; d.ldo = x.C;
        d.stats = sty;
        gemm(d);
        x = {y, x.C, Ho, Wo, sty};
        skips.push_back(x);
      }
      tap("down_blocks." + std::to_string(i), x);
    }
    // ---- 4. mid: UNET:568-572 ----
    {
      Act y = resnet(m.mid_res_[0], x, nullptr, temb_all, ldt);  // x is a skip: keep it
      Act z = transformer(m.mid_xf_, y, F);
      release(y.p);
      Act u = resnet(m.mid_res_[1], z, nullptr, temb_all, ldt);
      release(z.p);
      x = u;
    }
    tap("mid_block", x);
    // ---- 5. up: UNET:575-587 ----
    for (int i = 0; i < 4; ++i) {
      const int nf = i < cfg.num_3d_attn_blocks ? F : 1;
      for (int j = 0; j <= L; ++j) {
        const Act sk = skips.back();
        skips.pop_back();
        Act y = resnet(m.up_res_[i][j], x, &sk, temb_all, ldt);
        release(x.p);
        release(sk.p);
        if (i > 0) {
          Act z = transformer(m.up_xf_[i][j], y, nf);
          release(y.p);
          y = z;
        }
        x = y;
      }
      if (i < 3) {  // Upsample2D (nearest x2, then 3x3 conv) as four sub-pixel phases on the low-resolution tensor
        const int H2 = 2 * x.H, W2 = 2 * x.W;
        Act y{alloc(static_cast<size_t>(B) * H2 * W2 * x.C), x.C, H2, W2, stats_alloc(B, x.C, x.H, x.W)};
        {
          GemmDesc d;
          d.conv = 1; d.conv_kind = 3;
          d.A = x.p; d.n_img = B; d.H = x.H; d.W = x.W; d.Cin = x.C;
          d.Wt = m.up_us_[i].w; d.N = x.C; d.bias = m.up_us_[i].b; d.out = y.p; d.ldo = x.C;
          d.stats = y.stats;
          gemm(d);
        }
        release(x.p);
        x = y;
      }
      tap("up_blocks." + std::to_string(i), x);
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
  float* gn_partials_ = nullptr;
  long long* stats_pool_ = nullptr;
  size_t stats_used_ = 0;
  int rc_ = 0;
};

Plan* Model::find_plan(int n_domains, int B, int F, int h, int w) {
  for (auto& kv : plans_) {
    Plan* p = kv.second.get();
    if (p->n_domains == n_domains && p->B == B && p->F == F && p->h == h && p->w == w) return p;
  }
  return nullptr;
}

int Model::get_plan(const int* domain_ids, int n_domains, int B, int F, int h, int w, Plan** out, int F_total, bool pose_shared_neg) {
  if (!finalized_) {
    set_error("weights not finalized (call d4d_finalize_weights)");
    return 3;
  }
  D4D_REQUIRE(B > 0 && F > 0 && n_domains > 0, "empty batch");
  if (n_domains * F != B) {
    // same message as the reference's ValueError (unet_multiview_condition.py:524-525)
    set_error("num_frames: " + std::to_string(F) + " * len(domains): " + std::to_string(n_domains) + " != len(emb): " + std::to_string(B));
    return 1;
  }
  D4D_REQUIRE(h % 8 == 0 && w % 8 == 0 && h > 0 && w > 0, "latent height/width must be divisible by 8");
  for (int i = 0; i < n_domains; ++i) D4D_REQUIRE(domain_ids[i] == 0 || domain_ids[i] == 1, "Invalid domain for temporal embedding");
  const bool sharded = F_total > F;
  if (sharded) {
    D4D_REQUIRE(xch_.ready && xch_.world > 1, "frame-sharded forward needs d4d_exchange_open first");
    D4D_REQUIRE(F * xch_.world == F_total, "F_total must equal world * local frames");
  }
  const std::string key = plan_key(domain_ids, n_domains, B, F, h, w) + (sharded ? "_sh" + std::to_string(F_total) : std::string()) + (pose_shared_neg ? "_pn" : "");
  auto it = plans_.find(key);
  if (it != plans_.end()) {
    *out = it->second.get();
    return 0;
  }
  D4D_CUDA_OK(cudaSetDevice(device_));
  std::unique_ptr<Plan> p(new Plan());
  p->n_domains = n_domains; p->B = B; p->F = F; p->h = h; p->w = w;
  p->domains.assign(domain_ids, domain_ids + n_domains);
  if (sharded) { p->F_total = F_total; p->rank = xch_.rank; p->world = xch_.world; }
  p->pose_shared_neg = pose_shared_neg && cfg_.enable_pose_encoder && n_domains == 2;
  size_t peak = 0;
  {
    Plan scratch;
    scratch.n_domains = n_domains; scratch.B = B; scratch.F = F; scratch.h = h; scratch.w = w;
    scratch.domains = p->domains;
    scratch.F_total = p->F_total; scratch.rank = p->rank; scratch.world = p->world;
    scratch.pose_shared_neg = p->pose_shared_neg;
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

int Model::forward(const bf16* sample, const long long* timestep, const bf16* skeletons, const int* domain_ids,
                   int n_domains, int B, int F, int h, int w, bf16* out, cudaStream_t stream, int F_total, bool pose_shared_neg) {
  D4D_REQUIRE(sample && timestep && out && domain_ids, "null argument");
  D4D_REQUIRE(!cfg_.enable_pose_encoder || skeletons != nullptr, "skeletons are required when enable_pose_encoder");
  D4D_REQUIRE(!cfg_.center_input_sample, "center_input_sample is not supported");
  Plan* p = nullptr;
  if (int rc = get_plan(domain_ids, n_domains, B, F, h, w, &p, F_total, pose_shared_neg)) return rc;
  D4D_CUDA_OK(cudaSetDevice(device_));
  p->sample = sample;
  p->timestep = timestep;
  p->skeletons = skeletons;
  p->out = out;
  p->epoch0 = xch_.epoch_base;  // global, monotonic exchange counter: every rank runs the same forwards in the same order
  for (auto& f : p->ops)
    if (int rc = f(stream)) return rc;
  p->run_index++;
  xch_.epoch_base += static_cast<unsigned int>(p->n3d);
  return 0;
}

int Model::debug_tap(const bf16* sample, const long long* timestep, const bf16* skeletons, const int* domain_ids, int n_domains,
                     int B, int F, int h, int w, int tap, bf16* out, char* name64, int* dims3, cudaStream_t stream) {
  D4D_REQUIRE(domain_ids != nullptr, "null argument");
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
  D4D_REQUIRE(sample && timestep, "null argument");
  D4D_REQUIRE(!cfg_.enable_pose_encoder || skeletons != nullptr, "skeletons are required when enable_pose_encoder");
  D4D_CUDA_OK(cudaSetDevice(device_));
  p->sample = sample; p->timestep = timestep; p->skeletons = skeletons; p->out = nullptr;
  for (size_t i = 0; i < t.n_ops; ++i)
    if (int rc = p->ops[i](stream)) return rc;
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
  D4D_REQUIRE(sample && timestep && out && domain_ids && ms_by_kind && launches_by_kind && flops_by_kind, "null argument");
  Plan* p = nullptr;
  if (int rc = get_plan(domain_ids, n_domains, B, F, h, w, &p)) return rc;
  D4D_CUDA_OK(cudaSetDevice(device_));
  p->sample = sample; p->timestep = timestep; p->skeletons = skeletons; p->out = out;
  const size_t n = p->ops.size();
  while (p->events.size() < n + 1) {
    cudaEvent_t e;
    D4D_CUDA_OK(cudaEventCreate(&e));
    p->events.push_back(e);
  }
  for (size_t i = 0; i < n; ++i) {
    D4D_CUDA_OK(cudaEventRecord(p->events[i], stream));
    if (int rc = p->ops[i](stream)) return rc;
  }
  D4D_CUDA_OK(cudaEventRecord(p->events[n], stream));
  D4D_CUDA_OK(cudaEventSynchronize(p->events[n]));
  for (int k = 0; k < 6; ++k) { ms_by_kind[k] = 0.f; launches_by_kind[k] = 0; flops_by_kind[k] = 0.0; }
  for (size_t i = 0; i < n; ++i) {
    float ms = 0.f;
    D4D_CUDA_OK(cudaEventElapsedTime(&ms, p->events[i], p->events[i + 1]));
    const int k = p->op_kind[i];
    ms_by_kind[k] += ms;
    launches_by_kind[k] += 1;
    flops_by_kind[k] += p->op_flops[i];
  }
  return 0;
}

int Model::denoise_window(bf16* latents, const bf16* pixel, const bf16* plucker, const bf16* skeletons, const bf16* mask,
                          long long* ts_idx, const d4d_sched& sched, float guidance, int domain, int F, int h, int w,
                          int num_steps, cudaStream_t stream, int F_total) {
  D4D_REQUIRE(latents && pixel && plucker && mask && ts_idx, "null argument");
  D4D_REQUIRE(sched.timesteps_table && sched.alphas_cumprod && sched.n_steps > 0, "scheduler tables");
  D4D_REQUIRE(domain == 0 || domain == 1, "Invalid domain");
  const bool cfg_on = guidance > 1.0f;
  const int B = cfg_on ? 2 * F : F;
  const bool pose = cfg_.enable_pose_encoder != 0;
  const int Cin = 4 + 6 + (pose ? 0 : 4) + 1;
  D4D_REQUIRE(Cin == cfg_.in_channels, "in_channels does not match the latent/plucker/skeleton/mask channel layout");
  D4D_REQUIRE(skeletons != nullptr, "skeletons required");
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
    D4D_CUDA_OK(cudaMalloc(&wb->noise, sizeof(bf16) * B * cfg_.out_channels * hw));
    D4D_CUDA_OK(cudaMalloc(&wb->latents_tmp, sizeof(bf16) * F * 4 * hw));
    D4D_CUDA_OK(cudaMalloc(&wb->ts_tmp, sizeof(long long) * F));
    it = wbufs_.emplace(key, std::move(wb)).first;
  }
  WindowBufs& wb = *it->second;
  const int doms[2] = {domain, domain};
  const int hw = h * w;
  for (int step = 0; step < num_steps; ++step) {
    AssembleArgs a;
    a.latents = latents; a.pixel = pixel; a.plucker = plucker; a.skel_latents = pose ? nullptr : skeletons; a.mask = mask;
    a.timestep_indices = ts_idx; a.timesteps_table = reinterpret_cast<const long long*>(sched.timesteps_table);
    a.n_steps = sched.n_steps; a.F = F; a.h = h; a.w = w; a.cfg = cfg_on ? 1 : 0;
    a.sample = wb.sample; a.timestep_out = wb.timestep;
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
    if (int rc = forward(wb.sample, wb.timestep, skel_in, doms, cfg_on ? 2 : 1, B, F, h, w, wb.noise, stream, F_total, pose && cfg_on)) return rc;
    DdimArgs d;
    d.noise = wb.noise; d.latents = latents; d.mask = mask; d.timestep_indices = ts_idx;
    d.timesteps_table = reinterpret_cast<const long long*>(sched.timesteps_table); d.alphas_cumprod = sched.alphas_cumprod;
    d.n_steps = sched.n_steps; d.T = sched.num_train_timesteps; d.final_alpha_cumprod = sched.final_alpha_cumprod;
    d.F = F; d.chw = 4 * hw; d.hw = hw; d.cfg = cfg_on ? 1 : 0; d.guidance = guidance;
    d.prediction_type = sched.prediction_type; d.clip_sample = sched.clip_sample; d.clip_range = sched.clip_sample_range;
    d.emulate_bf16 = sched.emulate_bf16; d.out = wb.latents_tmp;
    if (int rc = cfg_ddim_step_run(d, wb.ts_tmp, stream)) return rc;
    D4D_CUDA_OK(cudaMemcpyAsync(latents, wb.latents_tmp, sizeof(bf16) * F * 4 * hw, cudaMemcpyDeviceToDevice, stream));
    D4D_CUDA_OK(cudaMemcpyAsync(ts_idx, wb.ts_tmp, sizeof(long long) * F, cudaMemcpyDeviceToDevice, stream));
  }
  return 0;
}

}  // namespace d4d
