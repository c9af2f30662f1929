"""CPU ORACLE (test infrastructure, NOT the product) for the Diffuman4D UNet forward.

A pure-torch restatement of ``UNetMultiviewConditionModel.forward`` and everything it
delegates to.  Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
cpu_baseline / ``--impl reference`` legs may import this module.

PARITY STATUS: the reference has no tests, golden vectors or fixtures for this path, and
its leaf arithmetic lives in the un-vendored dependency ``diffusers==0.33.1`` (pinned in
requirements.txt:5 of the reference) which is not installed here (no network).  Pinned against
code RUN from the reference checkout (tests/golden/gen_golden.py, fixtures committed, tests in
tests/test_oracle.py):
  * the whole UNet wiring -- the reference's own ``UNetMultiviewConditionModel`` constructor and
    forward, its block classes, ``TransformerMultiviewModel``, ``MultiviewTransformerBlock`` and
    ``PoseEncoder`` executed on stubs of the upstream LEAF classes only (three configurations,
    spatial+CFG and temporal inputs, max deviation < 2e-4), including the diffusers key layout
    (``load_state_dict(strict=True)`` of the product's key/shape spec into the reference model);
  * ``PoseEncoder`` and ``MultiviewTransformerBlock.forward`` individually.
Still **parity unpinned**: the arithmetic INSIDE the upstream leaf classes (ResnetBlock2D,
Down/Upsample2D, Transformer2DModel helpers, BasicTransformerBlock constructor, Attention +
AttnProcessor2_0, GEGLU, Timesteps, TimestepEmbedding), restated here from the published 0.33.1
sources and anchored on the reference's call sites (see DESIGN.md section 2).

Module tree and ``state_dict`` keys follow the diffusers layout so a real checkpoint
(`unet/diffusion_pytorch_model.safetensors`) loads by name (SURVEY.md section 8b).

Citations: UNET = src/diffusers/models/unets/unet_multiview_condition.py,
BLK = .../unets/unet_multiview_blocks.py, TRF = .../transformers/transformer_multiview.py,
ATT = src/diffusers/models/attention.py, POSE = .../unets/pose_encoder.py (all in the reference checkout).
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F


# --------------------------------------------------------------------------- embeddings
def timestep_embedding(timesteps: torch.Tensor, dim: int, flip_sin_to_cos: bool, freq_shift: float,
                       max_period: float = 10000.0) -> torch.Tensor:
    """upstream ``get_timestep_embedding`` (diffusers/models/embeddings.py), used at UNET:464,255."""
    half = dim // 2
    exponent = -math.log(max_period) * torch.arange(0, half, dtype=torch.float32, device=timesteps.device)
    exponent = exponent / (half - freq_shift)
    emb = torch.exp(exponent)
    emb = timesteps[:, None].float() * emb[None, :]
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
    if flip_sin_to_cos:
        emb = torch.cat([emb[:, half:], emb[:, :half]], dim=-1)
    if dim % 2 == 1:
        emb = F.pad(emb, (0, 1, 0, 0))
    return emb


class TimestepEmbedding(nn.Module):
    """upstream ``TimestepEmbedding`` (act silu, no post-act, no cond proj) -- UNET:245,257."""

    def __init__(self, in_dim: int, dim: int):
        super().__init__()
        self.linear_1 = nn.Linear(in_dim, dim)
        self.linear_2 = nn.Linear(dim, dim)

    def forward(self, x):
        return self.linear_2(F.silu(self.linear_1(x)))


# --------------------------------------------------------------------------- pose encoder
class PoseEncoder(nn.Module):
    """Restatement of POSE:11-54 (8 conv+SiLU, zero-init 1x1 projection, learnable scalar scale)."""

    SPEC = [(3, 3, 3, 1), (3, 16, 4, 2), (16, 16, 3, 1), (16, 32, 4, 2),
            (32, 32, 3, 1), (32, 64, 4, 2), (64, 64, 3, 1), (64, 128, 3, 1)]  # (cin, cout, k, stride), pad 1

    def __init__(self, out_channels: int = 320):
        super().__init__()
        layers = []
        for cin, cout, k, s in self.SPEC:
            layers += [nn.Conv2d(cin, cout, kernel_size=k, stride=s, padding=1), nn.SiLU()]
        self.conv_layers = nn.Sequential(*layers)
        self.final_proj = nn.Conv2d(128, out_channels, kernel_size=1)
        self.scale = nn.Parameter(torch.ones(1) * 2.0)

    def forward(self, x):
        return self.final_proj(self.conv_layers(x)) * self.scale


# --------------------------------------------------------------------------- resnet / sampling
class ResnetBlock2D(nn.Module):
    """upstream ``ResnetBlock2D`` (time_embedding_norm="default", output_scale_factor 1) -- BLK:274,423,585."""

    def __init__(self, cin: int, cout: int, temb_dim: int, groups: int, eps: float):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin, eps=eps)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb_dim, cout)
        self.norm2 = nn.GroupNorm(groups, cout, eps=eps)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None

    def forward(self, x, temb):
        h = self.conv1(F.silu(self.norm1(x)))
        h = h + self.time_emb_proj(F.silu(temb))[:, :, None, None]
        h = self.conv2(F.silu(self.norm2(h)))
        if self.conv_shortcut is not None:
            x = self.conv_shortcut(x)
        return x + h


class Downsample2D(nn.Module):
    """upstream ``Downsample2D(use_conv=True, padding=1, name="op")`` -- BLK:460; key ``downsamplers.0.conv``."""

    def __init__(self, c: int):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=2, padding=1)

    def forward(self, x):
        return self.conv(x)


class Upsample2D(nn.Module):
    """upstream ``Upsample2D(use_conv=True)``: nearest x2 then 3x3 conv -- BLK:620."""

    def __init__(self, c: int):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, padding=1)

    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))


# --------------------------------------------------------------------------- attention
class Attention(nn.Module):
    """upstream ``Attention`` + ``AttnProcessor2_0`` with ``encoder_hidden_states=None`` -- ATT:73,116."""

    def __init__(self, dim: int, heads: int):
        super().__init__()
        self.heads = heads
        self.to_q = nn.Linear(dim, dim, bias=False)
        self.to_k = nn.Linear(dim, dim, bias=False)
        self.to_v = nn.Linear(dim, dim, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(dim, dim), nn.Dropout(0.0)])

    def forward(self, x):
        b, s, c = x.shape
        d = c // self.heads
        q = self.to_q(x).view(b, s, self.heads, d).transpose(1, 2)
        k = self.to_k(x).view(b, s, self.heads, d).transpose(1, 2)
        v = self.to_v(x).view(b, s, self.heads, d).transpose(1, 2)
        o = sdpa(q, k, v)
        o = o.transpose(1, 2).reshape(b, s, c)
        return self.to_out[0](o)


def sdpa(q, k, v, chunk: int = 4096):
    """softmax(q k^T / sqrt(d)) v, no mask -- same maths as F.scaled_dot_product_attention, evaluated in
    query chunks so the 3-D attention (seq = F*hw) fits in host RAM."""
    if q.shape[2] * k.shape[2] <= (1 << 24):
        return F.scaled_dot_product_attention(q, k, v)
    outs = []
    for i in range(0, q.shape[2], chunk):
        outs.append(F.scaled_dot_product_attention(q[:, :, i:i + chunk], k, v))
    return torch.cat(outs, dim=2)


class GEGLU(nn.Module):
    def __init__(self, dim: int, inner: int):
        super().__init__()
        self.proj = nn.Linear(dim, inner * 2)

    def forward(self, x):
        a, g = self.proj(x).chunk(2, dim=-1)
        return a * F.gelu(g)  # exact (erf) GELU, upstream activations.GEGLU


class FeedForward(nn.Module):
    """upstream ``FeedForward(activation_fn="geglu", mult=4)``; keys ``ff.net.0.proj`` / ``ff.net.2``."""

    def __init__(self, dim: int):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, dim * 4), nn.Dropout(0.0), nn.Linear(dim * 4, dim)])

    def forward(self, x):
        for m in self.net:
            x = m(x)
        return x


class MultiviewTransformerBlock(nn.Module):
    """ATT:22-153 on top of upstream ``BasicTransformerBlock`` (norm_type layer_norm, eps 1e-5)."""

    def __init__(self, dim: int, heads: int, attn2: bool):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=1e-5)
        self.attn1 = Attention(dim, heads)
        if attn2:
            self.norm2 = nn.LayerNorm(dim, eps=1e-5)
            self.attn2 = Attention(dim, heads)
        else:
            self.norm2 = None
            self.attn2 = None
        self.norm3 = nn.LayerNorm(dim, eps=1e-5)
        self.ff = FeedForward(dim)

    def forward(self, x, num_frames: int = 1):
        bt, hw, c = x.shape
        n = self.norm1(x)
        if num_frames > 1:  # ATT:68-71  "(b t) hw c -> b (t hw) c"
            n = n.reshape(bt // num_frames, num_frames * hw, c)
        a = self.attn1(n)
        if num_frames > 1:  # ATT:82-83
            a = a.reshape(bt, hw, c)
        x = a + x
        if self.attn2 is not None:  # ATT:104-123 with encoder_hidden_states=None => per-image self-attention
            x = self.attn2(self.norm2(x)) + x
        x = self.ff(self.norm3(x)) + x  # ATT:128-151
        return x


class TransformerMultiviewModel(nn.Module):
    """TRF:42-232 + upstream continuous-input helpers (GroupNorm eps 1e-6, proj_in/out, +residual)."""

    def __init__(self, dim: int, heads: int, groups: int, linear_proj: bool, attn2: bool):
        super().__init__()
        self.linear_proj = linear_proj
        self.norm = nn.GroupNorm(groups, dim, eps=1e-6)
        if linear_proj:
            self.proj_in = nn.Linear(dim, dim)
            self.proj_out = nn.Linear(dim, dim)
        else:
            self.proj_in = nn.Conv2d(dim, dim, 1)
            self.proj_out = nn.Conv2d(dim, dim, 1)
        self.transformer_blocks = nn.ModuleList([MultiviewTransformerBlock(dim, heads, attn2)])

    def forward(self, x, num_frames: int = 1):
        b, c, h, w = x.shape
        res = x
        y = self.norm(x)
        if not self.linear_proj:
            y = self.proj_in(y)
            y = y.permute(0, 2, 3, 1).reshape(b, h * w, c)
        else:
            y = y.permute(0, 2, 3, 1).reshape(b, h * w, c)
            y = self.proj_in(y)
        for blk in self.transformer_blocks:
            y = blk(y, num_frames=num_frames)
        if not self.linear_proj:
            y = y.reshape(b, h, w, c).permute(0, 3, 1, 2).contiguous()
            y = self.proj_out(y)
        else:
            y = self.proj_out(y)
            y = y.reshape(b, h, w, c).permute(0, 3, 1, 2).contiguous()
        return y + res


# --------------------------------------------------------------------------- blocks
class DownBlock(nn.Module):
    """CrossAttnDownBlockMultiview (BLK:386-541) when ``attn`` else upstream DownBlock2D (BLK:71-83)."""

    def __init__(self, cfg, cin, cout, heads, attn, downsample, attn2):
        super().__init__()
        temb = cfg.time_embed_dim
        self.resnets = nn.ModuleList()
        self.attentions = nn.ModuleList() if attn else None
        for j in range(cfg.layers_per_block):
            self.resnets.append(ResnetBlock2D(cin if j == 0 else cout, cout, temb, cfg.norm_num_groups, cfg.norm_eps))
            if attn:
                self.attentions.append(
                    TransformerMultiviewModel(cout, heads, cfg.norm_num_groups, cfg.use_linear_projection, attn2))
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if downsample else None

    def forward(self, x, temb, num_frames=1):
        outs = []
        for j, r in enumerate(self.resnets):
            x = r(x, temb)
            if self.attentions is not None:
                x = self.attentions[j](x, num_frames=num_frames)
            outs.append(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
            outs.append(x)
        return x, outs


class MidBlock(nn.Module):
    """UNetMidBlockMultiviewCrossAttn, BLK:233-383."""

    def __init__(self, cfg, c, heads, attn2):
        super().__init__()
        temb = cfg.time_embed_dim
        self.resnets = nn.ModuleList([ResnetBlock2D(c, c, temb, cfg.norm_num_groups, cfg.norm_eps),
                                      ResnetBlock2D(c, c, temb, cfg.norm_num_groups, cfg.norm_eps)])
        self.attentions = nn.ModuleList(
            [TransformerMultiviewModel(c, heads, cfg.norm_num_groups, cfg.use_linear_projection, attn2)])

    def forward(self, x, temb, num_frames=1):
        x = self.resnets[0](x, temb)
        x = self.attentions[0](x, num_frames=num_frames)
        return self.resnets[1](x, temb)


class UpBlock(nn.Module):
    """CrossAttnUpBlockMultiview (BLK:544-712) when ``attn`` else upstream UpBlock2D (BLK:192-205)."""

    def __init__(self, cfg, cin, cout, cprev, heads, attn, upsample, attn2):
        super().__init__()
        temb = cfg.time_embed_dim
        n = cfg.layers_per_block + 1
        self.resnets = nn.ModuleList()
        self.attentions = nn.ModuleList() if attn else None
        for j in range(n):
            skip = cin if j == n - 1 else cout
            rin = cprev if j == 0 else cout
            self.resnets.append(ResnetBlock2D(rin + skip, cout, temb, cfg.norm_num_groups, cfg.norm_eps))
            if attn:
                self.attentions.append(
                    TransformerMultiviewModel(cout, heads, cfg.norm_num_groups, cfg.use_linear_projection, attn2))
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if upsample else None

    def forward(self, x, skips: List[torch.Tensor], temb, num_frames=1):
        for j, r in enumerate(self.resnets):
            x = torch.cat([x, skips.pop()], dim=1)
            x = r(x, temb)
            if self.attentions is not None:
                x = self.attentions[j](x, num_frames=num_frames)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x)
        return x


# --------------------------------------------------------------------------- top level
class OracleUNet(nn.Module):
    """Restatement of ``UNetMultiviewConditionModel`` (UNET:149-598)."""

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        ch = cfg.block_out_channels
        self.conv_in = nn.Conv2d(cfg.in_channels, ch[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(ch[0], cfg.time_embed_dim)
        if cfg.enable_tem_embeds:
            self.temporal_pos_embed = TimestepEmbedding(ch[0], cfg.time_embed_dim)
            nn.init.zeros_(self.temporal_pos_embed.linear_2.weight)  # UNET:265-266
            nn.init.zeros_(self.temporal_pos_embed.linear_2.bias)
        if cfg.enable_pose_encoder:
            self.pose_encoder = PoseEncoder(ch[0])
            nn.init.zeros_(self.pose_encoder.final_proj.weight)  # POSE:47-49
            nn.init.zeros_(self.pose_encoder.final_proj.bias)
        nlev = len(ch)
        self.down_blocks = nn.ModuleList()
        cout = ch[0]
        for i in range(nlev):
            cin, cout = cout, ch[i]
            last = i == nlev - 1
            self.down_blocks.append(DownBlock(cfg, cin, cout, cfg.heads(i), attn=not last, downsample=not last,
                                              attn2=cfg.has_attn2(i)))
        self.mid_block = MidBlock(cfg, ch[-1], cfg.heads(nlev - 1), cfg.has_attn2(nlev - 1))
        self.up_blocks = nn.ModuleList()
        rch = list(reversed(ch))
        cout = rch[0]
        for i in range(nlev):
            cprev, cout = cout, rch[i]
            cin = rch[min(i + 1, nlev - 1)]
            lvl = nlev - 1 - i
            self.up_blocks.append(UpBlock(cfg, cin, cout, cprev, cfg.heads(lvl), attn=i > 0,
                                          upsample=i < nlev - 1, attn2=cfg.has_attn2(lvl)))
        self.conv_norm_out = nn.GroupNorm(cfg.norm_num_groups, ch[0], eps=cfg.norm_eps)
        self.conv_out = nn.Conv2d(ch[0], cfg.out_channels, 3, padding=1)

    # UNET:527-546
    @staticmethod
    def frame_indices(domains: List[str], num_frames: int, device=None) -> torch.Tensor:
        out = []
        for d in domains:
            if d == "spatial":
                out.append(torch.zeros(num_frames, device=device))
            elif d == "temporal":
                out.append(torch.arange(num_frames // 2, device=device).repeat(2))
            else:
                raise ValueError(f"Invalid domain for temporal embedding: {d}")
        return torch.cat(out)

    def forward(self, sample, timestep, skeletons=None, domains=None, num_frames: int = 1):
        cfg = self.cfg
        dtype = sample.dtype
        if cfg.center_input_sample:
            sample = 2 * sample - 1.0
        if not torch.is_tensor(timestep):
            timestep = torch.tensor([timestep], dtype=torch.int64)
        timestep = timestep.reshape(-1).expand(sample.shape[0]).to(sample.device)
        t_emb = timestep_embedding(timestep, cfg.block_out_channels[0], cfg.flip_sin_to_cos, cfg.freq_shift).to(dtype)
        emb = self.time_embedding(t_emb)
        if cfg.enable_tem_embeds:
            if len(domains) * num_frames != len(emb):
                raise ValueError(
                    f"num_frames: {num_frames} * len(domains): {len(domains)} != len(emb): {len(emb)}")
            idx = self.frame_indices(domains, num_frames, device=sample.device)
            f_emb = timestep_embedding(idx, cfg.block_out_channels[0], True, 0).to(dtype)
            emb = emb + self.temporal_pos_embed(f_emb)
        x = self.conv_in(sample)
        if cfg.enable_pose_encoder:
            x = x + self.pose_encoder(skeletons)
        skips = [x]
        nd = len(self.down_blocks)
        for i, blk in enumerate(self.down_blocks):
            nf = num_frames if (nd - i - 1) < cfg.num_3d_attn_blocks else 1  # UNET:560
            x, outs = blk(x, emb, num_frames=nf)
            skips += outs
        x = self.mid_block(x, emb, num_frames=num_frames)  # UNET:570
        for i, blk in enumerate(self.up_blocks):
            nf = num_frames if i < cfg.num_3d_attn_blocks else 1  # UNET:582
            x = blk(x, skips, emb, num_frames=nf)
        x = self.conv_out(F.silu(self.conv_norm_out(x)))
        return x


def build_oracle(cfg, seed: int = 1, dtype=torch.float32) -> OracleUNet:
    """Random-init oracle.  Zero-init branches (POSE:47-49, UNET:265-266) and all norm affines are
    re-randomised, otherwise those paths are untested no-ops (SURVEY.md section 8c)."""
    g = torch.Generator().manual_seed(seed)
    m = OracleUNet(cfg)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if name.endswith("scale"):
                p.fill_(2.0)
                continue
            is_norm = ".norm" in name or name.startswith("conv_norm_out")
            if is_norm and name.endswith("weight"):
                p.copy_(1.0 + 0.2 * torch.randn(p.shape, generator=g))
            elif is_norm and name.endswith("bias"):
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
            elif name.endswith("bias"):
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
            else:
                fan_in = p[0].numel()
                p.copy_(torch.randn(p.shape, generator=g) / math.sqrt(fan_in))
    return m.to(dtype).eval()
