"""The UNet's modules and the tensor-core launches of one forward, in plain Python (no torch, no library).

``modules(cfg)`` walks the network in forward order as the ``Model`` constructor (csrc/unet.cu) does, and
``launches(...)`` expands that walk into the GEMM, convolution and attention launches ``PlanBuilder::build`` makes.  The
weight keys (weights.state_dict_spec), the FLOPs bench.py reports (flops.unet_flops), the K/V exchange size
(sharded.exchange_bytes), the shape tables of the tuning tools and the tests' launch lists all read these two functions,
and tests/test_plan.py checks the launch counts and FLOPs against a profiled forward of the library.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import numpy as np


@dataclass(frozen=True)
class Module:
    path: str                        # diffusers module path
    type: str                        # "resnet", "transformer", "downsampler" or "upsampler"
    level: int                       # resolution level of the input: h >> level
    cin: int
    cout: int
    skip: int = 0                    # up-path ResNet: channels of the skip concatenated to the input
    skip_from: Optional[str] = None  # ... and the module whose output it is
    is3d: bool = False               # transformer: attn1 attends over all frames of a sequence
    attn2: bool = False              # transformer: has the per-image attn2


def modules(cfg) -> List[Module]:
    """The down / mid / up modules in forward order.  The stem (time and frame-index embeddings, pose encoder, conv_in)
    runs before them and the head (conv_norm_out, conv_out) after."""
    ch, L, n3d = cfg.block_out_channels, cfg.layers_per_block, cfg.num_3d_attn_blocks
    out: List[Module] = []
    skips = [("conv_in", ch[0])]

    def add(path, type, level, cin, cout=None, **kw):
        out.append(Module(path, type, level, cin, cin if cout is None else cout, **kw))
        return out[-1]

    def xf(path, level, is3d):
        add(path, "transformer", level, ch[level], is3d=is3d, attn2=cfg.has_attn2(level))

    c = ch[0]
    for i in range(4):
        p = f"down_blocks.{i}"
        for j in range(L):
            add(f"{p}.resnets.{j}", "resnet", i, c, ch[i])
            c = ch[i]
            if i < 3:
                xf(f"{p}.attentions.{j}", i, 3 - i < n3d)
            skips.append((out[-1].path, c))
        if i < 3:
            skips.append((add(f"{p}.downsamplers.0", "downsampler", i, c).path, c))
    add("mid_block.resnets.0", "resnet", 3, c)
    xf("mid_block.attentions.0", 3, True)
    add("mid_block.resnets.1", "resnet", 3, c)
    for i in range(4):
        lvl, p = 3 - i, f"up_blocks.{i}"
        for j in range(L + 1):
            src, cs = skips.pop()
            add(f"{p}.resnets.{j}", "resnet", lvl, c, ch[lvl], skip=cs, skip_from=src)
            c = ch[lvl]
            if i > 0:
                xf(f"{p}.attentions.{j}", lvl, i < n3d)
        if i < 3:
            add(f"{p}.upsamplers.0", "upsampler", lvl, c)
    assert not skips
    return out


def pad_head_dim(d: int) -> int:
    """The head dim the attention kernel runs (pad_head_dim of csrc/unet.cu)."""
    return 64 if d <= 64 else (128 if d <= 128 else 192)


@dataclass
class Launch:
    kind: str                 # "gemm", "conv" or "attention" (d4d_profile_forward's kinds 0, 1, 2)
    module: str               # owning module: a path of modules(), or a stem / head module
    op: str                   # which launch of the module
    level: int                # resolution level (0 for the stem and head)
    spec: dict                # gemm {M, N, K1, K2}, conv {n, H, W, Cin, Cout, mode}, attention
                              # {batch, seq, seq_kv, heads, dpad, head_dim, scale}: what the library receives
    feats: tuple = ()         # epilogue features
    flops: float = 0.0        # executed FLOPs: gemm_flops / attn_flops
    algo: float = 0.0         # algorithmic FLOPs (2 x MAC) that flops.unet_flops counts ...
    category: str = ""        # ... under this key
    launches: int = 1         # kernel launches (the frame-sharded QKV GEMM adds a flag signal and wait)


def launches(cfg, F: int, h: int, w: int, halves: int = 2, ranks: int = 1) -> List[Launch]:
    """The tensor-core launches of one forward of `halves` CFG halves of F frames at an h x w latent, in plan order.
    ranks > 1: one rank's launches of the frame-sharded forward, F / ranks frames local; a 3-D attention then has
    F / ranks * hw local queries per CFG half and F * hw gathered keys, and its QKV GEMM scatters K|V to every rank."""
    C0, TE = cfg.block_out_channels[0], cfg.time_embed_dim
    Fl = F // ranks
    B = halves * Fl
    out: List[Launch] = []

    def hw(lvl):
        return (h >> lvl) * (w >> lvl)

    def rec(kind, module, op, level, spec, feats, flops, algo=0.0, category="", n=1):
        out.append(Launch(kind, module, op, level, spec, tuple(feats), float(flops), float(algo), category, n))

    def gemm(module, op, level, M, N, K1, feats, K2=0, algo=0.0, category="linear", n=1):
        flops = 2.0 * M * N * 64 * (-(-K1 // 64) + -(-K2 // 64))
        rec("gemm", module, op, level, dict(M=M, N=N, K1=K1, K2=K2), feats, flops, algo, category, n)

    def conv(module, op, level, n_img, H, W, Cin, Cout, mode, feats, algo=0.0):
        oh, ow, phases, taps = (H // 2, W // 2, 1, 9) if mode == "s2" else (H, W, 4, 4) if mode == "up" else (H, W, 1, 9)
        flops = 2.0 * n_img * oh * ow * phases * Cout * 64 * taps * -(-Cin // 64)
        rec("conv", module, op, level, dict(n=n_img, H=H, W=W, Cin=Cin, Cout=Cout, mode=mode), feats, flops, algo,
            "conv3x3")

    def stats(lvl):
        """gemm_stats fuses the GroupNorm statistics where the grid its tiles walk has H > 1 and H * W % 32 == 0."""
        return ("stats",) if (h >> lvl) > 1 and hw(lvl) % 32 == 0 else ()

    def attention(module, op, lvl, C, heads, d, batch, seq, seq_kv, category):
        dp = pad_head_dim(d)
        scale = float(np.float32(1.0) / np.sqrt(np.float32(d)))   # 1.0f / sqrtf(head_dim), from the real head dim
        rec("attention", module, op, lvl, dict(batch=batch, seq=seq, seq_kv=seq_kv, heads=heads, dpad=dp, head_dim=d,
                                                scale=scale), (), 4.0 * batch * heads * seq * seq_kv * dp,
            4.0 * batch * seq * seq_kv * C, category)

    def self_attention(m, prefix, is3d):
        C, heads, d, lvl, n = m.cout, cfg.heads(m.level), cfg.head_dim(m.level), m.level, hw(m.level)
        Cp, M = heads * pad_head_dim(d), B * n
        sharded = is3d and ranks > 1
        gemm(m.path, prefix + "qkv", lvl, M, 3 * Cp, C, ("kv_scatter",) if sharded else (), algo=6.0 * C * C * M,
             n=3 if sharded else 1)
        if is3d:
            attention(m.path, prefix + "attention", lvl, C, heads, d, halves, Fl * n, F * n, "attn3d")
        else:
            attention(m.path, prefix + "attention", lvl, C, heads, d, B, n, n, "attn2d")
        gemm(m.path, prefix + "out-proj", lvl, M, C, Cp, ("bias", "residual"), algo=2.0 * C * C * M)

    # time (+ frame-index) embedding; every ResNet's time_emb_proj as one GEMM of N = sum of their widths
    gemm("time_embedding", "time1", 0, B, TE, C0, ("bias", "act"))
    gemm("time_embedding", "time2", 0, B, TE, TE, ("bias",))
    if cfg.enable_tem_embeds:
        gemm("temporal_pos_embed", "tem1", 0, B, TE, C0, ("bias", "act"))
        gemm("temporal_pos_embed", "tem2", 0, B, TE, TE, ("bias", "residual"))
    ldt = sum(m.cout for m in modules(cfg) if m.type == "resnet")
    gemm("time_emb_proj", "temb_all", 0, B, ldt, TE, ("bias",), algo=2.0 * TE * ldt * B)
    # pose encoder layers 5-7 and its projection (layers 0-4 run on CUDA cores); conv_in as a GEMM over im2col
    M0 = B * h * w
    if cfg.enable_pose_encoder:
        gemm("pose_encoder", "pose l5", 0, M0, 64, 512, ("bias", "act"))
        conv("pose_encoder", "pose l6", 0, B, h, w, 64, 64, "s1", ("bias", "act"))
        conv("pose_encoder", "pose l7", 0, B, h, w, 64, 128, "s1", ("bias", "act"))
        gemm("pose_encoder", "pose proj", 0, M0, C0, 128, ("bias", "scale"))
    gemm("conv_in", "conv_in", 0, M0, C0, 192, ("bias",) + ("residual",) * cfg.enable_pose_encoder + stats(0),
         algo=18.0 * cfg.in_channels * C0 * M0, category="conv3x3")
    for m in modules(cfg):
        lvl, n = m.level, hw(m.level)
        s = h >> lvl, w >> lvl
        if m.type == "resnet":
            cin = m.cin + m.skip
            conv(m.path, "conv1", lvl, B, *s, cin, m.cout, "s1", ("bias", "rowvec") + stats(lvl),
                 algo=18.0 * cin * m.cout * n * B)
            if cin != m.cout:
                gemm(m.path, "shortcut", lvl, B * n, m.cout, m.cin, ("bias", "two_source") if m.skip else ("bias",),
                     K2=m.skip, algo=2.0 * cin * m.cout * n * B)
            conv(m.path, "conv2", lvl, B, *s, m.cout, m.cout, "s1", ("bias", "residual") + stats(lvl),
                 algo=18.0 * m.cout * m.cout * n * B)
        elif m.type == "transformer":
            C, M = m.cout, B * n
            gemm(m.path, "proj_in", lvl, M, C, C, ("bias",), algo=2.0 * C * C * M)
            self_attention(m, "", m.is3d and F > 1)   # 3-D over the window, also when a rank holds one frame
            if m.attn2:
                self_attention(m, "attn2 ", False)
            gemm(m.path, "ff1 geglu", lvl, M, 8 * C, C, ("bias", "geglu"), algo=16.0 * C * C * M, category="ff")
            gemm(m.path, "ff2", lvl, M, C, 4 * C, ("bias", "residual"), algo=8.0 * C * C * M, category="ff")
            gemm(m.path, "proj_out", lvl, M, C, C, ("bias", "residual") + stats(lvl), algo=2.0 * C * C * M)
        elif m.type == "downsampler":
            conv(m.path, "downsample", lvl, B, *s, m.cin, m.cout, "s2", ("bias",) + stats(lvl + 1),
                 algo=18.0 * m.cin * m.cout * hw(lvl + 1) * B)
        else:   # nearest x2 then 3x3: four sub-pixel phases of 2x2 taps on the low-resolution grid
            conv(m.path, "upsample", lvl, B, *s, m.cin, m.cout, "up", ("bias",) + stats(lvl),
                 algo=18.0 * m.cin * m.cout * hw(lvl - 1) * B)
    conv("conv_out", "conv_out", 0, B, h, w, C0, 16, "s1", ("bias",), algo=18.0 * C0 * cfg.out_channels * M0)
    return out
