"""Weight-key contract of the UNet (diffusers layout, SURVEY.md section 8b) and seeded random weights.

``state_dict_spec`` lists every parameter of ``unet/diffusion_pytorch_model.safetensors`` for a given config with its
diffusers shape, module by module of plan.modules; the C++ loader (the ``Model`` constructor in csrc/unet.cu) and the CPU
oracle must agree with it (tested).
"""
from __future__ import annotations

import math
from collections import OrderedDict
from typing import Dict, Tuple

import torch

from .config import UNetConfig
from .plan import modules

POSE_SPEC = [(3, 3, 3), (3, 16, 4), (16, 16, 3), (16, 32, 4), (32, 32, 3), (32, 64, 4), (64, 64, 3), (64, 128, 3)]


def state_dict_spec(cfg: UNetConfig) -> "OrderedDict[str, Tuple[int, ...]]":
    spec: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    C0, TE = cfg.block_out_channels[0], cfg.time_embed_dim

    def lin(p, out, inp, bias=True):
        spec[p + ".weight"] = (out, inp)
        if bias:
            spec[p + ".bias"] = (out,)

    def conv(p, out, inp, k):
        spec[p + ".weight"] = (out, inp, k, k)
        spec[p + ".bias"] = (out,)

    def norm(p, c):
        spec[p + ".weight"] = (c,)
        spec[p + ".bias"] = (c,)

    def resnet(p, cin, cout):
        norm(p + ".norm1", cin)
        conv(p + ".conv1", cout, cin, 3)
        lin(p + ".time_emb_proj", cout, TE)
        norm(p + ".norm2", cout)
        conv(p + ".conv2", cout, cout, 3)
        if cin != cout:
            conv(p + ".conv_shortcut", cout, cin, 1)

    def xf(p, C, attn2):
        norm(p + ".norm", C)
        if cfg.use_linear_projection:
            lin(p + ".proj_in", C, C)
        else:
            conv(p + ".proj_in", C, C, 1)
        b = p + ".transformer_blocks.0"
        norm(b + ".norm1", C)
        for n in ("to_q", "to_k", "to_v"):
            lin(f"{b}.attn1.{n}", C, C, bias=False)
        lin(b + ".attn1.to_out.0", C, C)
        if attn2:
            norm(b + ".norm2", C)
            for n in ("to_q", "to_k", "to_v"):
                lin(f"{b}.attn2.{n}", C, C, bias=False)
            lin(b + ".attn2.to_out.0", C, C)
        norm(b + ".norm3", C)
        lin(b + ".ff.net.0.proj", 8 * C, C)
        lin(b + ".ff.net.2", C, 4 * C)
        if cfg.use_linear_projection:
            lin(p + ".proj_out", C, C)
        else:
            conv(p + ".proj_out", C, C, 1)

    conv("conv_in", C0, cfg.in_channels, 3)
    lin("time_embedding.linear_1", TE, C0)
    lin("time_embedding.linear_2", TE, TE)
    if cfg.enable_tem_embeds:
        lin("temporal_pos_embed.linear_1", TE, C0)
        lin("temporal_pos_embed.linear_2", TE, TE)
    if cfg.enable_pose_encoder:
        for i, (ci, co, k) in enumerate(POSE_SPEC):
            conv(f"pose_encoder.conv_layers.{2 * i}", co, ci, k)
        conv("pose_encoder.final_proj", C0, 128, 1)
        spec["pose_encoder.scale"] = (1,)
    for m in modules(cfg):
        if m.type == "resnet":
            resnet(m.path, m.cin + m.skip, m.cout)
        elif m.type == "transformer":
            xf(m.path, m.cout, m.attn2)
        else:
            conv(m.path + ".conv", m.cout, m.cin, 3)
    norm("conv_norm_out", C0)
    conv("conv_out", cfg.out_channels, C0, 3)
    return spec


def random_state_dict(cfg: UNetConfig, seed: int = 1, dtype=torch.bfloat16, device="cpu") -> Dict[str, torch.Tensor]:
    """Seeded random weights (no network for the real checkpoint).  Fan-in-scaled normal weights, small biases,
    randomised norm affines and NON-zero values for the reference's zero-initialised branches
    (pose_encoder.final_proj, temporal_pos_embed.linear_2) so those paths carry signal.  The values depend on the seed
    and on the device whose generator draws them; a CUDA draw of the full-width UNet takes a fraction of the host's
    seconds."""
    g = torch.Generator(device=device).manual_seed(seed)
    randn = lambda shape: torch.randn(shape, generator=g, device=device)
    sd: Dict[str, torch.Tensor] = {}
    for key, shape in state_dict_spec(cfg).items():
        if key.endswith("scale"):
            t = torch.full(shape, 2.0, device=device)
        else:
            is_norm = ".norm" in key or key.startswith("conv_norm_out")
            if is_norm and key.endswith("weight"):
                t = 1.0 + 0.2 * randn(shape)
            elif is_norm and key.endswith("bias"):
                t = 0.1 * randn(shape)
            elif key.endswith("bias"):
                t = 0.05 * randn(shape)
            else:
                fan_in = 1
                for s in shape[1:]:
                    fan_in *= s
                t = randn(shape) / math.sqrt(fan_in)
        sd[key] = t.to(dtype)
    return sd
