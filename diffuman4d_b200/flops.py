"""Algorithmic FLOPs (2 x MAC) of one UNet forward -- the single figure used for roofline numbers.

Formula of SURVEY.md section 8(d): with B images, F frames per 3-D sequence, levels C = block_out_channels,
n_l = (h / 2^l)(w / 2^l), F_l = F for 3-D blocks else 1:
    conv3(ci,co,n) = 18 ci co n        lin(ci,co,n) = 2 ci co n
    Resnet(ci,co,n) = conv3(ci,co,n) + conv3(co,co,n) + [ci != co] lin(ci,co,n) + 2*TE*co
    Transf(C,n,F_l) = 6 lin(C,C,n) + 4 n (F_l n) C + 24 C^2 n   [+ attn2: 4 lin(C,C,n) + 4 n^2 C]
Embedding MLPs, the pose encoder and elementwise work are excluded (< 0.1 %).  Each launch of plan.launches carries its
term of this sum.
"""
from __future__ import annotations

from typing import Dict

from .config import UNetConfig
from .plan import launches


def unet_flops(cfg: UNetConfig, B: int, F: int, h: int, w: int) -> Dict[str, float]:
    if B % F:
        raise ValueError(f"B ({B}) must be a whole number of CFG halves of F ({F}) frames")
    out = {"conv3x3": 0.0, "linear": 0.0, "attn3d": 0.0, "attn2d": 0.0, "ff": 0.0}
    for launch in launches(cfg, F, h, w, halves=B // F):
        if launch.algo:
            out[launch.category] += launch.algo
    out["total"] = sum(out.values())
    return out
