"""plan.modules / plan.launches: the one walk of the UNet on the Python side.

* On the CPU, everything read from the walk (the weight keys, unet_flops, exchange_bytes, the attention launch lists, the
  module plan and the tools' GEMM / conv shape tables) reproduces tests/golden/plan_walk.jsonl exactly, over a grid of
  configs and latent shapes.  gen_plan_walk.py wrote the fixture from the hand-written restatements the walk replaced.
* On the GPU, one profiled forward (d4d_profile_forward, the call bench.py makes) reports, for each of gemm, conv and
  attention, exactly the launch count and the executed FLOPs that plan.launches sums.
"""
import ctypes as C
import gc
import json
import os
import sys

import pytest
import torch

from diffuman4d_b200.config import UNetConfig
from diffuman4d_b200.plan import launches
from test_gpu_attention_fp64 import PLANS

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))

import gen_plan_walk  # noqa: E402

KINDS = ("gemm", "conv", "attention")   # d4d_profile_forward's kinds 0, 1, 2
PROFILED = dict(PLANS, **{
    "tiny-L1-F4@16": (UNetConfig.tiny(layers_per_block=1), 4, 16, 16),
    "tiny-3d4-F4@24": (UNetConfig.tiny(num_3d_attn_blocks=4), 4, 24, 24)})


@pytest.mark.parametrize("table", ["state_dict_spec", "module_plan", "unet_flops", "exchange_bytes",
                                   "attention_launches", "plan_shapes"])
def test_walk_reproduces_the_restatements(table):
    want = gen_plan_walk.read()[table]
    got = json.loads(json.dumps(gen_plan_walk.generate()))[table]
    assert got.keys() == want.keys()
    for key in want:
        assert got[key] == want[key], key


@pytest.mark.gpu
@pytest.mark.parametrize("plan", list(PROFILED))
def test_launches_match_profile(cuda, plan):
    """plan.launches is the library's plan: per kind, the same number of launches and the same executed FLOPs."""
    from diffuman4d_b200._lib import check, lib
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict
    cfg, F, h, w = PROFILED[plan]
    B = 2 * F
    unet = B200MultiviewUNet(cfg, device=0).load_state_dict(random_state_dict(cfg, seed=1, device="cuda"))
    try:
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randn(B, cfg.in_channels, h, w, generator=g, device="cuda").to(torch.bfloat16)
        t = torch.randint(0, 1000, (B,), generator=g, device="cuda")
        sk = (torch.rand(B, 3, 8 * h, 8 * w, generator=g, device="cuda") * 2 - 1).to(torch.bfloat16) \
            if cfg.enable_pose_encoder else None
        y = torch.empty(B, cfg.out_channels, h, w, device="cuda", dtype=torch.bfloat16)
        ms, n, fl = (C.c_float * 6)(), (C.c_int32 * 6)(), (C.c_double * 6)()
        check(lib().d4d_profile_forward(unet._h, x.data_ptr(), t.data_ptr(), None if sk is None else sk.data_ptr(),
                                        (C.c_int32 * 2)(0, 1), 2, B, F, h, w, y.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream, ms, n, fl), "d4d_profile_forward")
        plan_launches = launches(cfg, F, h, w)
        for k, kind in enumerate(KINDS):
            mine = [a for a in plan_launches if a.kind == kind]
            print(f"\n  [{plan}] {kind}: {n[k]} launches, {fl[k] / 1e12:.3f} TFLOP, {ms[k]:.2f} ms")
            assert n[k] == sum(a.launches for a in mine), kind
            assert fl[k] == sum(a.flops for a in mine), kind
    finally:
        del unet
        gc.collect()
        torch.cuda.empty_cache()
