"""The two launch counts of a plan come from one record of its ops.

d4d_forward_launches reports the plan's launch total; d4d_profile_forward adds each op's launches into its kernel kind.
For single-GPU plans of the benchmarked SD-2.1 layout, with CFG and the pose encoder, at a latent size where some
GroupNorm statistics need their own launch (32x32: 4x4 at the deepest level) and one where every producer accumulates
them (64x64), the per-kind launches sum to the forward's launches, and both equal the count the plan had when this test
was written: a change to the plan's launch list has to update LAUNCHES on purpose."""
import ctypes as C
import gc

import pytest
import torch

from diffuman4d_b200.config import UNetConfig

# (F, h, w) -> kernel launches of one forward (B = 2F: CFG halves)
LAUNCHES = {(4, 32, 32): 309, (4, 64, 64): 292}


@pytest.mark.gpu
def test_profile_launches_sum_to_forward_launches(cuda):
    from diffuman4d_b200._lib import check, lib
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict
    cfg = UNetConfig.sd21()
    assert cfg.enable_pose_encoder
    unet = B200MultiviewUNet(cfg, device=0).load_state_dict(random_state_dict(cfg, seed=1, device="cuda"))
    got = {}
    try:
        for F, h, w in LAUNCHES:
            B = 2 * F
            g = torch.Generator(device="cuda").manual_seed(0)
            x = torch.randn(B, cfg.in_channels, h, w, generator=g, device="cuda").to(torch.bfloat16)
            t = torch.randint(0, 1000, (B,), generator=g, device="cuda")
            sk = (torch.rand(B, 3, 8 * h, 8 * w, generator=g, device="cuda") * 2 - 1).to(torch.bfloat16)
            y = torch.empty(B, cfg.out_channels, h, w, device="cuda", dtype=torch.bfloat16)
            ms, n, fl = (C.c_float * 6)(), (C.c_int32 * 6)(), (C.c_double * 6)()
            check(lib().d4d_profile_forward(unet._h, x.data_ptr(), t.data_ptr(), sk.data_ptr(), (C.c_int32 * 2)(0, 0), 2,
                                            B, F, h, w, y.data_ptr(), torch.cuda.current_stream().cuda_stream, ms, n, fl),
                  "d4d_profile_forward")
            got[F, h, w] = {"by kind": list(n), "sum": sum(n), "forward": unet.forward_launches(2, B, F, h, w)}
            print(f"\n  [F={F} {h}x{w}] {got[F, h, w]}")
    finally:
        del unet
        gc.collect()
        torch.cuda.empty_cache()
    assert {k: (v["sum"], v["forward"]) for k, v in got.items()} == {k: (n, n) for k, n in LAUNCHES.items()}, got
