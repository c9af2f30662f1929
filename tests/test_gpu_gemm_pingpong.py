"""The ping-pong GEMM schedule against the cooperative one.

Under ping-pong each MMA warpgroup owns whole 128-row tiles (two 64-row blocks) and the two take turns; under the
cooperative schedule both warpgroups share each tile.  Every dot product still runs over the same k-blocks in the same
order, the epilogue body is the same per 64-row block, and the GroupNorm statistics are the same fixed-point sums of the same
16-row partials.  So the stored output and the statistics words must not depend on the schedule: they are compared byte for
byte, buffer guard bands included, for every epilogue feature set the UNet plan launches at every ping-pong width, and for
tile counts that split unevenly between the warpgroups.  Each case is also held to criterion (a) of test_gpu_gemm_conv_fp64.py
(a correct rounding of a value within the accumulation allowance of the fp64 result), which guards the case of both
schedules being wrong together.

The chooser (gemm_choose_tile) is checked against its mirror (tools/gemm_shapes.py::auto_tile) for every plain GEMM of the
W16@64², W24@64² and W16@128² plans; that test needs no device.
"""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

from test_gpu_gemm_conv_fp64 import Case, check_a  # noqa: E402
from test_gpu_kernel_edges import _check_guard, _check_ws, _guarded, _rand, _stats_ws, _stream  # noqa: E402

COOP, PP = 1, 2
FEATS = {"none": (), "bias": ("bias",), "bias+residual": ("bias", "residual"),
         "bias+residual in place": ("bias", "residual", "inplace"), "bias+residual+stats": ("bias", "residual", "stats"),
         "two-source": ("bias", "two_source"), "geglu+bias": ("bias", "geglu")}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _inputs(M, N, K1, feats, seed):
    K2 = 64 if "two_source" in feats else 0
    g = torch.Generator().manual_seed(seed + 2)
    return {"a": _rand((M, K1), seed), "a2": _rand((M, K2), seed + 5) if K2 else None, "K2": K2,
            "w": _rand((N, K1 + K2), seed + 1, std=(K1 + K2) ** -0.5),
            "bias": (0.5 * torch.randn(N, generator=g)).cuda() if "bias" in feats else None,
            "res": _rand((M, N), seed + 3) if "residual" in feats else None}


def _check_a(x, M, N, K1, feats, out, what):
    """Criterion (a) of test_gpu_gemm_conv_fp64.py on out [M, N or N / 2].  GEGLU weight rows and bias are interleaved
    in groups of 8 (a rows, then g rows); the reference takes them a rows first."""
    w, b = x["w"], x["bias"]
    if "geglu" in feats:
        w = w.view(N // 16, 2, 8, -1).transpose(0, 1).reshape(N, -1)
        b = None if b is None else b.view(N // 16, 2, 8).transpose(0, 1).reshape(N)
    case = Case("pingpong", "gemm", dict(M=M, N=N, K1=K1, K2=x["K2"]), feats, {"rows": 1})
    check_a(out, case, {"a": x["a"], "a2": x["a2"], "w": w, "bias": b, "res": x["res"], "scale": 1.0}, what)


def _run(x, M, N, K1, feats, schedule, bn, ldo, n_img):
    """One launch into a guarded [M + 8, ldo] output; returns (output buffer, statistics workspace or None)."""
    from diffuman4d_b200._lib import check, lib
    geglu = "geglu" in feats
    nout = N // 2 if geglu else N
    out = _guarded(M, nout, ldo, 8)
    res, ld_res = x["res"], N
    if "inplace" in feats:  # residual == out: the kernel reads each residual element before it stores over it
        out[:M, :N] = x["res"]
        res, ld_res = out, ldo
    ws = _stats_ws(n_img * N * 2) if "stats" in feats else None
    p = lambda t: None if t is None else t.data_ptr()
    check(lib().d4d_op_gemm_tiled(p(x["a"]), K1, K1, p(x["a2"]), x["K2"], x["K2"], p(x["w"]), M, N, p(x["bias"]), None, 0, 0,
                                  p(res), ld_res if res is not None else 0, p(out), ldo, int(geglu), 0, 1.0, bn, schedule,
                                  p(ws), M // n_img if ws is not None else 0, _stream()), "d4d_op_gemm_tiled")
    return out, ws


def _check_pair(M, N, K1, feats, bn, coop_bn=None, ldo=None, n_img=1, seed=700):
    """Cooperative at width coop_bn (default bn) and ping-pong at bn: byte-equal buffers and statistics, fp64-close."""
    nout = N // 2 if "geglu" in feats else N
    ldo = ldo or nout
    x = _inputs(M, N, K1, feats, seed)
    (oc, sc), (op, sp) = (_run(x, M, N, K1, feats, COOP, bn if coop_bn is None else coop_bn, ldo, n_img),
                          _run(x, M, N, K1, feats, PP, bn, ldo, n_img))
    what = f"M{M} N{N} K{K1} {'+'.join(feats) or '-'} bn{bn}"
    diff = oc.view(torch.int16) != op.view(torch.int16)
    assert not diff.any(), f"{what}: {int(diff.sum())} output words differ between the cooperative and ping-pong schedules"
    _check_guard(op, M, nout, what)
    if sp is not None:
        assert torch.equal(sc, sp), f"{what}: {int((sc != sp).sum())} statistics words differ between the schedules"
        _check_ws(sp, op[:M, :N], n_img, what)
    _check_a(x, M, N, K1, feats, op[:M, :nout], what)


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("feats", list(FEATS))
def test_pingpong_equals_cooperative_every_kernel(cuda, feats, bn):
    """Every feature set at every ping-pong width (GEGLU has a ping-pong kernel at 128 only); 5 k-blocks like the level-1
    projections, 30 tiles per SM at width 64 so that both warpgroups run many tiles."""
    if "geglu" in feats and bn != 128:
        pytest.skip("GEGLU runs ping-pong at block_n 128 only")
    _check_pair(32 * 256, 640, 320, FEATS[feats], bn, n_img=32)


# (M, N, K1, bn, coop_bn, ldo, feats): edges of the tile grid and of the buffers
EDGES = [(333, 640, 320, 128, None, None, "bias+residual"),          # M not a multiple of 128: the last tile's rows clip
         (77, 256, 192, 64, None, None, "bias+residual in place"),   # one partial tile: a single 64-row block is live
         (200, 320, 320, 0, 64, None, "bias+residual"),              # automatic width 128 over N = 320: the last tile overhangs
         (256, 320, 320, 0, 64, None, "geglu+bias"),                 # GEGLU overhang: 2 x 128 columns -> 160 outputs
         (288, 640, 256, 128, None, 704, "bias+residual+stats"),     # ldo > N: guard columns; 3 images of 96 rows straddle tiles
         (300, 640, 128, 128, None, 712, "geglu+bias")]


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K1,bn,coop_bn,ldo,feats", EDGES, ids=lambda v: str(v))
def test_pingpong_edges(cuda, M, N, K1, bn, coop_bn, ldo, feats):
    n_img = 3 if "stats" in FEATS[feats] else 1
    _check_pair(M, N, K1, FEATS[feats], bn, coop_bn, ldo, n_img)


@pytest.mark.gpu
@pytest.mark.parametrize("per_cta", ["one", "odd", "uneven", "many"])
def test_pingpong_tiles_per_cta(cuda, per_cta):
    """Tile counts per CTA (grid = min(tiles, SMs)): exactly one (warpgroup 1 idles), three (warpgroup 0 runs two), two or
    three across CTAs, and about forty."""
    sms = _sms()
    M, N = {"one": (128 * (sms // 2), 256), "odd": (128 * 3 * sms, 128), "uneven": (128 * (2 * sms + 5), 128),
            "many": (128 * 8 * sms, 640)}[per_cta]
    _check_pair(M, N, 320, FEATS["bias+residual+stats"], 128, n_img=M // 128)


@pytest.mark.gpu
def test_pingpong_refused_where_no_kernel_exists(cuda):
    """An explicit ping-pong launch is an argument error where the kernel does not exist, before anything is launched."""
    x = _inputs(256, 1280, 128, ("bias",), 800)
    for bn in (160, 192, 256):
        with pytest.raises(ValueError):
            _run(x, 256, 1280, 128, ("bias",), PP, bn, 1280, 1)
    with pytest.raises(ValueError):
        _run(_inputs(256, 1280, 128, ("bias", "geglu"), 801), 256, 1280, 128, ("bias", "geglu"), PP, 64, 640, 1)
    with pytest.raises(ValueError):
        _run(x, 256, 1280, 128, ("bias",), 3, 128, 1280, 1)
    torch.cuda.synchronize()


@pytest.mark.parametrize("plan", ["W16@64", "W24@64", "W16@128"])
def test_chooser_follows_the_model(plan):
    import gemm_schedule_sweep
    import gemm_shapes
    from diffuman4d_b200._lib import check, lib
    sms = 132
    for nm, cnt, spec in gemm_schedule_sweep.gemm_plan(plan):
        M, N, K1, K2, geglu = spec["M"], spec["N"], spec["K1"], spec["K2"], "geglu" in spec["feats"]
        bn, sched = ctypes.c_int(), ctypes.c_int()
        check(lib().d4d_gemm_tile_choice(M, N, K1, K2, int(geglu), sms, ctypes.byref(bn), ctypes.byref(sched)))
        assert (128, bn.value, sched.value) == gemm_shapes.auto_tile(N, sms, M=M, geglu=geglu, K=K1 + K2), (plan, nm)
        if sched.value == PP:
            assert bn.value in ((128,) if geglu else (64, 128)), (plan, nm)
        if -(-M // 128) * -(-N // bn.value) <= sms:
            assert sched.value == COOP, f"{plan} {nm}: one tile per SM overlaps nothing"
