"""256-row conv tiles against 128-row tiles.

A 256-row tile gives each MMA warpgroup two 64-row blocks against one weight tile; every dot product still runs over the
same k-blocks in the same order, and the GroupNorm statistics are the same fixed-point sums of the same 16-row partials.  So
the stored output and the statistics words must not depend on the tile rows: they are compared byte for byte, for the three
conv kinds (stride 1, stride 2 through the strided tensor map, four-phase upsampling), the four epilogue instantiations of
the conv kernels, both widths that have 256-row kernels, the level shapes of the UNet at a reduced image count, and grids
that overhang the tile.  Each case is also held to criterion (a) of test_gpu_gemm_conv_fp64.py (a correct rounding of a value
within the accumulation allowance of the fp64 result), which guards the case of both tiles being wrong together.

The tile chooser (gemm_choose_tile) is checked against its cost table (tools/gemm_shapes.py::auto_tile) for every conv of the
W16@64², W24@64² and W16@128² plans; that test needs no device.
"""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

from diffuman4d_b200.config import UNetConfig  # noqa: E402
from diffuman4d_b200.plan import launches  # noqa: E402
from test_gpu_gemm_conv_fp64 import Case, check_a  # noqa: E402
from test_gpu_kernel_edges import _check_ws, _rand, _stats_ws, _stream  # noqa: E402

KIND = {"s1": 0, "s2": 1, "up": 3}
FEATS = {"bias+rowvec+stats": ("bias", "rowvec", "stats"),       # resnet conv1
         "bias+residual+stats": ("bias", "residual", "stats"),   # resnet conv2
         "bias+stats": ("bias", "stats"),                        # down / up sampling
         "all": ("bias", "rowvec", "residual", "act", "stats")}  # the all-features kernel


def _conv_tiled(x, wt, Cout, kind, block_m, block_n, bias=None, rowvec=None, residual=None, act=0, stats=None):
    from diffuman4d_b200._lib import check, lib
    n, H, W, Cin = x.shape
    oh, ow = {"s1": (H, W), "s2": (H // 2, W // 2), "up": (2 * H, 2 * W)}[kind]
    out = torch.empty(n, oh, ow, Cout, device="cuda", dtype=torch.bfloat16)
    p = lambda t: None if t is None else t.data_ptr()
    check(lib().d4d_op_conv_tiled(p(x), n, H, W, Cin, p(wt), Cout, p(bias), p(rowvec), 0 if rowvec is None else rowvec.stride(0),
                                  p(residual), act, p(out), KIND[kind], block_m, block_n, p(stats), _stream()), "d4d_op_conv_tiled")
    return out


def _run_both(n, H, W, Cin, Cout, kind, feats, bn, seed=300):
    """The conv at 128 and at 256 rows: outputs and statistics workspaces, and the launch and operands for check_a."""
    from diffuman4d_b200 import ops
    x = _rand((n, H, W, Cin), seed)
    w = _rand((Cout, Cin, 3, 3), seed + 1, std=(9 * Cin) ** -0.5)
    wt = torch.stack(ops.upsample_phase_weights(w)).contiguous() if kind == "up" else ops.conv_weight_to_octi(w)
    oh, ow = {"s1": (H, W), "s2": (H // 2, W // 2), "up": (2 * H, 2 * W)}[kind]
    bias = (1.0 + 0.5 * torch.randn(Cout, generator=torch.Generator().manual_seed(seed + 2))).cuda() if "bias" in feats else None
    rowvec = _rand((n, Cout), seed + 3) if "rowvec" in feats else None
    res = _rand((n, oh, ow, Cout), seed + 4) if "residual" in feats else None
    act = int("act" in feats)
    case = Case("tile-rows", "conv", dict(n=n, H=H, W=W, Cin=Cin, Cout=Cout, mode=kind), feats, {"rows": oh * ow})
    inp = {"a": x, "a2": None, "w": w, "bias": bias, "rowvec": rowvec, "scale": 1.0,
           "res": None if res is None else res.view(-1, Cout)}
    got = {}
    for bm in (128, 256):
        ws = _stats_ws(n * Cout * 2) if "stats" in feats else None
        got[bm] = (_conv_tiled(x, wt, Cout, kind, bm, bn, bias, rowvec, res, act, ws), ws)
    return got, (case, inp)


def _check_pair(got, ref, n, what):
    """ref: (case, operands) of the launch, for criterion (a)."""
    (o128, s128), (o256, s256) = got[128], got[256]
    assert torch.equal(o128.view(torch.int16), o256.view(torch.int16)), \
        f"{what}: {int((o128.view(torch.int16) != o256.view(torch.int16)).sum())} output words differ between 128 and 256 rows"
    if s128 is not None:
        assert torch.equal(s128, s256), f"{what}: {int((s128 != s256).sum())} statistics words differ between 128 and 256 rows"
        _check_ws(s256, o256, n, what)
    check_a(o256.view(-1, o256.shape[-1]), *ref, what)


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [128, 160])
@pytest.mark.parametrize("feats", list(FEATS))
@pytest.mark.parametrize("kind", ["s1", "s2", "up"])
def test_rows_256_equal_128_every_kernel(cuda, kind, feats, bn):
    """Every 256-row instantiation (4 feature sets x 2 widths) under every conv kind; Cout = 640 divides by both widths."""
    n, H, W = (3, 32, 32) if kind != "s2" else (3, 64, 64)
    got, ref = _run_both(n, H, W, 128, 640, kind, FEATS[feats], bn)
    _check_pair(got, ref, n, f"{kind} {feats} bn{bn}")


# (n, H, W, Cin, Cout, kind): the level shapes of the SD-2.1 layout at 4 images, then grids that do not fill their tiles
LEVELS = [(4, 64, 64, 320, 320, "s1"), (4, 32, 32, 640, 640, "s1"), (4, 16, 16, 1280, 1280, "s1"), (4, 8, 8, 1280, 1280, "s1"),
          (4, 64, 64, 320, 320, "s2"), (4, 32, 32, 640, 640, "s2"), (4, 16, 16, 1280, 1280, "s2"),
          (4, 8, 8, 1280, 1280, "up"), (4, 16, 16, 1280, 1280, "up"), (4, 32, 32, 640, 640, "up")]
EDGES = [(32, 16, 16, 64, 1280, "s1"),   # 256 tiles of 256 rows: more than SMs, so a CTA walks several tiles through its ring
         (2, 24, 24, 64, 320, "s1"),     # 16x16 boxes overhang in x and y
         (2, 40, 24, 64, 320, "s1"),
         (7, 8, 8, 128, 640, "s1"),      # four images per tile, the last tile one image short
         (2, 16, 16, 64, 400, "s1"),     # N = 400: the last 160-wide tile overhangs (automatic width only)
         (3, 16, 16, 72, 320, "s1"),     # Cin not a multiple of 64: the last k-block of each tap is zero-filled
         (2, 48, 48, 64, 320, "s2"),     # 24x24 output grid
         (5, 8, 8, 72, 320, "up"),
         (2, 12, 24, 64, 320, "up")]


@pytest.mark.gpu
@pytest.mark.parametrize("n,H,W,Cin,Cout,kind", LEVELS + EDGES, ids=lambda v: str(v))
def test_rows_256_equal_128_shapes(cuda, n, H, W, Cin, Cout, kind):
    feats = FEATS["bias+rowvec+stats"] if kind == "s1" else FEATS["bias+stats"]
    bn = 160 if Cout % 160 == 0 else 0
    got, ref = _run_both(n, H, W, Cin, Cout, kind, feats, bn, seed=400)
    _check_pair(got, ref, n, f"{kind} {n}x{H}x{W} {Cin}->{Cout}")


@pytest.mark.gpu
def test_rows_256_refused_where_no_kernel_exists(cuda):
    """An explicit 256-row tile is an argument error where the kernel does not exist, before anything is launched."""
    x = _rand((2, 16, 16, 64), 500)
    wt = _rand((1280, 9, 64), 501)
    for bm, bn in [(256, 256), (256, 64), (256, 320), (64, 0), (192, 160)]:
        with pytest.raises(ValueError):
            _conv_tiled(x, wt, 1280, "s1", bm, bn)
    torch.cuda.synchronize()


def _plan_convs(n, s):
    """(n, H, W, Cin, Cout, mode) of every distinct conv of the SD-2.1 plan (plan.launches) on n images of s x s latents."""
    convs = (c for c in launches(UNetConfig.sd21(), n // 2, s, s) if c.kind == "conv")
    return list(dict.fromkeys(tuple(c.spec.values()) for c in convs))


@pytest.mark.parametrize("n,s", [(32, 64), (48, 64), (32, 128)], ids=["W16@64", "W24@64", "W16@128"])
def test_chooser_follows_the_cost_table(n, s):
    import gemm_shapes
    from diffuman4d_b200._lib import check, lib
    sms = 132
    for n_img, H, W, Cin, Cout, mode in _plan_convs(n, s):
        bm, bn = ctypes.c_int(), ctypes.c_int()
        check(lib().d4d_conv_tile_choice(n_img, H, W, Cin, Cout, KIND[mode], sms, ctypes.byref(bm), ctypes.byref(bn)))
        assert (bm.value, bn.value) == gemm_shapes.auto_tile(Cout, sms, conv=(n_img, H, W, Cin, mode)), (n_img, H, W, Cin, Cout, mode)
        oh = H // 2 if mode == "s2" else H
        tiles_256 = gemm_shapes.conv_tiles(256, n_img, oh, oh) * (4 if mode == "up" else 1) * -(-Cout // max(bn.value, 1))
        if bm.value == 256:
            assert bn.value in (128, 160) and tiles_256 >= sms, (n_img, H, W, Cout, mode)
        if Cin == 64:
            assert bm.value == 128, "the pose encoder's 9-k-block convs are epilogue-bound and keep 128 rows"
        if s == 64 and n == 32 and H == 8 and mode == "s1":
            assert bm.value == 128, "level 4 of W16@64² has fewer 256-row tiles than SMs"
        if mode == "s1" and Cout >= 320 and n_img * H * W >= 8192:
            assert (bm.value, bn.value) == (256, 160), (n_img, H, W, Cout, mode)
