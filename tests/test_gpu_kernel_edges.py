"""Tile edges of the sm_90a kernels, against plain fp64 references.

test_gpu_ops.py checks each op's values at a tolerance that fits bf16 rounding.  This file checks what that tolerance
cannot see:

* GroupNorm statistics.  Every GEMM / conv epilogue instantiation the UNet plan launches with statistics (conv
  E_BIAS|E_ROWVEC|E_STATS, conv E_BIAS|E_STATS for the stride-2 and four-phase upsampling convs, plain
  E_BIAS|E_RES|E_STATS; conv E_BIAS|E_RES|E_STATS is test_gpu_ops.py::test_conv3x3_fused_groupnorm_stats) and the
  stand-alone statistics kernel must produce the per-(image, channel) fixed-point
  sums of the STORED bf16 output to within the rounding of one fp32 16-term partial plus half a fixed-point unit per
  partial:
      |S * 2^-28 - sum x| <= 2^-20 sum|x| + hw 2^-28,    |Q * 2^-24 - sum x^2| <= 2^-20 sum x^2 + hw 2^-24.
  A dropped or doubled 16-row partial misses this by orders of magnitude.
* GroupNorm apply at its numeric edges (a mean of 64 standard deviations, a group whose stored values sit ~600 standard
  deviations from zero, sd 1e-3 at eps 1e-6, constant groups, groups split by the virtual concat): one bf16 ulp of the
  fp64 result (magnitudes below 2^-8 count as 2^-8), plus 2^-20 (|x - mean| + |mean|) |gamma| rstd for the fp32 affine,
  plus the effect of the statistics' own (separately bounded) rounding, measured from the sums the kernel read.
* Writes outside the logical output (overhanging M / N / pixel / image tiles, rows past seq, statistics words past
  [n_img][C][2]) into sentinel-filled guard bands, and reads of the lda slack of strided operands (filled with NaN).
* Attention with K/V from a separate matrix (the frame-sharded layout) by an exact key census: with K = 0 every softmax
  weight is exactly 1, so each output column is the number of keys whose V column is 1, divided by seq_kv.
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SENT16 = 0x7FA5                # bf16 NaN bit pattern that no kernel produces
SENT64 = 0x0123456789ABCDEF    # statistics guard word
GUARD_WORDS = 4096


# ------------------------------------------------------------------------------------------------ helpers
def _rand(shape, seed, std=1.0, mean=0.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * std + mean).to(torch.bfloat16).cuda()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _close(out, ref, rtol=8e-3, afrac=2e-3):
    """The value tolerance of test_gpu_ops.py: |out - ref| <= rtol |ref| + afrac max|ref|."""
    ref, out = ref.float(), out.float()
    assert out.shape == ref.shape, (out.shape, ref.shape)
    assert torch.isfinite(out).all(), "non-finite kernel output"
    scale = ref.abs().max().item() + 1e-12
    err = (out - ref).abs()
    bad = err > rtol * ref.abs() + afrac * scale
    assert not bad.any(), f"max err {err.max().item():.4g} (scale {scale:.4g}), {int(bad.sum())} / {bad.numel()} out of tolerance"


def _bf16_ulp(mag):
    return torch.exp2(torch.floor(torch.log2(mag)) - 7)


@contextlib.contextmanager
def _fp32_exact():
    """fp32 references without TF32 (cuDNN convolutions use it by default)."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _conv_ref(x_nhwc, w_oihw, bias, stride=1, up=False):
    with _fp32_exact():
        xc = x_nhwc.float().permute(0, 3, 1, 2)
        if up:
            xc = F.interpolate(xc, scale_factor=2.0, mode="nearest")
        return F.conv2d(xc, w_oihw.float(), bias, stride=stride, padding=1).permute(0, 2, 3, 1)


def _stats_ws(words):
    """Zeroed statistics workspace of `words` int64 followed by GUARD_WORDS sentinel words."""
    ws = torch.full((words + GUARD_WORDS,), SENT64, dtype=torch.int64, device="cuda")
    ws[:words] = 0
    return ws


def _check_stats(st, y, n_img, what=""):
    """st: n_img * C * 2 statistics words; y: the stored tensor they describe, [n_img, hw, C] in any shape."""
    C = y.shape[-1]
    y = y.reshape(n_img, -1, C).double()
    hw = y.shape[1]
    st = st.view(n_img, C, 2).double()
    s_ref, a_ref, q_ref = y.sum(1), y.abs().sum(1), (y * y).sum(1)
    es = (st[..., 0] * 2.0 ** -28 - s_ref).abs()
    eq = (st[..., 1] * 2.0 ** -24 - q_ref).abs()
    bs = 2.0 ** -20 * a_ref + hw * 2.0 ** -28
    bq = 2.0 ** -20 * q_ref + hw * 2.0 ** -24
    assert (es <= bs).all(), f"{what}: sum off by {(es / bs).max().item():.3g} x the bound at {int((es > bs).sum())} / {es.numel()} (image, channel)"
    assert (eq <= bq).all(), f"{what}: sum of squares off by {(eq / bq).max().item():.3g} x the bound at {int((eq > bq).sum())} / {eq.numel()} (image, channel)"


def _check_ws(ws, y, n_img, what=""):
    """ws from _stats_ws: exact statistics of y, guard words untouched."""
    words = n_img * y.shape[-1] * 2
    assert (ws[words:] == SENT64).all(), f"{what}: statistics written past [{n_img}][{y.shape[-1]}][2]"
    _check_stats(ws[:words], y, n_img, what)


def _check_standalone_stats(y, n_img):
    """The stand-alone statistics kernel (d4d_op_groupnorm's first launch) on the same stored tensor: same bound."""
    from diffuman4d_b200 import ops
    C = y.shape[-1]
    x = y.reshape(n_img, -1, C).contiguous()
    ws = _stats_ws(n_img * C * 2)
    ops.groupnorm(x, torch.ones(C, device="cuda"), torch.zeros(C, device="cuda"), 32, 1e-5, False, stats=ws)
    _check_ws(ws, x, n_img, "stand-alone statistics")


def _widths(N):
    """Tile widths to run: automatic, and every wgmma width that divides N."""
    return [0] + [bn for bn in (64, 128, 256) if N % bn == 0]


def _auto_block_n(rows, N):
    """gemm_prepare's automatic tile width (gemm_wgmma.cu)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    best = None
    for c in (64, 128, 256):
        n_tiles = -(-N // c)
        waves = -(-(-(-rows // 128) * n_tiles) // sms)
        cost = waves * (c + 64) + (n_tiles * c - N) // 4
        if best is None or cost <= best[0]:
            best = (cost, c)
    return best[1]


def _guarded(rows, cols, ld, guard_rows):
    """bf16 buffer [rows + guard_rows, ld] filled with SENT16; the kernel writes its [:rows, :cols] block."""
    return torch.full((rows + guard_rows, ld), SENT16, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def _check_guard(buf, rows, cols, what=""):
    bits = buf.view(torch.int16).clone()
    bits[:rows, :cols] = SENT16
    bad = bits != SENT16
    assert not bad.any(), f"{what}: {int(bad.sum())} bf16 words written outside the [{rows}, {cols}] output"


def _pad_params(cases, widths_of):
    return [pytest.param(*c, bn, id=f"{'x'.join(map(str, c))}-bn{bn}") for c in cases for bn in widths_of(c)]


# ------------------------------------------------------------------------------------------------ a. statistics are exact sums
CONV_ROWVEC = [(32, 64, 64, 320, 320),   # bench level 0 (auto width: an overhanging last N tile)
               (48, 8, 8, 1280, 1280),   # two images per tile
               (3, 8, 8, 128, 320),      # an image count that does not fill a tile
               (2, 24, 40, 64, 320),     # x overhang
               (5, 4, 8, 64, 640),       # four images per tile, the last tile 3 images short
               (2, 12, 12, 64, 320)]     # tile condition holds, hw % 32 != 0 (the plan uses the stand-alone kernel there)


@pytest.mark.parametrize("n,H,W,Cin,Cout,bn", _pad_params(CONV_ROWVEC, lambda c: _widths(c[4])))
def test_conv_rowvec_statistics(cuda, n, H, W, Cin, Cout, bn):
    """resnet conv1: conv3x3 + bias + time-embedding row vector, statistics in the epilogue (E_BIAS|E_ROWVEC|E_STATS)."""
    from diffuman4d_b200 import ops
    if bn == 0 and (n, H, W, Cout) == (32, 64, 64, 320):
        assert Cout % _auto_block_n(n * H * W, Cout) != 0, "the automatic width no longer overhangs N here"
    g = torch.Generator().manual_seed(100)
    x = _rand((n, H, W, Cin), 101)
    w = _rand((Cout, Cin, 3, 3), 102, std=(9 * Cin) ** -0.5)
    bias = (2.0 + 0.5 * torch.randn(Cout, generator=g)).cuda()     # a mean well away from zero
    ld = 4 * Cout + 1288                                           # temb_all + temb_off of the plan: large ld, column offset
    temb_all = _rand((n, ld), 103)
    off = 2 * Cout + 648
    rowvec = temb_all[:, off:off + Cout]
    ws = _stats_ws(n * Cout * 2)
    out = ops.conv3x3(x, ops.conv_weight_to_octi(w), bias, rowvec=rowvec, block_n=bn, stats=ws)
    _close(out, _conv_ref(x, w, bias) + rowvec.float()[:, None, None, :])
    _check_ws(ws, out, n, "conv+rowvec")
    _check_standalone_stats(out, n)


@pytest.mark.parametrize("n,H,W,C", [(32, 64, 64, 320), (48, 16, 16, 1280), (3, 24, 40, 320)])
def test_downsample_statistics(cuda, n, H, W, C):
    """Downsample2D: stride-2 conv (E_BIAS|E_STATS), output rows from every other input row."""
    from diffuman4d_b200 import ops
    g = torch.Generator().manual_seed(120)
    x = _rand((n, H, W, C), 121)
    w = _rand((C, C, 3, 3), 122, std=(9 * C) ** -0.5)
    bias = (2.0 + 0.5 * torch.randn(C, generator=g)).cuda()
    ws = _stats_ws(n * C * 2)
    out = ops.conv3x3_stride2(x, ops.conv_weight_to_octi(w), bias, stats=ws)
    _close(out, _conv_ref(x, w, bias, stride=2))
    _check_ws(ws, out, n, "stride-2 conv")
    _check_standalone_stats(out, n)


@pytest.mark.parametrize("n,H,W,C", [(32, 32, 32, 640), (48, 8, 8, 1280), (3, 4, 8, 1280)])
def test_upsample_statistics(cuda, n, H, W, C):
    """Upsample2D: the four sub-pixel phases in one launch (kind 3, E_BIAS|E_STATS)."""
    from diffuman4d_b200 import ops
    g = torch.Generator().manual_seed(130)
    x = _rand((n, H, W, C), 131)
    w = _rand((C, C, 3, 3), 132, std=(9 * C) ** -0.5)
    bias = (2.0 + 0.5 * torch.randn(C, generator=g)).cuda()
    ws = _stats_ws(n * C * 2)
    out = ops.upsample2x_conv3x3(x, w, bias, stats=ws)
    _close(out, _conv_ref(x, w, bias, up=True))
    _check_ws(ws, out, n, "upsample conv")
    _check_standalone_stats(out, n)


GEMM_STATS = [(8192, 320, 320, 4096),    # proj_out at level 0 of a 64x64 latent, two images
              (3072, 1280, 1280, 64),    # 48 images of 8x8
              (480, 640, 640, 96),       # 96 rows per image: 128-row tiles straddle images, the last M tile is ragged
              (8192, 320, 192, 4096)]    # conv_in (K = 192)


@pytest.mark.parametrize("M,N,K,rows,bn", _pad_params(GEMM_STATS, lambda c: _widths(c[1])))
def test_gemm_residual_statistics(cuda, M, N, K, rows, bn):
    """transformer proj_out / conv_in: plain GEMM + bias + residual, statistics in the epilogue (E_BIAS|E_RES|E_STATS)."""
    from diffuman4d_b200 import ops
    g = torch.Generator().manual_seed(140)
    a, w = _rand((M, K), 141), _rand((N, K), 142, std=K ** -0.5)
    bias = (2.0 + 0.5 * torch.randn(N, generator=g)).cuda()
    res = _rand((M, N), 143)
    n_img = M // rows
    ws = _stats_ws(n_img * N * 2)
    out = ops.gemm(a, w, bias, residual=res, block_n=bn, stats=ws, stats_rows=rows)
    _close(out, a.float() @ w.float().t() + bias + res.float())
    _check_ws(ws, out, n_img, "GEMM+residual")
    _check_standalone_stats(out, n_img)


def test_statistics_rejections(cuda):
    """Launches whose statistics cannot be exact are refused as argument errors, before anything is written."""
    from diffuman4d_b200 import ops
    x, w = _rand((256, 64), 150), _rand((128, 64), 151)
    b = torch.zeros(128, device="cuda")
    ws = _stats_ws(2 * 128 * 2)
    wi, bi = ops.interleave_geglu(w, b)
    with pytest.raises(ValueError, match="statistics"):
        ops.gemm(x, wi, bi, geglu=True, stats=ws, stats_rows=128)
    with pytest.raises(ValueError, match="rows-per-image % 32"):
        ops.gemm(x, w, b, stats=ws, stats_rows=48)
    with pytest.raises(ValueError, match="M % rows-per-image"):
        ops.gemm(x[:200], w, b, stats=ws, stats_rows=64)       # rows past the last whole image would overrun the workspace
    with pytest.raises(ValueError, match="stats needs"):
        ops.gemm(x, w, b, stats=_stats_ws(8)[:8], stats_rows=128)
    xc, wc = _rand((2, 4, 4, 64), 152), _rand((64, 64, 3, 3), 153)
    with pytest.raises(ValueError, match="32-row warps"):      # 16 pixels per image: a warp's rows span two images
        ops.conv3x3(xc, ops.conv_weight_to_octi(wc), stats=ws)
    with pytest.raises(ValueError, match="32-row warps"):
        ops.conv3x3_stride2(_rand((2, 8, 8, 64), 154), ops.conv_weight_to_octi(wc), stats=ws)
    with pytest.raises(ValueError, match="32-row warps"):
        ops.upsample2x_conv3x3(xc, wc, stats=ws)
    assert (ws[2 * 128 * 2:] == SENT64).all() and (ws[:2 * 128 * 2] == 0).all()


# ------------------------------------------------------------------------------------------------ b. one format
@pytest.mark.parametrize("n,hw,C1,C2", [(3, 4, 64, 0), (2, 16, 2560, 0), (4, 36, 1280, 1280), (5, 100, 320, 640),
                                        (2, 100, 2560, 0), (1, 4096, 320, 0)])
def test_standalone_statistics(cuda, n, hw, C1, C2):
    """gn_stats_kernel with partial 16-pixel groups (hw 4, 36, 100), up to 2560 channels, and a second source whose
    statistics follow the first's in d4d_op_groupnorm's workspace."""
    from diffuman4d_b200 import ops
    x1 = _rand((n, hw, C1), 160, std=1.5, mean=2.0)
    x2 = None if C2 == 0 else _rand((n, hw, C2), 161, std=0.7, mean=-1.0)
    C = C1 + C2
    ws = _stats_ws(n * C * 2)
    ops.groupnorm(x1, torch.ones(C, device="cuda"), torch.zeros(C, device="cuda"), 32, 1e-5, True, x2=x2, stats=ws)
    w1 = n * C1 * 2
    assert (ws[n * C * 2:] == SENT64).all(), "statistics written past [n_img][C1 + C2][2]"
    _check_stats(ws[:w1], x1, n, "source 1")
    if x2 is not None:
        _check_stats(ws[w1:n * C * 2], x2, n, "source 2")


# ------------------------------------------------------------------------------------------------ c. GroupNorm apply vs fp64
def _gn_edge_input(n, hw, C, cpg, seed):
    """Group g follows profile g % 5: 0 ordinary (mean 0.5, sd 1); 1 mean of 64 sd (32, sd 0.5); 2 sd 1e-3 (mean 1e-3);
    3 exactly constant (3.0); 4 mean 384, sd 0.6, which bf16 stores as 382 / 384 / 386: ~600 stored sd from zero, where
    E[x^2] - mean^2 in fp32 loses the variance."""
    g = torch.Generator().manual_seed(seed)
    prof = (torch.arange(C) // cpg) % 5
    mu = torch.tensor([0.5, 32.0, 1e-3, 3.0, 384.0])[prof] + (prof == 0) * 0.3 * torch.randn(C, generator=g)
    sd = torch.tensor([1.0, 0.5, 1e-3, 0.0, 0.6])[prof]
    return (mu + sd * torch.randn(n, hw, C, generator=g)).to(torch.bfloat16).cuda()


def _gn_ref64(x, groups, gamma, beta, eps, silu, st):
    """fp64 GroupNorm(+SiLU) of x [n, hw, C] and the allowance beyond one bf16 ulp:
    * 2^-20 (|x - mean| + |mean|) |gamma| rstd: the fp32 affine of the apply kernel;
    * |x - mean| |gamma| |rstd_st - rstd| + |gamma| rstd_st |mean_st - mean|: what the apply inherits from the statistics
      it reads (st [n, C, 2], whose own error test_standalone_statistics bounds).  The format resolves the sum of squares
      to 2^-24 per 16-pixel partial; for a group with sd 1e-3 that is up to ~1e-3 of its variance, more than one bf16 ulp
      of outputs near zero, where the ulp is 2^-15.  mean_st and rstd_st are evaluated in fp64 from the integer sums.
    Both terms x1.1 through SiLU, whose slope is below 1.1."""
    n, hw, C = x.shape
    cpg = C // groups
    xd = x.double().view(n, hw, groups, cpg)
    mu = xd.mean(dim=(1, 3), keepdim=True)
    var = ((xd - mu) ** 2).mean(dim=(1, 3), keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    gs = st.view(n, groups, cpg, 2).sum(2)                       # int64 group totals, as the kernel forms them
    mu_st = (gs[..., 0].double() * 2.0 ** -28 / (hw * cpg)).view(n, 1, groups, 1)
    var_st = (gs[..., 1].double() * 2.0 ** -24 / (hw * cpg)).view(n, 1, groups, 1) - mu_st ** 2
    rstd_st = 1.0 / torch.sqrt(var_st.clamp_min(0) + eps)
    gm, bt = gamma.double().view(1, 1, groups, cpg), beta.double().view(1, 1, groups, cpg)
    y = (xd - mu) * rstd * gm + bt
    slack = gm.abs() * (2.0 ** -20 * ((xd - mu).abs() + mu.abs()) * rstd
                        + (xd - mu).abs() * (rstd_st - rstd).abs() + rstd_st * (mu_st - mu).abs())
    if silu:
        y, slack = F.silu(y), 1.1 * slack
    return y.view(n, hw, C), slack.view(n, hw, C)


@pytest.mark.parametrize("n,hw,C1,C2,silu,eps", [
    (2, 16384, 320, 0, True, 1e-5),     # 128x128 latent, level 0: 10 channels per group
    (48, 64, 1280, 0, False, 1e-6),     # 48 images of 8x8: 40 channels per group
    (2, 1024, 640, 0, True, 1e-6),      # 20 channels per group
    (3, 256, 2560, 0, False, 1e-5),     # 80 channels per group
    (2, 1024, 328, 312, True, 1e-5),    # virtual concat splits group 16 (20 channels per group)
    (2, 4096, 640, 320, False, 1e-6),   # up-path concat 640 | 320: 30 channels per group, groups split
    (48, 64, 1280, 640, True, 1e-5),    # up-path concat 1280 | 640: 60 channels per group, groups split
])
def test_groupnorm_apply_edges(cuda, n, hw, C1, C2, silu, eps):
    """Every case holds groups of all five _gn_edge_input profiles."""
    from diffuman4d_b200 import ops
    C, groups = C1 + C2, 32
    x = _gn_edge_input(n, hw, C, C // groups, 170)
    g = torch.Generator().manual_seed(171)
    gamma = (1 + 0.3 * torch.randn(C, generator=g)).cuda()
    beta = (0.2 * torch.randn(C, generator=g)).cuda()
    x1 = x[..., :C1].contiguous()
    x2 = None if C2 == 0 else x[..., C1:].contiguous()
    ws = _stats_ws(n * C * 2)
    out = ops.groupnorm(x1, gamma, beta, groups, eps, silu, x2=x2, stats=ws).double()
    w1 = n * C1 * 2
    st = ws[:w1].view(n, C1, 2) if x2 is None else torch.cat([ws[:w1].view(n, C1, 2), ws[w1:n * C * 2].view(n, C2, 2)], 1)
    _check_stats(st, x, n, "GroupNorm statistics")
    ref, slack = _gn_ref64(x, groups, gamma, beta, eps, silu, st)
    bound = _bf16_ulp(torch.maximum(out.abs(), ref.abs()).clamp_min(2.0 ** -8)) + slack
    err = (out - ref).abs()
    bad = err > bound
    if bad.any():
        grp = (bad.nonzero()[:, 2] // (C // groups)).unique().tolist()
        raise AssertionError(f"{int(bad.sum())} / {bad.numel()} beyond the bound (max {(err / bound).max().item():.3g} x), "
                             f"groups {grp[:8]} (profiles {[k % 5 for k in grp[:8]]})")


# ------------------------------------------------------------------------------------------------ d. guard bands, poisoned slack
def _gemm_raw(A, lda, K1, W, M, N, out, ldo, A2=None, lda2=0, K2=0, bias=None, residual=None, ld_res=0, geglu=0, block_n=0):
    from diffuman4d_b200._lib import check, lib
    p = lambda t: None if t is None else t.data_ptr()
    check(lib().d4d_op_gemm(p(A), lda, K1, p(A2), lda2, K2, p(W), M, N, p(bias), None, 0, 0, p(residual), ld_res, p(out),
                            ldo, geglu, 0, 1.0, block_n, None, 0, _stream()), "d4d_op_gemm")


def _nan_slack(M, K, ld, seed):
    """[M, ld] bf16 whose first K columns are data and whose slack is NaN; returns (buffer, data view)."""
    buf = torch.full((M, ld), float("nan"), dtype=torch.bfloat16, device="cuda")
    buf[:, :K] = _rand((M, K), seed)
    return buf, buf[:, :K]


@pytest.mark.parametrize("K1,K2,bn", [(40, 0, 0), (72, 0, 64), (200, 0, 0), (64, 40, 0), (128, 72, 64), (192, 200, 0)])
def test_gemm_guard_and_nan_slack(cuda, K1, K2, bn):
    """K not a multiple of 64 (the ABI accepts K % 8 == 0), strided A / A2 whose lda slack holds NaN, output with guard
    columns (ldo > N) and guard rows past a ragged M."""
    M, N, ldo = 333, 192, 232
    A, a = _nan_slack(M, K1, K1 + 24, 180)
    A2, a2 = (None, None) if K2 == 0 else _nan_slack(M, K2, K2 + 40, 181)
    w = _rand((N, K1 + K2), 182, std=(K1 + K2) ** -0.5)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(183)).cuda()
    out = _guarded(M, N, ldo, 130)
    _gemm_raw(A, A.stride(0), K1, w, M, N, out, ldo, A2=A2, lda2=0 if A2 is None else A2.stride(0), K2=K2, bias=bias,
              block_n=bn)
    src = a.float() if a2 is None else torch.cat([a, a2], 1).float()
    _close(out[:M, :N], src @ w.float().t() + bias)
    _check_guard(out, M, N, "GEMM")


@pytest.mark.parametrize("M,N,bn", [(333, 320, 0), (333, 320, 64), (200, 1280, 256), (77, 48, 48)])
def test_gemm_residual_guard(cuda, M, N, bn):
    """bias + residual epilogue (strided residual): guard columns and rows stay untouched, including past an
    overhanging last N tile."""
    K, ldo, ld_res = 128, N + 40, N + 24
    a, w = _rand((M, K), 190), _rand((N, K), 191, std=K ** -0.5)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(192)).cuda()
    res_buf = _rand((M, ld_res), 193)
    out = _guarded(M, N, ldo, 140)
    _gemm_raw(a, K, K, w, M, N, out, ldo, bias=bias, residual=res_buf, ld_res=ld_res, block_n=bn)
    _close(out[:M, :N], a.float() @ w.float().t() + bias + res_buf[:, :N].float())
    _check_guard(out, M, N, "GEMM+residual")


@pytest.mark.parametrize("C,bn", [(64, 0), (320, 0), (320, 32)])
def test_gemm_geglu_guard(cuda, C, bn):
    from diffuman4d_b200 import ops
    M, ldo = 333, 4 * C + 56
    x = _rand((M, C), 200)
    w = _rand((8 * C, C), 201, std=C ** -0.5)
    b = torch.randn(8 * C, generator=torch.Generator().manual_seed(202)).cuda()
    wi, bi = ops.interleave_geglu(w, b)
    out = _guarded(M, 4 * C, ldo, 130)
    _gemm_raw(x, C, C, wi, M, 8 * C, out, ldo, bias=bi, geglu=1, block_n=bn)
    y = x.float() @ w.float().t() + b
    ya, yg = y.chunk(2, dim=-1)
    _close(out[:M, :4 * C], ya * F.gelu(yg))
    _check_guard(out, M, 4 * C, "GEGLU")


@pytest.mark.parametrize("kind", ["conv3x3", "stride2", "upsample", "conv3x3_groupnorm"])
@pytest.mark.parametrize("n,H,W", [(3, 12, 8), (5, 4, 8), (3, 20, 24)])
def test_conv_guard(cuda, kind, n, H, W):
    """Output grids whose last tile overhangs in y and in images, written into a buffer with a trailing guard of more
    than one tile; statistics workspaces with guard words."""
    from diffuman4d_b200 import ops
    from diffuman4d_b200._lib import check, lib
    Cin, Cout = 64, 128
    if kind == "stride2":
        H, W = 2 * H, 2 * W                       # the OUTPUT grid is (H, W) in every kind
    x = _rand((n, H, W, Cin), 210)
    w = _rand((Cout, Cin, 3, 3), 211, std=(9 * Cin) ** -0.5)
    bias = (1.0 + torch.randn(Cout, generator=torch.Generator().manual_seed(212))).cuda()
    if kind == "stride2":
        Ho, Wo = H // 2, W // 2
    elif kind == "upsample":
        Ho, Wo = 2 * H, 2 * W
    else:
        Ho, Wo = H, W
    rows = n * Ho * Wo
    out = _guarded(rows, Cout, Cout, 3 * 128)
    stats_ok = (Ho * Wo) % 32 == 0 if kind != "upsample" else (H * W) % 32 == 0
    ws = _stats_ws(n * Cout * 2) if stats_ok else None
    p = lambda t: None if t is None else t.data_ptr()
    if kind == "conv3x3":
        res = _rand((n, H, W, Cout), 213)
        check(lib().d4d_op_conv3x3(p(x), n, H, W, Cin, p(ops.conv_weight_to_octi(w)), Cout, p(bias), None, 0, p(res), 0,
                                   p(out), 0, p(ws), _stream()))
        ref = _conv_ref(x, w, bias) + res.float()
    elif kind == "stride2":
        check(lib().d4d_op_conv_resample(p(x), n, H, W, Cin, p(ops.conv_weight_to_octi(w)), Cout, p(bias), 1, 0, 0, p(out),
                                         p(ws), _stream()))
        ref = _conv_ref(x, w, bias, stride=2)
    elif kind == "upsample":
        wp = torch.stack(ops.upsample_phase_weights(w)).contiguous()
        check(lib().d4d_op_conv_resample(p(x), n, H, W, Cin, p(wp), Cout, p(bias), 3, 0, 0, p(out), p(ws), _stream()))
        ref = _conv_ref(x, w, bias, up=True)
    else:
        if ws is None:
            pytest.skip("conv3x3_groupnorm needs H*W % 32 == 0")
        gn = _guarded(rows, Cout, Cout, 3 * 128)
        gamma = torch.ones(Cout, device="cuda")
        beta = torch.zeros(Cout, device="cuda")
        check(lib().d4d_op_conv3x3_groupnorm(p(x), n, H, W, Cin, p(ops.conv_weight_to_octi(w)), Cout, p(bias), None, 32,
                                             1e-5, p(gamma), p(beta), 1, p(out), p(gn), p(ws), _stream()))
        ref = _conv_ref(x, w, bias)
        _check_guard(gn, rows, Cout, "conv3x3_groupnorm (normalised)")
        conv = out[:rows].view(n, Ho, Wo, Cout)
        gref = F.silu(F.group_norm(conv.float().permute(0, 3, 1, 2), 32, gamma, beta, 1e-5)).permute(0, 2, 3, 1)
        _close(gn[:rows].view(n, Ho, Wo, Cout), gref)
    _close(out[:rows].view(n, Ho, Wo, Cout), ref)
    _check_guard(out, rows, Cout, kind)
    if ws is not None:
        _check_ws(ws, out[:rows], n, kind)


@pytest.mark.parametrize("batch,seq,heads,d", [(2, 200, 2, 64), (3, 100, 1, 128), (1, 330, 2, 192)])
def test_attention_guard(cuda, batch, seq, heads, d):
    """Output with guard columns (ld_out > heads * d) and guard rows past batch * seq; seq is not a multiple of the
    128-row query tile."""
    from diffuman4d_b200._lib import check, lib
    C = heads * d
    qkv = _rand((batch * seq, 3 * C), 220)
    ld_out = C + 72
    out = _guarded(batch * seq, C, ld_out, 128)
    base = qkv.data_ptr()
    check(lib().d4d_op_attention(base, base + 2 * C, base + 4 * C, 3 * C, out.data_ptr(), ld_out, batch, seq, heads, d,
                                 d ** -0.5, 0, 0, _stream()))
    q, k, v = qkv.float().view(batch, seq, 3, heads, d).permute(2, 0, 3, 1, 4)
    ref = F.scaled_dot_product_attention(q, k, v).permute(0, 2, 1, 3).reshape(batch * seq, C)
    _close(out[:batch * seq, :C], ref, rtol=1e-2, afrac=5e-3)
    _check_guard(out, batch * seq, C, "attention")


@pytest.mark.parametrize("n,hw,C1,C2", [(3, 100, 320, 0), (2, 36, 640, 320), (48, 64, 1280, 0)])
def test_groupnorm_guard(cuda, n, hw, C1, C2):
    from diffuman4d_b200._lib import check, lib
    C = C1 + C2
    x1 = _rand((n, hw, C1), 230, mean=1.0)
    x2 = None if C2 == 0 else _rand((n, hw, C2), 231, mean=-0.5)
    gamma = (1 + 0.2 * torch.randn(C, generator=torch.Generator().manual_seed(232))).cuda()
    beta = torch.zeros(C, device="cuda")
    out = _guarded(n * hw, C, C, 64)
    ws = _stats_ws(n * C * 2)
    check(lib().d4d_op_groupnorm(x1.data_ptr(), C1, None if x2 is None else x2.data_ptr(), C2, n, hw, 32, 1e-5,
                                 gamma.data_ptr(), beta.data_ptr(), 1, out.data_ptr(), ws.data_ptr(), _stream()))
    xc = x1 if x2 is None else torch.cat([x1, x2], 2)
    ref = F.silu(F.group_norm(xc.float().permute(0, 2, 1), 32, gamma, beta, 1e-5)).permute(0, 2, 1)
    _close(out[:n * hw].view(n, hw, C), ref)
    _check_guard(out, n * hw, C, "GroupNorm")
    assert (ws[n * C * 2:] == SENT64).all()


@pytest.mark.parametrize("rows,C", [(77, 1280), (100, 64), (333, 320)])
def test_layernorm_guard(cuda, rows, C):
    from diffuman4d_b200._lib import check, lib
    x = _rand((rows, C), 240, std=2.0, mean=0.5)
    gamma = (1 + 0.2 * torch.randn(C, generator=torch.Generator().manual_seed(241))).cuda()
    beta = (0.1 * torch.randn(C, generator=torch.Generator().manual_seed(242))).cuda()
    out = _guarded(rows, C, C, 16)
    check(lib().d4d_op_layernorm(x.data_ptr(), rows, C, 1e-5, gamma.data_ptr(), beta.data_ptr(), out.data_ptr(), _stream()))
    _close(out[:rows], F.layer_norm(x.float(), (C,), gamma, beta, 1e-5))
    _check_guard(out, rows, C, "LayerNorm")


# ------------------------------------------------------------------------------------------------ attention key census
def census_v(rows, heads, D, pattern, device="cuda"):
    """V [rows, heads*D] of zeros and ones.  pattern 0: V[j, h*D + c] = 1 iff (j // 64 + h) % D == c (which key tile);
    pattern 1: iff j % 64 == c (which key inside its tile).  j is the row of the K/V matrix, so batch entries differ."""
    j = torch.arange(rows)[:, None]
    c = torch.arange(D)[None, :]
    cols = [((j // 64 + h) % D == c) if pattern == 0 else (j % 64 == c) for h in range(heads)]
    return torch.cat(cols, 1).to(torch.bfloat16).to(device)


def census_misses(out, v, batch, seq, seq_kv):
    """Entries of out [batch*seq, C] more than one bf16 ulp from the census: with K = 0, every query row of batch entry
    b holds the mean of that entry's rows of v [batch*seq_kv, C]."""
    C = v.shape[1]
    ref = v.double().view(batch, seq_kv, C).mean(1)[:, None, :].expand(batch, seq, C).reshape(batch * seq, C)
    out = out.double()
    ulp = _bf16_ulp(torch.maximum(out.abs(), ref.abs()).clamp_min(2.0 ** -126))
    return int(((out - ref).abs() > ulp).sum())


CENSUS = ([(1 if s > 200 else 2, s, s, 2, d) for s in (200, 4096, 8192) for d in (64, 128, 192)]
          + [(2, 256, 1024, 5, 64),      # frame-sharded: 4 frames of 256 tokens gathered, one local
             (2, 512, 2048, 2, 128),
             (2, 200, 520, 2, 128),      # batch > 1, seq_kv % 64 != 0
             (3, 100, 300, 1, 192),
             (3, 130, 130, 2, 64),       # same matrix, batch > 1, seq_kv % 64 != 0
             # the plan's 3-D sequences: W16@64^2 level 1 (SD-2.1 and padded head_dim 80), W24@64^2, W16@128^2
             (2, 16384, 16384, 10, 64),
             (2, 16384, 16384, 8, 128),
             (2, 24576, 24576, 10, 64),
             (2, 65536, 65536, 10, 64),
             # W16@64^2 level 1 frame-sharded over 2, 4 and 8 ranks: one rank's queries, all 16 frames' keys
             (2, 8192, 16384, 10, 64),
             (2, 4096, 16384, 10, 64),
             (2, 2048, 16384, 10, 64),
             # seq_kv % 64 != 0 past 8192 keys: separate K/V matrix (40 keys in the last tile), same matrix (4 keys)
             (2, 4100, 12328, 2, 128),
             (2, 8260, 8260, 1, 192)])


@pytest.mark.parametrize("pattern", [0, 1])
@pytest.mark.parametrize("batch,seq,seq_kv,heads,D", CENSUS)
def test_attention_key_census(cuda, batch, seq, seq_kv, heads, D, pattern):
    """K = 0 makes every softmax weight exactly 1, so output column (h, c) of every query row of batch entry b is the
    number of that entry's keys whose V is 1 there, over seq_kv.  A dropped, duplicated or wrongly masked key tile, or
    a key read from another batch entry or another head's columns, changes a count."""
    from diffuman4d_b200 import ops
    C = heads * D
    q = _rand((batch * seq, C), 250)
    v = census_v(batch * seq_kv, heads, D, pattern)
    kv_zero = torch.zeros(batch * seq_kv, C, dtype=torch.bfloat16, device="cuda")
    if seq_kv == seq:
        out = ops.attention(torch.cat([q, kv_zero, v], 1), batch, seq, heads, D, D ** -0.5)
    else:
        # queries from the QKV matrix, whose own K / V columns are NaN and must not be read; K / V from the gathered
        # [batch * seq_kv, 2C] matrix (ld_kv = 2C)
        nan = torch.full((batch * seq, 2 * C), float("nan"), dtype=torch.bfloat16, device="cuda")
        out = ops.attention(torch.cat([q, nan], 1), batch, seq, heads, D, D ** -0.5, kv=torch.cat([kv_zero, v], 1))
    bad = census_misses(out, v, batch, seq, seq_kv)
    assert bad == 0, f"{bad} / {out.numel()} entries beyond one ulp of the census"
