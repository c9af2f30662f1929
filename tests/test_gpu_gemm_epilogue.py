"""The staged GEMM epilogue (output tile through shared memory, TMA stores, residual by TMA) and the 160 / 192 tile widths.

Values against fp32 torch references at the tolerance of test_gpu_ops.py; GroupNorm statistics to the bound of
test_gpu_kernel_edges.py; sentinel guard bands around every output of the TMA-store path (ragged M, an overhanging last N
tile, ldo > N); and launches with many tiles per CTA, which reuse the staging slabs and prefetch the next residual tile.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SENT16 = 0x7FA5


def _rand(shape, seed, std=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * std).to(torch.bfloat16).cuda()


def _close(out, ref, rtol=8e-3, afrac=2e-3):
    ref, out = ref.float(), out.float()
    assert out.shape == ref.shape, (out.shape, ref.shape)
    assert torch.isfinite(out).all(), "non-finite kernel output"
    scale = ref.abs().max().item() + 1e-12
    err = (out - ref).abs()
    bad = err > rtol * ref.abs() + afrac * scale
    assert not bad.any(), f"max err {err.max().item():.4g} (scale {scale:.4g}), {int(bad.sum())} / {bad.numel()} out of tolerance"


def _check_stats(st, y, n_img):
    C = y.shape[-1]
    y = y.reshape(n_img, -1, C).double()
    hw = y.shape[1]
    st = st.view(n_img, C, 2).double()
    es = (st[..., 0] * 2.0 ** -28 - y.sum(1)).abs()
    eq = (st[..., 1] * 2.0 ** -24 - (y * y).sum(1)).abs()
    assert (es <= 2.0 ** -20 * y.abs().sum(1) + hw * 2.0 ** -28).all(), "sums"
    assert (eq <= 2.0 ** -20 * (y * y).sum(1) + hw * 2.0 ** -24).all(), "sums of squares"


def _gemm_raw(A, W, M, N, out, ldo, bias=None, residual=None, ld_res=0, geglu=0, block_n=0, a2=None):
    """d4d_op_gemm on caller-owned buffers (arbitrary ldo / ld_res, output may alias the residual)."""
    from diffuman4d_b200._lib import check, lib
    p = lambda t: None if t is None else t.data_ptr()
    K1, K2 = A.shape[1], 0 if a2 is None else a2.shape[1]
    check(lib().d4d_op_gemm(p(A), A.stride(0), K1, p(a2), 0 if a2 is None else a2.stride(0), K2, p(W), M, N, p(bias),
                            None, 0, 0, p(residual), ld_res, p(out), ldo, geglu, 0, 1.0, block_n, None, 0,
                            torch.cuda.current_stream().cuda_stream), "d4d_op_gemm")


# ------------------------------------------------------------------------------------------------ widths 160 and 192
@pytest.mark.parametrize("bn", [160, 192])
def test_epilogue_variants_at_width(cuda, bn):
    from diffuman4d_b200 import ops
    M, N, K, rpi = 1000, 2 * bn, 320, 250
    a, w = _rand((M, K), 1), _rand((N, K), 2, std=K ** -0.5)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(3)).cuda()
    rowvec = _rand((M // rpi, N), 4)
    res = _rand((M, N), 5)
    y = a.float() @ w.float().t()
    _close(ops.gemm(a, w, bias, block_n=bn), y + bias)
    _close(ops.gemm(a, w, None, block_n=bn), y)
    _close(ops.gemm(a, w, bias, residual=res, block_n=bn), y + bias + res.float())
    _close(ops.gemm(a, w, bias, rowvec=rowvec, rows_per_image=rpi, block_n=bn),
           y + bias + rowvec.float().repeat_interleave(rpi, 0))
    _close(ops.gemm(a, w, bias, act=1, out_scale=0.5, residual=res, block_n=bn), F.silu(y + bias) * 0.5 + res.float())
    a2 = _rand((M, 192), 6)
    w2 = _rand((N, K + 192), 7, std=(K + 192) ** -0.5)
    _close(ops.gemm(a, w2, bias, a2=a2, block_n=bn), torch.cat([a, a2], 1).float() @ w2.float().t() + bias)
    # in-place residual: the output overwrites the residual it reads
    buf = res.clone()
    _gemm_raw(a, w, M, N, buf, N, bias=bias, residual=buf, ld_res=N, block_n=bn)
    _close(buf, y + bias + res.float())


@pytest.mark.parametrize("bn", [160, 192, 0])
def test_geglu_at_width(cuda, bn):
    from diffuman4d_b200 import ops
    C, M = 240, 777
    x = _rand((M, C), 10)
    w = _rand((8 * C, C), 11, std=C ** -0.5)
    b = torch.randn(8 * C, generator=torch.Generator().manual_seed(12)).cuda()
    wi, bi = ops.interleave_geglu(w, b)
    g = x.float() @ w.float().t() + b
    h, gate = g.chunk(2, dim=-1)
    _close(ops.gemm(x, wi, bi, geglu=True, block_n=bn), h * F.gelu(gate))


@pytest.mark.parametrize("M,N,bn", [(4096 * 4, 320, 160), (1024 * 8, 640, 160), (64 * 64, 960, 192), (2048, 1280, 0)])
def test_statistics_at_width(cuda, M, N, bn):
    """proj_out: bias + residual + statistics (E_BIAS|E_RES|E_STATS) at the new widths, exact fixed-point sums."""
    from diffuman4d_b200 import ops
    n_img, K = 4, N
    a, w = _rand((M, K), 20), _rand((N, K), 21, std=K ** -0.5)
    bias = (2.0 + 0.5 * torch.randn(N, generator=torch.Generator().manual_seed(22))).cuda()
    res = _rand((M, N), 23)
    ws = torch.zeros(n_img * N * 2, dtype=torch.int64, device="cuda")
    out = ops.gemm(a, w, bias, residual=res, block_n=bn, stats=ws, stats_rows=M // n_img)
    _close(out, a.float() @ w.float().t() + bias + res.float())
    _check_stats(ws, out, n_img)


def test_conv_at_width_160(cuda):
    """Level-1 resnet conv (Cout 320): automatic width 160, conv1 and conv2 epilogues, exact statistics."""
    from diffuman4d_b200 import ops
    n, H, W, Cin, Cout = 3, 32, 32, 320, 320
    x = _rand((n, H, W, Cin), 30)
    wt = _rand((Cout, Cin, 3, 3), 31, std=(9 * Cin) ** -0.5)
    bias = (1.0 + torch.randn(Cout, generator=torch.Generator().manual_seed(32))).cuda()
    temb = _rand((n, Cout), 33)
    res = _rand((n, H, W, Cout), 34)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), bias, padding=1).permute(0, 2, 3, 1)
    for bn in (0, 160):
        ws = torch.zeros(n * Cout * 2, dtype=torch.int64, device="cuda")
        out = ops.conv3x3(x, ops.conv_weight_to_octi(wt), bias, rowvec=temb, block_n=bn, stats=ws)
        _close(out, ref + temb.float()[:, None, None, :])
        _check_stats(ws, out, n)
        ws.zero_()
        out = ops.conv3x3(x, ops.conv_weight_to_octi(wt), bias, residual=res, block_n=bn, stats=ws)
        _close(out, ref + res.float())
        _check_stats(ws, out, n)


# ------------------------------------------------------------------------------------------------ guard bands
def _guarded(rows, ld, guard_rows):
    return torch.full((rows + guard_rows, ld), SENT16, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def _check_guard(buf, rows, cols):
    bits = buf.view(torch.int16).clone()
    bits[:rows, :cols] = SENT16
    bad = bits != SENT16
    assert not bad.any(), f"{int(bad.sum())} bf16 words written outside the [{rows}, {cols}] output"


@pytest.mark.parametrize("M,N,bn", [(333, 320, 160), (333, 384, 192), (70, 512, 256), (200, 96, 96), (129, 336, 0),
                                    (16500, 336, 0), (9000, 1200, 0), (4000, 336, 0)])
def test_staged_store_guard(cuda, M, N, bn):
    """Ragged M, overhanging last N tiles (the automatic widths of 336 at M 129 / 4000 / 16500 are 64 / 128 / 192, of 1200
    at M 9000 it is 256), a width that is not a kernel width (96 on the 128 kernel, masked) and ldo > N: the TMA stores
    and the residual loads stay inside [M, N]."""
    K = 128
    a, w = _rand((M, K), 40), _rand((N, K), 41, std=K ** -0.5)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(42)).cuda()
    res_full = _rand((M + 3, N + 40), 43)
    ref = a.float() @ w.float().t() + bias
    ldo = N + 56
    out = _guarded(M, ldo, 130)
    _gemm_raw(a, w, M, N, out, ldo, bias=bias, block_n=bn)
    _close(out[:M, :N], ref)
    _check_guard(out, M, N)
    out = _guarded(M, ldo, 130)
    _gemm_raw(a, w, M, N, out, ldo, bias=bias, residual=res_full, ld_res=N + 40, block_n=bn)
    _close(out[:M, :N], ref + res_full[:M, :N].float())
    _check_guard(out, M, N)


@pytest.mark.parametrize("bn", [0, 256])
def test_staged_geglu_guard(cuda, bn):
    from diffuman4d_b200 import ops
    C, M = 320, 301
    x = _rand((M, C), 50)
    w = _rand((8 * C, C), 51, std=C ** -0.5)
    b = torch.randn(8 * C, generator=torch.Generator().manual_seed(52)).cuda()
    wi, bi = ops.interleave_geglu(w, b)
    g = x.float() @ w.float().t() + b
    h, gate = g.chunk(2, dim=-1)
    ldo = 4 * C + 64
    out = _guarded(M, ldo, 130)
    _gemm_raw(x, wi, M, 8 * C, out, ldo, bias=bi, geglu=1, block_n=bn)
    _close(out[:M, :4 * C], h * F.gelu(gate))
    _check_guard(out, M, 4 * C)


# ------------------------------------------------------------------------------------------------ persistent loop
@pytest.mark.parametrize("N,K,bn", [(320, 320, 0), (640, 2560, 160), (1280, 320, 256), (960, 320, 192)])
def test_persistent_tiles(cuda, N, K, bn):
    """M >> 132 x 128: every CTA walks many tiles, reusing its staging slabs and prefetching the next residual tile under
    the current tile's MMAs; the residual is also the output (in place)."""
    M = 132 * 128 * 6 + 64
    a, w = _rand((M, K), 60), _rand((N, K), 61, std=K ** -0.5)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(62)).cuda()
    res = _rand((M, N), 63)
    ref = a.float() @ w.float().t() + bias + res.float()
    buf = res.clone()
    _gemm_raw(a, w, M, N, buf, N, bias=bias, residual=buf, ld_res=N, block_n=bn)
    _close(buf, ref)
