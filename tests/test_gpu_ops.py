"""GPU parity tests of the individual sm_90a kernels, called through the C ABI (ctypes), against plain
torch fp32 references evaluated on the SAME bf16 inputs.

Tolerances (stated per the task contract): the kernels accumulate in fp32 and round ONCE to bf16, so the
only systematic error is the bf16 output rounding (2^-8 relative) plus fp32 summation-order noise:
  GEMM / conv / norms : |out - ref| <= 8e-3*|ref| + 2e-3*max|ref|
  attention           : |out - ref| <= 1e-2*|ref| + 5e-3*max|ref|   (P is rounded to bf16 before P.V, as in
                        every flash-attention implementation the reference dispatches to)
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _close(out, ref, rtol=8e-3, afrac=2e-3):
    ref = ref.float()
    out = out.float()
    assert out.shape == ref.shape, (out.shape, ref.shape)
    scale = ref.abs().max().item() + 1e-12
    err = (out - ref).abs()
    bound = rtol * ref.abs() + afrac * scale
    bad = (err > bound)
    assert not torch.isnan(out).any(), "NaN in kernel output"
    assert not bad.any(), f"max err {err.max().item():.4g} (scale {scale:.4g}), {int(bad.sum())} / {bad.numel()} out of tolerance"


def _rand(shape, seed, std=1.0, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * std).to(torch.bfloat16).to(device)


# ------------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("M,N,K", [(128, 64, 64), (256, 320, 320), (1000, 640, 320), (32, 1280, 320),
                                   (4096, 1920, 640), (384, 160, 2880), (8192, 1280, 1280), (128, 16, 64)])
def test_gemm_plain(cuda, M, N, K):
    from diffuman4d_b200 import ops
    a, w = _rand((M, K), 10), _rand((N, K), 11, std=K ** -0.5)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(12)).cuda()
    out = ops.gemm(a, w, bias)
    _close(out, a.float() @ w.float().t() + bias)


def test_gemm_epilogues(cuda):
    from diffuman4d_b200 import ops
    M, N, K, rpi = 1024, 640, 384, 256
    a, w = _rand((M, K), 20), _rand((N, K), 21, std=K ** -0.5)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(22)).cuda()
    rowvec = _rand((M // rpi, N + 64), 23)[:, 32:32 + N]          # strided view, 64-byte aligned offset
    res = _rand((M, N), 24)
    out = ops.gemm(a, w, bias, rowvec=rowvec, rows_per_image=rpi, residual=res)
    ref = a.float() @ w.float().t() + bias + rowvec.float().repeat_interleave(rpi, 0) + res.float()
    _close(out, ref)
    out = ops.gemm(a, w, bias, act=1, out_scale=2.0, residual=res)
    _close(out, F.silu(a.float() @ w.float().t() + bias) * 2.0 + res.float())
    out = ops.gemm(a, w, None)
    _close(out, a.float() @ w.float().t())


@pytest.mark.parametrize("M,N,K,bn", [(333, 240, 128, 240), (77, 48, 64, 48), (513, 400, 64, 80), (200, 96, 64, 32),
                                      (129, 320, 192, 160), (1, 16, 64, 16)])
def test_gemm_staged_epilogue_tails(cuda, M, N, K, bn):
    """Tile widths that are not a wgmma width (240, 48, 80, 32, 160, 16 columns run on a wider kernel with the extra
    columns masked), ragged M (rows past M must not be written) and the in-place residual."""
    from diffuman4d_b200 import ops
    a, w = _rand((M, K), 25), _rand((N, K), 26, std=K ** -0.5)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(27)).cuda()
    res = _rand((M, N), 28)
    ref = a.float() @ w.float().t() + bias
    _close(ops.gemm(a, w, bias, block_n=bn), ref)
    _close(ops.gemm(a, w, bias, residual=res, block_n=bn), ref + res.float())


def test_gemm_two_source(cuda):
    from diffuman4d_b200 import ops
    M, N, K1, K2 = 512, 320, 640, 320
    a1, a2 = _rand((M, K1), 30), _rand((M, K2), 31)
    w = _rand((N, K1 + K2), 32, std=(K1 + K2) ** -0.5)
    out = ops.gemm(a1, w, None, a2=a2)
    _close(out, torch.cat([a1, a2], 1).float() @ w.float().t())


@pytest.mark.parametrize("C", [64, 320])
def test_gemm_geglu(cuda, C):
    from diffuman4d_b200 import ops
    M = 640
    x = _rand((M, C), 40)
    w = _rand((8 * C, C), 41, std=C ** -0.5)
    b = torch.randn(8 * C, generator=torch.Generator().manual_seed(42)).cuda()
    wi, bi = ops.interleave_geglu(w, b)
    y = x.float() @ w.float().t() + b
    a, g = y.chunk(2, dim=-1)
    for bn in (0, 32, 256):   # automatic width, a width narrower than the kernel's (masked), the widest
        _close(ops.gemm(x, wi, bi, geglu=True, block_n=bn), a * F.gelu(g))


# ------------------------------------------------------------------------------------------------ conv
@pytest.mark.parametrize("n,H,W,Cin,Cout", [(2, 16, 16, 64, 64), (3, 8, 8, 128, 64), (1, 32, 32, 320, 320),
                                            (2, 24, 40, 64, 128), (5, 4, 4, 64, 64), (2, 64, 64, 64, 16)])
def test_conv3x3(cuda, n, H, W, Cin, Cout):
    from diffuman4d_b200 import ops
    x = _rand((n, H, W, Cin), 50)
    w = _rand((Cout, Cin, 3, 3), 51, std=(9 * Cin) ** -0.5)
    bias = torch.randn(Cout, generator=torch.Generator().manual_seed(52)).cuda()
    temb = _rand((n, Cout), 53)
    res = _rand((n, H, W, Cout), 54)
    out = ops.conv3x3(x, ops.conv_weight_to_octi(w), bias, rowvec=temb, residual=res)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1).permute(0, 2, 3, 1)
    ref = ref + temb.float()[:, None, None, :] + res.float()
    _close(out, ref)


# ------------------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("batch,seq,heads,d", [(1, 128, 1, 64), (2, 256, 3, 64), (1, 1024, 2, 64), (2, 200, 2, 64),
                                               (3, 64, 2, 64), (1, 4096, 5, 64), (2, 384, 2, 128), (1, 320, 1, 192)])
def test_attention(cuda, batch, seq, heads, d):
    from diffuman4d_b200 import ops
    C = heads * d
    qkv = _rand((batch * seq, 3 * C), 60)
    scale = 1.0 / math.sqrt(d)
    out = ops.attention(qkv, batch, seq, heads, d, scale)
    q, k, v = qkv.float().view(batch, seq, 3, heads, d).permute(2, 0, 3, 1, 4)
    ref = F.scaled_dot_product_attention(q, k, v).permute(0, 2, 1, 3).reshape(batch * seq, C)
    _close(out, ref, rtol=1e-2, afrac=5e-3)


def test_attention_sharp_softmax(cuda):
    """large logits: the running max grows from tile to tile, so O and the row sums are rescaled many times."""
    from diffuman4d_b200 import ops
    batch, seq, heads, d = 1, 512, 2, 64
    qkv = _rand((batch * seq, 3 * heads * d), 61, std=3.0)
    out = ops.attention(qkv, batch, seq, heads, d, 0.5)
    q, k, v = qkv.float().view(batch, seq, 3, heads, d).permute(2, 0, 3, 1, 4)
    ref = F.scaled_dot_product_attention(q, k, v, scale=0.5).permute(0, 2, 1, 3).reshape(batch * seq, heads * d)
    _close(out, ref, rtol=1e-2, afrac=5e-3)


# ------------------------------------------------------------------------------------------------ norms
@pytest.mark.parametrize("n,hw,C1,C2,silu,eps", [(2, 256, 64, 0, True, 1e-5), (3, 64, 320, 0, False, 1e-6),
                                                 (2, 1024, 640, 320, True, 1e-5), (2, 16, 1280, 1280, True, 1e-5),
                                                 (1, 4096, 320, 0, True, 1e-5), (2, 100, 1280, 640, True, 1e-5)])
def test_groupnorm(cuda, n, hw, C1, C2, silu, eps):
    from diffuman4d_b200 import ops
    g = torch.Generator().manual_seed(70)
    x1 = ((torch.randn(n, hw, C1, generator=g) * 1.5 + 3.0 * torch.randn(1, 1, C1, generator=g))).to(torch.bfloat16).cuda()
    x2 = None if C2 == 0 else (torch.randn(n, hw, C2, generator=g) * 0.7 - 1.0).to(torch.bfloat16).cuda()
    C = C1 + C2
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).cuda()
    beta = (0.1 * torch.randn(C, generator=g)).cuda()
    out = ops.groupnorm(x1, gamma, beta, 32, eps, silu, x2=x2)
    xc = x1 if x2 is None else torch.cat([x1, x2], dim=2)
    ref = F.group_norm(xc.float().permute(0, 2, 1), 32, gamma, beta, eps).permute(0, 2, 1)
    if silu:
        ref = F.silu(ref)
    _close(out, ref)


@pytest.mark.parametrize("n,H,W,Cin,Cout", [(2, 16, 16, 64, 64), (3, 8, 8, 320, 320), (2, 32, 32, 128, 128), (2, 16, 24, 64, 128),
                                            (1, 64, 64, 320, 320)])
def test_resampling_convs(cuda, n, H, W, Cin, Cout):
    """Downsample2D (3x3 stride 2 through a strided tensor map) and Upsample2D (nearest x2 + 3x3 as four sub-pixel phases)."""
    from diffuman4d_b200 import ops
    x = _rand((n, H, W, Cin), 91)
    w = _rand((Cout, Cin, 3, 3), 92, std=(9 * Cin) ** -0.5)
    bias = torch.randn(Cout, generator=torch.Generator().manual_seed(93)).cuda()
    xc = x.float().permute(0, 3, 1, 2)
    down = ops.conv3x3_stride2(x, ops.conv_weight_to_octi(w), bias)
    _close(down, F.conv2d(xc, w.float(), bias, stride=2, padding=1).permute(0, 2, 3, 1))
    ref = F.conv2d(F.interpolate(xc, scale_factor=2.0, mode="nearest"), w.float(), bias, padding=1).permute(0, 2, 3, 1)
    up = ops.upsample2x_conv3x3(x, w, bias)                                # all four phases in one launch (the UNet plan)
    _close(up, ref)
    assert torch.equal(up, ops.upsample2x_conv3x3(x, w, bias, single_launch=False))


@pytest.mark.parametrize("n,H,W,Cin,Cout,silu", [(2, 16, 16, 64, 64, True), (3, 8, 8, 320, 640, True), (2, 32, 32, 320, 320, False),
                                                 (2, 16, 24, 128, 256, True), (1, 64, 64, 320, 320, True)])
def test_conv3x3_fused_groupnorm_stats(cuda, n, H, W, Cin, Cout, silu):
    """conv epilogue accumulates per-(image, channel) sums; GroupNorm applies from them (the resnet pair of the UNet plan)."""
    from diffuman4d_b200 import ops
    g = torch.Generator().manual_seed(75)
    x = _rand((n, H, W, Cin), 71)
    w = _rand((Cout, Cin, 3, 3), 72, std=(9 * Cin) ** -0.5)
    bias = (torch.randn(Cout, generator=g) + 1.5).cuda()   # a mean well away from zero: E[x^2] - E[x]^2 must hold up
    res = _rand((n, H, W, Cout), 73)
    gamma = (1 + 0.2 * torch.randn(Cout, generator=g)).cuda()
    beta = (0.1 * torch.randn(Cout, generator=g)).cuda()
    conv_out, gn_out = ops.conv3x3_groupnorm(x, ops.conv_weight_to_octi(w), bias, gamma, beta, 32, 1e-5, silu, residual=res)
    ref_conv = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1).permute(0, 2, 3, 1) + res.float()
    _close(conv_out, ref_conv)
    # GroupNorm reference on the bf16 tensor the kernel actually stored (what the next layer of the reference sees)
    ref = F.group_norm(conv_out.float().permute(0, 3, 1, 2), 32, gamma, beta, 1e-5).permute(0, 2, 3, 1)
    if silu:
        ref = F.silu(ref)
    _close(gn_out, ref)


@pytest.mark.parametrize("rows,C", [(100, 64), (4096, 320), (1000, 640), (77, 1280)])
def test_layernorm(cuda, rows, C):
    from diffuman4d_b200 import ops
    g = torch.Generator().manual_seed(80)
    x = (torch.randn(rows, C, generator=g) * 2 + 0.5).to(torch.bfloat16).cuda()
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).cuda()
    beta = (0.1 * torch.randn(C, generator=g)).cuda()
    out = ops.layernorm(x, gamma, beta)
    _close(out, F.layer_norm(x.float(), (C,), gamma, beta, 1e-5))
