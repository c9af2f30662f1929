"""The pose encoder's own kernels against fp64 convolutions, layer by layer and through the weight loader.

The pose encoder runs at 8h x 8w per image, the largest spatial size of the network, and its first five layers are
hand-written kernels: conv_layers.0 on FMAs (pose_conv0_kernel, 4 pixels per thread, NCHW in, 4-channel NHWC out) and
conv_layers.2/4/6/8 on mma.sync (pose_conv_mma_kernel: 32-pixel warp tiles that straddle images, a stride-2 origin, a
hand-written pixel tail).  Through the whole UNet their signal is hard to see: with fan-in-scaled weights and 0.05
biases the skeleton-dependent part of the embedding shrinks ~4x per layer, so a one-pixel shift or a broken image border
stays under the whole-network drift tolerance.  This file checks them directly:

* Per layer vs fp64.  With S = sum |w x| + |b| over an output's receptive field (fp64), every element satisfies
      |out - ref| <= 1/2 ulp_bf16(max(|out|, |ref|)) + 2^-14 S,
  one output rounding plus worst-case fp32 accumulation of <= 288 products plus the __expf / __fdividef SiLU.
* Exact properties: conv_layers.0 writes +0.0 into the pad channel; conv_layers.2 ignores whatever the pad channel holds
  (its weights are zero); each image of a batched call is bit-identical to a call on that image alone.
* Guard bands of sentinel bf16 words before and after every output.
* End to end through the C++ weight loader: with conv_in zeroed, the conv_in debug tap IS the pose embedding, which must
  match an fp64 chain that rounds to bf16 where the plan stores an activation, and the fp32 oracle PoseEncoder.  One-ulp
  rounding flips compound over nine layers, so these bounds are 2^-6 max|ref| per element plus an rms bound (see the test).
"""
import contextlib
import ctypes as C
import gc
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SENT16 = 0x7FA5     # bf16 NaN bit pattern that no kernel produces
GUARD = 4096        # bf16 words of guard before and after an output (keeps 16-byte alignment)

# (Cin, Cout, k, stride) of conv_layers.2/4/6/8; Cin of conv_layers.2 is 3, read as 4-channel pixels
MMA_LAYERS = {1: (3, 16, 4, 2), 2: (16, 16, 3, 1), 3: (16, 32, 4, 2), 4: (32, 32, 3, 1)}


# ------------------------------------------------------------------------------------------------ helpers
@contextlib.contextmanager
def _no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _input(shape, seed, std=None):
    """Uniform [-1, 1] like skeleton images, or normal with `std` (reaches both SiLU tails), as bf16 on the GPU."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g) * std if std else torch.rand(shape, generator=g) * 2 - 1
    return x.to(torch.bfloat16).cuda()


def _weights(cout, cin, k, seed):
    """bf16-valued OIHW weights (std 1.7 / sqrt(fan_in): pre-activations of order 1) and an fp32 bias."""
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(cout, cin, k, k, generator=g) * 1.7 / math.sqrt(cin * k * k)).to(torch.bfloat16).cuda()
    b = (0.3 * torch.randn(cout, generator=g)).cuda()
    return w, b


def _ref64(x_nchw, w, b, stride):
    """fp64 conv (pad 1) + bias + SiLU of the same bf16 values, and S = sum |w x| + |b| per output (NCHW)."""
    xd, wd, bd = x_nchw.double(), w.double(), b.double()
    with _no_tf32():
        pre = F.conv2d(xd, wd, bd, stride=stride, padding=1)
        s = F.conv2d(xd.abs(), wd.abs(), bd.abs(), stride=stride, padding=1)
    return F.silu(pre), s


def _ulp(mag):
    return torch.exp2(torch.floor(torch.log2(mag)) - 7)


def _check_layer(out_nhwc, ref_nchw, s_nchw, what):
    cout = ref_nchw.shape[1]
    out = out_nhwc[..., :cout].double().permute(0, 3, 1, 2)
    assert out.shape == ref_nchw.shape, (out.shape, ref_nchw.shape)
    assert torch.isfinite(out).all(), f"{what}: non-finite output"
    bound = 0.5 * _ulp(torch.maximum(out.abs(), ref_nchw.abs())) + 2.0 ** -14 * s_nchw
    err = (out - ref_nchw).abs()
    bad = err > bound
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} / {bad.numel()} beyond the bound (max {(err / bound).max().item():.3g} x); "
                             f"first at [n, c, y, x] = {i}: out {out[tuple(i)].item():.6g} ref {ref_nchw[tuple(i)].item():.6g}")


def _nhwc4(x_nchw3):
    """[n, 3, H, W] -> [n, H, W, 4] with a zero pad channel (conv_layers.0's output layout)."""
    return F.pad(x_nchw3.permute(0, 2, 3, 1), (0, 1)).contiguous()


def _guarded_out(numel):
    """SENT16-filled buffer with GUARD words before and after a numel-word output; returns (buffer, output view)."""
    buf = torch.full((numel + 2 * GUARD,), SENT16, dtype=torch.int16, device="cuda")
    return buf, buf[GUARD:GUARD + numel].view(torch.bfloat16)


def _check_guard(buf, numel, what):
    bits = buf.view(torch.int16)
    ok = (bits[:GUARD] == SENT16).all() and (bits[GUARD + numel:] == SENT16).all()
    assert ok, f"{what}: {int((bits[:GUARD] != SENT16).sum() + (bits[GUARD + numel:] != SENT16).sum())} guard words written"


def _conv0_raw(x, wp, b, out):
    from diffuman4d_b200._lib import check, lib
    n, _, H, W = x.shape
    check(lib().d4d_op_pose_conv0(x.data_ptr(), n, H, W, wp.data_ptr(), b.data_ptr(), out.data_ptr(), _stream()))


def _conv_raw(x, wp, b, cout, k, s, out):
    from diffuman4d_b200._lib import check, lib
    n, H, W, cin = x.shape
    check(lib().d4d_op_pose_conv(x.data_ptr(), n, cin, H, W, wp.data_ptr(), b.data_ptr(), cout, k, s, out.data_ptr(),
                                 _stream()))


def _out_hw(H, W, k, s):
    return (H + 2 - k) // s + 1, (W + 2 - k) // s + 1


# ------------------------------------------------------------------------------------------------ a. conv_layers.0
CONV0 = [(2, 512, 512, None),   # the plan at 64x64 latents, CFG off, two images
         (1, 1024, 1024, None),  # 128x128 latents
         (3, 7, 5, None),        # W % 4 = 1
         (2, 9, 6, None),        # W % 4 = 2
         (1, 5, 11, None),       # W % 4 = 3
         (2, 1, 13, None),       # one row
         (3, 6, 1, None),        # one column
         (1, 1, 1, None),
         (4, 33, 30, 4.0)]       # std 4: both SiLU tails


@pytest.mark.parametrize("n,H,W,std", CONV0)
def test_pose_conv0_vs_fp64(cuda, n, H, W, std):
    from diffuman4d_b200 import ops
    x = _input((n, 3, H, W), 300 + H + W, std)
    w, b = _weights(3, 3, 3, 301)
    wp = ops.pose_conv_weights(w)
    buf, out = _guarded_out(n * H * W * 4)
    _conv0_raw(x, wp, b, out)
    _check_guard(buf, n * H * W * 4, "conv_layers.0")
    out = out.view(n, H, W, 4)
    assert (out[..., 3].view(torch.int16) == 0).all(), "pad channel is not +0.0"
    ref, s = _ref64(x, w, b, 1)
    _check_layer(out, ref, s, f"conv_layers.0 {n}x{H}x{W}")
    assert torch.equal(ops.pose_conv0(x, wp, b), out)
    for i in range(min(n, 3)):                           # a batched call computes each image as a call on it alone
        assert torch.equal(ops.pose_conv0(x[i:i + 1].contiguous(), wp, b)[0], out[i]), f"image {i}"


# ------------------------------------------------------------------------------------------------ b. conv_layers.2/4/6/8
MMA = ([(l, n, H, W, None) for l, (n, H, W) in [(1, (2, 512, 512)), (1, (1, 1024, 1024)), (2, (2, 256, 256)),
                                                 (2, (1, 512, 512)), (3, (2, 256, 256)), (3, (1, 512, 512)),
                                                 (4, (2, 128, 128)), (4, (1, 256, 256))]]    # the plan's shapes
       + [(l, 37, 10, 10, None) for l in (1, 2, 3, 4)]     # 25 / 100 pixels per image: warp tiles straddle images
       + [(l, 3, 11, 13, None) for l in (1, 2, 3, 4)]      # odd H and W; 90 / 143 output pixels
       + [(l, 2, 1, 7, None) for l in (2, 4)]              # one row
       + [(1, 5, 3, 3, None), (3, 4, 2, 5, None)]          # stride 2 on 1 x 1 and 1 x 2 outputs
       + [(l, 3, 18, 14, 4.0) for l in (1, 2, 3, 4)])      # std 4: both SiLU tails


def _mma_case(layer, n, H, W, std, seed):
    """Input NHWC (pad channel zero for conv_layers.2), OIHW weights, packed weights, bias."""
    from diffuman4d_b200 import ops
    cin, cout, k, s = MMA_LAYERS[layer]
    x = _input((n, cin, H, W), seed, std)
    xh = _nhwc4(x) if cin == 3 else x.permute(0, 2, 3, 1).contiguous()
    w, b = _weights(cout, cin, k, seed + 1)
    return x, xh, w, ops.pose_conv_weights(w), b


@pytest.mark.parametrize("layer,n,H,W,std", MMA)
def test_pose_conv_vs_fp64(cuda, layer, n, H, W, std):
    from diffuman4d_b200 import ops
    cin, cout, k, s = MMA_LAYERS[layer]
    x, xh, w, wp, b = _mma_case(layer, n, H, W, std, 310 + layer + H + W)
    Ho, Wo = _out_hw(H, W, k, s)
    numel = n * Ho * Wo * cout
    buf, out = _guarded_out(numel)
    _conv_raw(xh, wp, b, cout, k, s, out)
    _check_guard(buf, numel, f"conv_layers.{2 * layer}")
    out = out.view(n, Ho, Wo, cout)
    ref, sabs = _ref64(x, w, b, s)
    _check_layer(out, ref, sabs, f"conv_layers.{2 * layer} {n}x{H}x{W}")
    assert torch.equal(ops.pose_conv(xh, wp, b, k, s), out)
    for i in sorted({0, n // 2, n - 1}):                 # per-pixel accumulation order does not depend on the tile
        assert torch.equal(ops.pose_conv(xh[i:i + 1].contiguous(), wp, b, k, s)[0], out[i]), f"image {i}"


@pytest.mark.parametrize("n,H,W", [(2, 64, 64), (37, 10, 10)])
def test_pose_conv_pad_channel_is_ignored(cuda, n, H, W):
    """conv_layers.2 reads 4-channel pixels; finite garbage in channel 3 must not change a bit (zero pad weights)."""
    from diffuman4d_b200 import ops
    _, xh, _, wp, b = _mma_case(1, n, H, W, None, 330)
    clean = ops.pose_conv(xh, wp, b, 4, 2)
    g = torch.Generator().manual_seed(331)
    dirty = xh.clone()
    dirty[..., 3] = (torch.randn(n, H, W, generator=g) * 3e4).to(torch.bfloat16).cuda()
    assert torch.equal(ops.pose_conv(dirty, wp, b, 4, 2), clean)


def test_pose_conv_argument_errors(cuda):
    from diffuman4d_b200 import ops
    from diffuman4d_b200._lib import check, lib
    x = _input((1, 16, 8, 8), 340).permute(0, 2, 3, 1).contiguous()
    w, b = _weights(32, 16, 3, 341)
    wp = ops.pose_conv_weights(w)
    with pytest.raises(ValueError, match="unsupported layer 16->32 k3 s1"):
        ops.pose_conv(x, wp, b, 3, 1)
    with pytest.raises(ValueError, match="unsupported layer 16->32 k3 s2"):
        ops.pose_conv(x, wp, b, 3, 2)
    w16, b16 = _weights(16, 16, 4, 342)
    with pytest.raises(ValueError, match="unsupported layer 16->16 k4 s2"):
        ops.pose_conv(x, ops.pose_conv_weights(w16), b16, 4, 2)
    w2, b2 = _weights(16, 16, 3, 343)
    wp2 = ops.pose_conv_weights(w2)
    flat = torch.zeros(wp2.numel() + 8, dtype=torch.bfloat16, device="cuda")
    flat[4:4 + wp2.numel()] = wp2.flatten()
    out = torch.empty(1, 8, 8, 16, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError, match="16-byte aligned"):    # refused before anything is launched
        check(lib().d4d_op_pose_conv(x.data_ptr(), 1, 16, 8, 8, flat[4:].data_ptr(), b2.data_ptr(), 16, 3, 1,
                                     out.data_ptr(), _stream()))
    w0, b0 = _weights(3, 3, 3, 344)
    with pytest.raises(ValueError, match="empty pose conv"):     # the C entry point refuses an empty batch
        ops.pose_conv0(_input((0, 3, 8, 8), 345), ops.pose_conv_weights(w0), b0)
    with pytest.raises(ValueError, match="empty pose conv"):
        ops.pose_conv(x[:0], wp2, b2, 3, 1)


@pytest.mark.parametrize("H,W", [(1, 9), (9, 1)])
def test_pose_conv_refuses_kernel_larger_than_input(cuda, H, W):
    """A 4x4 kernel on a 1-row (1-column) input has no output pixel: 1 + 2 < 4.  C's truncating (1 + 2 - 4) / 2 + 1
    would still count one, so the entry point must refuse the shape.  The raw call gets a guarded buffer as large as
    that miscount, so a missing check shows as guard words or a missing error, not as a stray write."""
    from diffuman4d_b200 import ops
    from diffuman4d_b200._lib import check, lib
    n = 2
    _, xh, _, wp, b = _mma_case(1, n, H, W, None, 346)
    miscount = n * max((H - 2) // 2 + 1, 1) * max((W - 2) // 2 + 1, 1) * 16
    buf, out = _guarded_out(miscount)
    with pytest.raises(ValueError, match="kernel larger than the padded input"):
        check(lib().d4d_op_pose_conv(xh.data_ptr(), n, 4, H, W, wp.data_ptr(), b.data_ptr(), 16, 4, 2, out.data_ptr(),
                                     _stream()))
    torch.cuda.synchronize()
    _check_guard(buf, 0, "refused pose conv")
    with pytest.raises(ValueError, match="kernel larger than the padded input"):
        ops.pose_conv(xh, wp, b, 4, 2)


# ------------------------------------------------------------------------------------------------ c. through the loader
@pytest.fixture(scope="module")
def pose_model(cuda):
    """SD-2.1 UNet whose conv_in is zero (the conv_in tap is exactly the pose embedding: the GEMM adds it as the residual
    to 0) and whose pose convs carry the skeleton signal (std 1.7 / sqrt(fan_in), biases ~0.01).  Freed with the module."""
    from diffuman4d_b200.config import UNetConfig
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import POSE_SPEC, random_state_dict
    cfg = UNetConfig.sd21()
    sd = random_state_dict(cfg, seed=7)
    sd["conv_in.weight"].zero_()
    sd["conv_in.bias"].zero_()
    g = torch.Generator().manual_seed(350)
    for i, (ci, co, k) in enumerate(POSE_SPEC):
        p = f"pose_encoder.conv_layers.{2 * i}"
        sd[p + ".weight"] = (torch.randn(co, ci, k, k, generator=g) * 1.7 / math.sqrt(ci * k * k)).to(torch.bfloat16)
        sd[p + ".bias"] = (0.01 * torch.randn(co, generator=g)).to(torch.bfloat16)
    unet = B200MultiviewUNet(cfg, 0).load_state_dict(sd)
    yield cfg, sd, unet
    del unet
    gc.collect()
    torch.cuda.empty_cache()


def _conv_in_tap(unet, cfg, B, h, w, skel):
    from diffuman4d_b200._lib import check, lib
    g = torch.Generator().manual_seed(351)
    sample = torch.randn(B, cfg.in_channels, h, w, generator=g).to(torch.bfloat16).cuda()
    t = torch.randint(0, 1000, (B,), generator=g).cuda()
    dom = (C.c_int32 * 1)(0)
    name, dims = C.create_string_buffer(64), (C.c_int32 * 3)()
    out = torch.empty(B, cfg.block_out_channels[0], h, w, dtype=torch.bfloat16, device="cuda")
    check(lib().d4d_debug_tap(unet._h, sample.data_ptr(), t.data_ptr(), skel.data_ptr(), dom, 1, B, B, h, w, 0,
                              out.data_ptr(), name, dims, _stream()), "d4d_debug_tap")
    assert name.value == b"conv_in" and tuple(dims) == tuple(out.shape[1:])
    return out


def _chain64(sd, skel):
    """fp64 pose encoder on the bf16 weights, rounded to bf16 wherever the plan stores an activation: after each of the
    8 conv+SiLU layers and once after final_proj * scale."""
    from diffuman4d_b200.weights import POSE_SPEC
    from oracle.unet_oracle import PoseEncoder
    y = skel.double()
    with _no_tf32():
        for i, (ci, co, k) in enumerate(POSE_SPEC):
            p = f"pose_encoder.conv_layers.{2 * i}"
            s = PoseEncoder.SPEC[i][3]
            y = F.silu(F.conv2d(y, sd[p + ".weight"].cuda().double(), sd[p + ".bias"].cuda().double(), stride=s, padding=1))
            y = y.to(torch.bfloat16).double()
        y = F.conv2d(y, sd["pose_encoder.final_proj.weight"].cuda().double(), sd["pose_encoder.final_proj.bias"].cuda().double())
        return (y * sd["pose_encoder.scale"].double().item()).to(torch.bfloat16).double()


@pytest.mark.parametrize("B,h,w", [(4, 64, 64), (1, 128, 128)])
def test_pose_embedding_through_loader(pose_model, B, h, w):
    from oracle.unet_oracle import PoseEncoder
    cfg, sd, unet = pose_model
    g = torch.Generator().manual_seed(352 + h)
    skel = (torch.rand(B, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16).cuda()
    out = _conv_in_tap(unet, cfg, B, h, w, skel).double()
    ref = _chain64(sd, skel)
    # the test's power: most of the embedding varies with the skeleton, so a shift or a wrong image shows
    varying = ref - ref.mean(dim=(2, 3), keepdim=True)
    power = (varying.pow(2).mean() / ref.pow(2).mean()).sqrt().item()
    assert power >= 0.5, f"pixel-varying part is only {power:.3f} of the rms"
    assert torch.isfinite(out).all()
    # The chain rounds where the plan rounds, but fp32 and fp64 sums still round a few values the other way, and each
    # such one-ulp flip feeds every later layer.  By conv_layers.14 ~4% of the values differ, so ANY fp32-accumulating
    # implementation drifts from this chain by far more than 2 ulps: a CPU fp32 chain with the same rounding points is
    # 4.6x beyond 2 ulp + 2^-12 max|ref| at 16x16 latents, at 4.8e-3 max|ref| and 2e-3 rms, and the kernels measure
    # 4.8e-3 and 2.6e-3.  Hence 2 ulp + 2^-6 max|ref| per element and 2^-7 of the rms (~3x headroom each).  The loader
    # failures this test exists for (a permuted re-layout, a dropped scale) are errors of order max|ref|, as are a
    # shifted or wrong image.
    err = (out - ref).abs()
    ulp2 = 2 * _ulp(torch.maximum(out.abs(), ref.abs()).clamp_min(2.0 ** -126))
    bound = ulp2 + 2.0 ** -6 * ref.abs().max()
    rms = (err.pow(2).mean() / ref.pow(2).mean()).sqrt().item()
    print(f"\n[pose embedding B={B} {h}x{w}] vs fp64 chain: {(err / (ulp2 + 2.0 ** -12 * ref.abs().max())).max().item():.3g} x "
          f"(2 ulp + 2^-12 max|ref|), max err {err.max().item() / ref.abs().max().item():.3g} max|ref|, rms {rms:.3g}; "
          f"varying share {power:.3f}")
    assert not (err > bound).any(), (f"{int((err > bound).sum())} / {err.numel()} beyond 2 ulp + 2^-6 max|ref| "
                                     f"(max {(err / bound).max().item():.3g} x)")
    assert rms <= 2.0 ** -7, f"rms error {rms:.3g} of the rms"
    # The fp32 oracle (no intermediate rounding) ties the chain to the module the reference runs.  At these shapes the
    # fp64 chain itself is 2.5-2.8x test_gpu_ops.py's value tolerance (8e-3 |ref| + 2e-3 max|ref|) from it, at 6.0e-3
    # rms, and the kernels add their drift from the chain: 6.5e-3 to 7.7e-3 max|ref| from the oracle, 0.75-0.78 of
    # 8e-3 |ref| + 2^-7 max|ref|.  So the absolute term is 2^-6 max|ref| (kernels at 0.38-0.42 of the bound), with
    # 2^-6 of the rms.
    pe = PoseEncoder(out_channels=cfg.block_out_channels[0]).cuda().eval()
    pe.load_state_dict({k[len("pose_encoder."):]: v.float() for k, v in sd.items() if k.startswith("pose_encoder.")})
    with torch.no_grad(), _no_tf32():
        y32 = pe(skel.float()).double()
    e32 = (out - y32).abs()
    m32 = y32.abs().max()
    tol = 8e-3 * y32.abs() + 2.0 ** -6 * m32
    rms32 = (e32.pow(2).mean() / y32.pow(2).mean()).sqrt().item()
    close = 8e-3 * y32.abs() + 2e-3 * m32
    print(f"[pose embedding B={B} {h}x{w}] vs fp32 oracle: max err {e32.max().item() / m32.item():.3g} max|ref|, "
          f"rms {rms32:.3g}; x test_gpu_ops.py's tolerance: kernels {(e32 / close).max().item():.3g}, fp64 chain "
          f"{((ref - y32).abs() / close).max().item():.3g}; x (8e-3 |ref| + 2^-7 max|ref|): kernels "
          f"{(e32 / (8e-3 * y32.abs() + 2.0 ** -7 * m32)).max().item():.3g}, x the bound: {(e32 / tol).max().item():.3g}")
    assert not (e32 > tol).any(), f"vs fp32 oracle: {(e32 / tol).max().item():.3g} x (8e-3 |ref| + 2^-6 max|ref|)"
    assert rms32 <= 2.0 ** -6, f"vs fp32 oracle: rms error {rms32:.3g} of the rms"
