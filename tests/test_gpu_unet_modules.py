"""Every module of the UNet launch plan against fp64, on exactly the bf16 tensors the plan fed it.

The whole-network tests (test_gpu_unet.py, test_gpu_fullsize.py) compare the output, or the ten block outputs, with the
fp32 oracle after the errors of up to sixty layers have accumulated.  A wrong host re-layout or plan choice inside one
module (a GEGLU half swap in one 16-row group, one ResNet's time-embedding slice, an attention scale taken from the padded
head dim) can hide under that drift, and once it shows it can no longer be traced to a module.  Here ``debug_taps(...,
modules=True)`` exposes the output of every module, and each module m is checked on its own:

  K    the plan's output of m (its tap);
  R64  the oracle's submodule m in float64 on the GPU, on the bf16 tensors the plan fed m: the previous tap, or
       cat(previous, skip) on the up path with the skip popped from the down-path taps in UpBlock order; a ResNet also
       reads the time_embedding tap, a transformer gets its level's num_frames;
  E16  the same submodule in bf16 eager on the same inputs: the arithmetic the reference runs.

Per module:  rms(K - R64) <= 1.25 rms(E16 - R64),  max|K - R64| <= 1.5 max|E16 - R64|,  K finite and of R64's shape.
The same recipe checks time_embedding (restated from the oracle's embedding functions), conv_in (+ pose encoder) and the
output head conv_out(silu(conv_norm_out(up_blocks.3))) against the forward's output.  A table of both ratios is printed
per case; the kernels round at fewer points than eager, so most ratios sit below 1.  Measured on an H100 80GB HBM3 (400 W
power limit) over the six cases: rms ratios 0.57-1.016, max ratios 0.36-1.13.  The rms ratios above 1 are all Upsample2D
(1.002-1.016): the plan runs it as four sub-pixel 2x2 convolutions whose weights are sums of two or four 3x3 taps, rounded
to bf16 once more on upload, a rounding eager does not have.  The max ratios above 1 (up to 1.13) are single elements of
ResNets and transformers whose rms ratios are 0.73-0.91: the largest error lands where one of the two roundings is worse.
With the weights drawn on the host instead (seed for seed a different draw) the same holds: rms up to 1.026, max up to 1.38.

test_module_harness_rehearsal runs the same harness on the CPU with the fp32 oracle's own module outputs, stored in bf16 at
every module boundary, standing in for the taps: it passes on them, and fails exactly at a module whose stand-in is scaled
by 1.02 and at that module's two consumers (the next module and the up-path ResNet that pops it as a skip).
"""
import copy
import gc
import time

import pytest
import torch
import torch.nn.functional as F

from diffuman4d_b200.config import UNetConfig
from diffuman4d_b200.plan import modules
from diffuman4d_b200.weights import random_state_dict
from oracle.unet_oracle import (Downsample2D, OracleUNet, ResnetBlock2D, TransformerMultiviewModel, Upsample2D,
                                timestep_embedding)

RMS_RATIO = 1.25   # rms(K - R64) <= RMS_RATIO * rms(E16 - R64)
MAX_RATIO = 1.5    # max|K - R64| <= MAX_RATIO * max|E16 - R64|
MODULE_TYPES = (ResnetBlock2D, TransformerMultiviewModel, Downsample2D, Upsample2D)

# (config, F, h, w, domains): what each case adds is in the comment
CASES = {
    # pose encoder, frame-index embedding, linear proj, head dim 64, per-image timesteps; level 3 at 2x3 pixels takes the
    # stand-alone GroupNorm statistics path (6 pixels per image: no 32-row warp stays inside one image)
    "tiny_temporal_16x24": (UNetConfig.tiny(), 4, 16, 24, ["temporal", "temporal"]),
    # different frame positions per CFG half
    "tiny_spatial_temporal": (UNetConfig.tiny(), 4, 16, 16, ["spatial", "temporal"]),
    # attn2 (per-image self-attention, norm1/2/3), 1x1-conv proj, odd F in the 3-D attention (test_gpu_unet.py's config)
    "tiny_attn2_convproj_nopose": (UNetConfig.tiny(cross_attention_dim=(64, 128, 256, 256), use_linear_projection=False,
                                                   enable_pose_encoder=False, enable_tem_embeds=False, in_channels=15),
                                   3, 16, 16, ["spatial", "spatial"]),
    # head dims 40 / 80 padded to 64 / 128, batch-1 3-D attention (no CFG)
    "headdim40_80": (UNetConfig(block_out_channels=(320, 320, 640, 640), attention_head_dim=(8, 8, 8, 8),
                                enable_pose_encoder=False, in_channels=15), 4, 16, 16, ["temporal"]),
    # reference constructor defaults at full width: head dims 40/80/160 -> 64/128/192, conv proj, in_channels 15
    "ctor_default": (UNetConfig.ctor_default(), 2, 16, 16, ["spatial", "spatial"]),
    # the benchmarked SD-2.1 layout: 1024-token 2-D and 3-D attention at full widths
    "sd21": (UNetConfig.sd21(), 4, 32, 32, ["temporal", "temporal"]),
}


# ------------------------------------------------------------------------------------------------ harness
def module_plan(cfg, F):
    """The modules of plan.modules in forward order as (name, input tap names, num_frames).  A ResNet also reads
    time_embedding; an up-path ResNet reads cat(previous, skip)."""
    plan, prev = [], "conv_in"
    for m in modules(cfg):
        plan.append((m.path, [prev] + ([m.skip_from] if m.skip_from else []), F if m.is3d else 1))
        prev = m.path
    return plan


def oracle_module_names(net):
    return {"time_embedding"} | {n for n, m in net.named_modules() if isinstance(m, MODULE_TYPES)}


def _cast(mod, dtype, device):
    return copy.deepcopy(mod).to(device=device, dtype=dtype)


def _time_embedding(net, cfg, t, domains, F, dtype, device):
    """UNET:519-546 from the oracle's pieces, in `dtype`; [B, 4*C0, 1, 1] like the tap.  The sinusoids are fp32 as in the
    oracle (error < 1e-4, far below bf16's 2^-9)."""
    C0 = cfg.block_out_channels[0]
    s = timestep_embedding(t.to(device), C0, cfg.flip_sin_to_cos, cfg.freq_shift).to(dtype)
    emb = _cast(net.time_embedding, dtype, device)(s)
    if cfg.enable_tem_embeds:
        idx = OracleUNet.frame_indices(domains, F, device=device)
        emb = emb + _cast(net.temporal_pos_embed, dtype, device)(timestep_embedding(idx, C0, True, 0).to(dtype))
    return emb[:, :, None, None]


def _conv_in(net, cfg, x, sk, dtype, device):
    y = _cast(net.conv_in, dtype, device)(x.to(device, dtype))
    if cfg.enable_pose_encoder:
        y = y + _cast(net.pose_encoder, dtype, device)(sk.to(device, dtype))
    return y


def _module(net, name, xs, temb, nf, dtype, device):
    m = _cast(net.get_submodule(name), dtype, device)
    x = torch.cat([v.to(device, dtype) for v in xs], dim=1)
    if isinstance(m, ResnetBlock2D):
        return m(x, temb.to(device, dtype).flatten(1))
    if isinstance(m, TransformerMultiviewModel):
        return m(x, num_frames=nf)
    return m(x)


def _head(net, x, dtype, device):
    n = _cast(net.conv_norm_out, dtype, device)(x.to(device, dtype))
    return _cast(net.conv_out, dtype, device)(F.silu(n))


def _ratios(k, r64, e16):
    """(rms ratio, max ratio, failure or None) of the kernel's and eager's errors from R64."""
    nan = float("nan")
    if k is None:
        return nan, nan, "no tap"
    if tuple(k.shape) != tuple(r64.shape):
        return nan, nan, f"shape {tuple(k.shape)} != {tuple(r64.shape)}"
    k = k.to(r64.device, torch.float64)
    if not torch.isfinite(k).all():
        return nan, nan, "non-finite"
    dk, de = k - r64, e16.to(torch.float64) - r64
    tiny = torch.finfo(torch.float64).tiny
    rr = dk.pow(2).mean().sqrt().item() / max(de.pow(2).mean().sqrt().item(), tiny)
    mr = dk.abs().max().item() / max(de.abs().max().item(), tiny)
    return rr, mr, None


def check_modules(net, cfg, taps, x, t, sk, domains, F, out, device):
    """Rows (name, rms ratio, max ratio, failure) for time_embedding, conv_in, every module of module_plan and the output
    head, each computed from `taps` (name -> bf16 NCHW) alone."""
    rows = []

    def row(name, k, fn):
        with torch.no_grad():
            r64, e16 = fn(torch.float64), fn(torch.bfloat16)
        rows.append((name, *_ratios(k, r64, e16)))

    temb = taps.get("time_embedding")
    row("time_embedding", temb, lambda dt: _time_embedding(net, cfg, t, domains, F, dt, device))
    row("conv_in", taps.get("conv_in"), lambda dt: _conv_in(net, cfg, x, sk, dt, device))
    plan = module_plan(cfg, F)
    for name, inputs, nf in plan:
        if temb is None or any(i not in taps for i in inputs):
            rows.append((name, float("nan"), float("nan"), "input tap missing"))
            continue
        row(name, taps.get(name), lambda dt: _module(net, name, [taps[i] for i in inputs], temb, nf, dt, device))
    last = plan[-1][0]
    if last in taps:
        row("conv_out (output)", out, lambda dt: _head(net, taps[last], dt, device))
    return rows


def failures(rows):
    return [name for name, rr, mr, fail in rows if fail or not (rr <= RMS_RATIO and mr <= MAX_RATIO)]


def report(title, rows):
    print(f"\n  kernel / eager error ratios vs fp64 [{title}]   bounds: rms {RMS_RATIO}, max {MAX_RATIO}")
    print(f"  {'module':<36}{'rms':>8}{'max':>8}")
    for name, rr, mr, fail in rows:
        flag = fail or ("  <-- beyond the bound" if not (rr <= RMS_RATIO and mr <= MAX_RATIO) else "")
        print(f"  {name:<36}{rr:>8.3f}{mr:>8.3f}{flag}")
    ok = [(rr, mr, name) for name, rr, mr, fail in rows if not fail]
    wr, wm = max(ok), max(ok, key=lambda r: r[1])
    print(f"  worst rms ratio {wr[0]:.3f} ({wr[2]}), worst max ratio {wm[1]:.3f} ({wm[2]})")


# ------------------------------------------------------------------------------------------------ shared set-up
def _oracle(cfg, sd):
    """The oracle holding exactly the state dict's tensors (checks cast a deep copy of each submodule)."""
    with torch.device("meta"):
        net = OracleUNet(cfg)
    net.load_state_dict(sd, assign=True)
    return net.eval()


def _inputs(cfg, B, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cfg.in_channels, h, w, generator=g).to(torch.bfloat16)
    t = torch.randint(0, 1000, (B,), generator=g)            # one timestep per image
    sk = (torch.rand(B, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16) if cfg.enable_pose_encoder else None
    return x, t, sk


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("case", list(CASES))
def test_module_plan_covers_the_oracle(case):
    cfg, F = CASES[case][:2]
    with torch.device("meta"):
        net = OracleUNet(cfg)
    plan = module_plan(cfg, F)
    names = [n for n, _, _ in plan]
    assert len(names) == len(set(names))
    assert {"time_embedding", *names} == oracle_module_names(net)


def _standin_taps(net, x, t, sk, domains, F):
    """The fp32 oracle's forward with every module boundary stored in bf16, as the plan stores it: each module's tensor
    inputs and its output are rounded, and recorded under the tap names (conv_in and time_embedding from the first
    ResNet's inputs).  Returns (taps, output) in bf16."""
    taps, hooks = {}, []
    rnd = lambda v: v.to(torch.bfloat16).float() if torch.is_tensor(v) else v
    first = net.get_submodule("down_blocks.0.resnets.0")

    def pre(m, args):
        args = tuple(rnd(a) for a in args)
        if m is first:
            taps["conv_in"], taps["time_embedding"] = args[0], args[1][:, :, None, None]
        return args

    def post(name):
        def hook(m, args, out):
            taps[name] = rnd(out)
            return taps[name]
        return hook

    for name, m in net.named_modules():
        if isinstance(m, MODULE_TYPES):
            hooks += [m.register_forward_pre_hook(pre), m.register_forward_hook(post(name))]
    try:
        with torch.no_grad():
            y = net(x.float(), t, None if sk is None else sk.float(), domains, F)
    finally:
        for hk in hooks:
            hk.remove()
    return {k: v.to(torch.bfloat16) for k, v in taps.items()}, y.to(torch.bfloat16)


def test_module_harness_rehearsal():
    """The harness on the CPU, fed the oracle's own module outputs: the skip-stack order, num_frames per level and the
    time-embedding plumbing must reproduce every stand-in within the bounds, and a 2% error in one stand-in must be
    named at that module and at its two consumers only."""
    cfg, F, h, w, domains = UNetConfig.tiny(), 2, 8, 8, ["temporal", "spatial"]
    net = _oracle(cfg, random_state_dict(cfg, seed=3, dtype=torch.bfloat16)).float()
    x, t, sk = _inputs(cfg, len(domains) * F, h, w, seed=4)
    taps, y = _standin_taps(net, x, t, sk, domains, F)
    assert set(taps) == oracle_module_names(net) | {"conv_in"}
    rows = check_modules(net, cfg, taps, x, t, sk, domains, F, y, "cpu")
    report("CPU rehearsal, oracle stand-ins", rows)
    assert not failures(rows), failures(rows)
    scaled = "down_blocks.1.attentions.0"
    bad = dict(taps)
    bad[scaled] = (taps[scaled].float() * 1.02).to(torch.bfloat16)
    fails = failures(check_modules(net, cfg, bad, x, t, sk, domains, F, y, "cpu"))
    # read by down_blocks.1.resnets.1, and popped as the skip of up_blocks.2.resnets.1 (the 8th of 12 pops)
    assert set(fails) == {scaled, "down_blocks.1.resnets.1", "up_blocks.2.resnets.1"}, fails


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_unet_modules_vs_fp64(cuda, case):
    from diffuman4d_b200.unet import B200MultiviewUNet
    cfg, F, h, w, domains = CASES[case]
    B = len(domains) * F
    t0 = time.perf_counter()
    sd = random_state_dict(cfg, seed=1, dtype=torch.bfloat16, device="cuda")
    ours = B200MultiviewUNet(cfg, device=0).load_state_dict(sd)
    net = _oracle(cfg, sd)
    del sd
    try:
        x, t, sk = (None if v is None else v.cuda() for v in _inputs(cfg, B, h, w))
        y = ours(x, t, sk, domains, F, return_dict=False)[0]
        launches = ours.forward_launches(len(domains), B, F, h, w)
        blocks = ours.debug_taps(x, t, sk, domains, F)
        taps = ours.debug_taps(x, t, sk, domains, F, modules=True)
        names = list(taps)
        # the ten block taps keep their indices and names; the module taps follow in forward order
        assert names[:10] == list(blocks) == ["conv_in", *(f"down_blocks.{i}" for i in range(4)), "mid_block",
                                              *(f"up_blocks.{i}" for i in range(4))]
        assert all(torch.equal(taps[k], blocks[k]) for k in blocks)
        assert names[10:] == ["time_embedding", *(n for n, _, _ in module_plan(cfg, F))]
        assert set(names[10:]) == oracle_module_names(net)
        # taps read the plan's buffers and add no launch: a plain forward afterwards is bit-identical
        assert torch.equal(ours(x, t, sk, domains, F, return_dict=False)[0], y)
        assert ours.forward_launches(len(domains), B, F, h, w) == launches
        rows = check_modules(net, cfg, taps, x, t, sk, domains, F, y, "cuda")
        torch.cuda.synchronize()
    finally:
        del ours, net
        gc.collect()
        torch.cuda.empty_cache()
    report(f"{case}: F={F} {h}x{w} {'+'.join(domains)}, {launches} launches", rows)
    print(f"  [{case}] {time.perf_counter() - t0:.1f} s")
    fails = failures(rows)
    assert not fails, f"modules beyond rms {RMS_RATIO}x / max {MAX_RATIO}x of bf16 eager's error from fp64: {fails}"
