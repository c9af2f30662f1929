"""GPU parity tests of the whole hot path through the C ABI: UNet forward, input assembly, CFG+DDIM step, window
denoise step, sliding loop -- against the CPU oracle (oracle/), on the same seeded inputs and the same weights.

Tolerance for the whole UNet (stated per the task contract).  BASELINE.json asks for rtol 1e-3 / atol 1e-4 "bf16";
bf16 has 2^-8 = 3.9e-3 relative spacing, so two *correct* bf16 evaluations of a 60-layer network differ by far more
than 1e-3 (SURVEY.md section 7).  The bar used here is the reference's own precision: with
    e_ours  = max|ours - oracle_fp32| / max|oracle_fp32|
    e_eager = max|oracle_bf16(torch eager, what the reference runs) - oracle_fp32| / max|oracle_fp32|
we require e_ours <= 1.5 * e_eager + 2e-3 and e_ours <= 4e-2 absolute.  Both numbers are printed.
"""
import math
import re

import pytest
import torch

from diffuman4d_b200.config import SchedulerConfig, UNetConfig
from diffuman4d_b200.weights import random_state_dict

pytestmark = pytest.mark.gpu


def _inputs(cfg, F, h, w, cfg_on=True, seed=0):
    g = torch.Generator().manual_seed(seed)
    B = 2 * F if cfg_on else F
    x = torch.randn(B, cfg.in_channels, h, w, generator=g).to(torch.bfloat16)
    t = torch.randint(0, 1000, (B,), generator=g)
    sk = (torch.rand(B, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16) if cfg.enable_pose_encoder else None
    return x, t, sk


def _build(cfg, seed=1):
    from diffuman4d_b200.unet import B200MultiviewUNet
    from oracle.unet_oracle import OracleUNet
    sd = random_state_dict(cfg, seed=seed, dtype=torch.bfloat16)        # bf16-representable weights for both sides
    ours = B200MultiviewUNet(cfg, device=0).load_state_dict(sd)
    ref = OracleUNet(cfg).eval()
    ref.load_state_dict({k: v.float() for k, v in sd.items()})
    return ours, ref


def _rel(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max()).item()


CONFIGS = {
    "tiny_pose_tem_linear": UNetConfig.tiny(),
    "tiny_attn2_convproj_nopose": UNetConfig.tiny(cross_attention_dim=(64, 128, 256, 256), use_linear_projection=False,
                                                  enable_pose_encoder=False, enable_tem_embeds=False, in_channels=15),
    "headdim40_80": UNetConfig(block_out_channels=(320, 320, 640, 640), attention_head_dim=(8, 8, 8, 8),
                               enable_pose_encoder=False, in_channels=15),
}


@pytest.mark.parametrize("name,F,h,w,domain", [("tiny_pose_tem_linear", 4, 16, 16, "spatial"),
                                               ("tiny_pose_tem_linear", 4, 16, 24, "temporal"),
                                               ("tiny_attn2_convproj_nopose", 3, 16, 16, "spatial"),
                                               ("headdim40_80", 2, 8, 8, "temporal")])
def test_unet_forward_vs_oracle(cuda, name, F, h, w, domain):
    cfg = CONFIGS[name]
    ours, ref = _build(cfg)
    x, t, sk = _inputs(cfg, F, h, w)
    doms = [domain, domain]
    with torch.no_grad():
        y_ref = ref(x.float(), t, None if sk is None else sk.float(), doms, F)
        ref16 = ref.to("cuda").to(torch.bfloat16)
        y_eager = ref16(x.cuda(), t.cuda(), None if sk is None else sk.cuda(), doms, F).float().cpu()
    y = ours(x.cuda(), t.cuda(), None if sk is None else sk.cuda(), doms, F, return_dict=False)[0]
    torch.cuda.synchronize()
    assert y.shape == y_ref.shape and y.dtype == torch.bfloat16
    assert torch.isfinite(y.float()).all()
    e_ours, e_eager = _rel(y.cpu(), y_ref), _rel(y_eager, y_ref)
    print(f"\n[{name} F={F} {h}x{w} {domain}] e_ours={e_ours:.3e}  e_eager_bf16={e_eager:.3e}")
    assert e_ours <= 1.5 * e_eager + 2e-3, (e_ours, e_eager)
    assert e_ours <= 4e-2
    # second call on the cached plan gives the identical result (no stale state in the arena)
    y2 = ours(x.cuda(), t.cuda(), None if sk is None else sk.cuda(), doms, F, return_dict=False)[0]
    assert torch.equal(y, y2)


def test_unet_forward_interface_errors(cuda):
    cfg = CONFIGS["tiny_pose_tem_linear"]
    ours, _ = _build(cfg)
    x, t, sk = _inputs(cfg, 2, 8, 8)
    with pytest.raises(ValueError, match="num_frames"):
        ours(x.cuda(), t.cuda(), sk.cuda(), ["spatial"], 2)                    # UNET:524-525
    with pytest.raises(ValueError, match="Invalid domain"):
        ours(x.cuda(), t.cuda(), sk.cuda(), ["diagonal", "spatial"], 2)         # UNET:541
    with pytest.raises(ValueError):
        ours(x.cuda(), t.cuda(), None, ["spatial", "spatial"], 2)               # pose encoder needs skeletons
    with pytest.raises(ValueError):
        ours(x[:, :5].cuda(), t.cuda(), sk.cuda(), ["spatial", "spatial"], 2)
    with pytest.raises(ValueError):
        ours(x[..., :6].contiguous().cuda(), t.cuda(), sk[..., :48].contiguous().cuda(), ["spatial", "spatial"], 2)  # w % 8
    out = ours(x.cuda(), t.cuda(), sk.cuda(), ["spatial", "spatial"], 2)
    assert out.sample.shape == (4, 4, 8, 8)
    with pytest.raises(RuntimeError):
        from diffuman4d_b200.unet import B200MultiviewUNet
        B200MultiviewUNet(cfg, 0).load_state_dict({"conv_in.weight": torch.zeros(64, 11, 3, 3)})


@pytest.mark.parametrize("name", [*CONFIGS, "tiny_3d0", "tiny_3d1", "tiny_3d4"])
def test_weight_keys_and_load_refusals(cuda, name):
    """The library's weight keys are state_dict_spec's, in order; a transposed tensor (right element count) and an
    unknown key are refused, naming the key."""
    import ctypes as C
    from diffuman4d_b200._lib import check, lib
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import state_dict_spec
    cfg = CONFIGS[name] if name in CONFIGS else UNetConfig.tiny(num_3d_attn_blocks=int(name[-1]))
    unet = B200MultiviewUNet(cfg, 0)
    assert unet.expected_keys() == list(state_dict_spec(cfg))
    sd = random_state_dict(cfg, seed=1, device="cuda")
    for key in ("time_embedding.linear_1.weight", "conv_in.weight", "up_blocks.1.resnets.2.conv_shortcut.weight"):
        with pytest.raises(ValueError, match=f"shape mismatch for {re.escape(key)}"):
            unet.load_state_dict({**sd, key: sd[key].transpose(0, 1).contiguous()})
    with pytest.raises(RuntimeError, match="unexpected"):
        unet.load_state_dict({**sd, "down_blocks.0.bogus.weight": torch.zeros(4)})
    t = torch.zeros(4)
    with pytest.raises(ValueError, match="unknown weight key: down_blocks.0.bogus.weight"):
        check(lib().d4d_load_weight(unet._h, b"down_blocks.0.bogus.weight", t.data_ptr(), (C.c_int64 * 1)(4), 1, 0))


def _sched_pair(pred="epsilon", emulate=False):
    from diffuman4d_b200.scheduler import DDIMTables
    from oracle.pipeline_oracle import DDIMOracle
    sc = SchedulerConfig(prediction_type=pred)
    a, b = DDIMTables(sc, device="cuda:0"), DDIMOracle(sc)
    a.set_timesteps(18), b.set_timesteps(18)
    return a, b


@pytest.mark.parametrize("with_skel", [False, True])
def test_assemble_input_bit_exact(cuda, with_skel):
    import ctypes as C
    from diffuman4d_b200._lib import check, lib
    from oracle.pipeline_oracle import assemble_unet_input
    F, h, w = 6, 16, 8
    g = torch.Generator().manual_seed(5)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    lat, pix, plk, skl = r(F, 4, h, w), r(F, 4, h, w), r(F, 6, h, w), (r(F, 4, h, w) if with_skel else None)
    mask = torch.ones(F, 1, h, w, dtype=torch.bfloat16)
    mask[[0, 3]] = 0
    ts, _ = _sched_pair()
    ti = torch.tensor([0, 2, 5, 0, 17, 1])
    for cfg_on in (True, False):
        lat_ref = lat.clone()
        x_ref, _ = assemble_unet_input(lat_ref, pix, plk, skl, mask, mask[:, 0, 0, 0] == 0, cfg_on, concat_skeleton=with_skel)
        lat_d = lat.clone().cuda()
        B = 2 * F if cfg_on else F
        x_d = torch.empty(B, x_ref.shape[1], h, w, dtype=torch.bfloat16, device="cuda")
        t_d = torch.empty(B, dtype=torch.int64, device="cuda")
        tbl = ts.timesteps.cuda()
        pix_d, plk_d, msk_d, ti_d = pix.cuda(), plk.cuda(), mask.cuda(), ti.cuda()   # keep the device copies alive
        skl_d = skl.cuda() if with_skel else None
        check(lib().d4d_assemble_input(lat_d.data_ptr(), pix_d.data_ptr(), plk_d.data_ptr(),
                                       skl_d.data_ptr() if with_skel else None, msk_d.data_ptr(),
                                       ti_d.data_ptr(), tbl.data_ptr(), 18, F, h, w, int(cfg_on), x_d.data_ptr(),
                                       t_d.data_ptr(), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        assert torch.equal(x_d.cpu(), x_ref)
        assert torch.equal(lat_d.cpu(), lat_ref)                 # cond frames overwritten in place (PIPE:375-379)
        t_ref = ts.timesteps[ti].clone()
        t_ref[[0, 3]] = 0
        assert torch.equal(t_d.cpu(), torch.cat([t_ref] * 2) if cfg_on else t_ref)


@pytest.mark.parametrize("pred", ["epsilon", "v_prediction", "sample"])
def test_cfg_ddim_step(cuda, pred):
    import ctypes as C
    from diffuman4d_b200._lib import check, lib
    F, h, w = 5, 8, 16
    g = torch.Generator().manual_seed(6)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    noise, lat = r(2 * F, 4, h, w), r(F, 4, h, w)
    mask = torch.ones(F, 1, h, w, dtype=torch.bfloat16)
    mask[1] = 0
    ti = torch.tensor([17, 0, 3, 0, 9])
    for emulate in (True, False):
        ts, orc = _sched_pair(pred)
        # oracle: CFG combine + per-frame step, in bf16 (the reference's arithmetic) or fp32
        dt = torch.bfloat16 if emulate else torch.float32
        u, c = noise.to(dt).chunk(2)
        eps = u + 2.0 * (c - u)          # 2.0 and the differences are exact roundings in either dtype
        ref = []
        for j in range(F):
            if mask[j, 0, 0, 0] == 0:
                ref.append(lat[j:j + 1].to(dt))
            else:
                ref.append(orc.step(eps[j:j + 1], int(orc.timesteps[ti[j]]), lat[j:j + 1].to(dt)))
        ref = torch.cat(ref)
        out = torch.empty(F, 4, h, w, dtype=torch.bfloat16, device="cuda")
        ti_out = torch.empty(F, dtype=torch.int64, device="cuda")
        s = ts.c_struct(emulate)
        noise_d, lat_d, msk_d, ti_d = noise.cuda(), lat.cuda(), mask.cuda(), ti.cuda()   # keep the device copies alive
        check(lib().d4d_cfg_ddim_step(noise_d.data_ptr(), lat_d.data_ptr(), msk_d.data_ptr(),
                                      ti_d.data_ptr(), ti_out.data_ptr(), C.byref(s), 2.0, 1, F, h, w,
                                      out.data_ptr(), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        assert ti_out.cpu().tolist() == [ti[0] + 1, 0, ti[2] + 1, ti[3] + 1, ti[4] + 1]
        if emulate:
            assert torch.equal(out.cpu(), ref.to(torch.bfloat16)), (out.cpu().float() - ref.float()).abs().max()
        else:
            torch.testing.assert_close(out.cpu().float(), ref, rtol=8e-3, atol=8e-3)


def test_denoise_window_vs_oracle(cuda):
    """B-3: one C-ABI call == the oracle's window step driven with OUR UNet as the noise predictor (isolates the
    pipeline logic: assembly, CFG, per-frame timesteps, cond-frame aliasing, index update).  bf16-emulating scheduler
    => bit-exact."""
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from oracle.pipeline_oracle import denoise_window_oracle
    cfg = CONFIGS["tiny_pose_tem_linear"]
    ours, _ = _build(cfg)
    pipe = B200Diffuman4DPipeline(ours, SchedulerConfig(), emulate_bf16_scheduler=True)
    pipe.parepare_schedulers(18, 6)
    _, orc = _sched_pair()
    F, h, w = 6, 8, 8
    g = torch.Generator().manual_seed(7)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    lat, pix, plk = r(F, 4, h, w), r(F, 4, h, w), r(F, 6, h, w)
    skel = (torch.rand(F, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16)
    mask = torch.ones(F, 1, h, w, dtype=torch.bfloat16)
    mask[:2] = 0
    ti = torch.tensor([0, 0, 5, 5, 4, 3])

    def unet_cb(x, t, sk, doms, nf):
        return ours(x.cuda(), t.cuda(), sk.cuda(), doms, nf, return_dict=False)[0].cpu()

    for domain in ("spatial", "temporal"):
        ref_lat, ref_ti = denoise_window_oracle(unet_cb, orc, latents=lat.clone(), pixel_latents=pix, plucker=plk,
                                                skeletons=skel, cond_mask=mask, timestep_indices=ti, domain=domain,
                                                guidance_scale=2.0, num_inference_steps=2, enable_pose_encoder=True)
        l_d, t_d = lat.clone().cuda(), ti.clone().cuda()
        pipe.denoise_window(latents=l_d, pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skel,
                            cond_masks_latents=mask, timestep_indices=t_d, domain=domain, guidance_scale=2.0,
                            num_inference_steps=2)
        torch.cuda.synchronize()
        assert torch.equal(t_d.cpu(), ref_ti)
        assert torch.equal(l_d.cpu(), ref_lat), (l_d.cpu().float() - ref_lat.float()).abs().max()


def test_sliding_iterative_denoise_invariants(cuda):
    """B-4 on the GPU: the reference's own runtime invariants (PIPE:480-487, 546-551) and its ValueErrors."""
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    cfg = CONFIGS["tiny_pose_tem_linear"]
    ours, _ = _build(cfg)
    pipe = B200Diffuman4DPipeline(ours, SchedulerConfig())
    n, h, w = 12, 8, 8
    g = torch.Generator().manual_seed(8)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    mask = torch.ones(n, 1, h, w)
    mask[[1, 4, 7, 10]] = 0
    kw = dict(pixel_values_latents=r(n, 4, h, w), plucker_embeds=r(n, 6, h, w),
              skeletons=(torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1), cond_masks=mask, latents=r(n, 4, h, w),
              domain="spatial", timestep_indices=torch.zeros(n, dtype=torch.long), window_size=4, sliding_stride=2,
              bidirectional=False, alternation_rounds=3, guidance_scale=2.0)
    out = pipe.sliding_iterative_denoise(**kw)
    tgt = (mask[:, 0, 0, 0] != 0)
    assert (out["timestep_indices"].cpu()[tgt] == 2).all() and (out["timestep_indices"].cpu()[~tgt] == 0).all()
    assert torch.equal(out["latents"].cpu()[~tgt], kw["pixel_values_latents"][~tgt])
    assert torch.isfinite(out["latents"].float()).all() and not out["fully_denoised"].any()
    with pytest.raises(ValueError, match="divisible by the sliding stride"):
        pipe.sliding_iterative_denoise(**{**kw, "window_size": 3})
    bad = torch.zeros(n, dtype=torch.long)
    bad[0] = 1
    with pytest.raises(ValueError, match="same for all target samples"):
        pipe.sliding_iterative_denoise(**{**kw, "timestep_indices": bad})


def test_full_size_properties(cuda):
    """BASELINE-size (SD-2.1 layout, W16 @ 64x64, CFG => 32 images) size-independent properties:
    (1) spatial-domain frame-permutation equivariance (3-D attention sees a set of frames; all frame-index
        embeddings are equal in the spatial domain),  (2) the two CFG halves do not interact."""
    from diffuman4d_b200.unet import B200MultiviewUNet
    cfg = UNetConfig.sd21()
    unet = B200MultiviewUNet(cfg, 0).load_state_dict(random_state_dict(cfg, seed=1))
    F, h, w = 16, 64, 64
    x, t, sk = _inputs(cfg, F, h, w)
    x, t, sk = x.cuda(), t.cuda(), sk.cuda()
    doms = ["spatial", "spatial"]
    y = unet(x, t, sk, doms, F, return_dict=False)[0]
    assert torch.isfinite(y.float()).all()
    perm = torch.randperm(F, generator=torch.Generator().manual_seed(9)).cuda()
    p2 = torch.cat([perm, perm + F])
    yp = unet(x[p2].contiguous(), t[p2].contiguous(), sk[p2].contiguous(), doms, F, return_dict=False)[0]
    scale = y.float().abs().max().item()
    assert (yp.float() - y[p2].float()).abs().max().item() <= 2e-2 * scale      # summation order changes only
    x2 = x.clone()
    x2[F:] = torch.randn_like(x2[F:])
    y2 = unet(x2, t, sk, doms, F, return_dict=False)[0]
    assert torch.equal(y2[:F], y[:F])                                            # negative half untouched
    assert unet.forward_launches(2, 2 * F, F, h, w) > 250     # (61 GroupNorm statistics launches are fused away)
    # temporal window W24 (12 cond + 12 target frames => 48 images): finite, deterministic, and different from 'spatial'
    F = 24
    x, t, sk = _inputs(cfg, F, h, w, seed=3)
    x, t, sk = x.cuda(), t.cuda(), sk.cuda()
    yt = unet(x, t, sk, ["temporal", "temporal"], F, return_dict=False)[0]
    assert torch.isfinite(yt.float()).all()
    assert torch.equal(yt, unet(x, t, sk, ["temporal", "temporal"], F, return_dict=False)[0])
    ys = unet(x, t, sk, ["spatial", "spatial"], F, return_dict=False)[0]
    assert (ys.float() - yt.float()).abs().max() > 0


def test_reference_default_latent_size(cuda):
    """The reference's default latent size (1024^2 px => 128x128 latents, DATA:27-28) with the largest window the sampler
    builds (W24, CFG => 48 images; level-1 3-D attention over 98 304 tokens): runs, finite, cond/uncond halves independent."""
    from diffuman4d_b200.unet import B200MultiviewUNet
    cfg = UNetConfig.sd21(enable_pose_encoder=False, in_channels=15)
    unet = B200MultiviewUNet(cfg, 0).load_state_dict(random_state_dict(cfg, seed=2))
    F, h, w = 24, 128, 128
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(2 * F, 15, h, w, device="cuda", generator=g).to(torch.bfloat16)
    t = torch.randint(0, 1000, (2 * F,), device="cuda", generator=g)
    y = unet(x, t, None, ["temporal", "temporal"], F, return_dict=False)[0]
    assert y.shape == (2 * F, 4, h, w) and torch.isfinite(y.float()).all()
    x2 = x.clone()
    x2[:F] = torch.randn_like(x2[:F])
    y2 = unet(x2, t, None, ["temporal", "temporal"], F, return_dict=False)[0]
    assert torch.equal(y2[F:], y[F:])
