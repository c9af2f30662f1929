"""GPU tests of the UniPC step (upstream UniPCMultistepScheduler, predict_x0, bh1 / bh2): the fused CFG + step kernel
against UniPCOracle on the same bf16 inputs with frames in every solver state, the window step through the C ABI and
the sliding loop against the oracle driven by the same CUDA UNet, ``__call__`` with the per-frame handles,
load_pipelines on a checkpoint that names the scheduler, and the device sampler."""
import copy
import json
import os
import sys

import pytest
import torch

from diffuman4d_b200.config import UNetConfig, UniPCConfig
from diffuman4d_b200.weights import random_state_dict

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def _oracle_frame(cfg, n, idx, lon, x0_prev, x0_prev2, last_sample):
    """A per-frame oracle scheduler standing where the frame's own copy stands after ``lon`` steps ending at ``idx``."""
    from oracle.unipc_oracle import UniPCOracle
    s = UniPCOracle(cfg)
    s.set_timesteps(n)
    s.step_index = idx
    s.lower_order_nums = lon
    s.this_order = lon                         # the previous step's order: lon whenever a further step is taken
    s.model_outputs[-1] = x0_prev
    if cfg.solver_order == 2:
        s.model_outputs[-2] = x0_prev2
    s.last_sample = last_sample if lon >= 1 else None
    return s


@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("pred", ["epsilon", "v_prediction", "sample"])
@pytest.mark.parametrize("cfg_on", [True, False])
def test_cfg_unipc_step_vs_oracle(cuda, order, pred, cfg_on):
    from diffuman4d_b200.ops import cfg_unipc_step
    from diffuman4d_b200.scheduler import UniPCTables
    n = 10
    cfg = UniPCConfig(prediction_type=pred, solver_order=order, disable_corrector=(6,))   # final sigma 0, lower_order_final
    F, h, w = 7, 9, 13                                                    # 4*h*w = 468: no multiple of the block size
    g = torch.Generator().manual_seed(21)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    noise, lat = r((2 if cfg_on else 1) * F, 4, h, w), r(F, 4, h, w)
    x0_prev, x0_prev2, last = r(F, 4, h, w), r(F, 4, h, w), r(F, 4, h, w)
    lat[0] *= 60   # a high-noise frame at step 0
    mask = torch.ones(F, 1, h, w, dtype=torch.bfloat16)
    mask[2] = 0
    # frame: 0 fresh at step 0 | 1 lon 1 | 2 cond | 3 fresh mid-schedule | 4 lon 2 | 5 final step (sigma 0) |
    #        6 corrector disabled (its previous step index 6 is listed)
    ti = torch.tensor([0, 1, 4, 5, 4, 9, 7])
    lon = torch.tensor([0, 1, 2, 0, 2, 2, 2], dtype=torch.int32).clamp(max=order)
    tables = UniPCTables(cfg, device="cuda:0")
    tables.set_timesteps(n)
    guidance = 2.0 if cfg_on else 1.0
    for emulate in (True, False):
        dt = torch.bfloat16 if emulate else torch.float32
        if cfg_on:
            u, c = noise.to(dt).chunk(2)
            eps = u + 2.0 * (c - u)          # 2.0 and the differences are exact roundings in either dtype
        else:
            eps = noise.to(dt)
        ref, ref_x0, ref_x02, ref_last = [], [], [], []
        for j in range(F):
            if mask[j, 0, 0, 0] == 0:
                ref.append(lat[j:j + 1].to(dt))
                ref_x0.append(x0_prev[j:j + 1].to(dt))
                ref_x02.append(x0_prev2[j:j + 1].to(dt))
                ref_last.append(last[j:j + 1].to(dt))
                continue
            s = _oracle_frame(cfg, n, int(ti[j]), int(lon[j]), x0_prev[j:j + 1].to(dt), x0_prev2[j:j + 1].to(dt),
                              last[j:j + 1].to(dt))
            ref.append(s.step(eps[j:j + 1], int(s.timesteps[ti[j]]), lat[j:j + 1].to(dt)))
            ref_x0.append(s.model_outputs[-1])
            ref_x02.append(s.model_outputs[-2] if order == 2 else x0_prev2[j:j + 1].to(dt))
            ref_last.append(s.last_sample)
        ref, ref_x0, ref_x02, ref_last = (torch.cat(t).float() for t in (ref, ref_x0, ref_x02, ref_last))
        x0_d, last_d = x0_prev.cuda(), last.cuda()
        x02_d = x0_prev2.cuda() if order == 2 else None
        out, ti_out, lon_out = cfg_unipc_step(noise.cuda(), lat.cuda(), mask.cuda(), ti.cuda(), x0_d, x02_d, last_d,
                                              lon.cuda(), tables.c_struct(emulate), guidance, cfg_on)
        torch.cuda.synchronize()
        assert ti_out.cpu().tolist() == [1, 2, 0, 6, 5, 10, 8]
        assert lon_out.cpu().tolist() == [min(v, order) for v in (1, 2, 2, 1, 2, 2, 2)]
        got = {"out": (out, ref), "x0_prev": (x0_d, ref_x0), "last_sample": (last_d, ref_last)}
        if order == 2:
            got["x0_prev2"] = (x02_d, ref_x02)
        for name, (g_d, want) in got.items():
            g_c = g_d.cpu().float()
            if emulate:
                assert torch.equal(g_c, want), (name, (g_c - want).abs().max())
            else:
                bound = 1e-6 * want.abs().max() + _bf16_ulp(want)
                assert ((g_c - want).abs() <= bound).all(), (name, ((g_c - want).abs() - bound).max())
        assert torch.equal(x0_d.cpu()[2], x0_prev[2]) and torch.equal(last_d.cpu()[2], last[2])   # cond: untouched
        # the final step with sigma 0 returns the data prediction itself
        assert torch.equal(out.cpu()[5], x0_d.cpu()[5])


def _tiny_pipe(emulate=True, **kw):
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.unet import B200MultiviewUNet
    cfg = UNetConfig.tiny()
    unet = B200MultiviewUNet(cfg, device=0).load_state_dict(random_state_dict(cfg, seed=1, dtype=torch.bfloat16))
    return B200Diffuman4DPipeline(unet, UniPCConfig(**kw), emulate_bf16_scheduler=emulate), unet


def _unet_cb(unet):
    def cb(x, t, sk, doms, nf):
        return unet(x.cuda(), t.cuda(), sk.cuda(), doms, nf, return_dict=False)[0].cpu()
    return cb


@pytest.mark.parametrize("order", [1, 2])
def test_denoise_window_unipc_vs_oracle_bit_exact(cuda, order):
    """``d4d_denoise_window_unipc`` (three steps of one window, staggered step indices, fresh state) against the oracle's
    window step with per-frame scheduler copies, both driven by the same CUDA UNet; the state comes back updated."""
    from oracle.dpm_solver_oracle import denoise_window_oracle_per_frame
    from oracle.unipc_oracle import UniPCOracle
    pipe, unet = _tiny_pipe(solver_order=order)
    n, h, w = 5, 8, 8
    g = torch.Generator().manual_seed(22)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    pix, plk, lat = r(n, 4, h, w), r(n, 6, h, w), r(n, 4, h, w)
    skel = (torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16)
    mask = torch.ones(n, 1, h, w, dtype=torch.bfloat16)
    mask[1] = 0
    ti = torch.tensor([0, 0, 1, 2, 3])
    handles, _ = pipe.parepare_schedulers(8, n)
    state = handles[0].state.take(torch.arange(n), h, w)
    orc = UniPCOracle(pipe.scheduler.config)
    orc.set_timesteps(8)
    copies = [copy.deepcopy(orc) for _ in range(n)]
    want, want_ti = denoise_window_oracle_per_frame(
        _unet_cb(unet), copies, latents=lat.clone(), pixel_latents=pix, plucker=plk, skeletons=skel, cond_mask=mask,
        timestep_indices=ti, domain="spatial", guidance_scale=2.0, num_inference_steps=3)
    lat_d, ti_d = lat.cuda(), ti.cuda()
    pipe.denoise_window(latents=lat_d, pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skel,
                        cond_masks_latents=mask, timestep_indices=ti_d, domain="spatial", guidance_scale=2.0,
                        num_inference_steps=3, solver_state=state)
    torch.cuda.synchronize()
    assert torch.equal(ti_d.cpu(), want_ti)
    assert torch.equal(lat_d.cpu(), want), (lat_d.cpu().float() - want.float()).abs().max()
    assert state.lower_order_nums.cpu().tolist() == [c.lower_order_nums for c in copies]
    for j in (0, 2, 3, 4):
        assert torch.equal(state.x0_prev.cpu()[j:j + 1], copies[j].model_outputs[-1])
        assert torch.equal(state.last_sample.cpu()[j:j + 1], copies[j].last_sample)
        if order == 2:
            assert torch.equal(state.x0_prev2.cpu()[j:j + 1], copies[j].model_outputs[-2])


@pytest.mark.parametrize("kw", [dict(), dict(solver_order=1, solver_type="bh1", final_sigmas_type="sigma_min"),
                                dict(final_sigmas_type="sigma_min", lower_order_final=False, disable_corrector=(1, 4))])
def test_sliding_iterative_denoise_unipc_vs_oracle_bit_exact(cuda, kw):
    """Per-frame solver state carried across the windows of a task and reset per task: a spatial and then a bidirectional
    temporal task on one pipeline, against the oracle's sliding loop (per-frame scheduler copies) with our UNet."""
    from oracle.dpm_solver_oracle import sliding_iterative_denoise_oracle_per_frame
    from oracle.unipc_oracle import UniPCOracle
    pipe, unet = _tiny_pipe(**kw)
    h = w = 8
    g = torch.Generator().manual_seed(23)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    for domain, n_in, n_tg, ws, stride, bidir, rounds in (("spatial", 2, 4, 2, 1, False, 2),
                                                          ("temporal", 3, 3, 2, 1, True, 1)):
        n = n_in + n_tg
        mask = torch.ones(n, 1, h, w, dtype=torch.bfloat16)
        mask[:n_in] = 0
        args = dict(pixel_latents=r(n, 4, h, w), plucker=r(n, 6, h, w),
                    skeletons=(torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16), cond_mask=mask,
                    latents=r(n, 4, h, w), domain=domain, timestep_indices=torch.zeros(n, dtype=torch.long),
                    window_size=ws, sliding_stride=stride, bidirectional=bidir, alternation_rounds=rounds,
                    guidance_scale=2.0)
        ref = sliding_iterative_denoise_oracle_per_frame(_unet_cb(unet), UniPCOracle(pipe.scheduler.config), **args,
                                                         enable_pose_encoder=True)
        out = pipe.sliding_iterative_denoise(
            pixel_values_latents=args["pixel_latents"], plucker_embeds=args["plucker"], skeletons=args["skeletons"],
            cond_masks=mask, latents=args["latents"], domain=domain, timestep_indices=args["timestep_indices"],
            window_size=ws, sliding_stride=stride, bidirectional=bidir, alternation_rounds=rounds, guidance_scale=2.0)
        torch.cuda.synchronize()
        assert torch.equal(out["timestep_indices"].cpu(), ref["timestep_indices"])
        assert torch.equal(out["fully_denoised"].cpu(), ref["fully_denoised"])
        assert torch.equal(out["latents"].cpu(), ref["latents"]), (out["latents"].cpu().float() -
                                                                   ref["latents"].float()).abs().max()


def test_call_carries_state_through_scheduler_handles(cuda):
    """``__call__`` with the per-frame handles of ``parepare_schedulers``: three successive windows over overlapping frames
    == the reference's pattern with per-frame scheduler copies (PIPE:535)."""
    from oracle.dpm_solver_oracle import denoise_window_oracle_per_frame
    from oracle.unipc_oracle import UniPCOracle
    pipe, unet = _tiny_pipe()
    n, h, w = 5, 8, 8
    g = torch.Generator().manual_seed(24)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    pix, plk, lat = r(n, 4, h, w), r(n, 6, h, w), r(n, 4, h, w)
    skel = (torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16)
    mask = torch.ones(n, 1, h, w, dtype=torch.bfloat16)
    mask[0] = 0
    handles, timesteps = pipe.parepare_schedulers(12, n)
    orc = UniPCOracle(pipe.scheduler.config)
    orc.set_timesteps(12)
    copies = [copy.deepcopy(orc) for _ in range(n)]
    ti = torch.zeros(n, dtype=torch.long)
    lat_ours, lat_ref = lat.clone().cuda(), lat.clone()
    for window in (torch.tensor([0, 1, 2, 3]), torch.tensor([0, 2, 3, 4]), torch.tensor([0, 1, 3, 4])):
        got = pipe(pixel_values_latents=pix[window], plucker_embeds_latents=plk[window], skeletons_latents=skel[window],
                   cond_masks_latents=mask[window], latents=lat_ours[window.cuda()], domains=["spatial"],
                   num_inference_steps=2, schedulers=[handles[i] for i in window], timesteps=timesteps,
                   timestep_indices=ti[window], guidance_scale=2.0)
        want, _ = denoise_window_oracle_per_frame(
            _unet_cb(unet), [copies[i] for i in window], latents=lat_ref[window], pixel_latents=pix[window],
            plucker=plk[window], skeletons=skel[window], cond_mask=mask[window], timestep_indices=ti[window],
            domain="spatial", guidance_scale=2.0, num_inference_steps=2)
        tgt = window[mask[window, 0, 0, 0] != 0]
        ti[tgt] += 2
        lat_ours[window.cuda()] = got
        lat_ref[window] = want
        torch.cuda.synchronize()
        assert torch.equal(got.cpu(), want), (got.cpu().float() - want.float()).abs().max()
    assert handles[2].state.lower_order_nums.cpu().tolist() == [c.lower_order_nums for c in copies]


def _tiny_checkpoint(tmp_path):
    from safetensors.torch import save_file
    cfg = UNetConfig.tiny()
    os.makedirs(tmp_path / "unet")
    os.makedirs(tmp_path / "scheduler")
    json.dump(dict(in_channels=11, out_channels=4, block_out_channels=[64, 128, 256, 256], attention_head_dim=[1, 2, 4, 4],
                   cross_attention_dim=None, use_linear_projection=True, enable_pose_encoder=True, enable_tem_embeds=True,
                   layers_per_block=2, num_3d_attn_blocks=3), open(tmp_path / "unet" / "config.json", "w"))
    json.dump({"_class_name": "UniPCMultistepScheduler", "beta_schedule": "scaled_linear", "beta_start": 0.00085,
               "beta_end": 0.012, "solver_order": 2, "prediction_type": "epsilon", "predict_x0": True,
               "solver_type": "bh2", "timestep_spacing": "leading", "steps_offset": 1, "use_karras_sigmas": False,
               "lower_order_final": True, "disable_corrector": [], "solver_p": None, "final_sigmas_type": "zero"},
              open(tmp_path / "scheduler" / "scheduler_config.json", "w"))
    save_file({k: v.contiguous() for k, v in random_state_dict(cfg, seed=1).items()},
              str(tmp_path / "unet" / "diffusion_pytorch_model.safetensors"))


def test_load_pipelines_with_unipc_scheduler(cuda, tmp_path):
    from diffuman4d_b200.loader import load_pipelines
    from diffuman4d_b200.scheduler import UniPCTables
    _tiny_checkpoint(tmp_path)
    (pipe,) = load_pipelines(model_dir=str(tmp_path), torch_dtype="bf16", gpu_ids=[0])
    assert isinstance(pipe.scheduler, UniPCTables) and pipe.scheduler.config.beta_schedule == "scaled_linear"
    n, h, w = 6, 8, 8
    g = torch.Generator().manual_seed(25)
    mask = torch.ones(n, 1, h, w)
    mask[[1, 4]] = 0
    out = pipe.sliding_iterative_denoise(
        pixel_values_latents=torch.randn(n, 4, h, w, generator=g), plucker_embeds=torch.randn(n, 6, h, w, generator=g),
        skeletons=torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1, cond_masks=mask, latents=None, domain="spatial",
        timestep_indices=torch.zeros(n, dtype=torch.long), window_size=2, sliding_stride=1, bidirectional=True,
        alternation_rounds=1, guidance_scale=2.0, generator=torch.Generator(device="cuda").manual_seed(0))
    ti = out["timestep_indices"].cpu()
    assert ti[[1, 4]].eq(0).all() and ti[[0, 2, 3, 5]].eq(4).all() and out["fully_denoised"].cpu()[[0, 2, 3, 5]].all()
    assert torch.isfinite(out["latents"].float()).all()


def test_sampler_drives_a_unipc_pipeline(cuda):
    sys.path.insert(0, GOLD)
    from pool_vae import PoolVAE
    from synthetic_dataset import SyntheticSpaTemDataset
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.sampler import B200SlidingIterativeSampler
    from diffuman4d_b200.unet import B200MultiviewUNet

    cfg = UNetConfig.tiny()
    unet = B200MultiviewUNet(cfg, 0).load_state_dict(random_state_dict(cfg, seed=1))
    pipe = B200Diffuman4DPipeline(unet, UniPCConfig(), vae=PoolVAE())
    ds = SyntheticSpaTemDataset(8, h=16, w=16)
    s = B200SlidingIterativeSampler(ds, [pipe], output_dir=None, spa_label_range=[0, 6, 1], tem_label_range=[0, 4, 1],
                                    input_spa_labels=[1, 4], window_size=2, sliding_stride=1, bidirectional=True,
                                    alternation_rounds=3, guidance_scale=2.0)
    s.execute_tasks()
    torch.cuda.synchronize()
    assert s.grid_latents.shape == (6, 4, 4, 16, 16) and torch.isfinite(s.grid_latents.float()).all()
    ti = s.grid_timestep_indices.cpu()
    n_inf = 2 * 1 // 1 * 2 * 3                                   # window * steps / stride, bidirectional, 3 rounds
    for v, spa in enumerate(s.spa_labels):
        expect = 0 if spa in s.input_spa_labels else n_inf      # every target cell fully denoised, inputs untouched
        assert (ti[v] == expect).all(), (spa, ti[v])
