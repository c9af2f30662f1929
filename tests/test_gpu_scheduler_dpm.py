"""GPU tests of the DPM-Solver++ step (upstream DPMSolverMultistepScheduler, dpmsolver++ / midpoint): the fused CFG + step
kernel against DPMSolverOracle on the same bf16 inputs, the window loop with per-frame solver state against the oracle's
sliding loop driven by the same CUDA UNet, and load_pipelines on a checkpoint that names the scheduler."""
import copy
import json
import os

import pytest
import torch

from diffuman4d_b200.config import DPMSolverConfig, UNetConfig
from diffuman4d_b200.weights import random_state_dict

pytestmark = pytest.mark.gpu


def _bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def _oracle_frame(cfg, n, idx, lon, x0_prev):
    """A per-frame oracle scheduler standing where the frame's own copy stands after `idx` steps."""
    from oracle.dpm_solver_oracle import DPMSolverOracle
    s = DPMSolverOracle(cfg)
    s.set_timesteps(n)
    s.step_index = idx
    s.lower_order_nums = lon
    s.model_outputs[-1] = x0_prev
    return s


@pytest.mark.parametrize("pred", ["epsilon", "v_prediction", "sample"])
@pytest.mark.parametrize("cfg_on", [True, False])
def test_cfg_dpm_step_vs_oracle(cuda, pred, cfg_on):
    from diffuman4d_b200.ops import cfg_dpm_step
    from diffuman4d_b200.scheduler import DPMSolverTables
    n = 10
    cfg = DPMSolverConfig(prediction_type=pred, lower_order_final=False)   # final sigma 0 => last step first order
    F, h, w = 6, 9, 13                                                    # 4*h*w = 468: no multiple of the block size
    g = torch.Generator().manual_seed(11)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    noise, lat, x0_prev = r((2 if cfg_on else 1) * F, 4, h, w), r(F, 4, h, w), r(F, 4, h, w)
    lat[0] *= 60   # a high-noise frame at step 0
    mask = torch.ones(F, 1, h, w, dtype=torch.bfloat16)
    mask[2] = 0
    # frame: 0 first step | 1 second order | 2 cond | 3 first step mid-schedule | 4 second order | 5 final step (sigma 0)
    ti = torch.tensor([0, 1, 4, 5, 8, 9])
    lon = torch.tensor([0, 1, 2, 0, 2, 2], dtype=torch.int32)
    tables = DPMSolverTables(cfg, device="cuda:0")
    tables.set_timesteps(n)
    guidance = 2.0 if cfg_on else 1.0
    for emulate in (True, False):
        dt = torch.bfloat16 if emulate else torch.float32
        if cfg_on:
            u, c = noise.to(dt).chunk(2)
            eps = u + 2.0 * (c - u)          # 2.0 and the differences are exact roundings in either dtype
        else:
            eps = noise.to(dt)
        ref, ref_x0 = [], []
        for j in range(F):
            if mask[j, 0, 0, 0] == 0:
                ref.append(lat[j:j + 1].to(dt))
                ref_x0.append(x0_prev[j:j + 1].to(dt))
                continue
            s = _oracle_frame(cfg, n, int(ti[j]), int(lon[j]), x0_prev[j:j + 1].to(dt))
            ref.append(s.step(eps[j:j + 1], int(s.timesteps[ti[j]]), lat[j:j + 1].to(dt)))
            ref_x0.append(s.model_outputs[-1])
        ref, ref_x0 = torch.cat(ref).float(), torch.cat(ref_x0).float()
        x0_d = x0_prev.cuda()
        out, ti_out, lon_out = cfg_dpm_step(noise.cuda(), lat.cuda(), mask.cuda(), ti.cuda(), x0_d, lon.cuda(),
                                            tables.c_struct(emulate), guidance, cfg_on)
        torch.cuda.synchronize()
        assert ti_out.cpu().tolist() == [1, 2, 0, 6, 9, 10]
        assert lon_out.cpu().tolist() == [1, 2, 2, 1, 2, 2]
        out, x0_d = out.cpu().float(), x0_d.cpu().float()
        assert torch.equal(x0_d[2], x0_prev[2].float())                 # cond frame: history untouched
        if emulate:
            assert torch.equal(out, ref), (out - ref).abs().max()
            assert torch.equal(x0_d, ref_x0), (x0_d - ref_x0).abs().max()
        else:
            for got, want in ((out, ref), (x0_d, ref_x0)):
                bound = 1e-6 * want.abs().max() + _bf16_ulp(want)
                assert ((got - want).abs() <= bound).all(), ((got - want).abs() - bound).max()
        # the final step with sigma 0 returns the data prediction itself
        assert torch.equal(out[5], x0_d[5])


def _tiny_pipe(emulate=True, **kw):
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.unet import B200MultiviewUNet
    cfg = UNetConfig.tiny()
    unet = B200MultiviewUNet(cfg, device=0).load_state_dict(random_state_dict(cfg, seed=1, dtype=torch.bfloat16))
    return B200Diffuman4DPipeline(unet, DPMSolverConfig(**kw), emulate_bf16_scheduler=emulate), unet


def test_sliding_iterative_denoise_dpm_vs_oracle_bit_exact(cuda):
    """Per-frame solver state carried across the windows of a task and reset per task: a spatial and then a bidirectional
    temporal task on one pipeline, against the oracle's sliding loop (per-frame scheduler copies) with our UNet."""
    from oracle.dpm_solver_oracle import DPMSolverOracle, sliding_iterative_denoise_oracle_per_frame
    pipe, unet = _tiny_pipe(final_sigmas_type="sigma_min", lower_order_final=False)

    def unet_cb(x, t, sk, doms, nf):
        return unet(x.cuda(), t.cuda(), sk.cuda(), doms, nf, return_dict=False)[0].cpu()

    h = w = 8
    g = torch.Generator().manual_seed(12)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    for domain, n_in, n_tg, ws, stride, bidir, rounds in (("spatial", 2, 4, 2, 1, False, 2),
                                                          ("temporal", 3, 3, 2, 1, True, 1)):
        n = n_in + n_tg
        mask = torch.ones(n, 1, h, w, dtype=torch.bfloat16)
        mask[:n_in] = 0
        kw = dict(pixel_latents=r(n, 4, h, w), plucker=r(n, 6, h, w),
                  skeletons=(torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16), cond_mask=mask,
                  latents=r(n, 4, h, w), domain=domain, timestep_indices=torch.zeros(n, dtype=torch.long),
                  window_size=ws, sliding_stride=stride, bidirectional=bidir, alternation_rounds=rounds,
                  guidance_scale=2.0)
        ref = sliding_iterative_denoise_oracle_per_frame(unet_cb, DPMSolverOracle(pipe.scheduler.config), **kw,
                                                         enable_pose_encoder=True)
        out = pipe.sliding_iterative_denoise(
            pixel_values_latents=kw["pixel_latents"], plucker_embeds=kw["plucker"], skeletons=kw["skeletons"],
            cond_masks=mask, latents=kw["latents"], domain=domain, timestep_indices=kw["timestep_indices"],
            window_size=ws, sliding_stride=stride, bidirectional=bidir, alternation_rounds=rounds, guidance_scale=2.0)
        torch.cuda.synchronize()
        assert torch.equal(out["timestep_indices"].cpu(), ref["timestep_indices"])
        assert torch.equal(out["fully_denoised"].cpu(), ref["fully_denoised"])
        assert torch.equal(out["latents"].cpu(), ref["latents"]), (out["latents"].cpu().float() -
                                                                   ref["latents"].float()).abs().max()


def test_call_carries_state_through_scheduler_handles(cuda):
    """``__call__`` with the per-frame handles of ``parepare_schedulers``: two successive windows over overlapping frames
    == the reference's pattern with per-frame scheduler copies (PIPE:535)."""
    from oracle.dpm_solver_oracle import DPMSolverOracle, denoise_window_oracle_per_frame
    pipe, unet = _tiny_pipe()
    n, h, w = 5, 8, 8
    g = torch.Generator().manual_seed(13)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    pix, plk, lat = r(n, 4, h, w), r(n, 6, h, w), r(n, 4, h, w)
    skel = (torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16)
    mask = torch.ones(n, 1, h, w, dtype=torch.bfloat16)
    mask[0] = 0
    handles, timesteps = pipe.parepare_schedulers(12, n)
    orc = DPMSolverOracle(pipe.scheduler.config)
    orc.set_timesteps(12)
    copies = [copy.deepcopy(orc) for _ in range(n)]
    ti = torch.zeros(n, dtype=torch.long)
    lat_ours, lat_ref = lat.clone().cuda(), lat.clone()

    def unet_cb(x, t, sk, doms, nf):
        return unet(x.cuda(), t.cuda(), sk.cuda(), doms, nf, return_dict=False)[0].cpu()

    for window in (torch.tensor([0, 1, 2, 3]), torch.tensor([0, 2, 3, 4]), torch.tensor([0, 1, 3, 4])):
        got = pipe(pixel_values_latents=pix[window], plucker_embeds_latents=plk[window], skeletons_latents=skel[window],
                   cond_masks_latents=mask[window], latents=lat_ours[window.cuda()], domains=["spatial"],
                   num_inference_steps=2, schedulers=[handles[i] for i in window], timesteps=timesteps,
                   timestep_indices=ti[window], guidance_scale=2.0)
        want, _ = denoise_window_oracle_per_frame(
            unet_cb, [copies[i] for i in window], latents=lat_ref[window], pixel_latents=pix[window], plucker=plk[window],
            skeletons=skel[window], cond_mask=mask[window], timestep_indices=ti[window], domain="spatial",
            guidance_scale=2.0, num_inference_steps=2)
        tgt = window[mask[window, 0, 0, 0] != 0]
        ti[tgt] += 2
        lat_ours[window.cuda()] = got
        lat_ref[window] = want
        torch.cuda.synchronize()
        assert torch.equal(got.cpu(), want), (got.cpu().float() - want.float()).abs().max()
    assert handles[2].state.lower_order_nums.cpu().tolist() == [c.lower_order_nums for c in copies]


def test_load_pipelines_with_dpm_solver_scheduler(cuda, tmp_path):
    from safetensors.torch import save_file
    from diffuman4d_b200.loader import load_pipelines
    from diffuman4d_b200.scheduler import DPMSolverTables
    cfg = UNetConfig.tiny()
    os.makedirs(tmp_path / "unet")
    os.makedirs(tmp_path / "scheduler")
    json.dump(dict(in_channels=11, out_channels=4, block_out_channels=[64, 128, 256, 256], attention_head_dim=[1, 2, 4, 4],
                   cross_attention_dim=None, use_linear_projection=True, enable_pose_encoder=True, enable_tem_embeds=True,
                   layers_per_block=2, num_3d_attn_blocks=3), open(tmp_path / "unet" / "config.json", "w"))
    json.dump({"_class_name": "DPMSolverMultistepScheduler", "beta_schedule": "scaled_linear", "beta_start": 0.00085,
               "beta_end": 0.012, "solver_order": 2, "prediction_type": "epsilon", "algorithm_type": "dpmsolver++",
               "solver_type": "midpoint", "timestep_spacing": "leading", "steps_offset": 1, "use_karras_sigmas": False,
               "lower_order_final": True, "final_sigmas_type": "zero"},
              open(tmp_path / "scheduler" / "scheduler_config.json", "w"))
    save_file({k: v.contiguous() for k, v in random_state_dict(cfg, seed=1).items()},
              str(tmp_path / "unet" / "diffusion_pytorch_model.safetensors"))
    (pipe,) = load_pipelines(model_dir=str(tmp_path), torch_dtype="bf16", gpu_ids=[0])
    assert isinstance(pipe.scheduler, DPMSolverTables) and pipe.scheduler.config.beta_schedule == "scaled_linear"
    n, h, w = 6, 8, 8
    g = torch.Generator().manual_seed(14)
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
