"""GPU tests of the PNDM step (upstream PNDMScheduler with skip_prk_steps): the fused CFG + step kernel against PNDMOracle
on the same bf16 inputs with frames at every counter state in one launch (bit for bit when emulating bf16, against fp64
arithmetic in the fp32 mode), the window step through the C ABI and the sliding loop against the oracle driven by the
same CUDA UNet, ``__call__`` with the per-frame handles, load_pipelines on a checkpoint that names the scheduler, and the
device sampler."""
import copy
import json
import os
import sys

import pytest
import torch

from diffuman4d_b200.config import PNDMConfig, UNetConfig
from diffuman4d_b200.weights import random_state_dict

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")
SD_PNDM = dict(beta_schedule="scaled_linear", beta_start=0.00085, beta_end=0.012, set_alpha_to_one=False,
               steps_offset=1, timestep_spacing="leading")


def _bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def _positions(counter: int) -> range:
    """Ring positions of upstream's ``ets`` after ``counter`` steps, oldest first (position p is in plane ets{p % 4})."""
    return range(max(0, counter - 5), max(1, counter - 1)) if counter > 0 else range(0)


def _oracle_frame(cfg, n, counter, ets_planes, cur_sample):
    """A per-frame oracle scheduler standing where the frame's own copy stands after ``counter`` steps, its history read
    from the ring planes."""
    from oracle.pndm_oracle import PNDMOracle
    s = PNDMOracle(cfg)
    s.set_timesteps(n)
    s.counter = counter
    s.ets = [ets_planes[p % 4] for p in _positions(counter)]
    s.cur_sample = cur_sample if counter == 1 else None
    return s


@pytest.mark.parametrize("pred", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("cfg_on", [True, False])
def test_cfg_pndm_step_vs_oracle(cuda, pred, cfg_on):
    from diffuman4d_b200.ops import cfg_pndm_step
    from diffuman4d_b200.scheduler import PNDMTables
    n = 10
    cfg = PNDMConfig(**{**SD_PNDM, "prediction_type": pred})
    F, h, w = 9, 9, 13                                                    # 4*h*w = 468: no multiple of the block size
    g = torch.Generator().manual_seed(31)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    noise, lat = r((2 if cfg_on else 1) * F, 4, h, w), r(F, 4, h, w)
    ets, cur = [r(F, 4, h, w) for _ in range(4)], r(F, 4, h, w)
    lat[0] *= 60   # a high-noise frame at step 0
    mask = torch.ones(F, 1, h, w, dtype=torch.bfloat16)
    mask[6] = 0
    # frame: counters 0, 1, 2, 3, 4, 7 (the ring has wrapped) | 6 cond | 7: fresh at a late row | 8: counter 5 at the
    # last row the reference reaches
    ti = torch.tensor([0, 1, 2, 3, 4, 7, 3, 6, 9])
    counter = torch.tensor([0, 1, 2, 3, 4, 7, 2, 0, 5], dtype=torch.int32)
    tables = PNDMTables(cfg, device="cuda:0")
    tables.set_timesteps(n)
    guidance = 2.0 if cfg_on else 1.0
    for emulate in (True, False):
        dt = torch.bfloat16 if emulate else torch.float64   # fp32 mode: against fp64 arithmetic on fp32 tables
        if cfg_on:
            u, c = noise.to(dt).chunk(2)
            eps = u + 2.0 * (c - u)          # 2.0 and the differences are exact roundings in either dtype
        else:
            eps = noise.to(dt)
        ref = []
        ref_ets = [e.to(dt).clone() for e in ets]
        ref_cur = cur.to(dt).clone()
        for j in range(F):
            if mask[j, 0, 0, 0] == 0:
                ref.append(lat[j:j + 1].to(dt))
                continue
            cnt = int(counter[j])
            s = _oracle_frame(cfg, n, cnt, [e[j:j + 1].to(dt) for e in ets], cur[j:j + 1].to(dt))
            ref.append(s.step(eps[j:j + 1], int(s.timesteps[ti[j]]), lat[j:j + 1].to(dt)))
            if cnt != 1:
                ref_ets[(0 if cnt == 0 else cnt - 1) % 4][j] = eps[j]
            if cnt == 0:
                ref_cur[j] = lat[j].to(dt)
            assert s.counter == cnt + 1
        ets_d, cur_d = [e.cuda() for e in ets], cur.cuda()
        out, ti_out, cnt_out = cfg_pndm_step(noise.cuda(), lat.cuda(), mask.cuda(), ti.cuda(), ets_d, cur_d,
                                             counter.cuda(), tables.c_struct(emulate), guidance, cfg_on)
        torch.cuda.synchronize()
        assert ti_out.cpu().tolist() == [1, 2, 3, 4, 5, 8, 0, 7, 10]
        assert cnt_out.cpu().tolist() == [1, 2, 3, 4, 5, 8, 2, 1, 6]
        got = {"out": (out, torch.cat(ref)), "cur_sample": (cur_d, ref_cur)}
        got.update({f"ets{k}": (ets_d[k], ref_ets[k]) for k in range(4)})
        for name, (g_d, want) in got.items():
            g_c = g_d.cpu().double()
            want = want.double()
            if emulate:
                assert torch.equal(g_c, want), (name, (g_c - want).abs().max())
            else:   # one bf16 rounding of the stored result, plus fp32 arithmetic relative to the largest input
                bound = _bf16_ulp(want) + 1e-5 * max(want.abs().max().item(), lat.abs().max().item())
                assert ((g_c - want).abs() <= bound).all(), (name, ((g_c - want).abs() - bound).max())
        for k in range(4):   # cond: untouched
            assert torch.equal(ets_d[k].cpu()[6], ets[k][6])
        assert torch.equal(cur_d.cpu()[6], cur[6])


def _tiny_pipe(emulate=True, **kw):
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.unet import B200MultiviewUNet
    cfg = UNetConfig.tiny()
    unet = B200MultiviewUNet(cfg, device=0).load_state_dict(random_state_dict(cfg, seed=1, dtype=torch.bfloat16))
    return B200Diffuman4DPipeline(unet, PNDMConfig(**kw), emulate_bf16_scheduler=emulate), unet


def _unet_cb(unet):
    def cb(x, t, sk, doms, nf):
        return unet(x.cuda(), t.cuda(), sk.cuda(), doms, nf, return_dict=False)[0].cpu()
    return cb


def _assert_state_matches(state, frames, copies):
    """The device state of ``frames`` (indices into ``state``) equals the per-frame oracle copies: counter, the kept
    outputs in their ring planes, and cur_sample where upstream still holds one."""
    for j, c in zip(frames, copies):
        assert int(state.counter[j]) == c.counter
        for p, e in zip(_positions(c.counter), c.ets):
            assert torch.equal(getattr(state, f"ets{p % 4}").cpu()[j:j + 1], e), (j, p)
        if c.cur_sample is not None:
            assert torch.equal(state.cur_sample.cpu()[j:j + 1], c.cur_sample), j


def test_denoise_window_pndm_vs_oracle_bit_exact(cuda):
    """``d4d_denoise_window_pndm`` (five steps of one window, staggered step indices, fresh state, so that the frames
    pass through counters 0 .. 4) against the oracle's window step with per-frame scheduler copies, both driven by the
    same CUDA UNet; the state comes back updated."""
    from oracle.dpm_solver_oracle import denoise_window_oracle_per_frame
    from oracle.pndm_oracle import PNDMOracle
    pipe, unet = _tiny_pipe(**SD_PNDM)
    n, h, w = 5, 8, 8
    g = torch.Generator().manual_seed(32)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    pix, plk, lat = r(n, 4, h, w), r(n, 6, h, w), r(n, 4, h, w)
    skel = (torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16)
    mask = torch.ones(n, 1, h, w, dtype=torch.bfloat16)
    mask[1] = 0
    ti = torch.tensor([0, 0, 1, 2, 4])
    handles, _ = pipe.parepare_schedulers(10, n)
    state = handles[0].state.take(torch.arange(n), h, w)
    orc = PNDMOracle(pipe.scheduler.config)
    orc.set_timesteps(10)
    copies = [copy.deepcopy(orc) for _ in range(n)]
    want, want_ti = denoise_window_oracle_per_frame(
        _unet_cb(unet), copies, latents=lat.clone(), pixel_latents=pix, plucker=plk, skeletons=skel, cond_mask=mask,
        timestep_indices=ti, domain="spatial", guidance_scale=2.0, num_inference_steps=5)
    lat_d, ti_d = lat.cuda(), ti.cuda()
    pipe.denoise_window(latents=lat_d, pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skel,
                        cond_masks_latents=mask, timestep_indices=ti_d, domain="spatial", guidance_scale=2.0,
                        num_inference_steps=5, solver_state=state)
    torch.cuda.synchronize()
    assert torch.equal(ti_d.cpu(), want_ti)
    assert torch.equal(lat_d.cpu(), want), (lat_d.cpu().float() - want.float()).abs().max()
    assert state.counter.cpu().tolist() == [c.counter for c in copies]
    _assert_state_matches(state, (0, 2, 3, 4), [copies[j] for j in (0, 2, 3, 4)])


@pytest.mark.parametrize("kw", [SD_PNDM, dict(prediction_type="v_prediction", timestep_spacing="trailing"),
                                dict(timestep_spacing="linspace", set_alpha_to_one=True)])
def test_sliding_iterative_denoise_pndm_vs_oracle_bit_exact(cuda, kw):
    """Per-frame solver state carried across the windows of a task and reset per task: a spatial and then a bidirectional
    temporal task on one pipeline, against the oracle's sliding loop (per-frame scheduler copies) with our UNet.  The
    task's final state planes are compared too."""
    from oracle.dpm_solver_oracle import sliding_iterative_denoise_oracle_per_frame
    from oracle.pndm_oracle import PNDMOracle
    pipe, unet = _tiny_pipe(**kw)
    handles = []
    prepare = pipe.parepare_schedulers
    pipe.parepare_schedulers = lambda *a: handles.append(prepare(*a)[0]) or (handles[-1], None)
    copies = []

    class RecordingPNDM(PNDMOracle):   # keeps the per-frame copies the oracle's loop makes
        def __deepcopy__(self, memo):
            c = PNDMOracle.__new__(RecordingPNDM)
            c.__dict__.update(copy.deepcopy(self.__dict__, memo))
            copies.append(c)
            return c

    h = w = 8
    g = torch.Generator().manual_seed(33)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    # each target frame takes per-alternation steps: 8 (the ring wraps) in the spatial task, 4 in the temporal one
    for domain, n_in, n_tg, ws, stride, bidir, rounds in (("spatial", 2, 4, 4, 1, True, 2),
                                                          ("temporal", 3, 3, 2, 1, True, 1)):
        n = n_in + n_tg
        mask = torch.ones(n, 1, h, w, dtype=torch.bfloat16)
        mask[:n_in] = 0
        args = dict(pixel_latents=r(n, 4, h, w), plucker=r(n, 6, h, w),
                    skeletons=(torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16), cond_mask=mask,
                    latents=r(n, 4, h, w), domain=domain, timestep_indices=torch.zeros(n, dtype=torch.long),
                    window_size=ws, sliding_stride=stride, bidirectional=bidir, alternation_rounds=rounds,
                    guidance_scale=2.0)
        copies.clear()
        ref = sliding_iterative_denoise_oracle_per_frame(_unet_cb(unet), RecordingPNDM(pipe.scheduler.config), **args,
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
        assert len(copies) == n and max(c.counter for c in copies) >= 4
        state = handles[-1][0].state
        _assert_state_matches(state, range(n), copies)


def test_call_carries_state_through_scheduler_handles(cuda):
    """``__call__`` with the per-frame handles of ``parepare_schedulers``: three successive windows over overlapping frames
    == the reference's pattern with per-frame scheduler copies (PIPE:535); the first window starts its frames at
    nonzero timestep indices with fresh counters."""
    from oracle.dpm_solver_oracle import denoise_window_oracle_per_frame
    from oracle.pndm_oracle import PNDMOracle
    pipe, unet = _tiny_pipe(**SD_PNDM)
    n, h, w = 5, 8, 8
    g = torch.Generator().manual_seed(34)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    pix, plk, lat = r(n, 4, h, w), r(n, 6, h, w), r(n, 4, h, w)
    skel = (torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16)
    mask = torch.ones(n, 1, h, w, dtype=torch.bfloat16)
    mask[0] = 0
    handles, timesteps = pipe.parepare_schedulers(12, n)
    orc = PNDMOracle(pipe.scheduler.config)
    orc.set_timesteps(12)
    copies = [copy.deepcopy(orc) for _ in range(n)]
    ti = torch.tensor([0, 2, 1, 3, 2])
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
    state = handles[0].state
    assert state.counter.cpu().tolist() == [c.counter for c in copies]
    _assert_state_matches(state, range(1, n), copies[1:])


def _tiny_checkpoint(tmp_path):
    from safetensors.torch import save_file
    cfg = UNetConfig.tiny()
    os.makedirs(tmp_path / "unet")
    os.makedirs(tmp_path / "scheduler")
    json.dump(dict(in_channels=11, out_channels=4, block_out_channels=[64, 128, 256, 256], attention_head_dim=[1, 2, 4, 4],
                   cross_attention_dim=None, use_linear_projection=True, enable_pose_encoder=True, enable_tem_embeds=True,
                   layers_per_block=2, num_3d_attn_blocks=3), open(tmp_path / "unet" / "config.json", "w"))
    # Stable Diffusion v1.5's scheduler_config.json
    json.dump({"_class_name": "PNDMScheduler", "_diffusers_version": "0.6.0", "beta_end": 0.012,
               "beta_schedule": "scaled_linear", "beta_start": 0.00085, "num_train_timesteps": 1000,
               "set_alpha_to_one": False, "skip_prk_steps": True, "steps_offset": 1, "trained_betas": None,
               "clip_sample": False}, open(tmp_path / "scheduler" / "scheduler_config.json", "w"))
    save_file({k: v.contiguous() for k, v in random_state_dict(cfg, seed=1).items()},
              str(tmp_path / "unet" / "diffusion_pytorch_model.safetensors"))


def test_load_pipelines_with_pndm_scheduler(cuda, tmp_path):
    from diffuman4d_b200.loader import load_pipelines
    from diffuman4d_b200.scheduler import PNDMTables
    _tiny_checkpoint(tmp_path)
    (pipe,) = load_pipelines(model_dir=str(tmp_path), torch_dtype="bf16", gpu_ids=[0])
    assert isinstance(pipe.scheduler, PNDMTables) and pipe.scheduler.config == PNDMConfig(**SD_PNDM)
    n, h, w = 6, 8, 8
    g = torch.Generator().manual_seed(35)
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


def test_sampler_drives_a_pndm_pipeline(cuda):
    sys.path.insert(0, GOLD)
    from pool_vae import PoolVAE
    from synthetic_dataset import SyntheticSpaTemDataset
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.sampler import B200SlidingIterativeSampler
    from diffuman4d_b200.unet import B200MultiviewUNet

    cfg = UNetConfig.tiny()
    unet = B200MultiviewUNet(cfg, 0).load_state_dict(random_state_dict(cfg, seed=1))
    pipe = B200Diffuman4DPipeline(unet, PNDMConfig(**SD_PNDM), vae=PoolVAE())
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
