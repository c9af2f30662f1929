"""GPU tests of the DDPM step (upstream DDPMScheduler, fixed variances) and its counter-based noise.

* ``d4d_op_ddpm_noise`` against the host Philox + Box-Muller of oracle/ddpm_oracle.py: fp32 results equal, except at
  most 1 ulp on at most 1e-6 of the elements (fp64 log / cos / sin may differ by an ulp between the device and the host).
* The fused CFG + step kernel against ``DDPMOracle`` fed the host noise: bit for bit when emulating bf16, within one bf16
  rounding in the fp32 mode; every prediction type, clip on and off, the three variance types, the last row (no noise).
* The window step through the C ABI and a whole sliding task against the per-frame oracles driven by the same UNet.
* The same seed gives the same bits; another seed changes every target frame and no conditioning frame.
* The frame-sharded window, the CFG split and the CFG grid (one-rank loopbacks) are bit-identical to the single-GPU
  window and sliding loop.
* Several processes on one GPU (gloo, exchange buffers mapped across processes with cudaIpc): the CFG split on 2 ranks,
  the CFG grid on 4 (R = 2) and the frame-sharded window on 2 (two frames per rank, each with its shard of the frame
  ids) give every rank the single-GPU bits of a window step and of a sliding task whose ranks start from different
  generators, so the initial noise and the noise seed must be rank 0's.
* ``load_pipelines`` on a checkpoint whose scheduler is ``DDPMScheduler``.
"""
import copy
import json
import os

import pytest
import torch

from diffuman4d_b200.config import DDPMConfig, UNetConfig
from diffuman4d_b200.weights import random_state_dict

pytestmark = pytest.mark.gpu

H = W = 8


def _bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def test_device_noise_equals_host_noise(cuda):
    from diffuman4d_b200.ops import ddpm_noise
    from oracle.ddpm_oracle import ddpm_noise as host_noise
    total = mismatched = 0
    for seed, h, w in ((0, 64, 64), (2 ** 64 - 1, 16, 24), (-5, 9, 13), (0x0123456789ABCDEF, 32, 32)):
        ids = torch.tensor([0, 1, 7, 2 ** 31 + 3, 12345])
        ti = torch.tensor([0, 3, 3, 999, 17])
        got = ddpm_noise(seed, ids.cuda(), ti.cuda(), h, w).cpu()
        want = host_noise(seed, ids, ti, h, w, torch.float32)
        diff = got.view(torch.int32) - want.view(torch.int32)
        assert diff.abs().max() <= 1, seed
        mismatched += int((diff != 0).sum())
        total += diff.numel()
    assert total > 10 ** 5 and mismatched <= max(1, total // 10 ** 6), (mismatched, total)


def _oracle(cfg, n, seed=0):
    from oracle.ddpm_oracle import DDPMOracle
    s = DDPMOracle(cfg, seed=seed)
    s.set_timesteps(n)
    return s


CASES = [dict(), dict(prediction_type="v_prediction"), dict(prediction_type="sample", clip_sample=False),
         dict(clip_sample=False, variance_type="fixed_small_log"), dict(variance_type="fixed_large", clip_sample_range=0.5),
         dict(prediction_type="v_prediction", variance_type="fixed_large", timestep_spacing="trailing"),
         dict(beta_schedule="scaled_linear", beta_start=0.00085, beta_end=0.012, timestep_spacing="linspace")]


@pytest.mark.parametrize("kw", CASES, ids=[",".join(f"{k}={v}" for k, v in c.items()) or "default" for c in CASES])
@pytest.mark.parametrize("cfg_on", [True, False])
def test_cfg_ddpm_step_vs_oracle(cuda, kw, cfg_on):
    from diffuman4d_b200.ops import cfg_ddpm_step
    from diffuman4d_b200.scheduler import DDPMTables
    from oracle.ddpm_oracle import ddpm_noise as host_noise
    n, seed = 10, 0x5EED5EED5EED
    cfg = DDPMConfig(**kw)
    ti = torch.tensor([0, 1, 4, 9, 5, 8, 3])          # frame 4 conditions; row 9 is the last
    ids = torch.tensor([3, 0, 9, 4, 1, 2, 7])          # the frames' indices in their task
    F, h, w = len(ti), 9, 13                           # 4*h*w = 468: no multiple of the block size
    g = torch.Generator().manual_seed(41)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    noise, lat = r((2 if cfg_on else 1) * F, 4, h, w), r(F, 4, h, w)
    lat[0] *= 30
    mask = torch.ones(F, 1, h, w, dtype=torch.bfloat16)
    mask[4] = 0
    tables = DDPMTables(cfg, device="cuda:0")
    tables.set_timesteps(n)
    guidance = 2.0 if cfg_on else 1.0
    for emulate in (True, False):
        dt = torch.bfloat16 if emulate else torch.float64   # fp32 mode: against fp64 arithmetic on fp32 tables
        eps = noise.to(dt)
        if cfg_on:
            u, c = eps.chunk(2)
            eps = u + 2.0 * (c - u)
        ref = []
        for j in range(F):
            if mask[j, 0, 0, 0] == 0:
                ref.append(lat[j:j + 1].to(dt))
                continue
            s = _oracle(cfg, n)
            z = host_noise(seed, [int(ids[j])], [int(ti[j])], h, w, torch.bfloat16 if emulate else torch.float64)
            ref.append(s.step(eps[j:j + 1], int(s.timesteps[ti[j]]), lat[j:j + 1].to(dt), noise=z))
        out, ti_out = cfg_ddpm_step(noise.cuda(), lat.cuda(), mask.cuda(), ti.cuda(), ids.cuda(),
                                    tables.c_struct(emulate, seed), guidance, cfg_on)
        torch.cuda.synchronize()
        assert ti_out.cpu().tolist() == [0 if j == 4 else int(ti[j]) + 1 for j in range(F)]
        got, want = out.cpu().double(), torch.cat(ref).double()
        assert torch.equal(got[4], lat[4].double())
        if emulate:
            assert torch.equal(got, want), (got - want).abs().max()
        else:   # one bf16 rounding of the stored result, plus fp32 arithmetic relative to the largest value
            bound = _bf16_ulp(want) + 1e-6 * max(want.abs().max().item(), lat.abs().max().item())
            assert ((got - want).abs() <= bound).all(), ((got - want).abs() - bound).max()
        if emulate and int(tables.timesteps[-1]) == 0:   # the last row (frame 3) adds no noise
            x0 = _oracle(cfg, n).step(eps[3:4], 0, lat[3:4].to(dt), add_noise=False)
            assert torch.equal(out.cpu()[3:4], x0)


def _tiny_pipe(emulate=True, device=0, **kw):
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.unet import B200MultiviewUNet
    cfg = UNetConfig.tiny()
    unet = B200MultiviewUNet(cfg, device=device).load_state_dict(random_state_dict(cfg, seed=1, dtype=torch.bfloat16))
    return B200Diffuman4DPipeline(unet, DDPMConfig(**kw), emulate_bf16_scheduler=emulate), unet


def _unet_cb(unet):
    def cb(x, t, sk, doms, nf):
        return unet(x.cuda(), t.cuda(), sk.cuda(), doms, nf, return_dict=False)[0].cpu()
    return cb


def _window(n, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    pix, plk, lat = r(n, 4, H, W), r(n, 6, H, W), r(n, 4, H, W)
    skel = (torch.rand(n, 3, 8 * H, 8 * W, generator=g) * 2 - 1).to(torch.bfloat16)
    mask = torch.ones(n, 1, H, W, dtype=torch.bfloat16)
    mask[1] = 0
    return pix, plk, lat, skel, mask


def test_denoise_window_ddpm_vs_oracle_bit_exact(cuda):
    """``d4d_denoise_window_ddpm``: four steps of one window whose frames are frames 6, 2, 0, 4, 5 of their task, at
    staggered timestep indices that reach the last row, against the oracle's window step with per-frame copies keyed by
    the same task indices."""
    from oracle.dpm_solver_oracle import denoise_window_oracle_per_frame
    from diffuman4d_b200.scheduler import DDPMTask
    pipe, unet = _tiny_pipe()
    n, seed = 5, 987654321
    pix, plk, lat, skel, mask = _window(n, 42)
    ti = torch.tensor([0, 0, 2, 5, 6])
    ids = torch.tensor([6, 2, 0, 4, 5])
    pipe.parepare_schedulers(10, 7)
    orc = _oracle(pipe.scheduler.config, 10, seed)
    copies = [copy.deepcopy(orc) for _ in range(7)]
    want, want_ti = denoise_window_oracle_per_frame(
        _unet_cb(unet), [copies[i] for i in ids], latents=lat.clone(), pixel_latents=pix, plucker=plk, skeletons=skel,
        cond_mask=mask, timestep_indices=ti, domain="spatial", guidance_scale=2.0, num_inference_steps=4)
    lat_d, ti_d = lat.cuda(), ti.cuda()
    frames = DDPMTask(7, "cuda", seed).take(ids)
    pipe.denoise_window(latents=lat_d, pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skel,
                        cond_masks_latents=mask, timestep_indices=ti_d, domain="spatial", guidance_scale=2.0,
                        num_inference_steps=4, solver_state=frames)
    torch.cuda.synchronize()
    assert torch.equal(ti_d.cpu(), want_ti)
    assert torch.equal(lat_d.cpu(), want), (lat_d.cpu().float() - want.float()).abs().max()


@pytest.mark.parametrize("kw", [dict(), dict(prediction_type="v_prediction", timestep_spacing="trailing",
                                             variance_type="fixed_large")])
def test_sliding_iterative_denoise_ddpm_vs_oracle_bit_exact(cuda, kw):
    """A spatial and then a bidirectional temporal task on one pipeline against the oracle's sliding loop (per-frame
    copies, the k-th copy keyed as frame k) with the seed the loop draws from its generator."""
    from diffuman4d_b200.scheduler import draw_seed
    from oracle.ddpm_oracle import DDPMOracle
    from oracle.dpm_solver_oracle import sliding_iterative_denoise_oracle_per_frame
    pipe, unet = _tiny_pipe(**kw)
    g = torch.Generator().manual_seed(43)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    for k, (domain, n_in, n_tg, ws, stride, bidir, rounds) in enumerate((("spatial", 2, 4, 4, 1, True, 2),
                                                                           ("temporal", 3, 3, 2, 1, True, 1))):
        n = n_in + n_tg
        mask = torch.ones(n, 1, H, W, dtype=torch.bfloat16)
        mask[:n_in] = 0
        args = dict(pixel_latents=r(n, 4, H, W), plucker=r(n, 6, H, W),
                    skeletons=(torch.rand(n, 3, 8 * H, 8 * W, generator=g) * 2 - 1).to(torch.bfloat16), cond_mask=mask,
                    latents=r(n, 4, H, W), domain=domain, timestep_indices=torch.zeros(n, dtype=torch.long),
                    window_size=ws, sliding_stride=stride, bidirectional=bidir, alternation_rounds=rounds,
                    guidance_scale=2.0)
        seed = int(draw_seed(torch.Generator("cuda").manual_seed(k), "cuda").item())
        ref = sliding_iterative_denoise_oracle_per_frame(_unet_cb(unet), DDPMOracle(pipe.scheduler.config, seed=seed),
                                                         **args, enable_pose_encoder=True)
        out = pipe.sliding_iterative_denoise(
            pixel_values_latents=args["pixel_latents"], plucker_embeds=args["plucker"], skeletons=args["skeletons"],
            cond_masks=mask, latents=args["latents"], domain=domain, timestep_indices=args["timestep_indices"],
            window_size=ws, sliding_stride=stride, bidirectional=bidir, alternation_rounds=rounds, guidance_scale=2.0,
            generator=torch.Generator("cuda").manual_seed(k))
        torch.cuda.synchronize()
        assert torch.equal(out["timestep_indices"].cpu(), ref["timestep_indices"])
        assert torch.equal(out["fully_denoised"].cpu(), ref["fully_denoised"])
        assert torch.equal(out["latents"].cpu(), ref["latents"]), (out["latents"].cpu().float() -
                                                                   ref["latents"].float()).abs().max()


def test_seed_decides_the_noise(cuda):
    """Same seed, same bits (twice through ``__call__`` and the per-frame handles); another seed changes every target
    frame and leaves the conditioning frame alone."""
    pipe, _ = _tiny_pipe(emulate=False)
    n = 5
    pix, plk, lat, skel, mask = _window(n, 44)
    runs = []
    for gseed in (7, 7, 8):
        handles, ts = pipe.parepare_schedulers(12, n)
        out = pipe(pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skel, cond_masks_latents=mask,
                   latents=lat.cuda(), domains=["spatial"], num_inference_steps=3, schedulers=handles, timesteps=ts,
                   timestep_indices=torch.zeros(n, dtype=torch.long), guidance_scale=2.0,
                   generator=torch.Generator("cuda").manual_seed(gseed))
        torch.cuda.synchronize()
        assert handles[0].state.seed is not None
        runs.append(out.cpu())
    assert torch.equal(runs[0], runs[1])
    assert torch.equal(runs[2][1], runs[0][1]) and torch.equal(runs[0][1], pix[1])   # the conditioning frame
    for j in (0, 2, 3, 4):
        assert not torch.equal(runs[2][j], runs[0][j]), j


# ------------------------------------------------------------------------------------------------ multi-GPU loopbacks
@pytest.fixture
def gloo_world1(tmp_path):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"file://{tmp_path / 'store'}", rank=0, world_size=1)
    try:
        yield
    finally:
        dist.destroy_process_group()


def _pipes(emulate, kw):
    """A plain pipeline and loopbacks of the frame-sharded window, the CFG split and the CFG grid, each on its own
    handle, with the same weights."""
    from diffuman4d_b200.cfg_split import CFGGridPipeline, CFGSplitPipeline
    from diffuman4d_b200.sharded import FrameShardedPipeline
    new = lambda: _tiny_pipe(emulate, **kw)[0]
    plain = new()
    return plain, {"sharded": FrameShardedPipeline(new(), max_frames=6, h=H, w=W),
                   "split": CFGSplitPipeline(new(), max_frames=6, h=H, w=W),
                   "grid": CFGGridPipeline(new(), max_frames=6, h=H, w=W)}


@pytest.mark.parametrize("emulate", [True, False])
@pytest.mark.parametrize("kw", [dict(), dict(prediction_type="v_prediction", variance_type="fixed_large")])
def test_loopbacks_are_bit_identical(cuda, gloo_world1, emulate, kw):
    from diffuman4d_b200.scheduler import DDPMTask
    plain, multi = _pipes(emulate, kw)
    n = 5
    pix, plk, lat, skel, mask = _window(n, 45)
    ti = torch.tensor([0, 0, 3, 1, 2], device="cuda")
    conds = dict(pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skel, cond_masks_latents=mask)
    for p in (plain, *(m.pipe for m in multi.values())):
        p.parepare_schedulers(12, 9)
    frames = DDPMTask(9, "cuda", 1234).take(torch.tensor([8, 1, 3, 0, 5]))
    for dom in ("spatial", "temporal"):
        for steps in (1, 2):
            kw2 = dict(domain=dom, guidance_scale=2.0, num_inference_steps=steps, **conds)
            ref_l, ref_t = lat.cuda(), ti.clone()
            plain.denoise_window(latents=ref_l, timestep_indices=ref_t, solver_state=frames, **kw2)
            assert not torch.equal(ref_l.cpu(), lat)
            for name, m in multi.items():
                l_, t_ = lat.cuda(), ti.clone()
                extra = dict(F_total=n) if name == "sharded" else {}
                m.denoise_window(latents=l_, timestep_indices=t_, solver_state=frames, **extra, **kw2)
                assert torch.equal(l_, ref_l), f"{name} {dom} steps {steps}: latents differ"
                assert torch.equal(t_, ref_t), f"{name} {dom} steps {steps}: timestep indices differ"
    # sliding tasks: the frame-sharded loop slices the frame ids; every loop draws the same seed from the generator
    g = torch.Generator().manual_seed(46)
    for domain, n_in, n_tg, ws in (("spatial", 2, 4, 2), ("temporal", 3, 3, 3)):
        n = n_in + n_tg
        mask = torch.ones(n, 1, 8 * H, 8 * W)
        mask[:n_in] = 0
        task = dict(pixel_values_latents=torch.randn(n, 4, H, W, generator=g), plucker_embeds=torch.randn(
            n, 6, 8 * H, 8 * W, generator=g), skeletons=torch.rand(n, 3, 8 * H, 8 * W, generator=g) * 2 - 1,
            cond_masks=mask, domain=domain, timestep_indices=torch.zeros(n, dtype=torch.long), window_size=ws,
            sliding_stride=1, bidirectional=True, alternation_rounds=1, guidance_scale=2.0)
        run = lambda p: p.sliding_iterative_denoise(latents=None, generator=torch.Generator("cuda").manual_seed(3),
                                                    **task)
        ref = run(plain)
        assert ref["fully_denoised"][n_in:].all()
        for name, m in multi.items():
            got = run(m)
            for key in ("latents", "timestep_indices"):
                assert torch.equal(got[key], ref[key]), f"{name} {domain} sliding: {key} differ"
        assert torch.equal(run(multi["grid"].pipe)["latents"], ref["latents"]), "plain loop on the grid's handle"


# ------------------------------------------------------------------------------------------------ several processes
MP_F = 4   # the window: two frames per rank of the frame-sharded window, one CFG half's frame shard per grid rank


def _mp_worker(rank, world, store, out_dir, mode):
    """One rank of the CFG split (2 ranks), the CFG grid (4 ranks, R = 2) or the frame-sharded window (2 ranks, two
    frames each, with its shard of the frame ids) on one GPU: a window step, then a sliding task whose initial noise and
    seed each rank draws from its own generator; rank 0 also runs both on one GPU."""
    import torch.distributed as dist
    from diffuman4d_b200.cfg_split import CFGGridPipeline, CFGSplitPipeline
    from diffuman4d_b200.scheduler import DDPMTask
    from diffuman4d_b200.sharded import FrameShardedPipeline
    from diffuman4d_b200.sharding import frame_shard
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=world)
    try:
        pipe = _tiny_pipe()[0]
        kind = {"split": CFGSplitPipeline, "grid": CFGGridPipeline, "sharded": FrameShardedPipeline}[mode]
        multi = kind(pipe, max_frames=MP_F, h=H, w=W)
        pix, plk, lat, skel, mask = (t.cuda() for t in _window(MP_F, 45))
        ti = torch.tensor([0, 0, 3, 1], device="cuda")
        conds = dict(pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skel, cond_masks_latents=mask)
        pipe.parepare_schedulers(12, 9)
        frames = DDPMTask(9, "cuda", 1234).take(torch.tensor([8, 1, 3, 0]))
        out = {}
        for dom in ("spatial", "temporal"):
            kw = dict(domain=dom, guidance_scale=2.0, num_inference_steps=2)
            if mode == "sharded":
                lo, hi = frame_shard(MP_F, rank, world)
                l_, t_ = lat[lo:hi].clone(), ti[lo:hi].clone()
                multi.denoise_window(latents=l_, timestep_indices=t_, solver_state=frames.shard(lo, hi), F_total=MP_F,
                                     **{k: v[lo:hi].contiguous() for k, v in conds.items()}, **kw)
            else:
                l_, t_ = lat.clone(), ti.clone()
                multi.denoise_window(latents=l_, timestep_indices=t_, solver_state=frames, **conds, **kw)
            out[("multi", dom)] = (l_.cpu(), t_.cpu())
            if rank == 0:
                l_, t_ = lat.clone(), ti.clone()
                pipe.denoise_window(latents=l_, timestep_indices=t_, solver_state=frames, **conds, **kw)
                out[("ref", dom)] = (l_.cpu(), t_.cpu())
        g = torch.Generator().manual_seed(46)
        n_in, n_tg = 3, 3                                   # bidirectional temporal: every window holds 4 frames
        n = n_in + n_tg
        cmask = torch.ones(n, 1, 8 * H, 8 * W)
        cmask[:n_in] = 0
        task = dict(pixel_values_latents=torch.randn(n, 4, H, W, generator=g),
                    plucker_embeds=torch.randn(n, 6, 8 * H, 8 * W, generator=g),
                    skeletons=torch.rand(n, 3, 8 * H, 8 * W, generator=g) * 2 - 1, cond_masks=cmask, latents=None,
                    domain="temporal", timestep_indices=torch.zeros(n, dtype=torch.long), window_size=2,
                    sliding_stride=1, bidirectional=True, alternation_rounds=1, guidance_scale=2.0)
        res = multi.sliding_iterative_denoise(generator=torch.Generator("cuda").manual_seed(100 + rank), **task)
        out[("multi", "loop")] = (res["latents"].cpu(), res["timestep_indices"].cpu())
        if rank == 0:
            res = pipe.sliding_iterative_denoise(generator=torch.Generator("cuda").manual_seed(100), **task)
            out[("ref", "loop")] = (res["latents"].cpu(), res["timestep_indices"].cpu())
        torch.save(out, os.path.join(out_dir, f"rank{rank}.pt"))
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("mode,world", [("split", 2), ("grid", 4), ("sharded", 2)])
def test_processes_on_one_gpu_give_the_single_gpu_bits(cuda, tmp_path, mode, world):
    """Every rank's window step and sliding task equal rank 0's single-GPU run bit for bit; the frame-sharded ranks hold
    their rows of the window.  Each rank starts from another generator, so the task's noise and seed must be rank 0's."""
    from test_gpu_cfg_grid import _spawn
    from diffuman4d_b200.sharding import frame_shard
    got = _spawn(tmp_path, _mp_worker, world, mode)
    for key in (("ref", "spatial"), ("ref", "temporal"), ("ref", "loop")):
        want_l, want_t = got[0][key]
        assert want_t.max() > 0
        for r in range(world):
            lat, ti = got[r][("multi", key[1])]
            if mode == "sharded" and key[1] != "loop":
                lo, hi = frame_shard(MP_F, r, world)
                want_l_r, want_t_r = want_l[lo:hi], want_t[lo:hi]
            else:
                want_l_r, want_t_r = want_l, want_t
            assert torch.equal(ti, want_t_r), f"{mode} {key[1]} rank {r}: timestep indices differ"
            assert torch.equal(lat, want_l_r), f"{mode} {key[1]} rank {r}: latents differ from the single-GPU run"


def test_load_pipelines_with_ddpm_scheduler(cuda, tmp_path):
    from safetensors.torch import save_file
    from diffuman4d_b200.loader import load_pipelines
    from diffuman4d_b200.scheduler import DDPMTables
    cfg = UNetConfig.tiny()
    os.makedirs(tmp_path / "unet")
    os.makedirs(tmp_path / "scheduler")
    json.dump(dict(in_channels=11, out_channels=4, block_out_channels=[64, 128, 256, 256], attention_head_dim=[1, 2, 4, 4],
                   cross_attention_dim=None, use_linear_projection=True, enable_pose_encoder=True, enable_tem_embeds=True,
                   layers_per_block=2, num_3d_attn_blocks=3), open(tmp_path / "unet" / "config.json", "w"))
    json.dump({"_class_name": "DDPMScheduler", "_diffusers_version": "0.33.1", "num_train_timesteps": 1000,
               "beta_start": 0.00085, "beta_end": 0.012, "beta_schedule": "scaled_linear", "trained_betas": None,
               "variance_type": "fixed_small", "clip_sample": False, "prediction_type": "epsilon", "thresholding": False,
               "timestep_spacing": "leading", "steps_offset": 1, "rescale_betas_zero_snr": False},
              open(tmp_path / "scheduler" / "scheduler_config.json", "w"))
    save_file({k: v.contiguous() for k, v in random_state_dict(cfg, seed=1).items()},
              str(tmp_path / "unet" / "diffusion_pytorch_model.safetensors"))
    (pipe,) = load_pipelines(model_dir=str(tmp_path), torch_dtype="bf16", gpu_ids=[0])
    assert isinstance(pipe.scheduler, DDPMTables) and pipe.scheduler.config == DDPMConfig(
        beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False, steps_offset=1)
    n = 6
    g = torch.Generator().manual_seed(47)
    mask = torch.ones(n, 1, H, W)
    mask[[1, 4]] = 0
    out = pipe.sliding_iterative_denoise(
        pixel_values_latents=torch.randn(n, 4, H, W, generator=g), plucker_embeds=torch.randn(n, 6, H, W, generator=g),
        skeletons=torch.rand(n, 3, 8 * H, 8 * W, generator=g) * 2 - 1, cond_masks=mask, latents=None, domain="spatial",
        timestep_indices=torch.zeros(n, dtype=torch.long), window_size=2, sliding_stride=1, bidirectional=True,
        alternation_rounds=1, guidance_scale=2.0, generator=torch.Generator(device="cuda").manual_seed(0))
    ti = out["timestep_indices"].cpu()
    assert ti[[1, 4]].eq(0).all() and ti[[0, 2, 3, 5]].eq(4).all() and out["fully_denoised"].cpu()[[0, 2, 3, 5]].all()
    assert torch.isfinite(out["latents"].float()).all()
