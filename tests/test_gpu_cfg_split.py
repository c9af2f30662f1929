"""The CFG-split window (``CFGSplitPipeline``, DESIGN.md section 7) against the single-GPU window, bit for bit.

* One-rank loopback (``d4d_exchange_open`` with rank 0 of world 1: the rank runs the negative half, then the positive
  half, into its own exchange buffer):
  - one window step of every device scheduler (DDIM, DPM-Solver++ order 2, UniPC order 2 bh2, PNDM, DEIS order 3,
    DPM-Solver++ singlestep order 3), epsilon and v-prediction, pose encoder on and off, 1 and 2 denoising steps per
    call, from a mid-task state (staggered timestep indices, a conditioning frame, solver history from three earlier
    steps, so the multistep solvers run their higher-order branches): latents, timestep indices, every solver-state
    plane and ``lower_order_nums``;
  - guidance 1.0 through the split pipeline (no halves: the plain step);
  - ``sliding_iterative_denoise`` over a spatial and a bidirectional temporal task, for DDIM and for PNDM and DEIS,
    which the frame-sharded window does not run;
  - ``execute_tasks(cfg_split=True)`` gives the default mode's grid.
* Two processes on one GPU (gloo, both ranks on cuda:0, the exchange buffers mapped across processes with cudaIpc), and
  two processes on two GPUs when there are two: both ranks' window results equal each other and the single-GPU result,
  for DDIM and DPM-Solver++.
"""
import copy
import os
import sys

import pytest
import torch

from diffuman4d_b200.config import (DEISConfig, DPMSingleConfig, DPMSolverConfig, PNDMConfig, SchedulerConfig,
                                    UNetConfig, UniPCConfig)

GOLD = os.path.join(os.path.dirname(__file__), "golden")

SCHEDULERS = {
    "ddim": lambda pred: SchedulerConfig(prediction_type=pred),
    "dpm2": lambda pred: DPMSolverConfig(solver_order=2, prediction_type=pred),
    "unipc2-bh2": lambda pred: UniPCConfig(solver_order=2, solver_type="bh2", prediction_type=pred),
    "pndm": lambda pred: PNDMConfig(prediction_type=pred),
    "deis3": lambda pred: DEISConfig(solver_order=3, prediction_type=pred),
    "dpm-single3": lambda pred: DPMSingleConfig(solver_order=3, prediction_type=pred),
}
F, H, W = 4, 16, 16


@pytest.fixture
def gloo_world1(tmp_path):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"file://{tmp_path / 'store'}", rank=0, world_size=1)
    try:
        yield
    finally:
        dist.destroy_process_group()


def _cfg(pose=True):
    return UNetConfig.tiny() if pose else UNetConfig.tiny(enable_pose_encoder=False, in_channels=15)


def _pipes(cfg, sched, max_frames, h, w, device=0, emulate=True, vae=None, plain=True):
    """A plain pipeline (when ``plain``) and a CFGSplitPipeline with the same weights, each on its own handle."""
    from diffuman4d_b200.cfg_split import CFGSplitPipeline
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict
    sd = random_state_dict(cfg, seed=1)
    pipes = [B200Diffuman4DPipeline(B200MultiviewUNet(cfg, device).load_state_dict(sd), sched, vae=vae,
                                    emulate_bf16_scheduler=emulate) for _ in range(2 if plain else 1)]
    sp = CFGSplitPipeline(pipes[-1], max_frames=max_frames, h=h, w=w)
    return (pipes[0] if plain else None), sp


def _window_inputs(cfg, seed=3):
    g = torch.Generator().manual_seed(seed)
    lat, pix, plk = (torch.randn(F, c, H, W, generator=g).to(torch.bfloat16).cuda() for c in (4, 4, 6))
    skel = ((torch.rand(F, 3, 8 * H, 8 * W, generator=g) * 2 - 1) if cfg.enable_pose_encoder
            else torch.randn(F, 4, H, W, generator=g)).to(torch.bfloat16).cuda()
    mask = torch.ones(F, 1, H, W, dtype=torch.bfloat16, device="cuda")
    mask[1] = 0
    return lat, pix, plk, skel, mask


def _clone(state):
    if state is None:
        return None
    c = copy.copy(state)
    for name in (*state.planes, "lower_order_nums"):
        setattr(c, name, getattr(state, name).clone())
    return c


def _fields(lat, ti, state):
    out = {"latents": lat, "timestep_indices": ti}
    if state is not None:
        out.update({name: getattr(state, name) for name in (*state.planes, "lower_order_nums")})
    return out


def _mid_task(pipe, cfg, kw):
    """A mid-task window: staggered timestep indices, frame 1 conditioning, and the solver history of three plain
    steps from a new task's state."""
    lat, pix, plk, skel, mask = _window_inputs(cfg)
    ti = torch.tensor([0, 5, 2, 1], device="cuda")
    pipe.parepare_schedulers(18, F)
    state = pipe.scheduler.new_state(F).take(torch.arange(F), H, W) if pipe._multistep else None
    conds = dict(pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skel, cond_masks_latents=mask)
    pipe.denoise_window(latents=lat, timestep_indices=ti, solver_state=state, num_inference_steps=3, **conds, **kw)
    return lat, ti, state, conds


def _compare_window(plain, run_split, cfg, kw, what):
    lat, ti, state, conds = _mid_task(plain, cfg, kw)
    if state is not None:
        assert int(state.lower_order_nums.max()) >= 2, f"{what}: the history does not reach a higher-order branch"
    for steps in (1, 2):
        res = []
        for run in (plain.denoise_window, run_split):
            l_, t_, st = lat.clone(), ti.clone(), _clone(state)
            run(latents=l_, timestep_indices=t_, solver_state=st, num_inference_steps=steps, **conds, **kw)
            res.append(_fields(l_, t_, st))
        assert not torch.equal(res[0]["latents"], lat), f"{what}: the step changed nothing"
        for name, ref in res[0].items():
            assert torch.equal(res[1][name], ref), f"{what} steps {steps}: {name} differs from the single-GPU window"


@pytest.mark.gpu
@pytest.mark.parametrize("pose", [True, False], ids=["pose", "skeleton-latents"])
@pytest.mark.parametrize("pred", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("sched", list(SCHEDULERS))
def test_loopback_window_is_bit_identical(cuda, gloo_world1, sched, pred, pose):
    cfg = _cfg(pose)
    plain, sp = _pipes(cfg, SCHEDULERS[sched](pred), F, H, W)
    sp.pipe.parepare_schedulers(18, F)
    for dom in ("spatial", "temporal"):
        _compare_window(plain, sp.denoise_window, cfg, dict(domain=dom, guidance_scale=2.0), f"{sched} {pred} {dom}")


@pytest.mark.gpu
@pytest.mark.parametrize("sched", ["ddim", "dpm2"])
def test_guidance_one_is_the_plain_step(cuda, gloo_world1, sched):
    """guidance_scale 1.0 has no CFG halves: the split pipeline runs the plain single-GPU step."""
    cfg = _cfg()
    plain, sp = _pipes(cfg, SCHEDULERS[sched]("epsilon"), F, H, W)
    sp.pipe.parepare_schedulers(18, F)
    _compare_window(plain, sp.denoise_window, cfg, dict(domain="spatial", guidance_scale=1.0), f"{sched} guidance 1")


def _capture_state(pipe):
    box = []
    inner = pipe.parepare_schedulers

    def wrapped(n, frames):
        s, ts = inner(n, frames)
        box.append(s[0].state if pipe._multistep else None)
        return s, ts
    pipe.parepare_schedulers = wrapped
    return box


def _task(cfg, domain, n_in, n_tg, h, w, seed):
    n = n_in + n_tg
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    mask = torch.ones(n, 1, 8 * h, 8 * w)
    mask[:n_in] = 0
    skel = ((torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16) if cfg.enable_pose_encoder
            else r(n, 4, h, w))
    return dict(pixel_values_latents=r(n, 4, h, w), plucker_embeds=r(n, 6, 8 * h, 8 * w), skeletons_latents=skel,
                cond_masks=mask, latents=r(n, 4, h, w), domain=domain, timestep_indices=torch.zeros(n, dtype=torch.long))


# (domain, inputs, targets, window, stride, bidirectional, alternation rounds)
LOOP_TASKS = [("spatial", 2, 4, 2, 1, False, 2), ("temporal", 3, 3, 2, 1, True, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("sched", ["ddim", "pndm", "deis3"])
def test_loopback_sliding_loop_is_bit_identical(cuda, gloo_world1, sched):
    cfg = _cfg()
    h = w = 8
    plain, sp = _pipes(cfg, SCHEDULERS[sched]("epsilon"), 6, h, w)
    bp, bs = _capture_state(plain), _capture_state(sp.pipe)
    for steps in (1, 2):
        for k, (domain, n_in, n_tg, ws, stride, bidir, rounds) in enumerate(LOOP_TASKS):
            kw = dict(_task(cfg, domain, n_in, n_tg, h, w, seed=20 + k), window_size=ws, sliding_stride=stride,
                      bidirectional=bidir, num_denoising_steps=steps, alternation_rounds=rounds, guidance_scale=2.0)
            ref = plain.sliding_iterative_denoise(**kw)
            got = sp.sliding_iterative_denoise(**kw)
            tag = f"{sched} {domain} steps {steps}"
            assert ref["timestep_indices"].max() > 0
            for key in ("latents", "timestep_indices", "fully_denoised"):
                assert torch.equal(got[key], ref[key]), f"{tag}: {key} differ"
            if bp[-1] is not None:
                for name, t in _fields(None, None, bp[-1]).items():
                    if t is not None:
                        assert torch.equal(_fields(None, None, bs[-1])[name], t), f"{tag}: {name} differs"


@pytest.mark.gpu
def test_loopback_execute_tasks_cfg_split(cuda, gloo_world1):
    """Three alternation rounds of the sampler: cfg_split=True on the loopback pipeline gives the default mode's grid
    (fresh targets draw their noise from the device's default generator, reseeded before each run)."""
    sys.path.insert(0, GOLD)
    from pool_vae import PoolVAE
    from synthetic_dataset import SyntheticSpaTemDataset
    from diffuman4d_b200.sampler import B200SlidingIterativeSampler
    plain, sp = _pipes(_cfg(), SchedulerConfig(), 6, 16, 16, emulate=False, vae=PoolVAE())
    grids = []
    for pipe, split in ((plain, False), (sp, True)):
        saved = []
        s = B200SlidingIterativeSampler(SyntheticSpaTemDataset(8, h=16, w=16), [pipe], output_dir=None,
                                        spa_label_range=[0, 6, 1], tem_label_range=[0, 4, 1], input_spa_labels=[1, 4],
                                        window_size=2, sliding_stride=1, bidirectional=True, alternation_rounds=3,
                                        guidance_scale=2.0, save_fn=lambda smp, d: saved.append(smp["domain_label"]))
        torch.cuda.manual_seed(1234)
        s.execute_tasks(cfg_split=split)
        torch.cuda.synchronize()
        grids.append((s.grid_latents.clone(), s.grid_timestep_indices.clone(), saved))
    assert grids[0][1].max() > 0
    assert torch.equal(grids[1][1], grids[0][1]), "timestep index grids differ"
    assert torch.equal(grids[1][0], grids[0][0]), "latent grids differ"
    assert grids[1][2] == grids[0][2], "rank 0 saves every task, in order"


# ------------------------------------------------------------------------------------------------ two processes
def _worker(rank, world, store, out_dir, devices):
    import torch.distributed as dist
    dev = devices[rank]
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=world)
    try:
        cfg = _cfg()
        out = {}
        for sched in ("ddim", "dpm2"):
            _, sp = _pipes(cfg, SCHEDULERS[sched]("epsilon"), F, H, W, device=dev, plain=False)
            kw = dict(domain="spatial", guidance_scale=2.0)
            lat, ti, state, conds = _mid_task(sp.pipe, cfg, kw)   # plain steps on this rank's handle
            runs = [("split", sp.denoise_window)] + ([("ref", sp.pipe.denoise_window)] if rank == 0 else [])
            for name, run in runs:
                l_, t_, st = lat.clone(), ti.clone(), _clone(state)
                run(latents=l_, timestep_indices=t_, solver_state=st, num_inference_steps=2, **conds, **kw)
                out[(name, sched)] = {k: v.cpu() for k, v in _fields(l_, t_, st).items()}
        torch.save(out, os.path.join(out_dir, f"rank{rank}.pt"))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _two_ranks(tmp_path, devices):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_worker, args=(r, 2, str(tmp_path / "store"), str(tmp_path), devices)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        for p in procs:
            p.join(timeout=600)
        for r, p in enumerate(procs):
            assert p.exitcode == 0, f"rank {r} exited with {p.exitcode}"
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=30)
    got = [torch.load(tmp_path / f"rank{r}.pt") for r in range(2)]
    for sched in ("ddim", "dpm2"):
        ref = got[0][("ref", sched)]
        for r in range(2):
            res = got[r][("split", sched)]
            assert res.keys() == ref.keys()
            for k in ref:
                assert torch.equal(res[k], ref[k]), f"{sched} rank {r}: {k} differs from the single-GPU window"


@pytest.mark.gpu
def test_two_processes_on_one_gpu(cuda, tmp_path):
    _two_ranks(tmp_path, [0, 0])


@pytest.mark.gpu
def test_two_gpus(cuda, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _two_ranks(tmp_path, [0, 1])
