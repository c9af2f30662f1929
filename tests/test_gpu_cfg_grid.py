"""The CFG grid (``CFGGridPipeline``: the CFG-split window on 2R ranks, DESIGN.md section 7) against the single-GPU
window, bit for bit.

* One-rank loopback (world 1 is R = 1: the rank runs both halves into its own exchange buffer): one window step of every
  device scheduler, epsilon and v-prediction, pose encoder on and off, 1 and 2 denoising steps per call, from a mid-task
  state, equals the plain window and the CFG-split loopback (latents, timestep indices and every solver-state plane).
  Plain window steps run on the grid pipeline's handle between its grid calls.  Guidance 1.0 through the grid pipeline
  is the plain step.
* Four processes on one GPU (a 2x2 grid, gloo, every rank on cuda:0, the exchange buffers mapped across processes with
  cudaIpc), on the tiny UNet: spatial and temporal windows for DDIM, DPM-Solver++ 2, UniPC, PNDM and DEIS-3 from a
  mid-task state, and one bidirectional temporal sliding loop.  Every rank's latents, timestep indices and solver state
  equal rank 0's single-GPU result.  This is the one-GPU run with frame shards r > 0, noise stores across the two halves'
  groups and the K/V scatter limited to a half's ranks.
* Four processes on one GPU also run 2-frame windows (ranks holding a single frame of the window, whose 3-D layers
  must still attend over both frames), and two processes run the frame-sharded window on a 2-frame window (one frame per
  rank) for the same reason.
* Two processes on one GPU (a 2x1 grid, R = 1) give the CFG-split window's bits.
* The same four- and eight-rank runs on four and eight GPUs, skipped below that many devices.
"""
import os

import pytest
import torch

from test_gpu_cfg_split import (LOOP_TASKS, SCHEDULERS, _capture_state, _cfg, _clone, _fields, _mid_task,  # noqa: E402
                                _task, gloo_world1)  # noqa: F401  (gloo_world1 is a fixture)

F, H, W = 4, 16, 16


def _pipes(cfg, sched, max_frames, h, w, device=0, emulate=True, plain=True, split=True):
    """A plain pipeline, a CFGSplitPipeline (when ``split``) and a CFGGridPipeline with the same weights, each on its own
    handle (None where not asked for)."""
    from diffuman4d_b200.cfg_split import CFGGridPipeline, CFGSplitPipeline
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict
    sd = random_state_dict(cfg, seed=1)
    new = lambda: B200Diffuman4DPipeline(B200MultiviewUNet(cfg, device).load_state_dict(sd), sched,
                                         emulate_bf16_scheduler=emulate)
    p = new() if plain else None
    sp = CFGSplitPipeline(new(), max_frames=max_frames, h=h, w=w) if split else None
    gp = CFGGridPipeline(new(), max_frames=max_frames, h=h, w=w)
    return p, sp, gp


def _compare(plain, others, cfg, kw, what, interleave=None):
    """From a mid-task state, 1 and 2 steps of each of ``others`` (name, run) equal the plain window's.  ``interleave``:
    a plain step run on another handle before each of its runs."""
    lat, ti, state, conds = _mid_task(plain, cfg, kw)
    if state is not None:
        assert int(state.lower_order_nums.max()) >= 2, f"{what}: the history does not reach a higher-order branch"
    for steps in (1, 2):
        runs = []
        for name, run in (("plain", plain.denoise_window), *others):
            if interleave is not None and name == "grid":
                l_, t_, st = lat.clone(), ti.clone(), _clone(state)
                interleave(latents=l_, timestep_indices=t_, solver_state=st, num_inference_steps=1, **conds, **kw)
            l_, t_, st = lat.clone(), ti.clone(), _clone(state)
            run(latents=l_, timestep_indices=t_, solver_state=st, num_inference_steps=steps, **conds, **kw)
            runs.append((name, _fields(l_, t_, st)))
        ref = runs[0][1]
        assert not torch.equal(ref["latents"], lat), f"{what}: the step changed nothing"
        for name, res in runs[1:]:
            for k, t in ref.items():
                assert torch.equal(res[k], t), f"{what} steps {steps}: {name} {k} differs from the single-GPU window"


@pytest.mark.gpu
@pytest.mark.parametrize("pose", [True, False], ids=["pose", "skeleton-latents"])
@pytest.mark.parametrize("pred", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("sched", list(SCHEDULERS))
def test_loopback_grid_is_bit_identical(cuda, gloo_world1, sched, pred, pose):
    cfg = _cfg(pose)
    plain, sp, gp = _pipes(cfg, SCHEDULERS[sched](pred), F, H, W)
    for p in (sp.pipe, gp.pipe):
        p.parepare_schedulers(18, F)
    for dom in ("spatial", "temporal"):
        _compare(plain, [("split", sp.denoise_window), ("grid", gp.denoise_window)], cfg,
                 dict(domain=dom, guidance_scale=2.0), f"{sched} {pred} {dom}", interleave=gp.pipe.denoise_window)


@pytest.mark.gpu
@pytest.mark.parametrize("sched", ["ddim", "dpm2"])
def test_guidance_one_is_the_plain_step(cuda, gloo_world1, sched):
    """guidance_scale 1.0 has no CFG halves: the grid pipeline runs the plain single-GPU step."""
    cfg = _cfg()
    plain, _, gp = _pipes(cfg, SCHEDULERS[sched]("epsilon"), F, H, W, split=False)
    gp.pipe.parepare_schedulers(18, F)
    _compare(plain, [("grid", gp.denoise_window)], cfg, dict(domain="spatial", guidance_scale=1.0), f"{sched} guidance 1")


# ------------------------------------------------------------------------------------------------ several processes
GRID_SCHEDULERS = ["ddim", "dpm2", "unipc2-bh2", "pndm", "deis3"]
GRID_LOOP = LOOP_TASKS[1]   # bidirectional temporal: every window holds 4 frames
SMALL_F = 2                 # a 2-frame window: one frame per rank on a 2x2 grid or a two-rank frame shard


def _small_window(pipe, cfg, kw, seed=4):
    """A mid-task window of SMALL_F frames (frame 0 conditioning) after two plain steps on ``pipe``'s handle."""
    g = torch.Generator().manual_seed(seed)
    lat, pix, plk = (torch.randn(SMALL_F, c, H, W, generator=g).to(torch.bfloat16).cuda() for c in (4, 4, 6))
    skel = (torch.rand(SMALL_F, 3, 8 * H, 8 * W, generator=g) * 2 - 1).to(torch.bfloat16).cuda()
    mask = torch.ones(SMALL_F, 1, H, W, dtype=torch.bfloat16, device="cuda")
    mask[0] = 0
    ti = torch.tensor([0, 3], device="cuda")
    pipe.parepare_schedulers(18, SMALL_F)
    state = pipe.scheduler.new_state(SMALL_F).take(torch.arange(SMALL_F), H, W) if pipe._multistep else None
    conds = dict(pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skel, cond_masks_latents=mask)
    pipe.denoise_window(latents=lat, timestep_indices=ti, solver_state=state, num_inference_steps=2, **conds, **kw)
    return lat, ti, state, conds


def _worker(rank, world, store, out_dir, devices, scheds, loop, small=()):
    import torch.distributed as dist
    dev = devices[rank]
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=world)
    try:
        cfg = _cfg()
        out = {}
        for sched in scheds:
            _, _, gp = _pipes(cfg, SCHEDULERS[sched]("epsilon"), F, H, W, device=dev, plain=False, split=False)
            for dom in ("spatial", "temporal"):
                kw = dict(domain=dom, guidance_scale=2.0)
                lat, ti, state, conds = _mid_task(gp.pipe, cfg, kw)   # plain steps on this rank's handle
                runs = [("grid", gp.denoise_window)] + ([("ref", gp.pipe.denoise_window)] if rank == 0 else [])
                for name, run in runs:
                    l_, t_, st = lat.clone(), ti.clone(), _clone(state)
                    run(latents=l_, timestep_indices=t_, solver_state=st, num_inference_steps=2, **conds, **kw)
                    out[(name, sched, dom)] = {k: v.cpu() for k, v in _fields(l_, t_, st).items()}
        for sched in small:
            _, _, gp = _pipes(cfg, SCHEDULERS[sched]("epsilon"), SMALL_F, H, W, device=dev, plain=False, split=False)
            for dom in ("spatial", "temporal"):
                kw = dict(domain=dom, guidance_scale=2.0)
                lat, ti, state, conds = _small_window(gp.pipe, cfg, kw)
                runs = [("grid", gp.denoise_window)] + ([("ref", gp.pipe.denoise_window)] if rank == 0 else [])
                for name, run in runs:
                    l_, t_, st = lat.clone(), ti.clone(), _clone(state)
                    run(latents=l_, timestep_indices=t_, solver_state=st, num_inference_steps=2, **conds, **kw)
                    out[(name, sched, dom, SMALL_F)] = {k: v.cpu() for k, v in _fields(l_, t_, st).items()}
        if loop:
            h = w = 8
            domain, n_in, n_tg, ws, stride, bidir, rounds = GRID_LOOP
            _, _, gp = _pipes(cfg, SCHEDULERS["dpm2"]("epsilon"), n_in + ws, h, w, device=dev, plain=False,
                              split=False)
            box = _capture_state(gp.pipe)
            kw = dict(_task(cfg, domain, n_in, n_tg, h, w, seed=21), window_size=ws, sliding_stride=stride,
                      bidirectional=bidir, num_denoising_steps=1, alternation_rounds=rounds, guidance_scale=2.0)
            runs = [("grid", gp.sliding_iterative_denoise)]
            if rank == 0:
                runs.append(("ref", gp.pipe.sliding_iterative_denoise))
            for name, run in runs:
                res = run(**kw)
                fields = {k: res[k].cpu() for k in ("latents", "timestep_indices", "fully_denoised")}
                fields.update({k: v.cpu() for k, v in _fields(None, None, box[-1]).items() if v is not None})
                out[(name, "loop", domain)] = fields
        torch.save(out, os.path.join(out_dir, f"rank{rank}.pt"))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _spawn(tmp_path, target, world, *args):
    """Runs ``target(rank, world, store, out_dir, *args)`` in ``world`` processes and loads each rank's saved dict."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=target, args=(r, world, str(tmp_path / "store"), str(tmp_path), *args))
             for r in range(world)]
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
    return [torch.load(tmp_path / f"rank{r}.pt") for r in range(world)]


def _run_ranks(tmp_path, devices, scheds, loop, small=()):
    world = len(devices)
    got = _spawn(tmp_path, _worker, world, devices, scheds, loop, small)
    keys = [k for k in got[0] if k[0] == "ref"]
    assert len(keys) == 2 * len(scheds) + 2 * len(small) + (1 if loop else 0)
    for key in keys:
        ref = got[0][key]
        for r in range(world):
            res = got[r][("grid", *key[1:])]
            assert res.keys() == ref.keys()
            for k in ref:
                assert torch.equal(res[k], ref[k]), f"{key[1:]} rank {r} of {world}: {k} differs from the single-GPU result"


@pytest.mark.gpu
def test_four_processes_on_one_gpu(cuda, tmp_path):
    _run_ranks(tmp_path, [0] * 4, GRID_SCHEDULERS, loop=True, small=("ddim", "dpm2"))


def _sharded_worker(rank, world, store, out_dir):
    """The frame-sharded window with one frame per rank: each rank's stepped frame, and on rank 0 the single-GPU
    window."""
    import torch.distributed as dist
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.sharded import FrameShardedPipeline
    from diffuman4d_b200.sharding import frame_shard
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=world)
    try:
        cfg = _cfg()
        sd = random_state_dict(cfg, seed=1)
        out = {}
        for sched in ("ddim", "dpm2"):
            pipe = B200Diffuman4DPipeline(B200MultiviewUNet(cfg, 0).load_state_dict(sd), SCHEDULERS[sched]("epsilon"),
                                          emulate_bf16_scheduler=True)
            sh = FrameShardedPipeline(pipe, max_frames=SMALL_F, h=H, w=W)
            lo, hi = frame_shard(SMALL_F, rank, world)
            for dom in ("spatial", "temporal"):
                kw = dict(domain=dom, guidance_scale=2.0)
                lat, ti, state, conds = _small_window(pipe, cfg, kw)
                local = {k: v[lo:hi].contiguous() for k, v in conds.items()}
                st = None if state is None else type(state)(hi - lo, state.x0_prev.device,
                                                            state.x0_prev[lo:hi].contiguous(),
                                                            state.lower_order_nums[lo:hi].contiguous())
                l_, t_ = lat[lo:hi].contiguous(), ti[lo:hi].contiguous()
                sh.denoise_window(latents=l_, timestep_indices=t_, solver_state=st, num_inference_steps=2,
                                  F_total=SMALL_F, **local, **kw)
                out[("sharded", sched, dom)] = {k: v.cpu() for k, v in _fields(l_, t_, st).items()}
                if rank == 0:
                    l_, t_, st = lat.clone(), ti.clone(), _clone(state)
                    pipe.denoise_window(latents=l_, timestep_indices=t_, solver_state=st, num_inference_steps=2,
                                        **conds, **kw)
                    out[("ref", sched, dom)] = {k: v.cpu() for k, v in _fields(l_, t_, st).items()}
        torch.save(out, os.path.join(out_dir, f"rank{rank}.pt"))
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_frame_sharded_one_frame_per_rank(cuda, tmp_path):
    """Two ranks on one GPU, each holding one frame of a 2-frame window: the 3-D layers still attend over both frames,
    so each rank's frame equals its row of the single-GPU window."""
    got = _spawn(tmp_path, _sharded_worker, 2)
    keys = [k for k in got[0] if k[0] == "ref"]
    assert len(keys) == 4
    for key in keys:
        ref = got[0][key]
        for r in range(2):
            res = got[r][("sharded", *key[1:])]
            assert res.keys() == ref.keys()
            for k in ref:
                assert torch.equal(res[k], ref[k][r:r + 1]), f"{key[1:]} rank {r}: {k} differs from the single-GPU row"


@pytest.mark.gpu
def test_two_processes_on_one_gpu_give_the_split_bits(cuda, tmp_path):
    _run_ranks(tmp_path, [0, 0], ["ddim", "dpm2"], loop=False)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [4, 8])
def test_grid_on_gpus(cuda, tmp_path, world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    # on 8 GPUs (R = 4) the 4-frame windows already put one frame on each rank
    _run_ranks(tmp_path, list(range(world)), GRID_SCHEDULERS, loop=True, small=("ddim",) if world == 4 else ())
