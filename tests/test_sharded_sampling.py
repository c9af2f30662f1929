"""Host logic of the frame-sharded sliding loop (``FrameShardedPipeline.sliding_iterative_denoise``) on the CPU.

* Every window of the spatial, temporal and bidirectional schedules of ``build_windows`` is covered exactly once by the
  rank slices of ``frame_shard``, for every rank count that divides it.
* A window whose frame count the ranks do not divide is refused with the ``frame_shard`` message before any window runs.
* A gloo job of 2 and of 4 processes runs the sharded loop with its device seam (sharded step + window-result exchange)
  replaced by a per-frame stand-in denoiser and ``dist.all_gather``; the final latents, timestep indices, ``fully_denoised``
  and DPM-Solver++ state equal the single-process plain loop's with the same stand-in.  That covers the slicing,
  re-assembly, solver-state and noise bookkeeping for ranks above 0, which a one-GPU loopback (always rank 0) cannot.
"""
import os
import types

import pytest
import torch

from diffuman4d_b200.config import DPMSolverConfig, SchedulerConfig, UNetConfig
from diffuman4d_b200.pipeline import B200Diffuman4DPipeline, build_windows
from diffuman4d_b200.sharding import frame_shard

H = W = 8


# ------------------------------------------------------------------------------------------------ rank slices
SCHEDULES = [  # (domain, inputs, targets, window, stride, bidirectional)
    ("spatial", 4, 8, 4, 1, False),
    ("spatial", 4, 44, 12, 2, True),
    ("spatial", 2, 10, 6, 3, False),
    ("temporal", 8, 8, 4, 1, False),
    ("temporal", 16, 16, 12, 2, True),
    ("temporal", 24, 24, 24, 4, True),
]


@pytest.mark.parametrize("sched", SCHEDULES, ids=[f"{s[0]}-{s[1]}+{s[2]}-w{s[3]}-s{s[4]}-{'bi' if s[5] else 'uni'}"
                                                  for s in SCHEDULES])
def test_rank_slices_cover_every_window_once(sched):
    domain, n_in, n_tg, ws, stride, bidir = sched
    inputs, targets = torch.arange(n_in), torch.arange(n_in, n_in + n_tg)
    tws, iws = build_windows(targets, inputs, domain, ws, stride, 0, bidir)
    assert tws
    tested = 0
    for tw, iw in zip(tws, iws):
        window = torch.cat([iw, tw])
        F = len(window)
        for R in (1, 2, 3, 4, 6, 8):
            if F % R:
                with pytest.raises(ValueError, match="must be divisible by the number of ranks"):
                    frame_shard(F, 0, R)
                continue
            parts = [window[slice(*frame_shard(F, r, R))] for r in range(R)]
            assert all(len(p) == F // R for p in parts)
            assert torch.equal(torch.cat(parts), window), (R, window)
            tested += 1
    assert tested > len(tws)


# ------------------------------------------------------------------------------------------------ stand-in window step
class _UNetStub:
    """What the pipeline's host code reads of the UNet (no library call is made with it)."""

    def __init__(self):
        self.device = torch.device("cpu")
        self.config = UNetConfig.tiny()


def _pipe(dpm: bool):
    return B200Diffuman4DPipeline(_UNetStub(), DPMSolverConfig() if dpm else SchedulerConfig())


def _standin(lat, ts, x0, lon, pix, msk, steps):
    """A per-frame denoiser in place of the device step: each frame's result depends on that frame's own latents,
    conditioning, timestep index and solver state only.  Conditioning frames receive their image latents and timestep 0,
    and keep their solver state, as in the CFG + scheduler kernels."""
    cond = msk[:, 0, 0, 0] == 0
    c4 = cond.view(-1, 1, 1, 1)
    for _ in range(steps):
        new = lat.float() * 0.75 + pix.float() * 0.25 - 0.01 * ts.view(-1, 1, 1, 1).float()
        if x0 is not None:
            new = new + 0.5 * x0.float() * (lon.view(-1, 1, 1, 1) > 0)
            x0.copy_(torch.where(c4, x0, lat))
            lon.copy_(torch.where(cond, lon, (lon + 1).clamp(max=2)))
        lat.copy_(torch.where(c4, pix, new.to(torch.bfloat16)))
        ts.copy_(torch.where(cond, torch.zeros_like(ts), ts + 1))


def _plain_standin(*, latents, pixel_values_latents, cond_masks_latents, timestep_indices, num_inference_steps,
                   solver_state=None, **_):
    st = solver_state
    _standin(latents, timestep_indices, None if st is None else st.x0_prev, None if st is None else st.lower_order_nums,
             pixel_values_latents, cond_masks_latents, num_inference_steps)
    return latents, timestep_indices


def _gathered_standin(sh):
    """``FrameShardedPipeline._step_and_exchange`` with the stand-in step on the local frames and dist.all_gather as the
    window-result exchange."""
    import torch.distributed as dist
    from diffuman4d_b200.scheduler import DPMSolverState

    def gather(t):
        parts = [torch.empty_like(t) for _ in range(sh.world)]
        dist.all_gather(parts, t)
        return torch.cat(parts)

    def step(lat, ts, state, conds, F_total, *, domain, guidance_scale, num_inference_steps):
        assert lat.shape[0] * sh.world == F_total
        pix, _, _, msk = conds
        x0, lon = (None, None) if state is None else (state.x0_prev, state.lower_order_nums)
        _standin(lat, ts, x0, lon, pix, msk, num_inference_steps)
        out = None if state is None else DPMSolverState(F_total, lat.device, gather(x0), gather(lon))
        return gather(lat), gather(ts), out
    return step


def _sharded(pipe, rank, world):
    """A FrameShardedPipeline without an exchange buffer (its device calls are replaced)."""
    from diffuman4d_b200.sharded import FrameShardedPipeline
    sh = FrameShardedPipeline.__new__(FrameShardedPipeline)
    sh.pipe, sh.group, sh.rank, sh.world = pipe, None, rank, world
    return sh


def _capture_state(pipe):
    """Record the task's DPMSolverState that the loop creates through parepare_schedulers."""
    box = []
    inner = pipe.parepare_schedulers

    def wrapped(n, F):
        s, ts = inner(n, F)
        box.append(s[0].state if pipe._multistep else None)
        return s, ts
    pipe.parepare_schedulers = wrapped
    return box


# (name, domain, inputs, targets, window, stride, bidirectional, denoising steps, DPM, initial noise drawn by the loop)
TASKS = [
    ("spatial-ddim", "spatial", 4, 8, 4, 2, False, 1, False, False),
    ("spatial-dpm-2steps-noise", "spatial", 4, 8, 4, 2, True, 2, True, True),
    ("temporal-bidir-dpm", "temporal", 8, 8, 4, 1, True, 1, True, False),
    ("temporal-bidir-ddim-2steps-noise", "temporal", 8, 8, 4, 2, True, 2, False, True),
]


def _task_inputs(domain, n_in, n_tg, seed=5):
    n = n_in + n_tg
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    mask = torch.ones(n, 1, 8 * H, 8 * W)
    mask[:n_in] = 0
    return dict(pixel_values_latents=r(n, 4, H, W), plucker_embeds=r(n, 6, 8 * H, 8 * W), skeletons_latents=r(n, 4, H, W),
                cond_masks=mask, latents=r(n, 4, H, W), domain=domain, timestep_indices=torch.zeros(n, dtype=torch.long))


def _run(task, sh_or_pipe, generator):
    _, domain, n_in, n_tg, ws, stride, bidir, steps, dpm, noise = task
    kw = _task_inputs(domain, n_in, n_tg)
    if noise:
        kw["latents"] = None
    return sh_or_pipe.sliding_iterative_denoise(**kw, window_size=ws, sliding_stride=stride, bidirectional=bidir,
                                                num_denoising_steps=steps, alternation_rounds=2, guidance_scale=2.0,
                                                generator=generator)


def _result(out, state):
    res = {k: out[k].clone() for k in ("latents", "timestep_indices", "fully_denoised")}
    if state is not None:
        res["x0_prev"], res["lower_order_nums"] = state.x0_prev.clone(), state.lower_order_nums.clone()
    return res


def _gloo_worker(rank, world, store, out_dir):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=world)
    try:
        results = {}
        for task in TASKS:
            pipe = _pipe(task[8])
            box = _capture_state(pipe)
            sh = _sharded(pipe, rank, world)
            sh._step_and_exchange = _gathered_standin(sh)
            # each rank draws different noise: the loop must step rank 0's on every rank
            out = _run(task, sh, torch.Generator().manual_seed(100 + rank))
            results[task[0]] = _result(out, box[-1])
        torch.save(results, os.path.join(out_dir, f"rank{rank}.pt"))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_gloo_sharded_loop_equals_plain_loop(tmp_path, world):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, str(tmp_path / "store"), str(tmp_path)))
             for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0, f"gloo worker exited with {p.exitcode}"
    got = [torch.load(tmp_path / f"rank{r}.pt") for r in range(world)]
    for task in TASKS:
        pipe = _pipe(task[8])
        box = _capture_state(pipe)
        pipe.denoise_window = _plain_standin
        ref = _result(_run(task, pipe, torch.Generator().manual_seed(100)), box[-1])
        assert ref["timestep_indices"].max() > 0
        for r in range(world):
            res = got[r][task[0]]
            assert res.keys() == ref.keys()
            for k in ref:
                assert torch.equal(res[k], ref[k]), f"{task[0]} rank {r} of {world}: {k} differs from the plain loop"


def test_indivisible_window_is_refused_before_any_window(monkeypatch):
    """A 6-frame window on 4 ranks: the frame_shard message, raised before the loop prepares the task."""
    pipe = _pipe(False)
    sh = _sharded(pipe, 1, 4)

    def boom(*a, **k):
        raise AssertionError("the loop ran")
    monkeypatch.setattr(pipe, "_sliding", boom)
    sh._step_and_exchange = boom
    kw = _task_inputs("spatial", 2, 8)
    with pytest.raises(ValueError, match=r"num_frames \(6\) must be divisible by the number of ranks \(4\)"):
        sh.sliding_iterative_denoise(**kw, window_size=4, sliding_stride=1, bidirectional=False, alternation_rounds=1)
    # a divisible window reaches the loop
    with pytest.raises(AssertionError, match="the loop ran"):
        sh.sliding_iterative_denoise(**kw, window_size=6, sliding_stride=1, bidirectional=False, alternation_rounds=1)


WINDOW_REFUSALS = [  # (case, F_total, message); the frame-sharded step runs on rank 0 of 2 with 2 local frames
    ("invalid-domain", 4, "Invalid domain for temporal embedding: diagonal"),
    ("cpu-latents", 4, "latents must be a contiguous CUDA bfloat16 tensor (updated in place)"),
    ("F_total-mismatch", 6, "F_total (6) must equal world (2) * local frames (2)"),
]


@pytest.mark.parametrize("dpm", [False, True], ids=["ddim", "dpm"])
@pytest.mark.parametrize("case,F_total,msg", WINDOW_REFUSALS, ids=[r[0] for r in WINDOW_REFUSALS])
def test_sharded_window_refusals_before_any_library_call(monkeypatch, case, F_total, msg, dpm):
    """The frame-sharded window step refuses these inputs with the single-GPU step's message (the F_total mismatch has no
    single-GPU counterpart), before the library is loaded."""
    import diffuman4d_b200.pipeline as pipeline_mod
    monkeypatch.setattr(pipeline_mod, "lib", lambda: pytest.fail("the library was called"))
    pipe = _pipe(dpm)
    sh = _sharded(pipe, 0, 2)
    r = lambda c: torch.zeros(2, c, H, W, dtype=torch.bfloat16)
    kw = dict(latents=r(4), pixel_values_latents=r(4), plucker_embeds_latents=r(6), skeletons_latents=r(4),
              cond_masks_latents=r(1), timestep_indices=torch.zeros(2, dtype=torch.int64),
              domain="diagonal" if case == "invalid-domain" else "spatial", guidance_scale=2.0)
    calls = [lambda: sh.denoise_window(F_total=F_total, **kw)]
    if case != "F_total-mismatch":
        calls.append(lambda: pipe.denoise_window(**kw))
    for call in calls:
        with pytest.raises(ValueError) as e:
            call()
        assert str(e.value) == msg


def test_sampler_frame_sharded_needs_a_sharded_pipeline():
    from diffuman4d_b200.sampler import B200SlidingIterativeSampler
    ds = types.SimpleNamespace(scene_label="s")
    s = B200SlidingIterativeSampler(ds, [_pipe(False)], output_dir=None, spa_label_range=[0, 6, 1],
                                    tem_label_range=[0, 4, 1], input_spa_labels=[1, 4], window_size=2)
    with pytest.raises(ValueError, match="FrameShardedPipeline"):
        s.execute_tasks(frame_sharded=True)
