"""Host logic of the CFG grid (``CFGGridPipeline``: the CFG-split window on 2R ranks) on the CPU.

* Worlds: 3, 5, 7 and 9 are refused before the exchange opens; 1, 2, 4, 6 and 8 open it with ``grid_exchange_bytes``.
* The rank map: for every ``build_windows`` schedule of ``test_sharded_sampling.py`` and every R that divides a window,
  the 2R ranks' noise rows cover each of the window's 2F rows exactly once, in the (half, frame shard) order the library
  stores them.
* A window that R does not divide is refused before any library call, by the window step and by the sliding loop (before
  any window runs); with guidance 1 there are no halves and nothing is refused.
* Every scheduler's grid entry point is exported, and ``CFGSplitPipeline`` still refuses worlds other than 1 and 2.
* ``grid_exchange_bytes`` for the SD-2.1 layout at W16 and W24, 64x64 latents.
* ``execute_tasks(cfg_split=True)`` accepts a grid pipeline.
* A gloo job of 4 processes (a 2x2 grid) runs the grid sliding loop with its device step replaced by a stand-in; every
  rank ends with the single-process loop's result on rank 0's noise.
"""
import os
import types

import pytest
import torch

from diffuman4d_b200.config import (DEISConfig, DPMSingleConfig, DPMSolverConfig, PNDMConfig, SchedulerConfig,
                                    UNetConfig, UniPCConfig)
from diffuman4d_b200.pipeline import B200Diffuman4DPipeline, build_windows

from test_sharded_sampling import SCHEDULES  # noqa: E402

H = W = 8
CONFIGS = [SchedulerConfig(), DPMSolverConfig(), UniPCConfig(), PNDMConfig(), DEISConfig(), DPMSingleConfig()]


class _UNetStub:
    """What the pipeline's host code reads of the UNet (no library call is made with it)."""

    def __init__(self):
        self.device = torch.device("cpu")
        self.config = UNetConfig.tiny()
        self._h = None


def _pipe(sched=None):
    return B200Diffuman4DPipeline(_UNetStub(), sched)


def _grid(pipe, rank, world):
    """A CFGGridPipeline without an exchange buffer (its device calls are replaced)."""
    from diffuman4d_b200.cfg_split import CFGGridPipeline
    gp = CFGGridPipeline.__new__(CFGGridPipeline)
    gp.pipe, gp.group, gp.rank, gp.world = pipe, None, rank, world
    return gp


@pytest.fixture
def no_library(monkeypatch):
    import diffuman4d_b200.pipeline as pipeline_mod
    import diffuman4d_b200.sharded as sharded_mod
    fail = lambda: pytest.fail("the library was called")
    monkeypatch.setattr(pipeline_mod, "lib", fail)
    monkeypatch.setattr(sharded_mod, "lib", fail)


@pytest.fixture
def fake_dist(monkeypatch):
    """torch.distributed reporting an initialised world; ``open_exchange`` records its calls instead of opening."""
    import torch.distributed as dist
    import diffuman4d_b200.cfg_split as cs
    state = types.SimpleNamespace(world=1, opened=[])
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: state.world)

    def fake_open(pipe, nbytes, group=None):
        state.opened.append(nbytes)
        return 0, state.world
    monkeypatch.setattr(cs, "open_exchange", fake_open)
    return state


# ------------------------------------------------------------------------------------------------ worlds
@pytest.mark.parametrize("world", [3, 5, 7, 9])
def test_refuses_other_worlds_before_the_exchange_opens(no_library, fake_dist, world):
    from diffuman4d_b200.cfg_split import CFGGridPipeline
    fake_dist.world = world
    with pytest.raises(ValueError, match=f"runs on 2 \\* R ranks with R in 1..4 \\(or 1 as a loopback\\), not {world}"):
        CFGGridPipeline(_pipe(), 4, H, W)
    assert fake_dist.opened == []


@pytest.mark.parametrize("world", [1, 2, 4, 6, 8])
def test_accepts_grid_worlds(no_library, fake_dist, world):
    from diffuman4d_b200.cfg_split import CFGGridPipeline, grid_exchange_bytes
    fake_dist.world = world
    gp = CFGGridPipeline(_pipe(), 12, H, W)
    assert (gp.rank, gp.world) == (0, world)
    assert fake_dist.opened == [grid_exchange_bytes(UNetConfig.tiny(), 12, H, W)]


def test_split_pipeline_still_refuses_grid_worlds(no_library, fake_dist):
    from diffuman4d_b200.cfg_split import CFGSplitPipeline
    fake_dist.world = 4
    with pytest.raises(ValueError, match="runs on 2 ranks \\(or 1 as a loopback\\), not 4"):
        CFGSplitPipeline(_pipe(), 4, H, W)
    assert fake_dist.opened == []


# ------------------------------------------------------------------------------------------------ rank map
def test_grid_cell_matches_the_documented_layout():
    from diffuman4d_b200.cfg_split import grid_cell
    assert [grid_cell(g, 8) for g in range(8)] == [(g // 4, g % 4, 4) for g in range(8)]
    assert [grid_cell(g, 6)[:2] for g in range(6)] == [(0, 0), (0, 1), (0, 2), (1, 0), (1, 1), (1, 2)]
    assert [grid_cell(g, 2) for g in range(2)] == [(0, 0, 1), (1, 0, 1)]
    assert grid_cell(0, 1) == (0, 0, 1)


@pytest.mark.parametrize("sched", SCHEDULES, ids=[f"{s[0]}-{s[1]}+{s[2]}-w{s[3]}-s{s[4]}-{'bi' if s[5] else 'uni'}"
                                                  for s in SCHEDULES])
def test_rank_map_covers_every_noise_row_once(sched):
    from diffuman4d_b200.cfg_split import grid_noise_rows
    domain, n_in, n_tg, ws, stride, bidir = sched
    tws, iws = build_windows(torch.arange(n_in, n_in + n_tg), torch.arange(n_in), domain, ws, stride, 0, bidir)
    assert tws
    tested = 0
    for tw, iw in zip(tws, iws):
        F = len(tw) + len(iw)
        for R in (1, 2, 3, 4):
            world = 2 * R
            if F % R:
                with pytest.raises(ValueError, match="must be divisible by the number of ranks"):
                    grid_noise_rows(F, world - 1, world)
                continue
            hits = torch.zeros(2 * F, dtype=torch.int64)
            for g in range(world):
                lo, hi = grid_noise_rows(F, g, world)
                assert hi - lo == F // R
                # rank g's rows: half g // R, frames of shard g % R
                assert (lo // F, (lo % F) // (F // R)) == (g // R, g % R)
                hits[lo:hi] += 1
            assert torch.equal(hits, torch.ones(2 * F, dtype=torch.int64)), (R, F)
            tested += 1
        assert grid_noise_rows(F, 0, 1) == (0, 2 * F)   # the loopback runs both halves
    assert tested > len(tws)


# ------------------------------------------------------------------------------------------------ refusals
def _window_kw(F, guidance=2.0):
    r = lambda c: torch.zeros(F, c, H, W, dtype=torch.bfloat16)
    return dict(latents=r(4), pixel_values_latents=r(4), plucker_embeds_latents=r(6), skeletons_latents=r(4),
                cond_masks_latents=r(1), timestep_indices=torch.zeros(F, dtype=torch.int64), domain="spatial",
                guidance_scale=guidance)


@pytest.mark.parametrize("sched", CONFIGS, ids=lambda c: type(c).__name__)
def test_indivisible_window_is_refused_before_any_library_call(no_library, sched):
    """A 6-frame window on a 2x4 grid: frame_shard's message.  With guidance 1 there are no halves, so the window goes on
    to the step's own checks (here the single-GPU step's refusal of CPU latents)."""
    gp = _grid(_pipe(sched), 5, 8)
    with pytest.raises(ValueError, match=r"num_frames \(6\) must be divisible by the number of ranks \(4\)"):
        gp.denoise_window(**_window_kw(6))
    with pytest.raises(ValueError, match="latents must be a contiguous CUDA bfloat16 tensor"):
        gp.denoise_window(**_window_kw(6, guidance=1.0))
    with pytest.raises(ValueError, match="latents must be a contiguous CUDA bfloat16 tensor"):
        gp.denoise_window(**_window_kw(8))


def _task_inputs(domain="spatial", n_in=4, n_tg=8, seed=5):
    n = n_in + n_tg
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    mask = torch.ones(n, 1, 8 * H, 8 * W)
    mask[:n_in] = 0
    return dict(pixel_values_latents=r(n, 4, H, W), plucker_embeds=r(n, 6, 8 * H, 8 * W), skeletons_latents=r(n, 4, H, W),
                cond_masks=mask, latents=None, domain=domain, timestep_indices=torch.zeros(n, dtype=torch.long))


def test_sliding_loop_refuses_an_indivisible_window_before_any_window(monkeypatch):
    pipe = _pipe()
    gp = _grid(pipe, 5, 8)

    def boom(*a, **k):
        raise AssertionError("the loop ran")
    monkeypatch.setattr(pipe, "_sliding", boom)
    gp.denoise_window = boom
    kw = _task_inputs("spatial", 2, 8)
    # window 4 holds 4 targets and the 2 inputs: 6 frames on a 2x4 grid
    with pytest.raises(ValueError, match=r"num_frames \(6\) must be divisible by the number of ranks \(4\)"):
        gp.sliding_iterative_denoise(**kw, window_size=4, sliding_stride=1, bidirectional=False, alternation_rounds=1)
    # a divisible window, or no halves, reaches the loop
    for ws, guidance in ((6, 2.0), (4, 1.0)):
        with pytest.raises(AssertionError, match="the loop ran"):
            gp.sliding_iterative_denoise(**kw, window_size=ws, sliding_stride=1, bidirectional=False,
                                         alternation_rounds=1, guidance_scale=guidance)


# ------------------------------------------------------------------------------------------------ entry points, sizes
@pytest.mark.parametrize("sched", CONFIGS, ids=lambda c: type(c).__name__)
def test_every_scheduler_has_a_grid_entry_point(sched):
    from diffuman4d_b200._lib import EXPORTS
    plain = _pipe(sched).scheduler.window_entry_points[0]
    assert plain + "_cfg_grid" in EXPORTS


def test_grid_exchange_bytes():
    from diffuman4d_b200.cfg_split import grid_exchange_bytes, noise_exchange_bytes
    from diffuman4d_b200.sharded import exchange_bytes
    cfg = UNetConfig.sd21()
    # the largest 3-D layer is level 1 (32x32 tokens per frame, 10 heads x 64): one half at W16 is 16 x 1024 rows of
    # 2 x 640 bf16 = 40 MiB, at W24 60 MiB; the gathered noise (1 and 1.5 MiB) is smaller
    assert grid_exchange_bytes(cfg, 16, 64, 64) == 41943040
    assert grid_exchange_bytes(cfg, 24, 64, 64) == 62914560
    assert exchange_bytes(cfg, 16, 64, 64) == 2 * grid_exchange_bytes(cfg, 16, 64, 64)
    # a model without 3-D layers at this size still needs the noise
    tiny = UNetConfig.tiny()
    assert grid_exchange_bytes(tiny, 4, 8, 8) == max(exchange_bytes(tiny, 4, 8, 8, cfg_halves=1),
                                                     noise_exchange_bytes(tiny, 4, 8, 8))


def _sampler(pipe):
    from diffuman4d_b200.sampler import B200SlidingIterativeSampler
    ds = types.SimpleNamespace(scene_label="s")
    return B200SlidingIterativeSampler(ds, [pipe], output_dir=None, spa_label_range=[0, 6, 1],
                                       tem_label_range=[0, 4, 1], input_spa_labels=[1, 4], window_size=2)


def test_sampler_cfg_split_accepts_a_grid_pipeline():
    """The mode check passes and the sampler goes on to its first task (stopped there)."""
    s = _sampler(_grid(_pipe(), 0, 4))
    s.prefetch = False
    s._fetch = lambda **task: {}
    s._attach_grid = lambda raw: raw

    def first_task(*a, **k):
        raise AssertionError("the sampler ran a task")
    s.denoise = first_task
    with pytest.raises(AssertionError, match="the sampler ran a task"):
        s.execute_tasks(cfg_split=True)


# ------------------------------------------------------------------------------------------------ stand-in step
def _standin(*, latents, pixel_values_latents, cond_masks_latents, timestep_indices, num_inference_steps,
             solver_state=None, **_):
    """A per-frame denoiser in place of the device step; conditioning frames receive their image latents and index 0."""
    cond = cond_masks_latents[:, 0, 0, 0] == 0
    for _ in range(num_inference_steps):
        new = latents.float() * 0.75 + pixel_values_latents.float() * 0.25 - 0.01 * timestep_indices.view(-1, 1, 1, 1)
        latents.copy_(torch.where(cond.view(-1, 1, 1, 1), pixel_values_latents, new.to(torch.bfloat16)))
        timestep_indices.copy_(torch.where(cond, torch.zeros_like(timestep_indices), timestep_indices + 1))
    return latents, timestep_indices


LOOP = dict(window_size=4, sliding_stride=2, bidirectional=True, num_denoising_steps=1, alternation_rounds=2,
            guidance_scale=2.0)


def _gloo_worker(rank, world, store, out_dir):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=world)
    try:
        gp = _grid(_pipe(), rank, world)
        seen = []

        def step(**kw):
            seen.append(kw["latents"].shape[0])
            return _standin(**kw)
        gp.pipe._window_step = lambda cfg_grid, **kw: step(**kw)
        # each rank draws different noise: the loop must step rank 0's on every rank
        out = gp.sliding_iterative_denoise(**_task_inputs(), **LOOP, generator=torch.Generator().manual_seed(100 + rank))
        assert seen and all(f % 2 == 0 for f in seen)
        torch.save({k: out[k] for k in ("latents", "timestep_indices")}, os.path.join(out_dir, f"rank{rank}.pt"))
    finally:
        dist.destroy_process_group()


def test_gloo_grid_ranks_end_with_rank0_noise_result(tmp_path):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_gloo_worker, args=(r, 4, str(tmp_path / "store"), str(tmp_path))) for r in range(4)]
    for p in procs:
        p.start()
    try:
        for p in procs:
            p.join(timeout=300)
        for r, p in enumerate(procs):
            assert p.exitcode == 0, f"gloo worker {r} exited with {p.exitcode}"
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
    pipe = _pipe()
    pipe.denoise_window = _standin
    ref = pipe.sliding_iterative_denoise(**_task_inputs(), **LOOP, generator=torch.Generator().manual_seed(100))
    for r in range(4):
        got = torch.load(tmp_path / f"rank{r}.pt")
        for k in ("latents", "timestep_indices"):
            assert torch.equal(got[k], ref[k]), f"rank {r}: {k} differs from the loop on rank 0's noise"
