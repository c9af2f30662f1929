"""Host logic of the CFG-split window (``CFGSplitPipeline``) on the CPU.

* The refusals: an uninitialised ``torch.distributed`` and a world other than 1 or 2 before any library call, the
  window step's argument errors with the single-GPU step's messages, and the sampler's mode checks.
* Every scheduler tables class names a CFG-split entry point, and the library binding exports it.
* The exchange-size formula.
* A gloo job of 2 processes runs the split sliding loop with its device step replaced by a stand-in; the ranks draw
  different noise and both end with the single-process loop's result on rank 0's noise.
"""
import os
import types

import pytest
import torch

from diffuman4d_b200.config import (DEISConfig, DPMSingleConfig, DPMSolverConfig, PNDMConfig, SchedulerConfig,
                                    UNetConfig, UniPCConfig)
from diffuman4d_b200.pipeline import B200Diffuman4DPipeline

H = W = 8
CONFIGS = [SchedulerConfig(), DPMSolverConfig(), UniPCConfig(), PNDMConfig(), DEISConfig(), DPMSingleConfig()]


class _UNetStub:
    """What the pipeline's host code reads of the UNet (no library call is made with it)."""

    def __init__(self):
        self.device = torch.device("cpu")
        self.config = UNetConfig.tiny()


def _pipe(sched=None):
    return B200Diffuman4DPipeline(_UNetStub(), sched)


def _split(pipe, rank, world):
    """A CFGSplitPipeline without an exchange buffer (its device calls are replaced)."""
    from diffuman4d_b200.cfg_split import CFGSplitPipeline
    sp = CFGSplitPipeline.__new__(CFGSplitPipeline)
    sp.pipe, sp.group, sp.rank, sp.world = pipe, None, rank, world
    return sp


@pytest.fixture
def no_library(monkeypatch):
    import diffuman4d_b200.pipeline as pipeline_mod
    import diffuman4d_b200.sharded as sharded_mod
    fail = lambda: pytest.fail("the library was called")
    monkeypatch.setattr(pipeline_mod, "lib", fail)
    monkeypatch.setattr(sharded_mod, "lib", fail)


# ------------------------------------------------------------------------------------------------ refusals
def test_needs_torch_distributed(no_library):
    from diffuman4d_b200.cfg_split import CFGSplitPipeline
    import torch.distributed as dist
    assert not dist.is_initialized()
    with pytest.raises(RuntimeError, match="torch.distributed must be initialised"):
        CFGSplitPipeline(_pipe(), 4, H, W)


@pytest.mark.parametrize("world", [3, 4, 8])
def test_refuses_worlds_other_than_one_or_two(no_library, monkeypatch, world):
    import torch.distributed as dist
    from diffuman4d_b200.cfg_split import CFGSplitPipeline
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: world)
    monkeypatch.setattr(dist, "get_rank", lambda group=None: pytest.fail("the exchange was opened"))
    with pytest.raises(ValueError, match=f"runs on 2 ranks \\(or 1 as a loopback\\), not {world}"):
        CFGSplitPipeline(_pipe(), 4, H, W)


WINDOW_REFUSALS = [  # (case, message)
    ("invalid-domain", "Invalid domain for temporal embedding: diagonal"),
    ("cpu-latents", "latents must be a contiguous CUDA bfloat16 tensor (updated in place)"),
]


@pytest.mark.parametrize("sched", CONFIGS, ids=lambda c: type(c).__name__)
@pytest.mark.parametrize("case,msg", WINDOW_REFUSALS, ids=[r[0] for r in WINDOW_REFUSALS])
def test_window_refusals_before_any_library_call(no_library, case, msg, sched):
    """The split step refuses these inputs with the single-GPU step's message, before the library is loaded."""
    pipe = _pipe(sched)
    sp = _split(pipe, 1, 2)
    r = lambda c: torch.zeros(2, c, H, W, dtype=torch.bfloat16)
    kw = dict(latents=r(4), pixel_values_latents=r(4), plucker_embeds_latents=r(6), skeletons_latents=r(4),
              cond_masks_latents=r(1), timestep_indices=torch.zeros(2, dtype=torch.int64),
              domain="diagonal" if case == "invalid-domain" else "spatial", guidance_scale=2.0)
    for call in (lambda: sp.denoise_window(**kw), lambda: pipe.denoise_window(**kw)):
        with pytest.raises(ValueError) as e:
            call()
        assert str(e.value) == msg


def _sampler(pipe):
    from diffuman4d_b200.sampler import B200SlidingIterativeSampler
    ds = types.SimpleNamespace(scene_label="s")
    return B200SlidingIterativeSampler(ds, [pipe], output_dir=None, spa_label_range=[0, 6, 1],
                                       tem_label_range=[0, 4, 1], input_spa_labels=[1, 4], window_size=2)


def test_sampler_cfg_split_needs_a_split_pipeline():
    from diffuman4d_b200.sharded import FrameShardedPipeline
    with pytest.raises(ValueError, match="cfg_split=True needs a CFGSplitPipeline"):
        _sampler(_pipe()).execute_tasks(cfg_split=True)
    sh = FrameShardedPipeline.__new__(FrameShardedPipeline)
    sh.pipe, sh.group, sh.rank, sh.world = _pipe(), None, 0, 1
    with pytest.raises(ValueError, match="cfg_split=True needs a CFGSplitPipeline"):
        _sampler(sh).execute_tasks(cfg_split=True)


def test_sampler_refuses_both_modes():
    with pytest.raises(ValueError, match="pass one of them"):
        _sampler(_split(_pipe(), 0, 2)).execute_tasks(frame_sharded=True, cfg_split=True)


# ------------------------------------------------------------------------------------------------ entry points, sizes
@pytest.mark.parametrize("sched", CONFIGS, ids=lambda c: type(c).__name__)
def test_every_scheduler_has_a_split_entry_point(sched):
    from diffuman4d_b200._lib import EXPORTS
    plain, _, split = _pipe(sched).scheduler.window_entry_points
    assert split == plain + "_cfg_split"
    assert split in EXPORTS


def test_noise_exchange_bytes():
    from diffuman4d_b200.cfg_split import noise_exchange_bytes
    cfg = UNetConfig.sd21()
    # W16 at 64x64 latents: each half is 16 x 4 x 64 x 64 bf16 = 0.5 MiB, and the buffer holds both
    assert noise_exchange_bytes(cfg, 16, 64, 64) == 2 * (1 << 19)
    assert noise_exchange_bytes(cfg, 3, 8, 16) == 2 * 3 * cfg.out_channels * 8 * 16 * 2


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


def _task_inputs(seed=5):
    n_in, n_tg = 4, 8
    n = n_in + n_tg
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    mask = torch.ones(n, 1, 8 * H, 8 * W)
    mask[:n_in] = 0
    return dict(pixel_values_latents=r(n, 4, H, W), plucker_embeds=r(n, 6, 8 * H, 8 * W), skeletons_latents=r(n, 4, H, W),
                cond_masks=mask, latents=None, domain="spatial", timestep_indices=torch.zeros(n, dtype=torch.long),
                window_size=4, sliding_stride=2, bidirectional=True, num_denoising_steps=1, alternation_rounds=2,
                guidance_scale=2.0)


def _gloo_worker(rank, world, store, out_dir):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=world)
    try:
        sp = _split(_pipe(), rank, world)
        sp.denoise_window = _standin
        # each rank draws different noise: the loop must step rank 0's on every rank
        out = sp.sliding_iterative_denoise(**_task_inputs(), generator=torch.Generator().manual_seed(100 + rank))
        torch.save({k: out[k] for k in ("latents", "timestep_indices")}, os.path.join(out_dir, f"rank{rank}.pt"))
    finally:
        dist.destroy_process_group()


def test_gloo_ranks_end_with_rank0_noise_result(tmp_path):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, str(tmp_path / "store"), str(tmp_path))) for r in range(2)]
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
    ref = pipe.sliding_iterative_denoise(**_task_inputs(), generator=torch.Generator().manual_seed(100))
    other = pipe.sliding_iterative_denoise(**_task_inputs(), generator=torch.Generator().manual_seed(101))
    assert not torch.equal(other["latents"], ref["latents"]), "the two ranks' noise must differ"
    for r in range(2):
        got = torch.load(tmp_path / f"rank{r}.pt")
        for k in ("latents", "timestep_indices"):
            assert torch.equal(got[k], ref[k]), f"rank {r}: {k} differs from the loop on rank 0's noise"
