"""CFG-split window denoise step across two GPUs (DESIGN.md section 7).

With classifier-free guidance on, a window step runs the UNet on 2F images: the F negative images, then the F positive
ones.  The two halves never read each other (3-D attention runs one sequence per half); they meet in the CFG combine in
front of the scheduler step.  So rank 0 runs the UNet on the negative half and rank 1 on the positive half (one process
per GPU, torch.distributed); the UNet's output permute stores each half's noise into both ranks' exchange buffers over
peer memory, one flag round publishes it, and both ranks run the unchanged scheduler step on the whole window.  They
compute the step from the same bits, so every rank holds the same latents, timestep indices and solver state afterwards:
there is no state to exchange, and every device scheduler runs this way.

Each rank passes the whole window and gets the whole result, bit-identical to ``B200Diffuman4DPipeline``.  World 1 is a
loopback on one GPU (rank 0 runs both halves into its own buffer).  With ``guidance_scale <= 1`` there are no halves:
every rank runs the plain single-GPU step, exchanges nothing, and gains nothing from the second GPU.

``CFGGridPipeline`` runs the same window step on 2R ranks (R = 1, 2, 3 or 4): each CFG half is frame-sharded over R
ranks, whose 3-D attention layers exchange K|V among themselves like the frame-sharded window, and every rank's noise
shard still lands in every rank's exchange buffer, so the step stays replicated and no solver state moves.
"""
from __future__ import annotations

from typing import Callable

import torch
import torch.distributed as dist

from .pipeline import B200Diffuman4DPipeline, build_windows
from .sharded import FrameShardedPipeline, exchange_bytes, open_exchange
from .sharding import frame_shard


def noise_exchange_bytes(cfg, max_frames: int, h: int, w: int) -> int:
    """Size of one exchange buffer of the CFG-split window: the gathered noise of both halves, bf16
    [2 * max_frames, out_channels, h, w]."""
    return 2 * max_frames * cfg.out_channels * h * w * 2


def grid_exchange_bytes(cfg, max_frames: int, h: int, w: int) -> int:
    """Size of one exchange buffer of the CFG grid: the larger of one CFG half's largest gathered 3-D K|V layer and the
    gathered noise of both halves, for windows of up to ``max_frames`` frames."""
    return max(exchange_bytes(cfg, max_frames, h, w, cfg_halves=1), noise_exchange_bytes(cfg, max_frames, h, w))


def grid_cell(rank: int, world: int):
    """``(k, r, R)`` of global ``rank`` in the CFG grid of ``world`` = 2R ranks: CFG half k (0 negative) and frame shard r
    of R per half.  A world of 1 is a loopback (R = 1; the rank runs both halves)."""
    R = 1 if world == 1 else world // 2
    return rank // R, rank % R, R


def grid_noise_rows(F: int, rank: int, world: int):
    """Rows ``[lo, hi)`` of a window's gathered noise [2F] (the negative half, then the positive half) that ``rank`` of
    the CFG grid computes and stores into every rank's exchange buffer: the rows of its frame shard in its half, or all
    2F on a loopback.  Raises ``frame_shard``'s ValueError when R does not divide F."""
    if world == 1:
        return 0, 2 * F
    k, r, R = grid_cell(rank, world)
    lo, hi = frame_shard(F, r, R)
    return k * F + lo, k * F + hi


class CFGSplitPipeline:
    def __init__(self, pipe: B200Diffuman4DPipeline, max_frames: int, h: int, w: int, group=None):
        """Opens the noise exchange of ``pipe``'s handle for windows of up to ``max_frames`` frames of ``h`` x ``w``
        latents.  Every rank of ``group`` (2 ranks, or 1 for a loopback) constructs it (SPMD)."""
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed must be initialised (one process per GPU)")
        self._check_world(dist.get_world_size(group))
        self.pipe = pipe
        self.group = group
        self.rank, self.world = open_exchange(pipe, self._exchange_bytes(pipe.unet.config, max_frames, h, w), group)

    @staticmethod
    def _check_world(world: int):
        if world not in (1, 2):
            raise ValueError(f"the CFG-split window runs on 2 ranks (or 1 as a loopback), not {world}")

    _exchange_bytes = staticmethod(noise_exchange_bytes)

    device = FrameShardedPipeline.device
    vae = FrameShardedPipeline.vae
    _share_noise = FrameShardedPipeline._share_noise

    def denoise_window(self, **kw):
        """B-3 with this rank running the UNet on its CFG half: the arguments, checks and in-place updates of
        ``B200Diffuman4DPipeline.denoise_window``, on the whole window on every rank.  SPMD: both ranks make the same
        calls with the same arguments."""
        return self.pipe._window_step(cfg_split=True, **kw)

    def _task_window(self, window, lw, tiw, sw, conds, **kw):
        """``B200Diffuman4DPipeline._task_window`` with the CFG-split step."""
        pix, plk, skl, msk = (t[window] for t in conds)
        self.denoise_window(latents=lw, pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skl,
                            cond_masks_latents=msk, timestep_indices=tiw, solver_state=sw, **kw)
        return lw, sw

    @torch.no_grad()
    def sliding_iterative_denoise(self, pixel_values=None, plucker_embeds=None, skeletons=None, cond_masks=None,
                                  latents=None, domain: str = "spatial", timestep_indices=None, window_size: int = 12,
                                  sliding_stride: int = 1, sliding_shift: int = 0, bidirectional: bool = True,
                                  num_denoising_steps: int = 1, alternation_rounds: int = 3, guidance_scale: float = 2.0,
                                  tqdm: Callable = None, pixel_values_latents=None, skeletons_latents=None,
                                  generator=None):
        """B-4 (``B200Diffuman4DPipeline.sliding_iterative_denoise``: same arguments, errors and returned dict) with every
        window step split by CFG half over the ranks.  Every rank passes the whole task and gets the whole result,
        bit-identical to the single-GPU loop; freshly drawn initial noise is rank 0's on every rank."""
        return self.pipe._sliding(
            self._task_window, pixel_values=pixel_values, plucker_embeds=plucker_embeds, skeletons=skeletons,
            cond_masks=cond_masks, latents=latents, domain=domain, timestep_indices=timestep_indices,
            window_size=window_size, sliding_stride=sliding_stride, sliding_shift=sliding_shift,
            bidirectional=bidirectional, num_denoising_steps=num_denoising_steps, alternation_rounds=alternation_rounds,
            guidance_scale=guidance_scale, tqdm=tqdm, pixel_values_latents=pixel_values_latents,
            skeletons_latents=skeletons_latents, generator=generator, share_noise=self._share_noise)


class CFGGridPipeline(CFGSplitPipeline):
    """The CFG-split window on 2R ranks (R = 1, 2, 3 or 4): rank g runs CFG half ``g // R`` (ranks 0 .. R-1 the negative
    half) on frame shard ``g % R`` of the window.  Arguments, results and SPMD rules are those of ``CFGSplitPipeline``;
    with guidance above 1 every window's frame count must be divisible by R.  With R = 1 (world 1 or 2) it is the CFG
    split.  ``execute_tasks(cfg_split=True)`` runs it like its base class."""

    @staticmethod
    def _check_world(world: int):
        if world not in (1, 2, 4, 6, 8):
            raise ValueError(f"the CFG grid runs on 2 * R ranks with R in 1..4 (or 1 as a loopback), not {world}")

    _exchange_bytes = staticmethod(grid_exchange_bytes)

    def denoise_window(self, **kw):
        """B-3 with this rank running the UNet on its frame shard of its CFG half: the arguments, checks and in-place
        updates of ``B200Diffuman4DPipeline.denoise_window``, on the whole window on every rank.  SPMD: every rank makes
        the same calls with the same arguments."""
        lat = kw.get("latents")
        if torch.is_tensor(lat) and self.pipe.has_cfg_halves(kw.get("guidance_scale", 1.0)):
            grid_noise_rows(lat.shape[0], self.rank, self.world)
        return self.pipe._window_step(cfg_grid=True, **kw)

    @torch.no_grad()
    def sliding_iterative_denoise(self, pixel_values=None, plucker_embeds=None, skeletons=None, cond_masks=None,
                                  latents=None, domain: str = "spatial", timestep_indices=None, window_size: int = 12,
                                  sliding_stride: int = 1, sliding_shift: int = 0, bidirectional: bool = True,
                                  num_denoising_steps: int = 1, alternation_rounds: int = 3, guidance_scale: float = 2.0,
                                  tqdm: Callable = None, pixel_values_latents=None, skeletons_latents=None,
                                  generator=None):
        """``CFGSplitPipeline.sliding_iterative_denoise`` on the grid.  With guidance above 1, a window whose frame count
        R does not divide is refused before any window runs."""
        if cond_masks is not None and self.pipe.has_cfg_halves(guidance_scale):
            flag = cond_masks[:, 0, 0, 0].cpu()
            tws, iws = build_windows(torch.where(flag != 0.0)[0], torch.where(flag == 0.0)[0], domain, window_size,
                                     sliding_stride, sliding_shift, bidirectional)
            for tw, iw in zip(tws, iws):
                grid_noise_rows(len(tw) + len(iw), self.rank, self.world)
        return super().sliding_iterative_denoise(
            pixel_values=pixel_values, plucker_embeds=plucker_embeds, skeletons=skeletons, cond_masks=cond_masks,
            latents=latents, domain=domain, timestep_indices=timestep_indices, window_size=window_size,
            sliding_stride=sliding_stride, sliding_shift=sliding_shift, bidirectional=bidirectional,
            num_denoising_steps=num_denoising_steps, alternation_rounds=alternation_rounds,
            guidance_scale=guidance_scale, tqdm=tqdm, pixel_values_latents=pixel_values_latents,
            skeletons_latents=skeletons_latents, generator=generator)
