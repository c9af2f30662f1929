"""Frame-sharded window denoise step across the GPUs of one box (SURVEY.md section 8e.2, DESIGN.md section 7).

One process per GPU (torch.distributed).  Rank r owns frames [r*F/R, (r+1)*F/R) of the window (both CFG halves of a
frame stay on the rank).  Everything except 3-D attention is per image and needs no communication; at each 3-D block
the fused-QKV GEMM epilogue stores K|V straight into every rank's gathered buffer over NVLink (peer memory mapped with
cudaIpc) -- there is no NCCL call on the data path.  torch.distributed is used to exchange the IPC handles, and once
per task to share freshly drawn initial noise.

``sliding_iterative_denoise`` runs whole tasks this way: every rank holds the whole task, steps its shard of each
window, and the window-result exchange (``d4d_window_exchange``, the same peer buffers) hands every rank the updated
frames of the whole window before the next window is gathered.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, List, Optional

import torch
import torch.distributed as dist

from ._lib import check, lib
from .pipeline import B200Diffuman4DPipeline, _check_inplace, build_windows
from .plan import modules, pad_head_dim
from .scheduler import DPMSolverState
from .sharding import frame_shard


def exchange_bytes(cfg, F_total: int, h: int, w: int, cfg_halves: int = 2) -> int:
    """Size of one gathered K|V buffer: the largest 3-D attention layer, its K|V columns (heads x padded head dim each)
    for every token of the window."""
    return max((cfg_halves * F_total * (h >> m.level) * (w >> m.level) * 2 * cfg.heads(m.level)
                * pad_head_dim(cfg.head_dim(m.level)) * 2 for m in modules(cfg) if m.is3d), default=0)


def open_exchange(pipe: B200Diffuman4DPipeline, nbytes: int, group=None):
    """Allocates this rank's exchange buffers (``nbytes`` each) on ``pipe``'s handle, all-gathers the cudaIpc handles over
    ``group`` and maps the peers' buffers.  Returns ``(rank, world)``.  Every rank of the group calls it (SPMD)."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    mine = (C.c_ubyte * 192)()
    with torch.cuda.device(pipe.device):
        check(lib().d4d_exchange_alloc(pipe.unet._h, nbytes, mine), "d4d_exchange_alloc")
    blobs: List[bytes] = [b""] * world
    dist.all_gather_object(blobs, bytes(mine), group=group)
    allh = (C.c_ubyte * (192 * world)).from_buffer_copy(b"".join(blobs))
    with torch.cuda.device(pipe.device):
        check(lib().d4d_exchange_open(pipe.unet._h, rank, world, allh), "d4d_exchange_open")
    dist.barrier(group=group)
    return rank, world


def window_result_bytes(F_total: int, h: int, w: int, dpm: bool = True) -> int:
    """Size of one gathered window result (``d4d_window_exchange``): latents (and DPM-Solver++ ``x0_prev``) bf16
    [F_total, 4, h, w], int64 timestep indices (and int32 ``lower_order_nums``) [F_total]."""
    return F_total * (4 * h * w * 2 * (2 if dpm else 1) + 8 + (4 if dpm else 0))


class FrameShardedPipeline:
    def __init__(self, pipe: B200Diffuman4DPipeline, max_frames: int, h: int, w: int, group=None):
        if pipe.scheduler.window_entry_points[1] is None:
            raise NotImplementedError(f"the frame-sharded window does not run the {pipe.scheduler.name} scheduler; use "
                                      "B200Diffuman4DPipeline on one GPU per task")
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed must be initialised (one process per GPU)")
        self.pipe = pipe
        self.group = group
        if dist.get_world_size(group) > 8:
            raise ValueError("at most 8 ranks (one NVSwitch domain)")
        # the buffers also carry the window results of the sliding loop, far smaller than any real model's K/V
        kv_bytes = max(exchange_bytes(pipe.unet.config, max_frames, h, w), window_result_bytes(max_frames, h, w))
        self.rank, self.world = open_exchange(pipe, kv_bytes, group)

    def frames(self, F_total: int):
        return frame_shard(F_total, self.rank, self.world)

    def _check_world(self, F_local: int, F_total: int):
        if F_local * self.world != F_total:
            raise ValueError(f"F_total ({F_total}) must equal world ({self.world}) * local frames ({F_local})")

    def unet_forward(self, sample, timestep, skeletons, domains: List[str], F_local: int, F_total: int):
        """B-2 on this rank's frames: sample [len(domains)*F_local, Cin, h, w] (CFG-major like the reference batch);
        otherwise the arguments and checks of ``B200MultiviewUNet.forward``."""
        self._check_world(F_local, F_total)
        return self.pipe.unet._forward(sample, timestep, skeletons, domains, F_local, F_total)

    def denoise_window(self, *, latents, F_total: int, **kw):
        """B-3 on this rank's frames: every tensor, ``latents`` [F_local,4,h,w] and with DPM-Solver++ ``solver_state``
        included, holds the LOCAL frames and is updated in place; otherwise the arguments and checks of
        ``B200Diffuman4DPipeline.denoise_window``."""
        if torch.is_tensor(latents):   # anything else is refused with the single-GPU message
            self._check_world(latents.shape[0], F_total)
        return self.pipe._window_step(latents=latents, F_total=F_total, **kw)

    def window_exchange(self, latents, timestep_indices, solver_state: Optional[DPMSolverState], F_total: int):
        """Every rank's updated frames to every rank: the LOCAL ``latents`` [F_local,4,h,w], ``timestep_indices`` and
        (DPM-Solver++) ``solver_state`` in, the whole window's (F_total frames, window order) out as new tensors
        ``(latents, timestep_indices, solver_state or None)``.  SPMD: every rank calls it after the same window step."""
        _check_inplace(latents, "latents", torch.bfloat16)
        _check_inplace(timestep_indices, "timestep_indices", torch.int64)
        F_local, c, h, w = latents.shape
        dev = latents.device
        lat = torch.empty(F_total, c, h, w, dtype=torch.bfloat16, device=dev)
        ts = torch.empty(F_total, dtype=torch.int64, device=dev)
        out = None
        ptrs = [None] * 4
        if solver_state is not None:
            _check_inplace(solver_state.x0_prev, "solver_state.x0_prev", torch.bfloat16)
            _check_inplace(solver_state.lower_order_nums, "solver_state.lower_order_nums", torch.int32)
            out = DPMSolverState(F_total, dev, torch.empty_like(lat), torch.empty(F_total, dtype=torch.int32, device=dev))
            ptrs = [solver_state.x0_prev.data_ptr(), solver_state.lower_order_nums.data_ptr(), out.x0_prev.data_ptr(),
                    out.lower_order_nums.data_ptr()]
        with torch.cuda.device(self.pipe.device):
            check(lib().d4d_window_exchange(
                self.pipe.unet._h, latents.data_ptr(), timestep_indices.data_ptr(), ptrs[0], ptrs[1], F_local, F_total, h,
                w, lat.data_ptr(), ts.data_ptr(), ptrs[2], ptrs[3], torch.cuda.current_stream(self.pipe.device).cuda_stream),
                "d4d_window_exchange")
        return lat, ts, out

    # B-4 on frame shards ----------------------------------------------------------------------------------
    @property
    def device(self):
        return self.pipe.device

    @property
    def vae(self):
        return self.pipe.vae

    def _step_and_exchange(self, lat, ts, state, conds, F_total: int, **kw):
        """The device work of one window on this rank: the sharded step on the local frames, then the window-result
        exchange.  Returns the gathered ``(latents, timestep_indices, solver_state or None)``."""
        pix, plk, skl, msk = conds
        self.denoise_window(latents=lat, pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skl,
                            cond_masks_latents=msk, timestep_indices=ts, F_total=F_total, solver_state=state, **kw)
        return self.window_exchange(lat, ts, state, F_total)

    def _task_window(self, window, lw, tiw, sw, conds, **kw):
        """``B200Diffuman4DPipeline._task_window`` on this rank's shard: slice, step, exchange; the gathered window
        replaces ``lw`` / ``sw`` (the plain loop's in-place update)."""
        F_total = len(window)
        lo, hi = self.frames(F_total)
        mine = window[lo:hi]
        state = None
        if sw is not None:
            state = DPMSolverState(hi - lo, sw.device, sw.x0_prev[lo:hi].contiguous(),
                                   sw.lower_order_nums[lo:hi].contiguous())
        lat, _, out = self._step_and_exchange(lw[lo:hi].contiguous(), tiw[lo:hi].contiguous(), state,
                                              tuple(t[mine] for t in conds), F_total, **kw)
        return lat, out

    def _share_noise(self, latents):
        """Rank 0's initial noise on every rank: each rank steps only its frames of the noise it holds."""
        if self.world > 1:
            src = 0 if self.group is None else dist.get_global_rank(self.group, 0)
            dist.broadcast(latents.view(torch.uint8), src=src, group=self.group)   # bytes: every backend moves them

    @torch.no_grad()
    def sliding_iterative_denoise(self, pixel_values=None, plucker_embeds=None, skeletons=None, cond_masks=None,
                                  latents=None, domain: str = "spatial", timestep_indices=None, window_size: int = 12,
                                  sliding_stride: int = 1, sliding_shift: int = 0, bidirectional: bool = True,
                                  num_denoising_steps: int = 1, alternation_rounds: int = 3, guidance_scale: float = 2.0,
                                  tqdm: Callable = None, pixel_values_latents=None, skeletons_latents=None,
                                  generator=None):
        """B-4 (``B200Diffuman4DPipeline.sliding_iterative_denoise``: same arguments, errors and returned dict) with every
        window frame-sharded over the ranks.  Every rank passes the whole task and gets the whole result; the result is
        bit-identical to the single-GPU loop.  Every window's frame count must be divisible by the number of ranks."""
        flag = cond_masks[:, 0, 0, 0].cpu()
        tws, iws = build_windows(torch.where(flag != 0.0)[0], torch.where(flag == 0.0)[0], domain, window_size,
                                 sliding_stride, sliding_shift, bidirectional)
        for tw, iw in zip(tws, iws):
            frame_shard(len(tw) + len(iw), self.rank, self.world)
        return self.pipe._sliding(
            self._task_window, pixel_values=pixel_values, plucker_embeds=plucker_embeds, skeletons=skeletons,
            cond_masks=cond_masks, latents=latents, domain=domain, timestep_indices=timestep_indices,
            window_size=window_size, sliding_stride=sliding_stride, sliding_shift=sliding_shift,
            bidirectional=bidirectional, num_denoising_steps=num_denoising_steps, alternation_rounds=alternation_rounds,
            guidance_scale=guidance_scale, tqdm=tqdm, pixel_values_latents=pixel_values_latents,
            skeletons_latents=skeletons_latents, generator=generator, share_noise=self._share_noise)
