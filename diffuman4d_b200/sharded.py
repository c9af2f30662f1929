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
from .pipeline import B200Diffuman4DPipeline, _DOMAIN_IDS, build_windows
from .scheduler import DDIMTables, DPMSolverState
from .sharding import frame_shard


def exchange_bytes(cfg, F_total: int, h: int, w: int, cfg_halves: int = 2) -> int:
    """Size of one gathered K|V buffer: the largest 3-D attention layer.  The mid block (level 3) always runs one; level
    L < 3 runs them (down_blocks.L, up_blocks.3-L) when 3 - L < num_3d_attn_blocks, so level 0 with 4."""
    best = 0
    for lvl in (0, 1, 2, 3):
        if lvl < 3 and 3 - lvl >= cfg.num_3d_attn_blocks:
            continue
        d = cfg.head_dim(lvl)
        dpad = 64 if d <= 64 else (128 if d <= 128 else 192)
        cp = cfg.heads(lvl) * dpad
        tokens = cfg_halves * F_total * (h >> lvl) * (w >> lvl)
        best = max(best, tokens * 2 * cp * 2)
    return best


def window_result_bytes(F_total: int, h: int, w: int, dpm: bool = True) -> int:
    """Size of one gathered window result (``d4d_window_exchange``): latents (and DPM-Solver++ ``x0_prev``) bf16
    [F_total, 4, h, w], int64 timestep indices (and int32 ``lower_order_nums``) [F_total]."""
    return F_total * (4 * h * w * 2 * (2 if dpm else 1) + 8 + (4 if dpm else 0))


class FrameShardedPipeline:
    def __init__(self, pipe: B200Diffuman4DPipeline, max_frames: int, h: int, w: int, group=None):
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed must be initialised (one process per GPU)")
        self.pipe = pipe
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        if self.world > 8:
            raise ValueError("at most 8 ranks (one NVSwitch domain)")
        # the buffers also carry the window results of the sliding loop, far smaller than any real model's K/V
        kv_bytes = max(exchange_bytes(pipe.unet.config, max_frames, h, w), window_result_bytes(max_frames, h, w))
        mine = (C.c_ubyte * 192)()
        with torch.cuda.device(pipe.device):
            check(lib().d4d_exchange_alloc(pipe.unet._h, kv_bytes, mine), "d4d_exchange_alloc")
        blobs: List[bytes] = [b""] * self.world
        dist.all_gather_object(blobs, bytes(mine), group=group)
        allh = (C.c_ubyte * (192 * self.world)).from_buffer_copy(b"".join(blobs))
        with torch.cuda.device(pipe.device):
            check(lib().d4d_exchange_open(pipe.unet._h, self.rank, self.world, allh), "d4d_exchange_open")
        dist.barrier(group=group)

    def frames(self, F_total: int):
        return frame_shard(F_total, self.rank, self.world)

    def _bf16(self, t, name):
        """Same argument contract as the single-GPU path (pipeline.py ``denoise_window``): raw pointers cross the C ABI, so a
        CPU / strided / wrongly typed tensor must be rejected here instead of surfacing as a peer K/V-flag timeout."""
        if t is None:
            raise ValueError(f"{name} is required")
        t = t.to(device=self.pipe.device, dtype=torch.bfloat16)
        return t if t.is_contiguous() else t.contiguous()

    @staticmethod
    def _inplace(t, name, dtype):
        if not (torch.is_tensor(t) and t.is_cuda and t.dtype == dtype and t.is_contiguous()):
            raise ValueError(f"{name} must be a contiguous CUDA {str(dtype).replace('torch.', '')} tensor (updated in place)")

    def unet_forward(self, sample, timestep, skeletons, domains: List[str], F_local: int, F_total: int):
        """B-2 on this rank's frames: sample [len(domains)*F_local, Cin, h, w] (CFG-major like the reference batch)."""
        unet = self.pipe.unet
        sample = self._bf16(sample, "sample")
        if sample.dim() != 4 or sample.shape[1] != unet.config.in_channels:
            raise ValueError(f"sample must be [B, {unet.config.in_channels}, h, w]")
        B, _, H, W = sample.shape
        if len(domains) * F_local != B:
            raise ValueError(f"num_frames: {F_local} * len(domains): {len(domains)} != len(emb): {B}")
        if F_local * self.world != F_total:
            raise ValueError(f"F_total ({F_total}) must equal world ({self.world}) * local frames ({F_local})")
        for d in domains:
            if d not in _DOMAIN_IDS:
                raise ValueError(f"Invalid domain for temporal embedding: {d}")
        timestep = timestep.to(device=unet.device, dtype=torch.int64).reshape(-1).contiguous()
        if timestep.numel() != B:
            raise ValueError("timestep must have one entry per image")
        if unet.config.enable_pose_encoder:
            skeletons = self._bf16(skeletons, "skeletons")
            if tuple(skeletons.shape) != (B, 3, 8 * H, 8 * W):
                raise ValueError(f"skeletons must be [B, 3, 8H, 8W], got {tuple(skeletons.shape)}")
        else:
            skeletons = None
        dom = (C.c_int32 * len(domains))(*[_DOMAIN_IDS[d] for d in domains])
        out = torch.empty(B, unet.config.out_channels, H, W, device=unet.device, dtype=torch.bfloat16)
        with torch.cuda.device(unet.device):
            check(lib().d4d_unet_forward_sharded(unet._h, sample.data_ptr(), timestep.data_ptr(),
                                                 None if skeletons is None else skeletons.data_ptr(), dom, len(domains), B,
                                                 F_local, F_total, H, W, out.data_ptr(),
                                                 torch.cuda.current_stream().cuda_stream), "d4d_unet_forward_sharded")
        return out

    def denoise_window(self, *, latents, pixel_values_latents, plucker_embeds_latents, skeletons_latents, cond_masks_latents,
                       timestep_indices, domain: str, guidance_scale: float, F_total: int, num_inference_steps: int = 1,
                       solver_state: Optional[DPMSolverState] = None):
        """B-3 on this rank's frames (all tensors hold the LOCAL frames; updated in place like the single-GPU call).  With
        DPM-Solver++, ``solver_state`` is the local frames' ``DPMSolverState``, also updated in place."""
        pipe = self.pipe
        if domain not in _DOMAIN_IDS:
            raise ValueError(f"Invalid domain for temporal embedding: {domain}")
        self._inplace(latents, "latents", torch.bfloat16)
        self._inplace(timestep_indices, "timestep_indices", torch.int64)
        F_local, _, h, w = latents.shape
        if F_local * self.world != F_total:
            raise ValueError(f"F_total ({F_total}) must equal world ({self.world}) * local frames ({F_local})")
        pixel_values_latents = self._bf16(pixel_values_latents, "pixel_values_latents")
        plucker_embeds_latents = self._bf16(plucker_embeds_latents, "plucker_embeds_latents")
        skeletons_latents = self._bf16(skeletons_latents, "skeletons")
        cond_masks_latents = self._bf16(cond_masks_latents, "cond_masks_latents")
        sched = pipe.scheduler.c_struct(pipe.emulate_bf16_scheduler)
        stream = torch.cuda.current_stream(pipe.device).cuda_stream
        if isinstance(pipe.scheduler, DDIMTables):
            with torch.cuda.device(pipe.device):
                check(lib().d4d_denoise_window_sharded(
                    pipe.unet._h, latents.data_ptr(), pixel_values_latents.data_ptr(), plucker_embeds_latents.data_ptr(),
                    skeletons_latents.data_ptr(), cond_masks_latents.data_ptr(), timestep_indices.data_ptr(),
                    C.byref(sched), float(guidance_scale), _DOMAIN_IDS[domain], F_local, F_total, h, w,
                    int(num_inference_steps), stream), "d4d_denoise_window_sharded")
            return latents, timestep_indices
        # DPM-Solver++: the checks and the guidance of B200Diffuman4DPipeline.denoise_window
        pipe._guidance_scale = guidance_scale
        g = guidance_scale if pipe.do_classifier_free_guidance else 1.0
        st = solver_state
        if st is None:
            raise ValueError("the DPM-Solver++ scheduler needs the window frames' solver_state")
        if not (st.x0_prev is not None and st.x0_prev.is_cuda and st.x0_prev.dtype == torch.bfloat16
                and st.x0_prev.is_contiguous() and st.x0_prev.shape == latents.shape):
            raise ValueError("solver_state.x0_prev must be a contiguous CUDA bfloat16 tensor shaped like latents")
        lon = st.lower_order_nums
        if not (lon.is_cuda and lon.dtype == torch.int32 and lon.is_contiguous() and lon.numel() == F_local):
            raise ValueError("solver_state.lower_order_nums must be a contiguous CUDA int32 [F] tensor")
        with torch.cuda.device(pipe.device):
            check(lib().d4d_denoise_window_dpm_sharded(
                pipe.unet._h, latents.data_ptr(), pixel_values_latents.data_ptr(), plucker_embeds_latents.data_ptr(),
                skeletons_latents.data_ptr(), cond_masks_latents.data_ptr(), timestep_indices.data_ptr(), C.byref(sched),
                float(g), _DOMAIN_IDS[domain], F_local, F_total, h, w, int(num_inference_steps), st.x0_prev.data_ptr(),
                lon.data_ptr(), stream), "d4d_denoise_window_dpm_sharded")
        return latents, timestep_indices

    def window_exchange(self, latents, timestep_indices, solver_state: Optional[DPMSolverState], F_total: int):
        """Every rank's updated frames to every rank: the LOCAL ``latents`` [F_local,4,h,w], ``timestep_indices`` and
        (DPM-Solver++) ``solver_state`` in, the whole window's (F_total frames, window order) out as new tensors
        ``(latents, timestep_indices, solver_state or None)``.  SPMD: every rank calls it after the same window step."""
        self._inplace(latents, "latents", torch.bfloat16)
        self._inplace(timestep_indices, "timestep_indices", torch.int64)
        F_local, c, h, w = latents.shape
        dev = latents.device
        lat = torch.empty(F_total, c, h, w, dtype=torch.bfloat16, device=dev)
        ts = torch.empty(F_total, dtype=torch.int64, device=dev)
        out = None
        ptrs = [None] * 4
        if solver_state is not None:
            self._inplace(solver_state.x0_prev, "solver_state.x0_prev", torch.bfloat16)
            self._inplace(solver_state.lower_order_nums, "solver_state.lower_order_nums", torch.int32)
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
