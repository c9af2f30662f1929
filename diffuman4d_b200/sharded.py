"""Frame-sharded window denoise step across the GPUs of one box (SURVEY.md section 8e.2, DESIGN.md section 7).

One process per GPU (torch.distributed).  Rank r owns frames [r*F/R, (r+1)*F/R) of the window (both CFG halves of a
frame stay on the rank).  Everything except 3-D attention is per image and needs no communication; at each 3-D block
the fused-QKV GEMM epilogue stores K|V straight into every rank's gathered buffer over NVLink (peer memory mapped with
cudaIpc) -- there is no NCCL call on the data path.  torch.distributed is used once, to exchange the IPC handles.
"""
from __future__ import annotations

import ctypes as C
from typing import List

import torch
import torch.distributed as dist

from ._lib import check, lib
from .pipeline import B200Diffuman4DPipeline, _DOMAIN_IDS
from .scheduler import DDIMTables
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
        kv_bytes = exchange_bytes(pipe.unet.config, max_frames, h, w)
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
                       timestep_indices, domain: str, guidance_scale: float, F_total: int, num_inference_steps: int = 1):
        """B-3 on this rank's frames (all tensors hold the LOCAL frames; updated in place like the single-GPU call)."""
        pipe = self.pipe
        if not isinstance(pipe.scheduler, DDIMTables):
            raise NotImplementedError("the frame-sharded window runs the DDIM step only")
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
        with torch.cuda.device(pipe.device):
            check(lib().d4d_denoise_window_sharded(
                pipe.unet._h, latents.data_ptr(), pixel_values_latents.data_ptr(), plucker_embeds_latents.data_ptr(),
                skeletons_latents.data_ptr(), cond_masks_latents.data_ptr(), timestep_indices.data_ptr(), C.byref(sched),
                float(guidance_scale), _DOMAIN_IDS[domain], F_local, F_total, h, w, int(num_inference_steps),
                torch.cuda.current_stream().cuda_stream), "d4d_denoise_window_sharded")
        return latents, timestep_indices
