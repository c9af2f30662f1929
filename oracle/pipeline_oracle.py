"""CPU ORACLE (test infrastructure, NOT the product) for the window denoise step and the
sliding-window loop of ``Diffuman4DPipeline``.

Restates  PIPE = src/diffusers/pipelines/diffuman4d/pipeline_diffuman4d.py:
  * ``get_negative_latents``            PIPE:103-113
  * ``get_timestep``                    PIPE:273-278
  * ``__call__`` denoise loop           PIPE:345-425  (input assembly, CFG, per-frame scheduler step)
  * ``sliding_iterative_denoise``       PIPE:463-551  (window schedule + invariants)
and upstream diffusers==0.33.1 ``DDIMScheduler`` (set_timesteps / step, eta=0), which the
reference deep-copies per frame (PIPE:265-271).

PARITY STATUS: the pipeline logic is pinned against the reference's OWN ``Diffuman4DPipeline.__call__`` and
``sliding_iterative_denoise`` executed on stubs of the upstream plumbing (tests/golden/gen_golden.py::gen_pipeline ->
tests/golden/pipeline_ref.pt; tests/test_oracle.py): input assembly, CFG negatives, cond-frame aliasing, per-frame
stepping (epsilon and v-prediction), visited windows, timestep bookkeeping and the three ValueError texts all match.
The scheduler ARITHMETIC is not: the scheduler class of the shipped checkpoint is not in the repo and diffusers is not
installed; DDIM (SD-2.x default) is restated from the published 0.33.1 source -- **parity unpinned** for that class, see
DESIGN.md.

The VAE is outside the hot path (SURVEY section 8f) and is not restated: all functions take latents.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np
import torch


class DDIMOracle:
    """upstream ``DDIMScheduler`` (scheduling_ddim.py, diffusers 0.33.1), eta = 0, no thresholding."""

    def __init__(self, cfg):
        self.cfg = cfg
        T = cfg.num_train_timesteps
        if cfg.beta_schedule == "scaled_linear":
            betas = torch.linspace(cfg.beta_start ** 0.5, cfg.beta_end ** 0.5, T, dtype=torch.float32) ** 2
        elif cfg.beta_schedule == "linear":
            betas = torch.linspace(cfg.beta_start, cfg.beta_end, T, dtype=torch.float32)
        else:
            raise ValueError(cfg.beta_schedule)
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if cfg.set_alpha_to_one else self.alphas_cumprod[0]
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = None

    def set_timesteps(self, n: int):
        cfg = self.cfg
        T = cfg.num_train_timesteps
        if n > T:
            raise ValueError("num_inference_steps > num_train_timesteps")
        self.num_inference_steps = n
        if cfg.timestep_spacing == "leading":
            ratio = T // n
            ts = (np.arange(0, n) * ratio).round()[::-1].copy().astype(np.int64)
            ts += cfg.steps_offset
        elif cfg.timestep_spacing == "trailing":
            ratio = T / n
            ts = np.round(np.arange(T, 0, -ratio)).astype(np.int64) - 1
        elif cfg.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n).round()[::-1].copy().astype(np.int64)
        else:
            raise ValueError(cfg.timestep_spacing)
        self.timesteps = torch.from_numpy(ts)
        return self.timesteps

    def step(self, model_output: torch.Tensor, timestep: int, sample: torch.Tensor) -> torch.Tensor:
        """One DDIM update.  Arithmetic is done op-by-op in ``sample``'s dtype with 0-dim fp32
        coefficients, exactly like upstream (so a bf16 caller gets upstream's bf16 rounding)."""
        cfg = self.cfg
        prev_t = timestep - cfg.num_train_timesteps // self.num_inference_steps
        a_t = self.alphas_cumprod[timestep]
        a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        b_t = 1 - a_t
        if sample.dtype == torch.bfloat16:
            # The reference runs this on CUDA bf16 tensors with 0-dim fp32 CPU coefficients: TensorIterator keeps such
            # "cpu scalar" operands in fp32 (opmath) and rounds every op's result to bf16.  Restated explicitly so the
            # emulation does not depend on which CPU kernel torch happens to pick for mixed bf16/fp32 operands.
            r = lambda x: x.to(torch.bfloat16).float()
            x, e = sample.float(), model_output.float()
            sa, sb = float(a_t ** 0.5), float(b_t ** 0.5)
            sap, sd = float(a_prev ** 0.5), float((1 - a_prev) ** 0.5)
            f32 = lambda v: torch.tensor(v, dtype=torch.float32)
            if cfg.prediction_type == "epsilon":
                x0 = r(r(x - r(f32(sb) * e)) / f32(sa))
                eps = e
            elif cfg.prediction_type == "v_prediction":
                x0 = r(r(f32(sa) * x) - r(f32(sb) * e))
                eps = r(r(f32(sa) * e) + r(f32(sb) * x))
            elif cfg.prediction_type == "sample":
                x0 = e
                eps = r(r(x - r(f32(sa) * x0)) / f32(sb))
            else:
                raise ValueError(cfg.prediction_type)
            if cfg.clip_sample:
                x0 = x0.clamp(-cfg.clip_sample_range, cfg.clip_sample_range)
            return r(r(f32(sap) * x0) + r(f32(sd) * eps)).to(torch.bfloat16)
        if cfg.prediction_type == "epsilon":
            x0 = (sample - b_t ** 0.5 * model_output) / a_t ** 0.5
            eps = model_output
        elif cfg.prediction_type == "v_prediction":
            x0 = (a_t ** 0.5) * sample - (b_t ** 0.5) * model_output
            eps = (a_t ** 0.5) * model_output + (b_t ** 0.5) * sample
        elif cfg.prediction_type == "sample":
            x0 = model_output
            eps = (sample - a_t ** 0.5 * x0) / b_t ** 0.5
        else:
            raise ValueError(cfg.prediction_type)
        if cfg.clip_sample:
            x0 = x0.clamp(-cfg.clip_sample_range, cfg.clip_sample_range)
        direction = (1 - a_prev) ** 0.5 * eps
        return a_prev ** 0.5 * x0 + direction


def get_negative_latents(latents: torch.Tensor, color: str) -> torch.Tensor:
    """PIPE:103-113."""
    ones = torch.ones_like(latents)
    if color == "black":
        return -1.0 * ones
    if color == "white":
        return ones
    if color in ("grey", "random"):
        return 0.0 * ones
    raise ValueError(f"color: {color} not supported.")


def assemble_unet_input(latents, pixel_latents, plucker, skeleton_latents, cond_mask, is_cond, cfg_on: bool,
                        concat_skeleton: bool):
    """PIPE:375-395.  Mutates ``latents`` in place at cond frames exactly like the reference
    (``latent_model_input`` aliases ``latents``, PIPE:375-379)."""
    lmi = latents
    lmi[is_cond] = pixel_latents[is_cond]
    if cfg_on:
        neg = lmi.clone()
        neg[is_cond] = get_negative_latents(pixel_latents, "white")[is_cond]
        lmi = torch.cat([neg, lmi])
        plucker = torch.cat([get_negative_latents(plucker, "grey"), plucker])
        if skeleton_latents is not None:
            skeleton_latents = torch.cat([get_negative_latents(skeleton_latents, "black"), skeleton_latents])
        cond_mask = torch.cat([cond_mask] * 2)
    parts = [lmi, plucker]
    if skeleton_latents is not None and concat_skeleton:
        parts.append(skeleton_latents)
    parts.append(cond_mask)
    return torch.cat(parts, dim=1), skeleton_latents


def denoise_window_oracle(unet: Callable, sched: DDIMOracle, *, latents, pixel_latents, plucker, skeletons,
                          cond_mask, timestep_indices, domain: str, guidance_scale: float,
                          num_inference_steps: int = 1, enable_pose_encoder: bool = True,
                          out_dtype: Optional[torch.dtype] = None):
    """``Diffuman4DPipeline.__call__`` PIPE:345-425 for one window (latents given).

    ``unet(sample, timestep, skeletons, domains, num_frames) -> noise_pred``.
    Returns (new latents, new timestep_indices).  ``latents`` is mutated at cond frames like the reference.
    """
    F_ = latents.shape[0]
    out_dtype = out_dtype or latents.dtype
    is_cond = cond_mask[:, 0, 0, 0] == 0
    cfg_on = guidance_scale > 1
    timestep_indices = timestep_indices.clone().long()
    domains = [domain] * (2 if cfg_on else 1)
    for _ in range(num_inference_steps):
        timestep_indices[is_cond] = 0                      # PIPE:275
        timestep = sched.timesteps[timestep_indices].clone()
        timestep[is_cond] = 0                              # PIPE:277
        x, skel = assemble_unet_input(latents, pixel_latents, plucker, skeletons, cond_mask, is_cond, cfg_on,
                                      concat_skeleton=not enable_pose_encoder)
        t_in = torch.cat([timestep] * 2) if cfg_on else timestep
        noise = unet(x, t_in, skel, domains, F_)
        if cfg_on:                                         # PIPE:408-410
            u, c = noise.chunk(2)
            if noise.dtype == torch.bfloat16:      # CUDA bf16 semantics: fp32 opmath, one rounding per op
                r = lambda x: x.to(torch.bfloat16).float()
                noise = r(u.float() + r(guidance_scale * r(c.float() - u.float()))).to(torch.bfloat16)
            else:
                noise = u + guidance_scale * (c - u)
        new = []
        for j in range(F_):                                # PIPE:413-422
            lat = latents[j:j + 1]
            if not bool(is_cond[j]):
                lat = sched.step(noise[j:j + 1], int(timestep[j]), lat)
            new.append(lat.to(out_dtype))
        latents = torch.cat(new)
        timestep_indices[~is_cond] += 1                    # PIPE:423
    return latents, timestep_indices


def build_windows(target_indices: torch.Tensor, input_indices: torch.Tensor, domain: str, window_size: int,
                  sliding_stride: int, sliding_shift: int = 0, bidirectional: bool = False):
    """PIPE:503-518."""
    tw, iw = [], []
    directions = (-1, 1) if bidirectional else (-1,)
    for direction in directions:
        for shift in range(sliding_shift, sliding_shift + len(target_indices), sliding_stride):
            t = target_indices.roll(shifts=shift * direction)[:window_size]
            tw.append(t)
            if domain == "spatial":
                iw.append(input_indices)
            elif domain == "temporal":
                iw.append(t - len(input_indices))
            else:
                raise ValueError(domain)
    return tw, iw


def sliding_iterative_denoise_oracle(unet: Callable, sched: DDIMOracle, *, pixel_latents, plucker, skeletons,
                                     cond_mask, latents, domain, timestep_indices, window_size=12,
                                     sliding_stride=1, sliding_shift=0, bidirectional=False,
                                     num_denoising_steps=1, alternation_rounds=3, guidance_scale=2.0,
                                     enable_pose_encoder=True):
    """PIPE:439-551 on latents (VAE encode/decode stripped)."""
    if (window_size * num_denoising_steps) % sliding_stride != 0:
        raise ValueError(
            f"The window size ({window_size}) * num denoising steps ({num_denoising_steps}) "
            f"should be divisible by the sliding stride ({sliding_stride})")
    per_alt = window_size * num_denoising_steps // sliding_stride
    if bidirectional:
        per_alt *= 2
    n_inf = per_alt * alternation_rounds
    timestep_indices = timestep_indices.clone().long()
    tgt = torch.where(cond_mask[:, 0, 0, 0] != 0.0)[0]
    inp = torch.where(cond_mask[:, 0, 0, 0] == 0.0)[0]
    t_end = int(timestep_indices[tgt][0]) + per_alt
    if (timestep_indices[tgt] != timestep_indices[tgt][0]).any():
        raise ValueError(f"The timestep indices should be the same for all target samples, "
                         f"timestep_indices = {timestep_indices}")
    if (timestep_indices[inp] != 0).any():
        raise ValueError(f"The timestep indices should be 0 for all input samples, "
                         f"timestep_indices = {timestep_indices}")
    latents = latents.clone() * sched.init_noise_sigma
    sched.set_timesteps(n_inf)
    tws, iws = build_windows(tgt, inp, domain, window_size, sliding_stride, sliding_shift, bidirectional)
    for tw, iw in zip(tws, iws):
        win = torch.cat([iw, tw])
        sl = lambda x: x[win] if x is not None else None
        lw, _ = denoise_window_oracle(
            unet, sched, latents=sl(latents), pixel_latents=sl(pixel_latents), plucker=sl(plucker),
            skeletons=sl(skeletons), cond_mask=sl(cond_mask), timestep_indices=timestep_indices[win],
            domain=domain, guidance_scale=guidance_scale, num_inference_steps=num_denoising_steps,
            enable_pose_encoder=enable_pose_encoder)
        timestep_indices[tw] += num_denoising_steps
        latents[win] = lw
    if (timestep_indices[tgt] != t_end).any():
        raise ValueError(f"The denoised timesteps of target samples mismatch the config, "
                         f"timestep_indices = {timestep_indices}")
    if (timestep_indices[inp] != 0).any():
        raise ValueError(f"Timesteps of input samples have changed, timestep_indices = {timestep_indices}")
    return {"latents": latents, "timestep_indices": timestep_indices,
            "fully_denoised": timestep_indices == n_inf}
