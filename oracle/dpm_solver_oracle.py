"""CPU ORACLE (test infrastructure, NOT the product) for DPM-Solver++ sampling through ``Diffuman4DPipeline``.

Restates upstream diffusers==0.33.1 ``DPMSolverMultistepScheduler`` (scheduling_dpmsolver_multistep.py: set_timesteps,
convert_model_output, dpm_solver_first_order_update, multistep_dpm_solver_second_order_update, step) for
algorithm_type "dpmsolver++" / solver_type "midpoint", and the window step and sliding loop of the reference pipeline
with ONE SCHEDULER OBJECT PER FRAME, as the reference runs them: ``parepare_schedulers`` deep-copies the scheduler per
frame after ``set_timesteps`` (PIPE:265-271), every ``sliding_iterative_denoise`` call makes a fresh set (PIPE:501), the
copies of a window's frames are handed to ``__call__`` (PIPE:535) and frame j is stepped by its own copy (PIPE:420).
The single-scheduler functions of ``pipeline_oracle`` are reused for everything that does not depend on that.

PARITY STATUS: the per-frame copy, window and reset semantics are pinned against the reference's own pipeline code run
with a scheduler adapter backed by ``DPMSolverOracle`` (tests/golden/gen_golden_dpm.py -> tests/golden/pipeline_dpm_ref.pt,
tests/test_scheduler_dpm.py).  The solver ARITHMETIC is **parity unpinned** against diffusers (not installed): it restates
the published 0.33.1 source, with independent mathematical anchors in tests/test_scheduler_dpm.py (order 1 == DDIM, an
exact point-mass denoiser stays on its trajectory, convergence orders 1 and 2 on Gaussian data).

bf16 emulation (the rule ``pipeline_oracle.DDIMOracle.step`` states for DDIM, applied to this scheduler's source): the
reference runs the step on CUDA bf16 tensors with 0-dim fp32 CPU coefficients, so every ``coef * (bf16 tensor)`` and
every op between bf16 tensors is computed in fp32 and rounded once to bf16; ``convert_model_output`` runs in bf16, so the
data prediction x0 and the stored history are bf16; D1 = (1/r0) * (m0 - m1) rounds twice; ``sample`` is upcast to fp32
before the update, so ``(sigma_t / sigma_s) * sample`` and the two subtractions stay fp32 and the final cast rounds once.
Divisions are emulated as correctly rounded fp32 divisions, as in ``DDIMOracle.step``.
"""
from __future__ import annotations

import copy
from typing import Callable, List

import numpy as np
import torch

from .pipeline_oracle import assemble_unet_input, build_windows


class DPMSolverOracle:
    """upstream ``DPMSolverMultistepScheduler`` (scheduling_dpmsolver_multistep.py, diffusers 0.33.1) with
    algorithm_type "dpmsolver++", solver_type "midpoint", solver_order 1 or 2, no thresholding, sigmas from the beta
    schedule, lambda_min_clipped -inf, variance_type None.  Stateful like upstream (model_outputs, lower_order_nums,
    step_index), so the reference's per-frame ``deepcopy`` gives per-frame histories.

    **Parity with diffusers is unpinned** (diffusers is not installed): this restates the published source.  The
    bf16 path rounds like the reference's eager bf16 maths (see ``DDIMOracle.step``): x0 and the history in bf16, each
    ``coef * bf16 tensor`` rounded, ``(sigma_t / sigma_s) * sample`` and the subtractions in fp32, one final cast.
    ``table_dtype=torch.float64`` evaluates the sigma table and the coefficients in fp64 (mathematical anchors only;
    upstream is fp32), and non-bf16 samples then stay in their own dtype instead of being upcast to fp32."""

    def __init__(self, cfg, table_dtype=torch.float32):
        self.cfg = cfg
        T = cfg.num_train_timesteps
        if cfg.beta_schedule == "scaled_linear":
            betas = torch.linspace(cfg.beta_start ** 0.5, cfg.beta_end ** 0.5, T, dtype=torch.float32) ** 2
        elif cfg.beta_schedule == "linear":
            betas = torch.linspace(cfg.beta_start, cfg.beta_end, T, dtype=torch.float32)
        else:
            raise ValueError(cfg.beta_schedule)
        if cfg.solver_order not in (1, 2):
            raise ValueError(cfg.solver_order)
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.table_dtype = table_dtype
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = None
        self.sigmas = None
        self._reset()

    def _reset(self):
        self.model_outputs = [None] * self.cfg.solver_order
        self.lower_order_nums = 0
        self.step_index = None

    def set_timesteps(self, n: int):
        cfg = self.cfg
        T = cfg.num_train_timesteps
        if cfg.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif cfg.timestep_spacing == "leading":
            step_ratio = T // (n + 1)
            ts = (np.arange(0, n + 1) * step_ratio).round()[::-1][:-1].copy().astype(np.int64)
            ts += cfg.steps_offset
        elif cfg.timestep_spacing == "trailing":
            step_ratio = T / n
            ts = np.arange(T, 0, -step_ratio).round().copy().astype(np.int64)
            ts -= 1
        else:
            raise ValueError(cfg.timestep_spacing)
        if len(np.unique(ts)) != len(ts):
            raise ValueError(f"duplicate timesteps {ts.tolist()}")
        ac = self.alphas_cumprod.to(self.table_dtype)
        all_sigmas = ((1 - ac) / ac) ** 0.5
        last = torch.zeros(1, dtype=self.table_dtype) if cfg.final_sigmas_type == "zero" else all_sigmas[:1]
        self.num_inference_steps = n
        self.timesteps = torch.from_numpy(ts)
        self.sigmas = torch.cat([all_sigmas[self.timesteps], last])
        self._reset()
        return self.timesteps

    @staticmethod
    def _alpha_sigma_t(sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha_t, sigma * alpha_t

    def _lambda(self, i):
        alpha, sigma = self._alpha_sigma_t(self.sigmas[i])
        return torch.log(alpha) - torch.log(sigma)

    def step(self, model_output: torch.Tensor, timestep: int, sample: torch.Tensor) -> torch.Tensor:
        cfg = self.cfg
        if self.step_index is None:
            cand = (self.timesteps == int(timestep)).nonzero()
            self.step_index = int(cand[0]) if len(cand) else len(self.timesteps) - 1
        i, n = self.step_index, len(self.timesteps)
        final_first = i == n - 1 and (cfg.euler_at_final or (cfg.lower_order_final and n < 15)
                                      or cfg.final_sigmas_type == "zero")
        first = cfg.solver_order == 1 or self.lower_order_nums < 1 or final_first
        alpha_s, sigma_s = self._alpha_sigma_t(self.sigmas[i])
        alpha_t, sigma_t = self._alpha_sigma_t(self.sigmas[i + 1])
        h = self._lambda(i + 1) - self._lambda(i)
        ratio = sigma_t / sigma_s
        c = alpha_t * (torch.exp(-h) - 1.0)
        bf = model_output.dtype == torch.bfloat16
        r = (lambda x: x.to(torch.bfloat16).float()) if bf else (lambda x: x)
        m, x = (model_output.float(), sample.float()) if bf else (model_output, sample)
        # convert_model_output (in the model output's dtype)
        if cfg.prediction_type == "epsilon":
            x0 = r(r(x - r(sigma_s * m)) / alpha_s)
        elif cfg.prediction_type == "v_prediction":
            x0 = r(r(alpha_s * x) - r(sigma_s * m))
        elif cfg.prediction_type == "sample":
            x0 = m
        else:
            raise ValueError(cfg.prediction_type)
        x0 = x0.to(model_output.dtype)
        for k in range(cfg.solver_order - 1):
            self.model_outputs[k] = self.model_outputs[k + 1]
        self.model_outputs[-1] = x0
        # sample.to(torch.float32); fp64 anchors keep fp64
        xs = sample.float() if sample.dtype in (torch.bfloat16, torch.float16, torch.float32) else sample
        m0 = x0.float() if bf else x0
        if first:
            prev = ratio * xs - r(c * m0)
        else:
            m1 = self.model_outputs[-2].float() if bf else self.model_outputs[-2]
            r0 = (self._lambda(i) - self._lambda(i - 1)) / h
            d1 = r((1.0 / r0) * r(m0 - m1))
            prev = ratio * xs - r(c * m0) - r((0.5 * c) * d1)
        if self.lower_order_nums < cfg.solver_order:
            self.lower_order_nums += 1
        self.step_index += 1
        return prev.to(model_output.dtype)



def denoise_window_oracle_per_frame(unet: Callable, scheds: List, *, latents, pixel_latents, plucker, skeletons,
                                    cond_mask, timestep_indices, domain: str, guidance_scale: float,
                                    num_inference_steps: int = 1, enable_pose_encoder: bool = True):
    """``Diffuman4DPipeline.__call__`` PIPE:345-425 for one window with latents given and ``schedulers`` = ``scheds``
    (one scheduler object per frame of the window, each stepped only for its own frame, PIPE:420).
    Returns (new latents, new timestep_indices); ``latents`` is mutated at cond frames like the reference."""
    F_ = latents.shape[0]
    if len(scheds) != F_:
        raise ValueError("one scheduler per frame")
    out_dtype = latents.dtype
    is_cond = cond_mask[:, 0, 0, 0] == 0
    cfg_on = guidance_scale > 1
    timestep_indices = timestep_indices.clone().long()
    domains = [domain] * (2 if cfg_on else 1)
    for _ in range(num_inference_steps):
        timestep_indices[is_cond] = 0                      # PIPE:275
        timestep = scheds[0].timesteps[timestep_indices].clone()
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
                lat = scheds[j].step(noise[j:j + 1], int(timestep[j]), lat)
            new.append(lat.to(out_dtype))
        latents = torch.cat(new)
        timestep_indices[~is_cond] += 1                    # PIPE:423
    return latents, timestep_indices


def sliding_iterative_denoise_oracle_per_frame(unet: Callable, sched, *, pixel_latents, plucker, skeletons, cond_mask,
                                               latents, domain, timestep_indices, window_size=12, sliding_stride=1,
                                               sliding_shift=0, bidirectional=False, num_denoising_steps=1,
                                               alternation_rounds=3, guidance_scale=2.0, enable_pose_encoder=True):
    """PIPE:439-551 on latents (VAE encode/decode stripped), with ``sched`` deep-copied per frame after
    ``set_timesteps`` (PIPE:265-271, 501): a stateful scheduler starts every call fresh and keeps one history per frame."""
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
    scheds = [copy.deepcopy(sched) for _ in range(len(latents))]
    tws, iws = build_windows(tgt, inp, domain, window_size, sliding_stride, sliding_shift, bidirectional)
    for tw, iw in zip(tws, iws):
        win = torch.cat([iw, tw])
        sl = lambda x: x[win] if x is not None else None
        lw, _ = denoise_window_oracle_per_frame(
            unet, [scheds[i] for i in win], latents=sl(latents), pixel_latents=sl(pixel_latents), plucker=sl(plucker),
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
