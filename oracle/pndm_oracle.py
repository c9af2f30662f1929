"""CPU ORACLE (test infrastructure, NOT the product) for PNDM (PLMS) sampling through ``Diffuman4DPipeline``.

Restates upstream diffusers==0.33.1 ``PNDMScheduler`` (scheduling_pndm.py: __init__, set_timesteps, step_plms,
_get_prev_sample) with ``skip_prk_steps=True``, epsilon or v prediction.  The window step and the sliding loop with one
scheduler object per frame are ``oracle.dpm_solver_oracle.denoise_window_oracle_per_frame`` and
``sliding_iterative_denoise_oracle_per_frame``, which take any stateful scheduler.

PARITY STATUS: the per-frame copy, window and reset semantics are pinned against the reference's own pipeline code run
with a scheduler adapter backed by ``PNDMOracle`` (tests/golden/gen_golden_pndm.py -> tests/golden/pipeline_pndm_ref.pt,
tests/test_scheduler_pndm.py).  The solver ARITHMETIC is **parity unpinned** against diffusers (not installed): it restates
the published 0.33.1 source, with independent mathematical anchors in tests/test_scheduler_pndm.py (counter 0 == DDIM,
counter 1 == the averaged-epsilon re-step, an exact point-mass denoiser stays on its trajectory).

Upstream facts the restatement keeps:
  * ``set_timesteps(n)`` spaces n timesteps, then repeats the second-largest, giving n + 1 entries (1 for n = 1); a
    frame of the reference's loop takes n steps and so never reaches the last entry.
  * ``prev_t = t - T // n`` from the timestep VALUE, whatever the spacing.  At counter 1 nothing is appended to ``ets``
    and the step goes from ``t + T // n`` to ``t``, from the sample saved at counter 0, with the mean of the two outputs.
  * ``ets`` keeps the last 4 outputs; at counter 2 it holds the outputs of counters 0 and 2.

bf16 emulation (the reference runs the step on CUDA bf16 tensors with 0-dim fp32 CPU coefficients and Python-number
constants): nothing is upcast, so every ``coef * (bf16 tensor)``, every op between bf16 tensors and every op with a Python
number is computed in fp32 and rounded once to bf16 -- the Adams-Bashforth sums one operation at a time as upstream
writes them, including the ``(1 / 24) *`` of the four-output sum.  Divisions are emulated as correctly rounded fp32
divisions, as in ``DDIMOracle.step``.
"""
from __future__ import annotations

import numpy as np
import torch


class PNDMOracle:
    """upstream ``PNDMScheduler`` (diffusers 0.33.1) with ``skip_prk_steps``, stateful like upstream (``ets``,
    ``counter``, ``cur_sample``), so the reference's per-frame ``deepcopy`` gives per-frame histories.  ``cfg`` is a
    ``PNDMConfig``.  ``table_dtype=torch.float64`` evaluates alphas_cumprod and the step scalars in fp64 (mathematical
    anchors only; upstream is fp32)."""

    def __init__(self, cfg, table_dtype=torch.float32):
        self.cfg = cfg
        T = cfg.num_train_timesteps
        if cfg.beta_schedule == "scaled_linear":
            betas = torch.linspace(cfg.beta_start ** 0.5, cfg.beta_end ** 0.5, T, dtype=torch.float32) ** 2
        elif cfg.beta_schedule == "linear":
            betas = torch.linspace(cfg.beta_start, cfg.beta_end, T, dtype=torch.float32)
        else:
            raise ValueError(cfg.beta_schedule)
        if cfg.prediction_type not in ("epsilon", "v_prediction"):
            raise ValueError(cfg.prediction_type)   # upstream raises for "sample" in _get_prev_sample
        betas = betas.to(table_dtype)
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = (torch.tensor(1.0, dtype=table_dtype) if cfg.set_alpha_to_one
                                    else self.alphas_cumprod[0])
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = None
        self._reset()

    def _reset(self):
        self.ets = []
        self.counter = 0
        self.cur_sample = None

    def set_timesteps(self, n: int):
        cfg = self.cfg
        T = cfg.num_train_timesteps
        if cfg.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n).round().astype(np.int64)
        elif cfg.timestep_spacing == "leading":
            step_ratio = T // n
            ts = (np.arange(0, n) * step_ratio).round()
            ts += cfg.steps_offset
        elif cfg.timestep_spacing == "trailing":
            step_ratio = T / n
            ts = np.round(np.arange(T, 0, -step_ratio))[::-1].astype(np.int64)
            ts -= 1
        else:
            raise ValueError(cfg.timestep_spacing)
        plms = np.concatenate([ts[:-1], ts[-2:-1], ts[-1:]])[::-1].copy()
        self.num_inference_steps = n
        self.timesteps = torch.from_numpy(plms.astype(np.int64))
        self._reset()
        return self.timesteps

    def prev_sample_coefs(self, t: int, prev: int) -> list:
        """The scalars ``_get_prev_sample`` evaluates from ``t`` to ``prev`` (0-dim tensors, upstream's order):
        a_t^0.5, (1 - a_t)^0.5, sample_coeff, a_prev - a_t and model_output_denom_coeff."""
        alpha_prod_t = self.alphas_cumprod[t]
        alpha_prod_t_prev = self.alphas_cumprod[prev] if prev >= 0 else self.final_alpha_cumprod
        beta_prod_t = 1 - alpha_prod_t
        beta_prod_t_prev = 1 - alpha_prod_t_prev
        sample_coeff = (alpha_prod_t_prev / alpha_prod_t) ** (0.5)
        model_output_denom_coeff = alpha_prod_t * beta_prod_t_prev ** (0.5) + (
            alpha_prod_t * beta_prod_t * alpha_prod_t_prev) ** (0.5)
        return [alpha_prod_t ** 0.5, beta_prod_t ** 0.5, sample_coeff, alpha_prod_t_prev - alpha_prod_t,
                model_output_denom_coeff]

    def step(self, model_output: torch.Tensor, timestep: int, sample: torch.Tensor) -> torch.Tensor:
        """``step_plms``; ``timestep`` is the table value the reference passes."""
        ratio = self.cfg.num_train_timesteps // self.num_inference_steps
        t = int(timestep)
        prev_t = t - ratio
        if self.counter != 1:
            self.ets = self.ets[-3:]
            self.ets.append(model_output)
        else:
            prev_t, t = t, t + ratio
        bf = model_output.dtype == torch.bfloat16
        r = (lambda x: x.to(torch.bfloat16).float()) if bf else (lambda x: x)
        up = (lambda x: x.float()) if bf else (lambda x: x)
        e = [up(v) for v in self.ets]
        x = up(sample)
        if len(self.ets) == 1 and self.counter == 0:
            eps = up(model_output)
            self.cur_sample = sample
        elif len(self.ets) == 1 and self.counter == 1:
            eps = r(r(up(model_output) + e[-1]) / 2)
            x = up(self.cur_sample)
            self.cur_sample = None
        elif len(self.ets) == 2:
            eps = r(r(r(3 * e[-1]) - e[-2]) / 2)
        elif len(self.ets) == 3:
            eps = r(r(r(r(23 * e[-1]) - r(16 * e[-2])) + r(5 * e[-3])) / 12)
        else:
            eps = r((1 / 24) * r(r(r(r(55 * e[-1]) - r(59 * e[-2])) + r(37 * e[-3])) - r(9 * e[-4])))
        # _get_prev_sample
        sqrt_a, sqrt_b, sample_coef, alpha_diff, denom = self.prev_sample_coefs(t, prev_t)
        if self.cfg.prediction_type == "v_prediction":
            eps = r(r(sqrt_a * eps) + r(sqrt_b * x))
        prev = r(r(sample_coef * x) - r(r(alpha_diff * eps) / denom))
        self.counter += 1
        return prev.to(sample.dtype)
