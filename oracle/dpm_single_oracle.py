"""CPU ORACLE (test infrastructure, NOT the product) for DPM-Solver++ singlestep sampling through ``Diffuman4DPipeline``.

Restates upstream diffusers==0.33.1 ``DPMSolverSinglestepScheduler`` (scheduling_dpmsolver_singlestep.py: __init__,
set_timesteps, get_order_list, convert_model_output, dpm_solver_first_order_update,
singlestep_dpm_solver_second_order_update, singlestep_dpm_solver_third_order_update, singlestep_dpm_solver_update, step)
for algorithm_type "dpmsolver++", solver_type "midpoint", solver_order 1, 2 or 3, no thresholding, sigmas from the beta
schedule, final_sigmas_type "zero" or "sigma_min".  The window step and the sliding loop with one scheduler object per
frame are ``oracle.dpm_solver_oracle.denoise_window_oracle_per_frame`` and ``sliding_iterative_denoise_oracle_per_frame``,
which take any stateful scheduler.

PARITY STATUS: the per-frame copy, window and reset semantics are pinned against the reference's own pipeline code run
with a scheduler adapter backed by ``DPMSingleOracle`` (tests/golden/gen_golden_dpm_single.py ->
tests/golden/pipeline_dpm_single_ref.pt, tests/test_scheduler_dpm_single.py).  The solver ARITHMETIC is **parity
unpinned** against diffusers (not installed): it restates the published 0.33.1 source, with independent mathematical
anchors in tests/test_scheduler_dpm_single.py (order 1 == DDIM and == DPM-Solver++ multistep order 1, an exact
point-mass denoiser stays on its trajectory at orders 2 and 3, convergence orders 1, 2 and 3 on Gaussian data).

Details taken from the published source and NOT checked against an installed diffusers:
  * Timesteps.  The class has no ``timestep_spacing`` knob: ``set_timesteps`` takes ``np.linspace(0, T - 1 -
    clipped_idx, n + 1).round()[::-1][:-1]`` (clipped_idx = 0 with ``lambda_min_clipped`` = -inf), and ``np.interp`` at
    the integer timesteps returns the fp32 table entries themselves.  The final sigma is 0 ("zero") or that of
    ``alphas_cumprod[0]`` ("sigma_min").  Duplicate timesteps are refused, so that a frame's step index is its timestep
    index.
  * Order list.  ``get_order_list(n)`` fixes one order per step index: blocks [1, .., solver_order]; with
    ``lower_order_final`` the list ends on a whole (shorter) block -- order 3: [1, 2, 3] * (n // 3 - 1) + [1, 2] + [1]
    when 3 divides n, else [1, 2, 3] * (n // 3) + [1] or + [1, 2]; order 2: [1, 2] * (n // 2 - 1) + [1, 1] when n is
    even, else [1, 2] * (n // 2) + [1] -- and without it [1, .., solver_order] * (n // solver_order).  With
    ``final_sigmas_type="zero"`` the last entry is set to 1.
  * ``lower_order_final`` switched on.  ``set_timesteps`` calls ``register_to_config(lower_order_final=True)`` when
    ``n % solver_order != 0``, or when ``final_sigmas_type`` is "zero", before it builds the order list.  The change
    stays in that scheduler object's config, so later ``set_timesteps`` calls on it see ``lower_order_final`` on whatever
    their step count; this oracle keeps its own copy of the config for the same reason.
  * Order reduction.  ``step`` takes the row's order from the list and lowers it while ``model_outputs[-order] is
    None``: a frame whose first step falls on a second- or third-order row (``__call__`` at a nonzero timestep index)
    runs at order 1, and the next rows of that block at 2 and 3.  The effective order is min(row order, steps taken + 1).
  * Block-start sample.  A step at effective order 1 saves ``self.sample = sample``; every step updates from
    ``self.sample``, so the second- and third-order steps restart from the sample of their block's first step, over
    h = lambda(i + 1) - lambda(i - order + 1), with ``model_outputs[-order]`` as D0 (the block start's data prediction).
    The midpoint third-order update uses D1_1 = (m0 - m2) / r0 only (D1_0, D1 and D2 are Heun's).
  * History.  ``model_outputs`` shifts on every step, whatever the order: ``model_outputs[i] <- model_outputs[i + 1]``.
  * Upcast.  Unlike ``DPMSolverMultistepScheduler.step`` (``sample.to(torch.float32)``), ``step`` does NOT upcast the
    sample: every product and difference of the update rounds to bf16 when the model output and sample are bf16.
  * ``prediction_type="sample"`` is accepted (``convert_model_output`` takes the output as x0), as are "epsilon" and
    "v_prediction".

bf16 emulation (the reference runs the step on CUDA bf16 tensors with 0-dim fp32 CPU coefficients): every
``coef * (bf16 tensor)`` and every op between bf16 tensors is computed in fp32 and rounded once to bf16.
``convert_model_output`` runs in bf16 like DPM-Solver++ multistep's; the history holds the data predictions in bf16.  The
first-order update rounds (sigma_t / sigma_s) * x, the (alpha_t (e^-h - 1)) * x0 product and their difference; the
second-order one rounds m0 - m1, (1 / r0) * (m0 - m1), the three products and each difference left to right; the
third-order one rounds m0 - m2, (1 / r0) * (m0 - m2), the three products, the difference and the sum left to right.
Divisions are emulated as correctly rounded fp32 divisions, as in ``DDIMOracle.step``.
"""
from __future__ import annotations

import copy

import numpy as np
import torch


class DPMSingleOracle:
    """upstream ``DPMSolverSinglestepScheduler`` (diffusers 0.33.1), stateful like upstream (``model_outputs``,
    ``sample``, ``step_index``, and the config ``set_timesteps`` may change), so the reference's per-frame ``deepcopy``
    gives per-frame histories.  ``cfg`` is a ``DPMSingleConfig``; the oracle works on a copy of it.

    **Parity with diffusers is unpinned** (diffusers is not installed): this restates the published source; the
    assumptions and the rounding of the bf16 path are stated in the module docstring.  ``table_dtype=torch.float64``
    evaluates the sigma table and the coefficients in fp64 (mathematical anchors only; upstream is fp32)."""

    def __init__(self, cfg, table_dtype=torch.float32):
        self.cfg = cfg = copy.copy(cfg)
        T = cfg.num_train_timesteps
        if cfg.beta_schedule == "scaled_linear":
            betas = torch.linspace(cfg.beta_start ** 0.5, cfg.beta_end ** 0.5, T, dtype=torch.float32) ** 2
        elif cfg.beta_schedule == "linear":
            betas = torch.linspace(cfg.beta_start, cfg.beta_end, T, dtype=torch.float32)
        else:
            raise ValueError(cfg.beta_schedule)
        if cfg.solver_order not in (1, 2, 3):
            raise ValueError(cfg.solver_order)
        if cfg.prediction_type not in ("epsilon", "v_prediction", "sample"):
            raise ValueError(cfg.prediction_type)
        if cfg.final_sigmas_type not in ("zero", "sigma_min"):
            raise ValueError(cfg.final_sigmas_type)
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.table_dtype = table_dtype
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = None
        self.sigmas = None
        self.order_list = None
        self._reset()

    def _reset(self):
        self.model_outputs = [None] * self.cfg.solver_order
        self.sample = None
        self.step_index = None

    def get_order_list(self, num_inference_steps: int) -> list:
        steps = num_inference_steps
        order = self.cfg.solver_order
        if self.cfg.lower_order_final:
            if order == 3:
                if steps % 3 == 0:
                    orders = [1, 2, 3] * (steps // 3 - 1) + [1, 2] + [1]
                elif steps % 3 == 1:
                    orders = [1, 2, 3] * (steps // 3) + [1]
                else:
                    orders = [1, 2, 3] * (steps // 3) + [1, 2]
            elif order == 2:
                if steps % 2 == 0:
                    orders = [1, 2] * (steps // 2 - 1) + [1, 1]
                else:
                    orders = [1, 2] * (steps // 2) + [1]
            else:
                orders = [1] * steps
        else:
            if order == 3:
                orders = [1, 2, 3] * (steps // 3)
            elif order == 2:
                orders = [1, 2] * (steps // 2)
            else:
                orders = [1] * steps
        if self.cfg.final_sigmas_type == "zero":
            orders[-1] = 1
        return orders

    def set_timesteps(self, n: int):
        cfg = self.cfg
        T = cfg.num_train_timesteps
        ts = np.linspace(0, T - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        if len(np.unique(ts)) != len(ts):
            raise ValueError(f"duplicate timesteps {ts.tolist()}")
        ac = self.alphas_cumprod.to(self.table_dtype)
        all_sigmas = ((1 - ac) / ac) ** 0.5
        last = all_sigmas[:1] if cfg.final_sigmas_type == "sigma_min" else torch.zeros(1, dtype=self.table_dtype)
        self.num_inference_steps = n
        self.timesteps = torch.from_numpy(ts)
        self.sigmas = torch.cat([all_sigmas[self.timesteps], last])
        self._reset()
        if not cfg.lower_order_final and n % cfg.solver_order != 0:
            cfg.lower_order_final = True          # register_to_config: persists on this object
        if not cfg.lower_order_final and cfg.final_sigmas_type == "zero":
            cfg.lower_order_final = True
        self.order_list = self.get_order_list(n)
        return self.timesteps

    @staticmethod
    def _alpha_sigma_t(sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha_t, sigma * alpha_t

    def _lambda(self, j: int):
        alpha, sigma = self._alpha_sigma_t(self.sigmas[j])
        return torch.log(alpha) - torch.log(sigma)

    def first_order_coefs(self, i: int):
        """``dpm_solver_first_order_update``'s scalars at step index i: sigma_t / sigma_s and alpha_t (e^-h - 1)."""
        alpha_t, sigma_t = self._alpha_sigma_t(self.sigmas[i + 1])
        alpha_s, sigma_s = self._alpha_sigma_t(self.sigmas[i])
        h = self._lambda(i + 1) - self._lambda(i)
        return sigma_t / sigma_s, alpha_t * (torch.exp(-h) - 1.0)

    def second_order_coefs(self, i: int):
        """``singlestep_dpm_solver_second_order_update``'s scalars at step index i: sigma_t / sigma_s1, alpha_t (e^-h - 1),
        0.5 alpha_t (e^-h - 1) and 1 / r0."""
        alpha_t, sigma_t = self._alpha_sigma_t(self.sigmas[i + 1])
        alpha_s1, sigma_s1 = self._alpha_sigma_t(self.sigmas[i - 1])
        lambda_t, lambda_s0, lambda_s1 = self._lambda(i + 1), self._lambda(i), self._lambda(i - 1)
        h, h_0 = lambda_t - lambda_s1, lambda_s0 - lambda_s1
        r0 = h_0 / h
        c = alpha_t * (torch.exp(-h) - 1.0)
        return sigma_t / sigma_s1, c, 0.5 * c, 1.0 / r0

    def third_order_coefs(self, i: int):
        """``singlestep_dpm_solver_third_order_update``'s (midpoint) scalars at step index i: sigma_t / sigma_s2,
        alpha_t (e^-h - 1), alpha_t ((e^-h - 1) / h + 1) and 1 / r0."""
        alpha_t, sigma_t = self._alpha_sigma_t(self.sigmas[i + 1])
        alpha_s2, sigma_s2 = self._alpha_sigma_t(self.sigmas[i - 2])
        lambda_t, lambda_s0, lambda_s2 = self._lambda(i + 1), self._lambda(i), self._lambda(i - 2)
        h, h_0 = lambda_t - lambda_s2, lambda_s0 - lambda_s2
        r0 = h_0 / h
        return (sigma_t / sigma_s2, alpha_t * (torch.exp(-h) - 1.0), alpha_t * ((torch.exp(-h) - 1.0) / h + 1.0),
                1.0 / r0)

    def step(self, model_output: torch.Tensor, timestep: int, sample: torch.Tensor) -> torch.Tensor:
        cfg = self.cfg
        if self.step_index is None:
            cand = (self.timesteps == int(timestep)).nonzero()
            self.step_index = int(cand[0]) if len(cand) else len(self.timesteps) - 1
        i = self.step_index
        bf = model_output.dtype == torch.bfloat16
        r = (lambda x: x.to(torch.bfloat16).float()) if bf else (lambda x: x)
        up = (lambda x: x.float()) if bf else (lambda x: x)
        m, x = up(model_output), up(sample)
        # convert_model_output (in the model output's dtype)
        alpha_s, sigma_s = self._alpha_sigma_t(self.sigmas[i])
        if cfg.prediction_type == "epsilon":
            x0 = r(r(x - r(sigma_s * m)) / alpha_s)
        elif cfg.prediction_type == "v_prediction":
            x0 = r(r(alpha_s * x) - r(sigma_s * m))
        else:
            x0 = m
        for k in range(cfg.solver_order - 1):
            self.model_outputs[k] = self.model_outputs[k + 1]
        self.model_outputs[-1] = x0.to(model_output.dtype)
        order = self.order_list[i]
        while self.model_outputs[-order] is None:
            order -= 1
        if order == 1:
            self.sample = sample
        s = up(self.sample)
        if order == 1:
            ratio, c = self.first_order_coefs(i)
            prev = r(r(ratio * s) - r(c * x0))
        elif order == 2:
            ratio, c, half_c, inv_r0 = self.second_order_coefs(i)
            m0, m1 = up(self.model_outputs[-1]), up(self.model_outputs[-2])
            d1 = r(inv_r0 * r(m0 - m1))
            prev = r(r(r(ratio * s) - r(c * m1)) - r(half_c * d1))
        else:
            ratio, c, c_d1, inv_r0 = self.third_order_coefs(i)
            m0, m2 = up(self.model_outputs[-1]), up(self.model_outputs[-3])
            d1_1 = r(inv_r0 * r(m0 - m2))
            prev = r(r(r(ratio * s) - r(c * m2)) + r(c_d1 * d1_1))
        self.step_index += 1
        return prev.to(model_output.dtype)
