"""CPU ORACLE (test infrastructure, NOT the product) for DEIS sampling through ``Diffuman4DPipeline``.

Restates upstream diffusers==0.33.1 ``DEISMultistepScheduler`` (scheduling_deis_multistep.py: __init__, set_timesteps,
convert_model_output, deis_first_order_update, multistep_deis_second_order_update, multistep_deis_third_order_update,
step) for algorithm_type "deis", solver_type "logrho", solver_order 1, 2 or 3, no thresholding, sigmas from the beta
schedule.  The window step and the sliding loop with one scheduler object per frame are
``oracle.dpm_solver_oracle.denoise_window_oracle_per_frame`` and ``sliding_iterative_denoise_oracle_per_frame``, which take
any stateful scheduler.

PARITY STATUS: the per-frame copy, window and reset semantics are pinned against the reference's own pipeline code run
with a scheduler adapter backed by ``DEISOracle`` (tests/golden/gen_golden_deis.py -> tests/golden/pipeline_deis_ref.pt,
tests/test_scheduler_deis.py).  The solver ARITHMETIC is **parity unpinned** against diffusers (not installed): it restates
the published 0.33.1 source, with independent mathematical anchors in tests/test_scheduler_deis.py (order 1 == DDIM, an
exact point-mass denoiser stays on its trajectory at orders 2 and 3, convergence orders 1, 2 and 3 on Gaussian data).

Assumptions taken from the published source and NOT checked against an installed diffusers:
  * The final sigma.  ``set_timesteps`` appends ``((1 - alphas_cumprod[0]) / alphas_cumprod[0]) ** 0.5`` (sigma_min);
    DEIS has no ``final_sigmas_type`` knob, so the last step never reaches sigma 0 and every log rho is finite.
    Timesteps are spaced like DPM-Solver++'s (linspace / leading over n + 1 points without the last, trailing) and
    ``np.interp`` at the integer timesteps returns the fp32 table entries themselves; duplicate timesteps are refused, so
    that a frame's step index is its timestep index.
  * ``step`` does NOT upcast the sample (unlike DPM-Solver++'s ``sample.to(torch.float32)``): every product, sum and
    quotient of the update rounds to bf16 when the model output and sample are bf16.
  * The ``ind_fn`` coefficients: rho = sigma_t / alpha_t are 0-dim fp32 tensors, ``np.log`` of each is numpy's float32
    log, and every other operation of ``ind_fn`` and of the coefficient differences is an fp32 operation, in upstream's
    order (fp64 throughout with ``table_dtype=torch.float64``).
  * ``prediction_type="sample"`` is accepted (``convert_model_output`` takes the output as x0), as are "epsilon" and
    "v_prediction".

bf16 emulation (the reference runs the step on CUDA bf16 tensors with 0-dim fp32 CPU coefficients): every
``coef * (bf16 tensor)`` and every op between bf16 tensors is computed in fp32 and rounded once to bf16.
``convert_model_output`` runs in bf16: the data prediction x0 rounds like DPM-Solver++'s, and its epsilon form
(x - alpha_t * x0) / sigma_t rounds after each op; the history holds that epsilon form in bf16.  The first-order update
rounds (alpha_t / alpha_s) * x, the (sigma_t (e^h - 1)) * m0 product and their difference; the higher-order updates round
x / alpha_s0, each c_k * m_k, each partial sum left to right and the final alpha_t * (...).  Divisions are emulated as
correctly rounded fp32 divisions, as in ``DDIMOracle.step``.
"""
from __future__ import annotations

import numpy as np
import torch


def _log(v: torch.Tensor) -> torch.Tensor:
    """upstream ``np.log`` of a 0-dim tensor: numpy's log in the tensor's dtype"""
    return torch.from_numpy(np.asarray(np.log(v.numpy())))


class DEISOracle:
    """upstream ``DEISMultistepScheduler`` (diffusers 0.33.1), stateful like upstream (``model_outputs``,
    ``lower_order_nums``, ``step_index``), so the reference's per-frame ``deepcopy`` gives per-frame histories.  ``cfg`` is
    a ``DEISConfig``.

    **Parity with diffusers is unpinned** (diffusers is not installed): this restates the published source; the
    assumptions and the rounding of the bf16 path are stated in the module docstring.  ``table_dtype=torch.float64``
    evaluates the sigma table and the coefficients in fp64 (mathematical anchors only; upstream is fp32)."""

    def __init__(self, cfg, table_dtype=torch.float32):
        self.cfg = cfg
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
        self.num_inference_steps = n
        self.timesteps = torch.from_numpy(ts)
        self.sigmas = torch.cat([all_sigmas[self.timesteps], all_sigmas[:1]])   # sigma_last: alphas_cumprod[0]'s
        self._reset()
        return self.timesteps

    @staticmethod
    def _alpha_sigma_t(sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha_t, sigma * alpha_t

    def first_order_coefs(self, i: int):
        """``deis_first_order_update``'s scalars from sigma index i to i + 1: alpha_t / alpha_s and
        sigma_t * (exp(h) - 1)."""
        alpha_t, sigma_t = self._alpha_sigma_t(self.sigmas[i + 1])
        alpha_s, sigma_s = self._alpha_sigma_t(self.sigmas[i])
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s = torch.log(alpha_s) - torch.log(sigma_s)
        h = lambda_t - lambda_s
        return alpha_t / alpha_s, sigma_t * (torch.exp(h) - 1.0)

    def _rho(self, j: int):
        alpha, sigma = self._alpha_sigma_t(self.sigmas[j])
        return sigma / alpha

    def second_order_coefs(self, i: int):
        """``multistep_deis_second_order_update``'s coef1, coef2 at step index i."""
        rho_t, rho_s0, rho_s1 = self._rho(i + 1), self._rho(i), self._rho(i - 1)

        def ind_fn(t, b, c):
            # Integrate[(log(t) - log(c)) / (log(b) - log(c)), {t}]
            return t * (-_log(c) + _log(t) - 1) / (_log(b) - _log(c))

        coef1 = ind_fn(rho_t, rho_s0, rho_s1) - ind_fn(rho_s0, rho_s0, rho_s1)
        coef2 = ind_fn(rho_t, rho_s1, rho_s0) - ind_fn(rho_s0, rho_s1, rho_s0)
        return coef1, coef2

    def third_order_coefs(self, i: int):
        """``multistep_deis_third_order_update``'s coef1, coef2, coef3 at step index i."""
        rho_t, rho_s0, rho_s1, rho_s2 = self._rho(i + 1), self._rho(i), self._rho(i - 1), self._rho(i - 2)

        def ind_fn(t, b, c, d):
            # Integrate[(log(t) - log(c))(log(t) - log(d)) / (log(b) - log(c))(log(b) - log(d)), {t}]
            numerator = t * (
                _log(c) * (_log(d) - _log(t) + 1)
                - _log(d) * _log(t)
                + _log(d)
                + _log(t) ** 2
                - 2 * _log(t)
                + 2
            )
            denominator = (_log(b) - _log(c)) * (_log(b) - _log(d))
            return numerator / denominator

        coef1 = ind_fn(rho_t, rho_s0, rho_s1, rho_s2) - ind_fn(rho_s0, rho_s0, rho_s1, rho_s2)
        coef2 = ind_fn(rho_t, rho_s1, rho_s2, rho_s0) - ind_fn(rho_s0, rho_s1, rho_s2, rho_s0)
        coef3 = ind_fn(rho_t, rho_s2, rho_s0, rho_s1) - ind_fn(rho_s0, rho_s2, rho_s0, rho_s1)
        return coef1, coef2, coef3

    def step(self, model_output: torch.Tensor, timestep: int, sample: torch.Tensor) -> torch.Tensor:
        cfg = self.cfg
        if self.step_index is None:
            cand = (self.timesteps == int(timestep)).nonzero()
            self.step_index = int(cand[0]) if len(cand) else len(self.timesteps) - 1
        i, n = self.step_index, len(self.timesteps)
        lower_order_final = i == n - 1 and cfg.lower_order_final and n < 15
        lower_order_second = i == n - 2 and cfg.lower_order_final and n < 15
        bf = model_output.dtype == torch.bfloat16
        r = (lambda x: x.to(torch.bfloat16).float()) if bf else (lambda x: x)
        up = (lambda x: x.float()) if bf else (lambda x: x)
        m, x = up(model_output), up(sample)
        # convert_model_output (in the model output's dtype): x0, then back to its epsilon form
        alpha_s, sigma_s = self._alpha_sigma_t(self.sigmas[i])
        if cfg.prediction_type == "epsilon":
            x0 = r(r(x - r(sigma_s * m)) / alpha_s)
        elif cfg.prediction_type == "v_prediction":
            x0 = r(r(alpha_s * x) - r(sigma_s * m))
        else:
            x0 = m
        e = r(r(x - r(alpha_s * x0)) / sigma_s)
        for k in range(cfg.solver_order - 1):
            self.model_outputs[k] = self.model_outputs[k + 1]
        self.model_outputs[-1] = e.to(model_output.dtype)
        if cfg.solver_order == 1 or self.lower_order_nums < 1 or lower_order_final:
            ratio, c = self.first_order_coefs(i)
            prev = r(r(ratio * x) - r(c * e))
        else:
            alpha_t = self._alpha_sigma_t(self.sigmas[i + 1])[0]
            if cfg.solver_order == 2 or self.lower_order_nums < 2 or lower_order_second:
                coefs = self.second_order_coefs(i)
            else:
                coefs = self.third_order_coefs(i)
            acc = r(x / alpha_s)
            for k, coef in enumerate(coefs):
                acc = r(acc + r(coef * up(self.model_outputs[-1 - k])))
            prev = r(alpha_t * acc)
        if self.lower_order_nums < cfg.solver_order:
            self.lower_order_nums += 1
        self.step_index += 1
        return prev.to(model_output.dtype)
