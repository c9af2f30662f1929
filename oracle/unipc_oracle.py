"""CPU ORACLE (test infrastructure, NOT the product) for UniPC sampling through ``Diffuman4DPipeline``.

Restates upstream diffusers==0.33.1 ``UniPCMultistepScheduler`` (scheduling_unipc_multistep.py: set_timesteps,
convert_model_output, multistep_uni_p_bh_update, multistep_uni_c_bh_update, step) for predict_x0=True, solver_type "bh1"
or "bh2", solver_order 1 or 2, no solver_p and no thresholding.  The window step and the sliding loop with one scheduler
object per frame are ``oracle.dpm_solver_oracle.denoise_window_oracle_per_frame`` and
``sliding_iterative_denoise_oracle_per_frame``, which take any stateful scheduler.

PARITY STATUS: the per-frame copy, window and reset semantics are pinned against the reference's own pipeline code run
with a scheduler adapter backed by ``UniPCOracle`` (tests/golden/gen_golden_unipc.py -> tests/golden/pipeline_unipc_ref.pt,
tests/test_scheduler_unipc.py).  The solver ARITHMETIC is **parity unpinned** against diffusers (not installed): it restates
the published 0.33.1 source, with independent mathematical anchors in tests/test_scheduler_unipc.py (order 1 without the
corrector == DDIM, an exact point-mass denoiser stays on its trajectory, convergence orders on Gaussian data).

Timesteps and sigmas: upstream interpolates the fp32 sigma table at the integer timesteps (``np.interp``), which returns
the table entries themselves, so ``DPMSolverOracle.set_timesteps`` gives the same sigmas; duplicate timesteps are refused.

bf16 emulation (the reference runs the step on CUDA bf16 tensors with 0-dim fp32 CPU coefficients): every
``coef * (bf16 tensor)`` and every op between bf16 tensors is computed in fp32 and rounded once to bf16.  Unlike
DPM-Solver++, UniPC does NOT upcast ``sample``, so ``(sigma_t / sigma_s0) * x`` and both subtractions round to bf16 too.
``convert_model_output`` runs in bf16 (x0 and the history are bf16); the corrected sample is bf16 (``.to(x.dtype)``).
D1 = (m_i - m0) / rk rounds twice (difference, then division; divisions are emulated as correctly rounded fp32
divisions, as in ``DDIMOracle.step``).  The predictor's order-2 rho is the bf16 tensor [0.5]; the corrector's is [0.5] at
order 1 and ``torch.linalg.solve(R, b)`` in fp32 cast to the sample's dtype (bf16) at order 2; each rho times a bf16
tensor rounds.  The order-1 corrector adds its term to the integer 0, and the order-1 predictor subtracts
``alpha_t * B_h * 0`` (a signed zero), as upstream does.
"""
from __future__ import annotations

import types

import torch

from .dpm_solver_oracle import DPMSolverOracle


class UniPCOracle(DPMSolverOracle):
    """upstream ``UniPCMultistepScheduler`` (diffusers 0.33.1), stateful like upstream (``model_outputs``,
    ``timestep_list``, ``last_sample``, ``lower_order_nums``, ``this_order``, ``step_index``), so the reference's per-frame
    ``deepcopy`` gives per-frame histories.  ``cfg`` is a ``UniPCConfig``.

    **Parity with diffusers is unpinned** (diffusers is not installed): this restates the published source; the rounding
    of the bf16 path is stated in the module docstring.  ``table_dtype=torch.float64`` evaluates the sigma table and the
    coefficients in fp64 (mathematical anchors only; upstream is fp32)."""

    def __init__(self, cfg, table_dtype=torch.float32):
        if cfg.solver_type not in ("bh1", "bh2"):
            raise ValueError(cfg.solver_type)
        super().__init__(cfg, table_dtype)

    def _reset(self):
        self.model_outputs = [None] * self.cfg.solver_order
        self.timestep_list = [None] * self.cfg.solver_order
        self.lower_order_nums = 0
        self.last_sample = None
        self.this_order = None
        self.step_index = None

    def bh_coefs(self, t: int, s0: int, si: int = None):
        """The scalars of a UniP / UniC update from sigma index ``s0`` to ``t`` (and ``rk`` from ``si`` when given), as
        ``multistep_uni_p_bh_update`` / ``multistep_uni_c_bh_update`` evaluate them on 0-dim tensors."""
        alpha_t, sigma_t = self._alpha_sigma_t(self.sigmas[t])
        _, sigma_s0 = self._alpha_sigma_t(self.sigmas[s0])
        lambda_s0 = self._lambda(s0)
        h = self._lambda(t) - lambda_s0
        rk = (self._lambda(si) - lambda_s0) / h if si is not None else None
        hh = -h
        h_phi_1 = torch.expm1(hh)
        B_h = hh if self.cfg.solver_type == "bh1" else torch.expm1(hh)
        return types.SimpleNamespace(ratio=sigma_t / sigma_s0, cphi=alpha_t * h_phi_1, cB=alpha_t * B_h, rk=rk, hh=hh,
                                     h_phi_1=h_phi_1, B_h=B_h)

    @staticmethod
    def rhos_c(k) -> torch.Tensor:
        """``torch.linalg.solve(R, b)`` of the order-2 corrector (before upstream's cast to the sample dtype)."""
        rks = torch.stack([k.rk, torch.ones((), dtype=k.rk.dtype)])
        h_phi_k = k.h_phi_1 / k.hh - 1
        factorial_i = 1
        R, b = [], []
        for i in range(1, 3):
            R.append(torch.pow(rks, i - 1))
            b.append(h_phi_k * factorial_i / k.B_h)
            factorial_i *= i + 1
            h_phi_k = h_phi_k / k.hh - 1 / factorial_i
        return torch.linalg.solve(torch.stack(R), torch.stack(b))

    def step(self, model_output: torch.Tensor, timestep: int, sample: torch.Tensor) -> torch.Tensor:
        cfg = self.cfg
        if self.step_index is None:
            cand = (self.timesteps == int(timestep)).nonzero()
            self.step_index = int(cand[0]) if len(cand) else len(self.timesteps) - 1
        i, n = self.step_index, len(self.timesteps)
        bf = model_output.dtype == torch.bfloat16
        r = (lambda x: x.to(torch.bfloat16).float()) if bf else (lambda x: x)
        up = (lambda x: x.float()) if bf else (lambda x: x)
        use_corrector = i > 0 and (i - 1) not in cfg.disable_corrector and self.last_sample is not None
        m, x = up(model_output), up(sample)
        # convert_model_output (in the model output's dtype)
        alpha_s, sigma_s = self._alpha_sigma_t(self.sigmas[i])
        if cfg.prediction_type == "epsilon":
            x0 = r(r(x - r(sigma_s * m)) / alpha_s)
        elif cfg.prediction_type == "v_prediction":
            x0 = r(r(alpha_s * x) - r(sigma_s * m))
        elif cfg.prediction_type == "sample":
            x0 = m
        else:
            raise ValueError(cfg.prediction_type)
        if use_corrector:   # multistep_uni_c_bh_update of the previous step's result, at the previous step's order
            order = self.this_order
            k = self.bh_coefs(i, i - 1, i - 2 if order == 2 else None)
            m0 = up(self.model_outputs[-1])
            x_t_ = r(r(k.ratio * up(self.last_sample)) - r(k.cphi * m0))
            d1_t = r(x0 - m0)
            if order == 1:
                inner = r(0.0 + r(0.5 * d1_t))
            else:
                rho = up(self.rhos_c(k).to(sample.dtype))
                d1 = r(r(up(self.model_outputs[-2]) - m0) / k.rk)
                inner = r(r(rho[0] * d1) + r(rho[1] * d1_t))
            x = r(x_t_ - r(k.cB * inner))
        for j in range(cfg.solver_order - 1):
            self.model_outputs[j] = self.model_outputs[j + 1]
            self.timestep_list[j] = self.timestep_list[j + 1]
        self.model_outputs[-1] = x0.to(model_output.dtype)
        self.timestep_list[-1] = timestep
        this_order = min(cfg.solver_order, n - i) if cfg.lower_order_final else cfg.solver_order
        self.this_order = min(this_order, self.lower_order_nums + 1)
        self.last_sample = x.to(sample.dtype)
        # multistep_uni_p_bh_update
        k = self.bh_coefs(i + 1, i, i - 1 if self.this_order == 2 else None)
        x_t_ = r(r(k.ratio * x) - r(k.cphi * x0))
        if self.this_order == 1:
            prev = x_t_ - k.cB * 0
        else:
            d1 = r(r(up(self.model_outputs[-2]) - x0) / k.rk)
            prev = r(x_t_ - r(k.cB * r(0.5 * d1)))
        if self.lower_order_nums < cfg.solver_order:
            self.lower_order_nums += 1
        self.step_index += 1
        return prev.to(sample.dtype)
