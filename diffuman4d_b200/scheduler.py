"""Host-side scheduler tables for the fused CFG + scheduler-step kernels: DDIM, DPM-Solver++ (multistep and singlestep),
UniPC, PNDM and DEIS.

Mirrors what the reference obtains from ``self.scheduler.set_timesteps(n)`` + per-frame deep copies
(pipeline_diffuman4d.py:265-271) for upstream diffusers==0.33.1 ``DDIMScheduler``: the ``timesteps`` vector and
``alphas_cumprod`` / ``final_alpha_cumprod``.  Only table construction lives here (numpy, host); the update itself
runs on the GPU (csrc/elementwise.cu ``cfg_ddim_kernel``).

``DPMSolverTables`` does the same for ``DPMSolverMultistepScheduler`` (dpmsolver++ / midpoint, order 1 or 2): the timesteps,
the sigma table and the per-step solver coefficients (``cfg_dpm_kernel``).  That scheduler is stateful, which is why the
reference deep-copies it per frame; here the state of every frame of a task is a ``DPMSolverState`` on the device.
``UniPCTables`` / ``UniPCState`` do the same for ``UniPCMultistepScheduler`` (``cfg_unipc_kernel``), whose corrector also
needs each frame's previous sample and, at order 2, a second data prediction of history.  ``PNDMTables`` / ``PNDMState``
do the same for ``PNDMScheduler`` with ``skip_prk_steps`` (``cfg_pndm_kernel``), whose history is the last four model
outputs, the sample of the frame's first step and its step counter.  ``DEISTables`` / ``DEISState`` do the same for
``DEISMultistepScheduler`` (``cfg_deis_kernel``, up to third order), whose history is the last two model outputs in their
epsilon form.  ``DPMSingleTables`` / ``DPMSingleState`` do the same for ``DPMSolverSinglestepScheduler``
(``cfg_dpm_single_kernel``, up to third order), whose history is the last two data predictions and the sample the frame's
current block started from.

Each tables class names the C entry points of its window step (``window_entry_points``: plain, frame-sharded and
CFG-split, None where there is none) and the bf16 state planes they take, in ABI order (``state_planes``; None for the stateless DDIM).
"""
from __future__ import annotations

import copy
import dataclasses

import numpy as np
import torch

from ._lib import D4DDeisSched, D4DDpmSched, D4DDpmSingleSched, D4DPndmSched, D4DSched, D4DUniPCSched
from .config import DEISConfig, DPMSingleConfig, DPMSolverConfig, PNDMConfig, SchedulerConfig, UniPCConfig

_PRED = {"epsilon": 0, "v_prediction": 1, "sample": 2}


class DDIMTables:
    init_noise_sigma = 1.0  # DDIM: scale_model_input is the identity, init sigma 1 (reference PIPE:189,376)
    window_entry_points = ("d4d_denoise_window", "d4d_denoise_window_sharded", "d4d_denoise_window_cfg_split")
    state_planes = None     # stateless: one table serves every frame

    def __init__(self, cfg: SchedulerConfig = None, device="cuda:0"):
        self.config = cfg or SchedulerConfig()
        c = self.config
        betas = _betas(c)
        if c.prediction_type not in _PRED:
            raise ValueError(f"prediction_type given as {c.prediction_type} must be one of {list(_PRED)}")
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = 1.0 if c.set_alpha_to_one else float(self.alphas_cumprod[0])
        self.device = torch.device(device)
        self._alphas_dev = None
        self.num_inference_steps = None
        self.timesteps = None          # host int64, like scheduler.timesteps
        self._timesteps_dev = None

    def set_timesteps(self, n: int, device=None):
        c = self.config
        T = c.num_train_timesteps
        if n > T:
            raise ValueError(f"`num_inference_steps`: {n} cannot be larger than `self.config.train_timesteps`: {T}")
        self.num_inference_steps = n
        if c.timestep_spacing == "leading":
            ts = (np.arange(0, n) * (T // n)).round()[::-1].copy().astype(np.int64) + c.steps_offset
        elif c.timestep_spacing == "trailing":
            ts = np.round(np.arange(T, 0, -T / n)).astype(np.int64) - 1
        elif c.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n).round()[::-1].copy().astype(np.int64)
        else:
            raise ValueError(f"{c.timestep_spacing} is not supported")
        self.timesteps = torch.from_numpy(ts)
        self._timesteps_dev = None
        return self.timesteps

    def c_struct(self, emulate_bf16: bool = False) -> D4DSched:
        if self.timesteps is None:
            raise ValueError("call set_timesteps first")
        if self._alphas_dev is None:
            self._alphas_dev = self.alphas_cumprod.to(self.device)
        if self._timesteps_dev is None:
            self._timesteps_dev = self.timesteps.to(self.device)
        c = self.config
        s = D4DSched()
        s.timesteps_table = self._timesteps_dev.data_ptr()
        s.alphas_cumprod = self._alphas_dev.data_ptr()
        s.n_steps = int(self.num_inference_steps)
        s.num_train_timesteps = int(c.num_train_timesteps)
        s.final_alpha_cumprod = float(self.final_alpha_cumprod)
        s.prediction_type = _PRED[c.prediction_type]
        s.clip_sample = int(c.clip_sample)
        s.clip_sample_range = float(c.clip_sample_range)
        s.emulate_bf16 = int(emulate_bf16)
        return s


def _betas(c) -> torch.Tensor:
    T = c.num_train_timesteps
    if c.beta_schedule == "scaled_linear":
        return torch.linspace(c.beta_start ** 0.5, c.beta_end ** 0.5, T, dtype=torch.float32) ** 2
    if c.beta_schedule == "linear":
        return torch.linspace(c.beta_start, c.beta_end, T, dtype=torch.float32)
    raise ValueError(f"{c.beta_schedule} is not implemented")


def dpm_timesteps(c: DPMSolverConfig, n: int) -> np.ndarray:
    """``DPMSolverMultistepScheduler.set_timesteps(n)`` timesteps (lambda_min_clipped = -inf); duplicates are refused,
    so that a frame's step index is always its timestep index."""
    T = c.num_train_timesteps
    if n > T:
        raise ValueError(f"`num_inference_steps`: {n} cannot be larger than `self.config.train_timesteps`: {T}")
    if c.timestep_spacing == "linspace":
        ts = np.linspace(0, T - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
    elif c.timestep_spacing == "leading":
        ts = (np.arange(0, n + 1) * (T // (n + 1))).round()[::-1][:-1].copy().astype(np.int64) + c.steps_offset
    elif c.timestep_spacing == "trailing":
        ts = np.arange(T, 0, -T / n).round().copy().astype(np.int64) - 1
    else:
        raise ValueError(f"{c.timestep_spacing} is not supported")
    if len(np.unique(ts)) != len(ts):
        raise ValueError(f"{c.timestep_spacing} spacing gives duplicate timesteps for {n} steps of {T}: {ts.tolist()}")
    return ts


def dpm_step_coefficients(sigmas: torch.Tensor) -> torch.Tensor:
    """[n, 6] fp32 coefficients of the n steps over ``sigmas`` [n+1] (layout in include/d4d.h ``d4d_dpm_sched``), each
    evaluated on 0-dim fp32 tensors in the order ``DPMSolverMultistepScheduler``'s ``convert_model_output`` /
    ``dpm_solver_first_order_update`` / ``multistep_dpm_solver_second_order_update`` evaluate them."""
    def alpha_sigma(sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha_t, sigma * alpha_t

    def lam(sigma):
        a, s = alpha_sigma(sigma)
        return torch.log(a) - torch.log(s)

    n = sigmas.numel() - 1
    out = torch.zeros(n, 6, dtype=torch.float32)
    for i in range(n):
        alpha_s, sigma_s = alpha_sigma(sigmas[i])
        alpha_t, sigma_t = alpha_sigma(sigmas[i + 1])
        h = lam(sigmas[i + 1]) - lam(sigmas[i])
        c = alpha_t * (torch.exp(-h) - 1.0)
        inv_r0 = 1.0 / ((lam(sigmas[i]) - lam(sigmas[i - 1])) / h) if i > 0 else torch.tensor(0.0)
        out[i] = torch.stack([alpha_s, sigma_s, sigma_t / sigma_s, c, 0.5 * c, inv_r0])
    return out


class _MultistepTables:
    """What ``DPMSolverTables``, ``UniPCTables``, ``DEISTables`` and ``DPMSingleTables`` share: the config checks common to
    all, the sigma
    table, ``set_timesteps`` and the device copies behind ``c_struct``.  A subclass adds its own checks (``_check``), its
    coefficient rows (``_coefficients``) and its C struct (``_struct``, plus the fields of ``_struct_fields``)."""
    init_noise_sigma = 1.0  # upstream: init_noise_sigma 1, scale_model_input is the identity
    solver_orders = (1, 2)  # the orders the fused step implements

    def __init__(self, cfg, device):
        self.config = c = cfg
        if c.prediction_type not in _PRED:
            raise ValueError(f"prediction_type given as {c.prediction_type} must be one of {list(_PRED)}")
        if c.solver_order not in self.solver_orders:
            orders = ", ".join(str(o) for o in self.solver_orders[:-1])
            raise NotImplementedError(f"solver_order={c.solver_order}: the fused step implements orders {orders} and "
                                      f"{self.solver_orders[-1]}")
        if self.final_sigmas_type not in ("zero", "sigma_min"):
            raise ValueError(f"final_sigmas_type {self.final_sigmas_type!r} must be 'zero' or 'sigma_min'")
        self._check(c)
        self.alphas_cumprod = torch.cumprod(1.0 - _betas(c), dim=0)
        self.all_sigmas = ((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5   # fp32 [T]
        self.device = torch.device(device)
        self.num_inference_steps = None
        self.timesteps = None          # host int64 [n]
        self.sigmas = None             # host fp32 [n+1]
        self.coefs = None              # host fp32 [n, coefficients per step]
        self._dev = None

    def _check(self, c):
        pass

    @property
    def final_sigmas_type(self) -> str:
        """The last sigma of the table: 0 ("zero") or that of the first training timestep ("sigma_min")."""
        return self.config.final_sigmas_type

    def _struct_fields(self) -> dict:
        return {}

    def set_timesteps(self, n: int, device=None):
        c = self.config
        ts = dpm_timesteps(c, n)       # UniPC, DEIS and singlestep space their timesteps like DPM-Solver++
        last = 0.0 if self.final_sigmas_type == "zero" else float(self.all_sigmas[0])
        self.num_inference_steps = n
        self.timesteps = torch.from_numpy(ts)
        self.sigmas = torch.cat([self.all_sigmas[self.timesteps], torch.tensor([last], dtype=torch.float32)])
        self.coefs = self._coefficients(self.sigmas)
        self._dev = None
        return self.timesteps

    def c_struct(self, emulate_bf16: bool = False):
        if self.timesteps is None:
            raise ValueError("call set_timesteps first")
        if self._dev is None:
            self._dev = (self.timesteps.to(self.device), self.coefs.to(self.device).contiguous())
        c = self.config
        return self._struct(timesteps_table=self._dev[0].data_ptr(), coefs=self._dev[1].data_ptr(),
                            n_steps=int(self.num_inference_steps), prediction_type=_PRED[c.prediction_type],
                            solver_order=int(c.solver_order), emulate_bf16=int(emulate_bf16), **self._struct_fields())


class DPMSolverTables(_MultistepTables):
    """Timesteps, sigmas and step coefficients of ``DPMSolverMultistepScheduler`` (diffusers 0.33.1) for
    ``cfg_dpm_kernel``."""
    name = "DPM-Solver++"
    window_entry_points = ("d4d_denoise_window_dpm", "d4d_denoise_window_dpm_sharded",
                          "d4d_denoise_window_dpm_cfg_split")
    state_planes = ("x0_prev",)
    _struct = D4DDpmSched

    def __init__(self, cfg: DPMSolverConfig = None, device="cuda:0"):
        super().__init__(cfg or DPMSolverConfig(), device)

    def _coefficients(self, sigmas: torch.Tensor) -> torch.Tensor:
        return dpm_step_coefficients(sigmas)

    @property
    def final_first_order(self) -> bool:
        """The last step falls back to first order (upstream ``lower_order_final`` in ``step``)."""
        c = self.config
        return bool(c.euler_at_final or (c.lower_order_final and self.num_inference_steps < 15)
                    or c.final_sigmas_type == "zero")

    def _struct_fields(self) -> dict:
        return {"final_first_order": int(self.final_first_order)}

    def new_state(self, num_frames: int) -> "DPMSolverState":
        return DPMSolverState(num_frames, self.device)


class SolverState:
    """The multistep solver history of every frame of one task, on the device: the bf16 planes named by ``planes``, each
    [F,4,h,w] and allocated (zeroed) when the latent size is first known, and ``lower_order_nums`` [F] int32.  A new task
    starts from zeros, which is the state of a freshly deep-copied upstream scheduler.  ``take`` / ``put`` gather and
    scatter the frames of one window."""

    def __init__(self, num_frames: int, device, planes: tuple, lower_order_nums: torch.Tensor = None, **tensors):
        self.num_frames = num_frames
        self.device = torch.device(device)
        self.planes = planes
        for name, t in tensors.items():
            setattr(self, name, t)
        self.lower_order_nums = (torch.zeros(num_frames, dtype=torch.int32, device=self.device)
                                 if lower_order_nums is None else lower_order_nums)

    def frames(self) -> list:
        """One handle per frame: what ``parepare_schedulers`` hands out in place of the per-frame scheduler copies."""
        return [DPMSolverFrame(self, i) for i in range(self.num_frames)]

    def _ensure(self, h: int, w: int):
        for name in self.planes:
            t = getattr(self, name)
            if t is None:
                setattr(self, name, torch.zeros(self.num_frames, 4, h, w, dtype=torch.bfloat16, device=self.device))
            elif tuple(t.shape[2:]) != (h, w):
                raise ValueError(f"solver state holds {tuple(t.shape[2:])} latents, got {(h, w)}")

    def take(self, index: torch.Tensor, h: int, w: int):
        """The state of frames ``index`` as a new (contiguous) state of the same kind, for one window."""
        self._ensure(h, w)
        index = index.to(self.device)
        window = copy.copy(self)
        window.num_frames = len(index)
        for name in (*self.planes, "lower_order_nums"):
            setattr(window, name, getattr(self, name)[index].contiguous())
        return window

    def put(self, index: torch.Tensor, window: "SolverState"):
        index = index.to(self.device)
        for name in (*self.planes, "lower_order_nums"):
            getattr(self, name)[index] = getattr(window, name)


class DPMSolverState(SolverState):
    """The DPM-Solver++ history: ``x0_prev`` (each frame's previous data prediction) and ``lower_order_nums``."""

    def __init__(self, num_frames: int, device, x0_prev: torch.Tensor = None, lower_order_nums: torch.Tensor = None):
        super().__init__(num_frames, device, DPMSolverTables.state_planes, lower_order_nums, x0_prev=x0_prev)


class DPMSolverFrame:
    """Frame ``index`` of a task's ``DPMSolverState`` or ``UniPCState`` (the per-frame scheduler object of the reference's
    lists)."""
    __slots__ = ("state", "index")

    def __init__(self, state: SolverState, index: int):
        self.state, self.index = state, index


# ---- UniPC ------------------------------------------------------------------------------------------------------------
UNIPC_COEFS = 14   # row layout in include/d4d.h ``d4d_unipc_sched``


def unipc_step_coefficients(c: UniPCConfig, sigmas: torch.Tensor) -> torch.Tensor:
    """[n, 14] fp32 coefficients of the n steps over ``sigmas`` [n+1] (layout in include/d4d.h ``d4d_unipc_sched``), each
    evaluated on 0-dim fp32 tensors in the order ``UniPCMultistepScheduler``'s ``convert_model_output`` /
    ``multistep_uni_p_bh_update`` / ``multistep_uni_c_bh_update`` / ``step`` evaluate them."""
    def alpha_sigma(sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha_t, sigma * alpha_t

    def lam(j):
        a, s = alpha_sigma(sigmas[j])
        return torch.log(a) - torch.log(s)

    def bh(t, s0, si):
        alpha_t, sigma_t = alpha_sigma(sigmas[t])
        h = lam(t) - lam(s0)
        rk = (lam(si) - lam(s0)) / h if si is not None else torch.tensor(0.0)
        hh = -h
        h_phi_1 = torch.expm1(hh)
        B_h = hh if c.solver_type == "bh1" else torch.expm1(hh)
        return sigma_t / alpha_sigma(sigmas[s0])[1], alpha_t * h_phi_1, alpha_t * B_h, rk, hh, h_phi_1, B_h

    n = sigmas.numel() - 1
    zero = torch.tensor(0.0)
    out = torch.zeros(n, UNIPC_COEFS, dtype=torch.float32)
    for i in range(n):
        alpha_s, sigma_s = alpha_sigma(sigmas[i])
        p_ratio, p_cphi, p_cB, p_rk = bh(i + 1, i, i - 1 if i > 0 else None)[:4]
        c_ratio = c_cphi = c_cB = c_rk = rho0 = rho1 = zero
        if i > 0:
            c_ratio, c_cphi, c_cB, c_rk, hh, h_phi_1, B_h = bh(i, i - 1, i - 2 if i > 1 else None)
            if i > 1:   # torch.linalg.solve(R, b) of the order-2 corrector
                rks = torch.stack([c_rk, torch.ones(())])
                h_phi_k = h_phi_1 / hh - 1
                factorial_i = 1
                R, b = [], []
                for k in range(1, 3):
                    R.append(torch.pow(rks, k - 1))
                    b.append(h_phi_k * factorial_i / B_h)
                    factorial_i *= k + 1
                    h_phi_k = h_phi_k / hh - 1 / factorial_i
                rho0, rho1 = torch.linalg.solve(torch.stack(R), torch.stack(b))
        corrector = float(i > 0 and (i - 1) not in c.disable_corrector)
        order_cap = float(min(c.solver_order, n - i) if c.lower_order_final else c.solver_order)
        out[i] = torch.stack([alpha_s, sigma_s, p_ratio, p_cphi, p_cB, p_rk, c_ratio, c_cphi, c_cB, c_rk, rho0, rho1,
                              torch.tensor(corrector), torch.tensor(order_cap)])
    return out


def _unipc_planes(solver_order: int) -> tuple:
    """UniPC's bf16 state planes in the order ``d4d_denoise_window_unipc`` takes them; ``x0_prev2`` exists at order 2
    only (None: its argument is NULL)."""
    return ("x0_prev", "x0_prev2" if solver_order == 2 else None, "last_sample")


class UniPCTables(_MultistepTables):
    """Timesteps, sigmas and step coefficients of ``UniPCMultistepScheduler`` (diffusers 0.33.1) for
    ``cfg_unipc_kernel``."""
    name = "UniPC"
    # no frame-sharded window: its window-result exchange carries DPM-Solver++'s state only
    window_entry_points = ("d4d_denoise_window_unipc", None, "d4d_denoise_window_unipc_cfg_split")
    _struct = D4DUniPCSched

    def __init__(self, cfg: UniPCConfig = None, device="cuda:0"):
        super().__init__(cfg or UniPCConfig(), device)

    def _check(self, c):
        if c.solver_type not in ("bh1", "bh2"):
            raise ValueError(f"solver_type {c.solver_type!r} must be 'bh1' or 'bh2'")
        if c.final_sigmas_type == "zero" and c.solver_order == 2 and not c.lower_order_final:
            raise NotImplementedError("final_sigmas_type='zero' with lower_order_final=False at solver_order 2: the last "
                                      "step's second-order term divides by an infinite h")
        if c.final_sigmas_type == "zero" and c.solver_type == "bh1":
            raise NotImplementedError("final_sigmas_type='zero' with solver_type='bh1': the last step's B(h) = -h is "
                                      "infinite and upstream returns NaN")

    def _coefficients(self, sigmas: torch.Tensor) -> torch.Tensor:
        return unipc_step_coefficients(self.config, sigmas)

    @property
    def state_planes(self) -> tuple:
        return _unipc_planes(self.config.solver_order)

    def new_state(self, num_frames: int) -> "UniPCState":
        return UniPCState(num_frames, self.device, self.config.solver_order)


class UniPCState(SolverState):
    """The UniPC history: ``x0_prev`` and ``lower_order_nums`` as DPM-Solver++'s, plus ``x0_prev2`` (the data prediction
    before ``x0_prev``; order 2 only, else None) and ``last_sample`` (the sample each frame's last predictor started from,
    after correction)."""

    def __init__(self, num_frames: int, device, solver_order: int = 2, x0_prev: torch.Tensor = None,
                 lower_order_nums: torch.Tensor = None, x0_prev2: torch.Tensor = None, last_sample: torch.Tensor = None):
        super().__init__(num_frames, device, tuple(p for p in _unipc_planes(solver_order) if p), lower_order_nums,
                         x0_prev=x0_prev, x0_prev2=x0_prev2, last_sample=last_sample)
        self.solver_order = solver_order


# ---- PNDM -------------------------------------------------------------------------------------------------------------
PNDM_COEFS = 10   # row layout in include/d4d.h ``d4d_pndm_sched``


def pndm_timesteps(c: PNDMConfig, n: int) -> np.ndarray:
    """``PNDMScheduler.set_timesteps(n)`` timesteps with ``skip_prk_steps``: the n spaced timesteps, the second-largest
    repeated, in descending order (n + 1 entries from n = 2 on; the counter-1 step re-steps to the repeated one)."""
    T = c.num_train_timesteps
    if n < 1:
        raise ValueError(f"num_inference_steps must be positive, got {n}")
    if c.timestep_spacing == "linspace":
        ts = np.linspace(0, T - 1, n).round().astype(np.int64)
    elif c.timestep_spacing == "leading":
        ts = (np.arange(0, n) * (T // n)).round() + c.steps_offset
    elif c.timestep_spacing == "trailing":
        ts = np.round(np.arange(T, 0, -T / n))[::-1].astype(np.int64) - 1
    else:
        raise ValueError(f"{c.timestep_spacing} is not supported")
    return np.concatenate([ts[:-1], ts[-2:-1], ts[-1:]])[::-1].copy().astype(np.int64)


def pndm_prev_sample_coefficients(alphas_cumprod: torch.Tensor, final_alpha_cumprod: torch.Tensor, t: int,
                                  prev: int) -> list:
    """The five scalars of ``PNDMScheduler._get_prev_sample`` from timestep ``t`` to ``prev``, evaluated on 0-dim tensors
    in upstream's order: a_t^0.5, (1 - a_t)^0.5, (a_prev / a_t)^0.5, a_prev - a_t and the denominator
    a_t (1 - a_prev)^0.5 + (a_t (1 - a_t) a_prev)^0.5."""
    a_t = alphas_cumprod[t]
    a_prev = alphas_cumprod[prev] if prev >= 0 else final_alpha_cumprod
    b_t = 1 - a_t
    b_prev = 1 - a_prev
    return [a_t ** 0.5, b_t ** 0.5, (a_prev / a_t) ** 0.5, a_prev - a_t,
            a_t * b_prev ** 0.5 + (a_t * b_t * a_prev) ** 0.5]


def pndm_step_coefficients(alphas_cumprod: torch.Tensor, final_alpha_cumprod: torch.Tensor, timesteps, n: int
                           ) -> torch.Tensor:
    """[len(timesteps), 10] coefficients of ``cfg_pndm_kernel`` (layout in include/d4d.h ``d4d_pndm_sched``) for
    ``n`` inference steps: each row's step from t to t - T // n, then the counter-1 step from t + T // n to t (NaN where
    t + T // n is past the table, where upstream's lookup fails)."""
    T = alphas_cumprod.numel()
    ratio = T // n
    out = torch.full((len(timesteps), PNDM_COEFS), float("nan"), dtype=alphas_cumprod.dtype)
    for i, t in enumerate(int(v) for v in timesteps):
        out[i, :5] = torch.stack(pndm_prev_sample_coefficients(alphas_cumprod, final_alpha_cumprod, t, t - ratio))
        if t + ratio < T:
            out[i, 5:] = torch.stack(pndm_prev_sample_coefficients(alphas_cumprod, final_alpha_cumprod, t + ratio, t))
    return out


class PNDMTables:
    """Timesteps and step coefficients of ``PNDMScheduler`` with ``skip_prk_steps`` (diffusers 0.33.1) for
    ``cfg_pndm_kernel``."""
    name = "PNDM"
    init_noise_sigma = 1.0  # upstream: init_noise_sigma 1, scale_model_input is the identity
    # no frame-sharded window: its window-result exchange carries DPM-Solver++'s state only
    window_entry_points = ("d4d_denoise_window_pndm", None, "d4d_denoise_window_pndm_cfg_split")
    state_planes = ("ets0", "ets1", "ets2", "ets3", "cur_sample")

    def __init__(self, cfg: PNDMConfig = None, device="cuda:0"):
        self.config = c = cfg or PNDMConfig()
        if c.prediction_type not in ("epsilon", "v_prediction"):
            raise NotImplementedError(f"prediction_type {c.prediction_type!r}: PNDM steps 'epsilon' or 'v_prediction'")
        if c.timestep_spacing not in ("linspace", "leading", "trailing"):
            raise ValueError(f"{c.timestep_spacing} is not supported")
        self.alphas_cumprod = torch.cumprod(1.0 - _betas(c), dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if c.set_alpha_to_one else self.alphas_cumprod[0]
        self.device = torch.device(device)
        self.num_inference_steps = None
        self.timesteps = None          # host int64 [n + 1] (n = 1: [1])
        self.coefs = None              # host fp32 [len(timesteps), 10]
        self._dev = None

    def set_timesteps(self, n: int, device=None):
        ts = pndm_timesteps(self.config, n)
        self.num_inference_steps = n
        self.timesteps = torch.from_numpy(ts)
        self.coefs = pndm_step_coefficients(self.alphas_cumprod, self.final_alpha_cumprod, ts, n)
        self._dev = None
        return self.timesteps

    def c_struct(self, emulate_bf16: bool = False) -> D4DPndmSched:
        if self.timesteps is None:
            raise ValueError("call set_timesteps first")
        if self._dev is None:
            self._dev = (self.timesteps.to(self.device), self.coefs.to(self.device).contiguous())
        s = D4DPndmSched()
        s.timesteps_table = self._dev[0].data_ptr()
        s.coefs = self._dev[1].data_ptr()
        s.n_steps = len(self.timesteps)
        s.prediction_type = _PRED[self.config.prediction_type]
        s.emulate_bf16 = int(emulate_bf16)
        return s

    def new_state(self, num_frames: int) -> "PNDMState":
        return PNDMState(num_frames, self.device)


class PNDMState(SolverState):
    """The PNDM history: ``ets0`` .. ``ets3`` (a ring of each frame's last model outputs: the output of counter c, c != 1,
    is in ``ets{(0 if c == 0 else c - 1) % 4}``), ``cur_sample`` (the sample each frame's first step started from) and,
    in ``lower_order_nums``, each frame's step counter (upstream ``counter``, not capped)."""

    def __init__(self, num_frames: int, device, counter: torch.Tensor = None, **planes):
        super().__init__(num_frames, device, PNDMTables.state_planes, counter,
                         **{name: planes.get(name) for name in PNDMTables.state_planes})

    @property
    def counter(self) -> torch.Tensor:
        return self.lower_order_nums


# ---- DEIS -------------------------------------------------------------------------------------------------------------
DEIS_COEFS = 11   # row layout in include/d4d.h ``d4d_deis_sched``


def _np_log(v: torch.Tensor) -> torch.Tensor:
    """``np.log`` of a 0-dim tensor, as upstream's ``ind_fn`` takes it: numpy's log in the tensor's dtype."""
    return torch.from_numpy(np.asarray(np.log(v.numpy())))


def deis_ind_coefficients(rho_t: torch.Tensor, rho_s: list) -> list:
    """The ``ind_fn`` coefficients of ``multistep_deis_second_order_update`` (``rho_s`` = [rho_s0, rho_s1]) or
    ``multistep_deis_third_order_update`` (``rho_s`` = [rho_s0, rho_s1, rho_s2]), evaluated like upstream: np.log of
    each 0-dim rho, every other operation on 0-dim tensors, in upstream's order."""
    def ind2(t, b, c):
        lt, lb, lc = _np_log(t), _np_log(b), _np_log(c)
        return t * (-lc + lt - 1) / (lb - lc)

    def ind3(t, b, c, d):
        lt, lb, lc, ld = _np_log(t), _np_log(b), _np_log(c), _np_log(d)
        numerator = t * (lc * (ld - lt + 1) - ld * lt + ld + lt ** 2 - 2 * lt + 2)
        denominator = (lb - lc) * (lb - ld)
        return numerator / denominator

    s0 = rho_s[0]
    if len(rho_s) == 2:
        s1 = rho_s[1]
        return [ind2(rho_t, s0, s1) - ind2(s0, s0, s1), ind2(rho_t, s1, s0) - ind2(s0, s1, s0)]
    s1, s2 = rho_s[1], rho_s[2]
    return [ind3(rho_t, s0, s1, s2) - ind3(s0, s0, s1, s2), ind3(rho_t, s1, s2, s0) - ind3(s0, s1, s2, s0),
            ind3(rho_t, s2, s0, s1) - ind3(s0, s2, s0, s1)]


def deis_order_cap(c: DEISConfig, i: int, n: int) -> int:
    """The highest order step i of n may take: ``solver_order``; 1 at the last step and 2 at the one before with
    ``lower_order_final`` below 15 steps (upstream ``lower_order_final`` / ``lower_order_second``); at most i + 1, as a
    frame has never taken more steps than its step index."""
    cap = min(c.solver_order, i + 1)
    if c.lower_order_final and n < 15:
        cap = min(cap, 1 if i == n - 1 else 2 if i == n - 2 else cap)
    return cap


def deis_step_coefficients(c: DEISConfig, sigmas: torch.Tensor) -> torch.Tensor:
    """[n, 11] fp32 coefficients of the n steps over ``sigmas`` [n+1] (layout in include/d4d.h ``d4d_deis_sched``), each
    evaluated on 0-dim fp32 tensors in the order ``DEISMultistepScheduler``'s ``convert_model_output`` /
    ``deis_first_order_update`` / ``multistep_deis_second_order_update`` / ``multistep_deis_third_order_update``
    evaluate them."""
    def alpha_sigma(j):
        alpha_t = 1 / ((sigmas[j] ** 2 + 1) ** 0.5)
        return alpha_t, sigmas[j] * alpha_t

    def lam(j):
        a, s = alpha_sigma(j)
        return torch.log(a) - torch.log(s)

    def rho(j):
        a, s = alpha_sigma(j)
        return s / a

    n = sigmas.numel() - 1
    zero = torch.tensor(0.0)
    out = torch.zeros(n, DEIS_COEFS, dtype=torch.float32)
    for i in range(n):
        alpha_s, sigma_s = alpha_sigma(i)
        alpha_t, sigma_t = alpha_sigma(i + 1)
        h = lam(i + 1) - lam(i)
        second = deis_ind_coefficients(rho(i + 1), [rho(i), rho(i - 1)]) if i >= 1 else [zero] * 2
        third = deis_ind_coefficients(rho(i + 1), [rho(i), rho(i - 1), rho(i - 2)]) if i >= 2 else [zero] * 3
        out[i] = torch.stack([alpha_s, sigma_s, alpha_t / alpha_s, sigma_t * (torch.exp(h) - 1.0), alpha_t, *second,
                              *third, torch.tensor(float(deis_order_cap(c, i, n)))])
    return out


def _deis_planes(solver_order: int) -> tuple:
    """DEIS's bf16 state planes in the order ``d4d_denoise_window_deis`` takes them; ``m_prev2`` exists at order 3 only
    (None: its argument is NULL)."""
    return ("m_prev", "m_prev2" if solver_order == 3 else None)


class DEISTables(_MultistepTables):
    """Timesteps, sigmas and step coefficients of ``DEISMultistepScheduler`` (algorithm_type "deis", solver_type
    "logrho"; diffusers 0.33.1) for ``cfg_deis_kernel``."""
    name = "DEIS"
    solver_orders = (1, 2, 3)
    # no frame-sharded window: its window-result exchange carries DPM-Solver++'s state only
    window_entry_points = ("d4d_denoise_window_deis", None, "d4d_denoise_window_deis_cfg_split")
    final_sigmas_type = "sigma_min"   # upstream's table always ends on the sigma of the first training timestep
    _struct = D4DDeisSched

    def __init__(self, cfg: DEISConfig = None, device="cuda:0"):
        super().__init__(cfg or DEISConfig(), device)

    def _coefficients(self, sigmas: torch.Tensor) -> torch.Tensor:
        return deis_step_coefficients(self.config, sigmas)

    @property
    def state_planes(self) -> tuple:
        return _deis_planes(self.config.solver_order)

    def new_state(self, num_frames: int) -> "DEISState":
        return DEISState(num_frames, self.device, self.config.solver_order)


class DEISState(SolverState):
    """The DEIS history: ``m_prev`` (each frame's previous model output, converted to its epsilon form), ``m_prev2`` (the
    one before; order 3 only, else None) and ``lower_order_nums``."""

    def __init__(self, num_frames: int, device, solver_order: int = 2, m_prev: torch.Tensor = None,
                 m_prev2: torch.Tensor = None, lower_order_nums: torch.Tensor = None):
        super().__init__(num_frames, device, tuple(p for p in _deis_planes(solver_order) if p), lower_order_nums,
                         m_prev=m_prev, m_prev2=m_prev2)
        self.solver_order = solver_order


# ---- DPM-Solver++ singlestep ------------------------------------------------------------------------------------------
DPM_SINGLE_COEFS = 13   # row layout in include/d4d.h ``d4d_dpm_single_sched``


def dpm_single_order_list(solver_order: int, lower_order_final: bool, final_sigmas_type: str, n: int) -> list:
    """The order of each of the n steps (upstream ``DPMSolverSinglestepScheduler.get_order_list``): blocks 1, 2, ..,
    solver_order.  With ``lower_order_final`` the list ends on a shorter block: the last n % solver_order steps form one,
    and when that is none, the last full block is split into 1, .., solver_order - 1 and 1.  Without it n must be a
    multiple of solver_order (``set_timesteps`` switches it on otherwise).  A zero final sigma makes the last step first
    order."""
    block = list(range(1, solver_order + 1))
    full, rest = divmod(n, solver_order)
    if not lower_order_final:
        if rest:
            raise ValueError(f"{n} steps are not whole blocks of {solver_order} without lower_order_final")
        orders = block * full
    elif rest:
        orders = block * full + block[:rest]
    else:
        orders = block * (full - 1) + block[:-1] + [1]
    if final_sigmas_type == "zero":
        orders[-1] = 1
    return orders


def dpm_single_step_coefficients(orders: list, sigmas: torch.Tensor) -> torch.Tensor:
    """[n, 13] fp32 coefficients of the n steps over ``sigmas`` [n+1] with the rows' ``orders`` (layout in include/d4d.h
    ``d4d_dpm_single_sched``), each evaluated on 0-dim fp32 tensors in the order ``DPMSolverSinglestepScheduler``'s
    ``convert_model_output`` / ``dpm_solver_first_order_update`` / ``singlestep_dpm_solver_second_order_update`` /
    ``singlestep_dpm_solver_third_order_update`` evaluate them.  The first-order scalars are DPM-Solver++ multistep's.
    The update of order k at row i spans the block from row i - k + 1; entries of orders above the row's are 0."""
    def alpha_sigma(sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha_t, sigma * alpha_t

    def lam(j):
        a, s = alpha_sigma(sigmas[j])
        return torch.log(a) - torch.log(s)

    first = dpm_step_coefficients(sigmas)
    n = sigmas.numel() - 1
    out = torch.zeros(n, DPM_SINGLE_COEFS, dtype=torch.float32)
    out[:, :4] = first[:, :4]
    for i, order in enumerate(orders):
        alpha_t, sigma_t = alpha_sigma(sigmas[i + 1])
        lambda_t, lambda_s0 = lam(i + 1), lam(i)
        if order >= 2:
            lambda_s1 = lam(i - 1)
            h = lambda_t - lambda_s1
            r0 = (lambda_s0 - lambda_s1) / h
            c = alpha_t * (torch.exp(-h) - 1.0)
            out[i, 4:8] = torch.stack([sigma_t / alpha_sigma(sigmas[i - 1])[1], c, 0.5 * c, 1.0 / r0])
        if order == 3:
            lambda_s2 = lam(i - 2)
            h = lambda_t - lambda_s2
            r0 = (lambda_s0 - lambda_s2) / h
            c = alpha_t * (torch.exp(-h) - 1.0)
            out[i, 8:12] = torch.stack([sigma_t / alpha_sigma(sigmas[i - 2])[1], c,
                                        alpha_t * ((torch.exp(-h) - 1.0) / h + 1.0), 1.0 / r0])
        out[i, 12] = float(order)
    return out


def _dpm_single_planes(solver_order: int) -> tuple:
    """The singlestep solver's bf16 state planes in the order ``d4d_denoise_window_dpm_single`` takes them; ``x0_prev2``
    exists at order 3 only (None: its argument is NULL)."""
    return ("x0_prev", "x0_prev2" if solver_order == 3 else None, "cur_sample")


class DPMSingleTables(_MultistepTables):
    """Timesteps, sigmas, order list and step coefficients of ``DPMSolverSinglestepScheduler`` (algorithm_type
    "dpmsolver++", solver_type "midpoint"; diffusers 0.33.1) for ``cfg_dpm_single_kernel``.

    ``config`` is this object's own copy: like upstream's ``register_to_config``, ``set_timesteps`` switches its
    ``lower_order_final`` on when the step count is not a multiple of ``solver_order`` or the final sigma is zero, and
    the switch stays for later ``set_timesteps`` calls."""
    name = "DPM-Solver++ singlestep"
    solver_orders = (1, 2, 3)
    # no frame-sharded window: its window-result exchange carries DPM-Solver++ multistep's state only
    window_entry_points = ("d4d_denoise_window_dpm_single", None,
                          "d4d_denoise_window_dpm_single_cfg_split")
    _struct = D4DDpmSingleSched

    def __init__(self, cfg: DPMSingleConfig = None, device="cuda:0"):
        super().__init__(dataclasses.replace(cfg or DPMSingleConfig()), device)
        self.order_list = None          # the order of each step, after set_timesteps

    def _check(self, c):
        if c.timestep_spacing != "linspace":
            raise ValueError(f"timestep_spacing {c.timestep_spacing!r}: DPMSolverSinglestepScheduler spaces its timesteps "
                             "by 'linspace' only")

    def set_timesteps(self, n: int, device=None):
        c = self.config
        if not c.lower_order_final and (n % c.solver_order != 0 or c.final_sigmas_type == "zero"):
            c.lower_order_final = True
        self.order_list = dpm_single_order_list(c.solver_order, c.lower_order_final, c.final_sigmas_type, n)
        return super().set_timesteps(n, device)

    def _coefficients(self, sigmas: torch.Tensor) -> torch.Tensor:
        return dpm_single_step_coefficients(self.order_list, sigmas)

    @property
    def state_planes(self) -> tuple:
        return _dpm_single_planes(self.config.solver_order)

    def new_state(self, num_frames: int) -> "DPMSingleState":
        return DPMSingleState(num_frames, self.device, self.config.solver_order)


class DPMSingleState(SolverState):
    """The DPM-Solver++ singlestep history: ``x0_prev`` (each frame's previous data prediction), ``x0_prev2`` (the one
    before; order 3 only, else None), ``cur_sample`` (the sample the frame's current block started from) and
    ``lower_order_nums``."""

    def __init__(self, num_frames: int, device, solver_order: int = 2, x0_prev: torch.Tensor = None,
                 x0_prev2: torch.Tensor = None, cur_sample: torch.Tensor = None, lower_order_nums: torch.Tensor = None):
        super().__init__(num_frames, device, tuple(p for p in _dpm_single_planes(solver_order) if p), lower_order_nums,
                         x0_prev=x0_prev, x0_prev2=x0_prev2, cur_sample=cur_sample)
        self.solver_order = solver_order
