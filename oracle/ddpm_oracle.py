"""CPU ORACLE (test infrastructure, NOT the product) for DDPM ancestral sampling through ``Diffuman4DPipeline``.

Restates upstream diffusers==0.33.1 ``DDPMScheduler`` (scheduling_ddpm.py: __init__, set_timesteps, previous_timestep,
_get_variance, step) for the fixed variance types "fixed_small", "fixed_small_log" and "fixed_large", without
thresholding, and the device's counter-based noise (include/d4d.h ``d4d_ddpm_sched``): a numpy Philox4x32-10 and an
fp64 Box-Muller.  Upstream draws the noise with ``randn_tensor(generator=None)`` from the CUDA RNG of whichever thread
runs the frame, which no one can reproduce; ``step`` takes the noise instead, and the per-frame copies of this oracle
draw the device's noise for their own frame (``__deepcopy__``), so the per-frame window and sliding oracles of
``dpm_solver_oracle`` run it unchanged.

PARITY STATUS: the per-frame copy, window and reset semantics are pinned against the reference's own pipeline code run
with a scheduler adapter backed by ``DDPMOracle`` (tests/golden/gen_golden_ddpm.py -> tests/golden/pipeline_ddpm_ref.pt,
tests/test_scheduler_ddpm.py).  The step ARITHMETIC is **parity unpinned** against diffusers (not installed): it restates
the published 0.33.1 source, with independent anchors in tests/test_scheduler_ddpm.py (the last step returns x0 exactly,
the noise-free fp64 step is the closed-form posterior mean, ``fixed_large`` has std^2 = beta_t).

bf16 emulation (the rule ``pipeline_oracle.DDIMOracle.step`` states): the reference runs the step on CUDA bf16 tensors
with 0-dim fp32 coefficients, so every ``coef * (bf16 tensor)`` and every op between bf16 tensors is computed in fp32 and
rounded once to bf16, ``std * z`` and the final sum included; the noise is drawn in bf16 (the model output's dtype).
"""
from __future__ import annotations

import numpy as np
import torch

_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_MASK = 0xFFFFFFFF


def philox4x32_10(counter, key):
    """Philox4x32-10 (Random123) of uint32 ``counter`` [..., 4] under ``key`` (k0, k1): uint32 [..., 4]."""
    c = [np.asarray(counter, dtype=np.uint64)[..., i].copy() for i in range(4)]
    k0, k1 = np.uint64(int(key[0]) & _MASK), np.uint64(int(key[1]) & _MASK)
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(_W0)) & np.uint64(_MASK), (k1 + np.uint64(_W1)) & np.uint64(_MASK)
        p0, p1 = c[0] * np.uint64(_M0), c[2] * np.uint64(_M1)
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(_MASK)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(_MASK)
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return np.stack(c, axis=-1).astype(np.uint32)


def _round_to_bf16(z: np.ndarray) -> np.ndarray:
    """fp64 -> bf16 rounded once to nearest even, as the fp64 values that hold the results."""
    b = z.astype(np.float64).view(np.uint64)
    b = (b + np.uint64((1 << 44) - 1) + ((b >> np.uint64(45)) & np.uint64(1))) & ~np.uint64((1 << 45) - 1)
    return b.view(np.float64)


def ddpm_noise_fp64(seed: int, frame_ids, timestep_indices, h: int, w: int) -> np.ndarray:
    """The device noise z in fp64, [F, 4, h, w]: element e of frame f takes word e % 4 of Philox4x32-10 with key = seed
    (low word first) and counter (e // 4, frame_ids[f], timestep_indices[f], 0); u = (x + 0.5) * 2^-32; Box-Muller
    (u0, u1) -> z0, z1 and (u2, u3) -> z2, z3."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    frame_ids = np.asarray(frame_ids, dtype=np.int64).reshape(-1)
    timestep_indices = np.asarray(timestep_indices, dtype=np.int64).reshape(-1)
    F, quads = len(frame_ids), h * w
    ctr = np.zeros((F, quads, 4), dtype=np.uint64)
    ctr[..., 0] = np.arange(quads, dtype=np.uint64)[None]
    ctr[..., 1] = (frame_ids.astype(np.uint64) & np.uint64(_MASK))[:, None]
    ctr[..., 2] = (timestep_indices.astype(np.uint64) & np.uint64(_MASK))[:, None]
    x = philox4x32_10(ctr, (seed & _MASK, seed >> 32)).astype(np.float64)
    u = (x + 0.5) * 2.0 ** -32
    z = np.empty_like(u)
    for p in range(2):
        r = np.sqrt(-2.0 * np.log(u[..., 2 * p]))
        a = 2.0 * np.pi * u[..., 2 * p + 1]
        z[..., 2 * p], z[..., 2 * p + 1] = r * np.cos(a), r * np.sin(a)
    return z.reshape(F, 4, h, w)


def ddpm_noise(seed: int, frame_ids, timestep_indices, h: int, w: int, dtype=torch.float32) -> torch.Tensor:
    """``ddpm_noise_fp64`` rounded once to ``dtype`` (float32, bfloat16 or float64)."""
    z = ddpm_noise_fp64(seed, frame_ids, timestep_indices, h, w)
    if dtype == torch.bfloat16:
        return torch.from_numpy(_round_to_bf16(z)).float().to(torch.bfloat16)   # both conversions are exact
    if dtype == torch.float32:
        return torch.from_numpy(z.astype(np.float32))
    return torch.from_numpy(z).to(dtype)


class DDPMOracle:
    """upstream ``DDPMScheduler`` (scheduling_ddpm.py, diffusers 0.33.1), fixed variances, no thresholding.

    ``table_dtype`` float64 builds ``alphas_cumprod`` in fp64 (for the anchors); upstream's is fp32.  ``seed`` and
    ``frame_id`` key the noise ``step`` draws when none is given: ``set_timesteps`` restarts the frame count, and each
    ``copy.deepcopy`` after it is the next frame of the task, as the k-th copy of PIPE:269 is frame k."""

    def __init__(self, cfg, seed: int = 0, table_dtype=torch.float32):
        self.cfg = cfg
        T = cfg.num_train_timesteps
        if cfg.beta_schedule == "scaled_linear":
            betas = torch.linspace(cfg.beta_start ** 0.5, cfg.beta_end ** 0.5, T, dtype=table_dtype) ** 2
        elif cfg.beta_schedule == "linear":
            betas = torch.linspace(cfg.beta_start, cfg.beta_end, T, dtype=table_dtype)
        else:
            raise ValueError(cfg.beta_schedule)
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.one = torch.tensor(1.0, dtype=table_dtype)
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = None
        self.seed = seed
        self.frame_id = None
        self._copies = 0

    def __deepcopy__(self, memo):
        new = object.__new__(type(self))
        new.__dict__.update(self.__dict__)
        new.frame_id = self._copies
        self._copies += 1
        return new

    def set_timesteps(self, n: int):
        cfg = self.cfg
        T = cfg.num_train_timesteps
        if n > T:
            raise ValueError("num_inference_steps > num_train_timesteps")
        self.num_inference_steps = n
        if cfg.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n).round()[::-1].copy().astype(np.int64)
        elif cfg.timestep_spacing == "leading":
            ts = (np.arange(0, n) * (T // n)).round()[::-1].copy().astype(np.int64)
            ts += cfg.steps_offset
        elif cfg.timestep_spacing == "trailing":
            ts = np.round(np.arange(T, 0, -T / n)).astype(np.int64) - 1
        else:
            raise ValueError(cfg.timestep_spacing)
        self.timesteps = torch.from_numpy(ts)
        self._copies = 0
        return self.timesteps

    def index_of(self, t: int) -> int:
        return int((self.timesteps == t).nonzero(as_tuple=True)[0][0])

    def previous_timestep(self, t: int) -> int:
        i = self.index_of(t)
        return -1 if i == self.timesteps.shape[0] - 1 else int(self.timesteps[i + 1])

    def _alphas(self, t: int):
        prev_t = self.previous_timestep(t)
        alpha_prod_t = self.alphas_cumprod[t]
        alpha_prod_t_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.one
        return alpha_prod_t, alpha_prod_t_prev

    def _get_variance(self, t: int):
        alpha_prod_t, alpha_prod_t_prev = self._alphas(t)
        current_beta_t = 1 - alpha_prod_t / alpha_prod_t_prev
        variance = torch.clamp((1 - alpha_prod_t_prev) / (1 - alpha_prod_t) * current_beta_t, min=1e-20)
        vt = self.cfg.variance_type
        if vt == "fixed_small":
            return variance
        if vt == "fixed_small_log":
            return torch.exp(0.5 * torch.log(variance))
        if vt == "fixed_large":
            return current_beta_t
        raise NotImplementedError(vt)

    def noise_std(self, t: int):
        """The 0-dim factor upstream multiplies the noise by: ``_get_variance ** 0.5`` (``fixed_small_log``: the value
        itself, already a standard deviation)."""
        v = self._get_variance(t)
        return v if self.cfg.variance_type == "fixed_small_log" else v ** 0.5

    def step(self, model_output: torch.Tensor, timestep: int, sample: torch.Tensor, noise: torch.Tensor = None,
             add_noise: bool = True) -> torch.Tensor:
        """One DDPM update of ``sample`` [1,4,h,w] (op by op in its dtype with 0-dim coefficients, as upstream).
        ``noise`` None: this frame's device noise (``ddpm_noise`` in the model output's dtype).  ``add_noise`` False
        leaves out the noise term (the posterior mean)."""
        cfg = self.cfg
        t = int(timestep)
        alpha_prod_t, alpha_prod_t_prev = self._alphas(t)
        beta_prod_t = 1 - alpha_prod_t
        beta_prod_t_prev = 1 - alpha_prod_t_prev
        current_alpha_t = alpha_prod_t / alpha_prod_t_prev
        current_beta_t = 1 - current_alpha_t
        c0 = (alpha_prod_t_prev ** 0.5 * current_beta_t) / beta_prod_t
        c1 = current_alpha_t ** 0.5 * beta_prod_t_prev / beta_prod_t
        sa, sb = alpha_prod_t ** 0.5, beta_prod_t ** 0.5
        bf16 = sample.dtype == torch.bfloat16
        if bf16:   # fp32 opmath, one bf16 rounding per op (see the module docstring)
            r = lambda x: x.to(torch.bfloat16).float()
            x, m = sample.float(), model_output.float()
            sa, sb, c0, c1 = (v.float() for v in (sa, sb, c0, c1))
        else:
            r = lambda x: x
            x, m = sample, model_output
        if cfg.prediction_type == "epsilon":
            x0 = r(r(x - r(sb * m)) / sa)
        elif cfg.prediction_type == "sample":
            x0 = m
        elif cfg.prediction_type == "v_prediction":
            x0 = r(r(sa * x) - r(sb * m))
        else:
            raise ValueError(cfg.prediction_type)
        if cfg.clip_sample:
            x0 = x0.clamp(-cfg.clip_sample_range, cfg.clip_sample_range)
        prev = r(r(c0 * x0) + r(c1 * x))
        if t > 0 and add_noise:
            if noise is None:
                h, w = sample.shape[-2:]
                noise = ddpm_noise(self.seed, [self.frame_id], [self.index_of(t)], h, w, model_output.dtype)
            std = self.noise_std(t)
            z = noise.reshape(prev.shape)
            prev = r(prev + r((std.float() if bf16 else std) * (z.float() if bf16 else z)))
        return prev.to(sample.dtype)
