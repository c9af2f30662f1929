"""UNet configuration for the Diffuman4D multiview denoiser hot path.

Mirrors the constructor knobs of the reference's ``UNetMultiviewConditionModel``
(reference: src/diffusers/models/unets/unet_multiview_condition.py:149-212).  Only the
knobs that change the arithmetic of the hot path are kept; everything the reference
never varies (dropout 0, act_fn silu, "default" time-scale-shift, layer_norm blocks,
geglu feed-forward, one transformer layer per block) is fixed here and stated in
DESIGN.md.

The shipped checkpoint's ``unet/config.json`` lives on Hugging Face and is not in the
repo (SURVEY.md section 0.3), so both plausible layouts are expressible:
``sd21()`` (heads 5/10/20/20 => head_dim 64, Linear proj) and ``ctor_default()``
(8 heads per level => head_dim 40/80/160, 1x1-conv proj).
"""
from __future__ import annotations

from dataclasses import dataclass, field, asdict
from typing import Optional, Tuple


@dataclass
class UNetConfig:
    in_channels: int = 11
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    layers_per_block: int = 2
    # "attention_head_dim" in the reference config is (mis)used as the number of heads
    # (unet_multiview_condition.py:219-225).
    attention_head_dim: Tuple[int, ...] = (5, 10, 20, 20)
    # None => no attn2 (block = 3-D self-attn + FF).  A per-level tuple equal to
    # block_out_channels => attn2 is an extra per-image self-attention (SURVEY 0.5).
    cross_attention_dim: Optional[Tuple[int, ...]] = None
    use_linear_projection: bool = True
    norm_num_groups: int = 32
    norm_eps: float = 1e-5
    flip_sin_to_cos: bool = True
    freq_shift: int = 0
    num_3d_attn_blocks: int = 3
    enable_tem_embeds: bool = True
    enable_pose_encoder: bool = True
    # reference pipelines read this (pipeline_diffuman4d.py:151)
    time_cond_proj_dim: Optional[int] = None
    center_input_sample: bool = False

    def __post_init__(self):
        self.block_out_channels = tuple(self.block_out_channels)
        n = len(self.block_out_channels)
        if isinstance(self.attention_head_dim, int):
            self.attention_head_dim = (self.attention_head_dim,) * n
        self.attention_head_dim = tuple(self.attention_head_dim)
        if isinstance(self.cross_attention_dim, int):
            self.cross_attention_dim = (self.cross_attention_dim,) * n
        if self.cross_attention_dim is not None:
            self.cross_attention_dim = tuple(self.cross_attention_dim)
        if n != 4:
            raise ValueError("the reference topology has exactly 4 resolution levels")
        if len(self.attention_head_dim) != n:
            raise ValueError("attention_head_dim must have one entry per level")
        for c, h in zip(self.block_out_channels, self.attention_head_dim):
            if c % h != 0:
                raise ValueError(f"channels {c} not divisible by heads {h}")
            if c % self.norm_num_groups != 0:
                raise ValueError(f"channels {c} not divisible by norm groups")
        if self.cross_attention_dim is not None:
            for c, x in zip(self.block_out_channels, self.cross_attention_dim):
                if x is not None and x != c:
                    raise ValueError(
                        "cross_attention_dim must equal block_out_channels per level: the pipeline never "
                        "passes encoder_hidden_states, so attn2 consumes width-C tokens (SURVEY 0.5)"
                    )

    # ---- derived -----------------------------------------------------------------
    @property
    def time_embed_dim(self) -> int:
        return self.block_out_channels[0] * 4

    def heads(self, level: int) -> int:
        return self.attention_head_dim[level]

    def head_dim(self, level: int) -> int:
        return self.block_out_channels[level] // self.attention_head_dim[level]

    def has_attn2(self, level: int) -> bool:
        return self.cross_attention_dim is not None and self.cross_attention_dim[level] is not None

    def to_dict(self) -> dict:
        return asdict(self)

    # ---- presets -----------------------------------------------------------------
    @classmethod
    def sd21(cls, **kw) -> "UNetConfig":
        """Stable-Diffusion-2.1 channel/head layout (the layout BASELINE.md's FLOP table uses)."""
        return cls(**kw)

    @classmethod
    def ctor_default(cls, **kw) -> "UNetConfig":
        """Reference constructor defaults: 8 heads per level, 1x1-conv projections."""
        base = dict(attention_head_dim=(8, 8, 8, 8), use_linear_projection=False,
                    enable_tem_embeds=False, enable_pose_encoder=False, in_channels=15)
        base.update(kw)
        return cls(**base)

    @classmethod
    def tiny(cls, **kw) -> "UNetConfig":
        """Small channel counts for CPU-speed tests (same topology, head_dim 64)."""
        base = dict(block_out_channels=(64, 128, 256, 256), attention_head_dim=(1, 2, 4, 4))
        base.update(kw)
        return cls(**base)


@dataclass
class SchedulerConfig:
    """DDIM scheduler knobs (upstream diffusers==0.33.1 ``DDIMScheduler`` defaults as used by SD-2.x)."""
    num_train_timesteps: int = 1000
    beta_start: float = 0.00085
    beta_end: float = 0.012
    beta_schedule: str = "scaled_linear"
    prediction_type: str = "epsilon"      # or "v_prediction"
    set_alpha_to_one: bool = False
    steps_offset: int = 1
    timestep_spacing: str = "leading"
    clip_sample: bool = False
    clip_sample_range: float = 1.0


@dataclass
class DPMSolverConfig:
    """DPM-Solver++ scheduler knobs (upstream diffusers==0.33.1 ``DPMSolverMultistepScheduler`` defaults) that the fused
    step implements: algorithm_type "dpmsolver++", solver_type "midpoint", solver_order 1 or 2, no thresholding, sigmas
    straight from the beta schedule."""
    num_train_timesteps: int = 1000
    beta_start: float = 0.0001
    beta_end: float = 0.02
    beta_schedule: str = "linear"         # or "scaled_linear"
    solver_order: int = 2                 # 1 or 2
    prediction_type: str = "epsilon"      # or "v_prediction", "sample"
    lower_order_final: bool = True
    euler_at_final: bool = False
    final_sigmas_type: str = "zero"       # or "sigma_min"
    timestep_spacing: str = "linspace"    # or "leading", "trailing"
    steps_offset: int = 0


@dataclass
class UniPCConfig:
    """UniPC scheduler knobs (upstream diffusers==0.33.1 ``UniPCMultistepScheduler`` defaults) that the fused step
    implements: predict_x0, solver_type "bh1" or "bh2", solver_order 1 or 2, no solver_p, no thresholding, sigmas straight
    from the beta schedule."""
    num_train_timesteps: int = 1000
    beta_start: float = 0.0001
    beta_end: float = 0.02
    beta_schedule: str = "linear"         # or "scaled_linear"
    solver_order: int = 2                 # 1 or 2
    prediction_type: str = "epsilon"      # or "v_prediction", "sample"
    solver_type: str = "bh2"              # or "bh1"
    lower_order_final: bool = True
    disable_corrector: Tuple[int, ...] = ()   # step indices whose result is not corrected by the next step
    final_sigmas_type: str = "zero"       # or "sigma_min"
    timestep_spacing: str = "linspace"    # or "leading", "trailing"
    steps_offset: int = 0

    def __post_init__(self):
        self.disable_corrector = tuple(int(i) for i in self.disable_corrector)


@dataclass
class PNDMConfig:
    """PNDM scheduler knobs (upstream diffusers==0.33.1 ``PNDMScheduler`` defaults, except ``skip_prk_steps``) that the
    fused step implements: skip_prk_steps (the PLMS steps only, as Stable Diffusion ships it), epsilon or v prediction,
    betas from a linear or scaled-linear schedule."""
    num_train_timesteps: int = 1000
    beta_start: float = 0.0001
    beta_end: float = 0.02
    beta_schedule: str = "linear"         # or "scaled_linear"
    prediction_type: str = "epsilon"      # or "v_prediction"
    set_alpha_to_one: bool = False
    timestep_spacing: str = "leading"     # or "linspace", "trailing"
    steps_offset: int = 0


@dataclass
class DEISConfig:
    """DEIS scheduler knobs (upstream diffusers==0.33.1 ``DEISMultistepScheduler`` defaults) that the fused step
    implements: algorithm_type "deis", solver_type "logrho", solver_order 1, 2 or 3, no thresholding, sigmas straight from
    the beta schedule (the last one is sigma_min: upstream has no final_sigmas_type knob for DEIS)."""
    num_train_timesteps: int = 1000
    beta_start: float = 0.0001
    beta_end: float = 0.02
    beta_schedule: str = "linear"         # or "scaled_linear"
    solver_order: int = 2                 # 1, 2 or 3
    prediction_type: str = "epsilon"      # or "v_prediction", "sample"
    lower_order_final: bool = True
    timestep_spacing: str = "linspace"    # or "leading", "trailing"
    steps_offset: int = 0


@dataclass
class DPMSingleConfig:
    """DPM-Solver++ singlestep scheduler knobs (upstream diffusers==0.33.1 ``DPMSolverSinglestepScheduler`` defaults) that
    the fused step implements: algorithm_type "dpmsolver++", solver_type "midpoint", solver_order 1, 2 or 3, no
    thresholding, sigmas straight from the beta schedule.  Upstream spaces the timesteps one way only (linspace over n + 1
    points, without the last), and its ``set_timesteps`` switches ``lower_order_final`` on when n is not a multiple of
    ``solver_order`` or the final sigma is zero."""
    num_train_timesteps: int = 1000
    beta_start: float = 0.0001
    beta_end: float = 0.02
    beta_schedule: str = "linear"         # or "scaled_linear"
    solver_order: int = 2                 # 1, 2 or 3
    prediction_type: str = "epsilon"      # or "v_prediction", "sample"
    lower_order_final: bool = False
    final_sigmas_type: str = "zero"       # or "sigma_min"
    timestep_spacing: str = "linspace"    # the only spacing upstream has


@dataclass
class DDPMConfig:
    """DDPM scheduler knobs (upstream diffusers==0.33.1 ``DDPMScheduler`` defaults) that the fused step implements:
    ancestral sampling with a fixed variance ("fixed_small", "fixed_small_log" or "fixed_large"), no thresholding, betas
    from a linear or scaled-linear schedule, DDIM's timestep spacings.  The noise of each step is counter-based
    (include/d4d.h ``d4d_ddpm_sched``), not torch's RNG stream."""
    num_train_timesteps: int = 1000
    beta_start: float = 0.0001
    beta_end: float = 0.02
    beta_schedule: str = "linear"         # or "scaled_linear"
    variance_type: str = "fixed_small"    # or "fixed_small_log", "fixed_large"
    clip_sample: bool = True
    clip_sample_range: float = 1.0
    prediction_type: str = "epsilon"      # or "v_prediction", "sample"
    timestep_spacing: str = "leading"     # or "linspace", "trailing"
    steps_offset: int = 0
