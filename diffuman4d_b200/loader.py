"""``load_pipelines`` -- drop-in for the reference's Hydra ``model`` target (seam B-1, SURVEY.md section 8b).

Reference: src/samplers/utils/sampling_utils.py:17-51 (``_target_`` of configs/model/diffuman4d.yaml:1).  A config
file ``configs/model/diffuman4d_b200.yaml`` with ``_target_: diffuman4d_b200.loader.load_pipelines`` makes the
reference's ``inference.py`` build the CUDA pipelines without source edits (see INTEGRATION.md).

Reads the diffusers-layout checkpoint directory:  ``unet/config.json``, ``unet/diffusion_pytorch_model.safetensors``
and ``scheduler/scheduler_config.json``.  No network access is attempted here; if ``huggingface_hub`` is importable the
snapshot download of the reference is mirrored, otherwise the directory must already exist.
"""
from __future__ import annotations

import importlib
import json
import math
import os
import warnings
from typing import Callable, List, Optional, Union

import torch

from .config import (DDPMConfig, DEISConfig, DPMSingleConfig, DPMSolverConfig, PNDMConfig, SchedulerConfig, UNetConfig,
                     UniPCConfig)
from .pipeline import B200Diffuman4DPipeline
from .unet import B200MultiviewUNet


def unet_config_from_json(d: dict) -> UNetConfig:
    """Map a diffusers ``unet/config.json`` onto ``UNetConfig``; refuse knobs the CUDA path does not implement."""
    def want(key, allowed, default):
        v = d.get(key, default)
        if v not in allowed:
            raise NotImplementedError(f"unet config {key}={v!r} is not supported by the CUDA path (supported: {allowed})")
        return v

    want("act_fn", ("silu", "swish"), "silu")
    want("resnet_time_scale_shift", ("default",), "default")
    want("time_embedding_type", ("positional",), "positional")
    want("class_embed_type", (None,), None)
    want("addition_embed_type", (None,), None)
    want("dual_cross_attention", (False,), False)
    want("transformer_layers_per_block", (1,), 1)
    want("mid_block_scale_factor", (1, 1.0), 1)
    want("resnet_out_scale_factor", (1, 1.0), 1.0)
    want("only_cross_attention", (False,), False)
    want("time_cond_proj_dim", (None,), None)
    want("conv_in_kernel", (3,), 3)
    want("conv_out_kernel", (3,), 3)
    heads = d.get("attention_head_dim", 8)
    if d.get("num_attention_heads") is not None:
        raise ValueError("num_attention_heads must be None (reference unet_multiview_condition.py:214-217)")
    return UNetConfig(
        in_channels=d.get("in_channels", 4), out_channels=d.get("out_channels", 4),
        block_out_channels=tuple(d.get("block_out_channels", (320, 640, 1280, 1280))),
        layers_per_block=d.get("layers_per_block", 2), attention_head_dim=heads,
        cross_attention_dim=d.get("cross_attention_dim", 1280),
        use_linear_projection=d.get("use_linear_projection", False), norm_num_groups=d.get("norm_num_groups", 32),
        norm_eps=d.get("norm_eps", 1e-5), flip_sin_to_cos=d.get("flip_sin_to_cos", True),
        freq_shift=d.get("freq_shift", 0), num_3d_attn_blocks=d.get("num_3d_attn_blocks", 3),
        enable_tem_embeds=d.get("enable_tem_embeds", False), enable_pose_encoder=d.get("enable_pose_encoder", False),
        center_input_sample=d.get("center_input_sample", False))


def dpm_solver_config_from_json(d: dict) -> DPMSolverConfig:
    """Map a diffusers ``DPMSolverMultistepScheduler`` config; every knob the fused step does not implement raises
    ``NotImplementedError`` naming the key."""
    def refuse(key, why):
        raise NotImplementedError(f"DPMSolverMultistepScheduler {key}={d.get(key)!r} is not supported by the CUDA path "
                                  f"({why})")

    def want(key, allowed, default):
        v = d.get(key, default)
        if v not in allowed:
            refuse(key, f"supported: {allowed}")
        return v

    if d.get("thresholding", False):
        refuse("thresholding", "dynamic thresholding is not implemented")
    for key in ("use_karras_sigmas", "use_exponential_sigmas", "use_beta_sigmas", "use_lu_lambdas", "use_flow_sigmas"):
        if d.get(key, False):
            refuse(key, "sigmas come straight from the beta schedule")
    if d.get("rescale_betas_zero_snr", False):
        refuse("rescale_betas_zero_snr", "zero-SNR rescaling is not implemented")
    lmc = d.get("lambda_min_clipped", -math.inf)
    if lmc is not None and math.isfinite(float(lmc)):
        refuse("lambda_min_clipped", "only -inf (no clipping)")
    if d.get("variance_type") is not None:
        refuse("variance_type", "only None")
    want("algorithm_type", ("dpmsolver++",), "dpmsolver++")
    want("solver_type", ("midpoint",), "midpoint")
    want("solver_order", (1, 2), 2)
    want("beta_schedule", ("linear", "scaled_linear"), "linear")
    want("prediction_type", ("epsilon", "v_prediction", "sample"), "epsilon")
    want("final_sigmas_type", ("zero", "sigma_min"), "zero")
    want("timestep_spacing", ("linspace", "leading", "trailing"), "linspace")
    if d.get("trained_betas") is not None:
        refuse("trained_betas", "betas come from beta_schedule")
    return DPMSolverConfig(
        num_train_timesteps=d.get("num_train_timesteps", 1000), beta_start=d.get("beta_start", 0.0001),
        beta_end=d.get("beta_end", 0.02), beta_schedule=d.get("beta_schedule", "linear"),
        solver_order=d.get("solver_order", 2), prediction_type=d.get("prediction_type", "epsilon"),
        lower_order_final=d.get("lower_order_final", True), euler_at_final=d.get("euler_at_final", False),
        final_sigmas_type=d.get("final_sigmas_type", "zero"), timestep_spacing=d.get("timestep_spacing", "linspace"),
        steps_offset=d.get("steps_offset", 0))


def unipc_config_from_json(d: dict) -> UniPCConfig:
    """Map a diffusers ``UniPCMultistepScheduler`` config; every knob the fused step does not implement raises
    ``NotImplementedError`` naming the key."""
    def refuse(key, why):
        raise NotImplementedError(f"UniPCMultistepScheduler {key}={d.get(key)!r} is not supported by the CUDA path "
                                  f"({why})")

    def want(key, allowed, default):
        v = d.get(key, default)
        if v not in allowed:
            refuse(key, f"supported: {allowed}")
        return v

    if not d.get("predict_x0", True):
        refuse("predict_x0", "only the data-prediction (predict_x0=True) form is implemented")
    if d.get("solver_p") is not None:
        refuse("solver_p", "only UniPC's own predictor")
    if d.get("thresholding", False):
        refuse("thresholding", "dynamic thresholding is not implemented")
    for key in ("use_karras_sigmas", "use_exponential_sigmas", "use_beta_sigmas", "use_flow_sigmas"):
        if d.get(key, False):
            refuse(key, "sigmas come straight from the beta schedule")
    if d.get("rescale_betas_zero_snr", False):
        refuse("rescale_betas_zero_snr", "zero-SNR rescaling is not implemented")
    if d.get("trained_betas") is not None:
        refuse("trained_betas", "betas come from beta_schedule")
    order = want("solver_order", (1, 2), 2)
    solver_type = want("solver_type", ("bh1", "bh2"), "bh2")
    want("beta_schedule", ("linear", "scaled_linear"), "linear")
    want("prediction_type", ("epsilon", "v_prediction", "sample"), "epsilon")
    final = want("final_sigmas_type", ("zero", "sigma_min"), "zero")
    want("timestep_spacing", ("linspace", "leading", "trailing"), "linspace")
    lower_order_final = d.get("lower_order_final", True)
    if final == "zero" and order == 2 and not lower_order_final:
        refuse("final_sigmas_type", "'zero' with lower_order_final=False at solver_order 2: the last step's "
                                    "second-order term divides by an infinite h")
    if final == "zero" and solver_type == "bh1":
        refuse("final_sigmas_type", "'zero' with solver_type='bh1': the last step's B(h) = -h is infinite")
    return UniPCConfig(
        num_train_timesteps=d.get("num_train_timesteps", 1000), beta_start=d.get("beta_start", 0.0001),
        beta_end=d.get("beta_end", 0.02), beta_schedule=d.get("beta_schedule", "linear"), solver_order=order,
        prediction_type=d.get("prediction_type", "epsilon"), solver_type=solver_type,
        lower_order_final=lower_order_final, disable_corrector=tuple(d.get("disable_corrector") or ()),
        final_sigmas_type=final, timestep_spacing=d.get("timestep_spacing", "linspace"),
        steps_offset=d.get("steps_offset", 0))


def pndm_config_from_json(d: dict) -> PNDMConfig:
    """Map a diffusers ``PNDMScheduler`` config; every knob the fused step does not implement raises
    ``NotImplementedError`` naming the key."""
    def refuse(key, why):
        raise NotImplementedError(f"PNDMScheduler {key}={d.get(key)!r} is not supported by the CUDA path ({why})")

    def want(key, allowed, default):
        v = d.get(key, default)
        if v not in allowed:
            refuse(key, f"supported: {allowed}")
        return v

    if not d.get("skip_prk_steps", False):
        refuse("skip_prk_steps", "only the PLMS steps (skip_prk_steps=True) are implemented, not the Runge-Kutta warm-up")
    if d.get("trained_betas") is not None:
        refuse("trained_betas", "betas come from beta_schedule")
    want("beta_schedule", ("linear", "scaled_linear"), "linear")
    want("prediction_type", ("epsilon", "v_prediction"), "epsilon")
    want("timestep_spacing", ("linspace", "leading", "trailing"), "leading")
    return PNDMConfig(
        num_train_timesteps=d.get("num_train_timesteps", 1000), beta_start=d.get("beta_start", 0.0001),
        beta_end=d.get("beta_end", 0.02), beta_schedule=d.get("beta_schedule", "linear"),
        prediction_type=d.get("prediction_type", "epsilon"), set_alpha_to_one=d.get("set_alpha_to_one", False),
        timestep_spacing=d.get("timestep_spacing", "leading"), steps_offset=d.get("steps_offset", 0))


def deis_config_from_json(d: dict) -> DEISConfig:
    """Map a diffusers ``DEISMultistepScheduler`` config; every knob the fused step does not implement raises
    ``NotImplementedError`` naming the key."""
    def refuse(key, why):
        raise NotImplementedError(f"DEISMultistepScheduler {key}={d.get(key)!r} is not supported by the CUDA path ({why})")

    def want(key, allowed, default):
        v = d.get(key, default)
        if v not in allowed:
            refuse(key, f"supported: {allowed}")
        return v

    if d.get("thresholding", False):
        refuse("thresholding", "dynamic thresholding is not implemented")
    for key in ("use_karras_sigmas", "use_exponential_sigmas", "use_beta_sigmas", "use_flow_sigmas",
                "use_dynamic_shifting"):
        if d.get(key, False):
            refuse(key, "sigmas come straight from the beta schedule")
    if d.get("rescale_betas_zero_snr", False):
        refuse("rescale_betas_zero_snr", "zero-SNR rescaling is not implemented")
    if d.get("trained_betas") is not None:
        refuse("trained_betas", "betas come from beta_schedule")
    want("algorithm_type", ("deis",), "deis")
    want("solver_type", ("logrho",), "logrho")
    order = want("solver_order", (1, 2, 3), 2)
    want("beta_schedule", ("linear", "scaled_linear"), "linear")
    want("prediction_type", ("epsilon", "v_prediction", "sample"), "epsilon")
    want("timestep_spacing", ("linspace", "leading", "trailing"), "linspace")
    return DEISConfig(
        num_train_timesteps=d.get("num_train_timesteps", 1000), beta_start=d.get("beta_start", 0.0001),
        beta_end=d.get("beta_end", 0.02), beta_schedule=d.get("beta_schedule", "linear"), solver_order=order,
        prediction_type=d.get("prediction_type", "epsilon"), lower_order_final=d.get("lower_order_final", True),
        timestep_spacing=d.get("timestep_spacing", "linspace"), steps_offset=d.get("steps_offset", 0))


def dpm_single_config_from_json(d: dict) -> DPMSingleConfig:
    """Map a diffusers ``DPMSolverSinglestepScheduler`` config; every knob the fused step does not implement raises
    ``NotImplementedError`` naming the key."""
    def refuse(key, why):
        raise NotImplementedError(f"DPMSolverSinglestepScheduler {key}={d.get(key)!r} is not supported by the CUDA path "
                                  f"({why})")

    def want(key, allowed, default):
        v = d.get(key, default)
        if v not in allowed:
            refuse(key, f"supported: {allowed}")
        return v

    if d.get("thresholding", False):
        refuse("thresholding", "dynamic thresholding is not implemented")
    for key in ("use_karras_sigmas", "use_exponential_sigmas", "use_beta_sigmas", "use_flow_sigmas",
                "use_dynamic_shifting"):
        if d.get(key, False):
            refuse(key, "sigmas come straight from the beta schedule")
    lmc = d.get("lambda_min_clipped", -math.inf)
    if lmc is not None and math.isfinite(float(lmc)):
        refuse("lambda_min_clipped", "only -inf (no clipping)")
    if d.get("variance_type") is not None:
        refuse("variance_type", "only None")
    if d.get("trained_betas") is not None:
        refuse("trained_betas", "betas come from beta_schedule")
    want("algorithm_type", ("dpmsolver++",), "dpmsolver++")
    want("solver_type", ("midpoint",), "midpoint")
    order = want("solver_order", (1, 2, 3), 2)
    want("beta_schedule", ("linear", "scaled_linear"), "linear")
    want("prediction_type", ("epsilon", "v_prediction", "sample"), "epsilon")
    want("final_sigmas_type", ("zero", "sigma_min"), "zero")
    want("timestep_spacing", ("linspace",), "linspace")    # upstream has no other spacing for this class
    return DPMSingleConfig(
        num_train_timesteps=d.get("num_train_timesteps", 1000), beta_start=d.get("beta_start", 0.0001),
        beta_end=d.get("beta_end", 0.02), beta_schedule=d.get("beta_schedule", "linear"), solver_order=order,
        prediction_type=d.get("prediction_type", "epsilon"), lower_order_final=d.get("lower_order_final", False),
        final_sigmas_type=d.get("final_sigmas_type", "zero"))


def ddpm_config_from_json(d: dict) -> DDPMConfig:
    """Map a diffusers ``DDPMScheduler`` config; every knob the fused step does not implement raises
    ``NotImplementedError`` naming the key."""
    def refuse(key, why):
        raise NotImplementedError(f"DDPMScheduler {key}={d.get(key)!r} is not supported by the CUDA path ({why})")

    def want(key, allowed, default):
        v = d.get(key, default)
        if v not in allowed:
            refuse(key, f"supported: {allowed}")
        return v

    if d.get("thresholding", False):
        refuse("thresholding", "dynamic thresholding is not implemented")
    if d.get("rescale_betas_zero_snr", False):
        refuse("rescale_betas_zero_snr", "zero-SNR rescaling is not implemented")
    if d.get("trained_betas") is not None:
        refuse("trained_betas", "betas come from beta_schedule")
    vt = d.get("variance_type", "fixed_small")
    if vt in ("learned", "learned_range"):
        refuse("variance_type", "a learned variance needs a UNet with 2 * out_channels outputs")
    if vt == "fixed_large_log":
        refuse("variance_type", "upstream takes the square root of a log there")
    want("variance_type", ("fixed_small", "fixed_small_log", "fixed_large"), "fixed_small")
    want("beta_schedule", ("linear", "scaled_linear"), "linear")
    want("prediction_type", ("epsilon", "v_prediction", "sample"), "epsilon")
    want("timestep_spacing", ("leading", "linspace", "trailing"), "leading")
    return DDPMConfig(
        num_train_timesteps=d.get("num_train_timesteps", 1000), beta_start=d.get("beta_start", 0.0001),
        beta_end=d.get("beta_end", 0.02), beta_schedule=d.get("beta_schedule", "linear"), variance_type=vt,
        clip_sample=d.get("clip_sample", True), clip_sample_range=d.get("clip_sample_range", 1.0),
        prediction_type=d.get("prediction_type", "epsilon"), timestep_spacing=d.get("timestep_spacing", "leading"),
        steps_offset=d.get("steps_offset", 0))


def scheduler_config_from_json(d: dict) -> Union[SchedulerConfig, DPMSolverConfig, UniPCConfig, PNDMConfig, DEISConfig,
                                                 DPMSingleConfig, DDPMConfig]:
    cls = d.get("_class_name", "DDIMScheduler")
    if cls == "DPMSolverMultistepScheduler":
        return dpm_solver_config_from_json(d)
    if cls == "UniPCMultistepScheduler":
        return unipc_config_from_json(d)
    if cls == "PNDMScheduler":
        return pndm_config_from_json(d)
    if cls == "DEISMultistepScheduler":
        return deis_config_from_json(d)
    if cls == "DPMSolverSinglestepScheduler":
        return dpm_single_config_from_json(d)
    if cls == "DDPMScheduler":
        return ddpm_config_from_json(d)
    if cls != "DDIMScheduler":
        raise NotImplementedError(
            f"scheduler {cls} is not fused on the CUDA path (DDIMScheduler, DDPMScheduler, DPMSolverMultistepScheduler, "
            "UniPCMultistepScheduler, PNDMScheduler, DEISMultistepScheduler and DPMSolverSinglestepScheduler only); run "
            "the reference's Python scheduler loop for other classes")
    if d.get("thresholding", False):
        raise NotImplementedError("dynamic thresholding is not supported")
    return SchedulerConfig(
        num_train_timesteps=d.get("num_train_timesteps", 1000), beta_start=d.get("beta_start", 0.0001),
        beta_end=d.get("beta_end", 0.02), beta_schedule=d.get("beta_schedule", "linear"),
        prediction_type=d.get("prediction_type", "epsilon"), set_alpha_to_one=d.get("set_alpha_to_one", True),
        steps_offset=d.get("steps_offset", 0), timestep_spacing=d.get("timestep_spacing", "leading"),
        clip_sample=d.get("clip_sample", True), clip_sample_range=d.get("clip_sample_range", 1.0))


class StockVAEAdapter:
    """``encode_latents`` / ``decode_latents`` over a stock diffusers ``AutoencoderKL`` with the reference's exact
    semantics: ``encode_vae`` / ``decode_vae`` (PIPE:47-72: batches of 8, ``latent_dist.sample() * scaling_factor``,
    ``decode(z / scaling_factor)``) and the ``output_type="pt"`` post-processing of ``post_process`` (PIPE:280-285:
    ``(x / 2 + 0.5).clamp(0, 1)``).  The VAE is SURVEY.md section 8f row 1 ("next"), not part of the CUDA hot path."""

    def __init__(self, vae, batch_size: int = 8):
        self.vae, self.batch_size = vae, batch_size

    def encode_latents(self, images):
        out = [self.vae.encode(x).latent_dist.sample() for x in images.split(self.batch_size)]
        return torch.cat(out, dim=0) * self.vae.config.scaling_factor

    def decode_latents(self, latents):
        sf = self.vae.config.scaling_factor
        out = [self.vae.decode(z / sf, return_dict=False)[0] for z in latents.split(self.batch_size)]
        return (torch.cat(out, dim=0) / 2 + 0.5).clamp(0, 1)


def default_vae_factory(model_dir: str, gpu_id: int):
    """Stock ``AutoencoderKL`` from ``model_dir/vae`` (what ``Diffuman4DPipeline.from_pretrained`` loads, SUTIL:45-47).
    Returns None (with a warning) when the checkpoint has no ``vae/`` or diffusers is not importable: the pipeline then
    accepts latents only and raises "no VAE attached" for image inputs."""
    if not os.path.isdir(os.path.join(model_dir, "vae")):
        return None
    try:
        from diffusers import AutoencoderKL
    except Exception as e:  # noqa: BLE001
        warnings.warn(f"{model_dir}/vae exists but diffusers is not importable ({e}); pipelines accept latents only")
        return None
    vae = AutoencoderKL.from_pretrained(os.path.join(model_dir, "vae"), torch_dtype=torch.bfloat16).to(f"cuda:{gpu_id}")
    return StockVAEAdapter(vae.eval())


def _resolve_factory(vae_factory: Union[None, str, Callable]) -> Callable:
    """``vae_factory``: None (default above), a callable ``(model_dir, gpu_id) -> vae`` or -- so that a Hydra yaml can
    name it -- a dotted path ``"package.module.function"`` to such a callable.  The returned ``vae`` object must offer
    ``encode_latents(images)`` and ``decode_latents(latents)``."""
    if vae_factory is None:
        return default_vae_factory
    if isinstance(vae_factory, str):
        mod, _, attr = vae_factory.rpartition(".")
        if not mod:
            raise ValueError(f"vae_factory must be a dotted path 'module.function', got {vae_factory!r}")
        vae_factory = getattr(importlib.import_module(mod), attr)
    if not callable(vae_factory):
        raise ValueError("vae_factory must be None, a dotted path or a callable (model_dir, gpu_id) -> vae")
    return vae_factory


def load_pipelines(repo_id: str = "krahets/Diffuman4D", model_dir: str = "./models/krahets-Diffuman4D",
                   torch_dtype: str = "bf16", gpu_ids: Optional[List[int]] = None,
                   vae_factory: Union[None, str, Callable] = None):
    """Same signature as the reference factory (+ ``vae_factory``, see ``_resolve_factory``); returns one
    ``B200Diffuman4DPipeline`` per GPU."""
    make_vae = _resolve_factory(vae_factory)
    if torch_dtype != "bf16":
        raise ValueError(f"Unsupported torch_dtype: {torch_dtype}. The B200 path supports 'bf16' only.")
    if gpu_ids is None:
        gpu_ids = list(range(torch.cuda.device_count()))
    if not os.path.isdir(os.path.join(model_dir, "unet")):
        try:  # mirror of sampling_utils.py:37-41
            from huggingface_hub import snapshot_download
            snapshot_download(repo_id, local_dir=model_dir, allow_patterns=["*.json", "*model.safetensors"])
        except Exception as e:  # noqa: BLE001
            raise FileNotFoundError(f"{model_dir}/unet not found and download of {repo_id} failed: {e}") from e
    with open(os.path.join(model_dir, "unet", "config.json")) as f:
        ucfg = unet_config_from_json(json.load(f))
    spath = os.path.join(model_dir, "scheduler", "scheduler_config.json")
    scfg = scheduler_config_from_json(json.load(open(spath))) if os.path.exists(spath) else SchedulerConfig()
    from safetensors.torch import load_file
    sd = load_file(os.path.join(model_dir, "unet", "diffusion_pytorch_model.safetensors"))
    pipelines = []
    for gpu_id in gpu_ids:
        unet = B200MultiviewUNet(ucfg, device=gpu_id).load_state_dict(sd)
        vae = make_vae(model_dir, gpu_id)
        pipelines.append(B200Diffuman4DPipeline(unet, scfg, vae=vae))
    return pipelines
