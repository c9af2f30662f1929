"""``B200Diffuman4DPipeline`` -- the denoise part of the reference's ``Diffuman4DPipeline`` on one H100.

Seams (SURVEY.md section 8b):
  B-3  ``denoise_window``  == ``Diffuman4DPipeline.__call__`` with latents given
       (reference src/diffusers/pipelines/diffuman4d/pipeline_diffuman4d.py:345-425): input assembly, UNet, CFG
       combine and the F per-frame scheduler steps run as ONE C-ABI call (no per-frame host sync).
  B-4  ``sliding_iterative_denoise`` == PIPE:439-559: same arguments, same ValueErrors, same returned dict.  The VAE
       (stock AutoencoderKL, out of scope per SURVEY section 8f) is pluggable: pass ``vae`` with ``encode_latents(x)`` /
       ``decode_latents(z)`` callables, or feed latents directly (``pixel_values_latents=...``).

Host code here is window scheduling only (index arithmetic mirroring PIPE:503-518); all tensor arithmetic is in
libd4d.so.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, List, Optional

import torch

from ._lib import check, lib
from .config import SchedulerConfig
from .scheduler import DDIMTables
from .unet import B200MultiviewUNet

_DOMAIN_IDS = {"spatial": 0, "temporal": 1}


def build_windows(target_indices: torch.Tensor, input_indices: torch.Tensor, domain: str, window_size: int,
                  sliding_stride: int, sliding_shift: int = 0, bidirectional: bool = False):
    """Window index lists of PIPE:503-518 (pure index arithmetic)."""
    target_windows, input_windows = [], []
    directions = (-1, 1) if bidirectional else (-1,)
    for direction in directions:
        for shift in range(sliding_shift, sliding_shift + len(target_indices), sliding_stride):
            tw = target_indices.roll(shifts=shift * direction)[:window_size]
            target_windows.append(tw)
            if domain == "spatial":
                input_windows.append(input_indices)
            elif domain == "temporal":
                input_windows.append(tw - len(input_indices))
            else:
                raise ValueError(f"Invalid domain: {domain}")
    return target_windows, input_windows


def resize_conditions(plucker_embeds: torch.Tensor, cond_masks: torch.Tensor, h: int, w: int, dtype: torch.dtype):
    """Latent-resolution conditioning maps on whatever device the inputs live on (PIPE:90-100, 215-226): Pluecker channels
    bilinearly, masks with nearest; both resizes run in the SOURCE dtype and are cast afterwards, like the reference."""
    plk, msk = plucker_embeds, cond_masks
    if plk.shape[-2:] != (h, w):
        plk = torch.nn.functional.interpolate(plk, size=(h, w), mode="bilinear")
    if msk.shape[-2:] != (h, w):
        msk = torch.nn.functional.interpolate(msk, size=(h, w), mode="nearest")
    return plk.to(dtype), msk.to(dtype)


class B200Diffuman4DPipeline:
    def __init__(self, unet: B200MultiviewUNet, scheduler_config: Optional[SchedulerConfig] = None, vae=None,
                 emulate_bf16_scheduler: bool = False):
        self.unet = unet
        self.vae = vae
        self.device = unet.device
        self.dtype = torch.bfloat16
        self.scheduler = DDIMTables(scheduler_config, device=self.device)
        self.emulate_bf16_scheduler = emulate_bf16_scheduler
        self._guidance_scale = 1.0

    # reference surface ------------------------------------------------------------------------------
    def to(self, *a, **k):
        return self

    def set_progress_bar_config(self, **kwargs):
        return None

    @property
    def guidance_scale(self):
        return self._guidance_scale

    @property
    def do_classifier_free_guidance(self):
        return self._guidance_scale > 1 and self.unet.config.time_cond_proj_dim is None

    def parepare_schedulers(self, num_inference_steps: int, num_frames: int):
        """PIPE:265-271.  The per-frame deep copies exist in the reference only because scheduler objects are
        stateful; DDIM is stateless, so one table serves all frames."""
        ts = self.scheduler.set_timesteps(num_inference_steps)
        return [self.scheduler] * num_frames, ts

    # B-3 -----------------------------------------------------------------------------------------------
    def denoise_window(self, *, latents, pixel_values_latents, plucker_embeds_latents, skeletons_latents,
                       cond_masks_latents, timestep_indices, domain: str, guidance_scale: float,
                       num_inference_steps: int = 1):
        """One window: ``num_inference_steps`` x (assemble -> UNet -> CFG -> per-frame DDIM).  ``latents`` [F,4,h,w] and
        ``timestep_indices`` [F] (int64, device) are updated IN PLACE and returned."""
        if domain not in _DOMAIN_IDS:
            raise ValueError(f"Invalid domain for temporal embedding: {domain}")
        F_, _, h, w = latents.shape
        dev = self.device

        def prep(t, name):
            if t is None:
                raise ValueError(f"{name} is required")
            t = t.to(device=dev, dtype=torch.bfloat16)
            return t if t.is_contiguous() else t.contiguous()

        if not (latents.is_cuda and latents.dtype == torch.bfloat16 and latents.is_contiguous()):
            raise ValueError("latents must be a contiguous CUDA bfloat16 tensor (updated in place)")
        if not (timestep_indices.is_cuda and timestep_indices.dtype == torch.int64 and timestep_indices.is_contiguous()):
            raise ValueError("timestep_indices must be a contiguous CUDA int64 tensor (updated in place)")
        pix = prep(pixel_values_latents, "pixel_values_latents")
        plk = prep(plucker_embeds_latents, "plucker_embeds_latents")
        skl = prep(skeletons_latents, "skeletons")
        msk = prep(cond_masks_latents, "cond_masks_latents")
        sched = self.scheduler.c_struct(self.emulate_bf16_scheduler)
        self._guidance_scale = guidance_scale
        g = guidance_scale if self.do_classifier_free_guidance else 1.0
        with torch.cuda.device(dev):
            check(lib().d4d_denoise_window(self.unet._h, latents.data_ptr(), pix.data_ptr(), plk.data_ptr(),
                                           skl.data_ptr(), msk.data_ptr(), timestep_indices.data_ptr(), C.byref(sched),
                                           float(g), _DOMAIN_IDS[domain], F_, h, w, int(num_inference_steps),
                                           torch.cuda.current_stream().cuda_stream), "d4d_denoise_window")
        return latents, timestep_indices

    # Diffuman4DPipeline.__call__ with latents given (PIPE:289-437) ----------------------------------------
    @torch.no_grad()
    def __call__(self, pixel_values_latents=None, plucker_embeds_latents=None, skeletons_latents=None,
                 cond_masks_latents=None, latents=None, domains: List[str] = None, num_inference_steps: int = 1,
                 schedulers=None, timesteps=None, timestep_indices=None, guidance_scale: float = 1.0,
                 output_type: str = "latent", **unused):
        if output_type != "latent":
            raise ValueError("only output_type='latent' is on the CUDA path (VAE decode is out of scope)")
        if domains is None or len(domains) != 1:
            raise ValueError("domains must be a one-element list, e.g. ['spatial']")
        F_ = pixel_values_latents.shape[0]
        if schedulers is None:
            self.parepare_schedulers(num_inference_steps, F_)
            timestep_indices = torch.zeros(F_)
        if latents is None:        # PIPE:172-183 prepare_latents: draw the initial noise
            latents = torch.randn(tuple(pixel_values_latents.shape), generator=unused.get("generator"), device=self.device,
                                  dtype=torch.bfloat16)
        lat = (latents * self.scheduler.init_noise_sigma).to(device=self.device, dtype=torch.bfloat16).contiguous().clone()
        ti = timestep_indices.to(device=self.device, dtype=torch.int64).contiguous().clone()
        self.denoise_window(latents=lat, pixel_values_latents=pixel_values_latents,
                            plucker_embeds_latents=plucker_embeds_latents, skeletons_latents=skeletons_latents,
                            cond_masks_latents=cond_masks_latents, timestep_indices=ti, domain=domains[0],
                            guidance_scale=guidance_scale, num_inference_steps=num_inference_steps)
        return lat

    # B-4 -------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def sliding_iterative_denoise(self, pixel_values=None, plucker_embeds=None, skeletons=None, cond_masks=None,
                                  latents=None, domain: str = "spatial", timestep_indices=None, window_size: int = 12,
                                  sliding_stride: int = 1, sliding_shift: int = 0, bidirectional: bool = True,
                                  num_denoising_steps: int = 1, alternation_rounds: int = 3, guidance_scale: float = 2.0,
                                  tqdm: Callable = None, pixel_values_latents=None, skeletons_latents=None,
                                  generator=None):
        dev = self.device
        if (window_size * num_denoising_steps) % sliding_stride != 0:
            raise ValueError(
                f"The window size ({window_size}) * num denoising steps ({num_denoising_steps}) "
                f"should be divisible by the sliding stride ({sliding_stride})")
        per_alt = window_size * num_denoising_steps // sliding_stride
        if bidirectional:
            per_alt *= 2
        num_inference_steps = per_alt * alternation_rounds

        timestep_indices = timestep_indices.to(device=dev, dtype=torch.int64).clone()
        flag = cond_masks[:, 0, 0, 0].to(dev)
        target_indices = torch.where(flag != 0.0)[0]
        input_indices = torch.where(flag == 0.0)[0]
        tgt_ti = timestep_indices[target_indices]
        inp_ti = timestep_indices[input_indices]
        timestep_id_end = tgt_ti[0].item() + per_alt
        if (tgt_ti != tgt_ti[0]).any():
            raise ValueError(
                f"The timestep indices should be the same for all target samples, timestep_indices = {timestep_indices}")
        if (inp_ti != 0).any():
            raise ValueError(
                f"The timestep indices should be 0 for all input samples, timestep_indices = {timestep_indices}")

        # ---- latent preparation (PIPE:193-263: prepare_all_latents).  Resizes run in the SOURCE dtype and are cast
        # afterwards, like the reference's encode_image_resizing (PIPE:90-100) ----
        if pixel_values_latents is None:
            if self.vae is None:
                raise ValueError("no VAE attached: pass pixel_values_latents (and skeletons_latents) instead of images")
            pixel_values_latents = self.vae.encode_latents(pixel_values.to(dev, torch.bfloat16))
        pixel_values_latents = pixel_values_latents.to(dev, torch.bfloat16)
        n, _, h, w = pixel_values_latents.shape
        plk, msk = resize_conditions(plucker_embeds.to(dev), cond_masks.to(dev), h, w, torch.bfloat16)
        if skeletons_latents is not None:                      # same precedence as PIPE:228-241
            skl = skeletons_latents.to(dev, torch.bfloat16)
        elif self.unet.config.enable_pose_encoder:
            skl = skeletons.to(dev, torch.bfloat16)
        else:
            if self.vae is None:
                raise ValueError("no VAE attached: pass skeletons_latents")
            skl = self.vae.encode_latents(skeletons.to(dev, torch.bfloat16))
        if latents is None:
            latents = torch.randn(n, 4, h, w, generator=generator, device=dev, dtype=torch.bfloat16)
        latents = (latents.to(dev, torch.bfloat16) * self.scheduler.init_noise_sigma).contiguous().clone()

        self.parepare_schedulers(num_inference_steps, n)
        target_windows, input_windows = build_windows(target_indices, input_indices, domain, window_size,
                                                      sliding_stride, sliding_shift, bidirectional)
        it = zip(target_windows, input_windows)
        if tqdm is not None:
            it = tqdm(it, total=len(target_windows))
        for tw, iw in it:
            window = torch.cat([iw, tw])
            lw = latents[window].contiguous()
            tiw = timestep_indices[window].contiguous()
            self.denoise_window(latents=lw, pixel_values_latents=pixel_values_latents[window],
                                plucker_embeds_latents=plk[window], skeletons_latents=skl[window],
                                cond_masks_latents=msk[window], timestep_indices=tiw, domain=domain,
                                guidance_scale=guidance_scale, num_inference_steps=num_denoising_steps)
            timestep_indices[tw] += num_denoising_steps
            latents[window] = lw

        if (timestep_indices[target_indices] != timestep_id_end).any():
            raise ValueError(
                f"The denoised timesteps of target samples mismatch the config, timestep_indices = {timestep_indices}")
        if (timestep_indices[input_indices] != 0).any():
            raise ValueError(f"Timesteps of input samples have changed, timestep_indices = {timestep_indices}")
        images = self.vae.decode_latents(latents) if self.vae is not None else None
        return {"images": images, "latents": latents, "timestep_indices": timestep_indices,
                "fully_denoised": timestep_indices == num_inference_steps}
