"""``B200Diffuman4DPipeline`` -- the denoise part of the reference's ``Diffuman4DPipeline`` on one H100.

Seams (SURVEY.md section 8b):
  B-3  ``denoise_window``  == ``Diffuman4DPipeline.__call__`` with latents given
       (reference src/diffusers/pipelines/diffuman4d/pipeline_diffuman4d.py:345-425): input assembly, UNet, CFG
       combine and the F per-frame scheduler steps run as ONE C-ABI call (no per-frame host sync).  The scheduler is DDIM
       (``SchedulerConfig``), DPM-Solver++ (``DPMSolverConfig``), UniPC (``UniPCConfig``), PNDM (``PNDMConfig``), DEIS
       (``DEISConfig``), DPM-Solver++ singlestep (``DPMSingleConfig``) or DDPM (``DDPMConfig``); the stateful ones keep a
       per-frame history on the device (``DPMSolverState`` / ``UniPCState`` / ``PNDMState`` / ``DEISState`` /
       ``DPMSingleState``) in place of the reference's per-frame scheduler copies, and DDPM's per-frame handles carry
       the task's noise seed and the frames' indices in the task (``DDPMTask``).
  B-4  ``sliding_iterative_denoise`` == PIPE:439-559: same arguments, same ValueErrors, same returned dict.  The VAE
       (stock AutoencoderKL, out of scope per SURVEY section 8f) is pluggable: pass ``vae`` with ``encode_latents(x)`` /
       ``decode_latents(z)`` callables, or feed latents directly (``pixel_values_latents=...``).

Host code here is window scheduling only (index arithmetic mirroring PIPE:503-518); all tensor arithmetic is in
libd4d.so.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, List, Optional, Union

import torch

from ._lib import check, lib
from .config import DDPMConfig, DEISConfig, DPMSingleConfig, DPMSolverConfig, PNDMConfig, SchedulerConfig, UniPCConfig
from .scheduler import (DDIMTables, DDPMFrames, DDPMTables, DEISTables, DPMSingleTables, DPMSolverFrame, DPMSolverTables,
                        PNDMTables, SolverState, UniPCTables, draw_seed)
from .unet import _DOMAIN_IDS, B200MultiviewUNet


def _check_inplace(t, name: str, dtype: torch.dtype):
    """Raw pointers of tensors the library updates in place cross the C ABI: they must be contiguous CUDA tensors of
    ``dtype`` (a copy would not receive the update)."""
    if not (torch.is_tensor(t) and t.is_cuda and t.dtype == dtype and t.is_contiguous()):
        raise ValueError(f"{name} must be a contiguous CUDA {str(dtype).replace('torch.', '')} tensor (updated in place)")


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
    def __init__(self, unet: B200MultiviewUNet,
                 scheduler_config: Union[SchedulerConfig, DPMSolverConfig, UniPCConfig, PNDMConfig, DEISConfig,
                                         DPMSingleConfig, DDPMConfig, None] = None,
                 vae=None, emulate_bf16_scheduler: bool = False):
        self.unet = unet
        self.vae = vae
        self.device = unet.device
        self.dtype = torch.bfloat16
        if isinstance(scheduler_config, DPMSolverConfig):
            self.scheduler = DPMSolverTables(scheduler_config, device=self.device)
        elif isinstance(scheduler_config, UniPCConfig):
            self.scheduler = UniPCTables(scheduler_config, device=self.device)
        elif isinstance(scheduler_config, PNDMConfig):
            self.scheduler = PNDMTables(scheduler_config, device=self.device)
        elif isinstance(scheduler_config, DEISConfig):
            self.scheduler = DEISTables(scheduler_config, device=self.device)
        elif isinstance(scheduler_config, DPMSingleConfig):
            self.scheduler = DPMSingleTables(scheduler_config, device=self.device)
        elif isinstance(scheduler_config, DDPMConfig):
            self.scheduler = DDPMTables(scheduler_config, device=self.device)
        else:
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
        return self.has_cfg_halves(self._guidance_scale)

    def has_cfg_halves(self, guidance_scale) -> bool:
        """Whether a window step at ``guidance_scale`` runs the UNet on two CFG halves (otherwise on the F frames once)."""
        return guidance_scale > 1 and self.unet.config.time_cond_proj_dim is None

    @property
    def _multistep(self) -> bool:
        return self.scheduler.state_planes is not None

    @property
    def _ddpm(self) -> bool:
        return isinstance(self.scheduler, DDPMTables)

    @property
    def _per_frame(self) -> bool:
        """Whether ``parepare_schedulers`` hands out per-frame handles (a multistep solver or DDPM)."""
        return self._multistep or self._ddpm

    def parepare_schedulers(self, num_inference_steps: int, num_frames: int):
        """PIPE:265-271.  The per-frame deep copies exist in the reference only because scheduler objects are
        stateful; DDIM is stateless, so one table serves all frames.  DPM-Solver++ (multistep and singlestep), UniPC,
        PNDM and DEIS get a fresh (zeroed) device state for the frames, and one ``DPMSolverFrame`` handle per frame in
        place of each copy.  DDPM's handles belong to a fresh ``DDPMTask``, whose noise seed is drawn when the task first
        runs (``__call__`` or the sliding loop)."""
        ts = self.scheduler.set_timesteps(num_inference_steps)
        if self._per_frame:
            return self.scheduler.new_state(num_frames).frames(), ts
        return [self.scheduler] * num_frames, ts

    # B-3 -----------------------------------------------------------------------------------------------
    def denoise_window(self, *, latents, pixel_values_latents, plucker_embeds_latents, skeletons_latents,
                       cond_masks_latents, timestep_indices, domain: str, guidance_scale: float,
                       num_inference_steps: int = 1, solver_state: Optional[SolverState] = None):
        """One window: ``num_inference_steps`` x (assemble -> UNet -> CFG -> per-frame scheduler step).  ``latents``
        [F,4,h,w] and ``timestep_indices`` [F] (int64, device) are updated IN PLACE and returned.  With DPM-Solver++,
        UniPC, PNDM, DEIS or DPM-Solver++ singlestep, ``solver_state`` is the window frames' ``DPMSolverState`` /
        ``UniPCState`` / ``PNDMState`` / ``DEISState`` / ``DPMSingleState`` (``take``), also updated in place.  With
        DDPM it is the window's ``DDPMFrames`` (``DDPMTask.take``): the task's noise seed and the frames' task indices."""
        return self._window_step(latents=latents, pixel_values_latents=pixel_values_latents,
                                 plucker_embeds_latents=plucker_embeds_latents, skeletons_latents=skeletons_latents,
                                 cond_masks_latents=cond_masks_latents, timestep_indices=timestep_indices, domain=domain,
                                 guidance_scale=guidance_scale, num_inference_steps=num_inference_steps,
                                 solver_state=solver_state)

    def _window_step(self, *, latents, pixel_values_latents, plucker_embeds_latents, skeletons_latents,
                     cond_masks_latents, timestep_indices, domain: str, guidance_scale: float,
                     num_inference_steps: int = 1, solver_state: Optional[SolverState] = None,
                     F_total: Optional[int] = None, cfg_split: bool = False, cfg_grid: bool = False):
        """``denoise_window``'s checks and library call.  ``F_total`` given: the tensors hold this rank's frames of a
        frame-sharded window of ``F_total`` frames (``FrameShardedPipeline.denoise_window``).  ``cfg_split``: the whole
        window, with this rank running the UNet on its CFG half (``CFGSplitPipeline.denoise_window``).  ``cfg_grid``: the
        whole window, with this rank running the UNet on its frame shard of its CFG half
        (``CFGGridPipeline.denoise_window``)."""
        if cfg_grid:
            name = self.scheduler.window_entry_points[0] + "_cfg_grid"
        else:
            name = self.scheduler.window_entry_points[2 if cfg_split else F_total is not None]
        if name is None:
            raise NotImplementedError(f"the frame-sharded window does not run the {self.scheduler.name} scheduler")
        if domain not in _DOMAIN_IDS:
            raise ValueError(f"Invalid domain for temporal embedding: {domain}")
        dev = self.device

        def prep(t, name):
            if t is None:
                raise ValueError(f"{name} is required")
            t = t.to(device=dev, dtype=torch.bfloat16)
            return t if t.is_contiguous() else t.contiguous()

        _check_inplace(latents, "latents", torch.bfloat16)
        _check_inplace(timestep_indices, "timestep_indices", torch.int64)
        F_, _, h, w = latents.shape
        pix = prep(pixel_values_latents, "pixel_values_latents")
        plk = prep(plucker_embeds_latents, "plucker_embeds_latents")
        skl = prep(skeletons_latents, "skeletons")
        msk = prep(cond_masks_latents, "cond_masks_latents")
        extra = []
        if self._ddpm:   # the noise seed in the table struct, the frames' task indices after num_inference_steps
            st = solver_state
            if not isinstance(st, DDPMFrames):
                raise ValueError("the DDPM scheduler needs the window's DDPMFrames as solver_state")
            ids = st.frame_ids
            if not (ids.is_cuda and ids.dtype == torch.int64 and ids.is_contiguous() and ids.numel() == F_):
                raise ValueError("solver_state.frame_ids must be a contiguous CUDA int64 [F] tensor")
            sched = self.scheduler.c_struct(self.emulate_bf16_scheduler, st.seed)
            extra.append(ids.data_ptr())
        else:
            sched = self.scheduler.c_struct(self.emulate_bf16_scheduler)
        self._guidance_scale = guidance_scale
        g = guidance_scale if self.do_classifier_free_guidance else 1.0
        frames = (F_,) if F_total is None else (F_, F_total)
        args = [self.unet._h, latents.data_ptr(), pix.data_ptr(), plk.data_ptr(), skl.data_ptr(), msk.data_ptr(),
                timestep_indices.data_ptr(), C.byref(sched), float(g), _DOMAIN_IDS[domain], *frames, h, w,
                int(num_inference_steps), *extra]
        if self._multistep:   # the state planes in ABI order (None: passed as NULL), then lower_order_nums
            st = solver_state
            if st is None:
                raise ValueError(f"the {self.scheduler.name} scheduler needs the window frames' solver_state")

            def state_plane(plane):
                t = getattr(st, plane, None)
                if not (t is not None and t.is_cuda and t.dtype == torch.bfloat16 and t.is_contiguous()
                        and t.shape == latents.shape):
                    raise ValueError(f"solver_state.{plane} must be a contiguous CUDA bfloat16 tensor shaped like latents")
                return t.data_ptr()

            args += [None if plane is None else state_plane(plane) for plane in self.scheduler.state_planes]
            lon = st.lower_order_nums
            if not (lon.is_cuda and lon.dtype == torch.int32 and lon.is_contiguous() and lon.numel() == F_):
                raise ValueError("solver_state.lower_order_nums must be a contiguous CUDA int32 [F] tensor")
            args.append(lon.data_ptr())
        with torch.cuda.device(dev):
            check(getattr(lib(), name)(*args, torch.cuda.current_stream().cuda_stream), name)
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
            schedulers, _ = self.parepare_schedulers(num_inference_steps, F_)
            timestep_indices = torch.zeros(F_)
        if latents is None:        # PIPE:172-183 prepare_latents: draw the initial noise
            latents = torch.randn(tuple(pixel_values_latents.shape), generator=unused.get("generator"), device=self.device,
                                  dtype=torch.bfloat16)
        lat = (latents * self.scheduler.init_noise_sigma).to(device=self.device, dtype=torch.bfloat16).contiguous().clone()
        ti = timestep_indices.to(device=self.device, dtype=torch.int64).contiguous().clone()
        task, frames, window_state = None, None, None
        if self._per_frame:   # the frames' solver history or task indices travel with the `schedulers` handles
            if len(schedulers) != F_ or not all(isinstance(s, DPMSolverFrame) for s in schedulers):
                raise ValueError("schedulers must be the per-frame handles of parepare_schedulers, one per frame")
            task = schedulers[0].state
            if any(s.state is not task for s in schedulers):
                raise ValueError("schedulers must all come from one parepare_schedulers call")
            frames = torch.tensor([s.index for s in schedulers], dtype=torch.int64)
            if self._ddpm and task.seed is None:
                task.seed = int(draw_seed(unused.get("generator"), self.device).item())
            window_state = task.take(frames, *lat.shape[2:])
        self.denoise_window(latents=lat, pixel_values_latents=pixel_values_latents,
                            plucker_embeds_latents=plucker_embeds_latents, skeletons_latents=skeletons_latents,
                            cond_masks_latents=cond_masks_latents, timestep_indices=ti, domain=domains[0],
                            guidance_scale=guidance_scale, num_inference_steps=num_inference_steps,
                            solver_state=window_state)
        if task is not None:
            task.put(frames, window_state)
        return lat

    # B-4 -------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def sliding_iterative_denoise(self, pixel_values=None, plucker_embeds=None, skeletons=None, cond_masks=None,
                                  latents=None, domain: str = "spatial", timestep_indices=None, window_size: int = 12,
                                  sliding_stride: int = 1, sliding_shift: int = 0, bidirectional: bool = True,
                                  num_denoising_steps: int = 1, alternation_rounds: int = 3, guidance_scale: float = 2.0,
                                  tqdm: Callable = None, pixel_values_latents=None, skeletons_latents=None,
                                  generator=None):
        return self._sliding(self._task_window, pixel_values=pixel_values, plucker_embeds=plucker_embeds,
                             skeletons=skeletons, cond_masks=cond_masks, latents=latents, domain=domain,
                             timestep_indices=timestep_indices, window_size=window_size, sliding_stride=sliding_stride,
                             sliding_shift=sliding_shift, bidirectional=bidirectional,
                             num_denoising_steps=num_denoising_steps, alternation_rounds=alternation_rounds,
                             guidance_scale=guidance_scale, tqdm=tqdm, pixel_values_latents=pixel_values_latents,
                             skeletons_latents=skeletons_latents, generator=generator)

    def _task_window(self, window, lw, tiw, sw, conds, **kw):
        """One window of the sliding loop: ``lw`` / ``tiw`` / ``sw`` (the window frames' latents, timestep indices and
        solver state) are updated in place; ``conds`` are the task's conditioning tensors, indexed by ``window``."""
        pix, plk, skl, msk = (t[window] for t in conds)
        self.denoise_window(latents=lw, pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skl,
                            cond_masks_latents=msk, timestep_indices=tiw, solver_state=sw, **kw)
        return lw, sw

    def _sliding(self, window_step: Callable, *, pixel_values, plucker_embeds, skeletons, cond_masks, latents, domain,
                 timestep_indices, window_size, sliding_stride, sliding_shift, bidirectional, num_denoising_steps,
                 alternation_rounds, guidance_scale, tqdm, pixel_values_latents, skeletons_latents, generator,
                 share_noise: Optional[Callable] = None):
        """The B-4 loop around ``window_step(window, lw, tiw, sw, conds, ...) -> (lw, sw)``, which returns the window's
        updated latents and solver state (``FrameShardedPipeline`` runs it on a frame shard).  ``share_noise`` is applied
        to freshly drawn initial noise and, with DDPM, to every task's noise seed."""
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
            if share_noise is not None:
                share_noise(latents)
        latents = (latents.to(dev, torch.bfloat16) * self.scheduler.init_noise_sigma).contiguous().clone()

        schedulers, _ = self.parepare_schedulers(num_inference_steps, n)   # a fresh solver state per task (PIPE:501)
        task = schedulers[0].state if self._per_frame else None
        if self._ddpm:   # the task's noise seed, drawn after the initial noise; rank 0's on every rank
            seed = draw_seed(generator, dev)
            if share_noise is not None:
                share_noise(seed)
            task.seed = int(seed.item())
        target_windows, input_windows = build_windows(target_indices, input_indices, domain, window_size,
                                                      sliding_stride, sliding_shift, bidirectional)
        it = zip(target_windows, input_windows)
        if tqdm is not None:
            it = tqdm(it, total=len(target_windows))
        conds = (pixel_values_latents, plk, skl, msk)
        for tw, iw in it:
            window = torch.cat([iw, tw])
            lw = latents[window].contiguous()
            tiw = timestep_indices[window].contiguous()
            sw = task.take(window, h, w) if task is not None else None
            lw, sw = window_step(window, lw, tiw, sw, conds, domain=domain, guidance_scale=guidance_scale,
                                 num_inference_steps=num_denoising_steps)
            if task is not None:
                task.put(window, sw)
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
