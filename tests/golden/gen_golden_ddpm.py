"""Generate tests/golden/pipeline_ddpm_ref.pt by RUNNING the reference pipeline code with a DDPM scheduler (only possible
in a container that has a checkout of the reference; the tests never read it, so the output is committed).

  pipeline_ddpm_ref.pt -- the reference ``Diffuman4DPipeline.__call__`` (PIPE:345-425) and ``sliding_iterative_denoise``
                          (PIPE:439-559) on the stubs of tests/golden/gen_golden.py, with a DDPMScheduler
                          (``oracle.ddpm_oracle.DDPMOracle`` behind the upstream ``set_timesteps`` / ``scale_model_input``
                          / ``step`` surface) whose noise is the device's counter-based noise keyed by frame: the k-th
                          deep copy of PIPE:269 is frame k of the task.  Pins what the per-frame copies see through the
                          reference -- which frame each copy steps, that conditioning frames are never stepped and draw
                          nothing, the timestep each frame steps at and its index advance -- not the step arithmetic.

Run:  DIFFUMAN4D_REFERENCE=<reference checkout> python tests/golden/gen_golden_ddpm.py      (from the repo root)
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_golden import _load_ref_pipeline, save_sharded  # noqa: E402


def gen_pipeline_ddpm():
    from diffuman4d_b200.config import DDPMConfig
    from oracle.ddpm_oracle import DDPMOracle
    pipe_mod, make_pipe = _load_ref_pipeline()

    class RefDDPM(DDPMOracle):
        """the upstream scheduler surface the reference touches (PIPE:265-271,376,420)"""

        def set_timesteps(self, n, device=None):
            super().set_timesteps(n)

        def scale_model_input(self, x, t):
            return x

        def step(self, noise, t, latent, return_dict=False):
            return (super().step(noise, int(t), latent),)

    def make_ddpm_pipe(cfg, seed):
        pipe, cin = make_pipe(True)
        pipe.scheduler = RefDDPM(cfg, seed=seed)   # what register_modules(scheduler=...) stores (PIPE:138)
        return pipe

    out = {"cases": {}}
    h = w = 4
    g = torch.Generator().manual_seed(2031)
    rn = lambda *s: torch.randn(*s, generator=g)
    skel = lambda n: (torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16)

    # ---- one window through __call__ at staggered timestep indices, reaching the last row (t = 0: no noise)
    for tag, guidance, ckw in (("call_cfg_eps", 2.0, dict()),
                               ("call_nocfg_v_large", 1.0, dict(prediction_type="v_prediction",
                                                                variance_type="fixed_large", clip_sample=False))):
        cfg = DDPMConfig(**ckw)
        pipe = make_ddpm_pipe(cfg, seed=77)
        F_ = 5
        mask = torch.ones(F_, 1, h, w)
        mask[:2] = 0
        inp = {"latents": rn(F_, 4, h, w), "pixel_latents": rn(F_, 4, h, w), "plucker": rn(F_, 6, h, w).clamp(-1, 1),
               "skeletons": skel(F_), "cond_mask": mask, "timestep_indices": torch.tensor([0, 0, 1, 4, 7])}
        schedulers, timesteps = pipe.parepare_schedulers(10, F_)
        ti = inp["timestep_indices"].clone()
        res = pipe(pixel_values_latents=inp["pixel_latents"].clone(), plucker_embeds_latents=inp["plucker"].clone(),
                   skeletons_latents=inp["skeletons"].float(), cond_masks_latents=inp["cond_mask"].clone(),
                   latents=inp["latents"].clone(), domains=["spatial"], num_inference_steps=3, schedulers=schedulers,
                   timesteps=timesteps, timestep_indices=ti, guidance_scale=guidance, output_type="latent")
        out["cases"][tag] = {"config": vars(cfg), "seed": 77, "guidance": guidance, "n_steps_table": 10,
                             "num_inference_steps": 3, "in": inp, "timesteps_table": timesteps.clone(),
                             "out_latents": res, "out_timestep_indices": ti}
        print("pipeline_ddpm", tag, float(res.abs().mean()), ti.tolist())

    # ---- sliding_iterative_denoise: two tasks on one pipeline object (the copies and their frame count reset per call)
    cases = (("slide_spatial_eps_cfg", "spatial", 2, 4, 2, 1, True, 1, 2.0, dict()),
             ("slide_temporal_bidir_v_nocfg", "temporal", 3, 3, 2, 1, True, 1, 1.0,
              dict(prediction_type="v_prediction", variance_type="fixed_small_log", timestep_spacing="trailing")))
    for tag, domain, n_in, n_tg, ws, stride, bidir, rounds, guidance, ckw in cases:
        cfg = DDPMConfig(**ckw)
        pipe = make_ddpm_pipe(cfg, seed=123456789)
        n = n_in + n_tg
        tasks = []
        for _ in range(2):
            mask = torch.ones(n, 1, 8 * h, 8 * w)
            mask[:n_in] = 0
            pixel = torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1
            inp = {"pixel_values": pixel, "plucker": rn(n, 6, h, w).clamp(-1, 1), "skeletons": skel(n),
                   "cond_masks": mask, "latents": rn(n, 4, h, w), "timestep_indices": torch.zeros(n, dtype=torch.int64)}
            res = pipe.sliding_iterative_denoise(
                pixel_values=inp["pixel_values"].clone(), plucker_embeds=inp["plucker"].clone(),
                skeletons=inp["skeletons"].float(), cond_masks=inp["cond_masks"].clone(), latents=inp["latents"].clone(),
                domain=domain, timestep_indices=inp["timestep_indices"].clone(), window_size=ws, sliding_stride=stride,
                sliding_shift=0, bidirectional=bidir, num_denoising_steps=1, alternation_rounds=rounds,
                guidance_scale=guidance, tqdm=lambda it, total=None: it)
            z = torch.nn.functional.avg_pool2d(pixel, 8)
            inp["pixel_latents"] = torch.cat([z, z.mean(dim=1, keepdim=True)], dim=1)  # what the fake VAE encoded
            inp["cond_mask_latents"] = torch.nn.functional.interpolate(mask, size=(h, w), mode="nearest")
            del inp["pixel_values"], inp["cond_masks"]
            tasks.append({"in": inp, "window_size": ws, "out_latents": res["latents"],
                          "out_timestep_indices": res["timestep_indices"], "fully_denoised": res["fully_denoised"]})
            print("pipeline_ddpm", tag, float(res["latents"].abs().mean()), res["timestep_indices"].tolist())
        out["cases"][tag] = {"config": vars(cfg), "seed": 123456789, "domain": domain, "sliding_stride": stride,
                             "bidirectional": bidir, "alternation_rounds": rounds, "guidance": guidance, "tasks": tasks}
    save_sharded(out, "pipeline_ddpm_ref")


if __name__ == "__main__":
    gen_pipeline_ddpm()
