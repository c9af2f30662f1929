"""Generate tests/golden/pipeline_dpm_single_ref.pt by RUNNING the reference pipeline code with a stateful DPM-Solver++
singlestep scheduler (only possible in a container that has a checkout of the reference; the tests never read it, so the
output is committed).

  pipeline_dpm_single_ref.pt -- the reference ``Diffuman4DPipeline.__call__`` (PIPE:345-425) and
                        ``sliding_iterative_denoise`` (PIPE:439-559) on the stubs of tests/golden/gen_golden.py, with a
                        DPMSolverSinglestepScheduler (our ``oracle.dpm_single_oracle.DPMSingleOracle`` behind the upstream
                        ``set_timesteps`` / ``scale_model_input`` / ``step`` surface).  Pins what a STATEFUL scheduler sees
                        through the reference -- one deep copy per frame (PIPE:265-271), the copies of a window's frames
                        handed to ``__call__`` (PIPE:535), a fresh set per ``sliding_iterative_denoise`` call (PIPE:501), a
                        frame's step index starting from its first timestep whatever that index is (so that its first
                        steps run below the row's order), and the ``lower_order_final`` switch that ``set_timesteps``
                        leaves on the pipeline's scheduler for its later calls -- not the solver arithmetic itself.

Run:  DIFFUMAN4D_REFERENCE=<reference checkout> python tests/golden/gen_golden_dpm_single.py      (from the repo root)
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_golden import _load_ref_pipeline, save_sharded  # noqa: E402

SCALED_LINEAR = dict(beta_schedule="scaled_linear", beta_start=0.00085, beta_end=0.012)


def gen_pipeline_dpm_single():
    """The reference pipeline with a per-frame deep-copyable singlestep scheduler; see the module docstring."""
    from diffuman4d_b200.config import DPMSingleConfig
    from oracle.dpm_single_oracle import DPMSingleOracle
    pipe_mod, make_pipe = _load_ref_pipeline()

    def make_single_pipe(cfg):
        pipe, cin = make_pipe(True)
        pipe.scheduler = RefDPMSingle(cfg)      # what register_modules(scheduler=...) stores (PIPE:138)
        return pipe, cin

    class RefDPMSingle(DPMSingleOracle):
        """the upstream scheduler surface the reference touches (PIPE:265-271,376,420)"""

        def set_timesteps(self, n, device=None):
            super().set_timesteps(n)

        def scale_model_input(self, x, t):
            return x

        def step(self, noise, t, latent, return_dict=False):
            return (super().step(noise, int(t), latent),)

    out = {"cases": {}}
    h = w = 4
    g = torch.Generator().manual_seed(2029)
    rn = lambda *s: torch.randn(*s, generator=g)
    # skeleton images are most of the fixture: stored as bf16, and the reference runs on those values widened to fp32
    skel = lambda n: (torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16)

    # ---- one window through __call__: fresh per-frame copies at staggered (nonzero) timestep indices, 5 inference
    # steps of a 10-step table, so that frames start on second- and third-order rows and run them at a lower order
    for tag, guidance, ckw in (("call_cfg_eps_order3", 2.0, dict(solver_order=3)),
                               ("call_nocfg_v_order2_sigma_min", 1.0, dict(prediction_type="v_prediction",
                                                                           final_sigmas_type="sigma_min"))):
        cfg = DPMSingleConfig(**ckw)
        pipe, cin = make_single_pipe(cfg)
        F_ = 5
        mask = torch.ones(F_, 1, h, w)
        mask[:2] = 0
        inp = {"latents": rn(F_, 4, h, w), "pixel_latents": rn(F_, 4, h, w), "plucker": rn(F_, 6, h, w).clamp(-1, 1),
               "skeletons": skel(F_), "cond_mask": mask,
               "timestep_indices": torch.tensor([0, 0, 1, 4, 5])}
        schedulers, timesteps = pipe.parepare_schedulers(10, F_)
        ti = inp["timestep_indices"].clone()
        res = pipe(pixel_values_latents=inp["pixel_latents"].clone(), plucker_embeds_latents=inp["plucker"].clone(),
                   skeletons_latents=inp["skeletons"].float(), cond_masks_latents=inp["cond_mask"].clone(),
                   latents=inp["latents"].clone(), domains=["spatial"], num_inference_steps=5, schedulers=schedulers,
                   timesteps=timesteps, timestep_indices=ti, guidance_scale=guidance, output_type="latent")
        out["cases"][tag] = {"config": vars(cfg), "guidance": guidance, "n_steps_table": 10, "num_inference_steps": 5,
                             "in": inp, "timesteps_table": timesteps.clone(), "out_latents": res,
                             "out_timestep_indices": ti, "order_list": list(pipe.scheduler.order_list),
                             "lower_order_final": pipe.scheduler.cfg.lower_order_final}
        print("pipeline_dpm_single", tag, float(res.abs().mean()), ti.tolist(), pipe.scheduler.order_list)

    # ---- sliding_iterative_denoise: every task runs on the same pipeline object (the copies reset per call, the
    # lower_order_final switch of set_timesteps stays).  window_sizes: one per task.
    cases = (
        ("slide_spatial_eps_cfg_order3", "spatial", 2, 6, (3, 3), 1, False, 2, 2.0, dict(solver_order=3)),
        ("slide_temporal_bidir_v_nocfg", "temporal", 4, 4, (2, 2), 2, True, 2, 1.0, dict(prediction_type="v_prediction")),
        ("slide_spatial_order1_sample", "spatial", 2, 4, (2, 2), 1, True, 1, 2.0,
         dict(solver_order=1, prediction_type="sample", **SCALED_LINEAR)),
        ("slide_spatial_order3_nolof_sigma_min", "spatial", 2, 4, (3, 3), 1, True, 1, 2.0,
         dict(solver_order=3, final_sigmas_type="sigma_min")),
        # 3 steps of order 2 switch lower_order_final on; the second task's 4 steps then end on [.., 1, 1], not [.., 1, 2]
        ("slide_order2_switch_persists", "spatial", 2, 4, (3, 4), 1, False, 1, 2.0, dict(final_sigmas_type="sigma_min")),
    )
    for tag, domain, n_in, n_tg, wss, stride, bidir, rounds, guidance, ckw in cases:
        cfg = DPMSingleConfig(**ckw)
        config = dict(vars(cfg))
        pipe, cin = make_single_pipe(cfg)
        n = n_in + n_tg
        tasks = []
        for ws in wss:
            mask = torch.ones(n, 1, 8 * h, 8 * w)
            mask[:n_in] = 0
            pixel = torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1
            inp = {"pixel_values": pixel, "plucker": rn(n, 6, h, w).clamp(-1, 1),
                   "skeletons": skel(n), "cond_masks": mask,
                   "latents": rn(n, 4, h, w), "timestep_indices": torch.zeros(n, dtype=torch.int64)}
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
                          "out_timestep_indices": res["timestep_indices"], "fully_denoised": res["fully_denoised"],
                          "order_list": list(pipe.scheduler.order_list),
                          "lower_order_final": pipe.scheduler.cfg.lower_order_final})
            print("pipeline_dpm_single", tag, float(res["latents"].abs().mean()), res["timestep_indices"].tolist(),
                  pipe.scheduler.order_list)
        out["cases"][tag] = {"config": config, "domain": domain, "sliding_stride": stride, "bidirectional": bidir,
                             "alternation_rounds": rounds, "guidance": guidance, "tasks": tasks}
    save_sharded(out, "pipeline_dpm_single_ref")


if __name__ == "__main__":
    gen_pipeline_dpm_single()
