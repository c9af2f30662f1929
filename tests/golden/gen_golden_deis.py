"""Generate tests/golden/pipeline_deis_ref.pt by RUNNING the reference pipeline code with a stateful DEIS scheduler (only
possible in a container that has a checkout of the reference; the tests never read it, so the output is committed).

  pipeline_deis_ref.pt -- the reference ``Diffuman4DPipeline.__call__`` (PIPE:345-425) and ``sliding_iterative_denoise``
                        (PIPE:439-559) on the stubs of tests/golden/gen_golden.py, with a DEIS scheduler (our
                        ``oracle.deis_oracle.DEISOracle`` behind the upstream ``set_timesteps`` / ``scale_model_input`` /
                        ``step`` surface).  Pins what a STATEFUL scheduler sees through the reference -- one deep copy
                        per frame (PIPE:265-271), the copies of a window's frames handed to ``__call__`` (PIPE:535), a
                        fresh set per ``sliding_iterative_denoise`` call (PIPE:501), a frame's step index and order count
                        starting from its first timestep whatever that index is -- not the solver arithmetic itself.

Run:  DIFFUMAN4D_REFERENCE=<reference checkout> python tests/golden/gen_golden_deis.py      (from the repo root)
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_golden import _load_ref_pipeline, save_sharded  # noqa: E402

SCALED_LINEAR = dict(beta_schedule="scaled_linear", beta_start=0.00085, beta_end=0.012)


def gen_pipeline_deis():
    """The reference pipeline with a per-frame deep-copyable DEIS scheduler; see the module docstring."""
    from diffuman4d_b200.config import DEISConfig
    from oracle.deis_oracle import DEISOracle
    pipe_mod, make_pipe = _load_ref_pipeline()

    def make_deis_pipe(cfg):
        pipe, cin = make_pipe(True)
        pipe.scheduler = RefDEIS(cfg)      # what register_modules(scheduler=...) stores (PIPE:138)
        return pipe, cin

    class RefDEIS(DEISOracle):
        """the upstream scheduler surface the reference touches (PIPE:265-271,376,420)"""

        def set_timesteps(self, n, device=None):
            super().set_timesteps(n)

        def scale_model_input(self, x, t):
            return x

        def step(self, noise, t, latent, return_dict=False):
            return (super().step(noise, int(t), latent),)

    out = {"cases": {}}
    h = w = 4
    g = torch.Generator().manual_seed(2028)
    rn = lambda *s: torch.randn(*s, generator=g)

    # ---- one window through __call__: fresh per-frame copies at staggered (nonzero) timestep indices, 5 inference
    # steps of a 10-step table, so that the frames pass through orders 1 .. 3 and one reaches the last two rows
    for tag, guidance, ckw in (("call_cfg_eps_order3", 2.0, dict(solver_order=3)),
                               ("call_nocfg_v_order3_nolof", 1.0, dict(prediction_type="v_prediction", solver_order=3,
                                                                       lower_order_final=False))):
        cfg = DEISConfig(**ckw)
        pipe, cin = make_deis_pipe(cfg)
        F_ = 5
        mask = torch.ones(F_, 1, h, w)
        mask[:2] = 0
        inp = {"latents": rn(F_, 4, h, w), "pixel_latents": rn(F_, 4, h, w), "plucker": rn(F_, 6, h, w).clamp(-1, 1),
               "skeletons": torch.rand(F_, 3, 8 * h, 8 * w, generator=g) * 2 - 1, "cond_mask": mask,
               "timestep_indices": torch.tensor([0, 0, 1, 3, 5])}
        schedulers, timesteps = pipe.parepare_schedulers(10, F_)
        ti = inp["timestep_indices"].clone()
        res = pipe(pixel_values_latents=inp["pixel_latents"].clone(), plucker_embeds_latents=inp["plucker"].clone(),
                   skeletons_latents=inp["skeletons"].clone(), cond_masks_latents=inp["cond_mask"].clone(),
                   latents=inp["latents"].clone(), domains=["spatial"], num_inference_steps=5, schedulers=schedulers,
                   timesteps=timesteps, timestep_indices=ti, guidance_scale=guidance, output_type="latent")
        out["cases"][tag] = {"config": vars(cfg), "guidance": guidance, "n_steps_table": 10, "num_inference_steps": 5,
                             "in": inp, "timesteps_table": timesteps.clone(), "out_latents": res,
                             "out_timestep_indices": ti, "lower_order_nums": [s.lower_order_nums for s in schedulers]}
        print("pipeline_deis", tag, float(res.abs().mean()), ti.tolist())

    # ---- sliding_iterative_denoise: every task runs twice on the same pipeline object (the copies reset per call)
    cases = (
        ("slide_spatial_eps_cfg_order3", "spatial", 2, 6, 3, 1, False, 2, 2.0, dict(solver_order=3)),
        ("slide_temporal_bidir_v_nocfg", "temporal", 4, 4, 2, 2, True, 2, 1.0, dict(prediction_type="v_prediction")),
        ("slide_spatial_order1_leading_sample", "spatial", 2, 4, 2, 1, True, 1, 2.0,
         dict(solver_order=1, timestep_spacing="leading", steps_offset=1, prediction_type="sample", **SCALED_LINEAR)),
        ("slide_spatial_order3_nolof_trailing", "spatial", 2, 4, 2, 1, True, 1, 2.0,
         dict(solver_order=3, lower_order_final=False, timestep_spacing="trailing")),
    )
    for tag, domain, n_in, n_tg, ws, stride, bidir, rounds, guidance, ckw in cases:
        cfg = DEISConfig(**ckw)
        pipe, cin = make_deis_pipe(cfg)
        n = n_in + n_tg
        tasks = []
        for _task in range(2):
            mask = torch.ones(n, 1, 8 * h, 8 * w)
            mask[:n_in] = 0
            pixel = torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1
            inp = {"pixel_values": pixel, "plucker": rn(n, 6, h, w).clamp(-1, 1),
                   "skeletons": torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1, "cond_masks": mask,
                   "latents": rn(n, 4, h, w), "timestep_indices": torch.zeros(n, dtype=torch.int64)}
            res = pipe.sliding_iterative_denoise(
                pixel_values=inp["pixel_values"].clone(), plucker_embeds=inp["plucker"].clone(),
                skeletons=inp["skeletons"].clone(), cond_masks=inp["cond_masks"].clone(), latents=inp["latents"].clone(),
                domain=domain, timestep_indices=inp["timestep_indices"].clone(), window_size=ws, sliding_stride=stride,
                sliding_shift=0, bidirectional=bidir, num_denoising_steps=1, alternation_rounds=rounds,
                guidance_scale=guidance, tqdm=lambda it, total=None: it)
            z = torch.nn.functional.avg_pool2d(pixel, 8)
            inp["pixel_latents"] = torch.cat([z, z.mean(dim=1, keepdim=True)], dim=1)  # what the fake VAE encoded
            inp["cond_mask_latents"] = torch.nn.functional.interpolate(mask, size=(h, w), mode="nearest")
            del inp["pixel_values"], inp["cond_masks"]
            tasks.append({"in": inp, "out_latents": res["latents"], "out_timestep_indices": res["timestep_indices"],
                          "fully_denoised": res["fully_denoised"]})
            print("pipeline_deis", tag, float(res["latents"].abs().mean()), res["timestep_indices"].tolist())
        out["cases"][tag] = {"config": vars(cfg), "domain": domain, "window_size": ws, "sliding_stride": stride,
                             "bidirectional": bidir, "alternation_rounds": rounds, "guidance": guidance, "tasks": tasks}
    save_sharded(out, "pipeline_deis_ref")


if __name__ == "__main__":
    gen_pipeline_deis()
