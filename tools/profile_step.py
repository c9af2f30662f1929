"""One warm window step, then ONE profiled window step (cudaProfilerStart/Stop) -- the command ncu wraps.
    ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv --log-file launches.csv python tools/profile_step.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from diffuman4d_b200.config import SchedulerConfig, UNetConfig  # noqa: E402
from diffuman4d_b200.pipeline import B200Diffuman4DPipeline  # noqa: E402
from diffuman4d_b200.unet import B200MultiviewUNet  # noqa: E402
from diffuman4d_b200.weights import random_state_dict  # noqa: E402

cfg = UNetConfig.sd21()
wl = bench.WORKLOAD
unet = B200MultiviewUNet(cfg, 0).load_state_dict(random_state_dict(cfg, seed=1))
pipe = B200Diffuman4DPipeline(unet, SchedulerConfig())
pipe.parepare_schedulers(wl["n_steps"], wl["F"])
d = {k: (v.to(torch.bfloat16) if v.dtype.is_floating_point else v).cuda()
     for k, v in bench.synth_inputs(wl["F"], wl["n_cond"], wl["h"], wl["w"]).items()}


def step():
    lat, ts = d["latents"].clone(), d["ts"].clone()
    pipe.denoise_window(latents=lat, pixel_values_latents=d["pixel"], plucker_embeds_latents=d["plucker"],
                        skeletons_latents=d["skel"], cond_masks_latents=d["mask"], timestep_indices=ts,
                        domain=wl["domain"], guidance_scale=wl["guidance"])
    torch.cuda.synchronize()


step()
torch.cuda.profiler.start()
step()
torch.cuda.profiler.stop()
print("profiled one window step")
