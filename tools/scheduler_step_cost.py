"""What the DPM-Solver++, UniPC, PNDM, DEIS, singlestep DPM-Solver++ and DDPM steps cost against DDIM in the window step of
bench.py's workload (W16 @ 64x64 latents, CFG 2.0, SD-2.1 channel layout, random weights), on one GPU in one process.

The seven pipelines share one UNet; rounds alternate DDIM, DPM-Solver++, UniPC, PNDM, DEIS, singlestep DPM-Solver++ and
DDPM, in an order rotated by one arm each round, so that clock drift and the position in a round hit all alike.
Each step restores its inputs (latents, timestep indices and, for the multistep schedulers, the frames' solver state) from
device copies and then makes ONE public ``denoise_window`` call.  The multistep frames start with a full history, so the
timed step is the second-order one; the UniPC target frames also sit two steps further into the schedule, so that both
its corrector and its predictor run at order 2, the PNDM frames have taken five steps, so that they combine four
model outputs, the DEIS (solver_order 3) frames sit at the UniPC rows with a full history, so that every one takes
the third-order step, and the singlestep (solver_order 3) frames sit on third-order rows of its order list with a full
history, so that every one takes the third-order update from its block's start sample; every DDPM target frame sits on a
row with t > 0, so that every one draws its noise.  Also times the seven fused step kernels alone.  Prints one JSON line (and writes it to --out) with the
card's name, power limit and max SM clock beside the numbers.

    python tools/scheduler_step_cost.py --rounds 8 --steps 10 --out /tmp/scheduler_step_cost.json
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10, help="window steps per round and scheduler")
    ap.add_argument("--kernel-iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs an H100: there is no CPU fallback")

    from bench import WORKLOAD, gpu_identity, synth_inputs
    from diffuman4d_b200 import ops
    from diffuman4d_b200._lib import check, lib
    from diffuman4d_b200.config import (DDPMConfig, DEISConfig, DPMSingleConfig, DPMSolverConfig, PNDMConfig,
                                        SchedulerConfig, UNetConfig, UniPCConfig)
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.scheduler import (DDPMTask, DEISState, DPMSingleState, DPMSolverState, PNDMState,
                                           UniPCState)
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    wl = WORKLOAD
    F, h, w, n_cond = wl["F"], wl["h"], wl["w"], wl["n_cond"]
    cfg = UNetConfig.sd21()
    unet = B200MultiviewUNet(cfg, 0).load_state_dict(random_state_dict(cfg, seed=1))
    ddim = B200Diffuman4DPipeline(unet, SchedulerConfig())
    dpm = B200Diffuman4DPipeline(unet, DPMSolverConfig())
    unipc = B200Diffuman4DPipeline(unet, UniPCConfig())
    pndm = B200Diffuman4DPipeline(unet, PNDMConfig())
    deis = B200Diffuman4DPipeline(unet, DEISConfig(solver_order=3))
    single = B200Diffuman4DPipeline(unet, DPMSingleConfig(solver_order=3))
    ddpm = B200Diffuman4DPipeline(unet, DDPMConfig())
    for p in (ddim, dpm, unipc, pndm, deis, single, ddpm):
        p.parepare_schedulers(wl["n_steps"], F)

    inp = {k: (v.to(torch.bfloat16) if v.dtype.is_floating_point else v).to(dev)
           for k, v in synth_inputs(F, n_cond, h, w).items()}
    lat, ts = inp["latents"].clone(), inp["ts"].clone()
    g = torch.Generator(device=dev).manual_seed(0)
    x0_init = torch.randn(F, 4, h, w, device=dev, generator=g).to(torch.bfloat16)
    lon_init = torch.full((F,), 1, dtype=torch.int32, device=dev)          # every frame has a history: second order
    state = DPMSolverState(F, dev).take(torch.arange(F), h, w)
    ts_unipc = inp["ts"].clone()
    ts_unipc[n_cond:] += 2                                                 # rows with an order-2 corrector
    lon2_init = torch.full((F,), 2, dtype=torch.int32, device=dev)
    x0_init2 = torch.randn(F, 4, h, w, device=dev, generator=g).to(torch.bfloat16)
    last_init = torch.randn(F, 4, h, w, device=dev, generator=g).to(torch.bfloat16)
    state_u = UniPCState(F, dev).take(torch.arange(F), h, w)
    ets_init = [torch.randn(F, 4, h, w, device=dev, generator=g).to(torch.bfloat16) for _ in range(4)]
    cnt_init = torch.full((F,), 5, dtype=torch.int32, device=dev)           # four kept outputs: the 4-term sum
    state_p = PNDMState(F, dev).take(torch.arange(F), h, w)
    lon3_init = torch.full((F,), 3, dtype=torch.int32, device=dev)         # two outputs of history: third order
    state_d = DEISState(F, dev, solver_order=3).take(torch.arange(F), h, w)
    ts_single = inp["ts"].clone()
    ts_single[n_cond:] = ts_single[n_cond:] // 3 * 3 + 2                   # the third row of each block: order 3
    assert all(single.scheduler.order_list[int(i)] == 3 for i in ts_single[n_cond:])
    cur_init = torch.randn(F, 4, h, w, device=dev, generator=g).to(torch.bfloat16)
    state_s = DPMSingleState(F, dev, solver_order=3).take(torch.arange(F), h, w)
    frames_p = DDPMTask(F, dev, seed=1234).take(torch.arange(F))   # every target row has t > 0: the noise is drawn

    def window(p, solver_state=None, ts_init=inp["ts"]):
        def step():
            lat.copy_(inp["latents"])
            ts.copy_(ts_init)
            if isinstance(solver_state, DPMSingleState):
                solver_state.x0_prev.copy_(x0_init)
                solver_state.x0_prev2.copy_(x0_init2)
                solver_state.cur_sample.copy_(cur_init)
                solver_state.lower_order_nums.copy_(lon3_init)
            elif isinstance(solver_state, DEISState):
                solver_state.m_prev.copy_(x0_init)
                solver_state.m_prev2.copy_(x0_init2)
                solver_state.lower_order_nums.copy_(lon3_init)
            elif isinstance(solver_state, PNDMState):
                for k in range(4):
                    getattr(solver_state, f"ets{k}").copy_(ets_init[k])
                solver_state.lower_order_nums.copy_(cnt_init)
            elif isinstance(solver_state, UniPCState):
                solver_state.x0_prev2.copy_(x0_init2)
                solver_state.last_sample.copy_(last_init)
                solver_state.x0_prev.copy_(x0_init)
                solver_state.lower_order_nums.copy_(lon2_init)
            elif isinstance(solver_state, DPMSolverState):   # DDPM's frames have no state to restore
                solver_state.x0_prev.copy_(x0_init)
                solver_state.lower_order_nums.copy_(lon_init)
            p.denoise_window(latents=lat, pixel_values_latents=inp["pixel"], plucker_embeds_latents=inp["plucker"],
                             skeletons_latents=inp["skel"], cond_masks_latents=inp["mask"], timestep_indices=ts,
                             domain=wl["domain"], guidance_scale=wl["guidance"], solver_state=solver_state)
        return step

    # the fused step kernels alone, on the window's shapes (CFG noise [2F,4,h,w])
    noise = torch.randn(2 * F, 4, h, w, device=dev, generator=g).to(torch.bfloat16)
    ddim_s, dpm_s, unipc_s = ddim.scheduler.c_struct(), dpm.scheduler.c_struct(), unipc.scheduler.c_struct()
    pndm_s, deis_s, single_s = pndm.scheduler.c_struct(), deis.scheduler.c_struct(), single.scheduler.c_struct()
    ddpm_s = ddpm.scheduler.c_struct(False, frames_p.seed)
    out = torch.empty_like(lat)
    ts_out = torch.empty_like(ts)
    x0_k, lon_k = x0_init.clone(), lon_init.clone()
    x0_u, x02_u, last_u, lon_u = x0_init.clone(), x0_init2.clone(), last_init.clone(), lon2_init.clone()
    ts_u = ts_unipc.clone()
    ets_p, cur_p, cnt_p = [e.clone() for e in ets_init], x0_init.clone(), cnt_init.clone()
    m_d, m2_d, lon_d = x0_init.clone(), x0_init2.clone(), lon3_init.clone()
    x0_s, x02_s, cur_s, lon_s = x0_init.clone(), x0_init2.clone(), cur_init.clone(), lon3_init.clone()
    ts_s = ts_single.clone()
    stream = lambda: torch.cuda.current_stream().cuda_stream

    def ddim_kernel():
        check(lib().d4d_cfg_ddim_step(noise.data_ptr(), lat.data_ptr(), inp["mask"].data_ptr(), ts.data_ptr(),
                                      ts_out.data_ptr(), C.byref(ddim_s), wl["guidance"], 1, F, h, w, out.data_ptr(),
                                      stream()))

    def dpm_kernel():
        ops.cfg_dpm_step(noise, lat, inp["mask"], ts, x0_k, lon_k, dpm_s, wl["guidance"], True)

    def unipc_kernel():
        ops.cfg_unipc_step(noise, lat, inp["mask"], ts_u, x0_u, x02_u, last_u, lon_u, unipc_s, wl["guidance"], True)

    def pndm_kernel():
        ops.cfg_pndm_step(noise, lat, inp["mask"], ts, ets_p, cur_p, cnt_p, pndm_s, wl["guidance"], True)

    def deis_kernel():
        ops.cfg_deis_step(noise, lat, inp["mask"], ts_u, m_d, m2_d, lon_d, deis_s, wl["guidance"], True)

    def single_kernel():
        ops.cfg_dpm_single_step(noise, lat, inp["mask"], ts_s, x0_s, x02_s, cur_s, lon_s, single_s, wl["guidance"], True)

    def ddpm_kernel():
        ops.cfg_ddpm_step(noise, lat, inp["mask"], ts, frames_p.frame_ids, ddpm_s, wl["guidance"], True)

    def timed(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    arms = {"ddim": window(ddim), "dpm_solver++": window(dpm, state), "unipc": window(unipc, state_u, ts_unipc),
            "pndm": window(pndm, state_p), "deis": window(deis, state_d, ts_unipc),
            "dpm_single": window(single, state_s, ts_single), "ddpm": window(ddpm, frames_p)}
    for fn in arms.values():                                             # warm-up: plans, buffers, clocks
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    per_round = {k: [] for k in arms}
    kernel = {"ddim": [], "dpm_solver++": [], "unipc": [], "pndm": [], "deis": [], "dpm_single": [], "ddpm": []}
    names = list(arms)
    for r in range(args.rounds):
        for k in names[r % len(names):] + names[:r % len(names)]:   # rotated: no arm always runs first in a round
            per_round[k].append(timed(arms[k], args.steps))
        kernel["ddim"].append(timed(ddim_kernel, args.kernel_iters))
        kernel["dpm_solver++"].append(timed(dpm_kernel, args.kernel_iters))
        kernel["unipc"].append(timed(unipc_kernel, args.kernel_iters))
        kernel["pndm"].append(timed(pndm_kernel, args.kernel_iters))
        kernel["deis"].append(timed(deis_kernel, args.kernel_iters))
        kernel["dpm_single"].append(timed(single_kernel, args.kernel_iters))
        kernel["ddpm"].append(timed(ddpm_kernel, args.kernel_iters))
    med = {k: statistics.median(v) for k, v in per_round.items()}
    kmed = {k: statistics.median(v) for k, v in kernel.items()}
    res = {"workload": wl["name"], "gpu": gpu_identity(0), "rounds": args.rounds, "steps_per_round": args.steps,
           "window_step_ms_median": med, "window_step_ms_rounds": per_round,
           "dpm_minus_ddim_ms": med["dpm_solver++"] - med["ddim"],
           "dpm_over_ddim": med["dpm_solver++"] / med["ddim"],
           "unipc_minus_ddim_ms": med["unipc"] - med["ddim"],
           "unipc_minus_dpm_ms": med["unipc"] - med["dpm_solver++"],
           "pndm_minus_ddim_ms": med["pndm"] - med["ddim"],
           "deis_minus_ddim_ms": med["deis"] - med["ddim"],
           "dpm_single_minus_ddim_ms": med["dpm_single"] - med["ddim"],
           "ddpm_minus_ddim_ms": med["ddpm"] - med["ddim"],
           "step_kernel_us_median": {k: 1e3 * v for k, v in kmed.items()},
           "note": "DPM-Solver++ and UniPC steps timed in their second-order branches (every frame has a full history, "
                   "UniPC corrects at order 2), PNDM in its four-output branch, DEIS and singlestep DPM-Solver++ in "
                   "their third-order branches, DDPM with noise drawn on every target frame; the kernel-only multistep times include the op wrappers' output "
                   "allocations"}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
