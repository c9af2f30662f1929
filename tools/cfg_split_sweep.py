"""Time a window step split by CFG half over two ranks against the single-GPU step, after checking both give the same bits.

The window is W16 at 64x64 latents (12 targets + 4 conditioning frames, the demo_3d window), one DDIM step, CFG 2.0,
on the SD-2.1 UNet layout with random weights.

    torchrun --nproc-per-node 2 tools/cfg_split_sweep.py [--latent 64] [--frames 16] [--repeats 5] [--out split.json]
    python tools/cfg_split_sweep.py --bound [--latent 64] [--frames 16]     # one GPU

Rank k uses cuda:k when there are two devices, otherwise both ranks share cuda:0.  Rank 0 also runs the single-GPU step
(``B200Diffuman4DPipeline`` on its own handle).  Before any timing, both ranks' split results (latents and timestep
indices) must equal it bit for bit, or the script exits with an error.  Then single-GPU and split steps alternate for
``--repeats`` rounds; the JSON line reports the median of each, the card, its power limit and maximum SM clock.  When
both ranks share one device, the split time says nothing about two GPUs and is reported as "not measured".

``--bound``: on one GPU, the UNet forward at B = F (one CFG half: what each rank of the split computes) against B = 2F
(the whole window, domains [d] against [d, d]), timed with CUDA events.  That is the per-rank compute of the split
against the whole window, without the exchange.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card(dev: int) -> dict:
    """The device's name, power limit and maximum SM clock, read with the measurement."""
    q = subprocess.run(["nvidia-smi", f"--id={dev}", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = ([s.strip() for s in q.stdout.strip().split(",")] + ["?"] * 3)[:3]
    return {"gpu": name or torch.cuda.get_device_name(dev), "power_limit": power, "max_sm_clock": clock}


def window(cfg, F: int, lat: int, seed: int = 0):
    g = torch.Generator().manual_seed(seed)
    mask = torch.ones(F, 1, lat, lat, dtype=torch.bfloat16)
    mask[:4] = 0
    return dict(latents=torch.randn(F, 4, lat, lat, generator=g).to(torch.bfloat16),
                pixel_values_latents=torch.randn(F, 4, lat, lat, generator=g).to(torch.bfloat16),
                plucker_embeds_latents=torch.randn(F, 6, lat, lat, generator=g).to(torch.bfloat16),
                skeletons_latents=(torch.rand(F, 3, 8 * lat, 8 * lat, generator=g) * 2 - 1).to(torch.bfloat16),
                cond_masks_latents=mask, timestep_indices=torch.tensor([0] * 4 + [3] * (F - 4)))


def bound(args):
    from diffuman4d_b200.config import UNetConfig
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict
    cfg = UNetConfig.sd21()
    unet = B200MultiviewUNet(cfg, 0).load_state_dict(random_state_dict(cfg, seed=1))
    F, lat = args.frames, args.latent
    g = torch.Generator().manual_seed(0)
    ms = {}
    for halves in (1, 2):
        B = halves * F
        x = torch.randn(B, cfg.in_channels, lat, lat, generator=g).to(torch.bfloat16).cuda()
        t = torch.full((B,), 500, dtype=torch.int64).cuda()
        sk = (torch.rand(B, 3, 8 * lat, 8 * lat, generator=g) * 2 - 1).to(torch.bfloat16).cuda()
        run = lambda: unet(x, t, sk, ["spatial"] * halves, F, return_dict=False)
        for _ in range(3):
            run()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            run()
        e1.record()
        e1.synchronize()
        ms[halves] = e0.elapsed_time(e1) / args.iters
    res = {"workload": f"UNet forward, SD-2.1 layout, random weights, pose encoder, {F} frames @ {lat}x{lat} latents",
           **card(0), "one_half_B_F_ms": round(ms[1], 3), "whole_window_B_2F_ms": round(ms[2], 3),
           "half_over_whole": round(ms[1] / ms[2], 3), "iters": args.iters}
    print(json.dumps(res))
    return res


def sweep(args):
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    dev = rank if torch.cuda.device_count() >= world else 0
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("gloo")
    else:
        store = os.path.join(tempfile.mkdtemp(prefix="d4d-split-"), "store")
        dist.init_process_group("gloo", init_method=f"file://{store}", rank=0, world_size=1)
    from diffuman4d_b200.cfg_split import CFGSplitPipeline
    from diffuman4d_b200.config import SchedulerConfig, UNetConfig
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict

    cfg = UNetConfig.sd21()
    sd = random_state_dict(cfg, seed=1)
    F, lat = args.frames, args.latent
    inputs = {k: v.cuda() for k, v in window(cfg, F, lat).items()}
    kw = dict(domain="spatial", guidance_scale=2.0, num_inference_steps=1)
    pipe = B200Diffuman4DPipeline(B200MultiviewUNet(cfg, dev).load_state_dict(sd), SchedulerConfig())
    split = CFGSplitPipeline(pipe, max_frames=F, h=lat, w=lat)
    single = B200Diffuman4DPipeline(B200MultiviewUNet(cfg, dev).load_state_dict(sd), SchedulerConfig()) if rank == 0 else None
    for p in (pipe, single):
        if p is not None:
            p.parepare_schedulers(18, F)

    def step(run):
        x = {k: v.clone() for k, v in inputs.items()}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run(**x, **kw)
        torch.cuda.synchronize()
        return x, time.perf_counter() - t0

    # correctness first (these runs also build the plans)
    got, _ = step(split.denoise_window)
    ref = step(single.denoise_window)[0] if rank == 0 else {k: torch.empty_like(v) for k, v in got.items()}
    ok = torch.ones(1)
    for k in ("latents", "timestep_indices"):
        r = ref[k].cpu()
        dist.broadcast(r.view(torch.uint8) if r.dtype == torch.bfloat16 else r, src=0)
        ok[0] = min(ok[0].item(), float(torch.equal(got[k].cpu(), r)))
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    if ok.item() != 1.0:
        raise SystemExit("the CFG-split window step differs from the single-GPU step")

    t_single, t_split = [], []
    for _ in range(args.repeats):
        if rank == 0:
            t_single.append(step(single.denoise_window)[1])
        dist.barrier()
        t_split.append(step(split.denoise_window)[1])
        dist.barrier()
    shared = world > 1 and torch.cuda.device_count() < world
    if rank == 0:
        s, c = statistics.median(t_single), statistics.median(t_split)
        res = {"workload": f"one window step of {F} frames ({F - 4} targets) @ {lat}x{lat} latents, DDIM, CFG 2.0, "
                           "SD-2.1 UNet layout with pose encoder, random weights",
               **card(dev), "ranks": world, "ranks_share_one_device": shared, "bit_identical": True,
               "single_gpu_ms": round(1e3 * s, 2),
               "cfg_split_ms": "not measured" if shared or world == 1 else round(1e3 * c, 2),
               "speedup": "not measured" if shared or world == 1 else round(s / c, 3), "repeats": args.repeats}
        print(json.dumps(res))
        return res
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--latent", type=int, default=64)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20, help="--bound: forwards per timing")
    ap.add_argument("--bound", action="store_true")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    res = bound(args) if args.bound else sweep(args)
    if res is not None and args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
