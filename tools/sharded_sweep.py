"""Time one demo_3d-shaped task frame-sharded against the single-GPU loop, after checking that both give the same bits.

The task is the spatial task of the reference's demo_3d sampling run (SURVEY.md section 6): 48 cameras, 4 of them inputs,
window 12 (+4 conditioning views = 16 frames), stride 1, one direction: 44 windows of one DDIM step, CFG 2.0, on the
SD-2.1 UNet layout with random weights.

    torchrun --nproc-per-node R tools/sharded_sweep.py [--latent 64] [--repeats 3] [--out sweep.json]
    python tools/sharded_sweep.py ...          # R = 1: the sharded plan on one GPU, exchanging with itself

R must divide the 16 frames of a window (1, 2, 4, 8).  Rank 0 also runs the single-GPU loop (``B200Diffuman4DPipeline``
on its own handle) while the other ranks wait; before any timing, the sharded result of every rank must equal it bit for
bit, or the script exits with an error.  Prints one JSON line: the median wall time of the task each way, the speed-up,
and windows per second.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--latent", type=int, default=64)
    ap.add_argument("--cams", type=int, default=48)
    ap.add_argument("--window", type=int, default=12)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()

    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    else:
        store = os.path.join(tempfile.mkdtemp(prefix="d4d-sweep-"), "store")
        dist.init_process_group("gloo", init_method=f"file://{store}", rank=0, world_size=1)

    from diffuman4d_b200.config import SchedulerConfig, UNetConfig
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.sharded import FrameShardedPipeline
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict

    cfg = UNetConfig.sd21()
    sd = random_state_dict(cfg, seed=1)
    n, lat = args.cams, args.latent
    inputs = [1, 13, 25, 37] if n >= 48 else sorted({(n * k) // 4 + 1 for k in range(4)})
    F = len(inputs) + args.window
    if F % world:
        raise SystemExit(f"{world} ranks do not divide the {F} frames of a window")
    g = torch.Generator().manual_seed(0)
    mask = torch.ones(n, 1, lat, lat)
    mask[inputs] = 0
    task = dict(pixel_values_latents=torch.randn(n, 4, lat, lat, generator=g).to(torch.bfloat16),
                plucker_embeds=torch.randn(n, 6, lat, lat, generator=g),
                skeletons_latents=(torch.rand(n, 3, 8 * lat, 8 * lat, generator=g) * 2 - 1).to(torch.bfloat16),
                cond_masks=mask, latents=torch.randn(n, 4, lat, lat, generator=g), domain="spatial",
                timestep_indices=torch.zeros(n, dtype=torch.long), window_size=args.window, sliding_stride=1,
                bidirectional=False, num_denoising_steps=1, alternation_rounds=1, guidance_scale=2.0)

    pipe = B200Diffuman4DPipeline(B200MultiviewUNet(cfg, local).load_state_dict(sd), SchedulerConfig())
    sharded = FrameShardedPipeline(pipe, max_frames=F, h=lat, w=lat)
    single = B200Diffuman4DPipeline(B200MultiviewUNet(cfg, local).load_state_dict(sd), SchedulerConfig()) if rank == 0 else None

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn(**task)
        torch.cuda.synchronize()
        return out, time.perf_counter() - t0

    # correctness first (these runs also build the plans)
    got, _ = timed(sharded.sliding_iterative_denoise)
    ok = torch.ones(1, device="cuda")
    if rank == 0:
        ref, _ = timed(single.sliding_iterative_denoise)
    ref_lat = ref["latents"] if rank == 0 else torch.empty_like(got["latents"])
    ref_ti = ref["timestep_indices"] if rank == 0 else torch.empty_like(got["timestep_indices"])
    dist.broadcast(ref_lat.view(torch.uint8), src=0)
    dist.broadcast(ref_ti, src=0)
    ok[0] = float(torch.equal(got["latents"], ref_lat) and torch.equal(got["timestep_indices"], ref_ti))
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    if ok.item() != 1.0:
        raise SystemExit("the frame-sharded task differs from the single-GPU task")

    t_single, t_sharded = [], []
    for _ in range(args.repeats):
        if rank == 0:
            t_single.append(timed(single.sliding_iterative_denoise)[1])
        dist.barrier()
        t_sharded.append(timed(sharded.sliding_iterative_denoise)[1])
        dist.barrier()
    windows = n - len(inputs)
    if rank == 0:
        s, f = statistics.median(t_single), statistics.median(t_sharded)
        res = {"workload": f"demo_3d-shaped spatial task: {n} cameras ({len(inputs)} inputs), {windows} windows of {F} "
                           f"frames @ {lat}x{lat} latents, 1 DDIM step each, CFG 2.0, SD-2.1 UNet layout, random weights",
               "gpu": torch.cuda.get_device_name(local), "ranks": world, "bit_identical": True,
               "single_gpu_s": round(s, 3), "frame_sharded_s": round(f, 3), "speedup": round(s / f, 3),
               "windows_per_s_single": round(windows / s, 2), "windows_per_s_sharded": round(windows / f, 2),
               "repeats": args.repeats}
        if args.out:
            os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
            json.dump(res, open(args.out, "w"), indent=1)
        print(json.dumps(res))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
