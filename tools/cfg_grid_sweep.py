"""Time a window step on the CFG grid (each CFG half frame-sharded over R = world / 2 ranks) against the single-GPU step
and the frame-sharded window on the same ranks, after checking the grid gives the single-GPU bits.

The window is W16 at 64x64 latents (12 targets + 4 conditioning frames, the demo_3d window), one DDIM step, CFG 2.0, on
the SD-2.1 UNet layout with random weights.

    torchrun --nproc-per-node 4 tools/cfg_grid_sweep.py [--latent 64] [--frames 16] [--repeats 5] [--out grid.json]
    torchrun --nproc-per-node 8 tools/cfg_grid_sweep.py

Rank g uses cuda:g when there are as many devices as ranks, otherwise every rank shares cuda:0.  Rank 0 also runs the
single-GPU step (``B200Diffuman4DPipeline`` on its own handle).  Before any timing, every rank's grid result (latents and
timestep indices) must equal it bit for bit, or the script exits with an error.  Then the single-GPU, grid and
frame-sharded steps alternate (the frame-sharded time includes its window-result exchange, so that, like the grid, every
rank ends with the whole window) for ``--repeats`` rounds; rank 0 prints one JSON line with the median of each, the card,
its power limit and maximum SM clock.  When the ranks share one device, the multi-rank times say nothing about several
GPUs and are reported as "not measured"; so is the frame-sharded step when the ranks do not divide the window.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from cfg_split_sweep import card, window  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--latent", type=int, default=64)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()

    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    dev = rank if torch.cuda.device_count() >= world else 0
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("gloo")
    else:
        store = os.path.join(tempfile.mkdtemp(prefix="d4d-grid-"), "store")
        dist.init_process_group("gloo", init_method=f"file://{store}", rank=0, world_size=1)
    from diffuman4d_b200.cfg_split import CFGGridPipeline, grid_cell
    from diffuman4d_b200.config import SchedulerConfig, UNetConfig
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.sharded import FrameShardedPipeline
    from diffuman4d_b200.sharding import frame_shard
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict

    cfg = UNetConfig.sd21()
    sd = random_state_dict(cfg, seed=1)
    F, lat = args.frames, args.latent
    _, _, R = grid_cell(rank, world)
    if F % R:
        raise SystemExit(f"--frames {F} must be divisible by the {R} ranks of each CFG half")
    new = lambda: B200Diffuman4DPipeline(B200MultiviewUNet(cfg, dev).load_state_dict(sd), SchedulerConfig())
    inputs = {k: v.cuda() for k, v in window(cfg, F, lat).items()}
    kw = dict(domain="spatial", guidance_scale=2.0, num_inference_steps=1)
    grid = CFGGridPipeline(new(), max_frames=F, h=lat, w=lat)
    sharded = FrameShardedPipeline(new(), max_frames=F, h=lat, w=lat) if F % world == 0 else None
    single = new() if rank == 0 else None
    for p in (grid.pipe, None if sharded is None else sharded.pipe, single):
        if p is not None:
            p.parepare_schedulers(18, F)

    def step(run, rows=None, **extra):
        x = {k: (v[slice(*rows)] if rows else v).clone() for k, v in inputs.items()}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run(**x, **kw, **extra)
        torch.cuda.synchronize()
        return x, time.perf_counter() - t0

    # correctness first (these runs also build the plans)
    got, _ = step(grid.denoise_window)
    ref = step(single.denoise_window)[0] if rank == 0 else {k: torch.empty_like(v) for k, v in got.items()}
    ok = torch.ones(1)
    for k in ("latents", "timestep_indices"):
        r = ref[k].cpu()
        dist.broadcast(r.view(torch.uint8) if r.dtype == torch.bfloat16 else r, src=0)
        ok[0] = min(ok[0].item(), float(torch.equal(got[k].cpu(), r)))
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    if ok.item() != 1.0:
        raise SystemExit("the CFG-grid window step differs from the single-GPU step")
    shard_rows = frame_shard(F, rank, world) if sharded is not None else None

    def sharded_step(latents, pixel_values_latents, plucker_embeds_latents, skeletons_latents, cond_masks_latents,
                     timestep_indices, **kw_):
        """The frame-sharded step on this rank's frames and the window-result exchange that gives every rank the whole
        window, as the grid step does."""
        conds = (pixel_values_latents, plucker_embeds_latents, skeletons_latents, cond_masks_latents)
        return sharded._step_and_exchange(latents, timestep_indices, None, conds, F, **kw_)

    if sharded is not None:
        step(sharded_step, shard_rows)

    t_single, t_grid, t_sharded = [], [], []
    for _ in range(args.repeats):
        if rank == 0:
            t_single.append(step(single.denoise_window)[1])
        dist.barrier()
        t_grid.append(step(grid.denoise_window)[1])
        dist.barrier()
        if sharded is not None:
            t_sharded.append(step(sharded_step, shard_rows)[1])
            dist.barrier()
    shared = world > 1 and torch.cuda.device_count() < world
    res = None
    if rank == 0:
        measured = not shared and world > 1
        s, g = statistics.median(t_single), statistics.median(t_grid)
        sh = statistics.median(t_sharded) if t_sharded else None
        ms = lambda t: round(1e3 * t, 2) if measured and t is not None else "not measured"
        res = {"workload": f"one window step of {F} frames ({F - 4} targets) @ {lat}x{lat} latents, DDIM, CFG 2.0, "
                           "SD-2.1 UNet layout with pose encoder, random weights",
               **card(dev), "ranks": world, "ranks_per_cfg_half": R, "ranks_share_one_device": shared,
               "bit_identical": True, "single_gpu_ms": round(1e3 * s, 2), "cfg_grid_ms": ms(g),
               "frame_sharded_ms": ms(sh),
               "grid_speedup_over_single": round(s / g, 3) if measured else "not measured",
               "grid_speedup_over_frame_sharded": round(sh / g, 3) if measured and sh is not None else "not measured",
               "repeats": args.repeats}
        print(json.dumps(res))
        if args.out:
            os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
            json.dump(res, open(args.out, "w"), indent=1)
    dist.barrier()
    dist.destroy_process_group()
    return res


if __name__ == "__main__":
    main()
