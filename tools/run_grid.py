"""BASELINE config 2 / 3 end to end: the `demo_4d_tiny` sampling run (reference configs/exp/demo_4d_tiny.yaml +
configs/sampler/sliding_default.yaml: 48 cameras x 16 frames, 4 input cameras, window 12, stride 1, 3 alternation rounds,
CFG 2.0) driven by B200SlidingIterativeSampler (the device-resident mirror of src/samplers/sliding_iterative_sampler.py)
through B200Diffuman4DPipeline.sliding_iterative_denoise on the SD-2.1 UNet layout with random weights, a synthetic dataset
with the reference's get_item contract and a pooling stand-in for the VAE (the VAE is out of scope, SURVEY 8f-1).

    python tools/run_grid.py [--latent 64] [--cams 48] [--frames 16] [--out grid.json]
    torchrun --nproc-per-node N tools/run_grid.py ...     # replicas: tasks of a round sharded over the ranks
    torchrun --nproc-per-node N tools/run_grid.py --frame-sharded ...   # every task on all ranks, windows split by frames

Prints one JSON line (and writes it to --out when given): window steps executed (W16 spatial / W24 temporal), device time inside denoise_window, wall time of execute_tasks.
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--latent", type=int, default=64)
    ap.add_argument("--cams", type=int, default=48)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    ap.add_argument("--prefetch", action="store_true", help="load the next task's dataset item on a helper thread")
    ap.add_argument("--frame-sharded", action="store_true",
                    help="run every task on all ranks with each window split by frames (windows of 16 spatial / 24 temporal "
                         "frames need a rank count that divides 8)")
    args = ap.parse_args()

    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))

    from pool_vae import PoolVAE
    from synthetic_dataset import SyntheticSpaTemDataset
    from diffuman4d_b200.config import SchedulerConfig, UNetConfig
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.sampler import B200SlidingIterativeSampler
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict

    cfg = UNetConfig.sd21()
    unet = B200MultiviewUNet(cfg, local).load_state_dict(random_state_dict(cfg, seed=1))
    pipe = B200Diffuman4DPipeline(unet, SchedulerConfig(), vae=PoolVAE())
    ds = SyntheticSpaTemDataset(args.cams, h=args.latent, w=args.latent)
    inputs = [1, 13, 25, 37] if args.cams >= 48 else sorted({(args.cams * k) // 4 + 1 for k in range(4)})
    driver = pipe
    if args.frame_sharded:
        if world == 1:   # one rank exchanging with itself
            import tempfile
            import torch.distributed as dist
            store = os.path.join(tempfile.mkdtemp(prefix="d4d-grid-"), "store")
            dist.init_process_group("gloo", init_method=f"file://{store}", rank=0, world_size=1)
        from diffuman4d_b200.sharded import FrameShardedPipeline
        driver = FrameShardedPipeline(pipe, max_frames=max(len(inputs) + 12, 24), h=args.latent, w=args.latent)
    sampler = B200SlidingIterativeSampler(ds, [driver], output_dir=None, spa_label_range=[0, args.cams, 1],
                                          tem_label_range=[0, args.frames, 1], input_spa_labels=inputs, window_size=12,
                                          sliding_stride=1, bidirectional=False, alternation_rounds=3, guidance_scale=2.0,
                                          prefetch=args.prefetch)

    # count window steps and their device time (CUDA events around every denoise_window call)
    stats = {"spatial": [0, 0.0], "temporal": [0, 0.0]}
    events = []
    inner = driver.denoise_window   # frame-sharded: the local frames of each window step

    def counted(**kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = inner(**kw)
        e1.record()
        events.append((kw["domain"], int(kw["latents"].shape[0]), e0, e1))
        return out

    driver.denoise_window = counted
    torch.cuda.synchronize()
    t0 = time.time()
    sampler.execute_tasks(rank, world, frame_sharded=args.frame_sharded)
    torch.cuda.synchronize()
    wall = time.time() - t0
    frames = {}
    for dom, f, e0, e1 in events:
        stats[dom][0] += 1
        stats[dom][1] += e0.elapsed_time(e1)
        frames.setdefault(dom, set()).add(f)
    ti = sampler.grid_timestep_indices.cpu()
    lat = sampler.grid_latents
    res = {
        "workload": f"demo_4d_tiny-shaped grid: {args.cams} cameras x {args.frames} frames @ {args.latent}x{args.latent} latents, "
                    "window 12 (+4 / +12 cond), stride 1, 3 alternation rounds, CFG 2.0, SD-2.1 UNet layout, random weights, "
                    "synthetic dataset, pooling stand-in for the VAE",
        "n_gpus": world, "rank": rank, "prefetch": bool(args.prefetch), "frame_sharded": bool(args.frame_sharded),
        "window_steps": {d: stats[d][0] for d in stats}, "frames_per_window": {d: sorted(frames.get(d, [])) for d in stats},
        "device_ms_in_denoise_window": {d: round(stats[d][1], 1) for d in stats},
        "ms_per_window_step": {d: round(stats[d][1] / max(1, stats[d][0]), 2) for d in stats},
        "wall_s_execute_tasks": round(wall, 2),
        "window_steps_per_s_wall": round(sum(stats[d][0] for d in stats) / wall, 2),
        "all_targets_fully_denoised": bool((ti.max() == ti[ti > 0].min()).item()) if (ti > 0).any() else False,
        "timestep_index_of_targets": int(ti.max()), "grid_finite": bool(torch.isfinite(lat.float()).all().item()),
    }
    if world > 1:
        import torch.distributed as dist
        allr = [None] * world
        dist.all_gather_object(allr, res)
        if rank == 0:
            # frame-sharded: every rank steps (its shard of) every window, so the windows are rank 0's
            steps = {d: (allr[0]["window_steps"][d] if args.frame_sharded else sum(r["window_steps"][d] for r in allr))
                     for d in stats}
            res = {"ranks": allr, "wall_s_execute_tasks": max(r["wall_s_execute_tasks"] for r in allr),
                   "window_steps_total": steps, "n_gpus": world, "frame_sharded": bool(args.frame_sharded),
                   "workload": res["workload"]}
            tot = sum(res["window_steps_total"].values())
            res["window_steps_per_s_wall"] = round(tot / res["wall_s_execute_tasks"], 2)
    if world > 1 or args.frame_sharded:
        import torch.distributed as dist
        dist.destroy_process_group()
    if rank == 0:
        if args.out:
            os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
            json.dump(res, open(args.out, "w"), indent=1)
        print(json.dumps(res))


if __name__ == "__main__":
    main()
