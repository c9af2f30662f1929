"""2-GPU test of the frame-sharded window (skipped on single-GPU boxes): the sharded UNet forward / window step on
every rank's frames must be BIT-IDENTICAL to the single-GPU call on the gathered window (all non-attention work is per
image; attention sees the same K/V tiles in the same order)."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, q, n3d=3):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from diffuman4d_b200.config import SchedulerConfig, UNetConfig
        from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
        from diffuman4d_b200.sharded import FrameShardedPipeline
        from diffuman4d_b200.unet import B200MultiviewUNet
        from diffuman4d_b200.weights import random_state_dict
        cfg = UNetConfig.tiny(num_3d_attn_blocks=n3d)
        sd = random_state_dict(cfg, seed=1)
        F, h, w = 4, 16, 16
        g = torch.Generator().manual_seed(0)
        x = torch.randn(2 * F, cfg.in_channels, h, w, generator=g).to(torch.bfloat16)
        t = torch.randint(0, 1000, (2 * F,), generator=g)
        sk = (torch.rand(2 * F, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16)
        lat, pix, plk = (torch.randn(F, c, h, w, generator=g).to(torch.bfloat16) for c in (4, 4, 6))
        skel = (torch.rand(F, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16)
        mask = torch.ones(F, 1, h, w, dtype=torch.bfloat16)
        mask[0] = 0
        ti = torch.tensor([0, 3, 2, 1])

        unet = B200MultiviewUNet(cfg, rank).load_state_dict(sd)
        pipe = B200Diffuman4DPipeline(unet, SchedulerConfig(), emulate_bf16_scheduler=True)
        pipe.parepare_schedulers(18, F)
        sh = FrameShardedPipeline(pipe, max_frames=F, h=h, w=w)
        lo, hi = sh.frames(F)
        idx = torch.cat([torch.arange(lo, hi), torch.arange(lo, hi) + F])   # my frames of both CFG halves
        res = {}
        for dom in ("spatial", "temporal"):
            y = sh.unet_forward(x[idx].cuda().contiguous(), t[idx].cuda().contiguous(), sk[idx].cuda().contiguous(),
                                [dom, dom], hi - lo, F)
            l_d, t_d = lat[lo:hi].clone().cuda(), ti[lo:hi].clone().cuda()
            for _ in range(2):
                sh.denoise_window(latents=l_d, pixel_values_latents=pix[lo:hi].cuda().contiguous(),
                                  plucker_embeds_latents=plk[lo:hi].cuda().contiguous(),
                                  skeletons_latents=skel[lo:hi].cuda().contiguous(),
                                  cond_masks_latents=mask[lo:hi].cuda().contiguous(), timestep_indices=t_d, domain=dom,
                                  guidance_scale=2.0, F_total=F)
            torch.cuda.synchronize()
            res[dom] = (y.cpu(), l_d.cpu(), t_d.cpu())
        if rank == 0:   # single-GPU reference on the gathered window (fresh handle, no exchange)
            ref_unet = B200MultiviewUNet(cfg, 0).load_state_dict(sd)
            ref_pipe = B200Diffuman4DPipeline(ref_unet, SchedulerConfig(), emulate_bf16_scheduler=True)
            ref_pipe.parepare_schedulers(18, F)
            ref = {}
            for dom in ("spatial", "temporal"):
                y = ref_unet(x.cuda(), t.cuda(), sk.cuda(), [dom, dom], F, return_dict=False)[0]
                l_d, t_d = lat.clone().cuda(), ti.clone().cuda()
                for _ in range(2):
                    ref_pipe.denoise_window(latents=l_d, pixel_values_latents=pix, plucker_embeds_latents=plk,
                                            skeletons_latents=skel, cond_masks_latents=mask, timestep_indices=t_d, domain=dom,
                                            guidance_scale=2.0)
                torch.cuda.synchronize()
                ref[dom] = (y.cpu(), l_d.cpu(), t_d.cpu())
            q.put(("ref", {k: tuple(v.float().tolist() if v.is_floating_point() else v.tolist() for v in vs) for k, vs in ref.items()}))
        q.put((rank, (lo, hi), {k: tuple(v.float().tolist() if v.is_floating_point() else v.tolist() for v in vs) for k, vs in res.items()}))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _run_two_ranks(n3d):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29600 + (os.getpid() % 1000) + 7 * n3d
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q, n3d)) for r in range(2)]
    for p in procs:
        p.start()
    items = [q.get(timeout=600) for _ in range(3)]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    ref = next(i[1] for i in items if i[0] == "ref")
    F = 4
    for it in items:
        if it[0] == "ref":
            continue
        _, (lo, hi), res = it
        for dom in ("spatial", "temporal"):
            y, lat, ti = (torch.tensor(v) for v in res[dom])
            ry, rlat, rti = (torch.tensor(v) for v in ref[dom])
            idx = torch.cat([torch.arange(lo, hi), torch.arange(lo, hi) + F])
            assert torch.equal(y, ry[idx]), f"UNet output differs on frames {lo}:{hi} ({dom}): {(y - ry[idx]).abs().max()}"
            assert torch.equal(lat, rlat[lo:hi]) and torch.equal(ti, rti[lo:hi])


def test_two_rank_frame_sharded_window_is_bit_identical(cuda):
    _run_two_ranks(3)


def test_two_rank_frame_sharded_window_with_level0_3d_attention(cuda):
    """num_3d_attn_blocks = 4: down_blocks.0 and up_blocks.3 exchange full-resolution K/V, the largest layer of the
    window (sharded.exchange_bytes)."""
    _run_two_ranks(4)
