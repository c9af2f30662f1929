"""The UNet alone (seam B-2) on the CFG split and the CFG grid (``CFGSplitPipeline.unet_forward``, ``CFGGridPipeline``
and their ``.unet`` object) against ``pipe.unet`` on one GPU, bit for bit (``torch.equal``).

* One-rank loopback of the split and of the grid (world 1: the rank forwards both CFG halves into its own exchange
  buffer): the tiny UNet with the pose encoder on and off; the CFG batch [2F] with spatial, temporal and mixed domains,
  and the [F] batch without halves; per-image timesteps and a negative half whose skeletons are not constant.  Two
  consecutive calls each, through ``unet_forward`` and through ``.unet(...)``.
* The same handle alternating B-2 calls, CFG-split / grid window steps and plain forwards: every result equals its
  single-GPU counterpart, so the exchange epochs and buffer parities of the two paths agree.
* Two processes (split) and four processes (a 2x2 grid) on one GPU (gloo, the exchange buffers mapped across processes
  with cudaIpc): two B-2 calls with a window step between them; every rank's outputs equal rank 0's single-GPU results.
  The same runs on two and four GPUs are skipped below that many devices.
* Three steps of the reference's window loop (``oracle.pipeline_oracle.denoise_window_oracle``, the restatement of
  ``Diffuman4DPipeline.__call__``) with the loopback ``.unet`` as its UNet equal the same loop with ``pipe.unet``.
"""
import os

import pytest
import torch

from test_gpu_cfg_split import _cfg, _fields, _mid_task, gloo_world1  # noqa: F401  (gloo_world1 is a fixture)

F, H, W = 4, 16, 16
DOMAINS = [("spatial", "spatial"), ("temporal", "temporal"), ("spatial", "temporal")]


def _pipes(cfg, device=0, plain=True, modes=("split", "grid"), max_frames=F):
    """A plain pipeline (when ``plain``) and one CFGSplitPipeline / CFGGridPipeline per mode, each on its own handle."""
    from diffuman4d_b200.cfg_split import CFGGridPipeline, CFGSplitPipeline
    from diffuman4d_b200.config import SchedulerConfig
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict
    sd = random_state_dict(cfg, seed=1)
    new = lambda: B200Diffuman4DPipeline(B200MultiviewUNet(cfg, device).load_state_dict(sd), SchedulerConfig(),
                                         emulate_bf16_scheduler=True)
    cls = {"split": CFGSplitPipeline, "grid": CFGGridPipeline}
    return (new() if plain else None), {m: cls[m](new(), max_frames=max_frames, h=H, w=W) for m in modes}


def _batch(cfg, n_img, seed):
    """sample [n, Cin, H, W], per-image timesteps [n] and (pose encoder) per-image skeletons, all different."""
    g = torch.Generator().manual_seed(seed)
    sample = torch.randn(n_img, cfg.in_channels, H, W, generator=g).to(torch.bfloat16).cuda()
    t = torch.randint(0, 1000, (n_img,), generator=g).cuda()
    skel = ((torch.rand(n_img, 3, 8 * H, 8 * W, generator=g) * 2 - 1).to(torch.bfloat16).cuda()
            if cfg.enable_pose_encoder else None)
    return sample, t, skel


def _b2_calls(cfg):
    """(domains, num_frames, inputs) of the B-2 calls each mode is checked on: the CFG batch, then the [F] batch."""
    calls = [(list(d), F, _batch(cfg, 2 * F, seed=10 + i)) for i, d in enumerate(DOMAINS)]
    calls += [([d], F, _batch(cfg, F, seed=20 + i)) for i, d in enumerate(("spatial", "temporal"))]
    return calls


@pytest.mark.gpu
@pytest.mark.parametrize("pose", [True, False], ids=["pose", "skeleton-latents"])
def test_loopback_unet_is_bit_identical(cuda, gloo_world1, pose):
    cfg = _cfg(pose)
    plain, modes = _pipes(cfg)
    for doms, nf, (x, t, s) in _b2_calls(cfg):
        ref = plain.unet(x, t, s, doms, nf, return_dict=False)[0]
        assert ref.shape == (len(doms) * nf, cfg.out_channels, H, W)
        for name, sp in modes.items():
            for k in range(2):   # two consecutive calls: the second reads the other buffer parity
                got = (sp.unet_forward(x, t, s, doms, nf) if k == 0 else
                       sp.unet(x, timestep=t, skeletons=s, domains=doms, num_frames=nf, return_dict=False)[0])
                assert got.data_ptr() != ref.data_ptr()
                assert torch.equal(got, ref), f"{name} {doms} call {k}: the noise differs from the single-GPU forward"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["split", "grid"])
def test_b2_calls_interleaved_with_window_steps(cuda, gloo_world1, mode):
    """On one handle: B-2 call, window step, plain forward, B-2 call, window step, B-2 call."""
    cfg = _cfg()
    plain, modes = _pipes(cfg, modes=(mode,))
    sp = modes[mode]
    kw = dict(domain="temporal", guidance_scale=2.0)
    lat, ti, state, conds = _mid_task(plain, cfg, kw)
    sp.pipe.parepare_schedulers(18, F)
    calls = _b2_calls(cfg)
    win_ref = []
    l_, t_ = lat.clone(), ti.clone()
    for _ in range(2):
        plain.denoise_window(latents=l_, timestep_indices=t_, num_inference_steps=1, **conds, **kw)
        win_ref.append((l_.clone(), t_.clone()))
    l_, t_ = lat.clone(), ti.clone()
    step = 0
    for i, op in enumerate(["b2", "window", "plain", "b2", "window", "b2"]):
        doms, nf, (x, t, s) = calls[i % len(calls)]
        if op == "window":
            sp.denoise_window(latents=l_, timestep_indices=t_, num_inference_steps=1, **conds, **kw)
            assert torch.equal(l_, win_ref[step][0]) and torch.equal(t_, win_ref[step][1]), f"{mode} window {step}"
            step += 1
            continue
        ref = plain.unet(x, t, s, doms, nf, return_dict=False)[0]
        got = sp.unet_forward(x, t, s, doms, nf) if op == "b2" else sp.pipe.unet(x, t, s, doms, nf, return_dict=False)[0]
        assert torch.equal(got, ref), f"{mode} op {i} ({op}, {doms}) differs from the single-GPU forward"


# ------------------------------------------------------------------------------------------------ several processes
def _worker(rank, world, store, out_dir, devices, mode):
    import torch.distributed as dist
    dev = devices[rank]
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=world)
    try:
        cfg = _cfg()
        _, modes = _pipes(cfg, device=dev, plain=False, modes=(mode,))
        sp = modes[mode]
        out = {}
        kw = dict(domain="spatial", guidance_scale=2.0)
        lat, ti, state, conds = _mid_task(sp.pipe, cfg, kw)   # plain steps on this rank's handle
        sp.pipe.parepare_schedulers(18, F)
        calls = [(["spatial", "spatial"], F, _batch(cfg, 2 * F, seed=30)),
                 (["temporal", "temporal"], F, _batch(cfg, 2 * F, seed=31)),
                 (["temporal"], F, _batch(cfg, F, seed=32))]
        for i, (op, c) in enumerate([("b2", 0), ("window", None), ("b2", 1), ("b2", 2)]):
            if op == "window":
                runs = [(mode, sp.denoise_window)] + ([("ref", sp.pipe.denoise_window)] if rank == 0 else [])
                for name, run in runs:
                    l_, t_ = lat.clone(), ti.clone()
                    run(latents=l_, timestep_indices=t_, num_inference_steps=2, **conds, **kw)
                    out[(name, i)] = {k: v.cpu() for k, v in _fields(l_, t_, None).items()}
                continue
            doms, nf, (x, t, s) = calls[c]
            out[(mode, i)] = {"noise": sp.unet(x, t, s, doms, nf).sample.cpu()}
            if rank == 0:
                out[("ref", i)] = {"noise": sp.pipe.unet(x, t, s, doms, nf).sample.cpu()}
        torch.save(out, os.path.join(out_dir, f"rank{rank}.pt"))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _run_ranks(tmp_path, devices, mode):
    from test_gpu_cfg_grid import _spawn
    world = len(devices)
    got = _spawn(tmp_path, _worker, world, devices, mode)
    keys = [k for k in got[0] if k[0] == "ref"]
    assert len(keys) == 4
    for key in keys:
        ref = got[0][key]
        for r in range(world):
            res = got[r][(mode, key[1])]
            assert res.keys() == ref.keys()
            for k in ref:
                assert torch.equal(res[k], ref[k]), f"{mode} op {key[1]} rank {r} of {world}: {k} differs"


@pytest.mark.gpu
def test_two_processes_on_one_gpu_split(cuda, tmp_path):
    _run_ranks(tmp_path, [0, 0], "split")


@pytest.mark.gpu
def test_four_processes_on_one_gpu_grid(cuda, tmp_path):
    _run_ranks(tmp_path, [0] * 4, "grid")


@pytest.mark.gpu
@pytest.mark.parametrize("mode,world", [("split", 2), ("grid", 4)])
def test_on_gpus(cuda, tmp_path, mode, world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    _run_ranks(tmp_path, list(range(world)), mode)


# ------------------------------------------------------------------------------------------------ the Python loop
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["split", "grid"])
def test_reference_loop_with_the_loopback_unet(cuda, gloo_world1, mode):
    from diffuman4d_b200.config import SchedulerConfig
    from oracle.pipeline_oracle import DDIMOracle, denoise_window_oracle
    cfg = _cfg()
    plain, modes = _pipes(cfg, modes=(mode,))
    g = torch.Generator().manual_seed(7)
    lat, pix, plk = (torch.randn(F, c, H, W, generator=g) for c in (4, 4, 6))
    skel = torch.rand(F, 3, 8 * H, 8 * W, generator=g) * 2 - 1
    mask = torch.ones(F, 1, H, W)
    mask[1] = 0
    ti = torch.tensor([0, 0, 2, 1])
    results = []
    for unet in (plain.unet, modes[mode].unet):
        sched = DDIMOracle(SchedulerConfig())
        sched.set_timesteps(18)

        def call(x, t, s, doms, nf, unet=unet):
            return unet(x, timestep=t, skeletons=s, domains=doms, num_frames=nf, return_dict=False)[0].float().cpu()
        results.append(denoise_window_oracle(call, sched, latents=lat.clone(), pixel_latents=pix, plucker=plk,
                                             skeletons=skel, cond_mask=mask, timestep_indices=ti, domain="spatial",
                                             guidance_scale=2.0, num_inference_steps=3))
    (ref_lat, ref_ti), (got_lat, got_ti) = results
    assert not torch.equal(ref_lat, lat)
    assert torch.equal(got_ti, ref_ti)
    assert torch.equal(got_lat, ref_lat), f"{mode}: the loop's latents differ from the loop with the single-GPU UNet"
