"""Whole tasks on the frame-sharded window (DESIGN.md section 7), on one GPU and, when there are two, on two.

* ``d4d_op_window_scatter`` (the store kernel of the window-result exchange) for every rank of R = 2, 3, 4 and 8, with
  and without DPM-Solver++ state, 1-3 local frames and two latent sizes: every destination holds the source frames at
  the rank's rows bit for bit; the other ranks' rows and a guard band behind the window stay untouched.  Its argument
  rejections return 1 with nothing written.
* One-rank loopback (``d4d_exchange_open`` with rank 0 of world 1 on the handle's own buffers), with plain forwards
  interleaved on the same handle so the epoch accounting of the exchanges carries across them:
  - the DPM-Solver++ window on a shard equals ``denoise_window`` with DPM-Solver++ bit for bit (order 1 and 2, epsilon and
    v, CFG on and off, fp32 and bf16-emulating);
  - ``FrameShardedPipeline.sliding_iterative_denoise`` equals the plain loop over a spatial and a bidirectional temporal
    task (DDIM and DPM-Solver++, pose encoder on and off, 1 and 2 denoising steps per window): latents, timestep indices,
    ``fully_denoised`` and the solver state;
  - ``execute_tasks(frame_sharded=True)`` gives the default mode's grid.
* Two ranks on two GPUs (skipped below two devices): the sliding loop is bit-identical to the single-GPU loop.

A loopback always stores at row 0; ranks above 0 are covered by the op test here and by the gloo test of the host loop
(test_sharded_sampling.py), and through real peer memory only by the two-GPU case.
"""
import ctypes as C
import os
import sys

import pytest
import torch

from diffuman4d_b200.config import DPMSolverConfig, SchedulerConfig, UNetConfig

SENT = 0xA5
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _layout(buf, F_total, h, w, dpm):
    """Views of a gathered window in a uint8 buffer (include/d4d.h, d4d_op_window_scatter)."""
    rows = F_total * 4 * h * w * 2
    lat = buf[:rows].view(torch.bfloat16).view(F_total, 4, h, w)
    off = rows
    x0 = None
    if dpm:
        x0 = buf[off:off + rows].view(torch.bfloat16).view(F_total, 4, h, w)
        off += rows
    ts = buf[off:off + 8 * F_total].view(torch.int64)
    off += 8 * F_total
    lon = None
    if dpm:
        lon = buf[off:off + 4 * F_total].view(torch.int32)
        off += 4 * F_total
    return lat, x0, ts, lon, off


def _frames(F, h, w, dpm, seed):
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(F, 4, h, w, generator=g).to(torch.bfloat16).cuda()
    ts = torch.randint(0, 1 << 40, (F,), generator=g).cuda()
    x0 = torch.randn(F, 4, h, w, generator=g).to(torch.bfloat16).cuda() if dpm else None
    lon = torch.randint(0, 3, (F,), generator=g, dtype=torch.int32).cuda() if dpm else None
    return lat, ts, x0, lon


def _ptr(t):
    """A device address: a tensor's, or a plain integer (the dummy operands of the rejection test)."""
    return t if t is None or isinstance(t, int) else t.data_ptr()


def _scatter(lib, lat, ts, x0, lon, F_local, F_total, h, w, world, rank, ptrs, nbytes):
    arr = (C.c_void_p * max(1, len(ptrs)))(*ptrs)
    return lib.d4d_op_window_scatter(_ptr(lat), _ptr(ts), _ptr(x0), _ptr(lon), F_local, F_total, h, w, world, rank, arr,
                                     nbytes, torch.cuda.current_stream().cuda_stream if torch.cuda.is_available() else None)


@pytest.fixture(scope="module")
def libd4d():
    from diffuman4d_b200 import build
    build.build(verbose=False)
    from diffuman4d_b200._lib import lib
    return lib()


# ------------------------------------------------------------------------------------------------ the store kernel
@pytest.mark.gpu
@pytest.mark.parametrize("hw", [(8, 8), (16, 24)], ids=["8x8", "16x24"])
@pytest.mark.parametrize("dpm", [False, True], ids=["ddim", "dpm"])
@pytest.mark.parametrize("R", [2, 3, 4, 8])
def test_window_scatter_every_rank(cuda, libd4d, R, dpm, hw):
    from diffuman4d_b200._lib import check
    from diffuman4d_b200.sharded import window_result_bytes
    h, w = hw
    guard = 4096
    for F_local in (1, 2, 3):
        F_total = F_local * R
        need = window_result_bytes(F_total, h, w, dpm)
        dst = [torch.full((need + guard,), SENT, dtype=torch.uint8, device="cuda") for _ in range(R)]
        expect = torch.full_like(dst[0], SENT)
        e_lat, e_x0, e_ts, e_lon, end = _layout(expect, F_total, h, w, dpm)
        assert end == need
        for r in range(R):
            lat, ts, x0, lon = _frames(F_local, h, w, dpm, seed=31 * r + F_local)
            check(_scatter(libd4d, lat, ts, x0, lon, F_local, F_total, h, w, R, r, [t.data_ptr() for t in dst], need),
                  "d4d_op_window_scatter")
            torch.cuda.synchronize()
            rows = slice(r * F_local, (r + 1) * F_local)
            e_lat[rows], e_ts[rows] = lat, ts
            if dpm:
                e_x0[rows], e_lon[rows] = x0, lon
            what = f"R {R} rank {r} F_local {F_local} {'dpm' if dpm else 'ddim'} {h}x{w}"
            for k, t in enumerate(dst):
                assert torch.equal(t, expect), f"{what}: destination {k} differs (other ranks' rows or the guard band)"
        assert not (expect[:need] == SENT).all()


# (id, argument overrides, message).  Base: R = 2, rank 1, F_local 2, F_total 4, 8x8, DPM state, buffers of the exact size.
REJECT = [
    ("world-0", dict(world=0), "world"),
    ("world-9", dict(world=9), "world"),
    ("rank-equals-world", dict(rank=2), "rank"),
    ("negative-rank", dict(rank=-1), "rank"),
    ("F_total-not-world-x-F_local", dict(F_total=5), "F_total must equal"),
    ("F_local-0", dict(F_local=0, F_total=0), "F_total must equal"),
    ("result-larger-than-buffer", dict(short=1), "does not fit"),
    ("ddim-result-larger-than-buffer", dict(dpm=False, short=1), "does not fit"),
    ("x0-without-lower_order_nums", dict(no_lon=1), "together"),
    ("null-destination", dict(null_dst=1), "null destination"),
]


@pytest.mark.parametrize("case,over,match", REJECT, ids=[c[0] for c in REJECT])
def test_window_scatter_rejections(libd4d, case, over, match):
    """Argument errors (status 1, ValueError) before any launch.  Without a GPU the operands are dummy addresses, so a
    call that is not rejected fails with a CUDA error instead; on a GPU they are real buffers, checked unwritten after
    the call, and the null destination is only tried without one."""
    from diffuman4d_b200._lib import check
    from diffuman4d_b200.sharded import window_result_bytes
    a = dict(world=2, rank=1, F_local=2, F_total=4, dpm=True, short=0, no_lon=0, null_dst=0)
    a.update(over)
    h = w = 8
    on_gpu = torch.cuda.is_available()
    if on_gpu and a["null_dst"]:
        pytest.skip("a null destination is only passed where no kernel can run")
    nbytes = window_result_bytes(4, h, w, a["dpm"]) - a["short"]
    if on_gpu:
        lat, ts, x0, lon = _frames(2, h, w, a["dpm"], seed=1)
        dst = [torch.full((window_result_bytes(4, h, w, True) + 4096,), SENT, dtype=torch.uint8, device="cuda")
               for _ in range(9)]
        ptrs = [t.data_ptr() for t in dst]
        src = [lat, ts, x0, lon]
    else:
        src = [0x100000, 0x200000, 0x300000 if a["dpm"] else None, 0x400000 if a["dpm"] else None]
        ptrs = [0x1000000 * (r + 1) for r in range(9)]
    if a["no_lon"]:
        src[3] = None
    if a["null_dst"]:
        ptrs[1] = None
    with pytest.raises(ValueError, match=match):
        check(_scatter(libd4d, *src, a["F_local"], a["F_total"], h, w, a["world"], a["rank"], ptrs[:max(1, min(a["world"], 9))],
                       nbytes), "d4d_op_window_scatter")
    if on_gpu:
        torch.cuda.synchronize()
        assert all(bool((t == SENT).all()) for t in dst), "a rejected scatter wrote"


# ------------------------------------------------------------------------------------------------ one-rank loopback
@pytest.fixture
def gloo_world1(tmp_path):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"file://{tmp_path / 'store'}", rank=0, world_size=1)
    try:
        yield
    finally:
        dist.destroy_process_group()


def _cfg(pose=True):
    return UNetConfig.tiny() if pose else UNetConfig.tiny(enable_pose_encoder=False, in_channels=15)


def _pipes(cfg, sched, max_frames, h, w, emulate=True, vae=None):
    """A plain pipeline and a loopback FrameShardedPipeline (world 1) with the same weights."""
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.sharded import FrameShardedPipeline
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict
    sd = random_state_dict(cfg, seed=1)
    pipes = [B200Diffuman4DPipeline(B200MultiviewUNet(cfg, 0).load_state_dict(sd), sched, vae=vae,
                                    emulate_bf16_scheduler=emulate) for _ in range(2)]
    sh = FrameShardedPipeline(pipes[1], max_frames=max_frames, h=h, w=w)
    assert sh.world == 1 and sh.rank == 0
    return pipes[0], sh


def _plain_forward(pipe, h, w, seed=9):
    """A plain forward on the loopback handle between sharded calls (it must not disturb the exchange epochs)."""
    cfg = pipe.unet.config
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(4, cfg.in_channels, h, w, generator=g).to(torch.bfloat16).cuda()
    t = torch.randint(0, 1000, (4,), generator=g).cuda()
    sk = (torch.rand(4, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16).cuda() if cfg.enable_pose_encoder else None
    return pipe.unet(x, t, sk, ["temporal"] * 2, 2, return_dict=False)[0]


def _window_inputs(cfg, F, h, w, seed=3):
    g = torch.Generator().manual_seed(seed)
    lat, pix, plk = (torch.randn(F, c, h, w, generator=g).to(torch.bfloat16).cuda() for c in (4, 4, 6))
    skel = ((torch.rand(F, 3, 8 * h, 8 * w, generator=g) * 2 - 1) if cfg.enable_pose_encoder
            else torch.randn(F, 4, h, w, generator=g)).to(torch.bfloat16).cuda()
    mask = torch.ones(F, 1, h, w, dtype=torch.bfloat16, device="cuda")
    mask[1] = 0
    x0 = torch.randn(F, 4, h, w, generator=g).to(torch.bfloat16).cuda()
    return lat, pix, plk, skel, mask, x0


@pytest.mark.gpu
@pytest.mark.parametrize("pred", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("order", [1, 2])
def test_loopback_dpm_window_is_bit_identical(cuda, gloo_world1, order, pred):
    """Three DPM-Solver++ window steps from a mid-task state (per-frame step indices and order counts differ), CFG on
    and off, fp32 and bf16-emulating, both domains; plain forwards on the loopback handle in between."""
    from diffuman4d_b200.scheduler import DPMSolverState
    cfg = _cfg()
    F, h, w = 4, 16, 16
    plain, sh = _pipes(cfg, DPMSolverConfig(solver_order=order, prediction_type=pred), F, h, w)
    lat, pix, plk, skel, mask, x0 = _window_inputs(cfg, F, h, w)
    ti = torch.tensor([0, 5, 2, 1], device="cuda")
    lon = torch.tensor([0, 2, 1, 1], dtype=torch.int32, device="cuda")
    for pipe in (plain, sh.pipe):
        pipe.parepare_schedulers(18, F)
    fwd_ref = _plain_forward(plain, h, w)
    for emulate in (True, False):
        for gs in (2.0, 1.0):
            for dom in ("spatial", "temporal"):
                kw = dict(pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skel,
                          cond_masks_latents=mask, domain=dom, guidance_scale=gs, num_inference_steps=3)
                plain.emulate_bf16_scheduler = sh.pipe.emulate_bf16_scheduler = emulate
                res = []
                for run in (plain.denoise_window, lambda **k: sh.denoise_window(F_total=F, **k)):
                    l_, t_, st = lat.clone(), ti.clone(), DPMSolverState(F, "cuda", x0.clone(), lon.clone())
                    run(latents=l_, timestep_indices=t_, solver_state=st, **kw)
                    res.append((l_, t_, st.x0_prev, st.lower_order_nums))
                what = f"emulate {emulate} guidance {gs} {dom}"
                for name, a, b in zip(("latents", "timestep_indices", "x0_prev", "lower_order_nums"), *res):
                    assert torch.equal(a, b), f"{what}: {name} differ"
                assert not torch.equal(res[0][0], lat)
                assert torch.equal(_plain_forward(sh.pipe, h, w), fwd_ref), f"{what}: plain forward on the loopback handle"


def _capture_state(pipe):
    box = []
    inner = pipe.parepare_schedulers

    def wrapped(n, F):
        s, ts = inner(n, F)
        box.append(s[0].state if pipe._multistep else None)
        return s, ts
    pipe.parepare_schedulers = wrapped
    return box


def _task(cfg, domain, n_in, n_tg, h, w, seed):
    n = n_in + n_tg
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    mask = torch.ones(n, 1, 8 * h, 8 * w)
    mask[:n_in] = 0
    skel = ((torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16) if cfg.enable_pose_encoder
            else r(n, 4, h, w))
    return dict(pixel_values_latents=r(n, 4, h, w), plucker_embeds=r(n, 6, 8 * h, 8 * w), skeletons_latents=skel,
                cond_masks=mask, latents=r(n, 4, h, w), domain=domain, timestep_indices=torch.zeros(n, dtype=torch.long))


# (domain, inputs, targets, window, stride, bidirectional, alternation rounds)
LOOP_TASKS = [("spatial", 2, 4, 2, 1, False, 2), ("temporal", 3, 3, 2, 1, True, 1)]


def _compare_loops(plain, sh, cfg, h, w, steps, what):
    bp, bs = _capture_state(plain), _capture_state(sh.pipe)
    for k, (domain, n_in, n_tg, ws, stride, bidir, rounds) in enumerate(LOOP_TASKS):
        kw = dict(_task(cfg, domain, n_in, n_tg, h, w, seed=20 + k), window_size=ws, sliding_stride=stride,
                  bidirectional=bidir, num_denoising_steps=steps, alternation_rounds=rounds, guidance_scale=2.0)
        ref = plain.sliding_iterative_denoise(**kw)
        got = sh.sliding_iterative_denoise(**kw)
        torch.cuda.synchronize()
        tag = f"{what} {domain} steps {steps}"
        assert ref["timestep_indices"].max() > 0
        for key in ("latents", "timestep_indices", "fully_denoised"):
            assert torch.equal(got[key], ref[key]), f"{tag}: {key} differ"
        if bp[-1] is not None:
            assert torch.equal(bs[-1].x0_prev, bp[-1].x0_prev), f"{tag}: x0_prev differs"
            assert torch.equal(bs[-1].lower_order_nums, bp[-1].lower_order_nums), f"{tag}: lower_order_nums differ"
        # the plain loop on the loopback handle, between sharded loops
        again = sh.pipe.sliding_iterative_denoise(**kw)
        assert torch.equal(again["latents"], ref["latents"]), f"{tag}: plain loop on the loopback handle"


@pytest.mark.gpu
@pytest.mark.parametrize("pose", [True, False], ids=["pose", "skeleton-latents"])
@pytest.mark.parametrize("sched", ["ddim", "dpm"])
def test_loopback_sliding_loop_is_bit_identical(cuda, gloo_world1, sched, pose):
    cfg = _cfg(pose)
    h = w = 8
    sc = DPMSolverConfig(final_sigmas_type="sigma_min", lower_order_final=False) if sched == "dpm" else SchedulerConfig()
    plain, sh = _pipes(cfg, sc, 6, h, w)
    for steps in (1, 2):
        _compare_loops(plain, sh, cfg, h, w, steps, f"{sched} pose {pose}")


@pytest.mark.gpu
def test_loopback_execute_tasks_frame_sharded(cuda, gloo_world1):
    """Three alternation rounds of the sampler: frame_sharded=True on the loopback pipeline gives the default mode's grid
    (fresh targets draw their noise from the device's default generator, reseeded before each run)."""
    sys.path.insert(0, GOLD)
    from pool_vae import PoolVAE
    from synthetic_dataset import SyntheticSpaTemDataset
    from diffuman4d_b200.sampler import B200SlidingIterativeSampler
    plain, sh = _pipes(_cfg(), SchedulerConfig(), 6, 16, 16, emulate=False, vae=PoolVAE())
    grids = []
    for pipe, fs in ((plain, False), (sh, True)):
        saved = []
        s = B200SlidingIterativeSampler(SyntheticSpaTemDataset(8, h=16, w=16), [pipe], output_dir=None,
                                        spa_label_range=[0, 6, 1], tem_label_range=[0, 4, 1], input_spa_labels=[1, 4],
                                        window_size=2, sliding_stride=1, bidirectional=True, alternation_rounds=3,
                                        guidance_scale=2.0, save_fn=lambda smp, d: saved.append(smp["domain_label"]))
        torch.cuda.manual_seed(1234)
        s.execute_tasks(frame_sharded=fs)
        torch.cuda.synchronize()
        grids.append((s.grid_latents.clone(), s.grid_timestep_indices.clone(), saved))
        _plain_forward(sh.pipe, 16, 16)
    assert grids[0][1].max() > 0
    assert torch.equal(grids[1][1], grids[0][1]), "timestep index grids differ"
    assert torch.equal(grids[1][0], grids[0][0]), "latent grids differ"
    assert grids[1][2] == grids[0][2], "rank 0 saves every task, in order"


# ------------------------------------------------------------------------------------------------ two GPUs
def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
        from diffuman4d_b200.sharded import FrameShardedPipeline
        from diffuman4d_b200.unet import B200MultiviewUNet
        from diffuman4d_b200.weights import random_state_dict
        cfg = _cfg()
        h = w = 8
        sd = random_state_dict(cfg, seed=1)
        out = {}
        for sched in ("ddim", "dpm"):
            sc = DPMSolverConfig(final_sigmas_type="sigma_min", lower_order_final=False) if sched == "dpm" else SchedulerConfig()
            pipe = B200Diffuman4DPipeline(B200MultiviewUNet(cfg, rank).load_state_dict(sd), sc, emulate_bf16_scheduler=True)
            sh = FrameShardedPipeline(pipe, max_frames=6, h=h, w=w)
            ref_pipe = None
            if rank == 0:
                ref_pipe = B200Diffuman4DPipeline(B200MultiviewUNet(cfg, 0).load_state_dict(sd), sc,
                                                  emulate_bf16_scheduler=True)
            # windows of 4 frames: spatial 2 inputs + 2 targets, temporal 2 + 2 (bidirectional)
            for k, (domain, n_in, n_tg, bidir) in enumerate((("spatial", 2, 4, False), ("temporal", 4, 4, True))):
                kw = dict(_task(cfg, domain, n_in, n_tg, h, w, seed=40 + k), window_size=2, sliding_stride=1,
                          bidirectional=bidir, num_denoising_steps=1, alternation_rounds=1, guidance_scale=2.0)
                kw["latents"] = None   # rank 0's initial noise must reach rank 1
                res = sh.sliding_iterative_denoise(**kw, generator=torch.Generator(device="cuda").manual_seed(7 + rank))
                torch.cuda.synchronize()
                out[(sched, domain)] = [res["latents"].cpu().view(torch.int16), res["timestep_indices"].cpu()]
                if rank == 0:
                    ref = ref_pipe.sliding_iterative_denoise(**kw, generator=torch.Generator(device="cuda").manual_seed(7))
                    torch.cuda.synchronize()
                    out[("ref", sched, domain)] = [ref["latents"].cpu().view(torch.int16), ref["timestep_indices"].cpu()]
        q.put((rank, {k: [t.tolist() for t in v] for k, v in out.items()}))
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_two_rank_sliding_loop_is_bit_identical(cuda):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + (os.getpid() % 1000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    items = dict(q.get(timeout=600) for _ in range(2))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    for sched in ("ddim", "dpm"):
        for domain in ("spatial", "temporal"):
            ref = items[0][("ref", sched, domain)]
            for r in (0, 1):
                assert items[r][(sched, domain)] == ref, f"rank {r} {sched} {domain}: differs from the single-GPU loop"
