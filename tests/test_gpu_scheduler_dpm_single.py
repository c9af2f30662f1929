"""GPU tests of the DPM-Solver++ singlestep step (upstream DPMSolverSinglestepScheduler, dpmsolver++ / midpoint, orders 1 to
3): the fused CFG + step kernel against DPMSingleOracle on the same bf16 inputs with frames at every row order and order
count in one launch, some of them below their row's order (bit for bit when emulating bf16, against fp64 arithmetic in
the fp32 mode), the window step through the C ABI and the sliding loop against the oracle driven by the same CUDA UNet,
``__call__`` with the per-frame handles, load_pipelines on a checkpoint that names the scheduler, and the device
sampler."""
import copy
import json
import os
import sys

import pytest
import torch

from diffuman4d_b200.config import DPMSingleConfig, UNetConfig
from diffuman4d_b200.weights import random_state_dict

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def _oracle_frame(cfg, n, idx, lon, x0_prev, x0_prev2, cur_sample):
    """A per-frame oracle scheduler standing where the frame's own copy stands at step index ``idx`` after taking
    ``lon`` steps (capped at solver_order), its history read from the state planes: the data predictions it holds
    (None where the frame has not taken that many steps) and the sample of its block's first step."""
    from oracle.dpm_single_oracle import DPMSingleOracle
    s = DPMSingleOracle(cfg)
    s.set_timesteps(n)
    s.step_index = idx
    held = [x0_prev2 if lon >= 2 else None, x0_prev if lon >= 1 else None]
    s.model_outputs = ([None] + held)[-cfg.solver_order:]
    s.sample = cur_sample
    return s


# (timestep index, order count) per frame for a 10-step table with a zero final sigma; at order 3 the rows have orders
# 1 2 3 1 2 3 1 2 3 1 and at order 2 orders 1 2 1 2 1 2 1 2 1 1; frame 7 is a conditioning frame.  Frames 3, 4 and 10
# stand on rows above their order count + 1 (upstream's order reduction).
FRAMES = [(0, 0), (1, 1), (2, 2), (2, 1), (5, 0), (8, 3), (9, 3), (3, 2), (4, 3), (7, 1), (6, 2)]


@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("pred", ["epsilon", "v_prediction", "sample"])
@pytest.mark.parametrize("cfg_on", [True, False])
def test_cfg_dpm_single_step_vs_oracle(cuda, order, pred, cfg_on):
    from diffuman4d_b200.ops import cfg_dpm_single_step
    from diffuman4d_b200.scheduler import DPMSingleTables
    n = 10
    cfg = DPMSingleConfig(solver_order=order, prediction_type=pred)
    F, h, w = len(FRAMES), 9, 13                                          # 4*h*w = 468: no multiple of the block size
    g = torch.Generator().manual_seed(51)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    noise, lat = r((2 if cfg_on else 1) * F, 4, h, w), r(F, 4, h, w)
    m1, m2, cur = r(F, 4, h, w), r(F, 4, h, w), r(F, 4, h, w)
    lat[0] *= 60   # a high-noise frame at step 0
    mask = torch.ones(F, 1, h, w, dtype=torch.bfloat16)
    mask[7] = 0
    ti = torch.tensor([f[0] for f in FRAMES])
    lon = torch.tensor([min(f[1], order) for f in FRAMES], dtype=torch.int32)
    tables = DPMSingleTables(cfg, device="cuda:0")
    tables.set_timesteps(n)
    guidance = 2.0 if cfg_on else 1.0
    orders = set()
    for emulate in (True, False):
        dt = torch.bfloat16 if emulate else torch.float64   # fp32 mode: against fp64 arithmetic on fp32 tables
        if cfg_on:
            u, c = noise.to(dt).chunk(2)
            eps = u + 2.0 * (c - u)          # 2.0 and the differences are exact roundings in either dtype
        else:
            eps = noise.to(dt)
        ref, ref_m1, ref_m2, ref_cur = [], m1.to(dt).clone(), m1.to(dt).clone(), cur.to(dt).clone()
        for j in range(F):
            if mask[j, 0, 0, 0] == 0:
                ref.append(lat[j:j + 1].to(dt))
                ref_m2[j] = m2[j].to(dt)
                continue
            s = _oracle_frame(cfg, n, int(ti[j]), int(lon[j]), m1[j:j + 1].to(dt), m2[j:j + 1].to(dt),
                              cur[j:j + 1].to(dt))
            ref.append(s.step(eps[j:j + 1], int(s.timesteps[ti[j]]), lat[j:j + 1].to(dt)))
            ref_m1[j] = s.model_outputs[-1][0]
            if order == 3 and s.model_outputs[-2] is not None:   # the kernel shifts x0_prev into x0_prev2 regardless
                assert torch.equal(s.model_outputs[-2][0], ref_m2[j])
            ref_cur[j] = s.sample[0]
            orders.add(min(tables.order_list[int(ti[j])], int(lon[j]) + 1))
        m1_d, cur_d = m1.cuda(), cur.cuda()
        m2_d = m2.cuda() if order == 3 else None
        out, ti_out, lon_out = cfg_dpm_single_step(noise.cuda(), lat.cuda(), mask.cuda(), ti.cuda(), m1_d, m2_d, cur_d,
                                                   lon.cuda(), tables.c_struct(emulate), guidance, cfg_on)
        torch.cuda.synchronize()
        assert ti_out.cpu().tolist() == [0 if j == 7 else int(ti[j]) + 1 for j in range(F)]
        assert lon_out.cpu().tolist() == [int(lon[j]) if j == 7 else min(int(lon[j]) + 1, order) for j in range(F)]
        got = {"out": (out, torch.cat(ref)), "x0_prev": (m1_d, ref_m1), "cur_sample": (cur_d, ref_cur)}
        if order == 3:
            got["x0_prev2"] = (m2_d, ref_m2)
        for name, (g_d, want) in got.items():
            g_c = g_d.cpu().double()
            want = want.double()
            if emulate or name in ("x0_prev2", "cur_sample"):   # moved bf16 planes are exact in either mode
                assert torch.equal(g_c, want), (name, (g_c - want).abs().max())
            else:   # one bf16 rounding of the stored result, plus fp32 arithmetic relative to the largest value
                bound = _bf16_ulp(want) + 1e-6 * max(want.abs().max().item(), lat.abs().max().item())
                assert ((g_c - want).abs() <= bound).all(), (name, ((g_c - want).abs() - bound).max())
        assert torch.equal(m1_d.cpu()[7], m1[7]) and torch.equal(cur_d.cpu()[7], cur[7])   # cond: untouched
    assert orders == set(range(1, order + 1))   # every order the config allows ran in the one launch


def _tiny_pipe(emulate=True, **kw):
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.unet import B200MultiviewUNet
    cfg = UNetConfig.tiny()
    unet = B200MultiviewUNet(cfg, device=0).load_state_dict(random_state_dict(cfg, seed=1, dtype=torch.bfloat16))
    return B200Diffuman4DPipeline(unet, DPMSingleConfig(**kw), emulate_bf16_scheduler=emulate), unet


def _unet_cb(unet):
    def cb(x, t, sk, doms, nf):
        return unet(x.cuda(), t.cuda(), sk.cuda(), doms, nf, return_dict=False)[0].cpu()
    return cb


def _assert_state_matches(state, frames, copies):
    """The device state of ``frames`` (indices into ``state``) equals the per-frame oracle copies: the order count (the
    history entries upstream holds), the data predictions and the sample of the current block."""
    for j, c in zip(frames, copies):
        held = sum(m is not None for m in c.model_outputs)
        assert int(state.lower_order_nums[j]) == held, j
        if held >= 1:
            assert torch.equal(state.x0_prev.cpu()[j:j + 1], c.model_outputs[-1]), j
            assert torch.equal(state.cur_sample.cpu()[j:j + 1], c.sample), j
        if c.cfg.solver_order == 3 and held >= 2:
            assert torch.equal(state.x0_prev2.cpu()[j:j + 1], c.model_outputs[-2]), j


def test_denoise_window_dpm_single_vs_oracle_bit_exact(cuda):
    """``d4d_denoise_window_dpm_single`` (five steps of one window at order 3, staggered step indices of a 10-step table,
    fresh state, so that frames start on second- and third-order rows below their order and pass through every order)
    against the oracle's window step with per-frame scheduler copies, both driven by the same CUDA UNet; the state comes
    back updated."""
    from oracle.dpm_single_oracle import DPMSingleOracle
    from oracle.dpm_solver_oracle import denoise_window_oracle_per_frame
    pipe, unet = _tiny_pipe(solver_order=3)
    n, h, w = 5, 8, 8
    g = torch.Generator().manual_seed(52)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    pix, plk, lat = r(n, 4, h, w), r(n, 6, h, w), r(n, 4, h, w)
    skel = (torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16)
    mask = torch.ones(n, 1, h, w, dtype=torch.bfloat16)
    mask[1] = 0
    ti = torch.tensor([0, 0, 1, 4, 5])
    handles, _ = pipe.parepare_schedulers(10, n)
    state = handles[0].state.take(torch.arange(n), h, w)
    orc = DPMSingleOracle(DPMSingleConfig(solver_order=3))
    orc.set_timesteps(10)
    copies = [copy.deepcopy(orc) for _ in range(n)]
    want, want_ti = denoise_window_oracle_per_frame(
        _unet_cb(unet), copies, latents=lat.clone(), pixel_latents=pix, plucker=plk, skeletons=skel, cond_mask=mask,
        timestep_indices=ti, domain="spatial", guidance_scale=2.0, num_inference_steps=5)
    lat_d, ti_d = lat.cuda(), ti.cuda()
    pipe.denoise_window(latents=lat_d, pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skel,
                        cond_masks_latents=mask, timestep_indices=ti_d, domain="spatial", guidance_scale=2.0,
                        num_inference_steps=5, solver_state=state)
    torch.cuda.synchronize()
    assert torch.equal(ti_d.cpu(), want_ti)
    assert torch.equal(lat_d.cpu(), want), (lat_d.cpu().float() - want.float()).abs().max()
    _assert_state_matches(state, (0, 2, 3, 4), [copies[j] for j in (0, 2, 3, 4)])


@pytest.mark.parametrize("kw", [dict(solver_order=3), dict(prediction_type="v_prediction", final_sigmas_type="sigma_min"),
                                dict(solver_order=3, final_sigmas_type="sigma_min", prediction_type="sample"),
                                dict(solver_order=1)])
def test_sliding_iterative_denoise_dpm_single_vs_oracle_bit_exact(cuda, kw):
    """Per-frame solver state carried across the windows of a task and reset per task: a spatial and then a bidirectional
    temporal task on one pipeline, against the oracle's sliding loop on one scheduler object (per-frame copies; the loop
    tests/test_scheduler_dpm_single.py pins against the reference pipeline's golden) with our UNet.  The spatial task's 16
    steps switch lower_order_final on at order 3 and the switch stays for the temporal task's 6.  The task's final state
    planes are compared too."""
    from oracle.dpm_single_oracle import DPMSingleOracle
    from oracle.dpm_solver_oracle import sliding_iterative_denoise_oracle_per_frame
    pipe, unet = _tiny_pipe(**kw)
    handles = []
    prepare = pipe.parepare_schedulers
    pipe.parepare_schedulers = lambda *a: handles.append(prepare(*a)[0]) or (handles[-1], None)
    copies = []

    class RecordingDPMSingle(DPMSingleOracle):   # keeps the per-frame copies the oracle's loop makes
        def __deepcopy__(self, memo):
            c = DPMSingleOracle.__new__(RecordingDPMSingle)
            c.__dict__.update(copy.deepcopy(self.__dict__, memo))
            copies.append(c)
            return c

    orc = RecordingDPMSingle(DPMSingleConfig(**kw))
    h = w = 8
    g = torch.Generator().manual_seed(53)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    # each target frame takes per-alternation steps: 8 in the spatial task, 6 in the temporal one
    for domain, n_in, n_tg, ws, stride, bidir, rounds in (("spatial", 2, 4, 4, 1, True, 2),
                                                          ("temporal", 3, 3, 3, 1, True, 1)):
        n = n_in + n_tg
        mask = torch.ones(n, 1, h, w, dtype=torch.bfloat16)
        mask[:n_in] = 0
        args = dict(pixel_latents=r(n, 4, h, w), plucker=r(n, 6, h, w),
                    skeletons=(torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16), cond_mask=mask,
                    latents=r(n, 4, h, w), domain=domain, timestep_indices=torch.zeros(n, dtype=torch.long),
                    window_size=ws, sliding_stride=stride, bidirectional=bidir, alternation_rounds=rounds,
                    guidance_scale=2.0)
        copies.clear()
        ref = sliding_iterative_denoise_oracle_per_frame(_unet_cb(unet), orc, **args, enable_pose_encoder=True)
        out = pipe.sliding_iterative_denoise(
            pixel_values_latents=args["pixel_latents"], plucker_embeds=args["plucker"], skeletons=args["skeletons"],
            cond_masks=mask, latents=args["latents"], domain=domain, timestep_indices=args["timestep_indices"],
            window_size=ws, sliding_stride=stride, bidirectional=bidir, alternation_rounds=rounds, guidance_scale=2.0)
        torch.cuda.synchronize()
        assert pipe.scheduler.config.lower_order_final == orc.cfg.lower_order_final
        assert pipe.scheduler.order_list == orc.order_list
        assert torch.equal(out["timestep_indices"].cpu(), ref["timestep_indices"])
        assert torch.equal(out["fully_denoised"].cpu(), ref["fully_denoised"])
        assert torch.equal(out["latents"].cpu(), ref["latents"]), (out["latents"].cpu().float() -
                                                                   ref["latents"].float()).abs().max()
        assert len(copies) == n
        _assert_state_matches(handles[-1][0].state, range(n), copies)


def test_call_carries_state_through_scheduler_handles(cuda):
    """``__call__`` with the per-frame handles of ``parepare_schedulers``: three successive windows over overlapping frames
    == the reference's pattern with per-frame scheduler copies (PIPE:535); the first window starts its frames at
    nonzero timestep indices with fresh histories."""
    from oracle.dpm_single_oracle import DPMSingleOracle
    from oracle.dpm_solver_oracle import denoise_window_oracle_per_frame
    pipe, unet = _tiny_pipe(solver_order=3)
    n, h, w = 5, 8, 8
    g = torch.Generator().manual_seed(54)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)
    pix, plk, lat = r(n, 4, h, w), r(n, 6, h, w), r(n, 4, h, w)
    skel = (torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16)
    mask = torch.ones(n, 1, h, w, dtype=torch.bfloat16)
    mask[0] = 0
    handles, timesteps = pipe.parepare_schedulers(12, n)
    orc = DPMSingleOracle(DPMSingleConfig(solver_order=3))
    orc.set_timesteps(12)
    copies = [copy.deepcopy(orc) for _ in range(n)]
    ti = torch.tensor([0, 2, 1, 4, 2])
    lat_ours, lat_ref = lat.clone().cuda(), lat.clone()
    for window in (torch.tensor([0, 1, 2, 3]), torch.tensor([0, 2, 3, 4]), torch.tensor([0, 1, 3, 4])):
        got = pipe(pixel_values_latents=pix[window], plucker_embeds_latents=plk[window], skeletons_latents=skel[window],
                   cond_masks_latents=mask[window], latents=lat_ours[window.cuda()], domains=["spatial"],
                   num_inference_steps=2, schedulers=[handles[i] for i in window], timesteps=timesteps,
                   timestep_indices=ti[window], guidance_scale=2.0)
        want, _ = denoise_window_oracle_per_frame(
            _unet_cb(unet), [copies[i] for i in window], latents=lat_ref[window], pixel_latents=pix[window],
            plucker=plk[window], skeletons=skel[window], cond_mask=mask[window], timestep_indices=ti[window],
            domain="spatial", guidance_scale=2.0, num_inference_steps=2)
        tgt = window[mask[window, 0, 0, 0] != 0]
        ti[tgt] += 2
        lat_ours[window.cuda()] = got
        lat_ref[window] = want
        torch.cuda.synchronize()
        assert torch.equal(got.cpu(), want), (got.cpu().float() - want.float()).abs().max()
    state = handles[0].state
    _assert_state_matches(state, range(1, n), copies[1:])
    assert int(state.lower_order_nums[0]) == 0


def _tiny_checkpoint(tmp_path):
    from safetensors.torch import save_file
    cfg = UNetConfig.tiny()
    os.makedirs(tmp_path / "unet")
    os.makedirs(tmp_path / "scheduler")
    json.dump(dict(in_channels=11, out_channels=4, block_out_channels=[64, 128, 256, 256], attention_head_dim=[1, 2, 4, 4],
                   cross_attention_dim=None, use_linear_projection=True, enable_pose_encoder=True, enable_tem_embeds=True,
                   layers_per_block=2, num_3d_attn_blocks=3), open(tmp_path / "unet" / "config.json", "w"))
    json.dump({"_class_name": "DPMSolverSinglestepScheduler", "_diffusers_version": "0.33.1", "num_train_timesteps": 1000,
               "beta_start": 0.00085, "beta_end": 0.012, "beta_schedule": "scaled_linear", "trained_betas": None,
               "solver_order": 3, "prediction_type": "epsilon", "thresholding": False, "algorithm_type": "dpmsolver++",
               "solver_type": "midpoint", "lower_order_final": False, "final_sigmas_type": "zero",
               "lambda_min_clipped": float("-inf"), "variance_type": None},
              open(tmp_path / "scheduler" / "scheduler_config.json", "w"))
    save_file({k: v.contiguous() for k, v in random_state_dict(cfg, seed=1).items()},
              str(tmp_path / "unet" / "diffusion_pytorch_model.safetensors"))


def test_load_pipelines_with_dpm_single_scheduler(cuda, tmp_path):
    from diffuman4d_b200.loader import load_pipelines
    from diffuman4d_b200.scheduler import DPMSingleTables
    _tiny_checkpoint(tmp_path)
    (pipe,) = load_pipelines(model_dir=str(tmp_path), torch_dtype="bf16", gpu_ids=[0])
    assert isinstance(pipe.scheduler, DPMSingleTables) and pipe.scheduler.config == DPMSingleConfig(
        beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", solver_order=3)
    n, h, w = 6, 8, 8
    g = torch.Generator().manual_seed(55)
    mask = torch.ones(n, 1, h, w)
    mask[[1, 4]] = 0
    out = pipe.sliding_iterative_denoise(
        pixel_values_latents=torch.randn(n, 4, h, w, generator=g), plucker_embeds=torch.randn(n, 6, h, w, generator=g),
        skeletons=torch.rand(n, 3, 8 * h, 8 * w, generator=g) * 2 - 1, cond_masks=mask, latents=None, domain="spatial",
        timestep_indices=torch.zeros(n, dtype=torch.long), window_size=2, sliding_stride=1, bidirectional=True,
        alternation_rounds=1, guidance_scale=2.0, generator=torch.Generator(device="cuda").manual_seed(0))
    ti = out["timestep_indices"].cpu()
    assert ti[[1, 4]].eq(0).all() and ti[[0, 2, 3, 5]].eq(4).all() and out["fully_denoised"].cpu()[[0, 2, 3, 5]].all()
    assert torch.isfinite(out["latents"].float()).all()
    assert pipe.scheduler.config.lower_order_final and pipe.scheduler.order_list == [1, 2, 3, 1]


def test_sampler_drives_a_dpm_single_pipeline(cuda):
    sys.path.insert(0, GOLD)
    from pool_vae import PoolVAE
    from synthetic_dataset import SyntheticSpaTemDataset
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.sampler import B200SlidingIterativeSampler
    from diffuman4d_b200.unet import B200MultiviewUNet

    cfg = UNetConfig.tiny()
    unet = B200MultiviewUNet(cfg, 0).load_state_dict(random_state_dict(cfg, seed=1))
    pipe = B200Diffuman4DPipeline(unet, DPMSingleConfig(solver_order=3), vae=PoolVAE())
    ds = SyntheticSpaTemDataset(8, h=16, w=16)
    s = B200SlidingIterativeSampler(ds, [pipe], output_dir=None, spa_label_range=[0, 6, 1], tem_label_range=[0, 4, 1],
                                    input_spa_labels=[1, 4], window_size=2, sliding_stride=1, bidirectional=True,
                                    alternation_rounds=3, guidance_scale=2.0)
    s.execute_tasks()
    torch.cuda.synchronize()
    assert s.grid_latents.shape == (6, 4, 4, 16, 16) and torch.isfinite(s.grid_latents.float()).all()
    ti = s.grid_timestep_indices.cpu()
    n_inf = 2 * 1 // 1 * 2 * 3                                   # window * steps / stride, bidirectional, 3 rounds
    for v, spa in enumerate(s.spa_labels):
        expect = 0 if spa in s.input_spa_labels else n_inf      # every target cell fully denoised, inputs untouched
        assert (ti[v] == expect).all(), (spa, ti[v])
