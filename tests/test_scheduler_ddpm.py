"""Host side of DDPM sampling (``DDPMScheduler``) on the CPU.

* The loader's mapping and every refusal by key; other classes are still refused with the old message.
* ``DDPMTables`` rows against ``DDPMOracle``'s restatement of upstream, bit for bit; DDIM's spacing code is shared.
* Anchors in fp64: the last row (t = 0) returns x0 exactly; without the noise term the step is the closed-form posterior
  mean of x0 and x_t; ``fixed_large`` has std^2 = beta_t and ``fixed_small`` the posterior variance.
* The host Philox4x32-10 against the Random123 known-answer vectors, and the noise's statistics over 10^6 draws: mean,
  variance, a Kolmogorov-Smirnov test against N(0, 1), and no correlation across frame id, timestep index and seed.
* The per-frame semantics of the reference's own loops, pinned by tests/golden/pipeline_ddpm_ref.pt
  (tests/golden/gen_golden_ddpm.py).
* A gloo job of 2 processes runs the frame-sharded sliding loop with a stand-in step that records the frame ids and seed
  each rank passes: each rank gets its shard of every window's task indices and rank 0's seed, and the results equal the
  plain loop's.
"""
import copy
import os

import numpy as np
import pytest
import torch

from diffuman4d_b200.config import DDPMConfig, UNetConfig
from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
from diffuman4d_b200.scheduler import DDIMTables, DDPMTables, SchedulerConfig, draw_seed
from oracle.ddpm_oracle import DDPMOracle, ddpm_noise, ddpm_noise_fp64, philox4x32_10

GOLD = os.path.join(os.path.dirname(__file__), "golden")


# ------------------------------------------------------------------------------------------------ loader
DDPM_JSON = {"_class_name": "DDPMScheduler", "_diffusers_version": "0.33.1", "num_train_timesteps": 1000,
             "beta_start": 0.00085, "beta_end": 0.012, "beta_schedule": "scaled_linear", "trained_betas": None,
             "variance_type": "fixed_small_log", "clip_sample": False, "clip_sample_range": 2.0,
             "prediction_type": "v_prediction", "thresholding": False, "dynamic_thresholding_ratio": 0.995,
             "sample_max_value": 1.0, "timestep_spacing": "trailing", "steps_offset": 1, "rescale_betas_zero_snr": False}


def test_loader_maps_ddpm():
    from diffuman4d_b200.loader import scheduler_config_from_json
    assert scheduler_config_from_json(DDPM_JSON) == DDPMConfig(
        beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", variance_type="fixed_small_log",
        clip_sample=False, clip_sample_range=2.0, prediction_type="v_prediction", timestep_spacing="trailing",
        steps_offset=1)
    assert scheduler_config_from_json({"_class_name": "DDPMScheduler"}) == DDPMConfig()


@pytest.mark.parametrize("key,value", [("variance_type", "learned"), ("variance_type", "learned_range"),
                                       ("variance_type", "fixed_large_log"), ("variance_type", "other"),
                                       ("thresholding", True), ("rescale_betas_zero_snr", True),
                                       ("trained_betas", [0.1, 0.2]), ("beta_schedule", "squaredcos_cap_v2"),
                                       ("prediction_type", "flow"), ("timestep_spacing", "karras")])
def test_loader_refuses_by_key(key, value):
    from diffuman4d_b200.loader import scheduler_config_from_json
    with pytest.raises(NotImplementedError, match=f"DDPMScheduler {key}="):
        scheduler_config_from_json({**DDPM_JSON, key: value})


def test_other_classes_are_still_refused():
    from diffuman4d_b200.loader import scheduler_config_from_json
    with pytest.raises(NotImplementedError, match="DPMSolverSinglestepScheduler only"):
        scheduler_config_from_json({"_class_name": "EulerDiscreteScheduler"})
    with pytest.raises(NotImplementedError, match="DDPMScheduler, "):
        scheduler_config_from_json({"_class_name": "EulerAncestralDiscreteScheduler"})


# ------------------------------------------------------------------------------------------------ tables
CONFIGS = [DDPMConfig(), DDPMConfig(variance_type="fixed_small_log", prediction_type="v_prediction"),
           DDPMConfig(variance_type="fixed_large", timestep_spacing="trailing"),
           DDPMConfig(beta_schedule="scaled_linear", beta_start=0.00085, beta_end=0.012, timestep_spacing="linspace"),
           DDPMConfig(timestep_spacing="leading", steps_offset=1, prediction_type="sample")]


@pytest.mark.parametrize("cfg", CONFIGS)
@pytest.mark.parametrize("n", [1, 7, 10, 50])
def test_tables_match_the_oracle_bitwise(cfg, n):
    t = DDPMTables(cfg, device="cpu")
    ts = t.set_timesteps(n)
    o = DDPMOracle(cfg)
    assert torch.equal(ts, o.set_timesteps(n))
    assert torch.equal(t.alphas_cumprod, o.alphas_cumprod)
    for i, tv in enumerate(int(v) for v in ts):
        a_t, a_prev = o._alphas(tv)
        beta = 1 - a_t / a_prev
        row = torch.stack([a_t ** 0.5, (1 - a_t) ** 0.5, (a_prev ** 0.5 * beta) / (1 - a_t),
                           (a_t / a_prev) ** 0.5 * (1 - a_prev) / (1 - a_t), o.noise_std(tv),
                           torch.tensor(float(tv > 0))])
        assert torch.equal(t.coefs[i], row), (i, t.coefs[i], row)
        assert o.previous_timestep(tv) == (int(ts[i + 1]) if i + 1 < n else -1)


def test_timesteps_are_ddims():
    for spacing, offset in (("leading", 0), ("leading", 1), ("trailing", 0), ("linspace", 0)):
        d = DDIMTables(SchedulerConfig(timestep_spacing=spacing, steps_offset=offset), device="cpu")
        p = DDPMTables(DDPMConfig(timestep_spacing=spacing, steps_offset=offset), device="cpu")
        for n in (1, 9, 25):
            assert torch.equal(d.set_timesteps(n), p.set_timesteps(n))


def test_unsupported_variance_type_is_refused():
    with pytest.raises(NotImplementedError, match="variance_type"):
        DDPMTables(DDPMConfig(variance_type="learned"), device="cpu")


# ------------------------------------------------------------------------------------------------ fp64 anchors
def _orc64(cfg, n):
    o = DDPMOracle(cfg, table_dtype=torch.float64)
    o.set_timesteps(n)
    return o


@pytest.mark.parametrize("pred", ["epsilon", "v_prediction", "sample"])
def test_last_step_returns_x0(pred):
    cfg = DDPMConfig(prediction_type=pred, clip_sample=False)
    o = _orc64(cfg, 10)
    assert int(o.timesteps[-1]) == 0
    g = torch.Generator().manual_seed(1)
    x, m = torch.randn(1, 4, 5, 5, generator=g, dtype=torch.float64), torch.randn(1, 4, 5, 5, generator=g,
                                                                                   dtype=torch.float64)
    a = o.alphas_cumprod[0]
    x0 = {"epsilon": (x - (1 - a) ** 0.5 * m) / a ** 0.5, "v_prediction": a ** 0.5 * x - (1 - a) ** 0.5 * m,
          "sample": m}[pred]
    assert torch.equal(o.step(m, 0, x), x0)
    bf = DDPMOracle(cfg)
    bf.set_timesteps(10)
    xb, mb = x.to(torch.bfloat16), m.to(torch.bfloat16)
    assert torch.equal(bf.step(mb, 0, xb), bf.step(mb, 0, xb, add_noise=False))   # t = 0 draws nothing


@pytest.mark.parametrize("n", [5, 20])
def test_noise_free_step_is_the_posterior_mean(n):
    """mu(x0, x_t) = sqrt(a_prev) beta_t / (1 - a_t) x0 + sqrt(alpha_t) (1 - a_prev) / (1 - a_t) x_t (Ho et al. 2020,
    eq. 7, with alpha_t = a_t / a_prev over the skipped timesteps)."""
    o = _orc64(DDPMConfig(prediction_type="sample", clip_sample=False), n)
    g = torch.Generator().manual_seed(2)
    x0, xt = torch.randn(1, 4, 3, 3, generator=g, dtype=torch.float64), torch.randn(1, 4, 3, 3, generator=g,
                                                                                     dtype=torch.float64)
    for i, t in enumerate(int(v) for v in o.timesteps):
        a_t = float(o.alphas_cumprod[t])
        a_prev = float(o.alphas_cumprod[int(o.timesteps[i + 1])]) if i + 1 < n else 1.0
        alpha = a_t / a_prev
        mu = (a_prev ** 0.5 * (1 - alpha) / (1 - a_t)) * x0 + (alpha ** 0.5 * (1 - a_prev) / (1 - a_t)) * xt
        assert torch.allclose(o.step(x0, t, xt, add_noise=False), mu, rtol=1e-12, atol=1e-12), i


def test_variances():
    n = 10
    large, small = (_orc64(DDPMConfig(variance_type=v), n) for v in ("fixed_large", "fixed_small"))
    for i, t in enumerate(int(v) for v in large.timesteps[:-1]):
        a_t = float(large.alphas_cumprod[t])
        a_prev = float(large.alphas_cumprod[int(large.timesteps[i + 1])])
        beta = 1 - a_t / a_prev
        assert abs(float(large.noise_std(t)) ** 2 - beta) <= 1e-14
        assert abs(float(small.noise_std(t)) ** 2 - (1 - a_prev) / (1 - a_t) * beta) <= 1e-14


# ------------------------------------------------------------------------------------------------ noise
def test_philox_known_answers():
    hexs = lambda a: " ".join(f"{int(v):08x}" for v in a)
    assert hexs(philox4x32_10(np.zeros(4, np.uint64), (0, 0))) == "6627e8d5 e169c58d bc57ac4c 9b00dbd8"
    assert hexs(philox4x32_10(np.full(4, 0xFFFFFFFF, np.uint64), (0xFFFFFFFF, 0xFFFFFFFF))) == \
        "408f276d 41c83b0e a20bc7c6 6d5451fd"
    assert hexs(philox4x32_10(np.array([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], np.uint64),
                              (0xA4093822, 0x299F31D0))) == "d16cfe09 94fdcceb 5001e420 24126ea1"


def test_noise_statistics():
    from scipy import stats
    z = ddpm_noise_fp64(2024, np.arange(16), np.full(16, 3), 128, 128)   # 16 * 4 * 128 * 128 = 1 048 576 draws
    flat = z.reshape(-1)
    assert flat.size >= 10 ** 6
    assert abs(flat.mean()) < 5 / np.sqrt(flat.size)
    assert abs(flat.var() - 1) < 5 * np.sqrt(2 / flat.size)
    assert stats.kstest(flat, "norm").pvalue > 1e-3
    n = 4 * 64 * 64
    base = ddpm_noise_fp64(7, [0], [0], 64, 64).reshape(-1)
    for other in (ddpm_noise_fp64(7, [1], [0], 64, 64), ddpm_noise_fp64(7, [0], [1], 64, 64),
                  ddpm_noise_fp64(8, [0], [0], 64, 64), ddpm_noise_fp64(7 + 2 ** 32, [0], [0], 64, 64)):
        assert abs(np.corrcoef(base, other.reshape(-1))[0, 1]) < 5 / np.sqrt(n)
    # the four words of one call are independent too
    q = z.reshape(-1, 4)
    c = np.corrcoef(q.T)
    assert np.abs(c - np.eye(4)).max() < 5 / np.sqrt(q.shape[0])


def test_bf16_noise_is_the_fp64_draw_rounded_once():
    z = ddpm_noise_fp64(11, [2], [5], 16, 16)
    b = ddpm_noise(11, [2], [5], 16, 16, torch.bfloat16).double().numpy()
    ulp = 2.0 ** (np.floor(np.log2(np.abs(z))) - 7)
    assert (np.abs(b - z) <= ulp / 2).all()


def test_seed_draw():
    s = draw_seed(torch.Generator().manual_seed(0))
    assert s.dtype == torch.int64 and s.shape == (1,)
    assert torch.equal(s, draw_seed(torch.Generator().manual_seed(0)))
    assert not torch.equal(s, draw_seed(torch.Generator().manual_seed(1)))


# ------------------------------------------------------------------------------------------------ golden
def _fake_unet(cin):
    import sys
    sys.path.insert(0, GOLD)
    from fake_unet import make_fake_unet
    return make_fake_unet(cin)


def _golden():
    return torch.load(os.path.join(GOLD, "pipeline_ddpm_ref.pt"))


@pytest.mark.parametrize("tag", ["call_cfg_eps", "call_nocfg_v_large"])
def test_window_call_matches_reference_pipeline_golden(tag):
    """The reference's ``__call__`` with a ``DDPMOracle`` adapter (tests/golden/gen_golden_ddpm.py) against the oracle's
    per-frame window: the k-th copy is frame k, conditioning frames are never stepped, and frames reach the last row."""
    from oracle.dpm_solver_oracle import denoise_window_oracle_per_frame
    c = _golden()["cases"][tag]
    i = c["in"]
    s = DDPMOracle(DDPMConfig(**c["config"]), seed=c["seed"])
    assert torch.equal(s.set_timesteps(c["n_steps_table"]), c["timesteps_table"])
    scheds = [copy.deepcopy(s) for _ in range(len(i["latents"]))]
    lat, ti = denoise_window_oracle_per_frame(
        _fake_unet(11), scheds, latents=i["latents"].clone(), pixel_latents=i["pixel_latents"], plucker=i["plucker"],
        skeletons=i["skeletons"].float(), cond_mask=i["cond_mask"], timestep_indices=i["timestep_indices"], domain="spatial",
        guidance_scale=c["guidance"], num_inference_steps=c["num_inference_steps"], enable_pose_encoder=True)
    torch.testing.assert_close(lat, c["out_latents"], rtol=1e-5, atol=1e-6)
    assert torch.equal(ti, c["out_timestep_indices"])
    # the noise is keyed by frame: another frame order gives other latents
    scheds = [copy.deepcopy(s) for _ in range(len(i["latents"]))][::-1]
    lat2, _ = denoise_window_oracle_per_frame(
        _fake_unet(11), scheds, latents=i["latents"].clone(), pixel_latents=i["pixel_latents"], plucker=i["plucker"],
        skeletons=i["skeletons"].float(), cond_mask=i["cond_mask"], timestep_indices=i["timestep_indices"], domain="spatial",
        guidance_scale=c["guidance"], num_inference_steps=c["num_inference_steps"], enable_pose_encoder=True)
    assert (lat2 - c["out_latents"]).abs().max() > 1e-3


@pytest.mark.parametrize("tag", ["slide_spatial_eps_cfg", "slide_temporal_bidir_v_nocfg"])
def test_sliding_loop_matches_reference_pipeline_golden(tag):
    """Two tasks on one scheduler object: the copies, and the frame count that keys their noise, reset per task."""
    from oracle.dpm_solver_oracle import sliding_iterative_denoise_oracle_per_frame
    c = _golden()["cases"][tag]
    sched = DDPMOracle(DDPMConfig(**c["config"]), seed=c["seed"])
    for task in c["tasks"]:
        i = task["in"]
        out = sliding_iterative_denoise_oracle_per_frame(
            _fake_unet(11), sched, pixel_latents=i["pixel_latents"], plucker=i["plucker"],
            skeletons=i["skeletons"].float(), cond_mask=i["cond_mask_latents"], latents=i["latents"],
            domain=c["domain"], timestep_indices=i["timestep_indices"], window_size=task["window_size"],
            sliding_stride=c["sliding_stride"], bidirectional=c["bidirectional"], num_denoising_steps=1,
            alternation_rounds=c["alternation_rounds"], guidance_scale=c["guidance"], enable_pose_encoder=True)
        torch.testing.assert_close(out["latents"], task["out_latents"], rtol=1e-5, atol=1e-5)
        assert torch.equal(out["timestep_indices"], task["out_timestep_indices"])
        assert torch.equal(out["fully_denoised"], task["fully_denoised"])


# ------------------------------------------------------------------------------------------------ gloo sharded loop
class _UNetStub:
    def __init__(self):
        self.device = torch.device("cpu")
        self.config = UNetConfig.tiny()


def _standin(lat, ts, frames, pix, msk, steps, record):
    """A per-frame step whose result depends on the frame's latents, conditioning, timestep index, task index and the
    task seed; conditioning frames receive their image latents and timestep 0."""
    record.append((frames.seed, frames.frame_ids.tolist()))
    cond = (msk[:, 0, 0, 0] == 0).view(-1, 1, 1, 1)
    key = (frames.frame_ids * 7 + frames.seed % 1009).view(-1, 1, 1, 1).float()
    for _ in range(steps):
        new = lat.float() * 0.75 + pix.float() * 0.25 + 0.001 * key - 0.01 * ts.view(-1, 1, 1, 1).float()
        lat.copy_(torch.where(cond, pix, new.to(torch.bfloat16)))
        ts.copy_(torch.where(cond.view(-1), torch.zeros_like(ts), ts + 1))


def _task(n_in=4, n_tg=8):
    n = n_in + n_tg
    g = torch.Generator().manual_seed(5)
    mask = torch.ones(n, 1, 64, 64)
    mask[:n_in] = 0
    return dict(pixel_values_latents=torch.randn(n, 4, 8, 8, generator=g).to(torch.bfloat16),
                plucker_embeds=torch.randn(n, 6, 64, 64, generator=g), skeletons_latents=torch.randn(n, 4, 8, 8, generator=g),
                cond_masks=mask, latents=None, domain="spatial", timestep_indices=torch.zeros(n, dtype=torch.long),
                window_size=4, sliding_stride=2, bidirectional=True, num_denoising_steps=1, alternation_rounds=2,
                guidance_scale=2.0)


def _gloo_worker(rank, world, store, out_dir):
    import torch.distributed as dist
    from diffuman4d_b200.sharded import FrameShardedPipeline
    dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=world)
    try:
        pipe = B200Diffuman4DPipeline(_UNetStub(), DDPMConfig())
        sh = FrameShardedPipeline.__new__(FrameShardedPipeline)
        sh.pipe, sh.group, sh.rank, sh.world = pipe, None, rank, world
        record = []

        def step(lat, ts, state, conds, F_total, *, domain, guidance_scale, num_inference_steps):
            pix, _, _, msk = conds
            _standin(lat, ts, state, pix, msk, num_inference_steps, record)
            parts = [[torch.empty_like(t) for _ in range(world)] for t in (lat, ts)]
            dist.all_gather(parts[0], lat)
            dist.all_gather(parts[1], ts)
            return torch.cat(parts[0]), torch.cat(parts[1]), None
        sh._step_and_exchange = step
        # each rank's generator differs: the loop must use rank 0's noise and seed on every rank
        out = sh.sliding_iterative_denoise(**_task(), generator=torch.Generator().manual_seed(100 + rank))
        torch.save({"latents": out["latents"], "timestep_indices": out["timestep_indices"], "record": record},
                   os.path.join(out_dir, f"rank{rank}.pt"))
    finally:
        dist.destroy_process_group()


def test_gloo_sharded_loop_passes_frame_ids_and_seed(tmp_path):
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, str(tmp_path / "store"), str(tmp_path)))
             for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0, f"gloo worker exited with {p.exitcode}"
    got = [torch.load(tmp_path / f"rank{r}.pt") for r in range(world)]
    pipe = B200Diffuman4DPipeline(_UNetStub(), DDPMConfig())
    record = []

    def plain(*, latents, pixel_values_latents, cond_masks_latents, timestep_indices, num_inference_steps,
              solver_state=None, **_):
        _standin(latents, timestep_indices, solver_state, pixel_values_latents, cond_masks_latents,
                 num_inference_steps, record)
    pipe.denoise_window = plain
    ref = pipe.sliding_iterative_denoise(**_task(), generator=torch.Generator().manual_seed(100))
    seed = int(draw_seed(_seeded_after_noise(100, 12)).item())
    assert record and all(s == seed for s, _ in record)
    for r in range(world):
        assert torch.equal(got[r]["latents"], ref["latents"]) and torch.equal(got[r]["timestep_indices"],
                                                                            ref["timestep_indices"])
        assert len(got[r]["record"]) == len(record)
        for (s, ids), (_, want) in zip(got[r]["record"], record):
            assert s == seed
            k = len(want) // world
            assert ids == want[r * k:(r + 1) * k]


def _seeded_after_noise(seed, n):
    """A generator in the state the sliding loop leaves it in after drawing the initial noise of n frames."""
    g = torch.Generator().manual_seed(seed)
    torch.randn(n, 4, 8, 8, generator=g, dtype=torch.bfloat16)
    return g
