"""PNDM (upstream PNDMScheduler with skip_prk_steps: the PLMS steps) on the CPU: mathematical anchors for the restated
arithmetic in fp64, the oracle's per-frame window step and sliding loop against the reference pipeline run with a stateful
scheduler (tests/golden/pipeline_pndm_ref.pt from tests/golden/gen_golden_pndm.py), the host tables, the config loader
and the frame-sharded refusal."""
import copy
import os
import sys

import pytest
import torch

from diffuman4d_b200.config import PNDMConfig, SchedulerConfig
from oracle.dpm_solver_oracle import denoise_window_oracle_per_frame, sliding_iterative_denoise_oracle_per_frame
from oracle.pipeline_oracle import DDIMOracle
from oracle.pndm_oracle import PNDMOracle

GOLD = os.path.join(os.path.dirname(__file__), "golden")
SD_PNDM = dict(beta_schedule="scaled_linear", beta_start=0.00085, beta_end=0.012, set_alpha_to_one=False,
               steps_offset=1, timestep_spacing="leading")


def _golden():
    return torch.load(os.path.join(GOLD, "pipeline_pndm_ref.pt"))


def _fake_unet(cin):
    sys.path.insert(0, GOLD)
    from fake_unet import make_fake_unet
    return make_fake_unet(cin)


def _fp64_pndm(n, **kw):
    s = PNDMOracle(PNDMConfig(**kw), table_dtype=torch.float64)
    s.set_timesteps(n)
    return s


def _fp64_ddim(pndm: PNDMOracle, n: int) -> DDIMOracle:
    c = pndm.cfg
    d = DDIMOracle(SchedulerConfig(num_train_timesteps=c.num_train_timesteps, beta_start=c.beta_start,
                                   beta_end=c.beta_end, beta_schedule=c.beta_schedule, prediction_type=c.prediction_type,
                                   set_alpha_to_one=c.set_alpha_to_one, steps_offset=c.steps_offset,
                                   timestep_spacing="leading", clip_sample=False))
    d.set_timesteps(n)
    d.alphas_cumprod = pndm.alphas_cumprod
    d.final_alpha_cumprod = pndm.final_alpha_cumprod
    return d


def _close(got, want, rel=1e-12):
    return (got - want).abs().max().item() <= rel * (1 + want.abs().max().item())


# ---- anchors ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("spacing", ["leading", "linspace", "trailing"])
@pytest.mark.parametrize("pred", ["epsilon", "v_prediction"])
def test_counter0_step_is_ddim_to_t_minus_T_over_n(spacing, pred):
    """A frame's first step uses the model output as it is: DDIM (eta 0) from t to t - T // n, for every row of the
    table, whatever the spacing (the previous timestep comes from the value of t and T // n)."""
    n = 10
    for i in range(n):
        s = _fp64_pndm(n, prediction_type=pred, timestep_spacing=spacing, steps_offset=int(spacing == "leading"))
        ddim = _fp64_ddim(s, n)
        g = torch.Generator().manual_seed(i)
        x = torch.randn(2, 4, 3, 3, generator=g, dtype=torch.float64)
        m = torch.randn(2, 4, 3, 3, generator=g, dtype=torch.float64)
        t = int(s.timesteps[i])
        assert _close(s.step(m, t, x), ddim.step(m, t, x)), (i, spacing, pred)
        assert s.counter == 1 and torch.equal(s.cur_sample, x) and len(s.ets) == 1


@pytest.mark.parametrize("pred", ["epsilon", "v_prediction"])
def test_counter1_step_restarts_from_cur_sample_with_the_mean_output(pred):
    """The second step re-steps from the first step's sample, from t + T // n to t (t = the repeated table entry), with
    the mean of the two model outputs: DDIM from t + T // n with that mean.  The first step's result is discarded, and the
    second output is not kept in ``ets``."""
    n = 12
    s = _fp64_pndm(n, prediction_type=pred, **SD_PNDM)
    ddim = _fp64_ddim(s, n)
    g = torch.Generator().manual_seed(3)
    x, m0, m1, junk = (torch.randn(2, 4, 3, 3, generator=g, dtype=torch.float64) for _ in range(4))
    t0, t1 = int(s.timesteps[0]), int(s.timesteps[1])
    s.step(m0, t0, x)
    got = s.step(m1, t1, junk)
    r = s.cfg.num_train_timesteps // n
    want = ddim.step((m0 + m1) / 2, t1 + r, x)   # v: the mean of the two outputs, converted at t1 + T // n
    assert t1 + r == t0 and int(s.timesteps[2]) == t1
    assert _close(got, want)
    assert s.counter == 2 and len(s.ets) == 1 and s.cur_sample is None


@pytest.mark.parametrize("kw", [dict(set_alpha_to_one=True), SD_PNDM])
def test_exact_denoiser_of_a_point_mass_stays_on_the_trajectory(kw):
    """Data = one point x0*: the exact epsilon-prediction is eps* at every point of x_t = a_t^0.5 x0* + (1 - a_t)^0.5
    eps*, and every combination PLMS forms of a constant is that constant, so each step lands on the trajectory at its
    previous timestep, through counters 0, 1, 2, 3 and >= 4.  (Not so with v-prediction: counter 1 averages v outputs
    of two timesteps, which upstream converts at the earlier one.)"""
    n = 12
    s = _fp64_pndm(n, **kw)
    ac, final = s.alphas_cumprod, s.final_alpha_cumprod
    alpha = lambda t: ac[t] if t >= 0 else final
    g = torch.Generator().manual_seed(1)
    x0s = torch.randn(3, 4, 5, 5, generator=g, dtype=torch.float64)
    eps = torch.randn(3, 4, 5, 5, generator=g, dtype=torch.float64)
    on_traj = lambda t: alpha(t) ** 0.5 * x0s + (1 - alpha(t)) ** 0.5 * eps
    r = s.cfg.num_train_timesteps // n
    x = on_traj(int(s.timesteps[0]))
    for i in range(n):
        t = int(s.timesteps[i])
        e = (x - ac[t] ** 0.5 * x0s) / (1 - ac[t]) ** 0.5
        lands = t if i == 1 else t - r
        x = s.step(e, t, x)
        ref = on_traj(lands)
        assert (x - ref).abs().max().item() <= 1e-9 * ref.abs().max().item(), i
    assert s.counter == n and len(s.ets) == 4


# ---- the reference pipeline's per-frame scheduler copies (golden) ------------------------------------------------
def _config(c):
    return PNDMConfig(**c["config"])


def _call(c):
    i = c["in"]
    s = PNDMOracle(_config(c))
    s.set_timesteps(c["n_steps_table"])
    assert torch.equal(s.timesteps, c["timesteps_table"])
    scheds = [copy.deepcopy(s) for _ in range(len(i["latents"]))]
    lat, ti = denoise_window_oracle_per_frame(
        _fake_unet(11), scheds, latents=i["latents"].clone(), pixel_latents=i["pixel_latents"], plucker=i["plucker"],
        skeletons=i["skeletons"], cond_mask=i["cond_mask"], timestep_indices=i["timestep_indices"], domain="spatial",
        guidance_scale=c["guidance"], num_inference_steps=c["num_inference_steps"], enable_pose_encoder=True)
    return lat, ti, scheds


@pytest.mark.parametrize("tag", ["call_cfg_eps_sd", "call_nocfg_v_linspace"])
def test_window_call_matches_reference_pipeline_golden(tag):
    """``__call__`` with fresh per-frame copies handed over at nonzero timestep indices: each frame's counter starts at 0
    whatever its index."""
    c = _golden()["cases"][tag]
    lat, ti, scheds = _call(c)
    torch.testing.assert_close(lat, c["out_latents"], rtol=1e-5, atol=1e-6)
    assert torch.equal(ti, c["out_timestep_indices"])
    assert [f.counter for f in scheds] == c["counter"]


SLIDE_TAGS = ["slide_spatial_eps_cfg_sd", "slide_temporal_bidir_v_nocfg", "slide_spatial_trailing",
              "slide_spatial_linspace_v"]


@pytest.mark.parametrize("tag", SLIDE_TAGS)
def test_sliding_loop_matches_reference_pipeline_golden(tag):
    """Two successive tasks on one scheduler object: per-frame histories across windows, reset per task."""
    c = _golden()["cases"][tag]
    for task in c["tasks"]:
        i = task["in"]
        out = sliding_iterative_denoise_oracle_per_frame(
            _fake_unet(11), PNDMOracle(_config(c)), pixel_latents=i["pixel_latents"], plucker=i["plucker"],
            skeletons=i["skeletons"], cond_mask=i["cond_mask_latents"], latents=i["latents"], domain=c["domain"],
            timestep_indices=i["timestep_indices"], window_size=c["window_size"], sliding_stride=c["sliding_stride"],
            bidirectional=c["bidirectional"], num_denoising_steps=1, alternation_rounds=c["alternation_rounds"],
            guidance_scale=c["guidance"], enable_pose_encoder=True)
        torch.testing.assert_close(out["latents"], task["out_latents"], rtol=1e-5, atol=1e-5)
        assert torch.equal(out["timestep_indices"], task["out_timestep_indices"])
        assert torch.equal(out["fully_denoised"], task["fully_denoised"])


# ---- tables -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(), SD_PNDM, dict(timestep_spacing="linspace", prediction_type="v_prediction"),
                                dict(timestep_spacing="trailing", set_alpha_to_one=True),
                                dict(timestep_spacing="leading", steps_offset=1, num_train_timesteps=1000)])
@pytest.mark.parametrize("n", [1, 2, 7, 50])
def test_tables_equal_the_oracle_bit_for_bit(kw, n):
    from diffuman4d_b200.scheduler import PNDMTables
    t = PNDMTables(PNDMConfig(**kw), device="cpu")
    o = PNDMOracle(t.config)
    assert torch.equal(t.set_timesteps(n), o.set_timesteps(n))
    assert len(t.timesteps) == (n + 1 if n > 1 else 1)
    assert t.coefs.dtype == torch.float32 and t.coefs.shape == (len(t.timesteps), 10)
    r = t.config.num_train_timesteps // n
    for i, ts in enumerate(t.timesteps.tolist()):
        want = [v.item() for v in o.prev_sample_coefs(ts, ts - r)]
        want += ([v.item() for v in o.prev_sample_coefs(ts + r, ts)] if ts + r < t.config.num_train_timesteps
                 else [float("nan")] * 5)
        got = t.coefs[i].tolist()
        assert torch.equal(torch.tensor(got).isnan(), torch.tensor(want).isnan()), i
        assert [g for g in got if g == g] == [w for w in want if w == w], i


def test_tables_refuse_what_the_step_does_not_implement():
    from diffuman4d_b200.scheduler import PNDMTables
    with pytest.raises(NotImplementedError, match="sample"):
        PNDMTables(PNDMConfig(prediction_type="sample"), device="cpu")
    with pytest.raises(ValueError):
        PNDMTables(PNDMConfig(timestep_spacing="karras"), device="cpu")
    with pytest.raises(ValueError):
        PNDMTables(PNDMConfig(beta_schedule="squaredcos_cap_v2"), device="cpu")


# ---- loader -------------------------------------------------------------------------------------------------------
# scheduler/scheduler_config.json of Stable Diffusion v1.5, as diffusers saved it
SD15_SCHEDULER_CONFIG = {
    "_class_name": "PNDMScheduler", "_diffusers_version": "0.6.0", "beta_end": 0.012, "beta_schedule": "scaled_linear",
    "beta_start": 0.00085, "num_train_timesteps": 1000, "set_alpha_to_one": False, "skip_prk_steps": True,
    "steps_offset": 1, "trained_betas": None, "clip_sample": False,
}


def test_loader_maps_the_sd15_config():
    from diffuman4d_b200.loader import scheduler_config_from_json
    assert scheduler_config_from_json(SD15_SCHEDULER_CONFIG) == PNDMConfig(**SD_PNDM)
    assert scheduler_config_from_json({"_class_name": "PNDMScheduler", "skip_prk_steps": True,
                                       "prediction_type": "v_prediction", "timestep_spacing": "trailing"}) == PNDMConfig(
        prediction_type="v_prediction", timestep_spacing="trailing")


@pytest.mark.parametrize("key,value", [("skip_prk_steps", False), ("prediction_type", "sample"),
                                       ("trained_betas", [0.1, 0.2]), ("beta_schedule", "squaredcos_cap_v2"),
                                       ("timestep_spacing", "karras")])
def test_loader_rejects_unsupported_pndm_keys(key, value):
    from diffuman4d_b200.loader import scheduler_config_from_json
    with pytest.raises(NotImplementedError, match=key):
        scheduler_config_from_json({**SD15_SCHEDULER_CONFIG, key: value})


def test_loader_rejects_the_runge_kutta_warmup_by_default():
    """Upstream's default is skip_prk_steps=False."""
    from diffuman4d_b200.loader import scheduler_config_from_json
    with pytest.raises(NotImplementedError, match="skip_prk_steps"):
        scheduler_config_from_json({"_class_name": "PNDMScheduler"})


# ---- frame-sharded refusal --------------------------------------------------------------------------------------------
def test_frame_sharded_pipeline_refuses_pndm_before_any_allocation(monkeypatch):
    import diffuman4d_b200.sharded as sharded_mod
    from diffuman4d_b200.config import UNetConfig
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline

    class _UNetStub:
        device = torch.device("cpu")
        config = UNetConfig.tiny()

    pipe = B200Diffuman4DPipeline(_UNetStub(), PNDMConfig(**SD_PNDM))
    monkeypatch.setattr(sharded_mod, "lib", lambda: pytest.fail("the library was called"))
    monkeypatch.setattr(sharded_mod.dist, "is_initialized", lambda: pytest.fail("torch.distributed was consulted"))
    monkeypatch.setattr(torch.cuda, "device", lambda *a: pytest.fail("a device was selected"))
    with pytest.raises(NotImplementedError, match="PNDM"):
        sharded_mod.FrameShardedPipeline(pipe, max_frames=8, h=8, w=8)
