"""DEIS (upstream DEISMultistepScheduler, algorithm_type "deis", solver_type "logrho") on the CPU: mathematical anchors for
the restated arithmetic in fp64, the oracle's per-frame window step and sliding loop against the reference pipeline run
with a stateful scheduler (tests/golden/pipeline_deis_ref.pt from tests/golden/gen_golden_deis.py), the host tables, the
config loader and the frame-sharded refusal."""
import copy
import math
import os
import sys

import pytest
import torch

from diffuman4d_b200.config import DEISConfig, DPMSolverConfig, SchedulerConfig, UniPCConfig
from oracle.deis_oracle import DEISOracle
from oracle.dpm_solver_oracle import denoise_window_oracle_per_frame, sliding_iterative_denoise_oracle_per_frame
from oracle.pipeline_oracle import DDIMOracle

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _golden():
    return torch.load(os.path.join(GOLD, "pipeline_deis_ref.pt"))


def _fake_unet(cin):
    sys.path.insert(0, GOLD)
    from fake_unet import make_fake_unet
    return make_fake_unet(cin)


def _fp64_deis(n, **kw):
    s = DEISOracle(DEISConfig(**kw), table_dtype=torch.float64)
    s.set_timesteps(n)
    return s


def _alpha_sigma(s, i):
    a, sig = DEISOracle._alpha_sigma_t(s.sigmas[i])
    return float(a), float(sig)


# ---- anchors ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pred", ["epsilon", "v_prediction", "sample"])
@pytest.mark.parametrize("beta", [dict(), dict(beta_schedule="scaled_linear", beta_start=0.00085, beta_end=0.012)])
def test_first_order_is_ddim(pred, beta):
    """Order 1 is DDIM (eta 0) between the same timesteps: sigma_t (e^h - 1) = alpha_t sigma_s / alpha_s - sigma_t, so
    (alpha_t / alpha_s) x - sigma_t (e^h - 1) eps = alpha_t x0 + sigma_t eps.  Trailing spacing makes DDIM's previous
    timestep the next table entry; DEIS's final sigma is that of alphas_cumprod[0], DDIM's final alpha_cumprod without
    set_alpha_to_one."""
    n = 10
    deis = _fp64_deis(n, solver_order=1, prediction_type=pred, timestep_spacing="trailing", **beta)
    ddim = DDIMOracle(SchedulerConfig(**{"beta_start": 1e-4, "beta_end": 0.02, "beta_schedule": "linear", **beta},
                                      prediction_type=pred, set_alpha_to_one=False, steps_offset=0,
                                      timestep_spacing="trailing"))
    ddim.set_timesteps(n)
    ddim.alphas_cumprod = ddim.alphas_cumprod.double()
    ddim.final_alpha_cumprod = ddim.alphas_cumprod[0]
    assert torch.equal(deis.timesteps, ddim.timesteps)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 3, 3, generator=g, dtype=torch.float64) * (1 + float(deis.sigmas[0]))
    for i, t in enumerate(deis.timesteps.tolist()):
        m = torch.randn(2, 4, 3, 3, generator=g, dtype=torch.float64)
        got, want = deis.step(m, t, x), ddim.step(m, t, x)
        assert (got - want).abs().max().item() <= 1e-12 * (1 + want.abs().max().item()), (i, pred)
        x = got


@pytest.mark.parametrize("order,lof", [(2, True), (2, False), (3, True), (3, False)])
@pytest.mark.parametrize("pred", ["epsilon", "v_prediction"])
def test_exact_denoiser_of_a_point_mass_stays_on_the_trajectory(order, lof, pred):
    """Data = one point x0*: the exact model output converts to the same epsilon eps* at every point of x_t = alpha_t x0*
    + sigma_t eps*, and the Lagrange weights of the second- and third-order updates integrate a constant exactly, so every
    step lands on the trajectory at its next sigma."""
    n = 12
    s = _fp64_deis(n, solver_order=order, lower_order_final=lof, prediction_type=pred)
    g = torch.Generator().manual_seed(1)
    x0s = torch.randn(3, 4, 5, 5, generator=g, dtype=torch.float64)
    eps = torch.randn(3, 4, 5, 5, generator=g, dtype=torch.float64)
    a, sig = _alpha_sigma(s, 0)
    x = a * x0s + sig * eps
    for i, t in enumerate(s.timesteps.tolist()):
        a, sig = _alpha_sigma(s, i)
        out = (x - a * x0s) / sig if pred == "epsilon" else a * ((x - a * x0s) / sig) - sig * x0s
        x = s.step(out, t, x)
        a1, sig1 = _alpha_sigma(s, i + 1)
        ref = a1 * x0s + sig1 * eps
        assert (x - ref).abs().max().item() <= 1e-9 * ref.abs().max().item(), (i, order)
    assert s.lower_order_nums == order


def _gaussian_error_at_t500(n, order):
    """Data ~ N(mu, s^2) per element: eps(x) = sigma_t (x - alpha mu) / (alpha^2 s^2 + sigma_t^2) exactly, and the
    probability-flow ODE keeps (x - alpha mu) / sqrt(alpha^2 s^2 + sigma_t^2) constant.  The error is taken after the
    first n / 2 steps, at timestep 500 for every even n (linspace spacing): the last steps of a 1000-step schedule, down
    to the sigma of timestep 0, shrink in log-SNR far slower than 1 / n and would hide the order."""
    mu, sd = 0.3, 0.5
    s = _fp64_deis(n, solver_order=order, lower_order_final=False)
    z = torch.linspace(-2.5, 2.5, 101, dtype=torch.float64)
    scale = lambda a, sig: math.sqrt(a * a * sd * sd + sig * sig)
    a, sig = _alpha_sigma(s, 0)
    x = a * mu + scale(a, sig) * z
    for i, t in enumerate(s.timesteps.tolist()[:n // 2]):
        a, sig = _alpha_sigma(s, i)
        x = s.step(sig * (x - a * mu) / scale(a, sig) ** 2, t, x)
    assert int(s.timesteps[n // 2]) == 500
    a, sig = _alpha_sigma(s, n // 2)
    return (x - (a * mu + scale(a, sig) * z)).abs().max().item()


# Error ratio per doubling of the steps (80 -> 160 -> 320): order p should give 2^p.  The integer timesteps of a
# 1000-step training schedule keep the fp64 run just short of the asymptote: it measured 1.99 / 1.99 at order 1,
# 3.80 / 3.87 at order 2 and 7.31 / 7.43 at order 3.  The bands do not overlap between orders.
@pytest.mark.parametrize("order,lo,hi", [(1, 1.8, 2.2), (2, 3.5, 4.4), (3, 6.5, 9.0)])
def test_convergence_order_on_gaussian_data(order, lo, hi):
    errs = [_gaussian_error_at_t500(n, order) for n in (80, 160, 320)]
    ratios = [errs[k] / errs[k + 1] for k in range(len(errs) - 1)]
    print(f"\norder {order}: errors at t = 500 {errs}, ratios {ratios}")
    for r in ratios:
        assert lo <= r <= hi, (order, errs, ratios)


# ---- the reference pipeline's per-frame scheduler copies (golden) ------------------------------------------------
def _config(c):
    return DEISConfig(**c["config"])


@pytest.mark.parametrize("tag", ["call_cfg_eps_order3", "call_nocfg_v_order3_nolof"])
def test_window_call_matches_reference_pipeline_golden(tag):
    """``__call__`` with fresh per-frame copies handed over at nonzero timestep indices: each frame's step index starts at
    its timestep and its order count at 0."""
    c = _golden()["cases"][tag]
    i = c["in"]
    s = DEISOracle(_config(c))
    s.set_timesteps(c["n_steps_table"])
    assert torch.equal(s.timesteps, c["timesteps_table"])
    scheds = [copy.deepcopy(s) for _ in range(len(i["latents"]))]
    lat, ti = denoise_window_oracle_per_frame(
        _fake_unet(11), scheds, latents=i["latents"].clone(), pixel_latents=i["pixel_latents"], plucker=i["plucker"],
        skeletons=i["skeletons"], cond_mask=i["cond_mask"], timestep_indices=i["timestep_indices"], domain="spatial",
        guidance_scale=c["guidance"], num_inference_steps=c["num_inference_steps"], enable_pose_encoder=True)
    torch.testing.assert_close(lat, c["out_latents"], rtol=1e-5, atol=1e-6)
    assert torch.equal(ti, c["out_timestep_indices"])
    assert [f.lower_order_nums for f in scheds] == c["lower_order_nums"]


SLIDE_TAGS = ["slide_spatial_eps_cfg_order3", "slide_temporal_bidir_v_nocfg", "slide_spatial_order1_leading_sample",
              "slide_spatial_order3_nolof_trailing"]


def _slide(c, cfg, task):
    i = task["in"]
    return sliding_iterative_denoise_oracle_per_frame(
        _fake_unet(11), DEISOracle(cfg), pixel_latents=i["pixel_latents"], plucker=i["plucker"], skeletons=i["skeletons"],
        cond_mask=i["cond_mask_latents"], latents=i["latents"], domain=c["domain"],
        timestep_indices=i["timestep_indices"], window_size=c["window_size"], sliding_stride=c["sliding_stride"],
        bidirectional=c["bidirectional"], num_denoising_steps=1, alternation_rounds=c["alternation_rounds"],
        guidance_scale=c["guidance"], enable_pose_encoder=True)


@pytest.mark.parametrize("tag", SLIDE_TAGS)
def test_sliding_loop_matches_reference_pipeline_golden(tag):
    """Two successive tasks on one scheduler object: per-frame histories across windows, reset per task."""
    c = _golden()["cases"][tag]
    for task in c["tasks"]:
        out = _slide(c, _config(c), task)
        torch.testing.assert_close(out["latents"], task["out_latents"], rtol=1e-5, atol=1e-5)
        assert torch.equal(out["timestep_indices"], task["out_timestep_indices"])
        assert torch.equal(out["fully_denoised"], task["fully_denoised"])


@pytest.mark.parametrize("tag,flip", [("slide_spatial_order3_nolof_trailing", {"lower_order_final": True}),
                                      ("slide_spatial_order3_nolof_trailing", {"solver_order": 2}),
                                      ("slide_spatial_eps_cfg_order3", {"solver_order": 2})])
def test_golden_cases_pin_the_order_knobs(tag, flip):
    """Flipping the knob gives a different result, so the fixture does pin it."""
    c = _golden()["cases"][tag]
    out = _slide(c, DEISConfig(**{**c["config"], **flip}), c["tasks"][0])
    assert (out["latents"] - c["tasks"][0]["out_latents"]).abs().max() > 1e-3


# ---- tables -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(), dict(solver_order=1), dict(solver_order=3),
                                dict(solver_order=3, lower_order_final=False, timestep_spacing="trailing"),
                                dict(timestep_spacing="leading", steps_offset=1, prediction_type="v_prediction"),
                                dict(solver_order=3, beta_schedule="scaled_linear", beta_start=0.00085, beta_end=0.012)])
@pytest.mark.parametrize("n", [3, 10, 20])
def test_tables_equal_a_hand_evaluation_in_upstreams_order(kw, n):
    """Every coefficient equals the oracle's restatement of upstream's update functions evaluated at that row, bit for
    bit, and the order cap follows upstream's lower_order_final / lower_order_second rule."""
    from diffuman4d_b200.scheduler import DEISTables
    t = DEISTables(DEISConfig(**kw), device="cpu")
    o = DEISOracle(t.config)
    assert torch.equal(t.set_timesteps(n), o.set_timesteps(n))
    assert t.sigmas.dtype == torch.float32 and torch.equal(t.sigmas, o.sigmas)
    assert t.coefs.dtype == torch.float32 and t.coefs.shape == (n, 11)
    c = t.config
    for i in range(n):
        a_s, s_s = DEISOracle._alpha_sigma_t(o.sigmas[i])
        a_t = DEISOracle._alpha_sigma_t(o.sigmas[i + 1])[0]
        want = [a_s.item(), s_s.item(), *(v.item() for v in o.first_order_coefs(i)), a_t.item()]
        want += [v.item() for v in o.second_order_coefs(i)] if i >= 1 else [0.0] * 2
        want += [v.item() for v in o.third_order_coefs(i)] if i >= 2 else [0.0] * 3
        cap = min(c.solver_order, i + 1)
        if c.lower_order_final and n < 15:
            cap = min(cap, {n - 1: 1, n - 2: 2}.get(i, cap))
        assert t.coefs[i].tolist() == want + [float(cap)], i


def test_tables_refuse_what_the_step_does_not_implement():
    from diffuman4d_b200.scheduler import DEISTables, DPMSolverTables, UniPCTables
    with pytest.raises(NotImplementedError, match="orders 1, 2 and 3"):
        DEISTables(DEISConfig(solver_order=4), device="cpu")
    with pytest.raises(ValueError, match="duplicate"):
        DEISTables(DEISConfig(num_train_timesteps=10), device="cpu").set_timesteps(10)
    with pytest.raises(ValueError):
        DEISTables(DEISConfig(beta_schedule="squaredcos_cap_v2"), device="cpu")
    # DPM-Solver++ and UniPC keep their order-2 limit
    for tables, cfg in ((DPMSolverTables, DPMSolverConfig), (UniPCTables, UniPCConfig)):
        with pytest.raises(NotImplementedError, match="solver_order=3: the fused step implements orders 1 and 2$"):
            tables(cfg(solver_order=3), device="cpu")


# ---- loader -------------------------------------------------------------------------------------------------------
# a DEISMultistepScheduler config as diffusers 0.33.1 saves it, every key present
DEIS_SCHEDULER_CONFIG = {
    "_class_name": "DEISMultistepScheduler", "_diffusers_version": "0.33.1", "num_train_timesteps": 1000,
    "beta_start": 0.00085, "beta_end": 0.012, "beta_schedule": "scaled_linear", "trained_betas": None,
    "solver_order": 3, "prediction_type": "v_prediction", "thresholding": False, "dynamic_thresholding_ratio": 0.995,
    "sample_max_value": 1.0, "algorithm_type": "deis", "solver_type": "logrho", "lower_order_final": False,
    "use_karras_sigmas": False, "use_exponential_sigmas": False, "use_beta_sigmas": False, "use_flow_sigmas": False,
    "flow_shift": 1.0, "timestep_spacing": "leading", "steps_offset": 1, "use_dynamic_shifting": False,
    "time_shift_type": "exponential",
}


def test_loader_maps_a_full_deis_config():
    from diffuman4d_b200.loader import scheduler_config_from_json
    assert scheduler_config_from_json(DEIS_SCHEDULER_CONFIG) == DEISConfig(
        beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", solver_order=3, prediction_type="v_prediction",
        lower_order_final=False, timestep_spacing="leading", steps_offset=1)
    assert scheduler_config_from_json({"_class_name": "DEISMultistepScheduler"}) == DEISConfig()


@pytest.mark.parametrize("key,value", [("algorithm_type", "dpmsolver++"), ("solver_type", "midpoint"),
                                       ("solver_order", 4), ("thresholding", True), ("use_karras_sigmas", True),
                                       ("use_exponential_sigmas", True), ("use_beta_sigmas", True),
                                       ("use_flow_sigmas", True), ("use_dynamic_shifting", True),
                                       ("rescale_betas_zero_snr", True), ("trained_betas", [0.1, 0.2]),
                                       ("beta_schedule", "squaredcos_cap_v2"), ("timestep_spacing", "karras"),
                                       ("prediction_type", "flow_prediction")])
def test_loader_rejects_unsupported_deis_keys(key, value):
    from diffuman4d_b200.loader import scheduler_config_from_json
    with pytest.raises(NotImplementedError, match=key):
        scheduler_config_from_json({**DEIS_SCHEDULER_CONFIG, key: value})


# ---- frame-sharded refusal --------------------------------------------------------------------------------------------
def test_frame_sharded_pipeline_refuses_deis_before_any_allocation(monkeypatch):
    import diffuman4d_b200.sharded as sharded_mod
    from diffuman4d_b200.config import UNetConfig
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline

    class _UNetStub:
        device = torch.device("cpu")
        config = UNetConfig.tiny()

    pipe = B200Diffuman4DPipeline(_UNetStub(), DEISConfig(solver_order=3))
    monkeypatch.setattr(sharded_mod, "lib", lambda: pytest.fail("the library was called"))
    monkeypatch.setattr(sharded_mod.dist, "is_initialized", lambda: pytest.fail("torch.distributed was consulted"))
    monkeypatch.setattr(torch.cuda, "device", lambda *a: pytest.fail("a device was selected"))
    with pytest.raises(NotImplementedError, match="DEIS"):
        sharded_mod.FrameShardedPipeline(pipe, max_frames=8, h=8, w=8)
