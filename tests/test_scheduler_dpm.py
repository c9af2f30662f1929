"""DPM-Solver++ (upstream DPMSolverMultistepScheduler, dpmsolver++ / midpoint) on the CPU: mathematical anchors for the
restated arithmetic in fp64, the oracle's per-frame sliding loop against the reference pipeline run with a stateful
scheduler (tests/golden/pipeline_dpm_ref.pt from tests/golden/gen_golden_dpm.py), the config loader and the host tables."""
import copy
import math
import os
import sys

import numpy as np
import pytest
import torch

from diffuman4d_b200.config import DPMSolverConfig, SchedulerConfig
from oracle.dpm_solver_oracle import (DPMSolverOracle, denoise_window_oracle_per_frame,
                                      sliding_iterative_denoise_oracle_per_frame)
from oracle.pipeline_oracle import DDIMOracle

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _load_golden(name):
    g = torch.load(os.path.join(GOLD, f"{name}.pt"))
    i = 0
    while os.path.exists(os.path.join(GOLD, f"{name}.inputs{i}.pt")):
        for path, t in torch.load(os.path.join(GOLD, f"{name}.inputs{i}.pt")).items():
            *parents, leaf = path.split("/")
            node = g
            for k in parents:
                node = node[k]
            node[leaf] = t
        i += 1
    return g


def _fake_unet(cin):
    sys.path.insert(0, GOLD)
    from fake_unet import make_fake_unet
    return make_fake_unet(cin)


def _fp64_dpm(n, **kw):
    s = DPMSolverOracle(DPMSolverConfig(**kw), table_dtype=torch.float64)
    s.set_timesteps(n)
    return s


def _alpha_sigma(s, i):
    a, sig = DPMSolverOracle._alpha_sigma_t(s.sigmas[i])
    return float(a), float(sig)


# ---- anchors ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pred", ["epsilon", "v_prediction", "sample"])
def test_first_order_step_is_ddim(pred):
    """DPM-Solver++ of order 1 is DDIM (eta 0) between the same two timesteps: trailing spacing makes DDIM's previous
    timestep the next table entry, and a zero final sigma is DDIM's final alpha_cumprod of 1."""
    n = 10
    dpm = _fp64_dpm(n, solver_order=1, prediction_type=pred, timestep_spacing="trailing")
    ddim = DDIMOracle(SchedulerConfig(beta_start=1e-4, beta_end=0.02, beta_schedule="linear", prediction_type=pred,
                                      set_alpha_to_one=True, steps_offset=0, timestep_spacing="trailing"))
    ddim.set_timesteps(n)
    ddim.alphas_cumprod = ddim.alphas_cumprod.double()
    ddim.final_alpha_cumprod = torch.tensor(1.0, dtype=torch.float64)
    assert torch.equal(dpm.timesteps, ddim.timesteps)
    g = torch.Generator().manual_seed(0)
    for i, t in enumerate(dpm.timesteps.tolist()):
        x = torch.randn(2, 4, 3, 3, generator=g, dtype=torch.float64) * (1 + float(dpm.sigmas[i]))
        m = torch.randn(2, 4, 3, 3, generator=g, dtype=torch.float64)
        s = copy.deepcopy(dpm)
        s.step_index = i
        got, ref = s.step(m, t, x), ddim.step(m, t, x)
        assert (got - ref).abs().max().item() <= 1e-12 * (1 + ref.abs().max().item()), (i, pred)


@pytest.mark.parametrize("order,final", [(1, "zero"), (2, "zero"), (2, "sigma_min"), (1, "sigma_min")])
def test_exact_denoiser_of_a_point_mass_stays_on_the_trajectory(order, final):
    """Data = one point x0*: the exact epsilon-prediction makes both orders follow alpha_t x0* + sigma_t eps* exactly."""
    n = 12
    s = _fp64_dpm(n, solver_order=order, final_sigmas_type=final, lower_order_final=False)
    g = torch.Generator().manual_seed(1)
    x0s = torch.randn(3, 4, 5, 5, generator=g, dtype=torch.float64)
    eps = torch.randn(3, 4, 5, 5, generator=g, dtype=torch.float64)
    a, sig = _alpha_sigma(s, 0)
    x = a * x0s + sig * eps
    for i, t in enumerate(s.timesteps.tolist()):
        a, sig = _alpha_sigma(s, i)
        x = s.step((x - a * x0s) / sig, t, x)
        a1, sig1 = _alpha_sigma(s, i + 1)
        ref = a1 * x0s + sig1 * eps
        assert (x - ref).abs().max().item() <= 1e-9 * ref.abs().max().item(), (i, order, final)
    assert s.lower_order_nums == order


def _gaussian_endpoint_error(n, order):
    """Data ~ N(mu, s^2) per element: eps(x) = sigma_t (x - alpha mu) / (alpha^2 s^2 + sigma_t^2) exactly, and the
    probability-flow ODE keeps (x - alpha mu) / sqrt(alpha^2 s^2 + sigma_t^2) constant."""
    mu, sd = 0.3, 0.5
    s = _fp64_dpm(n, solver_order=order, final_sigmas_type="sigma_min", lower_order_final=False)
    z = torch.linspace(-2.5, 2.5, 101, dtype=torch.float64)
    scale = lambda a, sig: math.sqrt(a * a * sd * sd + sig * sig)
    a, sig = _alpha_sigma(s, 0)
    x = a * mu + scale(a, sig) * z
    for i, t in enumerate(s.timesteps.tolist()):
        a, sig = _alpha_sigma(s, i)
        x = s.step(sig * (x - a * mu) / scale(a, sig) ** 2, t, x)
    a, sig = _alpha_sigma(s, n)
    return (x - (a * mu + scale(a, sig) * z)).abs().max().item()


@pytest.mark.parametrize("order,lo,hi", [(1, 1.6, 2.6), (2, 3.3, 5.0)])
def test_convergence_order_on_gaussian_data(order, lo, hi):
    errs = [_gaussian_endpoint_error(n, order) for n in (50, 100, 200)]
    ratios = [errs[k] / errs[k + 1] for k in range(len(errs) - 1)]
    print(f"\norder {order}: endpoint errors {errs}, ratios {ratios}")
    for r in ratios:
        assert lo <= r <= hi, (order, errs, ratios)


# ---- the reference pipeline's per-frame scheduler copies (golden) ------------------------------------------------
@pytest.mark.parametrize("tag", ["call_cfg_eps", "call_nocfg_v"])
def test_window_call_matches_reference_pipeline_golden(tag):
    c = _load_golden("pipeline_dpm_ref")["cases"][tag]
    i = c["in"]
    s = DPMSolverOracle(DPMSolverConfig(**c["config"]))
    s.set_timesteps(c["n_steps_table"])
    assert torch.equal(s.timesteps, c["timesteps_table"])
    scheds = [copy.deepcopy(s) for _ in range(len(i["latents"]))]
    lat, ti = denoise_window_oracle_per_frame(
        _fake_unet(11), scheds, latents=i["latents"].clone(), pixel_latents=i["pixel_latents"], plucker=i["plucker"],
        skeletons=i["skeletons"], cond_mask=i["cond_mask"], timestep_indices=i["timestep_indices"], domain="spatial",
        guidance_scale=c["guidance"], num_inference_steps=3, enable_pose_encoder=True)
    torch.testing.assert_close(lat, c["out_latents"], rtol=1e-5, atol=1e-6)
    assert torch.equal(ti, c["out_timestep_indices"])
    assert [f.lower_order_nums for f in scheds] == c["lower_order_nums"]


@pytest.mark.parametrize("tag", ["slide_spatial_eps_cfg", "slide_temporal_bidir_v_nocfg", "slide_spatial_sigma_min_lof",
                                 "slide_spatial_sigma_min_nolof"])
def test_sliding_loop_matches_reference_pipeline_golden(tag):
    """Two successive tasks on one scheduler object: per-frame histories across windows, reset per task."""
    c = _load_golden("pipeline_dpm_ref")["cases"][tag]
    s = DPMSolverOracle(DPMSolverConfig(**c["config"]))
    for task in c["tasks"]:
        i = task["in"]
        out = sliding_iterative_denoise_oracle_per_frame(
            _fake_unet(11), s, pixel_latents=i["pixel_latents"], plucker=i["plucker"], skeletons=i["skeletons"],
            cond_mask=i["cond_mask_latents"], latents=i["latents"], domain=c["domain"],
            timestep_indices=i["timestep_indices"], window_size=c["window_size"], sliding_stride=c["sliding_stride"],
            bidirectional=c["bidirectional"], num_denoising_steps=1, alternation_rounds=c["alternation_rounds"],
            guidance_scale=c["guidance"], enable_pose_encoder=True)
        torch.testing.assert_close(out["latents"], task["out_latents"], rtol=1e-5, atol=1e-5)
        assert torch.equal(out["timestep_indices"], task["out_timestep_indices"])
        assert torch.equal(out["fully_denoised"], task["fully_denoised"])


def test_golden_lower_order_final_changes_the_last_step():
    """The sigma_min fixtures reach the last step with fewer than 15 steps, so lower_order_final decides its order: the
    flipped flag must give a different result (the two cases do pin both branches)."""
    c = _load_golden("pipeline_dpm_ref")["cases"]["slide_spatial_sigma_min_lof"]
    cfg = DPMSolverConfig(**{**c["config"], "lower_order_final": False})
    i = c["tasks"][0]["in"]
    out = sliding_iterative_denoise_oracle_per_frame(
        _fake_unet(11), DPMSolverOracle(cfg), pixel_latents=i["pixel_latents"], plucker=i["plucker"],
        skeletons=i["skeletons"], cond_mask=i["cond_mask_latents"], latents=i["latents"], domain=c["domain"],
        timestep_indices=i["timestep_indices"], window_size=c["window_size"], sliding_stride=c["sliding_stride"],
        bidirectional=c["bidirectional"], num_denoising_steps=1, alternation_rounds=c["alternation_rounds"],
        guidance_scale=c["guidance"], enable_pose_encoder=True)
    assert (out["latents"] - c["tasks"][0]["out_latents"]).abs().max() > 1e-3


# ---- loader -------------------------------------------------------------------------------------------------------
def test_loader_maps_dpm_solver_config():
    from diffuman4d_b200.loader import scheduler_config_from_json
    d = {"_class_name": "DPMSolverMultistepScheduler", "_diffusers_version": "0.33.1", "num_train_timesteps": 1000,
         "beta_start": 0.00085, "beta_end": 0.012, "beta_schedule": "scaled_linear", "solver_order": 2,
         "prediction_type": "v_prediction", "algorithm_type": "dpmsolver++", "solver_type": "midpoint",
         "lower_order_final": True, "euler_at_final": False, "final_sigmas_type": "zero", "timestep_spacing": "leading",
         "steps_offset": 1, "thresholding": False, "use_karras_sigmas": False, "use_exponential_sigmas": False,
         "use_beta_sigmas": False, "use_lu_lambdas": False, "use_flow_sigmas": False, "rescale_betas_zero_snr": False,
         "lambda_min_clipped": -math.inf, "variance_type": None, "dynamic_thresholding_ratio": 0.995,
         "sample_max_value": 1.0, "trained_betas": None}
    assert scheduler_config_from_json(d) == DPMSolverConfig(
        beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", solver_order=2, prediction_type="v_prediction",
        lower_order_final=True, euler_at_final=False, final_sigmas_type="zero", timestep_spacing="leading",
        steps_offset=1)
    assert scheduler_config_from_json({"_class_name": "DPMSolverMultistepScheduler"}) == DPMSolverConfig()
    assert isinstance(scheduler_config_from_json({"_class_name": "DDIMScheduler"}), SchedulerConfig)


@pytest.mark.parametrize("key,value", [("thresholding", True), ("use_karras_sigmas", True),
                                       ("use_exponential_sigmas", True), ("use_beta_sigmas", True),
                                       ("use_lu_lambdas", True), ("use_flow_sigmas", True),
                                       ("rescale_betas_zero_snr", True), ("lambda_min_clipped", -5.1),
                                       ("variance_type", "learned_range"), ("algorithm_type", "sde-dpmsolver++"),
                                       ("algorithm_type", "dpmsolver"), ("algorithm_type", "sde-dpmsolver"),
                                       ("solver_type", "heun"), ("solver_order", 3)])
def test_loader_rejects_unsupported_dpm_solver_keys(key, value):
    from diffuman4d_b200.loader import scheduler_config_from_json
    with pytest.raises(NotImplementedError, match=key):
        scheduler_config_from_json({"_class_name": "DPMSolverMultistepScheduler", key: value})


# ---- tables -------------------------------------------------------------------------------------------------------
def _hand_sigmas(ts):
    betas = np.linspace(1e-4, 0.02, 1000, dtype=np.float64)
    ac = np.cumprod(1 - betas)
    return np.sqrt((1 - ac) / ac)[ts]


@pytest.mark.parametrize("spacing,ts", [
    ("linspace", [999, 899, 799, 699, 599, 500, 400, 300, 200, 100]),
    ("leading", [901, 811, 721, 631, 541, 451, 361, 271, 181, 91]),      # 1000 // 11 = 90, steps_offset 1
    ("trailing", [999, 899, 799, 699, 599, 499, 399, 299, 199, 99]),
])
@pytest.mark.parametrize("final", ["zero", "sigma_min"])
def test_tables_timesteps_and_sigmas(spacing, ts, final):
    from diffuman4d_b200.scheduler import DPMSolverTables
    t = DPMSolverTables(DPMSolverConfig(timestep_spacing=spacing, steps_offset=1, final_sigmas_type=final), device="cpu")
    assert t.set_timesteps(10).tolist() == ts
    assert t.sigmas.dtype == torch.float32 and t.sigmas.shape == (11,)
    np.testing.assert_allclose(t.sigmas[:10].numpy(), _hand_sigmas(ts), rtol=2e-5)
    if final == "zero":
        assert float(t.sigmas[10]) == 0.0
    else:
        assert math.isclose(float(t.sigmas[10]), _hand_sigmas([0])[0], rel_tol=1e-4)   # fp32 cumprod, 1 - ac cancels
    assert t.final_first_order                                       # 10 < 15 steps with lower_order_final
    # the device coefficients are the oracle's step coefficients, bit for bit
    o = DPMSolverOracle(t.config)
    o.set_timesteps(10)
    assert torch.equal(o.sigmas, t.sigmas)
    for i in range(10):
        a_s, s_s = DPMSolverOracle._alpha_sigma_t(o.sigmas[i])
        a_t, s_t = DPMSolverOracle._alpha_sigma_t(o.sigmas[i + 1])
        h = o._lambda(i + 1) - o._lambda(i)
        c = a_t * (torch.exp(-h) - 1.0)
        assert t.coefs[i, :5].tolist() == [a_s.item(), s_s.item(), (s_t / s_s).item(), c.item(),
                                           (0.5 * c).item()]
        if i > 0:
            assert t.coefs[i, 5].item() == (1.0 / ((o._lambda(i) - o._lambda(i - 1)) / h)).item()


def test_tables_final_policy_and_duplicates():
    from diffuman4d_b200.scheduler import DPMSolverTables
    t = DPMSolverTables(DPMSolverConfig(final_sigmas_type="sigma_min"), device="cpu")
    t.set_timesteps(20)
    assert not t.final_first_order                                   # 20 >= 15 steps, sigma_min
    t.set_timesteps(14)
    assert t.final_first_order                                       # lower_order_final below 15 steps
    t = DPMSolverTables(DPMSolverConfig(final_sigmas_type="sigma_min", euler_at_final=True), device="cpu")
    t.set_timesteps(20)
    assert t.final_first_order
    with pytest.raises(ValueError, match="duplicate"):
        DPMSolverTables(DPMSolverConfig(num_train_timesteps=10), device="cpu").set_timesteps(10)
    with pytest.raises(ValueError, match="duplicate"):
        DPMSolverOracle(DPMSolverConfig(num_train_timesteps=10)).set_timesteps(10)
    with pytest.raises(NotImplementedError):
        DPMSolverTables(DPMSolverConfig(solver_order=3), device="cpu")
