"""UniPC (upstream UniPCMultistepScheduler, predict_x0, bh1 / bh2) on the CPU: mathematical anchors for the restated
arithmetic in fp64, the oracle's per-frame window step and sliding loop against the reference pipeline run with a stateful
scheduler (tests/golden/pipeline_unipc_ref.pt from tests/golden/gen_golden_unipc.py), the host tables, the config loader
and the frame-sharded refusal."""
import copy
import math
import os
import sys

import pytest
import torch

from diffuman4d_b200.config import DPMSolverConfig, SchedulerConfig, UniPCConfig
from oracle.dpm_solver_oracle import (DPMSolverOracle, denoise_window_oracle_per_frame,
                                      sliding_iterative_denoise_oracle_per_frame)
from oracle.pipeline_oracle import DDIMOracle
from oracle.unipc_oracle import UniPCOracle

GOLD = os.path.join(os.path.dirname(__file__), "golden")
NO_CORRECTOR = tuple(range(1000))


def _golden():
    return torch.load(os.path.join(GOLD, "pipeline_unipc_ref.pt"))


def _fake_unet(cin):
    sys.path.insert(0, GOLD)
    from fake_unet import make_fake_unet
    return make_fake_unet(cin)


def _fp64_unipc(n, **kw):
    s = UniPCOracle(UniPCConfig(**kw), table_dtype=torch.float64)
    s.set_timesteps(n)
    return s


def _alpha_sigma(s, i):
    a, sig = UniPCOracle._alpha_sigma_t(s.sigmas[i])
    return float(a), float(sig)


# ---- anchors ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pred", ["epsilon", "v_prediction", "sample"])
@pytest.mark.parametrize("solver_type", ["bh1", "bh2"])
def test_first_order_predictor_is_ddim_and_dpm_solver(pred, solver_type):
    """UniP of order 1 without the corrector is DDIM (eta 0) and DPM-Solver++ of order 1 between the same timesteps (B(h)
    only scales the second-order term).  Trailing spacing makes DDIM's previous timestep the next table entry; a zero
    final sigma is DDIM's final alpha_cumprod of 1."""
    n = 10
    uni = _fp64_unipc(n, solver_order=1, prediction_type=pred, timestep_spacing="trailing", solver_type=solver_type,
                      final_sigmas_type="sigma_min" if solver_type == "bh1" else "zero", disable_corrector=NO_CORRECTOR)
    dpm = DPMSolverOracle(DPMSolverConfig(**{k: v for k, v in vars(uni.cfg).items()
                                             if k in DPMSolverConfig.__dataclass_fields__}), table_dtype=torch.float64)
    dpm.set_timesteps(n)
    ddim = DDIMOracle(SchedulerConfig(beta_start=1e-4, beta_end=0.02, beta_schedule="linear", prediction_type=pred,
                                      set_alpha_to_one=True, steps_offset=0, timestep_spacing="trailing"))
    ddim.set_timesteps(n)
    ddim.alphas_cumprod = ddim.alphas_cumprod.double()
    ddim.final_alpha_cumprod = torch.tensor(1.0 if solver_type == "bh2" else float(ddim.alphas_cumprod[0]),
                                            dtype=torch.float64)
    assert torch.equal(uni.timesteps, ddim.timesteps)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 3, 3, generator=g, dtype=torch.float64) * (1 + float(uni.sigmas[0]))
    for i, t in enumerate(uni.timesteps.tolist()):
        m = torch.randn(2, 4, 3, 3, generator=g, dtype=torch.float64)
        s = copy.deepcopy(dpm)
        s.step_index = i
        got, want_dpm = uni.step(m, t, x), s.step(m, t, x)
        tol = 1e-12 * (1 + want_dpm.abs().max().item())
        assert (got - want_dpm).abs().max().item() <= tol, (i, pred)
        if i < n - 1 or solver_type == "bh2":      # DDIM's final alpha is alphas_cumprod[0] only at the last step
            want_ddim = ddim.step(m, t, x)
            assert (got - want_ddim).abs().max().item() <= tol, (i, pred)
        x = got


@pytest.mark.parametrize("order,final,lof", [(1, "zero", True), (2, "zero", True), (2, "sigma_min", False),
                                             (1, "sigma_min", False), (2, "sigma_min", True)])
@pytest.mark.parametrize("solver_type", ["bh1", "bh2"])
def test_exact_denoiser_of_a_point_mass_stays_on_the_trajectory(order, final, lof, solver_type):
    """Data = one point x0*: with the exact epsilon-prediction every data prediction is x0*, so the predictor and the
    corrector both follow alpha_t x0* + sigma_t eps* exactly, at either order."""
    if final == "zero" and solver_type == "bh1":
        pytest.skip("bh1 with a zero final sigma is refused (infinite B(h) at the last step)")
    n = 12
    s = _fp64_unipc(n, solver_order=order, final_sigmas_type=final, lower_order_final=lof, solver_type=solver_type)
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


def _gaussian_endpoint_error(n, order, **kw):
    """Data ~ N(mu, s^2) per element: eps(x) = sigma_t (x - alpha mu) / (alpha^2 s^2 + sigma_t^2) exactly, and the
    probability-flow ODE keeps (x - alpha mu) / sqrt(alpha^2 s^2 + sigma_t^2) constant."""
    mu, sd = 0.3, 0.5
    s = _fp64_unipc(n, solver_order=order, final_sigmas_type="sigma_min", lower_order_final=False, **kw)
    z = torch.linspace(-2.5, 2.5, 101, dtype=torch.float64)
    scale = lambda a, sig: math.sqrt(a * a * sd * sd + sig * sig)
    a, sig = _alpha_sigma(s, 0)
    x = a * mu + scale(a, sig) * z
    for i, t in enumerate(s.timesteps.tolist()):
        a, sig = _alpha_sigma(s, i)
        x = s.step(sig * (x - a * mu) / scale(a, sig) ** 2, t, x)
    a, sig = _alpha_sigma(s, n)
    return (x - (a * mu + scale(a, sig) * z)).abs().max().item()


# Error ratio per doubling of the steps (100 -> 200 -> 400).  Order p alone should give 2^p, and a predictor of order p
# plus the corrector 2^(p+1).  The integer timesteps of a 1000-step training schedule keep the fp64 run short of the
# asymptote: it measured 1.97 / 1.99 for order 1 alone, 3.21 / 3.37 (bh2) and 3.31 / 3.59 (bh1) for order 1 + corrector,
# and 4.94 / 5.78 (bh2) and 5.84 / 6.84 (bh1) for order 2 + corrector, against about 4 for order 2 alone.
@pytest.mark.parametrize("order,solver_type,corrector,lo,hi", [
    (1, "bh2", False, 1.8, 2.2),
    (1, "bh2", True, 2.9, 4.4), (1, "bh1", True, 2.9, 4.4),
    (2, "bh2", True, 4.5, 8.8), (2, "bh1", True, 4.5, 8.8),
])
def test_convergence_order_on_gaussian_data(order, solver_type, corrector, lo, hi):
    kw = dict(solver_type=solver_type, disable_corrector=() if corrector else NO_CORRECTOR)
    errs = [_gaussian_endpoint_error(n, order, **kw) for n in (100, 200, 400)]
    ratios = [errs[k] / errs[k + 1] for k in range(len(errs) - 1)]
    print(f"\norder {order} {solver_type} corrector={corrector}: endpoint errors {errs}, ratios {ratios}")
    for r in ratios:
        assert lo <= r <= hi, (order, errs, ratios)


# ---- the reference pipeline's per-frame scheduler copies (golden) ------------------------------------------------
def _config(c):
    return UniPCConfig(**c["config"])


@pytest.mark.parametrize("tag", ["call_cfg_eps", "call_nocfg_v_order1"])
def test_window_call_matches_reference_pipeline_golden(tag):
    c = _golden()["cases"][tag]
    i = c["in"]
    s = UniPCOracle(_config(c))
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


SLIDE_TAGS = ["slide_spatial_eps_cfg", "slide_temporal_bidir_v_nocfg", "slide_spatial_order1_bh1",
              "slide_spatial_sigma_min_nolof_disable_corrector"]


def _slide(c, cfg, task):
    i = task["in"]
    return sliding_iterative_denoise_oracle_per_frame(
        _fake_unet(11), UniPCOracle(cfg), pixel_latents=i["pixel_latents"], plucker=i["plucker"], skeletons=i["skeletons"],
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


@pytest.mark.parametrize("tag,flip", [("slide_spatial_sigma_min_nolof_disable_corrector", {"disable_corrector": ()}),
                                      ("slide_spatial_sigma_min_nolof_disable_corrector", {"lower_order_final": True})])
def test_golden_cases_pin_the_corrector_and_final_order_knobs(tag, flip):
    """Flipping the knob gives a different result, so the fixture does pin it."""
    c = _golden()["cases"][tag]
    out = _slide(c, UniPCConfig(**{**c["config"], **flip}), c["tasks"][0])
    assert (out["latents"] - c["tasks"][0]["out_latents"]).abs().max() > 1e-3


# ---- tables -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(), dict(solver_order=1), dict(timestep_spacing="leading", steps_offset=1),
                                dict(timestep_spacing="trailing", final_sigmas_type="sigma_min", solver_type="bh1"),
                                dict(lower_order_final=False, final_sigmas_type="sigma_min", disable_corrector=(2, 5)),
                                dict(beta_schedule="scaled_linear", beta_start=0.00085, beta_end=0.012)])
def test_tables_equal_the_oracle_bit_for_bit(kw):
    from diffuman4d_b200.scheduler import UniPCTables
    n = 10
    t = UniPCTables(UniPCConfig(**kw), device="cpu")
    o = UniPCOracle(t.config)
    assert torch.equal(t.set_timesteps(n), o.set_timesteps(n))
    assert t.sigmas.dtype == torch.float32 and torch.equal(t.sigmas, o.sigmas)
    c = t.config
    for i in range(n):
        a_s, s_s = UniPCOracle._alpha_sigma_t(o.sigmas[i])
        p = o.bh_coefs(i + 1, i, i - 1 if i > 0 else None)
        want = [a_s.item(), s_s.item(), p.ratio.item(), p.cphi.item(), p.cB.item(), p.rk.item() if i > 0 else 0.0]
        if i > 0:
            k = o.bh_coefs(i, i - 1, i - 2 if i > 1 else None)
            rho = o.rhos_c(k).tolist() if i > 1 else [0.0, 0.0]
            want += [k.ratio.item(), k.cphi.item(), k.cB.item(), k.rk.item() if i > 1 else 0.0, *rho]
        else:
            want += [0.0] * 6
        want += [float(i > 0 and i - 1 not in c.disable_corrector),
                 float(min(c.solver_order, n - i) if c.lower_order_final else c.solver_order)]
        assert t.coefs[i].tolist() == want, i


def test_tables_refuse_what_the_step_does_not_implement():
    from diffuman4d_b200.scheduler import UniPCTables
    with pytest.raises(NotImplementedError, match="lower_order_final"):
        UniPCTables(UniPCConfig(lower_order_final=False), device="cpu")
    with pytest.raises(NotImplementedError, match="bh1"):
        UniPCTables(UniPCConfig(solver_type="bh1"), device="cpu")
    with pytest.raises(NotImplementedError):
        UniPCTables(UniPCConfig(solver_order=3), device="cpu")
    with pytest.raises(ValueError, match="duplicate"):
        UniPCTables(UniPCConfig(num_train_timesteps=10), device="cpu").set_timesteps(10)


# ---- loader -------------------------------------------------------------------------------------------------------
def test_loader_maps_unipc_config():
    from diffuman4d_b200.loader import scheduler_config_from_json
    d = {"_class_name": "UniPCMultistepScheduler", "_diffusers_version": "0.33.1", "num_train_timesteps": 1000,
         "beta_start": 0.00085, "beta_end": 0.012, "beta_schedule": "scaled_linear", "solver_order": 2,
         "prediction_type": "v_prediction", "predict_x0": True, "solver_type": "bh1", "lower_order_final": True,
         "disable_corrector": [0, 3], "solver_p": None, "final_sigmas_type": "sigma_min", "timestep_spacing": "leading",
         "steps_offset": 1, "thresholding": False, "dynamic_thresholding_ratio": 0.995, "sample_max_value": 1.0,
         "use_karras_sigmas": False, "use_exponential_sigmas": False, "use_beta_sigmas": False,
         "use_flow_sigmas": False, "flow_shift": 1.0, "rescale_betas_zero_snr": False, "trained_betas": None}
    assert scheduler_config_from_json(d) == UniPCConfig(
        beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", solver_order=2, prediction_type="v_prediction",
        solver_type="bh1", lower_order_final=True, disable_corrector=(0, 3), final_sigmas_type="sigma_min",
        timestep_spacing="leading", steps_offset=1)
    assert scheduler_config_from_json({"_class_name": "UniPCMultistepScheduler"}) == UniPCConfig()


@pytest.mark.parametrize("key,value", [("predict_x0", False), ("solver_p", {"_class_name": "DDIMScheduler"}),
                                       ("solver_order", 3), ("thresholding", True), ("use_karras_sigmas", True),
                                       ("use_exponential_sigmas", True), ("use_beta_sigmas", True),
                                       ("use_flow_sigmas", True), ("rescale_betas_zero_snr", True),
                                       ("trained_betas", [0.1, 0.2]), ("solver_type", "bh3")])
def test_loader_rejects_unsupported_unipc_keys(key, value):
    from diffuman4d_b200.loader import scheduler_config_from_json
    with pytest.raises(NotImplementedError, match=key):
        scheduler_config_from_json({"_class_name": "UniPCMultistepScheduler", "final_sigmas_type": "sigma_min",
                                    key: value})


@pytest.mark.parametrize("extra", [{"lower_order_final": False}, {"solver_type": "bh1"}])
def test_loader_rejects_a_zero_final_sigma_it_cannot_step(extra):
    from diffuman4d_b200.loader import scheduler_config_from_json
    with pytest.raises(NotImplementedError, match="final_sigmas_type"):
        scheduler_config_from_json({"_class_name": "UniPCMultistepScheduler", "final_sigmas_type": "zero", **extra})


# ---- frame-sharded refusal --------------------------------------------------------------------------------------------
def test_frame_sharded_pipeline_refuses_unipc_before_any_allocation(monkeypatch):
    import diffuman4d_b200.sharded as sharded_mod
    from diffuman4d_b200.config import UNetConfig
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline

    class _UNetStub:
        device = torch.device("cpu")
        config = UNetConfig.tiny()

    pipe = B200Diffuman4DPipeline(_UNetStub(), UniPCConfig())
    monkeypatch.setattr(sharded_mod, "lib", lambda: pytest.fail("the library was called"))
    monkeypatch.setattr(sharded_mod.dist, "is_initialized", lambda: pytest.fail("torch.distributed was consulted"))
    monkeypatch.setattr(torch.cuda, "device", lambda *a: pytest.fail("a device was selected"))
    with pytest.raises(NotImplementedError, match="UniPC"):
        sharded_mod.FrameShardedPipeline(pipe, max_frames=8, h=8, w=8)
