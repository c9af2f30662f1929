"""DPM-Solver++ singlestep (upstream DPMSolverSinglestepScheduler, dpmsolver++ / midpoint) on the CPU: the order list and
the lower_order_final switch of set_timesteps, mathematical anchors for the restated arithmetic in fp64, the oracle's
per-frame window step and sliding loop against the reference pipeline run with a stateful scheduler
(tests/golden/pipeline_dpm_single_ref.pt from tests/golden/gen_golden_dpm_single.py), the host tables, the config loader
and the frame-sharded refusal."""
import copy
import math
import os
import sys

import pytest
import torch

from diffuman4d_b200.config import DPMSingleConfig, DPMSolverConfig, SchedulerConfig
from oracle.dpm_single_oracle import DPMSingleOracle
from oracle.dpm_solver_oracle import (DPMSolverOracle, denoise_window_oracle_per_frame,
                                      sliding_iterative_denoise_oracle_per_frame)
from oracle.pipeline_oracle import DDIMOracle

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _golden():
    return torch.load(os.path.join(GOLD, "pipeline_dpm_single_ref.pt"))


def _fake_unet(cin):
    sys.path.insert(0, GOLD)
    from fake_unet import make_fake_unet
    return make_fake_unet(cin)


def _fp64_single(n, **kw):
    s = DPMSingleOracle(DPMSingleConfig(**kw), table_dtype=torch.float64)
    s.set_timesteps(n)
    return s


def _alpha_sigma(s, i):
    a, sig = DPMSingleOracle._alpha_sigma_t(s.sigmas[i])
    return float(a), float(sig)


# ---- order list and the lower_order_final switch ---------------------------------------------------------------------
def _expected_orders(order, lof, final, n):
    """Upstream's rule, written from its description: blocks 1, 2, .., order in turn; with lower_order_final the list ends
    on a whole block that is shorter than a full one; a zero final sigma makes the last entry 1."""
    if not lof and n % order:
        return None
    orders = [k % order + 1 for k in range(n)]
    if lof and n % order == 0 and order > 1:
        orders[-1] = 1          # the last full block splits into 1, .., order - 1 and 1
    if final == "zero":
        orders[-1] = 1
    return orders


@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("lof", [True, False])
@pytest.mark.parametrize("final", ["zero", "sigma_min"])
def test_order_list_follows_upstreams_rules(order, lof, final):
    from diffuman4d_b200.scheduler import dpm_single_order_list
    for n in range(1, 41):
        want = _expected_orders(order, lof, final, n)
        o = DPMSingleOracle(DPMSingleConfig(solver_order=order, lower_order_final=lof, final_sigmas_type=final))
        if want is None:
            with pytest.raises(ValueError):
                dpm_single_order_list(order, lof, final, n)
        else:
            assert dpm_single_order_list(order, lof, final, n) == want == o.get_order_list(n), n
            # every row of order k > 1 follows one of order k - 1: a block never starts above order 1
            assert all(k == 1 or want[i - 1] == k - 1 for i, k in enumerate(want)), n
        # what set_timesteps builds, with the switch applied
        o.set_timesteps(n)
        switched = lof or n % order != 0 or final == "zero"
        assert o.cfg.lower_order_final == switched
        assert o.order_list == _expected_orders(order, switched, final, n), n


def test_lower_order_final_switch_persists_on_the_tables():
    """set_timesteps switches lower_order_final on (upstream register_to_config) for a step count that is not a multiple
    of solver_order, and the switch stays for a later step count that is one; the caller's config is not touched."""
    from diffuman4d_b200.scheduler import DPMSingleTables
    cfg = DPMSingleConfig(solver_order=2, final_sigmas_type="sigma_min")
    t = DPMSingleTables(cfg, device="cpu")
    t.set_timesteps(4)
    assert not t.config.lower_order_final and t.order_list == [1, 2, 1, 2]
    t.set_timesteps(5)
    assert t.config.lower_order_final and t.order_list == [1, 2, 1, 2, 1]
    t.set_timesteps(4)
    assert t.config.lower_order_final and t.order_list == [1, 2, 1, 1]
    assert t.coefs[3, 12] == 1 and t.coefs[3, 4:].abs().sum() == 1   # only the order entry of an order-1 row
    assert not cfg.lower_order_final
    # a zero final sigma switches it on at any step count
    z = DPMSingleTables(DPMSingleConfig(solver_order=3), device="cpu")
    z.set_timesteps(6)
    assert z.config.lower_order_final and z.order_list == [1, 2, 3, 1, 2, 1]


# ---- anchors ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pred", ["epsilon", "v_prediction", "sample"])
@pytest.mark.parametrize("beta", [dict(), dict(beta_schedule="scaled_linear", beta_start=0.00085, beta_end=0.012)])
def test_first_order_is_ddim_and_multistep_order_1(pred, beta):
    """Order 1 is DDIM (eta 0) between the same timesteps: sigma_t / sigma_s x - alpha_t (e^-h - 1) x0 = alpha_t x0 +
    sigma_t eps.  Nine steps of linspace spacing are DDIM's leading spacing with steps_offset 111 (999 = 9 * 111), and
    the sigma_min final sigma is DDIM's alphas_cumprod[0].  It is also DPM-Solver++ multistep at order 1, for either
    final sigma."""
    n = 9
    single = _fp64_single(n, solver_order=1, prediction_type=pred, final_sigmas_type="sigma_min", **beta)
    ddim = DDIMOracle(SchedulerConfig(**{"beta_start": 1e-4, "beta_end": 0.02, "beta_schedule": "linear", **beta},
                                      prediction_type=pred, set_alpha_to_one=False, steps_offset=111,
                                      timestep_spacing="leading"))
    ddim.set_timesteps(n)
    ddim.alphas_cumprod = ddim.alphas_cumprod.double()
    ddim.final_alpha_cumprod = ddim.alphas_cumprod[0]
    assert torch.equal(single.timesteps, ddim.timesteps)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 3, 3, generator=g, dtype=torch.float64) * (1 + float(single.sigmas[0]))
    for i, t in enumerate(single.timesteps.tolist()):
        m = torch.randn(2, 4, 3, 3, generator=g, dtype=torch.float64)
        got, want = single.step(m, t, x), ddim.step(m, t, x)
        assert (got - want).abs().max().item() <= 1e-12 * (1 + want.abs().max().item()), (i, pred)
        x = got
    for final in ("zero", "sigma_min"):
        n = 10
        single = _fp64_single(n, solver_order=1, prediction_type=pred, final_sigmas_type=final, **beta)
        multi = DPMSolverOracle(DPMSolverConfig(solver_order=1, prediction_type=pred, final_sigmas_type=final, **beta),
                                table_dtype=torch.float64)
        multi.set_timesteps(n)
        assert torch.equal(single.timesteps, multi.timesteps) and torch.equal(single.sigmas, multi.sigmas)
        x = torch.randn(2, 4, 3, 3, generator=g, dtype=torch.float64) * (1 + float(single.sigmas[0]))
        for i, t in enumerate(single.timesteps.tolist()):
            m = torch.randn(2, 4, 3, 3, generator=g, dtype=torch.float64)
            got, want = single.step(m, t, x), multi.step(m, t, x)
            assert (got - want).abs().max().item() <= 1e-12 * (1 + want.abs().max().item()), (i, pred, final)
            x = got


@pytest.mark.parametrize("order,lof,final", [(2, True, "zero"), (2, False, "sigma_min"), (3, True, "zero"),
                                             (3, True, "sigma_min"), (3, False, "sigma_min")])
@pytest.mark.parametrize("pred", ["epsilon", "v_prediction"])
def test_exact_denoiser_of_a_point_mass_stays_on_the_trajectory(order, lof, final, pred):
    """Data = one point x0*: the exact model output gives x0* at every point of x_t = alpha_t x0* + sigma_t eps*, the
    differences of the second- and third-order updates vanish, and the first-order update from the block's start sample
    lands on the trajectory at any later sigma, so every step does."""
    n = 12
    s = _fp64_single(n, solver_order=order, lower_order_final=lof, final_sigmas_type=final, prediction_type=pred)
    assert max(s.order_list) == order
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


def _gaussian_error_at_t480(n, order):
    """Data ~ N(mu, s^2) per element: eps(x) = sigma (x - alpha mu) / (alpha^2 s^2 + sigma^2) exactly, and the
    probability-flow ODE keeps (x - alpha mu) / sqrt(alpha^2 s^2 + sigma^2) constant.  The error is taken after the
    first n / 2 steps (whole blocks at every order), at timestep 480.  961 training timesteps make every timestep of
    these step counts an integer without rounding (960 = 2^6 * 15), so the rows of a block are evenly spaced in t as the
    midpoint third-order update assumes; with 1000, the rounding moves its r0 by up to half a timestep and the third-order
    rate falls away as the steps get finer."""
    mu, sd = 0.3, 0.5
    s = _fp64_single(n, num_train_timesteps=961, solver_order=order, final_sigmas_type="sigma_min")
    assert not s.cfg.lower_order_final
    z = torch.linspace(-2.5, 2.5, 101, dtype=torch.float64)
    scale = lambda a, sig: math.sqrt(a * a * sd * sd + sig * sig)
    a, sig = _alpha_sigma(s, 0)
    x = a * mu + scale(a, sig) * z
    for i, t in enumerate(s.timesteps.tolist()[:n // 2]):
        a, sig = _alpha_sigma(s, i)
        x = s.step(sig * (x - a * mu) / scale(a, sig) ** 2, t, x)
    assert int(s.timesteps[n // 2]) == 480
    a, sig = _alpha_sigma(s, n // 2)
    return (x - (a * mu + scale(a, sig) * z)).abs().max().item()


# Error ratio per doubling of the steps (24 -> 48 -> 96): order p should give 2^p.  The fp64 run measured 1.99 / 2.00 at
# order 1, 3.91 / 3.96 at order 2 and 7.91 / 7.99 at order 3.  The bands do not overlap between orders.
@pytest.mark.parametrize("order,lo,hi", [(1, 1.85, 2.15), (2, 3.6, 4.3), (3, 7.2, 8.8)])
def test_convergence_order_on_gaussian_data(order, lo, hi):
    errs = [_gaussian_error_at_t480(n, order) for n in (24, 48, 96)]
    ratios = [errs[k] / errs[k + 1] for k in range(len(errs) - 1)]
    print(f"\norder {order}: errors at t = 480 {errs}, ratios {ratios}")
    for r in ratios:
        assert lo <= r <= hi, (order, errs, ratios)


# ---- the reference pipeline's per-frame scheduler copies (golden) ------------------------------------------------
def _config(c):
    return DPMSingleConfig(**c["config"])


@pytest.mark.parametrize("tag", ["call_cfg_eps_order3", "call_nocfg_v_order2_sigma_min"])
def test_window_call_matches_reference_pipeline_golden(tag):
    """``__call__`` with fresh per-frame copies handed over at nonzero timestep indices: each frame's step index starts at
    its timestep, and a frame whose first step falls on a second- or third-order row runs it at a lower order."""
    c = _golden()["cases"][tag]
    i = c["in"]
    s = DPMSingleOracle(_config(c))
    s.set_timesteps(c["n_steps_table"])
    assert torch.equal(s.timesteps, c["timesteps_table"])
    assert s.order_list == c["order_list"] and s.cfg.lower_order_final == c["lower_order_final"]
    scheds = [copy.deepcopy(s) for _ in range(len(i["latents"]))]
    lat, ti = denoise_window_oracle_per_frame(
        _fake_unet(11), scheds, latents=i["latents"].clone(), pixel_latents=i["pixel_latents"], plucker=i["plucker"],
        skeletons=i["skeletons"].float(), cond_mask=i["cond_mask"], timestep_indices=i["timestep_indices"], domain="spatial",
        guidance_scale=c["guidance"], num_inference_steps=c["num_inference_steps"], enable_pose_encoder=True)
    torch.testing.assert_close(lat, c["out_latents"], rtol=1e-5, atol=1e-6)
    assert torch.equal(ti, c["out_timestep_indices"])


SLIDE_TAGS = ["slide_spatial_eps_cfg_order3", "slide_temporal_bidir_v_nocfg", "slide_spatial_order1_sample",
              "slide_spatial_order3_nolof_sigma_min", "slide_order2_switch_persists"]


def _slide(c, sched, task):
    i = task["in"]
    return sliding_iterative_denoise_oracle_per_frame(
        _fake_unet(11), sched, pixel_latents=i["pixel_latents"], plucker=i["plucker"], skeletons=i["skeletons"].float(),
        cond_mask=i["cond_mask_latents"], latents=i["latents"], domain=c["domain"],
        timestep_indices=i["timestep_indices"], window_size=task["window_size"], sliding_stride=c["sliding_stride"],
        bidirectional=c["bidirectional"], num_denoising_steps=1, alternation_rounds=c["alternation_rounds"],
        guidance_scale=c["guidance"], enable_pose_encoder=True)


@pytest.mark.parametrize("tag", SLIDE_TAGS)
def test_sliding_loop_matches_reference_pipeline_golden(tag):
    """Successive tasks on one scheduler object: per-frame histories across windows, reset per task, and the
    lower_order_final switch carried from one task to the next."""
    c = _golden()["cases"][tag]
    sched = DPMSingleOracle(_config(c))
    for task in c["tasks"]:
        out = _slide(c, sched, task)
        assert sched.order_list == task["order_list"] and sched.cfg.lower_order_final == task["lower_order_final"]
        torch.testing.assert_close(out["latents"], task["out_latents"], rtol=1e-5, atol=1e-5)
        assert torch.equal(out["timestep_indices"], task["out_timestep_indices"])
        assert torch.equal(out["fully_denoised"], task["fully_denoised"])


@pytest.mark.parametrize("tag,task,flip", [("slide_spatial_order3_nolof_sigma_min", 0, {"lower_order_final": True}),
                                           ("slide_spatial_order3_nolof_sigma_min", 0, {"solver_order": 2}),
                                           ("slide_spatial_eps_cfg_order3", 0, {"solver_order": 2}),
                                           ("slide_order2_switch_persists", 1, {})])
def test_golden_cases_pin_the_order_knobs(tag, task, flip):
    """Flipping the knob, or running the task on a fresh scheduler that never saw the switch, gives a different result,
    so the fixture does pin it."""
    c = _golden()["cases"][tag]
    t = c["tasks"][task]
    out = _slide(c, DPMSingleOracle(DPMSingleConfig(**{**c["config"], **flip})), t)
    assert (out["latents"] - t["out_latents"]).abs().max() > 1e-3


# ---- tables -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(), dict(solver_order=1), dict(solver_order=3),
                                dict(solver_order=3, final_sigmas_type="sigma_min"),
                                dict(final_sigmas_type="sigma_min", prediction_type="v_prediction"),
                                dict(solver_order=3, beta_schedule="scaled_linear", beta_start=0.00085, beta_end=0.012)])
@pytest.mark.parametrize("n", [1, 2, 3, 10, 12, 20])
def test_tables_equal_a_hand_evaluation_in_upstreams_order(kw, n):
    """Every coefficient equals the oracle's restatement of upstream's update functions evaluated at that row, bit for
    bit; entries of orders above the row's are 0; the order column is upstream's order list."""
    from diffuman4d_b200.scheduler import DPMSingleTables
    t = DPMSingleTables(DPMSingleConfig(**kw), device="cpu")
    o = DPMSingleOracle(DPMSingleConfig(**kw))
    assert torch.equal(t.set_timesteps(n), o.set_timesteps(n))
    assert t.config == o.cfg and t.order_list == o.order_list
    assert t.sigmas.dtype == torch.float32 and torch.equal(t.sigmas, o.sigmas)
    assert t.coefs.dtype == torch.float32 and t.coefs.shape == (n, 13)
    for i, order in enumerate(o.order_list):
        a_s, s_s = DPMSingleOracle._alpha_sigma_t(o.sigmas[i])
        want = [a_s.item(), s_s.item(), *(v.item() for v in o.first_order_coefs(i))]
        want += [v.item() for v in o.second_order_coefs(i)] if order >= 2 else [0.0] * 4
        want += [v.item() for v in o.third_order_coefs(i)] if order == 3 else [0.0] * 4
        assert t.coefs[i].tolist() == want + [float(order)], i
    assert torch.isfinite(t.coefs).all()


def test_tables_refuse_what_the_step_does_not_implement():
    from diffuman4d_b200.scheduler import DPMSingleTables
    with pytest.raises(NotImplementedError, match="orders 1, 2 and 3"):
        DPMSingleTables(DPMSingleConfig(solver_order=4), device="cpu")
    with pytest.raises(ValueError, match="duplicate"):
        DPMSingleTables(DPMSingleConfig(num_train_timesteps=10), device="cpu").set_timesteps(10)
    with pytest.raises(ValueError, match="linspace"):
        DPMSingleTables(DPMSingleConfig(timestep_spacing="trailing"), device="cpu")
    with pytest.raises(ValueError):
        DPMSingleTables(DPMSingleConfig(beta_schedule="squaredcos_cap_v2"), device="cpu")
    with pytest.raises(ValueError):
        DPMSingleTables(DPMSingleConfig(final_sigmas_type="denoise_to_zero"), device="cpu")


# ---- loader -------------------------------------------------------------------------------------------------------
# a DPMSolverSinglestepScheduler config as diffusers 0.33.1 saves it, every key present
SINGLE_SCHEDULER_CONFIG = {
    "_class_name": "DPMSolverSinglestepScheduler", "_diffusers_version": "0.33.1", "num_train_timesteps": 1000,
    "beta_start": 0.00085, "beta_end": 0.012, "beta_schedule": "scaled_linear", "trained_betas": None,
    "solver_order": 3, "prediction_type": "v_prediction", "thresholding": False, "dynamic_thresholding_ratio": 0.995,
    "sample_max_value": 1.0, "algorithm_type": "dpmsolver++", "solver_type": "midpoint", "lower_order_final": True,
    "use_karras_sigmas": False, "use_exponential_sigmas": False, "use_beta_sigmas": False, "use_flow_sigmas": False,
    "flow_shift": 1.0, "final_sigmas_type": "sigma_min", "lambda_min_clipped": -math.inf, "variance_type": None,
    "use_dynamic_shifting": False, "time_shift_type": "exponential",
}


def test_loader_maps_a_full_dpm_single_config():
    from diffuman4d_b200.loader import scheduler_config_from_json
    assert scheduler_config_from_json(SINGLE_SCHEDULER_CONFIG) == DPMSingleConfig(
        beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", solver_order=3, prediction_type="v_prediction",
        lower_order_final=True, final_sigmas_type="sigma_min")
    assert scheduler_config_from_json({"_class_name": "DPMSolverSinglestepScheduler"}) == DPMSingleConfig()
    assert scheduler_config_from_json({**SINGLE_SCHEDULER_CONFIG, "timestep_spacing": "linspace"}).solver_order == 3


@pytest.mark.parametrize("key,value", [("algorithm_type", "dpmsolver"), ("algorithm_type", "sde-dpmsolver++"),
                                       ("solver_type", "heun"), ("solver_order", 4), ("thresholding", True),
                                       ("use_karras_sigmas", True), ("use_exponential_sigmas", True),
                                       ("use_beta_sigmas", True), ("use_flow_sigmas", True),
                                       ("use_dynamic_shifting", True), ("lambda_min_clipped", -5.1),
                                       ("variance_type", "learned_range"), ("trained_betas", [0.1, 0.2]),
                                       ("beta_schedule", "squaredcos_cap_v2"), ("prediction_type", "flow_prediction"),
                                       ("final_sigmas_type", "denoise_to_zero"), ("timestep_spacing", "trailing")])
def test_loader_rejects_unsupported_dpm_single_keys(key, value):
    from diffuman4d_b200.loader import scheduler_config_from_json
    with pytest.raises(NotImplementedError, match=key):
        scheduler_config_from_json({**SINGLE_SCHEDULER_CONFIG, key: value})


def test_loader_names_the_fused_classes_when_refusing_one():
    from diffuman4d_b200.loader import scheduler_config_from_json
    with pytest.raises(NotImplementedError, match="DPMSolverSinglestepScheduler only"):
        scheduler_config_from_json({"_class_name": "EulerDiscreteScheduler"})


# ---- frame-sharded refusal --------------------------------------------------------------------------------------------
def test_frame_sharded_pipeline_refuses_dpm_single_before_any_allocation(monkeypatch):
    import diffuman4d_b200.sharded as sharded_mod
    from diffuman4d_b200.config import UNetConfig
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline

    class _UNetStub:
        device = torch.device("cpu")
        config = UNetConfig.tiny()

    pipe = B200Diffuman4DPipeline(_UNetStub(), DPMSingleConfig(solver_order=3))
    monkeypatch.setattr(sharded_mod, "lib", lambda: pytest.fail("the library was called"))
    monkeypatch.setattr(sharded_mod.dist, "is_initialized", lambda: pytest.fail("torch.distributed was consulted"))
    monkeypatch.setattr(torch.cuda, "device", lambda *a: pytest.fail("a device was selected"))
    with pytest.raises(NotImplementedError, match="singlestep"):
        sharded_mod.FrameShardedPipeline(pipe, max_frames=8, h=8, w=8)
