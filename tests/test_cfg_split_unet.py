"""Host logic of the UNet alone (seam B-2) on the CFG split and the CFG grid (``CFGSplitPipeline.unet_forward``,
``CFGGridPipeline.unet_forward`` and their ``.unet`` object) on the CPU.

* Every refusal of ``d4d_unet_forward_cfg_split`` / ``_cfg_grid`` is raised before any library call (the library binding
  is replaced by one that fails the test): other than one or two domains, a batch that is not ``len(domains)`` times
  ``num_frames``, a grid half that R does not divide, noise larger than the exchange buffer, one grid half's K/V layers
  larger than it, and worlds the mode does not run (refused when the pipeline is built).  Batches the library accepts
  reach it, with the entry point of the mode.
* Both entry points are in ``_lib.EXPORTS`` and declared in ``include/d4d.h``.
* The ``.unet`` object has the B-2 surface: ``.config``, ``.dtype``, ``.device``, ``.to()``, ``.eval()``, and
  ``__call__(sample, timestep=, skeletons=, domains=, num_frames=, return_dict=)`` returning ``(out,)`` or ``.sample``.
"""
import contextlib
import os
import types

import pytest
import torch

from diffuman4d_b200.config import UNetConfig

H = W = 8
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _unet(cfg):
    """A B200MultiviewUNet without a library handle, on the CPU (only its host-side checks run)."""
    from diffuman4d_b200.unet import B200MultiviewUNet
    u = B200MultiviewUNet.__new__(B200MultiviewUNet)
    u.config, u._device, u._dtype, u._h, u._finalized = cfg, torch.device("cpu"), torch.bfloat16, None, True
    return u


@pytest.fixture
def fake_dist(monkeypatch):
    """torch.distributed reporting an initialised world; ``open_exchange`` returns ``(0, world)`` instead of opening."""
    import torch.distributed as dist
    import diffuman4d_b200.cfg_split as cs
    state = types.SimpleNamespace(world=1)
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: state.world)
    monkeypatch.setattr(cs, "open_exchange", lambda pipe, nbytes, group=None: (0, state.world))
    return state


@pytest.fixture
def no_library(monkeypatch):
    import diffuman4d_b200.unet as unet_mod
    monkeypatch.setattr(unet_mod, "lib", lambda: pytest.fail("the library was called"))


@pytest.fixture
def calls(monkeypatch):
    """The library binding replaced by a recorder: each call's entry point, n_domains, B and F; it returns 0."""
    import diffuman4d_b200.unet as unet_mod
    seen = []

    class Lib:
        def __getattr__(self, name):
            def fn(h, sample, timestep, sk, dom, n_domains, B, F, h_, w_, out, stream):
                seen.append((name, n_domains, B, F))
                return 0
            return fn
    monkeypatch.setattr(unet_mod, "lib", lambda: Lib())
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: types.SimpleNamespace(cuda_stream=0))
    return seen


def _mode(fake_dist, grid: bool, world: int, rank: int = 0, max_frames: int = 4, pose: bool = False):
    from diffuman4d_b200.cfg_split import CFGGridPipeline, CFGSplitPipeline
    cfg = UNetConfig.tiny() if pose else UNetConfig.tiny(enable_pose_encoder=False, in_channels=15)
    fake_dist.world = world
    sp = (CFGGridPipeline if grid else CFGSplitPipeline)(types.SimpleNamespace(unet=_unet(cfg)), max_frames, H, W)
    sp.rank = rank
    return sp


def _batch(sp, n_img, h=H, w=W):
    cfg = sp.pipe.unet.config
    sample = torch.zeros(n_img, cfg.in_channels, h, w, dtype=torch.bfloat16)
    skel = torch.zeros(n_img, 3, 8 * h, 8 * w, dtype=torch.bfloat16) if cfg.enable_pose_encoder else None
    return sample, torch.zeros(n_img, dtype=torch.int64), skel


MODES = [("split", False, 2), ("grid", True, 4)]


# ------------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize("name,grid,world", MODES, ids=[m[0] for m in MODES])
def test_domain_count_refused_before_any_library_call(no_library, fake_dist, name, grid, world):
    sp = _mode(fake_dist, grid, world)
    x, t, s = _batch(sp, 6)
    with pytest.raises(ValueError, match=r"takes one domain \(no CFG halves\) or two .*, not 3$"):
        sp.unet_forward(x, t, s, ["spatial"] * 3, 2)


@pytest.mark.parametrize("name,grid,world", MODES, ids=[m[0] for m in MODES])
def test_batch_size_refused_with_the_reference_message(no_library, fake_dist, name, grid, world):
    sp = _mode(fake_dist, grid, world)
    x, t, s = _batch(sp, 6)
    with pytest.raises(ValueError) as e:
        sp.unet_forward(x, t, s, ["spatial", "spatial"], 4)
    assert str(e.value) == "num_frames: 4 * len(domains): 2 != len(emb): 6"


@pytest.mark.parametrize("world,rank", [(4, 1), (6, 3), (8, 6)])
def test_grid_refuses_a_half_that_R_does_not_divide(no_library, fake_dist, world, rank):
    sp = _mode(fake_dist, True, world, rank=rank, max_frames=8)
    R = world // 2
    F = R + 1
    x, t, s = _batch(sp, 2 * F)
    with pytest.raises(ValueError, match=rf"num_frames \({F}\) must be divisible by the number of ranks \({R}\)"):
        sp.unet_forward(x, t, s, ["spatial", "temporal"], F)


@pytest.mark.parametrize("name,grid,world", MODES + [("loopback", False, 1)], ids=[m[0] for m in MODES] + ["loopback"])
def test_noise_larger_than_the_exchange_buffer_is_refused(no_library, fake_dist, name, grid, world):
    from diffuman4d_b200.cfg_split import noise_exchange_bytes
    sp = _mode(fake_dist, grid, world, max_frames=2)
    sp.exchange_nbytes = noise_exchange_bytes(sp.pipe.unet.config, 2, H, W)
    x, t, s = _batch(sp, 8)
    with pytest.raises(ValueError, match=r"the batch's noise \(\d+ bytes\) does not fit the exchange buffer"):
        sp.unet_forward(x, t, s, ["spatial", "spatial"], 4)


def test_grid_refuses_kv_layers_larger_than_the_exchange_buffer(no_library, fake_dist):
    from diffuman4d_b200.cfg_split import noise_exchange_bytes
    sp = _mode(fake_dist, True, 4, max_frames=4)
    sp.exchange_nbytes = noise_exchange_bytes(sp.pipe.unet.config, 4, H, W)   # room for the noise only
    x, t, s = _batch(sp, 8)
    with pytest.raises(ValueError, match=r"one CFG half's K/V layers \(\d+ bytes\) do not fit the exchange buffer"):
        sp.unet_forward(x, t, s, ["spatial", "spatial"], 4)


@pytest.mark.parametrize("grid,world", [(False, 3), (False, 4), (False, 8), (True, 3), (True, 5), (True, 9)])
def test_worlds_the_mode_does_not_run_are_refused(no_library, fake_dist, grid, world):
    with pytest.raises(ValueError, match=f"not {world}$"):
        _mode(fake_dist, grid, world)


def test_invalid_domain_is_refused(no_library, fake_dist):
    sp = _mode(fake_dist, False, 2)
    x, t, s = _batch(sp, 8)
    with pytest.raises(ValueError, match="Invalid domain for temporal embedding: diagonal"):
        sp.unet_forward(x, t, s, ["spatial", "diagonal"], 4)


# ------------------------------------------------------------------------------------------------ accepted batches
@pytest.mark.parametrize("name,grid,world", MODES + [("loopback", False, 1), ("grid-8", True, 8)],
                         ids=[m[0] for m in MODES] + ["loopback", "grid-8"])
def test_accepted_batches_reach_the_mode_entry_point(calls, fake_dist, name, grid, world):
    sp = _mode(fake_dist, grid, world, max_frames=4, pose=True)
    entry = "d4d_unet_forward_cfg_grid" if grid else "d4d_unet_forward_cfg_split"
    for n_dom, F in ((2, 4), (1, 4), (1, 3)):   # one domain: no halves, so R need not divide F
        x, t, s = _batch(sp, n_dom * F)
        out = sp.unet_forward(x, t, s, ["temporal"] * n_dom, F)
        assert out.shape == (n_dom * F, sp.pipe.unet.config.out_channels, H, W)
        assert calls[-1] == (entry, n_dom, n_dom * F, F)


# ------------------------------------------------------------------------------------------------ exports
def test_entry_points_are_exported_and_declared():
    from diffuman4d_b200._lib import EXPORTS
    with open(os.path.join(ROOT, "include", "d4d.h")) as f:
        header = f.read()
    for name in ("d4d_unet_forward_cfg_split", "d4d_unet_forward_cfg_grid"):
        assert name in EXPORTS
        assert f"int {name}(" in header


# ------------------------------------------------------------------------------------------------ the .unet object
@pytest.mark.parametrize("grid", [False, True], ids=["split", "grid"])
def test_unet_object_has_the_b2_surface(no_library, fake_dist, grid):
    sp = _mode(fake_dist, grid, 2, pose=True)
    u = sp.unet
    assert u.config is sp.pipe.unet.config
    assert u.config.enable_pose_encoder and u.config.time_cond_proj_dim is None
    assert u.dtype == torch.bfloat16
    assert u.device == sp.pipe.unet.device
    assert u.to(torch.bfloat16) is u and u.to(u.device) is u and u.eval() is u
    with pytest.raises(ValueError, match="bfloat16 only"):
        u.to(torch.float32)
    seen = []

    def standin(sample, timestep, skeletons, domains, num_frames):
        seen.append((sample, timestep, skeletons, domains, num_frames))
        return torch.ones(2)
    sp.unet_forward = standin
    x, t, s = _batch(sp, 4)
    res = u(x, timestep=t, skeletons=s, domains=["spatial", "spatial"], num_frames=2, return_dict=False)
    assert isinstance(res, tuple) and len(res) == 1 and torch.equal(res[0], torch.ones(2))
    assert seen[-1][0] is x and seen[-1][1] is t and seen[-1][2] is s and seen[-1][3:] == (["spatial", "spatial"], 2)
    assert torch.equal(u(x, t, s, ["spatial", "spatial"], 2).sample, torch.ones(2))
