"""CPU tests of the host-side logic and of the C-ABI boundary (no GPU compute): the shared library loads, exports
exactly the symbols include/d4d.h declares, and fails loudly without a device."""
import ctypes as C
import os
import re

import pytest
import torch

from diffuman4d_b200.config import SchedulerConfig, UNetConfig
from diffuman4d_b200.weights import random_state_dict, state_dict_spec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def libd4d():
    from diffuman4d_b200 import build
    build.build(verbose=False)          # nvcc cross-compiles sm_90a without a GPU
    from diffuman4d_b200._lib import lib
    return lib()


def test_header_and_library_export_the_same_symbols(libd4d):
    from diffuman4d_b200._lib import EXPORTS
    hdr = open(os.path.join(ROOT, "include", "d4d.h")).read()
    declared = set(re.findall(r"\b(d4d_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(EXPORTS), declared ^ set(EXPORTS)
    for name in EXPORTS:
        assert hasattr(libd4d, name), f"libd4d.so does not export {name}"
    assert libd4d.d4d_version() >= 100


def test_product_library_carries_no_test_kernels_or_ablation_switches(libd4d):
    """Library hygiene: no measurement / probe kernels and no D4D_*_ABLATE environment switches in the library."""
    import subprocess
    from diffuman4d_b200._lib import LIB_PATH
    prod = subprocess.run(["strings", LIB_PATH], capture_output=True, text=True).stdout
    for sw in ("D4D_GEMM_ABLATE", "D4D_ATTN_ABLATE"):
        assert sw not in prod
    assert "microbench" not in prod and "probe_kernel" not in prod


def test_library_has_no_libcuda_or_torch_dependency(libd4d):
    import subprocess
    from diffuman4d_b200._lib import LIB_PATH
    out = subprocess.run(["ldd", LIB_PATH], capture_output=True, text=True).stdout
    assert "libcuda.so" not in out and "libtorch" not in out and "libc10" not in out, out


@pytest.mark.skipif(torch.cuda.is_available(), reason="only meaningful on a box without a GPU")
def test_create_fails_loudly_without_gpu(libd4d):
    from diffuman4d_b200._lib import D4DError
    from diffuman4d_b200.unet import B200MultiviewUNet
    with pytest.raises((D4DError, ValueError)):
        B200MultiviewUNet(UNetConfig.tiny(), device=0)
    with pytest.raises(ValueError):
        B200MultiviewUNet(UNetConfig.tiny(), device="cpu")


def test_create_rejects_bad_config(libd4d):
    from diffuman4d_b200._lib import D4DConfig
    c = D4DConfig()
    h = C.c_void_p()
    assert libd4d.d4d_create(C.byref(c), 0, C.byref(h)) == 1
    assert b"layers_per_block" in libd4d.d4d_last_error()
    assert libd4d.d4d_create(None, 0, C.byref(h)) == 1


def test_config_validation():
    with pytest.raises(ValueError):
        UNetConfig(block_out_channels=(320, 640, 1280))
    with pytest.raises(ValueError):
        UNetConfig(attention_head_dim=(7, 10, 20, 20))
    with pytest.raises(ValueError):
        UNetConfig(cross_attention_dim=1280)      # would crash at the 320/640 levels in the reference (SURVEY 0.5)
    c = UNetConfig.ctor_default()
    assert [c.head_dim(i) for i in range(4)] == [40, 80, 160, 160] and not c.has_attn2(0)
    c = UNetConfig.sd21(cross_attention_dim=(320, 640, 1280, 1280))
    assert c.has_attn2(2) and c.head_dim(0) == 64 and c.time_embed_dim == 1280


@pytest.mark.parametrize("cfg", [UNetConfig.tiny(), UNetConfig.tiny(cross_attention_dim=(64, 128, 256, 256),
                                                                     use_linear_projection=False,
                                                                     enable_pose_encoder=False, enable_tem_embeds=False,
                                                                     in_channels=15)])
def test_weight_key_contract_matches_oracle(cfg):
    from oracle.unet_oracle import build_oracle
    sd = build_oracle(cfg).state_dict()
    spec = state_dict_spec(cfg)
    assert set(sd) == set(spec)
    for k, v in sd.items():
        assert tuple(v.shape) == spec[k], k
    rs = random_state_dict(cfg, seed=3, dtype=torch.float32)
    assert set(rs) == set(spec) and rs["pose_encoder.scale"].item() == 2.0 if cfg.enable_pose_encoder else True


def test_full_size_spec_counts():
    spec = state_dict_spec(UNetConfig.sd21())
    n = sum(torch.Size(s).numel() for s in spec.values())
    assert 8.0e8 < n < 8.4e8 and len(spec) == 597
    assert spec["up_blocks.1.resnets.2.conv1.weight"] == (1280, 1920, 3, 3)      # concat-skip input channels
    assert spec["down_blocks.1.attentions.0.transformer_blocks.0.ff.net.0.proj.weight"] == (5120, 640)


def test_scheduler_tables_match_oracle():
    from diffuman4d_b200.scheduler import DDIMTables
    from oracle.pipeline_oracle import DDIMOracle
    for sc in (SchedulerConfig(), SchedulerConfig(prediction_type="v_prediction", set_alpha_to_one=True, steps_offset=0),
               SchedulerConfig(timestep_spacing="trailing"), SchedulerConfig(beta_schedule="linear", beta_start=1e-4, beta_end=0.02)):
        a, b = DDIMTables(sc, device="cpu"), DDIMOracle(sc)
        assert torch.equal(a.alphas_cumprod, b.alphas_cumprod)
        for n in (12, 18, 36, 60):
            assert torch.equal(a.set_timesteps(n), b.set_timesteps(n))
        assert abs(a.final_alpha_cumprod - float(b.final_alpha_cumprod)) == 0
    with pytest.raises(ValueError):
        DDIMTables(SchedulerConfig(), device="cpu").set_timesteps(5000)


def test_window_builder_matches_oracle():
    from diffuman4d_b200.pipeline import build_windows
    from oracle.pipeline_oracle import build_windows as ref
    mask = torch.ones(48)
    mask[[1, 13, 25, 37]] = 0
    tgt, inp = torch.where(mask != 0)[0], torch.where(mask == 0)[0]
    for kw in (dict(window_size=12, sliding_stride=2), dict(window_size=12, sliding_stride=1, bidirectional=True),
               dict(window_size=4, sliding_stride=1, sliding_shift=3)):
        a, b = build_windows(tgt, inp, "spatial", **kw), ref(tgt, inp, "spatial", **kw)
        assert len(a[0]) == len(b[0]) and all(torch.equal(x, y) for x, y in zip(a[0], b[0]))
    with pytest.raises(ValueError):
        build_windows(tgt, inp, "diagonal", 12, 2)


def test_loader_vae_factory_resolution(tmp_path):
    """B-1: the Hydra yaml can only carry strings, so ``vae_factory`` accepts a dotted path; the default builds the stock
    AutoencoderKL adapter only when ``model_dir/vae`` exists."""
    from diffuman4d_b200 import loader
    assert loader._resolve_factory(None) is loader.default_vae_factory
    assert loader.default_vae_factory(str(tmp_path), 0) is None                    # no vae/ directory -> latents only
    f = loader._resolve_factory("diffuman4d_b200.loader.default_vae_factory")
    assert f is loader.default_vae_factory
    with pytest.raises(ValueError):
        loader._resolve_factory("nodots")
    with pytest.raises(ValueError):
        loader._resolve_factory(3)

    class FakeVAE:                                   # the reference's encode_vae / decode_vae arithmetic (PIPE:47-72,280-285)
        class config:
            scaling_factor = 0.5

        def encode(self, x):
            from types import SimpleNamespace
            return SimpleNamespace(latent_dist=SimpleNamespace(sample=lambda: x[:, :, ::8, ::8] * 2))

        def decode(self, z, return_dict=False):
            return (z.repeat_interleave(8, 2).repeat_interleave(8, 3),)

    a = loader.StockVAEAdapter(FakeVAE(), batch_size=2)
    img = torch.rand(5, 3, 16, 16) * 2 - 1
    z = a.encode_latents(img)
    assert torch.equal(z, img[:, :, ::8, ::8] * 2 * 0.5)
    out = a.decode_latents(z)
    assert out.shape == img.shape and float(out.min()) >= 0 and float(out.max()) <= 1
    torch.testing.assert_close(out[:, :, ::8, ::8], (img[:, :, ::8, ::8] * 2 / 2 + 0.5).clamp(0, 1))


def test_loader_config_mapping():
    from diffuman4d_b200.loader import scheduler_config_from_json, unet_config_from_json
    c = unet_config_from_json(dict(in_channels=11, attention_head_dim=[5, 10, 20, 20], cross_attention_dim=None,
                                   use_linear_projection=True, enable_pose_encoder=True, enable_tem_embeds=True))
    assert c == UNetConfig.sd21()
    with pytest.raises(NotImplementedError):
        unet_config_from_json(dict(class_embed_type="timestep", cross_attention_dim=None))
    with pytest.raises(NotImplementedError):
        scheduler_config_from_json({"_class_name": "EulerDiscreteScheduler"})
    s = scheduler_config_from_json({"_class_name": "DDIMScheduler", "beta_schedule": "scaled_linear", "beta_start": 0.00085,
                                    "beta_end": 0.012, "clip_sample": False, "set_alpha_to_one": False, "steps_offset": 1,
                                    "prediction_type": "v_prediction"})
    assert s.prediction_type == "v_prediction" and s.steps_offset == 1


def test_plucker_embeds_match_reference_ray_utils():
    """diffuman4d_b200.rays against ``calc_plucker_embeds`` / ``calc_relative_poses`` run from the reference
    (src/data/utils/ray_utils.py:101-118; fixture tests/golden/plucker.pt)."""
    import os
    from diffuman4d_b200.rays import plucker_embeds, relative_poses
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "plucker.pt"))
    torch.testing.assert_close(plucker_embeds(16, 16, g["K"], g["c2w"]), g["plucker"], rtol=1e-5, atol=2e-6)
    rel = relative_poses(g["c2w"])
    torch.testing.assert_close(rel, g["rel_poses"], rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(plucker_embeds(16, 16, g["K"], rel), g["plucker_rel"], rtol=1e-5, atol=5e-6)


def test_upsample_phase_weights_reproduce_nearest2x_conv3x3():
    """The sub-pixel form the Upsample2D kernel executes (conv_kind 2 / 3, csrc/gemm_wgmma.cu) is an identity, not an
    approximation: with integer-valued inputs and weights (exact in bf16 and in the fp32 sums) the four 2x2 phase convs
    on the low-resolution tensor equal `F.interpolate(nearest, x2)` + 3x3 / pad 1 conv bit for bit (reference:
    diffusers Upsample2D as called at unet_multiview_blocks.py:620)."""
    import torch.nn.functional as F
    from diffuman4d_b200.ops import upsample_phase_weights
    g = torch.Generator().manual_seed(0)
    n, cin, cout, H, W = 2, 5, 3, 6, 7
    x = torch.randint(-4, 5, (n, cin, H, W), generator=g).float()
    w = torch.randint(-3, 4, (cout, cin, 3, 3), generator=g).float()
    ref = F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), w, padding=1)
    phases = upsample_phase_weights(w)                       # [a*2+b] -> [Cout, 4 (ty*2+tx), Cin] bf16
    out = torch.zeros_like(ref)
    xp = F.pad(x, (1, 1, 1, 1))
    for a in range(2):
        for b in range(2):
            wp = phases[a * 2 + b].float().view(cout, 2, 2, cin).permute(0, 3, 1, 2)     # OIHW 2x2
            # rows {-1, 0} for a = 0, {0, +1} for a = 1 (columns alike): a window of the padded input
            y = F.conv2d(xp[:, :, a:a + H + 1, b:b + W + 1], wp)
            out[:, :, a::2, b::2] = y
    assert torch.equal(out, ref)
