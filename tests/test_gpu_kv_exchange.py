"""The frame-sharded 3-D attention layer (DESIGN.md section 7) on one GPU.

* The QKV GEMM whose epilogue scatters its K|V columns into every rank's gathered buffer (d4d_op_gemm_kv_scatter, the
  E_KV / E_ALL register-store kernels), run for each rank r of R in one process: against A.W^T in fp64, bit for bit
  against the plain GEMM on the same rows, all R destinations identical, every row outside the rank's slice (both CFG
  halves, or one) untouched, the Q columns of `out` as the plain GEMM's and its K|V columns unwritten.
* Width independence: the K|V bits must not depend on the tile width, because a rank's GEMM (M = halves * F/R frames)
  and the single-GPU GEMM of the whole window may pick different widths, and the sharded window promises results
  bit-identical to the single-GPU window.
* Attention over the gathered buffer, rank by rank, equals the fused-QKV attention of the full window bit for bit and
  fp64 softmax attention within the attention tolerance.
* The sharded UNet plan through a one-rank loopback (d4d_exchange_open with rank 0 of world 1 on the handle's own
  buffers): scatter GEMM into the exchange buffer, flag signal / wait, both buffer parities and the epoch counter, and
  attention with ld_kv = 2 C' -- bit-identical to the plain plan, for forwards and DDIM window steps.
* The exchange buffer size (sharded.exchange_bytes) and the argument checks of the scatter, on the CPU.

What needs two GPUs (cudaIpc mappings, NVLink stores, cross-rank flag order) stays in test_gpu_sharded.py.
"""
import ctypes as C
import dataclasses

import pytest
import torch

from diffuman4d_b200.config import SchedulerConfig, UNetConfig
from diffuman4d_b200.plan import launches, pad_head_dim
from diffuman4d_b200.sharded import exchange_bytes

SENT16 = 0x7FA5       # bf16 NaN bit pattern that no kernel produces
WIDTHS = (64, 128, 160, 192, 256)


# ------------------------------------------------------------------------------------------------ exchange buffer size (CPU)
@pytest.mark.parametrize("n3d", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("name", ["tiny", "sd21", "ctor_default"])
def test_exchange_bytes_is_the_largest_3d_layer(name, n3d):
    """exchange_bytes equals the largest batch * rows_global * 2 C' * 2 bytes that sharded_qkv_attention (csrc/unet.cu)
    requires of the buffer, over the 3-D attention launches of the plan: too small fails every sharded forward, and
    num_3d_attn_blocks = 4 puts a 3-D layer on level 0 (full-resolution tokens)."""
    cfg = dataclasses.replace(getattr(UNetConfig, name)(), num_3d_attn_blocks=n3d)
    for F_total in (2, 4, 16, 24):
        for lat in (16, 24, 64, 128):
            # batch (CFG halves) * rows_global (every frame's tokens of one half) * K|V columns * bf16
            need = max(a.spec["batch"] * a.spec["seq_kv"] * 2 * a.spec["heads"] * a.spec["dpad"] * 2
                       for a in launches(cfg, F_total, lat, lat) if a.category == "attn3d")
            assert exchange_bytes(cfg, F_total, lat, lat) == need, (F_total, lat)


# ------------------------------------------------------------------------------------------------ argument checks
@pytest.fixture(scope="module")
def libd4d():
    from diffuman4d_b200 import build
    build.build(verbose=False)
    from diffuman4d_b200._lib import lib
    return lib()


# M = 64 rows, K = 64, N = 384 (Q | K | V of 128 columns), kv_ld = 256, two halves of 32 local rows at offset 32 of 96
_BASE = dict(M=64, N=384, kv_col0=128, kv_ld=256, rows_local=32, rows_global=96, row_offset=32, world=2)
REJECT = [
    ("kv_col0-not-16", dict(kv_col0=136, kv_ld=248), "K/V scatter arguments"),
    ("kv_ld-not-8", dict(kv_ld=260), "K/V scatter arguments"),
    ("world-0", dict(world=0), "world"),
    ("world-9", dict(world=9), "world"),
    ("M-not-multiple-of-rows_local", dict(rows_local=24, rows_global=48, row_offset=24), "multiple of rows_local"),
    ("rows_local-0", dict(rows_local=0), "multiple of rows_local"),
    ("slice-past-rows_global", dict(row_offset=72), "exceeds rows_global"),
    ("negative-row_offset", dict(row_offset=-1), "exceeds rows_global"),
    ("null-destination", dict(null_dst=1), "null destination"),
]


@pytest.mark.parametrize("case,over,match", REJECT, ids=[c[0] for c in REJECT])
def test_scatter_rejections(libd4d, case, over, match):
    """Arguments under which the scatter would store outside the gathered buffers are argument errors (status 1,
    ValueError) raised before any CUDA call.  Without a GPU the operands are dummy addresses, and anything that is not
    rejected fails with a CUDA error instead; on a GPU they are real buffers large enough for any of these launches,
    except that the null destination is only tried without one.  (GEGLU and GroupNorm statistics, which gemm_prepare
    also refuses with a scatter, cannot be expressed through this entry point.)"""
    from diffuman4d_b200._lib import check
    a = dict(_BASE, **over)
    null_dst = a.pop("null_dst", 0)
    on_gpu = torch.cuda.is_available()
    if on_gpu and null_dst:
        pytest.skip("a null destination is only passed where no kernel can run")
    if on_gpu:
        keep = [torch.zeros(a["M"], 64, dtype=torch.bfloat16, device="cuda"),
                torch.zeros(a["N"], 64, dtype=torch.bfloat16, device="cuda"),
                torch.zeros(a["M"], a["N"], dtype=torch.bfloat16, device="cuda")]
        dst = [torch.zeros(8 * 96 * 4, 512, dtype=torch.bfloat16, device="cuda") for _ in range(9)]
        A, W, out = (t.data_ptr() for t in keep)
        ptrs = [t.data_ptr() for t in dst]
        stream = torch.cuda.current_stream().cuda_stream
    else:
        A, W, out, stream = 0x100000, 0x200000, 0x300000, None
        ptrs = [0x1000000 * (r + 1) for r in range(9)]
    if null_dst:
        ptrs[1] = None
    arr = (C.c_void_p * 9)(*ptrs)
    with pytest.raises(ValueError, match=match):
        check(libd4d.d4d_op_gemm_kv_scatter(A, 64, 64, W, a["M"], a["N"], out, a["N"], a["kv_col0"], a["kv_ld"],
                                            a["rows_local"], a["rows_global"], a["row_offset"], a["world"], arr, 0, stream),
              "d4d_op_gemm_kv_scatter")
    if on_gpu:
        torch.cuda.synchronize()
        assert all(int(t.count_nonzero()) == 0 for t in keep[2:] + dst), "a rejected scatter wrote"


# ------------------------------------------------------------------------------------------------ the scatter GEMM
# (id, C = K, heads, head_dim, tokens per frame, F_total, rank counts R).  N = 3 C', C' = heads * padded head_dim.
SHAPES = [
    ("sd21-L1-64px-W16", 640, 10, 64, 32 * 32, 16, (2, 4, 8)),        # N 1920
    ("sd21-L2-64px-W16", 1280, 20, 64, 16 * 16, 16, (2, 4, 8)),       # N 3840
    ("sd21-L3-64px-W16", 1280, 20, 64, 8 * 8, 16, (2, 4, 8)),         # N 3840
    ("sd21-L3-64px-W24", 1280, 20, 64, 8 * 8, 24, (2, 3, 4, 8)),      # N 3840
    ("ctor-L0-32px-W8", 320, 8, 40, 32 * 32, 8, (2, 4, 8)),           # N 1536 (head_dim 40 -> 64)
    ("ctor-L1-64px-W16", 640, 8, 80, 32 * 32, 16, (2, 4, 8)),         # N 3072 (80 -> 128)
    ("ctor-L2-64px-W16", 1280, 8, 160, 16 * 16, 16, (2, 4, 8)),       # N 4608 (160 -> 192)
    ("tiny-L1-16px-W4", 128, 2, 64, 8 * 8, 4, (2, 4)),                # N 384
    ("tiny-L0-16px-W4", 64, 1, 64, 16 * 16, 4, (2, 4)),               # N 192: num_3d_attn_blocks = 4
    # 24x24 latents: 9 tokens per frame at level 3.  M is not a multiple of 128, a row tile holds both CFG halves, and
    # the tiles of width 160 / 192 straddle the Q|K column boundary (kv_col0 = 256)
    ("tiny-L3-24px-W6", 256, 4, 64, 3 * 3, 6, (2, 3)),                # N 768
]


def _scatter_params():
    out = []
    for s in SHAPES:
        N = 3 * s[2] * pad_head_dim(s[3])
        for bn in (0,) + tuple(b for b in WIDTHS if N % b == 0):
            out.append(pytest.param(s, bn, id=f"{s[0]}-bn{bn}"))
    return out


_CACHE = {}


def _layer(shape):
    """Inputs and full-window references of a layer, kept for the widths of the same shape."""
    if _CACHE.get("key") != shape[0]:
        _CACHE.clear()
        from diffuman4d_b200 import ops
        _, K, heads, d, hw, F_total, _ = shape
        dp = pad_head_dim(d)
        Cp = heads * dp
        g = torch.Generator().manual_seed(7)
        a = torch.randn(2 * F_total * hw, K, generator=g).to(torch.bfloat16).cuda()
        w = (torch.randn(3, heads, dp, K, generator=g) * K ** -0.5)
        w[:, :, d:] = 0                                     # the loader's zero rows of a padded head
        w = w.reshape(3 * Cp, K).to(torch.bfloat16).cuda()
        full = {bn: ops.gemm(a, w, block_n=bn) for bn in (0,) + tuple(b for b in WIDTHS if (3 * Cp) % b == 0)}
        _CACHE.update(key=shape[0], a=a, w=w, full=full, ref64=a.double() @ w.double().t())
    return _CACHE


def _close(out, ref, rtol=8e-3, afrac=2e-3, what=""):
    """DESIGN.md section 2: |out - ref| <= rtol |ref| + afrac max|ref| (GEMM 8e-3 / 2e-3, attention 1e-2 / 5e-3)."""
    out, ref = out.double(), ref.double()
    assert torch.isfinite(out).all(), f"{what}: non-finite values"
    err = (out - ref).abs()
    bad = err > rtol * ref.abs() + afrac * ref.abs().max()
    assert not bad.any(), f"{what}: {int(bad.sum())} / {bad.numel()} out of tolerance (max err {err.max().item():.3g})"


def _bits(t):
    return t.view(torch.int16)


def _rank_rows(halves, F_total, R, r, hw):
    """Rows of the full window ([half][frame][token], half-major) that rank r owns, in its local order."""
    F_loc = F_total // R
    per_half = torch.arange(r * F_loc * hw, (r + 1) * F_loc * hw)
    return torch.cat([per_half + h * F_total * hw for h in range(halves)]).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("shape,bn", _scatter_params())
def test_kv_scatter(cuda, shape, bn):
    """Every rank of every R, with both CFG halves and with one: the scatter against fp64 and the plain GEMM, R identical
    destinations, untouched rows, Q columns of `out` and its unwritten K|V columns; and the K|V bits of the full-window
    GEMM at every width equal at the automatic one."""
    from diffuman4d_b200 import ops
    _, K, heads, d, hw, F_total, Rs = shape
    Cp = heads * pad_head_dim(d)
    N = 3 * Cp
    L = _layer(shape)
    a, w, full, ref64 = L["a"], L["w"], L["full"], L["ref64"]
    assert torch.equal(_bits(full[bn][:, Cp:]), _bits(full[0][:, Cp:])), \
        f"the K|V columns of the full-window GEMM differ between block_n {bn} and the automatic width"
    guard = 64
    for halves in (2, 1):
        rows_global = F_total * hw
        for R in Rs:
            rows_local = F_total // R * hw
            dst = [torch.full((halves * rows_global + guard, 2 * Cp), SENT16, dtype=torch.int16, device="cuda")
                   for _ in range(R)]
            expect = torch.full_like(dst[0], SENT16)
            for r in range(R):
                rows = _rank_rows(halves, F_total, R, r, hw)
                a_loc = a[rows].contiguous()
                out = torch.full((rows.numel(), N), SENT16, dtype=torch.int16, device="cuda").view(torch.bfloat16)
                ops.gemm_kv_scatter(a_loc, w, kv_col0=Cp, rows_local=rows_local, rows_global=rows_global,
                                    row_offset=r * rows_local, dst=[t.view(torch.bfloat16) for t in dst], out=out, block_n=bn)
                plain = ops.gemm(a_loc, w, block_n=bn)
                what = f"halves {halves} R {R} rank {r}"
                got = dst[0][rows].view(torch.bfloat16)
                _close(got, ref64[rows, Cp:], what=what + " K|V vs fp64")
                assert torch.equal(_bits(got), _bits(plain[:, Cp:])), f"{what}: K|V differ from the plain GEMM's"
                assert torch.equal(_bits(out[:, :Cp]), _bits(plain[:, :Cp])), f"{what}: Q columns of out differ"
                assert (_bits(out[:, Cp:]) == SENT16).all(), f"{what}: the scatter wrote K|V columns of out"
                expect[rows] = dst[0][rows]
                for k, t in enumerate(dst):
                    assert torch.equal(t, expect), \
                        f"{what}: destination {k} differs outside the rank's rows or from destination 0"
            # the gathered window (half-major, as the full window's rows) is the full-window GEMM's K|V, at any width
            assert torch.equal(expect[:halves * rows_global], _bits(full[0][:halves * rows_global, Cp:])), \
                f"halves {halves} R {R}: gathered K|V at block_n {bn} differ from the full-window GEMM at the automatic width"


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [pytest.param(s, id=s[0]) for s in SHAPES])
def test_attention_over_gathered_kv(cuda, shape):
    """The R ranks' attention over one gathered buffer, concatenated, is the fused-QKV attention of the full window bit
    for bit, and fp64 softmax attention (on >= 64 sampled query rows per rank, its first and last among them) within the
    attention tolerance."""
    from diffuman4d_b200 import ops
    _, K, heads, d, hw, F_total, Rs = shape
    dp = pad_head_dim(d)
    Cp = heads * dp
    L = _layer(shape)
    a, w, qkv_full = L["a"], L["w"], L["full"][0]
    scale = d ** -0.5
    halves, rows_global = 2, F_total * hw
    o_full = ops.attention(qkv_full, halves, rows_global, heads, dp, scale)
    g = torch.Generator().manual_seed(11)
    for R in Rs:
        rows_local = F_total // R * hw
        gathered = torch.empty(halves * rows_global, 2 * Cp, dtype=torch.bfloat16, device="cuda")
        o_sh = torch.empty_like(o_full)
        q = []
        for r in range(R):
            rows = _rank_rows(halves, F_total, R, r, hw)
            q.append(ops.gemm_kv_scatter(a[rows].contiguous(), w, kv_col0=Cp, rows_local=rows_local,
                                         rows_global=rows_global, row_offset=r * rows_local, dst=[gathered]))
        for r in range(R):                                   # after every rank has scattered
            rows = _rank_rows(halves, F_total, R, r, hw)
            o_sh[rows] = ops.attention(q[r], halves, rows_local, heads, dp, scale, kv=gathered)
            M_loc = rows.numel()
            pick = torch.cat([torch.tensor([0, M_loc - 1]), 1 + torch.randperm(M_loc - 2, generator=g)[:62]]).sort()[0]
            for h in range(halves):
                sel = pick[(pick // rows_local) == h].cuda()
                if sel.numel() == 0:
                    continue
                kv = gathered[h * rows_global:(h + 1) * rows_global].double().view(rows_global, 2, heads, dp)
                qd = q[r][sel, :Cp].double().view(-1, heads, dp)
                p = torch.softmax(torch.einsum("nhd,khd->nhk", qd, kv[:, 0]) * scale, dim=-1)
                ref = torch.einsum("nhk,khd->nhd", p, kv[:, 1]).reshape(-1, Cp)
                _close(o_sh[rows[sel]], ref, rtol=1e-2, afrac=5e-3, what=f"R {R} rank {r} half {h} attention vs fp64")
        assert torch.equal(_bits(gathered), _bits(qkv_full[:, Cp:].contiguous())), f"R {R}: gathered K|V"
        assert torch.equal(_bits(o_sh), _bits(o_full)), f"R {R}: sharded attention differs from the full window's"


# ------------------------------------------------------------------------------------------------ one-rank loopback plan
LOOP_CONFIGS = {
    "tiny_pose_tem_linear": UNetConfig.tiny(),
    "tiny_attn2_convproj_nopose": UNetConfig.tiny(cross_attention_dim=(64, 128, 256, 256), use_linear_projection=False,
                                                  enable_pose_encoder=False, enable_tem_embeds=False, in_channels=15),
    "headdim40_80": UNetConfig(block_out_channels=(320, 320, 640, 640), attention_head_dim=(8, 8, 8, 8),
                               enable_pose_encoder=False, in_channels=15),
    "tiny_n3d0": UNetConfig.tiny(num_3d_attn_blocks=0),
    "tiny_n3d1": UNetConfig.tiny(num_3d_attn_blocks=1),
    "tiny_n3d4": UNetConfig.tiny(num_3d_attn_blocks=4),
}
LOOP_SHAPE = {"headdim40_80": (2, 8, 8)}                     # (F, h, w); the others (4, 16, 16)


@pytest.fixture
def gloo_world1(tmp_path):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"file://{tmp_path / 'store'}", rank=0, world_size=1)
    try:
        yield
    finally:
        dist.destroy_process_group()


def _handles(cfg, h, w, F):
    """A plain handle and a loopback handle (FrameShardedPipeline of world 1) with the same weights."""
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.sharded import FrameShardedPipeline
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict
    sd = random_state_dict(cfg, seed=1)
    pipes = [B200Diffuman4DPipeline(B200MultiviewUNet(cfg, 0).load_state_dict(sd), SchedulerConfig(),
                                    emulate_bf16_scheduler=True) for _ in range(2)]
    sh = FrameShardedPipeline(pipes[1], max_frames=F, h=h, w=w)
    assert sh.world == 1 and sh.frames(F) == (0, F)
    return pipes[0], pipes[1], sh


def _inputs(cfg, F, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2 * F, cfg.in_channels, h, w, generator=g).to(torch.bfloat16).cuda()
    t = torch.randint(0, 1000, (2 * F,), generator=g).cuda()
    sk = (torch.rand(2 * F, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16).cuda() if cfg.enable_pose_encoder else None
    return x, t, sk


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(LOOP_CONFIGS))
def test_loopback_unet_forward_is_bit_identical(cuda, gloo_world1, name):
    """The sharded plan of one rank equals the plain plan bit for bit, with sharded and plain forwards interleaved on the
    loopback handle and spatial / temporal plans alternating, so that the global epoch counter (and, with an odd number
    of 3-D layers, the buffer parity) carries across plan boundaries."""
    cfg = LOOP_CONFIGS[name]
    F, h, w = LOOP_SHAPE.get(name, (4, 16, 16))
    plain, loop, sh = _handles(cfg, h, w, F)
    x, t, sk = _inputs(cfg, F, h, w)
    ref = {dom: plain.unet(x, t, sk, [dom, dom], F, return_dict=False)[0] for dom in ("spatial", "temporal")}
    for dom, sharded in [("spatial", True), ("temporal", True), ("spatial", False), ("temporal", True),
                         ("temporal", False), ("spatial", True), ("spatial", True)]:
        y = sh.unet_forward(x, t, sk, [dom, dom], F, F) if sharded else loop.unet(x, t, sk, [dom, dom], F, return_dict=False)[0]
        assert torch.equal(y, ref[dom]), f"{'sharded' if sharded else 'plain'} {dom} forward on the loopback handle: " \
                                         f"max diff {(y.float() - ref[dom].float()).abs().max().item()}"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_pose_tem_linear", "tiny_attn2_convproj_nopose", "tiny_n3d4"])
def test_loopback_denoise_window_is_bit_identical(cuda, gloo_world1, name):
    """Three DDIM window steps, CFG on (pose encoder: the shared negative skeleton image) and off, both domains."""
    cfg = LOOP_CONFIGS[name]
    F, h, w = 4, 16, 16
    plain, _, sh = _handles(cfg, h, w, F)
    g = torch.Generator().manual_seed(3)
    lat, pix, plk = (torch.randn(F, c, h, w, generator=g).to(torch.bfloat16).cuda() for c in (4, 4, 6))
    skel = ((torch.rand(F, 3, 8 * h, 8 * w, generator=g) * 2 - 1) if cfg.enable_pose_encoder
            else torch.randn(F, 4, h, w, generator=g)).to(torch.bfloat16).cuda()
    mask = torch.ones(F, 1, h, w, dtype=torch.bfloat16, device="cuda")
    mask[1] = 0
    ti = torch.tensor([0, 3, 2, 1], device="cuda")
    for pipe in (plain, sh.pipe):
        pipe.parepare_schedulers(18, F)
    for dom in ("spatial", "temporal"):
        for gs in (2.0, 1.0):
            kw = dict(pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skel, cond_masks_latents=mask,
                      domain=dom, guidance_scale=gs, num_inference_steps=3)
            l_ref, t_ref = lat.clone(), ti.clone()
            plain.denoise_window(latents=l_ref, timestep_indices=t_ref, **kw)
            l_sh, t_sh = lat.clone(), ti.clone()
            sh.denoise_window(latents=l_sh, timestep_indices=t_sh, F_total=F, **kw)
            assert torch.equal(t_sh, t_ref) and torch.equal(l_sh, l_ref), \
                f"{dom} guidance {gs}: max diff {(l_sh.float() - l_ref.float()).abs().max().item()}"


@pytest.mark.gpu
@pytest.mark.parametrize("dpm", [False, True], ids=["ddim", "dpm"])
def test_loopback_refusals_match_the_single_gpu_calls(cuda, gloo_world1, dpm):
    """The sharded window step and forward refuse what denoise_window and forward refuse, with the same message."""
    from diffuman4d_b200.config import DPMSolverConfig
    from diffuman4d_b200.pipeline import B200Diffuman4DPipeline
    from diffuman4d_b200.scheduler import DPMSolverState
    from diffuman4d_b200.sharded import FrameShardedPipeline
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict
    cfg = LOOP_CONFIGS["tiny_pose_tem_linear"]
    F, h, w = 4, 16, 16
    pipe = B200Diffuman4DPipeline(B200MultiviewUNet(cfg, 0).load_state_dict(random_state_dict(cfg, seed=1)),
                                  DPMSolverConfig() if dpm else SchedulerConfig())
    sh = FrameShardedPipeline(pipe, max_frames=F, h=h, w=w)
    pipe.parepare_schedulers(18, F)
    g = torch.Generator().manual_seed(3)
    lat, pix, plk = (torch.randn(F, c, h, w, generator=g).to(torch.bfloat16).cuda() for c in (4, 4, 6))
    skel = (torch.rand(F, 3, 8 * h, 8 * w, generator=g) * 2 - 1).to(torch.bfloat16).cuda()
    ti = torch.zeros(F, dtype=torch.int64, device="cuda")
    state = lambda **k: DPMSolverState(F, "cuda", **{"x0_prev": torch.zeros_like(lat), **k})
    ok = dict(latents=lat, pixel_values_latents=pix, plucker_embeds_latents=plk, skeletons_latents=skel,
              cond_masks_latents=torch.ones(F, 1, h, w, dtype=torch.bfloat16, device="cuda"), timestep_indices=ti,
              domain="spatial", guidance_scale=2.0, solver_state=state() if dpm else None)
    refused = [(dict(latents=lat.float()), "latents must be"),
               (dict(latents=lat.transpose(2, 3)), "latents must be"),
               (dict(timestep_indices=ti.int()), "timestep_indices must be"),
               (dict(timestep_indices=torch.zeros(2 * F, dtype=torch.int64, device="cuda")[::2]), "timestep_indices must be")]
    if dpm:
        refused += [(dict(solver_state=None), "needs the window frames' solver_state"),
                    (dict(solver_state=state(x0_prev=torch.zeros_like(lat[:, :, : h // 2]))), "solver_state.x0_prev must be"),
                    (dict(solver_state=state(lower_order_nums=ti.clone())), "solver_state.lower_order_nums must be")]
    for change, msg in refused:
        kw = {**ok, **change}
        with pytest.raises(ValueError, match=msg) as single:
            pipe.denoise_window(**kw)
        with pytest.raises(ValueError) as sharded:
            sh.denoise_window(F_total=F, **kw)
        assert str(sharded.value) == str(single.value)

    x, t, sk = _inputs(cfg, F, h, w)
    doms = ["spatial", "spatial"]
    refused = [((x, t, sk, ["spatial"]), "num_frames"), ((x, t, sk, ["diagonal", "spatial"]), "Invalid domain"),
               ((x[:, :5], t, sk, doms), "channels"), ((x, t[:3], sk, doms), "one entry per image"),
               ((x, t, None, doms), "skeletons are required"), ((x, t, sk[..., : 4 * w], doms), "skeletons must be")]
    for args, msg in refused:
        with pytest.raises(ValueError, match=msg) as single:
            pipe.unet(*args, F)
        with pytest.raises(ValueError) as sharded:
            sh.unet_forward(*args, F, F)
        assert str(sharded.value) == str(single.value)


def _sharded_forward(unet, x, t, sk, doms, F):
    """The sharded forward of a handle whose exchange was opened by hand (no FrameShardedPipeline)."""
    return unet._forward(x, t, sk, doms, F, F_total=F)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_pose_tem_linear", "tiny_n3d4"])
def test_loopback_exchange_size_is_exact(cuda, name):
    """An exchange buffer of exchange_bytes runs the forward (bit-identical to the plain plan); 2 bytes less is refused
    with an argument error that names d4d_exchange_alloc."""
    from diffuman4d_b200._lib import check, lib
    from diffuman4d_b200.unet import B200MultiviewUNet
    from diffuman4d_b200.weights import random_state_dict
    cfg = LOOP_CONFIGS[name]
    F, h, w = 4, 16, 16
    sd = random_state_dict(cfg, seed=1)
    x, t, sk = _inputs(cfg, F, h, w)
    ref = B200MultiviewUNet(cfg, 0).load_state_dict(sd)(x, t, sk, ["temporal"] * 2, F, return_dict=False)[0]
    for short in (0, 2):
        unet = B200MultiviewUNet(cfg, 0).load_state_dict(sd)
        blob = (C.c_ubyte * 192)()
        check(lib().d4d_exchange_alloc(unet._h, exchange_bytes(cfg, F, h, w) - short, blob), "d4d_exchange_alloc")
        check(lib().d4d_exchange_open(unet._h, 0, 1, blob), "d4d_exchange_open")
        if short:
            with pytest.raises(ValueError, match="d4d_exchange_alloc"):
                _sharded_forward(unet, x, t, sk, ["temporal"] * 2, F)
        else:
            assert torch.equal(_sharded_forward(unet, x, t, sk, ["temporal"] * 2, F), ref)
