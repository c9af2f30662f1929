"""The GEMM and implicit-GEMM convolution kernels against fp64 at every launch of the benchmarked plans.

test_gpu_ops.py, test_gpu_kernel_edges.py and test_gpu_gemm_epilogue.py accept |out - ref| <= 8e-3 |ref| + 2e-3 max|ref|,
several bf16 roundings wide: a final pack that truncates, an fp32 bias rounded to bf16 before the add, or acc + bias
rounded to bf16 before the residual all pass it.  Here every distinct GEMM and convolution launch of the plans in PLANS
(plan.launches, which test_plan.py checks against the library's profiled launch counts) runs at the tile and schedule
the library picks for it, on seeded inputs in the plan's layout, and is compared with

  R64  the exact formula in float64 on the kernel's own bf16 operands: fp32 bias as passed, exact-erf GELU, exact SiLU,
       the same out_scale; convolutions through an explicit tap gather and float64 matmuls (no cuDNN: its fp32
       algorithms are not exact and its TF32 default rounds the operands);
  C    bf16_RN(R64), correctly rounded (decided between the two bf16 neighbours in float64: torch's float64 -> bfloat16
       rounds twice, through fp32);
  tau  the accumulation allowance c_acc 2^-24 sqrt(ceil(K/16)) (sum_k |a_k w_k| + |bias| + |rowvec| + |residual|),
       carried through SiLU (slope <= 1.1, plus 2^-21 relative for __expf / __fdividef), out_scale, and GEGLU
       (|gelu(g)| tau_a + |a| (1.13 tau_g + 1e-6); 1e-6 covers the fit's 7e-7 and ex2.approx).

Per launch and input distribution:

  (a) |K - R64| <= ulp(R64) / 2 + tau at every checked element: K is a correct rounding of a value within tau of R64;
      every output finite, the guard rows and columns of the output and the statistics guard words untouched;
  (b) the share of K != C among elements with |R64| >= 2^-6 rms(R64) is at most MISMATCH_MAX;
  (c) |mean((K - R64) sign(R64) / ulp(R64))| over the same elements is at most BIAS_MAX ulp.

Above REF_BUDGET multiply-adds the reference runs on sampled rows (all N columns): for GEMMs rows of every 128-row tile,
their positions rotating so that every position 0-255 of a pair of tiles appears, plus the last row; for convolutions
whole images (first, middle, last), so every in-tile position and every border pixel is checked.

The integer census has no tolerance.  With a, w in {-3..3}, bias a multiple of 0.5 up to 2048, small integer row vector
and residual, and out_scale 2, every partial sum is exact in fp32 in any order, so the whole output must be
bf16_RN(exact) bit for bit: a dropped, repeated or misplaced k-block, tap, padding pixel, sub-pixel phase, image row
vector or N-tile bias changes bits, and the ties (a few percent of the outputs) pin ties-to-even.  The upsampling
reference there is nearest x2 followed by the 3x3 conv with the original weights, which pins the host's sub-pixel
decomposition too.  A second draw (a, w in {-1, 0, 1}, integer epilogue operands, |output| < 1024) makes every 16-row
statistics partial exact, so the GroupNorm statistics words must equal sum x 2^28 and sum x^2 2^24 exactly.  The census
runs on every launch without SiLU or GEGLU.

test_gemm_conv_criteria_rehearsal sets C_ACC, MISMATCH_MAX and BIAS_MAX on a CPU emulation of the kernels (its docstring
has the numbers).  Measured on an H100 80GB HBM3 (700 W power limit) over the 198 plan launches and 8 edges: (a) holds
everywhere; the worst element needs c_acc 1.58 (ctor-W16@64 QKV GEMM, N 1536, K 320, "wide"), more than the truncating
emulation's 1.12 and below C_ACC = 2, at which the rehearsal still catches every defect; (b) up to 8.2e-3; (c) at most
0.004 ulp; every census and statistics census exact, with up to 88% of the outputs rounded and up to 14% exact ties.
This file takes 27 s on that card.
"""
import math
import os
import time
from collections import namedtuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from diffuman4d_b200.plan import launches, modules, pad_head_dim
from test_gpu_attention_fp64 import ATTN2, PLANS, SHARDED  # noqa: E402
from test_gpu_kernel_edges import _check_guard, _check_ws, _guarded, _stats_ws  # noqa: E402

C_ACC = 2.0                 # tau's constant (set by the rehearsal; see there)
MISMATCH_MAX = 0.05         # (b): share of K != bf16_RN(R64)
BIAS_MAX = 0.1              # (c): |signed mean error| in ulp
REF_BUDGET = 2 ** 35        # multiply-adds of the fp64 reference per launch and distribution; beyond it rows are sampled
DISTRIBUTIONS = ("unit", "offset", "wide", "epilogue")
HANDLED = ("bias", "act", "scale", "residual", "rowvec", "two_source", "geglu", "stats")
EXCLUDED = {"kv_scatter": "test_gpu_kv_exchange.py pins the K/V scatter bit-equal to the plain GEMM, which this file covers"}
OUT_SCALE = float(np.float32(0.7317))   # the pose projection's learned scale: not a power of two
CENSUS_SCALE = 2.0     # a power of two: integers stay integers
CONV_KIND = {"s1": 0, "s2": 1, "up": 3}

# kind "gemm" (spec M, N, K1, K2) or "conv" (n, H, W, Cin, Cout, mode); ctx: rows (rows per image of a GEMM's
# statistics / row vector), ldt and rv_off (the row vector's [B, ldt] matrix and column offset), pad (heads, d, dpad,
# "qkv" | "out") for padded-head projections
Case = namedtuple("Case", "name kind spec feats ctx")


# ------------------------------------------------------------------------------------------------ the plans' launches
def _plan_cases():
    """The distinct (kind, spec, feats) GEMM / conv launches of PLANS (tiny-attn2 aside: test_gpu_unet_modules.py runs
    it whole), each with the layout context of its first occurrence."""
    seen, cases = set(), []
    for name, (cfg, F_, h, w) in PLANS.items():
        if cfg is ATTN2:
            continue
        offs, ldt = {}, 0
        for m in modules(cfg):
            if m.type == "resnet":
                offs[m.path], ldt = ldt, ldt + m.cout
        for l in launches(cfg, F_, h, w):
            key = (l.kind, tuple(l.spec.values()), l.feats)
            if l.kind not in ("gemm", "conv") or key in seen or set(l.feats) & set(EXCLUDED):
                continue
            seen.add(key)
            ctx = {"rows": (h >> l.level) * (w >> l.level)}
            if "rowvec" in l.feats:
                ctx.update(ldt=ldt, rv_off=offs[l.module])
            d = cfg.head_dim(l.level)
            if l.op.endswith(("qkv", "out-proj")) and pad_head_dim(d) != d:
                ctx["pad"] = (cfg.heads(l.level), d, pad_head_dim(d), "qkv" if l.op.endswith("qkv") else "out")
            cases.append(Case(name, l.kind, dict(l.spec), l.feats, ctx))
    return cases


def _g(M, N, K1, K2=0):
    return dict(M=M, N=N, K1=K1, K2=K2)


def _c(n, H, W, Cin, Cout, mode):
    return dict(n=n, H=H, W=W, Cin=Cin, Cout=Cout, mode=mode)


# op-level edges the plans do not reach
EDGES = [Case("edge", "gemm", _g(333, 640, 320), ("bias", "residual"), {"rows": 1}),          # M % 128 != 0
         Case("edge", "gemm", _g(40, 1280, 320), ("bias", "act"), {"rows": 1}),               # M < 64
         Case("edge", "gemm", _g(1000, 400, 320), ("bias", "residual"), {"rows": 1}),         # N 400: the last tile overhangs
         Case("edge", "gemm", _g(333, 192, 72), ("bias",), {"rows": 1}),                      # K1 = 72 (ABI: K % 8 == 0)
         Case("edge", "gemm", _g(333, 192, 192, 200), ("bias", "two_source"), {"rows": 1}),   # K2 = 200
         Case("edge", "conv", _c(3, 20, 24, 72, 320, "s1"), ("bias", "rowvec", "stats"),      # Cin 72, box overhangs x and y
              {"rows": 480, "ldt": 2 * 320 + 40, "rv_off": 320 + 24}),
         Case("edge", "conv", _c(5, 4, 8, 72, 320, "up"), ("bias",), {"rows": 128}),          # images overhang the tile
         Case("edge", "conv", _c(2, 48, 40, 64, 320, "s2"), ("bias", "stats"), {"rows": 480})]
PLAN_CASES = _plan_cases()
GEMM_CONV_CASES = PLAN_CASES + EDGES


def _case_id(case):
    s = case.spec
    shape = (f"M{s['M']}-N{s['N']}-K{s['K1']}" + (f"+{s['K2']}" if s["K2"] else "") if case.kind == "gemm"
             else f"{s['mode']}-n{s['n']}-{s['H']}x{s['W']}-{s['Cin']}to{s['Cout']}")
    return f"{case.name}-{case.kind}-{shape}-{'+'.join(case.feats) or 'plain'}"


def test_launch_list_follows_the_plan():
    """GEMM_CONV_CASES holds exactly the distinct GEMM / conv launches plan.launches yields for the plans, and the input
    builder knows every epilogue feature the plans (frame-sharded ones included) use, bar the excluded K/V scatter."""
    want = set()
    for name, (cfg, F_, h, w) in PLANS.items():
        if cfg is not ATTN2:
            want |= {(l.kind, tuple(l.spec.values()), l.feats) for l in launches(cfg, F_, h, w) if l.kind != "attention"}
    got = [(c.kind, tuple(c.spec.values()), c.feats) for c in PLAN_CASES]
    assert len(got) == len(set(got)) and set(got) == want, set(got) ^ want
    feats = set()
    for cfg, F_, h, w, r in SHARDED.values():
        feats |= {f for l in launches(cfg, F_, h, w, ranks=r) if l.kind != "attention" for f in l.feats}
    feats |= {f for c in GEMM_CONV_CASES for f in c.feats}
    assert feats <= set(HANDLED) | set(EXCLUDED), feats - set(HANDLED) - set(EXCLUDED)
    assert set(EXCLUDED) == {"kv_scatter"} and "kv_scatter" in feats
    assert os.path.exists(os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_gpu_kv_exchange.py"))
    with pytest.raises(ValueError, match="dropout"):
        make_inputs(Case("x", "gemm", _g(64, 64, 64), ("bias", "dropout"), {"rows": 1}), "unit", 0, "cpu")
    print(f"\n  {len(PLAN_CASES)} plan launches ({sum(c.kind == 'gemm' for c in PLAN_CASES)} GEMM), {len(EDGES)} edges")


# ------------------------------------------------------------------------------------------------ inputs
def _dims(case):
    """(K of the dot products, N, output columns, output rows, images)."""
    s = case.spec
    if case.kind == "gemm":
        N = s["N"]
        return s["K1"] + s["K2"], N, N // 2 if "geglu" in case.feats else N, s["M"], s["M"] // case.ctx["rows"]
    oh, ow = {"s1": (s["H"], s["W"]), "s2": (s["H"] // 2, s["W"] // 2), "up": (2 * s["H"], 2 * s["W"])}[s["mode"]]
    return (4 if s["mode"] == "up" else 9) * s["Cin"], s["Cout"], s["Cout"], s["n"] * oh * ow, s["n"]


def make_inputs(case, dist, seed, device):
    """Seeded operands of one launch in the plan's layout.  Real-valued distributions (w ~ N(0, 1/K) scaled as noted):
    unit      a ~ N(0, 1); bias, row vector and residual of std 0.5;
    offset    a = 2 + N(0, 1), like post-SiLU activations: partial sums cancel;
    wide      a ~ N(0, 1) 2^U(-6, 6) per input channel: k-blocks contribute unevenly;
    epilogue  a product of std 0.5 against bias ~ N(0, 4^2), row vector and residual of std 2.
    SiLU launches get pre-activations of std 4, GEGLU launches gates of std 3.  Integer draws: "census" (a, w in
    {-3..3}, bias k/2 with |bias| <= 2048, row vector and residual in {-8..8}, out_scale 2) and "census_stats" (a, w in
    {-1, 0, 1}, bias in {-64..64}, row vector and residual in {-8..8}).
    Returns a dict: a / x, a2, w (natural layout: GEGLU a rows then g rows; conv [Cout, Cin, 3, 3]), bias (fp32),
    rv_buf ([images, ldt]) and rowvec (its column view), res, scale."""
    unknown = sorted(set(case.feats) - set(HANDLED))
    if unknown:
        raise ValueError(f"no input builder for epilogue feature(s) {unknown}")
    s, feats, ctx = case.spec, case.feats, case.ctx
    K, N, _, rows, n_img = _dims(case)
    g = torch.Generator(device=device).manual_seed(seed)
    rn = lambda *sh: torch.randn(*sh, generator=g, device=device)
    ri = lambda m, *sh: torch.randint(-m, m + 1, sh, generator=g, device=device).float()
    if case.kind == "gemm":
        in_shape, w_shape, K1 = (s["M"], s["K1"]), (N, K), s["K1"]
        res_shape = (s["M"], N)
    else:
        in_shape, w_shape, K1 = (s["n"], s["H"], s["W"], s["Cin"]), (N, s["Cin"], 3, 3), s["Cin"]
        res_shape = (rows, N)
    K2 = s.get("K2", 0)
    out = {"scale": 1.0}
    if dist in ("census", "census_stats"):
        m = 3 if dist == "census" else 1
        a, a2, w = ri(m, *in_shape), ri(m, s["M"], K2) if K2 else None, ri(m, *w_shape)
        bias = 0.5 * ri(4096, N) if dist == "census" else ri(64, N)
        rv, res = ri(8, n_img, ctx.get("ldt", N)), ri(8, *res_shape)
        if "scale" in feats:
            out["scale"] = CENSUS_SCALE
    elif dist in DISTRIBUTIONS:
        a, a2 = rn(*in_shape), rn(s["M"], K2) if K2 else None
        wscale = K ** -0.5
        if dist == "offset":
            a += 2.0
            a2 = None if a2 is None else a2 + 2.0
        elif dist == "wide":
            sc = torch.exp2(12 * torch.rand(K1 + K2, generator=g, device=device) - 6)
            a *= sc[:K1]
            a2 = None if a2 is None else a2 * sc[K1:]
            wscale /= sc.pow(2).mean().sqrt().item()
        elif dist == "epilogue":
            wscale *= 0.5
        w = rn(*w_shape) * wscale * (4.0 if "act" in feats else 1.0)
        if "geglu" in feats:
            w[N // 2:] *= 3.0
        sb, se = (4.0, 2.0) if dist == "epilogue" else (0.5, 0.5)
        bias, rv, res = sb * rn(N), se * rn(n_img, ctx.get("ldt", N)), se * rn(*res_shape)
        if "scale" in feats:
            out["scale"] = OUT_SCALE
    else:
        raise ValueError(dist)
    if "pad" in ctx:   # padded heads: the loader's zero weight rows (QKV) or columns (out-proj); attention writes 0 there
        heads, d, dp, role = ctx["pad"]
        if role == "qkv":
            w[(torch.arange(N, device=device) % (heads * dp)) % dp >= d] = 0
        else:
            dead = torch.arange(K1, device=device) % dp >= d
            w[:, dead] = 0
            a[:, dead] = 0
    bf = lambda t: None if t is None else t.to(torch.bfloat16)
    out.update(a=bf(a).contiguous(), a2=bf(a2), w=bf(w).contiguous(), bias=bias.float().contiguous())
    if "rowvec" in feats:
        off = ctx.get("rv_off", 0)
        out["rv_buf"] = bf(rv)
        out["rowvec"] = out["rv_buf"][:, off:off + N]
    if "residual" in feats:
        out["res"] = bf(res).contiguous()
    if "bias" not in feats:
        out["bias"] = None
    return out


# ------------------------------------------------------------------------------------------------ fp64 reference
def _conv_products(x, w, mode, need_abs, exact_up=False):
    """(sum a w, sum |a w|) of a 3x3 conv in float64 over x [n, H, W, Cin] (any float type), w [Cout, Cin, 3, 3]: one
    float64 matmul per tap.  mode "up": the four sub-pixel phases with the kernel's bf16 phase weights, or with
    exact_up nearest x2 followed by the conv with w itself.  Returns [n, Ho, Wo, Cout] tensors."""
    from diffuman4d_b200.ops import upsample_phase_weights
    xd = x.double()
    if mode == "up" and exact_up:
        xd, mode = xd.repeat_interleave(2, 1).repeat_interleave(2, 2), "s1"
    n, H, W, Cin = xd.shape
    Cout = w.shape[0]
    xp = F.pad(xd, (0, 0, 1, 1, 1, 1))
    taps = []   # (output slice [n, Ho', Wo'] of the result, input view, weight [Cout, Cin])
    if mode in ("s1", "s2"):
        st = 2 if mode == "s2" else 1
        Ho, Wo = H // st, W // st
        for ky in range(3):
            for kx in range(3):
                taps.append(((slice(None), slice(None)), xp[:, ky:ky + st * Ho:st, kx:kx + st * Wo:st], w[:, :, ky, kx]))
    else:
        Ho, Wo = 2 * H, 2 * W
        wp = torch.stack(upsample_phase_weights(w))          # [4, Cout, 4 taps, Cin]
        for pa in range(2):
            for pb in range(2):
                for ty in range(2):
                    for tx in range(2):
                        taps.append(((slice(pa, None, 2), slice(pb, None, 2)),
                                     xp[:, ty + pa:ty + pa + H, tx + pb:tx + pb + W], wp[2 * pa + pb][:, 2 * ty + tx]))
    Z = torch.zeros(n, Ho, Wo, Cout, dtype=torch.float64, device=x.device)
    S = torch.zeros_like(Z) if need_abs else None
    for (sy, sx), X, wt in taps:
        wt = wt.double()
        Z[:, sy, sx] += X @ wt.t()
        if need_abs:
            S[:, sy, sx] += X.abs() @ wt.abs().t()
    return Z, S


def reference64(case, inp, sel=None, need_abs=True, exact_up=False):
    """R64 over the selected output rows and its allowance tau = C_ACC tc + t0, as float64 [rows, output columns].
    sel: GEMM rows or conv images (None: all).  need_abs=False skips tau (tc, t0 None)."""
    s, feats = case.spec, case.feats
    K, N, _, rows, _ = _dims(case)
    if case.kind == "gemm":
        sel = torch.arange(s["M"], device=inp["a"].device) if sel is None else sel
        A = inp["a"][sel].double()
        if inp["a2"] is not None:
            A = torch.cat([A, inp["a2"][sel].double()], 1)
        Wd = inp["w"].double()
        Z, S = A @ Wd.t(), (A.abs() @ Wd.abs().t() if need_abs else None)
        img = sel // case.ctx["rows"]
        res_rows = lambda r: r[sel]
    else:
        sel = torch.arange(s["n"], device=inp["a"].device) if sel is None else sel
        Z, S = _conv_products(inp["a"][sel], inp["w"], s["mode"], need_abs, exact_up)
        hw = Z.shape[1] * Z.shape[2]
        Z, S = Z.reshape(-1, N), (S.reshape(-1, N) if need_abs else None)
        img = sel.repeat_interleave(hw)
        res_rows = lambda r: r.view(s["n"], hw, N)[sel].reshape(-1, N)
    v = 2.0 ** -24 * math.sqrt(math.ceil(K / 16))
    t0 = torch.zeros_like(Z) if need_abs else None
    if inp["bias"] is not None:
        Z += inp["bias"].double()
        S = None if S is None else S + inp["bias"].double().abs()
    if "rowvec" in feats:
        rv = inp["rowvec"].double()[img]
        Z += rv
        S = None if S is None else S + rv.abs()
    if "geglu" in feats:
        za, zg = Z[:, :N // 2], Z[:, N // 2:]
        gl = 0.5 * zg * torch.special.erfc(-zg / math.sqrt(2.0))
        R = za * gl
        if not need_abs:
            return R, None, None
        tc = v * (gl.abs() * S[:, :N // 2] + 1.13 * za.abs() * S[:, N // 2:])
        return R, tc, 1e-6 * za.abs() + 2.0 ** -24 * R.abs()
    R, tc = Z, (v * S if need_abs else None)
    if "act" in feats:
        R = Z * torch.sigmoid(Z)
        if need_abs:
            tc, t0 = 1.1 * tc, 2.0 ** -21 * R.abs()
    if inp["scale"] != 1.0:
        R = R * inp["scale"]
        if need_abs:
            tc, t0 = abs(inp["scale"]) * tc, abs(inp["scale"]) * t0 + 2.0 ** -24 * R.abs()
    if "residual" in feats:
        r = res_rows(inp["res"]).double()
        R = R + r
        if need_abs:
            tc, t0 = tc + v * r.abs(), t0 + 2.0 ** -24 * R.abs()
    return R, tc, t0


def _ulp(x):
    """bf16 ulp of float64 x: 2^(floor(log2 |x|) - 7), subnormals at 2^-133."""
    _, e = torch.frexp(x.abs())
    e = torch.where(x == 0, torch.full_like(e, -125), e).clamp_min(-125)
    return torch.exp2((e - 8).double())


def rn_bf16(x):
    """bf16 round-to-nearest-even of float64 x, in one rounding (torch's float64 -> bfloat16 rounds through fp32)."""
    u = _ulp(x)
    return torch.round(x / u) * u


def criteria(K, R, tc, t0):
    """K (kernel output) and R64, tau = C_ACC tc + t0 over the same elements, float64.  Returns {"a": worst |K - R64| /
    (ulp/2 + tau), "need": the c_acc (a) would need, "mism": (b), "bias": (c), "finite"}."""
    u = _ulp(R)
    err = torch.nan_to_num((K - R).abs(), nan=math.inf)
    frac = err / (0.5 * u + C_ACC * tc + t0)
    need = torch.where(err > 0.5 * u + t0, (err - 0.5 * u - t0) / tc.clamp_min(1e-300), torch.zeros_like(err))
    big = R.abs() >= 2.0 ** -6 * R.pow(2).mean().sqrt()
    return {"a": frac.max().item(), "need": need.max().item(),
            "mism": (K != rn_bf16(R))[big].double().mean().item(),
            "bias": ((K - R) * R.sign() / u)[big].mean().item(), "finite": bool(torch.isfinite(K).all())}


def failed(c):
    out = [] if c["finite"] else ["finite"]
    out += [] if c["a"] <= 1.0 else ["a"]
    out += [] if c["mism"] <= MISMATCH_MAX else ["b"]
    out += [] if abs(c["bias"]) <= BIAS_MAX else ["c"]
    return out


def check_a(K, case, inp, what, sel=None):
    """Criterion (a) on K (the kernel's [rows, output columns] over sel) against inp: used by the tests that compare two
    tilings or schedules with each other, against both being wrong together."""
    R, tc, t0 = reference64(case, inp, sel)
    c = criteria(K.double().reshape(R.shape), R, tc, t0)
    assert c["finite"] and c["a"] <= 1.0, f"{what}: criterion (a) at {c['a']:.3g} x the allowance (finite: {c['finite']})"


def census_expect(case, inp, sel=None):
    """The exact outputs of an integer draw, bf16_RN'd: upsampling through nearest x2 and the original weights."""
    R, _, _ = reference64(case, inp, sel, need_abs=False, exact_up=True)
    assert R.abs().max().item() < 2 ** 23, "census operands leave fp32's exact range"
    return rn_bf16(R)


def census_stats(C, n_img):
    """Exact GroupNorm statistics words of stored values C [rows, N] (integers) over n_img images, as int64 [n_img, N, 2];
    asserts that every 16-row fp32 partial of the kernel is exact (|x| < 1024: 16 x^2 < 2^24)."""
    assert C.abs().max().item() < 1024 and bool((C == C.round()).all()), "the statistics census needs integers below 1024"
    y = C.view(n_img, -1, C.shape[1])
    return torch.stack([(y.sum(1) * 2.0 ** 28).long(), (y.pow(2).sum(1) * 2.0 ** 24).long()], -1)


# ------------------------------------------------------------------------------------------------ row sampling
def sample_sel(case):
    """GEMM rows or conv images at which the fp64 reference runs (all while M N K <= REF_BUDGET)."""
    K, N, _, rows, n_img = _dims(case)
    if rows * N * K <= REF_BUDGET:
        return None
    if case.kind == "conv":
        return torch.tensor(sorted({0, n_img // 2, n_img - 1}))
    M = rows
    n_t = -(-M // 128)
    per = min(128, max(1, REF_BUDGET // (N * K * n_t)))
    t = torch.arange(n_t)[:, None]
    pos = ((t // 2) * per + torch.arange(per)[None, :]) % 128      # pairs of tiles share a start: positions 0-255 appear
    last = M - t * 128
    pos = torch.where(pos < last, pos, pos % last)
    return torch.cat([(t * 128 + pos).flatten(), torch.tensor([M - 1])]).unique()


# ------------------------------------------------------------------------------------------------ CPU emulation
def _trunc32(x):
    """float64 -> float32 toward zero."""
    f = x.float()
    return torch.where(f.double().abs() > x.abs(), torch.nextafter(f, torch.zeros_like(f)), f)


def _pack(f, mode):
    """fp32 -> bf16: "rn" (nearest even), "trunc", "away" (ties away from zero)."""
    if mode == "rn":
        return f.to(torch.bfloat16)
    b = f.view(torch.int32)
    b = b & -65536 if mode == "trunc" else (b + 0x8000) & -65536
    return b.view(torch.float32).to(torch.bfloat16)


def _gelu_fit32(g):
    """gelu_erf_f (csrc/common.cuh) in fp32: each fmaf rounded once."""
    f = lambda x: torch.tensor(x, dtype=torch.float32).double()
    u = g.abs().double()
    q = (f(-4.8811754095e-04) * u + f(7.1988063864e-03)).float().double()
    for c in (-5.2146803588e-02, -4.5959571004e-01, -1.1510006189e+00):
        q = (q * u + f(c)).float().double()
    e = torch.exp2((q * u).float()).double()
    return ((-0.5 * u).float().double() * e + g.clamp_min(0).double()).float()


def _emu_gather(case, inp, mutation):
    """The kernel's dot products as GEMMs over k-block-ordered columns: [(output row index, A [rows, Kp], W [N, Kp])],
    each source / tap zero-padded to whole 64-column k-blocks (the TMA fill)."""
    s = case.spec
    pad64 = lambda t: F.pad(t, (0, -t.shape[-1] % 64))
    if case.kind == "gemm":
        K1 = s["K1"]
        A = [pad64(inp["a"].double())] + ([pad64(inp["a2"].double())] if inp["a2"] is not None else [])
        Wd = inp["w"].double()
        W = [pad64(Wd[:, :K1])] + ([pad64(Wd[:, K1:])] if inp["a2"] is not None else [])
        return [(torch.arange(s["M"]), torch.cat(A, 1), torch.cat(W, 1))]
    x, w = inp["a"].double(), inp["w"].double()
    n, H, W_, Cin = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    if s["mode"] == "up":
        from diffuman4d_b200.ops import upsample_phase_weights
        wp = [t.double() for t in upsample_phase_weights(inp["w"])]
        if mutation == "phase_swap":
            wp[1], wp[2] = wp[2], wp[1]
        out = []
        for pa in range(2):
            for pb in range(2):
                taps = [xp[:, ty + pa:ty + pa + H, tx + pb:tx + pb + W_] for ty in range(2) for tx in range(2)]
                A = torch.cat([pad64(t.reshape(-1, Cin)) for t in taps], 1)
                Wt = torch.cat([pad64(wp[2 * pa + pb][:, t]) for t in range(4)], 1)
                oy, ox = torch.meshgrid(2 * torch.arange(H) + pa, 2 * torch.arange(W_) + pb, indexing="ij")
                idx = (torch.arange(n)[:, None, None] * (4 * H * W_) + oy * (2 * W_) + ox).flatten()
                out.append((idx, A, Wt))
        return out
    st = 2 if s["mode"] == "s2" else 1
    Ho, Wo = H // st, W_ // st
    taps = []
    for ky in range(3):
        for kx in range(3):
            if mutation == "pad_wrap":   # x +- 1 past the row reads the neighbouring row's pixel instead of zero
                xf = F.pad(x.reshape(n, H * W_, Cin), (0, 0, W_ + 1, W_ + 1))
                sh = (ky - 1) * W_ + (kx - 1)
                taps.append(xf[:, W_ + 1 + sh:W_ + 1 + sh + H * W_].reshape(n, H, W_, Cin))
            else:
                taps.append(xp[:, ky:ky + st * Ho:st, kx:kx + st * Wo:st])
    A = torch.cat([pad64(t.reshape(-1, Cin)) for t in taps], 1)
    Wt = torch.cat([pad64(w[:, :, ky, kx]) for ky in range(3) for kx in range(3)], 1)
    return [(torch.arange(n * Ho * Wo), A, Wt)]


def _emu_accumulate(A, W, acc_mode, drop_cols=None):
    """fp32 accumulation per k16 slice in k-block order; each slice's 16 products summed in fp64 (exact up to 2^-53),
    added to the accumulator with one rounding, to nearest ("rn") or toward zero ("trunc").  drop_cols: columns whose
    second k-block is left out."""
    M, Kp = A.shape
    S = Kp // 16
    P = torch.einsum("msk,nsk->smn", A.view(M, S, 16), W.view(-1, S, 16))
    acc = torch.zeros(M, W.shape[0], dtype=torch.float32)
    for i in range(S):
        x = acc.double() + P[i]
        if drop_cols is not None and 4 <= i < 8:
            x[:, drop_cols] = acc.double()[:, drop_cols]
        acc = x.float() if acc_mode == "rn" else _trunc32(x)
    return acc


def _conv_tile_images(case):
    """Images per 128-row conv tile (conv_tile in gemm_wgmma.cu)."""
    s = case.spec
    oh, ow = (s["H"] // 2, s["W"] // 2) if s["mode"] == "s2" else (s["H"], s["W"])
    bw = 16
    while bw > ow:
        bw //= 2
    bh = 128 // bw
    while bh > oh and bh > 1:
        bh //= 2
    return 128 // (bw * bh)


def emulate(case, inp, acc_mode="rn", mutation=None, cache=None):
    """The kernel on the CPU: (output bf16 [rows, output columns], statistics int64 [images, N, 2] or None).  Epilogue in
    the kernel's order: fp32 acc + bias + row vector, SiLU, out_scale, + residual, one pack; GEGLU a * gelu_erf_f(g).
    `mutation` plants one defect (MUTATIONS); `cache` keeps accumulators between calls."""
    K, N, n_out, rows, n_img = _dims(case)
    feats = case.feats
    gmut = mutation if mutation in ("pad_wrap", "phase_swap", "kblock_drop") else None
    key = (acc_mode, gmut)
    if cache is None or key not in cache:
        acc = torch.zeros(rows, N, dtype=torch.float32)
        for idx, A, W in _emu_gather(case, inp, gmut):
            acc[idx] = _emu_accumulate(A, W, acc_mode, torch.arange(N - 64, N) if gmut == "kblock_drop" else None)
        if cache is not None:
            cache[key] = acc
    acc = cache[key] if cache is not None else acc
    f = acc.clone()
    if inp["bias"] is not None:
        b = inp["bias"].to(torch.bfloat16).float() if mutation == "bias_bf16" else inp["bias"]
        f = f + b
    if "geglu" in feats:
        a, g = f[:, :N // 2], f[:, N // 2:]
        gl = (0.5 * g * (1 + torch.tanh(0.7978845608 * (g + 0.044715 * g ** 3)))) if mutation == "gelu_tanh" else _gelu_fit32(g)
        return _pack(a * gl, "rn"), None
    if "rowvec" in feats:
        img = torch.arange(rows) // (rows // n_img)
        if mutation == "rowvec_straddle":
            tile_imgs = _conv_tile_images(case)
            img = img - img % tile_imgs
        f = f + inp["rowvec"].float()[img]
    if "act" in feats:
        e = torch.exp(-f) * (1.001 if mutation == "silu_exp" else 1.0)
        f = f / (1.0 + e)
    if inp["scale"] != 1.0:
        f = f * inp["scale"]
    if "residual" in feats:
        if mutation == "double_round":
            f = f.to(torch.bfloat16).float()
        f = f + inp["res"].float().reshape(rows, N)
    out = _pack(f, {"out_trunc": "trunc", "ties_away": "away"}.get(mutation, "rn"))
    st = None
    if "stats" in feats:   # fp32 sums of 16 consecutive stored rows of an image, fixed point, integer totals
        y = out.float().view(n_img, -1, 16, N)
        part = torch.stack([y.sum(2) * 2.0 ** 28, y.pow(2).sum(2) * 2.0 ** 24], -1).double().round().long()
        if mutation == "stats_drop":
            part[0, 0] = 0
        st = part.sum(1)
    return out, st


MUTATIONS = ("out_trunc", "ties_away", "bias_bf16", "double_round", "kblock_drop", "rowvec_straddle", "gelu_tanh",
             "silu_exp", "pad_wrap", "phase_swap", "stats_drop")
# what must catch each (at least one of these, on at least one case and distribution, or in a census)
CATCHES = {"out_trunc": {"b", "c"}, "ties_away": {"census"}, "bias_bf16": {"b"}, "double_round": {"b"},
           "kblock_drop": {"a", "census"}, "rowvec_straddle": {"a", "census"}, "gelu_tanh": {"a"},
           "silu_exp": {"a", "b"}, "pad_wrap": {"a", "census"}, "phase_swap": {"a", "census"},
           "stats_drop": {"census-stats"}}
REHEARSAL = [Case("K2880", "gemm", _g(256, 320, 2880), ("bias", "residual"), {"rows": 64}),
             Case("K23040", "gemm", _g(64, 64, 23040), ("bias", "residual"), {"rows": 64}),
             Case("geglu", "gemm", _g(256, 512, 320), ("bias", "geglu"), {"rows": 64}),
             Case("silu", "gemm", _g(256, 64, 512), ("bias", "act"), {"rows": 64}),
             Case("scale+stats", "gemm", _g(256, 64, 320, 320), ("bias", "scale", "two_source", "stats"), {"rows": 64}),
             Case("conv1", "conv", _c(4, 8, 8, 72, 64, "s1"), ("bias", "rowvec", "stats"),
                  {"rows": 64, "ldt": 192, "rv_off": 72}),
             Case("conv2", "conv", _c(2, 12, 20, 128, 64, "s1"), ("bias", "residual"), {"rows": 240}),
             Case("down", "conv", _c(2, 16, 16, 64, 64, "s2"), ("bias", "stats"), {"rows": 64}),
             Case("up", "conv", _c(2, 4, 8, 64, 64, "up"), ("bias", "stats"), {"rows": 128})]


def _applies(mut, case):
    f = case.feats
    return {"double_round": "residual" in f, "rowvec_straddle": "rowvec" in f, "gelu_tanh": "geglu" in f,
            "silu_exp": "act" in f, "pad_wrap": case.kind == "conv" and case.spec["mode"] == "s1",
            "phase_swap": case.kind == "conv" and case.spec["mode"] == "up", "stats_drop": "stats" in f,
            "ties_away": not ({"act", "geglu"} & set(f))}.get(mut, True)


def _row(label, c):
    bad = failed(c)
    return (f"  {label:<34}{c['a']:>9.3f}{c['need']:>9.3f}{c['mism']:>10.2e}{c['bias']:>+9.3f}  "
            + ("ok" if not bad else "fails " + ",".join(bad)))


def _header(title, first):
    return (f"\n  {title}\n  bounds: (a) 1 at c_acc {C_ACC}, (b) {MISMATCH_MAX:.1e}, (c) {BIAS_MAX} ulp\n"
            f"  {first:<34}{'(a)':>9}{'c_acc':>9}{'(b)':>10}{'(c)':>9}")


def test_gemm_conv_criteria_rehearsal():
    """Criteria (a)-(c) and both censuses on the CPU emulation: the faithful emulation, with an accumulator that rounds
    to nearest and with one that truncates, passes everything on every case and distribution, and each MUTATIONS
    defect is caught as CATCHES says.  Measured here: a round-to-nearest accumulator needs c_acc 0.06, mismatches (b) up
    to 4.9e-4 and biases (c) 0.005 ulp; a truncating one needs c_acc 1.12 (K 2880, "wide"), mismatches up to 1.2e-2 and
    biases 0.007 ulp.  The mildest defect that only (a) sees, SiLU's 1e-3 exp error, would need c_acc 3.8: C_ACC = 2
    sits between (the H100 needs 1.58).  The mildest defect (b) must catch, the bias rounded to bf16, mismatches 17% or
    more: MISMATCH_MAX = 5% sits between.  Output truncation biases -0.50 ulp: BIAS_MAX = 0.1 ulp is 14 times the
    faithful worst.  About 8 s."""
    t0 = time.perf_counter()
    lines = [_header("CPU emulation of the GEMM / conv kernels vs fp64: worst over cases", "version / distribution")]
    versions = [("faithful rn", "rn", None), ("faithful trunc", "trunc", None)] + [(m, "rn", m) for m in MUTATIONS]
    caches = {}
    faithful, caught = [], {m: set() for m in MUTATIONS}
    for label, acc_mode, mut in versions:
        for dist in DISTRIBUTIONS:
            runs = []
            for i, case in enumerate(REHEARSAL):
                if mut is not None and not _applies(mut, case):
                    continue
                inp = make_inputs(case, dist, 10 + i, "cpu")
                K, _ = emulate(case, inp, acc_mode, mut, caches.setdefault((i, dist), {}))
                c = criteria(K.double(), *reference64(case, inp))
                runs.append(c)
                if mut is None:
                    faithful.append((label, dist, case.name, c))
                else:
                    caught[mut] |= {(crit, f"{case.name}/{dist}") for crit in failed(c)}
            if runs:
                w = {"a": max(c["a"] for c in runs), "need": max(c["need"] for c in runs),
                     "mism": max(c["mism"] for c in runs), "bias": max((c["bias"] for c in runs), key=abs),
                     "finite": all(c["finite"] for c in runs)}
                lines.append(_row(f"{label} / {dist}", w))
    census_lines = []
    for label, acc_mode, mut in versions:
        for i, case in enumerate(REHEARSAL):
            if {"act", "geglu"} & set(case.feats) or (mut is not None and not _applies(mut, case)):
                continue
            for dist in ("census", "census_stats") if "stats" in case.feats else ("census",):
                inp = make_inputs(case, dist, 50 + i, "cpu")
                K, st = emulate(case, inp, acc_mode, mut)
                C = census_expect(case, inp)
                miss = int((K.double() != C).sum())
                smiss = 0
                if dist == "census_stats":
                    smiss = int((st != census_stats(C, _dims(case)[4])).sum())
                if mut is None:
                    assert miss == 0 and smiss == 0, f"{label} misses the {dist} of {case.name}: {miss} outputs, {smiss} words"
                    if dist == "census":
                        R = reference64(case, inp, need_abs=False, exact_up=True)[0]
                        u = _ulp(R)
                        census_lines.append(f"  census {case.name:<12} rounded {(R != C).double().mean().item():.2f}, "
                                            f"ties {((R / u) % 1 == 0.5).double().mean().item():.3f}")
                else:
                    if miss:
                        caught[mut].add(("census", case.name))
                    if smiss:
                        caught[mut].add(("census-stats", case.name))
    print("\n".join(lines))
    print("\n".join(sorted(set(census_lines))))
    for name in ("faithful rn", "faithful trunc"):
        cs = [c for lab, *_, c in faithful if lab == name]
        print(f"  {name:<15} worst: (a) {max(c['a'] for c in cs):.3f} (needs c_acc {max(c['need'] for c in cs):.3f}), "
              f"(b) {max(c['mism'] for c in cs):.2e}, (c) {max((c['bias'] for c in cs), key=abs):+.3f} ulp")
    for mut in MUTATIONS:
        names = sorted({crit for crit, _ in caught[mut]})
        where = sorted({f"{crit}@{w}" for crit, w in caught[mut]})
        print(f"  {mut:<16} caught by {', '.join(names) or 'nothing'}: {', '.join(where[:6])}{' ...' if len(where) > 6 else ''}")
    print(f"  [rehearsal] {time.perf_counter() - t0:.1f} s")
    for label, dist, name, c in faithful:
        assert not failed(c), f"{label} fails {failed(c)} on {name} / {dist}: {c}"
    for mut in MUTATIONS:
        assert {crit for crit, _ in caught[mut]} & CATCHES[mut], f"{mut} not caught by {CATCHES[mut]}: {caught[mut]}"


# ------------------------------------------------------------------------------------------------ GPU
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def tile_choice(case):
    """The library's (block_m, block_n, schedule) for the launch, as text."""
    import ctypes
    from diffuman4d_b200._lib import check, lib
    s = case.spec
    a, b = ctypes.c_int(), ctypes.c_int()
    if case.kind == "gemm":
        check(lib().d4d_gemm_tile_choice(s["M"], s["N"], s["K1"], s["K2"], int("geglu" in case.feats), _sms(),
                                         ctypes.byref(a), ctypes.byref(b)))
        return f"128x{a.value} {'ping-pong' if b.value == 2 else 'cooperative'}"
    check(lib().d4d_conv_tile_choice(s["n"], s["H"], s["W"], s["Cin"], s["Cout"], CONV_KIND[s["mode"]], _sms(),
                                     ctypes.byref(a), ctypes.byref(b)))
    return f"{a.value}x{b.value}"


def run_kernel(case, inp):
    """One launch at block_n 0 through the C entry points ops.gemm / ops.conv3x3 / ops.conv3x3_stride2 /
    ops.upsample2x_conv3x3 call, into an output with guard rows (and, for GEMMs, guard columns) and a guarded statistics
    workspace.  Returns (output buffer, output [rows, output columns], workspace or None)."""
    from diffuman4d_b200 import ops
    from diffuman4d_b200._lib import check, lib
    s, feats = case.spec, case.feats
    K, N, n_out, rows, n_img = _dims(case)
    p = lambda t: None if t is None else t.data_ptr()
    stream = torch.cuda.current_stream().cuda_stream
    ws = _stats_ws(n_img * N * 2) if "stats" in feats else None
    rv = inp.get("rowvec")
    ld_rv = 0 if rv is None else rv.stride(0)
    if case.kind == "gemm":
        ldo = n_out + 64
        buf = _guarded(rows, n_out, ldo, 64)
        w, b = inp["w"], inp["bias"]
        if "geglu" in feats:
            w, b = ops.interleave_geglu(w, b)
        a2, res = inp["a2"], inp.get("res")
        check(lib().d4d_op_gemm(p(inp["a"]), inp["a"].stride(0), s["K1"], p(a2), 0 if a2 is None else a2.stride(0), s["K2"],
                                p(w), rows, N, p(b), p(rv), ld_rv, case.ctx["rows"] if rv is not None else 0, p(res),
                                0 if res is None else res.stride(0), p(buf), ldo, int("geglu" in feats),
                                int("act" in feats), float(inp["scale"]), 0, p(ws),
                                case.ctx["rows"] if ws is not None else 0, stream), "d4d_op_gemm")
        return buf, buf[:rows, :n_out], ws
    buf = _guarded(rows, N, N, 256)
    x = inp["a"]
    if s["mode"] == "s1":
        check(lib().d4d_op_conv3x3(p(x), s["n"], s["H"], s["W"], s["Cin"], p(ops.conv_weight_to_octi(inp["w"])), N,
                                   p(inp["bias"]), p(rv), ld_rv, p(inp.get("res")), int("act" in feats), p(buf), 0, p(ws),
                                   stream), "d4d_op_conv3x3")
    else:
        wt = (ops.conv_weight_to_octi(inp["w"]) if s["mode"] == "s2"
              else torch.stack(ops.upsample_phase_weights(inp["w"])).contiguous())
        check(lib().d4d_op_conv_resample(p(x), s["n"], s["H"], s["W"], s["Cin"], p(wt), N, p(inp["bias"]),
                                         CONV_KIND[s["mode"]], 0, 0, p(buf), p(ws), stream), "d4d_op_conv_resample")
    return buf, buf[:rows], ws


def _selected(case, out, sel):
    """The kernel's outputs at the reference's rows, float64."""
    if sel is None:
        return out.double()
    if case.kind == "gemm":
        return out[sel.to(out.device)].double()
    n = case.spec["n"]
    return out.view(n, -1, out.shape[1])[sel.to(out.device)].reshape(-1, out.shape[1]).double()


def _census_check(case, inp, out, keep_expected, chunk_elems=2 ** 27):
    """(outputs that differ from bf16_RN(exact), share that needed rounding, share of exact ties, and the expected
    outputs if keep_expected), reference in chunks of rows or images."""
    K, N, _, rows, n_img = _dims(case)
    unit = case.spec["M"] if case.kind == "gemm" else case.spec["n"]
    per = rows // unit
    step = max(1, chunk_elems // (per * K + per * N))
    miss = rounded = ties = 0
    keep = []
    for i in range(0, unit, step):
        sel = torch.arange(i, min(unit, i + step), device=out.device)
        R, _, _ = reference64(case, inp, sel, need_abs=False, exact_up=True)
        C = rn_bf16(R)
        u = _ulp(R)
        miss += int((_selected(case, out, sel) != C).sum())
        rounded += int((R != C).sum())
        ties += int(((R / u) % 1 == 0.5).sum())
        if keep_expected:
            keep.append(C)
    return miss, rounded / out.numel(), ties / out.numel(), torch.cat(keep) if keep_expected else None


@pytest.mark.gpu
@pytest.mark.parametrize("case", GEMM_CONV_CASES, ids=_case_id)
def test_gemm_conv_launch_vs_fp64(cuda, case):
    """One launch of the plans (or EDGES): criteria (a)-(c) at every distribution, finite outputs, untouched guards and
    statistics within test_gpu_kernel_edges.py's bound; the integer census over the whole output, and the statistics
    census where the launch has statistics."""
    t0 = time.perf_counter()
    K, N, n_out, rows, n_img = _dims(case)
    sel = sample_sel(case)
    if sel is not None and case.kind == "gemm" and rows >= 128 * 256:
        assert (sel % 256).unique().numel() == 256, "the sample misses a row position of a tile pair"
    n_sel = rows if sel is None else (len(sel) if case.kind == "gemm" else len(sel) * rows // n_img)
    lines = [f"\n  {_case_id(case)}: tile {tile_choice(case)}, fp64 on {n_sel} of {rows} rows",
             f"  {'distribution':<34}{'(a)':>9}{'c_acc':>9}{'(b)':>10}{'(c)':>9}"]
    fails = []
    for i, dist in enumerate(DISTRIBUTIONS):
        inp = make_inputs(case, dist, 2000 + i, "cuda")
        buf, out, ws = run_kernel(case, inp)
        _check_guard(buf, rows, n_out, f"{dist}")
        if ws is not None:
            _check_ws(ws, out, n_img, f"{dist} statistics")
        c = criteria(_selected(case, out, sel), *reference64(case, inp, None if sel is None else sel.cuda()))
        fails += [f"{dist}: {b}" for b in failed(c)]
        lines.append(_row(dist, c))
        del inp, buf, out, ws
    if not {"act", "geglu"} & set(case.feats):
        for dist in ("census", "census_stats") if "stats" in case.feats else ("census",):
            inp = make_inputs(case, dist, 3000, "cuda")
            buf, out, ws = run_kernel(case, inp)
            _check_guard(buf, rows, n_out, dist)
            miss, rounded, ties, C = _census_check(case, inp, out, dist == "census_stats")
            line = f"  {dist:<34}{miss} of {out.numel()} differ; {rounded:.2f} rounded, {ties:.3f} ties"
            if miss:
                fails.append(f"{dist}: {miss} outputs differ from bf16_RN(exact)")
            if dist == "census_stats":
                _check_ws(ws, out, n_img, "census statistics")
                bad = int((ws[:n_img * N * 2].view(n_img, N, 2) != census_stats(C, n_img)).sum())
                line += f"; {bad} statistics words differ"
                if bad:
                    fails.append(f"{dist}: {bad} statistics words differ from the exact sums")
            lines.append(line)
            del inp, buf, out, ws, C
    torch.cuda.synchronize()
    print("\n".join(lines) + f"\n  [{_case_id(case)}] {time.perf_counter() - t0:.1f} s")
    assert not fails, fails
