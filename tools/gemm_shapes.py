"""Per-shape timing of the GEMM / conv launches of one W16@64² UNet forward (SD-2.1 layout, 32 images, CFG).

    python tools/gemm_shapes.py [--reps 20] [--json OUT]

Every distinct GEMM / conv launch shape of the plan (diffuman4d_b200/plan.py, which mirrors PlanBuilder in csrc/unet.cu)
runs with the epilogue features the plan gives it, through the C ABI on pre-allocated buffers, captured `reps` times
into a CUDA graph and timed with CUDA events after warm-up.  Per shape: launches per forward, the tile rows and width gemm_prepare picks, µs per launch, TFLOP/s
(executed FLOPs: the upsampling convs run 4 taps per phase), compulsory HBM bytes and GB/s, and the least time the card
could take: the larger of FLOPs / tensor peak and bytes / 3.35 TB/s, naming which bounds the shape.  The tensor peak is
4096 dense BF16 FLOP/clk/SM at the card's maximum SM clock; a power-limited card runs below it under load.
The count-weighted totals are the `gemm` and `conv3x3` kinds of bench.py's roofline.by_kind_ms.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from diffuman4d_b200.config import UNetConfig  # noqa: E402
from diffuman4d_b200.plan import launches  # noqa: E402

HBM_BPS = 3.35e12
B = 32


def label(launch):
    """The short name of a launch: its op, after its level (L1..L4; the mid block's transformer: mid)."""
    if launch.op in ("time1", "tem1"):
        return "time1 / tem1"
    if "_blocks." not in launch.module and not launch.module.startswith("mid_block."):
        return launch.op
    tag = "mid" if launch.module.startswith("mid_block.attentions") else f"L{launch.level + 1}"
    return f"{tag} {launch.op}"


def plan_shapes(B=B, s0=64):
    """(kind, name, count, spec) of every distinct GEMM / conv launch of one forward of B images (B / 2 frames with CFG)
    of s0 x s0 latents, SD-2.1 layout (default: W16@64²), from plan.launches.
    spec: plain {M, N, K1, K2, feats} / conv {n, H, W, Cin, Cout, mode, feats}."""
    shapes = {}
    for launch in launches(UNetConfig.sd21(), B // 2, s0, s0):
        if launch.kind != "attention":
            spec = dict(launch.spec, feats=launch.feats)
            key = (launch.kind, tuple(sorted(spec.items())))
            if key in shapes:
                shapes[key][2] += 1
            else:
                shapes[key] = [launch.kind, label(launch), 1, spec]
    return list(shapes.values())


OPERAND_WEIGHT = 128  # kOperandWeight of csrc/gemm_wgmma.cu
MIN_K_BLOCKS_256 = 16  # kMinKBlocks256
EPILOGUE_WEIGHT = 3072  # kEpilogueWeight
COOPERATIVE, PINGPONG = 1, 2  # kSchedCooperative, kSchedPingPong


def conv_tiles(rows, n, oh, ow):
    """Tiles per phase of a conv on an oh x ow output grid at `rows` positions per tile (conv_tile of csrc/gemm_wgmma.cu)."""
    bw = 16
    while bw > ow:
        bw >>= 1
    bh = rows // bw
    while bh > oh and bh > 1:
        bh >>= 1
    bn_img = rows // (bw * bh)
    return -(-ow // bw) * -(-oh // bh) * -(-n // bn_img)


def tile_cost(r, c, tiles, N, sms):
    """Cost of running `tiles` r x c tiles on `sms` SMs (gemm_choose_tile): waves x tile time + the padded columns."""
    n_tiles = -(-N // c)
    return -(-tiles // sms) * (r * c + OPERAND_WEIGHT * (r + c)) + (n_tiles * c - N) * (r // 2)


def pingpong_width(c, geglu):
    return c == 128 or (c == 64 and not geglu)


def plain_time(pingpong, c, M, N, K, sms):
    """gemm_choose_tile's time of the tiles an SM runs on either schedule: ping-pong overlaps each epilogue with the next
    tile's main loop."""
    per_sm = -(-(-(-M // 128) * -(-N // c)) // sms)
    main = -(-K // 64) * (128 * c + OPERAND_WEIGHT * (128 + c))
    epi = EPILOGUE_WEIGHT * c
    return per_sm * max(main, epi) + min(main, epi) if pingpong else per_sm * (main + epi)


def auto_tile(N, sms, M=0, geglu=False, conv=None, K=0):
    """Mirror of gemm_choose_tile (csrc/gemm_wgmma.cu): the (rows, width) of an automatic launch.  conv = (n, H, W, Cin, mode)
    with mode "s1" / "s2" / "up" on the H x W input; else a plain GEMM of M rows and K = K1 + K2 columns, for which the
    schedule (COOPERATIVE or PINGPONG) comes third."""
    if not conv:
        coop = _best_tile(N, sms, M=M, geglu=geglu)
        pp = _best_tile(N, sms, M=M, geglu=geglu, pingpong=True)
        if N % pp[1] == 0 and plain_time(True, pp[1], M, N, K, sms) < plain_time(False, coop[1], M, N, K, sms):
            return pp + (PINGPONG,)
        return coop + (COOPERATIVE,)
    return _best_tile(N, sms, conv=conv)


def _best_tile(N, sms, M=0, geglu=False, conv=None, pingpong=False):
    if conv:
        n, H, W, Cin, mode = conv
        oh, ow, phases = (H // 2, W // 2, 1) if mode == "s2" else (H, W, 4 if mode == "up" else 1)
        k_blocks = (4 if mode == "up" else 9) * -(-Cin // 64)
    best = None
    for r in (128, 256) if conv else (128,):
        m_tiles = conv_tiles(r, n, oh, ow) * phases if conv else -(-M // r)
        for c in (64, 128, 160, 192, 256):
            if (geglu and c % 64) or (pingpong and not pingpong_width(c, geglu)):
                continue
            tiles = m_tiles * -(-N // c)
            if r == 256 and not (c in (128, 160) and tiles >= sms and k_blocks >= MIN_K_BLOCKS_256):
                continue
            cost = tile_cost(r, c, tiles, N, sms)
            if best is None or cost <= best[0]:
                best = (cost, r, c)
    return best[1], best[2]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return name, float(q[0]), float(q[1])
    except Exception:  # noqa: BLE001 - the tool may be missing; the numbers are then reported as unknown
        return name, float("nan"), float("nan")


def make_launch(kind, spec, dev):
    """A zero-argument callable that enqueues the launch, plus its executed FLOPs and compulsory bytes."""
    from diffuman4d_b200._lib import check, lib
    from diffuman4d_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(0)
    r = lambda *s: (torch.randn(*s, generator=g) * 0.5).to(torch.bfloat16).to(dev)
    stream = lambda: torch.cuda.current_stream().cuda_stream
    f = set(spec["feats"])
    if kind == "gemm":
        M, N, K1, K2 = spec["M"], spec["N"], spec["K1"], spec["K2"]
        geglu = "geglu" in f
        a, a2 = r(M, K1), (r(M, K2) if K2 else None)
        w = r(N, K1 + K2) * (K1 + K2) ** -0.5
        bias = torch.randn(N, generator=g).to(dev) if "bias" in f else None
        nout = N // 2 if geglu else N
        out = torch.empty(M, nout, device=dev, dtype=torch.bfloat16)
        res = r(M, N) if "residual" in f else None
        stats_rows = M // B if "stats" in f else 0  # rows per image
        stats = torch.zeros(B * N * 2, device=dev, dtype=torch.int64) if "stats" in f else None
        act = 1 if "act" in f else 0
        scale = 2.0 if "scale" in f else 1.0
        p = lambda t: None if t is None else t.data_ptr()

        def run():
            check(lib().d4d_op_gemm(a.data_ptr(), K1, K1, p(a2), K2, K2, w.data_ptr(), M, N, p(bias), None, 0, 0, p(res),
                                    N if res is not None else 0, out.data_ptr(), nout, int(geglu), act, scale, 0,
                                    p(stats), stats_rows, stream()), "d4d_op_gemm")
        K = K1 + K2
        flops = 2.0 * M * N * K
        byts = 2.0 * (M * K + N * K + M * nout + (M * N if res is not None else 0))
        return run, flops, byts, auto_tile(N, torch.cuda.get_device_properties(0).multi_processor_count, M=M, geglu=geglu, K=K)
    n, H, W, Cin, Cout, mode = spec["n"], spec["H"], spec["W"], spec["Cin"], spec["Cout"], spec["mode"]
    x = r(n, H, W, Cin)
    bias = torch.randn(Cout, generator=g).to(dev) if "bias" in f else None
    stats = torch.zeros(n * Cout * 2, device=dev, dtype=torch.int64) if "stats" in f else None
    # pointers are taken inside run(), so that its closure keeps every tensor alive for as long as the launch is replayed
    p = lambda t: None if t is None else t.data_ptr()
    if mode == "up":
        taps, Mo = 4, n * 4 * H * W
        wp = torch.stack(ops.upsample_phase_weights(r(Cout, Cin, 3, 3) * (9 * Cin) ** -0.5)).contiguous()
        out = torch.empty(n, 2 * H, 2 * W, Cout, device=dev, dtype=torch.bfloat16)

        def run():
            check(lib().d4d_op_conv_resample(x.data_ptr(), n, H, W, Cin, wp.data_ptr(), Cout, p(bias), 3, 0, 0, out.data_ptr(),
                                             p(stats), stream()), "d4d_op_conv_resample")
    elif mode == "s2":
        taps, Mo = 9, n * (H // 2) * (W // 2)
        wt = r(Cout, 9, Cin) * (9 * Cin) ** -0.5
        out = torch.empty(n, H // 2, W // 2, Cout, device=dev, dtype=torch.bfloat16)

        def run():
            check(lib().d4d_op_conv_resample(x.data_ptr(), n, H, W, Cin, wt.data_ptr(), Cout, p(bias), 1, 0, 0, out.data_ptr(),
                                             p(stats), stream()), "d4d_op_conv_resample")
    else:
        taps, Mo = 9, n * H * W
        wt = r(Cout, 9, Cin) * (9 * Cin) ** -0.5
        out = torch.empty(n, H, W, Cout, device=dev, dtype=torch.bfloat16)
        rowvec = r(n, Cout) if "rowvec" in f else None
        res = r(n, H, W, Cout) if "residual" in f else None
        act = 1 if "act" in f else 0

        def run():
            check(lib().d4d_op_conv3x3(x.data_ptr(), n, H, W, Cin, wt.data_ptr(), Cout, p(bias), p(rowvec), Cout, p(res), act,
                                       out.data_ptr(), 0, p(stats), stream()),
                  "d4d_op_conv3x3")
    flops = 2.0 * Mo * Cout * taps * Cin
    byts = 2.0 * (x.numel() + taps * Cin * Cout + Mo * Cout * (2 if "residual" in f else 1))
    return run, flops, byts, auto_tile(Cout, torch.cuda.get_device_properties(0).multi_processor_count, conv=(n, H, W, Cin, mode)) + (0,)


def time_launch(run, reps):
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(reps):
            run()
    graph.replay()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    graph.replay()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="launches per timed graph replay")
    ap.add_argument("--json", default=None, help="also write the table as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_shapes.py needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power_w, max_mhz = card()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    peak = 4096.0 * sms * max_mhz * 1e6
    print(f"# {name}, power limit {power_w:.0f} W, max SM clock {max_mhz:.0f} MHz, {sms} SMs; "
          f"tensor peak {peak / 1e12:.0f} TFLOP/s (4096 FLOP/clk/SM at max clock), HBM 3.35 TB/s")
    hdr = f"{'kind':5} {'shape':58} {'cnt':>3} {'rows':>4} {'bn':>4} {'sched':>5} {'us':>9} {'TFLOP/s':>8} {'MB':>8} {'GB/s':>7} {'min us':>8} {'bound':>6} {'eff':>5}"
    print(hdr)
    rows, tot = [], {"gemm": 0.0, "conv": 0.0}
    for kind, nm, cnt, spec in plan_shapes():
        run, flops, byts, (bm, bn, sched) = make_launch(kind, spec, dev)
        sched_name = {0: "-", COOPERATIVE: "coop", PINGPONG: "pp"}[sched]
        us = time_launch(run, args.reps)
        t_f, t_b = flops / peak * 1e6, byts / HBM_BPS * 1e6
        bound = "tensor" if t_f >= t_b else "HBM"
        tmin = max(t_f, t_b)
        dims = (f"M{spec['M']} N{spec['N']} K{spec['K1']}" + (f"+{spec['K2']}" if spec["K2"] else "")) if kind == "gemm" else \
            f"{spec['n']}x{spec['H']}x{spec['W']} {spec['Cin']}->{spec['Cout']} {spec['mode']}"
        label = f"{nm}: {dims} [{','.join(spec['feats']) or '-'}]"
        print(f"{kind:5} {label:58} {cnt:3d} {bm:4d} {bn:4d} {sched_name:>5} {us:9.1f} {flops / us / 1e6:8.1f} {byts / 1e6:8.1f} "
              f"{byts / us / 1e3:7.0f} {tmin:8.1f} {bound:>6} {tmin / us:5.2f}")
        tot[kind] += cnt * us
        rows.append({"kind": kind, "name": nm, "spec": {k: (list(v) if isinstance(v, tuple) else v) for k, v in spec.items()},
                     "count": cnt, "block_m": bm, "block_n": bn, "schedule": sched_name, "us": us, "tflops": flops / us / 1e6, "bytes": byts,
                     "gbps": byts / us / 1e3, "min_us": tmin, "bound": bound})
        del run
        torch.cuda.empty_cache()
    print(f"# count-weighted per forward: gemm {tot['gemm'] / 1e3:.2f} ms, conv3x3 {tot['conv'] / 1e3:.2f} ms")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": name, "power_limit_w": power_w, "max_sm_mhz": max_mhz, "rows": rows,
                       "total_ms": {k: v / 1e3 for k, v in tot.items()}}, fh, indent=1)


if __name__ == "__main__":
    main()
