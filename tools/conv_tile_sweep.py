"""Tile sweep of the 3x3 convolutions of one W16@64² UNet forward: every conv shape of tools/gemm_shapes.py at every
explicit tile (rows, width) the kernel has, to see how the time of a launch follows the operand bytes its CTAs pull from L2
per FLOP.

    python tools/conv_tile_sweep.py [--reps 20] [--rounds 5] [--json OUT]
    python tools/conv_tile_sweep.py --list          # shapes and tiles only; needs no device

Tiles: 128 rows at every width of 64 / 128 / 160 / 256 that divides Cout, and 256 rows at 128 / 160.  Every launch goes
through the op-level C ABI (d4d_op_conv_tiled) with the epilogue features the plan gives it, `reps` times in a CUDA graph,
timed with CUDA events after warm-up; the tiles of one shape are timed in turn, `rounds` times over, so that a change of
clock hits them alike.  Per tile: median µs (and the range over the rounds), TFLOP/s, and the operand bytes per FLOP of a
k-block, (rows + bn)·128 B per rows·bn·64 multiply-adds = (rows + bn) / (rows·bn) B/FLOP.  `auto` marks the tile
gemm_prepare picks.  The SM clock, power draw and throttle reasons are sampled with nvidia-smi while the loop runs (read,
never set).

The last lines fit the tile-time model of gemm_choose_tile (csrc/gemm_wgmma.cu),
    µs = s · waves · k-blocks · (rows·bn + G·(rows + bn)),
by least squares over all tiles of the shapes with at least one tile per SM, and print G next to the kOperandWeight the
library uses.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import gemm_shapes  # noqa: E402

KIND = {"s1": 0, "s2": 1, "up": 3}
SMS_H100 = 132


def tiles_of(cout):
    """(rows, bn) of every explicit tile a conv with `cout` output channels can run at."""
    t = [(128, bn) for bn in (64, 128, 160, 256) if cout % bn == 0]
    return t + [(256, bn) for bn in (128, 160) if cout % bn == 0]


def conv_shapes():
    return [(nm, cnt, spec) for kind, nm, cnt, spec in gemm_shapes.plan_shapes() if kind == "conv" and tiles_of(spec["Cout"])]


def geometry(spec, rows, bn, sms):
    """k-blocks, tiles and SM-waves of a launch, and its executed FLOPs."""
    n, H, W, Cin, Cout, mode = (spec[k] for k in ("n", "H", "W", "Cin", "Cout", "mode"))
    oh, ow, phases, taps = (H // 2, W // 2, 1, 9) if mode == "s2" else (H, W, 4, 4) if mode == "up" else (H, W, 1, 9)
    tiles = gemm_shapes.conv_tiles(rows, n, oh, ow) * phases * (Cout // bn)
    return taps * -(-Cin // 64), tiles, -(-tiles // sms), 2.0 * n * oh * ow * phases * Cout * taps * Cin


def label(nm, spec):
    return f"{nm}: {spec['n']}x{spec['H']}x{spec['W']} {spec['Cin']}->{spec['Cout']} {spec['mode']}"


class ClockSampler:
    """SM clock / power draw / throttle reasons of GPU 0, sampled by one nvidia-smi process while the loop runs."""

    def __init__(self):
        self.samples = []
        self.proc = None

    def __enter__(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", "--query-gpu=clocks.sm,power.draw,clocks_throttle_reasons.active", "--format=csv,noheader,nounits",
                 "-i", "0", "-lms", "500"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=lambda: self.samples.extend(self.proc.stdout), daemon=True).start()
        except OSError:
            self.proc = None
        return self

    def __exit__(self, *exc):
        if self.proc is not None:
            self.proc.terminate()
            self.proc.wait()

    def summary(self):
        rows = [[f.strip() for f in ln.split(",")] for ln in self.samples if ln.count(",") == 2]
        if not rows:
            return "SM clock under load: not sampled (no nvidia-smi)"
        mhz = sorted(float(r[0]) for r in rows)
        watts = sorted(float(r[1]) for r in rows)
        reasons = sorted({r[2] for r in rows})
        return (f"SM clock under load {mhz[0]:.0f}-{mhz[-1]:.0f} MHz (median {mhz[len(mhz) // 2]:.0f}), power draw "
                f"{watts[0]:.0f}-{watts[-1]:.0f} W, throttle reasons {' '.join(reasons)}; {len(rows)} samples")


def make_conv(spec, rows, bn, dev):
    """A zero-argument callable that enqueues the conv at tile (rows, bn)."""
    import torch
    from diffuman4d_b200 import ops
    from diffuman4d_b200._lib import check, lib
    g = torch.Generator(device="cpu").manual_seed(0)
    r = lambda *s: (torch.randn(*s, generator=g) * 0.5).to(torch.bfloat16).to(dev)
    n, H, W, Cin, Cout, mode = (spec[k] for k in ("n", "H", "W", "Cin", "Cout", "mode"))
    f = set(spec["feats"])
    x = r(n, H, W, Cin)
    if mode == "up":
        wt = torch.stack(ops.upsample_phase_weights(r(Cout, Cin, 3, 3) * (9 * Cin) ** -0.5)).contiguous()
        oh, ow = 2 * H, 2 * W
    else:
        wt = r(Cout, 9, Cin) * (9 * Cin) ** -0.5
        oh, ow = (H // 2, W // 2) if mode == "s2" else (H, W)
    out = torch.empty(n, oh, ow, Cout, device=dev, dtype=torch.bfloat16)
    bias = torch.randn(Cout, generator=g).to(dev) if "bias" in f else None
    rowvec = r(n, Cout) if "rowvec" in f else None
    res = r(n, oh, ow, Cout) if "residual" in f else None
    stats = torch.zeros(n * Cout * 2, device=dev, dtype=torch.int64) if "stats" in f else None
    p = lambda t: None if t is None else t.data_ptr()

    def run():  # the closure owns every tensor: keep it for as long as a graph of the launch is replayed
        check(lib().d4d_op_conv_tiled(p(x), n, H, W, Cin, p(wt), Cout, p(bias), p(rowvec), Cout, p(res), int("act" in f), p(out),
                                      KIND[mode], rows, bn, p(stats), torch.cuda.current_stream().cuda_stream),
              "d4d_op_conv_tiled")
    return run


def graph_of(run, reps):
    import torch
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(reps):
            run()
    graph.replay()
    torch.cuda.synchronize()
    return graph


def time_graph(graph, reps):
    import torch
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    graph.replay()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) * 1e3 / reps


def auto_choice(spec, sms):
    from diffuman4d_b200._lib import check, lib
    bm, bn = ctypes.c_int(), ctypes.c_int()
    check(lib().d4d_conv_tile_choice(spec["n"], spec["H"], spec["W"], spec["Cin"], spec["Cout"], KIND[spec["mode"]], sms, ctypes.byref(bm),
                                     ctypes.byref(bn)), "d4d_conv_tile_choice")
    return bm.value, bn.value


def fit_operand_weight(results, sms):
    """Least squares of µs / (waves · k-blocks) on [rows·bn, rows + bn] over the launches that fill the SMs."""
    import numpy as np
    X, y = [], []
    for r in results:
        if r["tiles"] >= sms:
            X.append([r["rows"] * r["bn"], r["rows"] + r["bn"]])
            y.append(r["us"] / (r["waves"] * r["k_blocks"]))
    if len(X) < 3:
        return None
    X, y = np.asarray(X, float), np.asarray(y, float)
    coef = np.linalg.lstsq(X, y, rcond=None)[0]
    rel = np.abs(X @ coef - y) / y
    return {"G": float(coef[1] / coef[0]), "ns_per_mac_column": float(coef[0] * 1e3), "launches": len(y),
            "median_rel_err": float(np.median(rel)), "max_rel_err": float(rel.max())}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--reps", type=int, default=20, help="launches per timed graph replay")
    ap.add_argument("--rounds", type=int, default=5, help="timed replays per tile, the tiles of a shape taken in turn")
    ap.add_argument("--json", default=None, help="also write the table as JSON here")
    ap.add_argument("--list", action="store_true", help="print the shapes and their tiles, then stop (needs no device)")
    args = ap.parse_args()
    shapes = conv_shapes()
    if args.list:
        for nm, cnt, spec in shapes:
            auto = auto_choice(spec, SMS_H100)
            tl = " ".join(f"{r}x{bn}{'*' if (r, bn) == auto else ''}" for r, bn in tiles_of(spec["Cout"]))
            print(f"{label(nm, spec):48} x{cnt:2d}  tiles {tl}   (* automatic on {SMS_H100} SMs: {auto[0]}x{auto[1]})")
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("conv_tile_sweep.py needs a CUDA device to time anything (--list runs without one)")
    dev = torch.device("cuda:0")
    name, power_w, max_mhz = gemm_shapes.card()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"# {name}, power limit {power_w:.0f} W, max SM clock {max_mhz:.0f} MHz, {sms} SMs")
    print(f"{'shape':48} {'cnt':>3} {'rows':>4} {'bn':>4} {'B/FLOP':>8} {'FLOP/B':>7} {'waves':>5} {'us':>9} {'min..max':>17} {'TFLOP/s':>8}")
    results, total = [], {"auto": 0.0, "best": 0.0, "rows128": 0.0}
    with ClockSampler() as clock:
        for nm, cnt, spec in shapes:
            auto = auto_choice(spec, sms)
            # a graph holds raw pointers, and entering a capture empties the allocator's cache: the launches (and with them
            # their tensors) stay alive next to their graphs until the shape is done
            runs = [(t, make_conv(spec, *t, dev)) for t in tiles_of(spec["Cout"])]
            graphs = [(t, graph_of(run, args.reps)) for t, run in runs]
            times = {t: [] for t, _ in graphs}
            for _ in range(args.rounds):
                for t, gr in graphs:
                    times[t].append(time_graph(gr, args.reps))
            med = {t: statistics.median(v) for t, v in times.items()}
            for (rows, bn), v in times.items():
                kb, tiles, waves, flops = geometry(spec, rows, bn, sms)
                bpf = (rows + bn) / (rows * bn)
                us = med[(rows, bn)]
                print(f"{label(nm, spec):48} {cnt:3d} {rows:4d} {bn:4d} {bpf:8.5f} {1 / bpf:7.1f} {waves:5d} {us:9.1f} "
                      f"{min(v):8.1f}..{max(v):<7.1f} {flops / us / 1e6:8.1f}{'  auto' if (rows, bn) == auto else ''}")
                results.append({"name": nm, "spec": {k: (list(x) if isinstance(x, tuple) else x) for k, x in spec.items()},
                                "count": cnt, "rows": rows, "bn": bn, "us": us, "us_min": min(v), "us_max": max(v),
                                "tflops": flops / us / 1e6, "k_blocks": kb, "tiles": tiles, "waves": waves,
                                "auto": (rows, bn) == auto})
            total["auto"] += cnt * med[auto]
            total["best"] += cnt * min(med.values())
            total["rows128"] += cnt * min(us for (rows, _), us in med.items() if rows == 128)
            del graphs, gr, runs
            torch.cuda.empty_cache()
    print(f"# {clock.summary()}")
    print(f"# count-weighted per forward: automatic tiles {total['auto'] / 1e3:.2f} ms, best tile of each shape "
          f"{total['best'] / 1e3:.2f} ms, best 128-row tile of each shape {total['rows128'] / 1e3:.2f} ms")
    fit = fit_operand_weight(results, sms)
    if fit:
        print(f"# fit of us = s * waves * k-blocks * (rows*bn + G*(rows + bn)) over {fit['launches']} launches: G = {fit['G']:.0f} "
              f"(the library uses {gemm_shapes.OPERAND_WEIGHT}), s = {fit['ns_per_mac_column']:.4f} ns, relative error median "
              f"{fit['median_rel_err']:.3f}, max {fit['max_rel_err']:.3f}")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": name, "power_limit_w": power_w, "max_sm_mhz": max_mhz, "clock": clock.summary(), "rows": results,
                       "total_ms": {k: v / 1e3 for k, v in total.items()}, "fit": fit}, fh, indent=1)


if __name__ == "__main__":
    main()
