"""Schedule sweep of the plain GEMMs of one UNet forward: every plain GEMM shape of tools/gemm_shapes.py at every explicit
(schedule, width) the kernel has, to see where the ping-pong schedule (one MMA warpgroup per tile, epilogue under the other
warpgroup's MMAs) beats the cooperative one (both warpgroups on one tile, epilogue after the MMAs) and by how much.

    python tools/gemm_schedule_sweep.py [--plan W16@64] [--reps 20] [--rounds 5] [--json OUT]
    python tools/gemm_schedule_sweep.py --list          # shapes and candidates only; needs no device

Candidates: cooperative at every width of 64 / 128 / 160 / 192 / 256 that divides N (GEGLU: 64 / 128 / 256), ping-pong at
64 / 128 (GEGLU: 128), and the automatic launch (which may overhang the last N tile).  Every launch goes through the op-level
C ABI (d4d_op_gemm_tiled) with the epilogue features the plan gives it, `reps` times in a CUDA graph, timed with CUDA events
after warm-up; the candidates of one shape are timed in turn, `rounds` times over, so that a change of clock hits them
alike.  Per candidate: median µs and the range over the rounds.  `auto` marks what gemm_prepare picks, `best` the fastest.

The last lines give the count-weighted time per forward of the automatic launches, of the best candidate of each shape and
of the best cooperative candidate, and the time the picks of gemm_choose_tile's model would take at other epilogue weights
(kEpilogueWeight), read from the measured table.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import gemm_shapes  # noqa: E402
from conv_tile_sweep import ClockSampler, graph_of, time_graph  # noqa: E402

SMS_H100 = 132
PLANS = {"W16@64": (32, 64), "W24@64": (48, 64), "W16@128": (32, 128)}
NAMES = {0: "auto", gemm_shapes.COOPERATIVE: "coop", gemm_shapes.PINGPONG: "pp"}


def candidates(spec):
    """(schedule, bn) of every explicit launch of a plain GEMM, then the automatic one (0, 0)."""
    N, geglu = spec["N"], "geglu" in spec["feats"]
    out = [(gemm_shapes.COOPERATIVE, c) for c in (64, 128, 160, 192, 256) if N % c == 0 and not (geglu and c % 64)]
    out += [(gemm_shapes.PINGPONG, c) for c in (64, 128) if N % c == 0 and gemm_shapes.pingpong_width(c, geglu)]
    return out + [(0, 0)]


def gemm_plan(plan):
    return [(nm, cnt, spec) for kind, nm, cnt, spec in gemm_shapes.plan_shapes(*PLANS[plan]) if kind == "gemm"]


def label(nm, spec):
    return f"{nm}: M{spec['M']} N{spec['N']} K{spec['K1']}" + (f"+{spec['K2']}" if spec["K2"] else "") + \
        f" [{','.join(spec['feats']) or '-'}]"


def auto_choice(spec, sms):
    from diffuman4d_b200._lib import check, lib
    bn, sched = ctypes.c_int(), ctypes.c_int()
    check(lib().d4d_gemm_tile_choice(spec["M"], spec["N"], spec["K1"], spec["K2"], int("geglu" in spec["feats"]), sms,
                                     ctypes.byref(bn), ctypes.byref(sched)), "d4d_gemm_tile_choice")
    return sched.value, bn.value


def make_gemm(spec, n_img, sched, bn, dev):
    """A zero-argument callable that enqueues the GEMM at (schedule, width); (0, 0) is the automatic launch."""
    import torch
    from diffuman4d_b200._lib import check, lib
    g = torch.Generator(device="cpu").manual_seed(0)
    r = lambda *s: (torch.randn(*s, generator=g) * 0.5).to(torch.bfloat16).to(dev)
    M, N, K1, K2 = spec["M"], spec["N"], spec["K1"], spec["K2"]
    f = set(spec["feats"])
    geglu = "geglu" in f
    a, a2 = r(M, K1), (r(M, K2) if K2 else None)
    w = r(N, K1 + K2) * (K1 + K2) ** -0.5
    bias = torch.randn(N, generator=g).to(dev) if "bias" in f else None
    nout = N // 2 if geglu else N
    out = torch.empty(M, nout, device=dev, dtype=torch.bfloat16)
    res = r(M, N) if "residual" in f else None
    stats_rows = M // n_img if "stats" in f else 0  # rows per image
    stats = torch.zeros(n_img * N * 2, device=dev, dtype=torch.int64) if "stats" in f else None
    p = lambda t: None if t is None else t.data_ptr()

    def run():  # the closure owns every tensor: keep it for as long as a graph of the launch is replayed
        check(lib().d4d_op_gemm_tiled(p(a), K1, K1, p(a2), K2, K2, p(w), M, N, p(bias), None, 0, 0, p(res),
                                      N if res is not None else 0, p(out), nout, int(geglu), int("act" in f),
                                      2.0 if "scale" in f else 1.0, bn, sched, p(stats), stats_rows,
                                      torch.cuda.current_stream().cuda_stream), "d4d_op_gemm_tiled")
    return run


def model_total(results, weight, sms):
    """Count-weighted µs per forward if gemm_choose_tile used epilogue weight `weight`: its pick, read from the table (shapes
    whose pick was not timed are skipped, and counted)."""
    saved = gemm_shapes.EPILOGUE_WEIGHT
    gemm_shapes.EPILOGUE_WEIGHT = weight
    total, missing = 0.0, 0
    try:
        for spec, cnt, times in results:
            bm, bn, sched = gemm_shapes.auto_tile(spec["N"], sms, M=spec["M"], geglu="geglu" in spec["feats"],
                                                  K=spec["K1"] + spec["K2"])
            if (sched, bn) in times:
                total += cnt * times[(sched, bn)]
            else:
                missing += 1
    finally:
        gemm_shapes.EPILOGUE_WEIGHT = saved
    return total, missing


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--plan", default="W16@64", choices=list(PLANS) + ["all"])
    ap.add_argument("--reps", type=int, default=20, help="launches per timed graph replay")
    ap.add_argument("--rounds", type=int, default=5, help="timed replays per candidate, the candidates of a shape taken in turn")
    ap.add_argument("--json", default=None, help="also write the table as JSON here")
    ap.add_argument("--list", action="store_true", help="print the shapes and their candidates, then stop (needs no device)")
    args = ap.parse_args()
    plans = list(PLANS) if args.plan == "all" else [args.plan]
    if args.list:
        for plan in plans:
            for nm, cnt, spec in gemm_plan(plan):
                auto = auto_choice(spec, SMS_H100)
                c = " ".join(f"{NAMES[s]}{bn}" for s, bn in candidates(spec)[:-1])
                print(f"{plan:8} {label(nm, spec):66} x{cnt:2d}  {c}   (automatic on {SMS_H100} SMs: {NAMES[auto[0]]}{auto[1]})")
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("gemm_schedule_sweep.py needs a CUDA device to time anything (--list runs without one)")
    dev = torch.device("cuda:0")
    name, power_w, max_mhz = gemm_shapes.card()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"# {name}, power limit {power_w:.0f} W, max SM clock {max_mhz:.0f} MHz, {sms} SMs")
    out = {"card": name, "power_limit_w": power_w, "max_sm_mhz": max_mhz, "plans": {}}
    with ClockSampler() as clock:
        for plan in plans:
            print(f"## {plan}")
            print(f"{'shape':66} {'cnt':>3} {'sched':>5} {'bn':>4} {'us':>9} {'min..max':>17}")
            rows, measured, total = [], [], {"auto": 0.0, "best": 0.0, "best_coop": 0.0}
            for nm, cnt, spec in gemm_plan(plan):
                auto = auto_choice(spec, sms)
                runs = [(t, make_gemm(spec, PLANS[plan][0], *t, dev)) for t in candidates(spec)]
                graphs = [(t, graph_of(run, args.reps)) for t, run in runs]
                times = {t: [] for t, _ in graphs}
                for _ in range(args.rounds):
                    for t, gr in graphs:
                        times[t].append(time_graph(gr, args.reps))
                med = {t: statistics.median(v) for t, v in times.items()}
                best = min((t for t in med if t != (0, 0)), key=med.get)
                for (sched, bn), v in times.items():
                    tag = "  auto" if (sched, bn) == auto else ""
                    tag += "  best" if (sched, bn) == best else ""
                    shown = f"{NAMES[auto[0]]}{auto[1]}" if sched == 0 else f"{NAMES[sched]}{bn}"
                    print(f"{label(nm, spec):66} {cnt:3d} {NAMES[sched]:>5} {bn:4d} {med[(sched, bn)]:9.1f} "
                          f"{min(v):8.1f}..{max(v):<7.1f}{tag if sched else '  = ' + shown}")
                    rows.append({"name": nm, "spec": {k: (list(x) if isinstance(x, tuple) else x) for k, x in spec.items()},
                                 "count": cnt, "schedule": NAMES[sched], "bn": bn, "us": med[(sched, bn)], "us_min": min(v),
                                 "us_max": max(v), "auto": [NAMES[auto[0]], auto[1]]})
                total["auto"] += cnt * med[(0, 0)]
                total["best"] += cnt * med[best]
                total["best_coop"] += cnt * min(us for (s, _), us in med.items() if s == gemm_shapes.COOPERATIVE)
                timed = dict(med)
                timed[auto] = med[(0, 0)]
                measured.append((spec, cnt, timed))
                del graphs, gr, runs
                torch.cuda.empty_cache()
            print(f"# {plan} count-weighted per forward: automatic {total['auto'] / 1e3:.3f} ms, best candidate of each shape "
                  f"{total['best'] / 1e3:.3f} ms, best cooperative candidate {total['best_coop'] / 1e3:.3f} ms")
            model = {}
            for wgt in (0, 512, 1024, 2048, 3072, 4096, 6144, 8192, 12288, 16384, 1 << 30):
                t, miss = model_total(measured, wgt, sms)
                model[wgt] = (t / 1e3, miss)
            print(f"# {plan} model picks at epilogue weight w (ms per forward, picks not timed): " +
                  ", ".join(f"w={w}: {t:.3f} ({m})" for w, (t, m) in model.items()))
            out["plans"][plan] = {"rows": rows, "total_ms": {k: v / 1e3 for k, v in total.items()}, "model_ms": model}
    print(f"# {clock.summary()}")
    out["clock"] = clock.summary()
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
