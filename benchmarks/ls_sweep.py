#!/usr/bin/env python
"""Line-search / fused-round variants on one GPU (experiment driver; not a bench line).

    python benchmarks/ls_sweep.py [--rows 50000000] [--loss bernoulli]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from spark_ensemble_b200 import _native as N  # noqa: E402
from spark_ensemble_b200.context import Context  # noqa: E402


def time_rounds(ctx, rounds, lr):
    for _ in range(2):
        ctx.gbm_round(lr, True, 1e-6, 100, residual=True)
    ctx.sync()
    ev = 0
    t0 = time.perf_counter()
    for _ in range(rounds):
        _, _, ne = ctx.gbm_round(lr, True, 1e-6, 100, residual=True)
        ev += ne
    ctx.sync()
    return 1e3 * (time.perf_counter() - t0) / rounds, ev / rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[50_000_000, 6_250_000])
    ap.add_argument("--loss", default="bernoulli")
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--squared-rows", type=int, nargs="+", default=[50_000_000, 25_000_000, 12_500_000, 6_250_000])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    ctx = Context(0)
    res = []
    print("persisting L2 max", ctx.get_option("l2_persist_max_bytes") / 1e6, "MB; window max",
          ctx.get_option("l2_window_max_bytes") / 1e6, "MB", flush=True)
    for n in args.rows:
        ctx.gbm_configure(n, 0, 1, args.loss, 0.0, False)
        ctx.fill_synthetic(N.SLOT_Y, "bernoulli", 1, 0.4, 1.0)
        ctx.fill(N.SLOT_F, 0.0)
        ctx.fill_synthetic(N.SLOT_H, "normal", 3, 0.0, 1.0)
        variants = [("per-eval launches (round 1)", dict(ls_mode=0)),
                    ("persistent", dict(ls_mode=1, l2_persist=0, ls_resident=1, ls_ctas_per_sm=4)),
                    ("persistent no-resident", dict(ls_mode=1, l2_persist=0, ls_resident=0, ls_ctas_per_sm=4)),
                    ("persistent 3 CTAs/SM", dict(ls_mode=1, l2_persist=0, ls_resident=1, ls_ctas_per_sm=3)),
                    ("persistent 2 CTAs/SM", dict(ls_mode=1, l2_persist=0, ls_resident=1, ls_ctas_per_sm=2)),
                    ("persistent + L2 persisting window (carve-out released after each search)",
                     dict(ls_mode=1, l2_persist=1, ls_resident=1, ls_ctas_per_sm=4))]
        for name, opts in variants:
            ctx.fill(N.SLOT_F, 0.0)
            for k, v in opts.items():
                ctx.set_option(k, v)
            ctx.kernel_timing(True)
            ctx.kernel_times_reset()
            ms, ev = time_rounds(ctx, args.rounds, 0.1)
            kt = ctx.kernel_times()
            ctx.kernel_timing(False)
            r = {"rows": n, "loss": args.loss, "variant": name, "ms_per_round": ms, "evals": ev,
                 "kernel_ms_per_round": {k: v["ms"] / (args.rounds + 2) for k, v in kt.items()},
                 "workers": ctx.get_option("last_ls_workers"), "hit_ratio": ctx.get_option("last_ls_hit_ratio")}
            res.append(r)
            print(json.dumps(r), flush=True)
    for n in args.squared_rows:
        ctx.gbm_configure(n, 0, 1, "squared", 0.0, False)
        ctx.fill_synthetic(N.SLOT_Y, "normal", 1, 0.0, 1.0)
        ctx.fill_synthetic(N.SLOT_H, "normal", 3, 0.0, 1.0)
        for name, opts in (("two launches + host Brent", dict(fused_round=0)),
                           ("one cooperative launch, no prefetch", dict(fused_round=1, fused_ctas_per_sm=3, fused_prefetch_mb=0)),
                           ("one cooperative launch, prefetch 32 MB", dict(fused_round=1, fused_ctas_per_sm=3, fused_prefetch_mb=32)),
                           ("one cooperative launch, prefetch 64 MB", dict(fused_round=1, fused_ctas_per_sm=3, fused_prefetch_mb=64)),
                           ("one cooperative launch, prefetch 96 MB", dict(fused_round=1, fused_ctas_per_sm=3, fused_prefetch_mb=96))):
            ctx.fill(N.SLOT_F, 0.0)
            ctx.gbm_pseudo_residuals(False)
            for k, v in opts.items():
                ctx.set_option(k, v)
            ms, ev = time_rounds(ctx, 50, 0.5)
            r = {"rows": n, "loss": "squared", "variant": name, "ms_per_round": ms, "evals": ev,
                 "gbs_28B_per_row": 28 * n / (ms * 1e-3) / 1e9}
            res.append(r)
            print(json.dumps(r), flush=True)
    ctx.close()
    if args.out:
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
