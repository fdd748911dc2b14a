#!/usr/bin/env python
"""Persistent line search: cp.async ring depth x CTAs per SM (experiment driver).

    python benchmarks/ls_ring.py [--rows 50000000 6250000] [--loss bernoulli huber] [--out /tmp/ls_ring.json]
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
    ev, us = 0, 0.0
    alphas = []
    t0 = time.perf_counter()
    for _ in range(rounds):
        a, _, ne = ctx.gbm_round(lr, True, 1e-6, 100, residual=True)
        alphas.append(a)
        ev += ne
    ctx.sync()
    return 1e3 * (time.perf_counter() - t0) / rounds, ev / rounds, alphas


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[50_000_000, 6_250_000])
    ap.add_argument("--loss", nargs="+", default=["bernoulli", "huber"])
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    ctx = Context(0)
    res = []
    for loss in args.loss:
        for n in args.rows:
            ctx.gbm_configure(n, 0, 1, loss, 0.9 if loss == "huber" else 0.0, False)
            ctx.fill_synthetic(N.SLOT_Y, "bernoulli" if loss == "bernoulli" else "normal", 1, 0.4, 1.0)
            ctx.fill_synthetic(N.SLOT_H, "normal", 3, 0.0, 1.0)
            ref = None
            for ctas in (4, 3):
                for ring in (0, 2, 3, 4):  # 0 = register prefetch (the default)
                    ctx.fill(N.SLOT_F, 0.0)
                    ctx.gbm_pseudo_residuals(False)
                    ctx.set_option("ls_mode", 1)
                    ctx.set_option("ls_ctas_per_sm", ctas)
                    ctx.set_option("ls_ring", ring)
                    ms, ev, alphas = time_rounds(ctx, args.rounds, 0.1)
                    if ref is None:
                        ref = alphas
                    # per-pass time of one more round, from the in-kernel %globaltimer stamps
                    ctx.set_option("fused_timing", 1)
                    _, _, ne = ctx.gbm_round(0.1, True, 1e-6, 100, residual=True)
                    t_pass, t_fold = ctx.get_option("last_fused_stats_us"), ctx.get_option("last_fused_brent_us")
                    ctx.set_option("fused_timing", 0)
                    bpr = 8 if loss in ("bernoulli", "exponential") else 12
                    r = {"rows": n, "loss": loss, "ctas_per_sm": ctas, "ring": ring, "ms_per_round": ms, "evals": ev,
                         "us_per_pass": t_pass / max(ne, 1), "us_fold_per_pass": t_fold / max(ne, 1),
                         "pass_gbs": bpr * n / (t_pass / max(ne, 1) * 1e-6) / 1e9,
                         "workers": ctx.get_option("last_ls_workers"),
                         "alphas_identical_to_first_variant": alphas == ref}
                    res.append(r)
                    print(json.dumps(r), flush=True)
    ctx.close()
    if args.out:
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
