#!/usr/bin/env python
"""Per-kernel roofline sweep over the BASELINE.json configurations (single GPU shard sizes).

    python benchmarks/kernels.py [--quick] [--out /tmp/kernels.json]

Each line: kernel family, configuration, algorithmic bytes/row (SURVEY.md §8d), average launch duration from
CUDA events on the library stream (se_ctx_kernel_timing), achieved GB/s and fraction of the measured HBM peak."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from spark_ensemble_b200 import _native as N  # noqa: E402
from spark_ensemble_b200.context import Context  # noqa: E402


def peak():
    try:
        return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        return 6650.0


def timed(ctx, family, fn, reps=10, warm=2):
    for _ in range(warm):
        fn()
    ctx.sync()
    ctx.kernel_timing(True)
    ctx.kernel_times_reset()
    for _ in range(reps):
        fn()
    kt = ctx.kernel_times()[family]
    ctx.kernel_timing(False)
    return kt["ms"] / kt["launches"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--out", default=None)
    ap.add_argument("--only", default="", help="comma list of sections: scalar,logloss,boost,agg (default: all)")
    args = ap.parse_args()
    only = set(x for x in args.only.split(",") if x)
    want = lambda sec: not only or sec in only
    scale = 0.1 if args.quick else 1.0
    pk = peak()
    ctx = Context(0)
    rows = []

    def rec(name, cfg, n, bpr, ms):
        gbs = bpr * n / (ms * 1e-3) / 1e9
        rows.append({"kernel": name, "config": cfg, "rows": n, "bytes_per_row": bpr, "ms": ms,
                     "rows_per_s": n / (ms * 1e-3), "achieved_gbs": gbs, "frac_of_measured_peak": gbs / pk})
        print(f"{name:34s} {cfg:38s} n={n:>11d} {bpr:5d} B/row {ms:9.4f} ms {gbs:8.1f} GB/s {gbs / pk:6.3f}", flush=True)

    # ---- GBM scalar losses
    for loss, n in () if not want("scalar") else (("squared", int(10e6)), ("squared", int(100e6 * scale)), ("bernoulli", int(50e6 * scale)),
                    ("exponential", int(50e6 * scale)), ("absolute", int(50e6 * scale)), ("logcosh", int(50e6 * scale))):
        ctx.gbm_configure(n, 0, 1, loss, 0.9, False)
        if loss in ("bernoulli", "exponential"):
            ctx.fill_synthetic(N.SLOT_Y, "bernoulli", 1, 0.4, 0)
        else:
            ctx.fill_synthetic(N.SLOT_Y, "normal", 1, 0, 1)
        ctx.fill_synthetic(N.SLOT_F, "normal", 2, 0, 0.5)
        ctx.fill_synthetic(N.SLOT_H, "normal", 3, 0, 1)
        cfg = f"{loss} dim=1"
        rec("K2 linesearch_eval", cfg, n, 12, timed(ctx, "eval", lambda: ctx.gbm_linesearch_eval([0.7])))
        if loss == "squared":
            rec("K2 sq_stats", cfg, n, 12, timed(ctx, "sq_stats", lambda: ctx.gbm_linesearch_stats()))
        rec("K1 update+resid+loss", cfg, n, 20, timed(ctx, "update", lambda: ctx.gbm_update([1e-3], residual=True, loss=True)))
        rec("pseudo_residuals", cfg, n, 12, timed(ctx, "resid", lambda: ctx.gbm_pseudo_residuals(False)))
        if loss in ("squared", "bernoulli"):
            rec("K1 newton (r, w', S)", cfg, n, 24, timed(ctx, "update", lambda: ctx.gbm_update([1e-3], newton=True, loss=True)))

    # ---- LogLoss(K)
    for K, n in () if not want("logloss") else ((2, int(50e6 * scale)), (8, int(20e6 * scale)), (16, int(10e6 * scale)),
                                                (26, int(10e6 * scale))):
        ctx.gbm_configure(n, 0, K, "logloss", 0.0, False)
        ctx.fill_synthetic(N.SLOT_Y, "randint", 1, 0, K)
        ctx.fill_synthetic(N.SLOT_F, "normal", 2, 0, 0.5)
        ctx.fill_synthetic(N.SLOT_H, "normal", 3, 0, 1)
        cfg = f"logloss K={K}"
        rec("K2 linesearch_eval", cfg, n, 4 * (2 * K + 1), timed(ctx, "eval", lambda: ctx.gbm_linesearch_eval(np.full(K, 0.7))))
        rec("K1 update+resid+loss", cfg, n, 4 * (4 * K + 1),
            timed(ctx, "update", lambda: ctx.gbm_update(np.full(K, 1e-3), residual=True, loss=True)))
        rec("pseudo_residuals", cfg, n, 4 * (2 * K + 1), timed(ctx, "resid", lambda: ctx.gbm_pseudo_residuals(False)))
        rec("K1 newton (r, w', S)", cfg, n, 4 * (5 * K + 1),
            timed(ctx, "update", lambda: ctx.gbm_update(np.full(K, 1e-3), newton=True, loss=True)))
    for s in (N.SLOT_F, N.SLOT_H, N.SLOT_R, N.SLOT_WOUT):
        ctx.free(s)

    if want("boost"):
        # ---- SAMME.R / SAMME (config 4: K = 26)
        K, n = 26, int(100e6 * scale)
        ctx.boost_configure(n, K, True)
        ctx.fill_synthetic(N.SLOT_Y, "randint", 1, 0, K)
        ctx.fill_synthetic(N.SLOT_PROBA, "uniform", 2, 0.001, 0.08)
        def samme_r():
            ctx.fill(N.SLOT_BW, 1.0)
            ctx.boost_real_update(float(n))
        rec("K3 SAMME.R update", f"K={K}", n, 4 * K + 12, timed(ctx, "boost_real", samme_r, reps=5))
        ctx.free(N.SLOT_PROBA)
        ctx.boost_configure(n, K, False)
        ctx.fill_synthetic(N.SLOT_PRED, "randint", 3, 0, K)
        ctx.fill(N.SLOT_BW, 1.0)
        rec("K3' SAMME error", f"K={K}", n, 12, timed(ctx, "boost_err", lambda: ctx.boost_discrete_error(float(n))))
        rec("K3' SAMME update", f"K={K}", n, 16, timed(ctx, "boost_upd", lambda: ctx.boost_discrete_update(1.0, 1.0)))

    if want("agg"):
        # ---- aggregation (config 5: M = 512)
        for kind, name, M, K, n in ((N.AGG_BAGGING_REGRESSOR, "bagging mean", 512, 0, int(6.25e6 * scale)),
                                    (N.AGG_GBM_REGRESSOR, "gbm weighted sum", 512, 0, int(6.25e6 * scale)),
                                    (N.AGG_GBM_REGRESSOR, "gbm weighted sum", 100, 0, int(25e6 * scale)),
                                    (N.AGG_BOOSTING_REAL, "boosting real", 10, 26, int(10e6 * scale)),
                                    (N.AGG_BAGGING_HARD, "bagging hard vote", 64, 26, int(10e6 * scale)),
                                    (N.AGG_BAGGING_SOFT, "bagging soft vote", 16, 26, int(10e6 * scale)),
                                    (N.AGG_BAGGING_SOFT, "bagging soft vote", 64, 2, int(25e6 * scale)),
                                    (N.AGG_BOOSTING_DISCRETE, "boosting discrete", 64, 26, int(10e6 * scale)),
                                    (N.AGG_BOOSTING_REG_MEDIAN, "weighted median", 32, 0, int(25e6 * scale))):
            ctx.agg_configure(kind, M, max(K, 2), 1, 0, n)
            if kind in (N.AGG_BAGGING_HARD, N.AGG_BOOSTING_DISCRETE):
                ctx.fill_synthetic(N.SLOT_P, "randint", 5, 0, K)
            else:
                ctx.fill_synthetic(N.SLOT_P, "uniform", 5, 0.01, 1.0)
            w = np.full(M, 1.0 / M)
            if kind == N.AGG_BOOSTING_REG_MEDIAN:
                w = np.linspace(0.5, 1.5, M)   # distinct estimator weights (log 1/beta): the margin-checked fast path
            width = K if kind in (N.AGG_BOOSTING_REAL, N.AGG_BAGGING_SOFT) else 1
            C = K if K else 1
            regr = kind in (N.AGG_GBM_REGRESSOR, N.AGG_BAGGING_REGRESSOR, N.AGG_BOOSTING_REG_MEDIAN)
            bpr = 4 * M * width + (4 * C if regr else 4 * (2 * C + 1))  # classifiers write raw, prob [C] and the label
            rec("K4 aggregation", f"{name} M={M}" + (f" K={K}" if K else ""), n, bpr,
                timed(ctx, "agg", lambda: ctx.agg_run(w if kind in (N.AGG_GBM_REGRESSOR, N.AGG_BOOSTING_DISCRETE,
                                                                   N.AGG_BOOSTING_REG_MEDIAN) else None, [0.1]), reps=5))
    ctx.close()
    if args.out:
        json.dump({"peak_gbs": pk, "rows": rows}, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
