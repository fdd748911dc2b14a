"""The device logistic fit on the GPU: one se_logistic_loss_grad evaluation, a whole DeviceLogisticRegression fit, and
a StackingClassifier fit and transform with a logistic stacker on both routes.  Card name and power limit are read in
the same process.

    python benchmarks/logistic_time.py [--reps 10] [--out results.json]

Evaluation rows: X [p][n] and the label filled on the device (uniform features; Bernoulli labels for D = 1, uniform
class indices otherwise), no weights; the time of one call (CUDA events around it, median of --reps after a warm-up)
includes its small uploads and the download of the 1 + D(p+1) sums.  Bytes n·(4p + 4) and fp64 flops 4·n·D·(p+1)
(margins and gradient, one multiply and one add each) are computed from the shapes; the bound is the larger of bytes
over the H100 SXM data sheet's 3.35 TB/s of HBM3 and flops over its 34 TFLOP/s of fp64 (non-tensor: FFMA64).
Shapes: n = 100 M with D = 1 and p in {4, 32, 128}; n = 10 M with p = 104 and D = 26 (a letter-style raw stack).

Fit: DeviceLogisticRegression(regParam 0.01) on the same device-filled data (wall time, evaluations).  Stacking:
host data [n, 16] with 26 classes from a random linear model, members DeviceDecisionTreeClassifier(maxDepth 6) and
DeviceLogisticRegression, stackMethod "raw", stacker DeviceLogisticRegression; wall time of one fit and one transform
after a warm-up at 100 000 rows, for residentFeatures=True (device route) and False (host route)."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from benchmarks.stacking_time import FP64_FLOPS, HBM_BPS, card  # noqa: E402
from spark_ensemble_b200 import _native as N  # noqa: E402
from spark_ensemble_b200.classification import StackingClassifier  # noqa: E402
from spark_ensemble_b200.context import Context  # noqa: E402
from spark_ensemble_b200.ensemble import DataFrame  # noqa: E402
from spark_ensemble_b200.learners import DeviceDecisionTreeClassifier, DeviceLogisticRegression  # noqa: E402


def _fill(ctx, n, p, D):
    ctx.alloc(N.SLOT_X, p, n)
    ctx.fill_synthetic(N.SLOT_X, "uniform", 1, -1.0, 1.0)
    ctx.alloc(N.SLOT_Y, n)
    if D == 1:
        ctx.fill_synthetic(N.SLOT_Y, "bernoulli", 2, 0.4, 0.0)
    else:
        ctx.fill_synthetic(N.SLOT_Y, "randint", 2, 0.0, float(D))


def evaluation(n, p, D, reps):
    rng = np.random.default_rng(0)
    with Context(0) as ctx:
        _fill(ctx, n, p, D)
        cols = np.arange(p, dtype=np.int32)
        coef = rng.standard_normal((D, p + 1)) * 0.1
        ctx.logistic_loss_grad(N.SLOT_X, cols, coef, N.SLOT_Y)  # warm-up
        ts = []
        for _ in range(reps):
            ctx.timer_start()
            ctx.logistic_loss_grad(N.SLOT_X, cols, coef, N.SLOT_Y)
            ts.append(ctx.timer_stop())
        t0 = time.perf_counter()
        model = DeviceLogisticRegression(regParam=0.01).fit_resident(ctx, N.SLOT_X, cols, max(D, 2), N.SLOT_Y, 0, -1, 0)
        fit_s = time.perf_counter() - t0
    ms = float(np.median(ts))
    nbytes, flops = n * (4 * p + 4), 4 * n * D * (p + 1)
    bound = "bytes" if nbytes / HBM_BPS >= flops / FP64_FLOPS else "flops"
    bound_ms = 1e3 * max(nbytes / HBM_BPS, flops / FP64_FLOPS)
    return {"n": n, "p": p, "D": D, "ms": ms, "ms_all": ts, "bytes": nbytes, "flops": flops,
            "GBps": nbytes / ms / 1e6, "GFLOPps": flops / ms / 1e6, "bound": bound, "bound_ms": bound_ms,
            "share_of_bound": bound_ms / ms, "fit_s": fit_s, "fit_evaluations": model.numEvaluations}


def stacking(n, d=16, K=26, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d), dtype=np.float32)
    y = np.argmax(X @ rng.standard_normal((d, K)) + rng.gumbel(size=(n, K)), axis=1).astype(np.float64)
    est = StackingClassifier().setBaseLearners([DeviceDecisionTreeClassifier(maxDepth=6), DeviceLogisticRegression()]) \
        .setStacker(DeviceLogisticRegression()).setStackMethod("raw")
    out = {}
    for resident in (True, False):
        e = est.copy().setResidentFeatures(resident)
        e.fit(DataFrame(features=X[:100_000], label=y[:100_000]))  # warm-up
        t0 = time.perf_counter()
        model = e.fit(DataFrame(features=X, label=y))
        t1 = time.perf_counter()
        pred = model.transform(DataFrame(features=X))["prediction"]
        t2 = time.perf_counter()
        out["device" if resident else "host"] = {"fit_s": t1 - t0, "transform_s": t2 - t1,
                                                 "accuracy": float(np.mean(pred == y))}
    out.update(n=n, d=d, K=K)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--multi-rows", type=int, default=10_000_000)
    ap.add_argument("--stack-rows", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "evaluations": [], "stacking": None}
    for n, p, D in [(a.rows, 4, 1), (a.rows, 32, 1), (a.rows, 128, 1), (a.multi_rows, 104, 26)]:
        r = evaluation(n, p, D, a.reps)
        res["evaluations"].append(r)
        print(json.dumps({k: v for k, v in r.items() if k != "ms_all"}), flush=True)
    res["stacking"] = stacking(a.stack_rows)
    print(json.dumps(res["stacking"]), flush=True)
    print(json.dumps({"card": res["card"]}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
