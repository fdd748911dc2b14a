"""Stacking on the GPU: the moment pass of the device linear fit (se_linear_moments) and a StackingRegressor fit and
transform on both routes.  Card name and power limit are read in the same process.

    python benchmarks/stacking_time.py [--rows 100000000] [--reps 5] [--stack-rows 10000000] [--out results.json]

Moment rows: X [p][n] and the label filled on the device (uniform, normal), every column in the list once, no weights
or bag; the time of one call (CUDA events around the launch, median of --reps after a warm-up) includes its small
uploads and the download of the (p+2)² matrix.  Bytes and flops are computed from the shapes: per row 4p + 4 bytes
read and (p+2)(p+3) flops for the upper triangle (one multiply and one add per entry).  Both are lower bounds of what
the kernels do: the tiled kernel (p + 2 > 8) computes whole 64×64 tiles.  The bounds divide them by the H100 SXM data
sheet's 3.35 TB/s of HBM3 and 34 TFLOP/s of fp64 (non-tensor: the kernels use FFMA64).

Stacking rows: host data [n, 32] (normal) with a linear-plus-sine label; members DeviceDecisionTreeRegressor(maxDepth
5), DeviceLinearRegression and GBMRegressor (5 rounds of depth-3 device trees, residentFeatures), stacker
DeviceLinearRegression; wall time of one fit and one transform after a warm-up at 100 000 rows, for
residentFeatures=True (device route) and False (host route: each member fits and predicts on its own)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from spark_ensemble_b200 import _native as N  # noqa: E402
from spark_ensemble_b200.context import Context  # noqa: E402
from spark_ensemble_b200.ensemble import DataFrame  # noqa: E402
from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor, DeviceLinearRegression  # noqa: E402
from spark_ensemble_b200.regression import GBMRegressor, StackingRegressor  # noqa: E402

HBM_BPS = 3.35e12
FP64_FLOPS = 34e12


def card(device=0):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(device)],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def moments(n, p, reps):
    with Context(0) as ctx:
        ctx.alloc(N.SLOT_X, p, n)
        ctx.fill_synthetic(N.SLOT_X, "uniform", 1, -1.0, 1.0)
        ctx.alloc(N.SLOT_Y, n)
        ctx.fill_synthetic(N.SLOT_Y, "normal", 2, 0.0, 1.0)
        cols = np.arange(p, dtype=np.int32)
        ctx.linear_moments(N.SLOT_X, cols, N.SLOT_Y)  # warm-up
        ts = []
        for _ in range(reps):
            ctx.timer_start()
            ctx.linear_moments(N.SLOT_X, cols, N.SLOT_Y)
            ts.append(ctx.timer_stop())
    ms = float(np.median(ts))
    nbytes, flops = n * (4 * p + 4), n * (p + 2) * (p + 3)
    bound_ms = 1e3 * max(nbytes / HBM_BPS, flops / FP64_FLOPS)
    return {"n": n, "p": p, "ms": ms, "ms_all": ts, "bytes": nbytes, "flops": flops,
            "GBps": nbytes / ms / 1e6, "GFLOPps": flops / ms / 1e6,
            "bound": "bytes" if nbytes / HBM_BPS >= flops / FP64_FLOPS else "flops", "bound_ms": bound_ms,
            "share_of_bound": bound_ms / ms}


def stacking(n, d=32, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d), dtype=np.float32)
    y = X[:, :8] @ rng.standard_normal(8) + np.sin(2 * X[:, 0]) + 0.1 * rng.standard_normal(n)
    gbm = GBMRegressor().setBaseLearner(DeviceDecisionTreeRegressor(maxDepth=3)).setNumBaseLearners(5) \
        .setResidentFeatures(True)
    est = StackingRegressor().setBaseLearners([DeviceDecisionTreeRegressor(maxDepth=5), DeviceLinearRegression(), gbm]) \
        .setStacker(DeviceLinearRegression())
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
                                                 "rmse": float(np.sqrt(np.mean((pred - y) ** 2)))}
    out.update(n=n, d=d)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--stack-rows", type=int, default=10_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "moments": [], "stacking": None}
    for p in (4, 32, 128):
        r = moments(a.rows, p, a.reps)
        res["moments"].append(r)
        print(json.dumps({k: v for k, v in r.items() if k != "ms_all"}), flush=True)
    res["stacking"] = stacking(a.stack_rows)
    print(json.dumps(res["stacking"]), flush=True)
    print(json.dumps({"card": res["card"]}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
