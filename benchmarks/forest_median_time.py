#!/usr/bin/env python
"""BoostingRegressionModel's weighted median over tree members: the one-pass route (se_forest_median: every tree walked
and every row's median taken on chip) against the member route it replaces (se_tree_predict per member into the
[M][n] SLOT_P, then se_agg_run(AGG_BOOSTING_REG_MEDIAN)).  Both routes run alternately in one process on the same
synthetic depth-6 forests, with X already resident for the kernel times (CUDA events) and from the host array for the
transform wall times (each route uploads X once).  Also times a BoostingRegressor fit with
DeviceDecisionTreeRegressor(maxDepth=5): the resident route (trees fitted on the device-resident weights) against
residentFeatures=False (learner.fit per round on the downloaded weights), in rounds/s.

    python benchmarks/forest_median_time.py [--reps 3] [--sizes 10000000,50000000] [--out /tmp/forest_median.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from spark_ensemble_b200 import DataFrame  # noqa: E402
from spark_ensemble_b200 import _native as N  # noqa: E402
from spark_ensemble_b200.context import Context  # noqa: E402
from spark_ensemble_b200.learners import DeviceDecisionTreeRegressionModel, DeviceDecisionTreeRegressor  # noqa: E402
from spark_ensemble_b200.regression import BoostingRegressionModel, BoostingRegressor, _resident_context  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--sizes", default="10000000,50000000")
ap.add_argument("--trees", default="10,32,64")
ap.add_argument("--fit-rows", type=int, default=10_000_000)
ap.add_argument("--fit-rounds", type=int, default=5)
ap.add_argument("--out", default=None)
args = ap.parse_args()
D, DEPTH = 32, 6


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        pl = "unknown"
    return name, pl


def tree(rng, depth, d, cands):
    n_int, n = 2 ** depth - 1, 2 ** (depth + 1) - 1
    f = np.full(n, -1, np.int32)
    c = rng.integers(0, d, n_int)
    f[:n_int] = c
    t = np.zeros(n, np.float32)
    t[:n_int] = cands[c, rng.integers(0, cands.shape[1], n_int)]
    l = np.zeros(n, np.int32)
    r = np.zeros(n, np.int32)
    l[:n_int] = 2 * np.arange(n_int) + 1
    r[:n_int] = 2 * np.arange(n_int) + 2
    return {"feature": f, "threshold": t, "left": l, "right": r, "value": rng.standard_normal(n).astype(np.float32)}


def forest(seed, M, depth, d):
    rng = np.random.default_rng(seed)
    cands = np.sort(rng.standard_normal((d, 31)), axis=1).astype(np.float32)  # maxBins 32
    return [tree(rng, depth, d, cands) for _ in range(M)]


def member_route(ctx, trees, w, n):
    ctx.agg_configure(N.AGG_BOOSTING_REG_MEDIAN, len(trees), 0, 1, 0, n)
    for i, t in enumerate(trees):
        ctx.tree_predict(t, N.SLOT_P, i)
    ctx.agg_run(w)


def member_transform(X, trees, w):
    """The member route end to end, as BoostingRegressionModel took it before the one-pass kernel."""
    with _resident_context(0, X) as ctx:
        member_route(ctx, trees, w, X.shape[0])
        return ctx.download(N.SLOT_RAW).astype(np.float64)


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return 1e3 * (time.perf_counter() - t0), out


name, power = card()
res = {"card": name, "power_limit": power, "runs": []}
for n in [int(s) for s in args.sizes.split(",")]:
    X = np.random.default_rng(n).standard_normal((n, D), dtype=np.float32)
    df = DataFrame(features=X)
    for M in [int(s) for s in args.trees.split(",")]:
        trees = forest(M, M, DEPTH, D)
        w = np.random.default_rng(M + 1).uniform(0.1, 1.0, M)
        # kernel times, X resident, the two routes alternated in one context
        with Context(0) as ctx:
            ctx.alloc(N.SLOT_X, D, n)
            ctx.upload_rowmajor(N.SLOT_X, X)
            ctx.alloc(N.SLOT_H, 1, n)
            ctx.forest_median(trees, N.SLOT_H, w)  # warm-up: ranks the columns, sizes the buffers
            member_route(ctx, trees, w, n)
            ctx.sync()
            one = ctx.download(N.SLOT_H)
            same = bool(np.array_equal(one.view(np.uint32), ctx.download(N.SLOT_RAW).view(np.uint32)))
            chunks = ctx.get_option("last_forest_chunks")
            ctx.kernel_timing(True)
            k1, k2, c1, c2 = [], [], [], []

            def kernels(fn):  # (Σ of the call's kernel times, the call's event window) in ms
                ctx.kernel_times_reset()
                ctx.timer_start()
                fn()
                window = ctx.timer_stop()
                return sum(v["ms"] for v in ctx.kernel_times().values()), window

            for _ in range(args.reps):
                k, c = kernels(lambda: ctx.forest_median(trees, N.SLOT_H, w))
                k1.append(k)
                c1.append(c)
                k, c = kernels(lambda: member_route(ctx, trees, w, n))
                k2.append(k)
                c2.append(c)
            ctx.kernel_timing(False)
        model = BoostingRegressionModel(w, [DeviceDecisionTreeRegressionModel(t) for t in trees]).setResidentFeatures(True)
        model.transform(df)  # warm-up
        t1, t2 = [], []
        for _ in range(args.reps):  # alternated
            ms, a = timed(lambda: model.transform(df)["prediction"])
            t1.append(ms)
            ms, b = timed(lambda: member_transform(X, trees, w))
            t2.append(ms)
            same = same and bool(np.array_equal(a, b))
        row = {"n": n, "d": D, "trees": M, "depth": DEPTH, "chunks": chunks, "bit_identical": same,
               "one_pass_kernel_ms": min(k1), "member_kernels_ms": min(k2),
               "one_pass_call_ms": min(c1), "member_calls_ms": min(c2),
               "one_pass_transform_ms": min(t1), "member_transform_ms": min(t2),
               "member_matrix_bytes_not_moved": 2 * 4 * M * n}  # [M][n] fp32 written and read back
        res["runs"].append(row)
        print(json.dumps(row), flush=True)
    del X, df

# BoostingRegressor fit: device tree on the resident weights vs learner.fit per round
n = args.fit_rows
rng = np.random.default_rng(7)
X = rng.standard_normal((n, D), dtype=np.float32)
y = (np.sin(2 * X[:, 0]) + X[:, 1] * X[:, 2] + 0.5 * rng.standard_normal(n, dtype=np.float32)).astype(np.float64)
df = DataFrame(features=X, label=y)
for resident in (True, False, True, False):
    est = (BoostingRegressor().setBaseLearner(DeviceDecisionTreeRegressor(maxDepth=5)).setLossType("linear")
           .setNumBaseLearners(args.fit_rounds).setResidentFeatures(resident))
    ms, m = timed(lambda: est.fit(df))
    rounds = len(m.trainingHistory)
    row = {"fit": "BoostingRegressor", "n": n, "d": D, "maxDepth": 5, "resident": resident, "rounds": rounds,
           "fit_ms": ms, "rounds_per_s": rounds / (ms / 1e3)}
    res["runs"].append(row)
    print(json.dumps(row), flush=True)
print(json.dumps({"card": name, "power_limit": power}))
if args.out:
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)
