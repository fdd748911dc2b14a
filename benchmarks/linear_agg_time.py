#!/usr/bin/env python
"""Ensembles of linear and logistic members: se_linear_agg (one pass over the resident X) against the device member
route (se_logistic_predict per member into SLOT_P, then se_agg_run), and model.transform with residentFeatures True
(se_linear_agg) against False (members scored on the host, outputs uploaded, se_agg_run).

Kernel times are CUDA events on the context's stream around each route (X already resident, filled on the device),
median of --reps after a warm-up.  Bytes = 4 B x union columns x n + the outputs; fp64 FMAs = sum of D·p x n.  The bound
is the larger of bytes / 3.35 TB/s and FMAs / the H100 SXM data-sheet fp64 rate (33.5 TFLOP/s = 16.75 T FMA/s), both
for a card at 700 W: the card's name and power limit are read in the same process and printed with the numbers.
A member route that does not fit the card (its [M][K][n] SLOT_P) is reported as such.

    python benchmarks/linear_agg_time.py [--reps 5] [--rows 10000000,100000000] [--out /tmp/linear_agg.json]
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

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--rows", default="10000000,100000000")
ap.add_argument("--e2e-rows", type=int, default=10_000_000)
ap.add_argument("--out", default=None)
args = ap.parse_args()

HBM = 3.35e12
FP64_FMA = 33.5e12 / 2


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        q = "unknown"
    return q


def members(rng, M, d, D, ratio):
    p = max(1, int(round(ratio * d)))
    subs = [np.sort(rng.choice(d, p, replace=False)).astype(np.int32) for _ in range(M)]
    mem = [{"coef": rng.normal(0, 0.3, (D, p)), "intercept": rng.normal(0, 0.1, D), "threshold": 0.5} for _ in subs]
    return mem, subs


def median(ctx, fn, reps):
    fn()
    ctx.sync()
    ts = []
    for _ in range(reps):
        ctx.timer_start()
        fn()
        ts.append(ctx.timer_stop())
    return float(np.median(ts))


# (name, kind, K, M, D, subspaceRatio)
CASES = [
    ("bagging soft K=8", N.AGG_BAGGING_SOFT, 8, 10, 8, 0.5),
    ("bagging soft K=26", N.AGG_BAGGING_SOFT, 26, 10, 26, 0.5),
    ("SAMME.R K=8", N.AGG_BOOSTING_REAL, 8, 10, 8, 1.0),
    ("bagging regressor", N.AGG_BAGGING_REGRESSOR, 0, 10, 1, 0.5),
    ("boosting median M=10", N.AGG_BOOSTING_REG_MEDIAN, 0, 10, 1, 1.0),
    ("boosting median M=64", N.AGG_BOOSTING_REG_MEDIAN, 0, 64, 1, 1.0),
]


def kernel_case(ctx, n, d, case, rng):
    name, kind, K, M, D, ratio = case
    mem, subs = members(rng, M, d, D, ratio)
    w = rng.uniform(0.2, 1.0, M)
    width = K if kind in (N.AGG_BAGGING_SOFT, N.AGG_BOOSTING_REAL) else 1
    reg = kind in (N.AGG_BAGGING_REGRESSOR, N.AGG_BOOSTING_REG_MEDIAN)
    union = len(np.unique(np.concatenate(subs)))
    fmas = sum(D * len(s) for s in subs) * n
    out_bytes = 4 * n * (1 if reg else 2 * K + 1)
    nbytes = 4 * union * n + out_bytes
    bound = max(nbytes / HBM, fmas / FP64_FMA)
    if reg:
        ctx.alloc(N.SLOT_RAW, 1, n)

    def one():
        ctx.linear_agg(kind, K, mem, N.SLOT_RAW if reg else -1, weights=w, subspaces=subs)
    t1 = median(ctx, one, args.reps)
    res = {"case": name, "n": n, "d": d, "union_cols": union, "bytes": nbytes, "fp64_fma": fmas,
           "one_pass_ms": t1, "bound": "fp64" if fmas / FP64_FMA > nbytes / HBM else "hbm",
           "one_pass_share_of_bound": bound / (t1 * 1e-3)}
    free = int(__import__("torch").cuda.mem_get_info()[0])
    if 4 * M * width * n + 4 * 2 * max(K, 2) * n > free * 0.9:
        res["member_route_ms"] = None
        res["member_route"] = "SLOT_P of %.0f GB does not fit" % (4 * M * width * n / 1e9)
        return res

    def member():
        ctx.agg_configure(kind, M, K, 1, 0, n)
        for i, (mb, s) in enumerate(zip(mem, subs)):
            a = (mb["coef"], mb["intercept"], mb["threshold"])
            if reg:
                ctx.logistic_predict(*a, raw=(N.SLOT_PROBA, 0), subspace=s)
                ctx.copy_rows(N.SLOT_P, i, N.SLOT_PROBA, 1, 1)
            else:
                ctx.logistic_predict(*a, prob=(N.SLOT_P, i * K), subspace=s)
        ctx.agg_run(w)
    ctx.alloc(N.SLOT_PROBA, 2, n)
    res["member_route_ms"] = median(ctx, member, args.reps)
    res["speedup"] = res["member_route_ms"] / t1
    ctx.alloc(N.SLOT_P, 1, 32)
    ctx.alloc(N.SLOT_PROBA, 1, 32)
    return res


def e2e(n, rng):
    from spark_ensemble_b200 import learners as L
    from spark_ensemble_b200.classification import BaggingClassificationModel, BoostingClassificationModel
    from spark_ensemble_b200.regression import BaggingRegressionModel, BoostingRegressionModel
    d = 32
    X = rng.standard_normal((n, d), dtype=np.float32)
    out = []
    for name, kind, K, M, D, ratio in CASES:
        mem, subs = members(rng, M, d, D, ratio)
        if kind == N.AGG_BAGGING_SOFT:
            mods = [L.LogisticRegressionModel(m["coef"], m["intercept"], K, True) for m in mem]
            model = BaggingClassificationModel(K, subs, mods).setVotingStrategy("soft")
        elif kind == N.AGG_BOOSTING_REAL:
            mods = [L.LogisticRegressionModel(m["coef"], m["intercept"], K, True) for m in mem]
            model = BoostingClassificationModel(K, np.ones(M), mods).setAlgorithm("real")
        elif kind == N.AGG_BAGGING_REGRESSOR:
            mods = [L.LinearRegressionModel(m["coef"][0], m["intercept"][0]) for m in mem]
            model = BaggingRegressionModel(subs, mods)
        else:
            mods = [L.LinearRegressionModel(m["coef"][0], m["intercept"][0]) for m in mem]
            model = BoostingRegressionModel(rng.uniform(0.2, 1.0, M), mods).setVotingStrategy("median")
        df = DataFrame(features=X)
        t = {}
        for res in (True, False, True, False):  # alternated; the first of each is the warm-up
            model.set("residentFeatures", res)
            t0 = time.perf_counter()
            model.transform(df)
            t.setdefault(res, []).append(time.perf_counter() - t0)
        out.append({"case": name, "n": n, "d": d, "resident_s": t[True][-1], "host_s": t[False][-1],
                    "speedup": t[False][-1] / t[True][-1]})
        print(json.dumps(out[-1]), flush=True)
    return out


def main():
    rng = np.random.default_rng(0)
    info = {"card": card()}
    print(json.dumps(info), flush=True)
    kern = []
    for n in [int(v) for v in args.rows.split(",") if v]:
        for d in (32, 128):
            with Context(0) as ctx:
                ctx.alloc(N.SLOT_X, d, n)
                ctx.fill_synthetic(N.SLOT_X, "normal", 1, 0.0, 1.0)
                for case in CASES:
                    r = kernel_case(ctx, n, d, case, rng)
                    kern.append(r)
                    print(json.dumps(r), flush=True)
    ends = e2e(args.e2e_rows, rng) if args.e2e_rows else []
    if args.out:
        with open(args.out, "w") as f:
            json.dump({**info, "kernel": kern, "end_to_end": ends}, f, indent=1)


main()
