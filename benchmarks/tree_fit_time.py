"""Device regression-tree fit (se_tree_fit): CUDA-event times per level and per tree, achieved bytes/s against the
byte model of DESIGN.md §3 "Device tree fit", and GBM rounds/s with the device learner against the host learner.
With --classes K, the same for the classification-tree fit (se_tree_fit_classifier, weighted, --impurity gini or
entropy) and BoostingClassifier (SAMME) rounds/s with the device learner against the host learner.

    python benchmarks/tree_fit_time.py [--rows 100000000] [--cols 128] [--gbm-rows 10000000] [--host-rows 1000000]
    python benchmarks/tree_fit_time.py --classes 26 [--impurity gini] [--rows ...] [--gbm-rows ...] [--host-rows ...]
    python benchmarks/tree_fit_time.py --devices 0,1 [--rows ...] [--depth 6] [--gbm-rows ...]

The feature matrix of the tree timings is filled on the device (uniform), labels are normal; the split candidates
come from the first 10000 rows of each column (the candidate rule's sample size at maxBins 32).  A level's time is
the difference between the fit times of trees one level apart, so it includes everything a level launches.

With --devices, the rows are sharded over those GPUs (ShardedContext: each level's histogram is all-reduced with NCCL)
and the benchmark reports, for the tree of --depth, the wall time of the sharded fit next to one GPU fitting all the
rows and one GPU fitting one shard's rows.  The sharded fit minus the one-shard fit, per level, is what the all-reduce
and the ranks' wait for the slowest shard add to a level.  Then GBMRegressor rounds/s with the device learner on one
GPU and on the listed GPUs."""
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
from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor, continuous_split_candidates  # noqa: E402


def card(device=0):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(device)],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return q
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def tree_times(n, d, max_bins, depths, reps, classes=0, impurity="gini"):
    out = {}
    with Context(0) as ctx:
        ctx.alloc(N.SLOT_X, d, n)
        ctx.fill_synthetic(N.SLOT_X, "uniform", 1, 0.0, 1.0)
        if classes:  # labels: class indices drawn on the host; weights uniform in [0.5, 1.5)
            ctx.alloc(N.SLOT_Y, 1, n)
            ctx.upload(N.SLOT_Y, np.random.default_rng(2).integers(0, classes, n).astype(np.float32))
            ctx.alloc(N.SLOT_W, 1, n)
            ctx.fill_synthetic(N.SLOT_W, "uniform", 3, 0.5, 1.5)
            ctx.alloc(N.SLOT_PRED, 1, n)
        else:
            ctx.alloc(N.SLOT_R, 1, n)
            ctx.fill_synthetic(N.SLOT_R, "normal", 2, 0.0, 1.0)
            ctx.alloc(N.SLOT_H, 1, n)
        m = min(n, 10000)
        cands = [continuous_split_candidates(ctx.download(N.SLOT_X, count=m, offset=j * n), max_bins) for j in range(d)]
        ctx.tree_fit_bins(cands)
        sub = np.arange(d, dtype=np.int32)

        def fit(depth):
            if classes:
                return ctx.tree_fit_classifier(N.SLOT_Y, classes, weight_slot=N.SLOT_W, subspace=sub, impurity=impurity,
                                               max_depth=depth, out_slot=N.SLOT_PRED)
            return ctx.tree_fit(N.SLOT_R, 0, subspace=sub, max_depth=depth, out_slot=N.SLOT_H)

        for depth in depths:
            fit(depth)  # warm-up
            ts = []
            for _ in range(reps):
                ctx.timer_start()
                t = fit(depth)
                ts.append(ctx.timer_stop())
            out[depth] = {"ms_median": float(np.median(ts)), "ms_min": float(np.min(ts)), "nodes": int(t["feature"].size)}
    return out


def gbm_rounds(n, d, learner, rounds, resident=True, devices=()):
    from spark_ensemble_b200.ensemble import DataFrame
    from spark_ensemble_b200.regression import GBMRegressor
    rng = np.random.default_rng(0)
    X = rng.random((n, d), dtype=np.float32)
    y = np.sin(6 * X[:, 0]) + X[:, 1] * X[:, 2] + 0.1 * rng.standard_normal(n)
    df = DataFrame(features=X, label=y)
    times = {}
    for k in (1, rounds):
        g = GBMRegressor().set("baseLearner", learner).set("numBaseLearners", k).set("residentFeatures", resident)
        if devices:
            g.set("devices", list(devices))
        t0 = time.perf_counter()
        g.fit(df)
        times[k] = time.perf_counter() - t0
    per_round = (times[rounds] - times[1]) / (rounds - 1)
    res = {"rows": n, "cols": d, "rounds": rounds, "fit_s": times[rounds], "s_per_round": per_round,
           "rounds_per_s": 1.0 / per_round}
    if devices:
        res["devices"] = list(devices)
    return res


def boosting_rounds(n, d, K, learner, rounds):
    from spark_ensemble_b200.classification import BoostingClassifier
    from spark_ensemble_b200.ensemble import DataFrame
    rng = np.random.default_rng(0)
    X = rng.random((n, d), dtype=np.float32)
    z = np.sin(6 * X[:, 0]) + X[:, 1] * X[:, 2] + 0.3 * rng.standard_normal(n)
    y = np.digitize(z, np.quantile(z, np.linspace(0, 1, K + 1)[1:-1])).astype(np.float64)
    df = DataFrame(features=X, label=y, weight=rng.uniform(0.5, 1.5, n))
    times = {}
    for k in (1, rounds):
        b = BoostingClassifier().set("baseLearner", learner).set("numBaseLearners", k).set("residentFeatures", True)
        b.set("weightCol", "weight")
        t0 = time.perf_counter()
        m = b.fit(df)
        times[k] = time.perf_counter() - t0
    per_round = (times[rounds] - times[1]) / (rounds - 1)
    return {"rows": n, "cols": d, "classes": K, "rounds": rounds, "fitted_rounds": len(m.trainingHistory),
            "fit_s": times[rounds], "s_per_round": per_round, "rounds_per_s": 1.0 / per_round}


def fit_wall_ms(devices, n, d, max_bins, depth, reps):
    """Median wall time of a regression-tree fit of `depth` over n rows (uniform features, normal labels; the same
    fills as tree_times), on one GPU (devices of length 1) or sharded over `devices`.  A fit returns when every rank's
    stream has finished, so the wall time covers the whole fit."""
    from spark_ensemble_b200.sharded import ShardedContext
    world = len(devices)
    c = ShardedContext(devices) if world > 1 else Context(devices[0])
    try:
        c.gbm_configure(n, 0, 1, "squared")
        c.alloc(N.SLOT_X, d, n)
        ranks = c.ctxs if world > 1 else [c]
        for rk, rc in enumerate(ranks):  # every rank fills its own rows: no host copy of the matrix
            rc.fill_synthetic(N.SLOT_X, "uniform", 1 + 10 * rk, 0.0, 1.0)
            rc.fill_synthetic(N.SLOT_R, "normal", 2 + 10 * rk, 0.0, 1.0)
        n0 = ranks[0].layout(N.SLOT_X)[1]
        m = min(n0, 10000)
        cands = [continuous_split_candidates(ranks[0].download(N.SLOT_X, count=m, offset=j * n0), max_bins)
                 for j in range(d)]
        c.tree_fit_bins(cands)
        sub = np.arange(d, dtype=np.int32)
        fit = lambda: c.tree_fit(N.SLOT_R, 0, subspace=sub, max_depth=depth, out_slot=N.SLOT_H)
        fit()  # warm-up
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            t = fit()
            ts.append((time.perf_counter() - t0) * 1e3)
        return {"ms_median": float(np.median(ts)), "ms_min": float(np.min(ts)), "nodes": int(t["feature"].size)}
    finally:
        c.close()


def main_devices(args):
    from spark_ensemble_b200.ensemble import row_partition
    devices = [int(x) for x in args.devices.split(",")]
    world = len(devices)
    n, d, depth = args.rows, args.cols, args.depth
    s0, s1 = row_partition(n, world, 0)
    res = {"cards": [card(x) for x in devices], "rows": n, "cols": d, "bins": args.bins, "depth": depth, "gpus": world}
    one = fit_wall_ms(devices[:1], n, d, args.bins, depth, args.reps)
    shard = fit_wall_ms(devices[:1], s1 - s0, d, args.bins, depth, args.reps)
    sharded = fit_wall_ms(devices, n, d, args.bins, depth, args.reps)
    levels = max(depth, 1)
    nb = args.bins + 1  # bins per column: maxBins - 1 candidates, the rank past the last one, and NaN
    res.update({"one_gpu_all_rows": one, "one_gpu_one_shard": shard, "sharded": sharded,
                "sharded_over_one_gpu": sharded["ms_median"] / one["ms_median"],
                "sharded_level_ms": sharded["ms_median"] / levels,
                "allreduce_and_wait_ms_per_level": (sharded["ms_median"] - shard["ms_median"]) / levels,
                "histogram_MB_per_level": [(1 << L) * d * nb * 4 * 8 / 1e6 for L in range(levels)]})
    print(json.dumps(res, indent=1), flush=True)
    for devs in (devices[:1], devices):
        g = gbm_rounds(args.gbm_rows, args.gbm_cols, DeviceDecisionTreeRegressor(maxDepth=5), 20,
                       devices=devs if len(devs) > 1 else ())
        res.setdefault("gbm_device", []).append(g)
        print(json.dumps({"gbm_device": g}), flush=True)


def main_classes(args):
    from spark_ensemble_b200.learners import DecisionTreeClassifier, DeviceDecisionTreeClassifier
    K = args.classes
    res = {"card": card(), "classes": K, "impurity": args.impurity}
    n, d = args.rows, args.cols
    tt = tree_times(n, d, args.bins, list(range(0, 7)), args.reps, classes=K, impurity=args.impurity)
    res["tree_ms"] = tt
    bytes_level = n * (d + 4 + 4 + 2 + 2 + 1)  # ranks, labels, weights, node index in and out, one gathered rank
    levels = {}
    for L in range(6):
        ms = tt[L + 1]["ms_median"] - tt[L]["ms_median"]
        levels[L] = {"ms": ms, "model_bytes": bytes_level, "achieved_GBps": bytes_level / (ms * 1e-3) / 1e9}
    res["levels"] = levels
    res["byte_model_ms_per_level_at_3.06TBps"] = bytes_level / 3.06e12 * 1e3
    print(json.dumps(res, indent=1), flush=True)
    dev = DeviceDecisionTreeClassifier(maxDepth=5, impurity=args.impurity)
    res["boost_device"] = boosting_rounds(args.gbm_rows, args.gbm_cols, K, dev, 10)
    print(json.dumps({"boost_device": res["boost_device"]}), flush=True)
    res["boost_host"] = boosting_rounds(args.host_rows, args.gbm_cols, K, DecisionTreeClassifier(maxDepth=5), 3)
    print(json.dumps({"boost_host": res["boost_host"]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--cols", type=int, default=128)
    ap.add_argument("--bins", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--gbm-rows", type=int, default=10_000_000)
    ap.add_argument("--gbm-cols", type=int, default=32)
    ap.add_argument("--host-rows", type=int, default=1_000_000)
    ap.add_argument("--classes", type=int, default=0, help="classification fit with this many classes (2..64)")
    ap.add_argument("--impurity", default="gini", choices=("gini", "entropy"))
    ap.add_argument("--devices", default="", help="shard the rows over these GPUs, e.g. 0,1 (regression fit)")
    ap.add_argument("--depth", type=int, default=6, help="with --devices: depth of the timed tree")
    args = ap.parse_args()
    if args.devices:
        return main_devices(args)
    if args.classes:
        return main_classes(args)
    res = {"card": card()}
    n, d = args.rows, args.cols
    tt = tree_times(n, d, args.bins, list(range(0, 7)), args.reps)
    res["tree_ms"] = tt
    bytes_level = n * (d + 4 + 2 + 2 + 1)  # ranks, labels, node index in and out, one gathered rank (no weights, no bag)
    levels = {}
    for L in range(6):
        ms = tt[L + 1]["ms_median"] - tt[L]["ms_median"]
        levels[L] = {"ms": ms, "model_bytes": bytes_level, "achieved_GBps": bytes_level / (ms * 1e-3) / 1e9}
    res["levels"] = levels
    res["byte_model_ms_per_level_at_3.06TBps"] = bytes_level / 3.06e12 * 1e3
    print(json.dumps(res, indent=1), flush=True)
    res["gbm_device"] = gbm_rounds(args.gbm_rows, args.gbm_cols, DeviceDecisionTreeRegressor(maxDepth=5), 20)
    print(json.dumps({"gbm_device": res["gbm_device"]}), flush=True)
    from spark_ensemble_b200.learners import DecisionTreeRegressor
    res["gbm_host"] = gbm_rounds(args.host_rows, args.gbm_cols, DecisionTreeRegressor(maxDepth=5), 3)
    print(json.dumps({"gbm_host": res["gbm_host"]}), flush=True)


if __name__ == "__main__":
    main()
