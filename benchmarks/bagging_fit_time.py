"""Bagging's training on the GPU: the forest fit (se_forest_fit, every member's tree in one launch sequence per batch)
against the same trees fitted one at a time, and BaggingRegressor / BaggingClassifier's device route against the
member route (one learner.fit per member: a host gather of the in-bag rows and the member's columns, candidates, a
context, an upload and a re-rank per member).  Card name and power limit are read in the same process.

    python benchmarks/bagging_fit_time.py [--reps 3] [--skip-large] [--out results.json]

In-context rows ("forest" vs "loop"): one context holds X (filled on the device, normal), the labels (normal, or class
indices for --classes), weights (uniform) and bag multiplicities (0, 1 or 2), and the candidates of maxBins 32 from
the first 10000 rows of every column.  "forest" is DeviceDecisionTree*.fit_forest_resident over the members'
subspaces, "loop" is fit_resident per member over the same context and candidates, which gives the same trees one at
a time.  Both end in a device synchronise.  Estimator rows time Bagging*.fit end to end (host data, numBaseLearners,
subsampleRatio 0.7 with replacement) with residentFeatures=True (device route) and False (member route)."""
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
from spark_ensemble_b200.ensemble import DataFrame, subspace  # noqa: E402
from spark_ensemble_b200.learners import (DeviceDecisionTreeClassifier, DeviceDecisionTreeRegressor,  # noqa: E402
                                          continuous_split_candidates)


def card(device=0):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(device)],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def _median_s(fn, reps):
    fn()  # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def in_context(n, d, depth, M, ratio, K, reps, seed=0x5eed):
    """forest vs loop over one context; returns seconds per fit of all M members and the trees' node counts."""
    subs = [subspace(ratio, d, seed + i) for i in range(M)]
    learner = (DeviceDecisionTreeClassifier(maxDepth=depth) if K else DeviceDecisionTreeRegressor(maxDepth=depth))
    with Context(0) as ctx:
        ctx.alloc(N.SLOT_X, d, n)
        ctx.fill_synthetic(N.SLOT_X, "normal", 1, 0.0, 1.0)
        for s in (N.SLOT_Y, N.SLOT_W, N.SLOT_BAG, N.SLOT_H):
            ctx.alloc(s, 1, n)
        if K:
            ctx.fill_synthetic(N.SLOT_Y, "randint", 2, 0, K)
        else:
            ctx.fill_synthetic(N.SLOT_Y, "normal", 2, 0.0, 1.0)
        ctx.fill_synthetic(N.SLOT_W, "uniform", 3, 0.5, 1.5)
        ctx.fill_synthetic(N.SLOT_BAG, "randint", 4, 0, 3)
        m = min(n, 10000)
        ctx.tree_fit_bins([continuous_split_candidates(ctx.download(N.SLOT_X, count=m, offset=j * n), 32)
                           for j in range(d)])
        if K:
            forest = lambda: learner.fit_forest_resident(ctx, K, N.SLOT_Y, 0, N.SLOT_W, 0, True, subs)
            loop = lambda: [learner.fit_resident(ctx, K, N.SLOT_Y, 0, N.SLOT_W, 0, True, s, N.SLOT_H, 0) for s in subs]
        else:
            forest = lambda: learner.fit_forest_resident(ctx, N.SLOT_Y, 0, N.SLOT_W, 0, True, subs)
            loop = lambda: [learner.fit_resident(ctx, N.SLOT_Y, 0, N.SLOT_W, 0, True, s, N.SLOT_H, 0) for s in subs]
        res = {"rows": n, "cols": d, "depth": depth, "members": M, "subspaceRatio": ratio, "classes": K,
               "distinct_subspaces": len({s.tobytes() for s in subs})}
        # alternate the two routes so that drift on a shared host hits both alike
        a1 = _median_s(forest, reps)
        b1 = _median_s(loop, reps)
        a2 = _median_s(forest, reps)
        res["forest_batches"] = int(ctx.get_option("last_forest_fit_batches"))
        b2 = _median_s(loop, reps)
        res.update({"forest_s": min(a1, a2), "loop_s": min(b1, b2), "forest_s_runs": [a1, a2], "loop_s_runs": [b1, b2]})
        res["loop_over_forest"] = res["loop_s"] / res["forest_s"]
        f = forest()
        res["nodes"] = [int(m_.numNodes) for m_ in f]
    return res


def estimator(n, d, depth, M, ratio, K, reps, member=True):
    from spark_ensemble_b200.classification import BaggingClassifier
    from spark_ensemble_b200.regression import BaggingRegressor
    rng = np.random.default_rng(0)
    X = rng.standard_normal((n, d), dtype=np.float32)
    z = np.sin(2 * X[:, 0]) + X[:, 1] * X[:, 2] + 0.3 * rng.standard_normal(n)
    y = np.digitize(z, np.quantile(z, np.linspace(0, 1, K + 1)[1:-1])).astype(np.float64) if K else z
    df = DataFrame(features=X, label=y)
    if K:
        est = BaggingClassifier().setBaseLearner(DeviceDecisionTreeClassifier(maxDepth=depth))
    else:
        est = BaggingRegressor().setBaseLearner(DeviceDecisionTreeRegressor(maxDepth=depth))
    est = est.setNumBaseLearners(M).setSubspaceRatio(ratio).setSubsampleRatio(0.7).setReplacement(True)
    res = {"rows": n, "cols": d, "depth": depth, "members": M, "subspaceRatio": ratio, "classes": K}
    res["device_route_s"] = _median_s(lambda: est.setResidentFeatures(True).fit(df), reps)
    if member:
        res["member_route_s"] = _median_s(lambda: est.setResidentFeatures(False).fit(df), max(1, reps - 1))
        res["member_over_device"] = res["member_route_s"] / res["device_route_s"]
    else:
        res["member_route_s"] = "not measured"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-large", action="store_true", help="leave out the 100 M x 128 shape")
    ap.add_argument("--out", default="", help="also write the results as one JSON file here")
    args = ap.parse_args()
    out = {"card": card()}
    print(json.dumps(out), flush=True)
    shapes = [("reg_10M", dict(n=10_000_000, d=32, depth=5, M=10, ratio=0.5, K=0)),
              ("reg_1M", dict(n=1_000_000, d=32, depth=5, M=10, ratio=0.5, K=0)),
              ("reg_10M_ratio1", dict(n=10_000_000, d=32, depth=5, M=10, ratio=1.0, K=0)),
              ("cls2_10M", dict(n=10_000_000, d=32, depth=5, M=10, ratio=0.5, K=2)),
              ("cls26_10M", dict(n=10_000_000, d=32, depth=5, M=10, ratio=0.5, K=26))]
    if not args.skip_large:
        shapes.append(("reg_100M_128", dict(n=100_000_000, d=128, depth=6, M=8, ratio=0.5, K=0)))
    for name, s in shapes:
        r = in_context(reps=args.reps, **s)
        out[f"in_context_{name}"] = r
        print(json.dumps({f"in_context_{name}": r}), flush=True)
    for name, s, member in (("reg_1M", dict(n=1_000_000, d=32, depth=5, M=10, ratio=0.5, K=0), True),
                            ("reg_10M", dict(n=10_000_000, d=32, depth=5, M=10, ratio=0.5, K=0), True),
                            ("reg_10M_ratio1", dict(n=10_000_000, d=32, depth=5, M=10, ratio=1.0, K=0), True),
                            ("cls2_10M", dict(n=10_000_000, d=32, depth=5, M=10, ratio=0.5, K=2), True),
                            ("cls26_10M", dict(n=10_000_000, d=32, depth=5, M=10, ratio=0.5, K=26), True)):
        r = estimator(reps=args.reps, member=member, **s)
        out[f"estimator_{name}"] = r
        print(json.dumps({f"estimator_{name}": r}), flush=True)
    out["card_after"] = card()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
