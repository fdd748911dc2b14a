#!/usr/bin/env python
"""GBMRegressionModel.transform for tree members: se_forest_predict (one pass) vs one se_tree_predict per member into
an [M][n] array + the aggregation kernel.

    python benchmarks/forest_time.py [--rows 50000000] [--out /tmp/forest.json]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from spark_ensemble_b200 import _native as N  # noqa: E402
from spark_ensemble_b200.context import Context  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=50_000_000)
ap.add_argument("--out", default=None)
args = ap.parse_args()
ctx = Context(0)
n, d = args.rows, 128
ctx.alloc(N.SLOT_X, d, n)
ctx.fill_synthetic(N.SLOT_X, "normal", 3, 0, 1)
ctx.alloc(N.SLOT_H, 1, n)
rng = np.random.default_rng(7)
grid = (np.arange(-15, 16) * 0.1).astype(np.float32)   # 31 candidate thresholds per column (Spark's default maxBins 32)
res = []
for M, depth in ((20, 5), (100, 5), (100, 6)):
    nn = 2 ** (depth + 1) - 1
    idx = np.arange(nn)
    leaf = idx >= 2 ** depth - 1
    trees = []
    for _ in range(M):
        feat = rng.integers(0, d, nn)
        trees.append({"feature": np.where(leaf, -1, feat).astype(np.int32),
                      "threshold": np.where(leaf, 0.0, grid[rng.integers(0, grid.size, nn)]).astype(np.float32),
                      "left": np.where(leaf, 0, 2 * idx + 1).astype(np.int32), "right": np.where(leaf, 0, 2 * idx + 2).astype(np.int32),
                      "value": rng.standard_normal(nn).astype(np.float32)})
    w = rng.random(M) + 0.1
    ctx.forest_predict(trees, N.SLOT_H, weights=w, init=0.5)
    ctx.sync()
    t0 = time.perf_counter()
    R = 3
    for _ in range(R):
        ctx.forest_predict(trees, N.SLOT_H, weights=w, init=0.5)
    ctx.sync()
    forest_ms = 1e3 * (time.perf_counter() - t0) / R
    chunks = int(ctx.get_option("last_forest_chunks"))
    sum_forest = ctx.slot_sum(N.SLOT_H)
    # member by member into P, then the weighted sum
    ctx.agg_configure(N.AGG_GBM_REGRESSOR, M, 0, 1, 0, n)
    for m, tr in enumerate(trees):
        ctx.tree_predict(tr, N.SLOT_P, m)
    ctx.agg_run(w, [0.5])
    ctx.sync()
    t0 = time.perf_counter()
    for m, tr in enumerate(trees):
        ctx.tree_predict(tr, N.SLOT_P, m)
    ctx.agg_run(w, [0.5])
    ctx.sync()
    member_ms = 1e3 * (time.perf_counter() - t0)
    sum_members = ctx.slot_sum(N.SLOT_RAW)
    r = {"rows": n, "columns": d, "trees": M, "depth": depth, "forest_ms": forest_ms, "forest_chunks": chunks,
         "per_member_plus_aggregation_ms": member_ms, "speedup": member_ms / forest_ms,
         "intermediate_bytes_avoided": 4 * M * n, "sum_rel_diff": abs(sum_forest - sum_members) / abs(sum_members)}
    res.append(r)
    print(json.dumps(r), flush=True)
    ctx.free(N.SLOT_P)
ctx.close()
if args.out:
    json.dump(res, open(args.out, "w"), indent=1)
