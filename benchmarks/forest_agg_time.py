#!/usr/bin/env python
"""Classifier transform over tree members: the resident route (residentFeatures=True: X uploaded once, se_forest_agg
walks every tree and finishes every row on chip) against the member route (each member walked on the host, the
[M][K][n] outputs stacked and uploaded, se_agg_run).  Both routes run alternately in one process on the same model;
wall time of model.transform includes everything each route does.  Also times se_forest_agg alone (CUDA events, X
already resident) and one size the member route cannot hold.

    python benchmarks/forest_agg_time.py [--reps 3] [--out /tmp/forest_agg.json]
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
from spark_ensemble_b200.classification import (BaggingClassificationModel, BoostingClassificationModel,  # noqa: E402
                                                GBMClassificationModel)
from spark_ensemble_b200.context import Context  # noqa: E402
from spark_ensemble_b200.learners import (DeviceDecisionTreeClassificationModel,  # noqa: E402
                                          DeviceDecisionTreeRegressionModel)

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--out", default=None)
args = ap.parse_args()


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        pl = "unknown"
    return name, pl


def tree(rng, depth, d, cands, K):
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
    p = rng.dirichlet(np.full(K, 0.3), n).astype(np.float32)
    return {"feature": f, "threshold": t, "left": l, "right": r, "value": np.argmax(p, axis=1).astype(np.float32),
            "values": p}


def forest(seed, M, depth, d, K):
    rng = np.random.default_rng(seed)
    cands = np.sort(rng.standard_normal((d, 31)), axis=1).astype(np.float32)  # maxBins 32
    return [tree(rng, depth, d, cands, K) for _ in range(M)]


def models(kind, trees, K, d):
    M = len(trees)
    cls = [DeviceDecisionTreeClassificationModel(t, K) for t in trees]
    if kind == "bagging_soft":
        return BaggingClassificationModel(K, [np.arange(d)] * M, cls).setVotingStrategy("soft"), M * K
    if kind == "boosting_real":
        return BoostingClassificationModel(K, np.ones(M), cls).setAlgorithm("real"), M * K
    rounds = M // K if M >= K else 1  # GBM logloss: one regression tree per class and round
    reg = [[DeviceDecisionTreeRegressionModel(dict(trees[(i * K + j) % M], value=trees[(i * K + j) % M]["values"][:, 0]))
            for j in range(K)] for i in range(rounds)]
    return GBMClassificationModel(K, [np.full(K, 0.1)] * rounds, [np.arange(d)] * rounds, reg, np.zeros(K), K), rounds * K


def wall(m, df, resident):
    m.set("residentFeatures", resident)
    t0 = time.perf_counter()
    m.transform(df)
    return 1e3 * (time.perf_counter() - t0)


def kernel_ms(X, kind_id, trees, K, **kw):
    n, d = X.shape
    with Context(0) as ctx:
        ctx.alloc(N.SLOT_X, d, n)
        ctx.upload_rowmajor(N.SLOT_X, X)
        ctx.forest_agg(kind_id, K, trees, **kw)  # warm-up: ranks the columns, sizes the buffers
        ctx.sync()
        best = float("inf")
        for _ in range(args.reps):
            ctx.timer_start()
            ctx.forest_agg(kind_id, K, trees, **kw)
            best = min(best, ctx.timer_stop())
        return best, ctx.get_option("last_forest_chunks")


name, power = card()
res = {"card": name, "power_limit": power, "runs": []}
KIND = {"bagging_soft": N.AGG_BAGGING_SOFT, "boosting_real": N.AGG_BOOSTING_REAL, "gbm_logloss": N.AGG_GBM_CLASSIFIER}
n, d, K, M, depth = 2_000_000, 32, 26, 32, 6
X = np.random.default_rng(1).standard_normal((n, d), dtype=np.float32)
df = DataFrame(features=X)
trees = forest(2, M, depth, d, K)
for kind in ("gbm_logloss", "bagging_soft", "boosting_real"):
    m, outputs = models(kind, trees, K, d)
    wall(m, df, True)  # warm-up (library load, first allocations)
    tr, tm = [], []
    for _ in range(args.reps):  # alternated
        tr.append(wall(m, df, True))
        tm.append(wall(m, df, False))
    if kind == "gbm_logloss":
        flat = [mm.tree_arrays() for ms in m.models for mm in ms]
        kms, chunks = kernel_ms(X, KIND[kind], flat, K, weights=np.full(len(flat), 0.1), init=np.zeros(K),
                                tree_class=np.tile(np.arange(K, dtype=np.int32), len(m.models)), dim=K, loss="logloss")
    else:
        kms, chunks = kernel_ms(X, KIND[kind], trees, K)
    row = {"kind": kind, "n": n, "d": d, "K": K, "trees": outputs // (K if kind != "gbm_logloss" else 1), "depth": depth,
           "resident_ms": min(tr), "member_ms": min(tm), "forest_agg_kernel_ms": kms, "chunks": chunks,
           "resident_rows_per_s": n / (min(tr) / 1e3), "member_rows_per_s": n / (min(tm) / 1e3),
           "kernel_rows_per_s": n / (kms / 1e3), "bytes_not_moved": 4 * outputs * n}
    res["runs"].append(row)
    print(json.dumps(row), flush=True)

# only the resident route: the member outputs would take 4·M·K·n bytes = 111 GB
n2, d2, M2 = 8 * 1024 * 1024, 16, 128
X2 = np.random.default_rng(3).standard_normal((n2, d2), dtype=np.float32)
trees2 = forest(4, M2, 6, d2, K)
kms, chunks = kernel_ms(X2, N.AGG_BAGGING_SOFT, trees2, K)
m2, outputs2 = models("bagging_soft", trees2, K, d2)
m2.set("residentFeatures", True)
t0 = time.perf_counter()
m2.transform(DataFrame(features=X2))
w2 = 1e3 * (time.perf_counter() - t0)
row = {"kind": "bagging_soft", "n": n2, "d": d2, "K": K, "trees": M2, "depth": 6, "resident_ms": w2, "member_ms": None,
       "forest_agg_kernel_ms": kms, "chunks": chunks, "resident_rows_per_s": n2 / (w2 / 1e3),
       "kernel_rows_per_s": n2 / (kms / 1e3), "bytes_not_moved": 4 * outputs2 * n2}
res["runs"].append(row)
print(json.dumps(row), flush=True)
print(json.dumps({"card": name, "power_limit": power}))
if args.out:
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)
