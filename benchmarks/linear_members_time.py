"""Linear and logistic base learners fitted where Bagging's and Boosting's data live, against the route through the
learners' own `fit` (residentFeatures=False).  Card name and power limit are read in the same process.

    python benchmarks/linear_members_time.py [--rows 10000000] [--eval-rows 100000000] [--reps 10] [--out r.json]

1. BaggingClassifier fit, 10 DeviceLogisticRegression members (regParam 0.01), subspaceRatio 0.5, subsampleRatio 1
   with replacement (Poisson bag), at --rows × 32 host features with K = 2 and K = 8 classes from a random linear
   model: wall time of one fit per route after a warm-up at 100 000 rows, and the members' evaluation counts.
2. One se_logistic_loss_grad_batch call over 10 binomial members of 64 columns drawn from 128 (subspaceRatio 0.5)
   against the same 10 members' se_logistic_loss_grad calls one after another, at --eval-rows × 128 features filled on
   the device (uniform features, Bernoulli labels, weights uniform in [0, 2)): CUDA events around the calls, median of
   --reps after a warm-up.  Bytes: the union of the members' columns, labels and weights read once, 4 B each.
3. A BoostingClassifier (SAMME) fit of 2 rounds with DeviceLogisticRegression at --rows × 32, K = 2, per route."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from benchmarks.stacking_time import HBM_BPS, card  # noqa: E402
from spark_ensemble_b200 import _native as N  # noqa: E402
from spark_ensemble_b200.classification import BaggingClassifier, BoostingClassifier  # noqa: E402
from spark_ensemble_b200.context import Context  # noqa: E402
from spark_ensemble_b200.ensemble import DataFrame, subspace  # noqa: E402
from spark_ensemble_b200.learners import DeviceLogisticRegression  # noqa: E402


def _data(n, d, K, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d), dtype=np.float32)
    z = X @ rng.standard_normal((d, K)).astype(np.float32)
    y = np.argmax(z + rng.gumbel(size=(n, K)).astype(np.float32), axis=1).astype(np.float64)
    return X, y


def _routes(est, X, y):
    out = {}
    for resident in (True, False):
        e = est.copy().setResidentFeatures(resident)
        e.fit(DataFrame(features=X[:100_000], label=y[:100_000]))  # warm-up
        t0 = time.perf_counter()
        model = e.fit(DataFrame(features=X, label=y))
        out["resident" if resident else "fit"] = {"fit_s": time.perf_counter() - t0, "model": model}
    return out


def bagging(n, K, M=10, d=32):
    X, y = _data(n, d, K, seed=K)
    est = (BaggingClassifier().setBaseLearner(DeviceLogisticRegression(regParam=0.01)).setNumBaseLearners(M)
           .setSubspaceRatio(0.5).setReplacement(True))
    r = _routes(est, X, y)
    res = {"n": n, "d": d, "K": K, "M": M}
    for k, v in r.items():
        res[k] = {"fit_s": v["fit_s"], "evaluations": [m.numEvaluations for m in v["model"].models]}
    res["speedup"] = r["fit"]["fit_s"] / r["resident"]["fit_s"]
    return res


def evaluation(n, reps, M=10, d=128):
    rng = np.random.default_rng(0)
    subs = [subspace(0.5, d, 7 + i) for i in range(M)]
    members = [(s, rng.standard_normal((1, s.size + 1)) * 0.1, None, None) for s in subs]
    with Context(0) as ctx:
        ctx.alloc(N.SLOT_X, d, n)
        ctx.fill_synthetic(N.SLOT_X, "uniform", 1, -1.0, 1.0)
        ctx.alloc(N.SLOT_Y, n)
        ctx.fill_synthetic(N.SLOT_Y, "bernoulli", 2, 0.4, 0.0)
        ctx.alloc(N.SLOT_W, n)
        ctx.fill_synthetic(N.SLOT_W, "uniform", 3, 0.0, 2.0)

        def batch():
            return ctx.logistic_loss_grad_batch(N.SLOT_X, members, N.SLOT_Y, 0, N.SLOT_W, 0)

        def lone():
            return [ctx.logistic_loss_grad(N.SLOT_X, c, th, N.SLOT_Y, 0, N.SLOT_W, 0) for c, th, _, _ in members]

        times = {}
        for name, fn in (("batch", batch), ("lone", lone)):
            fn()  # warm-up
            ts = []
            for _ in range(reps):
                ctx.timer_start()
                fn()
                ts.append(ctx.timer_stop())
            times[name] = float(np.median(ts))
        same = all(a[1].tobytes() == b[1].tobytes() for a, b in zip(batch(), lone()))
    union = len(set(np.concatenate(subs).tolist()))
    nbytes = n * 4 * (union + 2)
    return {"n": n, "d": d, "M": M, "p": [int(s.size) for s in subs], "union_cols": union,
            "batch_ms": times["batch"], "lone_ms": times["lone"], "speedup": times["lone"] / times["batch"],
            "batch_bytes_once": nbytes, "batch_GBps_once": nbytes / times["batch"] / 1e6,
            "hbm_bound_ms": 1e3 * nbytes / HBM_BPS, "batch_equals_lone_bits": same}


def boosting(n, d=32, rounds=2):
    X, y = _data(n, d, 2, seed=5)
    est = (BoostingClassifier().setBaseLearner(DeviceLogisticRegression(regParam=0.01)).setNumBaseLearners(rounds))
    r = _routes(est, X, y)
    return {"n": n, "d": d, "rounds": rounds, **{k: {"fit_s": v["fit_s"]} for k, v in r.items()},
            "speedup": r["fit"]["fit_s"] / r["resident"]["fit_s"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--eval-rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card()}
    print(json.dumps({"card": res["card"]}), flush=True)
    res["evaluation"] = evaluation(a.eval_rows, a.reps)
    print(json.dumps(res["evaluation"]), flush=True)
    res["bagging"] = [bagging(a.rows, K) for K in (2, 8)]
    for r in res["bagging"]:
        print(json.dumps(r), flush=True)
    res["boosting"] = boosting(a.rows)
    print(json.dumps(res["boosting"]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
