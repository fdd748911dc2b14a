"""Generates the committed fixtures under tests/golden/ from the reference's LIBSVM data files (the tests
read only the committed fixtures).

    python tests/golden/make_golden.py <reference checkout>/data

* cpusmall.npz / letter.npz / adult8k.npz — the reference's own test datasets
  (data/* of the reference repository, loaded at e.g. test/regression/GBMRegressorSuite.scala:54) as compact arrays.
* gbm_cpusmall_oracle.json — BASELINE config 1 (GBMRegressor, cpusmall, 20 rounds, squared loss,
  DecisionTree depth 5) run through the ORACLE-driven reference control flow (tests/ref_fit.py): per-round
  alpha, train loss and a prediction checksum.  These are oracle outputs, not outputs of the Scala
  reference (no JVM here: parity unpinned, see oracle/se_oracle.h).
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = sys.argv[1] if len(sys.argv) > 1 else "data"


def read_libsvm(path, d):
    ys, rows = [], []
    with open(path) as f:
        for line in f:
            parts = line.split()
            if not parts:
                continue
            ys.append(float(parts[0]))
            x = np.zeros(d, dtype=np.float32)
            for tok in parts[1:]:
                k, v = tok.split(":")
                x[int(k) - 1] = float(v)
            rows.append(x)
    return np.stack(rows), np.asarray(ys, dtype=np.float32)


def main():
    X, y = read_libsvm(f"{REF}/cpusmall/cpusmall.svm", 12)
    np.savez_compressed(f"{HERE}/cpusmall.npz", X=X, y=y)
    X, y = read_libsvm(f"{REF}/letter/letter.svm", 16)
    # letter.svm is the [-1,1]-scaled variant: x = code/7.5 - 1 with integer codes 0..15; store the codes
    codes = np.rint((X.astype(np.float64) + 1.0) * 7.5).astype(np.int8)
    assert np.max(np.abs((codes / 7.5 - 1.0) - X)) < 1e-5
    np.savez_compressed(f"{HERE}/letter.npz", X=codes, y=(y - 1).astype(np.int8))  # labels 1..26 -> 0..25
    X, y = read_libsvm(f"{REF}/adult/adult.svm", 123)
    X, y = X[:8000], y[:8000]
    np.savez_compressed(f"{HERE}/adult8k.npz", X=np.packbits(X.astype(bool), axis=1), y=((y + 1) / 2).astype(np.int8))

    from oracle.oracle import Oracle
    from tests.ref_fit import ref_gbm_regressor_fit
    from spark_ensemble_b200.learners import DecisionTreeRegressor
    d = np.load(f"{HERE}/cpusmall.npz")
    res = ref_gbm_regressor_fit(Oracle(), d["X"], d["y"].astype(np.float64), None,
                                DecisionTreeRegressor(maxDepth=5), loss="squared", num_learners=20)
    out = {"config": "GBMRegressor cpusmall 20 rounds squared loss, DecisionTreeRegressor(maxDepth=5), lr=1, tol=1e-6",
           "init": res["init"], "alpha": res["alpha"], "train_loss": res["train_loss"],
           "pred_sum": float(np.sum(res["F"])), "pred_sq_sum": float(np.sum(res["F"] ** 2)),
           "pred_head": [float(v) for v in res["F"][:8]]}
    with open(f"{HERE}/gbm_cpusmall_oracle.json", "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", os.listdir(HERE))


if __name__ == "__main__":
    main()
