#!/usr/bin/env python
"""Vote-aggregation kernels (BaggingClassifier hard votes, BoostingClassifier SAMME discrete) at M = 64, K = 26."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from spark_ensemble_b200 import _native as N  # noqa: E402
from spark_ensemble_b200.context import Context  # noqa: E402

ctx = Context(0)
M, K, n = 64, 26, 10_000_000
peak = 3350.0  # H100 SXM data sheet, GB/s
for kind, name, w in ((N.AGG_BAGGING_HARD, "hard votes", None), (N.AGG_BOOSTING_DISCRETE, "weighted votes", np.linspace(0.5, 1.5, M))):
    ctx.agg_configure(kind, M, K, 1, 0, n)
    ctx.fill_synthetic(N.SLOT_P, "randint", 5, 0, K)
    ctx.agg_run(w); ctx.sync()
    ctx.kernel_timing(True); ctx.kernel_times_reset()
    for _ in range(10):
        ctx.agg_run(w)
    kt = ctx.kernel_times()["agg"]; ctx.kernel_timing(False)
    ms = kt["ms"] / kt["launches"]
    b = 4 * M + 4 * (2 * K + 1)
    print(f"{name:16s} M={M} K={K} n={n}: {ms:.4f} ms  {b * n / ms / 1e6:.0f} GB/s  {b * n / ms / 1e6 / peak:.3f} of the measured HBM peak", flush=True)
ctx.close()
