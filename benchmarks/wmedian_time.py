#!/usr/bin/env python
"""Weighted median (BoostingRegressor.predict) over 25 M rows: fast path vs exact kernel, by weight pattern.

    python benchmarks/wmedian_time.py [--out /tmp/wmedian.json]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from spark_ensemble_b200 import _native as N  # noqa: E402
from spark_ensemble_b200.context import Context  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", default=None)
ap.add_argument("--rows", type=int, default=25_000_000)
args = ap.parse_args()
ctx = Context(0)
rng = np.random.default_rng(5)
res = []
for M in (8, 32, 64):
    n = args.rows if M <= 32 else args.rows // 2
    ctx.agg_configure(N.AGG_BOOSTING_REG_MEDIAN, M, 0, 1, 0, n)
    ctx.fill_synthetic(N.SLOT_P, "normal", 7, 0.0, 1.0)
    for pattern, a in (("random", rng.random(M) + 0.05), ("equal", np.full(M, 0.25)), ("integers 1..3", rng.integers(1, 4, M).astype(np.float64))):
        row = {"M": M, "rows": n, "weights": pattern}
        for fast in (1, 0):
            ctx.set_option("wm_fast", fast)
            ctx.agg_run(a)
            ctx.sync()
            ctx.kernel_timing(True)
            ctx.kernel_times_reset()
            for _ in range(5):
                ctx.agg_run(a)
            kt = ctx.kernel_times()
            ctx.kernel_timing(False)
            ms = kt["agg"]["ms"] / 5
            row["fast_ms" if fast else "exact_ms"] = ms
            if fast:
                row["mode"] = int(ctx.get_option("last_wm_mode"))
                row["deferred_rows"] = int(ctx.get_option("last_wm_deferred"))
        row["gbs_fast"] = (4 * M + 4) * n / row["fast_ms"] / 1e6
        res.append(row)
        print(json.dumps(row), flush=True)
ctx.set_option("wm_fast", 1)
ctx.close()
if args.out:
    json.dump(res, open(args.out, "w"), indent=1)
