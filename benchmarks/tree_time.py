#!/usr/bin/env python
"""Tree prediction over 100 M x 128 (the kernel-sweep shape) per depth, for both walks over the rank matrix.

    python benchmarks/tree_time.py

mask 1 is the all-nodes kernel (option `tree_mask` 1, the default for trees of <= 64 internal nodes), mask 0 the
level-by-level walk (`tree_mask` 0, the kernel deeper trees use).
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from spark_ensemble_b200 import _native as N  # noqa: E402
from spark_ensemble_b200.context import Context  # noqa: E402

ctx = Context(0)
n, d = 100_000_000, 128
ctx.alloc(N.SLOT_X, d, n)
ctx.fill_synthetic(N.SLOT_X, "normal", 3, 0, 1)
ctx.alloc(N.SLOT_H, 1, n)
ctx.set_option("tree_bins", 1)
for depth in (3, 5, 6):
    nn = 2 ** (depth + 1) - 1
    idx = np.arange(nn)
    leaf = idx >= 2 ** depth - 1
    tree = {"feature": np.where(leaf, -1, (idx * 37) % d), "threshold": np.where(leaf, 0.0, ((idx * 13) % 7 - 3) * 0.2),
            "left": np.where(leaf, 0, 2 * idx + 1), "right": np.where(leaf, 0, 2 * idx + 2), "value": np.linspace(-1, 1, nn)}
    for mask in (1, 0):
        ctx.set_option("tree_mask", mask)
        ctx.tree_predict(tree, N.SLOT_H, 0)
        ctx.sync()
        ctx.kernel_timing(True)
        ctx.kernel_times_reset()
        for _ in range(10):
            ctx.tree_predict(tree, N.SLOT_H, 0)
        kt = ctx.kernel_times()
        ctx.kernel_timing(False)
        ms = kt["tree"]["ms"] / kt["tree"]["launches"]
        internal = 2 ** depth - 1
        print("depth", depth, "mask", int(ctx.get_option("last_tree_mask")), "ms", round(ms, 4),
              "GB/s at (internal nodes + 4) B/row", round((internal + 4) * n / ms / 1e6, 1), flush=True)
ctx.close()
