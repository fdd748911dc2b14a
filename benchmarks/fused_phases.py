#!/usr/bin/env python
"""Where a one-launch squared-loss round spends its time: in-kernel %globaltimer stamps (statistics phase, fold +
exchange + Brent, update phase), the kernel's CUDA-event duration and the host wall clock per round.

The update phase re-reads r and h (8 B/row) and writes r' (4 B/row).  Each CTA carries its statistics pass's last tile
in registers and, with `fused_resident`, the groups before it in shared memory (`last_fused_resident_tiles` per CTA);
`phase_b_offchip_read_bytes` is what the update phase then still reads from the L2 or HBM."""
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from spark_ensemble_b200 import _native as N  # noqa: E402
from spark_ensemble_b200.context import Context  # noqa: E402

U, BLOCK = 4, 256  # float4 groups per thread per tile, threads per CTA (se_gbm_fused.cu)


def carried_float4s(n, grid, slots):
    """float4 groups of r (and as many of h) the update phase takes from registers or shared memory."""
    n4 = n // 4
    tile = U * BLOCK
    ntiles = math.ceil(n4 / tile)
    total = 0
    for b in range(min(grid, ntiles)):
        cnt = (ntiles - 1 - b) // grid + 1
        for p in range((cnt - 1) * U - min(slots, (cnt - 1) * U), cnt * U):
            i, u = divmod(p, U)
            total += max(0, min(BLOCK, n4 - ((b + i * grid) * tile + u * BLOCK)))
    return total


ctx = Context(0)
for n in (100_000_000, 50_000_000, 25_000_000, 12_500_000, 6_250_000):
    ctx.gbm_configure(n, 0, 1, "squared", 0.0, False)
    ctx.fill_synthetic(N.SLOT_Y, "normal", 1, 0.0, 1.0)
    ctx.fill_synthetic(N.SLOT_F, "normal", 2, 0.0, 0.5)
    ctx.copy_slot(N.SLOT_H, N.SLOT_Y)
    ctx.gbm_update([0.5], residual=False, loss=False)
    ctx.copy_slot(N.SLOT_H, N.SLOT_F)   # h = 0.5 y + N(0, 0.5)
    ctx.fill(N.SLOT_F, 0.0)
    ctx.gbm_pseudo_residuals(False)
    for fused, l2m, res in ((1, 0, 1), (1, 0, 0), (0, 0, 1)):
        ctx.set_option("fused_round", fused)
        ctx.set_option("fused_l2_mode", l2m)
        ctx.set_option("fused_resident", res)
        ctx.set_option("fused_timing", 0)
        for _ in range(5):
            ctx.gbm_round(0.01, True, 1e-6, 100, residual=True)
        ctx.sync()
        t0 = time.perf_counter()
        R = 200
        for _ in range(R):
            ctx.gbm_round(0.01, True, 1e-6, 100, residual=True)
        ctx.sync()
        wall = 1e6 * (time.perf_counter() - t0) / R
        ctx.kernel_timing(True); ctx.kernel_times_reset()
        for _ in range(50):
            ctx.gbm_round(0.01, True, 1e-6, 100, residual=True)
        kt = ctx.kernel_times(); ctx.kernel_timing(False)
        out = {"rows": n, "fused": fused, "l2_mode": l2m, "fused_resident": res, "wall_us_per_round": wall,
               "kernel_event_us": {k: 1e3 * v["ms"] / v["launches"] for k, v in kt.items()}}
        if fused:
            ctx.set_option("fused_timing", 1)
            ph = []
            for _ in range(100):
                _, _, ne = ctx.gbm_round(0.01, True, 1e-6, 100, residual=True)
                ph.append([ctx.get_option("last_fused_stats_us"), ctx.get_option("last_fused_brent_us"),
                           ctx.get_option("last_fused_update_us")])
            ph.sort(key=lambda p: sum(p))
            out["phases_us_median"] = ph[len(ph) // 2]
            out["brent_evals"] = ne
            grid, tiles = int(ctx.get_option("last_fused_grid")), ctx.get_option("last_fused_resident_tiles")
            carried = carried_float4s(n, grid, int(round(tiles * U)))
            out.update({"grid": grid, "last_fused_resident_tiles": tiles, "phase_b_carried_bytes": 32 * carried,
                        "phase_b_offchip_read_bytes": 8 * n - 32 * carried, "phase_b_write_bytes": 4 * n})
            ctx.set_option("fused_timing", 0)
        print(json.dumps(out), flush=True)
ctx.close()
