#!/usr/bin/env python
"""What leaving the residual pending costs and saves: carried squared-loss rounds store nothing (8 B/row instead of
12) until `sq_defer_max` steps are pending, and the first read of R applies them (a 12 B/row settle pass).

Every measurement alternates the settings in one process, three repeats each; times are CUDA events around the whole
sequence (us per round, or per sequence).

  * sweep: rounds over one direction with nothing read in between, sq_defer_max in {0, 4, 8, 16, 32}
  * k_then_read: K rounds over one direction, then one read of R (se_slot_sum: it settles, then reads 4 B/row)
  * round_then_read: a read of R after every round (the next carried round then stores: no settles)
  * new_direction: a fit's loop -- a new H (a copy into H), one round, one read of R -- which never runs a carried
    round and so never defers"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from spark_ensemble_b200 import _native as N  # noqa: E402
from spark_ensemble_b200.context import Context  # noqa: E402

LR, TOL = 0.1, 1e-6


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return q


def setup(ctx, n):
    """h = 0.5 y + N(0, 0.5), as bench.py builds it; a copy of h kept in SLOT_P for the new-direction loop."""
    ctx.gbm_configure(n, 0, 1, "squared", 0.0, False)
    ctx.fill_synthetic(N.SLOT_Y, "normal", 1, 0.0, 1.0)
    ctx.fill_synthetic(N.SLOT_F, "normal", 2, 0.0, 0.5)
    ctx.copy_slot(N.SLOT_H, N.SLOT_Y)
    ctx.gbm_update([0.5], residual=False, loss=False)
    ctx.copy_slot(N.SLOT_H, N.SLOT_F)
    ctx.fill(N.SLOT_F, 0.0)
    ctx.alloc(N.SLOT_P, 1, n)
    ctx.copy_slot(N.SLOT_P, N.SLOT_H)
    ctx.gbm_pseudo_residuals(False)


def rnd(ctx):
    ctx.gbm_round(LR, True, TOL, 100, residual=True)


def timed(ctx, fn, reps):
    ctx.sync()
    ctx.timer_start()
    for _ in range(reps):
        fn()
    ms = ctx.timer_stop()
    ctx.sync()
    return 1e3 * ms / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--quick", action="store_true", help="fewer rounds per measurement")
    args = ap.parse_args()
    ctx = Context(0)
    ctx.set_option("fused_round", 1)
    default = int(ctx.get_option("sq_defer_max"))
    print(json.dumps({"card": card(), "sq_defer_max_default": default}), flush=True)

    for n, reps in ((100_000_000, 40), (12_500_000, 200)):
        reps = max(4, reps // 10) if args.quick else reps
        setup(ctx, n)
        res = {}
        for _ in range(args.repeats):
            for m in (0, 4, 8, 16, 32):
                ctx.set_option("sq_defer_max", m)
                for _ in range(2 * m + 3):  # settles into the steady cycle of m deferred rounds and one flush
                    rnd(ctx)
                res.setdefault(m, []).append(timed(ctx, lambda: rnd(ctx), reps))
        print(json.dumps({"part": "sweep", "rows": n, "rounds": reps,
                          "us_per_round": {m: sorted(v) for m, v in res.items()},
                          "median_us": {m: statistics.median(v) for m, v in res.items()}}), flush=True)

    n = 100_000_000
    setup(ctx, n)

    def k_then_read(k):
        def seq():
            for _ in range(k):
                rnd(ctx)
            ctx.slot_sum(N.SLOT_R)
        return seq

    def round_then_read():
        rnd(ctx)
        ctx.slot_sum(N.SLOT_R)

    def new_direction():
        ctx.copy_slot(N.SLOT_H, N.SLOT_P)
        rnd(ctx)
        ctx.slot_sum(N.SLOT_R)

    cases = [("k_then_read", k, k_then_read(k), max(2, 40 // k)) for k in (1, 2, 4, 8, 20)]
    cases += [("round_then_read", 1, round_then_read, 20), ("new_direction", 1, new_direction, 20)]
    for part, k, fn, reps in cases:
        reps = max(2, reps // 4) if args.quick else reps
        res = {}
        for _ in range(args.repeats):
            for m in (0, default):
                ctx.set_option("sq_defer_max", m)
                fn()
                res.setdefault(m, []).append(timed(ctx, fn, reps))
        print(json.dumps({"part": part, "rows": n, "k": k, "sequences": reps,
                          "us_per_sequence": {m: sorted(v) for m, v in res.items()},
                          "median_us": {m: statistics.median(v) for m, v in res.items()}}), flush=True)
    ctx.set_option("sq_defer_max", default)
    ctx.close()


if __name__ == "__main__":
    main()
