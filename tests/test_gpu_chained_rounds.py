"""On one GPU a carried squared-loss round folds its predecessor's per-CTA statistics in every CTA and runs Brent
itself, so it is launched as a programmatic dependent of the kernel before it and may start while that kernel drains.
Nothing it computes may depend on how far the two overlap.

Each sequence of calls runs twice: back to back, and with ctx.sync() after every call, which leaves nothing to
overlap.  Alpha, the loss, the evaluation counts, every read of R, the sums and the final R and F must be the same bits,
and every R read must be the exact fp32 chain r <- fmaf(-c, h, r) of the steps c = (float)(lr * alpha) the rounds
reported.  The caps 0, 1, 2 and 16 make storing and deferring rounds alternate at different rates; the sequences
include a round after a new direction (statistics pass, then carried rounds), reads and sums of R, sums of Y and a
round that exceeds MaxEval."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LR = 0.7
TOL = 1e-6
CAPS = [0, 1, 2, 16]
# 1001: less than one tile; 409603: one tile per CTA on fewer CTAs than the GPU holds, n % 4 == 3; 4000001: several
# tiles per CTA, part of them in shared memory; 20000002: tens of millions of rows
SIZES = [1001, 409_603, 4_000_001, 20_000_002]
SEQ = (["round"] * 3 + ["ysum"] + ["round"] * 2 + ["rsum"] + ["round"] * 4 + ["fail"] + ["round"] * 3 + ["read_r"]
       + ["round"] * 2 + ["new_h"] + ["round"] * 19 + ["ysum", "round", "round", "read_r", "round", "rsum", "round"])


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    fused, m = c.get_option("fused_round"), c.get_option("sq_defer_max")
    c.set_option("fused_round", 1)
    yield c
    c.set_option("sq_defer_max", m)
    c.set_option("fused_round", fused)
    c.close()


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def d64(a):
    return np.asarray(a, dtype=np.float64)


def fma32(c, h, x):
    """fp32 fmaf(c, h, x): c h is exact in fp64, the sum is rounded to fp32."""
    return f32(d64(x) + d64(f32(c)) * d64(h))


def run(ctx, n, seed, synced):
    from spark_ensemble_b200 import _native as N
    rng = np.random.default_rng(seed)
    y = f32(rng.standard_normal(n))
    F = f32(0.7 * rng.standard_normal(n))
    h = f32(0.6 * (d64(y) - F) + 0.2 * rng.standard_normal(n))
    h2 = f32(0.3 * (d64(y) - F) + 0.1 * rng.standard_normal(n))
    ctx.gbm_configure(n, 0, 1, "squared", 0.0, False)
    ctx.upload(N.SLOT_Y, y)
    ctx.upload(N.SLOT_F, F)
    ctx.upload(N.SLOT_H, h)
    ctx.gbm_pseudo_residuals(False)
    ctx.sync()
    r = f32(d64(y) - d64(F))  # the fp32 chain of the reported steps
    hcur = h
    out, carried = [], 0
    for op in SEQ:
        if op == "round":
            a, loss, ne = ctx.gbm_round(LR, True, TOL, 100, residual=True)
            carried += int(ctx.get_option("last_round_stats_carried"))
            out.append((a, loss, ne, int(ctx.get_option("last_round_deferred"))))
            r = fma32(-f32(LR * a), hcur, r)
        elif op == "fail":
            with pytest.raises(N.ConvergenceError):
                ctx.gbm_round(LR, True, 1e-12, 1, residual=True)
            out.append(("fail", int(ctx.get_option("last_round_deferred"))))  # its 0 step leaves r as it was
        elif op == "read_r":
            got = ctx.download(N.SLOT_R).copy()
            np.testing.assert_array_equal(got, r)
            out.append(got)
        elif op == "rsum":
            out.append(ctx.slot_sum(N.SLOT_R))
        elif op == "ysum":
            out.append(ctx.slot_sum(N.SLOT_Y))
        elif op == "new_h":
            ctx.upload(N.SLOT_H, h2)
            hcur = h2
        if synced:
            ctx.sync()
    R = ctx.download(N.SLOT_R).copy()
    np.testing.assert_array_equal(R, r)
    return out, R, ctx.download(N.SLOT_F).copy(), carried


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("n", SIZES)
def test_back_to_back_equals_synced(ctx, cap, n):
    ctx.set_option("sq_defer_max", cap)
    out1, R1, F1, c1 = run(ctx, n, 1000 + n % 97, synced=False)
    out0, R0, F0, c0 = run(ctx, n, 1000 + n % 97, synced=True)
    assert c1 == c0 and c1 >= len([o for o in SEQ if o == "round"]) - 4  # rounds after a new direction or a failure
    assert len(out1) == len(out0)
    for a, b in zip(out1, out0):
        if isinstance(a, np.ndarray):
            np.testing.assert_array_equal(a, b)
        else:
            assert a == b
    np.testing.assert_array_equal(R1, R0)
    np.testing.assert_array_equal(F1, F0)
    deferred = [o[-1] for o in out1 if isinstance(o, tuple)]
    assert (max(deferred) == 0) == (cap == 0)
