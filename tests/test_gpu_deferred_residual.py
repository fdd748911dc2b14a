"""A carried squared-loss round (one over the direction of the round before it, with its statistics taken from that
round's update pass) may leave the residual slot pending: it stores nothing, and its fp32 step joins a chain on the
device that the next carried round applies in registers before its own.  The round that would exceed `sq_defer_max`
pending steps stores r' with all of them applied, and anything that reads R or F, or writes Y, F, R or H, settles
the chain first.

Each step is the fmaf(-c, h, r) a storing round applies, so every materialised R, and every alpha, loss and
evaluation count, must equal the rounds that store r' each time (sq_defer_max = 0) bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LR = 0.7
TOL = 1e-6
# 3: scalar tail only; 1001: less than one tile (n % 4 == 1); 40961: fewer tiles than CTAs; 10000001: several tiles
# per CTA, part of them in shared memory
SIZES = [3, 1001, 40961, 10_000_001]
N_SMALL = 40961
D = 3


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    c.set_option("fused_round", 1)
    yield c
    c.close()


@pytest.fixture
def cap(ctx):
    m = int(ctx.get_option("sq_defer_max"))
    assert m >= 2
    yield m
    ctx.set_option("sq_defer_max", m)


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def d64(a):
    return np.asarray(a, dtype=np.float64)


def fma32(c, h, x):
    """fp32 fmaf(c, h, x): c h is exact in fp64, the sum is rounded to fp32."""
    return f32(d64(x) + d64(f32(c)) * d64(h))


def problem(n, seed):
    rng = np.random.default_rng(seed)
    y = f32(rng.standard_normal(n))
    F = f32(0.7 * rng.standard_normal(n))
    h = f32(0.6 * (d64(y) - F) + 0.2 * rng.standard_normal(n))
    return y, F, h


def start(ctx, y, F, h):
    from spark_ensemble_b200 import _native as N
    ctx.gbm_configure(len(y), 0, 1, "squared", 0.0, False)
    ctx.upload(N.SLOT_Y, y)
    ctx.upload(N.SLOT_F, F)
    ctx.upload(N.SLOT_H, h)
    ctx.gbm_pseudo_residuals(False)


def rounds(ctx, k, read_r=False):
    """k rounds over the current direction; (alpha, loss, evaluations, deferred) per round."""
    from spark_ensemble_b200 import _native as N
    out = []
    for _ in range(k):
        a, loss, ne = ctx.gbm_round(LR, True, TOL, 100, residual=True)
        assert ctx.get_option("last_round_fused") == 1
        out.append((a, loss, ne, int(ctx.get_option("last_round_deferred"))))
        if read_r:
            ctx.download(N.SLOT_R)
    return out


@pytest.mark.parametrize("n", SIZES)
def test_deferred_rounds_are_bit_identical(ctx, cap, n):
    from spark_ensemble_b200 import _native as N
    y, F, h = problem(n, 3000 + n % 97)
    k = 2 * cap + 3
    runs = {}
    for name, m, read_r in (("deferred", cap, False), ("eager", 0, False), ("read_each", cap, True)):
        ctx.set_option("sq_defer_max", m)
        start(ctx, y, F, h)
        r0 = ctx.download(N.SLOT_R).copy()
        res = rounds(ctx, k, read_r)
        runs[name] = (res, r0, ctx.download(N.SLOT_R).copy(), ctx.download(N.SLOT_F).copy())
    res, r0, r, Fg = runs["deferred"]
    # the first carried round stores; then cap rounds defer, one flushes, cap more defer
    assert [x[3] for x in res] == [0, 0] + [1] * cap + [0] + [1] * cap
    assert all(x[3] == 0 for x in runs["eager"][0] + runs["read_each"][0])
    for other in ("eager", "read_each"):
        o_res, o_r0, o_r, o_F = runs[other]
        assert [x[:3] for x in res] == [x[:3] for x in o_res], other
        np.testing.assert_array_equal(r0, o_r0)
        np.testing.assert_array_equal(r, o_r, err_msg=other)
        np.testing.assert_array_equal(Fg, o_F, err_msg=other)
    want = r0
    for a, _, _, _ in res:
        want = fma32(-f32(LR * a), h, want)
    np.testing.assert_array_equal(r, want)


# ---- every way a pending R is settled, after a partial chain: the same calls on the eager path give the same bits
def _setup_features(ctx, n):
    from spark_ensemble_b200 import _native as N
    rng = np.random.default_rng(5)
    X = f32(rng.standard_normal((D, n)))
    ctx.alloc(N.SLOT_X, D, n)
    ctx.upload(N.SLOT_X, X)
    ctx.tree_fit_bins([np.unique(f32(np.quantile(X[j], np.linspace(0.05, 0.95, 15)))) for j in range(D)])
    ctx.alloc(N.SLOT_P, 1, n)


def _read_r(ctx, h):
    from spark_ensemble_b200 import _native as N
    return [ctx.download(N.SLOT_R).copy()]


def _read_f(ctx, h):
    from spark_ensemble_b200 import _native as N
    return [ctx.download(N.SLOT_F).copy()]


def _new_h(ctx, h):
    from spark_ensemble_b200 import _native as N
    ctx.upload(N.SLOT_H, f32(0.5 * d64(h) + 0.25))
    return [x[:3] for x in rounds(ctx, 3)]


def _device_ptr_r(ctx, h):
    from spark_ensemble_b200 import _native as N
    assert ctx.device_ptr(N.SLOT_R) != 0
    return []


def _device_ptr_h(ctx, h):
    from spark_ensemble_b200 import _native as N
    assert ctx.device_ptr(N.SLOT_H) != 0
    return []


def _update(ctx, h):
    ctx.gbm_update([0.3], residual=True, loss=False)
    return []


def _linesearch_eval(ctx, h):
    return list(ctx.gbm_linesearch_eval([0.4]))


def _pseudo_residuals(ctx, h):
    ctx.gbm_pseudo_residuals(False)
    return []


def _bagged_round(ctx, h):
    ctx.gbm_set_bag(f32(np.random.default_rng(9).poisson(1.0, N_SMALL)))
    try:
        return list(ctx.gbm_round(LR, True, TOL, 100, residual=True))
    finally:
        ctx.gbm_set_bag(None)


def _eager_round(ctx, h):
    return list(ctx.gbm_round(LR, True, TOL, 100, residual=False))


def _async_round(ctx, h):
    ctx.gbm_round_squared_async(LR)
    return list(ctx.gbm_round_result())


def _copy_slot(ctx, h):
    from spark_ensemble_b200 import _native as N
    ctx.copy_slot(N.SLOT_P, N.SLOT_R)
    return [ctx.download(N.SLOT_P).copy()]


def _tree_fit(ctx, h):
    from spark_ensemble_b200 import _native as N
    t = ctx.tree_fit(N.SLOT_R, 0, -1, 0, False, subspace=np.arange(D, dtype=np.int32), max_depth=3,
                     out_slot=N.SLOT_P)
    # the splits exactly; the fp64 node sums within their summation order
    return [t["feature"], t["threshold"], t["left"], t["right"],
            Approx(t["value"]), Approx(t["gain"]), Approx(ctx.download(N.SLOT_P).copy())]


class Approx:
    def __init__(self, a):
        self.a = np.asarray(a, dtype=np.float64)


def _configure(ctx, h):
    ctx.gbm_configure(N_SMALL, 0, 1, "squared", 0.0, False)
    return []


TRIGGERS = [_read_r, _read_f, _new_h, _device_ptr_r, _device_ptr_h, _update, _linesearch_eval, _pseudo_residuals,
            _bagged_round, _eager_round, _async_round, _copy_slot, _tree_fit, _configure]


@pytest.mark.parametrize("trigger", TRIGGERS, ids=lambda f: f.__name__.lstrip("_"))
def test_settle_triggers(ctx, cap, trigger):
    from spark_ensemble_b200 import _native as N
    y, F, h = problem(N_SMALL, 71)
    _setup_features(ctx, N_SMALL)
    seen = {}
    for m in (cap, 0):
        ctx.set_option("sq_defer_max", m)
        start(ctx, y, F, h)
        res = rounds(ctx, 5)  # FROM_R, a storing carried round, three deferred ones
        if m:
            assert [x[3] for x in res] == [0, 0, 1, 1, 1]
            assert ctx.get_option("r_pending") == 3
        out = trigger(ctx, h)
        assert ctx.get_option("r_pending") == 0 or trigger is _new_h
        after = [x[:3] for x in rounds(ctx, 2)]  # the state the trigger left carries on as the eager path's
        seen[m] = (res, out, after, ctx.download(N.SLOT_R).copy(), ctx.download(N.SLOT_F).copy())
    (res1, out1, after1, r1, F1), (res0, out0, after0, r0, F0) = seen[cap], seen[0]
    assert [x[:3] for x in res1] == [x[:3] for x in res0]
    assert len(out1) == len(out0)
    for a, b in zip(out1, out0):
        if isinstance(a, Approx):
            np.testing.assert_allclose(a.a, b.a, rtol=1e-9, atol=1e-12)
        else:
            np.testing.assert_array_equal(a, b)
    assert after1 == after0
    np.testing.assert_array_equal(r1, r0)
    np.testing.assert_array_equal(F1, F0)


def test_launch_counts(ctx, cap):
    from spark_ensemble_b200 import _native as N
    y, F, h = problem(N_SMALL, 81)
    start(ctx, y, F, h)
    rounds(ctx, 2)
    for k in range(cap + 1):
        lc = ctx.launch_count
        ctx.gbm_round(LR, True, TOL, 100, residual=True)
        assert ctx.launch_count == lc + 1, k  # deferring, and at k == cap flushing: one launch each
        assert ctx.get_option("last_round_deferred") == (1 if k < cap else 0), k
        assert ctx.get_option("r_pending") == (k + 1 if k < cap else 0), k
    rounds(ctx, 2)
    assert ctx.get_option("r_pending") == 2
    lc = ctx.launch_count
    ctx.download(N.SLOT_R)
    assert ctx.launch_count == lc + 1  # the settle
    lc = ctx.launch_count
    ctx.download(N.SLOT_R)
    assert ctx.launch_count == lc  # settled: a second read launches nothing
    # a round after a read of R stores: a caller that reads R every round pays no settles
    lc = ctx.launch_count
    assert rounds(ctx, 1)[0][3] == 0
    ctx.download(N.SLOT_R)
    assert ctx.launch_count == lc + 1


def test_failed_round_in_a_chain(ctx, cap):
    """MaxEval exceeded in the middle of a chain: the round's 0 step is part of it, and R ends as the eager path's."""
    from spark_ensemble_b200 import _native as N
    y, F, h = problem(N_SMALL, 91)
    seen = {}
    for m in (cap, 0):
        ctx.set_option("sq_defer_max", m)
        start(ctx, y, F, h)
        res = rounds(ctx, 4)
        with pytest.raises(N.ConvergenceError):
            ctx.gbm_round(LR, True, 1e-12, 1, residual=True)
        if m:
            assert ctx.get_option("last_round_deferred") == 1
            assert ctx.get_option("r_pending") == 3
        r = ctx.download(N.SLOT_R).copy()
        after = [x[:3] for x in rounds(ctx, 3)]
        seen[m] = (res, r, after, ctx.download(N.SLOT_R).copy(), ctx.download(N.SLOT_F).copy())
    for a, b in zip(seen[cap], seen[0]):
        if isinstance(a, np.ndarray):
            np.testing.assert_array_equal(a, b)
        else:
            assert [x[:3] for x in a] == [x[:3] for x in b]
