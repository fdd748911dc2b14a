"""A residual-mode squared-loss round without a bag sums, in its update pass, the statistics Σr'², Σhr', Σh² of what
it writes.  The next round over the same direction takes them instead of running its statistics pass
(`last_round_stats_carried`), and every write of Y, F, R or H (or anything else that stops them describing the slots)
drops them.

A carried round's statistics are the same fp32 group sums added in another fp64 order, so alpha may differ from a
round that runs its statistics pass in the last bits; r' is then still the exact fp32 r - f32(lr alpha) h of the
round's own alpha."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LR = 0.7
TOL = 1e-6
K = 5
# 3: scalar tail only; 1001: less than one tile (n % 4 == 1); 40961: fewer tiles than CTAs; 10000001: several tiles
# per CTA, part of them in shared memory
SIZES = [3, 1001, 40961, 10_000_001]


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    c.set_option("fused_round", 1)
    yield c
    c.close()


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


def stats64(d, h):
    d, h = d64(d), d64(h)
    return np.array([np.sum(d * d), np.sum(h * d), np.sum(h * h)])


def round_stats(ctx):
    return np.array([ctx.get_option(f"last_round_stat{i}") for i in range(3)])


def check_oracle(a, loss, r_before, h, r_after):
    """fp64 oracle: the squared-loss objective along h is a parabola with its minimum at Σhr / Σh²."""
    s = stats64(r_before, h)
    a_o = min(max(s[1] / s[2], 0.0), 100.0) if s[2] > 0 else 1.0
    assert abs(a - a_o) <= 1e-5 * max(abs(a_o), 1e-3) + 4 * TOL, (a, a_o)
    l_o = 0.5 * float(np.sum(d64(r_after) ** 2))
    assert loss == pytest.approx(l_o, rel=1e-5, abs=1e-30)


def chain(ctx, y, F, h, refresh_h):
    """K rounds over one direction; refresh_h uploads the same H between rounds, which drops the carried
    statistics.  Returns per round (alpha, loss, evals, carried, launches, r before, r after)."""
    from spark_ensemble_b200 import _native as N
    start(ctx, y, F, h)
    out = []
    r = ctx.download(N.SLOT_R).copy()
    for _ in range(K):
        lc = ctx.launch_count
        a, loss, ne = ctx.gbm_round(LR, True, TOL, 100, residual=True)
        launches = ctx.launch_count - lc
        assert ctx.get_option("last_round_fused") == 1
        carried = int(ctx.get_option("last_round_stats_carried"))
        r_new = ctx.download(N.SLOT_R).copy()
        out.append((a, loss, ne, carried, launches, r, r_new))
        r = r_new
        if refresh_h:
            ctx.upload(N.SLOT_H, h)
    return out


@pytest.mark.parametrize("n", SIZES)
def test_rounds_over_one_direction_chain(ctx, n):
    y, F, h = problem(n, 2000 + n % 89)
    carried = chain(ctx, y, F, h, refresh_h=False)
    fresh = chain(ctx, y, F, h, refresh_h=True)
    assert [c[3] for c in carried] == [0] + [1] * (K - 1)
    assert [c[3] for c in fresh] == [0] * K
    same_so_far = True
    for k, (c, f) in enumerate(zip(carried, fresh)):
        a1, l1, _, _, launches, r0, r1 = c
        a0, l0, _, _, _, q0, q1 = f
        if k > 0:
            assert launches == 1, k
        # each path's r' is the exact fp32 update with its own alpha
        np.testing.assert_array_equal(r1, fma32(-f32(LR * a1), h, r0), err_msg=f"round {k}")
        np.testing.assert_array_equal(q1, fma32(-f32(LR * a0), h, q0), err_msg=f"round {k}")
        assert a1 == pytest.approx(a0, rel=1e-12, abs=1e-300), k
        assert l1 == pytest.approx(l0, rel=1e-12, abs=1e-300), k
        # r' differs only where a differing f32(lr alpha) was applied
        same_so_far = same_so_far and f32(LR * a1) == f32(LR * a0)
        if same_so_far:
            np.testing.assert_array_equal(r1, q1, err_msg=f"round {k}")
        else:
            assert np.all(np.abs(d64(r1) - d64(q1)) <= k * np.spacing(np.maximum(np.abs(r1), np.abs(q1)))), k
        check_oracle(a1, l1, r0, h, r1)


def settled(y, r):
    """What rebuilding the owed F leaves: F = y - r, then R = y - F (both fp32)."""
    F = f32(d64(y) - r)
    return F, f32(d64(y) - F)


def _upload_h(ctx, y, F, h, r):
    from spark_ensemble_b200 import _native as N
    ctx.upload(N.SLOT_H, h)
    return r


def _device_ptr_h(ctx, y, F, h, r):
    from spark_ensemble_b200 import _native as N
    ctx.device_ptr(N.SLOT_H)
    return r


def _device_ptr_r(ctx, y, F, h, r):
    from spark_ensemble_b200 import _native as N
    ctx.device_ptr(N.SLOT_R)
    return settled(y, r)[1]


def _upload_r(ctx, y, F, h, r):
    from spark_ensemble_b200 import _native as N
    ctx.upload(N.SLOT_R, r)  # the same bytes: the round then reads y - F
    return settled(y, r)[1]


def _upload_y(ctx, y, F, h, r):
    from spark_ensemble_b200 import _native as N
    ctx.upload(N.SLOT_Y, y)
    return settled(y, r)[1]


def _upload_f(ctx, y, F, h, r):
    from spark_ensemble_b200 import _native as N
    ctx.upload(N.SLOT_F, F)
    return f32(d64(y) - F)


def _read_f(ctx, y, F, h, r):
    from spark_ensemble_b200 import _native as N
    ctx.download(N.SLOT_F)  # rebuilds F and rewrites R as y - F
    return settled(y, r)[1]


def _configure(ctx, y, F, h, r):
    ctx.gbm_configure(len(y), 0, 1, "squared", 0.0, False)
    return settled(y, r)[1]


def _bag_off(ctx, y, F, h, r):
    ctx.gbm_set_bag(None)
    return r


def _loss_param(ctx, y, F, h, r):
    ctx.gbm_set_loss_param(0.0)
    return settled(y, r)[1]


def _update(ctx, y, F, h, r):
    ctx.gbm_update([0.0], residual=True, loss=False)
    return settled(y, r)[1]


def _pseudo_residuals(ctx, y, F, h, r):
    ctx.gbm_pseudo_residuals(False)
    return settled(y, r)[1]


def _failed_round(ctx, y, F, h, r):
    from spark_ensemble_b200 import _native as N
    with pytest.raises(N.ConvergenceError):
        ctx.gbm_round(LR, True, 1e-12, 2, residual=True)
    assert ctx.get_option("last_round_stats_carried") == 1  # it was carried itself, and its step was 0
    return r


def _eager_round(ctx, y, F, h, r):
    a, _, _ = ctx.gbm_round(LR, True, TOL, 100, residual=False)
    assert ctx.get_option("last_round_stats_carried") == 0
    F1 = fma32(f32(LR * a), h, settled(y, r)[0])
    return f32(d64(y) - F1)


def _async_round(ctx, y, F, h, r):
    from spark_ensemble_b200 import _native as N
    ctx.gbm_round_squared_async(LR)
    ctx.gbm_round_result()
    return ctx.download(N.SLOT_R).copy()


INVALIDATIONS = [_upload_h, _device_ptr_h, _device_ptr_r, _upload_r, _upload_y, _upload_f, _read_f, _configure,
                 _bag_off, _loss_param, _update, _pseudo_residuals, _failed_round, _eager_round, _async_round]


@pytest.mark.parametrize("invalidate", INVALIDATIONS, ids=lambda f: f.__name__.lstrip("_"))
def test_writes_drop_the_carried_statistics(ctx, invalidate):
    from spark_ensemble_b200 import _native as N
    n = 40961
    y, F, h = problem(n, 31)
    start(ctx, y, F, h)
    for k in range(2):
        ctx.gbm_round(LR, True, TOL, 100, residual=True)
        assert ctx.get_option("last_round_stats_carried") == k
    r = ctx.download(N.SLOT_R).copy()  # reading R keeps them
    d = invalidate(ctx, y, F, h, r)
    ctx.gbm_round(LR, True, TOL, 100, residual=True)
    assert ctx.get_option("last_round_fused") == 1
    assert ctx.get_option("last_round_stats_carried") == 0
    np.testing.assert_allclose(round_stats(ctx), stats64(d, h), rtol=1e-6)
    # the round that ran its statistics pass carries again
    r = ctx.download(N.SLOT_R).copy()
    ctx.gbm_round(LR, True, TOL, 100, residual=True)
    assert ctx.get_option("last_round_stats_carried") == 1
    np.testing.assert_allclose(round_stats(ctx), stats64(r, h), rtol=1e-6)


def test_bagged_and_row_reduced_rounds_carry_nothing(ctx):
    from spark_ensemble_b200 import _native as N
    n = 40961
    y, F, h = problem(n, 41)
    start(ctx, y, F, h)
    ctx.gbm_set_bag(f32(np.random.default_rng(42).poisson(1.0, n)))
    try:
        for _ in range(2):
            ctx.gbm_round(LR, True, TOL, 100, residual=True)
            assert ctx.get_option("last_round_stats_carried") == 0
    finally:
        ctx.gbm_set_bag(None)
    ctx.set_option("fused_loss_reduce", 1)
    try:
        for _ in range(2):
            r = ctx.download(N.SLOT_R).copy()
            ctx.gbm_round(LR, True, TOL, 100, residual=True)
            assert ctx.get_option("last_round_stats_carried") == 0
            np.testing.assert_allclose(round_stats(ctx), stats64(r, h), rtol=1e-6)
    finally:
        ctx.set_option("fused_loss_reduce", 0)


def test_carried_stats_describe_the_slots(ctx):
    """A carried round reports the statistics it used: fp64 sums over the r and h it read."""
    from spark_ensemble_b200 import _native as N
    n = 4_866_047
    y, F, h = problem(n, 51)
    start(ctx, y, F, h)
    ctx.gbm_round(LR, True, TOL, 100, residual=True)
    for _ in range(3):
        r = ctx.download(N.SLOT_R).copy()
        ctx.gbm_round(LR, True, TOL, 100, residual=True)
        assert ctx.get_option("last_round_stats_carried") == 1
        np.testing.assert_allclose(round_stats(ctx), stats64(r, h), rtol=1e-9)


def test_sharded_carried_rounds_agree():
    """Row-sharded rounds: each GPU carries its own sums and the round exchanges them once; alpha is the same on every
    rank and matches the fp64 oracle over the concatenated rows."""
    from spark_ensemble_b200 import _native as N
    if N.device_count() < 2:
        pytest.skip("needs two GPUs")
    from spark_ensemble_b200.sharded import ShardedContext
    n = 2_000_003
    y, F, h = problem(n, 61)
    with ShardedContext([0, 1]) as sc:
        if not sc.comm_p2p_active():
            pytest.skip("no peer-memory exchange between the GPUs")
        sc.set_option("fused_round", 1)
        start(sc, y, F, h)
        r = sc.download(N.SLOT_R).copy()
        for k in range(K):
            a, loss, _ = sc.gbm_round(LR, True, TOL, 100, residual=True)  # asserts that the ranks agree on alpha
            assert [int(c.get_option("last_round_stats_carried")) for c in sc.ctxs] == [int(k > 0)] * 2
            r_new = sc.download(N.SLOT_R).copy()
            np.testing.assert_array_equal(r_new, fma32(-f32(LR * a), h, r))
            check_oracle(a, loss, r, h, r_new)
            r = r_new
