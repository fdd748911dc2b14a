"""The residual-mode squared-loss round in one launch (se_gbm_round, fused_round) updates only the residual:
r' = r - c h.  F is owed (F = y - r) and rebuilt the first time anything reads train F or writes Y, F or R.

These tests check the rows bit for bit against an fp32 emulation of the kernel arithmetic, that every read path sees
y - r, that reads of R, Y and H never rebuild F, and that writes, reconfiguration, bags and MaxEval keep F's value."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LR = 0.7
N_ROWS = 40961  # n % 4 == 1: the scalar tail of block 0 is covered
D = 4


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    c = Context(0)
    c.set_option("fused_round", 1)
    # resident features for the model writers, and a scratch row
    c.alloc(N.SLOT_X, D, N_ROWS)
    c.upload(N.SLOT_X, f32(np.random.default_rng(3).standard_normal((D, N_ROWS))))
    c.alloc(N.SLOT_P, 1, N_ROWS)
    yield c
    c.close()


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def d64(a):
    return np.asarray(a, dtype=np.float64)


def fma32(c, h, x):
    """fp32 fmaf(c, h, x): c h is exact in fp64, the sum is rounded to fp32."""
    return f32(d64(x) + d64(f32(c)) * d64(h))


def problem(ctx, seed, n=N_ROWS):
    from spark_ensemble_b200 import _native as N
    rng = np.random.default_rng(seed)
    y = f32(rng.standard_normal(n))
    F = f32(0.7 * rng.standard_normal(n))
    h = f32(0.6 * (d64(y) - F) + 0.2 * rng.standard_normal(n))
    ctx.gbm_configure(n, 0, 1, "squared", 0.0, False)
    ctx.upload(N.SLOT_Y, y)
    ctx.upload(N.SLOT_F, F)
    ctx.upload(N.SLOT_H, h)
    return y, F, h


def lazy_state(ctx, seed, rounds=2):
    """Rounds on a fresh problem; returns y, h, the residual slot (read without rebuilding F) and the owed F."""
    from spark_ensemble_b200 import _native as N
    y, _, h = problem(ctx, seed)
    for _ in range(rounds):
        ctx.gbm_round(LR, True, 1e-6, 100, residual=True)
        assert ctx.get_option("last_round_fused") == 1
    lc = ctx.launch_count
    r = ctx.download(N.SLOT_R).copy()
    assert ctx.launch_count == lc
    return y, h, r, f32(d64(y) - r)


@pytest.mark.parametrize("start", ["uploaded_F", "current_r"])
def test_lazy_rounds_bit_exact(ctx, start):
    from spark_ensemble_b200 import _native as N
    y, F, h = problem(ctx, 11)
    if start == "current_r":
        ctx.gbm_pseudo_residuals(False)
    r = f32(d64(y) - F)  # both starts: the first round's residual is fl(y - F)
    for k in range(4):
        alpha, _, _ = ctx.gbm_round(LR, True, 1e-6, 100, residual=True)
        r = fma32(-f32(LR * alpha), h, r)
        # the loop of a boosting fit: read R, write H, next round -- none of it rebuilds F
        lc = ctx.launch_count
        np.testing.assert_array_equal(ctx.download(N.SLOT_R), r)
        ctx.download(N.SLOT_Y)
        ctx.upload(N.SLOT_H, h)
        assert ctx.launch_count == lc, k
    lc = ctx.launch_count
    Fg = ctx.download(N.SLOT_F)
    assert ctx.launch_count == lc + 1  # one rebuild
    np.testing.assert_array_equal(Fg, f32(d64(y) - r))
    # R is re-derived from the rebuilt F, as an eager update of that F leaves it
    np.testing.assert_array_equal(ctx.download(N.SLOT_R), f32(d64(y) - Fg))
    lc = ctx.launch_count
    np.testing.assert_array_equal(ctx.download(N.SLOT_F), Fg)
    assert ctx.launch_count == lc  # settled: a second read launches nothing


def test_download_paths(ctx):
    from spark_ensemble_b200 import _native as N
    y, h, r, Fe = lazy_state(ctx, 21)
    np.testing.assert_array_equal(ctx.download(N.SLOT_F, count=1000, offset=37), Fe[37:1037])
    y, h, r, Fe = lazy_state(ctx, 21)
    np.testing.assert_array_equal(ctx.download(N.SLOT_F, scale=2.5), Fe * np.float32(2.5))
    y, h, r, Fe = lazy_state(ctx, 21)
    ctx.alloc(N.SLOT_BW, N_ROWS)
    ctx.copy_slot(N.SLOT_BW, N.SLOT_F)
    np.testing.assert_array_equal(ctx.download(N.SLOT_BW), Fe)
    y, h, r, Fe = lazy_state(ctx, 21)
    scale = float(np.sum(np.abs(d64(Fe))))
    assert ctx.slot_sum(N.SLOT_F) == pytest.approx(float(np.sum(d64(Fe))), rel=1e-6, abs=1e-6 * scale)
    y, h, r, Fe = lazy_state(ctx, 21)
    q = ctx.quantile(N.SLOT_F, 0.3)
    assert q == float(np.sort(Fe)[int(np.ceil(0.3 * N_ROWS)) - 1])
    y, h, r, Fe = lazy_state(ctx, 21)
    lc = ctx.launch_count
    assert ctx.device_ptr(N.SLOT_F) != 0
    assert ctx.launch_count == lc + 1
    np.testing.assert_array_equal(ctx.download(N.SLOT_F), Fe)


def test_gbm_reads_see_owed_F(ctx):
    from spark_ensemble_b200 import _native as N
    y, h, r, Fe = lazy_state(ctx, 31)
    d = d64(y) - d64(Fe)
    assert ctx.gbm_mean_loss() == pytest.approx(0.5 * np.mean(d * d), rel=1e-6)

    y, h, r, Fe = lazy_state(ctx, 31)
    a = 0.37
    loss, _ = ctx.gbm_linesearch_eval([a])
    e = d64(y) - d64(fma32(a, h, Fe))  # y - (F + a h), F + a h in fp32 as the evaluation forms it
    assert loss == pytest.approx(0.5 * np.mean(e * e), rel=1e-6)

    y, h, r, Fe = lazy_state(ctx, 31)
    ctx.gbm_update([0.25], residual=True, loss=False)
    np.testing.assert_allclose(ctx.download(N.SLOT_F), fma32(0.25, h, Fe), rtol=1e-6, atol=1e-6)

    # the two-launch round and the async round both start from F = y - r
    for mode in ("two_launch", "async"):
        y, h, r, Fe = lazy_state(ctx, 31)
        d = d64(y) - d64(Fe)
        star = float(np.clip(np.sum(d64(h) * d) / np.sum(d64(h) ** 2), 0.0, 100.0))
        if mode == "async":
            ctx.gbm_round_squared_async(LR)
            alpha, _ = ctx.gbm_round_result()
        else:
            ctx.set_option("fused_round", 0)
            try:
                alpha, _, _ = ctx.gbm_round(LR, True, 1e-6, 100, residual=True)
            finally:
                ctx.set_option("fused_round", 1)
            assert ctx.get_option("last_round_fused") == 0
        assert alpha == pytest.approx(star, rel=1e-5), mode
        Fo = d64(Fe) + LR * alpha * d64(h)
        np.testing.assert_allclose(ctx.download(N.SLOT_F), Fo, rtol=1e-5, atol=1e-5 * np.sqrt(np.mean(Fo * Fo)),
                                   err_msg=mode)


TREE = {"feature": [1, -1, -1], "threshold": [0.25, 0.0, 0.0], "left": [1, 0, 0], "right": [2, 0, 0],
        "value": [0.0, -1.25, 2.5]}
TREE2 = {"feature": [0, 3, -1, -1, -1], "threshold": [-0.5, 0.75, 0.0, 0.0, 0.0], "left": [1, 2, 0, 0, 0],
         "right": [4, 3, 0, 0, 0], "value": [0.0, 0.0, 1.5, -0.5, 0.75]}
WHOLE_ROW = ("copy_slot", "linear_predict", "tree_predict", "forest_predict")


def write(ctx, op, slot, lo, cnt):
    """Writes elements [lo, lo + cnt) of the [1][n] slot through `op` (the whole-row writers: all of them)."""
    from spark_ensemble_b200 import _native as N
    vals = np.linspace(-3.0, 3.0, cnt)
    if op == "upload":
        ctx.upload(slot, f32(vals), offset=lo)
    elif op == "upload_f64":
        ctx.upload(slot, vals, offset=lo)
    elif op == "upload_rowmajor":
        ctx.upload_rowmajor(slot, f32(vals).reshape(-1, 1), row_offset=lo)
    elif op == "fill":
        ctx.fill(slot, 1.5, count=cnt, offset=lo)
    elif op == "fill_synthetic":
        ctx.fill_synthetic(slot, "normal", 7, 0.5, 2.0, count=cnt, offset=lo)
    elif op == "copy_slot":
        ctx.copy_slot(slot, N.SLOT_P)
    elif op == "linear_predict":
        ctx.linear_predict([0.5, -2.0], 0.25, slot, subspace=[0, 2])
    elif op == "tree_predict":
        ctx.tree_predict(TREE, slot)
    else:
        ctx.forest_predict([TREE, TREE2], slot, weights=[0.5, 1.5], init=0.125)


@pytest.mark.parametrize("slot_name", ["SLOT_Y", "SLOT_R", "SLOT_F"])
@pytest.mark.parametrize("op", ["upload", "fill", "upload_f64", "upload_rowmajor", "fill_synthetic"] + list(WHOLE_ROW))
def test_partial_write_keeps_owed_rows(ctx, slot_name, op):
    from spark_ensemble_b200 import _native as N
    slot = getattr(N, slot_name)
    lo, cnt = (0, N_ROWS) if op in WHOLE_ROW else (1001, 500)
    # what the call writes, from the same call into a slot nothing is derived from (copy_slot copies that slot)
    write(ctx, "upload" if op == "copy_slot" else op, N.SLOT_P, lo, cnt)
    vals = ctx.download(N.SLOT_P, count=cnt, offset=lo).copy()
    y, h, r, Fe = lazy_state(ctx, 41)
    write(ctx, op, slot, lo, cnt)
    want = Fe.copy()
    if slot == N.SLOT_F:
        want[lo:lo + cnt] = vals
    np.testing.assert_array_equal(ctx.download(N.SLOT_F), want)
    # the next round starts from the slots as they are now (F, and the written Y), not from the stale residual
    yy = y.copy()
    if slot == N.SLOT_Y:
        yy[lo:lo + cnt] = vals
    alpha, _, _ = ctx.gbm_round(LR, True, 1e-6, 100, residual=True)
    d = d64(yy) - d64(want)
    assert ctx.get_option("last_round_stat1") == pytest.approx(float(np.sum(d64(h) * d)), rel=1e-6)
    Fo = d64(want) + LR * alpha * d64(h)
    np.testing.assert_allclose(ctx.download(N.SLOT_F), Fo, rtol=1e-5, atol=1e-5)


def test_reconfigure_keeps_owed_F(ctx):
    from spark_ensemble_b200 import _native as N
    y, h, r, Fe = lazy_state(ctx, 51)
    ctx.gbm_configure(N_ROWS, 0, 1, "squared", 0.0, False)
    np.testing.assert_array_equal(ctx.download(N.SLOT_F), Fe)
    np.testing.assert_array_equal(ctx.download(N.SLOT_Y), y)


def test_bag_round_is_lazy(ctx):
    from spark_ensemble_b200 import _native as N
    y, F, h = problem(ctx, 61)
    rng = np.random.default_rng(62)
    ctx.gbm_set_bag(f32(rng.poisson(1.0, N_ROWS)))
    try:
        r = f32(d64(y) - F)
        for _ in range(2):
            alpha, loss_sum, _ = ctx.gbm_round(0.5, True, 1e-6, 100, residual=True)
            r = fma32(-f32(0.5 * alpha), h, r)
            rg = ctx.download(N.SLOT_R)
            np.testing.assert_array_equal(rg, r)
            # the loss is reduced over all rows: Σ r'²/2
            assert loss_sum == pytest.approx(0.5 * float(np.sum(d64(r) ** 2)), rel=1e-6)
        np.testing.assert_array_equal(ctx.download(N.SLOT_F), f32(d64(y) - r))
    finally:
        ctx.gbm_set_bag(None)


def test_maxeval_leaves_F_and_R(ctx):
    from spark_ensemble_b200 import _native as N
    y, h, r, Fe = lazy_state(ctx, 71)
    with pytest.raises(N.ConvergenceError):
        ctx.gbm_round(LR, True, 1e-12, 2, residual=True)
    np.testing.assert_array_equal(ctx.download(N.SLOT_R), r)
    np.testing.assert_array_equal(ctx.download(N.SLOT_F), Fe)
    # and from a settled F: neither slot moves, and F stays current (a download rebuilds nothing)
    Fs, rs = ctx.download(N.SLOT_F).copy(), ctx.download(N.SLOT_R).copy()
    with pytest.raises(N.ConvergenceError):
        ctx.gbm_round(LR, True, 1e-12, 2, residual=True)
    lc = ctx.launch_count
    np.testing.assert_array_equal(ctx.download(N.SLOT_F), Fs)
    assert ctx.launch_count == lc
    np.testing.assert_array_equal(ctx.download(N.SLOT_R), rs)
