"""Every entry point that writes a caller-chosen slot drops what the context derived from the slot's old contents: the
line search's weight sum (W, BAG), the tree walks' rank matrix (X), se_download's 1/S factor (WOUT) and the labels'
class-index check (Y).  Each case writes a slot through one entry point and checks that the context then behaves as it
does after a plain upload of the same contents: how the contents got there must not matter."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_ROWS = 20011
D = 4
C = 2  # the column the probe tree splits on
CANDS = [0.25, 0.5, 0.75]  # the fit's split candidates of every column
PROBE = {"feature": [C, -1, -1], "threshold": [0.5, 0.0, 0.0], "left": [1, 0, 0], "right": [2, 0, 0],
         "value": [0.0, -1.0, 1.0]}
WRITERS = ["copy_slot", "upload_rowmajor", "linear_predict", "tree_predict", "forest_predict", "forest_median",
           "tree_fit"]


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    yield c
    c.close()


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def resident_features(ctx):
    """Uploads X (D x N_ROWS: column 0 holds 0 or 1, the others are uniform in [0, 1)) and the fit's candidates;
    allocates the scratch slots."""
    from spark_ensemble_b200 import _native as N
    X = f32(np.random.default_rng(5).random((D, N_ROWS)))
    X[0] = X[0] < 0.5
    for slot, rows in ((N.SLOT_X, D), (N.SLOT_VX, D), (N.SLOT_P, 1), (N.SLOT_PRED, 1)):
        ctx.alloc(slot, rows, N_ROWS)
    ctx.upload(N.SLOT_X, X)
    ctx.tree_fit_bins([CANDS] * D)
    return X


def step_tree(a, b):
    return {"feature": [0, -1, -1], "threshold": [0.5, 0.0, 0.0], "left": [1, 0, 0], "right": [2, 0, 0],
            "value": [0.0, a, b]}


def write(ctx, writer, X, slot, row, a, b):
    """Writes row `row` of `slot` through `writer`: a where column 0 of X is 0, b where it is 1.  The writers that
    read X read it from the device."""
    from spark_ensemble_b200 import _native as N
    want = f32(np.where(X[0] == 0, a, b))
    if writer in ("copy_slot", "upload_rowmajor"):
        rows = ctx.layout(slot)[0]
        full = ctx.download(slot).reshape(rows, N_ROWS) if rows > 1 else np.empty((1, N_ROWS), np.float32)
        full[row] = want
        if writer == "copy_slot":
            src = N.SLOT_VX if slot == N.SLOT_X else N.SLOT_PRED
            ctx.upload(src, full)
            ctx.copy_slot(slot, src)
        else:
            ctx.upload_rowmajor(slot, f32(full.T))
    elif writer == "linear_predict":
        ctx.linear_predict([b - a], a, slot, out_row=row, subspace=[0])
    elif writer == "tree_predict":
        ctx.tree_predict(step_tree(a, b), slot, out_row=row)
    elif writer == "forest_predict":
        ctx.forest_predict([step_tree(a, b)], slot, out_row=row)
    elif writer == "forest_median":
        ctx.forest_median([step_tree(a, b)], slot, [1.0], out_row=row)
    else:
        ctx.upload(N.SLOT_PRED, want)
        ctx.tree_fit(N.SLOT_PRED, subspace=[0], max_depth=1, out_slot=slot, out_row=row)


@pytest.mark.parametrize("writer", WRITERS)
@pytest.mark.parametrize("slot_name", ["SLOT_W", "SLOT_BAG"])
def test_weight_sum(ctx, writer, slot_name):
    from spark_ensemble_b200 import _native as N
    slot = getattr(N, slot_name)
    X = resident_features(ctx)
    rng = np.random.default_rng(11)
    ctx.gbm_configure(N_ROWS, 0, 1, "squared", 0.0, True)
    ctx.upload(N.SLOT_Y, f32(rng.standard_normal(N_ROWS)))
    ctx.upload(N.SLOT_F, f32(0.5 * rng.standard_normal(N_ROWS)))
    ctx.upload(N.SLOT_H, f32(rng.standard_normal(N_ROWS)))
    ctx.upload(N.SLOT_W, f32(rng.random(N_ROWS) + 0.1))
    if slot == N.SLOT_BAG:
        ctx.gbm_set_bag(f32(rng.poisson(1.0, N_ROWS)))
    try:
        ctx.gbm_linesearch_eval([0.4])  # the weight sum is computed here
        write(ctx, writer, X, slot, 0, 1.0, 2.0)
        got, _ = ctx.gbm_linesearch_eval([0.4])
        ctx.upload(slot, ctx.download(slot))
        want, _ = ctx.gbm_linesearch_eval([0.4])
        assert got == want
    finally:
        ctx.gbm_set_bag(None)


@pytest.mark.parametrize("writer", WRITERS)
def test_rank_matrix(ctx, writer):
    from spark_ensemble_b200 import _native as N
    X = resident_features(ctx)
    ctx.tree_predict(PROBE, N.SLOT_P)
    assert ctx.get_option("last_tree_binned") == 1
    # row C of X moves across the probe's threshold where column 0 does; the walkers walk X itself
    write(ctx, writer, X, N.SLOT_X, C, 0.25, 0.75)
    Xg = ctx.download(N.SLOT_X)
    host = np.where(Xg[C] <= 0.5, -1.0, 1.0).astype(np.float32)
    assert np.any(host != np.where(X[C] <= 0.5, -1.0, 1.0))
    ctx.tree_predict(PROBE, N.SLOT_P)
    assert ctx.get_option("last_tree_binned") == 1
    binned = ctx.download(N.SLOT_P).copy()
    ctx.set_option("tree_bins", 0)
    try:
        ctx.tree_predict(PROBE, N.SLOT_P)
        assert ctx.get_option("last_tree_binned") == 0
        fp32 = ctx.download(N.SLOT_P).copy()
    finally:
        ctx.set_option("tree_bins", 1)
    np.testing.assert_array_equal(fp32, host)
    np.testing.assert_array_equal(binned, host)


@pytest.mark.parametrize("writer", WRITERS)
def test_wout_scale(ctx, writer):
    from spark_ensemble_b200 import _native as N
    X = resident_features(ctx)
    rng = np.random.default_rng(13)
    ctx.gbm_configure(N_ROWS, 0, 1, "squared", 0.0, False)
    ctx.upload(N.SLOT_Y, f32(rng.standard_normal(N_ROWS)))
    ctx.upload(N.SLOT_F, f32(rng.standard_normal(N_ROWS)))
    ctx.upload(N.SLOT_H, f32(rng.standard_normal(N_ROWS)))
    ctx.gbm_pseudo_residuals(newton=True)  # WOUT is downloaded times 1/S from here on
    write(ctx, writer, X, N.SLOT_WOUT, 0, -0.75, 1.5)
    got = ctx.download(N.SLOT_WOUT).copy()
    write(ctx, writer, X, N.SLOT_P, 0, -0.75, 1.5)  # the same call into a slot nothing is derived from
    np.testing.assert_array_equal(got, ctx.download(N.SLOT_P))


@pytest.mark.parametrize("writer", WRITERS)
def test_label_check(ctx, writer):
    from spark_ensemble_b200 import _native as N
    X = resident_features(ctx)
    rng = np.random.default_rng(17)
    ctx.gbm_configure(N_ROWS, 0, 2, "logloss", 0.0, False)
    ctx.upload(N.SLOT_Y, f32(rng.random(N_ROWS) < 0.5))
    ctx.upload(N.SLOT_F, f32(rng.standard_normal((2, N_ROWS))))
    ctx.upload(N.SLOT_H, f32(rng.standard_normal((2, N_ROWS))))
    alpha = [0.3, -0.2]
    ctx.gbm_linesearch_eval(alpha)  # checks the labels

    def evaluate():
        lc = ctx.launch_count
        loss, grad = ctx.gbm_linesearch_eval(alpha)
        return ctx.launch_count - lc, loss, grad

    write(ctx, writer, X, N.SLOT_Y, 0, 0.0, 1.0)
    launches, loss, grad = evaluate()
    ctx.upload(N.SLOT_Y, ctx.download(N.SLOT_Y))
    want_launches, want_loss, want_grad = evaluate()
    assert launches == want_launches  # the validation pass included
    assert loss == want_loss
    np.testing.assert_array_equal(grad, want_grad)
