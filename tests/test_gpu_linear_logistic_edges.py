"""se_linear_moments, se_logistic_stats, se_logistic_loss_grad, se_logistic_predict and se_copy_rows at the shapes where
their kernels change: every side of a kernel switch or tile edge, p = 0, ragged row counts, label and weight rows
other than row 0 of multi-row slots (ld != n), labels outside 0..K-1, output rows other than row 0 of wider slots
(every other row must keep its sentinel bits), tied and non-finite margins, and the row-copy errors.  The sums are
checked against the fp64 numpy contracts of oracle/np_linear.py and oracle/np_logistic.py at 1e-12 of the sums of
absolute terms, and repeated calls must give identical bits."""
import numpy as np
import pytest

from oracle import np_linear
from oracle import np_logistic as O

pytestmark = pytest.mark.gpu

SENTINEL = np.float32(-1.2345678e9)


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    yield c
    c.close()


def _put_rows(ctx, slot, rows, n, values, rng):
    """A [rows][n] slot whose row r holds values[r] where given and unrelated data elsewhere: a kernel that addresses a
    row by the wrong stride reads the wrong numbers."""
    ctx.alloc(slot, rows, n)
    data = (rng.uniform(-7, 9, (rows, n))).astype(np.float32)
    for r, v in values.items():
        data[r] = v
    ctx.upload(slot, data)


def _load_x(ctx, src, X):
    from spark_ensemble_b200 import _native as N
    n, d = X.shape
    ctx.alloc(src, d, n)
    if src == N.SLOT_X:
        ctx.upload_rowmajor(src, X)
    else:
        ctx.upload(src, np.ascontiguousarray(X.T))


# ---- se_linear_moments ------------------------------------------------------------------------------------------------
# m = p + 2 on each side of the register kernel (m <= 8) and of the 64-wide output tiles (m = 64 | 65, 128 | 129)
MOMENT_P = [0, 6, 7, 62, 63, 64, 126, 127]


def _moments_case(n, p, seed):
    rng = np.random.default_rng(seed)
    d = max(p + 3, 2)
    X = (rng.standard_normal((n, d)) * 2 + 5).astype(np.float32)
    y = (rng.standard_normal(n) + 10).astype(np.float32)
    w = rng.uniform(0, 3, n).astype(np.float32)
    w[rng.random(n) < 0.3] = 0.0
    bag = rng.integers(0, 11, n).astype(np.float32)  # zeros and multiplicities up to 10
    cols = rng.integers(0, d, p).astype(np.int32)  # unsorted, with repeats
    if p > 1:
        cols[-1] = cols[0]
    shift = X[0, cols].astype(np.float64) + 0.25
    return rng, X, y, w, bag, cols, shift, float(y[0]) - 0.5


def _moments_check(ctx, src, X, y, cols, shift, ys, w, bag, label=(None, 0), weight=(None, 0)):
    from spark_ensemble_b200 import _native as N
    lslot, lrow = label
    wslot, wrow = weight
    args = (src, cols, N.SLOT_Y if lslot is None else lslot, lrow,
            -1 if w is None else (N.SLOT_W if wslot is None else wslot), wrow, bag is not None, shift, ys)
    got = ctx.linear_moments(*args)
    ref = np_linear.linear_moments(X, y, cols, w, bag, shift, ys)
    scale = np_linear.abs_moments(X, y, cols, w, bag, shift, ys)
    err = np.abs(got - ref) / np.maximum(scale, 1e-300)
    assert err.max() <= 1e-12, float(err.max())
    np.testing.assert_array_equal(got, got.T)
    again = ctx.linear_moments(*args)
    assert again.tobytes() == got.tobytes(), "two identical calls differ"


@pytest.mark.parametrize("n", [1, 3, 33, 4099])
@pytest.mark.parametrize("p", MOMENT_P)
def test_moments_at_kernel_and_tile_edges(ctx, n, p):
    from spark_ensemble_b200 import _native as N
    rng, X, y, w, bag, cols, shift, ys = _moments_case(n, p, n * 1009 + p)
    for i, (ww, bb) in enumerate(((w, None), (None, bag), (w, bag))):
        src = (N.SLOT_X, N.SLOT_P)[(i + p) % 2]
        _load_x(ctx, src, X)
        ctx.alloc(N.SLOT_Y, n)
        ctx.upload(N.SLOT_Y, y)
        if ww is not None:
            ctx.alloc(N.SLOT_W, n)
            ctx.upload(N.SLOT_W, ww)
        if bb is not None:
            ctx.alloc(N.SLOT_BAG, n)
            ctx.upload(N.SLOT_BAG, bb)
        _moments_check(ctx, src, X, y, cols, shift, ys, ww, bb)


@pytest.mark.parametrize("p", [6, 7, 63])
def test_moments_read_label_and_weight_rows_of_multirow_slots(ctx, p):
    """Labels in row 2 of a 4-row slot and weights in row 3 (then 1) of another, at n = 4099 (ld = 4128)."""
    from spark_ensemble_b200 import _native as N
    n = 4099
    rng, X, y, w, bag, cols, shift, ys = _moments_case(n, p, 77 + p)
    _load_x(ctx, N.SLOT_X, X)
    ctx.alloc(N.SLOT_BAG, n)
    ctx.upload(N.SLOT_BAG, bag)
    assert ctx.layout(N.SLOT_X)[2] != n
    _put_rows(ctx, N.SLOT_PROB, 4, n, {2: y}, rng)
    for wrow in (3, 1):
        _put_rows(ctx, N.SLOT_RAW, 4, n, {wrow: w}, rng)
        for bb in (None, bag):
            _moments_check(ctx, N.SLOT_X, X, y, cols, shift, ys, w, bb, label=(N.SLOT_PROB, 2),
                           weight=(N.SLOT_RAW, wrow))


def test_moments_near_a_million_rows_at_m_9(ctx):
    from spark_ensemble_b200 import _native as N
    n = 1_000_003
    rng, X, y, w, bag, cols, shift, ys = _moments_case(n, 7, 5)
    _load_x(ctx, N.SLOT_P, X)
    ctx.alloc(N.SLOT_Y, n)
    ctx.upload(N.SLOT_Y, y)
    _put_rows(ctx, N.SLOT_RAW, 2, n, {1: w}, rng)
    ctx.alloc(N.SLOT_BAG, n)
    ctx.upload(N.SLOT_BAG, bag)
    _moments_check(ctx, N.SLOT_P, X, y, cols, shift, ys, w, bag, weight=(N.SLOT_RAW, 1))


# ---- se_logistic_loss_grad --------------------------------------------------------------------------------------------
def _lg_case(n, p, D, seed):
    rng = np.random.default_rng(seed)
    d = max(p + 3, 2)
    X = (rng.standard_normal((n, d)) * 2 + 5).astype(np.float32)
    y = rng.integers(0, max(D, 2), n).astype(np.float32)
    w = rng.uniform(0, 3, n).astype(np.float32)
    w[rng.random(n) < 0.2] = 0.0
    cols = rng.integers(0, d, p).astype(np.int32)
    if p > 1:
        cols[-1] = cols[0]
    shift = X[0, cols].astype(np.float64) + 0.25
    scale = rng.uniform(0.2, 1.5, p)
    scale[rng.random(p) < 0.2] = 0.0
    coef = rng.standard_normal((D, p + 1)) * (2.0 / np.sqrt(p + 1))
    return rng, X, y, w, cols, shift, scale, coef


def _lg_check(ctx, src, X, y, w, cols, shift, scale, coef, label=(None, 0), weight=(None, 0)):
    from spark_ensemble_b200 import _native as N
    lslot, lrow = label
    wslot, wrow = weight
    args = (src, cols, coef, N.SLOT_Y if lslot is None else lslot, lrow,
            -1 if w is None else (N.SLOT_W if wslot is None else wslot), wrow, shift, scale)
    loss, g = ctx.logistic_loss_grad(*args)
    rl, rg = O.loss_grad(X, y, cols, coef, w, shift, scale)
    sl, sg = O.abs_terms(X, y, cols, coef, w, shift, scale)
    assert abs(loss - rl) <= 1e-12 * sl, (loss, rl, sl)
    err = np.abs(g - rg) / np.maximum(sg, 1e-300)
    assert err.max() <= 1e-12, float(err.max())
    again = ctx.logistic_loss_grad(*args)
    assert again[0] == loss and again[1].tobytes() == g.tobytes(), "two identical calls differ"


def _lg_run(ctx, n, p, D, seed, weighted=(False, True)):
    from spark_ensemble_b200 import _native as N
    rng, X, y, w, cols, shift, scale, coef = _lg_case(n, p, D, seed)
    if D == 1:
        y = (y > 0).astype(np.float32)
    ctx.alloc(N.SLOT_Y, n)
    ctx.upload(N.SLOT_Y, y)
    ctx.alloc(N.SLOT_W, n)
    ctx.upload(N.SLOT_W, w)
    for i, use_w in enumerate(weighted):
        src = (N.SLOT_X, N.SLOT_P)[(i + p + D) % 2]
        _load_x(ctx, src, X)
        _lg_check(ctx, src, X, y, w if use_w else None, cols, shift, scale, coef)


# (D, p + 1): the register kernels' widths at D = 1 (16 | 17, 40 | 41), then each side of the tiled kernel's j-tile
# TJ = 4·(256 / nk): 128 at D <= 32, 64 at D <= 64; for D <= 16 the tile is wider than the 255 columns allowed
LG_SHAPES = [(1, 1), (1, 16), (1, 17), (1, 40), (1, 41), (5, 255), (8, 255), (17, 128), (17, 129), (32, 128),
             (32, 129), (33, 64), (33, 65), (64, 64), (64, 65)]


@pytest.mark.parametrize("n", [3, 4099])
@pytest.mark.parametrize("D,P1", LG_SHAPES)
def test_loss_grad_at_kernel_and_tile_edges(ctx, n, D, P1):
    _lg_run(ctx, n, P1 - 1, D, n * 31 + D * 1000 + P1)


@pytest.mark.parametrize("D", [4, 5, 8, 9, 16])
def test_loss_grad_lane_and_class_tile_switches(ctx, D):
    """The lanes per margin L and the class rows nk change at D = 4, 5, 8, 9 and 16 (at p + 1 = 49)."""
    _lg_run(ctx, 4099, 48, D, 500 + D)


@pytest.mark.parametrize("D", [1, 7])
def test_loss_grad_without_columns(ctx, D):
    _lg_run(ctx, 1027, 0, D, 600 + D)


@pytest.mark.parametrize("D", [1, 2, 6, 40])
def test_loss_grad_labels_outside_the_classes(ctx, D):
    """Labels K, -1, 0.5 and NaN match no class (the contract's loss for them); no kernel indexes memory by a label."""
    from spark_ensemble_b200 import _native as N
    p = {1: 10, 2: 39, 6: 60, 40: 20}[D]
    n = 2051
    rng, X, y, w, cols, shift, scale, coef = _lg_case(n, p, D, 700 + D)
    K = max(D, 2)
    if D == 1:
        y = (y > 0).astype(np.float32)
    bad = rng.choice(n, 400, replace=False)
    y[bad] = np.array([K, -1, 0.5, np.nan], np.float32)[np.arange(bad.size) % 4]
    ctx.alloc(N.SLOT_Y, n)
    ctx.upload(N.SLOT_Y, y)
    ctx.alloc(N.SLOT_W, n)
    ctx.upload(N.SLOT_W, w)
    _load_x(ctx, N.SLOT_X, X)
    _lg_check(ctx, N.SLOT_X, X, y, w, cols, shift, scale, coef)


@pytest.mark.parametrize("D,p", [(1, 10), (1, 30), (1, 60), (3, 20), (64, 64)])
def test_loss_grad_reads_label_and_weight_rows_of_multirow_slots(ctx, D, p):
    from spark_ensemble_b200 import _native as N
    n = 4099
    rng, X, y, w, cols, shift, scale, coef = _lg_case(n, p, D, 800 + D + p)
    if D == 1:
        y = (y > 0).astype(np.float32)
    _load_x(ctx, N.SLOT_X, X)
    _put_rows(ctx, N.SLOT_PROB, 3, n, {1: y}, rng)
    _put_rows(ctx, N.SLOT_RAW, 4, n, {3: w}, rng)
    _lg_check(ctx, N.SLOT_X, X, y, w, cols, shift, scale, coef, label=(N.SLOT_PROB, 1), weight=(N.SLOT_RAW, 3))


# ---- se_logistic_stats ------------------------------------------------------------------------------------------------
def _stats_scale(X, y, cols, K, w, shift):
    """Σ|term| of every entry of the statistics."""
    c = np.abs(np.ones(y.size) if w is None else np.asarray(w, dtype=np.float64))
    Dv = np.abs(np.asarray(X, dtype=np.float64)[:, cols] - shift)
    return np.concatenate([[c.sum(), (c * c).sum()], (c[:, None] * Dv).sum(axis=0),
                           (c[:, None] * Dv * Dv).sum(axis=0), np.full(K, c.sum()), [0.0]])


@pytest.mark.parametrize("K", [1, 2, 64])
@pytest.mark.parametrize("p", [0, 1, 254])
@pytest.mark.parametrize("n", [33, 20_011])
def test_stats_ragged_rows_and_multirow_slots(ctx, n, p, K):
    """Labels in row 2 and weights in row 1 of multi-row slots; one bad label in the last, partial 32-row step of the
    last CTA must be counted and must stay out of the class histogram."""
    from spark_ensemble_b200 import _native as N
    rng = np.random.default_rng(n + 10 * p + K)
    d = p + 2
    X = (rng.standard_normal((n, d)) * 3 + 2).astype(np.float32)
    y = rng.integers(0, K, n).astype(np.float32)
    w = rng.uniform(0, 2, n).astype(np.float32)
    w[rng.random(n) < 0.1] = 0.0
    cols = rng.integers(0, d, p).astype(np.int32)
    shift = X[0, cols].astype(np.float64)
    _load_x(ctx, (N.SLOT_X, N.SLOT_P)[p % 2], X)
    src = (N.SLOT_X, N.SLOT_P)[p % 2]
    for bad in (False, True):
        yy = y.copy()
        if bad:
            yy[n - 1] = K
        _put_rows(ctx, N.SLOT_PROB, 3, n, {2: yy}, rng)
        _put_rows(ctx, N.SLOT_RAW, 2, n, {1: w}, rng)
        for ww in (None, w):
            got = ctx.logistic_stats(src, cols, K, N.SLOT_PROB, 2, -1 if ww is None else N.SLOT_RAW, 1, shift)
            ref = O.stats(X, yy, cols, K, ww, shift)
            scale = _stats_scale(X, yy, cols, K, ww, shift)
            assert got[-1] == ref[-1] == (1 if bad else 0)
            err = np.abs(got - ref) / np.maximum(scale, 1e-300)
            assert err.max() <= 1e-12, float(err.max())
            again = ctx.logistic_stats(src, cols, K, N.SLOT_PROB, 2, -1 if ww is None else N.SLOT_RAW, 1, shift)
            assert again.tobytes() == got.tobytes(), "two identical calls differ"


def test_stats_count_a_bad_weight_and_feature_in_the_last_partial_step(ctx):
    from spark_ensemble_b200 import _native as N
    n, K = 100_003, 3
    rng = np.random.default_rng(9)
    X = rng.standard_normal((n, 5)).astype(np.float32)
    y = rng.integers(0, K, n).astype(np.float32)
    w = rng.uniform(0, 2, n).astype(np.float32)
    cols = np.array([4, 0, 2], np.int32)
    w[n - 2] = np.nan
    X[n - 1, 2] = np.inf
    X[n - 3, 1] = np.nan  # a column outside the list does not count
    _load_x(ctx, N.SLOT_X, X)
    ctx.alloc(N.SLOT_Y, n)
    ctx.upload(N.SLOT_Y, y)
    ctx.alloc(N.SLOT_W, n)
    ctx.upload(N.SLOT_W, w)
    got = ctx.logistic_stats(N.SLOT_X, cols, K, N.SLOT_Y, 0, N.SLOT_W, 0, None)
    assert got[-1] == O.stats(X, y, cols, K, w)[-1] == 2


# ---- se_logistic_predict ----------------------------------------------------------------------------------------------
def _predict_into(ctx, model, X, sub, outputs, n_rows=6):
    """Scores model over SLOT_X = X with column j of the model at column sub[j]; outputs maps kind -> (slot, row).
    Every output slot is [n_rows][n] filled with SENTINEL first.  Returns {kind: [width][n]} and the slots' contents."""
    from spark_ensemble_b200 import _native as N
    n = X.shape[0]
    _load_x(ctx, N.SLOT_X, X)
    for slot in {s for s, _ in outputs.values()}:
        ctx.alloc(slot, n_rows, n)
        ctx.fill(slot, float(SENTINEL))
    ctx.logistic_predict(model.coefficientMatrix, model.interceptVector, model.threshold, subspace=sub,
                         **{k: v for k, v in outputs.items()})
    W = 2 if model.coefficientMatrix.shape[0] == 1 else model.coefficientMatrix.shape[0]
    slots = {s: ctx.download(s).reshape(n_rows, n) for s in {s for s, _ in outputs.values()}}
    got, written = {}, {s: np.zeros(n_rows, bool) for s in slots}
    for kind, (s, r) in outputs.items():
        width = 1 if kind == "label" else W
        got[kind] = slots[s][r:r + width]
        written[s][r:r + width] = True
    for s, rows in slots.items():
        untouched = rows[~written[s]]
        assert untouched.tobytes() == np.full(untouched.shape, SENTINEL, np.float32).tobytes(), f"slot {s}: other rows"
    return got


def _host_check(model, Xs, got):
    """The tolerances of test_gpu_logistic_fit.test_predict_matches_host_model."""
    D = model.coefficientMatrix.shape[0]
    n = Xs.shape[0]
    scale = np.abs(Xs.astype(np.float64)) @ np.abs(model.coefficientMatrix.T) + np.abs(model.interceptVector)
    if "raw" in got:
        raw = got["raw"].T
        ref = model.predictRaw(Xs)
        fin = np.isfinite(ref)
        tol = 4 * 2.0 ** -24 * (np.tile(scale, (1, 2)) if D == 1 else scale)
        assert np.all(np.abs(raw[fin] - ref[fin]) <= tol[fin])
        np.testing.assert_array_equal(raw[~fin], ref[~fin])
    if "prob" in got:
        np.testing.assert_allclose(got["prob"].T, model.predictProbability(Xs), rtol=0, atol=1e-6)
    if "label" in got:
        lab = got["label"][0]
        ref = model.predict(Xs)
        close = np.zeros(n, bool)
        if D == 1:
            close = np.abs(model.predictProbability(Xs)[:, 1] - model.threshold) < 1e-6
        else:
            M = np.sort(model._margins(Xs), axis=1)
            with np.errstate(invalid="ignore"):  # infinite margins: no tie
                close = (M[:, -1] - M[:, -2]) <= 1e-9 * (1.0 + np.abs(M[:, -1]))
        np.testing.assert_array_equal(lab[~close], ref[~close])
        assert close.sum() <= max(2, n // 1000), int(close.sum())


def _predict_outputs():
    from spark_ensemble_b200 import _native as N
    return [{"raw": (N.SLOT_RAW, 1)}, {"prob": (N.SLOT_PROB, 3)}, {"label": (N.SLOT_P, 4)},
            {"raw": (N.SLOT_P, 1), "prob": (N.SLOT_PROB, 2), "label": (N.SLOT_RAW, 5)}]


@pytest.mark.parametrize("D", [1, 2, 5, 64])
@pytest.mark.parametrize("p", [0, 1, 254])
def test_predict_rows_and_subspace(ctx, p, D):
    from spark_ensemble_b200.learners import LogisticRegressionModel
    rng = np.random.default_rng(p * 100 + D)
    n, d = 3001, p + 5
    X = rng.standard_normal((n, d)).astype(np.float32)
    sub = rng.integers(0, d, p).astype(np.int32)  # unsorted, with repeats
    if p > 1:
        sub[-1] = sub[0]
    beta, b = rng.standard_normal((D, p)) * (3.0 / np.sqrt(max(p, 1))), rng.standard_normal(D)
    model = LogisticRegressionModel(beta, b, max(D, 2), D > 1, threshold=0.4)
    for outputs in _predict_outputs():
        rows = 6 if D == 1 else D + 6
        got = _predict_into(ctx, model, X, sub, outputs, rows)
        _host_check(model, X[:, sub], got)


def test_predict_ties_go_to_the_first_maximum(ctx):
    """Two identical coefficient rows dominate every row's margins: the label is the first of them, as numpy's argmax
    and Spark's Vector.argmax give.  Integer features and coefficients make every margin exact on both sides."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.learners import LogisticRegressionModel
    rng = np.random.default_rng(3)
    n, p, D = 2049, 12, 6
    X = rng.integers(-4, 5, (n, p)).astype(np.float32)
    beta = rng.integers(-2, 3, (D, p)).astype(np.float64)
    beta[4] = beta[1]
    b = np.zeros(D)
    b[[1, 4]] = 1000.0
    model = LogisticRegressionModel(beta, b, D, True)
    got = _predict_into(ctx, model, X, None, {"label": (N.SLOT_P, 2), "prob": (N.SLOT_PROB, 1)}, D + 3)
    np.testing.assert_array_equal(got["label"][0], np.ones(n))
    np.testing.assert_array_equal(model.predict(X), np.ones(n))
    np.testing.assert_allclose(got["prob"][[1, 4]], 0.5, rtol=0, atol=1e-6)
    # ties without columns: equal intercepts
    model = LogisticRegressionModel(np.zeros((D, 0)), [0.5, 2.0, -1.0, 2.0, 2.0, 0.0], D, True)
    got = _predict_into(ctx, model, X, np.zeros(0, np.int32), {"label": (N.SLOT_RAW, 3)}, 5)
    np.testing.assert_array_equal(got["label"][0], np.ones(n))
    np.testing.assert_array_equal(model.predict(X[:, :0]), np.ones(n))


@pytest.mark.parametrize("case", ["all_minus_inf", "plus_and_minus_inf"])
def test_predict_non_finite_margins(ctx, case):
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.learners import LogisticRegressionModel
    rng = np.random.default_rng(4)
    n, p, D = 1031, 7, 5
    X = rng.standard_normal((n, p)).astype(np.float32)
    beta = rng.standard_normal((D, p))
    b = np.full(D, -np.inf) if case == "all_minus_inf" else np.array([-np.inf, np.inf, 0.0, np.inf, -np.inf])
    model = LogisticRegressionModel(beta, b, D, True)
    got = _predict_into(ctx, model, X, None, {"raw": (N.SLOT_RAW, 2), "prob": (N.SLOT_PROB, 1),
                                              "label": (N.SLOT_P, 3)}, D + 4)
    _host_check(model, X, got)
    np.testing.assert_array_equal(got["label"][0], np.full(n, 0.0 if case == "all_minus_inf" else 1.0))
    if case == "plus_and_minus_inf":  # raw2probabilityInPlace: 1 for every +inf class
        np.testing.assert_array_equal(got["prob"], np.isposinf(b)[:, None].repeat(n, axis=1).astype(np.float32))


@pytest.mark.parametrize("threshold", [0.0, 1.0])
def test_predict_thresholds_0_and_1_with_margins_beyond_745(ctx, threshold):
    """Binomial margins up to ±2000: the device label is σ(m) > threshold, as the host model's and Spark's
    LogisticRegressionModel.predict.  At threshold 0 both differ from Spark's raw2prediction rule (m > -inf) for
    m below about -709.8, where exp(-m) overflows and σ(m) is 0: DESIGN §4 records it."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.learners import LogisticRegressionModel
    rng = np.random.default_rng(5)
    n, p = 4099, 3
    X = rng.uniform(-1, 1, (n, p)).astype(np.float32)
    model = LogisticRegressionModel(np.array([[2000.0, 0.0, 0.0]]), [0.0], 2, False, threshold=threshold)
    got = _predict_into(ctx, model, X, None, {"label": (N.SLOT_P, 1), "raw": (N.SLOT_RAW, 2)}, 5)
    m = model._margins(X)[:, 0]
    assert m.min() < -745 and m.max() > 745
    with np.errstate(over="ignore"):
        np.testing.assert_array_equal(got["label"][0], model.predict(X))
        p1 = 1.0 / (1.0 + np.exp(-m))
    np.testing.assert_array_equal(got["label"][0], (p1 > threshold).astype(np.float32))
    _host_check(model, X, {"raw": got["raw"]})
    spark_raw_rule = (m > (-np.inf if threshold == 0.0 else np.inf)).astype(np.float32)
    differ = got["label"][0] != spark_raw_rule
    if threshold == 0.0:
        np.testing.assert_array_equal(differ, p1 == 0.0)  # exactly the rows where σ(m) underflows
        assert differ.any()
    else:
        assert not differ.any()


# ---- se_copy_rows -----------------------------------------------------------------------------------------------------
def _filled(ctx, slot, rows, n, seed):
    data = np.random.default_rng(seed).standard_normal((rows, n)).astype(np.float32)
    ctx.alloc(slot, rows, n)
    ctx.upload(slot, data)
    return data


def test_copy_rows_between_slots_of_different_row_counts(ctx):
    from spark_ensemble_b200 import _native as N
    n = 1000  # n mod 32 != 0: padded rows
    src = _filled(ctx, N.SLOT_PROBA, 5, n, 1)
    for dst_row, src_row, count in ((2, 1, 3), (0, 0, 5), (6, 4, 1), (3, 2, 0)):
        ctx.alloc(N.SLOT_P, 9, n)
        ctx.fill(N.SLOT_P, float(SENTINEL))
        ctx.copy_rows(N.SLOT_P, dst_row, N.SLOT_PROBA, src_row, count)
        got = ctx.download(N.SLOT_P).reshape(9, n)
        expect = np.full((9, n), SENTINEL, np.float32)
        expect[dst_row:dst_row + count] = src[src_row:src_row + count]
        assert got.tobytes() == expect.tobytes(), (dst_row, src_row, count)
        np.testing.assert_array_equal(ctx.download(N.SLOT_PROBA).reshape(5, n), src)
    # the whole of a slot into a slot of the same row count
    ctx.alloc(N.SLOT_RAW, 5, n)
    ctx.fill(N.SLOT_RAW, float(SENTINEL))
    ctx.copy_rows(N.SLOT_RAW, 0, N.SLOT_PROBA, 0, 5)
    assert ctx.download(N.SLOT_RAW).reshape(5, n).tobytes() == src.tobytes()
    # a one-row slot (ld = n) into a padded one and back
    one = _filled(ctx, N.SLOT_LABEL, 1, n, 2)
    ctx.copy_rows(N.SLOT_RAW, 3, N.SLOT_LABEL, 0, 1)
    expect = src.copy()
    expect[3] = one[0]
    assert ctx.download(N.SLOT_RAW).reshape(5, n).tobytes() == expect.tobytes()
    ctx.copy_rows(N.SLOT_LABEL, 0, N.SLOT_PROBA, 4, 1)
    assert ctx.download(N.SLOT_LABEL).tobytes() == src[4].tobytes()


def test_copy_rows_disjoint_ranges_within_one_slot(ctx):
    from spark_ensemble_b200 import _native as N
    n = 517
    data = _filled(ctx, N.SLOT_P, 8, n, 3)
    ctx.copy_rows(N.SLOT_P, 5, N.SLOT_P, 1, 3)  # rows 1..3 -> 5..7, touching neither end
    ctx.copy_rows(N.SLOT_P, 0, N.SLOT_P, 4, 1)
    expect = data.copy()
    expect[5:8] = data[1:4]
    expect[0] = data[4]
    assert ctx.download(N.SLOT_P).reshape(8, n).tobytes() == expect.tobytes()


def test_copy_rows_errors_leave_the_destination_unchanged(ctx):
    from spark_ensemble_b200 import _native as N
    n = 333
    data = _filled(ctx, N.SLOT_P, 6, n, 4)
    _filled(ctx, N.SLOT_PROBA, 3, n, 5)
    _filled(ctx, N.SLOT_RAW, 3, n + 1, 6)
    cases = [((N.SLOT_P, 2, N.SLOT_P, 0, 3), ValueError, "overlapping"),
             ((N.SLOT_P, 1, N.SLOT_P, 3, 3), ValueError, "overlapping"),
             ((N.SLOT_P, 4, N.SLOT_PROBA, 0, 3), ValueError, "out of range"),  # past the end of the destination
             ((N.SLOT_P, 0, N.SLOT_PROBA, 1, 3), ValueError, "out of range"),  # past the end of the source
             ((N.SLOT_P, 0, N.SLOT_RAW, 0, 2), N.NativeError, "same length")]  # rows of different lengths
    for args, exc, match in cases:
        with pytest.raises(exc, match=match) as e:
            ctx.copy_rows(*args)
        if exc is N.NativeError:
            assert e.value.code == N.SE_ERR_STATE
        assert ctx.download(N.SLOT_P).reshape(6, n).tobytes() == data.tobytes(), args
