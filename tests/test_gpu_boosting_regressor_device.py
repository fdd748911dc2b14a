"""BoostingRegressor (AdaBoost.R2) on the device at both ends: the weighted median of a tree forest in one pass
(se_forest_median, Context.forest_median) against the member route it replaces (se_tree_predict per member into
SLOT_P + se_agg_run(AGG_BOOSTING_REG_MEDIAN)) bit for bit, and the fit of DeviceDecisionTreeRegressor on the
device-resident labels and boosting weights against the residentFeatures=False route."""
import os

import numpy as np
import pytest

from oracle import np_tree as T

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _cpusmall():
    d = np.load(os.path.join(GOLD, "cpusmall.npz"))
    return d["X"].astype(np.float32), d["y"].astype(np.float64)


# ---------------------------------------------------------------- se_forest_median against the member route
def _tree(rng, depth, n_sub, cands, levels):
    """A full regression tree of the given depth in BFS order over subspace indices [0, n_sub), thresholds drawn from
    cands, leaf values from `levels` (few distinct values, -0 among them: ties between members are common)."""
    n_int, n = 2 ** depth - 1, 2 ** (depth + 1) - 1
    f = np.full(n, -1, np.int32)
    t = np.zeros(n, np.float32)
    l = np.zeros(n, np.int32)
    r = np.zeros(n, np.int32)
    f[:n_int] = rng.integers(0, n_sub, n_int)
    t[:n_int] = rng.choice(cands, n_int)
    l[:n_int] = 2 * np.arange(n_int) + 1
    r[:n_int] = 2 * np.arange(n_int) + 2
    v = rng.choice(levels, n).astype(np.float32)
    return {"feature": f, "threshold": t, "left": l, "right": r, "value": v}


def _forest(seed, M, d, depth=6, n_sub=5):
    rng = np.random.default_rng(seed)
    cands = np.sort(rng.standard_normal(40)).astype(np.float32)
    levels = np.concatenate([np.arange(-3, 4, dtype=np.float32), [-0.0, 0.5, 1.25]]).astype(np.float32)
    trees = [_tree(rng, depth, n_sub, cands, levels) for _ in range(M)]
    subs = [np.sort(rng.choice(d, n_sub, replace=False)).astype(np.int32) for _ in range(M)]
    return trees, subs


def _weights(kind, M, seed):
    rng = np.random.default_rng(seed)
    if kind == "generic":
        return rng.uniform(0.1, 1.5, M)
    if kind == "integer":  # an even total: cumulative sums meet half of it exactly, rows inside the margin
        w = rng.integers(1, 4, M).astype(np.float64)
        w[0] += w.sum() % 2
        return w
    if kind == "equal":
        return np.full(M, 0.7)
    if kind == "nonpositive":  # the weight log(1/β) <= 0 of a kept round with estimatorError >= 0.5
        w = rng.uniform(0.1, 1.5, M)
        w[M // 2] = -0.25 if M > 1 else 0.0
        return w
    if kind == "nan_leaves":
        return rng.uniform(0.1, 1.5, M)
    raise AssertionError(kind)


def _member_route(ctx, trees, w, subs, validation, n):
    from spark_ensemble_b200 import _native as N
    ctx.agg_configure(N.AGG_BOOSTING_REG_MEDIAN, len(trees), 0, 1, 0, n)
    for i, (t, s) in enumerate(zip(trees, subs)):
        ctx.tree_predict(t, N.SLOT_P, i, validation=validation, subspace=s)
    ctx.agg_run(w)
    return ctx.download(N.SLOT_RAW).copy()


@pytest.fixture(scope="module")
def data():
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    rng = np.random.default_rng(11)
    n, nv, d = 20011, 3001, 12
    X = rng.standard_normal((n, d)).astype(np.float32)
    X[rng.random((n, d)) < 0.01] = np.nan  # NaN features go right, as in every tree walk
    VX = rng.standard_normal((nv, d)).astype(np.float32)
    ctx = Context(0)
    ctx.alloc(N.SLOT_X, d, n)
    ctx.upload_rowmajor(N.SLOT_X, X)
    ctx.alloc(N.SLOT_VX, d, nv)
    ctx.upload_rowmajor(N.SLOT_VX, VX)
    ctx.alloc(N.SLOT_H, 3, n)
    ctx.alloc(N.SLOT_VH, 1, nv)
    yield ctx, X, VX
    ctx.close()


@pytest.mark.parametrize("M", [1, 2, 7, 33, 64])
@pytest.mark.parametrize("kind", ["generic", "integer", "equal", "nonpositive", "nan_leaves"])
def test_one_pass_equals_member_route(data, M, kind):
    from spark_ensemble_b200 import _native as N
    ctx, X, VX = data
    n, nv = X.shape[0], VX.shape[0]
    trees, subs = _forest(100 + M, M, X.shape[1])
    if kind == "nan_leaves":  # a member whose root has W = 0 outputs NaN: leaves of NaN in one tree
        v = trees[0]["value"].copy()
        v[1::3] = np.nan
        trees[0] = dict(trees[0], value=v)
    w = _weights(kind, M, M)
    ctx.forest_median(trees, N.SLOT_H, w, out_row=1, subspaces=subs)
    chunks, mode = ctx.get_option("last_forest_chunks"), ctx.get_option("last_wm_mode")
    deferred = ctx.get_option("last_wm_deferred")
    got = ctx.download(N.SLOT_H).reshape(3, n)[1].copy()
    ref = _member_route(ctx, trees, w, subs, False, n)
    np.testing.assert_array_equal(got.view(np.uint32), ref.view(np.uint32))
    # se_agg_run's choice: the exact sort for every row unless all weights are finite and >= 0, no margin if all equal
    assert mode == (0 if np.any(w < 0) else 2 if np.all(w == w[0]) else 1)
    assert mode == {"generic": 1, "integer": mode, "equal": 2, "nonpositive": 0, "nan_leaves": 1}[kind] or M == 1
    if kind == "integer" and M >= 7:
        assert deferred > 0  # the exact sort resolved the rows inside the margin
    if M == 64:
        assert chunks >= 2  # the kernel re-staged several chunks of trees for every tile
    if kind == "nan_leaves" and M == 1:  # NaN keys sort last: with more members the median is rarely NaN
        assert np.isnan(got).any()
    # the validation features (VX)
    ctx.forest_median(trees, N.SLOT_VH, w, validation=True, subspaces=subs)
    np.testing.assert_array_equal(ctx.download(N.SLOT_VH).view(np.uint32),
                                  _member_route(ctx, trees, w, subs, True, nv).view(np.uint32))


def test_exact_sort_for_every_row_equals_member_route(data):
    """With the fast path off (wm_fast 0) both routes take the exact (key, model) sort for every row."""
    from spark_ensemble_b200 import _native as N
    ctx, X, _ = data
    trees, subs = _forest(7, 33, X.shape[1])
    w = _weights("integer", 33, 3)
    ctx.set_option("wm_fast", 0)
    try:
        ctx.forest_median(trees, N.SLOT_H, w, subspaces=subs)
        assert ctx.get_option("last_wm_mode") == 0
        got = ctx.download(N.SLOT_H).reshape(3, -1)[0].copy()
        ref = _member_route(ctx, trees, w, subs, False, X.shape[0])
    finally:
        ctx.set_option("wm_fast", 1)
    np.testing.assert_array_equal(got.view(np.uint32), ref.view(np.uint32))


def test_against_the_oracle(oracle):
    """The weighted median of fp64 host walks (ensemble/Utils.scala:26-40 in the oracle)."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressionModel
    n, d, M = 20011, 9, 21
    X = np.random.default_rng(5).standard_normal((n, d)).astype(np.float32)
    trees, subs = _forest(8, M, d, depth=5, n_sub=4)
    P = np.stack([DeviceDecisionTreeRegressionModel(t).predict(X[:, s]) for t, s in zip(trees, subs)])
    a = np.random.default_rng(9).uniform(0.1, 1.0, M)
    with Context(0) as ctx:
        ctx.alloc(N.SLOT_X, d, n)
        ctx.upload_rowmajor(N.SLOT_X, X)
        ctx.alloc(N.SLOT_RAW, 1, n)
        ctx.forest_median(trees, N.SLOT_RAW, a, subspaces=subs)
        got = ctx.download(N.SLOT_RAW)
    np.testing.assert_array_equal(got, oracle.agg_weighted_median(P.astype(np.float32), a).astype(np.float32))


def test_above_64_trees_keeps_the_member_route(data):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressionModel
    from spark_ensemble_b200.regression import BoostingRegressionModel
    ctx, X, _ = data
    trees, _ = _forest(3, 65, X.shape[1], depth=4, n_sub=X.shape[1])
    w = _weights("generic", 65, 1)
    with pytest.raises(ValueError, match="serves 1..64 trees, got 65"):  # SE_ERR_ARG
        ctx.forest_median(trees, N.SLOT_H, w)
    m = BoostingRegressionModel(w, [DeviceDecisionTreeRegressionModel(t) for t in trees])
    df = DataFrame(features=X)
    on = m.setResidentFeatures(True).transform(df)["prediction"]
    off = m.setResidentFeatures(False).transform(df)["prediction"]
    np.testing.assert_array_equal(on, off)


def test_model_takes_the_one_pass_route(monkeypatch):
    """residentFeatures with at most 64 tree members: one forest_median call, no member walked into SLOT_P."""
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.context import Context
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressionModel
    from spark_ensemble_b200.regression import BoostingRegressionModel
    X, _ = _cpusmall()
    trees, _ = _forest(4, 10, X.shape[1], depth=5, n_sub=X.shape[1])
    m = BoostingRegressionModel(_weights("generic", 10, 2), [DeviceDecisionTreeRegressionModel(t) for t in trees])
    calls = []
    real = Context.forest_median
    monkeypatch.setattr(Context, "forest_median", lambda self, *a, **k: (calls.append(1), real(self, *a, **k))[1])
    monkeypatch.setattr(Context, "tree_predict", lambda *a, **k: pytest.fail("a member was walked into SLOT_P"))
    on = m.setResidentFeatures(True).transform(DataFrame(features=X))["prediction"]
    monkeypatch.undo()
    assert calls == [1]
    off = m.setResidentFeatures(False).transform(DataFrame(features=X))["prediction"]
    np.testing.assert_array_equal(on, off)


# ---------------------------------------------------------------- BoostingRegressor fits on the device
def _estimator(learner, resident, rounds=6, loss="linear"):
    from spark_ensemble_b200.regression import BoostingRegressor
    return (BoostingRegressor().setBaseLearner(learner).setNumBaseLearners(rounds).setLossType(loss)
            .setResidentFeatures(resident))


@pytest.mark.parametrize("learner", ["device", "host"])
def test_fitted_model_transform_on_equals_off(learner):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.learners import DecisionTreeRegressor, DeviceDecisionTreeRegressor
    X, y = _cpusmall()
    base = DeviceDecisionTreeRegressor(maxDepth=5) if learner == "device" else DecisionTreeRegressor(maxDepth=5)
    df = DataFrame(features=X, label=y)
    m = _estimator(base, True).setVotingStrategy("median").fit(df)
    assert m.numModels >= 2
    on = m.setResidentFeatures(True).transform(df)["prediction"]
    off = m.setResidentFeatures(False).transform(df)["prediction"]
    np.testing.assert_array_equal(on, off)


def test_weights_never_leave_the_device(monkeypatch):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor
    X, y = _cpusmall()
    real_download, real_upload = Context.download, Context.upload

    def download(self, slot, *a, **k):
        assert slot != N.SLOT_BW, "the boosting weights left the device"
        return real_download(self, slot, *a, **k)

    def upload(self, slot, *a, **k):
        assert slot != N.SLOT_PRED, "the predictions were uploaded"
        return real_upload(self, slot, *a, **k)

    monkeypatch.setattr(Context, "download", download)
    monkeypatch.setattr(Context, "upload", upload)
    m = _estimator(DeviceDecisionTreeRegressor(maxDepth=5), True).fit(DataFrame(features=X, label=y))
    monkeypatch.undo()
    assert m.numModels >= 2


@pytest.mark.parametrize("loss", ["linear", "squared", "exponential"])
def test_resident_fit_is_the_same_fit(monkeypatch, loss):
    """Same rounds as the residentFeatures=False route; every tree audited on the weights it was fitted on."""
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor
    X, y = _cpusmall()
    df = DataFrame(features=X, label=y)
    learner = DeviceDecisionTreeRegressor(maxDepth=5, seed=3)
    ref = _estimator(learner, False, loss=loss).fit(df)
    seen = []
    real_fit = DeviceDecisionTreeRegressor.fit_resident

    def fit_resident(self, ctx, label_slot, label_row, weight_slot, *a, **k):
        w = ctx.download(weight_slot).astype(np.float64)  # the weights this round fits on, read by the test
        model = real_fit(self, ctx, label_slot, label_row, weight_slot, *a, **k)
        seen.append((w, model, ctx.download(N.SLOT_PRED).copy()))
        return model

    monkeypatch.setattr(DeviceDecisionTreeRegressor, "fit_resident", fit_resident)
    dev = _estimator(learner, True, loss=loss).fit(df)
    monkeypatch.undo()
    hr, hd = ref.trainingHistory, dev.trainingHistory
    assert len(hr) == len(hd) >= 2
    for a, b in zip(hr, hd):
        for key in ("maxError", "estimatorError", "sumWeights"):
            np.testing.assert_allclose(b[key], a[key], rtol=1e-5, atol=1e-12)
    np.testing.assert_allclose(dev.weights, ref.weights, rtol=1e-5)
    cands = learner.split_candidates(X)
    params = dict(max_depth=5, min_instances=1, min_info_gain=0.0, min_weight_fraction=0.0)
    assert len(seen) == len(hd)
    for w, model, out in seen:
        t = model._arrays
        assert T.audit(t, X, cands, np.arange(X.shape[1]), y.astype(np.float32), w, None, params,
                       out=out) == t["feature"].size


def test_device_learner_without_resident_features_keeps_learner_fit(monkeypatch):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor
    X, y = _cpusmall()
    calls = []
    real_fit = DeviceDecisionTreeRegressor.fit
    monkeypatch.setattr(DeviceDecisionTreeRegressor, "fit",
                        lambda self, X, y, w=None: (calls.append(w.sum()), real_fit(self, X, y, w))[1])
    m = _estimator(DeviceDecisionTreeRegressor(maxDepth=4), False, rounds=4).fit(DataFrame(features=X, label=y))
    assert len(calls) == len(m.trainingHistory) >= 2
    np.testing.assert_allclose(calls, 1.0, rtol=1e-4)  # learner.fit on the normalised weights, every round
    calls.clear()
    _estimator(DeviceDecisionTreeRegressor(maxDepth=4), True, rounds=4).fit(DataFrame(features=X, label=y))
    assert calls == []


def test_max_depth_above_8_raises():
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor
    with pytest.raises(ValueError):
        DeviceDecisionTreeRegressor(maxDepth=9)
    X, y = _cpusmall()
    learner = DeviceDecisionTreeRegressor(maxDepth=5)
    learner.maxDepth = 9
    with pytest.raises(ValueError):
        _estimator(learner, True).fit(DataFrame(features=X, label=y))
