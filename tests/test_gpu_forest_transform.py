"""Scoring tree ensembles over the device-resident features (residentFeatures=True): se_forest_agg for the classifier
aggregations, se_forest_predict for the regressor sums, device tree walks + se_agg_run for the weighted median.  Each
route is checked against the member-by-member route on the same model, and one case per kind against the oracle's
aggregations over fp64 host walks."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _letter(n):
    d = np.load(os.path.join(GOLD, "letter.npz"))
    return (d["X"][:n].astype(np.float64) / 7.5 - 1.0).astype(np.float32), d["y"][:n].astype(np.float64)


def _cpusmall():
    d = np.load(os.path.join(GOLD, "cpusmall.npz"))
    return d["X"].astype(np.float32), d["y"].astype(np.float64)


def _synthetic_cls(n, d, K, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(np.float32)
    z = np.sin(2 * X[:, 0]) + X[:, 1] ** 2 + 0.3 * rng.standard_normal(n)
    y = np.minimum(np.digitize(z, np.quantile(z, np.linspace(0, 1, K + 1)[1:-1])), K - 1).astype(np.float64)
    return X, y


def _both(model, fn):
    """fn(model) with residentFeatures on, then off (the member route)."""
    model.set("residentFeatures", True)
    a = fn(model)
    model.set("residentFeatures", False)
    b = fn(model)
    return a, b


def _transform(X):
    from spark_ensemble_b200 import DataFrame
    return lambda m: m.transform(DataFrame(features=X))


def _check_classifier(res, mem, real=False, hard=False):
    raw_r, raw_m = np.asarray(res["rawPrediction"]), np.asarray(mem["rawPrediction"])
    if hard:
        np.testing.assert_array_equal(raw_r, raw_m)
    # SAMME.R sums terms of +-(K - 1)·52·ln 2: atol scales with them
    atol = 1e-5 * max(1.0, np.abs(raw_m).max()) if real else 1e-6
    np.testing.assert_allclose(raw_r, raw_m, rtol=1e-5, atol=atol)
    np.testing.assert_allclose(res["probability"], mem["probability"], rtol=1e-5, atol=1e-6)
    srt = np.sort(raw_m, axis=1)
    near_tie = (srt[:, -1] - srt[:, -2]) <= 1e-5 * np.maximum(1.0, np.abs(srt[:, -1])) + atol
    differ = np.asarray(res["prediction"]) != np.asarray(mem["prediction"])
    assert not np.any(differ & ~near_tie)


# ---------------------------------------------------------------- route equivalence on fitted models
@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("data", ["letter", "k3"])
def test_gbm_classifier_logloss(data, device):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.classification import GBMClassifier
    from spark_ensemble_b200.learners import DecisionTreeRegressor, DeviceDecisionTreeRegressor
    X, y = _letter(3000) if data == "letter" else _synthetic_cls(20011, 6, 3, 5)
    learner = DeviceDecisionTreeRegressor(maxDepth=4) if device else DecisionTreeRegressor(maxDepth=4)
    m = (GBMClassifier().setBaseLearner(learner).setNumBaseLearners(3).setSubspaceRatio(0.5)
         .setResidentFeatures(device).fit(DataFrame(features=X, label=y)))
    res, mem = _both(m, _transform(X))
    _check_classifier(res, mem)


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("loss", ["bernoulli", "exponential"])
def test_gbm_classifier_binary(loss, device):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.classification import GBMClassifier
    from spark_ensemble_b200.learners import DecisionTreeRegressor, DeviceDecisionTreeRegressor
    X, y = _synthetic_cls(20011, 5, 2, 7)
    learner = DeviceDecisionTreeRegressor(maxDepth=5) if device else DecisionTreeRegressor(maxDepth=5)
    m = (GBMClassifier().setBaseLearner(learner).setNumBaseLearners(4).setLoss(loss).setResidentFeatures(device)
         .fit(DataFrame(features=X, label=y)))
    res, mem = _both(m, _transform(X))
    _check_classifier(res, mem)


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("algorithm", ["discrete", "real"])
@pytest.mark.parametrize("data", ["letter", "k3"])
def test_boosting_classifier(data, algorithm, device):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.classification import BoostingClassifier
    from spark_ensemble_b200.learners import DecisionTreeClassifier, DeviceDecisionTreeClassifier
    X, y = _letter(3000) if data == "letter" else _synthetic_cls(20011, 6, 3, 9)
    learner = DeviceDecisionTreeClassifier(maxDepth=5) if device else DecisionTreeClassifier(maxDepth=5)
    m = (BoostingClassifier().setBaseLearner(learner).setNumBaseLearners(5).setAlgorithm(algorithm)
         .setResidentFeatures(device).fit(DataFrame(features=X, label=y)))
    assert m.numModels >= 2
    res, mem = _both(m, _transform(X))
    _check_classifier(res, mem, real=algorithm == "real")


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("strategy", ["hard", "soft"])
def test_bagging_classifier(strategy, device):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.classification import BaggingClassifier
    from spark_ensemble_b200.learners import DecisionTreeClassifier, DeviceDecisionTreeClassifier
    X, y = _letter(4000)
    learner = DeviceDecisionTreeClassifier(maxDepth=6) if device else DecisionTreeClassifier(maxDepth=6)
    m = (BaggingClassifier().setBaseLearner(learner).setNumBaseLearners(6).setVotingStrategy(strategy)
         .setSubspaceRatio(0.5).fit(DataFrame(features=X, label=y)))
    res, mem = _both(m, _transform(X))
    _check_classifier(res, mem, hard=strategy == "hard")


def _reg_check(m, X):
    res, mem = _both(m, _transform(X))
    np.testing.assert_allclose(res["prediction"], mem["prediction"], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("init", ["constant", "base"])
def test_gbm_regressor_stand_in(init):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.learners import DecisionTreeRegressor
    from spark_ensemble_b200.regression import GBMRegressor
    X, y = _cpusmall()
    m = (GBMRegressor().setBaseLearner(DecisionTreeRegressor(maxDepth=4)).setNumBaseLearners(5)
         .setSubspaceRatio(0.5).setInitStrategy(init).fit(DataFrame(features=X, label=y)))
    _reg_check(m, X)


def test_gbm_regressor_device_fitted():
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor
    from spark_ensemble_b200.regression import GBMRegressor
    X, y = _cpusmall()
    m = (GBMRegressor().setBaseLearner(DeviceDecisionTreeRegressor(maxDepth=5)).setNumBaseLearners(5)
         .setResidentFeatures(True).fit(DataFrame(features=X, label=y)))
    _reg_check(m, X)


@pytest.mark.parametrize("device", [False, True])
def test_bagging_regressor(device):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.learners import DecisionTreeRegressor, DeviceDecisionTreeRegressor
    from spark_ensemble_b200.regression import BaggingRegressor
    X, y = _cpusmall()
    learner = DeviceDecisionTreeRegressor(maxDepth=5) if device else DecisionTreeRegressor(maxDepth=5)
    m = (BaggingRegressor().setBaseLearner(learner).setNumBaseLearners(5).setSubspaceRatio(0.5)
         .fit(DataFrame(features=X, label=y)))
    _reg_check(m, X)


@pytest.mark.parametrize("voting", ["median", "mean"])
def test_boosting_regressor(voting):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.learners import DecisionTreeRegressor
    from spark_ensemble_b200.regression import BoostingRegressor
    X, y = _cpusmall()
    m = (BoostingRegressor().setBaseLearner(DecisionTreeRegressor(maxDepth=4)).setNumBaseLearners(5)
         .setVotingStrategy(voting).fit(DataFrame(features=X, label=y)))
    assert m.numModels >= 2
    _reg_check(m, X)


# ---------------------------------------------------------------- synthetic forests, oracle, nothing on the host
def _tree(rng, depth, cols, cands, K):
    """A full tree of the given depth in BFS order over columns `cols`, thresholds drawn from cands[col]; node
    probabilities [n_nodes, K] (a fifth of them pure, as pure leaves are) and labels (their argmax)."""
    n_int, n = 2 ** depth - 1, 2 ** (depth + 1) - 1
    f = np.full(n, -1, np.int32)
    t = np.zeros(n, np.float32)
    l = np.zeros(n, np.int32)
    r = np.zeros(n, np.int32)
    c = rng.choice(cols, n_int)
    f[:n_int] = c
    t[:n_int] = [rng.choice(cands[j]) for j in c]
    l[:n_int] = 2 * np.arange(n_int) + 1
    r[:n_int] = 2 * np.arange(n_int) + 2
    p = rng.dirichlet(np.full(K, 0.3), n).astype(np.float32)
    pure = rng.random(n) < 0.2
    p[pure] = np.eye(K, dtype=np.float32)[rng.integers(0, K, int(pure.sum()))]
    v = np.argmax(p, axis=1).astype(np.float32)
    return {"feature": f, "threshold": t, "left": l, "right": r, "value": v, "values": p,
            "gain": np.zeros(n), "class_weights": np.zeros((n, K))}


def _forest(seed, M, depth, d, K, n_cands=24):
    rng = np.random.default_rng(seed)
    cands = [np.sort(rng.standard_normal(n_cands)).astype(np.float32) for _ in range(d)]
    return [_tree(rng, depth, np.arange(d), cands, K) for _ in range(M)]


def _members(trees, K):
    from spark_ensemble_b200.learners import DeviceDecisionTreeClassificationModel
    return [DeviceDecisionTreeClassificationModel(t, K) for t in trees]


def test_each_kind_against_the_oracle(oracle):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.classification import (BaggingClassificationModel, BoostingClassificationModel,
                                                    GBMClassificationModel)
    K, M, n, d = 5, 9, 20011, 7
    X = np.random.default_rng(1).standard_normal((n, d)).astype(np.float32)
    trees = _forest(2, M, 5, d, K)
    mem = _members(trees, K)
    leaf = [m._leaf(X) for m in mem]
    P = np.stack([t["values"][lf].T for t, lf in zip(trees, leaf)]).astype(np.float64)  # [M][K][n]
    V = np.stack([t["value"][lf] for t, lf in zip(trees, leaf)]).astype(np.float64)     # [M][n]
    a = np.random.default_rng(3).uniform(0.2, 1.5, M)
    subs = [np.arange(d)] * M

    def run(model):
        model.set("residentFeatures", True)
        return model.transform(DataFrame(features=X))

    bag = BaggingClassificationModel(K, subs, mem)
    out = run(bag.setVotingStrategy("soft"))
    raw, prob = oracle.agg_bagging_soft(P)
    np.testing.assert_allclose(out["rawPrediction"], raw.T, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(out["probability"], prob.T, rtol=1e-5, atol=1e-6)
    out = run(bag.setVotingStrategy("hard"))
    raw, prob = oracle.agg_bagging_hard(V, K)
    np.testing.assert_array_equal(out["rawPrediction"], raw.T)
    np.testing.assert_allclose(out["probability"], prob.T, rtol=1e-6)
    boost = BoostingClassificationModel(K, a, mem)
    out = run(boost.setAlgorithm("real"))
    raw, prob = oracle.agg_boosting_real(P)
    np.testing.assert_allclose(out["rawPrediction"], raw.T, rtol=1e-5, atol=1e-5 * np.abs(raw).max())
    np.testing.assert_allclose(out["probability"], prob.T, rtol=1e-5, atol=1e-6)
    out = run(boost.setAlgorithm("discrete"))
    raw, prob = oracle.agg_boosting_discrete(V, a.astype(np.float32), K)
    np.testing.assert_allclose(out["rawPrediction"], raw.T, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(out["probability"], prob.T, rtol=1e-5, atol=1e-6)
    # GBM classifier: the trees' leaf probabilities of class 0 serve as regression values
    reg = [dict(t, value=t["values"][:, 0].copy()) for t in trees[:6]]
    Pg = np.stack([t["value"][m._leaf(X)] for t, m in zip(reg, _members(reg, K))]).astype(np.float64)
    for dim, loss in ((3, "logloss"), (1, "bernoulli"), (1, "exponential")):
        from spark_ensemble_b200.learners import DeviceDecisionTreeRegressionModel
        rounds = 6 // dim
        models = [[DeviceDecisionTreeRegressionModel(reg[i * dim + j]) for j in range(dim)] for i in range(rounds)]
        wts = [np.random.default_rng(i).uniform(0.1, 1.0, dim) for i in range(rounds)]
        init = np.linspace(-0.3, 0.4, dim)
        Kc = 3 if dim == 3 else 2
        g = GBMClassificationModel(Kc, wts, [np.arange(d)] * rounds, models, init, dim).setLoss(loss)
        out = run(g)
        raw = oracle.agg_gbm_classifier_raw(Pg[: rounds * dim].reshape(rounds, dim, n), np.stack(wts), init, Kc)
        np.testing.assert_allclose(out["rawPrediction"], raw.T, rtol=1e-5, atol=1e-6)
        prob = oracle.gbm_raw2prob(N.LOSS[loss], raw)
        np.testing.assert_allclose(out["probability"], prob.T, rtol=1e-5, atol=1e-6)


def test_regressors_against_the_oracle(oracle):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.ensemble import fit_dummy_regressor
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressionModel
    from spark_ensemble_b200.regression import BaggingRegressionModel, BoostingRegressionModel, GBMRegressionModel
    M, n, d = 7, 20011, 6
    X = np.random.default_rng(4).standard_normal((n, d)).astype(np.float32)
    trees = [dict(t, value=(10 * t["values"][:, 0] - 3).astype(np.float32)) for t in _forest(5, M, 6, d, 2)]
    mem = [DeviceDecisionTreeRegressionModel(t) for t in trees]
    P = np.stack([m.predict(X) for m in mem])
    a = np.random.default_rng(6).uniform(0.1, 1.0, M)
    subs = [np.arange(d)] * M
    df = DataFrame(features=X)
    init = fit_dummy_regressor("constant", np.zeros(3), constant=0.75)
    g = GBMRegressionModel(a, subs, mem, init).setResidentFeatures(True)
    np.testing.assert_allclose(g.transform(df)["prediction"], oracle.agg_weighted_sum(P, a, 0.75), rtol=1e-5, atol=1e-5)
    b = BaggingRegressionModel(subs, mem).setResidentFeatures(True)
    np.testing.assert_allclose(b.transform(df)["prediction"], oracle.agg_mean(P), rtol=1e-5, atol=1e-5)
    r = BoostingRegressionModel(a, mem).setResidentFeatures(True)
    np.testing.assert_allclose(r.setVotingStrategy("mean").transform(df)["prediction"], oracle.agg_weighted_mean(P, a),
                               rtol=1e-5, atol=1e-5)
    np.testing.assert_array_equal(r.setVotingStrategy("median").transform(df)["prediction"],
                                  oracle.agg_weighted_median(P.astype(np.float32), a).astype(np.float32))


def test_nothing_walked_or_stacked_on_the_host(monkeypatch):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200 import learners as L
    from spark_ensemble_b200.classification import (BaggingClassificationModel, BoostingClassificationModel,
                                                    GBMClassificationModel)
    from spark_ensemble_b200.context import Context
    from spark_ensemble_b200.ensemble import fit_dummy_regressor
    from spark_ensemble_b200.regression import BaggingRegressionModel, BoostingRegressionModel, GBMRegressionModel
    K, M, n, d = 4, 6, 5003, 5
    X = np.random.default_rng(8).standard_normal((n, d)).astype(np.float32)
    trees = _forest(9, M, 4, d, K)
    cls = _members(trees, K)
    reg = [L.DeviceDecisionTreeRegressionModel(dict(t, value=t["values"][:, 1].copy())) for t in trees]
    subs = [np.arange(d)] * M
    a = np.linspace(0.2, 1.0, M)
    models = [
        BaggingClassificationModel(K, subs, cls).setVotingStrategy("soft"),
        BaggingClassificationModel(K, subs, cls).setVotingStrategy("hard"),
        BoostingClassificationModel(K, a, cls).setAlgorithm("real"),
        BoostingClassificationModel(K, a, cls).setAlgorithm("discrete"),
        GBMClassificationModel(3, [np.ones(3)] * 2, subs[:2], [reg[:3], reg[3:]], np.zeros(3), 3),
        GBMRegressionModel(a, subs, reg, fit_dummy_regressor("constant", np.zeros(2), constant=1.0)),
        BaggingRegressionModel(subs, reg),
        BoostingRegressionModel(a, reg).setVotingStrategy("mean"),
    ]
    df = DataFrame(features=X)
    expected = [m.transform(df) for m in models]

    def boom(*a, **k):
        raise AssertionError("a member was evaluated on the host")

    for c in (L.DeviceDecisionTreeClassificationModel, L.DeviceDecisionTreeRegressionModel):
        for name in ("predict", "predictProbability"):
            if hasattr(c, name):
                monkeypatch.setattr(c, name, boom)
    real_upload, real_cfg = Context.upload, Context.agg_configure

    def upload(self, slot, *a, **k):
        assert slot != N.SLOT_P, "member outputs were uploaded"
        return real_upload(self, slot, *a, **k)

    def agg_configure(self, *a, **k):
        raise AssertionError("the member-output matrix was allocated")

    monkeypatch.setattr(Context, "upload", upload)
    monkeypatch.setattr(Context, "agg_configure", agg_configure)
    for m, exp in zip(models, expected):
        m.set("residentFeatures", True)
        got = m.transform(df)
        for col in ("rawPrediction", "probability", "prediction"):
            if col in exp:
                np.testing.assert_allclose(got[col], exp[col], rtol=1e-5, atol=1e-5 * max(1.0, np.abs(exp[col]).max()))


def test_chunks_and_single_rows():
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.classification import BaggingClassificationModel
    from spark_ensemble_b200.context import Context
    K, M, n, d = 6, 24, 9001, 128
    X = np.random.default_rng(10).standard_normal((n, d)).astype(np.float32)
    trees = _forest(11, M, 8, d, K)
    with Context(0) as ctx:
        ctx.alloc(N.SLOT_X, d, n)
        ctx.upload_rowmajor(N.SLOT_X, X)
        ctx.forest_agg(N.AGG_BAGGING_SOFT, K, trees)
        assert ctx.get_option("last_forest_chunks") >= 3
        raw = ctx.download(N.SLOT_RAW).reshape(K, n).T
    mem = _members(trees, K)
    ref = sum(t["values"][m._leaf(X)].astype(np.float64) for t, m in zip(trees, mem))
    np.testing.assert_allclose(raw, ref, rtol=1e-5, atol=1e-5)
    m = BaggingClassificationModel(K, [np.arange(d)] * M, mem).setVotingStrategy("soft")
    res, memr = _both(m, _transform(X))
    _check_classifier(res, memr)
    x = X[17]
    for fn in ("predict", "predictRaw", "predictProbability"):
        a, b = _both(m, lambda mm: getattr(mm, fn)(x))
        np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6)


# ---------------------------------------------------------------- fallbacks
def test_fallback_more_than_255_thresholds():
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.learners import DecisionTreeRegressor
    from spark_ensemble_b200.regression import BaggingRegressor
    rng = np.random.default_rng(12)
    X = rng.standard_normal((20000, 2)).astype(np.float32)
    y = np.sin(3 * X[:, 0]) + 0.1 * rng.standard_normal(20000)
    m = (BaggingRegressor().setBaseLearner(DecisionTreeRegressor(maxDepth=8)).setNumBaseLearners(4)
         .fit(DataFrame(features=X, label=y)))
    assert sum(int(np.sum(t.tree_arrays()["feature"] == 0)) for t in m.models) > 255
    a, b = _both(m, _transform(X))
    np.testing.assert_array_equal(a["prediction"], b["prediction"])


def test_fallback_linear_members():
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.learners import LinearRegression
    from spark_ensemble_b200.regression import BaggingRegressor
    X, y = _cpusmall()
    m = BaggingRegressor().setBaseLearner(LinearRegression()).setNumBaseLearners(3).fit(DataFrame(features=X, label=y))
    a, b = _both(m, _transform(X))
    np.testing.assert_array_equal(a["prediction"], b["prediction"])


def test_fallback_above_the_class_limit():
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.classification import BaggingClassificationModel
    K, M, n, d = N.FOREST_AGG_MAX_CLASSES + 3, 4, 3001, 5
    X = np.random.default_rng(13).standard_normal((n, d)).astype(np.float32)
    m = BaggingClassificationModel(K, [np.arange(d)] * M, _members(_forest(14, M, 4, d, K), K))
    for strategy in ("soft", "hard"):
        a, b = _both(m.setVotingStrategy(strategy), _transform(X))
        for col in ("rawPrediction", "probability", "prediction"):
            np.testing.assert_array_equal(a[col], b[col])


def test_leaf_label_outside_the_classes_is_an_error():
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.classification import BaggingClassificationModel, BoostingClassificationModel
    K, M, n, d = 3, 3, 2001, 4
    X = np.random.default_rng(15).standard_normal((n, d)).astype(np.float32)
    trees = _forest(16, M, 3, d, K)
    trees[1]["value"][trees[1]["feature"] < 0] = K  # every leaf of tree 1 votes for class K
    mem = _members(trees, K)
    for m in (BaggingClassificationModel(K, [np.arange(d)] * M, mem).setVotingStrategy("hard"),
              BoostingClassificationModel(K, np.ones(M), mem).setAlgorithm("discrete")):
        m.set("residentFeatures", True)
        with pytest.raises(ValueError, match="class index"):
            m.transform(DataFrame(features=X))


# ---------------------------------------------------------------- scale: a member-output matrix of 106 GB
def test_soft_bagging_at_scale():
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.classification import BaggingClassificationModel
    K, M, n, d = 26, 128, 8 * 1024 * 1024, 16
    assert 4 * M * K * n > 100e9
    rng = np.random.default_rng(17)
    X = rng.standard_normal((n, d), dtype=np.float32)
    trees = _forest(18, M, 6, d, K)
    mem = _members(trees, K)
    m = BaggingClassificationModel(K, [np.arange(d)] * M, mem).setVotingStrategy("soft").setResidentFeatures(True)
    out = m.transform(DataFrame(features=X))
    rows = rng.choice(n, 10000, replace=False)
    Xs = X[rows]
    raw = sum(t["values"][mm._leaf(Xs)].astype(np.float64) for t, mm in zip(trees, mem))
    np.testing.assert_allclose(out["rawPrediction"][rows], raw, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(out["probability"][rows], raw / M, rtol=1e-5, atol=1e-6)
    assert np.mean(out["prediction"][rows] == np.argmax(raw, axis=1)) > 0.999
