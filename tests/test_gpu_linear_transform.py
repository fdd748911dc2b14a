"""Ensembles of linear and logistic members scored in one pass over the resident features (se_linear_agg).

The kernel is checked against the device member route it replaces (se_logistic_predict per member into SLOT_P, then
se_agg_run): bit for bit for the sum kinds, the median, SAMME.R RAW and hard-vote RAW, at _check_classifier's
tolerances for the rest.  Then one case per kind against the oracle, the six ensemble models with residentFeatures on
and off, the fallbacks, the errors and the stacking route."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")
REG_KINDS = (0, 1, 7, 8)  # AGG_GBM_REGRESSOR, AGG_BAGGING_REGRESSOR, AGG_BOOSTING_REG_MEDIAN, AGG_BOOSTING_REG_MEAN


def _cpusmall():
    d = np.load(os.path.join(GOLD, "cpusmall.npz"))
    return d["X"].astype(np.float32), d["y"].astype(np.float64)


def _letter(n):
    d = np.load(os.path.join(GOLD, "letter.npz"))
    return (d["X"][:n].astype(np.float64) / 7.5 - 1.0).astype(np.float32), d["y"][:n].astype(np.float64)


def _adult():
    d = np.load(os.path.join(GOLD, "adult8k.npz"))
    return np.unpackbits(d["X"], axis=1)[:, :123].astype(np.float32), d["y"].astype(np.float64)


def _check_classifier(res, mem, real=False, hard=False):
    raw_r, raw_m = np.asarray(res["rawPrediction"]), np.asarray(mem["rawPrediction"])
    if hard:
        np.testing.assert_array_equal(raw_r, raw_m)
    atol = 1e-5 * max(1.0, np.abs(raw_m).max()) if real else 1e-6
    np.testing.assert_allclose(raw_r, raw_m, rtol=1e-5, atol=atol)
    np.testing.assert_allclose(res["probability"], mem["probability"], rtol=1e-5, atol=1e-6)
    srt = np.sort(raw_m, axis=1)
    near_tie = (srt[:, -1] - srt[:, -2]) <= 1e-5 * np.maximum(1.0, np.abs(srt[:, -1])) + atol
    differ = np.asarray(res["prediction"]) != np.asarray(mem["prediction"])
    assert not np.any(differ & ~near_tie)


def _members(rng, M, d, D, p_max, scale=0.5):
    """M random members of D coefficient sets over random columns of d (repeats allowed, some with p = 0)."""
    mem, subs = [], []
    for i in range(M):
        p = 0 if i % 7 == 3 else int(rng.integers(1, p_max + 1))
        subs.append(rng.integers(0, d, p).astype(np.int32))
        mem.append({"coef": rng.normal(0, scale, (D, p)), "intercept": rng.normal(0, 0.3, D),
                    "threshold": float(rng.uniform(0.2, 0.8))})
    return mem, subs


def _device_member_route(X, kind, K, mem, subs, weights=None, init=None, member_class=None, dim=1, loss=0):
    """SLOT_P filled by se_logistic_predict per member, then se_agg_run: (raw, prob, label) or the regressor's row."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.routes import resident_context
    n, M = X.shape[0], len(mem)
    with resident_context(0, X) as ctx:
        ctx.agg_configure(kind, M // dim if kind == N.AGG_GBM_CLASSIFIER else M, K, dim, loss, n)  # GBM: rounds
        ctx.alloc(N.SLOT_PROBA, max(K, 2), n)
        for i, (mb, s) in enumerate(zip(mem, subs)):
            args = (mb["coef"], mb["intercept"], mb["threshold"])
            if kind in REG_KINDS or kind == N.AGG_GBM_CLASSIFIER:
                ctx.logistic_predict(*args, raw=(N.SLOT_PROBA, 0), subspace=s)
                ctx.copy_rows(N.SLOT_P, i, N.SLOT_PROBA, 1, 1)
            elif kind in (N.AGG_BAGGING_SOFT, N.AGG_BOOSTING_REAL):
                ctx.logistic_predict(*args, prob=(N.SLOT_P, i * K), subspace=s)
            else:
                ctx.logistic_predict(*args, label=(N.SLOT_P, i), subspace=s)
        ctx.agg_run(weights, init)
        return _fetch(ctx, kind, K, dim, n)


def _fetch(ctx, kind, K, dim, n):
    from spark_ensemble_b200 import _native as N
    raw = ctx.download(N.SLOT_RAW)
    if kind in REG_KINDS:
        return raw.reshape(-1)[:n]
    C = 2 if (kind == N.AGG_GBM_CLASSIFIER and dim == 1) else (dim if kind == N.AGG_GBM_CLASSIFIER else K)
    return {"rawPrediction": raw.reshape(C, n).T, "probability": ctx.download(N.SLOT_PROB).reshape(C, n).T,
            "prediction": ctx.download(N.SLOT_LABEL).reshape(-1)}


def _linear_agg(X, kind, K, mem, subs, which=0, **kw):
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.routes import resident_context
    n = X.shape[0]
    with resident_context(0, X) as ctx:
        if which:
            ctx.alloc(N.SLOT_VX, X.shape[1], n)
            ctx.upload_rowmajor(N.SLOT_VX, X)
            ctx.upload_rowmajor(N.SLOT_X, np.zeros_like(X))  # the call must not read SLOT_X
        if kind in REG_KINDS:
            ctx.alloc(N.SLOT_RAW, 1, n)
            ctx.linear_agg(kind, K, mem, N.SLOT_RAW, validation=bool(which), subspaces=subs, **kw)
        else:
            ctx.linear_agg(kind, K, mem, validation=bool(which), subspaces=subs, **kw)
        return _fetch(ctx, kind, K, kw.get("dim", 1), n)


def _compare(X, kind, K, mem, subs, which=0, **kw):
    from spark_ensemble_b200 import _native as N
    got = _linear_agg(X, kind, K, mem, subs, which=which, **kw)
    exp = _device_member_route(X, kind, K, mem, subs, **kw)
    if kind in REG_KINDS:
        np.testing.assert_array_equal(got.view(np.uint32), exp.view(np.uint32))
    elif kind == N.AGG_BOOSTING_REAL:
        np.testing.assert_array_equal(got["rawPrediction"], exp["rawPrediction"])
        _check_classifier(got, exp, real=True)
    else:
        _check_classifier(got, exp, hard=kind == N.AGG_BAGGING_HARD)


# ---------------------------------------------------------------- the kernel against the device member route
@pytest.mark.parametrize("n", [1, 3, 127, 128, 129, 4099])
@pytest.mark.parametrize("kind", REG_KINDS)
def test_regressor_kinds_bit_for_bit(kind, n):
    rng = np.random.default_rng(100 + kind * 7 + n)
    d = 9
    X = rng.standard_normal((n, d)).astype(np.float32)
    for M in (1, 5, 17, 64 if kind == 7 else 200):
        mem, subs = _members(rng, M, d, 1, 12, scale=2.0)
        w = rng.uniform(0.1, 2.0, M)
        _compare(X, kind, 0, mem, subs, weights=w if kind != 1 else None, init=[0.37] if kind == 0 else None)


@pytest.mark.parametrize("K", [2, 3, 26, 32])
@pytest.mark.parametrize("kind", [2, 3, 4, 5, 6])
def test_classifier_kinds(kind, K):
    from spark_ensemble_b200 import _native as N
    rng = np.random.default_rng(10 * kind + K)
    n, d, M = 4099, 11, 9
    X = rng.standard_normal((n, d)).astype(np.float32)
    if kind == N.AGG_GBM_CLASSIFIER:
        dim = 1 if K == 2 else K
        mem, subs = _members(rng, M * dim, d, 1, 8)
        for loss in (["bernoulli", "exponential"] if dim == 1 else ["logloss"]):
            _compare(X, kind, K, mem, subs, weights=rng.uniform(0.1, 1.0, M * dim), init=rng.normal(0, 0.2, dim),
                     member_class=np.tile(np.arange(dim), M), dim=dim, loss=loss)
        return
    for D in ([1, K] if K == 2 else [K]):
        mem, subs = _members(rng, M, d, D, 8)
        _compare(X, kind, K, mem, subs, weights=rng.uniform(0.1, 1.5, M) if kind == N.AGG_BOOSTING_DISCRETE else None)


def test_mixed_binomial_and_multinomial_votes_and_which():
    from spark_ensemble_b200 import _native as N
    rng = np.random.default_rng(5)
    n, d, K = 3001, 7, 2
    X = rng.standard_normal((n, d)).astype(np.float32)
    mem = _members(rng, 4, d, 1, 5)[0] + _members(rng, 4, d, 2, 5)[0]
    subs = [rng.integers(0, d, np.atleast_2d(m["coef"]).shape[1]).astype(np.int32) for m in mem]
    for kind in (N.AGG_BAGGING_HARD, N.AGG_BOOSTING_DISCRETE, N.AGG_BAGGING_SOFT, N.AGG_BOOSTING_REAL):
        _compare(X, kind, K, mem, subs, which=1, weights=rng.uniform(0.2, 1.0, 8))


def test_many_members_and_a_wide_union():
    from spark_ensemble_b200 import _native as N
    rng = np.random.default_rng(6)
    n, d = 2053, 300
    X = rng.standard_normal((n, d)).astype(np.float32)
    subs = [np.sort(rng.choice(d, d // 2, replace=False)).astype(np.int32) for _ in range(210)]
    mem = [{"coef": rng.normal(0, 0.05, (1, d // 2)), "intercept": rng.normal(0, 0.1, 1), "threshold": 0.5}
           for _ in subs]
    _compare(X, N.AGG_BAGGING_REGRESSOR, 0, mem, subs)
    _compare(X, N.AGG_BOOSTING_REG_MEAN, 0, mem, subs, weights=rng.uniform(0.1, 1.0, len(mem)))
    memk = [{"coef": rng.normal(0, 0.05, (5, d // 2)), "intercept": rng.normal(0, 0.1, 5), "threshold": 0.5}
            for _ in subs[:40]]
    _compare(X, N.AGG_BAGGING_SOFT, 5, memk, subs[:40])


def test_non_finite_features_margins_and_median_weights():
    from spark_ensemble_b200 import _native as N
    rng = np.random.default_rng(7)
    n, d = 1031, 6
    X = rng.standard_normal((n, d)).astype(np.float32)
    X[::7, 0] = np.inf
    X[3::11, 1] = -np.inf
    X[5::13, 2] = np.nan
    mem, subs = _members(rng, 12, d, 1, 6, scale=1.0)
    for w in (rng.uniform(0.1, 1.0, 12), np.where(np.arange(12) % 3 == 0, -0.5, 1.0),
              np.where(np.arange(12) == 4, np.nan, 1.0), np.where(np.arange(12) == 2, np.inf, 0.5), np.ones(12)):
        _compare(X, N.AGG_BOOSTING_REG_MEDIAN, 0, mem, subs, weights=w)
    # +inf margins: members over one column with a huge coefficient
    memk = [{"coef": np.array([[1e308], [1e308], [0.0]]), "intercept": np.zeros(3), "threshold": 0.5}
            for _ in range(3)]
    Xi = np.abs(X)
    for kind in (N.AGG_BAGGING_SOFT, N.AGG_BAGGING_HARD, N.AGG_BOOSTING_REAL):
        _compare(np.where(np.isnan(Xi), 1, Xi).astype(np.float32), kind, 3, memk, [np.array([0], np.int32)] * 3)


def test_out_row_in_a_wider_slot_keeps_the_other_rows():
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.routes import resident_context
    rng = np.random.default_rng(8)
    n, d = 777, 5
    X = rng.standard_normal((n, d)).astype(np.float32)
    mem, subs = _members(rng, 6, d, 1, 4)
    exp = _device_member_route(X, N.AGG_BAGGING_REGRESSOR, 0, mem, subs)
    with resident_context(0, X) as ctx:
        ctx.alloc(N.SLOT_P, 4, n)
        ctx.upload(N.SLOT_P, np.full((4, n), -12345.5, dtype=np.float32))
        ctx.linear_agg(N.AGG_BAGGING_REGRESSOR, 0, mem, N.SLOT_P, 2, subspaces=subs)
        got = ctx.download(N.SLOT_P).reshape(4, -1)[:, :n]
    np.testing.assert_array_equal(got[2], exp)
    assert np.all(got[[0, 1, 3]] == np.float32(-12345.5))


# ---------------------------------------------------------------- against the oracle
def test_each_kind_against_the_oracle(oracle):
    from spark_ensemble_b200 import _native as N
    rng = np.random.default_rng(9)
    n, d, M, K = 5003, 8, 7, 4
    X = rng.standard_normal((n, d)).astype(np.float32)
    mem, subs = _members(rng, M, d, 1, 6)
    V = np.stack([X[:, s].astype(np.float64) @ m["coef"][0] + m["intercept"][0] for m, s in zip(mem, subs)])
    a = rng.uniform(0.2, 1.5, M)
    np.testing.assert_allclose(_linear_agg(X, N.AGG_GBM_REGRESSOR, 0, mem, subs, weights=a, init=[0.5]),
                               oracle.agg_weighted_sum(V, a, 0.5), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(_linear_agg(X, N.AGG_BAGGING_REGRESSOR, 0, mem, subs), oracle.agg_mean(V),
                               rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(_linear_agg(X, N.AGG_BOOSTING_REG_MEAN, 0, mem, subs, weights=a),
                               oracle.agg_weighted_mean(V, a), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(_linear_agg(X, N.AGG_BOOSTING_REG_MEDIAN, 0, mem, subs, weights=a),
                               oracle.agg_weighted_median(V.astype(np.float32), a), rtol=1e-5, atol=1e-5)
    memk, subsk = _members(rng, M, d, K, 6)
    Mg = np.stack([X[:, s].astype(np.float64) @ m["coef"].T + m["intercept"] for m, s in zip(memk, subsk)])  # [M][n][K]
    e = np.exp(Mg - Mg.max(axis=2, keepdims=True))
    P = (e / e.sum(axis=2, keepdims=True)).transpose(0, 2, 1)  # [M][K][n]
    votes = Mg.argmax(axis=2).astype(np.float64)
    out = _linear_agg(X, N.AGG_BAGGING_SOFT, K, memk, subsk)
    raw, prob = oracle.agg_bagging_soft(P)
    np.testing.assert_allclose(out["rawPrediction"], raw.T, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(out["probability"], prob.T, rtol=1e-5, atol=1e-5)
    out = _linear_agg(X, N.AGG_BAGGING_HARD, K, memk, subsk)
    raw, prob = oracle.agg_bagging_hard(votes, K)
    np.testing.assert_allclose(out["rawPrediction"], raw.T, rtol=1e-5, atol=1e-5)
    out = _linear_agg(X, N.AGG_BOOSTING_REAL, K, memk, subsk)
    raw, prob = oracle.agg_boosting_real(P)
    np.testing.assert_allclose(out["rawPrediction"], raw.T, rtol=1e-5, atol=1e-5 * np.abs(raw).max())
    np.testing.assert_allclose(out["probability"], prob.T, rtol=1e-5, atol=1e-5)
    out = _linear_agg(X, N.AGG_BOOSTING_DISCRETE, K, memk, subsk, weights=a)
    raw, prob = oracle.agg_boosting_discrete(votes, a.astype(np.float32), K)
    np.testing.assert_allclose(out["rawPrediction"], raw.T, rtol=1e-5, atol=1e-5)
    wts = rng.uniform(0.1, 1.0, (M, 1))
    out = _linear_agg(X, N.AGG_GBM_CLASSIFIER, 2, mem, subs, weights=wts.reshape(-1), init=[0.2],
                      member_class=np.zeros(M), dim=1, loss="bernoulli")
    raw = oracle.agg_gbm_classifier_raw(V.reshape(M, 1, n), wts, np.array([0.2]), 2)
    np.testing.assert_allclose(out["rawPrediction"], raw.T, rtol=1e-5, atol=1e-5)


# ---------------------------------------------------------------- fitted models: residentFeatures on and off
def _both(model, X):
    from spark_ensemble_b200 import DataFrame
    model.set("residentFeatures", True)
    a = model.transform(DataFrame(features=X))
    model.set("residentFeatures", False)
    b = model.transform(DataFrame(features=X))
    return a, b


@pytest.mark.parametrize("learner", ["device", "host"])
def test_fitted_regressors(learner):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.learners import DeviceLinearRegression, LinearRegression
    from spark_ensemble_b200.regression import (BaggingRegressor, BoostingRegressionModel, BoostingRegressor,
                                                GBMRegressor)
    X, y = _cpusmall()
    lr = DeviceLinearRegression() if learner == "device" else LinearRegression()
    df = DataFrame(features=X, label=y)
    res = learner == "device"
    fitted = [
        GBMRegressor().setBaseLearner(lr).setNumBaseLearners(3).setSubspaceRatio(0.5).setResidentFeatures(res).fit(df),
        BaggingRegressor().setBaseLearner(lr).setNumBaseLearners(4).setSubspaceRatio(0.6).setResidentFeatures(res).fit(df),
        BoostingRegressor().setBaseLearner(lr).setNumBaseLearners(4).setResidentFeatures(res).fit(df),
    ]
    fitted.append(BoostingRegressionModel(fitted[-1].weights, fitted[-1].models).setVotingStrategy("mean"))
    for m in fitted:
        a, b = _both(m, X)
        np.testing.assert_array_equal(a["prediction"], b["prediction"])
        one = []
        for res in (True, False):  # one row: se_agg_run's tail form on both routes
            m.set("residentFeatures", res)
            one.append(m.predict(X[5]))
        assert one[0] == one[1]


@pytest.mark.parametrize("data", ["adult8k", "letter"])
def test_fitted_classifiers(data):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.classification import BaggingClassifier, BoostingClassifier, GBMClassifier
    from spark_ensemble_b200.learners import DeviceLinearRegression, DeviceLogisticRegression
    X, y = _adult() if data == "adult8k" else _letter(4000)
    if data == "letter":
        y = y % 5
    df = DataFrame(features=X, label=y)
    lg = DeviceLogisticRegression(regParam=0.01, maxIter=30)
    fitted = []
    for s in ("soft", "hard"):
        fitted.append(BaggingClassifier().setBaseLearner(lg).setNumBaseLearners(3).setSubspaceRatio(0.5)
                      .setVotingStrategy(s).setResidentFeatures(True).fit(df))
    for alg in ("real", "discrete"):
        fitted.append(BoostingClassifier().setBaseLearner(lg).setNumBaseLearners(3).setAlgorithm(alg)
                      .setResidentFeatures(True).fit(df))
    fitted.append(GBMClassifier().setBaseLearner(DeviceLinearRegression()).setNumBaseLearners(3).setSubspaceRatio(0.5)
                  .setResidentFeatures(True).fit(df))
    for m in fitted:
        a, b = _both(m, X)
        real = m.hasParam("algorithm") and m("algorithm") == "real"
        hard = m.hasParam("votingStrategy") and m("votingStrategy") == "hard"
        _check_classifier(a, b, real=real, hard=hard)
        m.set("residentFeatures", True)
        np.testing.assert_array_equal(m.predictRaw(X[7]), a["rawPrediction"][7])
        np.testing.assert_array_equal(m.predictProbability(X[7]), a["probability"][7])
        assert m.predict(X[7]) == a["prediction"][7]


def test_nothing_scored_or_stacked_on_the_host(monkeypatch):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200 import learners as L
    from spark_ensemble_b200.classification import (BaggingClassificationModel, BoostingClassificationModel,
                                                    GBMClassificationModel)
    from spark_ensemble_b200.context import Context
    from spark_ensemble_b200.ensemble import fit_dummy_regressor
    from spark_ensemble_b200.regression import BaggingRegressionModel, BoostingRegressionModel, GBMRegressionModel
    rng = np.random.default_rng(11)
    K, M, n, d = 4, 6, 5003, 5
    X = rng.standard_normal((n, d)).astype(np.float32)
    cls = [L.LogisticRegressionModel(rng.normal(0, 0.5, (K, d)), rng.normal(0, 0.2, K), K, True) for _ in range(M)]
    reg = [L.LinearRegressionModel(rng.normal(0, 1, d), rng.normal()) for _ in range(M)]
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
        BoostingRegressionModel(a, reg).setVotingStrategy("median"),
    ]
    df = DataFrame(features=X)
    expected = [m.transform(df) for m in models]

    def boom(*a, **k):
        raise AssertionError("a member was scored on the host")

    for c, names in ((L.LogisticRegressionModel, ("predict", "predictProbability", "predictRaw", "_margins")),
                     (L.LinearRegressionModel, ("predict",))):
        for name in names:
            monkeypatch.setattr(c, name, boom)
    real_upload = Context.upload

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


# ---------------------------------------------------------------- fallbacks and errors
def test_fallbacks_take_the_member_route():
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200 import learners as L
    from spark_ensemble_b200.classification import BaggingClassificationModel
    from spark_ensemble_b200.regression import BaggingRegressionModel, BoostingRegressionModel
    rng = np.random.default_rng(12)
    n, d = 2001, 260
    X = rng.standard_normal((n, d)).astype(np.float32)
    K = N.FOREST_AGG_MAX_CLASSES + 1
    cls = [L.LogisticRegressionModel(rng.normal(0, 0.1, (K, 4)), rng.normal(0, 0.1, K), K, True) for _ in range(3)]
    m = BaggingClassificationModel(K, [np.arange(4)] * 3, cls).setVotingStrategy("soft")
    a, b = _both(m, X)
    for col in ("rawPrediction", "probability", "prediction"):
        np.testing.assert_array_equal(a[col], b[col])
    reg = [L.LinearRegressionModel(rng.normal(0, 0.1, 4), 0.1 * i) for i in range(N.FOREST_MEDIAN_MAX_TREES + 1)]
    a, b = _both(BoostingRegressionModel(rng.uniform(0.1, 1, len(reg)), [r for r in reg]).setVotingStrategy("median"),
                 X[:, :4])
    np.testing.assert_array_equal(a["prediction"], b["prediction"])
    wide = [L.LinearRegressionModel(rng.normal(0, 0.01, 255), 0.0), L.LinearRegressionModel(rng.normal(0, 0.01, 255), 1.0)]
    a, b = _both(BaggingRegressionModel([np.arange(255)] * 2, wide), X)
    np.testing.assert_array_equal(a["prediction"], b["prediction"])
    tree = L.DeviceDecisionTreeRegressionModel({"feature": np.array([0, -1, -1], np.int32),
                                                "threshold": np.array([0.0, 0, 0], np.float32),
                                                "left": np.array([1, 0, 0], np.int32), "right": np.array([2, 0, 0], np.int32),
                                                "value": np.array([0, -1.0, 1.0], np.float32)})
    a, b = _both(BaggingRegressionModel([np.arange(4)] * 2, [tree, reg[0]]), X[:, :4])
    np.testing.assert_array_equal(a["prediction"], b["prediction"])


def test_bad_arguments_are_argument_errors():
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.routes import resident_context
    rng = np.random.default_rng(13)
    n, d = 100, 5
    X = rng.standard_normal((n, d)).astype(np.float32)
    one = {"coef": np.ones((1, 2)), "intercept": np.zeros(1), "threshold": 0.5}
    three = {"coef": np.ones((3, 2)), "intercept": np.zeros(3), "threshold": 0.5}
    with resident_context(0, X) as ctx:
        ctx.alloc(N.SLOT_RAW, 1, n)
        cases = [
            lambda: ctx.linear_agg(N.AGG_BAGGING_REGRESSOR, 0, [one], N.SLOT_RAW, subspaces=[[0, d]]),
            lambda: ctx.linear_agg(N.AGG_BAGGING_REGRESSOR, 0, [one], N.SLOT_RAW, subspaces=[[-1, 0]]),
            lambda: ctx.linear_agg(N.AGG_BAGGING_REGRESSOR, 0, [three], N.SLOT_RAW, subspaces=[[0, 1]]),
            lambda: ctx.linear_agg(N.AGG_BAGGING_SOFT, 4, [three], subspaces=[[0, 1]]),
            lambda: ctx.linear_agg(N.AGG_BAGGING_SOFT, 33, [three], subspaces=[[0, 1]]),
            lambda: ctx.linear_agg(N.AGG_BOOSTING_REG_MEDIAN, 0, [one] * 65, N.SLOT_RAW, weights=np.ones(65),
                                   subspaces=[[0, 1]] * 65),
            lambda: ctx.linear_agg(N.AGG_BAGGING_REGRESSOR, 0, [{"coef": np.ones((1, 255)), "intercept": np.zeros(1)}],
                                   N.SLOT_RAW, subspaces=[np.zeros(255, np.int32)]),
            lambda: ctx.linear_agg(N.AGG_GBM_REGRESSOR, 0, [one], N.SLOT_RAW, subspaces=[[0, 1]]),  # no weights
            lambda: ctx.linear_agg(N.AGG_BAGGING_REGRESSOR, 0, [one], N.SLOT_X, subspaces=[[0, 1]]),
        ]
        for f in cases:
            with pytest.raises(ValueError, match="libse_b200"):
                f()


# ---------------------------------------------------------------- stacking members
def test_stacking_members_stay_on_the_device(monkeypatch):
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.classification import BaggingClassifier, StackingClassifier
    from spark_ensemble_b200.learners import DeviceLinearRegression, DeviceLogisticRegression
    from spark_ensemble_b200.regression import GBMRegressor, StackingRegressor
    from spark_ensemble_b200 import routes
    Xa, ya = _adult()
    Xa, ya = Xa[:3000], ya[:3000]
    X, y = _cpusmall()
    wrote = []
    real = routes.write_member_rows

    def spy(ctx, model, method, row, width):
        ok = real(ctx, model, method, row, width)
        wrote.append((type(model).__name__, ok))
        return ok

    monkeypatch.setattr(routes, "write_member_rows", spy)
    bag = BaggingClassifier().setBaseLearner(DeviceLogisticRegression(regParam=0.01, maxIter=20)).setNumBaseLearners(3)
    sc = StackingClassifier().setBaseLearners([bag.setVotingStrategy("soft")]).setStacker(
        DeviceLogisticRegression(maxIter=20)).setStackMethod("proba")
    gbm = GBMRegressor().setBaseLearner(DeviceLinearRegression()).setNumBaseLearners(3).setResidentFeatures(True)
    sr = StackingRegressor().setBaseLearners([gbm]).setStacker(DeviceLinearRegression())
    for est, Xs, ys, col in ((sc, Xa, ya, "prediction"), (sr, X, y, "prediction")):
        df = DataFrame(features=Xs, label=ys)
        model = est.setResidentFeatures(True).fit(df)
        wrote.clear()
        a = model.transform(df)[col]
        assert wrote and all(ok for _, ok in wrote), wrote
        model.set("residentFeatures", False)
        b = model.transform(df)[col]
        scale = max(1.0, np.abs(b).max())
        np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-5 * scale)


# ---------------------------------------------------------------- past 2^31 elements of X
def test_scale_past_2_31_elements():
    from spark_ensemble_b200 import _native as N
    rng = np.random.default_rng(14)
    n, d = 17_000_000, 128
    X = np.empty((n, d), dtype=np.float32)
    for i in range(0, n, 1_000_000):
        X[i:i + 1_000_000] = rng.standard_normal((min(1_000_000, n - i), d), dtype=np.float32)
    mem = [{"coef": rng.normal(0, 0.1, (1, 4)), "intercept": rng.normal(0, 0.1, 1), "threshold": 0.5} for _ in range(3)]
    subs = [np.array([0, 64, 126, 127], np.int32), np.array([127, 1, 100, 120], np.int32), np.array([125], np.int32)]
    mem[2]["coef"] = mem[2]["coef"][:, :1]
    _compare(X, N.AGG_BAGGING_REGRESSOR, 0, mem, subs)
