"""DeviceLinearRegression and DeviceLogisticRegression as the base learner of Bagging, Boosting and GBM with
residentFeatures: fitted where the estimators' data live (one context, X uploaded once) against the same estimators with
residentFeatures=False, whose members fit through the learners' own `fit` on the rows the reference hands them.  Golden
sets: cpusmall (regression), adult8k (binary) and letter (26 classes).

- Bagging: each linear member's predictions, at a tolerance from its normal equations' conditioning; each logistic
  member's final objective, evaluated in fp64 by oracle/np_logistic.py on the member's own in-bag rows, to the
  optimiser's tolerance; the ensemble's labels (a near-tie may go either way).  Out-of-bag rows holding non-finite
  features must not fail the fit.  The lock-step fit equals, bit for bit, the fit of every member in a batch of its own.
- Boosting (SAMME, SAMME.R, AdaBoost.R2): the per-round history and the outputs at 1e-5, as the tree tests do.
- GBM (every regressor and classifier loss, gradient and Newton updates): as `_gbm_routes` states."""
import numpy as np
import pytest

from oracle import np_logistic as O

pytestmark = pytest.mark.gpu

TOL = 1e-10  # the logistic members' L-BFGS tolerance


def _golden(name, n=None):
    import os
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", f"{name}.npz"))
    X, y = z["X"].astype(np.float64), z["y"].astype(np.float64)
    return (X, y) if n is None else (X[:n], y[:n])


def _frame(X, y, weighted, seed=0):
    from spark_ensemble_b200.ensemble import DataFrame
    cols = dict(features=X, label=y)
    if weighted:
        cols["weight"] = np.random.default_rng(seed).uniform(0.5, 2.0, y.size)
    return DataFrame(**cols)


def _bag_rows(est, n, w):
    """The bag bagging_fit draws: (in-bag rows, their weights)."""
    rng = np.random.default_rng(est("seed") & 0xFFFFFFFF)
    counts = (rng.poisson(est("subsampleRatio"), n) if est("replacement")
              else (rng.random(n) < est("subsampleRatio"))).astype(np.float64)
    bw = counts if w is None else counts * w
    return np.flatnonzero(bw > 0), bw


def _objective(model, X, y, w, cols, lam, K):
    """Spark's objective of a fitted model over rows X[:, cols] (raw space, L2 part with standardization)."""
    coef = np.concatenate([model.coefficientMatrix, model.interceptVector[:, None]], axis=1)
    loss, _ = O.loss_grad(X, y, cols, coef, w)
    st = O.stats(X, y, cols, K, w)
    p = len(cols)
    sw, sw2, d1, d2 = st[0], st[1], st[2:2 + p], st[2 + p:2 + 2 * p]
    sigma = np.sqrt(np.maximum(d2 - d1 * d1 / sw, 0.0) / (sw - sw2 / sw))
    return loss / sw + 0.5 * lam * float(np.sum((model.coefficientMatrix * sigma) ** 2))


def _bagging(kind, ratio, replacement, weighted, M=5):
    from spark_ensemble_b200.classification import BaggingClassifier
    from spark_ensemble_b200.learners import DeviceLinearRegression, DeviceLogisticRegression
    from spark_ensemble_b200.regression import BaggingRegressor
    if kind == "linear":
        est = BaggingRegressor().setBaseLearner(DeviceLinearRegression(regParam=0.0))
    else:
        est = BaggingClassifier().setBaseLearner(DeviceLogisticRegression(regParam=0.01, tol=TOL, maxIter=200))
    return (est.setNumBaseLearners(M).setSubspaceRatio(ratio).setSubsampleRatio(0.7).setReplacement(replacement)
            .setResidentFeatures(True))


BAG_DATA = {"linear": ("cpusmall", None), "binary": ("adult8k", None), "letter": ("letter", 6000)}


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("replacement", [True, False])
@pytest.mark.parametrize("ratio", [0.5, 1.0])
@pytest.mark.parametrize("kind", ["linear", "binary", "letter"])
def test_bagging_resident_route_equals_member_route(kind, ratio, replacement, weighted):
    name, n = BAG_DATA[kind]
    X, y = _golden(name, n)
    df = _frame(X, y, weighted, seed=int(10 * ratio))
    est = _bagging(kind, ratio, replacement, weighted)
    if weighted:
        est = est.setWeightCol("weight")
    resident = est.setResidentFeatures(True).fit(df)
    member = est.setResidentFeatures(False).fit(df)
    w = np.asarray(df["weight"]) if weighted else None
    rows, bw = _bag_rows(est, y.size, w)
    Xb = X.astype(np.float32)[rows]
    for sub, a, b in zip(resident.subspaces, resident.models, member.models):
        if kind == "linear":
            Z = Xb[:, sub].astype(np.float64)
            Zc = (Z - Z.mean(axis=0)) / np.maximum(Z.std(axis=0), 1e-300)
            cond = np.linalg.cond(Zc.T @ (bw[rows][:, None] * Zc)) if sub.size else 1.0
            pa, pb = a.predict(Z), b.predict(Z)
            tol = max(1e-9, 1e-13 * cond) * np.abs(pb).max()
            assert np.abs(pa - pb).max() <= tol, (np.abs(pa - pb).max(), tol, cond)
        else:
            K = int(y.max()) + 1
            fa = _objective(a, Xb, y[rows], bw[rows], sub, 0.01, K)
            fb = _objective(b, Xb, y[rows], bw[rows], sub, 0.01, K)
            assert abs(fa - fb) <= 1e3 * TOL * max(1.0, abs(fb)), (fa, fb)
    col = resident("predictionCol")
    pa, pb = np.asarray(resident.transform(df)[col]), np.asarray(member.transform(df)[col])
    if kind == "linear":
        np.testing.assert_allclose(pa, pb, rtol=1e-5, atol=1e-5 * np.abs(pb).max())
    else:
        assert np.mean(pa != pb) <= 2e-3, np.mean(pa != pb)  # near-ties only


@pytest.mark.parametrize("kind", ["linear", "binary"])
def test_bagging_out_of_bag_non_finite_features_do_not_fail(kind):
    X, y = _golden(*BAG_DATA[kind])
    est = _bagging(kind, 1.0, False, False)
    rows, _ = _bag_rows(est, y.size, None)
    out = np.setdiff1d(np.arange(y.size), rows)[:50]
    Xn = X.copy()
    Xn[out, 1] = np.inf
    Xn[out[::2], 3] = np.nan
    if kind == "binary":
        yn = y.copy()
        yn[out[:5]] = 7.5  # an out-of-bag label the member route never reads
    else:
        yn = y
    resident = est.setResidentFeatures(True).fit(_frame(Xn, yn, False))
    clean = est.setResidentFeatures(True).fit(_frame(np.where(np.isfinite(Xn), Xn, 0.0), yn, False))
    member = est.setResidentFeatures(False).fit(_frame(Xn, yn, False))
    for a, b, c in zip(resident.models, clean.models, member.models):
        if kind == "linear":
            assert a.coefficients.tobytes() == b.coefficients.tobytes()
            np.testing.assert_allclose(a.coefficients, c.coefficients, rtol=1e-4, atol=1e-8)
        else:
            assert a.coefficientMatrix.tobytes() == b.coefficientMatrix.tobytes()
    # an in-bag non-finite feature fails both routes
    Xn[rows[3], 2] = np.nan
    for resident_features in (True, False):
        with pytest.raises(ValueError):
            est.setResidentFeatures(resident_features).fit(_frame(Xn, yn, False))


@pytest.mark.parametrize("name,n", [("adult8k", None), ("letter", 4000)])
def test_lockstep_fit_equals_members_fitted_alone(name, n):
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    from spark_ensemble_b200.ensemble import subspace
    from spark_ensemble_b200.learners import DeviceLogisticRegression
    X, y = _golden(name, n)
    X = X.astype(np.float32)
    K = int(y.max()) + 1
    w = np.random.default_rng(1).uniform(0, 2, y.size)
    w[::7] = 0.0
    subs = [subspace(0.5, X.shape[1], 40 + i) for i in range(6)] + [np.arange(X.shape[1], dtype=np.int32)]
    learner = DeviceLogisticRegression(regParam=0.05, elasticNetParam=0.3, tol=1e-9)
    with Context(0) as ctx:
        ctx.alloc(N.SLOT_X, X.shape[1], X.shape[0])
        ctx.upload_rowmajor(N.SLOT_X, X)
        ctx.alloc(N.SLOT_Y, y.size)
        ctx.upload(N.SLOT_Y, y.astype(np.float32))
        ctx.alloc(N.SLOT_W, y.size)
        ctx.upload(N.SLOT_W, w.astype(np.float32))
        shifts = [X[0, s].astype(np.float64) for s in subs]
        together = learner.fit_members_resident(ctx, subs, K, N.SLOT_Y, 0, N.SLOT_W, 0, shifts)
        alone = [learner.fit_members_resident(ctx, [s], K, N.SLOT_Y, 0, N.SLOT_W, 0, [sh])[0]
                 for s, sh in zip(subs, shifts)]
    assert len({m.numEvaluations for m in together}) > 1
    for a, b in zip(together, alone):
        assert a.coefficientMatrix.tobytes() == b.coefficientMatrix.tobytes()
        assert a.interceptVector.tobytes() == b.interceptVector.tobytes()
        assert a.objectiveHistory == b.objectiveHistory


# ---- Boosting and GBM -------------------------------------------------------------------------------------------------
def _history_close(ha, hb, keys):
    assert len(ha) == len(hb)
    for a, b in zip(ha, hb):
        for k in keys:
            np.testing.assert_allclose(a[k], b[k], rtol=1e-5, atol=1e-5, err_msg=k)


@pytest.mark.parametrize("algorithm", ["discrete", "real"])
@pytest.mark.parametrize("weighted", [False, True])
def test_boosting_classifier_logistic(algorithm, weighted):
    from spark_ensemble_b200.classification import BoostingClassifier
    from spark_ensemble_b200.learners import DeviceLogisticRegression
    X, y = _golden("adult8k")
    df = _frame(X, y, weighted, seed=3)
    est = (BoostingClassifier().setBaseLearner(DeviceLogisticRegression(regParam=0.01, tol=TOL, maxIter=200))
           .setNumBaseLearners(4).setAlgorithm(algorithm))
    if weighted:
        est = est.setWeightCol("weight")
    resident = est.setResidentFeatures(True).fit(df)
    member = est.setResidentFeatures(False).fit(df)
    _history_close(resident.trainingHistory, member.trainingHistory, ("estimatorError", "sumWeights"))
    np.testing.assert_allclose(resident.weights, member.weights, rtol=1e-5, atol=1e-5)
    for col in (resident("probabilityCol"), resident("predictionCol")):
        np.testing.assert_allclose(resident.transform(df)[col], member.transform(df)[col], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("loss", ["exponential", "squared", "linear"])
@pytest.mark.parametrize("reg", [0.0, 0.5])
def test_boosting_regressor_linear(loss, reg):
    from spark_ensemble_b200.learners import DeviceLinearRegression
    from spark_ensemble_b200.regression import BoostingRegressor
    X, y = _golden("cpusmall")
    df = _frame(X, y, True, seed=4)
    est = (BoostingRegressor().setBaseLearner(DeviceLinearRegression(regParam=reg)).setNumBaseLearners(4)
           .setLossType(loss).setWeightCol("weight"))
    resident = est.setResidentFeatures(True).fit(df)
    member = est.setResidentFeatures(False).fit(df)
    _history_close(resident.trainingHistory, member.trainingHistory, ("maxError", "estimatorError", "sumWeights"))
    col = resident("predictionCol")
    np.testing.assert_allclose(resident.transform(df)[col], member.transform(df)[col], rtol=1e-5, atol=1e-5)


def _gbm_routes(monkeypatch, est, df, quadratic):
    """The member route's and the resident route's fits of a GBM.  With the squared loss, every round's α, trainLoss and
    validationLoss agree at 1e-5.  Elsewhere α comes from Brent or L-BFGS-B over a sum of fp32 per-row losses, which
    pins it only to the objective's resolution: the two routes' α of each round are compared through the objective
    instead, both evaluated on the resident fit's context, which holds that round's F and h, at 1e-5.  The first round
    starts both routes from the same F, so its losses agree at 1e-5; after it the routes' F differ by that resolution,
    and the next residuals (signs, clipped or saturated in F) carry it into the next directions: measured up to 3e-4 of
    the loss over five rounds on cpusmall, allowed 1e-3.  tests/test_gpu_resident_linear_gbm.py checks every round of
    the resident route against fp64 instead."""
    from spark_ensemble_b200.gbm_engine import GBMEngine
    member = est.setResidentFeatures(False).fit(df)
    alphas = [np.atleast_1d(h["alpha"]) for h in member.trainingHistory]
    f = []

    def spied(real):
        def run(eng, tol, max_iter):
            out = real(eng, tol, max_iter)
            a_mem = alphas[len(f)] if len(f) < len(alphas) else np.atleast_1d(out[0])
            f.append((eng.ctx.gbm_linesearch_eval(out[0])[0], eng.ctx.gbm_linesearch_eval(a_mem)[0]))
            return out
        return run

    if not quadratic:
        monkeypatch.setattr(GBMEngine, "line_search_brent", spied(GBMEngine.line_search_brent))
        monkeypatch.setattr(GBMEngine, "line_search_lbfgsb", spied(GBMEngine.line_search_lbfgsb))
    resident = est.setResidentFeatures(True).fit(df)
    monkeypatch.undo()
    ha, hb = resident.trainingHistory, member.trainingHistory
    if quadratic:
        _history_close(ha, hb, ("alpha", "trainLoss", "validationLoss"))
    else:
        assert len(ha) == len(hb)
        for i, (a, b) in enumerate(zip(ha, hb)):
            for k in ("trainLoss", "validationLoss"):
                np.testing.assert_allclose(a[k], b[k], rtol=1e-5 if i == 0 else 1e-3, err_msg=f"round {i} {k}")
    for i, (fa, fb) in enumerate(f):
        assert abs(fa - fb) <= 1e-5 * max(1.0, abs(fa)), (i, fa, fb)
    return resident, member


# standardised features: the device direction is scored with fp32 coefficients (se_linear_predict, as every resident
# linear direction is), and cpusmall's raw column scales (up to 4e5) turn their rounding into 1e-5 of α
@pytest.mark.parametrize("bagged,weighted", [(False, False), (True, True)])
@pytest.mark.parametrize("loss,updates,reg", [("squared", "gradient", 0.1), ("absolute", "gradient", 0.1),
                                              ("huber", "gradient", 0.1), ("quantile", "gradient", 0.1),
                                              ("squared", "newton", 0.5)])
def test_gbm_regressor_linear(monkeypatch, loss, updates, reg, bagged, weighted):
    from spark_ensemble_b200.learners import DeviceLinearRegression
    from spark_ensemble_b200.regression import GBMRegressor
    X, y = _golden("cpusmall")
    X = (X - X.mean(axis=0)) / X.std(axis=0)
    df = _frame(X, y, weighted, seed=6)
    val = np.zeros(y.size, dtype=bool)
    val[::5] = True
    df = df.__class__(**{**{k: df[k] for k in df.columns}, "val": val})
    est = (GBMRegressor().setBaseLearner(DeviceLinearRegression(regParam=reg)).setNumBaseLearners(5)
           .setLoss(loss).setSubspaceRatio(0.7).setValidationIndicatorCol("val").set("updates", updates))
    if bagged:
        est = est.setSubsampleRatio(0.8)
    if weighted:
        est = est.setWeightCol("weight")
    resident, member = _gbm_routes(monkeypatch, est, df, loss == "squared")
    col = resident("predictionCol")
    pa, pb = np.asarray(resident.transform(df)[col]), np.asarray(member.transform(df)[col])
    if loss == "squared":
        np.testing.assert_allclose(pa, pb, rtol=1e-5, atol=1e-5 * np.abs(pb).max())
    else:  # as the losses; rows far out along a direction carry its difference further (measured 4e-3 of the scale)
        assert np.abs(pa - pb).mean() <= 1e-3 * np.abs(pb).mean()
        assert np.abs(pa - pb).max() <= 1e-2 * np.abs(pb).max()


@pytest.mark.parametrize("updates", ["gradient", "newton"])
@pytest.mark.parametrize("loss", ["bernoulli", "exponential", "logloss"])
def test_gbm_classifier_linear(monkeypatch, loss, updates):
    from spark_ensemble_b200.classification import GBMClassifier
    from spark_ensemble_b200.learners import DeviceLinearRegression
    if loss == "logloss":  # 4 classes of letter, a ragged row count
        X, y = _golden("letter")
        keep = np.flatnonzero(y < 4)[:2501]
        X, y = X[keep], y[keep]
    else:
        X, y = _golden("adult8k")
    X = (X - X.mean(axis=0)) / np.maximum(X.std(axis=0), 1e-12)
    df = _frame(X, y, True, seed=8)
    val = np.zeros(y.size, dtype=bool)
    val[1::6] = True
    df = df.__class__(**{**{k: df[k] for k in df.columns}, "val": val})
    est = (GBMClassifier().setBaseLearner(DeviceLinearRegression(regParam=0.5)).setNumBaseLearners(4)
           .setLoss(loss).set("updates", updates).setSubspaceRatio(0.7).setSubsampleRatio(0.8)
           .setValidationIndicatorCol("val").setWeightCol("weight"))
    resident, member = _gbm_routes(monkeypatch, est, df, False)
    # the members' weights are L-BFGS-B's α, which the routes share only to the objective's resolution (as the losses)
    ta, tb = resident.transform(df), member.transform(df)
    for col in (resident("probabilityCol"), resident("rawPredictionCol")):
        np.testing.assert_allclose(ta[col], tb[col], rtol=1e-3, atol=1e-4)
    assert np.mean(np.asarray(ta[resident("predictionCol")]) != np.asarray(tb[resident("predictionCol")])) <= 2e-3
