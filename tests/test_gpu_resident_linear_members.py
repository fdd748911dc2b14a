"""DeviceLinearRegression and DeviceLogisticRegression as the base learner of Bagging, Boosting and GBM with
residentFeatures: fitted where the estimators' data live (one context, X uploaded once) against the same estimators with
residentFeatures=False, whose members fit through the learners' own `fit` on the rows the reference hands them.  Golden
sets: cpusmall (regression), adult8k (binary) and letter (26 classes).

- Bagging: each linear member's predictions, at a tolerance from its normal equations' conditioning; each logistic
  member's final objective, evaluated in fp64 by oracle/np_logistic.py on the member's own in-bag rows, to the
  optimiser's tolerance; the ensemble's labels (a near-tie may go either way).  Out-of-bag rows holding non-finite
  features must not fail the fit.  The lock-step fit equals, bit for bit, the fit of every member in a batch of its own.
- Boosting (SAMME, SAMME.R, AdaBoost.R2) and GBM: the per-round history and the outputs at 1e-5, as the tree tests do."""
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


@pytest.mark.parametrize("loss", ["squared"])
@pytest.mark.parametrize("bagged", [False, True])
def test_gbm_regressor_linear(loss, bagged):
    from spark_ensemble_b200.learners import DeviceLinearRegression
    from spark_ensemble_b200.regression import GBMRegressor
    X, y = _golden("cpusmall")
    # standardised features: the device direction is scored with fp32 coefficients (se_linear_predict, as every
    # resident linear direction is), and cpusmall's raw column scales (up to 4e5) turn their rounding into 1e-5 of α
    X = (X - X.mean(axis=0)) / X.std(axis=0)
    df = _frame(X, y, False)
    val = np.zeros(y.size, dtype=bool)
    val[::5] = True
    df = df.__class__(**{**{k: df[k] for k in ("features", "label")}, "val": val})
    est = (GBMRegressor().setBaseLearner(DeviceLinearRegression(regParam=0.1)).setNumBaseLearners(5)
           .setLoss(loss).setSubspaceRatio(0.7).setValidationIndicatorCol("val"))
    if bagged:
        est = est.setSubsampleRatio(0.8)
    resident = est.setResidentFeatures(True).fit(df)
    member = est.setResidentFeatures(False).fit(df)
    _history_close(resident.trainingHistory, member.trainingHistory, ("alpha", "trainLoss", "validationLoss"))
    col = resident("predictionCol")
    np.testing.assert_allclose(resident.transform(df)[col], member.transform(df)[col], rtol=1e-5, atol=1e-5)
