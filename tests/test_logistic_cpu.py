"""DeviceLogisticRegression's optimiser driven by the numpy evaluation of oracle/np_logistic.py, against
scikit-learn's LogisticRegression on adult8k (binomial) and letter (26 classes); the numpy evaluation against finite
differences; Spark's post-processing (centring, σ = 0 columns, a single class, no intercept) and Param validation."""
import os
import warnings

import numpy as np
import pytest

from oracle import np_logistic as O
from spark_ensemble_b200.learners import DeviceLogisticRegression, LogisticRegressionModel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _data(name, rows=None):
    z = np.load(os.path.join(ROOT, "tests", "golden", f"{name}.npz"))
    X, y = z["X"].astype(np.float32).astype(np.float64), z["y"].astype(np.float64)
    return (X, y) if rows is None else (X[:rows], y[:rows])


def _fit(est, X, y, w=None, K=None):
    K = int(y.max()) + 1 if K is None else K
    cols = np.arange(X.shape[1])
    shift = X[0].copy()
    st = O.stats(X, y, cols, K, w, shift)
    return est.optimize(O.evaluator(X, y, cols, w), st, shift, K)


def _sigma(X, w):
    c = np.ones(X.shape[0]) if w is None else w
    mu = c @ X / c.sum()
    return np.sqrt((c @ (X - mu) ** 2) / (c.sum() - (c @ c) / c.sum()))


def _objective(X, y, w, beta, b, lam, alpha, sigma):
    """Spark's objective in raw space (standardization on): the quantity both fits minimise."""
    c = np.ones(y.size) if w is None else w
    M = X @ np.atleast_2d(beta).T + b
    if M.shape[1] == 1:
        loss = np.logaddexp(0.0, M[:, 0]) - (y == 1) * M[:, 0]
    else:
        mx = M.max(axis=1)
        loss = mx + np.log(np.exp(M - mx[:, None]).sum(axis=1)) - M[np.arange(y.size), y.astype(int)]
    th = np.atleast_2d(beta) * sigma
    return (c @ loss) / c.sum() + lam * ((1 - alpha) / 2 * np.sum(th ** 2) + alpha * np.sum(np.abs(th)))


def _sklearn(X, y, w, lam, alpha, sigma):
    from sklearn.linear_model import LogisticRegression as SK
    sw = X.shape[0] if w is None else w.sum()
    C = np.inf if lam == 0 else 1.0 / (lam * sw)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sk = SK(C=C, l1_ratio=alpha, solver="lbfgs" if alpha == 0 else "saga", tol=1e-12, max_iter=20000)
        sk.fit(X / sigma, y, sample_weight=w)
    b = sk.intercept_
    if not np.any(sk.coef_):  # saga stops on unchanged coefficients before its intercept settles: the closed form
        c = np.ones(y.size) if w is None else w
        h = np.array([c[y == k].sum() for k in range(int(y.max()) + 1)])
        b = np.log(h[1:2] / h[0]) if sk.coef_.shape[0] == 1 else np.log(h) - np.log(h).mean()
    return sk.coef_ / sigma, b


CASES = [(0.0, 0.0), (0.01, 0.0), (0.01, 0.5), (0.01, 1.0), (0.5, 0.0), (0.5, 0.5), (0.5, 1.0)]


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("name,lam,alpha", [("adult8k", lam, a) for lam, a in CASES] +
                         [("letter", lam, a) for lam, a in CASES if lam > 0])  # 2000 letter rows: nearly separable
def test_optimum_matches_sklearn(name, lam, alpha, weighted):
    rows = 2000 if name == "letter" else None  # 26 classes over numpy and saga: a smaller problem
    X, y = _data(name, rows)
    w = np.random.default_rng(7).uniform(0.5, 2.0, y.size) if weighted else None
    sigma = _sigma(X, w)
    model = _fit(DeviceLogisticRegression(regParam=lam, elasticNetParam=alpha, tol=1e-10, maxIter=5000), X, y, w)
    beta_sk, b_sk = _sklearn(X, y, w, lam, alpha, sigma)
    f = _objective(X, y, w, model.coefficientMatrix, model.interceptVector, lam, alpha, sigma)
    f_sk = _objective(X, y, w, beta_sk, b_sk, lam, alpha, sigma)
    assert f <= f_sk + 1e-7 * abs(f_sk), (f, f_sk)
    assert model.isMultinomial == (name == "letter")
    if alpha == 0.0:  # lbfgs converges to 1e-10; saga (elastic net) stops well before that, so only the bound above
        assert abs(f - f_sk) <= 1e-7 * abs(f_sk), (f, f_sk)
        # strictly convex (the multinomial up to its centring, which both sides share)
        beta, bsk = model.coefficientMatrix, beta_sk
        if model.isMultinomial:
            bsk = bsk - bsk.mean(axis=0)
        scale = np.abs(bsk).max()
        assert np.abs(beta - bsk).max() <= 1e-4 * scale, float(np.abs(beta - bsk).max() / scale)
    assert model.objectiveHistory[-1] == pytest.approx(f, rel=1e-9)
    assert model.numEvaluations >= len(model.objectiveHistory) - 1


def test_numpy_evaluation_matches_finite_differences():
    rng = np.random.default_rng(3)
    X = rng.standard_normal((200, 5))
    for D, y in ((1, (rng.random(200) < 0.4).astype(float)), (4, rng.integers(0, 4, 200).astype(float))):
        coef = rng.standard_normal((D, 6)) * 0.3
        w = rng.uniform(0.1, 2, 200)
        shift, scale = rng.standard_normal(5), rng.uniform(0.5, 2, 5)
        cols = np.array([3, 0, 0, 4, 1])
        f, g = O.loss_grad(X, y, cols, coef, w, shift, scale)
        h = 1e-6
        num = np.zeros_like(coef)
        for i in np.ndindex(coef.shape):
            e = np.zeros_like(coef)
            e[i] = h
            num[i] = (O.loss_grad(X, y, cols, coef + e, w, shift, scale)[0] -
                      O.loss_grad(X, y, cols, coef - e, w, shift, scale)[0]) / (2 * h)
        np.testing.assert_allclose(g, num, rtol=1e-6, atol=1e-6 * np.abs(g).max())


def test_multinomial_centring_and_constant_columns():
    X, y = _data("letter", 2000)
    X = np.concatenate([X, np.full((X.shape[0], 1), 3.0)], axis=1)  # σ = 0
    m0 = _fit(DeviceLogisticRegression(tol=1e-8), X, y)
    np.testing.assert_allclose(m0.coefficientMatrix.sum(axis=0), 0.0, atol=1e-10)  # λ = 0: centred coefficients
    assert abs(m0.interceptVector.sum()) <= 1e-10
    assert np.all(m0.coefficientMatrix[:, -1] == 0.0)
    m1 = _fit(DeviceLogisticRegression(regParam=0.1, tol=1e-8), X, y)
    assert abs(m1.interceptVector.sum()) <= 1e-10  # intercepts always centred
    assert np.all(m1.coefficientMatrix[:, -1] == 0.0)
    # a binomial fit with the σ = 0 column and without standardization keeps it at 0 as well
    Xa, ya = _data("adult8k", 2000)
    Xa = np.concatenate([Xa, np.zeros((Xa.shape[0], 1))], axis=1)
    m2 = _fit(DeviceLogisticRegression(regParam=0.01, standardization=False, tol=1e-8), Xa, ya)
    assert m2.coefficients[-1] == 0.0


def test_single_class_model():
    X, y = _data("adult8k", 500)
    m = _fit(DeviceLogisticRegression(), X, np.ones(500), K=2)
    assert np.all(m.coefficients == 0) and m.intercept == np.inf and m.numEvaluations == 0
    np.testing.assert_array_equal(m.predict(X), 1.0)
    np.testing.assert_array_equal(m.predictProbability(X)[:, 1], 1.0)
    m0 = _fit(DeviceLogisticRegression(), X, np.zeros(500), K=2)
    assert m0.intercept == -np.inf
    np.testing.assert_array_equal(m0.predict(X), 0.0)
    mm = _fit(DeviceLogisticRegression(family="multinomial"), X, np.full(500, 2.0), K=3)
    assert mm.interceptVector.tolist() == [0.0, 0.0, np.inf]
    np.testing.assert_array_equal(mm.predictProbability(X), np.tile([0.0, 0.0, 1.0], (500, 1)))
    np.testing.assert_array_equal(mm.predict(X), 2.0)


def test_no_intercept():
    X, y = _data("adult8k", 3000)
    m = _fit(DeviceLogisticRegression(regParam=0.01, fitIntercept=False, tol=1e-10, maxIter=2000), X, y)
    assert m.intercept == 0.0
    from sklearn.linear_model import LogisticRegression as SK
    sigma = _sigma(X, None)
    sk = SK(C=1.0 / (0.01 * y.size), fit_intercept=False, tol=1e-12, max_iter=20000).fit(X / sigma, y)
    f = _objective(X, y, None, m.coefficients, 0.0, 0.01, 0.0, sigma)
    f_sk = _objective(X, y, None, sk.coef_[0] / sigma, 0.0, 0.01, 0.0, sigma)
    assert abs(f - f_sk) <= 1e-7 * f_sk, (f, f_sk)


def test_params_and_validation():
    d = DeviceLogisticRegression()
    assert (d.regParam, d.elasticNetParam, d.maxIter, d.tol, d.fitIntercept, d.standardization, d.family,
            d.threshold, d.device) == (0.0, 0.0, 100, 1e-6, True, True, "auto", 0.5, 0)
    for kw in ({"regParam": -1}, {"elasticNetParam": 1.5}, {"family": "poisson"}, {"threshold": 2}, {"maxIter": -1}):
        with pytest.raises(ValueError):
            DeviceLogisticRegression(**kw)
    X, y = _data("letter", 300)
    with pytest.raises(ValueError, match="binomial family"):
        _fit(DeviceLogisticRegression(family="binomial"), X, y)
    bad = y.copy()
    bad[5] = 0.5
    with pytest.raises(ValueError, match="1 rows"):
        _fit(DeviceLogisticRegression(), X, bad, K=26)
    from spark_ensemble_b200 import routes
    assert routes.is_classifier(DeviceLogisticRegression()) and routes.takes_weights(DeviceLogisticRegression())
    assert not getattr(DeviceLogisticRegression(), "device_learner", False)


def test_model_host_scoring_threshold_and_infinite_margins():
    m = LogisticRegressionModel([[1.0, -2.0]], [0.5], 2, False, threshold=0.7)
    X = np.array([[0.0, 0.0], [1.0, 0.0], [0.0, 1.0]])
    raw = m.predictRaw(X)
    np.testing.assert_allclose(raw[:, 1], [0.5, 1.5, -1.5])
    np.testing.assert_allclose(raw[:, 0], -raw[:, 1])
    p1 = 1 / (1 + np.exp(-raw[:, 1]))
    np.testing.assert_allclose(m.predictProbability(X)[:, 1], p1)
    np.testing.assert_array_equal(m.predict(X), (p1 > 0.7).astype(float))
    mm = LogisticRegressionModel(np.zeros((3, 2)), [np.inf, 0.0, np.inf], 3, True)
    np.testing.assert_array_equal(mm.predictProbability(X[:1]), [[1.0, 0.0, 1.0]])
    np.testing.assert_array_equal(mm.predict(X[:1]), [0.0])
