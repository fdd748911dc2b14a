"""StackingRegressor and StackingClassifier: the device route (residentFeatures=True) against the host route on the same
estimator, over binary and multiclass stacks of every classifier ensemble member, weighted fits, members without a
device form or whose thresholds overflow the rank matrix (their rows are uploaded between device-written rows),
collinear meta-features, and ragged row counts.  For every case:

- the meta-features a recording stacker is fitted on agree between the routes to a few fp32 ulps (linear and
  logistic members at the scale of their terms), and the weights reach the same fits;
- the device stacker equals the same stacker fitted over the downloaded meta-features: identical bits for a
  logistic stacker and for tree arrays, the linear solve's tolerance for a linear one;
- transform on other rows (a ragged count) writes the meta-features the host route computes, and predicts what the
  stack predicts over them."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ULP = 2.0 ** -24


def _golden(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", f"{name}.npz"))
    return z["X"].astype(np.float32), z["y"].astype(np.float64)


def _split(X, y, seed=2019):
    """A train set and a held-out set of 20 % of the rows plus 3: a row count that is not a multiple of 32."""
    rng = np.random.default_rng(seed)
    test = rng.random(y.size) < 0.2
    test[np.flatnonzero(~test)[:3]] = True
    return X[~test], y[~test], X[test]


class _Recorder:
    """A host stacker that records the meta-features and the weights it is fitted on."""

    def __init__(self, log):
        self.log = log

    def copy(self, extra=None):
        return _Recorder(self.log)

    def fit(self, X, y, w=None, num_classes=None):
        self.log.append((np.array(X, dtype=np.float64), None if w is None else np.array(w, dtype=np.float64)))
        from spark_ensemble_b200.learners import LinearRegression
        return LinearRegression().fit(X[:, :1], y)


class _Capture:
    """A stack that records the meta-features it predicts over (the device route downloads them for a stack it cannot
    score on the device)."""

    def __init__(self):
        self.F = None

    def predict(self, F):
        self.F = np.array(F, dtype=np.float64)
        return np.zeros(F.shape[0])


class _NearestMean:
    """A classifier with no device form and no weights: the class whose mean feature vector is nearest."""

    def copy(self, extra=None):
        return _NearestMean()

    def fit(self, X, y, num_classes=None):
        K = int(num_classes)
        X = np.asarray(X, dtype=np.float64)
        mu = np.stack([X[y == k].mean(axis=0) if np.any(y == k) else np.zeros(X.shape[1]) for k in range(K)])
        return _NearestMeanModel(mu / X.std(axis=0).clip(1e-12), X.std(axis=0).clip(1e-12))


class _NearestMeanModel:
    def __init__(self, mu, sd):
        self.mu, self.sd = mu, sd

    def predictRaw(self, X):
        Z = np.asarray(X, dtype=np.float64) / self.sd
        return -((Z[:, None, :] - self.mu[None]) ** 2).sum(axis=2)

    def predictProbability(self, X):
        r = self.predictRaw(X)
        e = np.exp(r - r.max(axis=1, keepdims=True))
        return e / e.sum(axis=1, keepdims=True)

    def predict(self, X):
        return np.argmax(self.predictRaw(X), axis=1).astype(np.float64)


class _ColumnMeans:
    """A regressor with no device form and no weights: the label mean of each half of the first column."""

    def copy(self, extra=None):
        return _ColumnMeans()

    def fit(self, X, y):
        c = float(np.median(X[:, 0]))
        lo = X[:, 0] <= c
        return _ColumnMeansModel(c, float(y[lo].mean()), float(y[~lo].mean()))


class _ColumnMeansModel:
    def __init__(self, c, a, b):
        self.c, self.a, self.b = c, a, b

    def predict(self, X):
        return np.where(np.asarray(X)[:, 0] <= self.c, self.a, self.b)


def _meta(est, df, resident):
    log = []
    est.copy().setStacker(_Recorder(log)).setResidentFeatures(resident).fit(df)
    return log[0]


def _tolerance(models, widths, X, host, classifier):
    """Per entry of the meta-features: a few fp32 ulps of the value (and the fits' tolerance, 1e-5, for classifier
    outputs), and for a linear or logistic member's values the fp32 rounding of their terms: the device forms the dot
    product of fp32 features in fp64 and rounds it once to fp32, the host keeps it in fp64."""
    from spark_ensemble_b200.learners import LogisticRegressionModel
    tol = (8 * 2.0 ** -23 * np.abs(host) + 1e-5) if classifier else (4 * 2.0 ** -23 * np.abs(host) + 1e-6)
    X64 = np.abs(X.astype(np.float64))
    col = 0
    for m, k in zip(models, widths):
        lin = m.linear_arrays() if hasattr(m, "linear_arrays") else None
        if lin is not None:
            terms = X64 @ np.abs(np.asarray(lin["coef"], dtype=np.float64)) + abs(float(lin["intercept"]))
            tol[:, col] += 16 * ULP * terms + 4 * ULP * np.abs(host[:, col])
        elif isinstance(m, LogisticRegressionModel) and k > 1:
            terms = X64 @ np.abs(m.coefficientMatrix.T) + np.abs(m.interceptVector)
            if terms.shape[1] == 1:
                terms = np.tile(terms, (1, 2))
            tol[:, col:col + k] += 16 * ULP * terms + 4 * ULP * np.abs(host[:, col:col + k])
        col += k
    return tol


def _assert_meta(dev, host, tol):
    assert dev.shape == host.shape
    bad = np.abs(dev - host) > tol
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:5].tolist())


def _host_meta(model, X):
    from spark_ensemble_b200.routes import model_outputs
    method = model("stackMethod").lower() if model.hasParam("stackMethod") else "class"
    return np.concatenate([model_outputs(m, X, method, k) for m, k in zip(model.models, model.widths)]).T


def _device_meta(model, X):
    from spark_ensemble_b200.ensemble import DataFrame
    stack, cap = model.stack, _Capture()
    model.stack = cap
    try:
        model.transform(DataFrame(features=X))
    finally:
        model.stack = stack
    return cap.F


def _same_stacker(stack, ref):
    from spark_ensemble_b200.learners import LogisticRegressionModel
    if isinstance(stack, LogisticRegressionModel):
        assert stack.coefficientMatrix.tobytes() == ref.coefficientMatrix.tobytes()
        assert stack.interceptVector.tobytes() == ref.interceptVector.tobytes()
    else:
        for k in ("feature", "threshold", "left", "right", "value"):
            np.testing.assert_array_equal(stack.tree_arrays()[k], ref.tree_arrays()[k])


def _check_classifier(est, X, y, w, Xt, stackers, K):
    from spark_ensemble_b200.ensemble import DataFrame
    from spark_ensemble_b200.learners import LogisticRegressionModel
    cols = {"features": X, "label": y}
    if w is not None:
        cols["w"] = w
        est = est.copy().setWeightCol("w")
    df = DataFrame(**cols)
    (host, hw), (dev, dw) = _meta(est, df, False), _meta(est, df, True)
    sw = np.ones(y.size) if w is None else w
    np.testing.assert_array_equal(hw, sw)
    np.testing.assert_array_equal(dw, sw)
    for stacker in stackers:
        model = est.copy().setStacker(stacker).setResidentFeatures(True).fit(df)
        _assert_meta(dev, host, _tolerance(model.models, model.widths, X, host, True))
        ref = stacker.fit(dev, y, sw, num_classes=K)  # the same stacker over the downloaded meta-features
        _same_stacker(model.stack, ref)
        # other rows: the meta-features the device route writes against the host route's, and the stack's labels
        mt_dev, mt_host = _device_meta(model, Xt), _host_meta(model, Xt)
        _assert_meta(mt_dev, mt_host, _tolerance(model.models, model.widths, Xt, mt_host, True))
        out = model.transform(DataFrame(features=Xt))["prediction"]
        expect = ref.predict(mt_dev)
        tie = np.zeros(Xt.shape[0], bool)
        if isinstance(ref, LogisticRegressionModel):
            # the same model scored in fp64 on the device and on the host: equal labels but for rows whose deciding
            # margins tie to rounding (the two sums run in different orders)
            M = ref._margins(mt_dev)
            if ref.coefficientMatrix.shape[0] == 1:
                p1 = 1.0 / (1.0 + np.exp(-M[:, 0]))
                tie = np.abs(p1 - ref.threshold) <= 1e-9
            else:
                M = np.sort(M, axis=1)
                tie = (M[:, -1] - M[:, -2]) <= 1e-9 * (1.0 + np.abs(M[:, -1]))
        np.testing.assert_array_equal(out[~tie], expect[~tie])
        assert tie.sum() <= 2, int(tie.sum())
    return dev


def _binary_members(boost_algorithm):
    from spark_ensemble_b200.classification import BaggingClassifier, BoostingClassifier, GBMClassifier
    from spark_ensemble_b200.learners import (DeviceDecisionTreeClassifier, DeviceDecisionTreeRegressor,
                                              DeviceLogisticRegression)
    gbm = GBMClassifier().setLoss("bernoulli").setBaseLearner(DeviceDecisionTreeRegressor(maxDepth=3)) \
        .setNumBaseLearners(4).setResidentFeatures(True)
    boost = BoostingClassifier().setAlgorithm(boost_algorithm).setBaseLearner(DeviceDecisionTreeClassifier(maxDepth=3)) \
        .setNumBaseLearners(4).setResidentFeatures(True)
    bag = BaggingClassifier().setBaseLearner(DeviceDecisionTreeClassifier(maxDepth=4)).setNumBaseLearners(3) \
        .setVotingStrategy("hard").setResidentFeatures(True)
    return [DeviceDecisionTreeClassifier(maxDepth=5), DeviceLogisticRegression(regParam=0.01), gbm, boost, bag]


@pytest.mark.parametrize("method,algorithm", [("class", "discrete"), ("raw", "real"), ("proba", "discrete"),
                                              ("proba", "real")])
def test_binary_stack_of_every_member_kind(method, algorithm):
    """adult8k, two classes: a binomial logistic member (raw (-m, m), proba (1 - p, p)), a dim-1 GBMClassifier
    (two output classes), SAMME or SAMME.R boosting and hard-vote bagging, under a binomial logistic stacker, one
    with threshold 0.3 and a tree stacker."""
    from spark_ensemble_b200.classification import StackingClassifier
    from spark_ensemble_b200.learners import DeviceDecisionTreeClassifier, DeviceLogisticRegression
    X, y = _golden("adult8k")
    X, y, Xt = _split(X, y)
    est = StackingClassifier().setBaseLearners(_binary_members(algorithm)).setStackMethod(method)
    stackers = [DeviceLogisticRegression(regParam=0.01), DeviceLogisticRegression(regParam=0.01, threshold=0.3),
                DeviceDecisionTreeClassifier(maxDepth=4)]
    dev = _check_classifier(est, X, y, None, Xt, stackers, 2)
    assert dev.shape[1] == (5 if method == "class" else 10)


def test_multiclass_stack_of_ensemble_members_on_ragged_letter():
    """4099 rows of letter (26 classes): a LogLoss GBMClassifier (26 trees a round), SAMME.R boosting, hard-vote bagging
    and a member with no device form between device members, proba meta-features, a logistic stacker."""
    from spark_ensemble_b200.classification import (BaggingClassifier, BoostingClassifier, GBMClassifier,
                                                    StackingClassifier)
    from spark_ensemble_b200.learners import (DeviceDecisionTreeClassifier, DeviceDecisionTreeRegressor,
                                              DeviceLogisticRegression)
    X, y = _golden("letter")
    X, y = X[:4099], y[:4099]
    Xt = _golden("letter")[0][4099:4099 + 1027]
    gbm = GBMClassifier().setLoss("logloss").setBaseLearner(DeviceDecisionTreeRegressor(maxDepth=3)) \
        .setNumBaseLearners(2).setResidentFeatures(True)
    boost = BoostingClassifier().setAlgorithm("real").setBaseLearner(DeviceDecisionTreeClassifier(maxDepth=5)) \
        .setNumBaseLearners(3).setResidentFeatures(True)
    bag = BaggingClassifier().setBaseLearner(DeviceDecisionTreeClassifier(maxDepth=5)).setNumBaseLearners(3) \
        .setVotingStrategy("hard").setResidentFeatures(True)
    for method in ("proba", "class"):
        members = [gbm, _NearestMean(), boost, bag, DeviceDecisionTreeClassifier(maxDepth=6)]
        est = StackingClassifier().setBaseLearners(members).setStackMethod(method)
        stackers = [DeviceLogisticRegression(regParam=0.01)] if method == "proba" else \
            [DeviceDecisionTreeClassifier(maxDepth=6)]
        dev = _check_classifier(est, X, y, None, Xt, stackers, 26)
        assert dev.shape == (4099, 5 * 26 if method == "proba" else 5)


@pytest.mark.parametrize("with_unweighted_member", [False, True])
def test_weighted_classifier_stack(with_unweighted_member):
    """weightCol with zero-weight rows: every member takes the weights, or (with a member that takes none) the members
    are fitted unweighted and only the stacker is weighted."""
    from spark_ensemble_b200.classification import BaggingClassifier, StackingClassifier
    from spark_ensemble_b200.learners import DeviceDecisionTreeClassifier, DeviceLogisticRegression
    X, y = _golden("adult8k")
    X, y, Xt = _split(X, y, seed=7)
    rng = np.random.default_rng(11)
    w = rng.uniform(0.2, 3.0, y.size)
    w[rng.random(y.size) < 0.1] = 0.0
    bag = BaggingClassifier().setBaseLearner(DeviceDecisionTreeClassifier(maxDepth=4)).setNumBaseLearners(3) \
        .setVotingStrategy("hard").setResidentFeatures(True)
    members = [DeviceDecisionTreeClassifier(maxDepth=5), DeviceLogisticRegression(regParam=0.01), bag]
    if with_unweighted_member:
        members.insert(1, _NearestMean())
    est = StackingClassifier().setBaseLearners(members).setStackMethod("raw")
    stackers = [DeviceLogisticRegression(regParam=0.01), DeviceDecisionTreeClassifier(maxDepth=4)]
    dev = _check_classifier(est, X, y, w, Xt, stackers, 2)
    # the weights reached the members exactly when every member takes them: the device tree member's raw rows are
    # its leaves' weighted class totals
    tree = DeviceDecisionTreeClassifier(maxDepth=5).fit(X, y, None if with_unweighted_member else w, num_classes=2)
    np.testing.assert_allclose(dev[:, :2], tree.predictRaw(X), rtol=4 * 2.0 ** -23, atol=1e-6)


# ---- regression -------------------------------------------------------------------------------------------------------
def _check_regressor(est, X, y, w, Xt, stackers):
    from spark_ensemble_b200.ensemble import DataFrame
    from spark_ensemble_b200.learners import DeviceLinearRegression
    cols = {"features": X, "label": y}
    if w is not None:
        cols["w"] = w
        est = est.copy().setWeightCol("w")
    df = DataFrame(**cols)
    (host, hw), (dev, dw) = _meta(est, df, False), _meta(est, df, True)
    sw = np.ones(y.size) if w is None else w
    np.testing.assert_array_equal(hw, sw)
    np.testing.assert_array_equal(dw, sw)
    scale = np.abs(y).max()
    for stacker in stackers:
        model = est.copy().setStacker(stacker).setResidentFeatures(True).fit(df)
        _assert_meta(dev, host, _tolerance(model.models, model.widths, X, host, False))
        ref = stacker.fit(dev, y, sw)  # the same stacker over the downloaded meta-features
        if isinstance(stacker, DeviceLinearRegression):
            np.testing.assert_allclose(model.stack.predict(dev), ref.predict(dev), rtol=1e-6, atol=1e-6 * scale)
        else:
            _same_stacker(model.stack, ref)
        mt_dev, mt_host = _device_meta(model, Xt), _host_meta(model, Xt)
        _assert_meta(mt_dev, mt_host, _tolerance(model.models, model.widths, Xt, mt_host, False))
        out = model.transform(DataFrame(features=Xt))["prediction"]
        np.testing.assert_allclose(out, ref.predict(mt_dev), rtol=1e-5, atol=1e-5 * scale)
    return dev


def test_regression_stack_uploads_rows_between_device_members():
    """A member with no device form and a host tree with more than 255 thresholds in a column (SE_ERR_STATE) are
    scored on the host and uploaded into their rows of the padded [W][n] slot, each between two device-written rows."""
    from spark_ensemble_b200.learners import DecisionTreeRegressor, DeviceDecisionTreeRegressor, DeviceLinearRegression
    from spark_ensemble_b200.regression import StackingRegressor
    rng = np.random.default_rng(12)
    n = 20_003
    X = rng.standard_normal((n, 3)).astype(np.float32)
    y = np.sin(3 * X[:, 0]) + 0.5 * X[:, 1] + 0.1 * rng.standard_normal(n)
    X, y, Xt = _split(X, y)
    members = [DeviceDecisionTreeRegressor(maxDepth=4), DecisionTreeRegressor(maxDepth=12), DeviceLinearRegression(),
               _ColumnMeans(), DeviceDecisionTreeRegressor(maxDepth=6)]
    est = StackingRegressor().setBaseLearners(members)
    dev = _check_regressor(est, X, y, None, Xt, [DeviceLinearRegression(), DeviceDecisionTreeRegressor(maxDepth=4)])
    deep = DecisionTreeRegressor(maxDepth=12).fit(X, y).tree_arrays()
    assert max(np.unique(deep["threshold"][deep["feature"] == c]).size for c in range(3)) > 255
    np.testing.assert_array_equal(dev[:, 1], DecisionTreeRegressor(maxDepth=12).fit(X, y).predict(X)
                                  .astype(np.float32))
    assert np.unique(dev[:, 3]).size == 2


@pytest.mark.parametrize("with_unweighted_member", [False, True])
def test_weighted_regression_stack(with_unweighted_member):
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor, DeviceLinearRegression
    from spark_ensemble_b200.regression import BoostingRegressor, StackingRegressor
    X, y = _golden("cpusmall")
    X, y, Xt = _split(X, y, seed=3)
    rng = np.random.default_rng(13)
    w = rng.uniform(0.2, 3.0, y.size)
    w[rng.random(y.size) < 0.1] = 0.0
    boost = BoostingRegressor().setBaseLearner(DeviceDecisionTreeRegressor(maxDepth=3)).setNumBaseLearners(4) \
        .setResidentFeatures(True)
    members = [DeviceDecisionTreeRegressor(maxDepth=5), DeviceLinearRegression(), boost]
    if with_unweighted_member:
        members.insert(2, _ColumnMeans())
    est = StackingRegressor().setBaseLearners(members)
    dev = _check_regressor(est, X, y, w, Xt, [DeviceLinearRegression(), DeviceDecisionTreeRegressor(maxDepth=4)])
    tree = DeviceDecisionTreeRegressor(maxDepth=5).fit(X, y, None if with_unweighted_member else w)
    np.testing.assert_allclose(dev[:, 0], tree.predict(X), rtol=4 * 2.0 ** -23, atol=1e-6)


def test_regression_stack_of_two_identical_members():
    """Two identical members give collinear meta-features: the linear stacker's normal equations are singular and
    solve_linear_moments falls back to least squares, on both routes."""
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor, DeviceLinearRegression, LinearRegression
    from spark_ensemble_b200.regression import StackingRegressor
    X, y = _golden("cpusmall")
    X, y, Xt = _split(X, y, seed=5)
    members = [DeviceDecisionTreeRegressor(maxDepth=5), DeviceDecisionTreeRegressor(maxDepth=5), LinearRegression()]
    est = StackingRegressor().setBaseLearners(members)
    dev = _check_regressor(est, X, y, None, Xt, [DeviceLinearRegression()])
    np.testing.assert_array_equal(dev[:, 0], dev[:, 1])
