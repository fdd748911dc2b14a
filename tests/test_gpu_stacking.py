"""StackingRegressor and StackingClassifier on the device route against the host route: the meta-features the members
write on the device, the device stackers against the same stacker fitted over the downloaded meta-features, the
reference suite's RMSE properties, and one upload of X per fit and per transform."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Recorder:
    """A host stacker that records the meta-features it is fitted on."""

    def __init__(self, log):
        self.log = log

    def copy(self, extra=None):
        return _Recorder(self.log)

    def fit(self, X, y, w=None, num_classes=None):
        self.log.append(np.array(X, dtype=np.float64))
        from spark_ensemble_b200.learners import LinearRegression
        return LinearRegression().fit(X[:, :1], y)


def _cpusmall():
    z = np.load(os.path.join(ROOT, "tests", "golden", "cpusmall.npz"))
    return z["X"].astype(np.float32), z["y"].astype(np.float64)


def _regression_members():
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor, LinearRegression
    from spark_ensemble_b200.regression import BoostingRegressor, GBMRegressor
    gbm = GBMRegressor().setBaseLearner(DeviceDecisionTreeRegressor(maxDepth=3)).setNumBaseLearners(8) \
        .setResidentFeatures(True)
    boost = BoostingRegressor().setBaseLearner(DeviceDecisionTreeRegressor(maxDepth=4)).setNumBaseLearners(8) \
        .setResidentFeatures(True)
    return [DeviceDecisionTreeRegressor(maxDepth=6), boost, gbm, LinearRegression()]


def _meta(est, df, resident):
    log = []
    est.copy().setStacker(_Recorder(log)).setResidentFeatures(resident).fit(df)
    return log[0]


def test_stacking_regressor_device_route_on_cpusmall():
    from spark_ensemble_b200.ensemble import DataFrame
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor, DeviceLinearRegression
    from spark_ensemble_b200.regression import StackingRegressor
    X, y = _cpusmall()
    df = DataFrame(features=X, label=y)
    est = StackingRegressor().setBaseLearners(_regression_members())
    host, dev = _meta(est, df, False), _meta(est, df, True)
    assert dev.shape == (X.shape[0], 4)
    np.testing.assert_allclose(dev[:, :3], host[:, :3], rtol=4 * 2.0 ** -23, atol=1e-6)  # a few fp32 ulps
    # the linear member's fp32 dot product on the device, at the scale of its terms
    from spark_ensemble_b200.learners import LinearRegression
    lin = LinearRegression().fit(X, y)
    terms = np.abs(X.astype(np.float64)) @ np.abs(lin.coefficients) + abs(lin.intercept)
    assert np.all(np.abs(dev[:, 3] - host[:, 3]) <= 16 * 2.0 ** -24 * terms + 4 * 2.0 ** -24 * np.abs(host[:, 3]))
    for stacker in (DeviceLinearRegression(), DeviceDecisionTreeRegressor(maxDepth=4)):
        model = est.copy().setStacker(stacker).setResidentFeatures(True).fit(df)
        ref = stacker.fit(dev, y, np.ones(y.size))  # the same stacker over the downloaded meta-features
        if isinstance(stacker, DeviceLinearRegression):
            np.testing.assert_allclose(model.stack.predict(dev), ref.predict(dev), rtol=1e-6, atol=1e-6 * np.abs(y).max())
        else:
            for k in ("feature", "threshold", "left", "right", "value"):
                np.testing.assert_array_equal(model.stack.tree_arrays()[k], ref.tree_arrays()[k])
        out = model.transform(DataFrame(features=X))["prediction"]
        np.testing.assert_allclose(out, ref.predict(dev), rtol=1e-5, atol=1e-5 * np.abs(y).max())


def test_stacking_regressor_beats_its_members_on_a_split():
    from spark_ensemble_b200.ensemble import DataFrame
    from spark_ensemble_b200.learners import DeviceLinearRegression, LinearRegression
    from spark_ensemble_b200.regression import StackingRegressor
    X, y = _cpusmall()
    rng = np.random.default_rng(2019)
    train = rng.random(y.size) < 0.8
    Xtr, ytr, Xte, yte = X[train], y[train], X[~train], y[~train]
    model = StackingRegressor().setBaseLearners(_regression_members()).setStacker(DeviceLinearRegression()) \
        .setResidentFeatures(True).fit(DataFrame(features=Xtr, label=ytr))
    rmse = lambda p: float(np.sqrt(np.mean((p - yte) ** 2)))
    stack = rmse(model.transform(DataFrame(features=Xte))["prediction"])
    members = [rmse(model_outputs_1d(m, Xte)) for m in model.models]
    linear = rmse(LinearRegression().fit(Xtr, ytr).predict(Xte))
    assert stack < min(members), (stack, members)
    assert stack < linear, (stack, linear)


def model_outputs_1d(m, X):
    from spark_ensemble_b200.routes import model_outputs
    return model_outputs(m, X, "class", 1)[0]


@pytest.mark.parametrize("method", ["class", "raw", "proba"])
def test_stacking_classifier_device_route_on_letter(method):
    from spark_ensemble_b200.classification import BaggingClassifier, StackingClassifier
    from spark_ensemble_b200.ensemble import DataFrame
    from spark_ensemble_b200.learners import DecisionTreeClassifier, DeviceDecisionTreeClassifier
    z = np.load(os.path.join(ROOT, "tests", "golden", "letter.npz"))
    X, y = z["X"].astype(np.float32), z["y"].astype(np.float64)
    df = DataFrame(features=X, label=y)
    bag = BaggingClassifier().setBaseLearner(DeviceDecisionTreeClassifier(maxDepth=5)).setNumBaseLearners(4) \
        .setVotingStrategy("soft").setResidentFeatures(True)
    members = [DeviceDecisionTreeClassifier(maxDepth=6), bag, DecisionTreeClassifier(maxDepth=5)]
    est = StackingClassifier().setBaseLearners(members).setStackMethod(method)
    host, dev = _meta(est, df, False), _meta(est, df, True)
    K = int(y.max()) + 1
    assert dev.shape == (X.shape[0], 3 if method == "class" else 3 * K)
    np.testing.assert_allclose(dev, host, rtol=4 * 2.0 ** -23, atol=1e-6)
    stacker = DeviceDecisionTreeClassifier(maxDepth=5)
    model = est.copy().setStacker(stacker).setResidentFeatures(True).fit(df)
    ref = stacker.fit(dev, y, np.ones(y.size), num_classes=K)
    for k in ("feature", "threshold", "left", "right", "value"):
        np.testing.assert_array_equal(model.stack.tree_arrays()[k], ref.tree_arrays()[k])
    out = model.transform(DataFrame(features=X))
    assert out.columns == ["features", "prediction"]
    np.testing.assert_array_equal(out["prediction"], ref.predict(dev))
    assert np.mean(out["prediction"] == y) > 3.0 / K  # well above chance


def test_device_route_uploads_x_once_per_fit_and_transform(monkeypatch):
    from spark_ensemble_b200.context import Context
    from spark_ensemble_b200.ensemble import DataFrame
    from spark_ensemble_b200.learners import (DecisionTreeRegressor, DeviceDecisionTreeRegressor, DeviceLinearRegression,
                                              LinearRegression)
    from spark_ensemble_b200.regression import StackingRegressor
    X, y = _cpusmall()
    calls = []
    orig = Context.upload_rowmajor

    def spy(self, slot, features, row_offset=0):
        calls.append(np.asarray(features).shape)
        return orig(self, slot, features, row_offset)
    monkeypatch.setattr(Context, "upload_rowmajor", spy)
    members = [DeviceDecisionTreeRegressor(maxDepth=5), DeviceLinearRegression(), DecisionTreeRegressor(maxDepth=4),
               LinearRegression()]
    est = StackingRegressor().setBaseLearners(members).setStacker(DeviceLinearRegression()).setResidentFeatures(True)
    model = est.fit(DataFrame(features=X, label=y))
    assert calls == [X.shape]
    calls.clear()
    model.transform(DataFrame(features=X))
    assert calls == [X.shape]
