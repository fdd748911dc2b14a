"""StackingRegressor / StackingClassifier on the host route, and the solve of DeviceLinearRegression from numpy moments:
everything here runs without a GPU."""
import numpy as np
import pytest

from oracle import np_linear
from spark_ensemble_b200.classification import StackingClassificationModel, StackingClassifier
from spark_ensemble_b200.ensemble import DataFrame
from spark_ensemble_b200.learners import (DecisionTreeClassifier, DecisionTreeRegressor, DeviceDecisionTreeClassifier,
                                          DeviceLinearRegression, LinearRegression, solve_linear_moments)
from spark_ensemble_b200.regression import StackingRegressionModel, StackingRegressor


class _Recorder:
    """A learner that records what it is fitted on; its model predicts the first meta-feature plus a constant."""

    def __init__(self, log, takes_w=True):
        self.log, self.takes_w = log, takes_w

    def copy(self, extra=None):
        return _Recorder(self.log, self.takes_w)

    def fit(self, X, y, w=None):
        self.log.append({"X": np.array(X, dtype=np.float64), "y": np.array(y), "w": None if w is None else np.array(w)})
        return _FirstColumn()


class _FirstColumn:
    def predict(self, X):
        return np.asarray(X, dtype=np.float64)[:, 0] + 0.5


class _NoWeights:
    """A learner whose fit takes no weights (not HasWeightCol)."""

    def copy(self, extra=None):
        return _NoWeights()

    def fit(self, X, y):
        return LinearRegression().fit(X, y)


def _regression_data(n=400, d=5, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)).astype(np.float32)
    y = X @ rng.normal(size=d) + 0.3 * np.sin(3 * X[:, 0]) + 0.1 * rng.normal(size=n)
    w = rng.uniform(0.5, 2.0, size=n)
    return X, y, w


def _classification_data(n=500, d=4, K=3, seed=1):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)).astype(np.float32)
    y = (np.digitize(X[:, 0] + 0.5 * X[:, 1], [-0.5, 0.5]) % K).astype(np.float64)
    return X, y


def test_params_defaults_uids_and_copy():
    r, c = StackingRegressor(), StackingClassifier()
    assert r.uid.startswith("StackingRegressor_") and c.uid.startswith("StackingClassifier_")
    for est in (r, c):
        assert est.getParallelism() == 1 and est.getResidentFeatures() is False
        assert est.getLabelCol() == "label" and est.getFeaturesCol() == "features"
        assert est.getPredictionCol() == "prediction" and not est.isDefined("weightCol")
        with pytest.raises(ValueError):
            est.setParallelism(0)
    assert c.getStackMethod() == "class"
    for m in ("class", "RAW", "Proba"):
        c.setStackMethod(m)
    with pytest.raises(ValueError):
        c.setStackMethod("votes")
    members = [DecisionTreeRegressor(maxDepth=3), LinearRegression(0.5)]
    r.setBaseLearners(members).setStacker(LinearRegression())
    r2 = r.copy()
    assert r2.uid == r.uid
    assert [type(m) for m in r2.getBaseLearners()] == [type(m) for m in members]
    assert all(a is not b for a, b in zip(r2.getBaseLearners(), members))
    assert r2.getBaseLearners()[0].maxDepth == 3 and r2.getBaseLearners()[1].regParam == 0.5
    assert r2.getStacker() is not r.getStacker()
    assert StackingRegressionModel([], None).uid.startswith("StackingRegressionModel_")
    assert StackingClassificationModel([], None, 2, []).uid.startswith("StackingClassificationModel_")


@pytest.mark.parametrize("method", ["class", "raw", "proba"])
def test_classifier_meta_features_are_the_reference_flatmap(method):
    X, y = _classification_data()
    K = 3
    log = []
    members = [DecisionTreeClassifier(maxDepth=2), LinearRegression(), DecisionTreeClassifier(maxDepth=4, seed=3)]
    est = StackingClassifier().setBaseLearners(members).setStacker(_Recorder(log)).setStackMethod(method.upper())
    model = est.fit(DataFrame(features=X, label=y))
    m0, m1, m2 = model.models

    def outputs(m, x):  # models.flatMap for one row
        if isinstance(m, type(m1)):
            return [float(m.predict(x[None])[0])]
        if method == "proba":
            return list(m.predictProbability(x[None])[0])
        if method == "raw":
            return list(m.predictRaw(x[None])[0])
        return [float(m.predict(x[None])[0])]

    expect = np.array([outputs(m0, x) + outputs(m1, x) + outputs(m2, x) for x in X])
    assert model.widths == ([1, 1, 1] if method == "class" else [K, 1, K])
    np.testing.assert_allclose(log[0]["X"], expect, rtol=1e-13, atol=1e-13)  # one row vs all rows: BLAS order
    if method == "raw":  # the leaf's weighted class counts, which sum to the rows the leaf holds
        assert np.all(log[0]["X"][:, :K].sum(axis=1) >= 1)
    out = model.transform(DataFrame(features=X, label=y))
    assert out.columns == ["features", "label", "prediction"]
    np.testing.assert_array_equal(out["prediction"], log[0]["X"][:, 0] + 0.5)


def test_raw_of_device_tree_model_is_its_class_weights():
    arrays = {"feature": np.array([0, -1, -1], np.int32), "threshold": np.array([0.0, 0, 0], np.float32),
              "left": np.array([1, 0, 0], np.int32), "right": np.array([2, 0, 0], np.int32),
              "value": np.array([0, 0, 1], np.float32),
              "values": np.array([[.5, .5], [.75, .25], [0, 1]], np.float32),
              "class_weights": np.array([[4, 4], [3, 1], [0, 3.5]]), "gain": np.zeros(3)}
    from spark_ensemble_b200.learners import DeviceDecisionTreeClassificationModel
    m = DeviceDecisionTreeClassificationModel(arrays, 2)
    np.testing.assert_array_equal(m.predictRaw(np.array([[-1.0], [2.0]])), [[3, 1], [0, 3.5]])


def test_regressor_host_route_predict_is_stack_of_member_outputs():
    X, y, w = _regression_data()
    members = [DecisionTreeRegressor(maxDepth=3), LinearRegression(), DecisionTreeRegressor(maxDepth=5, seed=1)]
    est = StackingRegressor().setBaseLearners(members).setStacker(LinearRegression()).setWeightCol("w")
    model = est.fit(DataFrame(features=X, label=y, w=w))
    meta = np.column_stack([m.predict(X) for m in model.models])
    np.testing.assert_array_equal(model.transform(DataFrame(features=X))["prediction"], model.stack.predict(meta))
    assert model.predict(X[7]) == model.stack.predict(meta[7:8])[0]
    assert model.parent is est and model.getWeightCol() == "w"


def test_weights_reach_members_only_when_every_member_takes_them():
    X, y, w = _regression_data(n=120)
    df = DataFrame(features=X, label=y, w=w)
    for extra, member_w in (([], w), ([_NoWeights()], None)):
        log, stack_log = [], []
        est = (StackingRegressor().setBaseLearners([_Recorder(log)] + extra).setStacker(_Recorder(stack_log))
               .setWeightCol("w"))
        est.fit(df)
        if member_w is None:
            assert log[0]["w"] is None
        else:
            np.testing.assert_array_equal(log[0]["w"], member_w)
        np.testing.assert_array_equal(stack_log[0]["w"], w)  # the stacker always gets the weights
    log, stack_log = [], []
    StackingRegressor().setBaseLearners([_Recorder(log)]).setStacker(_Recorder(stack_log)).fit(
        DataFrame(features=X, label=y))
    assert log[0]["w"] is None
    np.testing.assert_array_equal(stack_log[0]["w"], np.ones(X.shape[0]))  # ... or ones


def _device_solve(X, y, w=None, bag=None, reg=0.0, shift_row=0):
    """What DeviceLinearRegression.fit_resident computes, with the numpy moments standing in for the device's."""
    cols = np.arange(X.shape[1])
    shift = np.asarray(X, dtype=np.float32)[shift_row].astype(np.float64)
    ys = float(np.float32(y[shift_row]))
    M = np_linear.linear_moments(X, y, cols, w, bag, shift, ys)
    return solve_linear_moments(M, shift, ys, reg)


def test_solve_matches_host_linear_regression_well_conditioned():
    X, y, w = _regression_data(n=2000, d=6, seed=4)
    X = (X * np.float32(3) + np.float32(100)).astype(np.float32)  # offset columns: the shift keeps the centring exact
    y32 = y.astype(np.float32).astype(np.float64)
    for weights, reg in ((None, 0.0), (w.astype(np.float32).astype(np.float64), 0.0), (None, 2.5)):
        coef, b = _device_solve(X, y32, weights, reg=reg)
        host = LinearRegression(reg).fit(X.astype(np.float64), y32, weights)
        np.testing.assert_allclose(coef, host.coefficients, rtol=1e-9)
        np.testing.assert_allclose(b, host.intercept, rtol=1e-9)


def _pred_check(X, y, w=None, bag=None, Xh=None, yh=None, wh=None):
    coef, b = _device_solve(X, y, w, bag)
    host = LinearRegression().fit(X if Xh is None else Xh, y if yh is None else yh, w if wh is None else wh)
    Xd = np.asarray(X, dtype=np.float64)
    np.testing.assert_allclose(Xd @ coef + b, host.predict(Xd), rtol=1e-9, atol=1e-9 * np.abs(y).max())


def test_solve_predictions_match_on_degenerate_designs():
    rng = np.random.default_rng(7)
    n = 600
    a = rng.normal(size=n).astype(np.float32)
    c = rng.normal(size=n).astype(np.float32)
    y = (2 * a.astype(np.float64) - c + 0.05 * rng.normal(size=n)).astype(np.float32).astype(np.float64)
    # four identical columns (collinear stacking members)
    _pred_check(np.column_stack([a, a, a, a, c]), y)
    # a constant column
    _pred_check(np.column_stack([a, np.full(n, 3.25, np.float32), c]), y)
    # zero-weight rows
    w = rng.uniform(0.5, 2, size=n).astype(np.float32).astype(np.float64)
    w[::5] = 0.0
    _pred_check(np.column_stack([a, c]), y, w=w)
    # bag counts equal repeated rows
    counts = rng.poisson(1.0, size=n).astype(np.float64)
    X = np.column_stack([a, c])
    rep = np.repeat(np.arange(n), counts.astype(int))
    _pred_check(X, y, bag=counts, Xh=X[rep].astype(np.float64), yh=y[rep])


def test_device_linear_regression_is_not_a_resident_learner():
    lr = DeviceLinearRegression(regParam=0.1)
    assert not getattr(lr, "device_learner", False)
    assert lr.copy().regParam == 0.1
    with pytest.raises(ValueError):
        DeviceLinearRegression(regParam=-1.0)
    assert getattr(DeviceDecisionTreeClassifier(), "device_learner", False)
