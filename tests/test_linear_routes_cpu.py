"""CPU checks of how linear and logistic members are packed for se_linear_agg and when a model takes that route."""
import numpy as np


def test_margin_arrays_are_the_fp64_member_form():
    from spark_ensemble_b200.learners import LinearRegressionModel, LogisticRegressionModel
    lin = LinearRegressionModel([1.5, -2.0, 0.25], 0.75).margin_arrays()
    assert lin["coef"].shape == (1, 3) and lin["coef"].dtype == np.float64
    np.testing.assert_array_equal(lin["intercept"], [0.75])
    bino = LogisticRegressionModel([[0.1, 0.2]], [0.3], 2, False, threshold=0.3).margin_arrays()
    assert bino["coef"].shape == (1, 2) and bino["threshold"] == 0.3
    multi = LogisticRegressionModel(np.ones((4, 5)), np.zeros(4), 4, True).margin_arrays()
    assert multi["coef"].shape == (4, 5) and multi["intercept"].shape == (4,)


def test_route_selection():
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressionModel, LinearRegressionModel
    from spark_ensemble_b200.regression import BaggingRegressionModel
    from spark_ensemble_b200.routes import device_linear, linear_kw, linear_list
    lin = [LinearRegressionModel(np.ones(3), 0.0), LinearRegressionModel(np.ones(254), 1.0)]
    tree = DeviceDecisionTreeRegressionModel({"feature": np.array([-1], np.int32), "threshold": np.zeros(1, np.float32),
                                              "left": np.zeros(1, np.int32), "right": np.zeros(1, np.int32),
                                              "value": np.zeros(1, np.float32)})
    assert [a["coef"].shape for a in linear_list(lin)] == [(1, 3), (1, 254)]
    assert linear_list(lin + [tree]) is None                                     # mixed members
    assert linear_list([LinearRegressionModel(np.ones(255), 0.0)]) is None        # wider than the kernel takes
    assert linear_list([object()]) is None
    m = BaggingRegressionModel([np.arange(3), np.arange(254)], lin)
    assert device_linear(m, m.models) is None                                    # residentFeatures off
    m.set("residentFeatures", True)
    assert len(device_linear(m, m.models)) == 2
    assert device_linear(m, []) is None
    assert linear_kw({"tree_class": [0], "weights": None}) == {"member_class": [0], "weights": None}
