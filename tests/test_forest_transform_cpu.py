"""residentFeatures on every ensemble: declared with default False, copied from the estimator to its model, and the
classifier forest entry point bound wherever the other entry points are."""
import numpy as np
import pytest

from spark_ensemble_b200 import DataFrame


def _estimators():
    from spark_ensemble_b200.classification import BaggingClassifier, BoostingClassifier, GBMClassifier
    from spark_ensemble_b200.regression import BaggingRegressor, BoostingRegressor, GBMRegressor
    return [GBMRegressor, GBMClassifier, BoostingClassifier, BaggingRegressor, BaggingClassifier, BoostingRegressor]


def _models():
    from spark_ensemble_b200.classification import (BaggingClassificationModel, BoostingClassificationModel,
                                                    GBMClassificationModel)
    from spark_ensemble_b200.regression import BaggingRegressionModel, BoostingRegressionModel, GBMRegressionModel
    return [GBMRegressionModel, GBMClassificationModel, BoostingClassificationModel, BaggingRegressionModel,
            BaggingClassificationModel, BoostingRegressionModel]


@pytest.mark.parametrize("cls", _estimators() + _models(), ids=lambda c: c.__name__)
def test_resident_features_declared_default_false(cls):
    assert cls._params["residentFeatures"].doc == "evaluate base models on device over the HBM-resident feature matrix"
    assert cls._defaults["residentFeatures"] is False


@pytest.mark.parametrize("kind", ["bagging_regressor", "bagging_classifier"])
def test_resident_features_copied_to_the_bagging_models(kind):
    """The bagging fits run on the host (scikit-learn stand-ins): the Param only reaches the model."""
    from spark_ensemble_b200.classification import BaggingClassifier
    from spark_ensemble_b200.learners import DecisionTreeClassifier, DecisionTreeRegressor
    from spark_ensemble_b200.regression import BaggingRegressor
    rng = np.random.default_rng(0)
    X = rng.standard_normal((200, 3)).astype(np.float32)
    y = (X[:, 0] > 0).astype(np.float64)
    if kind == "bagging_regressor":
        est = BaggingRegressor().setBaseLearner(DecisionTreeRegressor(maxDepth=2)).setNumBaseLearners(2)
    else:
        est = BaggingClassifier().setBaseLearner(DecisionTreeClassifier(maxDepth=2)).setNumBaseLearners(2)
    assert est.fit(DataFrame(features=X, label=y))("residentFeatures") is False
    m = est.setResidentFeatures(True).fit(DataFrame(features=X, label=y))
    assert m("residentFeatures") is True and m.isSet("residentFeatures")


def test_resident_features_copied_by_copy_values():
    for est_cls, model_cls in zip(_estimators(), _models()):
        est = est_cls().setResidentFeatures(True)
        model = model_cls.__new__(model_cls)
        model.__init__(*_model_args(model_cls))
        est._copyValues(model)
        assert model("residentFeatures") is True, model_cls.__name__


def _model_args(model_cls):
    from spark_ensemble_b200.ensemble import fit_dummy_regressor
    name = model_cls.__name__
    if name == "GBMRegressionModel":
        return ([], [], [], fit_dummy_regressor("constant", np.zeros(1)))
    if name == "GBMClassificationModel":
        return (2, [], [], [], np.zeros(1), 1)
    if name in ("BoostingClassificationModel",):
        return (2, [], [])
    if name == "BaggingRegressionModel":
        return ([], [])
    if name == "BaggingClassificationModel":
        return (2, [], [])
    return ([], [])


def test_forest_agg_bound():
    from spark_ensemble_b200 import _native as N
    assert "se_forest_agg" in N.PROTOTYPES
    assert N.FOREST_AGG_MAX_CLASSES == 32
