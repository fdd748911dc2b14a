"""Minimal mirror of Spark ML's Params machinery (org.apache.spark.ml.param), enough to keep the
reference's Estimator/Model surface: typed Params with validators and defaults, fluent setX/getX,
UIDs with the reference's prefixes, copy/extractParamMap/explainParams.

Reference surface mirrored: boosting/GBMParams.scala:29-131, boosting/BoostingParams.scala:26-37,
bagging/BaggingParams.scala:27-37, ensemble/HasSubBag.scala:27-71, ensemble/ensembleParams.scala:32-81.
"""
from __future__ import annotations

import copy as _copy
import uuid
from typing import Any, Callable


class Param:
    def __init__(self, name: str, doc: str, validator: Callable[[Any], bool] | None = None,
                 convert: Callable[[Any], Any] | None = None):
        self.name, self.doc, self.validator, self.convert = name, doc, validator, convert

    def __repr__(self):
        return f"Param({self.name})"


class ParamValidators:
    @staticmethod
    def gt(lo):
        return lambda v: v > lo

    @staticmethod
    def gtEq(lo):
        return lambda v: v >= lo

    @staticmethod
    def inRange(lo, hi):
        return lambda v: lo <= v <= hi

    @staticmethod
    def inArray(values):
        vals = list(values)
        return lambda v: v in vals


def random_uid(prefix: str) -> str:
    """Identifiable.randomUID: prefix + "_" + 12 hex digits."""
    return prefix + "_" + uuid.uuid4().hex[:12]


class Params:
    """Each subclass lists its Params in `_params` (name -> Param) and defaults in `_defaults`."""

    _params: dict[str, Param] = {}
    _defaults: dict[str, Any] = {}

    def __init__(self, uid: str):
        self.uid = uid
        self._paramMap: dict[str, Any] = {}

    # -- class-level declaration helpers
    @classmethod
    def _declare(cls, params: list[Param], defaults: dict[str, Any]):
        merged_p, merged_d = {}, {}
        for base in reversed(cls.__mro__[1:]):
            merged_p.update(getattr(base, "_params", {}))
            merged_d.update(getattr(base, "_defaults", {}))
        merged_p.update({p.name: p for p in params})
        merged_d.update(defaults)
        cls._params, cls._defaults = merged_p, merged_d
        for p in merged_p.values():
            cap = p.name[0].upper() + p.name[1:]
            if not hasattr(cls, "set" + cap):
                setattr(cls, "set" + cap, (lambda name: lambda self, value: self.set(name, value))(p.name))
            if not hasattr(cls, "get" + cap):
                setattr(cls, "get" + cap, (lambda name: lambda self: self.getOrDefault(name))(p.name))

    # -- instance API (Spark names)
    def hasParam(self, name: str) -> bool:
        return name in self._params

    def set(self, name: str, value):
        if name not in self._params:
            raise ValueError(f"Param {name} does not belong to {self.uid}")
        p = self._params[name]
        if p.convert is not None:
            value = p.convert(value)
        if p.validator is not None and not p.validator(value):
            # Spark: IllegalArgumentException from ParamValidators
            raise ValueError(f"{self.uid} parameter {name} given invalid value {value}.")
        self._paramMap[name] = value
        return self

    def isSet(self, name: str) -> bool:
        return name in self._paramMap

    def isDefined(self, name: str) -> bool:
        return name in self._paramMap or name in self._defaults

    def getOrDefault(self, name: str):
        if name in self._paramMap:
            return self._paramMap[name]
        if name in self._defaults:
            return self._defaults[name]
        raise KeyError(f"Failed to find a default value for {name}")

    def __call__(self, name: str):  # `$(param)` in Scala
        return self.getOrDefault(name)

    def extractParamMap(self) -> dict:
        m = dict(self._defaults)
        m.update(self._paramMap)
        return m

    def explainParams(self) -> str:
        lines = []
        for n, p in sorted(self._params.items()):
            cur = f"current: {self._paramMap[n]}" if n in self._paramMap else ""
            dft = f"default: {self._defaults[n]}" if n in self._defaults else "undefined"
            lines.append(f"{n}: {p.doc} ({dft}{', ' + cur if cur else ''})")
        return "\n".join(lines)

    def _copyValues(self, to: "Params", extra: dict | None = None) -> "Params":
        for n, v in self._paramMap.items():
            if to.hasParam(n):
                to._paramMap[n] = v
        for n, v in (extra or {}).items():
            if to.hasParam(n):
                to.set(n, v)
        return to

    def copy(self, extra: dict | None = None):
        other = _copy.copy(self)
        other._paramMap = dict(self._paramMap)
        for n, v in (extra or {}).items():
            other.set(n, v)
        return other


# ---- shared Spark params used by the ensembles (org.apache.spark.ml.param.shared) -----------------
def shared_predictor_params():
    return [
        Param("labelCol", "label column name"),
        Param("featuresCol", "features column name"),
        Param("predictionCol", "prediction column name"),
        Param("weightCol", "weight column name. If this is not set or empty, we treat all instance weights as 1.0"),
    ], {"labelCol": "label", "featuresCol": "features", "predictionCol": "prediction"}


def shared_classifier_params():
    return [
        Param("rawPredictionCol", "raw prediction (a.k.a. confidence) column name"),
        Param("probabilityCol", "Column name for predicted class conditional probabilities"),
        Param("thresholds", "Thresholds in multi-class classification to adjust the probability of predicting each class"),
    ], {"rawPredictionCol": "rawPrediction", "probabilityCol": "probability"}


def subbag_params():
    """ensemble/HasSubBag.scala:27-71 (SubBag defaults: replacement=true, ratios 1)."""
    return [
        Param("replacement", "whether samples are drawn with replacement", convert=bool),
        Param("subsampleRatio", "ratio of rows sampled out of the dataset", ParamValidators.inRange(0, 1), float),
        Param("subspaceRatio", "ratio of features sampled out of the dataset", ParamValidators.inRange(0, 1), float),
        Param("seed", "random seed", convert=int),
    ], {"replacement": True, "subsampleRatio": 1.0, "subspaceRatio": 1.0}


def boosting_params():
    """boosting/BoostingParams.scala:26-37 + ensemble/ensembleParams.scala:32-81."""
    return [
        Param("numBaseLearners", "number of base learners that will be used by the ensemble learner", ParamValidators.gtEq(1), int),
        Param("baseLearner", "base learner that will get stacked with boosting"),
        Param("checkpointInterval", "set checkpoint interval (>= 1) or disable checkpoint (-1)", convert=int),
        Param("aggregationDepth", "suggested depth for treeAggregate (>= 2)", ParamValidators.gtEq(2), int),
    ], {"numBaseLearners": 10, "checkpointInterval": 10, "aggregationDepth": 2}


# ---- the expert Params this project adds to the reference's surface --------------------------------------------------
# SURVEY.md §5: keep the column-major feature matrix in HBM and evaluate fitted trees / linear models on device instead
# of model.predict on the host; with a device tree learner, fit the trees there too
RESIDENT_FEATURES = Param("residentFeatures", "evaluate base models on device over the HBM-resident feature matrix",
                          convert=bool)
# "brent" = the reference's optimiser (default); "newton" = curvature-based line search on the same objective (dim 1,
# losses with a hessian): same minimiser within tol, ~6x fewer data passes
LINE_SEARCH = Param("lineSearch", "line-search optimiser for dim 1: brent (reference) or newton",
                    lambda v: v in ("brent", "newton"), str)
# GPUs to shard the rows of a GBM fit over (one context per GPU, contiguous row blocks); [] = the estimator's `device`
DEVICES = Param("devices", "CUDA device ordinals to shard the training rows over", lambda v: all(int(d) >= 0 for d in v),
                lambda v: [int(d) for d in v])


def gbm_params():
    """boosting/GBMParams.scala:29-131 (defaults :121-129)."""
    return [
        Param("optimizedWeights", "whether weights are optimized to minimize loss for each baseModel or weights are fixed to 1", convert=bool),
        Param("updates", "updates, (case-insensitive). Supported options: newton,gradient",
              lambda v: v.lower() in ("newton", "gradient"), str),
        Param("learningRate", "learning rate for the estimator", ParamValidators.gt(0.0), float),
        Param("validationTol", "Threshold for stopping early when fit with validation is used.", ParamValidators.gtEq(0.0), float),
        Param("numRounds", "number of round waiting for next decrease in validation set", ParamValidators.gtEq(1), int),
        Param("maxIter", "maximum number of iterations (>= 0)", ParamValidators.gtEq(0), int),
        Param("tol", "the convergence tolerance for iterative algorithms (>= 0)", ParamValidators.gtEq(0), float),
        Param("validationIndicatorCol", "name of the column that indicates whether each row is for training or for validation"),
        Param("parallelism", "the number of threads to use when running parallel algorithms (>= 1)", ParamValidators.gtEq(1), int),
    ], {"optimizedWeights": True, "updates": "gradient", "learningRate": 1.0, "numBaseLearners": 10,
        "tol": 1e-6, "maxIter": 100, "numRounds": 1, "validationTol": 0.01, "replacement": False,
        "parallelism": 1}
