"""Host-side mirror of the reference's classification ensembles for the hot path:
GBMClassifier (classification/GBMClassifier.scala), BoostingClassifier SAMME / SAMME.R
(classification/BoostingClassifier.scala) and the predictRaw/probability aggregation of
GBM / Boosting / Bagging classification models — same names, UID prefixes, Params and defaults, with
the per-row RDD closures replaced by calls into libse_b200.
"""
from __future__ import annotations

import math

import numpy as np

from . import _native as N
from .context import Context
from .ensemble import DataFrame, fit_dummy_classifier, java_string_hash
from .gbm_engine import fit_rounds
from .params import (DEVICES, LINE_SEARCH, RESIDENT_FEATURES, Param, Params, ParamValidators, boosting_params,
                     gbm_params, random_uid, shared_classifier_params, shared_predictor_params, subbag_params)
from .routes import (STACK_METHODS, bagging_fit, device_fit, device_linear, device_trees, extract_instances,
                     linear_kw, linear_list, load_boosting, member_route, one_pass, resident_linear, split_validation,
                     stacking_fit, stacking_predict, tree_list)

_CLS_LOSSES = ("logloss", "exponential", "bernoulli")  # GBMClassifier.scala:102-103
_CLS_INIT = ("uniform", "prior")                        # :104-106


def _num_classes(y: np.ndarray) -> int:
    """Classifier.getNumClasses: max label + 1 (labels are 0..K-1 doubles)."""
    return int(np.max(y)) + 1 if y.size else 0


def _validate_labels(y: np.ndarray, num_classes: int):
    """Classifier.validateLabel: non-negative integers below numClasses."""
    if y.size and (np.any(y < 0) or np.any(y != np.floor(y)) or np.any(y >= num_classes)):
        raise ValueError(f"Classifier was given dataset with invalid label; labels must be integers in [0, {num_classes})")


class _ClassifierModelBase(Params):
    """ProbabilisticClassificationModel.transform: rawPrediction, probability, prediction columns."""

    numClasses: int

    def _raw_prob_label(self, X):  # -> (raw [n,C], prob [n,C], label [n])
        raise NotImplementedError

    def transform(self, dataset: DataFrame) -> DataFrame:
        X = np.asarray(dataset[self("featuresCol")])
        raw, prob, label = self._raw_prob_label(X)
        out = dataset
        if self("rawPredictionCol"):
            out = out.withColumn(self("rawPredictionCol"), raw)
        if self("probabilityCol"):
            out = out.withColumn(self("probabilityCol"), prob)
        if self("predictionCol"):
            out = out.withColumn(self("predictionCol"), label)
        return out

    def predictRaw(self, features) -> np.ndarray:
        return self._raw_prob_label(np.asarray(features).reshape(1, -1))[0][0]

    def predictProbability(self, features) -> np.ndarray:
        return self._raw_prob_label(np.asarray(features).reshape(1, -1))[1][0]

    def predict(self, features) -> float:
        return float(self._raw_prob_label(np.asarray(features).reshape(1, -1))[2][0])

    def _fetch(self, ctx: Context):
        raw = ctx.download(N.SLOT_RAW).astype(np.float64)
        prob = ctx.download(N.SLOT_PROB).astype(np.float64)
        label = ctx.download(N.SLOT_LABEL).astype(np.float64)
        C = self._out_classes
        return raw.reshape(C, -1).T, prob.reshape(C, -1).T, label

    def _forest_agg_resident(self, X, kind: int, trees, **kw):
        """Scores the tree members in one pass over the device-resident features (se_forest_agg): no member output
        is computed on the host or stacked.  None when the forest is outside the kernel's reach (more than
        FOREST_AGG_MAX_CLASSES classes, or more than 255 thresholds in a column): the caller scores member by member."""
        if self.numClasses > N.FOREST_AGG_MAX_CLASSES:
            return None
        return one_pass(self.device, X, trees, lambda ctx, t: ctx.forest_agg(kind, self.numClasses, t, **kw),
                        self._fetch)

    def _linear_agg_resident(self, X, kind: int, members, **kw):
        """Scores linear and logistic members in one pass over the device-resident features (se_linear_agg), with the
        keyword arguments of _forest_agg_resident.  None without such members (device_linear) or above
        FOREST_AGG_MAX_CLASSES classes: the caller scores member by member."""
        if self.numClasses > N.FOREST_AGG_MAX_CLASSES:
            return None
        return one_pass(self.device, X, members,
                        lambda ctx, mb: ctx.linear_agg(kind, self.numClasses, mb, **linear_kw(kw)), self._fetch)

    def _one_pass(self, X):
        """The tree route (se_forest_agg), then the linear route (se_linear_agg); None leaves the member route."""
        kind, members, kw = self._forest_agg_args()
        out = self._forest_agg_resident(X, kind, device_trees(self, members), **kw)
        if out is None:
            out = self._linear_agg_resident(X, kind, device_linear(self, members), **kw)
        return out

    def _forest_agg_args(self):  # -> (kind, the members in forest order, keyword arguments of forest_agg)
        raise NotImplementedError

    def write_rows(self, ctx: Context, method: str, out_slot: int, out_row: int) -> bool:
        """A stacking member's meta-features over ctx's SLOT_X, on the device, when every member is a tree (one
        se_forest_agg pass) or a linear or logistic model (one se_linear_agg pass): its probability (proba), raw (raw)
        or label rows are then copied into out_slot from out_row on.  False when the members are outside both."""
        kind, members, kw = self._forest_agg_args()
        if not members or self.numClasses > N.FOREST_AGG_MAX_CLASSES:
            return False
        trees = tree_list(members)
        lin = linear_list(members) if trees is None else None
        if trees is not None:
            ctx.forest_agg(kind, self.numClasses, trees, **kw)
        elif lin is not None:
            ctx.linear_agg(kind, self.numClasses, lin, **linear_kw(kw))
        else:
            return False
        src, count = {"proba": (N.SLOT_PROB, self._out_classes), "raw": (N.SLOT_RAW, self._out_classes)}.get(
            method, (N.SLOT_LABEL, 1))
        ctx.copy_rows(out_slot, out_row, src, 0, count)
        return True


# ================================================================================ GBMClassifier
class GBMClassifier(Params):
    """classification/GBMClassifier.scala:146-496.  UID prefix "GBMClassifier" (:211)."""

    def __init__(self, uid: str | None = None, device: int = 0):
        super().__init__(uid or random_uid("GBMClassifier"))
        self.device = device

    def copy(self, extra=None):
        c = super().copy(extra)
        if c.isDefined("baseLearner"):
            c.set("baseLearner", c("baseLearner").copy(extra))
        return c

    def fit(self, dataset: DataFrame) -> "GBMClassificationModel":
        train_df, valid_df = split_validation(self, dataset)
        X, y, w = extract_instances(self, train_df)
        Xv, yv, _ = extract_instances(self, valid_df) if valid_df is not None else (None, None, None)
        num_classes = _num_classes(np.asarray(dataset[self("labelCol")], dtype=np.float64))
        _validate_labels(y, num_classes)
        loss = self("loss").lower()
        dim = num_classes if loss == "logloss" else 1  # GBMLoss.scala:198,270,295
        if dim == 1 and num_classes != 2:
            raise ValueError(f"loss {loss} is binary; got numClasses={num_classes}")
        newton = self("updates").lower() == "newton"  # every classification loss HasHessian (:338)

        # init :275-288 — binary "prior" with dim 1 stores the FULL log-odds (reference quirk 5)
        init_strategy = self("initStrategy").lower()
        if init_strategy == "prior" and dim == 1 and num_classes == 2:
            p1 = float(np.mean(y == 1.0))
            logodds = math.log(p1 / (1 - p1))
            init_raw = np.array([logodds])
        else:
            init_raw = fit_dummy_classifier(init_strategy, y, num_classes).rawPrediction
            if init_raw.shape[0] != dim:
                raise ValueError("prior init needs every class present in the training labels")

        def line_search(eng):  # :413-431
            if self("lineSearch") == "newton" and dim == 1:
                return eng.line_search_newton(self("tol"), self("maxIter"))[0]
            return eng.line_search_lbfgsb(self("tol"), self("maxIter"))[0]

        learner = self("baseLearner")
        fit_on_device = device_fit(self, learner, require_resident=True)
        models, weights, subspaces, history = fit_rounds(
            self, X, y, w, Xv, yv, dim, loss, 0.0, init_raw, init_raw if Xv is not None else None, learner,
            fit_on_device, newton, line_search)
        model = GBMClassificationModel(num_classes, weights, subspaces, models, init_raw, dim, device=self.device)
        self._copyValues(model)
        model.parent = self
        model.trainingHistory = history
        return model


_p, _d = shared_predictor_params()
_pc, _dc = shared_classifier_params()
_ps, _ds = subbag_params()
_pb, _db = boosting_params()
_pg, _dg = gbm_params()
_pcls = [
    Param("loss", "loss function, (case-insensitive). Supported options:" + ",".join(_CLS_LOSSES),
          lambda v: v.lower() in _CLS_LOSSES, str),
    Param("initStrategy", "strategy for the init predictions (uniform, prior)", lambda v: v in _CLS_INIT, str),
    RESIDENT_FEATURES, LINE_SEARCH, DEVICES,
]
_GBM_CLS_DEFAULTS = {**_d, **_dc, **_ds, **_db, **_dg, "loss": "logloss", "initStrategy": "prior",
                     "residentFeatures": False, "lineSearch": "brent", "devices": [],
                     "seed": java_string_hash("org.apache.spark.ml.classification.GBMClassifier")}
GBMClassifier._declare(_p + _pc + _ps + _pb + _pg + _pcls, _GBM_CLS_DEFAULTS)


class GBMClassificationModel(_ClassifierModelBase):
    """classification/GBMClassifier.scala:532-612; predictRaw :567-589, raw2probability :564-565."""

    def __init__(self, numClasses, weights, subspaces, models, init_raw, dim, uid=None, device: int = 0):
        super().__init__(uid or random_uid("GBMClassificationModel"))
        self.numClasses = int(numClasses)
        self.weights = [np.asarray(wt, dtype=np.float64) for wt in weights]
        self.subspaces, self.models = list(subspaces), [list(m) for m in models]
        self.init = np.asarray(init_raw, dtype=np.float64)
        self.dim = int(dim)
        self.numModels = len(self.models)
        self.device = device
        self.parent = None
        self._out_classes = 2 if (self.dim == 1 and self.numClasses == 2) else self.dim

    def _forest_agg_args(self):
        M, dim = self.numModels, self.dim
        return N.AGG_GBM_CLASSIFIER, [m for ms in self.models for m in ms], dict(
            weights=np.concatenate([np.asarray(wt, dtype=np.float64).reshape(dim) for wt in self.weights]) if M else None,
            init=self.init, tree_class=np.tile(np.arange(dim, dtype=np.int32), M), dim=dim, loss=self("loss").lower(),
            subspaces=[s for s in self.subspaces[:M] for _ in range(dim)])

    def _raw_prob_label(self, X):
        n, M, dim = X.shape[0], self.numModels, self.dim
        out = self._one_pass(X)
        if out is not None:
            return out
        P = np.zeros((max(M, 1), dim, n), dtype=np.float32)
        for i in range(M):
            Xs = X[:, self.subspaces[i]]
            for j in range(dim):
                P[i, j] = self.models[i][j].predict(Xs)
        a = np.stack(self.weights) if M else np.zeros((1, dim))
        return member_route(self.device, N.AGG_GBM_CLASSIFIER, P, self.numClasses, dim, self("loss").lower(), a,
                            self.init, self._fetch)


GBMClassificationModel._declare(_p + _pc + _ps + _pb + _pg + _pcls, _GBM_CLS_DEFAULTS)


# ================================================================================ BoostingClassifier
class BoostingClassifier(Params):
    """classification/BoostingClassifier.scala:105-282: AdaBoost SAMME ("discrete") / SAMME.R ("real")."""

    def __init__(self, uid: str | None = None, device: int = 0):
        super().__init__(uid or random_uid("BoostingClassifier"))
        self.device = device

    def fit(self, dataset: DataFrame) -> "BoostingClassificationModel":
        X, y, w = extract_instances(self, dataset)
        K = _num_classes(y)
        _validate_labels(y, K)
        real = self("algorithm").lower() == "real"
        learner = self("baseLearner")
        fit_on_device = device_fit(self, learner, require_resident=True)
        linear_on_device = resident_linear(self, learner)
        resident = bool(self("residentFeatures"))
        out_slot = N.SLOT_PROBA if real else N.SLOT_PRED  # the member's probabilities (SAMME.R) or labels (SAMME)
        models, est_weights, history = [], [], []
        with Context(self.device) as ctx:
            ctx.boost_configure(y.shape[0], K, real)
            # column-major X in HBM whenever residentFeatures is set: host-fitted trees are evaluated on the device too
            # (no K x n upload per round)
            all_cols, sum_w = load_boosting(ctx, X, y, w, learner, fit_on_device, upload_features=resident)  # :168-175
            i, done = 0, False
            while i < self("numBaseLearners") and not done and sum_w > 0:  # :180
                if fit_on_device:  # fitted on SLOT_Y / SLOT_BW where they live, straight into out_slot; the splits
                    # are invariant under the common 1 / sumWeights scale of :184-187
                    model = learner.fit_resident(ctx, K, N.SLOT_Y, 0, N.SLOT_BW, 0, False, all_cols, out_slot, 0,
                                                 proba=real)
                elif linear_on_device:  # the same: Spark's logistic objective is divided by Σ c
                    model = learner.fit_resident(ctx, N.SLOT_X, np.arange(X.shape[1], dtype=np.int32), K, N.SLOT_Y, 0,
                                                 N.SLOT_BW, 0, out_slot, 0, "proba" if real else "class",
                                                 shift=np.asarray(X[0], dtype=np.float64))
                else:
                    wn = ctx.download(N.SLOT_BW, scale=1.0 / sum_w)  # weight = boostingWeight / sumWeights :184-187
                    model = learner.fit(X, y, wn, num_classes=K)    # third party :189-195
                if real and not hasattr(model, "predictProbability"):
                    raise RuntimeError('algorithm "real" is not compatible with base learner')  # :261-263
                if not (fit_on_device or linear_on_device):  # the output into out_slot: on the device for a tree
                    t = model.tree_arrays() if resident else None
                    if t is not None:
                        if real:
                            ctx.tree_predict_multi(t, out_slot)
                        else:
                            ctx.tree_predict(t, out_slot, 0)
                    elif real:
                        ctx.upload(out_slot, np.ascontiguousarray(model.predictProbability(X).T, dtype=np.float32))
                    else:
                        ctx.upload(out_slot, model.predict(X))
                models.append(model)
                if real:  # SAMME.R :198-230
                    err, new_sum = ctx.boost_real_update(sum_w)
                    if err <= 0:
                        done = True
                    est_weights.append(1.0)  # :212
                else:  # SAMME :231-260
                    err = ctx.boost_discrete_error(sum_w)
                    if err <= 0:
                        done = True
                    beta = err / ((1 - err) * (K - 1))
                    est_weights.append(1.0 if beta == 0.0 else math.log(1.0 / beta))
                    if err >= 1.0 - (1.0 / K):  # :252 drop this model and stop
                        i -= 1
                        done = True
                    new_sum = ctx.boost_discrete_update(sum_w, beta if beta != 0.0 else 0.0)
                history.append({"estimatorError": err, "sumWeights": new_sum})
                sum_w = new_sum  # :269
                i += 1
            keep = max(i, 0)
            model = BoostingClassificationModel(K, est_weights[:keep], models[:keep], device=self.device)
            self._copyValues(model)
            model.parent = self
            model.trainingHistory = history
            return model


_pboost = [Param("algorithm", "algorithm, (case-insensitive). Supported options: discrete,real",
                 lambda v: v.lower() in ("discrete", "real"), str),
           RESIDENT_FEATURES]
_BOOST_DEFAULTS = {**_d, **_dc, **_db, "algorithm": "discrete", "residentFeatures": False,
                   "seed": java_string_hash("org.apache.spark.ml.classification.BoostingClassifier")}
BoostingClassifier._declare(_p + _pc + _pb + _pboost + [Param("seed", "random seed", convert=int)], _BOOST_DEFAULTS)


class BoostingClassificationModel(_ClassifierModelBase):
    """classification/BoostingClassifier.scala:318-404; predictRawReal :348-364, predictRawDiscrete
    :366-382, raw2probabilityInPlace :342-346."""

    def __init__(self, numClasses, weights, models, uid=None, device: int = 0):
        super().__init__(uid or random_uid("BoostingClassificationModel"))
        self.numClasses = int(numClasses)
        self.weights = np.asarray(weights, dtype=np.float64)
        self.models = list(models)
        self.numModels = len(self.models)
        self.device = device
        self.parent = None
        self._out_classes = self.numClasses

    def _forest_agg_args(self):
        real = self("algorithm").lower() == "real"
        kind = N.AGG_BOOSTING_REAL if real else N.AGG_BOOSTING_DISCRETE
        return kind, self.models, dict(weights=None if real else self.weights)

    def _raw_prob_label(self, X):
        n, M, K = X.shape[0], self.numModels, self.numClasses
        real = self("algorithm").lower() == "real"
        out = self._one_pass(X)
        if out is not None:
            return out
        kind = self._forest_agg_args()[0]
        if real:
            P = np.zeros((max(M, 1), K, n), dtype=np.float32)
            for i, m in enumerate(self.models):
                P[i] = m.predictProbability(X).T
            if M == 0:
                P[:] = 1.0
            return member_route(self.device, kind, P, K, fetch=self._fetch)
        V = np.zeros((max(M, 1), n), dtype=np.float32)
        for i, m in enumerate(self.models):
            V[i] = m.predict(X)
        return member_route(self.device, kind, V, K, weights=self.weights if M else np.zeros(1), fetch=self._fetch)


BoostingClassificationModel._declare(_p + _pc + _pb + _pboost + [Param("seed", "random seed", convert=int)], _BOOST_DEFAULTS)


# ================================================================================ BaggingClassifier
class BaggingClassifier(Params):
    """classification/BaggingClassifier.scala:106-207.  With residentFeatures and a device tree learner every member's
    tree grows in one forest fit over the device-resident features; otherwise train is one learner.fit per member:
    routes.bagging_fit."""

    def __init__(self, uid: str | None = None, device: int = 0):
        super().__init__(uid or random_uid("BaggingClassifier"))
        self.device = device

    def fit(self, dataset: DataFrame) -> "BaggingClassificationModel":
        X, y, w = extract_instances(self, dataset)
        K = _num_classes(y)
        subs, models = bagging_fit(self, X, y, w, num_classes=K)
        m = BaggingClassificationModel(K, subs, models, device=self.device)
        self._copyValues(m)
        m.parent = self
        return m


_pbagc = [Param("numBaseLearners", "number of base learners", ParamValidators.gtEq(1), int),
          Param("baseLearner", "base learner"),
          Param("votingStrategy", "voting strategy, (case-insensitive). Supported options: soft,hard",
                lambda v: v.lower() in ("soft", "hard"), str),
          Param("parallelism", "threads", ParamValidators.gtEq(1), int),
          RESIDENT_FEATURES]
_BAG_CLS_DEFAULTS = {**_d, **_dc, **_ds, "numBaseLearners": 10, "votingStrategy": "hard", "parallelism": 1,
                     "residentFeatures": False,
                     "seed": java_string_hash("org.apache.spark.ml.classification.BaggingClassifier")}
BaggingClassifier._declare(_p + _pc + _ps + _pbagc, _BAG_CLS_DEFAULTS)


class BaggingClassificationModel(_ClassifierModelBase):
    """classification/BaggingClassifier.scala:243-300; predictRaw :260-283, raw2probability :285-287."""

    def __init__(self, numClasses, subspaces, models, uid=None, device: int = 0):
        super().__init__(uid or random_uid("BaggingClassificationModel"))
        self.numClasses = int(numClasses)
        self.subspaces, self.models = list(subspaces), list(models)
        self.numModels = len(self.models)
        self.device = device
        self.parent = None
        self._out_classes = self.numClasses

    def _forest_agg_args(self):
        soft = self("votingStrategy").lower() == "soft"
        kind = N.AGG_BAGGING_SOFT if soft else N.AGG_BAGGING_HARD
        return kind, self.models, dict(subspaces=self.subspaces)

    def _raw_prob_label(self, X):
        n, M, K = X.shape[0], self.numModels, self.numClasses
        soft = self("votingStrategy").lower() == "soft"
        out = self._one_pass(X)
        if out is not None:
            return out
        kind = self._forest_agg_args()[0]
        P = np.zeros((M, K, n) if soft else (M, n), dtype=np.float32)
        for i, m in enumerate(self.models):
            Xs = X[:, self.subspaces[i]]
            P[i] = m.predictProbability(Xs).T if soft else m.predict(Xs)
        return member_route(self.device, kind, P, K, fetch=self._fetch)


BaggingClassificationModel._declare(_p + _pc + _ps + _pbagc, _BAG_CLS_DEFAULTS)


# ================================================================================ StackingClassifier
class StackingClassifier(Params):
    """classification/StackingClassifier.scala: every base learner fits on the dataset, its outputs become the
    meta-features of each row (stackMethod: the members' labels, raw vectors or probabilities, member-major) and the
    stacker fits on them.  residentFeatures keeps X and the meta-features on the device (routes.stacking_fit)."""

    def __init__(self, uid: str | None = None, device: int = 0):
        super().__init__(uid or random_uid("StackingClassifier"))
        self.device = device

    def copy(self, extra=None):
        c = super().copy(extra)
        if c.isDefined("baseLearners"):
            c.set("baseLearners", [m.copy(extra) for m in c("baseLearners")])
        if c.isDefined("stacker"):
            c.set("stacker", c("stacker").copy(extra))
        return c

    def fit(self, dataset: DataFrame) -> "StackingClassificationModel":
        y = np.asarray(dataset[self("labelCol")], dtype=np.float64)
        K = _num_classes(y)
        _validate_labels(y, K)
        models, stack, widths = stacking_fit(self, dataset, num_classes=K)
        m = StackingClassificationModel(models, stack, K, widths, device=self.device)
        self._copyValues(m)
        m.parent = self
        return m


_pstack = [Param("baseLearners", "base learners that will be used by the ensemble learner", convert=list),
           Param("stacker", "stacker that will be used by the ensemble learner to aggregate results of base learner(s)"),
           Param("parallelism", "the number of threads to use when running parallel algorithms (>= 1)",
                 ParamValidators.gtEq(1), int),
           RESIDENT_FEATURES]
_pstackc = [Param("stackMethod", "stackMethod, (case-insensitive). Supported options:" + ",".join(STACK_METHODS),
                  lambda v: v.lower() in STACK_METHODS, str)]
_STACK_CLS_DEFAULTS = {**_d, **_dc, "parallelism": 1, "residentFeatures": False, "stackMethod": "class"}
StackingClassifier._declare(_p + _pc + _pstack + _pstackc, _STACK_CLS_DEFAULTS)


class StackingClassificationModel(Params):
    """classification/StackingClassifier.scala StackingClassificationModel: predict = stack.predict(the members'
    meta-features); transform writes the prediction column only (PredictionModel)."""

    def __init__(self, models, stack, numClasses, widths, uid=None, device: int = 0):
        super().__init__(uid or random_uid("StackingClassificationModel"))
        self.models, self.stack = list(models), stack
        self.numClasses = int(numClasses)
        self.widths = [int(k) for k in widths]
        self.device = device
        self.parent = None

    def copy(self, extra=None):
        c = super().copy(extra)
        c.parent = self.parent
        return c

    def _predict(self, X) -> np.ndarray:
        return stacking_predict(self, X)

    def transform(self, dataset: DataFrame) -> DataFrame:
        return dataset.withColumn(self("predictionCol"), self._predict(np.asarray(dataset[self("featuresCol")])))

    def predict(self, features) -> float:
        return float(self._predict(np.asarray(features).reshape(1, -1))[0])


StackingClassificationModel._declare(_p + _pc + _pstack + _pstackc, _STACK_CLS_DEFAULTS)
