"""Host-side mirror of the reference's regression ensembles for the hot path:
GBMRegressor / GBMRegressionModel (regression/GBMRegressor.scala) and BaggingRegressionModel.predict
(regression/BaggingRegressor.scala:221-228) — same class names, UID prefixes, Params and defaults; the
per-row RDD closures of train()/predict() are replaced by calls into libse_b200 (sm_90a kernels).

On a JVM host the same substitution is made in Scala (scala/ + jni/se_jni.cpp, see INTEGRATION.md).
"""
from __future__ import annotations

import numpy as np

from . import _native as N
from .context import Context
from .ensemble import DataFrame, exact_quantile, fit_dummy_regressor, java_string_hash
from .gbm_engine import fit_rounds
from .params import (DEVICES, LINE_SEARCH, RESIDENT_FEATURES, Param, Params, ParamValidators, boosting_params,
                     gbm_params, random_uid, shared_predictor_params, subbag_params)
from .routes import (bagging_fit, device_fit, device_linear, device_trees, download_raw, extract_instances, forest_sum,
                     linear_list, linear_sum, load_boosting, member_route, one_pass, resident_context, resident_linear,
                     split_validation, stack_outputs, stacking_fit, stacking_predict, tree_list)

_REG_LOSSES = ("squared", "absolute", "huber", "quantile")  # GBMRegressor.scala:119-120
_REG_INIT = ("constant", "zero", "base")                     # :121-123


class GBMRegressor(Params):
    """regression/GBMRegressor.scala:164-476.  UID prefix "GBMRegressor2" (sic, :229)."""

    def __init__(self, uid: str | None = None, device: int = 0):
        super().__init__(uid or random_uid("GBMRegressor2"))
        self.device = device

    def copy(self, extra=None):
        c = super().copy(extra)
        if c.isDefined("baseLearner"):
            c.set("baseLearner", c("baseLearner").copy(extra))  # :230-234
        return c

    def fit(self, dataset: DataFrame) -> "GBMRegressionModel":
        return self._train(dataset)

    # -- GBMRegressor.train :237-476
    def _train(self, dataset: DataFrame) -> "GBMRegressionModel":
        train_df, valid_df = split_validation(self, dataset)
        X, y, w = extract_instances(self, train_df)
        Xv, yv, _ = extract_instances(self, valid_df) if valid_df is not None else (None, None, None)
        loss = self("loss").lower()
        learner = self("baseLearner")

        # init model :287-303
        init_strategy = self("initStrategy").lower()
        if init_strategy == "base":
            init = learner.fit(X, y, w)
        elif init_strategy == "zero":
            init = fit_dummy_regressor("constant", y, constant=0.0)
        else:
            strat = {"squared": "mean", "absolute": "median", "huber": "median", "quantile": "quantile"}[loss]
            init = fit_dummy_regressor(strat, y, quantile=self("alpha"))

        # huber delta / quantile parameter :305-308
        param = exact_quantile(y, self("alpha")) if loss == "huber" else self("alpha")
        newton = self("updates").lower() == "newton" and loss == "squared"  # HasScalarHessian among selectable losses :369

        def line_search(eng):  # :398-425
            if self("lineSearch") == "newton" and loss == "squared":
                return eng.line_search_newton(self("tol"), self("maxIter"))[0]
            return eng.line_search_brent(self("tol"), self("maxIter"))[0]

        fit_on_device = device_fit(self, learner, require_resident=True)
        const_init = hasattr(init, "prediction")  # Dummy model: broadcast the constant on device
        F0 = init.prediction if const_init else init.predict(X)
        vF0 = (init.prediction if const_init else init.predict(Xv)) if Xv is not None else None
        models, weights, subspaces, history = fit_rounds(self, X, y, w, Xv, yv, 1, loss, param, F0, vF0, learner,
                                                         fit_on_device, newton, line_search)
        for h in history:
            h["alpha"] = float(h["alpha"][0])
        model = GBMRegressionModel([float(wt[0]) for wt in weights], subspaces, [m[0] for m in models], init,
                                   device=self.device)
        self._copyValues(model)
        model.parent = self
        model.trainingHistory = history
        return model


_p, _d = shared_predictor_params()
_ps, _ds = subbag_params()
_pb, _db = boosting_params()
_pg, _dg = gbm_params()
_preg = [
    Param("loss", "loss function, (case-insensitive). Supported options:" + ",".join(_REG_LOSSES),
          lambda v: v.lower() in _REG_LOSSES, str),
    Param("alpha", "The alpha-quantile of the loss function. Only for huber and quantile loss.", convert=float),
    Param("initStrategy", "strategy for the init predictions (constant, zero, base)",
          lambda v: v in _REG_INIT, str),
    RESIDENT_FEATURES, LINE_SEARCH, DEVICES,
]
_GBM_REG_DEFAULTS = {**_d, **_ds, **_db, **_dg, "loss": "squared", "alpha": 0.9, "initStrategy": "constant", "residentFeatures": False, "lineSearch": "brent",
                     "devices": [],
                     "seed": java_string_hash("org.apache.spark.ml.regression.GBMRegressor")}
GBMRegressor._declare(_p + _ps + _pb + _pg + _preg, _GBM_REG_DEFAULTS)


class GBMRegressionModel(Params):
    """regression/GBMRegressor.scala:512-556; predict :531-539 = init + Σ_i w_i·m_i(x[S_i])."""

    def __init__(self, weights, subspaces, models, init, uid: str | None = None, device: int = 0):
        super().__init__(uid or random_uid("GBMRegressionModel"))
        self.weights = np.asarray(weights, dtype=np.float64)
        self.subspaces = list(subspaces)
        self.models = list(models)
        self.init = init
        self.numModels = len(self.models)
        self.device = device
        self.parent = None

    def _forest(self):  # -> (members, subspaces, weights, init) of the one-pass sum
        const_init = hasattr(self.init, "prediction")  # else a tree init scores as one more member of weight 1
        members = self.models if const_init else [self.init] + self.models
        subs = list(self.subspaces) if const_init else [None] + list(self.subspaces)
        a = self.weights if const_init else np.concatenate([[1.0], self.weights])
        init = self.init.prediction if const_init else 0.0
        return members, subs, a, init

    def write_rows(self, ctx: Context, method: str, out_slot: int, out_row: int) -> bool:
        """Its prediction over ctx's SLOT_X into row out_row of out_slot in one pass when every member is a tree, or a
        linear model after a constant init (a stacking member's meta-feature)."""
        members, subs, a, init = self._forest()
        trees = tree_list(members) if members else None
        if trees is not None:
            ctx.forest_predict(trees, out_slot, weights=a, init=init, out_row=out_row, subspaces=subs)
            return True
        lin = linear_list(self.models) if (self.models and hasattr(self.init, "prediction")) else None
        if lin is None:
            return False
        ctx.linear_agg(N.AGG_GBM_REGRESSOR, 0, lin, out_slot, out_row, weights=self.weights, init=[init],
                       subspaces=self.subspaces)
        return True

    def _aggregate(self, X) -> np.ndarray:
        const_init = hasattr(self.init, "prediction")
        members, subs, a, init = self._forest()
        out = forest_sum(self.device, X, device_trees(self, members), subs, a, init)
        if out is None and const_init:
            out = linear_sum(self.device, X, device_linear(self, self.models), self.subspaces, N.AGG_GBM_REGRESSOR,
                             weights=self.weights, init=[init])
        if out is not None:
            return out
        P = stack_outputs(self.models, self.subspaces, X, None if const_init else self.init.predict(X))
        return member_route(self.device, N.AGG_GBM_REGRESSOR, P, weights=a, init=[init])

    def transform(self, dataset: DataFrame) -> DataFrame:
        X = np.asarray(dataset[self("featuresCol")])
        return dataset.withColumn(self("predictionCol"), self._aggregate(X))

    def predict(self, features) -> float:
        return float(self._aggregate(np.asarray(features).reshape(1, -1))[0])


GBMRegressionModel._declare(_p + _ps + _pb + _pg + _preg, _GBM_REG_DEFAULTS)


# ---- Bagging -------------------------------------------------------------------------------------------------------
class BaggingRegressor(Params):
    """regression/BaggingRegressor.scala:77-172.  With residentFeatures and a device tree learner every member's
    tree grows in one forest fit over the device-resident features; otherwise train is the minimal host loop (one
    learner.fit per member): routes.bagging_fit."""

    def __init__(self, uid: str | None = None, device: int = 0):
        super().__init__(uid or random_uid("BaggingRegressor"))
        self.device = device

    def fit(self, dataset: DataFrame) -> "BaggingRegressionModel":
        X, y, w = extract_instances(self, dataset)
        subs, models = bagging_fit(self, X, y, w)
        m = BaggingRegressionModel(subs, models, device=self.device)
        self._copyValues(m)
        m.parent = self
        return m


_pbag = [Param("numBaseLearners", "number of base learners", ParamValidators.gtEq(1), int),
         Param("baseLearner", "base learner"),
         Param("parallelism", "the number of threads to use when running parallel algorithms (>= 1)",
               ParamValidators.gtEq(1), int),
         RESIDENT_FEATURES]
_BAG_REG_DEFAULTS = {**_d, **_ds, "numBaseLearners": 10, "parallelism": 1, "residentFeatures": False,
                     "seed": java_string_hash("org.apache.spark.ml.regression.BaggingRegressor")}
BaggingRegressor._declare(_p + _ps + _pbag, _BAG_REG_DEFAULTS)


class BaggingRegressionModel(Params):
    """regression/BaggingRegressor.scala:208-235; predict :221-228 = (Σ_i m_i(x[S_i])) / numModels."""

    def __init__(self, subspaces, models, uid: str | None = None, device: int = 0):
        super().__init__(uid or random_uid("BaggingRegressionModel"))
        self.subspaces, self.models = list(subspaces), list(models)
        self.numModels = len(self.models)
        self.device = device
        self.parent = None

    def write_rows(self, ctx: Context, method: str, out_slot: int, out_row: int) -> bool:
        """Its prediction over ctx's SLOT_X into row out_row of out_slot in one forest pass when every member is a tree
        (a stacking member's meta-feature): Σ_t tree_t(x) / M as weights 1/M."""
        trees = tree_list(self.models) if self.models else None
        if trees is not None:
            ctx.forest_predict(trees, out_slot, weights=np.full(len(trees), 1.0 / len(trees)), out_row=out_row,
                               subspaces=self.subspaces)
            return True
        lin = linear_list(self.models) if self.models else None
        if lin is None:
            return False
        ctx.linear_agg(N.AGG_BAGGING_REGRESSOR, 0, lin, out_slot, out_row, subspaces=self.subspaces)
        return True

    def _aggregate(self, X) -> np.ndarray:
        s = forest_sum(self.device, X, device_trees(self, self.models), self.subspaces, None, 0.0)
        if s is not None:  # (Σ_t tree_t(x)) / M in one pass over the device-resident features
            return s / self.numModels
        s = linear_sum(self.device, X, device_linear(self, self.models), self.subspaces, N.AGG_BAGGING_REGRESSOR)
        if s is not None:
            return s
        P = stack_outputs(self.models, self.subspaces, X)
        return member_route(self.device, N.AGG_BAGGING_REGRESSOR, P)

    def transform(self, dataset: DataFrame) -> DataFrame:
        return dataset.withColumn(self("predictionCol"), self._aggregate(np.asarray(dataset[self("featuresCol")])))

    def predict(self, features) -> float:
        return float(self._aggregate(np.asarray(features).reshape(1, -1))[0])


BaggingRegressionModel._declare(_p + _ps + _pbag, _BAG_REG_DEFAULTS)


# ---- BoostingRegressor (AdaBoost.R2, Drucker 1997): SURVEY.md §8f-2 -----------------------------------
class BoostingRegressor(Params):
    """regression/BoostingRegressor.scala:138-282.  Per round: maxError, estimatorError = Σ wₙ·loss, weight
    update wₙ·β^(1-loss), Σw' — three streaming passes on the device instead of four RDD jobs."""

    def __init__(self, uid: str | None = None, device: int = 0):
        super().__init__(uid or random_uid("BoostingRegressor"))
        self.device = device

    def fit(self, dataset: DataFrame) -> "BoostingRegressionModel":
        X, y, w = extract_instances(self, dataset)
        loss_type = self("lossType").lower()
        learner = self("baseLearner")
        # A device learner fits where the boosting weights live when the features are resident.  Without
        # residentFeatures it keeps the learner.fit route below (its own context per round) rather than raising.
        fit_on_device = device_fit(self, learner, require_resident=False)
        linear_on_device = resident_linear(self, learner)
        models, est_weights, history = [], [], []
        with Context(self.device) as ctx:
            ctx.boostreg_configure(y.shape[0])
            # X only for the device fit: a host-fitted tree is not walked on the device here (BoostingClassifier does)
            all_cols, sum_w = load_boosting(ctx, X, y, w, learner, fit_on_device,  # :205-212
                                            upload_features=fit_on_device or linear_on_device)
            if linear_on_device:  # the shifts learner.fit takes: the column means
                cols = np.arange(X.shape[1], dtype=np.int32)
                shift = np.asarray(X, dtype=np.float32).mean(axis=0, dtype=np.float64)
            i, best, done = 0, 0, False
            while i < self("numBaseLearners") and not done and sum_w > 0:  # :218
                if fit_on_device:  # fitted on SLOT_Y / SLOT_BW where they live, straight into SLOT_PRED; the splits are
                    # invariant under the common 1 / sumWeights scale of :222-225
                    model = learner.fit_resident(ctx, N.SLOT_Y, 0, N.SLOT_BW, 0, False, all_cols, N.SLOT_PRED, 0)
                elif linear_on_device:  # on the normalised weights of :222-225, since regParam > 0 depends on their scale
                    model = learner.fit_resident(ctx, N.SLOT_X, cols, N.SLOT_Y, 0, N.SLOT_BW, 0, False, N.SLOT_PRED, 0,
                                                 shift=shift, weight_scale=1.0 / sum_w)
                else:
                    wn = ctx.download(N.SLOT_BW, scale=1.0 / sum_w)  # :222-225
                    model = learner.fit(X, y, wn)                     # third party :231-233
                    ctx.upload(N.SLOT_PRED, model.predict(X))
                max_error = ctx.boostreg_max_error()                 # :235-238
                if max_error == 0:                                   # :240-243
                    best, done = i, True
                est_err = ctx.boostreg_error(sum_w, loss_type, max_error)  # :248-254
                if est_err >= 0.5:                                   # :256
                    best, done = i - 1, True
                beta = est_err / (1 - est_err)
                est_weight = 1.0 if beta == 0.0 else float(np.log(1.0 / beta))
                sum_w = ctx.boostreg_update(sum_w, loss_type, max_error, beta) if beta > 0 else 0.0  # :261-268
                est_weights.append(est_weight)
                models.append(model)
                history.append({"maxError": max_error, "estimatorError": est_err, "sumWeights": sum_w})
                best = i
                i += 1
            best += 1
            m = BoostingRegressionModel(est_weights[:best], models[:best], device=self.device)
            self._copyValues(m)
            m.parent = self
            m.trainingHistory = history
            return m


_pbr = [Param("lossType", "loss function, exponential by default (case-insensitive). Supported: exponential,squared,linear",
              lambda v: v.lower() in ("exponential", "squared", "linear"), str),
        Param("votingStrategy", "voting strategy, (case-insensitive). Supported options: median,mean",
              lambda v: v.lower() in ("median", "mean"), str),
        Param("seed", "random seed", convert=int),
        RESIDENT_FEATURES]
_BOOST_REG_DEFAULTS = {**_d, **_db, "lossType": "exponential", "votingStrategy": "median", "residentFeatures": False,
                       "seed": java_string_hash("org.apache.spark.ml.regression.BoostingRegressor")}
BoostingRegressor._declare(_p + _pb + _pbr, _BOOST_REG_DEFAULTS)


class BoostingRegressionModel(Params):
    """regression/BoostingRegressor.scala:318-360: weighted median (ensemble/Utils.scala:26-40) or weighted
    mean of the members' predictions."""

    def __init__(self, weights, models, uid: str | None = None, device: int = 0):
        super().__init__(uid or random_uid("BoostingRegressionModel"))
        self.weights = np.asarray(weights, dtype=np.float64)
        self.models = list(models)
        self.numModels = len(self.models)
        self.device = device
        self.parent = None

    def write_rows(self, ctx: Context, method: str, out_slot: int, out_row: int) -> bool:
        """Its prediction over ctx's SLOT_X into row out_row of out_slot in one forest pass when every member is a tree
        (a stacking member's meta-feature): the weighted median of at most 64 trees, or the weighted mean."""
        trees = tree_list(self.models) if self.models else None
        median = self("votingStrategy").lower() == "median"
        if trees is None:
            lin = linear_list(self.models) if self.models else None
            if lin is None or (median and len(lin) > N.FOREST_MEDIAN_MAX_TREES):
                return False
            ctx.linear_agg(N.AGG_BOOSTING_REG_MEDIAN if median else N.AGG_BOOSTING_REG_MEAN, 0, lin, out_slot, out_row,
                           weights=self.weights)
            return True
        if median:
            if len(trees) > N.FOREST_MEDIAN_MAX_TREES:
                return False
            ctx.forest_median(trees, out_slot, self.weights, out_row=out_row)
        else:
            ctx.forest_predict(trees, out_slot, weights=self.weights / float(np.sum(self.weights)), out_row=out_row)
        return True

    def _aggregate_resident(self, X, median: bool) -> np.ndarray | None:
        """Members evaluated over the device-resident features when every one is a tree: the weighted mean in one
        forest pass, and the median of at most 64 trees too (se_forest_median).  Above 64 trees, or when the rank
        matrix cannot hold the thresholds, each tree writes its row of SLOT_P on the device before the aggregation."""
        trees = device_trees(self, self.models)
        if trees is None:
            return None
        if not median:
            s = forest_sum(self.device, X, trees, None, self.weights, 0.0)
            return None if s is None else s / float(np.sum(self.weights))
        n = X.shape[0]

        def score(ctx, trees):
            ctx.alloc(N.SLOT_RAW, 1, n)
            ctx.forest_median(trees, N.SLOT_RAW, self.weights)
        out = one_pass(self.device, X, trees if len(trees) <= N.FOREST_MEDIAN_MAX_TREES else None, score, download_raw)
        if out is not None:
            return out
        with resident_context(self.device, X) as ctx:
            ctx.agg_configure(N.AGG_BOOSTING_REG_MEDIAN, len(trees), 0, 1, 0, n)
            for i, t in enumerate(trees):
                ctx.tree_predict(t, N.SLOT_P, i)
            ctx.agg_run(self.weights)
            return download_raw(ctx)

    def _aggregate(self, X) -> np.ndarray:
        median = self("votingStrategy").lower() == "median"
        out = self._aggregate_resident(X, median)
        if out is None and (not median or len(self.models) <= N.FOREST_MEDIAN_MAX_TREES):
            out = linear_sum(self.device, X, device_linear(self, self.models), None,
                             N.AGG_BOOSTING_REG_MEDIAN if median else N.AGG_BOOSTING_REG_MEAN, weights=self.weights)
        if out is not None:
            return out
        P = np.ascontiguousarray(np.stack([m.predict(X) for m in self.models]), dtype=np.float32)
        return member_route(self.device, N.AGG_BOOSTING_REG_MEDIAN if median else N.AGG_BOOSTING_REG_MEAN, P,
                            weights=self.weights)

    def transform(self, dataset: DataFrame) -> DataFrame:
        return dataset.withColumn(self("predictionCol"), self._aggregate(np.asarray(dataset[self("featuresCol")])))

    def predict(self, features) -> float:
        return float(self._aggregate(np.asarray(features).reshape(1, -1))[0])


BoostingRegressionModel._declare(_p + _pb + _pbr, _BOOST_REG_DEFAULTS)


# ---- Stacking ------------------------------------------------------------------------------------------------------
class StackingRegressor(Params):
    """regression/StackingRegressor.scala: every base learner fits on the dataset, its predictions become the
    meta-features of each row and the stacker fits on them.  residentFeatures keeps X and the meta-features on the
    device (routes.stacking_fit)."""

    def __init__(self, uid: str | None = None, device: int = 0):
        super().__init__(uid or random_uid("StackingRegressor"))
        self.device = device

    def copy(self, extra=None):
        c = super().copy(extra)
        if c.isDefined("baseLearners"):
            c.set("baseLearners", [m.copy(extra) for m in c("baseLearners")])
        if c.isDefined("stacker"):
            c.set("stacker", c("stacker").copy(extra))
        return c

    def fit(self, dataset: DataFrame) -> "StackingRegressionModel":
        models, stack, widths = stacking_fit(self, dataset)
        m = StackingRegressionModel(models, stack, device=self.device)
        self._copyValues(m)
        m.parent = self
        return m


_pstack = [Param("baseLearners", "base learners that will be used by the ensemble learner", convert=list),
           Param("stacker", "stacker that will be used by the ensemble learner to aggregate results of base learner(s)"),
           Param("parallelism", "the number of threads to use when running parallel algorithms (>= 1)",
                 ParamValidators.gtEq(1), int),
           RESIDENT_FEATURES]
_STACK_REG_DEFAULTS = {**_d, "parallelism": 1, "residentFeatures": False}
StackingRegressor._declare(_p + _pstack, _STACK_REG_DEFAULTS)


class StackingRegressionModel(Params):
    """regression/StackingRegressor.scala StackingRegressionModel: predict = stack.predict(every member's prediction)."""

    def __init__(self, models, stack, uid: str | None = None, device: int = 0):
        super().__init__(uid or random_uid("StackingRegressionModel"))
        self.models, self.stack = list(models), stack
        self.widths = [1] * len(self.models)
        self.device = device
        self.parent = None

    def copy(self, extra=None):
        c = super().copy(extra)
        c.parent = self.parent
        return c

    def _aggregate(self, X) -> np.ndarray:
        return stacking_predict(self, X)

    def transform(self, dataset: DataFrame) -> DataFrame:
        return dataset.withColumn(self("predictionCol"), self._aggregate(np.asarray(dataset[self("featuresCol")])))

    def predict(self, features) -> float:
        return float(self._aggregate(np.asarray(features).reshape(1, -1))[0])


StackingRegressionModel._declare(_p + _pstack, _STACK_REG_DEFAULTS)
