"""Base learners for the host-side mirror.

In the reference the base learner is ANY third-party Spark ML Predictor (ensemble/ensembleParams.scala:
64-81) — its fit/predict are not part of the hot path; only its per-row outputs are the hot path's
inputs.  There is no Spark here, so scikit-learn estimators stand in for Spark's DecisionTree*/Linear*
(also third party).  Fitted trees / linear models expose array forms so the product can evaluate them
ON DEVICE over the column-major feature matrix (se_tree_predict / se_linear_predict).
"""
from __future__ import annotations

import numpy as np


def _floor_f32(t64: np.ndarray) -> np.ndarray:
    """Largest fp32 <= each fp64 value, so `x <= t32` equals `x <= t64` for every fp32 x."""
    t64 = np.asarray(t64, dtype=np.float64)
    t32 = t64.astype(np.float32)
    up = t32.astype(np.float64) > t64
    t32[up] = np.nextafter(t32[up], np.float32(-np.inf))
    return t32


def _tree_arrays(tree) -> dict:
    t = tree.tree_
    leaf = t.children_left < 0
    thr32 = _floor_f32(t.threshold)
    return {
        "feature": np.where(leaf, -1, t.feature).astype(np.int32),
        "threshold": np.where(leaf, 0.0, thr32).astype(np.float32),
        "left": np.maximum(t.children_left, 0).astype(np.int32),
        "right": np.maximum(t.children_right, 0).astype(np.int32),
    }


class _Model:
    def tree_arrays(self):
        return None

    def linear_arrays(self):
        return None


class DecisionTreeRegressionModel(_Model):
    def __init__(self, sk):
        self.sk = sk

    def predict(self, X) -> np.ndarray:
        return self.sk.predict(np.asarray(X, dtype=np.float32)).astype(np.float64)

    def tree_arrays(self):
        d = _tree_arrays(self.sk)
        d["value"] = self.sk.tree_.value.reshape(-1).astype(np.float32)
        return d


class DecisionTreeRegressor:
    """Stand-in for org.apache.spark.ml.regression.DecisionTreeRegressor (maxDepth default 5)."""

    def __init__(self, maxDepth: int = 5, minInstancesPerNode: int = 1, seed: int = 0):
        self.maxDepth, self.minInstancesPerNode, self.seed = maxDepth, minInstancesPerNode, seed

    def copy(self, extra=None):
        return DecisionTreeRegressor(self.maxDepth, self.minInstancesPerNode, self.seed)

    def fit(self, X, y, w=None) -> DecisionTreeRegressionModel:
        from sklearn.tree import DecisionTreeRegressor as SK
        sk = SK(max_depth=self.maxDepth, min_samples_leaf=self.minInstancesPerNode, random_state=self.seed)
        sk.fit(np.asarray(X, dtype=np.float32), np.asarray(y, dtype=np.float64),
               sample_weight=None if w is None else np.asarray(w, dtype=np.float64))
        return DecisionTreeRegressionModel(sk)


def continuous_split_candidates(values, max_bins: int) -> np.ndarray:
    """Spark's findSplitsForContinuousFeature over one column's sample values (DESIGN.md §3 "Device tree fit"): sorted
    distinct non-NaN values v_0 < ... < v_m with counts c_i (-0 counted as +0); every fp64 midpoint when m <= maxBins - 1,
    else the midpoints where the running count passes the next multiple of N_s / maxBins.  Each midpoint is stored as the
    largest fp32 below it; an infinite midpoint (a column holding +-inf) as +-FLT_MAX, so that it still separates the
    infinite value from its finite neighbour and the lists stay finite."""
    v = np.asarray(values, dtype=np.float64).reshape(-1)
    v = v[~np.isnan(v)] + 0.0  # + 0.0 turns -0 into +0
    vals, counts = np.unique(v, return_counts=True)
    m = vals.size - 1
    if m <= 0:
        return np.zeros(0, dtype=np.float32)
    mids = (vals[:-1] + vals[1:]) / 2.0
    if m > max_bins - 1:
        stride = counts.sum() / max_bins
        cum = np.cumsum(counts)
        keep = []
        target = stride
        for i in range(1, m + 1):  # the target moves only when a midpoint is emitted: sequential by nature
            if abs(cum[i - 1] - target) < abs(cum[i] - target):
                keep.append(i - 1)
                target += stride
        mids = mids[np.asarray(keep, dtype=np.int64)]
    fmax = float(np.finfo(np.float32).max)
    out = _floor_f32(np.clip(mids, -fmax, fmax))
    return np.unique(out)  # sorted; clamping can only merge two candidates at the extremes


class DeviceDecisionTreeRegressionModel(_Model):
    """A regression tree fitted on the device, in the array form of se_tree_predict."""

    def __init__(self, arrays: dict):
        self._arrays = {k: np.asarray(v).copy() for k, v in arrays.items()}
        self.numNodes = int(self._arrays["feature"].size)

    def tree_arrays(self):
        return {k: self._arrays[k] for k in ("feature", "threshold", "left", "right", "value")}

    @property
    def gains(self) -> np.ndarray:
        return self._arrays["gain"]

    def predict(self, X) -> np.ndarray:
        """Host walk of the same arrays: left when x <= threshold (NaN goes right), fp32 features and values."""
        X = np.asarray(X, dtype=np.float32)
        f, t = self._arrays["feature"], self._arrays["threshold"]
        l, r, v = self._arrays["left"], self._arrays["right"], self._arrays["value"]
        node = np.zeros(X.shape[0], dtype=np.int64)
        rows = np.arange(X.shape[0])
        while True:
            live = f[node] >= 0
            if not live.any():
                break
            idx = rows[live]
            nd = node[idx]
            go_left = X[idx, f[nd]] <= t[nd]
            node[idx] = np.where(go_left, l[nd], r[nd])
        return v[node].astype(np.float64)


class _DeviceTreeLearner:
    """What the device tree learners share: the tree Params' validators and the split candidates of a fit."""

    device_learner = True

    def _check(self):
        if not 0 <= self.maxDepth <= 8:
            raise ValueError(f"maxDepth must be in [0, 8], got {self.maxDepth}")
        if not 2 <= self.maxBins <= 256:
            raise ValueError(f"maxBins must be in [2, 256], got {self.maxBins}")
        if self.minInstancesPerNode < 1:
            raise ValueError(f"minInstancesPerNode must be >= 1, got {self.minInstancesPerNode}")
        if not 0.0 <= self.minWeightFractionPerNode < 0.5:
            raise ValueError(f"minWeightFractionPerNode must be in [0, 0.5), got {self.minWeightFractionPerNode}")

    def sample_rows(self, n: int):
        """Rows the candidates are drawn from: all of them when n <= max(maxBins², 10000), else Spark's Bernoulli
        sample at fraction max(maxBins², 10000) / n with this learner's seed.  None means every row."""
        required = max(self.maxBins * self.maxBins, 10000)
        if n <= required:
            return None
        import ctypes
        from . import _native as N
        c = np.zeros(n, dtype=np.float32)
        s64 = int(self.seed) & 0xFFFFFFFFFFFFFFFF
        s64 = s64 - (1 << 64) if s64 >= (1 << 63) else s64
        N.check(N.load().se_spark_bernoulli_sample(ctypes.c_int64(s64), required / n, n, 0, N.fptr(c)))
        return np.flatnonzero(c > 0)

    def split_candidates(self, X) -> list:
        """Split candidates of every column of X, computed once per fit from the feature values only."""
        self._check()
        X = np.asarray(X, dtype=np.float32)
        rows = self.sample_rows(X.shape[0])
        S = X if rows is None else X[rows]
        return [continuous_split_candidates(S[:, j], self.maxBins) for j in range(X.shape[1])]


class DeviceDecisionTreeRegressor(_DeviceTreeLearner):
    """org.apache.spark.ml.regression.DecisionTreeRegressor fitted on the GPU: variance impurity, continuous features,
    level-wise best split over at most maxBins - 1 candidates per column (se_tree_fit).  Params keep Spark's names and
    defaults.  Inside GBMRegressor / GBMClassifier (residentFeatures=True) it fits on the device-resident residuals;
    `fit` alone opens a context on `device`, uploads X, fits and closes it."""

    def __init__(self, maxDepth: int = 5, maxBins: int = 32, minInstancesPerNode: int = 1, minInfoGain: float = 0.0,
                 minWeightFractionPerNode: float = 0.0, seed: int | None = None, device: int = 0):
        from .ensemble import java_string_hash
        self.maxDepth, self.maxBins = int(maxDepth), int(maxBins)
        self.minInstancesPerNode, self.minInfoGain = int(minInstancesPerNode), float(minInfoGain)
        self.minWeightFractionPerNode = float(minWeightFractionPerNode)
        self.seed = java_string_hash("org.apache.spark.ml.regression.DecisionTreeRegressor") if seed is None else int(seed)
        self.device = int(device)
        self._check()

    def copy(self, extra=None):
        c = DeviceDecisionTreeRegressor(self.maxDepth, self.maxBins, self.minInstancesPerNode, self.minInfoGain,
                                        self.minWeightFractionPerNode, self.seed, self.device)
        for k, v in (extra or {}).items():
            setattr(c, k, v)
        c._check()
        return c

    def fit_resident(self, ctx, label_slot: int, label_row: int, weight_slot: int, weight_row: int, use_bag: bool,
                     subspace, out_slot: int, out_row: int) -> DeviceDecisionTreeRegressionModel:
        """Fit over a context whose SLOT_X already holds this learner's candidates (Context.tree_fit_bins)."""
        self._check()
        t = ctx.tree_fit(label_slot, label_row, weight_slot, weight_row, use_bag, subspace=subspace,
                         max_depth=self.maxDepth, min_instances=self.minInstancesPerNode,
                         min_info_gain=self.minInfoGain, min_weight_fraction=self.minWeightFractionPerNode,
                         out_slot=out_slot, out_row=out_row)
        return DeviceDecisionTreeRegressionModel(t)

    def fit(self, X, y, w=None) -> DeviceDecisionTreeRegressionModel:
        from . import _native as N
        from .context import Context
        X = np.asarray(X, dtype=np.float32)
        n, d = X.shape
        if n == 0 or d == 0:
            raise ValueError("DeviceDecisionTreeRegressor.fit needs at least one row and one column")
        cands = self.split_candidates(X)
        with Context(self.device) as ctx:
            ctx.alloc(N.SLOT_X, d, n)
            ctx.upload_rowmajor(N.SLOT_X, X)
            ctx.alloc(N.SLOT_Y, n)
            ctx.upload(N.SLOT_Y, np.asarray(y, dtype=np.float32))
            if w is not None:
                ctx.alloc(N.SLOT_W, n)
                ctx.upload(N.SLOT_W, np.asarray(w, dtype=np.float32))
            ctx.alloc(N.SLOT_H, n)
            ctx.tree_fit_bins(cands)
            return self.fit_resident(ctx, N.SLOT_Y, 0, N.SLOT_W if w is not None else -1, 0, False,
                                     np.arange(d, dtype=np.int32), N.SLOT_H, 0)


class DecisionTreeClassificationModel(_Model):
    def __init__(self, sk, num_classes: int):
        self.sk, self.numClasses = sk, num_classes

    def predictProbability(self, X) -> np.ndarray:
        p = self.sk.predict_proba(np.asarray(X, dtype=np.float32))
        out = np.zeros((p.shape[0], self.numClasses))
        out[:, self.sk.classes_.astype(int)] = p
        return out

    def predict(self, X) -> np.ndarray:
        return np.argmax(self.predictProbability(X), axis=1).astype(np.float64)

    def tree_arrays(self):
        """Array form with per-node class-probability vectors ("values" [n_nodes, K]) and the predicted label
        ("value" [n_nodes]) so both predictProbability and predict can be evaluated on device."""
        d = _tree_arrays(self.sk)
        v = self.sk.tree_.value[:, 0, :].astype(np.float64)
        v = v / np.maximum(v.sum(axis=1, keepdims=True), 1e-300)
        full = np.zeros((v.shape[0], self.numClasses))
        full[:, self.sk.classes_.astype(int)] = v
        d["values"] = full.astype(np.float32)
        d["value"] = np.argmax(full, axis=1).astype(np.float32)
        return d


class DecisionTreeClassifier:
    """Stand-in for org.apache.spark.ml.classification.DecisionTreeClassifier."""

    def __init__(self, maxDepth: int = 5, seed: int = 0):
        self.maxDepth, self.seed = maxDepth, seed
        self.numClasses = None

    def copy(self, extra=None):
        return DecisionTreeClassifier(self.maxDepth, self.seed)

    def fit(self, X, y, w=None, num_classes: int | None = None) -> DecisionTreeClassificationModel:
        from sklearn.tree import DecisionTreeClassifier as SK
        sk = SK(max_depth=self.maxDepth, random_state=self.seed)
        yi = np.asarray(y).astype(int)
        sk.fit(np.asarray(X, dtype=np.float32), yi, sample_weight=None if w is None else np.asarray(w, dtype=np.float64))
        return DecisionTreeClassificationModel(sk, int(num_classes or (yi.max() + 1)))


class DeviceDecisionTreeClassificationModel(_Model):
    """A classification tree fitted on the device, in the array form of se_tree_predict ("value": the label) and
    se_tree_predict_multi ("values": [n_nodes, K] class probabilities), as DecisionTreeClassificationModel gives."""

    def __init__(self, arrays: dict, num_classes: int):
        self._arrays = {k: np.asarray(v).copy() for k, v in arrays.items()}
        self.numClasses = int(num_classes)
        self.numNodes = int(self._arrays["feature"].size)

    def tree_arrays(self):
        return {k: self._arrays[k] for k in ("feature", "threshold", "left", "right", "value", "values")}

    @property
    def gains(self) -> np.ndarray:
        return self._arrays["gain"]

    @property
    def class_weights(self) -> np.ndarray:
        return self._arrays["class_weights"]

    def _leaf(self, X) -> np.ndarray:
        """Host walk of the arrays: left when x <= threshold (NaN goes right), fp32 features."""
        X = np.asarray(X, dtype=np.float32)
        f, t = self._arrays["feature"], self._arrays["threshold"]
        l, r = self._arrays["left"], self._arrays["right"]
        node = np.zeros(X.shape[0], dtype=np.int64)
        rows = np.arange(X.shape[0])
        while True:
            live = f[node] >= 0
            if not live.any():
                break
            idx = rows[live]
            nd = node[idx]
            go_left = X[idx, f[nd]] <= t[nd]
            node[idx] = np.where(go_left, l[nd], r[nd])
        return node

    def predict(self, X) -> np.ndarray:
        return self._arrays["value"][self._leaf(X)].astype(np.float64)

    def predictProbability(self, X) -> np.ndarray:
        return self._arrays["values"][self._leaf(X)].astype(np.float64)


class DeviceDecisionTreeClassifier(_DeviceTreeLearner):
    """org.apache.spark.ml.classification.DecisionTreeClassifier fitted on the GPU: gini or entropy impurity,
    continuous features, level-wise best split over at most maxBins - 1 candidates per column, Spark's pruning
    (se_tree_fit_classifier).  Params keep Spark's names and defaults; 2..64 classes.  Inside BoostingClassifier
    (residentFeatures=True) it fits on the device-resident labels and boosting weights; `fit` alone opens a context on
    `device`, uploads X, fits and closes it (BaggingClassifier uses it that way)."""

    def __init__(self, maxDepth: int = 5, maxBins: int = 32, impurity: str = "gini", minInstancesPerNode: int = 1,
                 minInfoGain: float = 0.0, minWeightFractionPerNode: float = 0.0, seed: int | None = None,
                 device: int = 0):
        from .ensemble import java_string_hash
        self.maxDepth, self.maxBins, self.impurity = int(maxDepth), int(maxBins), str(impurity)
        self.minInstancesPerNode, self.minInfoGain = int(minInstancesPerNode), float(minInfoGain)
        self.minWeightFractionPerNode = float(minWeightFractionPerNode)
        self.seed = (java_string_hash("org.apache.spark.ml.classification.DecisionTreeClassifier") if seed is None
                     else int(seed))
        self.device = int(device)
        self._check()

    def _check(self):
        super()._check()
        if self.impurity.lower() not in ("gini", "entropy"):
            raise ValueError(f"impurity must be gini or entropy, got {self.impurity!r}")

    def copy(self, extra=None):
        c = DeviceDecisionTreeClassifier(self.maxDepth, self.maxBins, self.impurity, self.minInstancesPerNode,
                                         self.minInfoGain, self.minWeightFractionPerNode, self.seed, self.device)
        for k, v in (extra or {}).items():
            setattr(c, k, v)
        c._check()
        return c

    @staticmethod
    def _check_classes(K: int):
        if not 2 <= K <= 64:
            raise ValueError(f"the device classification tree supports 2..64 classes, got {K}")

    def fit_resident(self, ctx, num_classes: int, label_slot: int, label_row: int, weight_slot: int, weight_row: int,
                     use_bag: bool, subspace, out_slot: int, out_row: int,
                     proba: bool = False) -> DeviceDecisionTreeClassificationModel:
        """Fit over a context whose SLOT_X already holds this learner's candidates (Context.tree_fit_bins); writes
        every row's label (or, with proba, its K probabilities from row out_row on) into out_slot."""
        self._check()
        self._check_classes(int(num_classes))
        t = ctx.tree_fit_classifier(label_slot, num_classes, label_row, weight_slot, weight_row, use_bag,
                                    subspace=subspace, impurity=self.impurity.lower(), max_depth=self.maxDepth,
                                    min_instances=self.minInstancesPerNode, min_info_gain=self.minInfoGain,
                                    min_weight_fraction=self.minWeightFractionPerNode, proba=proba,
                                    out_slot=out_slot, out_row=out_row)
        return DeviceDecisionTreeClassificationModel(t, num_classes)

    def fit(self, X, y, w=None, num_classes: int | None = None) -> DeviceDecisionTreeClassificationModel:
        from . import _native as N
        from .context import Context
        X = np.asarray(X, dtype=np.float32)
        n, d = X.shape
        if n == 0 or d == 0:
            raise ValueError("DeviceDecisionTreeClassifier.fit needs at least one row and one column")
        y = np.asarray(y, dtype=np.float64).reshape(-1)
        K = int(num_classes) if num_classes is not None else int(y.max()) + 1
        if y.size != n or np.any(y < 0) or np.any(y != np.floor(y)) or np.any(y >= K):
            raise ValueError(f"labels must be integer class indices in [0, {K}) and one per row")
        self._check_classes(K)
        cands = self.split_candidates(X)
        with Context(self.device) as ctx:
            ctx.alloc(N.SLOT_X, d, n)
            ctx.upload_rowmajor(N.SLOT_X, X)
            ctx.alloc(N.SLOT_Y, n)
            ctx.upload(N.SLOT_Y, y.astype(np.float32))
            if w is not None:
                ctx.alloc(N.SLOT_W, n)
                ctx.upload(N.SLOT_W, np.asarray(w, dtype=np.float32))
            ctx.alloc(N.SLOT_PRED, n)
            ctx.tree_fit_bins(cands)
            return self.fit_resident(ctx, K, N.SLOT_Y, 0, N.SLOT_W if w is not None else -1, 0, False,
                                     np.arange(d, dtype=np.int32), N.SLOT_PRED, 0)


class LinearRegressionModel(_Model):
    def __init__(self, coef, intercept):
        self.coefficients = np.asarray(coef, dtype=np.float64)
        self.intercept = float(intercept)

    def predict(self, X) -> np.ndarray:
        return np.asarray(X, dtype=np.float64) @ self.coefficients + self.intercept

    def linear_arrays(self):
        return {"coef": self.coefficients.astype(np.float32), "intercept": np.float32(self.intercept)}


class LinearRegression:
    """Stand-in for org.apache.spark.ml.regression.LinearRegression (ridge via regParam)."""

    def __init__(self, regParam: float = 0.0):
        self.regParam = regParam

    def copy(self, extra=None):
        return LinearRegression(self.regParam)

    def fit(self, X, y, w=None) -> LinearRegressionModel:
        from sklearn.linear_model import Ridge
        sk = Ridge(alpha=max(self.regParam, 1e-12))
        sk.fit(np.asarray(X, dtype=np.float64), np.asarray(y, dtype=np.float64),
               sample_weight=None if w is None else np.asarray(w, dtype=np.float64))
        return LinearRegressionModel(sk.coef_, sk.intercept_)
