"""Base learners for the host-side mirror.

In the reference the base learner is ANY third-party Spark ML Predictor (ensemble/ensembleParams.scala:
64-81) — its fit/predict are not part of the hot path; only its per-row outputs are the hot path's
inputs.  There is no Spark here, so scikit-learn estimators stand in for Spark's DecisionTree*/Linear*
(also third party).  Fitted trees / linear models expose array forms so the product can evaluate them
ON DEVICE over the column-major feature matrix (se_tree_predict / se_linear_predict).
"""
from __future__ import annotations

import numpy as np

from . import _native as N
from .context import Context
from .ensemble import java_string_hash, spark_bernoulli_sample


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

    def margin_arrays(self):
        """{coef [D][p], intercept [D] (fp64), threshold}: the form in which se_linear_agg scores a linear or logistic
        member; None for other models."""
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


def distinct_subspaces(subspaces):
    """The distinct subspaces (each fitted once) and, per member, the index of its distinct subspace."""
    keys, first, index = {}, [], []
    for s in subspaces:
        s = np.asarray(s, dtype=np.int32).reshape(-1)
        key = s.tobytes()
        if key not in keys:
            keys[key] = len(first)
            first.append(s)
        index.append(keys[key])
    return first, index


def check_class_labels(y: np.ndarray, num_classes: int, n: int):
    """The device classification tree's labels: n of them, each an integer class index in [0, num_classes)."""
    if y.size != n or np.any(y < 0) or np.any(y != np.floor(y)) or np.any(y >= num_classes):
        raise ValueError(f"labels must be integer class indices in [0, {num_classes}) and one per row")


class _DeviceTreeModel(_Model):
    """A tree fitted on the device, in the array form of se_tree_predict, with the gain of every node."""

    def __init__(self, arrays: dict):
        self._arrays = {k: np.asarray(v).copy() for k, v in arrays.items()}
        self.numNodes = int(self._arrays["feature"].size)

    @property
    def gains(self) -> np.ndarray:
        return self._arrays["gain"]

    def _leaf(self, X) -> np.ndarray:
        """Host walk of the arrays: the leaf of every row, left when x <= threshold (NaN goes right), fp32 features."""
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


class DeviceDecisionTreeRegressionModel(_DeviceTreeModel):
    """A regression tree fitted on the device, in the array form of se_tree_predict."""

    def tree_arrays(self):
        return {k: self._arrays[k] for k in ("feature", "threshold", "left", "right", "value")}

    def predict(self, X) -> np.ndarray:
        return self._arrays["value"][self._leaf(X)].astype(np.float64)


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
        return np.flatnonzero(spark_bernoulli_sample(n, required / n, self.seed) > 0)

    def split_candidates(self, X, rows=None) -> list:
        """Split candidates of every column of X, computed once per fit from the feature values only.  With `rows`
        (row indices), exactly those of X[rows], without copying X[rows]: the candidate sample of len(rows) rows is
        taken through `rows`, so only the sampled rows are gathered."""
        self._check()
        if rows is None:
            X = np.asarray(X, dtype=np.float32)
            sample = self.sample_rows(X.shape[0])
            S = X if sample is None else X[sample]
        else:
            rows = np.asarray(rows, dtype=np.int64).reshape(-1)
            sample = self.sample_rows(rows.size)
            S = np.asarray(X[rows if sample is None else rows[sample]], dtype=np.float32)
        return [continuous_split_candidates(S[:, j], self.maxBins) for j in range(S.shape[1])]

    def _tree_params(self) -> dict:
        """This learner's Params as the keyword arguments of Context.tree_fit / forest_fit."""
        return {"max_depth": self.maxDepth, "min_instances": self.minInstancesPerNode, "min_info_gain": self.minInfoGain,
                "min_weight_fraction": self.minWeightFractionPerNode}

    def _fit_alone(self, X, y, w, out_slot: int, fit):
        """`fit` alone: a context of its own on `device` holding X (fp32, checked by _rows), the labels y (fp32) in
        SLOT_Y, the weights w (if any) in SLOT_W, out_slot for every row's output and this learner's candidates;
        fit(ctx, weight_slot, columns) fits over it, and the context is closed."""
        n, d = X.shape
        cands = self.split_candidates(X)
        with Context(self.device) as ctx:
            ctx.alloc(N.SLOT_X, d, n)
            ctx.upload_rowmajor(N.SLOT_X, X)
            ctx.alloc(N.SLOT_Y, n)
            ctx.upload(N.SLOT_Y, y)
            if w is not None:
                ctx.alloc(N.SLOT_W, n)
                ctx.upload(N.SLOT_W, np.asarray(w, dtype=np.float32))
            ctx.alloc(out_slot, n)
            ctx.tree_fit_bins(cands)
            return fit(ctx, N.SLOT_W if w is not None else -1, np.arange(d, dtype=np.int32))

    def _rows(self, X) -> np.ndarray:
        X = np.asarray(X, dtype=np.float32)
        if X.shape[0] == 0 or X.shape[1] == 0:
            raise ValueError(f"{type(self).__name__}.fit needs at least one row and one column")
        return X

    _forest_subspaces = staticmethod(distinct_subspaces)


class DeviceDecisionTreeRegressor(_DeviceTreeLearner):
    """org.apache.spark.ml.regression.DecisionTreeRegressor fitted on the GPU: variance impurity, continuous features,
    level-wise best split over at most maxBins - 1 candidates per column (se_tree_fit).  Params keep Spark's names and
    defaults.  Inside GBMRegressor / GBMClassifier (residentFeatures=True) it fits on the device-resident residuals,
    inside BaggingRegressor (residentFeatures=True) every member's tree grows in one forest fit
    (fit_forest_resident); `fit` alone opens a context on `device`, uploads X, fits and closes it."""

    def __init__(self, maxDepth: int = 5, maxBins: int = 32, minInstancesPerNode: int = 1, minInfoGain: float = 0.0,
                 minWeightFractionPerNode: float = 0.0, seed: int | None = None, device: int = 0):
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
                         out_slot=out_slot, out_row=out_row, **self._tree_params())
        return DeviceDecisionTreeRegressionModel(t)

    def fit_forest_resident(self, ctx, label_slot: int, label_row: int, weight_slot: int, weight_row: int,
                            use_bag: bool, subspaces) -> list:
        """One tree per subspace over the same labels, weights and bag of a context whose SLOT_X holds this learner's
        candidates, fitted together (Context.forest_fit).  Equal subspaces are fitted once: their trees would be
        fits of the same data.  Returns one model per subspace, with subspace-local features."""
        self._check()
        distinct, index = self._forest_subspaces(subspaces)
        trees = ctx.forest_fit(distinct, label_slot, label_row, weight_slot, weight_row, use_bag, **self._tree_params())
        return [DeviceDecisionTreeRegressionModel(trees[i]) for i in index]

    def fit(self, X, y, w=None) -> DeviceDecisionTreeRegressionModel:
        return self._fit_alone(self._rows(X), np.asarray(y, dtype=np.float32), w, N.SLOT_H,
                               lambda ctx, wslot, cols: self.fit_resident(ctx, N.SLOT_Y, 0, wslot, 0, False, cols,
                                                                          N.SLOT_H, 0))


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

    def node_raw(self) -> np.ndarray:
        """[n_nodes, numClasses] weighted class counts of every node: Spark's rawPrediction of a leaf."""
        t = self.sk.tree_
        v = t.value[:, 0, :].astype(np.float64)
        v = v / np.maximum(v.sum(axis=1, keepdims=True), 1e-300) * t.weighted_n_node_samples[:, None]
        full = np.zeros((v.shape[0], self.numClasses))
        full[:, self.sk.classes_.astype(int)] = v
        return full

    def predictRaw(self, X) -> np.ndarray:
        return self.node_raw()[self.sk.apply(np.asarray(X, dtype=np.float32))]

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


class DeviceDecisionTreeClassificationModel(_DeviceTreeModel):
    """A classification tree fitted on the device, in the array form of se_tree_predict ("value": the label) and
    se_tree_predict_multi ("values": [n_nodes, K] class probabilities), as DecisionTreeClassificationModel gives."""

    def __init__(self, arrays: dict, num_classes: int):
        super().__init__(arrays)
        self.numClasses = int(num_classes)

    def tree_arrays(self):
        return {k: self._arrays[k] for k in ("feature", "threshold", "left", "right", "value", "values")}

    @property
    def class_weights(self) -> np.ndarray:
        return self._arrays["class_weights"]

    def predict(self, X) -> np.ndarray:
        return self._arrays["value"][self._leaf(X)].astype(np.float64)

    def predictProbability(self, X) -> np.ndarray:
        return self._arrays["values"][self._leaf(X)].astype(np.float64)

    def node_raw(self) -> np.ndarray:
        """[n_nodes, numClasses] class weights of every node: Spark's rawPrediction of a leaf."""
        return self.class_weights

    def predictRaw(self, X) -> np.ndarray:
        return self.class_weights[self._leaf(X)]


class DeviceDecisionTreeClassifier(_DeviceTreeLearner):
    """org.apache.spark.ml.classification.DecisionTreeClassifier fitted on the GPU: gini or entropy impurity,
    continuous features, level-wise best split over at most maxBins - 1 candidates per column, Spark's pruning
    (se_tree_fit_classifier).  Params keep Spark's names and defaults; 2..64 classes.  Inside BoostingClassifier
    (residentFeatures=True) it fits on the device-resident labels and boosting weights, and inside BaggingClassifier
    (residentFeatures=True) every member's tree grows in one forest fit (fit_forest_resident); `fit` alone opens a
    context on `device`, uploads X, fits and closes it (BaggingClassifier without residentFeatures uses it that way)."""

    def __init__(self, maxDepth: int = 5, maxBins: int = 32, impurity: str = "gini", minInstancesPerNode: int = 1,
                 minInfoGain: float = 0.0, minWeightFractionPerNode: float = 0.0, seed: int | None = None,
                 device: int = 0):
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

    def _tree_params(self) -> dict:
        return {**super()._tree_params(), "impurity": self.impurity.lower()}

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
                                    subspace=subspace, proba=proba, out_slot=out_slot, out_row=out_row,
                                    **self._tree_params())
        return DeviceDecisionTreeClassificationModel(t, num_classes)

    def fit_forest_resident(self, ctx, num_classes: int, label_slot: int, label_row: int, weight_slot: int,
                            weight_row: int, use_bag: bool, subspaces) -> list:
        """One tree per subspace over the same labels, weights and bag of a context whose SLOT_X holds this learner's
        candidates, fitted together (Context.forest_fit).  Equal subspaces are fitted once: their trees would be
        fits of the same data.  Returns one model per subspace, with subspace-local features."""
        self._check()
        self._check_classes(int(num_classes))
        distinct, index = self._forest_subspaces(subspaces)
        trees = ctx.forest_fit(distinct, label_slot, label_row, weight_slot, weight_row, use_bag,
                               num_classes=int(num_classes), **self._tree_params())
        return [DeviceDecisionTreeClassificationModel(trees[i], num_classes) for i in index]

    def fit(self, X, y, w=None, num_classes: int | None = None) -> DeviceDecisionTreeClassificationModel:
        X = self._rows(X)
        y = np.asarray(y, dtype=np.float64).reshape(-1)
        K = int(num_classes) if num_classes is not None else int(y.max()) + 1
        check_class_labels(y, K, X.shape[0])
        self._check_classes(K)
        return self._fit_alone(X, y.astype(np.float32), w, N.SLOT_PRED,
                               lambda ctx, wslot, cols: self.fit_resident(ctx, K, N.SLOT_Y, 0, wslot, 0, False, cols,
                                                                          N.SLOT_PRED, 0))


class LinearRegressionModel(_Model):
    def __init__(self, coef, intercept):
        self.coefficients = np.asarray(coef, dtype=np.float64)
        self.intercept = float(intercept)

    def predict(self, X) -> np.ndarray:
        return np.asarray(X, dtype=np.float64) @ self.coefficients + self.intercept

    def linear_arrays(self):
        return {"coef": self.coefficients.astype(np.float32), "intercept": np.float32(self.intercept)}

    def margin_arrays(self):
        return {"coef": self.coefficients.reshape(1, -1), "intercept": np.array([self.intercept]), "threshold": 0.5}


def solve_linear_moments(M, shift, label_shift: float, reg_param: float = 0.0):
    """(coefficients, intercept) minimising Σ w·(y − xβ − b)² + α‖β‖², α = max(reg_param, 1e-12), b unpenalised, from the
    moment matrix M of se_linear_moments (z = (x − shift, 1, y − label_shift)): the centred normal equations in fp64,
    by Cholesky, or by a least-squares solve when they are singular to working precision (collinear columns)."""
    from scipy.linalg import LinAlgError, cho_factor, cho_solve
    M = np.asarray(M, dtype=np.float64)
    p = M.shape[0] - 2
    sw = M[p, p]
    if not sw > 0:
        raise ValueError("the linear fit needs a positive total weight")
    sx, sy = M[:p, p], M[p + 1, p]
    A = M[:p, :p] - np.outer(sx, sx) / sw
    b = M[:p, p + 1] - sx * (sy / sw)
    A[np.diag_indices(p)] += max(float(reg_param), 1e-12)
    try:
        beta = cho_solve(cho_factor(A, lower=True, check_finite=True), b) if p else np.zeros(0)
    except LinAlgError:
        beta = np.linalg.lstsq(A, b, rcond=None)[0]
    shift = np.zeros(p) if shift is None else np.asarray(shift, dtype=np.float64)
    intercept = (label_shift + sy / sw) - float((shift + sx / sw) @ beta)
    return beta, intercept


class DeviceLinearRegression:
    """org.apache.spark.ml.regression.LinearRegression fitted on the GPU, with the objective of the host stand-in
    LinearRegression:

        minimise Σ w·(y − xβ − b)² + α‖β‖², with α = max(regParam, 1e-12) and b unpenalised

    which, with the default regParam = 0, is Spark's default (least squares with an intercept) on full-rank data.  One
    pass over the resident columns forms the fp64 moment matrix of (x − s, 1, y − s_y) (se_linear_moments); the host
    solves its (p+1)-sized centred normal equations (solve_linear_moments).  Its model is LinearRegressionModel, scored
    on the device by se_linear_predict.  With residentFeatures the GBM, Bagging and Boosting loops fit it where their data
    live: GBM on the round's residuals (fit_resident), Boosting on the boosting weights (weight_scale = 1 / sumWeights),
    Bagging every member from one moment pass over the union of their columns (fit_members_resident).  Without it
    they call `fit`, which opens a context on `device`."""

    def __init__(self, regParam: float = 0.0, device: int = 0):
        self.regParam, self.device = float(regParam), int(device)
        if self.regParam < 0:
            raise ValueError(f"regParam must be >= 0, got {self.regParam}")

    def copy(self, extra=None):
        return DeviceLinearRegression(self.regParam, self.device)

    def fit_resident(self, ctx, src_slot: int, cols, label_slot: int, label_row: int, weight_slot: int,
                     weight_row: int, use_bag: bool, out_slot: int | None, out_row: int = 0,
                     shift=None, weight_scale: float = 1.0) -> LinearRegressionModel:
        """Fit over columns `cols` of src_slot in ctx: one se_linear_moments call, then the host solve.  The shifts
        default to the values of row 0 (a few downloads), which keeps the centring well away from cancellation.  The
        weights are multiplied by weight_scale (the moments are linear in them): with regParam > 0 the objective
        depends on their scale.  With out_slot, every row's prediction goes to its row out_row (src_slot must then be
        SLOT_X)."""
        cols = np.asarray(cols, dtype=np.int32).reshape(-1)
        n = ctx.layout(src_slot)[1]
        if shift is None:
            shift = np.array([ctx.download(src_slot, count=1, offset=int(c) * n)[0] for c in cols], dtype=np.float64)
        label_shift = float(ctx.download(label_slot, count=1, offset=int(label_row) * n)[0])
        M = ctx.linear_moments(src_slot, cols, label_slot, label_row, weight_slot, weight_row, use_bag, shift,
                               label_shift)
        if weight_scale != 1.0:
            M = M * float(weight_scale)
        coef, intercept = solve_linear_moments(M, shift, label_shift, self.regParam)
        model = LinearRegressionModel(coef, intercept)
        if out_slot is not None:
            if src_slot != N.SLOT_X:
                raise ValueError("predictions are written from SLOT_X only")
            a = model.linear_arrays()
            ctx.linear_predict(a["coef"], float(a["intercept"]), out_slot, out_row, subspace=cols)
        return model

    def fit_members_resident(self, ctx, subspaces, label_slot: int, label_row: int, weight_slot: int, weight_row: int,
                             shift, label_shift: float) -> list:
        """One model per subspace over columns of SLOT_X, the same labels and weights: one se_linear_moments pass per
        group of subspaces whose union holds at most 254 columns, each member's matrix sliced out of it (a moment of
        two columns does not depend on the others).  shift holds one value per column of SLOT_X."""
        shift = np.asarray(shift, dtype=np.float64).reshape(-1)
        subs = [np.asarray(c, dtype=np.int32).reshape(-1) for c in subspaces]
        models = [None] * len(subs)
        for group in column_groups(subs, N.LINEAR_MOMENTS_MAX_COLS):
            U = np.unique(np.concatenate([subs[i] for i in group])).astype(np.int32)
            M = ctx.linear_moments(N.SLOT_X, U, label_slot, label_row, weight_slot, weight_row, False, shift[U],
                                   label_shift)
            for i in group:
                idx = np.concatenate([np.searchsorted(U, subs[i]), [U.size, U.size + 1]])
                coef, b = solve_linear_moments(M[np.ix_(idx, idx)], shift[subs[i]], label_shift, self.regParam)
                models[i] = LinearRegressionModel(coef, b)
        return models

    def fit(self, X, y, w=None) -> LinearRegressionModel:
        X = np.asarray(X, dtype=np.float32)
        n, d = X.shape
        if n == 0:
            raise ValueError("DeviceLinearRegression.fit needs at least one row")
        with Context(self.device) as ctx:
            ctx.alloc(N.SLOT_X, d, n)
            ctx.upload_rowmajor(N.SLOT_X, X)
            ctx.alloc(N.SLOT_Y, n)
            ctx.upload(N.SLOT_Y, np.asarray(y, dtype=np.float32))
            if w is not None:
                ctx.alloc(N.SLOT_W, n)
                ctx.upload(N.SLOT_W, np.asarray(w, dtype=np.float32))
            return self.fit_resident(ctx, N.SLOT_X, np.arange(d, dtype=np.int32), N.SLOT_Y, 0,
                                     N.SLOT_W if w is not None else -1, 0, False, None,
                                     shift=X.mean(axis=0, dtype=np.float64))


class LogisticRegressionModel(_Model):
    """org.apache.spark.ml.classification.LogisticRegressionModel: coefficientMatrix [D][p] and interceptVector [D] in
    raw feature space, D = 1 (binomial: the margin of class 1) or numClasses (multinomial).  Host scoring is fp64;
    write_rows scores on the device over SLOT_X (se_logistic_predict)."""

    def __init__(self, coef, intercept, num_classes: int, multinomial: bool, threshold: float = 0.5,
                 objective_history=(), num_evaluations: int = 0):
        self.coefficientMatrix = np.atleast_2d(np.asarray(coef, dtype=np.float64))
        self.interceptVector = np.atleast_1d(np.asarray(intercept, dtype=np.float64))
        self.numClasses, self.isMultinomial = int(num_classes), bool(multinomial)
        self.threshold = float(threshold)
        self.objectiveHistory = list(objective_history)
        self.numEvaluations = int(num_evaluations)

    @property
    def coefficients(self) -> np.ndarray:
        if self.isMultinomial:
            raise ValueError("a multinomial model has a coefficient matrix: use coefficientMatrix")
        return self.coefficientMatrix[0]

    @property
    def intercept(self) -> float:
        if self.isMultinomial:
            raise ValueError("a multinomial model has an intercept vector: use interceptVector")
        return float(self.interceptVector[0])

    def _margins(self, X) -> np.ndarray:
        return np.asarray(X, dtype=np.float64) @ self.coefficientMatrix.T + self.interceptVector

    def predictRaw(self, X) -> np.ndarray:
        m = self._margins(X)
        return np.concatenate([-m, m], axis=1) if not self.isMultinomial else m

    def predictProbability(self, X) -> np.ndarray:
        m = self._margins(X)
        if not self.isMultinomial:
            p1 = 1.0 / (1.0 + np.exp(-m[:, 0]))
            return np.stack([1.0 - p1, p1], axis=1)
        mx = m.max(axis=1, keepdims=True)
        inf = np.isposinf(mx[:, 0])
        with np.errstate(invalid="ignore"):
            e = np.exp(m - mx)
            p = e / e.sum(axis=1, keepdims=True)
        p[inf] = np.isposinf(m[inf]).astype(np.float64)  # raw2probabilityInPlace: 1 for every +inf class
        return p

    def predict(self, X) -> np.ndarray:
        if not self.isMultinomial:
            return (self.predictProbability(X)[:, 1] > self.threshold).astype(np.float64)
        return np.argmax(self._margins(X), axis=1).astype(np.float64)

    def margin_arrays(self):
        return {"coef": self.coefficientMatrix, "intercept": self.interceptVector, "threshold": self.threshold}

    def write_rows(self, ctx, method: str, out_slot: int, out_row: int, subspace=None) -> bool:
        """Every row's label ("class"), raw vector ("raw") or probabilities ("proba") over the context's SLOT_X into
        out_slot from row out_row (se_logistic_predict); column j of the model is column subspace[j] of X (None: j)."""
        kind = {"class": "label", "raw": "raw", "proba": "prob"}[method]
        ctx.logistic_predict(self.coefficientMatrix, self.interceptVector, self.threshold,
                             subspace=subspace, **{kind: (out_slot, out_row)})
        return True


class DeviceLogisticRegression:
    """org.apache.spark.ml.classification.LogisticRegression fitted on the GPU, with Spark's Params, defaults and
    objective (λ = regParam, α = elasticNetParam, t_j = σ_j with standardization, else 1):

        f = (1/Σc)·Σ c·ℓ + λ·[(1−α)/2·Σ_{k,j} (t_j·β_kj)² + α·Σ_{k,j} t_j·|β_kj|], intercepts unpenalised

    One pass over the resident columns gives the weighted means, Spark's unbiased weighted σ_j, the class histogram and
    the input checks (se_logistic_stats).  The fit then runs in Spark's standardised space, θ_kj = σ_j·β_kj over
    z_j = (x_j − μ_j)/σ_j (μ = 0 without fitIntercept; a column with σ_j = 0 keeps β_kj = 0), and every loss and
    gradient evaluation is one pass over the columns (se_logistic_loss_grad).  Breeze's L-BFGS / OWL-QN are third
    party: SciPy's L-BFGS-B (m = 10) stands in, with the L1 part written exactly as split variables θ = θ⁺ − θ⁻,
    θ± >= 0.  Its iterates differ from Breeze's; the optimum is the same.  Post-processing as Spark: multinomial
    coefficients centred across classes when regParam = 0, multinomial intercepts always centred, and with fitIntercept
    a single present class gives zero coefficients and an infinite intercept without any evaluation.

    With residentFeatures, Boosting fits it on the labels and boosting weights where they live (fit_resident: the
    objective is divided by Σc, so the 1 / sumWeights scale does not change it), and Bagging fits every member in one
    context, their L-BFGS runs in lock step so that one se_logistic_loss_grad_batch call serves every member's
    evaluation (fit_members_resident).  Without it they call `fit`, which opens a context on `device`."""

    def __init__(self, regParam: float = 0.0, elasticNetParam: float = 0.0, maxIter: int = 100, tol: float = 1e-6,
                 fitIntercept: bool = True, standardization: bool = True, family: str = "auto",
                 threshold: float = 0.5, device: int = 0):
        self.regParam, self.elasticNetParam = float(regParam), float(elasticNetParam)
        self.maxIter, self.tol = int(maxIter), float(tol)
        self.fitIntercept, self.standardization = bool(fitIntercept), bool(standardization)
        self.family, self.threshold, self.device = str(family), float(threshold), int(device)
        self._check()

    def _check(self):
        if not self.regParam >= 0:
            raise ValueError(f"regParam must be >= 0, got {self.regParam}")
        if not 0.0 <= self.elasticNetParam <= 1.0:
            raise ValueError(f"elasticNetParam must be in [0, 1], got {self.elasticNetParam}")
        if self.maxIter < 0:
            raise ValueError(f"maxIter must be >= 0, got {self.maxIter}")
        if not self.tol >= 0:
            raise ValueError(f"tol must be >= 0, got {self.tol}")
        if self.family.lower() not in ("auto", "binomial", "multinomial"):
            raise ValueError(f"family must be auto, binomial or multinomial, got {self.family!r}")
        if not 0.0 <= self.threshold <= 1.0:
            raise ValueError(f"threshold must be in [0, 1], got {self.threshold}")

    def copy(self, extra=None):
        c = DeviceLogisticRegression(self.regParam, self.elasticNetParam, self.maxIter, self.tol, self.fitIntercept,
                                     self.standardization, self.family, self.threshold, self.device)
        for k, v in (extra or {}).items():
            setattr(c, k, v)
        c._check()
        return c

    def _multinomial(self, K: int) -> bool:
        fam = self.family.lower()
        if fam == "binomial" and K > 2:
            raise ValueError(f"binomial family only supports 1 or 2 outcome classes but found {K}")
        return fam == "multinomial" or (fam == "auto" and K > 2)

    def optimize(self, evaluate, stats, shift, num_classes: int) -> LogisticRegressionModel:
        """The fit from the statistics pass `stats` (se_logistic_stats's layout, over columns shifted by `shift`) and
        evaluate(shift, scale, coef [D][p+1]) -> (Σ c·ℓ, gradient [D][p+1]) (se_logistic_loss_grad's contract)."""
        from scipy.optimize import fmin_l_bfgs_b
        self._check()
        K = int(num_classes)
        if not 1 <= K <= N.LOGISTIC_MAX_CLASSES:
            raise ValueError(f"the device logistic fit supports 1..{N.LOGISTIC_MAX_CLASSES} classes, got {K}")
        multi = self._multinomial(K)
        st = np.asarray(stats, dtype=np.float64)
        p = (st.size - 3 - K) // 2
        if st[-1] > 0:
            raise ValueError(f"{int(st[-1])} rows have a label outside the integers 0..{K - 1}, a negative or "
                             f"non-finite weight, or a non-finite feature")
        sw, sw2 = st[0], st[1]
        if not sw > 0:
            raise ValueError("the logistic fit needs a positive total weight")
        s = np.zeros(p) if shift is None else np.asarray(shift, dtype=np.float64).reshape(-1)
        d1, d2, hist = st[2:2 + p], st[2 + p:2 + 2 * p], st[2 + 2 * p:2 + 2 * p + K]
        mean = s + d1 / sw
        denom = sw - sw2 / sw
        var = np.maximum(d2 - d1 * d1 / sw, 0.0) / denom if denom > 0 else np.zeros(p)
        sigma = np.sqrt(var)
        live = sigma > 0
        inv = np.where(live, 1.0 / np.where(live, sigma, 1.0), 0.0)
        D = K if multi else 1
        hist_mask = hist != 0
        if self.fitIntercept and hist_mask.sum() == 1:  # a single class present: Spark's constant-label model
            c = int(np.argmax(hist_mask))
            b = np.zeros(D)
            if multi:
                b[c] = np.inf
            else:
                b[0] = np.inf if c == 1 else -np.inf
            return LogisticRegressionModel(np.zeros((D, p)), b, K, multi, self.threshold, [], 0)
        kshift = mean if self.fitIntercept else np.zeros(p)
        lam, alpha = self.regParam, self.elasticNetParam
        q2 = np.ones(p) if self.standardization else inv * inv
        q1 = np.ones(p) if self.standardization else inv
        l2, l1 = lam * (1.0 - alpha), lam * alpha
        split = l1 > 0
        nt, nb = D * p, (D if self.fitIntercept else 0)
        b0 = np.zeros(D)
        if self.fitIntercept:
            if multi:
                r = np.log1p(hist)
                b0 = r - r.mean()
            elif hist[0] > 0 and hist[1] > 0:
                b0[0] = np.log(hist[1] / hist[0])
        evals, history, last = [0], [], [np.nan]

        def unpack(x):
            th = (x[:nt] - x[nt:2 * nt]) if split else x[:nt]
            b = x[(2 if split else 1) * nt:] if nb else np.zeros(D)
            return th.reshape(D, p), b

        def fun(x):
            th, b = unpack(x)
            loss, g = evaluate(kshift, inv, np.concatenate([th, b[:, None]], axis=1))
            evals[0] += 1
            g = np.asarray(g, dtype=np.float64).reshape(D, p + 1) / sw
            gt = g[:, :p] + l2 * q2 * th
            f = loss / sw + 0.5 * l2 * float(np.sum(q2 * th * th))
            parts = [gt.reshape(-1)]
            if split:
                f += l1 * float(np.sum(q1 * (x[:nt] + x[nt:2 * nt]).reshape(D, p)))
                parts = [(gt + l1 * q1).reshape(-1), (-gt + l1 * q1).reshape(-1)]
            if nb:
                parts.append(g[:, p])
            last[0] = f
            return f, np.concatenate(parts)

        x0 = np.concatenate([np.zeros(nt * (2 if split else 1)), b0[:nb]])
        bounds = [(0.0, None)] * (2 * nt) + [(None, None)] * nb if split else None
        history.append(fun(x0)[0])
        x, _, _ = fmin_l_bfgs_b(fun, x0, bounds=bounds, m=10, pgtol=self.tol,
                                factr=max(self.tol / np.finfo(float).eps, 1.0), maxiter=self.maxIter,
                                callback=lambda xk: history.append(last[0]))
        th, b = unpack(x)
        th, b = th.copy(), b.copy()
        if multi and lam == 0.0:
            th -= th.mean(axis=0, keepdims=True)
        if multi and self.fitIntercept:
            b -= b.mean()
        beta = th * inv
        intercept = (b - beta @ kshift) if self.fitIntercept else np.zeros(D)
        return LogisticRegressionModel(beta, intercept, K, multi, self.threshold, history, evals[0])

    def fit_resident(self, ctx, src_slot: int, cols, num_classes: int, label_slot: int, label_row: int,
                     weight_slot: int, weight_row: int, out_slot: int | None = None, out_row: int = 0,
                     method: str = "class", shift=None) -> LogisticRegressionModel:
        """Fit over columns `cols` of src_slot in ctx: one se_logistic_stats pass, then one se_logistic_loss_grad call
        per evaluation.  The stats shifts default to the values of row 0 (a few downloads).  With out_slot, every row's
        label, raw vector or probabilities (method "class", "raw", "proba") go to out_slot from row out_row (src_slot
        must then be SLOT_X)."""
        cols = np.asarray(cols, dtype=np.int32).reshape(-1)
        if cols.size > N.LOGISTIC_MAX_COLS:
            raise ValueError(f"the device logistic fit supports up to {N.LOGISTIC_MAX_COLS} columns, got {cols.size}")
        if out_slot is not None and src_slot != N.SLOT_X:
            raise ValueError("outputs are written from SLOT_X only")
        n = ctx.layout(src_slot)[1]
        if shift is None:
            shift = np.array([ctx.download(src_slot, count=1, offset=int(c) * n)[0] for c in cols], dtype=np.float64)
        st = ctx.logistic_stats(src_slot, cols, num_classes, label_slot, label_row, weight_slot, weight_row, shift)

        def evaluate(kshift, scale, coef):
            return ctx.logistic_loss_grad(src_slot, cols, coef, label_slot, label_row, weight_slot, weight_row,
                                          kshift, scale)
        model = self.optimize(evaluate, st, shift, num_classes)
        if out_slot is not None:
            model.write_rows(ctx, method, out_slot, out_row, subspace=cols)
        return model

    def fit_members_resident(self, ctx, subspaces, num_classes: int, label_slot: int, label_row: int,
                             weight_slot: int, weight_row: int, shifts) -> list:
        """One model per subspace over columns of SLOT_X, the same labels and weights: one se_logistic_stats pass per
        member (shifts: one array per member), then every member's optimize in lock step (lockstep), each evaluation
        round one se_logistic_loss_grad_batch call over the live members.  A member's fit is the one fit_resident
        gives over its columns, since its bits do not depend on the other members of a batch."""
        self._check()
        subs = [np.asarray(c, dtype=np.int32).reshape(-1) for c in subspaces]
        for c in subs:
            if c.size > N.LOGISTIC_MAX_COLS:
                raise ValueError(f"the device logistic fit supports up to {N.LOGISTIC_MAX_COLS} columns, got {c.size}")
        stats = [ctx.logistic_stats(N.SLOT_X, c, num_classes, label_slot, label_row, weight_slot, weight_row, s)
                 for c, s in zip(subs, shifts)]

        def evaluate_batch(requests):
            out = []
            for k in range(0, len(requests), N.LOGISTIC_MAX_BATCH):
                out += ctx.logistic_loss_grad_batch(
                    N.SLOT_X, [(subs[i], coef, kshift, scale) for i, kshift, scale, coef in
                               requests[k:k + N.LOGISTIC_MAX_BATCH]],
                    label_slot, label_row, weight_slot, weight_row)
            return out

        jobs = [lambda evaluate, st=st, s=s: self.optimize(evaluate, st, s, num_classes) for st, s in zip(stats, shifts)]
        return lockstep(jobs, evaluate_batch)

    def fit(self, X, y, w=None, num_classes: int | None = None) -> LogisticRegressionModel:
        X = np.asarray(X, dtype=np.float32)
        n, d = X.shape
        if n == 0:
            raise ValueError("DeviceLogisticRegression.fit needs at least one row")
        y = np.asarray(y, dtype=np.float64).reshape(-1)
        K = int(num_classes) if num_classes is not None else int(np.nanmax(y)) + 1
        with Context(self.device) as ctx:
            ctx.alloc(N.SLOT_X, d, n)
            ctx.upload_rowmajor(N.SLOT_X, X)
            ctx.alloc(N.SLOT_Y, n)
            ctx.upload(N.SLOT_Y, y.astype(np.float32))
            if w is not None:
                ctx.alloc(N.SLOT_W, n)
                ctx.upload(N.SLOT_W, np.asarray(w, dtype=np.float32))
            # row 0's values, the shifts fit_resident downloads by default: a fit over the same resident data in
            # another context (a stacker fitted in the stacking context) follows the same path to the same bits
            return self.fit_resident(ctx, N.SLOT_X, np.arange(d, dtype=np.int32), K, N.SLOT_Y, 0,
                                     N.SLOT_W if w is not None else -1, 0, shift=X[0].astype(np.float64))


def column_groups(subspaces, max_cols: int) -> list:
    """Indices of subspaces in consecutive groups whose union of columns holds at most max_cols columns (a subspace
    with more than max_cols distinct columns makes a group of its own)."""
    groups, cur, union = [], [], set()
    for i, c in enumerate(subspaces):
        u = union | {int(v) for v in c}
        if cur and len(u) > max_cols:
            groups.append(cur)
            cur, u = [], {int(v) for v in c}
        cur.append(i)
        union = u
    if cur:
        groups.append(cur)
    return groups


class _Stop(Exception):
    """Raised in a lock-step job's evaluate once another job or the batch evaluation has failed."""


def lockstep(jobs, evaluate_batch) -> list:
    """Runs jobs (job(evaluate) -> result, e.g. a member's DeviceLogisticRegression.optimize) in lock step, one thread
    each.  A job's evaluate(kshift, scale, coef) posts its request and waits; once every job still running has posted,
    evaluate_batch([(job index, kshift, scale, coef), ...]) (in job order) answers all of them with one list of
    (loss, gradient).  A job that returns leaves the batch.  An exception in a job or in evaluate_batch stops every
    other job at its next evaluation and is raised here (the lowest job's, evaluate_batch's first) once all threads
    have ended.  evaluate_batch runs on the calling thread, so a context is only used from the thread that owns it.
    As long as evaluate_batch answers a request independently of the rest of its batch, each job's result is the one
    it gets alone."""
    import threading
    cond = threading.Condition()
    live = set(range(len(jobs)))
    posted, answers, errors = {}, {}, {}
    results = [None] * len(jobs)
    stop = [False]

    def evaluate_of(i):
        def evaluate(kshift, scale, coef):
            with cond:
                if stop[0]:
                    raise _Stop()
                posted[i] = (kshift, scale, coef)
                cond.notify_all()
                while i not in answers and not stop[0]:
                    cond.wait()
                if i not in answers:
                    raise _Stop()
                return answers.pop(i)
        return evaluate

    def run(i):
        try:
            r = jobs[i](evaluate_of(i))
            with cond:
                results[i] = r
        except _Stop:
            pass
        except BaseException as e:  # noqa: BLE001 - handed to the caller below
            with cond:
                errors[i] = e
                stop[0] = True
        finally:
            with cond:
                live.discard(i)
                cond.notify_all()

    threads = [threading.Thread(target=run, args=(i,), daemon=True) for i in range(len(jobs))]
    for t in threads:
        t.start()
    try:
        while True:
            with cond:
                while not stop[0] and live and len(posted) < len(live):
                    cond.wait()
                if stop[0] or not live:
                    break
                batch = sorted(posted.items())
                posted.clear()
            try:
                out = evaluate_batch([(i,) + req for i, req in batch])
            except BaseException as e:  # noqa: BLE001
                with cond:
                    errors[-1] = e
                    stop[0] = True
                    cond.notify_all()
                break
            with cond:
                for (i, _), r in zip(batch, out):
                    answers[i] = r
                cond.notify_all()
    finally:
        with cond:
            stop[0] = stop[0] or bool(live)
            cond.notify_all()
        for t in threads:
            t.join()
    if errors:
        raise errors[min(errors)]
    return results


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
