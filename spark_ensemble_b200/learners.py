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

    def _forest_subspaces(self, subspaces):
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
    on the device by se_linear_predict.  It is not a resident learner of the GBM, Bagging or Boosting loops: they call
    its `fit`, which opens a context on `device`."""

    def __init__(self, regParam: float = 0.0, device: int = 0):
        self.regParam, self.device = float(regParam), int(device)
        if self.regParam < 0:
            raise ValueError(f"regParam must be >= 0, got {self.regParam}")

    def copy(self, extra=None):
        return DeviceLinearRegression(self.regParam, self.device)

    def fit_resident(self, ctx, src_slot: int, cols, label_slot: int, label_row: int, weight_slot: int,
                     weight_row: int, use_bag: bool, out_slot: int | None, out_row: int = 0,
                     shift=None) -> LinearRegressionModel:
        """Fit over columns `cols` of src_slot in ctx: one se_linear_moments call, then the host solve.  The shifts
        default to the values of row 0 (a few downloads), which keeps the centring well away from cancellation.  With
        out_slot, every row's prediction goes to its row out_row (src_slot must then be SLOT_X)."""
        cols = np.asarray(cols, dtype=np.int32).reshape(-1)
        n = ctx.layout(src_slot)[1]
        if shift is None:
            shift = np.array([ctx.download(src_slot, count=1, offset=int(c) * n)[0] for c in cols], dtype=np.float64)
        label_shift = float(ctx.download(label_slot, count=1, offset=int(label_row) * n)[0])
        M = ctx.linear_moments(src_slot, cols, label_slot, label_row, weight_slot, weight_row, use_bag, shift,
                               label_shift)
        coef, intercept = solve_linear_moments(M, shift, label_shift, self.regParam)
        model = LinearRegressionModel(coef, intercept)
        if out_slot is not None:
            if src_slot != N.SLOT_X:
                raise ValueError("predictions are written from SLOT_X only")
            a = model.linear_arrays()
            ctx.linear_predict(a["coef"], float(a["intercept"]), out_slot, out_row, subspace=cols)
        return model

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
