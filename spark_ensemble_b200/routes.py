"""What the estimator mirrors (regression, classification) share: their instances and bags, the choice of the device
fit, the set-up of a Bagging or Boosting fit, and the two routes by which a model scores its members:

- one pass over the device-resident features when every member is a tree (se_forest_predict / se_forest_median /
  se_forest_agg), which returns None when the forest's thresholds do not fit the rank matrix;
- the member route: every member's output stacked on the host, uploaded as SLOT_P and aggregated on the device
  (se_agg_run).

Each decision lives here once, so the estimators that make it differently make that visible at their call sites.
"""
from __future__ import annotations

import numpy as np

from . import _native as N
from .context import Context
from .ensemble import DataFrame, spark_bernoulli_sample, subspace
from .learners import check_class_labels
from .params import Params


# ---- instances and bags ------------------------------------------------------------------------------------------------
def extract_instances(est: Params, dataset: DataFrame):
    """Predictor.extractInstances: label cast to double, weight = weightCol if set and non-empty else 1."""
    X = np.asarray(dataset[est("featuresCol")])
    y = np.asarray(dataset[est("labelCol")], dtype=np.float64)
    wc = est("weightCol") if est.isDefined("weightCol") else ""
    w = np.asarray(dataset[wc], dtype=np.float64) if wc else None
    return X, y, w


def split_validation(est: Params, dataset: DataFrame):
    """(train, validation) frames of a GBM fit: the rows validationIndicatorCol flags are held out; validation is None
    without that column."""
    vc = est("validationIndicatorCol") if est.isDefined("validationIndicatorCol") else ""
    if vc:
        mask = np.asarray(dataset[vc], dtype=bool)
        return dataset.filter(~mask), dataset.filter(mask)
    return dataset, None


def bag_counts(n: int, subsample_ratio: float, replacement: bool, seed: int):
    """GBM's bag: multiplicity of every train row in `RDD.sample(replacement, ratio, seed)`; None when the bag is the
    whole set.  Drawn once, because the reference passes the same seed every round (quirk 3).
    Without replacement: Spark's own sampler for rows in ONE partition (ensemble.spark_bernoulli_sample; unpinned: no
    Spark here).  With replacement Spark uses commons-math3's PoissonDistribution over a Well19937c generator, which is
    not restated: numpy draws Poisson(ratio).  On a Spark host the multiplicities come from Spark itself
    (GBMRegressorNative.scala).  Bagging draws its bag with numpy either way (bagging_fit)."""
    if subsample_ratio == 1.0 and not replacement:
        return None
    if not replacement:
        return spark_bernoulli_sample(n, subsample_ratio, seed)
    rng = np.random.default_rng(seed & 0xFFFFFFFF)
    return rng.poisson(subsample_ratio, n).astype(np.float32)


# ---- the device fit ----------------------------------------------------------------------------------------------------
def device_fit(est: Params, learner, require_resident: bool) -> bool:
    """True when the base learner fits on the device (learners.DeviceDecisionTreeRegressor / Classifier).  It reads the
    residuals (or labels and weights) and the features where they live, so it needs residentFeatures=True; without it,
    require_resident raises, and otherwise the learner's own `fit` is used (it opens a context per call).  With Param
    `devices` naming two or more GPUs it fits over all of their rows at once (sharded.ShardedContext.tree_fit: each
    level's histogram is all-reduced across the GPUs)."""
    if not getattr(learner, "device_learner", False):
        return False
    if not est("residentFeatures"):
        if require_resident:
            raise ValueError("the device tree learner fits over the device-resident features: set residentFeatures=True")
        return False
    devices = [int(d) for d in est("devices")] if est.hasParam("devices") else []
    if len(devices) >= 2:  # every rank joins each level's all-reduce: the GPUs must exist and be distinct (NCCL)
        if len(set(devices)) != len(devices):
            raise ValueError(f"the device tree learner shards its fit over `devices`, which must name distinct GPUs: "
                             f"{devices}")
        visible = N.device_count()
        missing = [d for d in devices if d >= visible]
        if missing:
            raise ValueError(f"the device tree learner shards its fit over `devices` {devices}, but GPU {missing[0]} is "
                             f"not one of the {visible} visible")
    return True


# ---- Bagging: every member sees the same bag (reference quirk 3) and differs only in its subspace -----------------
def bagging_fit(est: Params, X, y, w, num_classes: int | None = None):
    """(subspaces, models) of a Bagging fit.  The bag is drawn once with numpy.  With residentFeatures and a device tree
    learner every member's tree grows in one forest fit (_bagging_forest_fit); otherwise each member is one
    learner.fit on the in-bag rows of its subspace.  num_classes goes to the classifier's learner."""
    n, d = X.shape
    seed, M = est("seed"), est("numBaseLearners")
    learner = est("baseLearner")
    subs = [subspace(est("subspaceRatio"), d, seed + i) for i in range(M)]
    rng = np.random.default_rng(seed & 0xFFFFFFFF)
    counts = (rng.poisson(est("subsampleRatio"), n) if est("replacement")
              else (rng.random(n) < est("subsampleRatio"))).astype(np.float64)
    bw = counts if w is None else counts * w
    if device_fit(est, learner, require_resident=False):
        return subs, _bagging_forest_fit(est.device, learner, X, y, bw, subs, num_classes)
    keep = bw > 0
    kw = {} if num_classes is None else {"num_classes": num_classes}
    return subs, [learner.fit(X[keep][:, subs[i]], y[keep], bw[keep], **kw) for i in range(M)]


def _bagging_forest_fit(device: int, learner, X, y, bw, subs, num_classes: int | None) -> list:
    """Bagging's members fitted together on the device: X is uploaded once, the candidates come from the in-bag rows,
    and one forest fit grows every member's tree.  The labels sit in SLOT_Y, the weights bw in SLOT_W and the in-bag
    indicator in SLOT_BAG, so a node's rawCount counts distinct in-bag rows and its weight is Σ bw: the statistics
    learner.fit(X[keep][:, sub], y[keep], bw[keep]) sees, hence the same trees.  Raises the ValueError that route
    raises for no in-bag row, an empty subspace, bad labels or Params."""
    keep = bw > 0
    rows = np.flatnonzero(keep)
    if rows.size == 0 or any(len(s) == 0 for s in subs):
        raise ValueError(f"{type(learner).__name__}.fit needs at least one row and one column")
    n, d = X.shape
    if num_classes is not None:
        K = int(num_classes)
        check_class_labels(np.asarray(y, dtype=np.float64).reshape(-1)[rows], K, rows.size)
        learner._check_classes(K)
    cands = learner.split_candidates(X, rows=rows)
    with Context(device) as ctx:
        ctx.alloc(N.SLOT_X, d, n)
        ctx.upload_rowmajor(N.SLOT_X, X)
        ctx.alloc(N.SLOT_Y, n)
        ctx.upload(N.SLOT_Y, np.asarray(y, dtype=np.float32))
        ctx.alloc(N.SLOT_W, n)
        ctx.upload(N.SLOT_W, np.asarray(bw, dtype=np.float32))
        ctx.alloc(N.SLOT_BAG, n)
        ctx.upload(N.SLOT_BAG, keep.astype(np.float32))
        ctx.tree_fit_bins(cands)
        if num_classes is None:
            return learner.fit_forest_resident(ctx, N.SLOT_Y, 0, N.SLOT_W, 0, True, subs)
        return learner.fit_forest_resident(ctx, int(num_classes), N.SLOT_Y, 0, N.SLOT_W, 0, True, subs)


# ---- Boosting ----------------------------------------------------------------------------------------------------------
def load_boosting(ctx: Context, X, y, w, learner, device_fit: bool, upload_features: bool):
    """The state of a Boosting fit, after its *_configure call: X column-major in SLOT_X when upload_features, the
    device learner's split candidates (set once for every round) when device_fit, the labels in SLOT_Y and the boosting
    weights (the instance weights, else 1) in SLOT_BW.  Returns (every column, for the device fit; Σ boosting weights)."""
    n, d = X.shape
    if upload_features:
        ctx.alloc(N.SLOT_X, d, n)
        ctx.upload_rowmajor(N.SLOT_X, X)
    all_cols = None
    if device_fit:
        ctx.tree_fit_bins(learner.split_candidates(X))
        all_cols = np.arange(d, dtype=np.int32)
    ctx.upload(N.SLOT_Y, y)
    ctx.upload(N.SLOT_BW, np.ones(n) if w is None else w)
    return all_cols, ctx.slot_sum(N.SLOT_BW)


# ---- scoring -----------------------------------------------------------------------------------------------------------
def device_trees(model: Params, members) -> list | None:
    """The tree arrays of every member when the model scores them on the device: residentFeatures is set, there is
    at least one member, and every member exposes tree_arrays().  None keeps the member-by-member route."""
    if not model("residentFeatures") or not members:
        return None
    trees = []
    for m in members:
        fn = getattr(m, "tree_arrays", None)
        t = fn() if fn is not None else None
        if t is None:
            return None
        trees.append(t)
    return trees


def resident_context(device: int, X) -> Context:
    """A context whose SLOT_X holds the rows of X column-major: the matrix the forest kernels walk."""
    X = np.asarray(X, dtype=np.float32)
    ctx = Context(device)
    try:
        ctx.alloc(N.SLOT_X, X.shape[1], X.shape[0])
        ctx.upload_rowmajor(N.SLOT_X, X)
    except BaseException:
        ctx.close()
        raise
    return ctx


def download_raw(ctx: Context) -> np.ndarray:
    return ctx.download(N.SLOT_RAW).astype(np.float64)


def one_pass(device: int, X, trees, score, fetch):
    """score(ctx, trees) over a resident context of X, then fetch(ctx).  None without trees (device_trees), or when the
    forest's thresholds do not fit the uint8 rank matrix (more than 255 in a column: SE_ERR_STATE), so that the
    caller scores member by member."""
    if trees is None:
        return None
    with resident_context(device, X) as ctx:
        try:
            score(ctx, trees)
        except N.NativeError as e:
            if e.code == N.SE_ERR_STATE:
                return None
            raise
        return fetch(ctx)


def forest_sum(device: int, X, trees, subspaces, weights, init: float) -> np.ndarray | None:
    """init + Σ_t weights[t] · tree_t(x) through se_forest_predict; None as one_pass."""
    def score(ctx, trees):
        ctx.alloc(N.SLOT_RAW, 1, X.shape[0])
        ctx.forest_predict(trees, N.SLOT_RAW, weights=weights, init=init, subspaces=subspaces)
    return one_pass(device, X, trees, score, download_raw)


def stack_outputs(models, subspaces, X, extra=None) -> np.ndarray:
    """[M][n] fp32: every member's predictions on its subspace of X, after `extra` (a row) when given."""
    rows = [] if extra is None else [extra]
    for m, s in zip(models, subspaces):
        rows.append(m.predict(X[:, s]))
    if not rows:
        return np.zeros((0, X.shape[0]), dtype=np.float32)
    return np.ascontiguousarray(np.stack(rows), dtype=np.float32)


def member_route(device: int, kind: int, P, num_classes: int = 0, dim: int = 1, loss=0, weights=None, init=None,
                 fetch=download_raw):
    """The members' outputs P ([M][...][n], stacked on the host) aggregated on the device by agg_run: SLOT_RAW for a
    regressor, or whatever fetch reads."""
    with Context(device) as ctx:
        ctx.agg_configure(kind, P.shape[0], num_classes, dim, loss, P.shape[-1])
        if P.shape[0]:
            ctx.upload(N.SLOT_P, P)
        ctx.agg_run(weights, init)
        return fetch(ctx)
