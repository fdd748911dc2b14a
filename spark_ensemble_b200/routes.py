"""What the estimator mirrors (regression, classification) share: their instances and bags, the choice of the device
fit, the set-up of a Bagging or Boosting fit, and the two routes by which a model scores its members:

- one pass over the device-resident features when every member is a tree (se_forest_predict / se_forest_median /
  se_forest_agg), which returns None when the forest's thresholds do not fit the rank matrix;
- one pass over them when every member is a linear or logistic model (se_linear_agg);
- the member route: every member's output stacked on the host, uploaded as SLOT_P and aggregated on the device
  (se_agg_run).

Each decision lives here once, so the estimators that make it differently make that visible at their call sites.
"""
from __future__ import annotations

import inspect

import numpy as np

from . import _native as N
from .context import Context
from .ensemble import DataFrame, spark_bernoulli_sample, subspace
from .learners import check_class_labels, distinct_subspaces
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


def resident_linear(est: Params, learner) -> bool:
    """True when a DeviceLinearRegression or DeviceLogisticRegression base learner fits in the estimator's own context,
    over the data already there: residentFeatures is set and Param `devices`, if the estimator has it, names at most
    one GPU (sharded.ShardedContext has no linear or logistic calls).  Otherwise the learner's `fit` is used."""
    from .learners import DeviceLinearRegression, DeviceLogisticRegression
    if not isinstance(learner, (DeviceLinearRegression, DeviceLogisticRegression)) or not est("residentFeatures"):
        return False
    return not (est.hasParam("devices") and len(est("devices")) >= 2)


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
    if resident_linear(est, learner):
        return subs, _bagging_linear_fit(est.device, learner, X, y, bw, subs, num_classes)
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


def _bagging_linear_fit(device: int, learner, X, y, bw, subs, num_classes: int | None) -> list:
    """Bagging's linear or logistic members fitted in one context: X is uploaded once, the weights bw go to SLOT_W (0
    outside the bag) and equal subspaces are fitted once.  A member sees what learner.fit(X[keep][:, sub], y[keep],
    bw[keep]) sees: the same weighted sums, with the same shifts (the in-bag column means for a linear member, the
    first in-bag row for a logistic one), since rows of weight 0 add exact zeros.  The out-of-bag rows' labels and
    non-finite features, which that route never reads, are replaced by 0 in what is uploaded, so they fail nothing;
    an in-bag one fails the fit as it does there."""
    from .learners import DeviceLogisticRegression
    keep = bw > 0
    rows = np.flatnonzero(keep)
    if rows.size == 0:
        raise ValueError(f"{type(learner).__name__}.fit needs at least one row")
    X = np.asarray(X, dtype=np.float32)
    n, d = X.shape
    finite = np.isfinite(X).all(axis=1)
    if not finite[~keep].all():
        X = np.where((keep | finite)[:, None], X, np.where(np.isfinite(X), X, np.float32(0)))
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    distinct, index = distinct_subspaces(subs)
    with Context(device) as ctx:
        ctx.alloc(N.SLOT_X, d, n)
        ctx.upload_rowmajor(N.SLOT_X, X)
        ctx.alloc(N.SLOT_Y, n)
        ctx.upload(N.SLOT_Y, np.where(keep, y, 0.0).astype(np.float32))
        ctx.alloc(N.SLOT_W, n)
        ctx.upload(N.SLOT_W, np.where(keep, bw, 0.0).astype(np.float32))
        if isinstance(learner, DeviceLogisticRegression):
            K = int(num_classes) if num_classes is not None else int(np.nanmax(y[rows])) + 1
            first = X[rows[0]].astype(np.float64)
            models = learner.fit_members_resident(ctx, distinct, K, N.SLOT_Y, 0, N.SLOT_W, 0,
                                                  [first[c] for c in distinct])
        else:
            shift = X[rows].mean(axis=0, dtype=np.float64)
            models = learner.fit_members_resident(ctx, distinct, N.SLOT_Y, 0, N.SLOT_W, 0, shift,
                                                  float(np.float32(y[rows[0]])))
    return [models[i] for i in index]


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


def linear_list(members) -> list | None:
    """The fp64 margin arrays (margin_arrays()) of every member, or None when one of them is not a linear or logistic
    model, or reads more columns than se_linear_agg takes."""
    out = []
    for m in members:
        a = m.margin_arrays() if hasattr(m, "margin_arrays") else None
        if a is None or np.atleast_2d(a["coef"]).shape[1] > N.LOGISTIC_MAX_COLS:
            return None
        out.append(a)
    return out


def device_linear(model: Params, members) -> list | None:
    """The packed members when the model scores them in one se_linear_agg pass: residentFeatures is set, there is at
    least one member, and every member is a linear or logistic model (linear_list).  None keeps the member route."""
    if not model("residentFeatures") or not members:
        return None
    return linear_list(members)


def linear_kw(kw: dict) -> dict:
    """forest_agg's keyword arguments as linear_agg takes them: a member's GBM class is its member_class."""
    return {("member_class" if k == "tree_class" else k): v for k, v in kw.items()}


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


def linear_sum(device: int, X, members, subspaces, kind: int, weights=None, init=None) -> np.ndarray | None:
    """A regressor kind's aggregate of linear members (device_linear) through se_linear_agg: what agg_run gives over
    their outputs, without them; None without members."""
    def score(ctx, members):
        ctx.alloc(N.SLOT_RAW, 1, X.shape[0])
        ctx.linear_agg(kind, 0, members, N.SLOT_RAW, weights=weights, init=init, subspaces=subspaces)
    return one_pass(device, X, members, score, download_raw)


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


# ---- Stacking ----------------------------------------------------------------------------------------------------------
STACK_METHODS = ("class", "raw", "proba")  # classification/StackingClassifier.scala supportedStackMethod


def is_classifier(member) -> bool:
    """A classification estimator mirror (it has rawPredictionCol) or a learner whose fit takes num_classes."""
    if isinstance(member, Params):
        return member.hasParam("rawPredictionCol")
    return "num_classes" in inspect.signature(member.fit).parameters


def takes_weights(member) -> bool:
    """HasWeightCol: an estimator mirror with weightCol, or a learner whose fit takes w."""
    if isinstance(member, Params):
        return member.hasParam("weightCol")
    return "w" in inspect.signature(member.fit).parameters


def member_width(member, method: str, num_classes: int | None) -> int:
    """Meta-features a member contributes (the reference's models.flatMap): its K probabilities (proba) or its K-wide
    raw vector (raw) for a classifier, else its one prediction."""
    if num_classes is not None and method in ("raw", "proba") and is_classifier(member):
        return int(num_classes)
    return 1


def fit_member(est: Params, member, dataset: DataFrame, X, y, w, num_classes: int | None, weight_col: str = ""):
    """fitBaseLearner: an estimator mirror fits on the frame with the stacking estimator's label, features and
    prediction columns (and weight_col when w is given); a learner fits on (X, y, w)."""
    if isinstance(member, Params):
        m = member.copy()
        for name in ("labelCol", "featuresCol", "predictionCol"):
            m.set(name, est(name))
        if w is not None:
            m.set("weightCol", weight_col)
        return m.fit(dataset)
    kw = {"num_classes": num_classes} if (num_classes is not None and is_classifier(member)) else {}
    return member.fit(X, y, w, **kw) if takes_weights(member) else member.fit(X, y, **kw)


def model_outputs(model, X, method: str, width: int) -> np.ndarray:
    """[width][n] fp64 meta-features of one member model on the host."""
    if hasattr(model, "_raw_prob_label"):  # a classification estimator model
        raw, prob, label = model._raw_prob_label(X)
        out = prob.T if (width > 1 and method == "proba") else raw.T if width > 1 else label[None]
    elif hasattr(model, "_aggregate"):  # a regression estimator model
        out = model._aggregate(X)[None]
    elif width > 1 and method == "proba":
        out = model.predictProbability(X).T
    elif width > 1:
        out = model.predictRaw(X).T
    else:
        out = np.asarray(model.predict(X))[None]
    out = np.asarray(out, dtype=np.float64)
    if out.shape[0] != width:
        raise ValueError(f"{type(model).__name__} gives {out.shape[0]} meta-features where {width} are expected")
    return out


def model_predict(model, F) -> np.ndarray:
    """The stack's predict over meta-features F [n, W]."""
    return model_outputs(model, F, "class", 1)[0]


def write_member_rows(ctx: Context, model, method: str, row: int, width: int) -> bool:
    """A fitted member's meta-features into rows row .. row + width - 1 of SLOT_P over the context's SLOT_X, on the
    device: single trees (se_tree_predict / se_tree_predict_multi), linear models (se_linear_predict) and the estimator
    models of trees (their write_rows).  False when the model has no device form, or when its thresholds do not fit
    the rank matrix (SE_ERR_STATE): the caller predicts it on the host then."""
    try:
        t = model.tree_arrays() if hasattr(model, "tree_arrays") else None
        if t is not None:
            if width == 1:
                ctx.tree_predict(t, N.SLOT_P, row)
                return True
            vals = t["values"] if method == "proba" else model.node_raw()
            ctx.alloc(N.SLOT_PROBA, width, ctx.layout(N.SLOT_P)[1])
            ctx.tree_predict_multi({**t, "values": np.asarray(vals, dtype=np.float32)}, N.SLOT_PROBA)
            ctx.copy_rows(N.SLOT_P, row, N.SLOT_PROBA, 0, width)
            return True
        lin = model.linear_arrays() if hasattr(model, "linear_arrays") else None
        if lin is not None:
            ctx.linear_predict(lin["coef"], float(lin["intercept"]), N.SLOT_P, row)
            return True
        write = getattr(model, "write_rows", None)
        return bool(write is not None and write(ctx, method, N.SLOT_P, row))
    except N.NativeError as e:
        if e.code == N.SE_ERR_STATE:
            return False
        raise


def tree_list(members) -> list | None:
    """The tree arrays of every member, or None when one of them is not a tree."""
    trees = []
    for m in members:
        t = m.tree_arrays() if hasattr(m, "tree_arrays") else None
        if t is None:
            return None
        trees.append(t)
    return trees


def _stacker_fit_device(ctx: Context, stacker, n: int, W: int, weighted: bool, num_classes: int | None):
    """The stacker fitted over the meta-features in the context's SLOT_X; None for a stacker without a device fit."""
    from .learners import DeviceLinearRegression, DeviceLogisticRegression
    cols = np.arange(W, dtype=np.int32)
    wslot = N.SLOT_W if weighted else -1
    if isinstance(stacker, DeviceLinearRegression):
        return stacker.fit_resident(ctx, N.SLOT_X, cols, N.SLOT_Y, 0, wslot, 0, False, None)
    if isinstance(stacker, DeviceLogisticRegression) and num_classes is not None:
        return stacker.fit_resident(ctx, N.SLOT_X, cols, int(num_classes), N.SLOT_Y, 0, wslot, 0)
    if not getattr(stacker, "device_learner", False):
        return None
    # candidates from the meta-features of the sampled rows, as stacker.fit over the downloaded matrix draws them
    ctx.tree_fit_bins(stacker.split_candidates(ctx.download(N.SLOT_X).reshape(W, n).T))
    ctx.alloc(N.SLOT_RAW, 1, n)
    if num_classes is None:
        return stacker.fit_resident(ctx, N.SLOT_Y, 0, wslot, 0, False, cols, N.SLOT_RAW, 0)
    return stacker.fit_resident(ctx, int(num_classes), N.SLOT_Y, 0, wslot, 0, False, cols, N.SLOT_RAW, 0)


def stacking_fit(est: Params, dataset: DataFrame, num_classes: int | None = None):
    """(member models, stack, widths) of a Stacking fit.  Members get the weights only when every member takes them; the
    stacker always gets them (or ones).  Host route (residentFeatures=False): the reference's data flow.  Device route:
    one context holds X (uploaded once), the labels and weights; device learners fit in it and write their outputs into
    their rows of SLOT_P, other members are fitted on their own and scored into their rows on the device when they have
    a device form (on the host otherwise); the meta-features then become SLOT_X and a device stacker fits over them."""
    X, y, w = extract_instances(est, dataset)
    X = np.asarray(X, dtype=np.float32)
    n, d = X.shape
    members = list(est("baseLearners"))
    stacker = est("stacker")
    method = est("stackMethod").lower() if est.hasParam("stackMethod") else "class"
    mw = w if (w is not None and all(takes_weights(m) for m in members)) else None
    wc = mw is not None and est("weightCol")
    sw = np.ones(n) if w is None else w
    widths = [member_width(m, method, num_classes) for m in members]
    if not est("residentFeatures"):
        models = [fit_member(est, m, dataset, X, y, mw, num_classes, wc) for m in members]
        meta = np.concatenate([model_outputs(mod, X, method, k) for mod, k in zip(models, widths)])
        return models, _fit_stacker_host(est, stacker, meta.T, y, sw, num_classes), widths
    from .learners import DeviceLinearRegression, DeviceLogisticRegression
    W = sum(widths)
    models = []
    with resident_context(est.device, X) as ctx:
        ctx.alloc(N.SLOT_Y, n)
        ctx.upload(N.SLOT_Y, y)
        if w is not None:
            ctx.alloc(N.SLOT_W, n)
            ctx.upload(N.SLOT_W, w)
        ctx.alloc(N.SLOT_P, W, n)
        all_cols = np.arange(d, dtype=np.int32)
        mslot = N.SLOT_W if mw is not None else -1
        row = 0
        for m, k in zip(members, widths):
            if isinstance(m, DeviceLinearRegression):
                model = m.fit_resident(ctx, N.SLOT_X, all_cols, N.SLOT_Y, 0, mslot, 0, False, N.SLOT_P, row)
            elif isinstance(m, DeviceLogisticRegression) and num_classes is not None:
                model = m.fit_resident(ctx, N.SLOT_X, all_cols, int(num_classes), N.SLOT_Y, 0, mslot, 0, N.SLOT_P, row,
                                       method if k > 1 else "class")
            elif getattr(m, "device_learner", False):
                ctx.tree_fit_bins(m.split_candidates(X))
                if not is_classifier(m):
                    model = m.fit_resident(ctx, N.SLOT_Y, 0, mslot, 0, False, all_cols, N.SLOT_P, row)
                else:
                    check_class_labels(y, int(num_classes), n)
                    model = m.fit_resident(ctx, int(num_classes), N.SLOT_Y, 0, mslot, 0, False, all_cols, N.SLOT_P,
                                           row, proba=(k > 1))
                    if k > 1 and method == "raw" and not write_member_rows(ctx, model, method, row, k):
                        ctx.upload(N.SLOT_P, model_outputs(model, X, method, k), offset=row * n)
            else:
                model = fit_member(est, m, dataset, X, y, mw, num_classes, wc)
                if not write_member_rows(ctx, model, method, row, k):
                    ctx.upload(N.SLOT_P, model_outputs(model, X, method, k), offset=row * n)
            models.append(model)
            row += k
        ctx.alloc(N.SLOT_X, W, n)
        ctx.copy_slot(N.SLOT_X, N.SLOT_P)
        stack = _stacker_fit_device(ctx, stacker, n, W, w is not None, num_classes)
        if stack is None:
            meta = ctx.download(N.SLOT_P).reshape(W, n).T.astype(np.float64)
    if stack is None:
        stack = _fit_stacker_host(est, stacker, meta, y, sw, num_classes)
    return models, stack, widths


def _fit_stacker_host(est: Params, stacker, F, y, w, num_classes: int | None):
    """The stacker fitted on the host over meta-features F [n, W] with weights w: an estimator mirror on a frame of
    the label, the meta-features and the weights under the stacking estimator's column names (weightCol, or "weight"
    when it is unset), a learner on (F, y, w)."""
    wc = (est("weightCol") if est.isDefined("weightCol") else "") or "weight"
    frame = DataFrame(**{est("labelCol"): y, est("featuresCol"): F, wc: w})
    return fit_member(est, stacker, frame, F, y, w, num_classes, wc)


def stacking_predict(model: Params, X) -> np.ndarray:
    """stack.predict(meta-features) of every row of X.  Host route: each member's outputs on the host.  Device route
    (residentFeatures): X is uploaded once; members with a device form write their rows of SLOT_P on the device, the
    others are predicted on the host and uploaded; the meta-features become SLOT_X and a tree, linear or logistic stack
    scores them there."""
    X = np.asarray(X, dtype=np.float32)
    n = X.shape[0]
    method = model("stackMethod").lower() if model.hasParam("stackMethod") else "class"
    if not model("residentFeatures"):
        meta = np.concatenate([model_outputs(m, X, method, k) for m, k in zip(model.models, model.widths)])
        return model_predict(model.stack, meta.T)
    W = sum(model.widths)
    with resident_context(model.device, X) as ctx:
        ctx.alloc(N.SLOT_P, W, n)
        row = 0
        for m, k in zip(model.models, model.widths):
            if not write_member_rows(ctx, m, method, row, k):
                ctx.upload(N.SLOT_P, model_outputs(m, X, method, k), offset=row * n)
            row += k
        ctx.alloc(N.SLOT_X, W, n)
        ctx.copy_slot(N.SLOT_X, N.SLOT_P)
        ctx.alloc(N.SLOT_RAW, 1, n)
        if write_stack_rows(ctx, model.stack, N.SLOT_RAW):
            return download_raw(ctx)
        meta = ctx.download(N.SLOT_P).reshape(W, n).T.astype(np.float64)
    return model_predict(model.stack, meta)


def write_stack_rows(ctx: Context, stack, out_slot: int) -> bool:
    """The stack's prediction (a tree's value or label, a linear model, or a logistic regression's label) of every row
    of SLOT_X into out_slot; False for any other stack, which is then predicted on the host."""
    try:
        t = stack.tree_arrays() if hasattr(stack, "tree_arrays") else None
        if t is not None:
            ctx.tree_predict(t, out_slot, 0)
            return True
    except N.NativeError as e:
        if e.code == N.SE_ERR_STATE:
            return False
        raise
    lin = stack.linear_arrays() if hasattr(stack, "linear_arrays") else None
    if lin is not None:
        ctx.linear_predict(lin["coef"], float(lin["intercept"]), out_slot, 0)
        return True
    from .learners import LogisticRegressionModel
    if isinstance(stack, LogisticRegressionModel):  # its write_rows writes only the label row of out_slot
        return stack.write_rows(ctx, "class", out_slot, 0)
    return False
