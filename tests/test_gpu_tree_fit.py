"""The device regression-tree fit (se_tree_fit) against the numpy restatement in oracle/np_tree.py, and GBM fits with
the device learner against a host loop that fits the restatement on the downloaded residuals."""
import numpy as np
import pytest

from oracle import np_tree as T

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    yield c
    c.close()


def _data(n, d, seed, special=False, dyadic=False):
    rng = np.random.default_rng(seed)
    if dyadic:
        X = rng.integers(0, 8, (n, d)).astype(np.float32)
        r = (rng.integers(-8, 8, n) / 4).astype(np.float32)
        return X, r
    X = rng.standard_normal((n, d)).astype(np.float32)
    if special:
        X[rng.random((n, d)) < 0.05] = np.nan
        X[rng.random((n, d)) < 0.02] = np.inf
        X[rng.random((n, d)) < 0.02] = -np.inf
    z = np.nan_to_num(X[:, : min(d, 3)], nan=0.0, posinf=3.0, neginf=-3.0)
    r = (np.sin(2 * z[:, 0]) + z[:, -1] ** 2 + 0.3 * rng.standard_normal(n)).astype(np.float32)
    return X, r


def _fit(ctx, X, r, *, w=None, bag=None, sub=None, max_depth=3, max_bins=32, min_instances=1, min_info_gain=0.0,
         min_weight_fraction=0.0, exact=False):
    """Device fit and oracle fit of the same problem; returns (device tree, device out, oracle tree, oracle ranks).
    Every node of the device tree is audited (np_tree.audit) from the rows it receives, whatever the near ties."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor
    n, d = X.shape
    sub = np.arange(d, dtype=np.int32) if sub is None else np.asarray(sub, dtype=np.int32)
    cands = DeviceDecisionTreeRegressor(maxBins=max_bins, seed=11).split_candidates(X)
    ctx.alloc(N.SLOT_X, d, n)
    ctx.upload_rowmajor(N.SLOT_X, X)
    ctx.alloc(N.SLOT_R, 1, n)
    ctx.upload(N.SLOT_R, r)
    ctx.alloc(N.SLOT_H, 1, n)
    ctx.alloc(N.SLOT_RAW, 1, n)
    if w is not None:
        ctx.alloc(N.SLOT_W, 1, n)
        ctx.upload(N.SLOT_W, w)
    if bag is not None:
        ctx.alloc(N.SLOT_BAG, 1, n)
        ctx.upload(N.SLOT_BAG, bag)
    ctx.tree_fit_bins(cands)
    t = ctx.tree_fit(N.SLOT_R, 0, N.SLOT_W if w is not None else -1, 0, bag is not None, subspace=sub,
                     max_depth=max_depth, min_instances=min_instances, min_info_gain=min_info_gain,
                     min_weight_fraction=min_weight_fraction, out_slot=N.SLOT_H, out_row=0)
    out = ctx.download(N.SLOT_H)
    ctx.tree_predict(t, N.SLOT_RAW, 0, subspace=sub)
    walk = ctx.download(N.SLOT_RAW)
    np.testing.assert_array_equal(out.view(np.uint32), walk.view(np.uint32))  # the fit's output IS the tree's output
    params = dict(max_depth=max_depth, min_instances=min_instances, min_info_gain=min_info_gain,
                  min_weight_fraction=min_weight_fraction)
    assert T.audit(t, X, cands, sub, r, w, bag, params, out=out, exact=exact) == t["feature"].size
    ranks = [T.ranks(X[:, c], cands[c]) for c in sub]
    o = T.fit(ranks, [cands[c].size for c in sub], r, w=w, counts=bag, **params)
    return t, out, o, ranks, [cands[c] for c in sub]


def _near_tie(info):
    """A searched node whose best and second-best gains are within 1e-7, or whose best is noise: fp64 rounding may
    decide it either way."""
    return info is not None and np.isfinite(info[0]) and (info[0] - info[1] <= 1e-7 * abs(info[0]) or info[0] < 1e-10)


def _compare(t, o, ranks, cands, rows, i=0, j=0, counts=None):
    """Walks the device tree (i) and the oracle tree (j) together.  Returns (nodes compared, nodes skipped): the
    subtree of a near tie is skipped (the audit checks it)."""
    if _near_tie(o["info"][j]):
        return 0, 1
    dev_leaf, or_leaf = t["feature"][i] < 0, o["feature"][j] < 0
    assert dev_leaf == or_leaf, (i, j)
    if dev_leaf:
        np.testing.assert_allclose(t["value"][i], o["pred"][j], rtol=1e-6, atol=1e-6)
        return 1, 0
    fo, bo = o["feature"][j], o["bin"][j]
    go = ranks[fo][rows] <= bo
    fd = t["feature"][i]
    bd = int(np.searchsorted(cands[fd], t["threshold"][i]))
    assert cands[fd][bd] == t["threshold"][i]  # a candidate, and its rank threshold
    # the first maximum: the same column and candidate, or (rounding of equal sums) another column splitting alike
    gd = ranks[fd][rows] <= bd
    if counts is not None:
        inb = counts[rows] > 0
        assert np.array_equal(go[inb], gd[inb])
    else:
        assert np.array_equal(go, gd)
        if fd == fo:
            assert bd == bo
    a = _compare(t, o, ranks, cands, rows[go], t["left"][i], o["left"][j], counts)
    b = _compare(t, o, ranks, cands, rows[~go], t["right"][i], o["right"][j], counts)
    return 1 + a[0] + b[0], a[1] + b[1]


CASES = [
    # n, |S|, maxDepth, maxBins, weights, bag, non-finite features
    (1, 1, 3, 32, False, None, False),
    (7, 5, 3, 4, True, None, False),
    (1000, 5, 0, 32, False, None, False),
    (1000, 1, 1, 2, False, None, False),
    (1000, 40, 5, 32, True, "poisson", False),
    (1000, 5, 8, 256, False, "bernoulli", True),
    (65537, 5, 5, 255, True, "bernoulli", True),
    (65537, 40, 3, 2, False, None, False),
    (65537, 5, 8, 256, True, None, False),   # deep levels: one column's histogram overflows shared memory
    (1_000_000, 5, 5, 32, True, "poisson", True),
]


@pytest.mark.parametrize("n,S,depth,bins,weighted,bag,special", CASES)
def test_device_fit_matches_oracle(ctx, n, S, depth, bins, weighted, bag, special):
    rng = np.random.default_rng(n + S + depth)
    d = S + 3
    X, r = _data(n, d, seed=n + depth, special=special)
    sub = rng.permutation(d)[:S].astype(np.int32)  # a non-identity subspace
    w = rng.uniform(0.25, 4.0, n).astype(np.float32) if weighted else None
    counts = None
    if bag == "poisson":
        counts = rng.poisson(1.0, n).astype(np.float32)
    elif bag == "bernoulli":
        counts = (rng.random(n) < 0.7).astype(np.float32)
    if counts is not None and counts.sum() == 0:
        counts[0] = 1
    t, out, o, ranks, cands = _fit(ctx, X, r, w=w, bag=counts, sub=sub, max_depth=depth, max_bins=bins)
    done, skipped = _compare(t, o, ranks, cands, np.arange(n), counts=counts)
    print(f"nodes {t['feature'].size}: all audited, {done} compared with the restatement, {skipped} subtrees skipped")
    # nodes of a handful of rows tie often, and deep trees over 1000 rows are made of them: the near ties must be
    # rare in the large fits and a minority everywhere
    assert done >= 1
    if n >= 100:
        assert skipped <= (done // 3 if n < 10000 else max(1, done // 10)), (done, skipped)
    if skipped == 0:
        np.testing.assert_allclose(out, T.predict(o, ranks), rtol=1e-6, atol=1e-6)
    assert t["feature"].size <= 2 ** (depth + 1) - 1
    assert np.all(t["gain"][t["feature"] >= 0] > 0)


@pytest.mark.parametrize("seed", range(4))
def test_exact_ties_first_max_and_pruning(ctx, seed):
    """Dyadic labels and integer features: every sum is exact, so equal gains are equal bit for bit.  A duplicated
    column and the equal candidates of sparse nodes must resolve to the first maximum, and no internal node keeps two
    leaf children with equal predictions."""
    X, r = _data(4096, 3, seed=seed, dyadic=True)
    X = np.concatenate([X[:, :1], X], axis=1)  # column 1 duplicates column 0
    t, out, o, ranks, cands = _fit(ctx, X, r, max_depth=6, max_bins=8, exact=True)
    done, skipped = _compare(t, o, ranks, cands, np.arange(X.shape[0]))
    assert skipped <= max(1, done // 10)
    assert 1 not in set(t["feature"].tolist()), "the duplicated column must lose every tie to the first"
    f, l, rr, v = t["feature"], t["left"], t["right"], t["value"]
    for i in np.flatnonzero(f >= 0):
        assert not (f[l[i]] < 0 and f[rr[i]] < 0 and v[l[i]] == v[rr[i]])


def test_validity_rules_bind(ctx):
    X, r = _data(20000, 4, seed=3)
    base, _, _, _, _ = _fit(ctx, X, r, max_depth=4)
    for kw in ({"min_instances": 3000}, {"min_info_gain": float(np.median(base["gain"][base["feature"] >= 0]))},
               {"min_weight_fraction": 0.15}):
        t, out, o, ranks, cands = _fit(ctx, X, r, max_depth=4, w=np.linspace(0.5, 1.5, 20000, dtype=np.float32), **kw)
        done, skipped = _compare(t, o, ranks, cands, np.arange(20000))
        assert skipped <= 1
        assert t["feature"].size < base["feature"].size, kw  # the rule removed splits


def test_errors(ctx):
    from spark_ensemble_b200 import _native as N
    X, r = _data(500, 3, seed=1)
    _fit(ctx, X, r, max_depth=2)
    for kw in ({"max_depth": 9}, {"max_depth": -1}, {"min_instances": 0}, {"min_weight_fraction": 0.5},
               {"min_weight_fraction": -0.01}):
        args = dict(max_depth=2, min_instances=1, min_weight_fraction=0.0)
        args.update(kw)
        with pytest.raises(ValueError):
            ctx.tree_fit(N.SLOT_R, 0, -1, 0, False, subspace=[0, 1], out_slot=N.SLOT_H, **args)
    with pytest.raises(ValueError):  # candidates must be sorted and finite
        ctx.tree_fit_bins([np.array([1.0, 0.0]), np.zeros(0), np.zeros(0)])
    with pytest.raises(ValueError):
        ctx.tree_fit_bins([np.array([np.inf]), np.zeros(0), np.zeros(0)])
    # a host tree whose threshold is not a candidate lands in column 1: fitting over column 1 is refused
    host = {"feature": np.array([1, -1, -1], np.int32), "threshold": np.array([0.123456], np.float32).repeat(3),
            "left": np.array([1, 0, 0], np.int32), "right": np.array([2, 0, 0], np.int32),
            "value": np.array([0, 1, 2], np.float32)}
    ctx.tree_predict(host, N.SLOT_RAW, 0)
    with pytest.raises(N.NativeError) as e:
        ctx.tree_fit(N.SLOT_R, 0, -1, 0, False, subspace=[0, 1], max_depth=2, out_slot=N.SLOT_H)
    assert e.value.code == N.SE_ERR_STATE
    ctx.tree_fit(N.SLOT_R, 0, -1, 0, False, subspace=[0, 2], max_depth=2, out_slot=N.SLOT_H)  # other columns still fit


# ---- GBM end to end --------------------------------------------------------------------------------------------
class _OracleTree:
    """Host learner: the restatement fitted on the downloaded residuals, over the same candidates.  A near tie would
    let fp64 rounding pick another split than the device: fail loudly instead of diverging quietly."""

    def __init__(self, cands, max_depth):
        self.cands, self.max_depth = cands, max_depth

    def copy(self, extra=None):
        return self

    def fit(self, X, y, w=None):
        from spark_ensemble_b200.learners import DeviceDecisionTreeRegressionModel
        ranks = [T.ranks(X[:, j], self.cands[j]) for j in range(X.shape[1])]
        o = T.fit(ranks, [c.size for c in self.cands], y, w=w, max_depth=self.max_depth)
        ties = [i for i in o["info"] if _near_tie(i)]
        assert not ties, f"a near tie in the host loop: {ties}"
        thr = np.array([self.cands[f][b] if f >= 0 else 0.0 for f, b in zip(o["feature"], o["bin"])], np.float32)
        return DeviceDecisionTreeRegressionModel({"feature": o["feature"].astype(np.int32), "threshold": thr,
                                                  "left": o["left"].astype(np.int32), "right": o["right"].astype(np.int32),
                                                  "value": o["pred"].astype(np.float32), "gain": o["gain"]})


E2E = [("reg", "squared", "gradient"), ("reg", "huber", "gradient"), ("reg", "squared", "newton"),
       ("cls", "bernoulli", "gradient"), ("cls", "logloss", "gradient"),
       # two-valued residuals (sign, {q, q - 1}), and Newton weights in WOUT rows 1 .. K - 1
       ("reg", "absolute", "gradient"), ("reg", "quantile", "gradient"), ("cls", "logloss", "newton")]


@pytest.mark.parametrize("kind,loss,updates", E2E)
def test_gbm_with_device_learner_matches_host_loop(monkeypatch, kind, loss, updates):
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.classification import GBMClassifier
    from spark_ensemble_b200.context import Context
    from spark_ensemble_b200.ensemble import DataFrame
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor
    from spark_ensemble_b200.regression import GBMRegressor
    rng = np.random.default_rng(7)
    n, d = 6000, 6
    X = rng.standard_normal((n, d)).astype(np.float32)
    z = np.sin(2 * X[:, 0]) + X[:, 1] * X[:, 2]
    if kind == "reg":
        y = z + 0.3 * rng.standard_normal(n)
    elif loss == "bernoulli":
        y = (z + 0.5 * rng.standard_normal(n) > 0).astype(np.float64)
    else:
        y = np.digitize(z + 0.5 * rng.standard_normal(n), [-0.5, 0.5]).astype(np.float64)
    valid = rng.random(n) < 0.25
    # two-valued residuals (sign, {q, q - 1}, one-hot minus a prior) make a gain a function of counts alone, and equal
    # counts tie exactly between different splits: continuous row weights break those ties
    weighted = loss in ("absolute", "quantile", "logloss")
    df = DataFrame(features=X, label=y, valid=valid, weight=rng.uniform(0.5, 2.0, n)) if weighted else \
        DataFrame(features=X, label=y, valid=valid)
    dev = DeviceDecisionTreeRegressor(maxDepth=3, maxBins=32, seed=5)
    cands = dev.split_candidates(X[~valid])
    est_cls = GBMRegressor if kind == "reg" else GBMClassifier

    def make(learner):
        e = est_cls().set("baseLearner", learner).set("numBaseLearners", 8).set("loss", loss).set("updates", updates)
        e.set("residentFeatures", True).set("validationIndicatorCol", "valid").set("numRounds", 2)
        if weighted:
            e.set("weightCol", "weight")
        e.set("subsampleRatio", 0.8).set("learningRate", 0.5)
        return e

    host = make(_OracleTree(cands, 3)).fit(df)
    real_download = Context.download

    def guarded(self, slot, *a, **k):
        assert slot not in (N.SLOT_R, N.SLOT_WOUT), "residuals left the device"
        return real_download(self, slot, *a, **k)

    monkeypatch.setattr(Context, "download", guarded)
    devm = make(dev).fit(df)
    monkeypatch.undo()
    hh, dh = host.trainingHistory, devm.trainingHistory
    assert len(hh) == len(dh) and len(dh) >= 2
    # Newton weights are continuous: a leaf value may differ from the host's by an fp32 ulp (same trees otherwise), and
    # L-BFGS-B (K = 3 step sizes), which stops at tol 1e-6, pins α only to ~sqrt(tol): the losses carry the 1e-5 check
    a_rtol = 1e-3 if (kind, updates) == ("cls", "newton") else 1e-5
    for a, b in zip(hh, dh):
        np.testing.assert_allclose(np.atleast_1d(b["alpha"]), np.atleast_1d(a["alpha"]), rtol=a_rtol, atol=1e-7)
        np.testing.assert_allclose(b["trainLoss"], a["trainLoss"], rtol=1e-5)
        np.testing.assert_allclose(b["validationLoss"], a["validationLoss"], rtol=1e-5)
