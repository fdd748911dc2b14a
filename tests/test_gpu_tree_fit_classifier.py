"""The device classification-tree fit (se_tree_fit_classifier) against the numpy restatement in
oracle/np_tree_cls.py, and BoostingClassifier / BaggingClassifier with the device learner: boosting against a host loop
that fits the restatement on the downloaded normalised weights."""
import os

import numpy as np
import pytest

from oracle import np_tree as T
from oracle import np_tree_cls as TC

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    yield c
    c.close()


def _data(n, d, K, seed, special=False, exact=False):
    rng = np.random.default_rng(seed)
    if exact:
        X = rng.integers(0, 8, (n, d)).astype(np.float32)
        z = X[:, 0] + 0.5 * X[:, 1] + rng.integers(0, 3, n)
    else:
        X = rng.standard_normal((n, d)).astype(np.float32)
        if special:
            X[rng.random((n, d)) < 0.05] = np.nan
            X[rng.random((n, d)) < 0.02] = np.inf
            X[rng.random((n, d)) < 0.02] = -np.inf
        zz = np.nan_to_num(X[:, : min(d, 3)], nan=0.0, posinf=3.0, neginf=-3.0)
        z = np.sin(2 * zz[:, 0]) + zz[:, -1] ** 2 + 0.4 * rng.standard_normal(n)
    if n == 1:
        return X, np.zeros(1, np.float32)
    y = np.digitize(z, np.quantile(z, np.linspace(0, 1, K + 1)[1:-1]))
    return X, np.minimum(y, K - 1).astype(np.float32)


def _fit(ctx, X, y, K, *, w=None, bag=None, sub=None, impurity="gini", max_depth=3, max_bins=32, min_instances=1,
         min_info_gain=0.0, min_weight_fraction=0.0, exact=False):
    """Device fits (label and probability outputs) and the oracle fit of the same problem.  Every node of both device
    trees is audited (np_tree_cls.audit) from the rows it receives, whatever the near ties."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.learners import DeviceDecisionTreeClassifier
    n, d = X.shape
    sub = np.arange(d, dtype=np.int32) if sub is None else np.asarray(sub, dtype=np.int32)
    cands = DeviceDecisionTreeClassifier(maxBins=max_bins, seed=11).split_candidates(X)
    ctx.alloc(N.SLOT_X, d, n)
    ctx.upload_rowmajor(N.SLOT_X, X)
    ctx.alloc(N.SLOT_Y, 1, n)
    ctx.upload(N.SLOT_Y, y)
    ctx.alloc(N.SLOT_PRED, 1, n)
    ctx.alloc(N.SLOT_RAW, 1, n)
    ctx.alloc(N.SLOT_PROBA, K, n)
    ctx.alloc(N.SLOT_P, K, n)
    if w is not None:
        ctx.alloc(N.SLOT_W, 1, n)
        ctx.upload(N.SLOT_W, w)
    if bag is not None:
        ctx.alloc(N.SLOT_BAG, 1, n)
        ctx.upload(N.SLOT_BAG, bag)
    ctx.tree_fit_bins(cands)
    kw = dict(subspace=sub, impurity=impurity, max_depth=max_depth, min_instances=min_instances,
              min_info_gain=min_info_gain, min_weight_fraction=min_weight_fraction)
    wslot = N.SLOT_W if w is not None else -1
    t = ctx.tree_fit_classifier(N.SLOT_Y, K, 0, wslot, 0, bag is not None, out_slot=N.SLOT_PRED, **kw)
    tp = ctx.tree_fit_classifier(N.SLOT_Y, K, 0, wslot, 0, bag is not None, proba=True, out_slot=N.SLOT_PROBA, **kw)
    out = ctx.download(N.SLOT_PRED)
    outp = ctx.download(N.SLOT_PROBA).reshape(K, n)
    ctx.tree_predict(t, N.SLOT_RAW, 0, subspace=sub)
    np.testing.assert_array_equal(out.view(np.uint32), ctx.download(N.SLOT_RAW).view(np.uint32))
    ctx.tree_predict_multi(tp, N.SLOT_P, subspace=sub)
    np.testing.assert_array_equal(outp.view(np.uint32), ctx.download(N.SLOT_P).reshape(K, n).view(np.uint32))
    params = dict(num_classes=K, impurity=impurity, max_depth=max_depth, min_instances=min_instances,
                  min_info_gain=min_info_gain, min_weight_fraction=min_weight_fraction)
    assert TC.audit(t, X, cands, sub, y, w, bag, params, out=out, exact=exact) == t["feature"].size
    assert TC.audit(tp, X, cands, sub, y, w, bag, params, out_proba=outp, exact=exact) == tp["feature"].size
    ranks = [T.ranks(X[:, c], cands[c]) for c in sub]
    o = TC.fit(ranks, [cands[c].size for c in sub], y, K, w=w, counts=bag, impurity_kind=impurity,
               max_depth=max_depth, min_instances=min_instances, min_info_gain=min_info_gain,
               min_weight_fraction=min_weight_fraction)
    if not any(_near_tie(i) for i in o["info"]):  # fp64 atomics cannot flip a clear split: both fits chose one tree
        for key in ("feature", "threshold", "left", "right", "value"):
            np.testing.assert_array_equal(t[key], tp[key])
    return t, out, outp, o, ranks, [cands[c] for c in sub]


def _near_tie(info):
    return info is not None and np.isfinite(info[0]) and (info[0] - info[1] <= 1e-7 * abs(info[0]) or info[0] < 1e-10)


def _compare(t, o, ranks, cands, rows, i=0, j=0, counts=None):
    """Walks the device tree (i) and the oracle tree (j) together; returns (nodes compared, nodes skipped)."""
    if _near_tie(o["info"][j]):
        return 0, 1
    dev_leaf, or_leaf = t["feature"][i] < 0, o["feature"][j] < 0
    assert dev_leaf == or_leaf, (i, j)
    assert t["value"][i] == o["label"][j], (i, j)
    np.testing.assert_allclose(t["values"][i], o["proba"][j], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(t["class_weights"][i], o["cw"][j], rtol=1e-9, atol=1e-9)
    if dev_leaf:
        return 1, 0
    fo, bo = o["feature"][j], o["bin"][j]
    go = ranks[fo][rows] <= bo
    fd = t["feature"][i]
    bd = int(np.searchsorted(cands[fd], t["threshold"][i]))
    assert cands[fd][bd] == t["threshold"][i]
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
    # n, |S|, K, impurity, maxDepth, maxBins, weights, bag, non-finite features
    (1, 1, 2, "gini", 3, 32, False, None, False),
    (7, 5, 3, "entropy", 3, 4, True, None, False),
    (1000, 5, 2, "gini", 0, 32, False, None, False),
    (1000, 1, 3, "entropy", 1, 2, False, None, False),
    (1000, 40, 26, "gini", 5, 32, True, "poisson", False),
    (1000, 5, 64, "entropy", 8, 256, True, "bernoulli", True),  # weighted: ~11 rows a class tie often unweighted
    (65537, 5, 3, "gini", 5, 255, True, "bernoulli", True),
    (65537, 40, 2, "entropy", 3, 2, False, None, False),
    (65537, 4, 26, "gini", 8, 256, True, None, False),   # one column's histogram overflows shared memory
    (200000, 6, 64, "gini", 6, 32, True, None, False),
    (1_000_000, 5, 3, "entropy", 5, 32, True, "poisson", True),
]


@pytest.mark.parametrize("n,S,K,impurity,depth,bins,weighted,bag,special", CASES)
def test_device_fit_matches_oracle(ctx, n, S, K, impurity, depth, bins, weighted, bag, special):
    rng = np.random.default_rng(n + S + depth + K)
    d = S + 3
    X, y = _data(n, d, K, seed=n + depth, special=special)
    sub = rng.permutation(d)[:S].astype(np.int32)  # a non-identity subspace
    w = rng.uniform(0.25, 4.0, n).astype(np.float32) if weighted else None
    counts = None
    if bag == "poisson":
        counts = rng.poisson(1.0, n).astype(np.float32)
    elif bag == "bernoulli":
        counts = (rng.random(n) < 0.7).astype(np.float32)
    if counts is not None and counts.sum() == 0:
        counts[0] = 1
    t, out, outp, o, ranks, cands = _fit(ctx, X, y, K, w=w, bag=counts, sub=sub, impurity=impurity, max_depth=depth,
                                         max_bins=bins)
    done, skipped = _compare(t, o, ranks, cands, np.arange(n), counts=counts)
    print(f"nodes {t['feature'].size}: all audited, {done} compared with the restatement, {skipped} subtrees skipped")
    assert done >= 1
    if n >= 100:
        assert skipped <= (done // 3 if n < 10000 else max(1, done // 10)), (done, skipped)
    if skipped == 0:
        leaf = TC.leaf_of(o, ranks)
        np.testing.assert_array_equal(out, o["label"][leaf].astype(np.float32))
        np.testing.assert_allclose(outp.T, o["proba"][leaf], rtol=1e-6, atol=1e-6)
    assert t["feature"].size <= 2 ** (depth + 1) - 1
    assert np.all(t["gain"][t["feature"] >= 0] > 0)


def _exact(ctx, seed, impurity):
    """Integer features and labels, unweighted: every sum is exact.  A duplicated column must lose every tie to the
    first; no internal node keeps two leaf children with equal labels; every leaf's probabilities are the class
    distribution of all the rows that reach it, so a merged leaf carries its parent's, not a child's.  Returns the
    number of merged leaves."""
    K = 3
    X, y = _data(4096, 3, K, seed=seed, exact=True)
    X = np.concatenate([X[:, :1], X], axis=1)  # column 1 duplicates column 0
    t, out, outp, o, ranks, cands = _fit(ctx, X, y, K, impurity=impurity, max_depth=6, max_bins=8, exact=True)
    done, skipped = _compare(t, o, ranks, cands, np.arange(X.shape[0]))
    assert skipped <= max(1, done // 10)
    assert 1 not in set(t["feature"].tolist()), "the duplicated column must lose every tie to the first"
    f, l, rr, v = t["feature"], t["left"], t["right"], t["value"]
    for i in np.flatnonzero(f >= 0):
        assert not (f[l[i]] < 0 and f[rr[i]] < 0 and v[l[i]] == v[rr[i]])
    from spark_ensemble_b200.learners import DeviceDecisionTreeClassificationModel
    leaf = DeviceDecisionTreeClassificationModel(t, K)._leaf(X)
    for i in np.unique(leaf):
        cnt = np.bincount(y[leaf == i].astype(int), minlength=K).astype(np.float64)
        np.testing.assert_array_equal(t["values"][i], (cnt / cnt.sum()).astype(np.float32))
        np.testing.assert_array_equal(t["class_weights"][i], cnt)
    return int(np.sum(o["merged"]))


def test_exact_ties_first_max_and_pruning(ctx):
    merged = sum(_exact(ctx, s, imp) for s, imp in [(0, "gini"), (1, "entropy"), (2, "gini"), (3, "entropy")])
    assert merged > 0, "the exact data must exercise merged leaves"


def test_validity_rules_bind(ctx):
    X, y = _data(20000, 4, 3, seed=3)
    base, *_ = _fit(ctx, X, y, 3, max_depth=4)
    for kw in ({"min_instances": 3000}, {"min_info_gain": float(np.median(base["gain"][base["feature"] >= 0]))},
               {"min_weight_fraction": 0.15}):
        t, out, outp, o, ranks, cands = _fit(ctx, X, y, 3, max_depth=4, w=np.linspace(0.5, 1.5, 20000, dtype=np.float32),
                                             **kw)
        done, skipped = _compare(t, o, ranks, cands, np.arange(20000))
        assert skipped <= 1
        assert t["feature"].size < base["feature"].size, kw


def test_errors(ctx):
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.learners import DeviceDecisionTreeClassifier
    X, y = _data(500, 3, 3, seed=1)
    _fit(ctx, X, y, 3, max_depth=2)
    for K, depth in ((1, 2), (65, 2), (3, 9)):
        with pytest.raises(ValueError):
            ctx.tree_fit_classifier(N.SLOT_Y, K, subspace=[0, 1], max_depth=depth, out_slot=N.SLOT_PRED)
    with pytest.raises(ValueError):  # a label outside [0, K) on the device: flagged, the call fails
        ctx.tree_fit_classifier(N.SLOT_Y, 2, subspace=[0, 1], max_depth=2, out_slot=N.SLOT_PRED)
    ctx.tree_fit_classifier(N.SLOT_Y, 3, subspace=[0, 1], max_depth=2, out_slot=N.SLOT_PRED)  # and recovers
    with pytest.raises(ValueError):
        DeviceDecisionTreeClassifier(maxDepth=2).fit(X, np.where(y == 2, 3, y), num_classes=3)
    host = {"feature": np.array([1, -1, -1], np.int32), "threshold": np.array([0.123456], np.float32).repeat(3),
            "left": np.array([1, 0, 0], np.int32), "right": np.array([2, 0, 0], np.int32),
            "value": np.array([0, 1, 2], np.float32)}
    ctx.tree_predict(host, N.SLOT_RAW, 0)
    with pytest.raises(N.NativeError) as e:
        ctx.tree_fit_classifier(N.SLOT_Y, 3, subspace=[0, 1], max_depth=2, out_slot=N.SLOT_PRED)
    assert e.value.code == N.SE_ERR_STATE
    ctx.tree_fit_classifier(N.SLOT_Y, 3, subspace=[0, 2], max_depth=2, out_slot=N.SLOT_PRED)


# ---- BoostingClassifier / BaggingClassifier end to end ---------------------------------------------------------
class _OracleTree:
    """Host learner: the restatement fitted on the downloaded normalised weights, over the same candidates.  A near
    tie would let fp64 rounding pick another split than the device: fail loudly instead of diverging quietly."""

    def __init__(self, cands, max_depth, impurity):
        self.cands, self.max_depth, self.impurity = cands, max_depth, impurity

    def copy(self, extra=None):
        return self

    def fit(self, X, y, w=None, num_classes=None):
        from spark_ensemble_b200.learners import DeviceDecisionTreeClassificationModel
        ranks = [T.ranks(X[:, j], self.cands[j]) for j in range(X.shape[1])]
        o = TC.fit(ranks, [c.size for c in self.cands], y, num_classes, w=w, impurity_kind=self.impurity,
                   max_depth=self.max_depth)
        ties = [i for i in o["info"] if _near_tie(i)]
        assert not ties, f"a near tie in the host loop: {ties}"
        thr = np.array([self.cands[f][b] if f >= 0 else 0.0 for f, b in zip(o["feature"], o["bin"])], np.float32)
        return DeviceDecisionTreeClassificationModel(
            {"feature": o["feature"].astype(np.int32), "threshold": thr, "left": o["left"].astype(np.int32),
             "right": o["right"].astype(np.int32), "value": o["label"].astype(np.float32), "values": o["proba"],
             "class_weights": o["cw"], "gain": o["gain"]}, num_classes)


def _letter(n):
    d = np.load(os.path.join(GOLD, "letter.npz"))
    return (d["X"][:n].astype(np.float64) / 7.5 - 1.0).astype(np.float32), d["y"][:n].astype(np.float64)


@pytest.mark.parametrize("data,algorithm,impurity", [("letter", "discrete", "entropy"), ("letter", "real", "entropy"),
                                                     ("binary", "discrete", "entropy"), ("binary", "real", "gini")])
def test_boosting_with_device_learner_matches_host_loop(monkeypatch, data, algorithm, impurity):
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.classification import BoostingClassifier
    from spark_ensemble_b200.context import Context
    from spark_ensemble_b200.ensemble import DataFrame
    from spark_ensemble_b200.learners import DeviceDecisionTreeClassifier
    rng = np.random.default_rng(3)
    if data == "letter":
        # SAMME.R drives letter's weights apart by 1e13 within a few rounds, and integer features then meet near ties
        # in some subsets: these have none in five rounds
        X, y = _letter(4000 if algorithm == "real" else 3000)
        w = None
        depth = 4
    else:
        n = 6000
        X = rng.standard_normal((n, 5)).astype(np.float32)
        y = (np.sin(2 * X[:, 0]) + X[:, 1] * X[:, 2] + 0.5 * rng.standard_normal(n) > 0).astype(np.float64)
        w = rng.uniform(0.5, 2.0, n)
        depth = 3
    df = DataFrame(features=X, label=y) if w is None else DataFrame(features=X, label=y, weight=w)
    dev = DeviceDecisionTreeClassifier(maxDepth=depth, maxBins=32, impurity=impurity, seed=5)
    cands = dev.split_candidates(X)

    def make(learner):
        e = BoostingClassifier().set("baseLearner", learner).set("numBaseLearners", 5).set("algorithm", algorithm)
        e.set("residentFeatures", True)
        if w is not None:
            e.set("weightCol", "weight")
        return e

    host = make(_OracleTree(cands, depth, impurity)).fit(df)
    real_download = Context.download

    def guarded(self, slot, *a, **k):
        assert slot != N.SLOT_BW, "the boosting weights left the device"
        return real_download(self, slot, *a, **k)

    monkeypatch.setattr(Context, "download", guarded)
    devm = make(dev).fit(df)
    monkeypatch.undo()
    hh, dh = host.trainingHistory, devm.trainingHistory
    assert len(hh) == len(dh) >= 2
    for a, b in zip(hh, dh):
        np.testing.assert_allclose(b["estimatorError"], a["estimatorError"], rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(b["sumWeights"], a["sumWeights"], rtol=1e-5)
    np.testing.assert_allclose(devm.weights, host.weights, rtol=1e-5)
    oh, od = host.transform(df), devm.transform(df)
    for col in ("rawPrediction", "probability"):  # SAMME.R sums terms of +-(K - 1)·52·ln 2: scale atol to them
        np.testing.assert_allclose(od[col], oh[col], rtol=1e-5, atol=1e-5 * max(1.0, np.abs(oh[col]).max()))
    assert np.mean(od["prediction"] == oh["prediction"]) > 0.999


def test_bagging_with_device_learner_aggregates_members():
    from spark_ensemble_b200 import DataFrame
    from spark_ensemble_b200.classification import BaggingClassifier
    from spark_ensemble_b200.learners import DeviceDecisionTreeClassificationModel, DeviceDecisionTreeClassifier
    Xl, yl = _letter(3000)
    for strategy in ("hard", "soft"):
        bcl = (BaggingClassifier().setBaseLearner(DeviceDecisionTreeClassifier(maxDepth=8)).setNumBaseLearners(5)
               .setVotingStrategy(strategy))
        mc = bcl.fit(DataFrame(features=Xl, label=yl))
        assert all(isinstance(m, DeviceDecisionTreeClassificationModel) and m.numClasses == 26 for m in mc.models)
        out = mc.transform(DataFrame(features=Xl))
        if strategy == "hard":
            votes = np.stack([mm.predict(Xl[:, s]) for mm, s in zip(mc.models, mc.subspaces)])
            cnt = np.stack([(votes == c).sum(axis=0) for c in range(26)], axis=1).astype(np.float64)
            np.testing.assert_array_equal(out["rawPrediction"], cnt)
            np.testing.assert_allclose(out["probability"], cnt / 5, rtol=1e-6)
        else:
            P = np.stack([mm.predictProbability(Xl[:, s]) for mm, s in zip(mc.models, mc.subspaces)])
            np.testing.assert_allclose(out["rawPrediction"], P.sum(axis=0), rtol=1e-5, atol=1e-6)
        assert np.mean(out["prediction"] == yl) > 0.4
