"""CPU checks of the regression-tree learner's specification (DESIGN.md §3 "Device tree fit"): the numpy restatement in
oracle/np_tree.py against scikit-learn's exact tree and against brute force, hand-worked split candidates, the
validity rules and pruning, and the learner's Params."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import np_tree as T
from spark_ensemble_b200 import learners as Lr


def _fit_cols(X, y, max_bins=256, **kw):
    cands = [T.candidates(X[:, j], max_bins) for j in range(X.shape[1])]
    ranks = [T.ranks(X[:, j], cands[j]) for j in range(X.shape[1])]
    return T.fit(ranks, [c.size for c in cands], y, **kw), cands, ranks


def _thresholds(tree, cands):
    return np.array([cands[f][b] if f >= 0 else 0.0 for f, b in zip(tree["feature"], tree["bin"])], dtype=np.float32)


# ---- candidates ------------------------------------------------------------------------------------------------
def test_candidates_hand_worked():
    assert T.candidates([1, 2, 3, 4], 32).tolist() == [1.5, 2.5, 3.5]
    assert T.candidates([5, 5, 5], 32).size == 0                          # constant column: never splits
    assert T.candidates([np.nan, np.nan], 32).size == 0
    assert T.candidates([1, 1, 1, 2, 2, 3], 32).tolist() == [1.5, 2.5]   # duplicates count once as values
    assert T.candidates([-0.0, 0.0, 1.0], 32).tolist() == [0.5]          # -0 is +0
    assert T.candidates([1, np.nan, 3], 32).tolist() == [2.0]            # NaN is not a value
    # stride branch: 10 distinct values of count 1, maxBins 4: stride 2.5, emits at cumulative counts 3, 5 and 8
    assert T.candidates(np.arange(10), 4).tolist() == [2.5, 4.5, 7.5]
    # counts matter: 7 of 12 samples on 0 (stride 4) put both candidates next to it
    assert T.candidates([0] * 7 + [1, 2, 3, 4, 5], 3).tolist() == [0.5, 1.5]
    # fp64 midpoint of two adjacent floats is stored as the largest float below it
    a = np.float32(1.0)
    b = np.nextafter(a, np.float32(2))
    assert T.candidates([a, b], 32).tolist() == [1.0]
    # +-inf: the midpoint is clamped to +-FLT_MAX and still separates the infinite value
    fmax = float(np.finfo(np.float32).max)
    assert T.candidates([-np.inf, 0.0, np.inf], 32).tolist() == [-fmax, fmax]


@pytest.mark.parametrize("max_bins", [2, 4, 32, 255, 256])
def test_product_candidates_equal_oracle(max_bins):
    rng = np.random.default_rng(max_bins)
    cols = [rng.standard_normal(3000), rng.integers(0, 50, 3000), np.round(rng.exponential(size=3000), 2),
            np.r_[rng.standard_normal(100), [np.nan, np.inf, -np.inf, -0.0, 0.0]], np.full(10, 3.0)]
    for c in cols:
        c = np.asarray(c, dtype=np.float32)
        np.testing.assert_array_equal(Lr.continuous_split_candidates(c, max_bins), T.candidates(c, max_bins))


def test_candidates_sample_rule():
    m = Lr.DeviceDecisionTreeRegressor(maxBins=32, seed=7)
    assert m.sample_rows(10000) is None                     # n <= max(maxBins², 10000): every row
    m2 = Lr.DeviceDecisionTreeRegressor(maxBins=200, seed=7)
    assert m2.sample_rows(40000) is None                    # maxBins² = 40000
    rows = m.sample_rows(200000)
    assert rows is not None and 8000 < rows.size < 12000   # fraction 10000 / n
    np.testing.assert_array_equal(rows, m.sample_rows(200000))


# ---- the fit ---------------------------------------------------------------------------------------------------
def _walk_equal_sklearn(tree, cands, sk, X, rows, i=0, j=0):
    """Same structure, same partition of the node's rows at every split, same leaf values.  scikit-learn puts its
    threshold halfway between the two values adjacent WITHIN the node; the restatement takes the first of the global
    candidates between them (all of which split the node alike): it must be the lowest one that does."""
    t = sk.tree_
    info = tree["info"][i]
    if info is not None and info[0] - info[1] <= 1e-9 * abs(info[0]):
        return 0  # a gain tie between different splits: scikit-learn breaks it at random
    leaf_sk = t.children_left[j] < 0
    assert (tree["feature"][i] < 0) == leaf_sk
    if leaf_sk:
        np.testing.assert_allclose(tree["pred"][i], t.value[j].reshape(-1)[0], rtol=1e-9, atol=1e-12)
        return 1
    f = tree["feature"][i]
    thr = cands[f][tree["bin"][i]]
    x = X[rows, f]
    go = x <= thr
    # another column that splits the node's rows identically is the same split (scikit-learn picks one at random)
    np.testing.assert_array_equal(go, X[rows, t.feature[j]] <= Lr._floor_f32(np.array([t.threshold[j]]))[0])
    assert thr >= x[go].max() and (tree["bin"][i] == 0 or cands[f][tree["bin"][i] - 1] < x[go].max())
    return (1 + _walk_equal_sklearn(tree, cands, sk, X, rows[go], tree["left"][i], t.children_left[j])
            + _walk_equal_sklearn(tree, cands, sk, X, rows[~go], tree["right"][i], t.children_right[j]))


@pytest.mark.parametrize("seed,depth,weighted", [(0, 3, False), (1, 4, False), (2, 5, True), (3, 2, True)])
def test_oracle_equals_sklearn_exact_tree(seed, depth, weighted):
    """With every midpoint a candidate (maxBins - 1 >= distinct values) and continuous data (no gain ties), the
    restatement is an exact CART regression tree: scikit-learn's, node for node."""
    from sklearn.tree import DecisionTreeRegressor
    rng = np.random.default_rng(seed)
    n, d = 150, 3
    X = rng.standard_normal((n, d)).astype(np.float32)
    y = (X[:, 0] * 2 + np.sin(3 * X[:, 1]) + 0.3 * rng.standard_normal(n)).astype(np.float32)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32) if weighted else None
    cands = [T.candidates(X[:, j], 256) for j in range(d)]
    assert all(c.size == n - 1 for c in cands)
    ranks = [T.ranks(X[:, j], cands[j]) for j in range(d)]
    tree = T.fit(ranks, [c.size for c in cands], y, w=w, max_depth=depth)
    tree = T.fit(ranks, [c.size for c in cands], y, w=w, max_depth=depth, min_instances=3)
    sk = DecisionTreeRegressor(max_depth=depth, min_samples_leaf=3, random_state=0).fit(
        X, y.astype(np.float64), sample_weight=w)
    compared = _walk_equal_sklearn(tree, cands, sk, X, np.arange(n))
    assert compared >= 0.8 * sk.tree_.node_count and sk.tree_.node_count == tree["feature"].size


def _brute(ranks, ncand, r, c, depth, max_depth, min_inst):
    """Direct recursion over every (column, candidate) with masked sums: no histograms, no prefix sums."""
    W = c.sum()
    S = (c * r).sum()
    Q = (c * r * r).sum()
    pred = S / W
    imp = (Q - S * S / W) / W
    if depth == max_depth:
        return ("leaf", pred)
    best = None
    for k in range(len(ranks)):
        for j in range(ncand[k]):
            m = ranks[k] <= j
            cl, cr = c * m, c * ~m
            if cl.sum() < min_inst or cr.sum() < min_inst:
                continue
            stats = []
            for cc in (cl, cr):
                w_, s_, q_ = cc.sum(), (cc * r).sum(), (cc * r * r).sum()
                stats.append((w_, (q_ - s_ * s_ / w_) / w_))
            g = imp - stats[0][0] / W * stats[0][1] - stats[1][0] / W * stats[1][1]
            if best is None or g > best[0]:
                best = (g, k, j, cl, cr, stats)
    if best is None or best[0] <= 0:
        return ("leaf", pred)
    g, k, j, cl, cr, stats = best
    kids = []
    for cc, (_, ci) in zip((cl, cr), stats):
        if depth + 1 == max_depth or abs(ci) < T.EPS:
            kids.append(("leaf", (cc * r).sum() / cc.sum()))
        else:
            kids.append(_brute(ranks, ncand, r, cc, depth + 1, max_depth, min_inst))
    if kids[0][0] == kids[1][0] == "leaf" and kids[0][1] == kids[1][1]:
        return ("leaf", kids[0][1])
    return ("split", k, j, kids[0], kids[1])


def _as_nested(tree, i=0):
    if tree["feature"][i] < 0:
        return ("leaf", tree["pred"][i])
    return ("split", int(tree["feature"][i]), int(tree["bin"][i]), _as_nested(tree, tree["left"][i]),
            _as_nested(tree, tree["right"][i]))


def _same(a, b):
    if a[0] != b[0]:
        return False
    if a[0] == "leaf":
        return abs(a[1] - b[1]) <= 1e-9 * max(1.0, abs(a[1]))
    return a[1:3] == b[1:3] and _same(a[3], b[3]) and _same(a[4], b[4])


@pytest.mark.parametrize("seed", range(6))
def test_oracle_equals_brute_force(seed):
    rng = np.random.default_rng(100 + seed)
    n = 10
    X = rng.integers(0, 5, (n, 2)).astype(np.float32)
    r = rng.standard_normal(n).astype(np.float32)
    c = rng.integers(0, 3, n).astype(np.float32) if seed % 2 else np.ones(n, dtype=np.float32)
    cands = [T.candidates(X[:, j], 3) for j in range(2)]
    ranks = [T.ranks(X[:, j], cands[j]) for j in range(2)]
    for max_depth, min_inst in [(1, 1), (3, 1), (3, 2)]:
        tree = T.fit(ranks, [x.size for x in cands], r, counts=c, max_depth=max_depth, min_instances=min_inst)
        brute = _brute([np.asarray(q) for q in ranks], [x.size for x in cands], r.astype(np.float64),
                       c.astype(np.float64), 0, max_depth, min_inst)
        assert _same(_as_nested(tree), brute), (_as_nested(tree), brute)


def test_first_max_tie_rule_and_pruning():
    # two identical columns: every gain ties, the first column wins; within a column the first candidate wins
    x = np.array([0, 1, 2, 3], dtype=np.float32)
    X = np.stack([x, x], axis=1)
    y = np.array([0, 0, 1, 1], dtype=np.float32)
    tree, cands, _ = _fit_cols(X, y, max_depth=2)
    assert tree["feature"][0] == 0 and tree["bin"][0] == 1
    sym = np.array([1, 0, 0, 1], dtype=np.float32)  # candidates 0 and 2 give the same gain: the first is kept
    tree, _, _ = _fit_cols(x[:, None], sym, max_depth=1)
    assert tree["feature"][0] == 0 and tree["bin"][0] == 0
    # pruning: on decimal data a split whose children have equal fp64 means can carry a rounding-positive gain; the
    # fitted tree then never keeps two leaf siblings with equal predictions
    rng = np.random.default_rng(0)
    pruned = 0
    for _ in range(1500):
        xx = rng.integers(0, 4, 8).astype(np.float32)
        yy = (rng.integers(0, 4, 8) / 10).astype(np.float32)
        t, _, _ = _fit_cols(xx[:, None], yy, max_depth=3)
        for i in np.flatnonzero(t["feature"] >= 0):
            a, b = t["left"][i], t["right"][i]
            assert not (t["feature"][a] < 0 and t["feature"][b] < 0 and t["pred"][a] == t["pred"][b])
        pruned += sum(1 for i, f in zip(t["info"], t["feature"]) if f < 0 and i is not None and i[0] > 0)
    assert pruned > 0


def test_validity_rules_bind():
    rng = np.random.default_rng(5)
    n = 200
    X = rng.standard_normal((n, 2)).astype(np.float32)
    y = (X[:, 0] > 1.5).astype(np.float32) * 5 + 0.1 * rng.standard_normal(n).astype(np.float32)
    base, _, _ = _fit_cols(X, y, max_bins=64, max_depth=1)
    assert base["feature"][0] == 0
    # minInstancesPerNode larger than the best split's small side: another (worse) split wins
    small = int(min(base["left"].size, (X[:, 0] > 1.5).sum()))
    t, _, _ = _fit_cols(X, y, max_bins=64, max_depth=1, min_instances=(X[:, 0] > 1.5).sum() + 1)
    assert t["feature"].size == 1 or t["bin"][0] != base["bin"][0]
    assert small >= 1
    # minInfoGain above the best gain: the root stays a leaf
    t, _, _ = _fit_cols(X, y, max_bins=64, max_depth=1, min_info_gain=base["gain"][0] * 1.01)
    assert t["feature"].size == 1
    # minWeightFractionPerNode: both sides must carry that fraction of the root weight
    t, _, _ = _fit_cols(X, y, max_bins=64, max_depth=1, min_weight_fraction=0.2)
    assert t["feature"].size == 3
    lw = (T.ranks(X[:, t["feature"][0]], T.candidates(X[:, t["feature"][0]], 64)) <= t["bin"][0]).mean()
    assert 0.2 <= lw <= 0.8
    # maxDepth 0: the root is a leaf with the weighted mean
    t, _, _ = _fit_cols(X, y, max_depth=0)
    assert t["feature"].tolist() == [-1] and abs(t["pred"][0] - y.astype(np.float64).mean()) < 1e-12


# ---- the audit of a fitted tree (oracle/np_tree.audit) --------------------------------------------------------
def _audit_problem(seed, weighted, bagged):
    rng = np.random.default_rng(300 + seed)
    n, d = 3000, 5
    X = rng.standard_normal((n, d)).astype(np.float32)
    X[rng.random((n, d)) < 0.03] = np.nan
    z = np.nan_to_num(X)
    r = (np.sin(2 * z[:, 1]) + z[:, 3] ** 2 + 0.3 * rng.standard_normal(n)).astype(np.float32)
    w = rng.uniform(0.25, 4.0, n).astype(np.float32) if weighted else None
    c = rng.poisson(1.0, n).astype(np.float32) if bagged else None
    cands = [T.candidates(X[:, j], 32) for j in range(d)]
    sub = np.array([4, 1, 0, 3], np.int32)
    R = [T.ranks(X[:, j], cands[j]) for j in sub]
    params = dict(max_depth=4, min_instances=1, min_info_gain=0.0, min_weight_fraction=0.0)
    o = T.fit(R, [cands[j].size for j in sub], r, w=w, counts=c, **params)
    return T.arrays(o, [cands[j] for j in sub]), X, cands, sub, r, w, c, params, T.predict(o, R), R


def _mutations(a, X, cands, sub, r, w, c, params, R):
    """The tree with one thing wrong, five ways: (name, arrays)."""
    f, left, right = a["feature"], a["left"], a["right"]
    splits = np.flatnonzero(f >= 0)
    leaves = np.flatnonzero(f < 0)
    out = []
    b = a.copy()
    b["value"] = b["value"].copy()
    i = leaves[0]
    b["value"][i] = np.float32(b["value"][i]) + 4 * np.spacing(np.float32(b["value"][i]))
    out.append(("leaf value + 4 ulps", b))
    b = {k: v.copy() for k, v in a.items()}
    i = splits[0]
    cc = cands[sub[f[i]]]
    j = int(np.searchsorted(cc, b["threshold"][i]))
    b["threshold"][i] = cc[j + 1] if j + 1 < cc.size else cc[j - 1]
    out.append(("threshold on the neighbouring candidate", b))
    b = {k: v.copy() for k, v in a.items()}
    i = next(i for i in splits if abs(a["value"][left[i]] - a["value"][right[i]]) > 1e-3)
    b["left"][i], b["right"][i] = a["right"][i], a["left"][i]
    out.append(("children swapped", b))
    b = {k: v.copy() for k, v in a.items()}
    cw = (np.ones(r.size) if c is None else c.astype(np.float64)) * (np.ones(r.size) if w is None else w)
    ib = np.flatnonzero(cw > 0) if c is not None else np.arange(r.size)
    cand = T._node_search(R, [cands[j].size for j in sub], ib, np.ones(r.size) if c is None else c.astype(np.float64),
                          cw, r.astype(np.float64), params, cw.sum())
    g, k2, j2 = next(x for x in cand if x[1] != f[0])
    assert cand[0][0] - g > 1e-6
    b["feature"][0], b["threshold"][0] = k2, cands[sub[k2]][j2]
    out.append(("root split on the runner-up column", b))
    for i in splits:  # the value stays fp32(S/W) of the node's rows: only the missing split is wrong
        out.append((f"internal node {i} collapsed into a leaf", T.cut(a, i)[0]))
    return out


@pytest.mark.parametrize("seed,weighted,bagged", [(0, False, False), (1, True, False), (2, True, True)])
def test_audit_passes_restatement_fits_and_fails_each_corruption(seed, weighted, bagged):
    a, X, cands, sub, r, w, c, params, pred, R = _audit_problem(seed, weighted, bagged)
    assert T.audit(a, X, cands, sub, r, w, c, params, out=pred.astype(np.float32)) == a["feature"].size
    for name, b in _mutations(a, X, cands, sub, r, w, c, params, R):
        with pytest.raises(AssertionError):
            T.audit(b, X, cands, sub, r, w, c, params)
            pytest.fail(f"the audit accepted: {name}")


def test_audit_exact_and_degenerate_fits():
    """Dyadic data: values exact, so a 1-ulp error fails; a root without in-bag weight is a NaN leaf; a pure node
    split by a rounding-positive gain passes (Spark's rule) while a false leaf with a real gain does not."""
    rng = np.random.default_rng(9)
    X = rng.integers(0, 8, (2000, 3)).astype(np.float32)
    r = (rng.integers(-8, 8, 2000) / 4).astype(np.float32)
    cands = [T.candidates(X[:, j], 8) for j in range(3)]
    sub = np.arange(3)
    R = [T.ranks(X[:, j], cands[j]) for j in sub]
    params = dict(max_depth=5)
    o = T.fit(R, [x.size for x in cands], r, max_depth=5)
    a = T.arrays(o, cands)
    T.audit(a, X, cands, sub, r, params=params, exact=True)
    b = {k: v.copy() for k, v in a.items()}
    i = np.flatnonzero((a["feature"] < 0) & (a["value"] != 0))[0]
    b["value"][i] = np.nextafter(b["value"][i], np.float32(np.inf))
    T.audit(b, X, cands, sub, r, params=params)  # 1 ulp passes on inexact data ...
    with pytest.raises(AssertionError):
        T.audit(b, X, cands, sub, r, params=params, exact=True)  # ... not on exact data
    leaf = {"feature": np.array([-1], np.int32), "threshold": np.zeros(1, np.float32), "left": np.zeros(1, np.int32),
            "right": np.zeros(1, np.int32), "value": np.array([np.nan], np.float32), "gain": np.zeros(1)}
    T.audit(leaf, X, cands, sub, r, counts=np.zeros(2000, np.float32), params=params)
    T.audit(leaf, X, cands, sub, r, w=np.zeros(2000, np.float32), params=params)
    with pytest.raises(AssertionError):  # the root has a real split: a leaf there is wrong
        T.audit(dict(leaf, value=np.float32([r.astype(np.float64).mean()])), X, cands, sub, r, params=params)
    # a pure node (quantile residuals {0.9, -0.1} all equal) split on a noise-level gain passes the audit
    q = np.float32(0.9) * np.ones(64, np.float32)
    Xq = np.arange(64, dtype=np.float32)[:, None]
    cq = [T.candidates(Xq[:, 0], 4)]
    t1 = {"feature": np.array([0, -1, -1], np.int32), "threshold": np.array([cq[0][0], 0, 0], np.float32),
          "left": np.array([1, 0, 0], np.int32), "right": np.array([2, 0, 0], np.int32),
          "value": np.full(3, q[0], np.float32), "gain": np.array([1e-18, 0, 0])}
    T.audit(t1, Xq, cq, [0], q, params=dict(max_depth=1))


# ---- Params ----------------------------------------------------------------------------------------------------
def test_device_learner_params():
    m = Lr.DeviceDecisionTreeRegressor()
    assert (m.maxDepth, m.maxBins, m.minInstancesPerNode, m.minInfoGain, m.minWeightFractionPerNode) == (5, 32, 1, 0.0, 0.0)
    from spark_ensemble_b200.ensemble import java_string_hash
    assert m.seed == java_string_hash("org.apache.spark.ml.regression.DecisionTreeRegressor")
    c = m.copy({"maxDepth": 3})
    assert c.maxDepth == 3 and m.maxDepth == 5 and c.maxBins == 32
    for bad in ({"maxDepth": 9}, {"maxDepth": -1}, {"maxBins": 1}, {"maxBins": 257}, {"minInstancesPerNode": 0},
                {"minWeightFractionPerNode": 0.5}, {"minWeightFractionPerNode": -0.1}):
        with pytest.raises(ValueError):
            Lr.DeviceDecisionTreeRegressor(**bad)


def test_device_model_host_predict_walk():
    arrays = {"feature": np.array([1, -1, 0, -1, -1], np.int32), "threshold": np.array([0.5, 0, 2.0, 0, 0], np.float32),
              "left": np.array([1, 0, 3, 0, 0], np.int32), "right": np.array([2, 0, 4, 0, 0], np.int32),
              "value": np.array([0, 10, 0, 20, 30], np.float32), "gain": np.zeros(5)}
    m = Lr.DeviceDecisionTreeRegressionModel(arrays)
    X = np.array([[0, 0.5], [0, 0.6], [2, 1], [3, 1], [0, np.nan], [np.nan, 9]], dtype=np.float32)
    assert m.predict(X).tolist() == [10, 20, 20, 30, 20, 30]  # NaN goes right at every node


def test_gbm_rejects_device_learner_without_resident_features():
    from spark_ensemble_b200.ensemble import DataFrame
    from spark_ensemble_b200.regression import GBMRegressor
    rng = np.random.default_rng(0)
    df = DataFrame(features=rng.standard_normal((50, 3)).astype(np.float32), label=rng.standard_normal(50))
    g = GBMRegressor().set("baseLearner", Lr.DeviceDecisionTreeRegressor(maxDepth=2)).set("numBaseLearners", 2)
    with pytest.raises(ValueError, match="residentFeatures"):
        g.fit(df)
    g.set("residentFeatures", True).set("devices", [0, 1])
    with pytest.raises(ValueError, match="devices"):
        g.fit(df)
