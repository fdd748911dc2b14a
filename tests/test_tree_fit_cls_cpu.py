"""CPU checks of the classification-tree learner's specification (DESIGN.md §3 "Device classification-tree fit"): the
numpy restatement in oracle/np_tree_cls.py against scikit-learn's exact tree and against brute force, a hand-worked
cascade of pruning merges, the validity rules, and the learner's Params."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import np_tree as T
from oracle import np_tree_cls as TC
from spark_ensemble_b200 import learners as Lr


def _fit_cols(X, y, K, max_bins=256, **kw):
    cands = [T.candidates(X[:, j], max_bins) for j in range(X.shape[1])]
    ranks = [T.ranks(X[:, j], cands[j]) for j in range(X.shape[1])]
    return TC.fit(ranks, [c.size for c in cands], y, K, **kw), cands, ranks


def _sk_leaves(t, j):
    if t.children_left[j] < 0:
        return [j]
    return _sk_leaves(t, t.children_left[j]) + _sk_leaves(t, t.children_right[j])


def _sk_dist(t, j):
    v = t.value[j, 0].astype(np.float64)
    return v / v.sum()


def _walk_equal_sklearn(tree, cands, sk, X, rows, i=0, j=0):
    """Same partition at every split; a leaf of the restatement is a leaf of scikit-learn with the same label and
    probabilities, or (pruned) a scikit-learn subtree whose leaves all carry its label and whose root has its
    probabilities.  Near ties are skipped: scikit-learn breaks them at random."""
    t = sk.tree_
    info = tree["info"][i]
    if info is not None and np.isfinite(info[0]) and info[0] - info[1] <= 1e-9 * abs(info[0]):
        return 0
    if tree["feature"][i] < 0:
        for leaf in _sk_leaves(t, j):
            assert int(np.argmax(t.value[leaf, 0])) == tree["label"][i]
        if not tree["merged"][i]:
            assert t.children_left[j] < 0
        np.testing.assert_allclose(tree["proba"][i], _sk_dist(t, j), rtol=1e-6, atol=1e-7)
        return 1
    assert t.children_left[j] >= 0
    f = tree["feature"][i]
    go = X[rows, f] <= cands[f][tree["bin"][i]]
    np.testing.assert_array_equal(go, X[rows, t.feature[j]] <= Lr._floor_f32(np.array([t.threshold[j]]))[0])
    return (1 + _walk_equal_sklearn(tree, cands, sk, X, rows[go], tree["left"][i], t.children_left[j])
            + _walk_equal_sklearn(tree, cands, sk, X, rows[~go], tree["right"][i], t.children_right[j]))


@pytest.mark.parametrize("seed,depth,K,impurity,weighted", [(0, 3, 2, "gini", False), (1, 4, 3, "entropy", False),
                                                            (2, 5, 4, "gini", True), (3, 3, 3, "entropy", True)])
def test_oracle_equals_sklearn_exact_tree(seed, depth, K, impurity, weighted):
    """Every midpoint a candidate and continuous data: the restatement is an exact CART classification tree,
    scikit-learn's, up to Spark's pruning of equal-label leaf siblings."""
    from sklearn.tree import DecisionTreeClassifier
    rng = np.random.default_rng(seed)
    n, d = 200, 3
    X = rng.standard_normal((n, d)).astype(np.float32)
    z = X[:, 0] * 2 + np.sin(3 * X[:, 1]) + 0.7 * rng.standard_normal(n)
    y = np.digitize(z, np.quantile(z, np.linspace(0, 1, K + 1)[1:-1])).astype(np.float32)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32) if weighted else None
    tree, cands, _ = _fit_cols(X, y, K, max_depth=depth, impurity_kind=impurity)
    assert all(c.size == n - 1 for c in cands)
    sk = DecisionTreeClassifier(criterion=impurity, max_depth=depth, random_state=0).fit(
        X, y.astype(int), sample_weight=None if w is None else w.astype(np.float64))
    if weighted:
        tree, _, _ = _fit_cols(X, y, K, max_depth=depth, impurity_kind=impurity, w=w)
    compared = _walk_equal_sklearn(tree, cands, sk, X, np.arange(n))
    assert compared >= 3


def _brute(ranks, ncand, y, c, K, depth, max_depth, kind):
    """Direct recursion over every (column, candidate) with masked sums and Spark's pruning: no histograms."""
    n = (np.eye(K)[y] * c[:, None]).sum(axis=0)
    if depth == max_depth:
        return ("leaf", TC.label_of(n), TC.proba_of(n))
    imp = TC.impurity(n, kind)
    best = None
    for k in range(len(ranks)):
        for j in range(ncand[k]):
            m = ranks[k] <= j
            cl, cr = c * m, c * ~m
            if cl.sum() < 1 or cr.sum() < 1:
                continue
            nl, nr = (np.eye(K)[y] * cl[:, None]).sum(axis=0), (np.eye(K)[y] * cr[:, None]).sum(axis=0)
            tw = nl.sum() + nr.sum()
            g = imp - nl.sum() / tw * TC.impurity(nl, kind) - nr.sum() / tw * TC.impurity(nr, kind)
            if best is None or g > best[0]:
                best = (g, k, j, cl, cr, nl, nr)
    if best is None or best[0] <= 0:
        return ("leaf", TC.label_of(n), TC.proba_of(n))
    g, k, j, cl, cr, nl, nr = best
    kids = []
    for cc, nn in ((cl, nl), (cr, nr)):
        if depth + 1 == max_depth or abs(TC.impurity(nn, kind)) < T.EPS:
            kids.append(("leaf", TC.label_of(nn), TC.proba_of(nn)))
        else:
            kids.append(_brute(ranks, ncand, y, cc, K, depth + 1, max_depth, kind))
    if kids[0][0] == kids[1][0] == "leaf" and kids[0][1] == kids[1][1]:
        return ("leaf", kids[0][1], TC.proba_of(n))  # the children's label, the node's own distribution
    return ("split", k, j, kids[0], kids[1])


def _as_nested(tree, i=0):
    if tree["feature"][i] < 0:
        return ("leaf", int(tree["label"][i]), tree["proba"][i])
    return ("split", int(tree["feature"][i]), int(tree["bin"][i]), _as_nested(tree, tree["left"][i]),
            _as_nested(tree, tree["right"][i]))


def _same(a, b):
    if a[0] != b[0]:
        return False
    if a[0] == "leaf":
        return a[1] == b[1] and np.array_equal(a[2], b[2])
    return a[1:3] == b[1:3] and _same(a[3], b[3]) and _same(a[4], b[4])


@pytest.mark.parametrize("seed", range(8))
def test_oracle_equals_brute_force(seed):
    rng = np.random.default_rng(200 + seed)
    n, K = 12, 2 + seed % 3
    X = rng.integers(0, 5, (n, 2)).astype(np.float32)
    y = rng.integers(0, K, n)
    c = rng.integers(0, 3, n).astype(np.float32) if seed % 2 else np.ones(n, dtype=np.float32)
    cands = [T.candidates(X[:, j], 3) for j in range(2)]
    ranks = [np.asarray(T.ranks(X[:, j], cands[j])) for j in range(2)]
    kind = "gini" if seed < 4 else "entropy"
    for max_depth in (1, 2, 3):
        tree = TC.fit(ranks, [x.size for x in cands], y, K, counts=c, max_depth=max_depth, impurity_kind=kind)
        brute = _brute(ranks, [x.size for x in cands], y, c.astype(np.float64), K, 0, max_depth, kind)
        assert _same(_as_nested(tree), brute), (_as_nested(tree), brute)


def _groups(spec):
    """Rows from {(x0, x1): (count of class 0, count of class 1)}."""
    X, y = [], []
    for (a, b), counts in spec.items():
        for k, m in enumerate(counts):
            X += [(a, b)] * m
            y += [k] * m
    return np.asarray(X, dtype=np.float32), np.asarray(y, dtype=np.float32)


def test_hand_worked_cascade_of_merges():
    """x0 splits the root ([8, 4], gini gain 0.0254 against 0.0069 for x1), then x1 splits both halves:
    [4, 1] -> [2, 0] | [2, 1] and [4, 3] -> [3, 3] | [1, 0].  All four leaves have label 0 (a [3, 3] tie goes to the
    first class), so both halves merge, and then the root: one leaf, label 0, with the ROOT's distribution."""
    X, y = _groups({(0, 0): (2, 0), (0, 1): (2, 1), (1, 0): (3, 3), (1, 1): (1, 0)})
    t, _, _ = _fit_cols(X, y, 2, max_depth=2)
    assert t["feature"].tolist() == [-1] and t["label"].tolist() == [0] and t["merged"].tolist() == [True]
    np.testing.assert_array_equal(t["proba"][0], np.float32([8 / 12, 4 / 12]))
    assert abs(t["info"][0][0] - (36 / 121 * 0 + 4 / 9 - (5 / 12 * 0.32 + 7 / 12 * 24 / 49))) < 1e-12
    # maxDepth 1: the root's children [4, 1] and [4, 3] are leaves with label 0: one merge, same leaf
    t1, _, _ = _fit_cols(X, y, 2, max_depth=1)
    assert t1["feature"].tolist() == [-1] and t1["label"].tolist() == [0]
    # one class-1 row instead of the class-0 row at (1, 1): [3, 4] -> [3, 3] | [0, 1] keeps its split (labels 0 | 1)
    # while [4, 1] still merges into a leaf with ITS distribution [0.8, 0.2], not a child's ([1, 0] or [2/3, 1/3])
    X2, y2 = _groups({(0, 0): (2, 0), (0, 1): (2, 1), (1, 0): (3, 3), (1, 1): (0, 1)})
    t2, _, _ = _fit_cols(X2, y2, 2, max_depth=2)
    assert t2["feature"][0] == 0
    left = t2["left"][0]
    assert t2["feature"][left] == -1 and t2["merged"][left] and t2["label"][left] == 0
    np.testing.assert_array_equal(t2["proba"][left], np.float32([0.8, 0.2]))
    right = t2["right"][0]
    assert t2["feature"][right] == 1


def test_impurities_and_label_rule():
    assert TC.impurity([0, 0, 0], "gini") == 0.0 and TC.impurity([0, 0], "entropy") == 0.0
    assert TC.impurity([5, 0], "gini") == 0.0 and TC.impurity([0, 5], "entropy") == 0.0
    assert abs(TC.impurity([1, 1], "gini") - 0.5) < 1e-15 and abs(TC.impurity([2, 2], "entropy") - 1.0) < 1e-15
    assert abs(TC.impurity([1, 1, 1, 1], "entropy") - 2.0) < 1e-15
    assert TC.label_of([1, 3, 3]) == 1 and TC.label_of([0, 0]) == 0
    np.testing.assert_array_equal(TC.proba_of([0, 0, 0]), np.zeros(3, np.float32))  # W == 0: all-zero probabilities
    np.testing.assert_array_equal(TC.proba_of([1, 2]), np.float32([1 / 3, 2 / 3]))


def test_validity_rules_bind():
    rng = np.random.default_rng(5)
    n = 300
    X = rng.standard_normal((n, 2)).astype(np.float32)
    y = ((X[:, 0] > 1.2) | (rng.random(n) < 0.05)).astype(np.float32)
    base, cands, ranks = _fit_cols(X, y, 2, max_bins=64, max_depth=1)
    assert base["feature"][0] == 0
    small = int(min((ranks[0] <= base["bin"][0]).sum(), (ranks[0] > base["bin"][0]).sum()))
    t, _, _ = _fit_cols(X, y, 2, max_bins=64, max_depth=1, min_instances=small + 1)
    assert t["feature"].size == 1 or t["bin"][0] != base["bin"][0] or t["feature"][0] != base["feature"][0]
    t, _, _ = _fit_cols(X, y, 2, max_bins=64, max_depth=1, min_info_gain=base["gain"][0] * 1.01)
    assert t["feature"].size == 1
    t, _, _ = _fit_cols(X, y, 2, max_bins=64, max_depth=1, min_weight_fraction=0.3)
    if t["feature"][0] >= 0:
        f = t["feature"][0]
        lw = (T.ranks(X[:, f], T.candidates(X[:, f], 64)) <= t["bin"][0]).mean()
        assert 0.3 <= lw <= 0.7
    t, _, _ = _fit_cols(X, y, 2, max_depth=0)
    assert t["feature"].tolist() == [-1]
    np.testing.assert_array_equal(t["proba"][0], np.float32([(y == 0).mean(), (y == 1).mean()]))


# ---- the audit of a fitted tree (oracle/np_tree_cls.audit) ----------------------------------------------------
@pytest.mark.parametrize("seed,K,kind,weighted,bagged", [(0, 3, "gini", False, False), (1, 5, "entropy", True, False),
                                                         (2, 2, "gini", True, True), (3, 26, "entropy", False, True)])
def test_audit_passes_restatement_fits_and_fails_each_corruption(seed, K, kind, weighted, bagged):
    rng = np.random.default_rng(400 + seed)
    n, d = 4000, 5
    X = rng.standard_normal((n, d)).astype(np.float32)
    X[rng.random((n, d)) < 0.03] = np.nan
    z = np.sin(2 * np.nan_to_num(X[:, 1])) + np.nan_to_num(X[:, 3]) ** 2 + 0.4 * rng.standard_normal(n)
    y = np.minimum(np.digitize(z, np.quantile(z, np.linspace(0, 1, K + 1)[1:-1])), K - 1).astype(np.float32)
    w = rng.uniform(0.25, 4.0, n).astype(np.float32) if weighted else None
    c = rng.poisson(1.0, n).astype(np.float32) if bagged else None
    cands = [T.candidates(X[:, j], 32) for j in range(d)]
    sub = np.array([4, 1, 0, 3], np.int32)
    R = [T.ranks(X[:, j], cands[j]) for j in sub]
    params = dict(num_classes=K, impurity=kind, max_depth=4, min_instances=1, min_info_gain=0.0,
                  min_weight_fraction=0.0)
    o = TC.fit(R, [cands[j].size for j in sub], y, K, w=w, counts=c, impurity_kind=kind, max_depth=4)
    a = TC.arrays(o, [cands[j] for j in sub])
    leaf = TC.leaf_of(o, R)
    assert TC.audit(a, X, cands, sub, y, w, c, params, out=o["label"][leaf], out_proba=o["proba"][leaf].T) == \
        a["feature"].size
    f = a["feature"]
    splits, leaves = np.flatnonzero(f >= 0), np.flatnonzero(f < 0)
    muts = []
    b = {k: v.copy() for k, v in a.items()}
    i = next(i for i in leaves if b["values"][i].max() > 0.1)
    kk = int(np.argmax(b["values"][i]))
    b["values"][i, kk] += 4 * np.spacing(b["values"][i, kk])
    muts.append(("probability + 4 ulps", b))
    b = {k: v.copy() for k, v in a.items()}
    cc = cands[sub[f[0]]]
    j = int(np.searchsorted(cc, b["threshold"][0]))
    b["threshold"][0] = cc[j + 1] if j + 1 < cc.size else cc[j - 1]
    muts.append(("threshold on the neighbouring candidate", b))
    b = {k: v.copy() for k, v in a.items()}
    i = splits[0]
    b["left"][i], b["right"][i] = a["right"][i], a["left"][i]
    muts.append(("children swapped", b))
    b = {k: v.copy() for k, v in a.items()}
    cw = (np.ones(n) if c is None else c.astype(np.float64)) * (np.ones(n) if w is None else w)
    ib = np.flatnonzero(cw > 0)
    cnt = np.ones(n) if c is None else c.astype(np.float64)
    gains = []
    for k in range(len(R)):
        g = TC._column_gains(R[k][ib], y.astype(np.int64)[ib], cnt[ib], cw[ib], K, cands[sub[k]].size, kind, params,
                             cw.sum())
        gains += [(float(g[jj]), k, int(jj)) for jj in np.flatnonzero(np.isfinite(g))]
    gains.sort(key=lambda x: (-x[0], x[1], x[2]))
    g2, k2, j2 = next(x for x in gains if x[1] != f[0])
    assert gains[0][0] - g2 > 1e-6
    b["feature"][0], b["threshold"][0] = k2, cands[sub[k2]][j2]
    muts.append(("root split on the runner-up column", b))
    b = {k: v.copy() for k, v in a.items()}
    b["class_weights"][0, int(np.argmax(b["class_weights"][0]))] *= 1 + 1e-9
    muts.append(("class weight x (1 + 1e-9)", b))
    b = {k: v.copy() for k, v in a.items()}
    i = next(i for i in leaves if np.sort(b["values"][i])[-1] - np.sort(b["values"][i])[-2] > 0.01)
    b["value"][i] = np.argsort(b["values"][i])[-2]
    muts.append(("label of the second-largest class", b))
    for i in splits:  # a pruned tree's internal nodes all have leaves of two labels below them
        b, q = T.cut(a, i)
        b["value"][q] = TC.label_of(b["class_weights"][q])
        muts.append((f"internal node {i} collapsed into a leaf with its own statistics", b))
    for name, b in muts:
        with pytest.raises(AssertionError):
            TC.audit(b, X, cands, sub, y, w, c, params)
            pytest.fail(f"the audit accepted: {name}")


def test_audit_merged_leaf_and_zero_weight_root():
    """The hand-worked cascade (one merged leaf with the root's distribution) passes; the same leaf with a child's
    distribution, or with a label the subtree does not give, fails.  A root without in-bag weight is label 0 with
    all-zero probabilities."""
    X, y = _groups({(0, 0): (2, 0), (0, 1): (2, 1), (1, 0): (3, 3), (1, 1): (1, 0)})
    cands = [T.candidates(X[:, j], 256) for j in range(2)]
    R = [T.ranks(X[:, j], cands[j]) for j in range(2)]
    o = TC.fit(R, [x.size for x in cands], y, 2, max_depth=2)
    a = TC.arrays(o, cands)
    params = dict(num_classes=2, max_depth=2)
    assert TC.audit(a, X, cands, [0, 1], y, params=params, exact=True) == 1
    b = {k: v.copy() for k, v in a.items()}
    b["values"][0] = np.float32([1.0, 0.0])
    b["class_weights"][0] = [2.0, 0.0]
    with pytest.raises(AssertionError):
        TC.audit(b, X, cands, [0, 1], y, params=params)
    # the same data with the (1, 1) row of class 1: the root keeps its split, a leaf there is wrong
    X2, y2 = _groups({(0, 0): (2, 0), (0, 1): (2, 1), (1, 0): (3, 3), (1, 1): (0, 1)})
    with pytest.raises(AssertionError):
        TC.audit(dict(a, class_weights=np.array([[7.0, 5.0]]), values=np.float32([[7 / 12, 5 / 12]])), X2, cands,
                 [0, 1], y2, params=params)
    zero = dict(a, class_weights=np.zeros((1, 2)), values=np.zeros((1, 2), np.float32), value=np.zeros(1, np.float32))
    TC.audit(zero, X, cands, [0, 1], y, w=np.zeros(12, np.float32), params=params, exact=True)


@pytest.mark.parametrize("kind,weighted", [("gini", False), ("entropy", True)])
def test_audit_fails_every_wrongly_collapsed_subtree(kind, weighted):
    """Small deep nodes of integer labels meet near ties often.  A tie below an internal node must not excuse
    collapsing it: every internal node of restatement fits, made a leaf with its own statistics, fails the audit."""
    collapsed = 0
    for seed in range(6):
        rng = np.random.default_rng(500 + seed)
        n, d, K = 1500, 4, 3
        X = rng.standard_normal((n, d)).astype(np.float32)
        z = np.sin(2 * X[:, 0]) + X[:, 1] * X[:, 2] + 0.5 * rng.standard_normal(n)
        y = np.minimum(np.digitize(z, np.quantile(z, [1 / 3, 2 / 3])), K - 1).astype(np.float32)
        w = rng.uniform(0.25, 4.0, n).astype(np.float32) if weighted else None
        cands = [T.candidates(X[:, j], 32) for j in range(d)]
        R = [T.ranks(X[:, j], cands[j]) for j in range(d)]
        o = TC.fit(R, [x.size for x in cands], y, K, w=w, impurity_kind=kind, max_depth=5)
        a = TC.arrays(o, cands)
        params = dict(num_classes=K, impurity=kind, max_depth=5)
        TC.audit(a, X, cands, np.arange(d), y, w, params=params)
        for i in np.flatnonzero(a["feature"] >= 0):
            b, q = T.cut(a, i)
            b["value"][q] = TC.label_of(b["class_weights"][q])
            with pytest.raises(AssertionError):
                TC.audit(b, X, cands, np.arange(d), y, w, params=params)
                pytest.fail(f"seed {seed}: the audit accepted internal node {i} collapsed into a leaf")
            collapsed += 1
    assert collapsed > 100


# ---- Params ----------------------------------------------------------------------------------------------------
def test_device_classifier_params():
    from spark_ensemble_b200.ensemble import java_string_hash
    m = Lr.DeviceDecisionTreeClassifier()
    assert (m.maxDepth, m.maxBins, m.impurity, m.minInstancesPerNode, m.minInfoGain, m.minWeightFractionPerNode) == \
        (5, 32, "gini", 1, 0.0, 0.0)
    assert m.seed == java_string_hash("org.apache.spark.ml.classification.DecisionTreeClassifier")
    c = m.copy({"maxDepth": 3, "impurity": "entropy"})
    assert c.maxDepth == 3 and c.impurity == "entropy" and m.maxDepth == 5 and m.impurity == "gini"
    for bad in ({"maxDepth": 9}, {"maxDepth": -1}, {"maxBins": 1}, {"maxBins": 257}, {"minInstancesPerNode": 0},
                {"minWeightFractionPerNode": 0.5}, {"minWeightFractionPerNode": -0.1}, {"impurity": "variance"}):
        with pytest.raises(ValueError):
            Lr.DeviceDecisionTreeClassifier(**bad)
    with pytest.raises(ValueError):
        m.copy({"maxDepth": 9})
    # the candidates are the regressor's: one implementation
    X = np.random.default_rng(0).standard_normal((500, 3)).astype(np.float32)
    r = Lr.DeviceDecisionTreeRegressor(maxBins=16, seed=3)
    k = Lr.DeviceDecisionTreeClassifier(maxBins=16, seed=3)
    for a, b in zip(r.split_candidates(X), k.split_candidates(X)):
        np.testing.assert_array_equal(a, b)


def test_device_classification_model_host_walk():
    arrays = {"feature": np.array([1, -1, -1], np.int32), "threshold": np.array([0.5, 0, 0], np.float32),
              "left": np.array([1, 0, 0], np.int32), "right": np.array([2, 0, 0], np.int32),
              "value": np.array([0, 1, 0], np.float32),
              "values": np.array([[0.5, 0.5], [0.25, 0.75], [1, 0]], np.float32), "gain": np.zeros(3),
              "class_weights": np.zeros((3, 2))}
    m = Lr.DeviceDecisionTreeClassificationModel(arrays, 2)
    X = np.array([[0, 0.5], [0, 0.6], [0, np.nan]], dtype=np.float32)
    assert m.predict(X).tolist() == [1, 0, 0]  # NaN goes right
    np.testing.assert_array_equal(m.predictProbability(X), [[0.25, 0.75], [1, 0], [1, 0]])
    assert set(m.tree_arrays()) == {"feature", "threshold", "left", "right", "value", "values"}


def test_standalone_fit_and_boosting_validate_on_the_host():
    from spark_ensemble_b200.classification import BoostingClassifier
    from spark_ensemble_b200.ensemble import DataFrame
    X = np.zeros((4, 2), np.float32)
    m = Lr.DeviceDecisionTreeClassifier(maxDepth=2)
    for y, K in (([0, 1, 2, 3], 3), ([0, 1, 0.5, 1], 2), ([0, -1, 0, 1], 2), ([0, 0, 0, 0], 1)):
        with pytest.raises(ValueError):
            m.fit(X, np.asarray(y, np.float64), num_classes=K)
    df = DataFrame(features=np.random.default_rng(0).standard_normal((40, 3)).astype(np.float32),
                   label=np.arange(40) % 2 * 1.0)
    b = BoostingClassifier().set("baseLearner", m).set("numBaseLearners", 2)
    with pytest.raises(ValueError, match="residentFeatures"):
        b.fit(df)
