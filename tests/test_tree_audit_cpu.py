"""The chunked audit of a fitted tree (oracle/tree_audit.py): the OpenMP accumulator of per-node statistics against
numpy, for any chunking, and its verdicts against np_tree.audit / np_tree_cls.audit on fits of the restatements and on
trees with one thing wrong."""
import numpy as np
import pytest

from oracle import np_tree as T
from oracle import np_tree_cls as TC
from oracle import tree_audit as TA


@pytest.fixture(scope="module")
def orc():
    from oracle.oracle import Oracle
    return Oracle(omp=True)


def _chunks(R, lab, w, c, bounds):
    """A chunks() function over in-memory rows, cut at `bounds`."""
    R = np.stack(R).astype(np.uint8)
    edges = [0] + list(bounds) + [lab.size]

    def gen():
        for a, b in zip(edges[:-1], edges[1:]):
            yield (np.ascontiguousarray(R[:, a:b]), lab[a:b].astype(np.float64),
                   None if w is None else w[a:b].astype(np.float64), None if c is None else c[a:b].astype(np.float64))
    return gen


def test_ranks_and_walk_match_numpy(orc):
    rng = np.random.default_rng(1)
    x = rng.standard_normal(10_001).astype(np.float32)
    x[::97] = np.nan
    x[5], x[6] = -0.0, np.inf
    cands = np.sort(np.append(rng.standard_normal(39), 0.0)).astype(np.float32)
    x[7:9] = cands[3], np.nextafter(cands[3], np.float32(np.inf))  # on a candidate, one ulp past it
    np.testing.assert_array_equal(orc.ranks(x, cands), T.ranks(x, cands))
    np.testing.assert_array_equal(orc.ranks(x, cands[:0]), T.ranks(x, cands[:0]))
    X = rng.standard_normal((3000, 4)).astype(np.float32)
    cc = [T.candidates(X[:, j], 16) for j in range(4)]
    R = [T.ranks(X[:, j], cc[j]) for j in range(4)]
    o = T.fit(R, [c.size for c in cc], X[:, 0] * X[:, 2] + X[:, 3], max_depth=4)
    leaf = orc.tree_walk(np.stack(R).astype(np.uint8), o["feature"], o["bin"], o["left"], o["right"])
    np.testing.assert_array_equal(o["pred"][leaf], T.predict(o, R))


@pytest.mark.parametrize("K,weighted,bagged", [(0, False, False), (0, True, True), (5, True, False), (2, False, True)])
def test_accumulator_equals_bincount_for_any_chunking(orc, K, weighted, bagged):
    """Random ranks and a node list with alternative splits of one node (a row reaches several children): the C sums
    equal numpy's per node, column and rank, and do not depend on the chunking beyond fp64 reassociation."""
    rng = np.random.default_rng(10 + K)
    n, S = 20_000, 6
    R = [rng.integers(0, 40, n).astype(np.int64) for _ in range(S)]
    R[2][rng.random(n) < 0.05] = 255  # NaN ranks
    lab = rng.integers(0, K, n).astype(np.float32) if K else rng.standard_normal(n).astype(np.float32)
    w = rng.uniform(0.25, 4.0, n).astype(np.float32) if weighted else None
    c = rng.integers(0, 3, n).astype(np.float32) if bagged else None
    nodes = T.Nodes()
    a = nodes.child(0, 1, 17, 1)
    nodes.child(0, 1, 17, 0)
    nodes.child(a, 4, 5, 0)
    nodes.child(a, 2, 30, 1)  # two different splits of node a
    b = nodes.child(0, 3, 2, 1)  # a second split of the root
    nodes.child(b, 3, 0, 0)
    want = {0, 1, 3, 4, 5, 6}
    tot0, h0 = T.row_stats(R, K, lab, w, c)(nodes, want)
    for bounds in ([], [1], [7777, 7778, 15000], list(range(1000, n, 1000))):
        tot, h = TA.chunk_stats(orc, _chunks(R, lab, w, c, bounds), S, K)(nodes, want)
        np.testing.assert_allclose(tot, tot0, rtol=1e-12, atol=1e-9)
        assert set(h) == want
        for v in want:
            np.testing.assert_allclose(h[v], h0[v], rtol=1e-12, atol=1e-9)
    assert tot0[5, -1] > 0 and tot0[6, -1] > 0 and 0 < tot0[3, -1] + tot0[4, -1]


def _reg_problem(seed, weighted, bagged):
    rng = np.random.default_rng(500 + seed)
    n, d = 3000, 5
    X = rng.standard_normal((n, d)).astype(np.float32)
    X[rng.random((n, d)) < 0.03] = np.nan
    z = np.nan_to_num(X)
    r = (np.sin(2 * z[:, 1]) + z[:, 3] ** 2 + 0.3 * rng.standard_normal(n)).astype(np.float32)
    w = rng.uniform(0.25, 4.0, n).astype(np.float32) if weighted else None
    c = rng.integers(0, 3, n).astype(np.float32) if bagged else None
    cands = [T.candidates(X[:, j], 32) for j in range(d)]
    sub = np.array([4, 1, 0, 3], np.int32)
    R = [T.ranks(X[:, j], cands[j]) for j in sub]
    params = dict(max_depth=4, min_instances=1, min_info_gain=0.0, min_weight_fraction=0.0)
    o = T.fit(R, [cands[j].size for j in sub], r, w=w, counts=c, **params)
    return T.arrays(o, [cands[j] for j in sub]), X, cands, sub, r, w, c, params, R


def _cls_problem(seed, K, kind, weighted, bagged):
    rng = np.random.default_rng(600 + seed)
    n, d = 4000, 5
    X = rng.standard_normal((n, d)).astype(np.float32)
    z = np.sin(2 * X[:, 1]) + X[:, 3] ** 2 + 0.4 * rng.standard_normal(n)
    y = np.minimum(np.digitize(z, np.quantile(z, np.linspace(0, 1, K + 1)[1:-1])), K - 1).astype(np.float32)
    w = rng.uniform(0.25, 4.0, n).astype(np.float32) if weighted else None
    c = rng.integers(0, 3, n).astype(np.float32) if bagged else None
    cands = [T.candidates(X[:, j], 32) for j in range(d)]
    sub = np.array([4, 1, 0, 3], np.int32)
    R = [T.ranks(X[:, j], cands[j]) for j in sub]
    params = dict(num_classes=K, impurity=kind, max_depth=4, min_instances=1, min_info_gain=0.0,
                  min_weight_fraction=0.0)
    o = TC.fit(R, [cands[j].size for j in sub], y, K, w=w, counts=c, impurity_kind=kind, max_depth=4)
    return TC.arrays(o, [cands[j] for j in sub]), X, cands, sub, y, w, c, params, R


def _mutations(a, cands, sub, classifier):
    """The tree with one thing wrong: (name, arrays)."""
    f = a["feature"]
    splits, leaves = np.flatnonzero(f >= 0), np.flatnonzero(f < 0)
    out = []
    b = {k: v.copy() for k, v in a.items()}
    cc = cands[sub[f[0]]]
    j = int(np.searchsorted(cc, b["threshold"][0]))
    b["threshold"][0] = cc[j + 1] if j + 1 < cc.size else cc[j - 1]
    out.append(("root threshold on the next candidate", b))
    b = {k: v.copy() for k, v in a.items()}
    if classifier:
        i = next(i for i in leaves if b["values"][i].max() > 0.1)
        kk = int(np.argmax(b["values"][i]))
        b["values"][i, kk] += 4 * np.spacing(b["values"][i, kk])
    else:
        i = leaves[0]
        b["value"][i] = np.float32(b["value"][i]) + 4 * np.spacing(np.float32(b["value"][i]))
    out.append(("a leaf value 4 ulps off", b))
    b = {k: v.copy() for k, v in a.items()}
    others = [k for k in range(len(sub)) if k != f[0] and cands[sub[k]].size]
    k2 = others[0]
    b["feature"][0], b["threshold"][0] = k2, cands[sub[k2]][cands[sub[k2]].size // 2]
    out.append(("root split on another column", b))
    for i in splits:
        b, q = T.cut(a, i)
        if classifier:
            b["value"][q] = TC.label_of(b["class_weights"][q])
        out.append((f"internal node {i} made a leaf", b))
    return out


@pytest.mark.parametrize("seed,weighted,bagged", [(0, False, False), (1, True, False), (2, True, True)])
def test_chunked_audit_agrees_on_regression_fits(orc, seed, weighted, bagged):
    a, X, cands, sub, r, w, c, params, R = _reg_problem(seed, weighted, bagged)
    chunks = _chunks(R, r, w, c, [999, 2000])
    cs = [cands[j] for j in sub]
    leaves = []
    assert TA.audit(a, chunks, cs, params, orc, out=leaves.append) == T.audit(a, X, cands, sub, r, w, c, params) == \
        a["feature"].size
    np.testing.assert_array_equal(np.concatenate(leaves), T.leaf_of(a, R, T.bins_of(a, cs)))
    for name, b in _mutations(a, cands, sub, False):
        verdicts = []
        for run in (lambda: T.audit(b, X, cands, sub, r, w, c, params), lambda: TA.audit(b, chunks, cs, params, orc)):
            try:
                run()
                verdicts.append(True)
            except AssertionError:
                verdicts.append(False)
        assert verdicts == [False, False], (name, verdicts)


@pytest.mark.parametrize("seed,K,kind,weighted,bagged", [(0, 3, "gini", False, False), (1, 5, "entropy", True, False),
                                                         (2, 2, "gini", True, True), (3, 26, "entropy", False, True)])
def test_chunked_audit_agrees_on_classification_fits(orc, seed, K, kind, weighted, bagged):
    a, X, cands, sub, y, w, c, params, R = _cls_problem(seed, K, kind, weighted, bagged)
    chunks = _chunks(R, y, w, c, [1234])
    cs = [cands[j] for j in sub]
    assert TA.audit(a, chunks, cs, params, orc, num_classes=K) == TC.audit(a, X, cands, sub, y, w, c, params) == \
        a["feature"].size
    for name, b in _mutations(a, cands, sub, True):
        verdicts = []
        for run in (lambda: TC.audit(b, X, cands, sub, y, w, c, params),
                    lambda: TA.audit(b, chunks, cs, params, orc, num_classes=K)):
            try:
                run()
                verdicts.append(True)
            except AssertionError:
                verdicts.append(False)
        assert verdicts == [False, False], (name, verdicts)


def test_chunked_audit_grows_pruned_subtrees():
    """A pruned leaf of a classifier fit is checked by growing, round by round, what the fit may have grown below
    it: the chunked audit asks for those nodes' statistics and agrees with the in-memory audit."""
    from oracle.oracle import Oracle
    orc = Oracle(omp=True)
    rng = np.random.default_rng(7)
    n = 6000
    X = rng.standard_normal((n, 3)).astype(np.float32)
    y = (X[:, 0] > 0).astype(np.float32)
    noise = rng.random(n) < 0.1
    y[noise] = rng.integers(0, 3, noise.sum())
    cands = [T.candidates(X[:, j], 16) for j in range(3)]
    R = [T.ranks(X[:, j], cands[j]) for j in range(3)]
    params = dict(num_classes=3, impurity="gini", max_depth=4)
    o = TC.fit(R, [c.size for c in cands], y, 3, max_depth=4)
    assert o["merged"].any()
    a = TC.arrays(o, cands)
    calls = []
    stats = TA.chunk_stats(orc, _chunks(R, y, None, None, [3000]), 3, 3)

    def counted(nodes, want):
        calls.append(len(want))
        return stats(nodes, want)
    TC.check(a, T.bins_of(a, cands), [c.size for c in cands], counted, params)
    assert len(calls) >= 2, calls
    TC.audit(a, X, cands, np.arange(3), y, params=params)
