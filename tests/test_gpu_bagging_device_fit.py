"""The forest fit (se_forest_fit: several trees over the same rows, labels, weights and bag, one subspace each, in
one launch sequence per batch) against one-tree fits in the same context, every tree audited from fp64 sums over the
rows each node receives, and BaggingRegressor / BaggingClassifier's device route against their member route."""
import numpy as np
import pytest

from oracle import np_tree as T
from oracle import np_tree_cls as TC

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    yield c
    c.close()


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _same_tree(got, want, K):
    for k in ("feature", "threshold", "left", "right"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    # a gain is a difference of impurities: fp64 atomic order moves it by ulps of the largest terms, not of itself
    np.testing.assert_allclose(got["gain"], want["gain"], rtol=1e-9, atol=1e-9 * np.abs(want["gain"]).max(initial=0))
    if K:
        np.testing.assert_array_equal(got["value"], want["value"])  # labels
        assert _ulps(got["values"], want["values"]).max(initial=0) <= 1
        np.testing.assert_allclose(got["class_weights"], want["class_weights"], rtol=1e-9, atol=1e-300)
    else:
        assert _ulps(got["value"], want["value"]).max(initial=0) <= 1


def _problem(ctx, n, d, K, rows, seed, max_bins=32):
    """Continuous features (no gain ties) with one constant column (no candidates), labels, weights and bag on the
    device; returns what the audits read."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(np.float32)
    X[:, d - 1] = 0.5
    z = np.sin(2 * X[:, 0]) + X[:, 1] ** 2 - X[:, 2] * X[:, 3] + 0.3 * rng.standard_normal(n)
    if K:
        y = np.digitize(z, np.quantile(z, np.linspace(0, 1, K + 1)[1:-1])).astype(np.float32)
    else:
        y = z.astype(np.float32)
    w = rng.uniform(0.25, 4.0, n).astype(np.float32) if rows in ("weighted", "weighted_bag") else None
    bag = rng.poisson(1.0, n).astype(np.float32) if rows in ("bag", "weighted_bag") else None
    cands = DeviceDecisionTreeRegressor(maxBins=max_bins, seed=3).split_candidates(X)
    assert cands[d - 1].size == 0
    ctx.alloc(N.SLOT_X, d, n)
    ctx.upload_rowmajor(N.SLOT_X, X)
    ctx.alloc(N.SLOT_Y, 1, n)
    ctx.upload(N.SLOT_Y, y)
    ctx.alloc(N.SLOT_H, 1, n)
    ctx.alloc(N.SLOT_PRED, 1, n)
    if w is not None:
        ctx.alloc(N.SLOT_W, 1, n)
        ctx.upload(N.SLOT_W, w)
    if bag is not None:
        ctx.alloc(N.SLOT_BAG, 1, n)
        ctx.upload(N.SLOT_BAG, bag)
    ctx.tree_fit_bins(cands)
    return X, y, w, bag, cands


def _fits(ctx, subs, K, impurity, w, bag, depth):
    """The forest fit and the one-tree fit of every subspace, same context, same arguments."""
    from spark_ensemble_b200 import _native as N
    wslot = N.SLOT_W if w is not None else -1
    kw = dict(max_depth=depth, min_instances=1, min_info_gain=0.0, min_weight_fraction=0.0)
    forest = ctx.forest_fit(subs, N.SLOT_Y, 0, wslot, 0, bag is not None, num_classes=K, impurity=impurity, **kw)
    assert len(forest) == len(subs)
    single = []
    for s in subs:
        if K:
            single.append(ctx.tree_fit_classifier(N.SLOT_Y, K, 0, wslot, 0, bag is not None, subspace=s,
                                                  impurity=impurity, out_slot=N.SLOT_PRED, **kw))
        else:
            single.append(ctx.tree_fit(N.SLOT_Y, 0, wslot, 0, bag is not None, subspace=s, out_slot=N.SLOT_H, **kw))
    return forest, single


def _audit(tree, X, cands, sub, y, w, bag, K, impurity, depth):
    params = dict(max_depth=depth, min_instances=1, min_info_gain=0.0, min_weight_fraction=0.0)
    f64 = lambda a: None if a is None else a.astype(np.float64)
    if K:
        params.update(num_classes=K, impurity=impurity)
        return TC.audit(tree, X, cands, sub, y.astype(np.float64), f64(w), f64(bag), params)
    return T.audit(tree, X, cands, sub, y.astype(np.float64), f64(w), f64(bag), params)


KINDS = [(0, "variance"), (2, "gini"), (2, "entropy"), (26, "gini"), (26, "entropy")]


@pytest.mark.parametrize("depth", [0, 1, 5, 8])
@pytest.mark.parametrize("rows", ["plain", "weighted", "bag", "weighted_bag"])
@pytest.mark.parametrize("K,impurity", KINDS, ids=[f"K{k}-{i}" for k, i in KINDS])
def test_forest_fit_equals_one_tree_fits(ctx, K, impurity, rows, depth):
    """Mixed subspace sizes: one column, the column with no candidates alone and with others, repeated columns of
    other trees, the whole matrix.  Every forest tree equals its one-tree fit and passes the audit."""
    n, d = 6_001, 10
    X, y, w, bag, cands = _problem(ctx, n, d, K, rows, seed=K * 10 + depth + len(rows))
    rng = np.random.default_rng(depth)
    subs = [np.array([2], np.int32), np.array([d - 1], np.int32), np.array([d - 1, 1, 0], np.int32),
            np.arange(d, dtype=np.int32)] + [np.sort(rng.choice(d, rng.integers(2, d), replace=False)).astype(np.int32)
                                             for _ in range(4)]
    forest, single = _fits(ctx, subs, K, impurity if K else "gini", w, bag, depth)
    assert int(ctx.get_option("last_forest_fit_batches")) == 1
    for got, want in zip(forest, single):
        _same_tree(got, want, K)
    for got, s in zip(forest, subs):
        assert _audit(got, X, cands, s, y, w, bag, K, impurity, depth) == got["feature"].size
    assert forest[1]["feature"].size == 1, "a tree over a column without candidates is a leaf"
    if depth >= 5:
        assert forest[3]["feature"].size > 7, "the whole-matrix tree grows"


def test_forest_fit_in_several_batches(ctx):
    """70 distinct subspaces (d = 32, subspaceRatio 0.5) are more than one batch holds."""
    from spark_ensemble_b200.ensemble import subspace
    n, d = 20_000, 32
    X, y, w, bag, cands = _problem(ctx, n, d, 0, "weighted_bag", seed=70)
    subs = [subspace(0.5, d, 1000 + i) for i in range(70)]
    assert len({s.tobytes() for s in subs}) == 70 and min(s.size for s in subs) >= 1
    forest, single = _fits(ctx, subs, 0, "gini", w, bag, 4)
    assert int(ctx.get_option("last_forest_fit_batches")) >= 2
    for got, want, s in zip(forest, single, subs):
        _same_tree(got, want, 0)
    for t in (0, 63, 64, 69):  # the first and last trees of both batches
        assert _audit(forest[t], X, cands, subs[t], y, w, bag, 0, "gini", 4) == forest[t]["feature"].size


def test_forest_fit_errors(ctx):
    from spark_ensemble_b200 import _native as N
    _problem(ctx, 1_000, 6, 3, "plain", seed=1)
    with pytest.raises(ValueError, match="tree 1: empty subspace"):  # SE_ERR_ARG
        ctx.forest_fit([[0, 1], [], [2]], N.SLOT_Y)
    with pytest.raises(ValueError, match="tree 2: subspace entry 1: column 6 outside"):
        ctx.forest_fit([[0, 1], [3], [2, 6]], N.SLOT_Y)
    with pytest.raises(ValueError, match="numClasses"):
        ctx.forest_fit([[0, 1]], N.SLOT_Y, num_classes=65)
    with pytest.raises(ValueError, match="maxDepth 9"):
        ctx.forest_fit([[0, 1]], N.SLOT_Y, max_depth=9)


def test_forest_fit_past_2_31_bytes_of_node_ids(ctx):
    """70 M rows and 9 trees: tree t's node ids start at t · 2 · 4⌈n/4⌉ · 2 B, so tree 8's lie past 2^31 bytes.  Every
    tree is audited over 4 M-row chunks (oracle/tree_audit.py)."""
    from oracle import tree_audit as TA
    from oracle.oracle import Oracle
    from spark_ensemble_b200 import _native as N
    n, d, depth = 70_000_001, 40, 4
    C = np.asarray([-1.5, -0.8, -0.3, 0.0, 0.2, 0.6, 1.1, 1.7], np.float32)
    cols = np.array([0, 7, 13, 21, 29, 39], np.int32)  # the columns the trees split on
    rng = np.random.default_rng(9)
    subs = [np.sort(rng.choice(cols, 3, replace=False)).astype(np.int32) for _ in range(9)]
    ctx.alloc(N.SLOT_X, d, n)
    ctx.fill_synthetic(N.SLOT_X, "normal", 91, 0.0, 1.0)
    ctx.tree_fit_bins([C] * d)
    for s in (N.SLOT_Y, N.SLOT_W, N.SLOT_BAG, N.SLOT_H):
        ctx.alloc(s, 1, n)
    ctx.linear_predict([1.0, -2.0, 0.5, 1.5, -1.0, 2.0], 0.0, N.SLOT_Y, 0, subspace=cols.tolist())
    ctx.fill_synthetic(N.SLOT_W, "uniform", 92, 0.25, 4.0)
    ctx.fill_synthetic(N.SLOT_BAG, "randint", 93, 0, 3)
    assert 8 * 2 * 4 * ((n + 3) // 4) * 2 > 2 ** 31
    forest = ctx.forest_fit(subs, N.SLOT_Y, 0, N.SLOT_W, 0, True, max_depth=depth)
    assert int(ctx.get_option("last_forest_fit_batches")) == 1
    # host copies of what the audits read: the ranks of the split columns, labels, weights, bag
    orc = Oracle(omp=True)
    CH = 4_000_000
    R = np.empty((cols.size, n), np.uint8)
    h = {s: np.empty(n, np.float32) for s in (N.SLOT_Y, N.SLOT_W, N.SLOT_BAG)}
    for a in range(0, n, CH):
        b = min(n, a + CH)
        for s in h:
            ctx.download(s, count=b - a, offset=a, out=h[s][a:b])
        x = np.empty(b - a, np.float32)
        for k, c in enumerate(cols):
            ctx.download(N.SLOT_X, count=b - a, offset=int(c) * n + a, out=x)
            R[k, a:b] = orc.ranks(x, C)
    pos = {int(c): k for k, c in enumerate(cols)}
    params = dict(max_depth=depth, min_instances=1, min_info_gain=0.0, min_weight_fraction=0.0)
    for t, s in enumerate(subs):
        idx = np.asarray([pos[int(c)] for c in s])

        def gen(idx=idx):
            for a in range(0, n, CH):
                b = min(n, a + CH)
                yield (np.ascontiguousarray(R[idx, a:b]), h[N.SLOT_Y][a:b].astype(np.float64),
                       h[N.SLOT_W][a:b].astype(np.float64), h[N.SLOT_BAG][a:b].astype(np.float64))
        tree = forest[t]
        assert tree["feature"].size > 7
        assert TA.audit(tree, gen, [C] * s.size, params, orc) == tree["feature"].size
    ctx.free(N.SLOT_X)


# ---- the estimators -------------------------------------------------------------------------------------------------
def _frame(n, d, K, weighted, seed):
    from spark_ensemble_b200.ensemble import DataFrame
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d))
    z = np.sin(2 * X[:, 0]) + X[:, 1] ** 2 - X[:, 2] + 0.3 * rng.standard_normal(n)
    y = np.digitize(z, np.quantile(z, np.linspace(0, 1, K + 1)[1:-1])).astype(np.float64) if K else z
    cols = dict(features=X, label=y)
    if weighted:
        cols["weight"] = rng.uniform(0.5, 2.0, n)
    return DataFrame(**cols)


def _estimator(kind, ratio, replacement, weighted, M=6, depth=4):
    from spark_ensemble_b200.classification import BaggingClassifier
    from spark_ensemble_b200.learners import DeviceDecisionTreeClassifier, DeviceDecisionTreeRegressor
    from spark_ensemble_b200.regression import BaggingRegressor
    if kind == "regressor":
        est = BaggingRegressor().setBaseLearner(DeviceDecisionTreeRegressor(maxDepth=depth))
    else:
        est = (BaggingClassifier().setBaseLearner(DeviceDecisionTreeClassifier(maxDepth=depth, impurity="entropy"))
               .setVotingStrategy(kind))
    est = est.setNumBaseLearners(M).setSubspaceRatio(ratio).setSubsampleRatio(0.7).setReplacement(replacement)
    if weighted:
        est = est.setWeightCol("weight")
    return est


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("replacement", [True, False])
@pytest.mark.parametrize("ratio", [0.5, 1.0])
@pytest.mark.parametrize("kind", ["regressor", "hard", "soft"])
def test_bagging_device_route_equals_member_route(kind, ratio, replacement, weighted):
    K = 0 if kind == "regressor" else 3
    df = _frame(30_000, 8, K, weighted, seed=len(kind) + int(10 * ratio))
    est = _estimator(kind, ratio, replacement, weighted)
    member = est.setResidentFeatures(False).fit(df)
    device = est.setResidentFeatures(True).fit(df)
    assert len(device.models) == len(member.models) == 6
    for sa, sb in zip(device.subspaces, member.subspaces):
        np.testing.assert_array_equal(sa, sb)
    for a, b in zip(device.models, member.models):
        ta, tb = a.tree_arrays(), b.tree_arrays()
        for k in ("feature", "threshold", "left", "right"):
            np.testing.assert_array_equal(ta[k], tb[k])
        assert _ulps(ta["value"], tb["value"]).max(initial=0) <= 1
        if K:
            assert _ulps(ta["values"], tb["values"]).max(initial=0) <= 1
    col = device("predictionCol")
    np.testing.assert_allclose(device.transform(df)[col], member.transform(df)[col], rtol=1e-5, atol=1e-5)
    if K:
        pc = device("probabilityCol")
        np.testing.assert_allclose(device.transform(df)[pc], member.transform(df)[pc], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("kind", ["regressor", "hard"])
def test_bagging_device_route_uploads_features_once(monkeypatch, kind):
    """X goes up once per fit and nothing of it comes back; at subspaceRatio 1 every member shares one subspace and
    the forest fit is asked for exactly one tree."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    calls = {"x_up": 0, "x_down": 0, "trees": []}
    up, down, ff = Context.upload_rowmajor, Context.download, Context.forest_fit

    def upload_rowmajor(self, slot, *a, **k):
        calls["x_up"] += slot == N.SLOT_X
        return up(self, slot, *a, **k)

    def download(self, slot, *a, **k):
        calls["x_down"] += slot in (N.SLOT_X,)
        return down(self, slot, *a, **k)

    def forest_fit(self, subspaces, *a, **k):
        calls["trees"].append(len(subspaces))
        return ff(self, subspaces, *a, **k)
    monkeypatch.setattr(Context, "upload_rowmajor", upload_rowmajor)
    monkeypatch.setattr(Context, "download", download)
    monkeypatch.setattr(Context, "forest_fit", forest_fit)
    K = 0 if kind == "regressor" else 3
    df = _frame(5_000, 16, K, True, seed=2)  # 16 columns: no member draws an empty subspace at ratio 0.5
    for ratio, want in ((0.5, None), (1.0, 1)):
        calls.update(x_up=0, x_down=0, trees=[])
        m = _estimator(kind, ratio, True, True, M=10).setResidentFeatures(True).fit(df)
        assert calls["x_up"] == 1 and calls["x_down"] == 0 and len(calls["trees"]) == 1
        distinct = len({np.asarray(s).tobytes() for s in m.subspaces})
        assert calls["trees"][0] == distinct
        if want is not None:
            assert calls["trees"][0] == want and len(m.models) == 10


@pytest.mark.parametrize("kind", ["regressor", "hard"])
@pytest.mark.parametrize("case", ["empty_subspace", "no_in_bag_row", "classes", "max_depth"])
def test_bagging_device_route_errors_match_member_route(kind, case):
    K = 0 if kind == "regressor" else 3
    if case == "classes" and not K:
        pytest.skip("classifier only")
    df = _frame(500, 4, K, False, seed=3)
    if case == "classes":
        from spark_ensemble_b200.ensemble import DataFrame
        df = DataFrame(features=df["features"], label=np.zeros(500))  # one class: K = 1
    est = _estimator(kind, 1.0, False, False, M=3)
    if case == "empty_subspace":
        est = est.setSubspaceRatio(1e-9)
    elif case == "no_in_bag_row":
        est = est.setSubsampleRatio(1e-12)
    elif case == "max_depth":
        est("baseLearner").maxDepth = 9
    msgs = []
    for resident in (False, True):
        with pytest.raises(ValueError) as e:
            est.setResidentFeatures(resident).fit(df)
        msgs.append(str(e.value))
    assert msgs[0] == msgs[1]
