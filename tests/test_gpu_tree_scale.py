"""Device tree fits and forest scoring on one benchmark-sized shard: 34,000,003 rows x 128 columns, so the uint8 rank
matrix (ld8 = 34,000,128) puts column 63 just below 2^31 bytes, column 64 above it and column 127 above 2^32, and the
row count is a multiple of neither 4 nor 128.  Every node of every fit is audited from fp64 sums over the rows it
receives (oracle/tree_audit.py, summed over 4 M-row chunks), the fit's output row is checked against a host walk and
se_tree_predict on every row, and the one-pass forest kernels are checked against the member route on every row and
against a numpy walk of the downloaded features on three 1 M-row windows.

All data is generated on the device; the host downloads the ranks of the subspace columns, the labels, weights and
bag multiplicities, and the feature windows.  The fits are chosen so that, between them, every histogram path of
tree_fit_run runs (several columns per CTA, one column per CTA, opt-in shared memory at 2 and at 1 CTA per SM, global
fp64 atomics), with tens of millions of rows per CTA grid."""
import numpy as np
import pytest
from scipy.special import ndtri

from oracle import tree_audit as TA

pytestmark = pytest.mark.gpu

N_ROWS, D = 34_000_003, 128
CHUNK = 4_000_000
WIN = 1_000_000
KEY = (0, 63, 64, 127)  # byte offsets of the rank matrix: 0, just below 2^31, above 2^31, above 2^32


def _quantiles(bins):
    """bins - 1 fp32 quantiles of N(0, 1): the split candidates of every column (k/32 is 8k/256: the 31 candidates
    are a subset of the 255)."""
    c = ndtri(np.arange(1, bins) / bins).astype(np.float32)
    assert np.all(np.diff(c) > 0)
    return c


C31, C255 = _quantiles(32), _quantiles(256)
SUB = np.random.default_rng(5).permutation(np.concatenate([np.asarray(KEY), np.random.default_rng(4).choice(
    np.setdiff1d(np.arange(D), KEY), 44, replace=False)])).astype(np.int32)
PEAK = {"used": 0}


def _note_memory():
    import torch
    free, total = torch.cuda.mem_get_info(0)
    PEAK["used"] = max(PEAK["used"], total - free)


def chunks(n, size=CHUNK):
    for a in range(0, n, size):
        yield a, min(n, a + size)


def rows(ctx, slot, a, b, dim=1, row0=0):
    """Rows [a, b) of rows row0 .. row0 + dim - 1 of a [.][n] slot as float32 [dim][b - a]."""
    _, n, _ = ctx.layout(slot)
    out = np.empty((dim, b - a), dtype=np.float32)
    for j in range(dim):
        ctx.download(slot, count=b - a, offset=(row0 + j) * n + a, out=out[j])
    return out


def _windows(n):
    return (0, (n // 2 // 4) * 4 + 1, n - WIN)


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    yield c
    c.close()
    print(f"\npeak device memory in use: {PEAK['used'] / 2 ** 30:.2f} GiB")


@pytest.fixture(scope="module")
def orc():
    from oracle.oracle import Oracle
    import os
    o = Oracle(omp=True)
    n = len(os.sched_getaffinity(0))
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if q != "max":
            n = max(1, min(n, int(float(q) / float(p) + 0.5)))
    except Exception:
        pass
    o.lib.orc_set_num_threads(n)
    return o


def _planted(depth, seed, values):
    """A complete tree over the KEY columns (global indices) with candidate thresholds near the middle."""
    rng = np.random.default_rng(seed)
    nn = 2 ** (depth + 1) - 1
    idx = np.arange(nn)
    leaf = idx >= 2 ** depth - 1
    feat = np.where(leaf, -1, np.asarray(KEY)[(idx * 3 + 1) % 4])
    feat[0] = 127
    thr = np.where(leaf, 0.0, C31[rng.integers(8, 23, nn)]).astype(np.float32)
    return {"feature": feat.astype(np.int32), "threshold": thr, "left": np.where(leaf, 0, 2 * idx + 1).astype(np.int32),
            "right": np.where(leaf, 0, 2 * idx + 2).astype(np.int32), "value": np.asarray(values(rng, nn), np.float32)}


@pytest.fixture(scope="module")
def shard(ctx, orc):
    """The shard on the device and, on the host, what the audits read: the ranks of the subspace columns under both
    candidate sets, the regression labels, weights and bag multiplicities."""
    from spark_ensemble_b200 import _native as N
    n = N_ROWS
    ctx.alloc(N.SLOT_X, D, n)
    ctx.fill_synthetic(N.SLOT_X, "normal", 71, 0.0, 1.0)
    ctx.tree_fit_bins([C255] * D)
    for s in (N.SLOT_W, N.SLOT_BAG, N.SLOT_R, N.SLOT_H, N.SLOT_F, N.SLOT_RAW, N.SLOT_Y, N.SLOT_PRED):
        ctx.alloc(s, 1, n)
    ctx.fill_synthetic(N.SLOT_W, "uniform", 72, 0.25, 4.0)
    ctx.fill_synthetic(N.SLOT_BAG, "randint", 73, 0, 3)
    # regression labels: a linear term over the KEY columns, a planted tree, noise
    ctx.linear_predict([1.5, -2.0, 1.0, 2.5], 0.1, N.SLOT_R, 0, subspace=list(KEY))
    ctx.tree_predict(_planted(4, 74, lambda rng, m: 3.0 * rng.standard_normal(m)), N.SLOT_H, 0)
    ctx.fill_synthetic(N.SLOT_F, "normal", 75, 0.0, 0.3)
    h = {"r": np.empty(n, np.float32), "w": np.empty(n, np.float32), "bag": np.empty(n, np.float32),
         "R255": np.empty((SUB.size, n), np.uint8), "R31": np.empty((SUB.size, n), np.uint8)}
    for a, b in chunks(n):
        r = (rows(ctx, N.SLOT_R, a, b)[0].astype(np.float64) + rows(ctx, N.SLOT_H, a, b)[0] +
             rows(ctx, N.SLOT_F, a, b)[0]).astype(np.float32)
        ctx.upload(N.SLOT_R, r, offset=a)
        h["r"][a:b] = r
        h["w"][a:b] = rows(ctx, N.SLOT_W, a, b)[0]
        h["bag"][a:b] = rows(ctx, N.SLOT_BAG, a, b)[0]
        for k, c in enumerate(SUB):
            x = rows(ctx, N.SLOT_X, a, b, row0=int(c))[0]
            h["R255"][k, a:b] = orc.ranks(x, C255)
            h["R31"][k, a:b] = orc.ranks(x, C31)
    assert set(np.unique(h["bag"][:CHUNK]).tolist()) == {0.0, 1.0, 2.0}
    assert h["w"].min() >= 0.25 and h["w"].max() < 4.0
    ctx.free(N.SLOT_F)
    _note_memory()
    return h


def _chunks_of(h, R, lab, w, bag):
    def gen():
        for a, b in chunks(N_ROWS):
            yield (np.ascontiguousarray(h[R][:, a:b]), lab[a:b].astype(np.float64),
                   None if w is None else w[a:b].astype(np.float64), None if bag is None else bag[a:b].astype(np.float64))
    return gen


def _hist_paths(ctx, depth):
    v = int(ctx.get_option("last_tree_fit_hist"))
    return [(v >> (3 * L)) & 7 for L in range(max(depth, 1))]


def _depths(tree):
    d = np.zeros(tree["feature"].size, np.int64)
    for i in range(tree["feature"].size):  # BFS order: parents first
        if tree["feature"][i] >= 0:
            d[tree["left"][i]] = d[tree["right"][i]] = d[i] + 1
    return d


def _fit_and_audit(ctx, orc, h, *, cands, R, depth, weighted, bagged, paths, K=0, labels=None, impurity="gini",
                   mutate=False):
    """One device fit over the subspace, its histogram path per level, every node audited over 4 M-row chunks, its
    output row against the host walk and against se_tree_predict of the returned arrays on every row."""
    from spark_ensemble_b200 import _native as N
    wslot = N.SLOT_W if weighted else -1
    if K:
        t = ctx.tree_fit_classifier(N.SLOT_Y, K, weight_slot=wslot, use_bag=bagged, subspace=SUB, impurity=impurity,
                                    max_depth=depth, out_slot=N.SLOT_PRED)
        out_slot, lab = N.SLOT_PRED, labels
    else:
        t = ctx.tree_fit(N.SLOT_R, 0, wslot, 0, bagged, subspace=SUB, max_depth=depth, out_slot=N.SLOT_H)
        out_slot, lab = N.SLOT_H, h["r"]
    got_paths = _hist_paths(ctx, depth)
    _note_memory()
    print(f"\nfit K={K} depth {depth}, {len(cands[0]) + 1} bins: {t['feature'].size} nodes, histogram path per level "
          f"{got_paths} (0 several columns / CTA, 1 one column / CTA, 2 opt-in 2 CTAs/SM, 3 opt-in 1 CTA/SM, 4 global)")
    assert got_paths == paths
    # a regression tree splits down to the deepest searched level; a classifier's deepest splits on noise are pruned
    assert _depths(t)[t["feature"] >= 0].max() >= (3 if K else depth - 1), "the deep levels are split"
    assert set(KEY) & {int(SUB[f]) for f in t["feature"][t["feature"] >= 0]}, "the tree splits on a far column"
    ctx.tree_predict(t, N.SLOT_RAW, 0, subspace=SUB)
    pos = [0]

    def check_out(leaf):
        a, b = pos[0], pos[0] + leaf.size
        got = rows(ctx, out_slot, a, b)[0]
        np.testing.assert_array_equal(got.view(np.uint32), rows(ctx, N.SLOT_RAW, a, b)[0].view(np.uint32))
        np.testing.assert_array_equal(got, t["value"][leaf].astype(np.float32))
        pos[0] = b
    params = dict(max_depth=depth, min_instances=1, min_info_gain=0.0, min_weight_fraction=0.0)
    if K:
        params["impurity"] = impurity
    gen = _chunks_of(h, R, lab, h["w"] if weighted else None, h["bag"] if bagged else None)
    assert TA.audit(t, gen, cands, params, orc, num_classes=K, out=check_out) == t["feature"].size
    assert pos[0] == N_ROWS
    if mutate:  # one thing wrong in the returned arrays, nothing else changed: the audit must refuse each
        f = t["feature"]
        b = {k: v.copy() for k, v in t.items()}
        j = int(np.searchsorted(cands[f[0]], b["threshold"][0]))
        b["threshold"][0] = cands[f[0]][j + 1 if j + 1 < len(cands[f[0]]) else j - 1]
        c = {k: v.copy() for k, v in t.items()}
        leaf = int(np.flatnonzero(f < 0)[0])
        v = c["values"][leaf] if K else c["value"]  # a class probability, or the regression value
        q = int(np.argmax(v)) if K else leaf
        v[q] = np.float32(v[q]) + 3 * np.spacing(np.float32(v[q]))
        for name, bad in (("root threshold on the next candidate", b), ("a leaf value 3 ulps off", c)):
            with pytest.raises(AssertionError):
                TA.audit(bad, gen, cands, params, orc, num_classes=K)
                pytest.fail(f"the audit accepted: {name}")
    return t


def _class_labels(ctx, K, seed):
    """Class labels in SLOT_Y: a planted classification tree, then about 10 % of the rows overwritten with random
    classes over five row ranges; returns them as host fp32."""
    from spark_ensemble_b200 import _native as N
    ctx.tree_predict(_planted(5, seed, lambda rng, m: rng.integers(0, K, m)), N.SLOT_Y, 0)
    span = N_ROWS // 50
    for q, a in enumerate(np.linspace(0, N_ROWS - span, 5).astype(np.int64)):
        ctx.fill_synthetic(N.SLOT_Y, "randint", seed + 1 + q, 0, K, count=span, offset=int(a))
    y = np.empty(N_ROWS, np.float32)
    for a, b in chunks(N_ROWS):
        y[a:b] = rows(ctx, N.SLOT_Y, a, b)[0]
    assert set(np.unique(y[:CHUNK]).tolist()) <= set(range(K)) and np.unique(y).size == K
    return y


# ---- fits ------------------------------------------------------------------------------------------------------
def test_fit_b_regression_256_bins(ctx, orc, shard):
    """255 candidates, no weights, no bag: several columns per CTA (L 0, 1), one column (L 2), opt-in at 2 CTAs/SM
    (L 3, 64 KB) and at 1 CTA/SM (L 4, 128 KB), global fp64 atomics (L 5, 256 KB)."""
    _fit_and_audit(ctx, orc, shard, cands=[C255] * SUB.size, R="R255", depth=6, weighted=False, bagged=False,
                   paths=[0, 0, 1, 2, 3, 4])
    del shard["R255"]  # the later fits and forests use the 31 candidates


def test_fit_a_regression_32_bins(ctx, orc, shard):
    """31 candidates, weights and bag, maxDepth 7: several columns per CTA (L 0-4), one column (L 5), opt-in at 2
    CTAs/SM (L 6, 66 KB).  A mutated copy of the returned tree fails the audit."""
    ctx.tree_fit_bins([C31] * D)
    _fit_and_audit(ctx, orc, shard, cands=[C31] * SUB.size, R="R31", depth=7, weighted=True, bagged=True,
                   paths=[0, 0, 0, 0, 0, 1, 2], mutate=True)


def test_fit_c_classifier_k26_gini(ctx, orc, shard):
    """K = 26, gini, weights: 27 doubles per bin, one column per CTA (L 3, 56 KB), opt-in at 2 CTAs/SM (L 4, 111 KB)
    and at 1 CTA/SM (L 5, 223 KB), global (L 6)."""
    y = _class_labels(ctx, 26, 80)
    _fit_and_audit(ctx, orc, shard, cands=[C31] * SUB.size, R="R31", depth=7, weighted=True, bagged=False,
                   paths=[0, 0, 0, 1, 2, 3, 4], K=26, labels=y, mutate=True)


def test_fit_d_classifier_k2_entropy(ctx, orc, shard):
    """K = 2, entropy, bag: the binary entropy path, every level several columns per CTA."""
    y = _class_labels(ctx, 2, 90)
    _fit_and_audit(ctx, orc, shard, cands=[C31] * SUB.size, R="R31", depth=6, weighted=False, bagged=True,
                   paths=[0] * 6, K=2, labels=y, impurity="entropy")


# ---- forests ---------------------------------------------------------------------------------------------------
def _forest(seed, M, depth, K=0):
    """M complete trees of the given depth over candidate thresholds: the root of tree t splits on KEY[t % 4], the
    other nodes on the KEY columns or a few others (global indices)."""
    rng = np.random.default_rng(seed)
    cols = np.concatenate([np.asarray(KEY), SUB[-6:]])
    out = []
    for t in range(M):
        nn = 2 ** (depth + 1) - 1
        idx = np.arange(nn)
        leaf = idx >= 2 ** depth - 1
        feat = np.where(leaf, -1, cols[rng.integers(0, cols.size, nn)])
        feat[0] = KEY[t % 4]
        tr = {"feature": feat.astype(np.int32), "threshold": np.where(leaf, 0.0, C31[rng.integers(0, C31.size, nn)])
              .astype(np.float32), "left": np.where(leaf, 0, 2 * idx + 1).astype(np.int32),
              "right": np.where(leaf, 0, 2 * idx + 2).astype(np.int32),
              "value": rng.standard_normal(nn).astype(np.float32)}
        if K:
            tr["values"] = rng.dirichlet(np.full(K, 0.5), nn).astype(np.float32)
            tr["value"] = tr["values"].argmax(axis=1).astype(np.float32)
        out.append(tr)
    return out


def _features(ctx, a, b):
    """Columns [0, D) of rows [a, b) as fp32 [b - a][D] (only the forest's columns are downloaded; others are NaN)."""
    from spark_ensemble_b200 import _native as N
    cols = np.concatenate([np.asarray(KEY), SUB[-6:]])
    X = np.full((b - a, D), np.nan, np.float32)
    for c in cols:
        X[:, c] = rows(ctx, N.SLOT_X, a, b, row0=int(c))[0]
    return X


def _leaf(tree, X):
    node = np.zeros(X.shape[0], np.int64)
    for _ in range(64):
        f = tree["feature"][node]
        live = f >= 0
        if not live.any():
            break
        x = X[np.arange(X.shape[0]), np.maximum(f, 0)]
        node = np.where(live, np.where(x <= tree["threshold"][node], tree["left"][node], tree["right"][node]), node)
    return node


def _members(ctx, trees, K=0):
    """The member route's P: tree_predict of every member (and class) into rows of SLOT_P."""
    from spark_ensemble_b200 import _native as N
    for m, tr in enumerate(trees):
        if K:
            for k in range(K):
                ctx.tree_predict(dict(tr, value=tr["values"][:, k].copy()), N.SLOT_P, m * K + k)
        else:
            ctx.tree_predict(tr, N.SLOT_P, m)


def test_forest_predict_past_4g(ctx, shard):
    """se_forest_predict over 24 trees of depth 7 (two chunks of trees) against tree_predict per member into an
    [M][n] P and se_agg_run(GBM_REGRESSOR) on every row, and against fp64 numpy walks on three windows."""
    from spark_ensemble_b200 import _native as N
    M, n, init = 24, N_ROWS, 0.25
    trees = _forest(101, M, 7)
    w = np.random.default_rng(102).random(M) + 0.1
    ctx.forest_predict(trees, N.SLOT_H, weights=w, init=init)
    nch = int(ctx.get_option("last_forest_chunks"))
    assert nch >= 2
    ctx.agg_configure(N.AGG_GBM_REGRESSOR, M, 0, 1, 0, n)
    _members(ctx, trees)
    ctx.agg_run(w, [init])
    _note_memory()
    scale = float(np.abs(w).sum() * 4.5 + abs(init))
    for a, b in chunks(n):
        got, mem = rows(ctx, N.SLOT_H, a, b)[0].astype(np.float64), rows(ctx, N.SLOT_RAW, a, b)[0].astype(np.float64)
        assert np.max(np.abs(got - mem)) <= 1.5e-7 * scale * (nch + 1), a
    for a in _windows(n):
        X = _features(ctx, a, a + WIN)
        want = np.full(WIN, init)
        P = rows(ctx, N.SLOT_P, a, a + WIN, M)
        for m, tr in enumerate(trees):
            v = tr["value"][_leaf(tr, X)]
            np.testing.assert_array_equal(P[m], v)  # every member's leaf, exactly
            want = want + w[m] * v.astype(np.float64)
        got = rows(ctx, N.SLOT_H, a, a + WIN)[0].astype(np.float64)
        assert np.max(np.abs(got - want)) <= 1.5e-7 * scale * nch, a
    ctx.free(N.SLOT_P)


def test_forest_median_past_4g(ctx, orc, shard):
    """se_forest_median, M = 32: bit for bit the member route (tree_predict per member + se_agg_run
    BOOSTING_REG_MEDIAN) on every row, and the oracle's weighted median of numpy walks on three windows."""
    from spark_ensemble_b200 import _native as N
    M, n = 32, N_ROWS
    trees = _forest(111, M, 5)
    a_w = np.random.default_rng(112).random(M) + 0.05
    ctx.forest_median(trees, N.SLOT_H, a_w)
    ctx.agg_configure(N.AGG_BOOSTING_REG_MEDIAN, M, 0, 1, 0, n)
    _members(ctx, trees)
    ctx.agg_run(a_w)
    _note_memory()
    for a, b in chunks(n):
        np.testing.assert_array_equal(rows(ctx, N.SLOT_H, a, b)[0].view(np.uint32),
                                      rows(ctx, N.SLOT_RAW, a, b)[0].view(np.uint32))
    for a in _windows(n):
        X = _features(ctx, a, a + WIN)
        P = np.stack([tr["value"][_leaf(tr, X)] for tr in trees])
        np.testing.assert_array_equal(rows(ctx, N.SLOT_P, a, a + WIN, M), P)
        np.testing.assert_array_equal(rows(ctx, N.SLOT_H, a, a + WIN)[0].astype(np.float64),
                                      orc.agg_weighted_median(P.astype(np.float64), a_w))
    ctx.free(N.SLOT_P)


@pytest.mark.parametrize("kind,K,M", [("soft", 8, 6), ("real", 26, 4)])
def test_forest_agg_past_4g(ctx, orc, shard, kind, K, M):
    """se_forest_agg, bagging soft and SAMME.R: RAW, PROB and LABEL against the member route (tree_predict per
    member and class into [M][K][n] P + se_agg_run) on every row, and against the oracle's aggregation of numpy walks
    on three windows, with the tolerances of the model-level checks."""
    from spark_ensemble_b200 import _native as N
    n = N_ROWS
    agg = N.AGG_BAGGING_SOFT if kind == "soft" else N.AGG_BOOSTING_REAL
    trees = _forest(121 + K, M, 6, K)
    ctx.forest_agg(agg, K, trees)
    raw = np.empty((K, n), np.float32)
    prob = np.empty((K, n), np.float32)
    lab = np.empty(n, np.float32)
    for a, b in chunks(n):
        raw[:, a:b], prob[:, a:b] = rows(ctx, N.SLOT_RAW, a, b, K), rows(ctx, N.SLOT_PROB, a, b, K)
        lab[a:b] = rows(ctx, N.SLOT_LABEL, a, b)[0]
    ctx.agg_configure(agg, M, K, 1, 0, n)
    _members(ctx, trees, K)
    ctx.agg_run()
    _note_memory()

    def close(r_got, p_got, l_got, r_want, p_want):
        atol = 1e-5 * max(1.0, float(np.abs(r_want).max())) if kind == "real" else 1e-6
        np.testing.assert_allclose(r_got, r_want, rtol=1e-5, atol=atol)
        np.testing.assert_allclose(p_got, p_want, rtol=1e-5, atol=1e-6)
        srt = np.sort(r_want, axis=0)
        near_tie = (srt[-1] - srt[-2]) <= 1e-5 * np.maximum(1.0, np.abs(srt[-1])) + atol
        assert not np.any((l_got != np.argmax(r_want, axis=0)) & ~near_tie)
    for a, b in chunks(n):
        close(raw[:, a:b], prob[:, a:b], lab[a:b], rows(ctx, N.SLOT_RAW, a, b, K), rows(ctx, N.SLOT_PROB, a, b, K))
    for a in _windows(n):
        X = _features(ctx, a, a + WIN)
        P = np.stack([tr["values"][_leaf(tr, X)].T for tr in trees])  # [M][K][WIN]
        np.testing.assert_array_equal(rows(ctx, N.SLOT_P, a, a + WIN, M * K).reshape(M, K, WIN), P)
        r_o, p_o = (orc.agg_bagging_soft if kind == "soft" else orc.agg_boosting_real)(P.astype(np.float64))
        close(raw[:, a:a + WIN], prob[:, a:a + WIN], lab[a:a + WIN], r_o, p_o)
    ctx.free(N.SLOT_P)


def test_tree_walks_past_4g(ctx, shard):
    """The three single-tree walks (mask, rank-matrix walk, fp32) on a tree whose root reads column 127 (byte offset
    above 2^32): sums and three windows bit for bit, a window against a numpy walk."""
    from spark_ensemble_b200 import _native as N
    tree = _planted(6, 131, lambda rng, m: np.linspace(-1, 1, m))
    got = {}
    try:
        for name, bins, mask in (("mask", 1, 1), ("walk", 1, 0), ("fp32", 0, 0)):
            ctx.set_option("tree_bins", bins)
            ctx.set_option("tree_mask", mask)
            ctx.tree_predict(tree, N.SLOT_H, 0)
            assert ctx.get_option("last_tree_binned") == bins and ctx.get_option("last_tree_mask") == (bins and mask)
            got[name] = (ctx.slot_sum(N.SLOT_H), [rows(ctx, N.SLOT_H, a, a + WIN)[0] for a in _windows(N_ROWS)])
    finally:
        ctx.set_option("tree_bins", 1)
        ctx.set_option("tree_mask", 1)
    for name in ("walk", "fp32"):
        assert got[name][0] == got["mask"][0], name
        for u, v in zip(got[name][1], got["mask"][1]):
            np.testing.assert_array_equal(u, v)
    for q, a in enumerate(_windows(N_ROWS)):
        np.testing.assert_array_equal(got["mask"][1][q], tree["value"][_leaf(tree, _features(ctx, a, a + WIN))])


def test_fit_after_forests_reranks_nothing(ctx, orc, shard):
    """The forests and walks used candidate thresholds only: a fit afterwards re-ranks no column and is accepted."""
    from spark_ensemble_b200 import _native as N
    t = ctx.tree_fit(N.SLOT_R, 0, N.SLOT_W, 0, True, subspace=SUB, max_depth=3, out_slot=N.SLOT_H)
    assert ctx.get_option("last_tree_rebinned_cols") == 0
    assert t["feature"].size == 15
    assert TA.audit(t, _chunks_of(shard, "R31", shard["r"], shard["w"], shard["bag"]), [C31] * SUB.size,
                    dict(max_depth=3), orc) == 15
    _note_memory()
