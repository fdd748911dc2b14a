"""Device tree fits over row-sharded GPUs: each level's histogram is all-reduced, so a fit over a ShardedContext (or
over per-rank contexts joined by a communicator) is the fit of the union of the shards.  On data whose fp64 sums are
exact in any order it equals the one-GPU fit bit for bit; on general data every node is audited (oracle.np_tree /
np_tree_cls) over the whole rows.  Ranks that disagree on the fit's shape fail together instead of blocking."""
import concurrent.futures as cf
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import np_tree as T
from oracle import np_tree_cls as TC

pytestmark = pytest.mark.gpu
TREE_KEYS = ("feature", "threshold", "left", "right", "value", "gain")


def _worlds():
    """2, and every count up to 4 that the machine has."""
    from spark_ensemble_b200 import _native as N
    g = N.device_count()
    if g < 2:
        pytest.skip("needs >= 2 GPUs")
    return list(range(2, min(g, 4) + 1))


@pytest.fixture(scope="module")
def one():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def sharded():
    """ShardedContext per world size, opened once for the module."""
    from spark_ensemble_b200.sharded import ShardedContext
    made = {}

    def get(world):
        if world not in made:
            made[world] = ShardedContext(list(range(world)))
        return made[world]
    yield get
    for sc in made.values():
        sc.close()


def _exact(n, d, seed, levels=8):
    """Integer features, quarter labels, small integer weights and bag counts: every fp64 histogram sum is exact."""
    rng = np.random.default_rng(seed)
    X = rng.integers(0, levels, (n, d)).astype(np.float32)
    r = ((X[:, 0] > levels // 2) * 4 + (X[:, 1] % 3) + rng.integers(-4, 4, n)).astype(np.float32) / 4
    w = rng.integers(1, 5, n).astype(np.float32)
    bag = rng.integers(0, 4, n).astype(np.float32)
    return X, r.astype(np.float32), w, bag


def _load(c, X, r, w=None, bag=None):
    """The same calls on a Context or a ShardedContext (whole host arrays; the latter splits them)."""
    from spark_ensemble_b200 import _native as N
    n, d = X.shape
    c.gbm_configure(n, 0, 1, "squared", 0.0, w is not None)
    c.alloc(N.SLOT_X, d, n)
    c.upload_rowmajor(N.SLOT_X, X)
    c.upload(N.SLOT_R, r)
    if w is not None:
        c.upload(N.SLOT_W, w)
    c.gbm_set_bag(bag)


def _fit(c, X, r, cands, *, w=None, bag=None, sub=None, **params):
    from spark_ensemble_b200 import _native as N
    _load(c, X, r, w, bag)
    c.tree_fit_bins(cands)
    sub = np.arange(X.shape[1], dtype=np.int32) if sub is None else sub
    t = c.tree_fit(N.SLOT_R, 0, N.SLOT_W if w is not None else -1, 0, bag is not None, subspace=sub,
                   out_slot=N.SLOT_H, **params)
    return t, np.asarray(c.download(N.SLOT_H)).reshape(-1).copy()


def _same(t, out, t1, out1):
    for k in TREE_KEYS:
        np.testing.assert_array_equal(t[k], t1[k], err_msg=k)
    np.testing.assert_array_equal(out.view(np.uint32), out1.view(np.uint32))


def _cands(X, max_bins):
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor
    return DeviceDecisionTreeRegressor(maxBins=max_bins, seed=11).split_candidates(X)


# ---- 1. exact data: the sharded fit IS the one-GPU fit ----------------------------------------------------------
EXACT = [
    # id, n, d, levels, maxBins, weights, bag, subspace, params
    ("plain", 20011, 6, 8, 32, False, False, False, dict(max_depth=5)),
    ("weighted", 20011, 6, 8, 32, True, False, False, dict(max_depth=5)),
    ("bag", 20011, 6, 8, 32, False, True, False, dict(max_depth=5)),
    ("weighted-bag-subspace", 20011, 9, 8, 32, True, True, True, dict(max_depth=5)),
    ("depth0", 20011, 4, 8, 32, True, True, False, dict(max_depth=0)),
    ("depth1", 20011, 4, 8, 32, True, False, False, dict(max_depth=1)),
    ("depth8-256-bins", 40000, 4, 256, 256, True, True, False, dict(max_depth=8)),
    ("minInstances", 20011, 6, 8, 32, True, False, False, dict(max_depth=6, min_instances=400)),
]


@pytest.mark.parametrize("case", EXACT, ids=[c[0] for c in EXACT])
def test_sharded_fit_equals_one_gpu_fit(one, sharded, case):
    _, n, d, levels, bins, weighted, bagged, subspaced, params = case
    worlds = _worlds()
    X, r, w, bag = _exact(n, d, seed=n + d + levels, levels=levels)
    w = w if weighted else None
    bag = bag if bagged else None
    sub = np.array([5, 0, 7, 2, 3], np.int32) if subspaced else None
    cands = _cands(X, bins)
    t1, out1 = _fit(one, X, r, cands, w=w, bag=bag, sub=sub, **params)
    assert t1["feature"].size >= (3 if params["max_depth"] >= 1 else 1)
    for world in worlds:
        t, out = _fit(sharded(world), X, r, cands, w=w, bag=bag, sub=sub, **params)
        _same(t, out, t1, out1)


def test_sharded_fit_uses_the_global_root_weight(one, sharded):
    """minWeightFractionPerNode is a fraction of the root weight of ALL rows: the first half of the rows weighs 4x
    the second, so a shard's own root weight would bound the children differently."""
    X, r, w, _ = _exact(20011, 5, seed=3)
    w = np.where(np.arange(X.shape[0]) < X.shape[0] // 2, 4.0, 1.0).astype(np.float32)
    cands = _cands(X, 32)
    free, _ = _fit(one, X, r, cands, w=w, max_depth=5)
    t1, out1 = _fit(one, X, r, cands, w=w, max_depth=5, min_weight_fraction=0.2)
    assert t1["feature"].size < free["feature"].size  # the rule binds
    for world in _worlds():
        t, out = _fit(sharded(world), X, r, cands, w=w, max_depth=5, min_weight_fraction=0.2)
        _same(t, out, t1, out1)


def test_sharded_fit_with_an_out_of_bag_shard_and_a_pure_shard(one, sharded):
    """A shard with no in-bag row adds nothing to any histogram; a shard whose labels are all equal is pure on its
    own but not in the union."""
    from spark_ensemble_b200.ensemble import row_partition
    n = 20011
    X, r0, w, bag0 = _exact(n, 6, seed=5)
    cands = _cands(X, 32)
    for world in _worlds():
        bag = bag0.copy()
        s0, s1 = row_partition(n, world, 0)
        bag[s0:s1] = 0
        r = r0.copy()
        p0, p1 = row_partition(n, world, world - 1)
        r[p0:p1] = 0.75
        for kw in (dict(bag=bag), dict(w=w, bag=bag)):
            t1, out1 = _fit(one, X, r, cands, max_depth=5, **kw)
            t, out = _fit(sharded(world), X, r, cands, max_depth=5, **kw)
            _same(t, out, t1, out1)


# ---- 2. general data: every node audited over the whole rows -----------------------------------------------------
@pytest.mark.parametrize("labels", ["normal", "absolute-residual"])
@pytest.mark.parametrize("depth,bins", [(5, 32), (8, 256)])
def test_sharded_fit_audited(sharded, labels, depth, bins):
    rng = np.random.default_rng(depth + bins)
    n, d = 30011, 7
    X = rng.standard_normal((n, d)).astype(np.float32)
    if labels == "normal":
        r = rng.standard_normal(n).astype(np.float32)
    else:  # the residual of the absolute loss: sign(y - F)
        y = np.sin(2 * X[:, 0]) + X[:, 1] * X[:, 2] + 0.3 * rng.standard_normal(n)
        r = np.sign(y - 0.1).astype(np.float32)
    w = np.abs(rng.standard_normal(n)).astype(np.float32) + 0.05
    bag = rng.poisson(1.0, n).astype(np.float32)
    sub = rng.permutation(d)[:5].astype(np.int32)
    cands = _cands(X, bins)
    params = dict(max_depth=depth, min_instances=1, min_info_gain=0.0, min_weight_fraction=0.0)
    for world in _worlds():
        for kw in (dict(), dict(w=w, bag=bag)):
            t, out = _fit(sharded(world), X, r, cands, sub=sub, **kw, **params)
            assert T.audit(t, X, cands, sub, r, kw.get("w"), kw.get("bag"), params, out=out) == t["feature"].size
            assert t["feature"].size > 7


# ---- 3. the classifier through per-rank contexts joined by a communicator -----------------------------------------
def _fit_cls_ranks(sc, X, y, K, cands, w, impurity, depth, proba):
    """tree_fit_classifier on every rank of sc at once, each on its own rows; returns every rank's tree and the
    concatenated output ([n] labels, or [K, n] probabilities)."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.ensemble import row_partition
    n, d = X.shape
    sub = np.arange(d, dtype=np.int32)

    def f(rk, c):
        s0, s1 = row_partition(n, sc.world, rk)
        c.alloc(N.SLOT_X, d, s1 - s0)
        c.upload_rowmajor(N.SLOT_X, X[s0:s1])
        c.alloc(N.SLOT_Y, 1, s1 - s0)
        c.upload(N.SLOT_Y, y[s0:s1])
        c.alloc(N.SLOT_W, 1, s1 - s0)
        c.upload(N.SLOT_W, w[s0:s1])
        slot = N.SLOT_PROBA if proba else N.SLOT_PRED
        c.alloc(slot, K if proba else 1, s1 - s0)
        c.tree_fit_bins(cands)
        t = c.tree_fit_classifier(N.SLOT_Y, K, 0, N.SLOT_W, 0, False, subspace=sub, impurity=impurity,
                                  max_depth=depth, proba=proba, out_slot=slot)
        return t, np.asarray(c.download(slot)).reshape(K if proba else 1, s1 - s0)
    res = sc._all(f)
    out = np.concatenate([o for _, o in res], axis=1)
    return [t for t, _ in res], (out if proba else out[0])


def _fit_cls_one(c, X, y, K, cands, w, impurity, depth, proba):
    from spark_ensemble_b200 import _native as N
    n, d = X.shape
    c.alloc(N.SLOT_X, d, n)
    c.upload_rowmajor(N.SLOT_X, X)
    c.alloc(N.SLOT_Y, 1, n)
    c.upload(N.SLOT_Y, y)
    c.alloc(N.SLOT_W, 1, n)
    c.upload(N.SLOT_W, w)
    slot = N.SLOT_PROBA if proba else N.SLOT_PRED
    c.alloc(slot, K if proba else 1, n)
    c.tree_fit_bins(cands)
    t = c.tree_fit_classifier(N.SLOT_Y, K, 0, N.SLOT_W, 0, False, subspace=np.arange(d, dtype=np.int32),
                              impurity=impurity, max_depth=depth, proba=proba, out_slot=slot)
    out = np.asarray(c.download(slot)).reshape(K if proba else 1, n)
    return t, (out if proba else out[0])


CLS_KEYS = ("feature", "threshold", "left", "right", "value", "values", "class_weights", "gain")


@pytest.mark.parametrize("K", [2, 26])
@pytest.mark.parametrize("impurity", ["gini", "entropy"])
def test_sharded_classifier_exact_and_audited(one, sharded, K, impurity):
    n, d, depth = 20011, 6, 5
    rng = np.random.default_rng(K)
    # exact: integer features and class weights, so the sums are exact in any order
    X = rng.integers(0, 8, (n, d)).astype(np.float32)
    y = ((3 * X[:, 0] + X[:, 1] + rng.integers(0, 3, n)) % K).astype(np.float32)
    w = rng.integers(1, 5, n).astype(np.float32)
    cands = _cands(X, 32)
    # general: normal features, continuous weights
    Xg = rng.standard_normal((n, d)).astype(np.float32)
    zg = np.sin(2 * Xg[:, 0]) + Xg[:, 1] ** 2 + 0.4 * rng.standard_normal(n)
    yg = np.minimum(np.digitize(zg, np.quantile(zg, np.linspace(0, 1, K + 1)[1:-1])), K - 1).astype(np.float32)
    wg = rng.uniform(0.25, 4.0, n).astype(np.float32)
    cg = _cands(Xg, 32)
    params = dict(num_classes=K, impurity=impurity, max_depth=depth, min_instances=1, min_info_gain=0.0,
                  min_weight_fraction=0.0)
    sub = np.arange(d, dtype=np.int32)
    for proba in (False, True):
        t1, out1 = _fit_cls_one(one, X, y, K, cands, w, impurity, depth, proba)
        for world in _worlds():
            ts, out = _fit_cls_ranks(sharded(world), X, y, K, cands, w, impurity, depth, proba)
            for t in ts:
                for k in CLS_KEYS:
                    np.testing.assert_array_equal(t[k], t1[k], err_msg=k)
            np.testing.assert_array_equal(out.view(np.uint32), out1.view(np.uint32))
            ts, out = _fit_cls_ranks(sharded(world), Xg, yg, K, cg, wg, impurity, depth, proba)
            for t in ts[1:]:
                for k in CLS_KEYS:
                    np.testing.assert_array_equal(t[k], ts[0][k], err_msg=k)
            kw = dict(out_proba=out) if proba else dict(out=out)
            assert TC.audit(ts[0], Xg, cg, sub, yg, wg, None, params, **kw) == ts[0]["feature"].size


# ---- 4. estimators with devices=[0, 1] and the device learner -------------------------------------------------------
def _audited_learner(X_train, n, **kw):
    """DeviceDecisionTreeRegressor that audits every round's tree against the residuals (and weights, bag) it was fitted
    on, downloaded whole from the (sharded) context just before the fit."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor

    class Audited(DeviceDecisionTreeRegressor):
        audited = 0

        def copy(self, extra=None):
            return self

        def fit_resident(self, ctx, label_slot, label_row, weight_slot, weight_row, use_bag, subspace, out_slot, out_row):
            r = np.asarray(ctx.download(label_slot)).reshape(-1, n)[label_row].copy()
            w = None if weight_slot < 0 else np.asarray(ctx.download(weight_slot)).reshape(-1, n)[weight_row].copy()
            bag = np.asarray(ctx.download(N.SLOT_BAG)).reshape(-1).copy() if use_bag else None
            m = super().fit_resident(ctx, label_slot, label_row, weight_slot, weight_row, use_bag, subspace, out_slot,
                                     out_row)
            out = np.asarray(ctx.download(out_slot)).reshape(-1, n)[out_row]
            params = dict(max_depth=self.maxDepth, min_instances=self.minInstancesPerNode, min_info_gain=self.minInfoGain,
                          min_weight_fraction=self.minWeightFractionPerNode)
            cands = self.split_candidates(X_train)
            assert T.audit(m._arrays, X_train, cands, subspace, r, w, bag, params, out=out) == m.numNodes
            Audited.audited += 1
            return m
    return Audited(**kw)


@pytest.mark.parametrize("loss", ["squared", "absolute"])
def test_gbm_regressor_sharded_with_device_learner(loss):
    from spark_ensemble_b200 import DataFrame, _native as N
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor
    from spark_ensemble_b200.regression import GBMRegressor
    if N.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    rng = np.random.default_rng(17)
    n, d = 20011, 8
    X = rng.integers(0, 8, (n, d)).astype(np.float32)  # few candidates, splits that win by a wide margin
    y = 3.0 * (X[:, 0] > 3) + 2.0 * (X[:, 1] > 5) - 1.5 * (X[:, 2] < 2) + 0.05 * rng.standard_normal(n)
    val = rng.random(n) < 0.2
    wt = rng.uniform(0.5, 2.0, n)
    df = DataFrame(features=X, label=y, validation=val, weight=wt)
    fits = []
    for devices in ([], [0, 1]):
        learner = _audited_learner(X[~val], int((~val).sum()), maxDepth=3, seed=5) if devices else \
            DeviceDecisionTreeRegressor(maxDepth=3, seed=5)
        g = (GBMRegressor().setBaseLearner(learner).setNumBaseLearners(6).setValidationIndicatorCol("validation")
             .setLearningRate(0.5))
        g.set("loss", loss).set("residentFeatures", True).set("subsampleRatio", 0.8).set("subspaceRatio", 0.75)
        if loss == "absolute":
            g.set("weightCol", "weight")
        g.set("devices", devices)
        fits.append(g.fit(df))
        if devices:
            assert type(learner).audited == 6
    base, m = fits
    assert m.numModels == base.numModels
    pb = base.transform(df)["prediction"]
    np.testing.assert_allclose(m.transform(df)["prediction"], pb, rtol=1e-5, atol=1e-5 * float(np.abs(pb).max()))


def test_gbm_classifier_sharded_with_device_learner():
    from spark_ensemble_b200 import DataFrame, _native as N
    from spark_ensemble_b200.classification import GBMClassifier
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor
    if N.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    rng = np.random.default_rng(23)
    n, d = 20011, 6
    X = rng.integers(0, 8, (n, d)).astype(np.float32)
    z = 2.0 * (X[:, 0] > 3) + 1.0 * (X[:, 1] > 5) + 0.3 * rng.standard_normal(n)
    y = np.digitize(z, [0.9, 2.1]).astype(np.float64)
    df = DataFrame(features=X, label=y)
    ms = []
    for devices in ([], [0, 1]):
        learner = _audited_learner(X, n, maxDepth=3, seed=5) if devices else DeviceDecisionTreeRegressor(maxDepth=3, seed=5)
        g = GBMClassifier().setBaseLearner(learner).setNumBaseLearners(4).setLoss("logloss")
        g.set("residentFeatures", True).set("devices", devices)
        ms.append(g.fit(df))
        if devices:
            assert type(learner).audited == 4 * 3  # one tree per class dimension and round
    assert len(ms[0].weights) == len(ms[1].weights)
    for w0, w1 in zip(ms[0].weights, ms[1].weights):
        np.testing.assert_allclose(w1, w0, rtol=1e-4, atol=1e-5)
    np.testing.assert_array_equal(ms[0].transform(df)["prediction"], ms[1].transform(df)["prediction"])


# ---- 5. one rank per process ----------------------------------------------------------------------------------------
def test_tree_fit_one_rank_per_process():
    from spark_ensemble_b200 import _native as N
    if N.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", "29541",
                          os.path.join(root, "tests", "mgpu_tree_check.py")], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "MGPU_TREE_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


# ---- 6. ranks that disagree fail together ---------------------------------------------------------------------------
def _each(sc, fn):
    """fn(rank, ctx) on every rank at once; returns every rank's result or exception."""
    futs = [sc._pool.submit(fn, rk, c) for rk, c in enumerate(sc.ctxs)]
    cf.wait(futs)
    return [f.exception() or f.result() for f in futs]


def test_ranks_that_disagree_fail_together(sharded):
    from spark_ensemble_b200 import _native as N
    _worlds()
    sc = sharded(2)
    X, r, w, _ = _exact(20011, 5, seed=9)
    cands = _cands(X, 32)
    _load(sc, X, r, w)
    sub = np.arange(5, dtype=np.int32)
    fit = lambda rk, c: c.tree_fit(N.SLOT_R, 0, N.SLOT_W, 0, False, subspace=sub, max_depth=5, out_slot=N.SLOT_H)
    sc.tree_fit_bins(cands)
    good = sc.tree_fit(N.SLOT_R, 0, N.SLOT_W, 0, False, subspace=sub, max_depth=5, out_slot=N.SLOT_H)
    shifted = [c + 0.25 for c in cands]  # the same counts (and bins per column), other values: only the hash differs
    fewer = _cands(X, 4)
    for other in (shifted, fewer):
        sc.tree_fit_bins(cands)
        sc.ctxs[1].tree_fit_bins(other)
        res = _each(sc, fit)
        assert all(isinstance(e, N.NativeError) and e.code == N.SE_ERR_ARG for e in res), res
        assert all("ranks disagree on the fit" in str(e) for e in res), res
    # one rank fails its own checks (a weight slot of the wrong length): it keeps its error, its peer is told
    sc.tree_fit_bins(cands)
    sc.ctxs[1].alloc(N.SLOT_WOUT, 1, 7)
    res = _each(sc, lambda rk, c: c.tree_fit(N.SLOT_R, 0, N.SLOT_WOUT if rk == 1 else N.SLOT_W, 0, False, subspace=sub,
                                             max_depth=5, out_slot=N.SLOT_H))
    assert isinstance(res[0], N.NativeError) and "another rank failed" in str(res[0]), res
    assert isinstance(res[1], N.NativeError) and res[1].code == N.SE_ERR_STATE, res
    # different depths
    res = _each(sc, lambda rk, c: c.tree_fit(N.SLOT_R, 0, N.SLOT_W, 0, False, subspace=sub, max_depth=5 + rk,
                                             out_slot=N.SLOT_H))
    assert all(isinstance(e, N.NativeError) and "maxDepth" in str(e) for e in res), res
    # the same contexts fit again once the ranks agree
    t = sc.tree_fit(N.SLOT_R, 0, N.SLOT_W, 0, False, subspace=sub, max_depth=5, out_slot=N.SLOT_H)
    for k in TREE_KEYS:
        np.testing.assert_array_equal(t[k], good[k])
