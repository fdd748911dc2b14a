"""The device tree fits (se_tree_fit, se_tree_fit_classifier) on what boosting feeds them: the residuals the losses
produce, rows of multi-row slots, SAMME-like weights, wide and degenerate subspaces, one context reused across fits, and
the residual a one-launch squared round leaves.  Every fit is audited at every node (oracle/np_tree.audit,
np_tree_cls.audit) and, below the near ties, compared with the restatement node by node."""
import numpy as np
import pytest

from oracle import np_tree as T
from oracle import np_tree_cls as TC
from tests.test_gpu_tree_fit import _compare as _compare_reg
from tests.test_gpu_tree_fit import _near_tie
from tests.test_gpu_tree_fit_classifier import _compare as _compare_cls

pytestmark = pytest.mark.gpu

REG = ("max_depth", "min_instances", "min_info_gain", "min_weight_fraction")


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    yield c
    c.close()


def _params(depth=5, **kw):
    p = dict(max_depth=depth, min_instances=1, min_info_gain=0.0, min_weight_fraction=0.0)
    p.update(kw)
    return p


def _features(n, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(np.float32)
    z = np.sin(2 * X[:, 0]) + X[:, 1] * X[:, min(2, d - 1)] + 0.5 * rng.standard_normal(n)
    return X, z, rng


def _cands(X, bins):
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor
    return DeviceDecisionTreeRegressor(maxBins=bins, seed=11).split_candidates(X)


def _load_x(ctx, X, cands):
    from spark_ensemble_b200 import _native as N
    ctx.alloc(N.SLOT_X, X.shape[1], X.shape[0])
    ctx.upload_rowmajor(N.SLOT_X, X)
    ctx.tree_fit_bins(cands)


def _put(ctx, slot, v, rows=1):
    ctx.alloc(slot, rows, v.size // rows)
    ctx.upload(slot, np.ascontiguousarray(v, dtype=np.float32).reshape(-1))


def _reg(ctx, X, r, cands, *, w=None, bag=None, sub=None, params=None, wslot=None, load=True, exact=False):
    """Device regression fit on SLOT_R (weights in wslot, default SLOT_W), audited; returns (tree, out)."""
    from spark_ensemble_b200 import _native as N
    n, d = X.shape
    sub = np.arange(d, dtype=np.int32) if sub is None else np.asarray(sub, dtype=np.int32)
    params = params or _params()
    wslot = N.SLOT_W if wslot is None else wslot
    if load:
        _load_x(ctx, X, cands)
    _put(ctx, N.SLOT_R, r)
    ctx.alloc(N.SLOT_H, 1, n)
    if w is not None:
        _put(ctx, wslot, w)
    if bag is not None:
        _put(ctx, N.SLOT_BAG, bag)
    t = ctx.tree_fit(N.SLOT_R, 0, wslot if w is not None else -1, 0, bag is not None, subspace=sub,
                     out_slot=N.SLOT_H, out_row=0, **{k: params[k] for k in REG})
    out = ctx.download(N.SLOT_H)
    assert T.audit(t, X, cands, sub, r, w, bag, params, out=out, exact=exact) == t["feature"].size
    return t, out


def _reg_compare(t, X, r, cands, *, w=None, bag=None, sub=None, params=None):
    """The restatement's fit, node by node below the near ties; returns (compared, skipped, restatement tree)."""
    n, d = X.shape
    sub = np.arange(d) if sub is None else np.asarray(sub)
    ranks = [T.ranks(X[:, c], cands[c]) for c in sub]
    o = T.fit(ranks, [cands[c].size for c in sub], r, w=w, counts=bag, **(params or _params()))
    done, skipped = _compare_reg(t, o, ranks, [cands[c] for c in sub], np.arange(n), counts=bag)
    return done, skipped, o


def _cls(ctx, X, y, K, cands, *, w=None, bag=None, sub=None, params=None, wslot=None, load=True, proba=False,
         impurity="gini", exact=False):
    """Device classification fit on SLOT_Y (weights in wslot, default SLOT_W), audited; returns (tree, out)."""
    from spark_ensemble_b200 import _native as N
    n, d = X.shape
    sub = np.arange(d, dtype=np.int32) if sub is None else np.asarray(sub, dtype=np.int32)
    params = dict(params or _params(), num_classes=K, impurity=impurity)
    wslot = N.SLOT_W if wslot is None else wslot
    if load:
        _load_x(ctx, X, cands)
    _put(ctx, N.SLOT_Y, y)
    ctx.alloc(N.SLOT_PRED, 1, n)
    ctx.alloc(N.SLOT_PROBA, K, n)
    if w is not None:
        _put(ctx, wslot, w)
    if bag is not None:
        _put(ctx, N.SLOT_BAG, bag)
    t = ctx.tree_fit_classifier(N.SLOT_Y, K, 0, wslot if w is not None else -1, 0, bag is not None, subspace=sub,
                                impurity=impurity, proba=proba, out_slot=N.SLOT_PROBA if proba else N.SLOT_PRED,
                                **{k: params[k] for k in REG})
    out = ctx.download(N.SLOT_PROBA if proba else N.SLOT_PRED)
    if proba:
        assert TC.audit(t, X, cands, sub, y, w, bag, params, out_proba=out, exact=exact) == t["feature"].size
    else:
        assert TC.audit(t, X, cands, sub, y, w, bag, params, out=out, exact=exact) == t["feature"].size
    return t, out


def _cls_compare(t, X, y, K, cands, *, w=None, bag=None, sub=None, params=None, impurity="gini"):
    n, d = X.shape
    sub = np.arange(d) if sub is None else np.asarray(sub)
    ranks = [T.ranks(X[:, c], cands[c]) for c in sub]
    o = TC.fit(ranks, [cands[c].size for c in sub], y, K, w=w, counts=bag, impurity_kind=impurity,
               **(params or _params()))
    done, skipped = _compare_cls(t, o, ranks, [cands[c] for c in sub], np.arange(n), counts=bag)
    return done, skipped, o


def _classes(z, K):
    return np.minimum(np.digitize(z, np.quantile(z, np.linspace(0, 1, K + 1)[1:-1])), K - 1).astype(np.float32)


# ---- residuals the losses produce ------------------------------------------------------------------------------
def _residual(loss, z, rng, X):
    """Residuals of `loss`; for the two-valued ones, every row with X[:, 3] > 0.5 is on the positive side, so that the
    fit meets pure nodes."""
    F = (0.3 * z + 0.5 * rng.standard_normal(z.size)).astype(np.float32)
    e = z.astype(np.float32) - F
    if loss in ("absolute", "quantile"):
        e = np.where(X[:, 3] > 0.5, np.float32(1.0), e)
    if loss == "absolute":
        return np.where(e > 0, 1.0, -1.0).astype(np.float32)
    if loss == "quantile":  # {q, q - 1} in fp32, q = 0.9: not dyadic
        return np.where(e > 0, np.float32(0.9), np.float32(0.9) - np.float32(1.0)).astype(np.float32)
    if loss == "huber":  # clipped at the 20 % quantile of |e|: most rows at +-delta
        delta = np.float32(np.quantile(np.abs(e), 0.2))
        return np.clip(e, -delta, delta).astype(np.float32)
    if loss == "bernoulli":  # the first round: y - p0
        y = ((z > 0.3) | (X[:, 3] > 0.5)).astype(np.float32)
        return (y - np.float32(y.mean())).astype(np.float32)
    if loss == "logcosh":
        return np.tanh(e).astype(np.float32)
    assert loss == "offset"  # raw targets of DeviceDecisionTreeRegressor.fit: a large common offset
    return (1e5 + 1e3 * np.tanh(z)).astype(np.float32)


def _pure_nodes(t, X, cands, sub, r, bag):
    """Nodes of a fitted tree whose in-bag rows (two or more) all carry one residual value: the audit passes them as
    leaves, or as splits of noise-level gain whose children keep the node's mean."""
    R, _, bins = T.route(t, X, cands, sub)
    inb = np.ones(r.size, bool) if bag is None else bag > 0
    it, pure = T.walk(t, r.size), 0
    step = next(it)
    while step is not None:
        i, rows, _ = step
        v = r[rows[inb[rows]]]
        pure += int(v.size > 1 and bool((v == v[0]).all()))
        f = t["feature"][i]
        step = next(it, None) if f < 0 else T.send(it, R[f][rows] <= bins[i])
    return pure


LOSSES = ["absolute", "quantile", "huber", "bernoulli", "logcosh", "offset"]
MODES = ["plain", "weighted", "bagged"]


@pytest.mark.parametrize("loss", LOSSES)
@pytest.mark.parametrize("mode", MODES)
def test_loss_residuals(ctx, loss, mode):
    n = 20001
    X, z, rng = _features(n, 8, seed=10 * LOSSES.index(loss) + MODES.index(mode))
    r = _residual(loss, z, rng, X)
    w = rng.uniform(0.25, 4.0, n).astype(np.float32) if mode == "weighted" else None
    bag = rng.poisson(1.0, n).astype(np.float32) if mode == "bagged" else None
    cands = _cands(X, 32)
    sub = np.array([5, 0, 7, 1, 2, 3], np.int32)
    t, out = _reg(ctx, X, r, cands, w=w, bag=bag, sub=sub)
    done, skipped, o = _reg_compare(t, X, r, cands, w=w, bag=bag, sub=sub)
    pure = _pure_nodes(t, X, cands, sub, r, bag)
    print(f"{loss} {mode}: nodes {t['feature'].size}, all audited, {done} compared, {skipped} subtrees skipped, "
          f"{pure} pure")
    assert t["feature"][0] >= 0 and done >= 1
    if loss in ("absolute", "quantile", "bernoulli"):
        assert pure >= 1, "the two-valued residuals must meet a pure node"


# ---- rows of multi-row slots -----------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [3, 9])
def test_regression_on_rows_of_a_multi_row_slot(ctx, K):
    """R row j with WOUT row j as weights (the Newton step of a K-class LogLoss fit) and without weights (the gradient
    step), written to H row j: n = 10001 pads each row to 10016 values.  No other row of H changes."""
    from spark_ensemble_b200 import _native as N
    n = 10001
    X, z, rng = _features(n, 6, seed=K)
    cands = _cands(X, 32)
    _load_x(ctx, X, cands)
    logits = rng.standard_normal((K, n)) + np.outer(np.arange(K), z) / K
    p = np.exp(logits - logits.max(axis=0))
    p /= p.sum(axis=0)
    y = rng.integers(0, K, n)
    R = (np.eye(K)[y].T - p).astype(np.float32)           # -g of LogLoss
    WO = np.maximum(p * (1 - p), 1e-16).astype(np.float32)  # the Newton weights
    _put(ctx, N.SLOT_R, R, K)
    _put(ctx, N.SLOT_WOUT, WO, K)
    H0 = rng.standard_normal((K, n)).astype(np.float32)
    _put(ctx, N.SLOT_H, H0, K)
    assert ctx.layout(N.SLOT_H)[2] > n
    H = H0.copy()
    for j in (1, K - 1):
        for wslot in (N.SLOT_WOUT, -1):  # Newton weights, and the unweighted gradient step
            t = ctx.tree_fit(N.SLOT_R, j, wslot, j, False, subspace=np.arange(6, dtype=np.int32), max_depth=4,
                             out_slot=N.SLOT_H, out_row=j)
            got = ctx.download(N.SLOT_H).reshape(K, n)
            H[j] = got[j]
            np.testing.assert_array_equal(got.view(np.uint32), H.view(np.uint32))  # only row j changed
            wj = WO[j] if wslot >= 0 else None
            assert T.audit(t, X, cands, np.arange(6), R[j], wj, None, _params(4), out=got[j]) == t["feature"].size


def test_classifier_out_rows_of_a_multi_row_slot(ctx):
    from spark_ensemble_b200 import _native as N
    n, K = 10002, 4
    X, z, rng = _features(n, 5, seed=4)
    y = _classes(z, K)
    cands = _cands(X, 32)
    _load_x(ctx, X, cands)
    _put(ctx, N.SLOT_Y, y)
    sub = np.arange(5, dtype=np.int32)
    params = dict(_params(4), num_classes=K, impurity="entropy")
    P0 = rng.standard_normal((K + 3, n)).astype(np.float32)
    _put(ctx, N.SLOT_P, P0, K + 3)
    t = ctx.tree_fit_classifier(N.SLOT_Y, K, subspace=sub, impurity="entropy", max_depth=4, proba=True,
                                out_slot=N.SLOT_P, out_row=2)
    got = ctx.download(N.SLOT_P).reshape(K + 3, n)
    np.testing.assert_array_equal(got[[0, 1, K + 2]].view(np.uint32), P0[[0, 1, K + 2]].view(np.uint32))
    TC.audit(t, X, cands, sub, y, params=params, out_proba=got[2:2 + K])
    t2 = ctx.tree_fit_classifier(N.SLOT_Y, K, subspace=sub, impurity="entropy", max_depth=4, out_slot=N.SLOT_P,
                                 out_row=K + 2)
    got2 = ctx.download(N.SLOT_P).reshape(K + 3, n)
    np.testing.assert_array_equal(got2[:K + 2].view(np.uint32), got[:K + 2].view(np.uint32))
    TC.audit(t2, X, cands, sub, y, params=params, out=got2[K + 2])


# ---- weights ---------------------------------------------------------------------------------------------------
def _weights(kind, n, rng):
    if kind == "zeros":  # 20 % exact zeros
        return np.where(rng.random(n) < 0.2, 0.0, rng.uniform(0.5, 2.0, n)).astype(np.float32)
    if kind == "span":  # 1e-30 .. 1, log-uniform: SAMME's weights after many rounds
        return (10.0 ** rng.uniform(-30, 0, n)).astype(np.float32)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32)  # one row carries most of the weight
    w[7] = 1e6
    return w


@pytest.mark.parametrize("kind", ["zeros", "span", "dominant"])
def test_weights(ctx, kind):
    n = 20000
    X, z, rng = _features(n, 6, seed=len(kind))
    w = _weights(kind, n, rng)
    cands = _cands(X, 32)
    r = (z + 0.2 * rng.standard_normal(n)).astype(np.float32)
    t, _ = _reg(ctx, X, r, cands, w=w)
    done, skipped, _ = _reg_compare(t, X, r, cands, w=w)
    print(f"regression {kind}: nodes {t['feature'].size}, all audited, {done} compared, {skipped} subtrees skipped")
    y = _classes(z, 3)
    for impurity in ("gini", "entropy"):
        t, _ = _cls(ctx, X, y, 3, cands, w=w, impurity=impurity, load=False)
        t, _ = _cls(ctx, X, y, 3, cands, w=w, impurity=impurity, load=False, proba=True)
        done, skipped, _ = _cls_compare(t, X, y, 3, cands, w=w, impurity=impurity)
        print(f"classification {kind} {impurity}: nodes {t['feature'].size}, {done} compared, {skipped} skipped")


def test_weight_scale_does_not_change_the_fit(ctx):
    """Weights x 2^-60 and x 2^60 are exact in fp32, and on dyadic data every sum is exact: the same tree and the same
    output, bit for bit -- WOUT for the regressor (the Newton weights without their 1/S), BW for the classifier (the
    unnormalised SAMME weights)."""
    from spark_ensemble_b200 import _native as N
    rng = np.random.default_rng(60)
    n = 8191
    X = rng.integers(0, 16, (n, 4)).astype(np.float32)
    r = (rng.integers(-8, 8, n) / 4).astype(np.float32)
    y = (rng.integers(0, 3, n)).astype(np.float32)
    w = rng.integers(1, 5, n).astype(np.float32)
    cands = _cands(X, 32)
    _load_x(ctx, X, cands)
    ref = None
    for s in (1.0, 2.0 ** -60, 2.0 ** 60):
        t, out = _reg(ctx, X, r, cands, w=(w * np.float32(s)).astype(np.float32), wslot=N.SLOT_WOUT, load=False,
                      exact=True)
        tc, outc = _cls(ctx, X, y, 3, cands, w=(w * np.float32(s)).astype(np.float32), wslot=N.SLOT_BW, load=False,
                        proba=True, exact=True)
        got = (t, out, tc, outc)
        if ref is None:
            ref = got
            continue
        for a, b in zip(got, ref):
            if isinstance(a, dict):
                for k in ("feature", "threshold", "left", "right", "value", "gain"):
                    np.testing.assert_array_equal(a[k], b[k])
                if "values" in a:
                    np.testing.assert_array_equal(a["values"], b["values"])
                    np.testing.assert_array_equal(a["class_weights"] / s, b["class_weights"])
            else:
                np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))


# ---- all-zero weights and a root with no in-bag weight -----------------------------------------------------------
@pytest.mark.parametrize("how", ["weights", "bag"])
def test_root_without_in_bag_weight(ctx, how):
    """The regressor's prediction is S / W = 0 / 0: a NaN leaf, NaN in every row of the output; the classifier's is
    label 0 with all-zero probabilities (DESIGN.md §3)."""
    n = 1003
    X, z, rng = _features(n, 3, seed=5)
    cands = _cands(X, 32)
    zero = np.zeros(n, np.float32)
    kw = {"w": zero} if how == "weights" else {"bag": zero}
    t, out = _reg(ctx, X, z.astype(np.float32), cands, **kw)
    assert t["feature"].tolist() == [-1] and np.isnan(t["value"][0]) and np.isnan(out).all()
    y = _classes(z, 3)
    t, out = _cls(ctx, X, y, 3, cands, load=False, **kw)
    assert t["feature"].tolist() == [-1] and t["value"][0] == 0 and (out == 0).all()
    t, out = _cls(ctx, X, y, 3, cands, load=False, proba=True, **kw)
    assert (t["values"] == 0).all() and (out == 0).all()


# ---- shapes ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,depth,bins", [(128, 4, 32), (300, 3, 32), (300, 6, 256)])
def test_wide_subspaces(ctx, S, depth, bins):
    """|S| above the 256 threads of tree_split_kernel and the 8 warps of tree_split_cls_kernel; (300, 6, 256): the
    regressor's level 5 and the 64-class classifier's levels >= 1 take the global-atomics histograms."""
    n = 6001
    X, z, rng = _features(n, S + 2, seed=S + depth)
    z = z + X[:, S // 2] + np.sin(X[:, S])  # informative columns spread over the subspace
    sub = rng.permutation(S + 2)[:S].astype(np.int32)
    cands = _cands(X, bins)
    r = z.astype(np.float32)
    t, _ = _reg(ctx, X, r, cands, sub=sub, params=_params(depth))
    K = 64 if bins == 256 else 5
    y = _classes(z, K)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32)
    tc, _ = _cls(ctx, X, y, K, cands, sub=sub, w=w, params=_params(min(depth, 3)), load=False)
    if S < 300:  # the restatement loops over candidates in Python: the audit alone is the check at |S| = 300
        _reg_compare(t, X, r, cands, sub=sub, params=_params(depth))
        _cls_compare(tc, X, y, K, cands, sub=sub, w=w, params=_params(min(depth, 3)))


def test_columns_without_candidates_and_a_full_column(ctx):
    """Constant and all-NaN columns (0 candidates) first in the subspace, where the root's totals are read, and
    interleaved; a column of exactly 255 candidates whose last rank (255) holds both +inf and NaN rows."""
    n = 5003
    X, z, rng = _features(n, 4, seed=255)
    full = rng.permutation(np.r_[np.arange(255, dtype=np.float32), np.float32(np.inf)])[np.arange(n) % 256]
    full[rng.random(n) < 0.05] = np.nan
    X = np.column_stack([np.full(n, 3.0), np.full(n, np.nan), X[:, 0], np.full(n, -1.0), full, X[:, 1:]])
    X = X.astype(np.float32)
    z = z + 0.01 * np.nan_to_num(full, nan=300, posinf=400)
    cands = _cands(X, 256)
    assert cands[0].size == cands[1].size == cands[3].size == 0 and cands[4].size == 255
    for sub in ([0, 1, 2, 3, 4, 5, 6, 7], [1, 4, 0, 2, 3, 6], [3, 0], [0, 4]):
        sub = np.asarray(sub, np.int32)
        r = z.astype(np.float32)
        t, _ = _reg(ctx, X, r, cands, sub=sub)
        if len(sub) == 2 and 4 not in sub:
            assert t["feature"].tolist() == [-1]
        y = _classes(z, 3)
        _cls(ctx, X, y, 3, cands, sub=sub, load=False)
        _cls(ctx, X, y, 3, cands, sub=sub, load=False, proba=True, impurity="entropy")


@pytest.mark.parametrize("n", [4097, 4098, 4099])
def test_row_counts_off_the_four_row_tiles(ctx, n):
    X, z, rng = _features(n, 5, seed=n)
    cands = _cands(X, 32)
    bag = rng.poisson(1.0, n).astype(np.float32)
    bag[-3:] = 5.0  # the last rows weigh: a tail lost from a tile would show in every statistic
    t, _ = _reg(ctx, X, z.astype(np.float32), cands, bag=bag)
    _reg_compare(t, X, z.astype(np.float32), cands, bag=bag)
    _cls(ctx, X, _classes(z, 3), 3, cands, bag=bag, load=False)


# ---- one context, many fits ------------------------------------------------------------------------------------
def test_one_context_many_fits():
    """n, |S|, depth, maxBins and K grow and shrink in one context (reallocating X and the scratch, then reusing the
    larger scratch); X is re-uploaded between fits (fitted straight after the upload) and the candidates are set again
    after a tree walk took a column off the fit.  Each fit equals the same fit in a fresh context (where there is no near tie: the audit covers it)."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    seq = [(3000, 6, 3, 32, 3), (20000, 24, 6, 64, 26), (1001, 2, 1, 2, 2), (30000, 40, 2, 256, 64),
           (5000, 12, 5, 64, 5)]
    shared = Context(0)
    try:
        for i, (n, S, depth, bins, K) in enumerate(seq):
            X, z, rng = _features(n, S, seed=i)
            r = z.astype(np.float32)
            y = _classes(z, K)
            cands = _cands(X, bins)
            p = _params(depth)
            t, out = _reg(shared, X, r, cands, params=p)
            tc, outc = _cls(shared, X, y, K, cands, params=p, load=False, proba=True)
            # X re-uploaded with its rows reversed and fitted with no se_tree_fit_bins in between: the fit must re-rank
            # the rewritten X itself (the candidates are unchanged: the same values); stale ranks fail the audit
            X2 = X[::-1].copy()
            shared.upload_rowmajor(N.SLOT_X, X2)
            _reg(shared, X2, r[::-1].copy(), cands, params=p, load=False)
            shared.upload_rowmajor(N.SLOT_X, X)
            _reg(shared, X, r, cands, params=p, load=False)
            host = {"feature": np.array([0, -1, -1], np.int32), "threshold": np.float32([0.123456, 0, 0]),
                    "left": np.array([1, 0, 0], np.int32), "right": np.array([2, 0, 0], np.int32),
                    "value": np.float32([0, 1, 2])}
            shared.alloc(N.SLOT_RAW, 1, n)
            shared.tree_predict(host, N.SLOT_RAW, 0)  # column 0 no longer holds the fit's candidates
            shared.tree_fit_bins(cands)
            t2, out2 = _reg(shared, X, r, cands, params=p, load=False)
            with Context(0) as fresh:
                tf, outf = _reg(fresh, X, r, cands, params=p)
                tcf, outcf = _cls(fresh, X, y, K, cands, params=p, load=False, proba=True)
            ranks = [T.ranks(X[:, c], cands[c]) for c in range(S)]
            o = T.fit(ranks, [c.size for c in cands], r, **p)
            oc = TC.fit(ranks, [c.size for c in cands], y, K, **p)
            if not any(_near_tie(x) for x in o["info"]):
                for a in (t, t2):
                    for k in ("feature", "threshold", "left", "right", "value"):
                        np.testing.assert_array_equal(a[k], tf[k])
                np.testing.assert_array_equal(out.view(np.uint32), outf.view(np.uint32))
                np.testing.assert_array_equal(out2.view(np.uint32), outf.view(np.uint32))
            if not any(_near_tie(x) for x in oc["info"]):
                for k in ("feature", "threshold", "left", "right", "value", "values"):
                    np.testing.assert_array_equal(tc[k], tcf[k])
                np.testing.assert_array_equal(outc.view(np.uint32), outcf.view(np.uint32))
    finally:
        shared.close()


# ---- after a one-launch squared round ----------------------------------------------------------------------------
def test_fit_on_the_residual_a_one_launch_round_leaves():
    """The residual-mode one-launch squared round leaves F owed (F = y - r, rebuilt when read).  A fit on R reads r
    without rebuilding F, and equals the fit on the downloaded R in a fresh context."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    n = 40961
    X, z, rng = _features(n, 6, seed=41)
    cands = _cands(X, 32)
    y = z.astype(np.float32)
    with Context(0) as c:
        c.set_option("fused_round", 1)
        c.gbm_configure(n, 0, 1, "squared", 0.0, False)
        c.upload(N.SLOT_Y, y)
        c.upload(N.SLOT_F, (0.3 * z).astype(np.float32))
        c.upload(N.SLOT_H, (0.5 * z + 0.3 * rng.standard_normal(n)).astype(np.float32))
        for _ in range(2):
            c.gbm_round(0.7, True, 1e-6, 100, residual=True)
            assert c.get_option("last_round_fused") == 1
        _load_x(c, X, cands)
        r = c.download(N.SLOT_R).copy()
        sub = np.arange(6, dtype=np.int32)
        counts = []
        for _ in range(2):
            lc = c.launch_count
            t = c.tree_fit(N.SLOT_R, 0, -1, 0, False, subspace=sub, max_depth=4, out_slot=N.SLOT_H)
            counts.append(c.launch_count - lc)
            out = c.download(N.SLOT_H)
        lc = c.launch_count
        F = c.download(N.SLOT_F)  # the owed F: one settling launch, so the fits above did not settle it
        assert c.launch_count == lc + 1
        assert counts[0] == counts[1]
        np.testing.assert_array_equal(F, (y.astype(np.float64) - r).astype(np.float32))
    assert T.audit(t, X, cands, sub, r, params=_params(4), out=out) == t["feature"].size
    with Context(0) as fresh:
        tf, outf = _reg(fresh, X, r, cands, params=_params(4))
    ranks = [T.ranks(X[:, k], cands[k]) for k in sub]
    if not any(_near_tie(x) for x in T.fit(ranks, [k.size for k in cands], r, max_depth=4)["info"]):
        for k in ("feature", "threshold", "left", "right", "value"):
            np.testing.assert_array_equal(t[k], tf[k])
        np.testing.assert_array_equal(out.view(np.uint32), outf.view(np.uint32))
