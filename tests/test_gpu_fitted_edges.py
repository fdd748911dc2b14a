"""GPU tests in the regimes the broad parity suite does not reach: LogLoss on well-fitted rows (the label class leads
by a margin of up to 20, the per-row loss and gradients shrink like exp(-margin)), scalar losses at large |F| and at
exact ties y == F, and tree walks over non-finite, signed-zero and denormal features.

Every kernel output is compared with an fp64 reference computed from the SAME fp32 inputs the kernel sees (p = F + c h
is rounded to fp32 exactly as the kernel's fma does), element by element, at 1e-5 relative.  The only absolute floor is
FLT_MIN: the approximate SFU ops flush denormal results to zero.  LogLoss is referenced to the stable fp64 form of
oracle/np_oracle.py (logloss_stable), which the CPU suite pins against the C oracle up to a margin of 20."""
import numpy as np
import pytest

from oracle import np_oracle as NP
from tests.test_gpu_parity import _random_unbalanced_tree, _walk

pytestmark = pytest.mark.gpu

RTOL = 1e-5
FLT_MIN = float(np.finfo(np.float32).tiny)
FLT_MAX = float(np.finfo(np.float32).max)
KS = [2, 3, 4, 5, 8, 9, 16, 17, 26, 32, 33, 64, 65, 200]   # register kernel, every tiled KMAX bucket, generic kernel
MARGINS = [0, 4, 8, 12, 16, 20]


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    yield c
    c.close()


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def d64(a):
    return np.asarray(a, dtype=np.float64)


def rel_close(got, want, what):
    """|got - want| <= 1e-5 |want| + FLT_MIN, element by element."""
    got, want = d64(got), d64(want)
    bad = ~(np.abs(got - want) <= RTOL * np.abs(want) + FLT_MIN)
    if bad.any():
        i = np.flatnonzero(bad.ravel())[0]
        worst = np.max(np.abs(got - want)[bad] / np.maximum(np.abs(want)[bad], FLT_MIN))
        raise AssertionError(f"{what}: {bad.sum()} / {want.size} beyond 1e-5 relative; worst {worst:.3e}; first at flat "
                             f"index {i}: got {got.ravel()[i]!r}, want {want.ravel()[i]!r}")


def fma32(F, c, h):
    """fp32 fmaf(c, h, F) of the kernels: the exact value rounded once (c h is exact in fp64)."""
    c = d64(f32(c))
    return d64(f32(d64(F) + c.reshape(-1, 1) * d64(h)))


# ------------------------------------------------------------------ LogLoss on well-fitted rows
def fitted_rows(rng, K, n, margin, mixed):
    """Classes N(0, 0.5); the label class at +margin.  mixed: one row in eight has ANOTHER class at +margin, so its
    label is not the argmax (its loss is about the margin and hides the fitted rows in the sums: both cases run)."""
    y = rng.integers(0, K, n)
    top = y.copy()
    if mixed:
        other = rng.random(n) < 0.125
        top[other] = (y[other] + rng.integers(1, K, int(other.sum()))) % K
    F = rng.normal(0.0, 0.5, (K, n))
    F[top, np.arange(n)] += margin
    # a direction along the negative gradient (label class up, the others down): every h g has one sign, so the
    # line-search gradient sums do not cancel and compare at 1e-5 relative like single elements
    sign = np.where(np.arange(K)[:, None] == y[None, :], 1.0, -1.0)
    h = sign * rng.uniform(0.5, 1.5, (K, n)) * 0.3
    return f32(y), f32(F), f32(h)


def ll_ref(y, P):
    return NP.logloss_stable(y.astype(np.int64), d64(P))


@pytest.mark.parametrize("n", [257, 40961])
@pytest.mark.parametrize("mixed", [False, True])
@pytest.mark.parametrize("margin", MARGINS)
@pytest.mark.parametrize("K", KS)
def test_logloss_fitted_rows(ctx, rng, K, margin, mixed, n):
    """Every LogLoss entry point on well-fitted rows: mean loss (train / validation), the validation update, the
    line-search loss and gradient sums (weighted, with and without a bag), gradient and newton residuals, and the
    fused update in plain / residual / newton mode with its loss."""
    from spark_ensemble_b200 import _native as N
    y, F, h = fitted_rows(rng, K, n, margin, mixed)
    vy, vF, vh = fitted_rows(rng, K, n, margin, mixed)
    w = f32(rng.random(n) + 0.5)
    ctx.gbm_configure(n, n, K, "logloss", 0.0, True)
    for slot, v in ((N.SLOT_Y, y), (N.SLOT_F, F), (N.SLOT_H, h), (N.SLOT_W, w), (N.SLOT_VY, vy), (N.SLOT_VF, vF),
                    (N.SLOT_VH, vh)):
        ctx.upload(slot, v)
    w64 = d64(w)

    # mean loss, train and validation
    lo, g, hs = ll_ref(y, F)
    rel_close(ctx.gbm_mean_loss(False), lo.mean(), "mean train loss")
    rel_close(ctx.gbm_mean_loss(True), ll_ref(vy, vF)[0].mean(), "mean validation loss")

    # line search: loss (counted K times per row) and Σ c h g over Σ c w, without and with a bag
    alpha = f32(rng.uniform(0.2, 1.0, K))
    p = fma32(F, alpha, h)
    lp, gp, _ = ll_ref(y, p)
    bag = f32(rng.poisson(1.0, n))
    for c in (None, bag):
        cc = np.ones(n) if c is None else d64(c)
        ctx.gbm_set_bag(c)
        lg, gg = ctx.gbm_linesearch_eval(d64(alpha))
        ws = np.sum(cc * w64)
        rel_close(lg, K * np.sum(cc * lp) / ws, f"line-search loss (bag={c is not None})")
        rel_close(gg, (cc * d64(h) * gp).sum(axis=1) / ws, f"line-search gradient sums (bag={c is not None})")
    ctx.gbm_set_bag(None)

    # residuals at F: gradient mode, then newton mode (R = -g / hc, WOUT = hc w / 2S, S = Σ hc)
    ctx.gbm_pseudo_residuals(newton=False)
    rel_close(ctx.download(N.SLOT_R).reshape(K, n), -g, "gradient residuals")
    S = ctx.gbm_pseudo_residuals(newton=True)
    hc = np.maximum(hs, 1e-2)
    rel_close(S, hc.sum(axis=1), "newton S")
    rel_close(ctx.download(N.SLOT_R).reshape(K, n), -g / hc, "newton residuals")
    rel_close(ctx.download(N.SLOT_WOUT).reshape(K, n), 0.5 * hc / hc.sum(axis=1)[:, None] * w64, "newton weights")

    # fused update F' = F + step h (one fp32 rounding) with the loss and the next residuals at F'
    step = f32(rng.uniform(0.1, 0.6, K))
    for mode in ("plain", "residual", "newton"):
        ctx.upload(N.SLOT_F, F)
        ls, S = ctx.gbm_update(d64(step), residual=(mode == "residual"), newton=(mode == "newton"), loss=True)
        Fg = ctx.download(N.SLOT_F).reshape(K, n)
        np.testing.assert_array_equal(Fg, f32(fma32(F, step, h)))
        lo2, g2, hs2 = ll_ref(y, Fg)
        rel_close(ls / n, lo2.mean(), f"{mode} update loss")
        if mode == "residual":
            rel_close(ctx.download(N.SLOT_R).reshape(K, n), -g2, "residuals after the update")
        if mode == "newton":
            hc2 = np.maximum(hs2, 1e-2)
            rel_close(S, hc2.sum(axis=1), "newton S after the update")
            rel_close(ctx.download(N.SLOT_R).reshape(K, n), -g2 / hc2, "newton residuals after the update")
            rel_close(ctx.download(N.SLOT_WOUT).reshape(K, n), 0.5 * hc2 / hc2.sum(axis=1)[:, None] * w64,
                      "newton weights after the update")

    # validation update
    vstep = f32(rng.uniform(0.1, 0.6, K))
    lv = ctx.gbm_update_validation(d64(vstep))
    vFg = ctx.download(N.SLOT_VF).reshape(K, n)
    np.testing.assert_array_equal(vFg, f32(fma32(vF, vstep, vh)))
    rel_close(lv, ll_ref(vy, vFg)[0].mean(), "validation update loss")


# ------------------------------------------------------------------ scalar losses at large margins and at ties
PARAM = {"huber": 0.9, "quantile": 0.9, "scaledlogcosh": 0.9}
HESS = ("logcosh", "scaledlogcosh", "bernoulli", "exponential")


def scalar_rows(rng, name, n):
    if name in ("bernoulli", "exponential"):           # |F| up to 40: margins far beyond the N(0, 0.7) of the suite
        y = f32(rng.random(n) < 0.4)
        F = f32(rng.uniform(-40.0, 40.0, n))
        F[: n // 8] = f32(rng.standard_normal(n // 8))
    elif name in ("logcosh", "scaledlogcosh"):         # |y - F| from 1e-3 to 60, across the 0.25 series / exp switch
        y = f32(rng.standard_normal(n))
        d = np.exp(rng.uniform(np.log(1e-3), np.log(60.0), n)) * rng.choice([-1.0, 1.0], n)
        F = f32(y - d)
    else:                                              # F = median(y): round 1 of a fit; a quarter of the rows tie exactly
        y = f32(rng.standard_normal(n))
        F = np.full(n, np.median(y), np.float32)
        F[: n // 4] = y[: n // 4]
    return y, F


def scalar_ref(name, y, p):
    par = PARAM.get(name, 0.0)
    ye = NP.encode(name, d64(y))
    p = d64(p)
    hs = NP.hessian(name, par, ye, p) if name in HESS else None
    return NP.loss(name, par, ye, p), NP.gradient(name, par, ye, p), hs


@pytest.mark.parametrize("n", [257, 40961])
@pytest.mark.parametrize("name", ["bernoulli", "exponential", "logcosh", "scaledlogcosh", "absolute", "quantile", "huber"])
def test_scalar_losses_large_margins_and_ties(ctx, rng, name, n):
    from spark_ensemble_b200 import _native as N
    par = PARAM.get(name, 0.0)
    y, F = scalar_rows(rng, name, n)
    vy, vF = scalar_rows(rng, name, n)
    h = f32(rng.standard_normal(n))
    vh = f32(rng.standard_normal(n))
    w = f32(rng.random(n) + 0.5)
    w64 = d64(w)
    ctx.gbm_configure(n, n, 1, name, par, True)
    for slot, v in ((N.SLOT_Y, y), (N.SLOT_F, F), (N.SLOT_H, h), (N.SLOT_W, w), (N.SLOT_VY, vy), (N.SLOT_VF, vF),
                    (N.SLOT_VH, vh)):
        ctx.upload(slot, v)
    lo, g, hs = scalar_ref(name, y, F)
    rel_close(ctx.gbm_mean_loss(False), lo.mean(), "mean train loss")
    rel_close(ctx.gbm_mean_loss(True), scalar_ref(name, vy, vF)[0].mean(), "mean validation loss")
    if name in ("absolute", "quantile", "huber"):
        tie = y == F
        assert tie.sum() >= n // 4
        want = {"absolute": 0.0, "quantile": 1.0 - par, "huber": 0.0}[name]
        assert np.all(g[tie] == want)

    # line search at alpha = 0 (p = F: the ties stay ties) and at two alphas, without and with a bag.  The gradient
    # sums Σ c h g cancel (h is random): they are held to 1e-5 of Σ |c h g|, the scale of their rounding
    bag = f32(rng.poisson(1.0, n))
    for c in (None, bag):
        cc = np.ones(n) if c is None else d64(c)
        ctx.gbm_set_bag(c)
        ws = np.sum(cc * w64)
        for a in (0.0, 0.375, 1.75):
            p = fma32(F.reshape(1, n), [a], h.reshape(1, n))[0]
            lp, gp, _ = scalar_ref(name, y, p)
            lg, gg = ctx.gbm_linesearch_eval([a])
            rel_close(lg, np.sum(cc * lp) / ws, f"line-search loss (alpha={a}, bag={c is not None})")
            terms = cc * d64(h) * gp
            assert abs(gg[0] - terms.sum() / ws) <= RTOL * np.abs(terms).sum() / ws + FLT_MIN, \
                (a, c is not None, gg[0], terms.sum() / ws)
    ctx.gbm_set_bag(None)

    ctx.gbm_pseudo_residuals(newton=False)
    rel_close(ctx.download(N.SLOT_R), -g, "gradient residuals")
    if name in HESS:
        S = ctx.gbm_pseudo_residuals(newton=True)
        hc = np.maximum(hs, 1e-2)
        rel_close(S, [hc.sum()], "newton S")
        rel_close(ctx.download(N.SLOT_R), -g / hc, "newton residuals")
        rel_close(ctx.download(N.SLOT_WOUT), 0.5 * hc / hc.sum() * w64, "newton weights")

    step = f32([0.25])
    for mode in ("plain", "residual") + (("newton",) if name in HESS else ()):
        ctx.upload(N.SLOT_F, F)
        ls, S = ctx.gbm_update(d64(step), residual=(mode == "residual"), newton=(mode == "newton"), loss=True)
        Fg = ctx.download(N.SLOT_F)
        np.testing.assert_array_equal(Fg, f32(fma32(F.reshape(1, n), step, h.reshape(1, n))[0]))
        lo2, g2, hs2 = scalar_ref(name, y, Fg)
        rel_close(ls / n, lo2.mean(), f"{mode} update loss")
        if mode == "residual":
            rel_close(ctx.download(N.SLOT_R), -g2, "residuals after the update")
        if mode == "newton":
            hc2 = np.maximum(hs2, 1e-2)
            rel_close(S, [hc2.sum()], "newton S after the update")
            rel_close(ctx.download(N.SLOT_R), -g2 / hc2, "newton residuals after the update")
    lv = ctx.gbm_update_validation([0.5])
    vFg = ctx.download(N.SLOT_VF)
    rel_close(lv, scalar_ref(name, vy, vFg)[0].mean(), "validation update loss")

    # the persistent device line search (ls_mode 1): the objective it reports at its minimiser, against the fp64
    # objective at that alpha; and the host Brent over single-evaluation launches of the same kernel, bit for bit
    ctx.upload(N.SLOT_F, F)
    try:
        ctx.set_option("ls_mode", 1)
        a, l, ne = ctx.gbm_linesearch_brent()
        assert ne >= 1
        p = fma32(F.reshape(1, n), [a], h.reshape(1, n))[0]
        rel_close(l, np.sum(scalar_ref(name, y, p)[0]) / np.sum(w64), "device line search objective")
        ctx.set_option("ls_mode", 2)
        assert ctx.gbm_linesearch_brent() == (a, l, ne)
    finally:
        ctx.set_option("ls_mode", 1)


# ------------------------------------------------------------------ tree walks on edge features
DENORMS = [1e-45, -1e-45, 1e-40, -1e-40, FLT_MIN / 2, -FLT_MIN / 2]
SPECIAL_X = [np.nan, np.inf, -np.inf, FLT_MAX, -FLT_MAX, 0.0, -0.0, FLT_MIN, -FLT_MIN] + DENORMS
SPECIAL_T = [np.inf, -np.inf, 0.0, -0.0]


def edge_matrix(rng, n, d, cand):
    """Columns mixing N(0,1) values, the special values above and the column's own thresholds (rows ON a threshold)."""
    X = rng.standard_normal((n, d)).astype(np.float32)
    for f in range(d):
        pool = np.array(SPECIAL_X + list(cand[f]), dtype=np.float32)
        pick = rng.random(n) < 0.7
        X[pick, f] = pool[rng.integers(0, pool.size, int(pick.sum()))]
    X[:len(SPECIAL_X), 0] = np.array(SPECIAL_X, np.float32)   # every special value at least once
    return X


def edge_candidates(rng, d):
    return [SPECIAL_T + list(rng.standard_normal(6).astype(np.float32)) for _ in range(d)]


def assert_all_paths(ctx, N, tree, X, sub=None):
    """tree_bins 0 (fp32 walk), rank walk (tree_mask 0), all-nodes mask kernel, multi-output: the numpy walk's leaf."""
    Xs = X if sub is None else X[:, sub]
    want = tree["value"][_walk(tree, Xs)]
    try:
        for bins, mask in ((0, 1), (1, 0), (1, 1)):
            ctx.set_option("tree_bins", bins)
            ctx.set_option("tree_mask", mask)
            ctx.tree_predict(tree, N.SLOT_H, 0, subspace=sub)
            assert ctx.get_option("last_tree_binned") == bins
            n_internal = int(np.sum(np.asarray(tree["feature"]) >= 0))
            assert ctx.get_option("last_tree_mask") == (1 if bins and mask and n_internal <= 64 else 0)
            np.testing.assert_array_equal(ctx.download(N.SLOT_H), want, err_msg=f"tree_bins={bins} tree_mask={mask}")
        if "values" in tree:
            k = tree["values"].shape[1]
            ctx.alloc(N.SLOT_PROBA, k, X.shape[0])
            ctx.tree_predict_multi(tree, N.SLOT_PROBA, subspace=sub)
            np.testing.assert_array_equal(ctx.download(N.SLOT_PROBA).reshape(k, -1), tree["values"][_walk(tree, Xs)].T)
    finally:
        ctx.set_option("tree_bins", 1)
        ctx.set_option("tree_mask", 1)


@pytest.mark.parametrize("n", [19, 4099])
def test_tree_walks_on_edge_features(rng, n):
    """NaN, +-inf, +-FLT_MAX, +-0 and denormal features against thresholds of +-inf, +0 and -0 (and ordinary ones):
    every walk must pick the leaf of `x <= t` (NaN goes right at every node, like Spark's shouldGoLeft)."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    d = 6
    cand = edge_candidates(rng, d)
    X = edge_matrix(rng, n, d, cand)
    ctx = Context(0)
    try:
        ctx.alloc(N.SLOT_X, d, n)
        ctx.upload_rowmajor(N.SLOT_X, X)
        ctx.alloc(N.SLOT_H, 1, n)
        # stumps: one special threshold at a time on the column that holds every special value
        for t in SPECIAL_T + [FLT_MIN / 2]:
            stump = {"feature": np.array([0, -1, -1], np.int32), "threshold": np.array([t, 0, 0], np.float32),
                     "left": np.array([1, 0, 0], np.int32), "right": np.array([2, 0, 0], np.int32),
                     "value": np.array([0.0, 1.0, 2.0], np.float32)}
            assert_all_paths(ctx, N, stump, X)
        for n_internal in (5, 40, 64, 90):
            tree = _random_unbalanced_tree(rng, n_internal, d, cand)
            tree["values"] = rng.random((tree["feature"].size, 3)).astype(np.float32)
            assert_all_paths(ctx, N, tree, X)
        sub = np.array([0, 2, 3, 5], np.int32)
        tree = _random_unbalanced_tree(rng, 30, sub.size, [cand[c] for c in sub])
        assert_all_paths(ctx, N, tree, X, sub)
    finally:
        ctx.close()


@pytest.mark.parametrize("n", [19, 4099])
def test_forest_on_edge_features(rng, n):
    """se_forest_predict over the rank matrix of X and of VX, with subspaces, on the same edge features: the fp64 sum
    init + Σ w_t leaf_t in model order, rounded once to fp32, bit for bit."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    d, T = 6, 9
    cand = edge_candidates(rng, d)
    X = edge_matrix(rng, n, d, cand)
    VX = edge_matrix(rng, n, d, cand)
    trees, subs = [], []
    for t in range(T):
        sub = np.sort(rng.choice(d, size=3, replace=False)).astype(np.int32) if t % 2 else None
        cc = cand if sub is None else [cand[c] for c in sub]
        trees.append(_random_unbalanced_tree(rng, int(rng.integers(1, 40)), d if sub is None else sub.size, cc))
        subs.append(sub)
    w = rng.random(T) + 0.1
    init = 0.37
    ctx = Context(0)
    try:
        for slot, out, M, validation in ((N.SLOT_X, N.SLOT_H, X, False), (N.SLOT_VX, N.SLOT_VH, VX, True)):
            ctx.alloc(slot, d, n)
            ctx.upload_rowmajor(slot, M)
            ctx.alloc(out, 1, n)
            ctx.forest_predict(trees, out, weights=w, init=init, validation=validation, subspaces=subs)
            assert ctx.get_option("last_forest_chunks") == 1
            want = np.full(n, init)
            for tr, sub, wt in zip(trees, subs, w):
                want = want + wt * tr["value"][_walk(tr, M if sub is None else M[:, sub])].astype(np.float64)
            np.testing.assert_array_equal(ctx.download(out), want.astype(np.float32), err_msg=f"validation={validation}")
    finally:
        ctx.close()


@pytest.mark.parametrize("n_thr", [255, 256])
def test_rank_matrix_threshold_capacity(rng, n_thr):
    """A column with 255 distinct thresholds still fits the uint8 ranks (rank 255 is left to NaN and values above every
    threshold); with 256 the tree falls back to the fp32 walk and the forest kernel refuses.  Either way: exact."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    n = 3001
    thr = np.sort(np.unique(rng.standard_normal(n_thr + 50).astype(np.float32)))[:n_thr]
    assert thr.size == n_thr

    def bst(lo, hi, nodes):                  # balanced tree over the sorted thresholds thr[lo:hi]: every one is used
        i = len(nodes["feature"])
        for k in nodes:
            nodes[k].append(0)
        if lo == hi:
            nodes["feature"][i], nodes["value"][i] = -1, float(lo)
            return i
        mid = (lo + hi) // 2
        nodes["feature"][i], nodes["threshold"][i] = 0, thr[mid]
        nodes["left"][i] = bst(lo, mid, nodes)
        nodes["right"][i] = bst(mid + 1, hi, nodes)
        return i

    nodes = {"feature": [], "threshold": [], "left": [], "right": [], "value": []}
    bst(0, n_thr, nodes)
    tree = {"feature": np.array(nodes["feature"], np.int32), "threshold": np.array(nodes["threshold"], np.float32),
            "left": np.array(nodes["left"], np.int32), "right": np.array(nodes["right"], np.int32),
            "value": np.array(nodes["value"], np.float32)}
    assert np.unique(tree["threshold"][tree["feature"] >= 0]).size == n_thr
    X = rng.standard_normal((n, 1)).astype(np.float32)
    X[: n // 3, 0] = thr[rng.integers(0, n_thr, n // 3)]                 # rows ON thresholds
    X[n // 3: n // 3 + len(SPECIAL_X), 0] = np.array(SPECIAL_X, np.float32)
    want = tree["value"][_walk(tree, X)]
    ctx = Context(0)
    try:
        ctx.alloc(N.SLOT_X, 1, n)
        ctx.upload_rowmajor(N.SLOT_X, X)
        ctx.alloc(N.SLOT_H, 1, n)
        ctx.tree_predict(tree, N.SLOT_H, 0)
        assert ctx.get_option("last_tree_binned") == (1 if n_thr <= 255 else 0)
        np.testing.assert_array_equal(ctx.download(N.SLOT_H), want)
        if n_thr <= 255:
            ctx.forest_predict([tree], N.SLOT_H, weights=[1.0], init=0.0)
            np.testing.assert_array_equal(ctx.download(N.SLOT_H), want)
        else:
            with pytest.raises(N.NativeError):
                ctx.forest_predict([tree], N.SLOT_H, weights=[1.0], init=0.0)
    finally:
        ctx.close()
