"""GPU tests of the BoostingClassifier and AdaBoost.R2 weight updates and of the classifier aggregations on the outputs
Spark's tree classifiers actually produce: pure leaves (probability vectors of exact 0s and one 1), well-fitted rows
(late rounds: most probabilities clamp to EPSILON = 2^-52, each log is about -36), exact ties, and class counts on
both sides of every kernel switch.

Every output is compared with an fp64 reference computed from the SAME fp32 inputs the kernel sees (the C oracle, or
the pure-leaf closed forms of oracle/np_oracle.py, which the CPU suite pins against the oracle), element by element:
|got - want| <= 1e-5 |want| + FLT_MIN.  Vote counts and labels are exact."""
import numpy as np
import pytest
from scipy.special import expit

from oracle import np_oracle as NP
from oracle import oracle as O

pytestmark = pytest.mark.gpu

RTOL = 1e-5
FLT_MIN = float(np.finfo(np.float32).tiny)
EPS = 2.0 ** -52


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


def rel_close(got, want, what, rtol=RTOL, floor=FLT_MIN):
    """|got - want| <= rtol |want| + floor, element by element (floor may be an array)."""
    got, want = d64(got), d64(want)
    floor = np.broadcast_to(d64(floor), want.shape)
    bad = ~(np.abs(got - want) <= rtol * np.abs(want) + floor)
    if bad.any():
        i = np.flatnonzero(bad.ravel())[0]
        worst = np.max(np.abs(got - want)[bad] / np.maximum(np.abs(want)[bad], FLT_MIN))
        raise AssertionError(f"{what}: {bad.sum()} / {want.size} beyond {rtol:g} relative; worst {worst:.3e}; first at "
                             f"flat index {i}: got {got.ravel()[i]!r}, want {want.ravel()[i]!r}")


def onehot(K, cls):
    return (np.arange(K)[:, None] == np.asarray(cls)[None, :]).astype(np.float64)


def other_class(rng, K, y):
    return (y + rng.integers(1, K, y.size)) % K


# ------------------------------------------------------------------ A. SAMME.R weight update
SAMME_KS = [2, 3, 4, 5, 8, 26, 32, 33, 64, 100, 200, 201, 256]   # register kernel K <= 4 and K > 200, tiled between
REGIMES = ["onehot_correct", "onehot_wrong", "fitted0", "fitted5", "fitted10", "fitted20", "fitted30", "fitted40",
           "mixed", "uniform", "denormal", "exact_one"]


def samme_rows(rng, K, n, regime):
    """(y, P[K][n]) for one regime.  fitted<m>: label logit +m over N(0, 0.5) logits (from about +36 every non-label
    probability is below EPSILON); mixed: fitted10 with one row in eight led by another class."""
    y = rng.integers(0, K, n)
    if regime == "onehot_correct":
        return y, onehot(K, y)
    if regime == "onehot_wrong":
        return y, onehot(K, other_class(rng, K, y))
    if regime == "uniform":                                           # exact tie: argmax is class 0, the loss is 0
        return y, np.full((K, n), np.float32(1.0 / K), dtype=np.float64)
    if regime.startswith("fitted") or regime in ("mixed", "denormal", "exact_one"):
        margin = {"mixed": 10.0, "denormal": 5.0, "exact_one": 20.0}.get(regime) or float(regime[6:])
        top = y.copy()
        if regime == "mixed":
            sel = rng.random(n) < 0.125
            top[sel] = other_class(rng, K, y[sel])
        Z = rng.normal(0.0, 0.5, (K, n))
        Z[top, np.arange(n)] += margin
        P = d64(f32(NP.softmax_cols(Z)))
        if regime == "denormal":                                      # non-label entries at and below EPSILON
            pool = np.array([0.0, 1e-45, 1e-40, FLT_MIN / 2, FLT_MIN, 1e-30, 1e-20, EPS, EPS * (1 - 2 ** -23),
                             EPS * (1 + 2 ** -23)], np.float32)
            pick = (rng.random((K, n)) < 0.6) & (np.arange(K)[:, None] != y[None, :])
            P[pick] = pool[rng.integers(0, pool.size, int(pick.sum()))]
        if regime == "exact_one":                                     # p == 1 on the label, or on another class
            a = rng.random(n)
            right, wrong = a < 0.5, a > 0.75
            P[:, right] = d64(f32(P[:, right] * 1e-3))
            P[y[right], np.flatnonzero(right)] = 1.0
            o = other_class(rng, K, y[wrong])
            P[:, wrong] = d64(f32(P[:, wrong] * 1e-3))
            P[o, np.flatnonzero(wrong)] = 1.0
        return y, P
    raise ValueError(regime)


def run_samme_r(ctx, oracle, rng, K, n, regime):
    from spark_ensemble_b200 import _native as N
    y, P = samme_rows(rng, K, n, regime)
    P = d64(f32(P))
    w = f32(rng.random(n) + 0.1)
    w[1::7] = 0.0                                                     # zero weights stay zero
    ctx.boost_configure(n, K, True)
    ctx.upload(N.SLOT_Y, f32(y)); ctx.upload(N.SLOT_BW, w); ctx.upload(N.SLOT_PROBA, f32(P))
    sw = ctx.slot_sum(N.SLOT_BW)
    e, s = ctx.boost_real_update(sw)
    out, eo, so = oracle.samme_r_update(K, d64(y), d64(w), sw, P)
    if regime in ("onehot_correct", "onehot_wrong"):                  # the closed form, independent of the oracle
        rel_close(out, NP.samme_r_pure_leaf(K, d64(w) / sw, regime == "onehot_correct"), "oracle vs closed form",
                  rtol=1e-12)
    if regime == "uniform":
        rel_close(out, d64(w) / sw, "oracle at the tie", rtol=1e-12)
        assert eo == pytest.approx(np.sum((d64(w) / sw)[y != 0]), rel=1e-12)
    rel_close(ctx.download(N.SLOT_BW), out, f"weights (K={K}, n={n}, {regime})")
    assert abs(e - eo) <= RTOL * eo + (1e-12 if eo == 0 else 0.0), (e, eo)
    rel_close(s, so, "new sum")


@pytest.mark.parametrize("n", [257, 40961])
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("K", SAMME_KS)
def test_samme_r_update_regimes(ctx, oracle, rng, K, regime, n):
    run_samme_r(ctx, oracle, rng, K, n, regime)


@pytest.mark.parametrize("n", [1, 3, 255, 256])
@pytest.mark.parametrize("regime", ["onehot_wrong", "mixed"])
@pytest.mark.parametrize("K", [2, 4, 5, 200, 201, 256])
def test_samme_r_update_row_tails(ctx, oracle, rng, K, regime, n):
    """Row counts below one 4-row group and one 256-row tile, on both sides of the register / tiled switches."""
    run_samme_r(ctx, oracle, rng, K, n, regime)


# ------------------------------------------------------------------ B. SAMME.R aggregation
AGG_KS = [2, 5, 26, 32, 33, 40]          # tile kernel up to 32 classes, streaming sum + finalize above


def tie_votes(rng, K, M, n):
    """votes[M][n]: a third of the rows alternate two classes (an exact count tie when M is even), a third alternate
    two classes and give the last vote to a third one (counts differing by 1), the rest vote at random."""
    votes = rng.integers(0, K, (M, n))
    kind = rng.integers(0, 3, n)
    k1 = rng.integers(0, K, n)
    k2 = other_class(rng, K, k1) if K > 1 else k1
    k3 = np.where(K > 2, (k1 + 2) % K, k1)
    k3 = np.where((k3 == k2) & (K > 2), (k3 + 1) % K, k3)
    alt = np.where(np.arange(M)[:, None] % 2 == 0, k1[None, :], k2[None, :])
    for t in (0, 1):
        sel = kind == t
        votes[:, sel] = alt[:, sel]
        if t == 1 and M % 2 == 0:
            votes[M - 1, sel] = k3[sel]
    return votes


def check_labels(label, counts, what):
    """Exact count ties: the label is one of the tied classes; otherwise the argmax."""
    label = np.asarray(label).astype(np.int64)
    top = counts.max(axis=0)
    ok = counts[label, np.arange(label.size)] == top
    if not ok.all():
        i = np.flatnonzero(~ok)[0]
        raise AssertionError(f"{what}: {np.sum(~ok)} labels not a maximum; row {i}: label {label[i]}, counts "
                             f"{counts[:, i].tolist()}")


@pytest.mark.parametrize("M", [1, 8, 16, 17, 64, 512])
@pytest.mark.parametrize("K", AGG_KS)
def test_boosting_real_pure_leaves(ctx, rng, K, M):
    """One-hot base models: raw_k = (K-1) L (c_k - M/K), prob = softmax(L c) from the vote counts c."""
    from spark_ensemble_b200 import _native as N
    n = 257
    votes = tie_votes(rng, K, M, n)
    P = np.stack([onehot(K, v) for v in votes])
    counts = P.sum(axis=0)
    raw, prob = NP.boosting_real_pure_leaf(counts)
    ctx.agg_configure(N.AGG_BOOSTING_REAL, M, K, 1, 0, n)
    ctx.upload(N.SLOT_P, f32(P))
    ctx.agg_run()
    g = ctx.download(N.SLOT_RAW).reshape(K, n)
    rel_close(g, raw, "raw", rtol=0.0, floor=RTOL * np.abs(raw).max(axis=0))
    rs = np.abs(d64(g).sum(axis=0))
    assert np.all(rs <= RTOL * np.abs(d64(g)).sum(axis=0) + FLT_MIN), rs.max()
    rel_close(ctx.download(N.SLOT_PROB).reshape(K, n), prob, "prob")
    check_labels(ctx.download(N.SLOT_LABEL), counts, "label")


@pytest.mark.parametrize("M", [1, 8, 17, 64])
@pytest.mark.parametrize("K", AGG_KS)
def test_boosting_real_impure_leaves(ctx, oracle, rng, K, M):
    """Leaf frequencies p = j / leafsize, each model's output on a row one-hot (pure leaf) with probability 1/2.
    prob at 1e-5 relative where it is at least 1e-6 of its row's largest, at 1e-11 of that largest below; raw at 1e-5
    of the largest |raw| (a near tie of two classes has a raw far below the rounding of the logs it is made of)."""
    from spark_ensemble_b200 import _native as N
    n = 257
    P = np.empty((M, K, n))
    for m in range(M):
        size = rng.integers(2, 60, n)
        cnt = np.stack([rng.multinomial(s, rng.dirichlet(np.full(K, 0.3))) for s in size], axis=1)
        P[m] = cnt / size
        pure = rng.random(n) < 0.5
        P[m][:, pure] = onehot(K, rng.integers(0, K, int(pure.sum())))
    P = d64(f32(P))
    raw, prob = oracle.agg_boosting_real(P)
    ctx.agg_configure(N.AGG_BOOSTING_REAL, M, K, 1, 0, n)
    ctx.upload(N.SLOT_P, f32(P))
    ctx.agg_run()
    rel_close(ctx.download(N.SLOT_RAW).reshape(K, n), raw, "raw", rtol=0.0, floor=RTOL * np.abs(raw).max())
    pmax = prob.max(axis=0)
    big = prob >= 1e-6 * pmax
    got = d64(ctx.download(N.SLOT_PROB).reshape(K, n))
    rel_close(got[big], prob[big], "prob (>= 1e-6 of the row maximum)")
    small = ~big
    lim = (1e-11 * np.broadcast_to(pmax, prob.shape))[small]
    assert np.all(np.abs(got[small] - prob[small]) <= lim), np.max(np.abs(got[small] - prob[small]) / lim)
    lab = ctx.download(N.SLOT_LABEL)
    srt = np.sort(raw, axis=0)
    clear = (srt[-1] - srt[-2]) > 1e-6 * np.abs(raw).max(axis=0)
    np.testing.assert_array_equal(lab[clear], oracle.argmax(raw)[clear])


# ------------------------------------------------------------------ C. vote aggregations
@pytest.mark.parametrize("M", [1, 8, 255, 256, 300])
@pytest.mark.parametrize("K", [2, 26, 98, 99, 160, 161, 200, 1000])
def test_vote_aggregations(ctx, rng, K, M):
    """Bagging hard votes and SAMME discrete votes with equal model weights, past the packed kernel's M <= 255 and
    K <= 160 and past the shared-memory histograms: exact counts, first-maximum labels."""
    from spark_ensemble_b200 import _native as N
    n = 1029
    votes = tie_votes(rng, K, M, n)
    counts = np.zeros((K, n))
    np.add.at(counts, (votes, np.broadcast_to(np.arange(n), votes.shape)), 1.0)
    first = np.argmax(counts, axis=0)                                   # numpy: the first maximum

    ctx.agg_configure(N.AGG_BAGGING_HARD, M, K, 1, 0, n)
    ctx.upload(N.SLOT_P, f32(votes))
    ctx.agg_run()
    np.testing.assert_array_equal(ctx.download(N.SLOT_RAW).reshape(K, n), counts)
    rel_close(ctx.download(N.SLOT_PROB).reshape(K, n), counts / M, "hard-vote prob")
    np.testing.assert_array_equal(ctx.download(N.SLOT_LABEL), first)

    a = 0.375                                                           # equal weights: ties exact in fp64 too
    raw = a * (K * counts - M) / (K - 1)
    ctx.agg_configure(N.AGG_BOOSTING_DISCRETE, M, K, 1, 0, n)
    ctx.upload(N.SLOT_P, f32(votes))
    ctx.agg_run(np.full(M, a))
    rel_close(ctx.download(N.SLOT_RAW).reshape(K, n), raw, "discrete raw")
    rel_close(ctx.download(N.SLOT_PROB).reshape(K, n), NP.softmax_cols(raw / (K - 1)), "discrete prob")
    np.testing.assert_array_equal(ctx.download(N.SLOT_LABEL), first)


# ------------------------------------------------------------------ D. AdaBoost.R2 and SAMME updates
@pytest.mark.parametrize("beta", [1e-8, 0.3, 0.999])
@pytest.mark.parametrize("loss_type", ["exponential", "linear", "squared"])
def test_adaboost_r2_edges(ctx, oracle, rng, loss_type, beta):
    """maxError = 2 on exactly one row (linear and squared loss 1: the weight is only normalised), e / maxError at
    0.25 (1 +- 2^-23) and
    0.25 (the exponential loss's series / SFU switch), tiny errors, |y| about 1e6, zero weights; then the update with
    maxError == 0, which multiplies every weight by beta."""
    from spark_ensemble_b200 import _native as N
    n = 4099
    y = f32(rng.standard_normal(n))
    pred = f32(y + f32(rng.uniform(-1.5, 1.5, n)))
    big = slice(100, 1100)                                              # |y| about 1e6: differences of large values
    y[big] = f32(rng.uniform(0.5e6, 2e6, 1000) * rng.choice([-1, 1], 1000))
    pred[big] = f32(y[big] + f32(rng.uniform(-1.5, 1.5, 1000)))
    D = 2.0
    q = np.float32(0.25)
    special = [D, D * q * (1 - 2 ** -23), D * q, D * q * (1 + 2 ** -23), D * 1e-6, D * 3e-7, 0.0]
    for j, d in enumerate(special):                                     # y = 0: e = |pred| exactly
        y[j], pred[j] = 0.0, -np.float32(d)
    tiny = slice(1200, 1400)
    pred[tiny] = f32(y[tiny] + f32(rng.uniform(1e-7, 3e-6, 200) * D))
    assert np.max(np.abs(d64(y) - d64(pred))) == D and np.sum(np.abs(d64(y) - d64(pred)) == D) == 1
    w = f32(rng.random(n) + 0.1)
    w[::5] = 0.0
    w[0] = 0.7
    ctx.boostreg_configure(n)
    ctx.upload(N.SLOT_Y, y); ctx.upload(N.SLOT_PRED, pred); ctx.upload(N.SLOT_BW, w)
    sw = ctx.slot_sum(N.SLOT_BW)
    mx = ctx.boostreg_max_error()
    assert mx == D
    e = ctx.boostreg_error(sw, loss_type, mx)
    rel_close(e, oracle.r2_estimator_error(loss_type, y, pred, w, sw, mx), "estimator error")
    s = ctx.boostreg_update(sw, loss_type, mx, beta)
    out, so = oracle.r2_update(loss_type, y, pred, w, sw, mx, beta)
    got = ctx.download(N.SLOT_BW)
    rel_close(got, out, f"weights ({loss_type}, beta={beta})")
    if loss_type != "exponential":                                     # loss(1) = 1: the weight is only normalised
        rel_close(got[0], d64(w[0]) / sw, "loss-1 row: beta^0")
    rel_close(s, so, "new sum")

    ctx.upload(N.SLOT_PRED, y); ctx.upload(N.SLOT_BW, w)               # maxError == 0
    assert ctx.boostreg_max_error() == 0.0
    assert ctx.boostreg_error(sw, loss_type, 0.0) == 0.0
    s = ctx.boostreg_update(sw, loss_type, 0.0, beta)
    out, so = oracle.r2_update(loss_type, y, y, w, sw, 0.0, beta)
    rel_close(out, d64(w) / sw * beta, "oracle, maxError == 0", rtol=1e-12)
    rel_close(ctx.download(N.SLOT_BW), out, "weights, maxError == 0")
    rel_close(s, so, "new sum, maxError == 0")


@pytest.mark.parametrize("beta", [1e-8, 0.5])
def test_samme_discrete_small_beta(ctx, oracle, rng, beta):
    """SAMME update with beta about 1e-8: misclassified weights grow by 1/beta about 1e8."""
    from spark_ensemble_b200 import _native as N
    n, K = 40961, 7
    y = f32(rng.integers(0, K, n))
    pred = f32(np.where(rng.random(n) < 0.7, y, rng.integers(0, K, n)))
    w = f32(rng.random(n))
    w[::9] = 0.0
    ctx.boost_configure(n, K, False)
    ctx.upload(N.SLOT_Y, y); ctx.upload(N.SLOT_BW, w); ctx.upload(N.SLOT_PRED, pred)
    sw = ctx.slot_sum(N.SLOT_BW)
    rel_close(ctx.boost_discrete_error(sw), oracle.samme_error(y, w, sw, pred), "error")
    s = ctx.boost_discrete_update(sw, beta)
    out, so = oracle.samme_update(y, w, sw, pred, beta)
    rel_close(ctx.download(N.SLOT_BW), out, "weights")
    rel_close(s, so, "new sum")


# ------------------------------------------------------------------ E. GBM classifier aggregation at fitted margins
@pytest.mark.parametrize("M", [1, 9])
@pytest.mark.parametrize("loss,R", [("bernoulli", 40.0), ("exponential", 20.0)])
def test_gbm_binary_aggregation_large_margins(ctx, oracle, rng, loss, R, M):
    """dim 1: raw = (-F, F) with |F| up to R; the small probability keeps full relative precision.  The reference is
    the stable fp64 logistic of the oracle's raw (1 - p in fp64 would round the small one away)."""
    from spark_ensemble_b200 import _native as N
    n = 3001
    s = rng.uniform(-R, R, n)
    a = f32(rng.uniform(0.9, 1.1, (M, 1))).astype(np.float64)
    P = f32((s / M)[None, None, :] / a[:, :, None] + rng.normal(0.0, 0.01, (M, 1, n)))
    init = f32([0.03]).astype(np.float64)
    ctx.agg_configure(N.AGG_GBM_CLASSIFIER, M, 2, 1, loss, n)
    ctx.upload(N.SLOT_P, P)
    ctx.agg_run(a, init)
    raw = oracle.agg_gbm_classifier_raw(P, a, init, 2)
    rel_close(ctx.download(N.SLOT_RAW).reshape(2, n), raw, "raw", floor=RTOL)        # 1e-5 of max(|raw|, 1)
    x = -2.0 * raw[0] if loss == "exponential" else raw[0]             # p1 = 1 / (1 + e^x)
    rel_close(ctx.download(N.SLOT_PROB).reshape(2, n), np.stack([expit(x), expit(-x)]), "prob")
    lab = ctx.download(N.SLOT_LABEL)
    np.testing.assert_array_equal(lab[raw[1] != raw[0]], (raw[1] > raw[0])[raw[1] != raw[0]])


@pytest.mark.parametrize("M", [1, 9])
@pytest.mark.parametrize("K", [2, 3, 5, 26, 32, 33, 40])
def test_gbm_logloss_aggregation_fitted(ctx, oracle, rng, K, M):
    """dim = K: the label logit leads by 0-20; every probability at 1e-5 relative (no absolute floor but FLT_MIN)."""
    from spark_ensemble_b200 import _native as N
    n = 1029
    top = rng.integers(0, K, n)
    Z = rng.normal(0.0, 0.5, (K, n))
    Z[top, np.arange(n)] += rng.uniform(0.0, 20.0, n)
    a = f32(rng.uniform(0.9, 1.1, (M, K))).astype(np.float64)
    P = f32((Z / M)[None, :, :] / a[:, :, None] + rng.normal(0.0, 0.01, (M, K, n)))
    init = f32(rng.normal(0.0, 0.1, K)).astype(np.float64)
    ctx.agg_configure(N.AGG_GBM_CLASSIFIER, M, K, K, O.LOSS_IDS["logloss"], n)
    ctx.upload(N.SLOT_P, P)
    ctx.agg_run(a, init)
    raw = oracle.agg_gbm_classifier_raw(P, a, init, K)
    rel_close(ctx.download(N.SLOT_RAW).reshape(K, n), raw, "raw", rtol=0.0,
              floor=RTOL * np.maximum(1.0, np.abs(raw).max(axis=0)))
    rel_close(ctx.download(N.SLOT_PROB).reshape(K, n), oracle.gbm_raw2prob(O.LOSS_IDS["logloss"], raw), "prob")
    lab = ctx.download(N.SLOT_LABEL)
    srt = np.sort(raw, axis=0)
    clear = (srt[-1] - srt[-2]) > 1e-4
    np.testing.assert_array_equal(lab[clear], oracle.argmax(raw)[clear])
