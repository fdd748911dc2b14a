"""CPU tests that pin the oracle (no GPU): the portable properties the reference's own tests assert,
a cross-check against the independent numpy restatement, and closed forms.
Reference tests mirrored: test/boosting/GBMLossSuite.scala:84-125 (finite differences),
test/classification/BoostingClassifierSuite.scala:126-154 (zero-sum raw predictions)."""
import numpy as np
import pytest

from oracle import np_oracle as NP
from oracle import oracle as O

SCALAR = ["squared", "absolute", "huber", "quantile", "logcosh", "scaledlogcosh", "bernoulli",
          "exponential"]
PARAM = {"huber": 0.9, "quantile": 0.9, "scaledlogcosh": 0.9}


def _labels(name, rng, n):
    if name in ("bernoulli", "exponential"):
        return (rng.random(n) < 0.4).astype(np.float64)
    return rng.standard_normal(n)


@pytest.mark.parametrize("name", SCALAR)
def test_c_matches_numpy_pointwise(oracle, rng, name):
    n = 2000
    y = _labels(name, rng, n)
    p = rng.standard_normal(n) * 2
    par = PARAM.get(name, 0.0)
    ye = NP.encode(name, y)
    lid = O.LOSS_IDS[name]
    lc = np.array([oracle.loss(lid, par, a, b) for a, b in zip(ye, p)])
    gc = np.array([oracle.gradient(lid, par, a, b) for a, b in zip(ye, p)])
    np.testing.assert_allclose(lc, NP.loss(name, par, ye, p), rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(gc, NP.gradient(name, par, ye, p), rtol=1e-13, atol=1e-15)
    if name in ("squared", "logcosh", "scaledlogcosh", "bernoulli", "exponential"):
        hc = np.array([oracle.hessian(lid, par, a, b) for a, b in zip(ye, p)])
        np.testing.assert_allclose(hc, NP.hessian(name, par, ye, p), rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("name", ["squared", "absolute", "huber", "quantile", "logcosh",
                                  "scaledlogcosh"])
def test_finite_difference_property(oracle, rng, name):
    """GBMLossSuite.scala:107-123: 1000 N(0,1) labels, prediction=[0], direction=[pred], weight 1,
    Breeze GradientTester at x=1: relative error of d/dalpha vs forward difference < 1e-5."""
    n = 1000
    y = rng.standard_normal(n)
    h = rng.standard_normal(n)
    F = np.zeros(n)
    lid, par = O.LOSS_IDS[name], PARAM.get(name, 0.0)
    eps = 1e-5  # Breeze GradientTester default epsilon
    f0, g0 = oracle.linesearch_eval(lid, par, y, None, F, h, [1.0])
    f1, _ = oracle.linesearch_eval(lid, par, y, None, F, h, [1.0 + eps])
    fd = (f1 - f0) / eps
    rel = abs(fd - g0[0]) / max(abs(fd), abs(g0[0]), 1e-4)
    assert rel < 1e-4 if name in ("absolute", "quantile", "huber") else rel < 1e-5, rel


@pytest.mark.parametrize("name", ["squared", "logcosh", "scaledlogcosh", "bernoulli", "exponential"])
def test_hessian_is_derivative_of_gradient(oracle, rng, name):
    """GBMLossSuite's (gradient -> hessian) pairs: hessian == d(gradient)/d(prediction)."""
    lid, par = O.LOSS_IDS[name], PARAM.get(name, 0.0)
    for _ in range(200):
        y = float(oracle.encode_label(lid, _labels(name, rng, 1)[0]))
        p = float(rng.standard_normal())
        e = 1e-6
        fd = (oracle.gradient(lid, par, y, p + e) - oracle.gradient(lid, par, y, p - e)) / (2 * e)
        assert abs(fd - oracle.hessian(lid, par, y, p)) < 1e-6 * max(1.0, abs(fd))


@pytest.mark.parametrize("name", SCALAR + ["logloss"])
@pytest.mark.parametrize("weighted", [False, True])
def test_linesearch_eval_matches_numpy(oracle, rng, name, weighted):
    n, K = 777, 5
    dim = K if name == "logloss" else 1
    y = rng.integers(0, K, n).astype(np.float64) if name == "logloss" else _labels(name, rng, n)
    F = rng.standard_normal((dim, n))
    h = rng.standard_normal((dim, n))
    w = rng.random(n) + 0.5 if weighted else None
    alpha = rng.random(dim) * 2
    par = PARAM.get(name, 0.0)
    lc, gc = oracle.linesearch_eval(O.LOSS_IDS[name], par, y, w, F, h, alpha)
    ln, gn = NP.linesearch_eval(name, par, y, w, F, h, alpha)
    assert lc == pytest.approx(ln, rel=1e-12)
    np.testing.assert_allclose(gc, gn, rtol=1e-11, atol=1e-14)


def _fitted_logloss_rows(rng, K, n, margin):
    """Label class at +margin over N(0, 0.5) classes: the late-round regime of a boosted classifier."""
    y = rng.integers(0, K, n)
    F = rng.normal(0.0, 0.5, (K, n))
    F[y, np.arange(n)] += margin
    return y, F


@pytest.mark.parametrize("K", [2, 9, 100])
def test_logloss_stable_form_and_where_the_unshifted_oracle_departs(oracle, rng, K):
    """The stable fp64 LogLoss of np_oracle (max term kept out of the exp-sum) is the reference the GPU tests use on
    well-fitted rows.  Up to a margin of 20 the C oracle's unshifted form (the reference's arithmetic) agrees with it
    to 1e-6 on the mean loss and the line-search sums, and on every residual up to a margin of 16; from a margin of
    about 30 the unshifted form itself loses the loss and the label-class gradient to the rounding of log Σ exp(p_k).
    That is why the GPU tests stop at a margin of 20."""
    n = 4000
    for margin in (0, 4, 8, 12, 16, 20, 30, 40):
        y, F = _fitted_logloss_rows(rng, K, n, margin)
        yf = y.astype(np.float64)
        ls, gs, hs = NP.logloss_stable(y, F)
        lu, gu, hu = NP.logloss_parts(y, F)
        lc = oracle.mean_loss(O.LOGLOSS, 0.0, K, yf, F)
        rc, _, _ = oracle.pseudo_residuals(O.LOGLOSS, 0.0, K, yf, None, F, False)
        rel_loss = abs(lc - ls.mean()) / ls.mean()
        rel_res = float(np.max(np.abs(rc + gs) / np.abs(gs)))
        if margin <= 20:
            assert rel_loss <= 1e-6, (margin, rel_loss)
            h = np.abs(gs) * rng.uniform(0.5, 1.5, (K, n))       # a direction along the residual: no cancellation
            lsum, gsum = oracle.linesearch_eval(O.LOGLOSS, 0.0, yf, None, F, h, np.zeros(K))
            assert lsum == pytest.approx(K * ls.mean(), rel=1e-6)
            np.testing.assert_allclose(gsum, (h * gs).sum(axis=1) / n, rtol=1e-6)
            assert lu.mean() == pytest.approx(lc, rel=1e-12)      # the numpy restatement of the unshifted form
        if margin <= 16:
            assert rel_res <= 1e-6, (margin, rel_res)
            np.testing.assert_allclose(hu, hs, rtol=1e-6)
        if margin == 30:
            assert rel_res > 1e-4, rel_res                         # label-class gradient: 1 - softmax cancels in fp64
        if margin == 40:
            assert rel_loss > 0.5, rel_loss                        # log Σ exp(p_k) rounds to m: the loss is lost
        # the stable form itself: loss = log1p(S) + m - p_y > 0, gradients of a row sum to 0 to its own precision
        assert np.all(ls >= 0)
        assert np.all(np.abs(gs.sum(axis=0)) <= 1e-15 * np.abs(gs).sum(axis=0) * K)


def test_logloss_stable_ties_and_non_argmax_labels():
    """Tied maxima count in S beyond the first; a label that is not the argmax keeps its O(margin) loss."""
    P = np.array([[3.0, 0.0, 0.0], [3.0, 25.0, 0.0], [-1.0, 0.0, 25.0]])
    y = np.array([1, 0, 2])
    lo, g, hs = NP.logloss_stable(y, P)
    lu, gu, hu = NP.logloss_parts(y, P)
    np.testing.assert_allclose(lo[:2], lu[:2], rtol=1e-14)
    np.testing.assert_allclose(g[:, 0], gu[:, 0], rtol=1e-14)
    assert lo[0] == pytest.approx(np.log(2.0 + np.exp(-4.0)), rel=1e-15)
    assert lo[1] == pytest.approx(25.0 + np.log1p(2.0 * np.exp(-25.0)), rel=1e-15)
    assert lo[2] == pytest.approx(np.log1p(np.exp(-25.0) + np.exp(-25.0)), rel=1e-14)
    s = 2.0 * np.exp(-25.0)
    assert g[2, 2] == pytest.approx(-s / (1.0 + s), rel=1e-14)
    assert hs[2, 2] == pytest.approx(s / (1.0 + s) ** 2, rel=1e-14)


def test_logloss_loss_counted_dim_times(oracle, rng):
    """Reference quirk (GBMLoss.scala:60-64): lossSum accumulates loss `dim` times per row."""
    n, K = 100, 4
    y = rng.integers(0, K, n).astype(np.float64)
    F = rng.standard_normal((K, n))
    h = np.zeros((K, n))
    l, _ = oracle.linesearch_eval(O.LOGLOSS, 0.0, y, None, F, h, np.ones(K))
    assert l == pytest.approx(K * oracle.mean_loss(O.LOGLOSS, 0.0, K, y, F), rel=1e-12)


@pytest.mark.parametrize("name", ["squared", "logcosh", "bernoulli", "exponential", "logloss",
                                  "absolute", "quantile"])
@pytest.mark.parametrize("newton", [False, True])
def test_pseudo_residuals_match_numpy(oracle, rng, name, newton):
    if newton and name in ("absolute", "quantile"):
        pytest.skip("no hessian")
    n, K = 513, 3
    dim = K if name == "logloss" else 1
    y = rng.integers(0, K, n).astype(np.float64) if name == "logloss" else _labels(name, rng, n)
    F = rng.standard_normal((dim, n))
    w = rng.random(n) + 0.5
    par = PARAM.get(name, 0.0)
    r, wo, S = oracle.pseudo_residuals(O.LOSS_IDS[name], par, dim, y, w, F, newton)
    rn, won, Sn = NP.pseudo_residuals(name, par, dim, y, w, F, newton)
    np.testing.assert_allclose(r, rn, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(wo, won, rtol=1e-12, atol=1e-16)
    if newton:
        np.testing.assert_allclose(S, Sn, rtol=1e-12)
        assert np.all(wo > 0)  # weights are 1/2*h/S*w: positive


def test_brent_squared_matches_closed_form(oracle, rng):
    """For squared loss the line-search objective is a parabola; Brent (rel=abs=1e-6, [0,100], start 1)
    must land within its own tolerance of clip(sum(h(y-F))/sum(h^2))."""
    n = 4096
    y = rng.standard_normal(n)
    F = rng.standard_normal(n) * 0.3
    for scale in (0.05, 0.7, 1.0, 3.0):
        h = (y - F) * scale + 0.1 * rng.standard_normal(n)
        star = float(np.clip(np.sum(h * (y - F)) / np.sum(h * h), 0, 100))
        f = lambda a: oracle.linesearch_eval(O.SQUARED, 0.0, y, None, F, h, [a])[0]
        x, ne, st = oracle.brent(f)
        assert st == 0 and ne <= 100
        assert abs(x - star) <= 3 * (1e-6 * abs(star) + 1e-6)


def test_brent_vs_scipy_on_nonquadratic(oracle, rng):
    from scipy.optimize import minimize_scalar
    n = 2000
    y = (rng.random(n) < 0.5).astype(np.float64)
    F = rng.standard_normal(n) * 0.1
    h = (2 * y - 1) * 0.5 + 0.3 * rng.standard_normal(n)
    f = lambda a: oracle.linesearch_eval(O.BERNOULLI, 0.0, y, None, F, h, [a])[0]
    x, ne, st = oracle.brent(f)
    ref = minimize_scalar(f, bounds=(0, 100), method="bounded", options={"xatol": 1e-9})
    assert st == 0
    assert abs(x - ref.x) < 1e-4
    assert f(x) <= ref.fun + 1e-12


def test_brent_max_eval_status(oracle):
    x, ne, st = oracle.brent(lambda a: (a - 37.123) ** 2, max_eval=3)
    assert st == 1 and ne == 3


def test_samme_r_matches_numpy_and_invariants(oracle, rng):
    n, K = 1500, 26
    y = rng.integers(0, K, n).astype(np.float64)
    Z = rng.standard_normal((K, n))
    Z[y.astype(int), np.arange(n)] += 2.0
    P = NP.softmax_cols(Z)
    P[3, :10] = 0.0  # exercises max(p, EPSILON)
    w = rng.random(n) + 0.1
    sw = oracle.sum(w)
    assert sw == pytest.approx(w.sum(), rel=1e-13)
    out, e, s = oracle.samme_r_update(K, y, w, sw, P)
    outn, en, sn = NP.samme_r_update(K, y, w, sw, P)
    np.testing.assert_allclose(out, outn, rtol=1e-12)
    assert e == pytest.approx(en, rel=1e-12) and s == pytest.approx(sn, rel=1e-12)
    assert 0 <= e <= 1 and np.all(out > 0)


@pytest.mark.parametrize("K", [2, 5, 26, 201, 256])
def test_samme_r_pure_leaf_closed_form(oracle, rng, K):
    """One-hot base-model outputs (pure leaves): the C oracle's weights are wn e^{-(K-1)L/K} on rows whose vote is the
    label and wn e^{L/K} elsewhere, L = -log(EPSILON), to 1e-12."""
    n = 300
    y = rng.integers(0, K, n)
    vote = np.where(rng.random(n) < 0.6, y, (y + rng.integers(1, K, n)) % K)
    P = (np.arange(K)[:, None] == vote[None, :]).astype(np.float64)
    w = rng.random(n) + 0.1
    sw = w.sum()
    out, e, s = oracle.samme_r_update(K, y.astype(np.float64), w, sw, P)
    want = NP.samme_r_pure_leaf(K, w / sw, vote == y)
    np.testing.assert_allclose(out, want, rtol=1e-12, atol=0)
    assert e == pytest.approx(np.sum((w / sw)[vote != y]), rel=1e-12)
    assert s == pytest.approx(want.sum(), rel=1e-12)


@pytest.mark.parametrize("K,M", [(2, 1), (2, 16), (5, 17), (26, 64), (33, 8), (40, 512)])
def test_boosting_real_pure_leaf_closed_form(oracle, rng, K, M):
    """M one-hot models: the C oracle's SAMME.R raw and probabilities are the vote-count closed form to 1e-12, and
    classes with equal counts get equal probabilities (the rows alternate two classes, so half of them tie).
    The oracle's probabilities are exponentials of differences of fp64 sums of M K terms of size L: where that
    rounding bound, 4 M K L 2^-53, exceeds 1e-12 (M = 512), it is the tolerance."""
    n = 200
    votes = rng.integers(0, K, (M, n))
    alt = rng.random(n) < 0.5
    k1 = rng.integers(0, K, n)
    k2 = (k1 + rng.integers(1, K, n)) % K
    votes[:, alt] = np.where(np.arange(M)[:, None] % 2 == 0, k1[alt][None, :], k2[alt][None, :])
    P = (np.arange(K)[None, :, None] == votes[:, None, :]).astype(np.float64)
    counts = P.sum(axis=0)
    raw, prob = oracle.agg_boosting_real(P)
    rw, pw = NP.boosting_real_pure_leaf(counts)
    assert np.all(np.abs(raw - rw) <= 1e-12 * np.abs(rw).max(axis=0))
    ok = pw > 1e-300
    np.testing.assert_allclose(prob[ok], pw[ok], rtol=max(1e-12, 4.0 * M * K * NP.L_EPS * 2.0 ** -53))
    assert np.all(prob[~ok] <= 1e-300)
    if M % 2 == 0:
        np.testing.assert_array_equal(pw[k1[alt], np.flatnonzero(alt)], pw[k2[alt], np.flatnonzero(alt)])


def test_samme_discrete_matches_numpy(oracle, rng):
    n, K = 1000, 5
    y = rng.integers(0, K, n).astype(np.float64)
    pred = np.where(rng.random(n) < 0.7, y, rng.integers(0, K, n)).astype(np.float64)
    w = rng.random(n)
    sw = w.sum()
    e = oracle.samme_error(y, w, sw, pred)
    assert e == pytest.approx(NP.samme_error(y, w, sw, pred), rel=1e-12)
    beta = e / ((1 - e) * (K - 1))
    out, s = oracle.samme_update(y, w, sw, pred, beta)
    outn, sn = NP.samme_update(y, w, sw, pred, beta)
    np.testing.assert_allclose(out, outn, rtol=1e-13)
    # analytic: sum w' = (1 - e) + e / beta
    assert s == pytest.approx((1 - e) + e / beta, rel=1e-10)


def test_boosting_raw_predictions_sum_to_zero(oracle, rng):
    """BoostingClassifierSuite.scala:126-154: every rawPrediction sums to 0 +- 1e-6, both algorithms."""
    M, K, n = 7, 26, 400
    P = NP.softmax_cols(rng.standard_normal((M * K, n)).reshape(M, K, n).reshape(M * K, n)).reshape(M, K, n)
    P = P / P.sum(axis=1, keepdims=True)
    raw, prob = oracle.agg_boosting_real(P)
    assert np.max(np.abs(raw.sum(axis=0))) < 1e-6
    rawn, probn = NP.agg_boosting_real(P)
    np.testing.assert_allclose(raw, rawn, rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(prob, probn, rtol=1e-10, atol=1e-14)
    votes = rng.integers(0, K, (M, n)).astype(np.float64)
    a = rng.random(M) + 0.1
    raw, prob = oracle.agg_boosting_discrete(votes, a, K)
    assert np.max(np.abs(raw.sum(axis=0))) < 1e-6
    rawn, probn = NP.agg_boosting_discrete(votes, a, K)
    np.testing.assert_allclose(raw, rawn, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(prob, probn, rtol=1e-10, atol=1e-14)
    np.testing.assert_allclose(prob.sum(axis=0), 1.0, rtol=1e-12)


def test_aggregations(oracle, rng):
    M, K, n = 9, 4, 300
    P = rng.standard_normal((M, n))
    a = rng.random(M)
    np.testing.assert_allclose(oracle.agg_weighted_sum(P, a, 0.25), 0.25 + (a[:, None] * P).sum(0),
                               rtol=1e-12, atol=1e-13)
    np.testing.assert_allclose(oracle.agg_mean(P), P.mean(axis=0), rtol=1e-12, atol=1e-14)
    votes = rng.integers(0, K, (M, n)).astype(np.float64)
    raw, prob = oracle.agg_bagging_hard(votes, K)
    rawn, probn = NP.agg_bagging_hard(votes, K)
    np.testing.assert_array_equal(raw, rawn)
    np.testing.assert_allclose(prob, probn, rtol=1e-15)
    assert np.all(raw.sum(axis=0) == M)
    Pk = rng.random((M, K, n))
    raw, prob = oracle.agg_bagging_soft(Pk)
    np.testing.assert_allclose(raw, Pk.sum(axis=0), rtol=1e-13)
    np.testing.assert_allclose(prob, Pk.mean(axis=0), rtol=1e-13)
    # GBM classifier raw: binary dim 1 -> (-res, res)
    Pd = rng.standard_normal((M, 1, n))
    ad = rng.random((M, 1))
    raw = oracle.agg_gbm_classifier_raw(Pd, ad, np.array([0.3]), 2)
    res = 0.3 + (ad[:, :, None] * Pd).sum(axis=0)[0]
    np.testing.assert_allclose(raw[1], res, rtol=1e-12, atol=1e-13)
    np.testing.assert_allclose(raw[0], -res, rtol=1e-12, atol=1e-13)
    pb = oracle.gbm_raw2prob(O.BERNOULLI, raw)
    np.testing.assert_allclose(pb[1], 1 / (1 + np.exp(-res)), rtol=1e-12)  # p1 = sigma(F): quirk 6
    pe = oracle.gbm_raw2prob(O.EXPONENTIAL, raw)
    np.testing.assert_allclose(pe[1], 1 / (1 + np.exp(2 * res)), rtol=1e-12)  # decreasing in F: quirk 6
    Pm = rng.standard_normal((M, K, n))
    am = rng.random((M, K))
    init = rng.standard_normal(K)
    raw = oracle.agg_gbm_classifier_raw(Pm, am, init, K)
    np.testing.assert_allclose(raw, init[:, None] + (am[:, :, None] * Pm).sum(axis=0), rtol=1e-12,
                               atol=1e-13)
    pl = oracle.gbm_raw2prob(O.LOGLOSS, raw)
    np.testing.assert_allclose(pl, NP.softmax_cols(raw), rtol=1e-12)
    np.testing.assert_array_equal(oracle.argmax(raw), np.argmax(raw, axis=0).astype(np.float64))


def test_openmp_build_agrees(rng):
    o1, o2 = O.Oracle(omp=False), O.Oracle(omp=True)
    n = 20000
    y = rng.standard_normal(n); F = rng.standard_normal(n); h = rng.standard_normal(n)
    a, ga = o1.linesearch_eval(O.LOGCOSH, 0.0, y, None, F, h, [0.7])
    b, gb = o2.linesearch_eval(O.LOGCOSH, 0.0, y, None, F, h, [0.7])
    assert a == pytest.approx(b, rel=1e-12) and ga[0] == pytest.approx(gb[0], rel=1e-11)
    assert o2.num_threads() >= 1


def test_weighted_median_properties(oracle, rng):
    """test/ensemble/UtilsSuite.scala:29-67: weighted median == median under uniform weights; 0/1 weights
    select among the kept values; scaling the weights changes nothing."""
    M, n = 9, 200
    P = rng.standard_normal((M, n))
    np.testing.assert_array_equal(oracle.agg_weighted_median(P, np.ones(M)), np.sort(P, axis=0)[(M - 1) // 2])
    keep = np.array([1, 0, 1, 1, 0, 0, 1, 1, 0], dtype=float)
    med = oracle.agg_weighted_median(P, keep)
    sub = np.sort(P[keep > 0], axis=0)
    np.testing.assert_array_equal(med, sub[(int(keep.sum()) - 1) // 2])
    a = rng.random(M) + 0.1
    np.testing.assert_array_equal(oracle.agg_weighted_median(P, a), oracle.agg_weighted_median(P, 7.5 * a))
    np.testing.assert_allclose(oracle.agg_weighted_mean(P, a), (a[:, None] * P).sum(0) / a.sum(), rtol=1e-13)


def test_adaboost_r2_oracle(oracle, rng):
    n = 1000
    y = rng.standard_normal(n); pred = y + 0.3 * rng.standard_normal(n); w = rng.random(n) + 0.1
    sw = w.sum()
    mx = oracle.r2_max_error(y, pred)
    assert mx == np.max(np.abs(y - pred))
    for lt, f in (("linear", lambda e: e), ("squared", lambda e: e ** 2), ("exponential", lambda e: 1 - np.exp(-e))):
        e = oracle.r2_estimator_error(lt, y, pred, w, sw, mx)
        L = f(np.abs(y - pred) / mx)
        assert e == pytest.approx(np.sum(w / sw * L), rel=1e-12)
        beta = e / (1 - e)
        out, s = oracle.r2_update(lt, y, pred, w, sw, mx, beta)
        np.testing.assert_allclose(out, w / sw * beta ** (1 - L), rtol=1e-12)
        assert s == pytest.approx(out.sum(), rel=1e-12)
