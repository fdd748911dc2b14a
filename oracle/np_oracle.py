"""Independent numpy (fp64, vectorised) restatement of the same reference formulas as se_oracle.c.

TEST INFRASTRUCTURE ONLY.  Exists so the C oracle is cross-checked by a second, separately written
restatement (different language, vectorised instead of per-row).  PARITY UNPINNED like the C oracle.
Citations relative to core/src/main/scala/org/apache/spark/ml/ of the reference repository.
"""
from __future__ import annotations

import numpy as np

EPS = 2.0 ** -52  # Spark ml.impl.Utils.EPSILON


def encode(loss: str, y):
    return 2.0 * y - 1.0 if loss in ("bernoulli", "exponential") else y  # GBMLoss.scala:272,297


def _log1pexp(x):
    return np.where(x > 0, x + np.log1p(np.exp(-np.abs(x))), np.log1p(np.exp(np.minimum(x, 0))))


def loss(name, param, y, p):
    d = y - p
    if name == "squared":
        return d * d / 2.0
    if name == "absolute":
        return np.abs(d)
    if name == "huber":
        return np.where(np.abs(d) <= param, d * d / 2.0, param * (np.abs(d) - param / 2.0))
    if name == "quantile":
        return np.where(y > p, param * d, (param - 1.0) * d)
    if name == "logcosh":
        return np.log(np.cosh(d))
    if name == "scaledlogcosh":
        return np.where(y > p, param, 1.0 - param) * np.log(np.cosh(d))
    if name == "bernoulli":
        return _log1pexp(-2.0 * y * p)
    if name == "exponential":
        return np.exp(-y * p)
    raise ValueError(name)


def gradient(name, param, y, p):
    d = y - p
    if name == "squared":
        return -d
    if name == "absolute":
        return -np.sign(d)
    if name == "huber":
        return np.where(np.abs(d) <= param, -d, -param * np.sign(d))
    if name == "quantile":
        return np.where(y > p, -param, 1.0 - param)
    if name == "logcosh":
        return -np.tanh(d)
    if name == "scaledlogcosh":
        return np.where(y > p, param, 1.0 - param) * -np.tanh(d)
    if name == "bernoulli":
        return -2.0 * y / (1.0 + np.exp(2.0 * y * p))
    if name == "exponential":
        return -y * np.exp(-y * p)
    raise ValueError(name)


def hessian(name, param, y, p):
    d = y - p
    if name == "squared":
        return np.ones_like(d)
    if name == "logcosh":
        return 1.0 / np.cosh(d) ** 2
    if name == "scaledlogcosh":
        return np.where(y > p, param, 1.0 - param) / np.cosh(d) ** 2
    if name == "bernoulli":
        e = np.exp(2.0 * p * y)
        return 4.0 * e * y * y / (1.0 + e) ** 2
    if name == "exponential":
        return y * y * np.exp(-y * p)
    raise ValueError(name)


def logloss_parts(y_idx, P):
    """P [K][n]. Returns (loss[n], grad[K][n], hess[K][n]) per GBMLoss.scala:206-256 (no max-shift)."""
    K, n = P.shape
    lse = np.log(np.exp(P).sum(axis=0))
    onehot = (np.arange(K)[:, None] == y_idx[None, :]).astype(np.float64)
    lo = -(onehot * (P - lse)).sum(axis=0)
    s = np.exp(P - lse)
    return lo, s - onehot, s * (1.0 - s)


def logloss_stable(y_idx, P):
    """P [K][n]. The same (loss[n], grad[K][n], hess[K][n]) as logloss_parts, in a form that keeps full relative
    precision on well-fitted rows, where the label class leads the others by a wide margin and the loss, the gradient
    and 1 - softmax_argmax all shrink like exp(-margin):
        S = Σ_{k != argmax} exp(p_k - m),  loss = log1p(S) + m - p_y,  1 - softmax_argmax = S / (1 + S).
    The argmax is the first maximum; tied maxima beyond it count in S.  The unshifted form of the reference (and of
    logloss_parts / se_oracle.c) loses the loss to the rounding of log Σ exp(p_k) once exp(-margin) nears the fp64
    epsilon of the margin, i.e. from a margin of about 25-30."""
    K, n = P.shape
    cols = np.arange(n)
    am = np.argmax(P, axis=0)
    m = P[am, cols]
    E = np.exp(P - m)
    E[am, cols] = 0.0
    S = E.sum(axis=0)
    inv = 1.0 / (1.0 + S)
    sm = E * inv
    sm[am, cols] = inv
    om = S * inv  # 1 - softmax_argmax
    onehot = np.arange(K)[:, None] == y_idx[None, :]
    g = sm - onehot
    top_is_label = am == y_idx
    g[am[top_is_label], cols[top_is_label]] = -om[top_is_label]
    hs = sm * (1.0 - sm)
    hs[am, cols] = sm[am, cols] * om
    return np.log1p(S) + (m - P[y_idx, cols]), g, hs


def linesearch_eval(name, param, y, w, F, h, alpha):
    """(lossSum/weightSum, gradSum/weightSum) with the dim-times loss quirk (GBMLoss.scala:50-74)."""
    alpha = np.atleast_1d(np.asarray(alpha, dtype=np.float64))
    dim = alpha.shape[0]
    n = y.shape[0]
    F = F.reshape(dim, n)
    h = h.reshape(dim, n)
    wsum = float(n) if w is None else float(np.sum(w))
    p = F + alpha[:, None] * h
    if name == "logloss":
        lo, g, _ = logloss_parts(y.astype(np.int64), p)
        return dim * lo.sum() / wsum, (h * g).sum(axis=1) / wsum
    ye = encode(name, y)
    return loss(name, param, ye, p[0]).sum() / wsum, np.array(
        [(h[0] * gradient(name, param, ye, p[0])).sum() / wsum])


def pseudo_residuals(name, param, dim, y, w, F, newton):
    n = y.shape[0]
    F = F.reshape(dim, n)
    wv = np.ones(n) if w is None else w
    if name == "logloss":
        _, g, hs = logloss_parts(y.astype(np.int64), F)
    else:
        ye = encode(name, y)
        g = gradient(name, param, ye, F[0])[None, :]
        hs = hessian(name, param, ye, F[0])[None, :] if newton else None
    if not newton:
        return -g, np.broadcast_to(wv, (dim, n)).copy(), None
    hc = np.maximum(hs, 1e-2)
    S = hc.sum(axis=1)
    return -g / hc, 0.5 * hc / S[:, None] * wv[None, :], S


def samme_r_update(K, y, w, sum_w, P):
    wn = w / sum_w
    am = np.argmax(P, axis=0)
    err = float(np.sum(wn * (am != y)))
    code = np.where(np.arange(K)[:, None] == y[None, :], 1.0, -1.0 / (K - 1.0))
    lo = (code * np.log(np.maximum(P, EPS))).sum(axis=0)
    out = wn * np.exp(-((K - 1.0) / K) * lo)
    return out, err, float(out.sum())


def samme_error(y, w, sum_w, pred):
    return float(np.sum((w / sum_w) * (y != pred)))


def samme_update(y, w, sum_w, pred, beta):
    out = (w / sum_w) * np.power(1.0 / beta, (y != pred).astype(np.float64))
    return out, float(out.sum())


def softmax_cols(raw):
    m = raw.max(axis=0)
    e = np.exp(raw - m)
    return e / e.sum(axis=0)


def agg_boosting_real(P):
    M, K, n = P.shape
    lp = np.log(np.maximum(P, EPS))
    raw = ((K - 1) * (lp - lp.sum(axis=1, keepdims=True) / K)).sum(axis=0)
    return raw, softmax_cols(raw / (K - 1.0))


# Pure-leaf closed forms.  A pure tree leaf returns a probability vector of exact 0s and one 1, so every clamped log
# is 0 or -L with L = -log(EPSILON) = 52 ln 2, and the SAMME.R sums reduce to vote counts.
L_EPS = -np.log(EPS)


def samme_r_pure_leaf(K, wn, correct):
    """SAMME.R weight of a row whose base model put probability 1 on one class: wn e^{-(K-1)L/K} when that class is
    the label, wn e^{L/K} when it is not."""
    return wn * np.where(correct, np.exp(-(K - 1.0) * L_EPS / K), np.exp(L_EPS / K))


def boosting_real_pure_leaf(counts):
    """SAMME.R aggregation of M one-hot models from the vote counts c[K][n]: raw_k = (K-1) L (c_k - M/K) and
    prob = softmax(L c).  Independent of the order of summation: equal counts give equal values."""
    counts = np.asarray(counts, dtype=np.float64)
    K = counts.shape[0]
    M = counts.sum(axis=0)
    return (K - 1) * L_EPS * (counts - M / K), softmax_cols(L_EPS * counts)


def agg_boosting_discrete(votes, a, K):
    M, n = votes.shape
    onehot = (np.arange(K)[None, :, None] == votes[:, None, :].astype(np.int64))
    contrib = np.where(onehot, a[:, None, None], -a[:, None, None] / (K - 1))
    raw = contrib.sum(axis=0)
    return raw, softmax_cols(raw / (K - 1.0))


def agg_bagging_hard(votes, K):
    M, n = votes.shape
    raw = (np.arange(K)[None, :, None] == votes[:, None, :].astype(np.int64)).sum(axis=0).astype(np.float64)
    return raw, raw / M
