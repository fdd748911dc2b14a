"""numpy fp64 restatement of se_logistic_stats and se_logistic_loss_grad.

X is [n, d] (fp32 values, as the device holds them), the columns `cols` any order with repeats, y the labels and w the
weights (None: 1).  With z_j = (x_{cols[j]} − shift_j)·scale_j, z_p = 1 and m = coef @ z:
  binomial (D = 1):  ℓ = log1pExp(m) − [y=1]·m, log1pExp(m) = max(m, 0) + log1p(exp(−|m|)), π = σ(m);
  multinomial:       ℓ = logsumexp(m) − m_y (the maximum subtracted), π = softmax(m);
and loss_grad returns (Σ c·ℓ, [D][p+1] of Σ c·(π_k − [y=k])·z_j).  abs_terms gives Σ|term| of both for tolerances.
"""
from __future__ import annotations

import numpy as np


def _z(X, cols, shift=None, scale=None) -> np.ndarray:
    cols = np.asarray(cols, dtype=np.int64).reshape(-1)
    Z = np.asarray(X, dtype=np.float64)[:, cols]
    if shift is not None:
        Z = Z - np.asarray(shift, dtype=np.float64)
    if scale is not None:
        Z = Z * np.asarray(scale, dtype=np.float64)
    return np.concatenate([Z, np.ones((Z.shape[0], 1))], axis=1)


def _weights(w, n) -> np.ndarray:
    return np.ones(n) if w is None else np.asarray(w, dtype=np.float64).reshape(-1)


def stats(X, y, cols, num_classes: int, w=None, shift=None) -> np.ndarray:
    """[Σc, Σc², Σc(x−s) per column, Σc(x−s)² per column, Σc[y=k] per class, invalid rows]."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    c = _weights(w, y.size)
    cols = np.asarray(cols, dtype=np.int64).reshape(-1)
    D = X[:, cols] - (0.0 if shift is None else np.asarray(shift, dtype=np.float64))
    K = int(num_classes)
    good_y = (y >= 0) & (y < K) & (y == np.floor(y))
    bad = ~good_y | ~np.isfinite(c) | (c < 0) | ~np.all(np.isfinite(X[:, cols]), axis=1)
    hist = [float(np.sum(np.where(good_y & (y == k), c, 0.0))) for k in range(K)]
    return np.concatenate([[c.sum(), (c * c).sum()], (c[:, None] * D).sum(axis=0), (c[:, None] * D * D).sum(axis=0),
                           hist, [float(bad.sum())]])


def _margins(X, cols, coef, shift, scale):
    Z = _z(X, cols, shift, scale)
    th = np.atleast_2d(np.asarray(coef, dtype=np.float64))
    return Z, Z @ th.T  # [n, p+1], [n, D]


def loss_grad(X, y, cols, coef, w=None, shift=None, scale=None):
    """(Σ c·ℓ, gradient [D][p+1]) in the kernel's contract."""
    Z, M = _margins(X, cols, coef, shift, scale)
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    c = _weights(w, y.size)
    if M.shape[1] == 1:
        m = M[:, 0]
        yy = (y == 1).astype(np.float64)
        e = np.exp(-np.abs(m))
        loss = np.maximum(m, 0.0) + np.log1p(e) - yy * m
        pi = np.where(m >= 0, 1.0 / (1.0 + e), e / (1.0 + e))
        R = (c * (pi - yy))[:, None]
    else:
        mx = M.max(axis=1, keepdims=True)
        E = np.exp(M - mx)
        S = E.sum(axis=1, keepdims=True)
        Y = (y[:, None] == np.arange(M.shape[1])[None, :]).astype(np.float64)
        loss = mx[:, 0] + np.log(S[:, 0]) - (M * Y).sum(axis=1)
        R = c[:, None] * (E / S - Y)
    return float((c * loss).sum()), R.T @ Z


def abs_terms(X, y, cols, coef, w=None, shift=None, scale=None):
    """(Σ|c|·(|terms of ℓ|), [D][p+1] of Σ|c|·(π_k + [y=k])·|z_j|): the scales the device sums are compared at."""
    Z, M = _margins(X, cols, coef, shift, scale)
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    c = np.abs(_weights(w, y.size))
    if M.shape[1] == 1:
        m = M[:, 0]
        yy = (y == 1).astype(np.float64)
        e = np.exp(-np.abs(m))
        lsc = np.abs(m) + np.log1p(e) + yy * np.abs(m)
        P = np.where(m >= 0, 1.0 / (1.0 + e), e / (1.0 + e))[:, None] + yy[:, None]
    else:
        mx = M.max(axis=1, keepdims=True)
        E = np.exp(M - mx)
        S = E.sum(axis=1, keepdims=True)
        Y = (y[:, None] == np.arange(M.shape[1])[None, :]).astype(np.float64)
        lsc = np.abs(mx[:, 0]) + np.abs(np.log(S[:, 0])) + np.abs(M * Y).sum(axis=1)
        P = E / S + Y
    return float((c * lsc).sum()), (c[:, None] * P).T @ np.abs(Z)


def evaluator(X, y, cols, w=None):
    """evaluate(shift, scale, coef) -> (Σ c·ℓ, gradient) over columns `cols` of host data: the CPU stand-in for
    Context.logistic_loss_grad that drives the same optimiser."""
    def evaluate(shift, scale, coef):
        return loss_grad(X, y, cols, coef, w, shift, scale)
    return evaluate
