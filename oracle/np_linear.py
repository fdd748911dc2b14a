"""numpy fp64 restatement of se_linear_moments: the weighted moment matrix of shifted columns.

For columns `cols` of X ([n, d]), labels y, weights w (None: 1) and bag multiplicities (None: 1):
z_i = (X[i, cols] − shift, 1, y_i − label_shift) and M = Σ_i c_i z_i z_iᵀ with c_i = w_i · bag_i, all in fp64.
`abs_moments` gives Σ_i |c_i z_i z_iᵀ| entry by entry, the scale the device result is compared at.
"""
from __future__ import annotations

import numpy as np


def _z(X, y, cols, shift, label_shift):
    X = np.asarray(X, dtype=np.float32).astype(np.float64)
    cols = np.asarray(cols, dtype=np.int64).reshape(-1)
    shift = np.zeros(cols.size) if shift is None else np.asarray(shift, dtype=np.float64)
    y = np.asarray(y, dtype=np.float32).astype(np.float64)
    return np.column_stack([X[:, cols] - shift, np.ones(X.shape[0]), y - float(label_shift)])


def _c(n, w, bag):
    c = np.ones(n)
    if w is not None:
        c = c * np.asarray(w, dtype=np.float32).astype(np.float64)
    if bag is not None:
        c = c * np.asarray(bag, dtype=np.float32).astype(np.float64)
    return c


def linear_moments(X, y, cols, w=None, bag=None, shift=None, label_shift: float = 0.0) -> np.ndarray:
    Z = _z(X, y, cols, shift, label_shift)
    return (Z * _c(Z.shape[0], w, bag)[:, None]).T @ Z


def abs_moments(X, y, cols, w=None, bag=None, shift=None, label_shift: float = 0.0) -> np.ndarray:
    Z = np.abs(_z(X, y, cols, shift, label_shift))
    return (Z * np.abs(_c(Z.shape[0], w, bag))[:, None]).T @ Z
