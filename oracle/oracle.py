"""ctypes binding of the CPU oracle (oracle/se_oracle.c).

TEST INFRASTRUCTURE ONLY — may be imported from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs, never from the product package.  PARITY UNPINNED (no JVM in
this image; the reference's tests hold no golden numbers) — see se_oracle.h.

All arrays are float64, C-contiguous, layout [dim][n] / [M][n] / [M][K][n].
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))

SQUARED, ABSOLUTE, HUBER, QUANTILE, LOGCOSH, SCALED_LOGCOSH, BERNOULLI, EXPONENTIAL, LOGLOSS = range(9)
LOSS_IDS = {
    "squared": SQUARED, "absolute": ABSOLUTE, "huber": HUBER, "quantile": QUANTILE,
    "logcosh": LOGCOSH, "scaledlogcosh": SCALED_LOGCOSH, "bernoulli": BERNOULLI,
    "exponential": EXPONENTIAL, "logloss": LOGLOSS,
}

_dp = C.POINTER(C.c_double)
_FN1 = C.CFUNCTYPE(C.c_double, C.c_double, C.c_void_p)


def build(force: bool = False) -> None:
    """Compile liboracle.so / liboracle_omp.so with the committed Makefile."""
    libs = [os.path.join(_HERE, f) for f in ("liboracle.so", "liboracle_omp.so")]
    srcs = [os.path.join(_HERE, f) for f in ("se_oracle.c", "se_oracle.h", "Makefile")]
    need = force or not all(os.path.exists(l) for l in libs) or \
        max(os.path.getmtime(s) for s in srcs if os.path.exists(s)) > min(os.path.getmtime(l) for l in libs)
    if need:
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))


def _p(a):
    if a is None:
        return None
    assert a.dtype == np.float64 and a.flags["C_CONTIGUOUS"], (a.dtype, a.flags)
    return a.ctypes.data_as(_dp)


def _f64(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64)


class Oracle:
    def __init__(self, omp: bool = False):
        build()
        self.lib = C.CDLL(os.path.join(_HERE, "liboracle_omp.so" if omp else "liboracle.so"))
        L = self.lib
        i64, i32, d = C.c_int64, C.c_int, C.c_double
        L.orc_encode_label.restype = d; L.orc_encode_label.argtypes = [i32, d]
        for nm in ("orc_loss", "orc_gradient", "orc_hessian"):
            getattr(L, nm).restype = d
            getattr(L, nm).argtypes = [i32, d, d, d]
        L.orc_has_hessian.restype = i32; L.orc_has_hessian.argtypes = [i32]
        L.orc_linesearch_eval.restype = None
        L.orc_linesearch_eval.argtypes = [i32, d, i32, i64, _dp, _dp, _dp, _dp, _dp, _dp, _dp]
        L.orc_pseudo_residuals.restype = None
        L.orc_pseudo_residuals.argtypes = [i32, d, i32, i64, _dp, _dp, _dp, i32, _dp, _dp, _dp]
        L.orc_update.restype = None; L.orc_update.argtypes = [i32, i64, _dp, _dp, _dp]
        L.orc_mean_loss.restype = d; L.orc_mean_loss.argtypes = [i32, d, i32, i64, _dp, _dp]
        L.orc_brent_minimize.restype = d
        L.orc_brent_minimize.argtypes = [_FN1, C.c_void_p, d, d, d, d, d, i32,
                                         C.POINTER(i32), C.POINTER(i32)]
        L.orc_sum.restype = d; L.orc_sum.argtypes = [i64, _dp]
        L.orc_samme_r_update.restype = None
        L.orc_samme_r_update.argtypes = [i32, i64, _dp, _dp, d, _dp, _dp, _dp, _dp]
        L.orc_samme_error.restype = d; L.orc_samme_error.argtypes = [i64, _dp, _dp, d, _dp]
        L.orc_samme_update.restype = None
        L.orc_samme_update.argtypes = [i64, _dp, _dp, d, _dp, d, _dp, _dp]
        L.orc_agg_weighted_sum.restype = None
        L.orc_agg_weighted_sum.argtypes = [i32, i64, _dp, _dp, d, _dp]
        L.orc_agg_mean.restype = None; L.orc_agg_mean.argtypes = [i32, i64, _dp, _dp]
        L.orc_agg_gbm_classifier_raw.restype = None
        L.orc_agg_gbm_classifier_raw.argtypes = [i32, i32, i32, i64, _dp, _dp, _dp, _dp]
        L.orc_gbm_raw2prob.restype = None; L.orc_gbm_raw2prob.argtypes = [i32, i32, i64, _dp, _dp]
        L.orc_agg_bagging_soft.restype = None
        L.orc_agg_bagging_soft.argtypes = [i32, i32, i64, _dp, _dp, _dp]
        L.orc_agg_bagging_hard.restype = None
        L.orc_agg_bagging_hard.argtypes = [i32, i32, i64, _dp, _dp, _dp]
        L.orc_agg_boosting_real.restype = None
        L.orc_agg_boosting_real.argtypes = [i32, i32, i64, _dp, _dp, _dp]
        L.orc_agg_boosting_discrete.restype = None
        L.orc_agg_boosting_discrete.argtypes = [i32, i32, i64, _dp, _dp, _dp, _dp]
        L.orc_argmax.restype = None; L.orc_argmax.argtypes = [i32, i64, _dp, _dp]
        L.orc_r2_max_error.restype = d; L.orc_r2_max_error.argtypes = [i64, _dp, _dp]
        L.orc_r2_estimator_error.restype = d
        L.orc_r2_estimator_error.argtypes = [i32, i64, _dp, _dp, _dp, d, d]
        L.orc_r2_update.restype = None
        L.orc_r2_update.argtypes = [i32, i64, _dp, _dp, _dp, d, d, d, _dp, _dp]
        L.orc_agg_weighted_median.restype = None; L.orc_agg_weighted_median.argtypes = [i32, i64, _dp, _dp, _dp]
        L.orc_agg_weighted_mean.restype = None; L.orc_agg_weighted_mean.argtypes = [i32, i64, _dp, _dp, _dp]
        _u8, _i32p = C.POINTER(C.c_uint8), C.POINTER(C.c_int32)
        L.orc_ranks.restype = None; L.orc_ranks.argtypes = [i64, C.POINTER(C.c_float), i32, C.POINTER(C.c_float), _u8]
        L.orc_tree_walk.restype = None; L.orc_tree_walk.argtypes = [i64, _u8, _i32p, _i32p, _i32p, _i32p, _i32p]
        L.orc_tree_hist.restype = None
        L.orc_tree_hist.argtypes = [i64, i32, _u8, i32, _dp, _dp, _dp, i32, _i32p, _i32p, _i32p, _i32p, _i32p, _dp, _dp]
        L.orc_num_threads.restype = i32
        L.orc_set_num_threads.argtypes = [i32]

    # ---- scalar helpers
    def num_threads(self) -> int:
        return int(self.lib.orc_num_threads())

    def loss(self, loss, param, label, pred):
        return self.lib.orc_loss(loss, param, label, pred)

    def gradient(self, loss, param, label, pred):
        return self.lib.orc_gradient(loss, param, label, pred)

    def hessian(self, loss, param, label, pred):
        return self.lib.orc_hessian(loss, param, label, pred)

    def encode_label(self, loss, label):
        return self.lib.orc_encode_label(loss, label)

    # ---- GBM
    def linesearch_eval(self, loss, param, y, w, F, h, alpha):
        """Returns (lossSum/weightSum, gradSum/weightSum) exactly as Spark's RDDLossFunction."""
        y, w, F, h = _f64(y), _f64(w), _f64(F), _f64(h)
        alpha = _f64(np.atleast_1d(alpha))
        dim = alpha.shape[0]
        n = y.shape[0]
        assert F.size == dim * n and h.size == dim * n
        out_l = C.c_double()
        g = np.zeros(dim)
        self.lib.orc_linesearch_eval(loss, param, dim, n, _p(y), _p(w), _p(F), _p(h), _p(alpha),
                                     C.cast(C.byref(out_l), _dp), _p(g))
        return out_l.value, g

    def pseudo_residuals(self, loss, param, dim, y, w, F, newton, out_r=None, want_weights=True):
        """Returns (r[dim][n], wout[dim][n] or None, sum_hess[dim]).  `out_r` reuses a caller buffer and
        want_weights=False skips the (gradient-mode) copy of the instance weights — both only matter for
        the timed CPU baseline, which must not be dominated by page-faulting fresh arrays."""
        y, w, F = _f64(y), _f64(w), _f64(F)
        n = y.shape[0]
        r = np.zeros((dim, n)) if out_r is None else out_r
        wout = np.zeros((dim, n)) if (want_weights or newton) else None
        sh = np.zeros(dim)
        self.lib.orc_pseudo_residuals(loss, param, dim, n, _p(y), _p(w), _p(F), int(newton),
                                      _p(r), _p(wout), _p(sh))
        return r, wout, sh

    def update(self, F, h, step):
        step = _f64(np.atleast_1d(step))
        dim = step.shape[0]
        assert F.dtype == np.float64 and F.flags["C_CONTIGUOUS"]
        h = _f64(h)
        n = F.size // dim
        self.lib.orc_update(dim, n, _p(F), _p(h), _p(step))
        return F

    def mean_loss(self, loss, param, dim, y, F):
        y, F = _f64(y), _f64(F)
        return self.lib.orc_mean_loss(loss, param, dim, y.shape[0], _p(y), _p(F))

    def brent(self, fn, lo=0.0, hi=100.0, start=1.0, rel=1e-6, abs_tol=1e-6, max_eval=100):
        cb = _FN1(lambda x, _u: float(fn(x)))
        ne, st = C.c_int(), C.c_int()
        x = self.lib.orc_brent_minimize(cb, None, lo, hi, start, rel, abs_tol, max_eval,
                                        C.byref(ne), C.byref(st))
        return x, ne.value, st.value

    # ---- Boosting
    def sum(self, w):
        w = _f64(w)
        return self.lib.orc_sum(w.shape[0], _p(w))

    def samme_r_update(self, K, y, w, sum_w, P):
        y, w, P = _f64(y), _f64(w), _f64(P)
        n = y.shape[0]
        out = np.zeros(n)
        e, s = C.c_double(), C.c_double()
        self.lib.orc_samme_r_update(K, n, _p(y), _p(w), sum_w, _p(P), _p(out),
                                    C.cast(C.byref(e), _dp), C.cast(C.byref(s), _dp))
        return out, e.value, s.value

    def samme_error(self, y, w, sum_w, pred):
        y, w, pred = _f64(y), _f64(w), _f64(pred)
        return self.lib.orc_samme_error(y.shape[0], _p(y), _p(w), sum_w, _p(pred))

    def samme_update(self, y, w, sum_w, pred, beta):
        y, w, pred = _f64(y), _f64(w), _f64(pred)
        n = y.shape[0]
        out = np.zeros(n)
        s = C.c_double()
        self.lib.orc_samme_update(n, _p(y), _p(w), sum_w, _p(pred), beta, _p(out),
                                  C.cast(C.byref(s), _dp))
        return out, s.value

    # ---- BoostingRegressor (AdaBoost.R2)
    R2_LOSS = {"exponential": 0, "linear": 1, "squared": 2}

    def r2_max_error(self, y, pred):
        y, pred = _f64(y), _f64(pred)
        return self.lib.orc_r2_max_error(y.shape[0], _p(y), _p(pred))

    def r2_estimator_error(self, loss_type, y, pred, w, sum_w, max_error):
        y, pred, w = _f64(y), _f64(pred), _f64(w)
        return self.lib.orc_r2_estimator_error(self.R2_LOSS[loss_type], y.shape[0], _p(y), _p(pred), _p(w),
                                               sum_w, max_error)

    def r2_update(self, loss_type, y, pred, w, sum_w, max_error, beta):
        y, pred, w = _f64(y), _f64(pred), _f64(w)
        out = np.zeros(y.shape[0])
        s = C.c_double()
        self.lib.orc_r2_update(self.R2_LOSS[loss_type], y.shape[0], _p(y), _p(pred), _p(w), sum_w, max_error,
                               beta, _p(out), C.cast(C.byref(s), _dp))
        return out, s.value

    def agg_weighted_median(self, P, a):
        P, a = _f64(P), _f64(a)
        M, n = P.shape
        out = np.zeros(n)
        self.lib.orc_agg_weighted_median(M, n, _p(P), _p(a), _p(out))
        return out

    def agg_weighted_mean(self, P, a):
        P, a = _f64(P), _f64(a)
        M, n = P.shape
        out = np.zeros(n)
        self.lib.orc_agg_weighted_mean(M, n, _p(P), _p(a), _p(out))
        return out

    # ---- aggregation
    def agg_weighted_sum(self, P, a, init):
        P, a = _f64(P), _f64(a)
        M, n = P.shape
        out = np.zeros(n)
        self.lib.orc_agg_weighted_sum(M, n, _p(P), _p(a), init, _p(out))
        return out

    def agg_mean(self, P):
        P = _f64(P)
        M, n = P.shape
        out = np.zeros(n)
        self.lib.orc_agg_mean(M, n, _p(P), _p(out))
        return out

    def agg_gbm_classifier_raw(self, P, a, init, num_classes):
        P, a, init = _f64(P), _f64(a), _f64(init)
        M, dim, n = P.shape
        C_out = 2 if (dim == 1 and num_classes == 2) else dim
        raw = np.zeros((C_out, n))
        self.lib.orc_agg_gbm_classifier_raw(M, dim, num_classes, n, _p(P), _p(a), _p(init), _p(raw))
        return raw

    def gbm_raw2prob(self, loss, raw):
        raw = _f64(raw)
        Cn, n = raw.shape
        prob = np.zeros((Cn, n))
        self.lib.orc_gbm_raw2prob(loss, Cn, n, _p(raw), _p(prob))
        return prob

    def agg_bagging_soft(self, P):
        P = _f64(P)
        M, K, n = P.shape
        raw, prob = np.zeros((K, n)), np.zeros((K, n))
        self.lib.orc_agg_bagging_soft(M, K, n, _p(P), _p(raw), _p(prob))
        return raw, prob

    def agg_bagging_hard(self, votes, K):
        votes = _f64(votes)
        M, n = votes.shape
        raw, prob = np.zeros((K, n)), np.zeros((K, n))
        self.lib.orc_agg_bagging_hard(M, K, n, _p(votes), _p(raw), _p(prob))
        return raw, prob

    def agg_boosting_real(self, P):
        P = _f64(P)
        M, K, n = P.shape
        raw, prob = np.zeros((K, n)), np.zeros((K, n))
        self.lib.orc_agg_boosting_real(M, K, n, _p(P), _p(raw), _p(prob))
        return raw, prob

    def agg_boosting_discrete(self, votes, a, K):
        votes, a = _f64(votes), _f64(a)
        M, n = votes.shape
        raw, prob = np.zeros((K, n)), np.zeros((K, n))
        self.lib.orc_agg_boosting_discrete(M, K, n, _p(votes), _p(a), _p(raw), _p(prob))
        return raw, prob

    def argmax(self, raw):
        raw = _f64(raw)
        Cn, n = raw.shape
        out = np.zeros(n)
        self.lib.orc_argmax(Cn, n, _p(raw), _p(out))
        return out

    # ---- audit of a fitted tree over row chunks (oracle/tree_audit.py)
    def ranks(self, x, cands) -> np.ndarray:
        """uint8 rank of every fp32 x among the sorted fp32 candidates (#{cand < x}; 255 for NaN)."""
        x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1)
        c = np.ascontiguousarray(cands, dtype=np.float32).reshape(-1)
        out = np.empty(x.size, np.uint8)
        self.lib.orc_ranks(x.size, x.ctypes.data_as(C.POINTER(C.c_float)), c.size,
                           c.ctypes.data_as(C.POINTER(C.c_float)), out.ctypes.data_as(C.POINTER(C.c_uint8)))
        return out

    def tree_walk(self, R, feature, bins, left, right) -> np.ndarray:
        """Leaf index of every row of R ([S][m] uint8 ranks) in a tree (bins: rank thresholds)."""
        R = np.ascontiguousarray(R, dtype=np.uint8)
        a = [np.ascontiguousarray(v, dtype=np.int32) for v in (feature, bins, left, right)]
        out = np.empty(R.shape[1], np.int32)
        self.lib.orc_tree_walk(R.shape[1], R.ctypes.data_as(C.POINTER(C.c_uint8)),
                               *[v.ctypes.data_as(C.POINTER(C.c_int32)) for v in a],
                               out.ctypes.data_as(C.POINTER(C.c_int32)))
        return out

    def tree_hist(self, R, K, lab, w, c, parent, col, bins, left, hist_of, totals, hist):
        """Adds one chunk of rows (R [S][m] uint8 ranks, fp64 labels, weights and counts, None: 1) to the statistics
        of a node list (se_oracle.h orc_tree_hist): totals [n_nodes][stats + 2] and hist [h][S][256][stats]."""
        R = np.ascontiguousarray(R, dtype=np.uint8)
        lab, w, c = _f64(lab), _f64(w), _f64(c)
        a = [np.ascontiguousarray(v, dtype=np.int32) for v in (parent, col, bins, left, hist_of)]
        assert totals.dtype == np.float64 and totals.flags["C_CONTIGUOUS"] and hist.flags["C_CONTIGUOUS"]
        self.lib.orc_tree_hist(R.shape[1], R.shape[0], R.ctypes.data_as(C.POINTER(C.c_uint8)), int(K), _p(lab),
                               _p(w), _p(c), a[0].size, *[v.ctypes.data_as(C.POINTER(C.c_int32)) for v in a],
                               _p(totals), _p(hist))
