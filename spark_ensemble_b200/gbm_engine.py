"""Host-side driver of one GBM fit on one GPU shard: the glue between the estimator mirrors
(regression.GBMRegressor, classification.GBMClassifier) and the C ABI.

It mirrors the data flow of the reference's train() loop (regression/GBMRegressor.scala:340-469,
classification/GBMClassifier.scala:325-483) with the RDD closures replaced by native calls:
state (y, w, F, h, r) lives in HBM for the whole fit; per round only the base learner's inputs
(pseudo-residuals -> host) and outputs (directions -> device, or a tree evaluated on device) move.
"""
from __future__ import annotations

import numpy as np

from . import _native as N
from .context import Context


class GBMEngine:
    def __init__(self, ctx: Context, n: int, nv: int, dim: int, loss: str, param: float = 0.0,
                 has_weights: bool = False):
        self.ctx, self.n, self.nv, self.dim, self.loss = ctx, n, nv, dim, loss
        self.has_weights = has_weights
        ctx.gbm_configure(n, nv, dim, loss, param, has_weights)
        self._x_resident = False
        self._X_host = None
        self._fit_bins = None  # the device learner whose split candidates SLOT_X holds

    # ---- data in
    def load(self, y, w=None, F0=None, vy=None, vF0=None):
        c = self.ctx
        c.upload(N.SLOT_Y, y)
        if self.has_weights:
            c.upload(N.SLOT_W, w)
        self._load_pred(N.SLOT_F, F0, self.n)
        if self.nv > 0:
            c.upload(N.SLOT_VY, vy)
            self._load_pred(N.SLOT_VF, vF0, self.nv)

    def _load_pred(self, slot, F0, n):
        c = self.ctx
        F0 = np.asarray(F0, dtype=np.float64)
        if F0.ndim == 0 or F0.shape == (self.dim,):
            vals = np.broadcast_to(F0, (self.dim,))
            for j in range(self.dim):  # constant init model: broadcast on device
                c.fill(slot, float(vals[j]), n, j * n)
        else:
            c.upload(slot, np.ascontiguousarray(F0.reshape(self.dim, n), dtype=np.float32))

    def load_features(self, X, Xv=None):
        """Column-major feature matrix to HBM (enables on-device base-model evaluation)."""
        c = self.ctx
        X = np.asarray(X)
        c.alloc(N.SLOT_X, X.shape[1], X.shape[0])
        c.upload_rowmajor(N.SLOT_X, X)  # transposed on the device, chunked + double buffered
        self._X_host = X
        self._fit_bins = None
        if Xv is not None and self.nv > 0:
            Xv = np.asarray(Xv)
            c.alloc(N.SLOT_VX, Xv.shape[1], Xv.shape[0])
            c.upload_rowmajor(N.SLOT_VX, Xv)
        self._x_resident = True

    # ---- per-round pieces
    def residuals(self, newton: bool = False):
        return self.ctx.gbm_pseudo_residuals(newton)

    def fetch_residuals(self, newton: bool = False, out=None):
        r = self.ctx.download(N.SLOT_R, out=out).reshape(self.dim, self.n)
        wout = self.ctx.download(N.SLOT_WOUT).reshape(self.dim, self.n) if newton else None
        return r, wout

    def fit_direction(self, j: int, learner, subspace, newton: bool = False, bag: bool = False):
        """Fit the device tree learner on R row j (weights: WOUT row j in newton mode, else W when the fit has
        weights; the bag's multiplicities when `bag`) and write its output into H row j.  The split candidates are
        set once per fit, on the first call.  Nothing but the fitted tree crosses PCIe."""
        if not self._x_resident:
            raise ValueError("the device tree learner needs the features on the device (residentFeatures=True)")
        c = self.ctx
        if self._fit_bins is None:
            c.tree_fit_bins(learner.split_candidates(self._X_host))
            self._fit_bins = learner
        if newton:
            wslot, wrow = N.SLOT_WOUT, j
        elif self.has_weights:
            wslot, wrow = N.SLOT_W, 0
        else:
            wslot, wrow = -1, 0
        return learner.fit_resident(c, N.SLOT_R, j, wslot, wrow, bag, subspace, N.SLOT_H, j)

    def set_direction(self, h, validation: bool = False):
        self.ctx.upload(N.SLOT_VH if validation else N.SLOT_H,
                        np.ascontiguousarray(h, dtype=np.float32).reshape(-1))

    def set_direction_from_model(self, j: int, model, subspace, X_host=None, validation: bool = False):
        """Direction of dimension j: on device when X is resident and the model has an array form,
        otherwise model.predict on the host + upload (the reference's path)."""
        c = self.ctx
        slot = N.SLOT_VH if validation else N.SLOT_H
        if self._x_resident:
            t = model.tree_arrays()
            if t is not None:
                c.tree_predict(t, slot, j, validation=validation, subspace=subspace)
                return
            lin = model.linear_arrays()
            if lin is not None:
                c.linear_predict(lin["coef"], float(lin["intercept"]), slot, j, validation=validation,
                                 subspace=subspace)
                return
        n = self.nv if validation else self.n
        h = model.predict(X_host[:, subspace])
        c.upload(slot, np.ascontiguousarray(h, dtype=np.float32), offset=j * n)

    def line_search_brent(self, tol: float, max_iter: int):
        """GBMRegressor.scala:411-421: Brent on [0,100] from 1, rel=abs=tol, MaxEval(maxIter)."""
        alpha, loss, n_eval = self.ctx.gbm_linesearch_brent(0.0, 100.0, 1.0, tol, tol, max_iter)
        return alpha, loss, n_eval

    def line_search_newton(self, tol: float, max_iter: int):
        """Opt-in (Param lineSearch="newton"): safeguarded Newton on the same objective and interval, using the
        curvature Σ h²·H returned by the evaluation pass; ~5 passes instead of Brent's 20-40.  Same minimiser to
        the same tolerance, different iterates (not the reference's optimiser)."""
        alpha, loss, n_eval = self.ctx.gbm_linesearch_newton(0.0, 100.0, 1.0, tol, tol, max_iter)
        return alpha, loss, n_eval

    def line_search_lbfgsb(self, tol: float, max_iter: int):
        """GBMClassifier.scala:290-292,427: L-BFGS-B on [0,inf)^dim from 1, m=10.  Breeze's LBFGSB is
        third party; SciPy's L-BFGS-B (the original Byrd-Lu-Nocedal code) stands in on this host."""
        from scipy.optimize import fmin_l_bfgs_b
        evals = [0]

        def fun(a):
            evals[0] += 1
            l, g = self.ctx.gbm_linesearch_eval(a)
            return l, g

        x, f, info = fmin_l_bfgs_b(fun, np.ones(self.dim), bounds=[(0.0, None)] * self.dim, m=10,
                                   pgtol=tol, factr=max(tol / np.finfo(float).eps, 1.0),
                                   maxiter=max_iter)
        return x, f, evals[0]

    def update(self, step, residual: bool = True, newton: bool = False):
        return self.ctx.gbm_update(np.atleast_1d(step), residual=residual, newton=newton, loss=True)

    def update_validation(self, step) -> float:
        return self.ctx.gbm_update_validation(np.atleast_1d(step))

    # ---- the per-round body with HOST buffers (bench.py's e2e step, dim == 1)
    def boost_round(self, h_host: np.ndarray, learning_rate: float, tol: float, max_iter: int,
                    r_out: np.ndarray):
        """h (host) -> device; line search; F += lr·α·h fused with next residuals and loss; residuals
        (the next base learner's labels) -> host.  Returns (alpha, train_loss_sum)."""
        self.ctx.upload(N.SLOT_H, h_host)
        alpha, loss_sum, _ = self.ctx.gbm_round(learning_rate, True, tol, max_iter, residual=True)
        self.ctx.download(N.SLOT_R, out=r_out)
        return alpha, loss_sum
