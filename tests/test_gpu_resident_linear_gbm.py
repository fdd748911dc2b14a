"""Every round of a GBM fit whose DeviceLinearRegression learner fits where the residuals live (residentFeatures=True,
GBMEngine.fit_direction) against fp64: the fp64 C oracle (oracle/se_oracle.c) on the device's own F for the residuals,
the learner's weights, the line-search objective and the update, and a numpy weighted ridge solve for the fit.

A spy around GBMEngine.fit_direction, the line searches, GBMEngine.update / update_validation and
Context.gbm_set_loss_param records each round: F, R, the learner's weights (WOUT as downloaded, i.e. ×1/S_j, in Newton
mode), the fitted models, H, α and the state after the update.  Then, per round:

(a) R equals the oracle's pseudo-residuals at 1e-5 of the row's scale, WOUT the oracle's normalised Newton weights at
    1e-6; huber's δ equals the exact α-quantile of |y − F|.
(b) each fitted model predicts, on its in-bag rows, what an fp64 least-squares solve of Σ c·(r − xβ − b)² +
    regParam·‖β‖² predicts, with r and c (weights × bag multiplicities) from the oracle; a fit that read unscaled Newton
    weights, ignored the bag or read another dimension's weights fails here.  H equals the model's fp64 prediction to
    the fp32 rounding of its coefficients.
(c) α: at 1e-5 of the closed form for the squared loss; otherwise the device objective is within 1e-6 of the oracle's
    around α, and the oracle's objective at the device's α is within a few times that evaluation error, plus the
    optimiser's tolerance, of where the same optimiser ends on the oracle's objective (Brent for the regressor, its
    minimum; L-BFGS-B for the classifier, with the estimator's settings and start).
(d) F and VF after the update equal F + lr·α·H to fp32, and trainLoss / validationLoss the oracle's mean loss at 1e-5.

A guarded fit per estimator checks that neither R nor WOUT leaves the device, bar the one label value fit_resident reads
to shift the labels.  Data: cpusmall standardised (one raw-scale case), adult8k and ragged letter slices of 3 and 5
classes."""
import math
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROUNDS = 3
TOL = 1e-6  # the estimators' default tol: Brent's and L-BFGS-B's tolerance


def _golden(name):
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", f"{name}.npz"))
    return z["X"].astype(np.float64), z["y"].astype(np.float64)


def _standardise(X):
    return (X - X.mean(axis=0)) / np.maximum(X.std(axis=0), 1e-12)


def _data(data):
    """(X, y) of a case: cpusmall (standardised or raw), adult8k standardised, or letter's rows of its first K classes,
    cut to an odd row count."""
    if data in ("cpusmall", "cpusmall-raw"):
        X, y = _golden("cpusmall")
        return (X if data == "cpusmall-raw" else _standardise(X)), y
    if data == "adult8k":
        X, y = _golden("adult8k")
        return _standardise(X), y
    K, n = {"letter3": (3, 1999), "letter5": (5, 3001)}[data]
    X, y = _golden("letter")
    keep = np.flatnonzero(y < K)[:n]
    return _standardise(X[keep]), y[keep]


def _estimator(kind, loss, updates, reg, weighted, bag, rounds=ROUNDS):
    from spark_ensemble_b200.classification import GBMClassifier
    from spark_ensemble_b200.learners import DeviceLinearRegression
    from spark_ensemble_b200.regression import GBMRegressor
    est = GBMRegressor() if kind == "reg" else GBMClassifier()
    est.set("baseLearner", DeviceLinearRegression(regParam=reg)).set("numBaseLearners", rounds).set("loss", loss)
    est.set("updates", updates).set("subspaceRatio", 0.7).set("residentFeatures", True)
    # every round runs: no early stop on the validation loss
    est.set("validationIndicatorCol", "val").set("numRounds", rounds + 1).set("validationTol", 0.0)
    est.set("learningRate", 0.7)
    if weighted:
        est.set("weightCol", "weight")
    if bag == "bag":
        est.set("subsampleRatio", 0.8)
    elif bag == "poisson":  # multiplicities above 1
        est.set("subsampleRatio", 0.8).set("replacement", True)
    return est


def _frame(X, y, weighted, seed):
    from spark_ensemble_b200.ensemble import DataFrame
    rng = np.random.default_rng(seed)
    cols = dict(features=X, label=y, val=rng.random(y.size) < 0.2)
    if weighted:
        cols["weight"] = rng.uniform(0.5, 2.0, y.size)
    return DataFrame(**cols)


class _Spy:
    """Records each round of fit_rounds on the device (downloads allowed: this is not the guarded run)."""

    def __init__(self, monkeypatch):
        from spark_ensemble_b200 import _native as N
        from spark_ensemble_b200.context import Context
        from spark_ensemble_b200.gbm_engine import GBMEngine
        self.rounds, self.params, self.static = [], [], None
        spy = self

        def f64(ctx, slot, dim):
            return ctx.download(slot).astype(np.float64).reshape(dim, -1)

        real_param = Context.gbm_set_loss_param

        def set_loss_param(ctx, param):
            spy.params.append(float(param))
            return real_param(ctx, param)

        real_fit = GBMEngine.fit_direction

        def fit_direction(eng, j, learner, sub, newton=False, bag=False):
            c, dim = eng.ctx, eng.dim
            if j == 0:
                if spy.static is None:
                    spy.static = dict(
                        X=np.asarray(eng._X_host, dtype=np.float32).astype(np.float64),
                        y=c.download(N.SLOT_Y).astype(np.float64),
                        w=c.download(N.SLOT_W).astype(np.float64) if eng.has_weights else None,
                        vy=c.download(N.SLOT_VY).astype(np.float64) if eng.nv else None)
                spy.rounds.append(dict(
                    F=f64(c, N.SLOT_F, dim), R=f64(c, N.SLOT_R, dim),
                    WOUT=f64(c, N.SLOT_WOUT, dim) if newton else None,
                    bag=c.download(N.SLOT_BAG).astype(np.float64) if bag else None,
                    param=spy.params[-1] if spy.params else None, newton=newton, sub=np.asarray(sub), models=[]))
            model = real_fit(eng, j, learner, sub, newton=newton, bag=bag)
            spy.rounds[-1]["models"].append(model)
            return model

        def line_search(real):
            def run(eng, tol, max_iter):
                rec = spy.rounds[-1]
                rec["H"] = f64(eng.ctx, N.SLOT_H, eng.dim)
                out = real(eng, tol, max_iter)
                alpha = np.atleast_1d(np.asarray(out[0], dtype=np.float64))
                # the device objective around α, for the oracle to bound its evaluation error
                pts = [alpha, alpha * (1 + 1e-3), alpha * (1 - 1e-3) + 1e-3, alpha * (1 + 1e-2),
                       alpha * (1 - 1e-2) + 1e-3, np.ones_like(alpha)]
                rec["evals"] = [(a, eng.ctx.gbm_linesearch_eval(a)[0]) for a in pts]
                return out
            return run

        real_update, real_vupdate = GBMEngine.update, GBMEngine.update_validation

        def update(eng, step, residual=True, newton=False):
            out = real_update(eng, step, residual=residual, newton=newton)
            rec = spy.rounds[-1]
            rec["step"] = np.atleast_1d(np.asarray(step, dtype=np.float64))
            rec["F_next"] = f64(eng.ctx, N.SLOT_F, eng.dim)
            return out

        def update_validation(eng, step):
            rec = spy.rounds[-1]
            rec["VF"] = f64(eng.ctx, N.SLOT_VF, eng.dim)
            rec["VH"] = f64(eng.ctx, N.SLOT_VH, eng.dim)
            out = real_vupdate(eng, step)
            rec["VF_next"] = f64(eng.ctx, N.SLOT_VF, eng.dim)
            return out

        monkeypatch.setattr(Context, "gbm_set_loss_param", set_loss_param)
        monkeypatch.setattr(GBMEngine, "fit_direction", fit_direction)
        monkeypatch.setattr(GBMEngine, "line_search_brent", line_search(GBMEngine.line_search_brent))
        monkeypatch.setattr(GBMEngine, "line_search_lbfgsb", line_search(GBMEngine.line_search_lbfgsb))
        monkeypatch.setattr(GBMEngine, "update", update)
        monkeypatch.setattr(GBMEngine, "update_validation", update_validation)


def _rep(a, counts):
    """Rows of a ([dim][n] or [n]) repeated by the bag's multiplicities: the line search sums each sampled copy."""
    if counts is None:
        return a
    c = counts.astype(np.int64)
    return np.repeat(a, c, axis=-1)


def _ridge_predict(Z, r, c, reg):
    """fp64 predictions on Z of argmin Σ c·(r − Zβ − b)² + max(reg, 1e-12)·‖β‖² (b unpenalised): lstsq on the
    √c-scaled system stacked over √reg·I — independent of the normal equations the device fit solves."""
    n, p = Z.shape
    lam = max(float(reg), 1e-12)
    s = np.sqrt(c)
    A = np.vstack([np.hstack([s[:, None] * Z, s[:, None]]),
                   np.hstack([math.sqrt(lam) * np.eye(p), np.zeros((p, 1))])])
    rhs = np.concatenate([s * r, np.zeros(p)])
    sol = np.linalg.lstsq(A, rhs, rcond=None)[0]
    Zc = Z - (c @ Z) / c.sum()
    G = Zc.T @ (c[:, None] * Zc) + lam * np.eye(p)
    d = np.sqrt(np.diag(G))
    cond = np.linalg.cond(G / np.outer(d, d)) if p else 1.0  # the scaled conditioning Cholesky's error follows
    return Z @ sol[:p] + sol[p], cond


def _check_rounds(O, spy, est, hist, loss, dim):
    """Checks (a) to (d) of every recorded round."""
    lid = O_LOSS[loss]
    st = spy.static
    X, y, w, vy = st["X"], st["y"], st["w"], st["vy"]
    n = y.size
    assert len(spy.rounds) == len(hist) == ROUNDS
    for i, (rec, h) in enumerate(zip(spy.rounds, hist)):
        F, newton, bag = rec["F"], rec["newton"], rec["bag"]
        msg = f"round {i}"
        # ---- (a) residuals and the learner's weights
        if loss == "huber":
            k = int(math.ceil(est("alpha") * n)) - 1
            delta = float(np.partition(np.abs(y - F[0]), k)[k])
            assert rec["param"] == pytest.approx(delta, rel=1e-6, abs=1e-30), (msg, rec["param"], delta)
            param = rec["param"]
        else:
            param = est("alpha") if loss == "quantile" else 0.0
        r, wout, S = O.pseudo_residuals(lid, param, dim, y, w, F.reshape(-1), newton)
        r, wout = r.reshape(dim, n), wout.reshape(dim, n)
        if newton and bag is not None:  # S_j sums the hessians of the bag's rows, each copy once (GBMRegressor.scala:373)
            S_bag = O.pseudo_residuals(lid, param, dim, _rep(y, bag), None, _rep(F, bag).reshape(-1), True)[2]
            wout *= (S / S_bag)[:, None]
        for j in range(dim):
            np.testing.assert_allclose(rec["R"][j], r[j], rtol=0, atol=1e-5 * np.abs(r[j]).max(),
                                       err_msg=f"{msg} R row {j}")
            if newton:
                np.testing.assert_allclose(rec["WOUT"][j], wout[j], rtol=1e-6, atol=1e-6 * wout[j].max(),
                                           err_msg=f"{msg} WOUT row {j}")
        if bag is not None:
            assert np.all(bag >= 0) and np.all(bag == np.round(bag)), msg
        # ---- (b) the fit, and H as its fp32-coefficient scoring
        sub = rec["sub"]
        rows = np.flatnonzero(bag > 0) if bag is not None else np.arange(n)
        Z = X[rows][:, sub]
        for j in range(dim):
            c = wout[j][rows] * (bag[rows] if bag is not None else 1.0)
            ref, cond = _ridge_predict(Z, r[j][rows], c, est("baseLearner").regParam)
            model = rec["models"][j]
            got = model.predict(Z)
            mag = np.abs(Z * model.coefficients).sum(axis=1) + abs(model.intercept)
            tol = 2e-6 * np.abs(r[j][rows]).max() + 1e-13 * cond * mag.max()
            err = np.abs(got - ref).max()
            assert err <= tol, (f"{msg} fit of dimension {j}: max |device − fp64| = {err:.3e} > {tol:.3e}",
                                float(np.abs(ref).max()), cond)
            Zall = X[:, sub]
            p64 = model.predict(Zall)
            htol = (len(sub) + 4) * 2.0 ** -24 * (np.abs(Zall * model.coefficients).sum(axis=1) + abs(model.intercept))
            assert np.all(np.abs(rec["H"][j] - p64) <= htol + 1e-30), (msg, j, np.abs(rec["H"][j] - p64).max())
        # ---- (c) the line search, on the oracle's objective over the device's F and H
        yb, wb = _rep(y, bag), (_rep(w, bag) if w is not None else None)
        Fb, Hb = _rep(F, bag), _rep(rec["H"], bag)

        def f_or(a):
            return O.linesearch_eval(lid, param, yb, wb, Fb.reshape(-1), Hb.reshape(-1), np.atleast_1d(a))[0]

        alpha = np.atleast_1d(np.asarray(h["alpha"], dtype=np.float64))
        if loss == "squared":
            res = (yb - Fb[0]) * Hb[0]
            a_star = min(max(float(res.sum() / (Hb[0] * Hb[0]).sum()), 0.0), 100.0)
            assert alpha[0] == pytest.approx(a_star, rel=1e-5, abs=1e-7), (msg, alpha[0], a_star)
        else:
            # E: the device objective's evaluation error, measured around α (and at the start point 1)
            E = max(abs(fd - f_or(a)) for a, fd in rec["evals"])
            if est.__class__.__name__ == "GBMRegressor":
                a_or = O.brent(f_or, 0.0, 100.0, 1.0, TOL, TOL, 100)[0]
                dx = 2 * (TOL * abs(a_or) + TOL)
                f_star = f_or(a_or)
                # Brent's x tolerance, and its parabolic steps over an objective that differs from the oracle's by up
                # to E near a flat (absolute, quantile: piecewise linear) minimum: measured up to 3E, allowed 8E
                slack = max(f_or(a_or + dx), f_or(max(a_or - dx, 0.0))) - f_star + 6 * E
            else:
                # L-BFGS-B (GBMClassifier.scala:427) stops when one step lowers the objective by less than tol
                # relative, which can be well short of the minimum: the reference point is the same optimiser, with
                # the same settings and start, on the oracle's objective
                from scipy.optimize import fmin_l_bfgs_b

                def fg(a):
                    return O.linesearch_eval(lid, param, yb, wb, Fb.reshape(-1), Hb.reshape(-1), a)
                a_or, f_star, _ = fmin_l_bfgs_b(fg, np.ones(dim), bounds=[(0.0, None)] * dim, m=10, pgtol=TOL,
                                                factr=TOL / np.finfo(float).eps, maxiter=100)
                slack = 10 * TOL * max(1.0, abs(f_star))
                assert f_or(alpha) <= f_or(np.ones(dim)) + 2 * E, (msg, "no descent from α = 1")
            f_dev = f_or(alpha)
            assert E <= 1e-6 * max(1.0, abs(f_star)), (msg, "device objective vs oracle", E)
            assert f_dev <= f_star + 2 * E + slack, (msg, alpha, a_or, f_dev, f_star, E, slack)
        # ---- (d) the update and the losses
        step = rec["step"]
        np.testing.assert_allclose(step, est("learningRate") * alpha, rtol=1e-15)
        Fn = O.update(F.reshape(-1).copy(), rec["H"].reshape(-1), step).reshape(dim, n)
        scale = np.abs(F) + np.abs(step[:, None] * rec["H"]) + (np.abs(y) if dim == 1 else 0.0)
        assert np.all(np.abs(rec["F_next"] - Fn) <= 2.0 ** -21 * scale), (msg, np.abs(rec["F_next"] - Fn).max())
        assert h["trainLoss"] == pytest.approx(O.mean_loss(lid, param, dim, y, rec["F_next"].reshape(-1)), rel=1e-5)
        VFn = O.update(rec["VF"].reshape(-1).copy(), rec["VH"].reshape(-1), step).reshape(dim, -1)
        vscale = np.abs(rec["VF"]) + np.abs(step[:, None] * rec["VH"])
        assert np.all(np.abs(rec["VF_next"] - VFn) <= 2.0 ** -21 * vscale), msg
        assert h["validationLoss"] == pytest.approx(
            O.mean_loss(lid, param, dim, vy, rec["VF_next"].reshape(-1)), rel=1e-5)


O_LOSS = {"squared": 0, "absolute": 1, "huber": 2, "quantile": 3, "bernoulli": 6, "exponential": 7, "logloss": 8}

# (estimator, data, loss, updates, regParam, weighted, bag)
CASES = (
    # every regressor loss; between them weighted and unweighted fits, no bag, a bag and Poisson multiplicities
    [("reg", "cpusmall", loss, "gradient", 0.1, weighted, bag) for loss, weighted, bag in (
        ("squared", False, "none"), ("squared", True, "poisson"), ("absolute", True, "bag"),
        ("absolute", False, "poisson"), ("huber", False, "bag"), ("huber", True, "poisson"),
        ("quantile", True, "none"), ("quantile", False, "bag"))]
    + [("reg", "cpusmall", "squared", "newton", reg, weighted, "bag") for reg in (0.0, 0.5) for weighted in (False, True)]
    + [("reg", "cpusmall-raw", "squared", "gradient", 0.1, True, "bag")]
    + [("cls", "adult8k", loss, updates, reg, reg > 0, "none")
       for loss in ("bernoulli", "exponential") for updates in ("gradient", "newton") for reg in (0.0, 0.5)]
    + [("cls", data, "logloss", updates, 0.5, True, "bag")
       for data, updates in (("letter3", "gradient"), ("letter3", "newton"), ("letter5", "newton"))]
)


@pytest.mark.parametrize("kind,data,loss,updates,reg,weighted,bag", CASES,
                         ids=["-".join(str(v) for v in c) for c in CASES])
def test_resident_linear_gbm_rounds_match_fp64(oracle, monkeypatch, kind, data, loss, updates, reg, weighted, bag):
    X, y = _data(data)
    est = _estimator(kind, loss, updates, reg, weighted, bag)
    spy = _Spy(monkeypatch)
    model = est.fit(_frame(X, y, weighted, seed=len(data) + 7 * weighted))
    monkeypatch.undo()
    dim = int(y.max()) + 1 if loss == "logloss" else 1
    if bag == "poisson":
        assert spy.rounds[0]["bag"].max() > 1
    _check_rounds(oracle, spy, est, model.trainingHistory, loss, dim)


@pytest.mark.parametrize("kind", ["reg", "cls"])
def test_resident_linear_gbm_keeps_residuals_and_weights_on_device(monkeypatch, kind):
    """Only the fitted model leaves the device in a round: no download of R or WOUT, bar fit_resident's one-value read
    of the label shift."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    if kind == "reg":
        X, y = _data("cpusmall")
        est = _estimator("reg", "squared", "newton", 0.5, True, "poisson")
    else:
        X, y = _data("letter3")
        est = _estimator("cls", "logloss", "newton", 0.5, True, "bag")
    real_download = Context.download
    reads = []

    def guarded(self, slot, *a, **k):
        if slot == N.SLOT_R:
            count = k.get("count", a[0] if a else None)
            assert count == 1, "residuals left the device"
            reads.append(slot)
        assert slot != N.SLOT_WOUT, "Newton weights left the device"
        return real_download(self, slot, *a, **k)

    monkeypatch.setattr(Context, "download", guarded)
    model = est.fit(_frame(X, y, True, seed=5))
    monkeypatch.undo()
    dim = int(y.max()) + 1 if kind == "cls" else 1
    assert len(model.trainingHistory) == ROUNDS and len(reads) == ROUNDS * dim
