"""se_logistic_loss_grad and se_logistic_stats against the fp64 numpy contract of oracle/np_logistic.py, their argument
checks, a scale case past 2^32-byte column offsets, se_logistic_predict against the host model, DeviceLogisticRegression
against the same optimiser driven by numpy, and StackingClassifier with logistic members and stackers."""
import os

import numpy as np
import pytest

from oracle import np_logistic as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    yield c
    c.close()


def _load(ctx, src, X, y, w=None):
    from spark_ensemble_b200 import _native as N
    n, d = X.shape
    ctx.alloc(src, d, n)
    if src == N.SLOT_X:
        ctx.upload_rowmajor(src, X)
    else:
        ctx.upload(src, np.ascontiguousarray(X.T))
    ctx.alloc(N.SLOT_Y, n)
    ctx.upload(N.SLOT_Y, y)
    if w is not None:
        ctx.alloc(N.SLOT_W, n)
        ctx.upload(N.SLOT_W, w)


def _case(n, p, D, seed):
    rng = np.random.default_rng(seed)
    d = p + 3 if n < 1000 else min(p + 3, 64)
    X = (rng.standard_normal((n, d)) * 2 + 5).astype(np.float32)
    K = max(D, 2)
    y = rng.integers(0, K, n).astype(np.float32)
    w = rng.uniform(0, 3, n).astype(np.float32)
    cols = rng.integers(0, d, p).astype(np.int32)  # unsorted, with repeats
    if p > 1:
        cols[-1] = cols[0]
    shift = X[0, cols].astype(np.float64) + 0.25
    scale = rng.uniform(0.2, 1.5, p)
    scale[rng.random(p) < 0.2] = 0.0
    coef = rng.standard_normal((D, p + 1)) * (2.0 / np.sqrt(p + 1))
    return X, y, w, cols, shift, scale, coef


def _check(ctx, src, X, y, w, cols, shift, scale, coef, tol=1e-12):
    from spark_ensemble_b200 import _native as N
    _load(ctx, src, X, y, w)
    wslot = N.SLOT_W if w is not None else -1
    loss, g = ctx.logistic_loss_grad(src, cols, coef, N.SLOT_Y, 0, wslot, 0, shift, scale)
    rl, rg = O.loss_grad(X, y, cols, coef, w, shift, scale)
    sl, sg = O.abs_terms(X, y, cols, coef, w, shift, scale)
    assert abs(loss - rl) <= tol * sl, (loss, rl, sl)
    err = np.abs(g - rg) / np.maximum(sg, 1e-300)
    assert err.max() <= tol, float(err.max())
    again = ctx.logistic_loss_grad(src, cols, coef, N.SLOT_Y, 0, wslot, 0, shift, scale)
    assert again[0] == loss and again[1].tobytes() == g.tobytes(), "two identical calls differ"


@pytest.mark.parametrize("D", [1, 2, 3, 26, 64])
@pytest.mark.parametrize("p", [1, 4, 33, 128, 254])
@pytest.mark.parametrize("n", [1, 31, 1_000_003])
def test_loss_grad_matches_numpy(ctx, n, p, D):
    from spark_ensemble_b200 import _native as N
    X, y, w, cols, shift, scale, coef = _case(n, p, D, n * 7 + p * 131 + D)
    if D == 1:
        y = (y > 0).astype(np.float32)
    for i, ww in enumerate((None, w)):
        _check(ctx, (N.SLOT_X, N.SLOT_P)[(i + p) % 2], X, y, ww, cols, shift, scale, coef)


@pytest.mark.parametrize("D", [1, 5])
def test_loss_grad_margins_beyond_700(ctx, D):
    from spark_ensemble_b200 import _native as N
    X, y, w, cols, shift, scale, coef = _case(4099, 6, D, 99 + D)
    if D == 1:
        y = (y > 0).astype(np.float32)
    coef = coef * 400.0  # |m| of several hundred to a few thousand
    Z = O._z(X, cols, shift, scale) @ coef.T
    assert np.abs(Z).max() > 700
    _check(ctx, N.SLOT_X, X, y, w, cols, shift, scale, coef)


def test_stats_match_numpy_and_count_invalid_rows(ctx):
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.learners import DeviceLogisticRegression
    rng = np.random.default_rng(5)
    n, d, K = 100_003, 40, 7
    X = (rng.standard_normal((n, d)) * 3 + 2).astype(np.float32)
    y = rng.integers(0, K, n).astype(np.float32)
    w = rng.uniform(0, 2, n).astype(np.float32)
    cols = rng.integers(0, d, 37).astype(np.int32)
    shift = X[0, cols].astype(np.float64)
    for src, ww in ((N.SLOT_X, None), (N.SLOT_P, w)):
        _load(ctx, src, X, y, ww)
        got = ctx.logistic_stats(src, cols, K, N.SLOT_Y, 0, N.SLOT_W if ww is not None else -1, 0, shift)
        ref = O.stats(X, y, cols, K, ww, shift)
        np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-9)
        assert got[-1] == 0
    yb, wb, Xb = y.copy(), w.copy(), X.copy()
    yb[[3, 10]] = [K, 0.5]
    wb[[10, 20]] = [-1.0, np.nan]
    Xb[30, cols[4]] = np.inf
    outside = [c for c in range(d) if c not in cols]
    Xb[31, outside[0]] = np.nan  # a column outside the list does not count
    _load(ctx, N.SLOT_X, Xb, yb, wb)
    got = ctx.logistic_stats(N.SLOT_X, cols, K, N.SLOT_Y, 0, N.SLOT_W, 0, shift)
    ref = O.stats(Xb, yb, cols, K, wb, shift)
    assert got[-1] == ref[-1] == 4
    with pytest.raises(ValueError, match="rows have a label"):
        DeviceLogisticRegression().fit_resident(ctx, N.SLOT_X, cols, K, N.SLOT_Y, 0, N.SLOT_W, 0)


def test_argument_errors(ctx):
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    n = 100
    with Context(0) as c:
        _load(c, N.SLOT_X, np.ones((n, 3), np.float32), np.ones(n, np.float32))
        coef = np.zeros((1, 3))
        with pytest.raises(ValueError, match="255 columns"):
            c.logistic_loss_grad(N.SLOT_X, np.zeros(255, np.int32), np.zeros((1, 256)), N.SLOT_Y)
        with pytest.raises(ValueError, match="only SE_SLOT_X or SE_SLOT_P"):
            c.logistic_loss_grad(N.SLOT_H, [0, 1], coef, N.SLOT_Y)
        with pytest.raises(ValueError, match="outside"):
            c.logistic_loss_grad(N.SLOT_X, [0, 3], coef, N.SLOT_Y)
        with pytest.raises(ValueError, match="weight slot"):
            c.logistic_loss_grad(N.SLOT_X, [0, 1], coef, N.SLOT_Y, weight_slot=N.SLOT_W)
        with pytest.raises(ValueError, match="no row 1"):
            c.logistic_stats(N.SLOT_X, [0, 1], 2, N.SLOT_Y, label_row=1)
        with pytest.raises(ValueError, match="65 coefficient sets"):
            c.logistic_loss_grad(N.SLOT_X, [0, 1], np.zeros((65, 3)), N.SLOT_Y)
        with pytest.raises(ValueError, match="65 classes"):
            c.logistic_stats(N.SLOT_X, [0, 1], 65, N.SLOT_Y)
        with pytest.raises(ValueError, match="0 classes"):
            c.logistic_stats(N.SLOT_X, [0, 1], 0, N.SLOT_Y)
        lib, h = c._lib, c._h
        out = np.zeros(8)
        assert lib.se_logistic_loss_grad(h, N.SLOT_X, 2, None, None, None, 1, N.dptr(out), N.SLOT_Y, 0, -1, 0,
                                         N.dptr(out)) == N.SE_ERR_ARG


def test_loss_grad_scale_50m_by_128(ctx):
    """50 M rows × 128 columns: column offsets past 2^32 bytes, against a torch fp64 computation on the same device."""
    import torch
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    n, p = 50_000_000, 128
    rng = np.random.default_rng(21)
    with Context(0) as c:
        c.alloc(N.SLOT_X, p, n)
        c.fill_synthetic(N.SLOT_X, "uniform", 11, -1.0, 3.0)
        c.alloc(N.SLOT_Y, n)
        c.fill_synthetic(N.SLOT_Y, "bernoulli", 12, 0.4, 0.0)
        cols = np.arange(p, dtype=np.int32)[::-1].copy()
        shift, scale = np.ones(p), rng.uniform(0.5, 1.5, p)
        coef = rng.standard_normal((1, p + 1)) * 0.2
        loss, g = c.logistic_loss_grad(N.SLOT_X, cols, coef, N.SLOT_Y, shift=shift, scale=scale)
        _, _, ld = c.layout(N.SLOT_X)

        class _Dev:  # the slots as torch tensors on the same device, without a copy
            def __init__(self, slot, shape):
                self.__cuda_array_interface__ = {"shape": shape, "typestr": "<f4", "version": 3,
                                                 "data": (c.device_ptr(slot), False)}
        dev = torch.device("cuda", 0)
        Xt = torch.as_tensor(_Dev(N.SLOT_X, (p, ld)), device=dev)
        yt = torch.as_tensor(_Dev(N.SLOT_Y, (n,)), device=dev)
        idx = torch.from_numpy(cols.astype(np.int64)).to(dev)
        th = torch.from_numpy(coef[0]).to(dev)
        sh, sc = torch.from_numpy(shift).to(dev), torch.from_numpy(scale).to(dev)
        rl = torch.zeros((), dtype=torch.float64, device=dev)
        rg = torch.zeros(p + 1, dtype=torch.float64, device=dev)
        sg = torch.zeros_like(rg)
        for r0 in range(0, n, 2_500_000):
            r1 = min(n, r0 + 2_500_000)
            Z = torch.ones((r1 - r0, p + 1), dtype=torch.float64, device=dev)
            Z[:, :p] = (Xt[idx, r0:r1].T.double() - sh) * sc
            m = Z @ th
            yy = (yt[r0:r1] == 1).double()
            e = torch.exp(-m.abs())
            rl += (m.clamp(min=0) + torch.log1p(e) - yy * m).sum()
            pi = torch.where(m >= 0, 1 / (1 + e), e / (1 + e))
            rg += (pi - yy) @ Z
            sg += (pi + yy) @ Z.abs()
            del Z
        assert int(cols[0]) * ld * 4 > 2 ** 32
        assert abs(loss - rl.item()) <= 1e-12 * n * 10
        err = np.abs(g[0] - rg.cpu().numpy()) / sg.cpu().numpy()
        assert err.max() <= 1e-12, float(err.max())


@pytest.mark.parametrize("D", [1, 26])
def test_predict_matches_host_model(ctx, D):
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.learners import LogisticRegressionModel
    rng = np.random.default_rng(D)
    n, p = 5001, 12
    X = rng.standard_normal((n, p)).astype(np.float32)
    beta, b = rng.standard_normal((D, p)), rng.standard_normal(D)
    if D > 1:
        b[3] = np.inf  # every row's probability goes to class 3
    models = [LogisticRegressionModel(beta, b, max(D, 2), D > 1, threshold=0.3)]
    if D == 1:
        models.append(LogisticRegressionModel(beta * 0, [np.inf], 2, False))
    for m in models:
        W = 2 if D == 1 else D
        ctx.alloc(N.SLOT_X, p, n)
        ctx.upload_rowmajor(N.SLOT_X, X)
        for slot, rows in ((N.SLOT_RAW, W), (N.SLOT_PROB, W), (N.SLOT_LABEL, 1)):
            ctx.alloc(slot, rows, n)
        ctx.logistic_predict(m.coefficientMatrix, m.interceptVector, m.threshold, raw=(N.SLOT_RAW, 0),
                             prob=(N.SLOT_PROB, 0), label=(N.SLOT_LABEL, 0))
        raw = ctx.download(N.SLOT_RAW).reshape(W, n).T
        prob = ctx.download(N.SLOT_PROB).reshape(W, n).T
        lab = ctx.download(N.SLOT_LABEL).reshape(-1)
        scale = np.abs(X.astype(np.float64)) @ np.abs(m.coefficientMatrix.T) + np.abs(m.interceptVector)
        ref_raw = m.predictRaw(X)
        fin = np.isfinite(ref_raw)
        tol = 4 * 2.0 ** -24 * (np.tile(scale, (1, 2)) if D == 1 else scale)
        assert np.all(np.abs(raw[fin] - ref_raw[fin]) <= tol[fin])
        np.testing.assert_array_equal(raw[~fin], ref_raw[~fin])
        np.testing.assert_allclose(prob, m.predictProbability(X), rtol=0, atol=1e-6)
        ref_lab = m.predict(X)
        close = np.zeros(n, bool)
        if D == 1:
            close = np.abs(m.predictProbability(X)[:, 1] - m.threshold) < 1e-6
        np.testing.assert_array_equal(lab[~close], ref_lab[~close])


@pytest.mark.parametrize("name,kw", [("adult8k", {}), ("adult8k", {"regParam": 0.01, "elasticNetParam": 0.5}),
                                     ("letter", {"regParam": 0.01})])
def test_device_fit_matches_cpu_driver(name, kw):
    from spark_ensemble_b200.learners import DeviceLogisticRegression
    z = np.load(os.path.join(ROOT, "tests", "golden", f"{name}.npz"))
    X, y = z["X"].astype(np.float32), z["y"].astype(np.float64)
    w = np.random.default_rng(1).uniform(0.5, 2, y.size).astype(np.float32).astype(np.float64)
    est = DeviceLogisticRegression(tol=1e-10, maxIter=2000, **kw)
    dev = est.fit(X, y, w)
    cols = np.arange(X.shape[1])
    X64 = X.astype(np.float64)
    shift = X64[0].copy()  # the shifts DeviceLogisticRegression.fit takes
    K = int(y.max()) + 1
    host = est.optimize(O.evaluator(X64, y, cols, w), O.stats(X64, y, cols, K, w, shift), shift, K)
    f, fh = dev.objectiveHistory[-1], host.objectiveHistory[-1]
    assert abs(f - fh) <= 1e-7 * abs(fh), (f, fh)
    scale = np.abs(host.coefficientMatrix).max()
    assert np.abs(dev.coefficientMatrix - host.coefficientMatrix).max() <= 1e-4 * scale
    assert dev.numEvaluations > 1


def _letter():
    z = np.load(os.path.join(ROOT, "tests", "golden", "letter.npz"))
    return z["X"].astype(np.float32), z["y"].astype(np.float64)


class _Recorder:
    """A host stacker that records the meta-features it is fitted on."""

    def __init__(self, log):
        self.log = log

    def copy(self, extra=None):
        return _Recorder(self.log)

    def fit(self, X, y, w=None, num_classes=None):
        self.log.append(np.array(X, dtype=np.float64))
        from spark_ensemble_b200.learners import DecisionTreeClassifier
        return DecisionTreeClassifier(maxDepth=1).fit(X[:, :1], y, w, num_classes)


@pytest.mark.parametrize("method", ["class", "raw", "proba"])
def test_stacking_classifier_with_logistic_member_and_stacker(method):
    from spark_ensemble_b200.classification import StackingClassifier
    from spark_ensemble_b200.ensemble import DataFrame
    from spark_ensemble_b200.learners import DeviceDecisionTreeClassifier, DeviceLogisticRegression
    X, y = _letter()
    X, y = X[:6000], y[:6000]
    df = DataFrame(features=X, label=y)
    members = [DeviceDecisionTreeClassifier(maxDepth=6), DeviceLogisticRegression(regParam=0.01)]
    est = StackingClassifier().setBaseLearners(members).setStackMethod(method)
    logs = {}
    for resident in (False, True):
        logs[resident] = []
        est.copy().setStacker(_Recorder(logs[resident])).setResidentFeatures(resident).fit(df)
    host, dev = logs[False][0], logs[True][0]
    np.testing.assert_allclose(dev, host, rtol=8 * 2.0 ** -23, atol=1e-5)  # a few fp32 ulps (and the fit's tolerance)
    stacker = DeviceLogisticRegression(regParam=0.01)
    model = est.copy().setStacker(stacker).setResidentFeatures(True).fit(df)
    ref = stacker.fit(dev, y, np.ones(y.size), num_classes=26)  # the same stacker over the downloaded meta-features
    np.testing.assert_array_equal(model.stack.coefficientMatrix, ref.coefficientMatrix)
    np.testing.assert_array_equal(model.stack.interceptVector, ref.interceptVector)
    out = model.transform(DataFrame(features=X))["prediction"]
    # the same model scored in fp64 on the device and on the host: equal labels, but for rows whose two best margins
    # tie to rounding (the two sums run in different orders)
    M = np.sort(ref._margins(dev), axis=1)
    tie = (M[:, -1] - M[:, -2]) <= 1e-9 * (1.0 + np.abs(M[:, -1]))
    np.testing.assert_array_equal(out[~tie], ref.predict(dev)[~tie])
    assert tie.sum() <= 2, int(tie.sum())
    assert np.mean(out == y) > 3.0 / 26


@pytest.mark.parametrize("ensemble", ["bagging", "boosting"])
def test_stacking_classifier_with_tree_ensemble_stacker_on_device_route(ensemble):
    """A classifier ensemble of trees as the stacker: the device route's transform scores it over the meta-features on
    the host, and gives the label of every row, as the stack predicts over the downloaded meta-features."""
    from spark_ensemble_b200.classification import BaggingClassifier, BoostingClassifier, StackingClassifier
    from spark_ensemble_b200.ensemble import DataFrame
    from spark_ensemble_b200.learners import DeviceDecisionTreeClassifier, DeviceLogisticRegression
    from spark_ensemble_b200.routes import model_predict
    X, y = _letter()
    X, y = X[:3000], y[:3000]
    df = DataFrame(features=X, label=y)
    members = [DeviceDecisionTreeClassifier(maxDepth=6), DeviceLogisticRegression(regParam=0.01)]
    est = StackingClassifier().setBaseLearners(members).setStackMethod("proba").setResidentFeatures(True)
    log = []
    est.copy().setStacker(_Recorder(log)).fit(df)
    cls = BaggingClassifier if ensemble == "bagging" else BoostingClassifier
    stacker = cls().setBaseLearner(DeviceDecisionTreeClassifier(maxDepth=4)).setNumBaseLearners(4) \
        .setResidentFeatures(True)
    model = est.copy().setStacker(stacker).fit(df)
    out = model.transform(DataFrame(features=X))["prediction"]
    assert out.shape == (X.shape[0],)
    np.testing.assert_array_equal(out, model_predict(model.stack, log[0]))


def test_device_route_uploads_x_once_with_logistic(monkeypatch):
    from spark_ensemble_b200.classification import StackingClassifier
    from spark_ensemble_b200.context import Context
    from spark_ensemble_b200.ensemble import DataFrame
    from spark_ensemble_b200.learners import DeviceDecisionTreeClassifier, DeviceLogisticRegression
    X, y = _letter()
    X, y = X[:3000], y[:3000]
    calls = []
    orig = Context.upload_rowmajor

    def spy(self, slot, features, row_offset=0):
        calls.append(np.asarray(features).shape)
        return orig(self, slot, features, row_offset)
    monkeypatch.setattr(Context, "upload_rowmajor", spy)
    est = StackingClassifier().setBaseLearners([DeviceDecisionTreeClassifier(maxDepth=4), DeviceLogisticRegression()]) \
        .setStacker(DeviceLogisticRegression()).setStackMethod("raw").setResidentFeatures(True)
    model = est.fit(DataFrame(features=X, label=y))
    assert calls == [X.shape]
    calls.clear()
    model.transform(DataFrame(features=X))
    assert calls == [X.shape]


def test_stacking_beats_its_members_on_letter():
    """The reference suite's first StackingClassifier test with device learners, a logistic member and a logistic
    stacker, stackMethod "raw", on an 80/20 split of letter."""
    from spark_ensemble_b200.classification import BoostingClassifier, GBMClassifier, StackingClassifier
    from spark_ensemble_b200.ensemble import DataFrame
    from spark_ensemble_b200.learners import (DeviceDecisionTreeClassifier, DeviceDecisionTreeRegressor,
                                              DeviceLogisticRegression)
    from spark_ensemble_b200.routes import model_outputs
    X, y = _letter()
    rng = np.random.default_rng(2019)
    train = rng.random(y.size) < 0.8
    Xtr, ytr, Xte, yte = X[train], y[train], X[~train], y[~train]
    boost = BoostingClassifier().setBaseLearner(DeviceDecisionTreeClassifier(maxDepth=5)).setNumBaseLearners(5) \
        .setResidentFeatures(True)
    gbm = GBMClassifier().setBaseLearner(DeviceDecisionTreeRegressor(maxDepth=4)).setNumBaseLearners(5) \
        .setResidentFeatures(True)
    members = [DeviceDecisionTreeClassifier(maxDepth=8), boost, gbm, DeviceLogisticRegression()]
    model = StackingClassifier().setBaseLearners(members).setStacker(DeviceLogisticRegression()) \
        .setStackMethod("raw").setResidentFeatures(True).fit(DataFrame(features=Xtr, label=ytr))
    acc = lambda p: float(np.mean(p == yte))
    stack = acc(model.transform(DataFrame(features=Xte))["prediction"])
    each = [acc(model_outputs(m, Xte, "class", 1)[0]) for m in model.models]
    print("letter accuracies: stack", stack, "members", each)
    assert stack > max(each), (stack, each)
