"""se_linear_moments against the fp64 numpy moments of oracle/np_linear.py, its argument checks, a scale case past
2^32-byte column offsets, and DeviceLinearRegression against the host learner."""
import os

import numpy as np
import pytest

from oracle import np_linear

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    yield c
    c.close()


def _load(ctx, src, X, y, w=None, bag=None):
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
    if bag is not None:
        ctx.alloc(N.SLOT_BAG, n)
        ctx.upload(N.SLOT_BAG, bag)


@pytest.mark.parametrize("n", [1, 31, 1_000_003])
@pytest.mark.parametrize("p", [1, 4, 33, 128, 254])
def test_moments_match_numpy(ctx, n, p):
    from spark_ensemble_b200 import _native as N
    rng = np.random.default_rng(n * 1000 + p)
    d = p + 3 if n < 1000 else min(p + 3, 160)
    if n * d > 120_000_000:
        d = p
    X = (rng.standard_normal((n, d)) * 2 + 5).astype(np.float32)
    y = (rng.standard_normal(n) + 10).astype(np.float32)
    w = rng.uniform(0, 3, n).astype(np.float32)
    bag = rng.poisson(1.0, n).astype(np.float32)
    cols = rng.integers(0, d, p).astype(np.int32)  # unsorted, with repeats
    if p > 1:
        cols[-1] = cols[0]
    shift = X[0, cols].astype(np.float64) + 0.25
    ys = float(y[0]) - 0.5
    cases = [("neither", None, None), ("weights", w, None), ("bag", None, bag)]
    for i, (name, ww, bb) in enumerate(cases):
        src = (N.SLOT_X, N.SLOT_P)[i % 2]
        _load(ctx, src, X, y, ww, bb)
        got = ctx.linear_moments(src, cols, N.SLOT_Y, 0, N.SLOT_W if ww is not None else -1, 0, bb is not None,
                                 shift, ys)
        ref = np_linear.linear_moments(X, y, cols, ww, bb, shift, ys)
        scale = np_linear.abs_moments(X, y, cols, ww, bb, shift, ys)
        err = np.abs(got - ref) / np.maximum(scale, 1e-300)
        assert err.max() <= 1e-12, (name, src, float(err.max()))
        np.testing.assert_array_equal(got, got.T)
        again = ctx.linear_moments(src, cols, N.SLOT_Y, 0, N.SLOT_W if ww is not None else -1, 0, bb is not None,
                                   shift, ys)
        assert again.tobytes() == got.tobytes(), "two identical calls differ"


def test_moment_argument_errors(ctx):
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    n = 100
    X = np.ones((n, 3), np.float32)
    with Context(0) as c:
        _load(c, N.SLOT_X, X, np.ones(n, np.float32))
        with pytest.raises(ValueError, match="255 columns"):
            c.linear_moments(N.SLOT_X, np.zeros(255, np.int32), N.SLOT_Y)
        with pytest.raises(ValueError, match="weight slot"):
            c.linear_moments(N.SLOT_X, [0, 1], N.SLOT_Y, weight_slot=N.SLOT_W)
        with pytest.raises(ValueError, match="bag slot"):
            c.linear_moments(N.SLOT_X, [0, 1], N.SLOT_Y, use_bag=True)
        with pytest.raises(ValueError, match="no row 1"):
            c.linear_moments(N.SLOT_X, [0, 1], N.SLOT_Y, label_row=1)
        with pytest.raises(ValueError, match="outside"):
            c.linear_moments(N.SLOT_X, [0, 3], N.SLOT_Y)
        with pytest.raises(ValueError, match="only SE_SLOT_X or SE_SLOT_P"):
            c.linear_moments(N.SLOT_H, [0], N.SLOT_Y)
        lib, h = c._lib, c._h
        out = np.zeros(2 * 2)
        assert lib.se_linear_moments(h, N.SLOT_X, 255, None, None, 0.0, N.SLOT_Y, 0, -1, 0, 0, N.dptr(out)) == N.SE_ERR_ARG


def test_moments_scale_50m_by_128(ctx):
    """50 M rows × 128 columns: column offsets past 2^32 bytes, against a torch fp64 matmul on the same device."""
    import torch
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    n, p = 50_000_000, 128
    with Context(0) as c:
        c.alloc(N.SLOT_X, p, n)
        c.fill_synthetic(N.SLOT_X, "uniform", 11, -1.0, 3.0)
        c.alloc(N.SLOT_Y, n)
        c.fill_synthetic(N.SLOT_Y, "normal", 12, 2.0, 1.0)
        cols = np.arange(p, dtype=np.int32)[::-1].copy()
        got = c.linear_moments(N.SLOT_X, cols, N.SLOT_Y, shift=np.ones(p), label_shift=2.0)
        _, _, ld = c.layout(N.SLOT_X)

        class _Dev:  # the slots as torch tensors on the same device, without a copy
            def __init__(self, slot, shape):
                self.__cuda_array_interface__ = {"shape": shape, "typestr": "<f4", "version": 3,
                                                 "data": (c.device_ptr(slot), False)}
        dev = torch.device("cuda", 0)
        Xt = torch.as_tensor(_Dev(N.SLOT_X, (p, ld)), device=dev)
        yt = torch.as_tensor(_Dev(N.SLOT_Y, (n,)), device=dev)
        ref = torch.zeros((p + 2, p + 2), dtype=torch.float64, device=dev)
        scale = torch.zeros_like(ref)
        idx = torch.from_numpy(cols.astype(np.int64)).to(dev)
        for r0 in range(0, n, 2_500_000):
            r1 = min(n, r0 + 2_500_000)
            Z = torch.empty((r1 - r0, p + 2), dtype=torch.float64, device=dev)
            Z[:, :p] = Xt[idx, r0:r1].T.double() - 1.0
            Z[:, p] = 1.0
            Z[:, p + 1] = yt[r0:r1].double() - 2.0
            ref += Z.T @ Z
            Z.abs_()
            scale += Z.T @ Z
            del Z
        ref, scale = ref.cpu().numpy(), scale.cpu().numpy()
        assert int(cols[0]) * ld * 4 > 2 ** 32
        err = np.abs(got - ref) / scale
        assert err.max() <= 1e-12, float(err.max())


def test_device_linear_regression_matches_host_on_cpusmall():
    from spark_ensemble_b200.learners import DeviceLinearRegression, LinearRegression
    z = np.load(os.path.join(ROOT, "tests", "golden", "cpusmall.npz"))
    X, y = z["X"].astype(np.float32), z["y"].astype(np.float32).astype(np.float64)
    w = np.random.default_rng(3).uniform(0.5, 2, y.size).astype(np.float32).astype(np.float64)
    for weights, reg in ((None, 0.0), (w, 0.0), (w, 10.0)):
        dev = DeviceLinearRegression(reg).fit(X, y, weights)
        host = LinearRegression(reg).fit(X.astype(np.float64), y, weights)
        np.testing.assert_allclose(dev.coefficients, host.coefficients, rtol=1e-7, atol=1e-9)
        np.testing.assert_allclose(dev.predict(X), host.predict(X), rtol=1e-9, atol=1e-9 * np.abs(y).max())
