"""se_logistic_loss_grad_batch (Context.logistic_loss_grad_batch): the loss and gradient of several logistic members
over the same rows in one call.  Every member is checked against the fp64 numpy contract of oracle/np_logistic.py at
1e-12 of the sums of absolute terms, at D = 1, 2, 26 and 64, members of p = 0, 1, 40, 41 and 254 columns (unsorted, with
repeats; the union of a batch's columns at 254), labels and weights read from rows other than row 0 of padded slots,
and rows of weight 0 whose features are ±inf or NaN, which must contribute nothing.  A member's bits must not change
between identical calls, nor when the batch is permuted, shrunk to that member alone or grown with other members."""
import numpy as np
import pytest

from oracle import np_logistic as O

pytestmark = pytest.mark.gpu

D_FEATURES = 254


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    yield c
    c.close()


def _member(rng, p, D):
    if p == D_FEATURES:
        cols = rng.permutation(D_FEATURES).astype(np.int32)  # every column once: the batch's union is 254
    else:
        cols = rng.integers(0, D_FEATURES, p).astype(np.int32)
        if p > 1:
            cols[-1] = cols[0]
    shift = rng.standard_normal(p) + 5.0
    scale = rng.uniform(0.2, 1.5, p)
    scale[rng.random(p) < 0.2] = 0.0
    coef = rng.standard_normal((D, p + 1)) * (2.0 / np.sqrt(p + 1))
    return cols, coef, shift, scale


def _case(ctx, n, D, ps, seed):
    """Loads X (SLOT_X), the labels (row 2 of a 3-row SLOT_PROB) and the weights (row 1 of a 4-row SLOT_RAW) and returns
    the host copies and the members."""
    from spark_ensemble_b200 import _native as N
    rng = np.random.default_rng(seed)
    X = (rng.standard_normal((n, D_FEATURES)) * 2 + 5).astype(np.float32)
    K = max(D, 2)
    y = rng.integers(0, K, n).astype(np.float32)
    w = rng.uniform(0, 3, n).astype(np.float32)
    w[rng.random(n) < 0.25] = 0.0
    zero = np.flatnonzero(w == 0)
    for k, r in enumerate(zero[:64]):  # out-of-bag rows holding non-finite features in the members' columns
        X[r, rng.choice(D_FEATURES, 40, replace=False)] = np.array([np.inf, -np.inf, np.nan], np.float32)[k % 3]
    ctx.alloc(N.SLOT_X, D_FEATURES, n)
    ctx.upload_rowmajor(N.SLOT_X, X)
    for slot, rows, row, v in ((N.SLOT_PROB, 3, 2, y), (N.SLOT_RAW, 4, 1, w)):
        data = rng.uniform(-7, 9, (rows, n)).astype(np.float32)
        data[row] = v
        ctx.alloc(slot, rows, n)
        ctx.upload(slot, data)
    members = [_member(rng, p, D) for p in ps]
    return X, y, w, members


def _call(ctx, members):
    from spark_ensemble_b200 import _native as N
    return ctx.logistic_loss_grad_batch(N.SLOT_X, members, N.SLOT_PROB, 2, N.SLOT_RAW, 1)


def _bits(r):
    return np.float64(r[0]).tobytes() + r[1].tobytes()


def _check(ctx, n, D, ps, seed):
    X, y, w, members = _case(ctx, n, D, ps, seed)
    got = _call(ctx, members)
    live = w != 0
    for (cols, coef, shift, scale), (loss, g) in zip(members, got):
        args = (X[live], y[live], cols, coef, w[live], shift, scale)
        rl, rg = O.loss_grad(*args)
        sl, sg = O.abs_terms(*args)
        assert g.shape == (D, cols.size + 1)
        assert abs(loss - rl) <= 1e-12 * sl, (loss, rl, sl)
        err = np.abs(g - rg) / np.maximum(sg, 1e-300)
        assert err.max() <= 1e-12, float(err.max())
    bits = [_bits(r) for r in got]
    assert [_bits(r) for r in _call(ctx, members)] == bits, "two identical calls differ"
    order = np.random.default_rng(seed + 1).permutation(len(members))
    permuted = _call(ctx, [members[i] for i in order])
    assert [_bits(permuted[k]) for k in np.argsort(order)] == bits, "a permuted batch changes a member's bits"
    for i, m in enumerate(members):
        assert _bits(_call(ctx, [m])[0]) == bits[i], f"member {i} alone differs from member {i} in the batch"
    rng = np.random.default_rng(seed + 2)
    extra = [_member(rng, p, D) for p in (3, 41, 200)]
    grown = _call(ctx, extra[:2] + members + extra[2:])
    assert [_bits(r) for r in grown[2:2 + len(members)]] == bits, "a grown batch changes a member's bits"


@pytest.mark.parametrize("n", [1, 33, 4099])
@pytest.mark.parametrize("D", [1, 2, 26, 64])
def test_batch_matches_the_contract(ctx, n, D):
    _check(ctx, n, D, [0, 1, 40, 41, 254], 1000 * D + n)


@pytest.mark.parametrize("D", [1, 26])
def test_batch_at_a_million_rows(ctx, D):
    _check(ctx, 10**6 + 3, D, [0, 1, 40, 41], 77 + D)


def test_batch_member_equals_the_lone_call_on_finite_rows(ctx):
    """Without non-finite features a member runs what se_logistic_loss_grad runs over the same rows: the same bits."""
    from spark_ensemble_b200 import _native as N
    n = 4099
    for D in (1, 5):
        X, y, w, members = _case(ctx, n, D, [7, 39, 41, 120], 900 + D)
        X = np.where(np.isfinite(X), X, np.float32(1))
        ctx.upload_rowmajor(N.SLOT_X, X)
        for (cols, coef, shift, scale), r in zip(members, _call(ctx, members)):
            lone = ctx.logistic_loss_grad(N.SLOT_X, cols, coef, N.SLOT_PROB, 2, N.SLOT_RAW, 1, shift, scale)
            assert _bits(lone) == _bits(r)


def test_batch_rejects_mixed_class_counts_and_bad_columns(ctx):
    X, y, w, members = _case(ctx, 33, 2, [3, 4], 5)
    rng = np.random.default_rng(6)
    with pytest.raises(ValueError):
        _call(ctx, [members[0], _member(rng, 3, 3)])
    cols, coef, shift, scale = members[1]
    with pytest.raises(ValueError, match="outside slot"):
        _call(ctx, [members[0], (np.array([0, D_FEATURES, 1], np.int32), coef[:, :4], shift[:3], scale[:3])])
