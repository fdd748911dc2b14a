"""Parity at BASELINE.json's shard sizes (VERDICT r1 'What's weak' 2): the code paths that only exist at scale —
multi-CTA-per-SM persistent grids, the L2 policy of shards larger than the L2, element offsets beyond 2^31 in [K][n] arrays, 32-bit TMA
tile coordinates near their range, M = 512 fp64 batch folding — checked against the fp64 OpenMP oracle evaluated in
row chunks on data generated on the device and downloaded chunk by chunk.

Sums (GLOBAL scalars) are accumulated over ALL chunks; per-row outputs are compared on every chunk (GBM) or on the
first / middle / last chunks (wide arrays).  Tolerance 1e-5 relative (north_star)."""
import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu

RTOL = 1e-5
CHUNK = 4_000_000


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def orc():
    from oracle.oracle import Oracle
    import os
    o = Oracle(omp=True)
    n = len(os.sched_getaffinity(0))
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if q != "max":
            n = max(1, min(n, int(float(q) / float(p) + 0.5)))
    except Exception:
        pass
    o.lib.orc_set_num_threads(n)
    return o


def chunks(n, size=CHUNK):
    for a in range(0, n, size):
        yield a, min(n, a + size)


def rows(ctx, slot, a, b, dim=1):
    """Rows [a, b) of a [dim][n] slot as float64 [dim][b-a]."""
    _, n, _ = ctx.layout(slot)
    out = np.empty((dim, b - a), dtype=np.float32)
    for j in range(dim):
        ctx.download(slot, count=b - a, offset=j * n + a, out=out[j])
    return out.astype(np.float64)


def max_rel(a, b, scale=1.0):
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), scale)))


def test_c2_squared_round_10m(ctx, orc):
    """Config 2 shard: 10 M rows, squared loss — one whole round (statistics, Brent, update, residuals, loss), both
    as one cooperative launch and as two launches."""
    from spark_ensemble_b200 import _native as N
    n = 10_000_000
    for fused in (1, 0):
        ctx.gbm_configure(n, 0, 1, "squared", 0.0, False)
        ctx.fill_synthetic(N.SLOT_Y, "normal", 11, 0.0, 1.0)
        ctx.fill_synthetic(N.SLOT_F, "normal", 12, 0.0, 0.5)
        ctx.copy_slot(N.SLOT_H, N.SLOT_Y)
        ctx.set_option("fused_round", 0)
        ctx.gbm_update([0.5], residual=False, loss=False)   # F = N(0, 0.5) + 0.5 y
        ctx.copy_slot(N.SLOT_H, N.SLOT_F)                   # direction correlated with the label
        ctx.fill_synthetic(N.SLOT_F, "normal", 13, 0.2, 0.3)
        y, F, h = rows(ctx, N.SLOT_Y, 0, n), rows(ctx, N.SLOT_F, 0, n), rows(ctx, N.SLOT_H, 0, n)
        ctx.set_option("fused_round", fused)
        try:
            a, ls, ne = ctx.gbm_round(0.3, True, 1e-6, 100, residual=True)
            assert ctx.get_option("last_round_fused") == fused
        finally:
            ctx.set_option("fused_round", -1)
        f = lambda x: orc.linesearch_eval(O.SQUARED, 0.0, y[0], None, F, h, [x])[0]
        ao, neo, st = orc.brent(f)
        assert st == 0 and abs(a - ao) <= 1e-5 * abs(ao) + 4e-6, (a, ao)
        orc.update(F, h, [0.3 * a])
        assert abs(ls / n - orc.mean_loss(O.SQUARED, 0.0, 1, y[0], F)) <= RTOL * (ls / n)
        assert max_rel(rows(ctx, N.SLOT_F, 0, n), F) <= RTOL
        r, _, _ = orc.pseudo_residuals(O.SQUARED, 0.0, 1, y[0], None, F, False, want_weights=False)
        assert max_rel(rows(ctx, N.SLOT_R, 0, n), r) <= RTOL


@pytest.mark.parametrize("name,dim", [("bernoulli", 1), ("logloss", 2)])
def test_c3_binary_50m(ctx, orc, name, dim):
    """Config 3 shard: 50 M rows (8 CTAs/SM grids, no L2 hints at this size): line-search objective and
    gradient, the device line search (bernoulli), fused update + residuals + loss."""
    from spark_ensemble_b200 import _native as N
    n = 50_000_000
    lid = O.LOSS_IDS[name]
    ctx.gbm_configure(n, 0, dim, name, 0.0, False)
    ctx.fill_synthetic(N.SLOT_Y, "bernoulli", 21, 0.4, 1.0)
    ctx.fill_synthetic(N.SLOT_F, "normal", 22, 0.0, 0.7)
    ctx.fill_synthetic(N.SLOT_H, "normal", 23, 0.1, 1.0)
    alpha = np.array([0.37, 0.81][:dim])
    lg, gg = ctx.gbm_linesearch_eval(alpha)
    dev = ctx.gbm_linesearch_brent() if dim == 1 else None
    step = 0.25 * alpha
    # oracle over chunks BEFORE the update (F is about to change): sums of the objective at alpha and at the device minimiser
    lsum, gsum, l_at_dev, wsum = 0.0, np.zeros(dim), 0.0, 0.0
    keep = {}
    for a, b in chunks(n):
        y, F, h = rows(ctx, N.SLOT_Y, a, b)[0], rows(ctx, N.SLOT_F, a, b, dim), rows(ctx, N.SLOT_H, a, b, dim)
        lo, go = orc.linesearch_eval(lid, 0.0, y, None, F, h, alpha)
        lsum += lo * (b - a); gsum += go * (b - a); wsum += b - a
        if dev is not None:
            l_at_dev += orc.linesearch_eval(lid, 0.0, y, None, F, h, [dev[0]])[0] * (b - a)
        if a in (0, (n // CHUNK // 2) * CHUNK) or b == n:
            keep[a] = (y, F, h)
    assert abs(lg - lsum / wsum) <= RTOL * abs(lsum / wsum), (lg, lsum / wsum)
    assert np.all(np.abs(gg - gsum / wsum) <= RTOL * np.maximum(np.abs(gsum / wsum), np.abs(gsum / wsum).max()))
    if dev is not None:
        assert abs(dev[1] - l_at_dev / wsum) <= RTOL * abs(l_at_dev / wsum), (dev, l_at_dev / wsum)
    ls, _ = ctx.gbm_update(step, residual=True, loss=True)
    # the loss sum needs every chunk of the NEW F: recompute from the kept inputs where possible, else from the device F
    tot = 0.0
    for a, b in chunks(n):
        y = keep[a][0] if a in keep else rows(ctx, N.SLOT_Y, a, b)[0]
        Fn = rows(ctx, N.SLOT_F, a, b, dim)
        tot += orc.mean_loss(lid, 0.0, dim, y, Fn) * (b - a)
        if a in keep:
            _, F, h = keep[a]
            Fo = F.copy(); orc.update(Fo, h, step)
            assert max_rel(Fn, Fo) <= RTOL
            r, _, _ = orc.pseudo_residuals(lid, 0.0, dim, y, None, Fo, False, want_weights=False)
            assert max_rel(rows(ctx, N.SLOT_R, a, b, dim), r) <= RTOL
    assert abs(ls - tot) <= RTOL * abs(tot), (ls, tot)
    for s in (N.SLOT_F, N.SLOT_H, N.SLOT_R):
        ctx.free(s)


def test_c4_samme_r_k26_beyond_2g_elements(ctx, orc):
    """Config 4: SAMME.R, K = 26, 84 M rows: P[26][n] holds 2.18 G elements (> 2^31), 8.7 GB."""
    from spark_ensemble_b200 import _native as N
    K, n = 26, 84_000_000
    assert K * n > 2 ** 31
    ctx.boost_configure(n, K, True)
    ctx.fill_synthetic(N.SLOT_Y, "randint", 31, 0, K)
    ctx.fill_synthetic(N.SLOT_PROBA, "uniform", 32, 0.001, 0.08)
    ctx.fill_synthetic(N.SLOT_BW, "uniform", 33, 0.5, 1.5)
    sw = ctx.slot_sum(N.SLOT_BW)
    # inputs of the sampled chunks before the in-place weight update
    sample = [0, (n // CHUNK // 2) * CHUNK, ((n - 1) // CHUNK) * CHUNK]
    before = {a: rows(ctx, N.SLOT_BW, a, min(n, a + CHUNK))[0] for a in sample}
    e, s = ctx.boost_real_update(sw)
    eo = so = swo = 0.0
    for a, b in chunks(n):
        w_new = rows(ctx, N.SLOT_BW, a, b)[0]
        so += float(np.sum(w_new))
        if a in before:
            y = rows(ctx, N.SLOT_Y, a, b)[0]
            P = rows(ctx, N.SLOT_PROBA, a, b, K)
            out, ec, sc = orc.samme_r_update(K, y, before[a], sw, P)
            assert max_rel(w_new, out, scale=1e-30) <= RTOL, a
            eo += ec
    assert abs(s - so) <= RTOL * so, (s, so)
    assert 0.0 < e < 1.0
    # the error sum over the sampled chunks must be consistent with the global one (uniform data): within 2 %
    assert abs(eo * (n / (len(sample) * CHUNK)) - e) <= 0.02 * e
    ctx.free(N.SLOT_PROBA)


def test_c5_aggregation_m512(ctx, orc):
    """Config 5 shard: 512 base-model outputs x 6.25 M rows (12.8 GB), Bagging mean and GBM weighted sum."""
    from spark_ensemble_b200 import _native as N
    M, n = 512, 6_250_000
    ctx.agg_configure(N.AGG_BAGGING_REGRESSOR, M, 0, 1, 0, n)
    ctx.fill_synthetic(N.SLOT_P, "normal", 41, 0.3, 1.0)
    ctx.agg_run()
    got_mean = rows(ctx, N.SLOT_RAW, 0, n)[0]
    wts = np.random.default_rng(5).random(M) * 0.2
    ctx.agg_configure(N.AGG_GBM_REGRESSOR, M, 0, 1, 0, n)
    ctx.agg_run(wts, [0.7])
    got_gbm = rows(ctx, N.SLOT_RAW, 0, n)[0]
    w32 = wts.astype(np.float32).astype(np.float64)  # the device holds fp32-narrowed weights
    C2 = 250_000
    for a in (0, (n // C2 // 2) * C2, n - C2):
        P = rows(ctx, N.SLOT_P, a, a + C2, M)
        assert max_rel(got_mean[a:a + C2], orc.agg_mean(P), scale=1e-3) <= RTOL
        assert max_rel(got_gbm[a:a + C2], orc.agg_weighted_sum(P, w32, 0.7), scale=1e-3) <= RTOL
    ctx.free(N.SLOT_P)


def test_tree_kernels_agree_beyond_2g_byte_offsets(ctx):
    """70 M rows x 40 columns: the uint8 rank matrix is 2.8 GB (column offsets beyond 2^31 bytes), the fp32 matrix 11.2
    GB.  The all-nodes kernel, the rank-matrix walk and the fp32 walk must pick the same leaf for every row (sums and
    three 1 M-row windows bit for bit), and a window must equal a plain numpy walk over the downloaded features."""
    from spark_ensemble_b200 import _native as N
    n, d, depth = 70_000_000, 40, 6
    ctx.alloc(N.SLOT_X, d, n)
    ctx.fill_synthetic(N.SLOT_X, "normal", 51, 0.0, 1.0)
    ctx.alloc(N.SLOT_H, 1, n)
    nn = 2 ** (depth + 1) - 1
    idx = np.arange(nn)
    leaf = idx >= 2 ** depth - 1
    feat = np.where(leaf, -1, (d - 1 - (idx * 7) % d))          # node 0 reads the LAST column
    thr = np.where(leaf, 0.0, ((idx * 13) % 9 - 4) * 0.25).astype(np.float32)
    tree = {"feature": feat.astype(np.int32), "threshold": thr, "left": np.where(leaf, 0, 2 * idx + 1).astype(np.int32),
            "right": np.where(leaf, 0, 2 * idx + 2).astype(np.int32), "value": np.linspace(-1, 1, nn).astype(np.float32)}
    W = 1_000_000
    wins = (0, (n // 2 // 4) * 4, n - W)
    got = {}
    try:
        for name, bins, mask in (("mask", 1, 1), ("walk", 1, 0), ("fp32", 0, 0)):
            ctx.set_option("tree_bins", bins)
            ctx.set_option("tree_mask", mask)
            ctx.tree_predict(tree, N.SLOT_H, 0)
            assert ctx.get_option("last_tree_binned") == bins and ctx.get_option("last_tree_mask") == (bins and mask)
            got[name] = (ctx.slot_sum(N.SLOT_H), [rows(ctx, N.SLOT_H, a, a + W)[0] for a in wins])
    finally:
        ctx.set_option("tree_bins", 1)
        ctx.set_option("tree_mask", 1)
    for name in ("walk", "fp32"):
        assert got[name][0] == got["mask"][0], name
        for u, v in zip(got[name][1], got["mask"][1]):
            np.testing.assert_array_equal(u, v)
    a, C2 = wins[1], 100_000
    X = rows(ctx, N.SLOT_X, a, a + C2, d).astype(np.float32)      # [d][C2]
    node = np.zeros(C2, dtype=np.int64)
    for _ in range(depth):
        f = np.maximum(feat[node], 0)
        node = np.where(X[f, np.arange(C2)] <= thr[node], tree["left"][node], tree["right"][node])
    np.testing.assert_array_equal(got["mask"][1][1][:C2], tree["value"][node].astype(np.float64))
    ctx.free(N.SLOT_X)


def test_weighted_median_fast_equals_exact_25m(ctx, orc):
    """BoostingRegressor.predict shard: 32 models x 25 M rows.  The margin-checked fast path and the exact kernel must
    return the same values (sum and windows bit for bit); a window against the oracle."""
    from spark_ensemble_b200 import _native as N
    M, n = 32, 25_000_000
    ctx.agg_configure(N.AGG_BOOSTING_REG_MEDIAN, M, 0, 1, 0, n)
    ctx.fill_synthetic(N.SLOT_P, "normal", 61, 0.0, 1.0)
    a = np.random.default_rng(9).random(M) + 0.05
    W = 1_000_000
    wins = (0, (n // 2 // 4) * 4, n - W)
    got = {}
    try:
        for fast in (1, 0):
            ctx.set_option("wm_fast", fast)
            ctx.agg_run(a)
            assert ctx.get_option("last_wm_mode") == fast
            got[fast] = (ctx.slot_sum(N.SLOT_RAW), [rows(ctx, N.SLOT_RAW, s, s + W)[0] for s in wins])
    finally:
        ctx.set_option("wm_fast", 1)
    assert got[1][0] == got[0][0]
    for u, v in zip(got[1][1], got[0][1]):
        np.testing.assert_array_equal(u, v)
    s, C2 = wins[1], 200_000
    P = rows(ctx, N.SLOT_P, s, s + C2, M)
    np.testing.assert_array_equal(got[1][1][1][:C2], orc.agg_weighted_median(P, a))
    ctx.free(N.SLOT_P)
