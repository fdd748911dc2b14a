"""The one-launch squared-loss round (residual mode, reading r, no bag) carries its statistics pass's last tile into
the update pass in registers and, with `fused_resident`, the groups before it in shared memory.  Where a group comes
from must not change a bit of the round: alpha, the loss, the evaluation count and r' are the same with the shared
memory carry on and off, and r' is the fp32 emulation of r - c h, round after round."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LR = 0.7
# 3: no full float4 group (scalar tail only); 40961: fewer tiles than CTAs; 4866047: at 3 CTAs per SM on 132 SMs
# every tile of a CTA is carried; 10000001: part carried, part streamed.  None is a multiple of 4 or of a tile.
SIZES = [3, 40961, 4_866_047, 10_000_001]


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    c.set_option("fused_round", 1)
    yield c
    c.close()


@pytest.fixture
def opts(ctx):
    """Options a test changes, restored afterwards (the context is shared by the module)."""
    keys = ("fused_resident", "fused_ctas_per_sm", "alternate_passes", "fused_loss_reduce")
    saved = {k: ctx.get_option(k) for k in keys}
    yield ctx
    for k, v in saved.items():
        ctx.set_option(k, v)


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def d64(a):
    return np.asarray(a, dtype=np.float64)


def fma32(c, h, x):
    """fp32 fmaf(c, h, x): c h is exact in fp64, the sum is rounded to fp32."""
    return f32(d64(x) + d64(f32(c)) * d64(h))


def problem(n, seed):
    rng = np.random.default_rng(seed)
    y = f32(rng.standard_normal(n))
    F = f32(0.7 * rng.standard_normal(n))
    h = f32(0.6 * (d64(y) - F) + 0.2 * rng.standard_normal(n))
    return y, F, h


def run_rounds(ctx, y, F, h, resident, rounds):
    """A fit's loop on the current residual: round, read R.  Returns per round (alpha, loss, evals, r, tiles)."""
    from spark_ensemble_b200 import _native as N
    ctx.set_option("fused_resident", resident)
    ctx.gbm_configure(len(y), 0, 1, "squared", 0.0, False)
    ctx.upload(N.SLOT_Y, y)
    ctx.upload(N.SLOT_F, F)
    ctx.upload(N.SLOT_H, h)
    ctx.gbm_pseudo_residuals(False)
    out = []
    for _ in range(rounds):
        a, loss, ne = ctx.gbm_round(LR, True, 1e-6, 100, residual=True)
        assert ctx.get_option("last_round_fused") == 1
        out.append((a, loss, ne, ctx.download(N.SLOT_R).copy(), ctx.get_option("last_fused_resident_tiles")))
    return out


@pytest.mark.parametrize("alternate", [1, 0])
@pytest.mark.parametrize("ctas", [3, 2])
@pytest.mark.parametrize("n", SIZES)
def test_carry_is_bit_identical(opts, n, ctas, alternate):
    ctx = opts
    ctx.set_option("fused_ctas_per_sm", ctas)
    ctx.set_option("alternate_passes", alternate)
    y, F, h = problem(n, 1000 + n % 97)
    on = run_rounds(ctx, y, F, h, 1, 4)
    off = run_rounds(ctx, y, F, h, 0, 4)
    r = f32(d64(y) - F)
    for k, ((a1, l1, ne1, r1, t1), (a0, l0, ne0, r0, t0)) in enumerate(zip(on, off)):
        assert (a1, l1, ne1) == (a0, l0, ne0), k
        np.testing.assert_array_equal(r1, r0, err_msg=f"round {k}")
        r = fma32(-f32(LR * a1), h, r)
        np.testing.assert_array_equal(r1, r, err_msg=f"round {k}")
        assert t0 == 0.0
        # shared memory holds groups only when a CTA has tiles before its last one
        assert (t1 > 0.0) == (n > 1_000_000), (n, t1)


def test_carry_with_row_reduced_loss(opts):
    """fused_loss_reduce sums r'^2/2 over the rows in the update pass: same tile order, same sum, bit for bit."""
    ctx = opts
    ctx.set_option("fused_loss_reduce", 1)
    y, F, h = problem(10_000_001, 7)
    on = run_rounds(ctx, y, F, h, 1, 2)
    off = run_rounds(ctx, y, F, h, 0, 2)
    for (a1, l1, ne1, r1, t1), (a0, l0, ne0, r0, _) in zip(on, off):
        assert (a1, l1, ne1) == (a0, l0, ne0)
        np.testing.assert_array_equal(r1, r0)
        assert t1 > 0.0
        assert l1 == pytest.approx(0.5 * float(np.sum(d64(r1) ** 2)), rel=1e-6)


def test_maxeval_leaves_r_with_carry(opts):
    from spark_ensemble_b200 import _native as N
    ctx = opts
    y, F, h = problem(10_000_001, 8)
    r = run_rounds(ctx, y, F, h, 1, 2)[-1][3]
    with pytest.raises(N.ConvergenceError):
        ctx.gbm_round(LR, True, 1e-12, 2, residual=True)
    assert ctx.get_option("last_fused_resident_tiles") > 0.0
    np.testing.assert_array_equal(ctx.download(N.SLOT_R), r)


def test_other_rounds_carry_nothing_in_shared_memory(opts):
    """Rounds that read y and F, bagged rounds and eager F updates keep their own path."""
    from spark_ensemble_b200 import _native as N
    ctx = opts
    n = 10_000_001
    y, F, h = problem(n, 9)
    ctx.set_option("fused_resident", 1)
    ctx.gbm_configure(n, 0, 1, "squared", 0.0, False)
    ctx.upload(N.SLOT_Y, y)
    ctx.upload(N.SLOT_F, F)
    ctx.upload(N.SLOT_H, h)
    a, _, _ = ctx.gbm_round(LR, True, 1e-6, 100, residual=True)  # the residual slot is not current: reads y, F
    assert ctx.get_option("last_fused_resident_tiles") == 0.0
    r = fma32(-f32(LR * a), h, f32(d64(y) - F))
    np.testing.assert_array_equal(ctx.download(N.SLOT_R), r)
    ctx.gbm_set_bag(f32(np.random.default_rng(10).poisson(1.0, n)))
    try:
        a, _, _ = ctx.gbm_round(LR, True, 1e-6, 100, residual=True)
        assert ctx.get_option("last_fused_resident_tiles") == 0.0
        np.testing.assert_array_equal(ctx.download(N.SLOT_R), fma32(-f32(LR * a), h, r))
    finally:
        ctx.gbm_set_bag(None)
