"""Seeded random walks of GBM context calls, checked call by call against an fp64 model of y, F, h, r and WOUT
(tests/gbm_walk.py).

The context keeps derived state between calls (an owed F, pending residual steps, carried statistics, WOUT's 1/S, the
weight sum, the rank matrix), and reads settle some of it.  So each walk runs three times: A with only the reads it
drew (plus a final read of everything), B with F, R, VF, H, VH and WOUT read after every call, C with R read after
every call.  All three must agree with the model; A and C, which differ only by reads of R, bit for bit.  Walks that
never flip the options documented as bit-identical run once per such setting and must match the default bits.

A failure prints the seed, the step and the calls up to it: `generate(seed, ...)` replays the walk."""
import numpy as np
import pytest

from tests import gbm_walk as W

pytestmark = pytest.mark.gpu

SIZES = (3, 1001, 40961)
SEEDS = [(3, 101), (3, 102), (1001, 201), (1001, 202), (1001, 203), (40961, 301), (40961, 302), (40961, 303)]
BIG = 10_000_001  # several tiles per CTA, part of them carried in shared memory
BIG_SEED = 404    # a walk with a chain of eight residual rounds over one direction
SHARDED_SEEDS = [(1001, 601), (40961, 602), (40961, 603)]


@pytest.fixture(scope="module")
def ctx():
    from spark_ensemble_b200.context import Context
    c = Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def oracle():
    from oracle import oracle as O
    return O.Oracle()


def _steps(seed):
    return 40 + seed % 41


def run(ctx, oracle, ops, seed, reads="drawn", options=None):
    w = W.Walker(ctx, reads=reads, options=options, oracle=oracle, seed=seed).run(ops)
    if reads == "drawn":
        w.observe("full")
    return w


def _same_bits(a, b, what, keys=None):
    """Every observation of walk `a` (or those in `keys`) equals the one of `b` at the same step bit for bit."""
    ib = {(s, k): v for s, k, v in b.observed}
    for s, k, v in a.observed:
        if keys is not None and not keys(k):
            continue
        assert (s, k) in ib, f"{what}: {k} at step {s} missing"
        if not np.array_equal(v, ib[(s, k)], equal_nan=True):
            bad = np.flatnonzero(~((v == ib[(s, k)]) | (np.isnan(v) & np.isnan(ib[(s, k)]))))
            raise AssertionError(f"{what}: {k} at step {s} (call {a.log[s - 1] if s else None}) differs in "
                                 f"{bad.size} values, first at {bad[0]}: {v.reshape(-1)[bad[0]]!r} vs "
                                 f"{ib[(s, k)].reshape(-1)[bad[0]]!r}")


def _drawn(what):
    """What walk A read that C read too: everything but A's final reads of F, H, VF, VH and WOUT."""
    return not what.startswith("obs:") or what == "obs:R"


@pytest.mark.parametrize("n,seed", SEEDS)
def test_walk_against_the_model(ctx, oracle, n, seed):
    ops = W.generate(seed, n, _steps(seed), sizes=SIZES if seed % 2 else None)
    a = run(ctx, oracle, ops, seed, "drawn")
    run(ctx, oracle, ops, seed, "full")
    c = run(ctx, oracle, ops, seed, "r")
    _same_bits(a, c, f"seed {seed}: reads of R changed what the walk computed", _drawn)


@pytest.mark.parametrize("n,seed", SEEDS[::2])
def test_bit_identical_settings(ctx, oracle, n, seed):
    """Walks drawn from their own seeds: the walks above flip the settings compared here, so they cannot be rerun
    with one of them held.  The generator is the same, with the flips of those four settings left out."""
    pinned = tuple(W.BIT_IDENTICAL)
    ops = W.generate(seed + 5000, n, _steps(seed), pinned=pinned)
    base = run(ctx, oracle, ops, seed + 5000)
    for key, val in W.BIT_IDENTICAL.items():
        other = run(ctx, oracle, ops, seed + 5000, options={key: val})
        _same_bits(base, other, f"seed {seed + 5000}: {key}={val}")
        _same_bits(other, base, f"seed {seed + 5000}: {key}={val}")


def test_walk_at_ten_million_rows(ctx, oracle):
    """The one walk whose carried rounds hold part of each CTA's tiles in shared memory: it never flips the settings
    documented as bit-identical, so that it can be rerun with sq_defer_max 0 and with fused_resident 0."""
    ops = W.generate(BIG_SEED, BIG, 30, pinned=tuple(W.BIT_IDENTICAL), losses=("squared",))
    a = run(ctx, oracle, ops, BIG_SEED, "drawn")
    assert any(carried and tiles > 0 for carried, tiles, _ in a.rounds), a.rounds
    assert any(deferred for _, _, deferred in a.rounds), a.rounds
    run(ctx, oracle, ops, BIG_SEED, "full")
    c = run(ctx, oracle, ops, BIG_SEED, "r")
    _same_bits(a, c, f"seed {BIG_SEED}: reads of R changed what the walk computed", _drawn)
    for key in ("sq_defer_max", "fused_resident"):
        other = run(ctx, oracle, ops, BIG_SEED, options={key: W.BIT_IDENTICAL[key]})
        assert not any(d for _, _, d in other.rounds) if key == "sq_defer_max" else \
            not any(t for _, t, _ in other.rounds), other.rounds
        _same_bits(a, other, f"seed {BIG_SEED}: {key}={W.BIT_IDENTICAL[key]}")
        _same_bits(other, a, f"seed {BIG_SEED}: {key}={W.BIT_IDENTICAL[key]}")


# ---- regression walks: the shortest walks that showed a broken rule
def _start(loss="squared", n=1001):
    s = 77
    return [{"op": "configure", "n": n, "nv": 0, "loss": loss, "param": 0.5, "has_w": False}, {"op": "features"},
            {"op": "upload", "slot": "Y", "kind": "label" if loss == "bernoulli" else "normal", "seed": s,
             "offset": 0, "count": n, "f64": False},
            {"op": "upload", "slot": "F", "kind": "normal", "seed": s + 1, "offset": 0, "count": n, "f64": False},
            {"op": "upload", "slot": "H", "kind": "dir", "seed": s + 2, "offset": 0, "count": n, "f64": False}]


REGRESSIONS = {
    # a one-launch residual round that fails MaxEval over a residual slot that is not current must not replace R with
    # y - F: the failed round leaves F and R as they were
    "failed_round_keeps_a_stale_r": _start() + [
        {"op": "resid", "newton": False}, {"op": "round", "lr": W.LR, "residual": False},
        {"op": "fail_maxeval", "residual": True}, {"op": "read", "what": "R"}],
    # a gradient-mode pseudo-residual call does not write WOUT, so it must not drop the 1/S its download applies
    "gradient_residuals_keep_wout_scaled": _start("bernoulli") + [
        {"op": "resid", "newton": True}, {"op": "resid", "newton": False}, {"op": "read", "what": "WOUT"}],
    # a write of WOUT drops the 1/S a download applies to the Newton weights it replaced
    "wout_write_drops_the_scale": _start("bernoulli") + [
        {"op": "resid", "newton": True},
        {"op": "upload", "slot": "WOUT", "kind": "weight", "seed": 5, "offset": 10, "count": 20, "f64": False},
        {"op": "read", "what": "WOUT"}],
    # carried rounds over one direction with a small cap: the chain is stored once it holds sq_defer_max steps
    "defer_cap": _start() + [{"op": "opt", "key": "sq_defer_max", "value": 1}, {"op": "resid", "newton": False}] +
    [{"op": "round", "lr": W.LR, "residual": True}] * 5 + [{"op": "read", "what": "R"}],
}


@pytest.mark.parametrize("name", sorted(REGRESSIONS))
def test_regression_walk(ctx, oracle, name):
    run(ctx, oracle, REGRESSIONS[name], name, "drawn")


# ---- walks over row-sharded GPUs: the calls ShardedContext exposes, the model over the union of the rows
@pytest.fixture(scope="module")
def sharded():
    from spark_ensemble_b200 import _native as N
    if N.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from spark_ensemble_b200.sharded import ShardedContext
    sc = ShardedContext([0, 1])
    yield sc
    sc.close()


@pytest.mark.parametrize("n,seed", SHARDED_SEEDS)
def test_sharded_walk(sharded, oracle, n, seed):
    ops = W.generate(seed, n, _steps(seed), sizes=(1001, 40961), sharded=True)
    a = run(sharded, oracle, ops, seed, "drawn")
    run(sharded, oracle, ops, seed, "full")
    c = run(sharded, oracle, ops, seed, "r")
    _same_bits(a, c, f"sharded seed {seed}: reads of R changed what the walk computed", _drawn)


def test_sharded_failed_round(sharded, oracle):
    """Every shard's R and F stay as they were when the one-launch round fails MaxEval: over a stale R, and in the
    middle of a chain of carried rounds."""
    ops = REGRESSIONS["failed_round_keeps_a_stale_r"] + [{"op": "resid", "newton": False}] + \
        [{"op": "round", "lr": W.LR, "residual": True}] * 4 + \
        [{"op": "fail_maxeval", "residual": True}, {"op": "round", "lr": W.LR, "residual": True},
         {"op": "read", "what": "R"}, {"op": "read", "what": "F"}]
    for reads in ("drawn", "full"):
        run(sharded, oracle, ops, "sharded_failed_round", reads)
