"""Known-answer vectors of the third-party pieces the oracle (and the product's host side) restate — commons-math3
BrentOptimizer, Spark's ml.impl.Utils (log1pExp / softmax / EPSILON), MurmurHash3 + XORShiftRandom — from their
PUBLISHED test suites / tables (tests/golden/thirdparty_*.json hold the citations; make_thirdparty_golden.py
re-derives every expectation).  This is what moves the oracle from "pinned by properties" to "pinned by published
vectors" for the pieces whose source is not part of the reference repository."""
import ctypes
import json
import math
import os

import numpy as np
import pytest

from oracle import np_oracle as NP
from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
FUNCS = {"sin": math.sin, "quintic": lambda x: (x - 1) * (x - 0.5) * x * (x + 0.5) * (x + 1),
         "math832": lambda x: 1e2 * math.sqrt(x) + 1e6 / x + 1e4 / math.sqrt(x)}


def _golden(name):
    return json.load(open(os.path.join(HERE, "golden", name)))


@pytest.fixture(scope="module")
def lib():
    from spark_ensemble_b200 import _native, build
    build.build()
    return _native.load()


def _product_brent(lib, fn, lo, hi, start, rel, abs_tol, max_eval):
    from spark_ensemble_b200 import _native as N
    cb = N.FN1(lambda x, _u: float(fn(x)))
    x, f, ne = ctypes.c_double(), ctypes.c_double(), ctypes.c_int()
    rc = lib.se_brent_minimize(cb, None, lo, hi, start, rel, abs_tol, max_eval, ctypes.byref(x), ctypes.byref(f),
                               ctypes.byref(ne))
    return rc, x.value, ne.value


@pytest.mark.parametrize("case", _golden("thirdparty_brent.json")["cases"], ids=lambda c: c["name"])
def test_brent_restatements_meet_the_published_commons_math_expectations(lib, oracle, case):
    """Both Brent restatements — the oracle's C (oracle/se_oracle.c) and the product's host/device template
    (csrc/se_brent.h; the device instantiation is tied to the host one bit for bit by the GPU tests) — must satisfy
    what BrentOptimizerTest asserts for the original, and agree with each other evaluation for evaluation."""
    fn = FUNCS[case["f"]]
    start = 0.5 * (case["lo"] + case["hi"])  # SearchInterval(lo, hi): commons-math starts at the midpoint
    rc, xp, nep = _product_brent(lib, fn, case["lo"], case["hi"], start, case["rel"], case["abs"], case["max_eval"])
    xo, neo, st = oracle.brent(fn, case["lo"], case["hi"], start, case["rel"], case["abs"], case["max_eval"])
    assert rc == 0 and st == 0
    assert abs(xp - case["expected"]) <= case["tol"], (xp, case["expected"])
    assert abs(xo - case["expected"]) <= case["tol"], (xo, case["expected"])
    assert nep <= case["max_evaluations_asserted"] and neo <= case["max_evaluations_asserted"]
    assert (xp, nep) == (xo, neo)


def test_spark_log1pexp_softmax_epsilon(oracle):
    g = _golden("thirdparty_spark_utils.json")
    for v in g["log1pExp"]:
        x = v["x"]
        # BernoulliLoss.loss(label 1 -> y~ = +1, prediction p) = log1pExp(-2 p)  (GBMLoss.scala:297-301)
        got_c = oracle.loss(O.BERNOULLI, 0.0, 1.0, -0.5 * x)
        got_np = float(NP.log1p_exp(np.array([x]))[0]) if hasattr(NP, "log1p_exp") else got_c
        for got in (got_c, got_np):
            if v["kind"] == "rel":
                assert abs(got - v["expected"]) <= v["tol"] * abs(v["expected"]), (x, got, v["expected"])
            else:
                assert abs(got - v["expected"]) <= v["tol"], (x, got, v["expected"])
    assert NP.EPS == g["epsilon"]["expected"]
    eps = 1.0
    while (1.0 + (eps / 2.0)) != 1.0:
        eps /= 2.0
    assert eps == g["epsilon"]["expected"]
    # SAMME.R clamps probabilities at EPSILON (BoostingClassifier.scala:215-228): a zero probability behaves like EPSILON
    K, y, w = 2, np.array([0.0]), np.array([1.0])
    out0, _, _ = oracle.samme_r_update(K, y, w, 1.0, np.array([[0.0], [1.0]]))
    oute, _, _ = oracle.samme_r_update(K, y, w, 1.0, np.array([[g["epsilon"]["expected"]], [1.0]]))
    assert out0[0] == oute[0]
    for v in g["softmax"]:
        raw = np.array(v["x"], dtype=np.float64).reshape(-1, 1)
        np.testing.assert_allclose(oracle.gbm_raw2prob(O.LOGLOSS, raw)[:, 0], v["expected"], rtol=1e-14, atol=0)
        np.testing.assert_allclose(NP.softmax_cols(raw)[:, 0], v["expected"], rtol=1e-14, atol=0)


def test_murmur3_published_vectors_and_xorshift_properties():
    from spark_ensemble_b200.ensemble import XORShiftRandom, _murmur3_bytes_hash
    g = _golden("thirdparty_murmur3.json")
    for v in g["vectors"]:
        assert _murmur3_bytes_hash(v["data"].encode(), v["seed"]) == v["expected"], v
    # Spark XORShiftRandomSuite: "XORShift with zero seed" and "hashSeed has random bits throughout"
    assert XORShiftRandom(0)._next(32) != 0
    total = 0
    for seed in range(10):
        bits = bin(XORShiftRandom(seed).seed).count("1")
        assert bits > 20, (seed, bits)
        total += bits
    assert total > 64 * 10 * 0.4
    # "XORShift generates valid random numbers": uniformity of nextDouble (chi-square over 10 bins, 100k draws)
    r = XORShiftRandom(12345)
    draws = np.array([r.next_double() for _ in range(100_000)])
    assert 0.0 <= draws.min() and draws.max() < 1.0
    counts = np.histogram(draws, bins=10, range=(0, 1))[0]
    chi2 = float(((counts - 10_000) ** 2 / 10_000).sum())
    assert chi2 < 27.88  # 99.9 % quantile of chi-square with 9 degrees of freedom


def test_spark_bernoulli_sampler_restatement(lib):
    """se_spark_bernoulli_sample (host-only) = java.util.Random -> per-partition seed -> XORShiftRandom ->
    BernoulliSampler.  Pinned pieces: java.util.Random by its specification (new Random(42).nextInt() == -1170105035 is
    the value the Java documentation's LCG gives; checked through the Python restatement below), XORShift / MurmurHash3
    by the vectors above; the sampler logic (gap sampling below 0.4, `nextDouble() <= fraction` above) is restated from
    the Spark 3.3.1 sources and only checked for self-consistency and its statistical contract here."""
    import ctypes as C
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.ensemble import XORShiftRandom

    class JavaRandom:  # java.util.Random as specified in the Java SE API documentation
        def __init__(self, seed):
            self.s = (seed ^ 0x5DEECE66D) & ((1 << 48) - 1)

        def next(self, bits):
            self.s = (self.s * 0x5DEECE66D + 0xB) & ((1 << 48) - 1)
            v = self.s >> (48 - bits)
            return v - (1 << bits) if v >= (1 << (bits - 1)) else v

        def next_long(self):
            return ((self.next(32) << 32) + self.next(32) + (1 << 63)) % (1 << 64) - (1 << 63)

    assert JavaRandom(42).next(32) == -1170105035          # widely published first nextInt() of new Random(42)
    assert JavaRandom(42).next_long() == -5025562857975149833

    def native(seed, fraction, n, part=0):
        c = np.zeros(n, dtype=np.float32)
        assert lib.se_spark_bernoulli_sample(C.c_int64(seed), fraction, n, part, N.fptr(c)) == 0
        return c

    n = 20000
    for seed, part in ((42, 0), (-7, 0), (123456789012345, 2)):
        jr = JavaRandom(seed)
        for _ in range(part + 1):
            pseed = jr.next_long()
        # fraction > 0.4: one draw per row, keep iff nextDouble() <= fraction
        rng = XORShiftRandom(pseed)
        want = np.array([1.0 if rng.next_double() <= 0.7 else 0.0 for _ in range(n)], dtype=np.float32)
        np.testing.assert_array_equal(native(seed, 0.7, n, part), want)
        # fraction <= 0.4: gap sampling
        rng = XORShiftRandom(pseed)
        lnq = math.log1p(-0.25)
        adv = lambda: int(math.log(max(rng.next_double(), 5e-11)) / lnq)
        drop, want = adv(), []
        for _ in range(n):
            if drop > 0:
                drop -= 1; want.append(0.0)
            else:
                drop = adv(); want.append(1.0)
        np.testing.assert_array_equal(native(seed, 0.25, n, part), np.array(want, dtype=np.float32))
    # statistical contract of RDD.sample: E[kept] = fraction * n
    for f in (0.1, 0.25, 0.5, 0.9):
        kept = native(2024, f, 200_000).mean()
        assert abs(kept - f) < 4 * math.sqrt(f * (1 - f) / 200_000)
    assert native(1, 1.0, 10).sum() == 10 and native(1, 0.0, 10).sum() == 0
    # the same seed draws the same bag every time (the reference reuses one seed per fit: quirk 3)
    np.testing.assert_array_equal(native(9, 0.6, 1000), native(9, 0.6, 1000))
