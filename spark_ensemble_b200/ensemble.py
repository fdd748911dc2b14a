"""Host-side pieces shared by the ensemble mirrors: the columnar DataFrame stand-in, sub-bagging
(ensemble/HasSubBag.scala:73-84 with Spark's XORShiftRandom restated), the row partitioner used for
multi-GPU sharding, and the Dummy init models (regression/DummyRegressor.scala:113-129,
classification/DummyClassifier.scala:90-123).  Nothing here touches per-row numerics of the hot path.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native as N


# ---- a minimal columnar stand-in for a Spark DataFrame ----------------------------------------------
class DataFrame:
    """Columns are numpy arrays with a common leading dimension (features: [n, d])."""

    def __init__(self, **columns):
        self._cols = {}
        n = None
        for k, v in columns.items():
            a = np.asarray(v)
            if n is None:
                n = a.shape[0]
            if a.shape[0] != n:
                raise ValueError(f"column {k} has {a.shape[0]} rows, expected {n}")
            self._cols[k] = a
        self._n = n or 0

    @property
    def columns(self):
        return list(self._cols)

    def count(self) -> int:
        return self._n

    def __contains__(self, name):
        return name in self._cols

    def __getitem__(self, name) -> np.ndarray:
        if name not in self._cols:
            raise KeyError(f"column {name} does not exist; available: {self.columns}")
        return self._cols[name]

    def withColumn(self, name, values) -> "DataFrame":
        cols = dict(self._cols)
        cols[name] = np.asarray(values)
        return DataFrame(**cols)

    def filter(self, mask) -> "DataFrame":
        mask = np.asarray(mask, dtype=bool)
        return DataFrame(**{k: v[mask] for k, v in self._cols.items()})


def java_string_hash(s: str) -> int:
    """java.lang.String.hashCode (Spark HasSeed default = class name hash)."""
    h = 0
    for ch in s:
        h = (31 * h + ord(ch)) & 0xFFFFFFFF
    return h - (1 << 32) if h & 0x80000000 else h


# ---- Spark XORShiftRandom (org.apache.spark.util.random.XORShiftRandom, Spark 3.3.1; not vendored) ---
def _rotl32(x, r):
    return ((x << r) | (x >> (32 - r))) & 0xFFFFFFFF


def _murmur3_bytes_hash(data: bytes, seed: int) -> int:
    """scala.util.hashing.MurmurHash3.bytesHash."""
    def mix_last(h, k):
        k = (k * 0xCC9E2D51) & 0xFFFFFFFF
        k = _rotl32(k, 15)
        k = (k * 0x1B873593) & 0xFFFFFFFF
        return h ^ k

    def mix(h, k):
        h = mix_last(h, k)
        h = _rotl32(h, 13)
        return (h * 5 + 0xE6546B64) & 0xFFFFFFFF

    h = seed & 0xFFFFFFFF
    n = len(data)
    i = 0
    while n - i >= 4:
        k = data[i] | (data[i + 1] << 8) | (data[i + 2] << 16) | (data[i + 3] << 24)
        h = mix(h, k)
        i += 4
    rem = n - i
    k = 0
    if rem == 3:
        k ^= data[i + 2] << 16
    if rem >= 2:
        k ^= data[i + 1] << 8
    if rem >= 1:
        k ^= data[i]
        h = mix_last(h, k)
    h ^= n
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & 0xFFFFFFFF
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & 0xFFFFFFFF
    h ^= h >> 16
    return h


class XORShiftRandom:
    _MASK = (1 << 64) - 1

    def __init__(self, init: int):
        b = (init & self._MASK).to_bytes(8, "big")  # ByteBuffer.putLong: big endian
        low = _murmur3_bytes_hash(b, 0x3C074A61)    # MurmurHash3.arraySeed
        high = _murmur3_bytes_hash(b, low)
        self.seed = ((high << 32) | low) & self._MASK

    def _next(self, bits: int) -> int:
        s = self.seed
        s ^= (s << 21) & self._MASK
        s ^= s >> 35
        s ^= (s << 4) & self._MASK
        self.seed = s
        return s & ((1 << bits) - 1)

    def next_double(self) -> float:
        """java.util.Random.nextDouble over the overridden next(bits)."""
        return ((self._next(26) << 27) + self._next(27)) * (1.0 / (1 << 53))


def subspace(subspace_ratio: float, num_features: int, seed: int) -> np.ndarray:
    """ensemble/HasSubBag.scala:73-79: keep feature j iff rng.nextDouble() < subspaceRatio."""
    rng = XORShiftRandom(seed)
    return np.array([j for j in range(num_features) if rng.next_double() < subspace_ratio], dtype=np.int32)


def spark_bernoulli_sample(n: int, fraction: float, seed: int) -> np.ndarray:
    """Multiplicity (0 or 1, fp32) of each of n rows in `RDD.sample(false, fraction, seed)` over ONE partition: Spark's
    own algorithm (java.util.Random -> per-partition seed -> XORShiftRandom -> BernoulliSampler with gap sampling below
    0.4), restated in the native library (se_spark_bernoulli_sample, host only)."""
    c = np.zeros(n, dtype=np.float32)
    s64 = int(seed) & 0xFFFFFFFFFFFFFFFF  # the Scala Long seed
    s64 = s64 - (1 << 64) if s64 >= (1 << 63) else s64
    N.check(N.load().se_spark_bernoulli_sample(C.c_int64(s64), float(fraction), n, 0, N.fptr(c)))
    return c


def slice_features(indices: np.ndarray, X: np.ndarray) -> np.ndarray:
    """ensemble/HasSubBag.scala:81-84 (dense case): features(indices)."""
    return X[:, indices]


# ---- row partitioner for multi-GPU sharding (SURVEY.md §8e) -----------------------------------------
def row_partition(n_rows: int, n_shards: int, shard: int, align: int = 4) -> tuple[int, int]:
    """Contiguous row blocks [start, stop) per shard; block size rounded up to a multiple of `align`
    rows so 128-bit loads stay aligned on every shard. Trailing shards may be short or empty."""
    if not (0 <= shard < n_shards):
        raise ValueError(f"shard {shard} outside [0,{n_shards})")
    per = -(-n_rows // n_shards)
    per = -(-per // align) * align
    start = min(n_rows, shard * per)
    stop = min(n_rows, start + per)
    return start, stop


# ---- Dummy init models -----------------------------------------------------------------------------
class DummyRegressionModel:
    """regression/DummyRegressor.scala: constant prediction."""

    def __init__(self, prediction: float):
        self.prediction = float(prediction)

    def predict(self, X) -> np.ndarray:
        return np.full(np.asarray(X).shape[0], self.prediction, dtype=np.float64)


def fit_dummy_regressor(strategy: str, labels: np.ndarray, constant: float = 0.0, quantile: float = 0.5):
    """DummyRegressor.train :113-129. mean = unweighted label mean; median/quantile use Spark's
    approxQuantile (Greenwald-Khanna, relative error tol) — restated here as the exact lower empirical
    quantile, which is what approxQuantile returns for tol -> 0 (rank ceil(q*n))."""
    y = np.asarray(labels, dtype=np.float64)
    if strategy == "mean":
        return DummyRegressionModel(float(np.mean(y)))
    if strategy in ("median", "quantile"):
        q = 0.5 if strategy == "median" else quantile
        return DummyRegressionModel(exact_quantile(y, q))
    if strategy == "constant":
        return DummyRegressionModel(constant)
    raise ValueError(f"unknown strategy {strategy}")


def exact_quantile(values: np.ndarray, q: float) -> float:
    s = np.sort(np.asarray(values, dtype=np.float64))
    if s.size == 0:
        return float("nan")
    rank = int(np.ceil(q * s.size))
    return float(s[min(max(rank - 1, 0), s.size - 1)])


class DummyClassificationModel:
    """classification/DummyClassifier.scala:130-175: constant rawPrediction / probability."""

    def __init__(self, num_classes: int, raw_prediction, probability):
        self.numClasses = num_classes
        self.rawPrediction = np.asarray(raw_prediction, dtype=np.float64)
        self.probability = np.asarray(probability, dtype=np.float64)

    def predictRaw(self, X) -> np.ndarray:
        return np.tile(self.rawPrediction, (np.asarray(X).shape[0], 1))


def fit_dummy_classifier(strategy: str, labels: np.ndarray, num_classes: int):
    """DummyClassifier.train :90-123."""
    if strategy == "uniform":
        return DummyClassificationModel(num_classes, np.zeros(num_classes), np.full(num_classes, 1.0 / num_classes))
    if strategy == "prior":
        y = np.asarray(labels).astype(np.int64)
        present = np.unique(y)
        pri = np.array([np.sum(y == c) / float(y.size) for c in present])  # only observed labels, sorted
        return DummyClassificationModel(num_classes, np.log(pri), pri)
    raise ValueError(f"unknown strategy {strategy}")
