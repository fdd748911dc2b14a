"""CPU tests of the host-side mirror logic (no GPU, no kernels): Params surface, sub-bagging,
row partitioner, and the world_size-2 gloo check of the sharded-reduction algebra (SURVEY.md §8e)."""
import os

import numpy as np
import pytest


def test_uid_prefixes_and_defaults_match_reference():
    """SURVEY.md §5: UID prefixes and Param defaults are part of the drop-in surface."""
    from spark_ensemble_b200.classification import (BaggingClassifier, BoostingClassifier, GBMClassifier)
    from spark_ensemble_b200.regression import BaggingRegressor, GBMRegressor
    g = GBMRegressor()
    assert g.uid.startswith("GBMRegressor2_") and len(g.uid) == len("GBMRegressor2_") + 12  # sic, :229
    d = g.extractParamMap()
    assert (d["numBaseLearners"], d["learningRate"], d["optimizedWeights"], d["updates"]) == (10, 1.0, True, "gradient")
    assert (d["tol"], d["maxIter"], d["numRounds"], d["validationTol"], d["replacement"]) == (1e-6, 100, 1, 0.01, False)
    assert (d["loss"], d["alpha"], d["initStrategy"]) == ("squared", 0.9, "constant")
    assert (d["subsampleRatio"], d["subspaceRatio"], d["checkpointInterval"], d["aggregationDepth"]) == (1.0, 1.0, 10, 2)
    c = GBMClassifier()
    assert c.uid.startswith("GBMClassifier_")
    assert (c.getLoss(), c.getInitStrategy(), c.getParallelism()) == ("logloss", "prior", 1)
    b = BoostingClassifier()
    assert b.uid.startswith("BoostingClassifier_") and b.getAlgorithm() == "discrete"
    assert BaggingRegressor().uid.startswith("BaggingRegressor_")
    bc = BaggingClassifier()
    assert bc.uid.startswith("BaggingClassifier_") and bc.getVotingStrategy() == "hard" and bc.getReplacement() is True


def test_param_validators_raise_like_spark():
    from spark_ensemble_b200.regression import GBMRegressor
    g = GBMRegressor()
    for name, bad in [("learningRate", 0.0), ("numBaseLearners", 0), ("loss", "poisson"), ("updates", "adam"),
                      ("subspaceRatio", 1.5), ("numRounds", 0), ("validationTol", -1.0), ("initStrategy", "mean")]:
        with pytest.raises(ValueError):
            g.set(name, bad)
    assert g.setLoss("Huber").getLoss() == "Huber" and g.setUpdates("Newton")("updates") == "Newton"
    g2 = g.copy({"learningRate": 0.3})
    assert g2.getLearningRate() == 0.3 and g.getLearningRate() == 1.0 and g2.uid == g.uid
    assert "learningRate" in g.explainParams()


def test_java_string_hash_and_default_seed():
    from spark_ensemble_b200.ensemble import java_string_hash
    assert java_string_hash("hello") == 99162322
    assert java_string_hash("") == 0
    assert java_string_hash("org.apache.spark.ml.regression.GBMRegressor") == 1243996765


def test_subspace_properties():
    """test/ensemble/HasSubBagSuite.scala:60-105: E|subspace| = ratio*d +- 0.1*d, sorted, ratio 1 => identity."""
    from spark_ensemble_b200.ensemble import XORShiftRandom, subspace
    d = 200
    for ratio in (0.1, 0.5, 0.9):
        sizes = [len(subspace(ratio, d, seed)) for seed in range(40)]
        assert abs(np.mean(sizes) / d - ratio) < 0.1
        s = subspace(ratio, d, 7)
        assert list(s) == sorted(set(s)) and s.dtype == np.int32
    np.testing.assert_array_equal(subspace(1.0, 17, 123), np.arange(17))
    assert len(subspace(0.0, 17, 123)) == 0
    # determinism + hashSeed bit spread (XORShiftRandomSuite "hashSeed has random bits throughout")
    assert list(subspace(0.5, 50, 42)) == list(subspace(0.5, 50, 42))
    assert list(subspace(0.5, 50, 42)) != list(subspace(0.5, 50, 43))
    for seed in range(10):
        r = XORShiftRandom(seed)
        assert bin(r.seed).count("1") > 20
        u = [r.next_double() for _ in range(1000)]
        assert 0.0 <= min(u) and max(u) < 1.0 and abs(np.mean(u) - 0.5) < 0.05


def test_row_partition_covers_rows_aligned():
    from spark_ensemble_b200.ensemble import row_partition
    for n in (0, 1, 5, 8192, 100_000_003):
        for g in (1, 2, 3, 8):
            spans = [row_partition(n, g, r) for r in range(g)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            for (a0, a1), (b0, b1) in zip(spans, spans[1:]):
                assert a1 == b0 and a0 <= a1
            assert all(s0 % 4 == 0 for s0, s1 in spans if s1 > s0)  # 128-bit alignment of non-empty shards
    with pytest.raises(ValueError):
        row_partition(10, 2, 2)


def test_dummy_init_models():
    """DummyRegressorSuite.scala:78-108 / DummyClassifier.train :90-123."""
    from spark_ensemble_b200.ensemble import exact_quantile, fit_dummy_classifier, fit_dummy_regressor
    y = np.array([3.0, 1.0, 2.0, 10.0])
    assert fit_dummy_regressor("mean", y).prediction == 4.0
    assert fit_dummy_regressor("median", y).prediction == 2.0
    assert fit_dummy_regressor("quantile", y, quantile=0.9).prediction == 10.0
    assert fit_dummy_regressor("constant", y, constant=0.0).prediction == 0.0
    assert exact_quantile(np.arange(1, 101), 0.9) == 90.0
    labels = np.array([0, 0, 1, 2, 2, 2], dtype=float)
    m = fit_dummy_classifier("prior", labels, 3)
    np.testing.assert_allclose(m.probability, [2 / 6, 1 / 6, 3 / 6])
    np.testing.assert_allclose(m.rawPrediction, np.log([2 / 6, 1 / 6, 3 / 6]))
    u = fit_dummy_classifier("uniform", labels, 3)
    np.testing.assert_allclose(u.rawPrediction, 0.0)
    assert u.predictRaw(np.zeros((4, 2))).shape == (4, 3)


def test_bag_counts_same_every_round():
    """Reference quirk 3: RDD.sample gets the same seed every round => one bag per fit."""
    from spark_ensemble_b200.routes import bag_counts
    assert bag_counts(100, 1.0, False, 7) is None
    a, b = bag_counts(10000, 0.6, False, 7), bag_counts(10000, 0.6, False, 7)
    np.testing.assert_array_equal(a, b)
    assert set(np.unique(a)) <= {0.0, 1.0} and abs(a.mean() - 0.6) < 0.03
    c = bag_counts(10000, 1.0, True, 7)
    assert c.max() >= 2 and abs(c.mean() - 1.0) < 0.05  # Poisson(1) bootstrap


def test_tree_arrays_threshold_rounding():
    """fp32 thresholds are rounded DOWN so `x <= thr32` equals sklearn's `x <= thr64` for fp32 x."""
    from spark_ensemble_b200.learners import DecisionTreeRegressor
    rng = np.random.default_rng(3)
    X = rng.standard_normal((2000, 5)).astype(np.float32)
    y = X[:, 0] + X[:, 1] ** 2
    m = DecisionTreeRegressor(maxDepth=7).fit(X, y)
    t = m.tree_arrays()
    node = np.zeros(len(X), dtype=np.int64)
    for _ in range(10):
        f = t["feature"][node]
        live = f >= 0
        x = X[np.arange(len(X)), np.maximum(f, 0)]
        nxt = np.where(x <= t["threshold"][node], t["left"][node], t["right"][node])
        node = np.where(live, nxt, node)
    np.testing.assert_allclose(t["value"][node], m.predict(X), rtol=1e-6)


def _gloo_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    from oracle import oracle as O
    from spark_ensemble_b200.ensemble import row_partition
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    orc = O.Oracle()
    rng = np.random.default_rng(5)  # every rank regenerates the same global dataset
    n, K = 10_007, 3
    res = {}
    for name, dim in (("bernoulli", 1), ("logloss", K), ("squared", 1)):
        y = (rng.integers(0, K, n) if name == "logloss" else (rng.random(n) < 0.5)).astype(np.float64)
        if name == "squared":
            y = rng.standard_normal(n)
        w = rng.random(n) + 0.5
        F = rng.standard_normal((dim, n))
        h = rng.standard_normal((dim, n))
        alpha = rng.random(dim) + 0.5
        s0, s1 = row_partition(n, world, rank)
        lid = O.LOSS_IDS[name]
        # per-shard partial sums exactly as a GPU shard produces them: (lossSum, weightSum, gradSum[dim])
        l, g = orc.linesearch_eval(lid, 0.0, y[s0:s1], w[s0:s1], np.ascontiguousarray(F[:, s0:s1]),
                                   np.ascontiguousarray(h[:, s0:s1]), alpha)
        ws = float(np.sum(w[s0:s1]))
        part = torch.tensor([l * ws, ws] + list(g * ws), dtype=torch.float64)
        dist.all_reduce(part)  # the ONE collective of a boosting round
        tot = part.numpy()
        full_l, full_g = orc.linesearch_eval(lid, 0.0, y, w, F, h, alpha)
        res[name] = (abs(tot[0] / tot[1] - full_l) / abs(full_l),
                     float(np.max(np.abs(tot[2:] / tot[1] - full_g) / (np.abs(full_g) + 1e-12))))
    dist.barrier()
    dist.destroy_process_group()
    q.put((rank, res))


def test_sharded_reduction_world2_gloo():
    """Rows shard contiguously; the only exchange is a sum-allreduce of dim+2 doubles: the combined result
    equals the unsharded aggregator (what se_comm_* does over NCCL on GPUs)."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for _, res in out:
        for name, (el, eg) in res.items():
            assert el < 1e-12 and eg < 1e-9, (name, el, eg)


def test_bench_reference_arm_json_contract():
    """`bench.py --impl reference` (the CPU arm: oracle port on the host cores) prints one JSON line with the
    contract's keys; runs without a GPU."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1",
                          "--warmup", "0", "--cpu-rows", "20000"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    d = json.loads(out.stdout.strip().splitlines()[-1])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
              "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["unit"] == "rows/s" and d["value"] > 0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert "workload" in d["config"] and d["vs_baseline"] is None


def test_no_product_module_imports_the_oracle():
    """The oracle is test infrastructure: nothing under spark_ensemble_b200/ may import it."""
    import re
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "spark_ensemble_b200")
    for dirpath, _, files in os.walk(root):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                src = open(os.path.join(dirpath, f), errors="replace").read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
                assert "se_oracle.h" not in src and "liboracle" not in src, f


def test_libsvm_reader_blocks_and_errors(tmp_path):
    """LIBSVM text -> dense fp32 row blocks (1-based ascending indices, comments, blank lines, ragged tail block)."""
    from spark_ensemble_b200.io import count_libsvm_rows, iter_libsvm_dense
    rng = np.random.default_rng(3)
    n, d = 23, 7
    X = np.where(rng.random((n, d)) < 0.5, rng.standard_normal((n, d)), 0.0).astype(np.float32)
    y = rng.standard_normal(n)
    p = tmp_path / "a.svm"
    with open(p, "w") as fh:
        fh.write("# header comment\n\n")
        for i in range(n):
            feats = " ".join(f"{j + 1}:{float(X[i, j])!r}" for j in range(d) if X[i, j] != 0.0)
            fh.write(f"{float(y[i])!r} {feats}  # row {i}\n")
    assert count_libsvm_rows(str(p)) == n
    blocks = list(iter_libsvm_dense(str(p), d, block_rows=10))
    assert [len(b[1]) for b in blocks] == [10, 10, 3]
    np.testing.assert_array_equal(np.concatenate([b[0] for b in blocks]), X)
    np.testing.assert_array_equal(np.concatenate([b[1] for b in blocks]), y)
    bad = tmp_path / "b.svm"
    bad.write_text("1.0 3:1.0 2:2.0\n")
    with pytest.raises(ValueError, match="ascending"):
        list(iter_libsvm_dense(str(bad), d))
    bad.write_text("1.0 9:1.0\n")
    with pytest.raises(ValueError, match="outside"):
        list(iter_libsvm_dense(str(bad), d))


# ------------------------------------------------------------------ JNI / Scala boundary (generated from one table)
def _jni_gen():
    import importlib.util
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("gen_jni", os.path.join(root, "jni", "gen_jni.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m, root


def test_jni_shim_scala_natives_and_abi_header_agree():
    """JNI symbol list == Scala @native list == the generator's table, and every function se_abi.h declares is either
    bound or listed (with a reason) as deliberately not bound."""
    import os
    import re
    g, root = _jni_gen()
    cpp, scala = g.generate()
    assert open(os.path.join(root, "jni", "se_jni.cpp")).read() == cpp, "jni/se_jni.cpp is stale: python jni/gen_jni.py"
    sp = os.path.join(root, "scala", "org", "apache", "spark", "ml", "se", "SeNative.scala")
    assert open(sp).read() == scala, "SeNative.scala is stale: python jni/gen_jni.py"
    jni_syms = re.findall(r"^SE_JNI\(\w+, (\w+)\)", cpp, flags=re.M)
    natives = re.findall(r"@native def (\w+)\(", scala)
    assert sorted(jni_syms) == sorted(natives) == sorted(g.native_names())
    assert len(set(natives)) == len(natives)
    declared = set(re.findall(r"^SE_API\s+[\w\s\*]+?\b(se_\w+)\(", open(os.path.join(root, "include", "se_abi.h")).read(), flags=re.M))
    bound = g.bound_abi()
    assert bound <= declared, bound - declared
    assert declared - bound == set(g.NOT_BOUND), (declared - bound, set(g.NOT_BOUND))
    # the entry points bench.py times are bound (VERDICT r1: se_gbm_round was not)
    for must in ("se_gbm_round", "se_upload_rowmajor", "se_tree_predict", "se_tree_predict_multi", "se_host_alloc",
                 "se_gbm_round_squared_async", "se_gbm_linesearch_brent", "se_ctx_set_option"):
        assert must in bound
    # every ABI call in the generated C++ exists in the header
    called = set(re.findall(r"\b(se_\w+)\(", cpp)) - {"se_ctx"}
    assert called <= declared, called - declared
    # no JNI critical regions (ADVICE r1): nothing may be pinned while a DMA, a kernel or a collective runs
    assert "GetPrimitiveArrayCritical" not in cpp.split("#ifdef SE_HAVE_JNI")[1]


def test_jni_shim_type_checks_against_stub_jni_h():
    """g++ -fsyntax-only with jni/jni_stub.h (the JNI types and the JNIEnv members the shim uses): the generated C++
    is at least well-formed and calls every ABI function with compatible argument types."""
    import os
    import shutil
    import subprocess
    _, root = _jni_gen()
    gxx = shutil.which("g++")
    assert gxx
    r = subprocess.run([gxx, "-std=c++17", "-fsyntax-only", "-Wall", "-DSE_JNI_STUB", "-I" + os.path.join(root, "jni"),
                        os.path.join(root, "jni", "se_jni.cpp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]


def test_rewired_scala_train_uses_only_existing_natives():
    import os
    import re
    _, root = _jni_gen()
    natives = set(re.findall(r"@native def (\w+)\(", open(os.path.join(root, "scala", "org", "apache", "spark", "ml", "se", "SeNative.scala")).read()))
    src = open(os.path.join(root, "scala", "org", "apache", "spark", "ml", "regression", "GBMRegressorNative.scala")).read()
    used = set(re.findall(r"SeNative\.(\w+)\(", src))
    assert used and used <= natives, used - natives
    # the per-row work of the reference's train() is delegated: every step of the hot path appears
    for call in ("gbmPseudoResiduals", "gbmLinesearchEval", "gbmRound", "gbmUpdate", "gbmUpdateValidation", "quantile",
                 "treePredict", "uploadRowmajor"):
        assert call in used
    # GBMRegressionModel.transform per partition: the forest route and the member-by-member route
    src = open(os.path.join(root, "scala", "org", "apache", "spark", "ml", "regression", "GBMRegressionModelNative.scala")).read()
    used = set(re.findall(r"SeNative\.(\w+)\(", src))
    assert used and used <= natives, used - natives
    for call in ("forestPredict", "uploadRowmajor", "aggConfigure", "aggRun", "download", "ctxDestroy"):
        assert call in used
    # BoostingClassifier.train() (SAMME / SAMME.R), rewired the same way
    src = open(os.path.join(root, "scala", "org", "apache", "spark", "ml", "classification", "BoostingClassifierNative.scala")).read()
    used = set(re.findall(r"SeNative\.(\w+)\(", src))
    assert used and used <= natives, used - natives
    for call in ("boostConfigure", "boostRealUpdate", "boostDiscreteError", "boostDiscreteUpdate", "slotSum", "downloadScaled"):
        assert call in used


# ------------------------------------------------------------------ row sharding over several contexts (Param `devices`)
class _FakeCtx:
    """Records what a Context would hold: slot -> float32 [rows][cols]."""

    def __init__(self, device):
        self.device, self.slots, self.calls = device, {}, []
        self.dim = 1

    def close(self):
        self.closed = True

    def sync(self):
        pass

    def comm_destroy(self):
        self.left = True

    def gbm_configure(self, n, nv, dim, loss, param=0.0, has_weights=False):
        import numpy as np
        from spark_ensemble_b200 import _native as N
        self.n, self.nv, self.dim = n, nv, dim
        for s, (r, c) in {N.SLOT_Y: (1, n), N.SLOT_W: (1, n), N.SLOT_F: (dim, n), N.SLOT_H: (dim, n), N.SLOT_R: (dim, n),
                          N.SLOT_VY: (1, nv), N.SLOT_VF: (dim, nv), N.SLOT_VH: (dim, nv)}.items():
            self.slots[s] = np.zeros((r, c), dtype=np.float32)

    def layout(self, slot):
        a = self.slots[slot]
        return a.shape[0], a.shape[1], a.shape[1]

    def upload(self, slot, host, offset=0):
        import numpy as np
        a = np.asarray(host, dtype=np.float32).reshape(-1)
        self.slots[slot].reshape(-1)[offset:offset + a.size] = a

    def fill(self, slot, value, count=None, offset=0):
        flat = self.slots[slot].reshape(-1)
        flat[offset:offset + (flat.size - offset if count is None else count)] = value

    def download(self, slot, scale=None):
        a = self.slots[slot]
        return a.copy() if a.shape[0] > 1 else a.reshape(-1).copy()

    def forest_predict(self, trees, out_slot, **kw):
        self.calls.append(("forest", len(trees), out_slot, kw.get("init", 0.0)))

    def gbm_update(self, step, residual=False, newton=False, loss=True):
        self.calls.append(("update", tuple(step)))
        return 1.25, None


def test_sharded_context_splits_and_reassembles_rows():
    import numpy as np
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.ensemble import row_partition
    from spark_ensemble_b200.sharded import ShardedContext
    for world, n, nv, dim in ((2, 1003, 10, 1), (3, 17, 2, 4), (4, 5, 0, 2)):
        sc = ShardedContext(list(range(world)), context_factory=_FakeCtx, join=False)
        sc.gbm_configure(n, nv, dim, "logloss" if dim > 1 else "squared")
        y = np.arange(n, dtype=np.float32)
        F = (np.arange(dim * n, dtype=np.float32) * 0.5).reshape(dim, n)
        sc.upload(N.SLOT_Y, y)
        sc.upload(N.SLOT_F, F)
        for j in range(dim):  # GBMEngine.set_direction_from_model's per-dimension upload and _load_pred's fill
            sc.upload(N.SLOT_H, F[j] + 1.0, offset=j * n)
            sc.fill(N.SLOT_R, float(j + 1), n, j * n)
        for r, c in enumerate(sc.ctxs):
            s0, s1 = row_partition(n, world, r)
            assert c.n == s1 - s0
            np.testing.assert_array_equal(c.slots[N.SLOT_Y][0], y[s0:s1])
            np.testing.assert_array_equal(c.slots[N.SLOT_F], F[:, s0:s1])
            np.testing.assert_array_equal(c.slots[N.SLOT_H], F[:, s0:s1] + 1.0)
            for j in range(dim):
                assert np.all(c.slots[N.SLOT_R][j] == j + 1)
        np.testing.assert_array_equal(np.asarray(sc.download(N.SLOT_F)).reshape(dim, n), F)
        np.testing.assert_array_equal(np.asarray(sc.download(N.SLOT_Y)).reshape(-1), y)
        assert sc.gbm_update([0.5] * dim, residual=True)[0] == 1.25
        assert all(c.calls == [("update", tuple([0.5] * dim))] for c in sc.ctxs)
        sc.forest_predict([{"feature": [-1]}] * 3, N.SLOT_H, init=0.25)   # every shard evaluates the same forest over its rows
        assert all(c.calls[-1] == ("forest", 3, N.SLOT_H, 0.25) for c in sc.ctxs)
        ctxs = list(sc.ctxs)
        sc.close()
        assert all(getattr(c, "left", False) and getattr(c, "closed", False) for c in ctxs)  # communicator left first


def test_gbm_regressor_has_devices_param():
    from spark_ensemble_b200.regression import GBMRegressor
    g = GBMRegressor()
    assert g("devices") == []
    g.set("devices", [0, 1]) if hasattr(g, "set") else None


def test_sort_network_sorts(tmp_path):
    """csrc/se_sortnet.h (Batcher's odd-even merge sort, the weighted-median kernels' network) compiled for the host:
    random, many-duplicate and 0/1 inputs (zero-one principle) for every size the kernels instantiate."""
    import shutil
    import subprocess
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    src = tmp_path / "sn.cpp"
    src.write_text(r"""
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <algorithm>
#include "se_sortnet.h"
template <int N> int run(int expect) {
  int ces = 0, bad = 0;
  for (int it = 0; it < 20000; ++it) {
    uint64_t v[N], r[N];
    for (int i = 0; i < N; ++i) v[i] = (it & 1) ? (uint64_t)(rand() & 1) : (rand() % (it % 7 + 2) == 0 ? (uint64_t)(rand() % 5) : ((uint64_t)rand() << 20) ^ (uint64_t)rand());
    for (int i = 0; i < N; ++i) r[i] = v[i];
    std::sort(r, r + N);
    ces = 0;
    se::sortnet_oddeven<N>(v, [&](uint64_t& a, uint64_t& b) { ++ces; const uint64_t lo = std::min(a, b), hi = std::max(a, b); a = lo; b = hi; });
    for (int i = 0; i < N; ++i) bad += v[i] != r[i];
  }
  if (N == 16) {  // exhaustive 0/1
    for (uint32_t m = 0; m < (1u << 16); ++m) {
      uint64_t v[N];
      for (int i = 0; i < N; ++i) v[i] = (m >> i) & 1;
      se::sortnet_oddeven<N>(v, [&](uint64_t& a, uint64_t& b) { const uint64_t lo = std::min(a, b), hi = std::max(a, b); a = lo; b = hi; });
      for (int i = 0; i + 1 < N; ++i) bad += v[i] > v[i + 1];
    }
  }
  std::printf("N=%d ces=%d bad=%d\n", N, ces, bad);
  return bad + (ces != expect);
}
int main() { return run<1>(0) + run<2>(1) + run<4>(5) + run<8>(19) + run<16>(63) + run<32>(191) + run<64>(543); }
""")
    exe = tmp_path / "sn"
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "spark_ensemble_b200", "csrc")
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", inc, "-o", str(exe), str(src)], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
