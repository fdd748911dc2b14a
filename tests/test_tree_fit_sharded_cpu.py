"""ShardedContext.tree_fit without a GPU: every rank is called, and the ranks' trees must be identical."""
import numpy as np
import pytest


class _TreeCtx:
    """Returns a fixed tree from tree_fit and records the calls; `tree` is set per rank by the test."""

    def __init__(self, device):
        self.device, self.calls = device, []
        self.tree = None

    def close(self):
        pass

    def sync(self):
        pass

    def comm_destroy(self):
        pass

    def tree_fit_bins(self, candidates):
        self.calls.append(("bins", len(candidates)))

    def tree_fit(self, *a, **k):
        self.calls.append(("fit", a, tuple(sorted(k))))
        return {key: np.copy(v) for key, v in self.tree.items()}


def _tree():
    return {"feature": np.array([0, -1, -1], np.int32), "threshold": np.array([0.5, 0, 0], np.float32),
            "left": np.array([1, 0, 0], np.int32), "right": np.array([2, 0, 0], np.int32),
            "value": np.array([0, -1.25, 2.5], np.float32), "gain": np.array([0.75, 0, 0])}


@pytest.mark.parametrize("world", [2, 3, 4])
def test_sharded_tree_fit_returns_rank0_tree_when_ranks_agree(world):
    from spark_ensemble_b200.sharded import ShardedContext
    with ShardedContext(list(range(world)), context_factory=_TreeCtx, join=False) as sc:
        for c in sc.ctxs:
            c.tree = _tree()
        sc.tree_fit_bins([np.array([0.5]), np.zeros(0)])
        t = sc.tree_fit(3, 0, -1, 0, False, subspace=[0, 1], max_depth=1)
        for k, v in _tree().items():
            np.testing.assert_array_equal(t[k], v)
        for c in sc.ctxs:  # every rank got the same candidates and the same fit call
            assert c.calls == sc.ctxs[0].calls == [("bins", 2), ("fit", (3, 0, -1, 0, False), ("max_depth", "subspace"))]


def test_gbm_device_learner_accepts_several_devices_that_exist(monkeypatch):
    """With the device learner, `devices` must name distinct GPUs that exist (every rank joins each level's
    all-reduce); such a list is accepted by GBMRegressor and GBMClassifier alike."""
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.classification import GBMClassifier
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor
    from spark_ensemble_b200.regression import GBMRegressor
    from spark_ensemble_b200.routes import device_fit
    learner = DeviceDecisionTreeRegressor(maxDepth=2)
    monkeypatch.setattr(N, "device_count", lambda: 4)
    for est in (GBMRegressor(), GBMClassifier()):
        est.set("residentFeatures", True)
        for devices in ([], [2], [0, 1], [3, 1, 2]):
            est.set("devices", devices)
            assert device_fit(est, learner, require_resident=True) is True
        est.set("devices", [0, 1, 0])
        with pytest.raises(ValueError, match="distinct"):
            device_fit(est, learner, require_resident=True)
        est.set("devices", [0, 4])
        with pytest.raises(ValueError, match="GPU 4 is not one of the 4 visible"):
            device_fit(est, learner, require_resident=True)
        est.set("residentFeatures", False)
        with pytest.raises(ValueError, match="residentFeatures"):
            device_fit(est, learner, require_resident=True)


@pytest.mark.parametrize("key", ["feature", "threshold", "value", "gain"])
def test_sharded_tree_fit_raises_when_ranks_differ(key):
    from spark_ensemble_b200.sharded import ShardedContext
    with ShardedContext([0, 1, 2], context_factory=_TreeCtx, join=False) as sc:
        for c in sc.ctxs:
            c.tree = _tree()
        bad = sc.ctxs[2].tree[key]
        bad[0] = np.nextafter(bad[0], np.inf, dtype=bad.dtype) if bad.dtype.kind == "f" else bad[0] + 1
        with pytest.raises(AssertionError, match="ranks disagree on the fitted tree"):
            sc.tree_fit(3, 0, -1, 0, False, subspace=[0, 1], max_depth=1)
