"""The pieces of BaggingRegressor / BaggingClassifier's device fit that need no GPU: the split candidates of a row
subset without copying it, the deduplication of equal subspaces, and the forest-fit prototype."""
import numpy as np
import pytest


def _learners():
    from spark_ensemble_b200.learners import DeviceDecisionTreeClassifier, DeviceDecisionTreeRegressor
    return [DeviceDecisionTreeRegressor(maxBins=32, seed=7), DeviceDecisionTreeClassifier(maxBins=64, seed=-3)]


@pytest.mark.parametrize("n", [3_000, 40_000])  # below and above max(maxBins², 10000): every row, then Spark's sample
@pytest.mark.parametrize("which", [0, 1])
def test_split_candidates_of_a_row_subset(n, which):
    learner = _learners()[which]
    rng = np.random.default_rng(n + which)
    X = rng.standard_normal((n, 5))
    X[rng.random((n, 5)) < 0.03] = np.nan
    X[:, 3] = np.round(X[:, 3])  # few distinct values: every midpoint
    X[:, 4] = 1.0                # one value: no candidate
    for keep in (rng.random(n) < 0.7, rng.poisson(1.0, n) > 0):
        rows = np.flatnonzero(keep)
        want = learner.split_candidates(X[rows])
        got = learner.split_candidates(X, rows=rows)
        assert len(got) == len(want) == X.shape[1]
        for g, w in zip(got, want):
            assert g.dtype == w.dtype == np.float32
            np.testing.assert_array_equal(g, w)
    required = max(learner.maxBins ** 2, 10000)
    assert (learner.sample_rows(rows.size) is None) == (rows.size <= required)


def test_split_candidates_rows_do_not_copy_the_subset():
    """Only the sampled rows are gathered: a subset past the sampling threshold never materialises X[rows]."""
    learner = _learners()[0]
    rng = np.random.default_rng(1)
    X = rng.standard_normal((200_000, 3)).astype(np.float32)
    rows = np.flatnonzero(rng.random(X.shape[0]) < 0.9)
    seen = []

    class Spy(np.ndarray):
        def __getitem__(self, idx):
            out = np.ndarray.__getitem__(self, idx)
            if isinstance(idx, np.ndarray):
                seen.append(idx.size)
            return out
    got = learner.split_candidates(X.view(Spy), rows=rows)
    assert seen and max(seen) < rows.size // 5
    for g, w in zip(got, learner.split_candidates(X[rows])):
        np.testing.assert_array_equal(g, w)


def test_forest_subspaces_fit_each_distinct_subspace_once():
    learner = _learners()[0]
    subs = [np.array([0, 2], np.int32), np.array([1], np.int32), np.array([0, 2], np.int32), np.array([2, 0], np.int32)]
    distinct, index = learner._forest_subspaces(subs)
    assert [d.tolist() for d in distinct] == [[0, 2], [1], [2, 0]]
    assert index == [0, 1, 0, 2]


def test_forest_fit_prototype_matches_header():
    import re
    from spark_ensemble_b200 import _native as N
    import os
    hdr = open(os.path.join(os.path.dirname(N.__file__), "..", "include", "se_abi.h")).read()
    m = re.search(r"SE_API int se_forest_fit\(([^;]*)\);", hdr, re.S)
    assert m, "se_forest_fit is declared"
    assert len(m.group(1).split(",")) == len(N.PROTOTYPES["se_forest_fit"])
