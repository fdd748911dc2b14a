"""learners.lockstep, the driver that runs Bagging's logistic members' L-BFGS fits together so that one batched call
answers every live member's evaluation: driven here by a numpy evaluate (oracle/np_logistic.py), without a GPU.  Members
fitted together must equal members fitted one by one, bit for bit, while they stop at different iterations; a batch of
one must reproduce the lone optimize; an exception in one member or in the batch evaluation must fail the whole fit
without leaving a thread behind."""
import threading

import numpy as np
import pytest

from oracle import np_logistic as O
from spark_ensemble_b200.learners import DeviceLogisticRegression, column_groups, lockstep


def _data(seed, n=600, d=8, K=2):
    rng = np.random.default_rng(seed)
    X = (rng.standard_normal((n, d)) * [1, 2, 3, 0.5, 1, 4, 1, 2][:d] + 3).astype(np.float32)
    logits = X @ rng.standard_normal((d, K))
    y = np.argmax(logits + rng.gumbel(size=(n, K)), axis=1).astype(np.float64)
    w = rng.uniform(0, 2, n)
    w[rng.random(n) < 0.2] = 0.0
    return X, y, w


SUBS = [np.array([0, 1, 2]), np.array([3, 4, 5, 6, 7]), np.array([1]), np.array([7, 2, 2, 5]), np.array([], np.int32)]


def _members(X, y, w, K, learner):
    """(job, evaluate over the member's columns) per subspace, with the device route's stats and shifts."""
    out = []
    for c in SUBS:
        shift = X[0, c].astype(np.float64)
        st = O.stats(X, y, c, K, w, shift)
        out.append((lambda ev, st=st, s=shift: learner.optimize(ev, st, s, K), O.evaluator(X, y, c, w)))
    return out


def _batch_of(evaluators, calls=None):
    def evaluate_batch(requests):
        if calls is not None:
            calls.append([i for i, *_ in requests])
        return [evaluators[i](kshift, scale, coef) for i, kshift, scale, coef in requests]
    return evaluate_batch


def _same(a, b):
    assert a.coefficientMatrix.tobytes() == b.coefficientMatrix.tobytes()
    assert a.interceptVector.tobytes() == b.interceptVector.tobytes()
    assert a.objectiveHistory == b.objectiveHistory
    assert a.numEvaluations == b.numEvaluations


@pytest.mark.parametrize("K", [2, 4])
def test_members_together_equal_members_alone(K):
    X, y, w = _data(3 + K, K=K)
    learner = DeviceLogisticRegression(regParam=0.01, tol=1e-9, maxIter=60)
    members = _members(X, y, w, K, learner)
    alone = [job(ev) for job, ev in members]
    calls = []
    together = lockstep([job for job, _ in members], _batch_of([ev for _, ev in members], calls))
    for a, b in zip(alone, together):
        _same(a, b)
    # the members stop at different evaluation counts, and the batches shrink as they do
    counts = [m.numEvaluations for m in alone]
    assert len(set(counts)) > 1, counts
    sizes = [len(c) for c in calls]
    assert sizes[0] == len(SUBS) and sizes[-1] == 1 and sizes == sorted(sizes, reverse=True)
    assert len(calls) == max(counts)
    for k in range(len(SUBS)):
        assert sum(k in c for c in calls) == counts[k]


def test_batch_of_one_is_the_lone_optimize():
    X, y, w = _data(11)
    learner = DeviceLogisticRegression(regParam=0.1, elasticNetParam=0.5, tol=1e-8)
    (job, ev), = _members(X, y, w, 2, learner)[1:2]
    _same(job(ev), lockstep([job], _batch_of([ev]))[0])


def test_no_members():
    assert lockstep([], _batch_of([])) == []


def test_member_exception_fails_the_fit():
    X, y, w = _data(5)
    learner = DeviceLogisticRegression(tol=1e-9)
    members = _members(X, y, w, 2, learner)
    evals = [ev for _, ev in members]
    n_seen = [0]

    def failing(ev):
        def evaluate(*a):
            n_seen[0] += 1
            if n_seen[0] == 3:
                raise ArithmeticError("member 2 failed")
            return ev(*a)
        return learner.optimize(evaluate, O.stats(X, y, SUBS[2], 2, w, X[0, SUBS[2]].astype(np.float64)),
                                X[0, SUBS[2]].astype(np.float64), 2)

    jobs = [job for job, _ in members]
    jobs[2] = failing
    before = threading.active_count()
    with pytest.raises(ArithmeticError, match="member 2 failed"):
        lockstep(jobs, _batch_of(evals))
    assert threading.active_count() == before


def test_batch_exception_fails_the_fit():
    X, y, w = _data(6)
    learner = DeviceLogisticRegression(tol=1e-9)
    members = _members(X, y, w, 2, learner)
    evals = [ev for _, ev in members]
    calls = [0]

    def evaluate_batch(requests):
        calls[0] += 1
        if calls[0] == 4:
            raise RuntimeError("device call failed")
        return [evals[i](*r) for i, *r in requests]

    before = threading.active_count()
    with pytest.raises(RuntimeError, match="device call failed"):
        lockstep([job for job, _ in members], evaluate_batch)
    assert threading.active_count() == before
    assert calls[0] == 4


def test_column_groups_keep_each_union_within_the_limit():
    subs = [np.arange(0, 100), np.arange(50, 200), np.arange(190, 260), np.arange(300, 320), np.arange(0, 300)]
    groups = column_groups(subs, 254)
    assert [i for g in groups for i in g] == list(range(len(subs)))
    for g in groups:
        union = set(np.concatenate([subs[i] for i in g]).tolist())
        assert len(union) <= 254 or len(g) == 1
    assert groups == [[0, 1], [2, 3], [4]]
