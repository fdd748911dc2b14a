"""The random GBM walks of test_gpu_gbm_state_walks.py, without a device: the generator is deterministic, draws only
calls that are valid where they are drawn (failing ones only on purpose), and the fp64 model's F, r and loss equal a
direct recomputation from the steps it applied."""
import numpy as np
import pytest

from oracle import np_oracle as NP
from tests import gbm_walk as W

SEEDS = list(range(40))


def _walk(seed):
    n = (3, 1001, 40961)[seed % 3]
    return W.generate(seed, n, 40 + seed % 41, sizes=(3, 1001, 40961) if seed % 4 == 0 else None), n


@pytest.mark.parametrize("seed", SEEDS[:8])
def test_generator_is_deterministic(seed):
    a, _ = _walk(seed)
    b, _ = _walk(seed)
    assert repr(a) == repr(b)
    assert repr(W.generate(seed, 1001, 60, pinned=tuple(W.BIT_IDENTICAL))) == \
        repr(W.generate(seed, 1001, 60, pinned=tuple(W.BIT_IDENTICAL)))


def _check_valid(ops, pinned=()):
    """An independent reading of each call's preconditions against the state the calls before it left."""
    n = nv = 0
    loss, has_w, wout, feats = None, False, False, False
    known = set()
    fails = 0
    for i, o in enumerate(ops):
        k = o["op"]
        where = f"step {i}: {o}"
        if i == 0:
            assert k == "configure", where
        if k == "configure":
            assert o["loss"] in W.LOSSES and o["nv"] >= 0 and o["n"] >= 1, where
            if (o["n"], o["nv"]) != (n, nv):
                known, feats, wout = set(), False, False
            elif o["has_w"] and not has_w:
                known.discard("W")
            n, nv, loss, has_w = o["n"], o["nv"], o["loss"], o["has_w"]
            continue
        if k == "features":
            feats = True
            continue
        if k in ("upload", "fill", "synth"):
            sl = o["slot"]
            size = nv if sl.startswith("V") else n
            assert 0 <= o["offset"] and o["count"] >= 1 and o["offset"] + o["count"] <= size, where
            assert sl != "W" or has_w, where
            assert not sl.startswith("V") or nv, where
            assert sl != "WOUT" or wout, where
            assert sl != "P" or feats, where
            if sl in ("Y", "VY") and loss == "bernoulli":
                assert o.get("kind") in ("label", "bernoulli") or o.get("value") in (0.0, 1.0), where
            if o["offset"] == 0 and o["count"] == size:
                known.add(sl)
            else:
                assert sl in known or sl == "P", where
            continue
        if k in ("copy_slot", "copy_rows"):
            assert feats and o["src"] in known | {"P"}, where
            known.add(o["dst"])
            continue
        # every call below reads the GBM problem
        need = {"Y", "F", "H"} | ({"W"} if has_w else set()) | ({"VY", "VF", "VH"} if nv else set())
        if k not in ("opt", "device_ptr", "set_bag", "set_param") and not k.startswith("fail"):
            assert need <= known, (where, need - known)
        if k in ("tree", "forest", "linear", "linear_v", "tree_fit"):
            assert feats, where
            assert k != "linear_v" or nv, where
            assert k != "tree_fit" or "R" in known, where
            known.add("H")
        elif k == "resid":
            assert not o["newton"] or loss in W.HESSIAN, where
            known |= {"R", "WOUT"} if o["newton"] else {"R"}
            wout = wout or o["newton"]
        elif k == "update":
            assert not o["newton"] or loss in W.HESSIAN, where
            known |= {"R", "WOUT"} if o["newton"] else set()
            wout = wout or o["newton"]
        elif k == "update_valid":
            assert nv, where
        elif k in ("async", "stats", "fail_tol"):
            assert loss == "squared", where
        elif k == "ls_newton":
            assert loss in W.HESSIAN, where
        elif k == "read":
            assert o["what"] != "WOUT" or wout, where
            assert o["what"] != "mean_v" or nv, where
            assert o["what"] not in ("R", "sumR") or "R" in known, where
        elif k == "opt":
            assert o["key"] not in pinned and o["value"] in W.OPTIONS[o["key"]], where
            assert o["key"] != "sq_defer_max" or o["value"] < 64, where
        elif k == "quantile":
            assert 0.0 <= o["q"] <= 1.0, where
        elif k == "absq":
            assert 0.0 <= o["q"] <= 1.0, where
        if k.startswith("fail"):
            fails += 1
        else:
            assert k in ("round", "brent", "eval", "eval2", "set_bag", "set_param", "device_ptr", "tree", "forest",
                         "linear", "linear_v", "tree_fit", "resid", "update", "update_valid", "async", "stats",
                         "ls_newton", "read", "opt", "quantile", "absq"), where
    return fails


def test_every_call_is_valid_where_it_is_drawn():
    fails = 0
    for seed in SEEDS:
        ops, _ = _walk(seed)
        fails += _check_valid(ops)
        _check_valid(W.generate(seed, 1001, 60, pinned=tuple(W.BIT_IDENTICAL)), pinned=tuple(W.BIT_IDENTICAL))
    assert fails > 0  # failing calls are drawn, on purpose, and only as fail_* calls


def test_walks_cover_the_operations():
    seen = set()
    for seed in SEEDS:
        seen |= {o["op"] for o in _walk(seed)[0]}
    assert {"configure", "upload", "fill", "synth", "copy_slot", "copy_rows", "device_ptr", "tree", "forest",
            "linear", "tree_fit", "resid", "round", "async", "brent", "ls_newton", "eval", "eval2", "stats",
            "update", "update_valid", "set_bag", "set_param", "absq", "quantile", "read", "opt", "fail_upload",
            "fail_quantile", "fail_maxeval", "fail_tol"} <= seen


def _replay(ops, alphas):
    """F, r and the loss of a walk recomputed from its calls alone, apart from the model: the writes as the calls give
    them, F as its last write plus the sum of the fp32 steps taken since, summed in one pass in reverse order, and r
    from np_oracle at the F of the last call that derived it.  `alphas` are the line searches' choices, in order."""
    n = nv = 0
    loss = param = None
    slot, steps, X, VX, cands = {}, [], None, None, None
    k = 0

    def F():
        if not steps:
            return slot["F"]
        return slot["F"] + np.sum(np.stack([c * h for c, h in reversed(steps)]), axis=0)

    def settle():
        f = F()
        steps.clear()
        slot["F"] = f
        return f

    def derive_r(newton):
        y = slot["Y"]
        r, _, _ = NP.pseudo_residuals(loss, param, 1, y, None, settle(), newton)
        slot["R"] = r[0]

    for o in ops:
        op = o["op"]
        if op == "configure":
            if (o["n"], o["nv"]) != (n, nv):
                slot, steps = {}, []
            n, nv, loss, param = o["n"], o["nv"], o["loss"], o["param"]
        elif op == "features":
            X, VX, cands = W.features(n, nv)
        elif op in ("upload", "fill", "synth"):
            sl = o["slot"]
            if op == "upload":
                vals = W.values(o["kind"], o["seed"], o["count"])
            elif op == "fill":
                vals = np.full(o["count"], np.float32(o["value"]))
            else:  # the model's stand-in for the device generator
                vals = W.values("label" if o["kind"] == "bernoulli" else "weight" if sl == "W" else "dir", o["seed"],
                                o["count"])
            if sl == "F" and steps:
                settle()
            cur = slot.get(sl)
            cur = np.zeros(nv if sl.startswith("V") else n) if cur is None else cur.copy()
            cur[o["offset"]:o["offset"] + o["count"]] = vals
            slot[sl] = cur
        elif op in ("copy_slot", "copy_rows"):
            # the device holds fp32: a direction copied into H is what the model then steps along
            slot[o["dst"]] = W.d64(W.f32(slot[o["src"]])) if o["dst"] == "H" else slot[o["src"]].copy()
        elif op in ("tree", "forest", "linear", "linear_v"):
            rng = np.random.default_rng(o["seed"])
            if op == "tree":
                slot["H"] = W.d64(W.f32(W.tree_eval(W.random_tree(rng, cands), X)[1]))
            elif op == "forest":
                ts = [W.random_tree(rng, cands) for _ in range(2)]
                slot["H"] = W.d64(W.f32(0.1 + 0.6 * W.tree_eval(ts[0], X)[1] - 0.3 * W.tree_eval(ts[1], X)[1]))
            else:
                coef, b = W.f32(rng.standard_normal(W.D) * 0.4), float(np.float32(rng.standard_normal() * 0.2))
                slot["VH" if op == "linear_v" else "H"] = W.d64(W.f32(W.d64(coef) @ W.d64(VX if op == "linear_v" else X) + b))
        elif op == "tree_fit":  # without a device the model's stand-in: the mean of r to three decimals
            slot["H"] = W.d64(W.f32(np.full(n, np.round(np.mean(slot["R"]), 3))))
        elif op == "resid":
            derive_r(o["newton"])
        elif op == "update":
            steps.append((float(np.float32(o["step"])), slot["H"]))
            if o["residual"] or o["newton"]:
                derive_r(o["newton"])
        elif op in ("round", "async"):
            steps.append((float(np.float32(o["lr"] * alphas[k])), slot["H"]))
            k += 1
            if op == "async" or o["residual"]:
                derive_r(False)
        elif op == "set_param":
            param = o["param"]
    assert k == len(alphas)
    f = F()
    return f, slot.get("R"), NP.loss(loss, param, NP.encode(loss, slot["Y"]), f).sum()


@pytest.mark.parametrize("seed", SEEDS[::5])
def test_model_matches_a_direct_recomputation(seed):
    """The model's F, r and train loss after a walk equal an independent recomputation from the calls and the
    alphas the model applied."""
    from oracle import oracle as O
    ops, n = _walk(seed)
    w = W.Walker(None, oracle=O.Oracle(), seed=seed).run(ops)
    F, r, lo = _replay(ops, w.alphas)
    scale = np.abs(w.v["F"]) + sum(np.abs(s[1] * s[2]) for s in w.steps if s[0] == "step")
    np.testing.assert_array_less(np.abs(w.v["F"] - F), 1e-13 * scale + 1e-300)
    np.testing.assert_allclose(w.v["R"], r, rtol=1e-9, atol=1e-12)
    got = NP.loss(w.loss, w.param, w._ye(), w.v["F"]).sum()
    assert got == pytest.approx(lo, rel=1e-11)
