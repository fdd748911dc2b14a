"""Seeded random walks of GBM context calls, and an fp64 host model of what they leave in y, F, h, r, w and the bag.

The native context keeps derived state between calls: an owed F (y - r), a residual slot with pending steps, the
squared round's carried statistics, the weight sum, WOUT's 1/S factor, the rank matrix.  None of it may show in what a
call returns.  A walk draws calls freely (rounds over one direction are common, so chains build), and `Walker` applies
each call to the model and, given a Context, to the device, checking every value the device returns against the model.

The model owns the values; the device only chooses: the model applies the step lr·alpha the device reports, after
checking alpha against the closed form (squared loss) or the fp64 objective at the oracle Brent's minimum.  Test
infrastructure only: no product module imports it.
"""
from __future__ import annotations

import numpy as np

from oracle import np_oracle as NP

EPS32 = float(np.finfo(np.float32).eps)
LOSSES = ("squared", "huber", "absolute", "bernoulli")
D = 3           # feature columns of the resident X
LR = 0.7
TOL = 1e-6
RTOL = 1e-5     # sums, losses and means (test_gpu_boost_edges.py)
# options a walk may flip between calls; the bit-identical pairs are run with walks that never flip the pinned ones
OPTIONS = {"sq_defer_max": (0, 1, 2, 16), "fused_round": (-1, 0, 1), "fused_resident": (0, 1), "host_mirror": (0, 1),
           "alternate_passes": (0, 1), "ls_mode": (0, 1, 2)}
DEFAULTS = {"sq_defer_max": 16, "fused_round": 1, "fused_resident": 1, "host_mirror": 1, "alternate_passes": 1,
            "ls_mode": 1}
# settings documented as giving the same bits as the default ones (sq_defer_max: test_gpu_deferred_residual.py,
# fused_resident: test_gpu_fused_resident.py; host_mirror serves the same doubles from mapped memory instead of a
# copy; ls_mode 2 runs the device Brent's template on the host over the same evaluations)
BIT_IDENTICAL = {"sq_defer_max": 0, "fused_resident": 0, "host_mirror": 0, "ls_mode": 2}
HESSIAN = ("squared", "bernoulli")
SLOTS = ("Y", "W", "F", "H", "R", "WOUT", "VY", "VF", "VH", "P")


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def d64(a):
    return np.asarray(a, dtype=np.float64)


def values(kind, seed, count):
    """Deterministic host data of a walk's writes (fp32)."""
    rng = np.random.default_rng(seed)
    if kind == "label":
        return f32(rng.random(count) < 0.45)
    if kind == "weight":
        return f32(rng.uniform(0.25, 2.0, count))
    if kind == "bag":
        return f32(rng.poisson(1.0, count))
    if kind == "dir":
        return f32(0.5 * rng.standard_normal(count) + 0.05)
    return f32(rng.standard_normal(count))


def features(n, nv):
    rng = np.random.default_rng(7 + n)
    X = f32(rng.standard_normal((D, n)))
    VX = f32(rng.standard_normal((D, nv))) if nv else None
    cands = [np.unique(f32(np.quantile(X[j], np.linspace(0.1, 0.9, 9)))) for j in range(D)]
    return X, VX, cands


def random_tree(rng, cands):
    f0, f1 = (int(x) for x in rng.integers(0, D, 2))
    t0, t1 = (float(c[rng.integers(0, c.size)]) for c in (cands[f0], cands[f1]))
    v = f32(rng.standard_normal(5) * 0.5)
    return {"feature": np.array([f0, -1, f1, -1, -1], np.int32), "threshold": f32([t0, 0, t1, 0, 0]),
            "left": np.array([1, -1, 3, -1, -1], np.int32), "right": np.array([2, -1, 4, -1, -1], np.int32),
            "value": v}


def tree_eval(tree, X):
    """Spark's walk: x <= threshold goes left.  Returns (leaf node per row, leaf value per row)."""
    node = np.zeros(X.shape[1], dtype=np.int64)
    for _ in range(64):
        f = tree["feature"][node]
        inner = f >= 0
        if not inner.any():
            break
        x = X[np.maximum(f, 0), np.arange(X.shape[1])]
        go_left = x <= tree["threshold"][node]
        nxt = np.where(go_left, tree["left"][node], tree["right"][node])
        node = np.where(inner, nxt, node)
    return node, d64(tree["value"][node])


# ---------------------------------------------------------------------------------------------------- the walk
def _pick(rng, seq):
    return seq[int(rng.integers(0, len(seq)))]


class _Shape:
    """What the generator needs to know to draw only valid calls: shapes, the loss, which slots hold known values."""

    def __init__(self):
        self.n = self.nv = 0
        self.loss = None
        self.has_w = False
        self.wout = False  # WOUT holds a Newton output of the current shape
        self.bag = False


def generate(seed: int, n: int, steps: int, pinned=(), sizes=None, losses=LOSSES, sharded=False) -> list:
    """The calls of walk `seed`: a list of dicts.  Rounds over one direction dominate; `pinned` options never flip.
    `sharded` keeps to what ShardedContext exposes: whole-slot uploads and fills, and no copies, synthetic fills, device
    pointers, slot sums, slot quantiles, asynchronous rounds or eval2."""
    rng = np.random.default_rng(seed)
    sizes = sizes or (n,)
    st = _Shape()
    ops = []

    def setup(new_n, nv, loss, has_w, param):
        ops.append({"op": "configure", "n": new_n, "nv": nv, "loss": loss, "param": param, "has_w": has_w})
        same = st.n == new_n and st.nv == nv
        st.wout = st.wout and same
        st.n, st.nv, st.loss, st.has_w, st.bag = new_n, nv, loss, has_w, False
        return same

    def fresh(loss):
        lab = "label" if loss == "bernoulli" else "normal"
        s = int(rng.integers(1 << 30))
        ops.append({"op": "features"})
        ops.append({"op": "upload", "slot": "Y", "kind": lab, "seed": s, "offset": 0, "count": st.n, "f64": False})
        ops.append({"op": "upload", "slot": "F", "kind": "normal", "seed": s + 1, "offset": 0, "count": st.n,
                    "f64": False})
        ops.append({"op": "upload", "slot": "H", "kind": "dir", "seed": s + 2, "offset": 0, "count": st.n,
                    "f64": False})
        if st.has_w:
            ops.append({"op": "upload", "slot": "W", "kind": "weight", "seed": s + 3, "offset": 0, "count": st.n,
                        "f64": False})
        if st.nv:
            for sl, k in (("VY", lab), ("VF", "normal"), ("VH", "dir")):
                ops.append({"op": "upload", "slot": sl, "kind": k, "seed": s + 4, "offset": 0, "count": st.nv,
                            "f64": False})
        ops.append({"op": "resid", "newton": False})

    loss0 = _pick(rng, losses)
    setup(n, int(_pick(rng, (0, 0, 5))) if n > 3 else 0, loss0, bool(rng.random() < 0.3), 0.5)
    fresh(loss0)
    flips = [k for k in OPTIONS if k not in pinned]
    table = [("round", 14), ("configure", 1.2), ("write", 4), ("dirwrite", 2.5), ("resid", 2), ("update", 2),
             ("async", 1), ("ls", 2.5), ("bag", 1), ("param", 1), ("quant", 1), ("read", 3), ("fail", 1.2),
             ("opt", 3 if flips else 0), ("misc", 2)]
    names = [t[0] for t in table]
    wts = np.array([t[1] for t in table], dtype=np.float64)
    wts /= wts.sum()
    while len(ops) < steps:
        kind = names[int(rng.choice(len(names), p=wts))]
        N_, loss = st.n, st.loss
        if kind == "round":
            k = int(rng.integers(1, 5)) if rng.random() < 0.5 else 1
            resid = bool(rng.random() < 0.8)
            for _ in range(k):
                ops.append({"op": "round", "lr": LR, "residual": resid})
        elif kind == "configure":
            new_n = N_ if rng.random() < 0.6 or len(sizes) == 1 else int(_pick(rng, [s for s in sizes if s != N_]))
            nv = st.nv if new_n == N_ and rng.random() < 0.7 else (int(_pick(rng, (0, 5))) if new_n > 3 else 0)
            new_loss = _pick(rng, losses)
            has_w = bool(rng.random() < 0.3)
            had_w = st.has_w and new_n == N_
            same = setup(new_n, nv, new_loss, has_w, float(_pick(rng, (0.3, 1.0))))
            if not same:
                fresh(new_loss)
            else:
                if new_loss == "bernoulli":
                    ops.append({"op": "upload", "slot": "Y", "kind": "label", "seed": int(rng.integers(1 << 30)),
                                "offset": 0, "count": new_n, "f64": False})
                    if nv:
                        ops.append({"op": "upload", "slot": "VY", "kind": "label", "seed": int(rng.integers(1 << 30)),
                                    "offset": 0, "count": nv, "f64": False})
                if has_w and not had_w:
                    ops.append({"op": "fill", "slot": "W", "value": 1.5, "offset": 0, "count": new_n})
        elif kind == "write":
            slots = ["Y", "F", "H", "R"] + (["W"] if st.has_w else []) + (["VY", "VF", "VH"] if st.nv else []) + \
                (["WOUT"] if st.wout else [])
            sl = _pick(rng, slots)
            cnt = st.nv if sl.startswith("V") else N_
            how = _pick(rng, ("upload", "upload", "fill", "synth", "copy"))
            part = rng.random() < 0.4 and cnt > 1 and not sharded
            if sharded and how in ("synth", "copy"):
                how = "upload"
            off = int(rng.integers(0, cnt)) if part else 0
            c = int(rng.integers(1, cnt - off + 1)) if part else cnt
            label = sl in ("Y", "VY") and loss == "bernoulli"
            vk = "label" if label else "weight" if sl in ("W", "WOUT") else "dir" if sl in ("H", "VH") else "normal"
            if how == "copy" and sl in ("R", "H"):
                if sl == "R":
                    ops.append({"op": "copy_slot", "dst": "P", "src": "R"})
                    ops.append({"op": "upload", "slot": "P", "kind": "normal", "seed": int(rng.integers(1 << 30)),
                                "offset": off, "count": c, "f64": False})
                    ops.append({"op": _pick(rng, ("copy_slot", "copy_rows")), "dst": "R", "src": "P"})
                else:
                    ops.append({"op": "copy_rows", "dst": "P", "src": "R"})
                    ops.append({"op": "copy_rows", "dst": "H", "src": "P"})
            elif how == "fill":
                v = float(_pick(rng, (0.0, 1.0))) if label else (1.25 if sl in ("W", "WOUT") else
                                                                  float(np.round(rng.uniform(-1, 1), 3)) or 0.5)
                ops.append({"op": "fill", "slot": sl, "value": v, "offset": off, "count": c})
            elif how == "synth" and sl in ("Y", "H", "W", "VH"):
                sk = "bernoulli" if label else "uniform"
                a, b = (0.5, 0.0) if label else ((0.25, 2.0) if sl == "W" else (-1.0, 1.0))
                ops.append({"op": "synth", "slot": sl, "kind": sk, "seed": int(rng.integers(1 << 30)), "a": a, "b": b,
                            "offset": off, "count": c})
            else:
                ops.append({"op": "upload", "slot": sl, "kind": vk, "seed": int(rng.integers(1 << 30)), "offset": off,
                            "count": c, "f64": bool(rng.random() < 0.3)})
        elif kind == "dirwrite":
            w = _pick(rng, ("tree", "forest", "linear", "linear_v", "tree_fit", "tree_fit"))
            if w == "linear_v" and not st.nv:
                w = "linear"
            ops.append({"op": w, "seed": int(rng.integers(1 << 30))})
        elif kind == "resid":
            ops.append({"op": "resid", "newton": bool(loss in HESSIAN and rng.random() < 0.4)})
            if ops[-1]["newton"]:
                st.wout = True
        elif kind == "update":
            newton = bool(loss in HESSIAN and rng.random() < 0.3)
            ops.append({"op": "update", "step": float(np.round(rng.uniform(0.05, 0.8), 3)),
                        "residual": bool(rng.random() < 0.6), "newton": newton, "loss": bool(rng.random() < 0.7)})
            st.wout = st.wout or newton
            if st.nv and rng.random() < 0.5:
                ops.append({"op": "update_valid", "step": float(np.round(rng.uniform(0.05, 0.8), 3))})
        elif kind == "async":
            if loss == "squared" and not sharded:
                ops.append({"op": "async", "lr": LR})
        elif kind == "ls":
            choices = ["brent", "eval"] + ([] if sharded else ["eval2"]) + (["stats"] if loss == "squared" else []) + \
                (["ls_newton"] if loss in HESSIAN else [])
            ops.append({"op": _pick(rng, choices), "alpha": float(np.round(rng.uniform(0, 2), 3))})
        elif kind == "bag":
            on = rng.random() < 0.6
            ops.append({"op": "set_bag", "seed": int(rng.integers(1 << 30)) if on else None})
            st.bag = on
        elif kind == "param":
            ops.append({"op": "set_param", "param": float(_pick(rng, (0.2, 0.5, 1.5)))})
        elif kind == "quant":
            q = float(_pick(rng, (0.0, 0.3, 0.5, 0.9, 1.0)))
            ops.append({"op": "absq", "q": q} if loss in ("huber", "squared", "absolute") and (sharded or rng.random() < 0.5)
                       else {"op": "quantile", "slot": _pick(rng, ("H", "Y")), "q": q})
        elif kind == "read":
            r = _pick(rng, ("F", "R", "R", "H", "sumF", "sumR", "mean", "mean_v", "WOUT"))
            if r == "WOUT" and not st.wout:
                r = "R"
            if r == "mean_v" and not st.nv:
                r = "mean"
            if sharded and r.startswith("sum"):
                r = r[3:]
            ops.append({"op": "read", "what": r})
        elif kind == "fail":
            choices = ([] if sharded else ["fail_upload", "fail_quantile"]) + ["fail_maxeval"] + \
                (["fail_tol"] if loss == "squared" else [])
            ops.append({"op": _pick(rng, choices), "residual": bool(rng.random() < 0.7)})
        elif kind == "opt":
            key = _pick(rng, flips)
            ops.append({"op": "opt", "key": key, "value": _pick(rng, OPTIONS[key])})
        elif kind == "misc" and not sharded:
            ops.append({"op": "device_ptr", "slot": _pick(rng, ("R", "H"))})
    return ops


# ---------------------------------------------------------------------------------------------------- the model
class WalkFailure(AssertionError):
    pass


class Walker:
    """Applies a walk's calls to the fp64 model and, when `ctx` is given, to the device.

    reads: "drawn" (only the walk's own reads), "full" (F, R, VF, WOUT, H and VH after every call) or "r" (R after
    every call).  `observed` records (step, what, value) of every device value, for bit-for-bit comparisons."""

    def __init__(self, ctx=None, reads="drawn", options=None, oracle=None, seed=None):
        self.ctx = ctx
        self.reads = reads
        self.oracle = oracle
        self.seed = seed
        self.v = {}          # slot -> fp64 values (None: unknown)
        self.m = {}          # slot -> per-element magnitude sum M; a value is checked to within 4·ε32·M
        self.n = self.nv = 0
        self.loss, self.param, self.has_w = "squared", 0.0, False
        self.bag = None
        self.S = None        # the Newton Σ hc of the last Newton call: WOUT is 1/2·hc·w/S
        self.wout_scaled = False  # a download of WOUT applies 1/S (until WOUT is next written)
        self.X = self.VX = None
        self.cands = None
        self.log = []        # the applied calls
        self.steps = []      # ("F-write", ...) / ("F-step", c, h): F's history since its last full write
        self.observed = []
        self.alphas = []     # the alpha of every round, in order: what the model applied
        self.rounds = []     # per device round: (carried, tiles per CTA held in shared memory, deferred)
        self.options = dict(DEFAULTS)
        self.options.update(options or {})
        if ctx is not None:
            for k, val in self.options.items():
                ctx.set_option(k, val)

    # ---- helpers
    def _ye(self, y=None):
        y = self.v["Y"] if y is None else y
        return NP.encode(self.loss, y)

    def _bagc(self):
        return np.ones(self.n) if self.bag is None else self.bag

    def _wsum(self):
        w = self.v["W"] if self.has_w else np.ones(self.n)
        return float(np.sum(self._bagc() * w))

    def _resid(self, F, newton=False):
        ye = self._ye()
        g = NP.gradient(self.loss, self.param, ye, F)
        if not newton:
            return -g, None
        hc = np.maximum(NP.hessian(self.loss, self.param, ye, F), 1e-2)
        return -g / hc, hc

    def _set_R_derived(self, newton=False):
        F = self.v["F"]
        r, hc = self._resid(F, newton)
        self.v["R"] = r
        lip = 1.0 if hc is None else 4.0 / hc
        self.m["R"] = lip * (self.m["F"] + np.abs(self.v["Y"])) + 4 * np.abs(r) + 1.0 * (hc is not None)
        if self.loss == "absolute":  # sign(y - F): rows within F's error of a tie may take either sign
            self.m["R"] = np.where(np.abs(self.v["Y"] - F) <= 8 * EPS32 * (self.m["F"] + np.abs(self.v["Y"])),
                                   np.inf, 0.0)
        if newton:
            w = self.v["W"] if self.has_w else np.ones(self.n)
            self.S = float(np.sum(self._bagc() * hc))
            self.wout_scaled = True
            self.v["WOUT"] = 0.5 * hc * w / self.S
            self.m["WOUT"] = 64 * np.abs(self.v["WOUT"]) * (1 + lip * (self.m["F"] + np.abs(self.v["Y"])))

    def _step_F(self, c):
        h = self.v["H"]
        F = self.v["F"] + c * h
        self.v["F"] = F
        self.m["F"] = self.m["F"] + np.abs(c * h) + np.abs(F) + np.abs(self.v["Y"])
        self.steps.append(("step", c, h.copy()))

    def _objective(self, a):
        p = self.v["F"] + a * self.v["H"]
        return float(np.sum(self._bagc() * NP.loss(self.loss, self.param, self._ye(), p)) / self._wsum())

    def _alpha_model(self):
        """The line search the model expects: the closed form for squared loss, the fp64 oracle Brent otherwise."""
        c, h = self._bagc(), self.v["H"]
        if self.loss == "squared":
            r = self.v["Y"] - self.v["F"]
            s2 = float(np.sum(c * h * h))
            return min(max(float(np.sum(c * r * h)) / s2, 0.0), 100.0) if s2 > 0 else 1.0
        x, _, st = self.oracle.brent(self._objective, 0.0, 100.0, 1.0, TOL, TOL, 100)
        assert st == 0
        return x

    def _check_alpha(self, a, what):
        want = self._alpha_model()
        if self.loss == "squared":
            assert abs(a - want) <= 1e-6 * (abs(want) + 1.0) + 2 * TOL, f"{what}: alpha {a!r}, closed form {want!r}"
        else:
            fa, fw = self._objective(a), self._objective(want)
            assert fa <= fw + RTOL * (abs(fw) + 1e-3), f"{what}: objective {fa!r} at alpha {a!r}, oracle {fw!r} at {want!r}"

    def _close(self, got, want, what, scale=None):
        scale = abs(want) if scale is None else scale
        assert abs(got - want) <= RTOL * scale + 1e-30, f"{what}: {got!r}, model {want!r}"

    def _check_slot(self, sl, got):
        want, m = self.v.get(sl), self.m.get(sl)
        assert want is not None, f"{sl} read while the model does not know it"
        got = d64(got).reshape(-1)
        assert got.shape == want.shape, f"{sl}: {got.shape} vs {want.shape}"
        if m is None:
            bad = got != f32(want)
        else:
            bad = ~(np.abs(got - want) <= 4 * EPS32 * m + 1e-30)
        if bad.any():
            i = int(np.flatnonzero(bad)[0])
            raise WalkFailure(f"{sl}: {int(bad.sum())} of {got.size} values off the model; first at {i}: device "
                              f"{got[i]!r}, model {want[i]!r}, bound {4 * EPS32 * (m[i] if m is not None else 0):.3g}")

    def _dev_read(self, sl, what=None):
        import spark_ensemble_b200._native as N
        out = self.ctx.download(getattr(N, "SLOT_" + sl)).reshape(-1).copy()
        self.observed.append((len(self.log), what or sl, out))
        return out

    def _exact_write(self, sl, vals, offset=0):
        cur = self.v.get(sl)
        if sl == "WOUT" and self.wout_scaled:  # a write drops the 1/S: the rows it leaves download as 1/2·hc·w
            cur, self.m["WOUT"] = cur * self.S, self.m["WOUT"] * self.S
            self.wout_scaled = False
        full = np.zeros(self._len(sl)) if cur is None else cur.copy()
        full[offset:offset + vals.size] = d64(vals)
        self.v[sl] = full
        if sl in ("F", "R", "VF", "P", "WOUT"):
            mm = self.m.get(sl)
            mm = np.zeros(full.size) if mm is None else mm.copy()
            mm[offset:offset + vals.size] = np.abs(d64(vals))
            self.m[sl] = mm
        else:
            self.m.pop(sl, None)
        if sl == "F":
            self.steps = [("write", full.copy())] if offset == 0 and vals.size == full.size else \
                self.steps + [("patch", offset, d64(vals).copy())]

    def _len(self, sl):
        return self.nv if sl.startswith("V") else self.n

    # ---- one call
    def apply(self, op):
        self.log.append(op)
        getattr(self, "op_" + op["op"])(op)
        if self.ctx is not None and self.reads != "drawn":
            self.observe(self.reads)

    def observe(self, which):
        # R first: a read of F rebuilds an owed F as y - r and re-derives R from it, which need not give r's bits
        slots = ["R"] if which == "r" else ["R", "F", "H"] + (["VF", "VH"] if self.nv else []) + \
            (["WOUT"] if self.v.get("WOUT") is not None else [])
        for sl in slots:
            if self.v.get(sl) is None:
                continue
            self._check_slot(sl, self._dev_read(sl, "obs:" + sl))

    def run(self, ops):
        for i, op in enumerate(ops):
            try:
                self.apply(op)
            except AssertionError as e:
                calls = "\n".join(f"  {j:3d} {o}" for j, o in enumerate(ops[:i + 1]))
                raise WalkFailure(f"walk seed {self.seed}, reads={self.reads}, options {self.options}: step {i} "
                                  f"{op}\n{e}\ncalls:\n{calls}") from None
        return self

    # ---- calls
    def op_configure(self, o):
        same = self.n == o["n"] and self.nv == o["nv"]
        if self.ctx is not None:
            self.ctx.gbm_configure(o["n"], o["nv"], 1, o["loss"], o["param"], o["has_w"])
        if not same:
            self.v = {"P": None}
            self.m = {}
            self.S = None
            self.wout_scaled = False
            self.X = None
        elif self.n != o["n"] or (o["has_w"] and not self.has_w):
            self.v["W"] = None
        if self.v.get("WOUT") is not None and self.n != o["n"]:
            self.v["WOUT"] = None
        self.n, self.nv, self.loss, self.param, self.has_w = o["n"], o["nv"], o["loss"], o["param"], o["has_w"]
        self.bag = None

    def op_features(self, o):
        import spark_ensemble_b200._native as N
        self.X, self.VX, self.cands = features(self.n, self.nv)
        if self.ctx is not None:
            self.ctx.alloc(N.SLOT_X, D, self.n)
            self.ctx.upload(N.SLOT_X, self.X)
            if self.nv:
                self.ctx.alloc(N.SLOT_VX, D, self.nv)
                self.ctx.upload(N.SLOT_VX, self.VX)
            self.ctx.tree_fit_bins(self.cands)
            if not hasattr(self.ctx, "ctxs"):  # ShardedContext shards only the GBM and feature slots
                self.ctx.alloc(N.SLOT_P, 1, self.n)

    def op_upload(self, o):
        import spark_ensemble_b200._native as N
        vals = values(o["kind"], o["seed"], o["count"])
        if self.ctx is not None:
            host = d64(vals) if o["f64"] else vals
            self.ctx.upload(getattr(N, "SLOT_" + o["slot"]), host, offset=o["offset"])
        if o["slot"] == "P" and self.v.get("P") is None:
            self.v["P"] = np.zeros(self.n)
        self._exact_write(o["slot"], vals, o["offset"])

    def op_fill(self, o):
        import spark_ensemble_b200._native as N
        if self.ctx is not None:
            self.ctx.fill(getattr(N, "SLOT_" + o["slot"]), o["value"], count=o["count"], offset=o["offset"])
        self._exact_write(o["slot"], np.full(o["count"], np.float32(o["value"])), o["offset"])

    def op_synth(self, o):
        import spark_ensemble_b200._native as N
        if self.ctx is None:  # the device's generator: the model takes any values of the right kind
            vals = values("label" if o["kind"] == "bernoulli" else "weight" if o["slot"] == "W" else "dir",
                          o["seed"], o["count"])
        else:
            slot = getattr(N, "SLOT_" + o["slot"])
            self.ctx.fill_synthetic(slot, o["kind"], o["seed"], o["a"], o["b"], count=o["count"], offset=o["offset"])
            # Y, H, W and VH are read without side effects: the model learns what the generator wrote
            vals = self.ctx.download(slot, count=o["count"], offset=o["offset"]).copy()
            if o["kind"] == "bernoulli":
                assert np.isin(vals, (0.0, 1.0)).all()
            else:
                assert (vals >= o["a"]).all() and (vals <= o["b"]).all()
        self._exact_write(o["slot"], vals, o["offset"])

    def op_copy_slot(self, o):
        import spark_ensemble_b200._native as N
        if self.ctx is not None:
            self.ctx.copy_slot(getattr(N, "SLOT_" + o["dst"]), getattr(N, "SLOT_" + o["src"]))
        self._copy(o)

    def op_copy_rows(self, o):
        import spark_ensemble_b200._native as N
        if self.ctx is not None:
            self.ctx.copy_rows(getattr(N, "SLOT_" + o["dst"]), 0, getattr(N, "SLOT_" + o["src"]), 0, 1)
        self._copy(o)

    def _copy(self, o):
        src, dst = o["src"], o["dst"]
        assert self.v.get(src) is not None, f"copy from unknown {src}"
        self.v[dst] = self.v[src].copy()
        if src in self.m:
            self.m[dst] = self.m[src].copy()
        else:
            self.m.pop(dst, None)
        if dst == "F":
            self.steps = [("write", self.v["F"].copy())]
        if dst == "H":  # a direction: the model takes the fp32 values the device holds, once they check out
            got = f32(self.v["H"]) if self.ctx is None else self._dev_read("H", "copy:H")
            if self.ctx is not None:
                self._check_slot("H", got)
            self._exact_write("H", got)

    def op_device_ptr(self, o):
        import spark_ensemble_b200._native as N
        if self.ctx is not None:
            assert self.ctx.device_ptr(getattr(N, "SLOT_" + o["slot"])) != 0

    def _learn_direction(self, sl, want, scale):
        """A direction writer's output: checked against the host evaluation, then the model takes the fp32 values."""
        if self.ctx is None:
            got = f32(want)
        else:
            got = self._dev_read(sl, "dir:" + sl)
            bad = np.abs(d64(got) - want) > RTOL * scale + 1e-30
            assert not bad.any(), f"{sl}: {int(bad.sum())} rows off the host evaluation"
        self._exact_write(sl, got)

    def op_tree(self, o):
        import spark_ensemble_b200._native as N
        t = random_tree(np.random.default_rng(o["seed"]), self.cands)
        if self.ctx is not None:
            self.ctx.tree_predict(t, N.SLOT_H)
        self._learn_direction("H", tree_eval(t, self.X)[1], 0.0)

    def op_forest(self, o):
        import spark_ensemble_b200._native as N
        rng = np.random.default_rng(o["seed"])
        ts = [random_tree(rng, self.cands) for _ in range(2)]
        w = [0.6, -0.3]
        if self.ctx is not None:
            self.ctx.forest_predict(ts, N.SLOT_H, weights=w, init=0.1)
        want = 0.1 + sum(wi * tree_eval(t, self.X)[1] for wi, t in zip(w, ts))
        self._learn_direction("H", want, 4.0)

    def op_linear(self, o, validation=False):
        import spark_ensemble_b200._native as N
        rng = np.random.default_rng(o["seed"])
        coef, b = f32(rng.standard_normal(D) * 0.4), float(np.float32(rng.standard_normal() * 0.2))
        X = self.VX if validation else self.X
        sl = "VH" if validation else "H"
        if self.ctx is not None:
            self.ctx.linear_predict(coef, b, getattr(N, "SLOT_" + sl), validation=validation)
        want = d64(coef) @ d64(X) + b
        self._learn_direction(sl, want, 10.0)

    def op_linear_v(self, o):
        self.op_linear(o, validation=True)

    def op_tree_fit(self, o):
        """A tree fit over R that writes its output into H: it reads R (settling pending steps along the old h)
        before it replaces h."""
        import spark_ensemble_b200._native as N
        assert self.v.get("R") is not None
        r = self.v["R"]
        if self.ctx is None:  # a stand-in direction, rounded so that r's last bits do not move it
            self._exact_write("H", f32(np.full(self.n, np.round(np.mean(r), 3))))
            return
        else:
            t = self.ctx.tree_fit(N.SLOT_R, 0, -1, 0, False, subspace=np.arange(D, dtype=np.int32), max_depth=2,
                                  out_slot=N.SLOT_H)
            self.observed.append((len(self.log), "tree", np.concatenate([t["feature"].astype(np.float64),
                                                                        d64(t["threshold"]), d64(t["value"])])))
            leaf, _ = tree_eval(t, self.X)
            out = self._dev_read("H", "tree_fit:H")
            np.testing.assert_array_equal(out, t["value"][leaf])
        mr = self.m.get("R")
        for k in np.unique(leaf):
            rows = leaf == k
            want = float(np.mean(r[rows]))
            err = 4 * EPS32 * float(np.max(mr[rows])) if mr is not None else 0.0
            got = float(t["value"][k])
            assert abs(got - want) <= RTOL * float(np.max(np.abs(r[rows]))) + err + 1e-30, \
                f"tree_fit leaf {k}: {got!r}, mean of the model's r {want!r}"
        self._exact_write("H", out)

    def op_resid(self, o):
        if self.ctx is not None:
            self.ctx.gbm_pseudo_residuals(o["newton"])
        self._set_R_derived(o["newton"])

    def op_update(self, o):
        c = float(np.float32(o["step"]))
        if self.ctx is not None:
            ls, sh = self.ctx.gbm_update([o["step"]], residual=o["residual"], newton=o["newton"], loss=o["loss"])
        self._step_F(c)
        if o["newton"] or o["residual"]:
            self._set_R_derived(o["newton"])
        if self.ctx is not None:
            if o["newton"]:
                self._close(float(sh[0]), self.S, "Σ hc")
            if o["loss"]:
                terms = NP.loss(self.loss, self.param, self._ye(), self.v["F"])
                self._close(ls, float(np.sum(terms)), "update loss")

    def op_update_valid(self, o):
        c = float(np.float32(o["step"]))
        if self.ctx is not None:
            ml = self.ctx.gbm_update_validation([o["step"]])
        VF = self.v["VF"] + c * self.v["VH"]
        self.m["VF"] = self.m["VF"] + np.abs(c * self.v["VH"]) + np.abs(VF)
        self.v["VF"] = VF
        if self.ctx is not None:
            want = float(np.mean(NP.loss(self.loss, self.param, self._ye(self.v["VY"]), VF)))
            self._close(ml, want, "validation loss")

    def _apply_round(self, a, lr, residual, loss_sum):
        c = float(np.float32(lr * a))
        self._step_F(c)
        if residual:
            self._set_R_derived(False)
        if loss_sum is not None:
            terms = NP.loss(self.loss, self.param, self._ye(), self.v["F"])
            scale = float(np.sum(terms))
            if self.loss == "squared":  # the closed form (s0 - 2c s1 + c² s2)/2 cancels: scale by its terms
                r = self.v["Y"] - self.v["F"] + c * self.v["H"]
                scale = float(np.sum(0.5 * r * r + np.abs(c * r * self.v["H"]) + 0.5 * (c * self.v["H"]) ** 2))
            self._close(loss_sum, float(np.sum(terms)), "round loss", scale)

    def op_round(self, o):
        if self.ctx is None:
            a, ls = self._alpha_model(), None
        else:
            a, ls, ne = self.ctx.gbm_round(o["lr"], True, TOL, 100, residual=o["residual"])
            self.observed.append((len(self.log), "round", np.array([a, ls, ne])))
            self._check_alpha(a, "round")
            g = self.ctx.get_option
            self.rounds.append((int(g("last_round_stats_carried")), g("last_fused_resident_tiles"),
                                int(g("last_round_deferred"))))
            # a round leaves no more steps pending than the cap in force when it ran (a lower cap set later applies
            # from the next round on)
            pend = g("r_pending")
            assert pend <= self.options["sq_defer_max"], f"{pend:g} steps pending, cap {self.options['sq_defer_max']}"
        self.alphas.append(a)
        self._apply_round(a, o["lr"], o["residual"], ls)

    def op_async(self, o):
        c, h = self._bagc(), self.v["H"]
        r = self.v["Y"] - self.v["F"]
        s2 = float(np.sum(c * h * h))
        want = min(max(float(np.sum(c * r * h)) / s2, 0.0), 100.0) if s2 > 0 else 1.0
        if self.ctx is None:
            a, ls = want, None
        else:
            self.ctx.gbm_round_squared_async(o["lr"])
            a, ls = self.ctx.gbm_round_result()
            self.observed.append((len(self.log), "async", np.array([a, ls])))
            # Σrh over fp32 rows cancels: bound it by the rows' rounding, Σ|r h| 4·ε32, over Σh²
            err = 4 * EPS32 * float(np.sum(c * (np.abs(r) + 4 * EPS32 * self.m["R"] + np.abs(self.v["Y"])) *
                                           np.abs(h))) / s2 if s2 > 0 else 0.0
            assert abs(a - want) <= 1e-6 * abs(want) + err + 1e-12, f"async alpha {a!r}, closed form {want!r}"
        self.alphas.append(a)
        c = float(np.float32(o["lr"] * a))
        self._step_F(c)
        self._set_R_derived(False)
        if ls is not None:
            self._close(ls, float(np.sum(0.5 * (self.v["Y"] - self.v["F"]) ** 2)), "async loss")

    def op_brent(self, o):
        if self.ctx is not None:
            a, obj, ne = self.ctx.gbm_linesearch_brent(0.0, 100.0, 1.0, TOL, TOL, 100)
            self.observed.append((len(self.log), "brent", np.array([a, obj, ne])))
            self._check_alpha(a, "brent")
            self._close(obj, self._objective(a), "brent objective", abs(self._objective(a)) + 1e-3)

    def op_ls_newton(self, o):
        if self.ctx is not None:
            a, obj, ne = self.ctx.gbm_linesearch_newton(0.0, 100.0, 1.0, TOL, TOL, 100)
            self.observed.append((len(self.log), "ls_newton", np.array([a, obj, ne])))
            fa, fw = self._objective(a), self._objective(self._alpha_model())
            assert fa <= fw + RTOL * (abs(fw) + 1e-3), f"newton line search: objective {fa!r}, oracle {fw!r}"

    def op_eval(self, o):
        if self.ctx is not None:
            lo, g = self.ctx.gbm_linesearch_eval([o["alpha"]])
            self.observed.append((len(self.log), "eval", np.array([lo, g[0]])))
            self._close(lo, self._objective(o["alpha"]), "linesearch_eval", abs(self._objective(o["alpha"])) + 1e-3)

    def op_eval2(self, o):
        if self.ctx is not None:
            lo, d1, d2 = self.ctx.gbm_linesearch_eval2(o["alpha"])
            self.observed.append((len(self.log), "eval2", np.array([lo, d1, d2])))
            want = self._objective(o["alpha"]) * self._wsum()
            self._close(lo * self._wsum(), want, "linesearch_eval2", abs(want) + 1e-3)

    def op_stats(self, o):
        if self.ctx is not None:
            s = self.ctx.gbm_linesearch_stats()
            self.observed.append((len(self.log), "stats", s.copy()))
            c, h = self._bagc(), self.v["H"]
            r = self.v["Y"] - self.v["F"]
            s0, s2 = float(np.sum(c * r * r)), float(np.sum(c * h * h))
            self._close(s[0], s0, "stats s0")
            self._close(s[1], float(np.sum(c * h * r)), "stats s1", float(np.sqrt(s0 * s2)))
            self._close(s[2], s2, "stats s2")
            self._close(s[3], self._wsum(), "stats wsum")

    def op_set_bag(self, o):
        if o["seed"] is None:
            if self.ctx is not None:
                self.ctx.gbm_set_bag(None)
            self.bag = None
        else:
            counts = values("bag", o["seed"], self.n)
            if self.ctx is not None:
                self.ctx.gbm_set_bag(counts)
            self.bag = d64(counts)

    def op_set_param(self, o):
        if self.ctx is not None:
            self.ctx.gbm_set_loss_param(o["param"])
        self.param = o["param"]

    def op_absq(self, o):
        if self.ctx is not None:
            got = self.ctx.gbm_abs_residual_quantile(o["q"])
            self.observed.append((len(self.log), "absq", np.array([got])))
            d = np.abs(self.v["Y"] - self.v["F"])
            from spark_ensemble_b200.ensemble import exact_quantile
            want = exact_quantile(d, o["q"])
            err = 4 * EPS32 * float(np.max(self.m["F"] + np.abs(self.v["Y"])))
            assert abs(got - want) <= err, f"|y - F| quantile {got!r}, model {want!r}"

    def op_quantile(self, o):
        import spark_ensemble_b200._native as N
        if self.ctx is not None:
            got = self.ctx.quantile(getattr(N, "SLOT_" + o["slot"]), o["q"])
            self.observed.append((len(self.log), "quantile", np.array([got])))
            from spark_ensemble_b200.ensemble import exact_quantile
            assert got == exact_quantile(f32(self.v[o["slot"]]), o["q"]), "quantile"

    def op_read(self, o):
        import spark_ensemble_b200._native as N
        w = o["what"]
        if self.ctx is None:
            return
        if w in ("F", "R", "H", "WOUT"):
            self._check_slot(w, self._dev_read(w))
        elif w.startswith("sum"):
            sl = w[3:]
            got = self.ctx.slot_sum(getattr(N, "SLOT_" + sl))
            self.observed.append((len(self.log), w, np.array([got])))
            want = float(np.sum(self.v[sl]))
            assert abs(got - want) <= RTOL * float(np.sum(np.abs(self.v[sl]))) + \
                4 * EPS32 * float(np.sum(self.m[sl])) + 1e-30, f"slot_sum {sl}: {got!r}, model {want!r}"
        else:
            val = w == "mean_v"
            got = self.ctx.gbm_mean_loss(validation=val)
            self.observed.append((len(self.log), w, np.array([got])))
            y, F = (self.v["VY"], self.v["VF"]) if val else (self.v["Y"], self.v["F"])
            self._close(got, float(np.mean(NP.loss(self.loss, self.param, self._ye(y), F))), "mean loss")

    def _unchanged(self, fn, exc):
        """A failing call raises `exc`.  The model leaves every value as it was: walk B's reads after the call, and every
        later read, check that the device did too."""
        if self.ctx is None:
            return
        try:
            fn()
        except exc:
            pass
        else:
            raise AssertionError(f"expected {exc.__name__}")

    def op_fail_upload(self, o):
        import spark_ensemble_b200._native as N
        self._unchanged(lambda: self.ctx.upload(N.SLOT_R, np.zeros(2, np.float32), offset=self.n - 1), ValueError)

    def op_fail_quantile(self, o):
        import spark_ensemble_b200._native as N
        self._unchanged(lambda: self.ctx.quantile(N.SLOT_H, 1.5), ValueError)

    def op_fail_tol(self, o):
        self._unchanged(lambda: self.ctx.gbm_round(LR, True, 1e-17, 100, residual=o["residual"]), ValueError)

    def op_fail_maxeval(self, o):
        import spark_ensemble_b200._native as N
        self._unchanged(lambda: self.ctx.gbm_round(LR, True, 1e-12, 1, residual=o["residual"]), N.ConvergenceError)

    def op_opt(self, o):
        if self.ctx is not None:
            self.ctx.set_option(o["key"], o["value"])
        self.options[o["key"]] = o["value"]

    # ---- an independent recomputation of F (CPU test)
    def replay_F(self):
        F = None
        for s in self.steps:
            if s[0] == "write":
                F = s[1].copy()
            elif s[0] == "patch":
                F[s[1]:s[1] + s[2].size] = s[2]
            else:
                F = F + s[1] * s[2]
        return F
