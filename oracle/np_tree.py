"""Plain numpy restatement of the device regression-tree learner (DESIGN.md §3 "Device tree fit"): Spark 3.3's
RandomForest.run for one DecisionTreeRegressor tree (variance impurity, continuous features, featureSubsetStrategy
"all", prune = true), over the split candidates of findSplitsForContinuousFeature.  Written for clarity, not speed:
loops over nodes, columns and candidates, fp64 sums with numpy.  Independent of the product code."""
from __future__ import annotations

import numpy as np

EPS = 2.0 ** -52  # Utils.EPSILON: a child this pure becomes a leaf without a search


def candidates(sample_values, max_bins: int) -> np.ndarray:
    """findSplitsForContinuousFeature over one column's sample values; returns the fp32 candidates."""
    vals = {}
    for x in np.asarray(sample_values, dtype=np.float64).reshape(-1):
        if np.isnan(x):
            continue
        x = 0.0 if x == 0.0 else float(x)  # -0 -> +0
        vals[x] = vals.get(x, 0) + 1
    v = sorted(vals)
    c = [vals[x] for x in v]
    m = len(v) - 1
    if m <= 0:
        return np.zeros(0, dtype=np.float32)
    if m <= max_bins - 1:
        mids = [(v[i - 1] + v[i]) / 2.0 for i in range(1, m + 1)]
    else:
        stride = sum(c) / max_bins
        target = stride
        cur = c[0]
        mids = []
        for i in range(1, m + 1):
            prev = cur
            cur += c[i]
            if abs(prev - target) < abs(cur - target):
                mids.append((v[i - 1] + v[i]) / 2.0)
                target += stride
    out = []
    fmax = float(np.finfo(np.float32).max)
    for t in mids:
        t = min(max(t, -fmax), fmax)
        f = np.float32(t)
        if float(f) > t:
            f = np.nextafter(f, np.float32(-np.inf))
        if not out or f > out[-1]:
            out.append(f)
    return np.asarray(out, dtype=np.float32)


def ranks(x, cands) -> np.ndarray:
    """rank(x) = #{candidates < x}; NaN ranks 255 (right of every candidate)."""
    x = np.asarray(x, dtype=np.float32)
    r = np.searchsorted(np.asarray(cands, dtype=np.float32), x, side="left").astype(np.int64)
    r[np.isnan(x)] = 255
    return r


def _stats(r, w, c):
    cw = c * w
    return np.array([c.sum(), cw.sum(), (cw * r).sum(), (cw * r * r).sum()], dtype=np.float64)


def _impurity(s) -> float:
    return 0.0 if s[1] == 0 else (s[3] - s[2] * s[2] / s[1]) / s[1]


def fit(rank_cols, ncand, r, w=None, counts=None, max_depth=5, min_instances=1, min_info_gain=0.0,
        min_weight_fraction=0.0):
    """One tree over the ranks: rank_cols[k] are the ranks of subspace column k, ncand[k] its candidate count.
    Returns the tree in the array form of se_tree_predict (BFS order) with `bin` (rank threshold) instead of the fp32
    threshold, `pred` (fp64 prediction) and `info`: per searched node, (best, second best) valid gain, where the
    second best is taken over the splits that partition the node's rows differently from the best."""
    r = np.asarray(r, dtype=np.float32).astype(np.float64)
    n = r.size
    w = np.ones(n) if w is None else np.asarray(w, dtype=np.float32).astype(np.float64)
    c = np.ones(n) if counts is None else np.asarray(counts, dtype=np.float32).astype(np.float64)
    R = [np.asarray(a, dtype=np.int64) for a in rank_cols]
    inbag = c > 0
    # node: dict(rows, stats, depth, leaf, col, bin, gain, left, right)
    root_rows = np.flatnonzero(inbag)
    nodes = [{"rows": root_rows, "stats": _stats(r[root_rows], w[root_rows], c[root_rows]), "depth": 0,
              "search": max_depth > 0}]
    w_root = nodes[0]["stats"][1]
    info = {}
    level = [0]
    while level:
        nxt = []
        for i in level:
            nd = nodes[i]
            nd["leaf"] = True
            if not nd["search"]:
                continue
            rows = nd["rows"]
            best, second, choice = -np.inf, -np.inf, None
            valid = []
            for k in range(len(R)):
                if ncand[k] == 0:
                    continue
                rk = R[k][rows]
                cw = c[rows] * w[rows]
                per_rank = np.stack([np.bincount(rk, weights=v, minlength=256)
                                     for v in (c[rows], cw, cw * r[rows], cw * r[rows] * r[rows])], axis=1)
                cum = np.cumsum(per_rank, axis=0)
                tot = cum[-1]
                imp = _impurity(tot)
                for j in range(ncand[k]):
                    if j > 0 and per_rank[j, 0] == 0:
                        continue  # no in-bag row ranks j: the same partition (and gain) as candidate j - 1
                    ls = cum[j]
                    rs = tot - ls
                    if ls[0] < min_instances or rs[0] < min_instances:
                        continue
                    if ls[1] < min_weight_fraction * w_root or rs[1] < min_weight_fraction * w_root:
                        continue
                    g = imp - ls[1] / tot[1] * _impurity(ls) - rs[1] / tot[1] * _impurity(rs)
                    if g < min_info_gain:
                        continue
                    valid.append((g, tuple(ls)))
                    if g > best:
                        best, choice = g, (k, j, ls, rs, rk <= j)
            if choice is not None:  # runner-up among the splits that send other rows left (not a duplicate column)
                second = max([g for g, key in valid if key != tuple(choice[2])], default=-np.inf)
            info[i] = (best, second)
            if choice is None or not best > 0:
                continue
            k, j, ls, rs, m = choice
            nd.update(leaf=False, col=k, bin=j, gain=best)
            d = nd["depth"] + 1
            for side, st, sel in (("left", ls, m), ("right", rs, ~m)):
                child = {"rows": rows[sel], "stats": st, "depth": d,
                         "search": d < max_depth and not abs(_impurity(st)) < EPS}
                nd[side] = len(nodes)
                nodes.append(child)
                nxt.append(nd[side])
        level = nxt
    for nd in nodes:
        nd["pred"] = nd["stats"][2] / nd["stats"][1] if nd["stats"][1] != 0 else np.nan
    # prune bottom-up: an internal node with two leaf children of equal prediction becomes a leaf
    for i in range(len(nodes) - 1, -1, -1):
        nd = nodes[i]
        if nd["leaf"]:
            continue
        a, b = nodes[nd["left"]], nodes[nd["right"]]
        if a["leaf"] and b["leaf"] and a["pred"] == b["pred"]:
            nd["leaf"] = True
            nd["pred"] = a["pred"]
    # BFS numbering of what is left
    order, q = [], [0]
    while q:
        i = q.pop(0)
        order.append(i)
        if not nodes[i]["leaf"]:
            q += [nodes[i]["left"], nodes[i]["right"]]
    pos = {i: p for p, i in enumerate(order)}
    T = {"feature": [], "bin": [], "left": [], "right": [], "pred": [], "gain": [], "info": []}
    for i in order:
        nd = nodes[i]
        leaf = nd["leaf"]
        T["feature"].append(-1 if leaf else nd["col"])
        T["bin"].append(0 if leaf else nd["bin"])
        T["left"].append(0 if leaf else pos[nd["left"]])
        T["right"].append(0 if leaf else pos[nd["right"]])
        T["pred"].append(nd["pred"])
        T["gain"].append(0.0 if leaf else nd["gain"])
        T["info"].append(info.get(i))
    out = {k: np.asarray(v) for k, v in T.items() if k != "info"}
    out["info"] = T["info"]
    return out


def predict(tree, rank_cols) -> np.ndarray:
    """Leaf prediction (fp64) of every row, walking the ranks: left when rank <= bin."""
    R = np.stack([np.asarray(a, dtype=np.int64) for a in rank_cols])
    n = R.shape[1]
    node = np.zeros(n, dtype=np.int64)
    for _ in range(64):
        f = tree["feature"][node]
        live = f >= 0
        if not live.any():
            break
        rk = R[np.maximum(f, 0), np.arange(n)]
        go = np.where(rk <= tree["bin"][node], tree["left"][node], tree["right"][node])
        node = np.where(live, go, node)
    return tree["pred"][node]
