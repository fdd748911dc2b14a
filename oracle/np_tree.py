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


def arrays(tree, cands) -> dict:
    """The restatement's tree in the array form a device fit returns: fp32 thresholds (cands[k] are the candidates of
    subspace column k), fp32 values."""
    thr = np.array([cands[f][b] if f >= 0 else 0.0 for f, b in zip(tree["feature"], tree["bin"])], np.float32)
    return {"feature": tree["feature"].astype(np.int32), "threshold": thr, "left": tree["left"].astype(np.int32),
            "right": tree["right"].astype(np.int32), "value": tree["pred"].astype(np.float32),
            "gain": tree["gain"].astype(np.float64)}


def cut(tree, i) -> tuple:
    """The array-form tree with the subtree below internal node i removed and i made a leaf (its statistics as they
    are; BFS order and child indices kept consistent).  Returns (tree, i's new index)."""
    f = tree["feature"]
    drop, stack = set(), [int(tree["left"][i]), int(tree["right"][i])]
    while stack:
        j = stack.pop()
        drop.add(j)
        if f[j] >= 0:
            stack += [int(tree["left"][j]), int(tree["right"][j])]
    keep = [j for j in range(f.size) if j not in drop]
    new = {j: q for q, j in enumerate(keep)}
    out = {k: np.asarray(v)[keep].copy() for k, v in tree.items()}
    for q, j in enumerate(keep):
        if f[j] >= 0 and j != i:
            out["left"][q], out["right"][q] = new[int(tree["left"][j])], new[int(tree["right"][j])]
    q = new[i]
    out["feature"][q], out["threshold"][q], out["left"][q], out["right"][q], out["gain"][q] = -1, 0, 0, 0, 0
    return out, q


# ---- audit of a fitted tree -------------------------------------------------------------------------------------
# τ, the rounding bound of a gain: TAU_C · 2⁻⁵² · (1 + √m) · scale, m the node's in-bag rows.  The kernels sum the
# node's fp64 statistics with atomics in no fixed order, the audit with numpy in another; each sum carries a rounding
# error that grows like √m (a random walk of 2⁻⁵³-relative steps), and the gain formula adds a few roundings of its
# own.  The regression scale is the node's second moment Q/W: the gain cancels terms of that size (Q/W − S²/W²), so
# its error scales with Q/W, not with the variance.  TAU_C = 32 covers the walk many times over.
TAU_C = 32.0


def ulps32(a, b) -> float:
    """Distance of two fp32 values in units in the last place; 0 for two NaNs, inf for a NaN and a number."""
    a, b = np.float32(a), np.float32(b)
    if np.isnan(a) or np.isnan(b):
        return 0.0 if np.isnan(a) and np.isnan(b) else np.inf

    def key(x):
        i = int(np.array(x, np.float32).view(np.int32))
        return i if i >= 0 else -(i & 0x7FFFFFFF)
    return float(abs(key(a) - key(b)))


def tau(m, scale) -> float:
    return TAU_C * EPS * (1.0 + np.sqrt(m)) * abs(scale)


def _gains(per, ncand, p, w_root):
    """Gain of every candidate of one column from the node's per-rank sums per [256][4] (c, c·w, c·w·r, c·w·r²):
    -inf where not valid, and where no row ranks j > 0 (candidate j then repeats candidate j - 1's partition, which
    the fit takes first)."""
    if ncand == 0:
        return np.full(0, -np.inf)
    cum = np.cumsum(per, axis=0)
    tot = cum[-1]
    ls = cum[:ncand]
    rs = tot - ls
    with np.errstate(all="ignore"):
        def imp(s):
            return np.where(s[..., 1] == 0, 0.0, (s[..., 3] - s[..., 2] * s[..., 2] / s[..., 1]) / s[..., 1])
        g = imp(tot) - ls[:, 1] / tot[1] * imp(ls) - rs[:, 1] / tot[1] * imp(rs)
        ok = (ls[:, 0] >= p["min_instances"]) & (rs[:, 0] >= p["min_instances"])
        ok &= (ls[:, 1] >= p["min_weight_fraction"] * w_root) & (rs[:, 1] >= p["min_weight_fraction"] * w_root)
        ok &= g >= p["min_info_gain"]
    ok &= (np.arange(ncand) == 0) | (per[:ncand, 0] > 0)
    return np.where(ok, g, -np.inf)


def _column_gains(rk, c, cw, r, ncand, p, w_root):
    """_gains over a node's in-bag rows (rk their ranks in the column)."""
    per = np.stack([np.bincount(rk, weights=v, minlength=256) for v in (c, cw, cw * r, cw * r * r)], axis=1)
    return _gains(per, ncand, p, w_root)


def _node_search(R, ncand, ib, c, cw, r, p, w_root):
    """search() over a node's in-bag rows ib."""
    return search([np.stack([np.bincount(R[k][ib], weights=v[ib], minlength=256) for v in (c, cw, cw * r, cw * r * r)],
                            axis=1) for k in range(len(R))], ncand, p, w_root)


def search(hist, ncand, p, w_root, gains=_gains):
    """(gain, column, candidate) of every valid split of a node (hist: its [S][256][stats] sums per column and rank),
    sorted by gain descending, then column, candidate."""
    out = []
    for k in range(len(ncand)):
        g = gains(hist[k], ncand[k], p, w_root)
        for j in np.flatnonzero(np.isfinite(g)):
            out.append((float(g[j]), k, int(j)))
    out.sort(key=lambda t: (-t[0], t[1], t[2]))
    return out


def route(tree, X, cands, sub):
    """Ranks of the subspace columns and, per node, the candidate index of its threshold (which must be one)."""
    X = np.asarray(X, dtype=np.float32)
    sub = np.asarray(sub).reshape(-1)
    R = [ranks(X[:, col], cands[col]) for col in sub]
    ncand = [np.asarray(cands[col]).size for col in sub]
    return R, ncand, bins_of(tree, [cands[col] for col in sub])


def bins_of(tree, cands):
    """Per node, the candidate index of its threshold, which must be a candidate of its column (cands[k]: the
    candidates of subspace column k)."""
    bins = np.zeros(tree["feature"].size, np.int64)
    for i in np.flatnonzero(tree["feature"] >= 0):
        cc = np.asarray(cands[tree["feature"][i]], np.float32)
        b = int(np.searchsorted(cc, np.float32(tree["threshold"][i])))
        assert b < cc.size and cc[b] == np.float32(tree["threshold"][i]), f"node {i}: threshold is not a candidate"
        bins[i] = b
    return bins


def walk(tree, n):
    """Yields (node, rows, depth) of every node reached from the root, checking that each node is reached once."""
    seen = np.zeros(tree["feature"].size, bool)
    stack = [(0, np.arange(n), 0)]
    while stack:
        i, rows, depth = stack.pop()
        assert not seen[i], f"node {i} is reached twice"
        seen[i] = True
        go = yield i, rows, depth
        if tree["feature"][i] >= 0:
            stack.append((int(tree["right"][i]), rows[~go], depth + 1))
            stack.append((int(tree["left"][i]), rows[go], depth + 1))
    assert seen.all(), f"nodes {np.flatnonzero(~seen).tolist()} are not reached from the root"


# ---- per-node statistics of a tree's rows ----------------------------------------------------------------------
class Nodes:
    """A list of row sets: node 0 holds every row, node v > 0 the rows of parent[v] whose rank in subspace column
    col[v] is <= bin[v] (left[v]) or > bin[v].  A tree's nodes are one such list; the classifier's audit adds the
    children of the splits a pruned node may have grown."""

    def __init__(self):
        self.parent, self.col, self.bin, self.left, self.depth = [-1], [0], [0], [1], [0]
        self._key = {}

    def __len__(self):
        return len(self.parent)

    def child(self, v, k, b, left) -> int:
        key = (int(v), int(k), int(b), int(bool(left)))
        if key not in self._key:
            self._key[key] = len(self.parent)
            self.parent.append(key[0]); self.col.append(key[1]); self.bin.append(key[2]); self.left.append(key[3])
            self.depth.append(self.depth[key[0]] + 1)
        return self._key[key]

    @classmethod
    def of_tree(cls, tree, bins):
        """The nodes of a tree, after checking that every node is reached from the root once.  Returns (nodes,
        order): node v here is node order[v] of the tree, parents before children."""
        f = tree["feature"]
        nodes, seen, order = cls(), np.zeros(f.size, bool), [0]
        seen[0] = True
        for v, i in enumerate(order):
            if f[i] < 0:
                continue
            for side, j in ((1, int(tree["left"][i])), (0, int(tree["right"][i]))):
                assert 0 <= j < f.size and not seen[j], f"node {j} is reached twice"
                seen[j] = True
                nodes.child(v, f[i], bins[i], side)
                order.append(j)
        assert seen.all(), f"nodes {np.flatnonzero(~seen).tolist()} are not reached from the root"
        return nodes, order


def row_stats(R, K, labels, w=None, counts=None):
    """Statistics of Nodes over rows held in memory (R[k]: the ranks of subspace column k), as
    oracle.Oracle.tree_hist sums them over chunks: a function (nodes, want) -> (totals, hists), totals[v] the node's
    sums (c, c·w, c·w·r, c·w·r²) or (c, c·w per class), then Σ c·w·|r| and its in-bag row count; hists[v] for v in
    want its [S][256][stats] sums per column and rank.  K == 0: regression labels, else class indices."""
    y = np.asarray(labels, dtype=np.float32).astype(np.float64)
    n = y.size
    w = np.ones(n) if w is None else np.asarray(w, dtype=np.float32).astype(np.float64)
    c = np.ones(n) if counts is None else np.asarray(counts, dtype=np.float32).astype(np.float64)
    cw = c * w
    if K:
        per_row = np.zeros((n, K + 1))
        per_row[:, 0] = c
        per_row[np.arange(n), 1 + y.astype(np.int64)] = cw
    else:
        per_row = np.stack([c, cw, cw * y, cw * y * y], axis=1)
    rows = {}

    def stats(nodes, want):
        tot, hists = np.zeros((len(nodes), per_row.shape[1] + 2)), {}
        for v in range(len(nodes)):
            if v not in rows:
                p = nodes.parent[v]
                rows[v] = np.flatnonzero(c > 0) if p < 0 else \
                    rows[p][(R[nodes.col[v]][rows[p]] <= nodes.bin[v]) == bool(nodes.left[v])]
            ib = rows[v]
            tot[v, :-2] = per_row[ib].sum(axis=0)
            tot[v, -2] = 0.0 if K else (cw[ib] * np.abs(y[ib])).sum()
            tot[v, -1] = ib.size
            if v in want:
                hists[v] = np.stack([np.stack([np.bincount(R[k][ib], weights=per_row[ib, s], minlength=256)
                                               for s in range(per_row.shape[1])], axis=1) for k in range(len(R))])
        return tot, hists
    return stats


def check(tree, bins, ncand, stats, params=None, exact=False) -> int:
    """The checks of audit() on a regression tree from the statistics of its nodes (stats: as row_stats returns);
    bins[i] is node i's candidate index (bins_of), ncand[k] the candidate count of subspace column k.  Returns the
    number of nodes checked (every node)."""
    p = {"max_depth": 5, "min_instances": 1, "min_info_gain": 0.0, "min_weight_fraction": 0.0}
    p.update(params or {})
    f, value, gain = tree["feature"], tree["value"], tree["gain"]
    nodes, order = Nodes.of_tree(tree, bins)
    want = {v for v, i in enumerate(order) if f[i] >= 0 or nodes.depth[v] < p["max_depth"]}
    tot, hist = stats(nodes, want)
    w_root = tot[0, 1]
    parent = {}  # per node: its parent's (relative rounding bound, Σ c·w·|r|, W)
    for v, i in enumerate(order):
        depth = nodes.depth[v]
        st, a_abs, m_rows = tot[v, :4], tot[v, 4], tot[v, 5]
        W = st[1]
        t = tau(m_rows, st[3] / W) if W != 0 else 0.0
        if i == 0:
            parent[0] = (tau(m_rows, 1.0), a_abs, W)
        if W == 0:
            assert np.isnan(value[i]), f"node {i}: no in-bag weight, value {value[i]} (S/W is NaN)"
        else:
            m = st[2] / W
            d = ulps32(value[i], np.float32(m))
            if exact:
                assert d == 0, f"node {i}: value {value[i]!r} is not fp32(S/W) = {m!r}"
            elif d > 1:  # a right child's S and W are the parent's minus the left's: the parent's rounding
                rel, a_p, w_p = parent[i]
                assert abs(float(value[i]) - m) <= float(np.spacing(np.float32(m))) + rel * (a_p + abs(m) * w_p) / W, \
                    f"node {i}: value {value[i]!r} is {d} ulps from fp32(S/W) = {m!r}, beyond the sums' rounding"
        if f[i] < 0:
            if depth < p["max_depth"] and not abs(_impurity(st)) < EPS + t:
                cand = search(hist[v], ncand, p, w_root)
                assert not cand or not cand[0][0] > t, f"node {i}: a leaf, but split {cand[0]} has gain > τ = {t:.3g}"
            continue
        assert depth < p["max_depth"], f"node {i}: a split at depth {depth}"
        k, b = int(f[i]), int(bins[i])
        per = hist[v][k]
        assert b == 0 or per[b, 0] > 0, f"node {i}: candidate {b} repeats candidate {b - 1}'s partition"
        ls = per[:b + 1].sum(axis=0)
        rs = st - ls
        slack = 1e-12 * w_root
        assert ls[0] >= p["min_instances"] and rs[0] >= p["min_instances"], f"node {i}: rawCount {ls[0]}, {rs[0]}"
        assert min(ls[1], rs[1]) >= p["min_weight_fraction"] * w_root - slack, f"node {i}: weights {ls[1]}, {rs[1]}"
        assert gain[i] >= p["min_info_gain"] and gain[i] > 0, f"node {i}: gain {gain[i]}"
        g = _impurity(st) - ls[1] / W * _impurity(ls) - rs[1] / W * _impurity(rs)
        assert abs(g - gain[i]) <= t, f"node {i}: gain {gain[i]!r}, recomputed {g!r}, τ = {t:.3g}"
        cand = search(hist[v], ncand, p, w_root)
        assert cand and cand[0][0] <= g + t, f"node {i}: split {cand[0]} beats gain {g!r} by more than τ = {t:.3g}"
        if len(cand) == 1 or cand[0][0] - cand[1][0] > t:
            assert (k, b) == cand[0][1:], f"node {i}: the clear winner is {cand[0]}, the fit took ({k}, {b})"
        parent[int(tree["left"][i])] = parent[int(tree["right"][i])] = (tau(m_rows, 1.0), a_abs, W)
    return len(nodes)


def audit(tree, X, cands, sub, labels, w=None, counts=None, params=None, out=None, exact=False) -> int:
    """Checks a fitted regression tree (the array form of a device fit: feature = subspace index, fp32 threshold and
    value, fp64 gain) from the rows each node receives, with fp64 numpy and nothing of the fit but its arrays; returns
    the number of nodes audited (every node).  Independent of which of two near-equal splits the fit took:
      statistics  every node's value is within 1 fp32 ulp of fp32(S/W) of its in-bag rows, plus what the parent's
                  rounding carries into S/W (a right child's S and W are the parent's minus the left's): the
                  relative bound τ/scale of the parent's sums times (Σ c·w·|r| + |S/W|·W) of the parent, over W
                  (equal when `exact`, the sums then being exact); NaN when W == 0;
      splits      the threshold is a candidate with an in-bag row at its rank (the first candidate of its partition);
                  rawCount >= minInstancesPerNode and W >= minWeightFractionPerNode · W_root on both sides;
                  gain >= minInfoGain and > 0; the recomputed gain equals the returned one within τ; no (column,
                  candidate) of the subspace beats it by more than τ; a clear winner (gap > τ) is the one taken;
      leaves      depth maxDepth, or |impurity| < 2⁻⁵² + τ, or no valid split with gain > τ (a pruned node's best
                  split has children of equal means: gain 0 up to rounding);
      output      out (when given) is every row's leaf value, bit for bit.
    cands are the candidates of every column of X, sub the subspace; params holds max_depth, min_instances,
    min_info_gain and min_weight_fraction.  The checks run on per-node sums (check); oracle/tree_audit.py takes the
    same sums over row chunks."""
    R, ncand, bins = route(tree, X, cands, sub)
    audited = check(tree, bins, ncand, row_stats(R, 0, labels, w, counts), params, exact)
    if out is not None:
        np.testing.assert_array_equal(np.asarray(out, np.float32),
                                      tree["value"][leaf_of(tree, R, bins)].astype(np.float32))
    return audited


def leaf_of(tree, rank_cols, bins) -> np.ndarray:
    """Index of every row's leaf in an array-form tree (bins: its candidate indices), walking the ranks."""
    Rk = np.stack([np.asarray(a, dtype=np.int64) for a in rank_cols])
    n = Rk.shape[1]
    node = np.zeros(n, dtype=np.int64)
    for _ in range(64):
        f = tree["feature"][node]
        live = f >= 0
        if not live.any():
            break
        rk = Rk[np.maximum(f, 0), np.arange(n)]
        go = np.where(rk <= bins[node], tree["left"][node], tree["right"][node])
        node = np.where(live, go, node)
    return node


def send(it, go):
    """The next node of walk() after a split that sends the rows `go` left; None after the last."""
    try:
        return it.send(go)
    except StopIteration:
        return None


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
