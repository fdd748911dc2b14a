"""Plain numpy restatement of the device classification-tree learner (DESIGN.md §3 "Device classification-tree fit"):
Spark 3.3's RandomForest.run for one DecisionTreeClassifier tree (gini or entropy impurity, continuous features,
featureSubsetStrategy "all", prune = true), over the split candidates of np_tree.candidates.  Written for clarity, not
speed: loops over nodes, columns, candidates and classes, fp64 sums with numpy.  Independent of the product code."""
from __future__ import annotations

import math

import numpy as np

from .np_tree import EPS, candidates, ranks  # noqa: F401  (the candidates and ranks are the regressor's)
from .np_tree import Nodes, route, row_stats, send, tau, ulps32, walk  # noqa: F401
from .np_tree import leaf_of as np_leaf_of


def impurity(n, kind: str) -> float:
    """Spark's Gini / Entropy calculate(): classes in order, classes with zero weight skipped, 0 when W == 0."""
    W = float(sum(n))
    if W == 0:
        return 0.0
    imp = 1.0 if kind == "gini" else 0.0
    for c in n:
        if c == 0:
            continue
        f = c / W
        imp -= f * f if kind == "gini" else f * (math.log(f) / math.log(2))
    return imp


def label_of(n) -> int:
    """indexOfLargestArrayElement: the first class of the largest weight."""
    return int(np.argmax(np.asarray(n, dtype=np.float64)))


def proba_of(n) -> np.ndarray:
    """predictRaw = class weights, then normalizeToProbabilitiesInPlace; fp32 of the fp64 quotients (0 when W == 0)."""
    n = np.asarray(n, dtype=np.float64)
    W = n.sum()
    return np.zeros(n.size, dtype=np.float32) if W == 0 else (n / W).astype(np.float32)


def fit(rank_cols, ncand, y, num_classes, w=None, counts=None, impurity_kind="gini", max_depth=5, min_instances=1,
        min_info_gain=0.0, min_weight_fraction=0.0):
    """One tree over the ranks: rank_cols[k] are the ranks of subspace column k, ncand[k] its candidate count, y the
    class indices.  Returns the pruned tree in BFS order: feature, bin (rank threshold), left, right, label, proba
    ([n, K] fp32), cw ([n, K] fp64 class weights), gain, and `info`: per searched node, (best, second best) valid gain,
    the second best over the splits that partition the node's rows differently from the best."""
    K = int(num_classes)
    y = np.asarray(y, dtype=np.float32).astype(np.int64)
    n = y.size
    w = np.ones(n) if w is None else np.asarray(w, dtype=np.float32).astype(np.float64)
    c = np.ones(n) if counts is None else np.asarray(counts, dtype=np.float32).astype(np.float64)
    R = [np.asarray(a, dtype=np.int64) for a in rank_cols]
    onehot = np.zeros((n, K))
    onehot[np.arange(n), y] = 1.0

    def stats(rows):  # (rawCount, class weights)
        return c[rows].sum(), (onehot[rows] * (c[rows] * w[rows])[:, None]).sum(axis=0)

    root_rows = np.flatnonzero(c > 0)
    rc, cw = stats(root_rows)
    nodes = [{"rows": root_rows, "count": rc, "cw": cw, "depth": 0, "search": max_depth > 0}]
    w_root = cw.sum()
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
                cnt_rank = np.bincount(rk, weights=c[rows], minlength=256)
                cls_rank = np.stack([np.bincount(rk, weights=onehot[rows, j] * c[rows] * w[rows], minlength=256)
                                     for j in range(K)], axis=1)
                cum_c, cum_cls = np.cumsum(cnt_rank), np.cumsum(cls_rank, axis=0)
                tot_c, tot = cum_c[-1], cum_cls[-1]
                imp = impurity(tot, impurity_kind)
                for j in range(ncand[k]):
                    if j > 0 and cnt_rank[j] == 0:
                        continue  # no in-bag row ranks j: the same partition (and gain) as candidate j - 1
                    left = cum_cls[j]
                    right = tot - left
                    lw, rw = left.sum(), right.sum()
                    if cum_c[j] < min_instances or tot_c - cum_c[j] < min_instances:
                        continue
                    if lw < min_weight_fraction * w_root or rw < min_weight_fraction * w_root:
                        continue
                    tw = lw + rw
                    g = imp - lw / tw * impurity(left, impurity_kind) - rw / tw * impurity(right, impurity_kind)
                    if g < min_info_gain:
                        continue
                    valid.append((g, tuple(left)))
                    if g > best:
                        best, choice = g, (k, j, rk <= j, tuple(left))
            if choice is not None:  # runner-up among the splits that send other rows left (not a duplicate column)
                second = max([g for g, key in valid if key != choice[3]], default=-np.inf)
            info[i] = (best, second)
            if choice is None or not best > 0:
                continue
            k, j, m, _ = choice
            nd.update(leaf=False, col=k, bin=j, gain=best)
            d = nd["depth"] + 1
            for side, sel in (("left", m), ("right", ~m)):
                crow = rows[sel]
                cc, ccw = stats(crow)
                child = {"rows": crow, "count": cc, "cw": ccw, "depth": d,
                         "search": d < max_depth and not abs(impurity(ccw, impurity_kind)) < EPS}
                nd[side] = len(nodes)
                nodes.append(child)
                nxt.append(nd[side])
        level = nxt
    for nd in nodes:
        nd["label"] = label_of(nd["cw"])
    # prune bottom-up (LearningNode.toNode): two leaf children with equal labels make the node a leaf that keeps the
    # children's label and its own class weights
    for i in range(len(nodes) - 1, -1, -1):
        nd = nodes[i]
        if nd["leaf"]:
            continue
        a, b = nodes[nd["left"]], nodes[nd["right"]]
        if a["leaf"] and b["leaf"] and a["label"] == b["label"]:
            nd["leaf"] = True
            nd["merged"] = True
            nd["label"] = a["label"]
    order, q = [], [0]
    while q:
        i = q.pop(0)
        order.append(i)
        if not nodes[i]["leaf"]:
            q += [nodes[i]["left"], nodes[i]["right"]]
    pos = {i: p for p, i in enumerate(order)}
    T = {"feature": [], "bin": [], "left": [], "right": [], "label": [], "proba": [], "cw": [], "gain": [],
         "merged": [], "info": []}
    for i in order:
        nd = nodes[i]
        leaf = nd["leaf"]
        T["feature"].append(-1 if leaf else nd["col"])
        T["bin"].append(0 if leaf else nd["bin"])
        T["left"].append(0 if leaf else pos[nd["left"]])
        T["right"].append(0 if leaf else pos[nd["right"]])
        T["label"].append(nd["label"])
        T["proba"].append(proba_of(nd["cw"]))
        T["cw"].append(nd["cw"])
        T["gain"].append(0.0 if leaf else nd["gain"])
        T["merged"].append(bool(nd.get("merged", False)))
        T["info"].append(info.get(i))
    out = {k: np.asarray(v) for k, v in T.items() if k != "info"}
    out["proba"] = out["proba"].reshape(len(order), K).astype(np.float32)
    out["cw"] = out["cw"].reshape(len(order), K)
    out["info"] = T["info"]
    return out


def arrays(tree, cands) -> dict:
    """The restatement's tree in the array form a device fit returns (cands[k]: candidates of subspace column k)."""
    thr = np.array([cands[f][b] if f >= 0 else 0.0 for f, b in zip(tree["feature"], tree["bin"])], np.float32)
    return {"feature": tree["feature"].astype(np.int32), "threshold": thr, "left": tree["left"].astype(np.int32),
            "right": tree["right"].astype(np.int32), "value": tree["label"].astype(np.float32),
            "values": tree["proba"].astype(np.float32), "class_weights": tree["cw"].astype(np.float64),
            "gain": tree["gain"].astype(np.float64)}


# ---- audit of a fitted tree -------------------------------------------------------------------------------------
CW_RTOL = 1e-12  # class weights, relative to the parent's weight: a right child's are the parent's minus the left's


def labels_like(nk, label, tol) -> bool:
    """Whether the first-arg-max rule over class weights nk, known within tol, may give `label`: it is a maximum
    within 2·tol, and no earlier class is larger, nor exactly equal (an exact tie goes to the first class)."""
    nk = np.asarray(nk, np.float64)
    if not nk[label] >= nk.max() - 2 * tol:
        return False
    e = nk[:label]
    return not np.any((e > nk[label] + 2 * tol) | (e == nk[label]))


def _impurity_rows(nm, kind):
    """impurity() of every row of nm ([m, K] class weights), vectorised (class terms summed in numpy's order)."""
    W = nm.sum(axis=-1)
    with np.errstate(all="ignore"):
        f = np.where(nm > 0, nm / W[..., None], 0.0)
        if kind == "gini":
            v = 1.0 - (f * f).sum(axis=-1)
        else:
            v = -np.where(f > 0, f * np.log2(np.where(f > 0, f, 1.0)), 0.0).sum(axis=-1)
    return np.where(W == 0, 0.0, v)


def _gains(per, ncand, kind, p, w_root):
    """Gain of every candidate of one column from the node's per-rank sums per [256][K + 1] (c, then c·w per class):
    -inf where not valid, and where no row ranks j > 0."""
    if ncand == 0:
        return np.full(0, -np.inf)
    cnt = per[:, 0]
    cum, cc = np.cumsum(per[:, 1:], axis=0), np.cumsum(cnt)
    tot = cum[-1]
    ls, lc = cum[:ncand], cc[:ncand]
    rs, rc = tot - ls, cc[-1] - lc
    lw, rw = ls.sum(axis=1), rs.sum(axis=1)
    with np.errstate(all="ignore"):
        tw = lw + rw
        g = _impurity_rows(tot, kind) - lw / tw * _impurity_rows(ls, kind) - rw / tw * _impurity_rows(rs, kind)
        ok = (lc >= p["min_instances"]) & (rc >= p["min_instances"])
        ok &= (lw >= p["min_weight_fraction"] * w_root) & (rw >= p["min_weight_fraction"] * w_root)
        ok &= g >= p["min_info_gain"]
    ok &= (np.arange(ncand) == 0) | (cnt[:ncand] > 0)
    return np.where(ok, g, -np.inf)


def _column_gains(rk, yk, c, cw, K, ncand, kind, p, w_root):
    per = np.concatenate([np.bincount(rk, weights=c, minlength=256)[:, None],
                          np.bincount(rk * K + yk, weights=cw, minlength=256 * K).reshape(256, K)], axis=1)
    return _gains(per, ncand, kind, p, w_root)


def audit(tree, X, cands, sub, labels, w=None, counts=None, params=None, out=None, out_proba=None,
          exact=False) -> int:
    """Checks a fitted classification tree (the array form of a device fit: feature = subspace index, fp32 threshold,
    label `value`, fp32 `values`, fp64 `class_weights` and gain) from the rows each node receives, with fp64 numpy and
    nothing of the fit but its arrays; returns the number of nodes audited (every node).  Independent of which of two
    near-equal splits the fit took:
      statistics  class_weights are Σ c·w of the node's in-bag rows per class within CW_RTOL of the parent's weight
                  (equal when `exact`); values are fp32(n_k / W) within 1 ulp plus what that rounding of n_k and W
                  carries into the quotient (equal when `exact`; 0 when W == 0);
                  the label is the first arg-max, up to classes within that rounding (an exact tie goes to the
                  first class); a pruned leaf's statistics are those of all its rows;
      splits      as np_tree.audit: a first candidate, Spark's validity rules, the gain within τ, nothing better by
                  more than τ, the clear winner taken;
      leaves      depth maxDepth, or |impurity| < 2⁻⁵² + τ, or no valid split with gain > τ, or a pruned node: a
                  subtree the fit can grow on its rows (the remaining depth) has every leaf of its label -- at a near
                  tie, one of the tied choices must lead there, not merely any choice;
      output      out / out_proba (when given, out_proba [K, n]) are every row's leaf label / values, bit for bit.
    τ = TAU_C · 2⁻⁵² · (1 + √m), times log₂K for entropy (np_tree.TAU_C).  params holds num_classes, impurity,
    max_depth, min_instances, min_info_gain and min_weight_fraction.  The checks run on per-node sums (check);
    oracle/tree_audit.py takes the same sums over row chunks."""
    K = int(params["num_classes"])
    R, ncand, bins = route(tree, X, cands, sub)
    audited = check(tree, bins, ncand, row_stats(R, K, labels, w, counts), params, exact)
    leaf = np_leaf_of(tree, R, bins)
    if out is not None:
        np.testing.assert_array_equal(np.asarray(out, np.float32), tree["value"][leaf].astype(np.float32))
    if out_proba is not None:
        np.testing.assert_array_equal(np.asarray(out_proba, np.float32).reshape(K, leaf.size),
                                      np.asarray(tree["values"], np.float32)[leaf].T)
    return audited


def check(tree, bins, ncand, stats, params, exact=False) -> int:
    """The checks of audit() on a classification tree from the statistics of its nodes (stats: as np_tree.row_stats
    returns), asked again for the children of the splits a pruned leaf may have grown.  Returns the number of nodes
    checked (every node)."""
    p = {"impurity": "gini", "max_depth": 5, "min_instances": 1, "min_info_gain": 0.0, "min_weight_fraction": 0.0}
    p.update(params or {})
    K, kind = int(p["num_classes"]), p["impurity"]
    f, gain = tree["feature"], tree["gain"]
    scale = 1.0 if kind == "gini" else math.log2(K)
    nodes, order = Nodes.of_tree(tree, bins)
    tot, hist = stats(nodes, {v for v, i in enumerate(order) if f[i] >= 0 or nodes.depth[v] < p["max_depth"]})
    tot = {v: tot[v] for v in range(len(order))}
    w_root = tot[0][1:K + 1].sum()
    parent_w = {0: w_root}

    def splits(v):
        out = []
        for kk in range(len(ncand)):
            gk = _gains(hist[v][kk], ncand[kk], kind, p, w_root)
            out += [(float(gk[j]), kk, int(j)) for j in np.flatnonzero(np.isfinite(gk))]
        out.sort(key=lambda x: (-x[0], x[1], x[2]))
        return out

    need = set()

    def collapses(v, label, pw):
        """Whether the fit, growing a subtree on node v's in-bag rows (pw: the parent's weight), can end with every
        leaf of it labelled `label`, so that pruning merges it into one leaf; None while the statistics of a node it
        depends on are not known yet (they are then in `need`).  Where rounding may decide (gains within τ or 1e-7 of
        the best, impurity within τ of the purity rule, a gain within τ of 0), every choice the fit may make is tried;
        anywhere else there is one."""
        depth = nodes.depth[v]
        if v not in tot or (depth < p["max_depth"] and v not in hist):
            need.add(v)
            return None
        nk = tot[v][1:K + 1]
        labelled = labels_like(nk, label, CW_RTOL * pw)
        t = tau(tot[v][-1], scale)
        imp = abs(impurity(nk, kind))
        if depth >= p["max_depth"] or imp < EPS - t:
            return labelled
        cand = splits(v)
        best = cand[0][0] if cand else -np.inf
        if labelled and (imp < EPS + t or not best > t):
            return True  # the fit may stop here: pure within rounding, or no split clearly above 0
        seen, unknown = set(), False
        for g, k, j in cand:
            if g < best - max(t, 1e-7 * abs(best)) or not g > -t:
                break
            key = tuple(hist[v][k][:j + 1].sum(axis=0))  # the partition, by the sums of its left side
            if key in seen:
                continue
            seen.add(key)
            W = nk.sum()
            a = collapses(nodes.child(v, k, j, 1), label, W)
            b = collapses(nodes.child(v, k, j, 0), label, W) if a is not False else False
            if a and b:
                return True
            unknown |= a is None or b is None
        return None if unknown else False

    pending = []
    for v, i in enumerate(order):
        depth = nodes.depth[v]
        nk = tot[v][1:K + 1]
        W = nk.sum()
        t = tau(tot[v][-1], scale)
        tol = 0.0 if exact else CW_RTOL * parent_w[v]
        dev_cw = np.asarray(tree["class_weights"][i], np.float64)
        assert np.all(np.abs(dev_cw - nk) <= tol), f"node {i}: class weights {dev_cw} against {nk}"
        want = np.zeros(K, np.float32) if W == 0 else (nk / W).astype(np.float32)
        d = max(ulps32(a, b) for a, b in zip(tree["values"][i], want))
        if exact or W == 0:
            assert d == 0, f"node {i}: values {tree['values'][i]} are {d} ulps from {want}"
        elif d > 1:  # a small class of a right child: n_k = parent's - left's carries the parent's rounding, tol
            err = np.abs(np.asarray(tree["values"][i], np.float64) - nk / W)
            assert np.all(err <= np.spacing(want).astype(np.float64) + 2 * tol / W), \
                f"node {i}: values {tree['values'][i]} are {d} ulps from {want}, beyond the class weights' rounding"
        label = int(tree["value"][i])
        assert label == tree["value"][i] and 0 <= label < K, f"node {i}: label {tree['value'][i]}"
        if exact:
            assert label == label_of(nk), f"node {i}: label {label}, the first arg-max is {label_of(nk)}"
        else:  # a pruned leaf too: its children's label beats every earlier class in each child, so in their sum
            assert labels_like(nk, label, tol), f"node {i}: label {label} is not the first arg-max of {nk}"
        imp = impurity(nk, kind)
        if f[i] < 0:
            if depth < p["max_depth"] and not abs(imp) < EPS + t:
                cand = splits(v)
                best = cand[0][0] if cand else -np.inf
                if best > t:  # only a pruned node: its subtree's leaves all carry one label
                    pending.append((i, v, label, parent_w[v], best, t))
            continue
        assert depth < p["max_depth"], f"node {i}: a split at depth {depth}"
        k, b = int(f[i]), int(bins[i])
        per = hist[v][k]
        assert b == 0 or per[b, 0] > 0, f"node {i}: candidate {b} repeats candidate {b - 1}'s partition"
        # each side summed over its own ranks: a class absent from a side weighs exactly 0 there (the parent's sum
        # minus the other side's, summed in another order, may leave -1e-16, outside the impurities' domain)
        left, right = per[:b + 1].sum(axis=0), per[b + 1:].sum(axis=0)
        lk, rk = left[1:], right[1:]
        lc, rc = left[0], right[0]
        slack = 1e-12 * w_root
        assert lc >= p["min_instances"] and rc >= p["min_instances"], f"node {i}: rawCount {lc}, {rc}"
        assert min(lk.sum(), rk.sum()) >= p["min_weight_fraction"] * w_root - slack, f"node {i}: weights"
        assert gain[i] >= p["min_info_gain"] and gain[i] > 0, f"node {i}: gain {gain[i]}"
        lw, rw = lk.sum(), rk.sum()
        g = imp - lw / (lw + rw) * impurity(lk, kind) - rw / (lw + rw) * impurity(rk, kind)
        assert abs(g - gain[i]) <= t, f"node {i}: gain {gain[i]!r}, recomputed {g!r}, τ = {t:.3g}"
        cand = splits(v)
        assert cand and cand[0][0] <= g + t, f"node {i}: split {cand[0]} beats gain {g!r} by more than τ = {t:.3g}"
        if len(cand) == 1 or cand[0][0] - cand[1][0] > t:
            assert (k, b) == cand[0][1:], f"node {i}: the clear winner is {cand[0]}, the fit took ({k}, {b})"
        parent_w[order.index(int(tree["left"][i]))] = parent_w[order.index(int(tree["right"][i]))] = W
    # pruned leaves: grow what the fit may have grown below them, one level of statistics per round
    while pending:
        need.clear()
        left_over = []
        for i, v, label, pw, best, t in pending:
            ok = collapses(v, label, pw)
            assert ok is not False, f"node {i}: a leaf, but a split of gain {best!r} > τ = {t:.3g} leads to other labels"
            if ok is None:
                left_over.append((i, v, label, pw, best, t))
        pending = left_over
        if pending:
            more_tot, more_hist = stats(nodes, {u for u in need if nodes.depth[u] < p["max_depth"]})
            tot.update({u: more_tot[u] for u in need})
            hist.update(more_hist)
    return len(order)


def leaf_of(tree, rank_cols) -> np.ndarray:
    """Index of every row's leaf, walking the ranks: left when rank <= bin."""
    Rk = np.stack([np.asarray(a, dtype=np.int64) for a in rank_cols])
    n = Rk.shape[1]
    node = np.zeros(n, dtype=np.int64)
    for _ in range(64):
        f = tree["feature"][node]
        live = f >= 0
        if not live.any():
            break
        rk = Rk[np.maximum(f, 0), np.arange(n)]
        go = np.where(rk <= tree["bin"][node], tree["left"][node], tree["right"][node])
        node = np.where(live, go, node)
    return node
