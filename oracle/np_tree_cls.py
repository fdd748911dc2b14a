"""Plain numpy restatement of the device classification-tree learner (DESIGN.md §3 "Device classification-tree fit"):
Spark 3.3's RandomForest.run for one DecisionTreeClassifier tree (gini or entropy impurity, continuous features,
featureSubsetStrategy "all", prune = true), over the split candidates of np_tree.candidates.  Written for clarity, not
speed: loops over nodes, columns, candidates and classes, fp64 sums with numpy.  Independent of the product code."""
from __future__ import annotations

import math

import numpy as np

from .np_tree import EPS, candidates, ranks  # noqa: F401  (the candidates and ranks are the regressor's)


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
