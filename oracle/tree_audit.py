"""The audit of a fitted tree (np_tree.audit, np_tree_cls.audit) over rows that do not fit in host memory at once:
the per-node statistics the checks read (np_tree.check, np_tree_cls.check) are summed chunk by chunk in fp64 by the
OpenMP oracle (orc_tree_hist), each row routed through the tree.  The checks are the same functions the in-memory
audit runs, so the two cannot disagree on the same sums.

A chunk is (R, labels, w, counts): R the [S][m] uint8 ranks of the subspace columns (Oracle.ranks), labels the
regression labels or class indices, w and counts the weights and bag multiplicities (None: 1)."""
from __future__ import annotations

import numpy as np

from . import np_tree as T
from . import np_tree_cls as TC


def chunk_stats(orc, chunks, S, K):
    """Statistics of np_tree.Nodes summed over the chunks `chunks()` yields (a function, called once per request:
    the classifier's audit asks again for the children a pruned leaf may have grown)."""
    ns = K + 1 if K else 4

    def stats(nodes, want):
        want = sorted(want)
        slot = np.full(len(nodes), -1, np.int32)
        slot[want] = np.arange(len(want), dtype=np.int32)
        tot = np.zeros((len(nodes), ns + 2))
        hist = np.zeros((len(want), S, 256, ns))
        par = np.asarray(nodes.parent, np.int32)
        for R, lab, w, c in chunks():
            orc.tree_hist(R, K, lab, w, c, par, nodes.col, nodes.bin, nodes.left, slot, tot, hist)
        return tot, {v: hist[h] for h, v in enumerate(want)}
    return stats


def audit(tree, chunks, cands, params, orc, num_classes=0, out=None, exact=False) -> int:
    """np_tree.audit (num_classes 0) or np_tree_cls.audit of a fitted tree over chunked rows: cands[k] are the
    candidates of subspace column k.  `out(leaf)`, when given, is called per chunk with the tree node of every row
    of it, in order, to check the fit's output.  Returns the number of nodes audited (every node)."""
    bins = T.bins_of(tree, cands)
    ncand = [np.asarray(c).size for c in cands]
    K = int(num_classes)
    stats = chunk_stats(orc, chunks, len(cands), K)
    if K:
        n = TC.check(tree, bins, ncand, stats, dict(params, num_classes=K), exact)
    else:
        n = T.check(tree, bins, ncand, stats, params, exact)
    if out is not None:
        for R, *_ in chunks():
            out(orc.tree_walk(R, tree["feature"], bins, tree["left"], tree["right"]))
    return n
