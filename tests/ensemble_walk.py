"""Numpy restatement of the ensemble walk (Tree::Predict / NumericalDecision, include/LightGBM/tree.h:329-347; GBDT::PredictRaw /
PredictLeafIndex) on the trees of gpboost_b200.booster.parse_model_string, and builders of synthetic model texts. Shared by the
prediction tests."""
import hashlib

import numpy as np

K_ZERO = float(np.float32(1e-35))


def digest(a, dtype):
    """sha256 of the array's bytes as `dtype` (little endian): a bitwise comparison against a stored result without storing it"""
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.dtype(dtype).newbyteorder("<")).tobytes()).hexdigest()


def iteration_range(total, start_iteration, num_iteration):
    b = max(0, min(start_iteration, total))
    c = total - b
    if num_iteration > 0:
        c = min(num_iteration, c)
    return b, c


def leaf_of_rows(tree, X):
    """leaf index of every row of X (float64, NaNs allowed) in one parsed tree"""
    n = X.shape[0]
    if tree["num_leaves"] <= 1:
        return np.zeros(n, dtype=np.int64)
    node = np.zeros(n, dtype=np.int64)
    rows = np.arange(n)
    dts = tree.get("decision_type")
    while True:
        act = node >= 0
        if not act.any():
            break
        nd = node[act]
        f = X[rows[act], tree["split_feature"][nd]].astype(np.float64)
        dt = dts[nd] if dts is not None else np.full(nd.shape, 2)
        missing = (dt >> 2) & 3
        isnan = np.isnan(f)
        f = np.where(isnan & (missing != 2), 0.0, f)
        with np.errstate(invalid="ignore"):
            use_default = ((missing == 1) & (f >= -K_ZERO) & (f <= K_ZERO)) | ((missing == 2) & isnan)
            left = np.where(use_default, (dt & 2) != 0, f <= tree["threshold"][nd])
        node[act] = np.where(left, tree["left_child"][nd], tree["right_child"][nd])
    return ~node


def predict(trees, X, start_iteration=0, num_iteration=-1, pred_leaf=False):
    """raw score (one fp64 add per tree, ensemble order, starting from 0.0) or the (nrow, trees) leaf indices"""
    X = np.asarray(X)
    X = X.astype(np.float64)  # float32 input is widened first
    first, count = iteration_range(len(trees), start_iteration, num_iteration)
    if pred_leaf:
        out = np.zeros((X.shape[0], count), dtype=np.int64)
        for k in range(count):
            out[:, k] = leaf_of_rows(trees[first + k], X)
        return out
    s = np.zeros(X.shape[0])
    for t in trees[first:first + count]:
        s = s + t["leaf_value"][leaf_of_rows(t, X)]
    return s


def _fmt(v):
    return " ".join(repr(float(x)) for x in v)


def tree_text(index, split_feature, threshold, decision_type, left_child, right_child, leaf_value):
    nl = len(leaf_value)
    lines = ["Tree=%d" % index, "num_leaves=%d" % nl, "num_cat=0"]
    if nl > 1:
        lines += ["split_feature=" + " ".join(str(int(v)) for v in split_feature),
                  "split_gain=" + " ".join("1" for _ in split_feature),
                  "threshold=" + _fmt(threshold),
                  "decision_type=" + " ".join(str(int(v)) for v in decision_type),
                  "left_child=" + " ".join(str(int(v)) for v in left_child),
                  "right_child=" + " ".join(str(int(v)) for v in right_child)]
    lines += ["leaf_value=" + _fmt(leaf_value), "leaf_count=" + " ".join("1" for _ in leaf_value), "is_linear=0", "shrinkage=1", "", ""]
    return "\n".join(lines)


def model_text(ncol, tree_texts):
    head = ["tree", "version=v3", "num_class=1", "num_tree_per_iteration=1", "label_index=0", "max_feature_idx=%d" % (ncol - 1),
            "objective=regression", "feature_names=" + " ".join("Column_%d" % j for j in range(ncol)),
            "feature_infos=" + " ".join("[-10:10]" for _ in range(ncol)), "", ""]
    return "\n".join(head) + "".join(tree_texts) + "end of trees\n"


def random_tree(rng, index, ncol, num_leaves, decision_types=(2,), thresholds=None):
    """a tree grown like Tree::Split: node i splits a random existing leaf (children of a node have larger indices)"""
    if num_leaves <= 1:
        return tree_text(index, [], [], [], [], [], [rng.standard_normal()])
    nn = num_leaves - 1
    left, right = np.zeros(nn, dtype=np.int64), np.zeros(nn, dtype=np.int64)
    left[0], right[0] = ~0, ~1
    parent_slot = {0: (0, 0), 1: (0, 1)}  # leaf -> (node, side)
    for i in range(1, nn):
        leaf = int(rng.integers(0, i + 1))
        node, side = parent_slot[leaf]
        (left if side == 0 else right)[node] = i
        left[i], right[i] = ~leaf, ~(i + 1)
        parent_slot[leaf] = (i, 0)
        parent_slot[i + 1] = (i, 1)
    feat = rng.integers(0, ncol, nn)
    thr = rng.standard_normal(nn) if thresholds is None else rng.choice(thresholds, nn)
    dt = rng.choice(np.asarray(decision_types), nn)
    return tree_text(index, feat, thr, dt, left, right, rng.standard_normal(num_leaves))


def chain_tree(rng, index, ncol, num_leaves, decision_types=(2,)):
    """degenerate tree of depth num_leaves - 1: every right child is the next node"""
    nn = num_leaves - 1
    left = np.array([~i for i in range(nn)], dtype=np.int64)
    right = np.array([i + 1 for i in range(nn)], dtype=np.int64)
    right[-1] = ~nn
    thr = np.sort(rng.standard_normal(nn))  # increasing thresholds on one feature: rows stop at every depth
    feat = np.full(nn, int(rng.integers(0, ncol)))
    return tree_text(index, feat, thr, rng.choice(np.asarray(decision_types), nn), left, right, rng.standard_normal(num_leaves))
