"""CPU definition of RandomForestClassifier.fit (scikit-learn 1.9, criterion='gini', dense rows without NaN), restated
in numpy so that the GPU fit (csrc/forest_fit.cu) has something exact to be compared with on a machine without a GPU.

The random numbers are scikit-learn's: `forest_fit_plan` (the package's host half of the fit) draws the per-tree seeds,
bootstrap indices and splitter states; this module restates the rest:

* DepthFirstTreeBuilder.build (sk:tree/_tree.pyx): a LIFO stack, right child pushed before the left, nodes numbered in
  pop order;
* node_split_best (sk:tree/_splitter.pyx) with the DensePartitioner (sk:tree/_partitioner.pyx): Fisher-Yates feature
  draws with our_rand_r, the known-constant bookkeeping carried through the tree, FEATURE_THRESHOLD as a float32 constant
  added in float32, candidate positions, strict-improvement choice, threshold as the sum of halves;
* Gini (sk:tree/_criterion.pyx): 1 - sum_c count_c^2 / w^2 in class order, the proxy -wr gini_r - wl gini_l and
  impurity_improvement in their operation order.

Every weight is an integer bootstrap count, so class sums are exact in fp64 whatever order they are added in; the order
of rows inside a node therefore never changes the tree, and this restatement sorts with numpy's stable sort.
"""
import numpy as np

from traffic_classifier_sdn_b200.estimators import forest_feature_importances, forest_fit_plan

FEATURE_THRESHOLD = np.float32(1e-7)
EPSILON = np.finfo(np.float64).eps
TREE_LEAF, TREE_UNDEFINED = -1, -2


class RandR:
    """sk:utils/_random.pxd our_rand_r, and sk:tree/_utils.pyx rand_int."""

    def __init__(self, seed):
        self.s = int(seed) & 0xFFFFFFFF

    def rand_int(self, low, high):
        s = self.s or 1
        s ^= (s << 13) & 0xFFFFFFFF
        s ^= s >> 17
        s ^= (s << 5) & 0xFFFFFFFF
        self.s = s
        return low + (s % 0x80000000) % (high - low)


def _gini(counts, w):
    sq = 0.0
    for c in counts:
        sq += float(c) * float(c)
    return 1.0 - sq / (w * w)


def build_tree(X32, y, n_classes, weight, seed, plan):
    """One tree: -> dict of the eight node arrays (left, right, feature, threshold, value, impurity, n_node_samples,
    weighted_n_node_samples).  X32 [n][d] float32, y [n] class index, weight [n] integer counts, seed the rand_r state."""
    n, d = X32.shape
    C = n_classes
    max_depth, mss, msl = plan["max_depth"], plan["min_samples_split"], plan["min_samples_leaf"]
    max_features, mid = plan["max_features"], plan["min_impurity_decrease"]
    w = np.asarray(weight, np.int64)
    samples = np.flatnonzero(w != 0)
    W = float(w.sum())
    onehot = np.zeros((n, C), np.int64)
    onehot[np.arange(n), y] = w
    features = np.arange(d)
    constant_features = np.zeros(d, np.int64)
    rng = RandR(seed)
    nodes = {k: [] for k in ("left", "right", "feature", "threshold", "value", "impurity", "n_node_samples",
                             "weighted_n_node_samples")}
    stack = [(0, len(samples), 0, -1, False, np.inf, 0)]
    first = True
    while stack:
        start, end, depth, parent, is_left, impurity, n_const = stack.pop()
        idx = samples[start:end]
        tot = onehot[idx].sum(axis=0)
        wn = float(w[idx].sum())
        m = end - start
        is_leaf = depth >= max_depth or m < mss or m < 2 * msl
        if first:
            impurity = _gini(tot, wn)
            first = False
        is_leaf = is_leaf or impurity <= EPSILON
        split = None
        if not is_leaf:
            split = _node_split(X32, onehot, w, samples, start, end, tot, wn, W, impurity, n_const, features,
                                constant_features, rng, max_features, msl, d)
            is_leaf = split["pos"] >= end or split["improvement"] + EPSILON < mid
        nid = len(nodes["left"])
        if parent >= 0:
            nodes["left" if is_left else "right"][parent] = nid
        nodes["left"].append(TREE_LEAF)
        nodes["right"].append(TREE_LEAF)
        nodes["feature"].append(TREE_UNDEFINED if is_leaf else split["feature"])
        nodes["threshold"].append(float(TREE_UNDEFINED) if is_leaf else split["threshold"])
        nodes["value"].append(tot / wn)
        nodes["impurity"].append(impurity)
        nodes["n_node_samples"].append(m)
        nodes["weighted_n_node_samples"].append(wn)
        if not is_leaf:
            nc = split["n_constant_features"]
            stack.append((split["pos"], end, depth + 1, nid, False, split["impurity_right"], nc))
            stack.append((start, split["pos"], depth + 1, nid, True, split["impurity_left"], nc))
    out = {k: np.asarray(v) for k, v in nodes.items()}
    for k in ("left", "right", "feature"):
        out[k] = out[k].astype(np.int32)
    out["n_node_samples"] = out["n_node_samples"].astype(np.int64)
    out["value"] = out["value"].reshape(-1, C).astype(np.float64)
    return out


def _node_split(X32, onehot, w, samples, start, end, tot, wn, W, impurity, n_known, features, constant_features, rng,
                max_features, msl, d):
    f_i = d
    n_visited = n_found = n_drawn = 0
    n_total = n_known
    best = dict(pos=end, proxy=-np.inf)
    while f_i > n_total and (n_visited < max_features or n_visited <= n_found + n_drawn):
        n_visited += 1
        f_j = rng.rand_int(n_drawn, f_i - n_found)
        if f_j < n_known:
            features[n_drawn], features[f_j] = features[f_j], features[n_drawn]
            n_drawn += 1
            continue
        f_j += n_found
        f = int(features[f_j])
        idx = samples[start:end].copy()
        order = np.argsort(X32[idx, f], kind="stable")
        samples[start:end] = idx[order]
        fv = X32[samples[start:end], f]
        if fv[-1] <= fv[0] + FEATURE_THRESHOLD:
            features[f_j], features[n_total] = features[n_total], features[f_j]
            n_found += 1
            n_total += 1
            continue
        f_i -= 1
        features[f_i], features[f_j] = features[f_j], features[f_i]
        # candidate p (absolute) has fv[p] > fv[p-1] + FEATURE_THRESHOLD, p - start >= msl, end - p >= msl
        q = np.flatnonzero(fv[1:] > fv[:-1] + FEATURE_THRESHOLD) + 1          # p - start
        q = q[(q >= msl) & ((end - start) - q >= msl)]
        if len(q) == 0:
            continue
        cum = np.cumsum(onehot[samples[start:end]], axis=0)
        left = cum[q - 1].astype(np.float64)                                  # [len(q)][C]
        wl = left.sum(axis=1)   # integer-valued: exact
        wr = wn - wl
        sql = np.zeros(len(q))
        sqr = np.zeros(len(q))
        for c in range(onehot.shape[1]):
            lc = left[:, c]
            rc = float(tot[c]) - lc
            sql = sql + lc * lc
            sqr = sqr + rc * rc
        gl = 1.0 - sql / (wl * wl)
        gr = 1.0 - sqr / (wr * wr)
        proxy = -wr * gr - wl * gl
        k = int(np.argmax(proxy))
        if proxy[k] > best["proxy"]:
            p = int(q[k])
            best = dict(pos=start + p, proxy=proxy[k], feature=f,
                        threshold=float(fv[p - 1]) / 2.0 + float(fv[p]) / 2.0)
    if best["pos"] < end:
        f, thr = best["feature"], best["threshold"]
        idx = samples[start:end].copy()
        go_left = X32[idx, f].astype(np.float64) <= thr
        samples[start:end] = np.concatenate([idx[go_left], idx[~go_left]])
        assert start + int(go_left.sum()) == best["pos"]
        cl = onehot[idx[go_left]].sum(axis=0)
        wl = float(w[idx[go_left]].sum())
        wr = wn - wl
        il, ir = _gini(cl, wl), _gini(tot - cl, wr)
        best["impurity_left"], best["impurity_right"] = il, ir
        best["improvement"] = (wn / W) * (impurity - (wr / wn * ir) - (wl / wn * il))
    features[:n_known] = constant_features[:n_known]
    constant_features[n_known:n_known + n_found] = features[n_known:n_known + n_found]
    best["n_constant_features"] = n_total
    return best


def fit_forest(X, y, **params):
    """-> (classes, forest dict): the concatenated tree arrays with ``tree_offsets`` and ``feature_importances``, for
    RandomForestClassifier(**params).fit(X, y)."""
    X32 = np.ascontiguousarray(np.asarray(X).astype(np.float32))
    classes, yi = np.unique(np.asarray(y), return_inverse=True)
    n, d = X32.shape
    plan = forest_fit_plan(params, n, d)
    trees = []
    for t in range(plan["n_trees"]):
        if plan["bootstrap_idx"] is not None:
            wt = np.bincount(plan["bootstrap_idx"][t], minlength=n)
        else:
            wt = np.ones(n, np.int64)
        trees.append(build_tree(X32, yi, len(classes), wt, plan["rand_r_seeds"][t], plan))
    offs = np.concatenate([[0], np.cumsum([len(t["left"]) for t in trees])]).astype(np.int64)
    out = {k: np.concatenate([t[k] for t in trees]) for k in trees[0]}
    out["tree_offsets"] = offs
    out["feature_importances"] = forest_feature_importances(offs, out["left"], out["right"], out["feature"],
                                                            out["impurity"], out["weighted_n_node_samples"], d)
    return classes, out


def sklearn_forest(est):
    """The same dict from a fitted sklearn.ensemble.RandomForestClassifier."""
    keys = ("left", "right", "feature", "threshold", "value", "impurity", "n_node_samples", "weighted_n_node_samples")
    trees = []
    for e in est.estimators_:
        t = e.tree_
        trees.append(dict(left=t.children_left.astype(np.int32), right=t.children_right.astype(np.int32),
                          feature=t.feature.astype(np.int32), threshold=t.threshold, value=t.value[:, 0, :],
                          impurity=t.impurity, n_node_samples=t.n_node_samples.astype(np.int64),
                          weighted_n_node_samples=t.weighted_n_node_samples))
    out = {k: np.concatenate([t[k] for t in trees]) for k in keys}
    out["tree_offsets"] = np.concatenate([[0], np.cumsum([len(t["left"]) for t in trees])]).astype(np.int64)
    out["feature_importances"] = est.feature_importances_
    return out


def forest_diff(a, b):
    """-> the names of the arrays that differ (np.array_equal), [] when the two forests are the same bits."""
    keys = ("tree_offsets", "left", "right", "feature", "threshold", "value", "impurity", "n_node_samples",
            "weighted_n_node_samples", "feature_importances")
    return [k for k in keys if not (np.shape(a[k]) == np.shape(b[k]) and np.array_equal(a[k], b[k]))]
