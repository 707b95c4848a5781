"""The KNN engine's pruning rule (csrc/knn_engine.cu, "KNN: spatial order and pruning"), restated in numpy on small data:
training rows in kd order -> tiles of 64 with centre and radius; queries sorted by kd leaf -> passes of 256; per pass the
tiles are visited by centre distance from the home tile and tile t is left out when

    (||x0 - c_t|| - r_t - rho)^2 > H          x0 = first row of the pass, rho = max ||x - x0||, H = max current k-th distance^2

(per lane: ||x - x0|| and the lane's own k-th distance).  The property the kernel relies on: a tile that is left out never
holds one of the k nearest rows of any query it was left out for -- whatever the (stale) H at the time of the test.  This is
a statement about the rule; the CUDA implementation is held to sklearn's answers by tests/test_engine_gpu.py."""
import numpy as np
import pytest

from traffic_classifier_sdn_b200 import synth

N = 64


def _kd_order(T, lo_hi_leaf=8):
    """same splitting rule as kd_build(): widest coordinate, median at a tile boundary above 64 rows, plain median below"""
    leaves, splits = [], []

    def rec(idx, lo):
        if len(idx) <= lo_hi_leaf:
            leaves.append((idx, lo // N))
            return ("leaf", len(leaves) - 1)
        sub = T[idx]
        j = int(np.argmax(sub.max(0) - sub.min(0)))
        n = len(idx)
        mid = ((n // 2 + N - 1) // N) * N if n > N else n // 2
        part = np.argpartition(sub[:, j], mid)
        split = sub[part[mid], j]
        return ("node", j, split, rec(idx[part[:mid]], lo), rec(idx[part[mid:]], lo + mid))

    tree = rec(np.arange(len(T)), 0)
    order = np.concatenate([l[0] for l in leaves])
    leaf_tile = np.array([l[1] for l in leaves])
    return tree, order, leaf_tile


def _descend(tree, X):
    key = np.empty(len(X), dtype=np.int64)

    def rec(t, ids):
        if t[0] == "leaf":
            key[ids] = t[1]
            return
        m = X[ids, t[1]] < t[2]
        rec(t[3], ids[m])
        rec(t[4], ids[~m])

    rec(tree, np.arange(len(X)))
    return key


@pytest.mark.parametrize("seed,k,lag", [(0, 5, 0), (1, 1, 4), (2, 9, 8)])
def test_skipped_tiles_never_hold_a_neighbour(seed, k, lag):
    T, _ = synth.make_flows(3000, seed=seed)
    X = synth.make_flows(1500, seed=seed + 50, return_labels=False)
    X[:64] = T[:64]                                              # queries that coincide with training rows
    tree, order, leaf_tile = _kd_order(T)
    nt = -(-len(T) // N)
    tiles = [order[i * N:(i + 1) * N] for i in range(nt)]
    cent = np.array([T[t].mean(0) for t in tiles])
    rad = np.array([np.sqrt(((T[t] - c) ** 2).sum(1).max()) for t, c in zip(tiles, cent)])
    key = _descend(tree, X)
    qs = np.argsort(key, kind="stable")
    Xs, ks = X[qs], key[qs]
    d2_all = ((Xs[:, None, :] - T[None, :, :]) ** 2).sum(2)
    kth_true = np.sort(d2_all, 1)[:, k - 1]
    tile_of_row = np.empty(len(T), dtype=np.int64)
    tile_of_row[order] = np.arange(len(T)) // N
    P = 256
    skipped_pass = skipped_lane = 0
    for p0 in range(0, len(Xs), P):
        Q = Xs[p0:p0 + P]
        x0 = Q[0]
        e = np.sqrt(((Q - x0) ** 2).sum(1))
        rho = e.max()
        home = leaf_tile[ks[p0]]
        tord = np.argsort(np.sqrt(((cent - cent[home]) ** 2).sum(1)), kind="stable")
        gap = np.sqrt(((cent - x0) ** 2).sum(1)) - rad           # <= ||x0 - row|| for every row of the tile
        best = np.full((len(Q), k), np.inf)
        hist = []                                                 # H after each visited tile; the producer sees it `lag` tiles late
        for t in tord:
            H = hist[len(hist) - 1 - lag] if len(hist) > lag else np.inf
            m = gap[t] - rho
            rows = tiles[t]
            if m > 0 and m * m > H:                               # left out for the whole pass
                skipped_pass += 1
                assert (d2_all[p0:p0 + len(Q)][:, rows].min(1) > kth_true[p0:p0 + len(Q)]).all()
                continue
            kth = best[:, -1]
            ml = gap[t] - e
            far = (ml > 0) & (ml * ml > kth)                      # per lane, with the lane's own k-th distance so far
            if far.any():
                skipped_lane += int(far.sum())
                sub = d2_all[p0:p0 + len(Q)][far][:, rows]
                assert (sub.min(1) > kth_true[p0:p0 + len(Q)][far]).all()
            d2 = d2_all[p0:p0 + len(Q)][:, rows]
            d2 = np.where(far[:, None], np.inf, d2)               # a lane that skipped the tile learns nothing from it
            best = np.sort(np.concatenate([best, d2], 1), 1)[:, :k]
            hist.append(best[:, -1].max())
        assert np.array_equal(best[:, -1], kth_true[p0:p0 + len(Q)])   # what was visited suffices
    assert skipped_pass > 0 and skipped_lane > 0, "the data should give the rule something to skip"


def test_tie_rule_flags_exactly_the_class_relevant_ties():
    """the engine's end-of-pass decision: a query needs sklearn's index-order heap iff a row left out at exactly the k-th
    distance and the kept rows at that distance do not all carry one class"""
    rng = np.random.default_rng(3)
    for _ in range(200):
        n, k = 40, int(rng.integers(1, 6))
        d = rng.integers(0, 6, n).astype(float)                  # many equal distances
        y = rng.integers(0, 3, n)
        order = rng.permutation(n)                               # the engine's visiting order
        hv, hi, tie_val, tie_cls = [], [], None, None

        def note(v, c):
            nonlocal tie_val, tie_cls
            if tie_val != v:
                tie_val, tie_cls = v, c
            elif tie_cls != c:
                tie_cls = -2

        for i in order:
            if len(hv) < k:
                hv.append(d[i]); hi.append(i)
                continue
            r = int(np.argmax(hv))
            if d[i] < hv[r]:
                ev, ei = hv[r], hi[r]
                hv[r], hi[r] = d[i], i
                if max(hv) == ev:
                    note(ev, y[ei])
            elif d[i] == hv[r]:
                note(d[i], y[i])
        vk = max(hv)
        tied = False
        if tie_val == vk:
            tied = tie_cls < 0 or any(y[j] != tie_cls for v, j in zip(hv, hi) if v == vk)
        # ground truth: do all rows at the k-th distance share a class, or are they all inside the kept set anyway?
        at = np.flatnonzero(d == vk)
        inside = sum(1 for v in hv if v == vk)
        relevant = len(at) > inside and len(set(y[at])) > 1
        assert tied == relevant
