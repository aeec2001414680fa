"""fp64 numpy restatement of the random-forest kernels (hebo_b200/csrc/forest.cu), operation for operation.

TEST INFRASTRUCTURE ONLY; never imported by hebo_b200/.  It fixes every choice the device makes where sklearn's
RandomForestRegressor leaves one open (the order of each sum, the tie rule, the node numbering), so the device forest must
equal it bit for bit; and it restates the reference's predict arithmetic (sklearn's sequential tree sum, numpy's pairwise
sums inside np.var / np.mean), which must equal numpy bit for bit.

A forest here is a list of trees; a tree is a dict of numpy arrays over its nodes: feature (int32, -2 at a leaf),
threshold (fp64, -2 at a leaf), left / right (int32, -1 at a leaf) and value (fp64, S / W of every node).
"""
from __future__ import annotations

import numpy as np

from oracle.rng_oracle import block

FEATURE_THRESHOLD = 1e-7                  # sklearn _splitter.pyx
EPS = np.finfo(np.float64).eps            # sklearn _tree.pyx EPSILON


RF_PHILOX_TAG = 0x52460000                # word 3 of the bootstrap counter (forest.cu)


# ---------------------------------------------------------------------------------------------------------------- bootstrap
def bootstrap_counts(seed: int, b: int, t: int, kept, n: int) -> np.ndarray:
    """hb_rf_fit's bootstrap counts of tree (b, t) over n rows: draw j of the n_b = len(kept) draws is
    kept[umulhi(w, n_b)], w = word j % 4 of the Philox4x32-10 block (j / 4, t, b, RF_PHILOX_TAG) under seed."""
    kept = np.asarray(kept, dtype=np.int64)
    nb = kept.size
    counts = np.zeros(n, dtype=np.int32)
    if nb == 0:
        return counts
    q = np.arange((nb + 3) // 4, dtype=np.uint64)
    words = np.stack(block(seed, q, np.uint64(t), np.uint64(b), np.uint64(RF_PHILOX_TAG)), axis=1).reshape(-1)[:nb]
    idx = (words.astype(np.uint64) * np.uint64(nb)) >> np.uint64(32)
    np.add.at(counts, kept[idx.astype(np.int64)], 1)
    return counts


# ---------------------------------------------------------------------------------------------------------------- inputs
def tree_inputs(Xc, Xe, num_uniqs) -> np.ndarray:
    """[Xc | one_hot(Xe)] as float32 (rf.py:27-35, layers.py:36)."""
    parts = []
    if Xc is not None and np.asarray(Xc).shape[1] > 0:
        parts.append(np.asarray(Xc, dtype=np.float32))
    if num_uniqs:
        Xe = np.asarray(Xe, dtype=np.int64)
        for c, u in enumerate(num_uniqs):
            parts.append((Xe[:, c:c + 1] == np.arange(u)[None, :]).astype(np.float32))
    return np.concatenate(parts, axis=1)


# ---------------------------------------------------------------------------------------------------------------- numpy sums
def pairwise_sum(a) -> float:
    """numpy's pairwise_sum of a 1-D fp64 array (eight accumulators, blocks of 128, halves above), as the device streams it."""
    a = np.asarray(a, dtype=np.float64)
    n = a.size
    if n < 8:
        r = 0.0
        for v in a:
            r = float(np.float64(r) + v)
        return r
    if n <= 128:
        r = [np.float64(v) for v in a[:8]]
        i = 8
        while i < n - n % 8:
            for j in range(8):
                r[j] = r[j] + a[i + j]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        while i < n:
            res = res + a[i]
            i += 1
        return float(res)
    n2 = n // 2
    n2 -= n2 % 8
    return float(np.float64(pairwise_sum(a[:n2])) + np.float64(pairwise_sum(a[n2:])))


def sequential_sum(a) -> float:
    r = np.float64(0.0)
    for v in np.asarray(a, dtype=np.float64):
        r = r + v
    return float(r)


# ---------------------------------------------------------------------------------------------------------------- growth
def grow_tree(X: np.ndarray, y: np.ndarray, w: np.ndarray) -> dict:
    """One tree of hb_rf_fit from float32 inputs X [n, width], float32 y [n] and integer weights w [n] (0 = out of bag)."""
    X = np.asarray(X, dtype=np.float32) + np.float32(0.0)        # -0 -> +0, as the presort keys it
    n, width = X.shape
    y64 = np.asarray(y, dtype=np.float32).astype(np.float64)
    w = np.asarray(w, dtype=np.int64)
    w64 = w.astype(np.float64)
    order = [np.argsort(X[:, f], kind="stable") for f in range(width)]
    feat, thr, left, right, val = [], [], [], [], []
    Wn, Sn, Qn, Cn = [], [], [], []

    def add_node(W, S, Q, C):
        for lst, v in ((feat, -2), (thr, -2.0), (left, -1), (right, -1), (val, 0.0), (Wn, W), (Sn, S), (Qn, Q), (Cn, C)):
            lst.append(v)
        return len(feat) - 1

    inbag = w > 0
    wy = w64 * np.where(inbag, y64, 0.0)
    sq = wy * np.where(inbag, y64, 0.0)
    rows = np.nonzero(inbag)[0]
    add_node(sequential_sum(w64[rows]), sequential_sum(wy[rows]), sequential_sum(sq[rows]), int(rows.size))
    nid = np.zeros(n, dtype=np.int64)
    lo, hi = 0, 1
    while lo < hi:
        open_nodes = []
        for k in range(lo, hi):
            W, S, Q = Wn[k], Sn[k], Qn[k]
            mean = S / W if W != 0 else np.nan
            imp = Q / W - mean * mean if W != 0 else np.nan
            val[k] = mean
            if Cn[k] < 2 or imp <= EPS:
                continue
            open_nodes.append(k)
        if not open_nodes:
            break
        best = {}
        for k in open_nodes:
            members = inbag & (nid == k)
            W, S = Wn[k], Sn[k]
            bp, bb = -np.inf, None
            for f in range(width):
                r = order[f][members[order[f]]]
                v = X[r, f].astype(np.float64)
                cw, cs, cq = np.cumsum(w64[r]), np.cumsum(wy[r]), np.cumsum(sq[r])
                j = np.arange(1, r.size)
                ok = v[j] > v[j - 1] + FEATURE_THRESHOLD
                if not ok.any():
                    continue
                j = j[ok]
                WL, SL = cw[j - 1], cs[j - 1]
                SR = S - SL
                proxy = SL * SL / WL + SR * SR / (W - WL)
                a = int(np.argmax(proxy))
                if proxy[a] > bp:
                    jj = int(j[a])
                    th = v[jj - 1] / 2.0 + v[jj] / 2.0
                    if th == v[jj] or np.isinf(th):
                        th = v[jj - 1]
                    bp, bb = proxy[a], (f, float(th), float(cw[jj - 1]), float(cs[jj - 1]), float(cq[jj - 1]), jj)
            best[k] = bb
        nx = hi
        for k in open_nodes:
            if best[k] is None:
                continue
            f, th, WL, SL, QL, cl = best[k]
            W, S, Q, C = Wn[k], Sn[k], Qn[k], Cn[k]
            l = add_node(WL, SL, QL, cl)
            r = add_node(W - WL, S - SL, Q - QL, C - cl)
            assert (l, r) == (nx, nx + 1)
            nx += 2
            feat[k], thr[k], left[k], right[k] = f, th, l, r
            sel = inbag & (nid == k)
            goes_left = X[:, f].astype(np.float64) <= th
            nid[sel & goes_left] = l
            nid[sel & ~goes_left] = r
        lo, hi = hi, nx
    return dict(feature=np.array(feat, dtype=np.int32), threshold=np.array(thr, dtype=np.float64),
                left=np.array(left, dtype=np.int32), right=np.array(right, dtype=np.int32),
                value=np.array(val, dtype=np.float64))


def apply(tree: dict, X: np.ndarray) -> np.ndarray:
    """Leaf index of every row of float32 X (DecisionTreeRegressor.apply: x <= threshold goes left, compared in fp64)."""
    X = np.asarray(X, dtype=np.float32)
    node = np.zeros(X.shape[0], dtype=np.int64)
    while True:
        f = tree["feature"][node]
        inner = f >= 0
        if not inner.any():
            return node
        idx = np.nonzero(inner)[0]
        x = X[idx, f[idx]].astype(np.float64)
        node[idx] = np.where(x <= tree["threshold"][node[idx]], tree["left"][node[idx]], tree["right"][node[idx]])


def tree_predict(tree: dict, X) -> np.ndarray:
    return tree["value"][apply(tree, X)]


# ---------------------------------------------------------------------------------------------------------------- forest
def fit(X, y, counts):
    """(trees, est_noise) of one output: X float32 [n, width], y float32 [n] (non-finite rows weigh 0), counts [T, n]."""
    y = np.asarray(y, dtype=np.float32)
    keep = np.isfinite(y)
    trees = [grow_tree(X, np.where(keep, y, 0.0).astype(np.float32), np.where(keep, np.maximum(c, 0), 0))
             for c in np.asarray(counts)]
    return trees, noise(trees, X[keep], y[keep])


def forest_mean64(trees, X) -> np.ndarray:
    """RandomForestRegressor.predict: the tree outputs summed sequentially in tree order from 0, then / T (fp64)."""
    s = np.zeros(np.asarray(X).shape[0], dtype=np.float64)
    for t in trees:
        s = s + tree_predict(t, X)
    return s / len(trees)


def noise(trees, Xk, yk) -> np.float32:
    """est_noise (rf.py:42-43) over the kept rows: fp32(np.mean((forest mean - y)^2)), numpy's pairwise sum."""
    d = forest_mean64(trees, Xk) - np.asarray(yk, dtype=np.float32).astype(np.float64)
    return np.float32(pairwise_sum(d * d) / d.size)


def predict(trees, X, noise_b) -> tuple:
    """RF.predict (rf.py:49-56) restated: (mean, var) fp32 [m] with the reference's summation orders."""
    P = np.stack([tree_predict(t, X) for t in trees], axis=1)          # [m, T]
    T = P.shape[1]
    mean = np.float32(0) + (forest_mean64(trees, X)).astype(np.float32)
    var = np.empty(P.shape[0], dtype=np.float32)
    for i in range(P.shape[0]):
        mu = pairwise_sum(P[i]) / T
        d = P[i] - mu
        var[i] = np.float32(pairwise_sum(d * d) / T)
    return mean, var + np.float32(noise_b)
