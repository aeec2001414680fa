"""fp64 numpy restatement of the random-forest kernels (hebo_b200/csrc/forest.cu), operation for operation.

TEST INFRASTRUCTURE ONLY; never imported by hebo_b200/.  It fixes every choice the device makes where sklearn's
RandomForestRegressor leaves one open (the order of each sum, the tie rule, the node numbering), so the device forest must
equal it bit for bit; and it restates the reference's predict arithmetic (sklearn's sequential tree sum, numpy's pairwise
sums inside np.var / np.mean), which must equal numpy bit for bit.

A forest here is a list of trees; a tree is a dict of numpy arrays over its nodes: feature (int32, -2 at a leaf),
threshold (fp64, -2 at a leaf), left / right (int32, -1 at a leaf), value (fp64, S / W of every node) and, optionally,
missing_go_to_left (int32, 1 where a NaN input goes left; sklearn sets it, for trees trained without NaN, where the split
leaves more distinct in-bag rows left than right).
"""
from __future__ import annotations

import os
from concurrent.futures import ThreadPoolExecutor

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
    feat, thr, left, right, val, nanl = [], [], [], [], [], []
    Wn, Sn, Qn, Cn = [], [], [], []

    def add_node(W, S, Q, C):
        for lst, v in ((feat, -2), (thr, -2.0), (left, -1), (right, -1), (val, 0.0), (nanl, 0), (Wn, W), (Sn, S), (Qn, Q),
                       (Cn, C)):
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
            feat[k], thr[k], left[k], right[k], nanl[k] = f, th, l, r, int(cl > C - cl)
            sel = inbag & (nid == k)
            goes_left = X[:, f].astype(np.float64) <= th
            nid[sel & goes_left] = l
            nid[sel & ~goes_left] = r
        lo, hi = hi, nx
    return dict(feature=np.array(feat, dtype=np.int32), threshold=np.array(thr, dtype=np.float64),
                left=np.array(left, dtype=np.int32), right=np.array(right, dtype=np.int32),
                value=np.array(val, dtype=np.float64), missing_go_to_left=np.array(nanl, dtype=np.int32))


def grow_tree_level(X: np.ndarray, y: np.ndarray, w: np.ndarray, chunk_elems: int = 1 << 21) -> dict:
    """grow_tree, level-synchronous and vectorised over features and nodes: the same tree, node numbering and bits.

    Every in-bag row of the level's open nodes sits in G [width, nl]: row f is feature f's presorted order filtered to
    those rows and grouped by node, the nodes' segments in node order at the same offsets for every feature.  A split
    partitions each segment stably into its children's, so a segment stays the presorted order of its node's rows.
    The split search pads the segments of a chunk of features into [features, nodes, L] blocks, one per power-of-two
    length class L, and scans them with np.cumsum(axis=-1), which adds sequentially along each segment as grow_tree does
    (trailing zero padding cannot change an earlier prefix).  Cut rule, proxy and tie rule are grow_tree's."""
    X = np.asarray(X, dtype=np.float32) + np.float32(0.0)
    n, width = X.shape
    y64 = np.asarray(y, dtype=np.float32).astype(np.float64)
    w = np.asarray(w, dtype=np.int64)
    w64 = w.astype(np.float64)
    inbag = w > 0
    wy = w64 * np.where(inbag, y64, 0.0)
    sq = wy * np.where(inbag, y64, 0.0)
    Xt = np.ascontiguousarray(X.T)
    feat, thr, left, right, val, nanl = [], [], [], [], [], []
    Wn, Sn, Qn, Cn = [], [], [], []

    def add_node(W, S, Q, C):
        for lst, v in ((feat, -2), (thr, -2.0), (left, -1), (right, -1), (val, 0.0), (nanl, 0), (Wn, W), (Sn, S), (Qn, Q),
                       (Cn, C)):
            lst.append(v)
        return len(feat) - 1

    rows = np.nonzero(inbag)[0]
    add_node(sequential_sum(w64[rows]), sequential_sum(wy[rows]), sequential_sum(sq[rows]), int(rows.size))
    # root level: every feature's stable presort filtered to the in-bag rows; V [width, nl] holds G's values
    order = np.argsort(Xt, axis=1, kind="stable").astype(np.int32)
    G = order[inbag[order]].reshape(width, rows.size)
    del order
    V = np.take_along_axis(Xt, G, axis=1)
    seg_nodes, seg_off = [0], [0]          # the level's nodes in order, and their column offsets in G
    pool = ThreadPoolExecutor(os.cpu_count() or 1)          # numpy releases the GIL inside these array operations
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
        # keep only the open nodes' segments
        off = dict(zip(seg_nodes, seg_off))
        keep = np.concatenate([np.arange(off[k], off[k] + Cn[k]) for k in open_nodes])
        G, V = np.ascontiguousarray(G[:, keep]), np.ascontiguousarray(V[:, keep])
        no = len(open_nodes)
        cnt = np.array([Cn[k] for k in open_nodes], dtype=np.int64)
        segoff = np.concatenate([[0], np.cumsum(cnt)[:-1]])
        Wv = np.array([Wn[k] for k in open_nodes], dtype=np.float64)
        Sv = np.array([Sn[k] for k in open_nodes], dtype=np.float64)
        nl = G.shape[1]
        # length classes: open nodes whose count rounds up to the same power of two
        L2 = 1 << np.ceil(np.log2(cnt)).astype(np.int64)
        classes = []
        for Lc in np.unique(L2):
            ks = np.nonzero(L2 == Lc)[0]
            j = np.arange(Lc)
            valid = j[None, :] < cnt[ks, None]
            idx = np.where(valid, segoff[ks, None] + j[None, :], 0)
            classes.append((ks, idx, valid, valid[:, 1:] & valid[:, :-1], Sv[ks][None, :, None], Wv[ks][None, :, None]))

        def search(f0, f1):
            """per (feature, node) of features f0 .. f1 - 1: the proxy at the first arg-max over the cuts, and that cut"""
            cp = np.full((f1 - f0, no), -np.inf)
            cj = np.zeros((f1 - f0, no), dtype=np.int64)
            with np.errstate(divide="ignore", invalid="ignore"):
                for ks, idx, valid, cut, S, W in classes:
                    r = G[f0:f1, idx]                                  # [features, nodes, Lc] rows
                    v = V[f0:f1, idx].astype(np.float64)
                    cw = np.cumsum(np.where(valid, w64[r], 0.0), axis=-1)
                    cs = np.cumsum(np.where(valid, wy[r], 0.0), axis=-1)
                    ok = cut & (v[..., 1:] > v[..., :-1] + FEATURE_THRESHOLD)
                    WL, SL = cw[..., :-1], cs[..., :-1]
                    SR = S - SL
                    proxy = np.where(ok, SL * SL / WL + SR * SR / (W - WL), -np.inf)
                    a = np.argmax(proxy, axis=-1)
                    cp[:, ks] = np.take_along_axis(proxy, a[..., None], axis=-1)[..., 0]
                    cj[:, ks] = a + 1
            return cp, cj

        fc = max(1, chunk_elems // (2 * nl))
        bp = np.full(no, -np.inf)
        bf = np.full(no, -1, dtype=np.int64)
        bj = np.zeros(no, dtype=np.int64)
        chunks = [(f0, min(width, f0 + fc)) for f0 in range(0, width, fc)]
        for (f0, _), (cp, cj) in zip(chunks, pool.map(lambda c: search(*c), chunks)):
            # ascending features, replace only on a strictly greater proxy (NaN never replaces)
            for i in range(cp.shape[0]):
                better = cp[i] > bp
                bp = np.where(better, cp[i], bp)
                bf = np.where(better, f0 + i, bf)
                bj = np.where(better, cj[i], bj)
        # children in breadth-first order, and each in-bag row's side
        nx = hi
        side = np.zeros(n, dtype=bool)
        child = np.full(no, -1, dtype=np.int64)
        for o, k in enumerate(open_nodes):
            if bf[o] < 0:
                continue
            f, jj = int(bf[o]), int(bj[o])
            seg = G[f, segoff[o]:segoff[o] + cnt[o]]
            v = X[seg, f].astype(np.float64)
            cw, cs, cq = np.cumsum(w64[seg]), np.cumsum(wy[seg]), np.cumsum(sq[seg])
            th = v[jj - 1] / 2.0 + v[jj] / 2.0
            if th == v[jj] or np.isinf(th):
                th = v[jj - 1]
            th, WL, SL, QL = float(th), float(cw[jj - 1]), float(cs[jj - 1]), float(cq[jj - 1])
            W, S, Q, C = Wn[k], Sn[k], Qn[k], Cn[k]
            l = add_node(WL, SL, QL, jj)
            r = add_node(W - WL, S - SL, Q - QL, C - jj)
            assert (l, r) == (nx, nx + 1)
            nx += 2
            feat[k], thr[k], left[k], right[k], nanl[k] = f, th, l, r, int(jj > C - jj)
            child[o] = l
            side[seg] = X[seg, f].astype(np.float64) <= th
        if nx == hi:
            break
        # stable partition of every split node's segment into its children's, for every feature
        nodeof = np.repeat(np.arange(no), cnt)
        split = child[nodeof] >= 0
        G, V = G[:, split], V[:, split]
        nodeof = nodeof[split]
        so = np.zeros(no, dtype=np.int64)                                       # split nodes' offsets in the new G
        so[child >= 0] = np.concatenate([[0], np.cumsum(cnt[child >= 0])[:-1]])
        lcnt = np.zeros(no, dtype=np.int64)
        for o in np.nonzero(child >= 0)[0]:
            lcnt[o] = Cn[int(child[o])]
        start = so[nodeof]                                                       # segment start of each column
        before = np.arange(G.shape[1]) - start
        rstart = start + lcnt[nodeof]
        Gn, Vn = np.empty_like(G), np.empty_like(V)

        def partition(f0, f1):
            sl = side[G[f0:f1]]
            cl = np.cumsum(sl, axis=1, dtype=np.int64) - sl                     # left entries before, whole row
            cl -= np.take_along_axis(cl, np.broadcast_to(start, cl.shape), axis=1)
            dest = np.where(sl, start + cl, rstart + (before - cl))
            np.put_along_axis(Gn[f0:f1], dest, G[f0:f1], axis=1)
            np.put_along_axis(Vn[f0:f1], dest, V[f0:f1], axis=1)

        fp = max(1, chunk_elems // G.shape[1])
        list(pool.map(lambda c: partition(*c), [(f0, min(width, f0 + fp)) for f0 in range(0, width, fp)]))
        G, V = Gn, Vn
        seg_nodes = [int(child[o]) + s for o in np.nonzero(child >= 0)[0] for s in (0, 1)]
        seg_off = [int(so[o]) + s * int(lcnt[o]) for o in np.nonzero(child >= 0)[0] for s in (0, 1)]
        lo, hi = hi, nx
    pool.shutdown()
    return dict(feature=np.array(feat, dtype=np.int32), threshold=np.array(thr, dtype=np.float64),
                left=np.array(left, dtype=np.int32), right=np.array(right, dtype=np.int32),
                value=np.array(val, dtype=np.float64), missing_go_to_left=np.array(nanl, dtype=np.int32))


def apply(tree: dict, X: np.ndarray) -> np.ndarray:
    """Leaf index of every row of float32 X (DecisionTreeRegressor.apply: x <= threshold goes left, compared in fp64; NaN
    goes left where missing_go_to_left is set, right elsewhere)."""
    X = np.asarray(X, dtype=np.float32)
    node = np.zeros(X.shape[0], dtype=np.int64)
    nanl = np.asarray(tree.get("missing_go_to_left", np.zeros(tree["feature"].size, np.int32))) != 0
    while True:
        f = tree["feature"][node]
        inner = f >= 0
        if not inner.any():
            return node
        idx = np.nonzero(inner)[0]
        x = X[idx, f[idx]].astype(np.float64)
        k = node[idx]
        node[idx] = np.where((x <= tree["threshold"][k]) | (np.isnan(x) & nanl[k]), tree["left"][k], tree["right"][k])


def tree_predict(tree: dict, X) -> np.ndarray:
    return tree["value"][apply(tree, X)]


# ---------------------------------------------------------------------------------------------------------------- forest
def fit(X, y, counts, grow=grow_tree):
    """(trees, est_noise) of one output: X float32 [n, width], y float32 [n] (non-finite rows weigh 0), counts [T, n].
    grow: grow_tree, or grow_tree_level for large inputs (the same trees)."""
    y = np.asarray(y, dtype=np.float32)
    keep = np.isfinite(y)
    trees = [grow(X, np.where(keep, y, 0.0).astype(np.float32), np.where(keep, np.maximum(c, 0), 0))
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


def predict_fast(trees, X, noise_b) -> tuple:
    """predict, vectorised over candidates with the reference's own expressions: P [m, T] of leaf values, the mean as
    forest_mean64's sequential tree sum, the variance as np.var(P, axis=1) (rf.py:55), then fp32 and + noise in fp32."""
    P = np.stack([tree_predict(t, X) for t in trees], axis=1)          # C-contiguous [m, T], as np.concatenate(axis=1)
    s = np.zeros(P.shape[0], dtype=np.float64)
    for t in range(P.shape[1]):
        s = s + P[:, t]
    mean = (s / P.shape[1]).astype(np.float32)
    return mean, np.var(P, axis=1).astype(np.float32) + np.float32(noise_b)
