"""The random-forest oracle (oracle/rf_oracle.py) against the reference's own sklearn forests
(tests/golden/ref_rf.npz, tests/golden/make_ref_rf.py) and against numpy: the oracle grown from the reference's bootstrap
counts splits the in-bag rows into the same leaves and predicts them alike; its restatement of RF.predict and of the
noise estimate equals the reference bit for bit on the reference's trees; its pairwise sum is numpy's."""
import os

import numpy as np
import pytest

from oracle import rf_oracle as R

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "ref_rf.npz"))
VARIANTS = [str(v) for v in GOLD["variants"]]


def variant(name):
    p = name + "/"
    g = {k[len(p):]: GOLD[k] for k in GOLD.files if k.startswith(p)}
    g["uniqs"] = [int(u) for u in g["uniqs"]]
    g["X"] = R.tree_inputs(g["Xc"], g["Xe"], g["uniqs"])
    g["X_test"] = R.tree_inputs(g["Xc_test"], g["Xe_test"], g["uniqs"])
    g["trees"] = [{k: g[k][t, :g["ncount"][t]] for k in ("feature", "threshold", "left", "right", "value")}
                  for t in range(int(g["T"]))]
    return g


def partition(leaves, rows):
    """The in-bag rows grouped by leaf, as a set of frozensets (invariant to node numbering)."""
    groups = {}
    for r in rows:
        groups.setdefault(int(leaves[r]), set()).add(int(r))
    return {frozenset(s) for s in groups.values()}


def same_partitions(trees, X, y, counts, ref_apply, ref_trees):
    for t, c in enumerate(counts):
        rows = np.nonzero(c > 0)[0]
        assert partition(R.apply(trees[t], X), rows) == partition(ref_apply[t], rows), f"tree {t}"
        mine, ref = R.tree_predict(trees[t], X)[rows], ref_trees[t]["value"][ref_apply[t][rows]]
        np.testing.assert_allclose(mine, ref, rtol=1e-12, atol=1e-12 * np.abs(y[np.isfinite(y)]).max())


@pytest.mark.parametrize("name", VARIANTS)
def test_oracle_partitions_match_reference(name):
    g = variant(name)
    y = g["y"].reshape(-1)
    trees, _ = R.fit(g["X"], y, g["counts"])
    same_partitions(trees, g["X"], y, g["counts"], g["apply"], g["trees"])


@pytest.mark.parametrize("name", VARIANTS)
def test_predict_restatement_is_the_reference(name):
    g = variant(name)
    y = g["y"].reshape(-1)
    keep = np.isfinite(y)
    nz = R.noise(g["trees"], g["X"][keep], y[keep])
    assert nz.tobytes() == g["noise"].astype(np.float32).tobytes()
    mean, var = R.predict(g["trees"], g["X_test"], nz)
    assert mean.tobytes() == g["mean"].reshape(-1).astype(np.float32).tobytes()
    assert var.tobytes() == g["var"].reshape(-1).astype(np.float32).tobytes()


def test_pairwise_sum_is_numpys():
    rng = np.random.default_rng(0)
    for T in list(range(1, 301)) + [511, 1023, 1024, 4097, 8192]:
        P = rng.standard_normal((4, T)) * 10.0 ** rng.uniform(-4, 4, (4, T))
        v = np.var(P, axis=1)
        for i in range(4):
            mu = R.pairwise_sum(P[i]) / T
            d = P[i] - mu
            assert R.pairwise_sum(d * d) / T == v[i], T
            assert R.pairwise_sum(P[i]) / T == np.mean(P[i]), T


def test_bootstrap_restatement():
    n, kept = 40, np.array([0, 3, 4, 9, 10, 11, 20, 21, 39])
    c = R.bootstrap_counts(123, 1, 7, kept, n)
    assert c.sum() == kept.size and np.all(c[np.setdiff1d(np.arange(n), kept)] == 0)
    assert not np.array_equal(c, R.bootstrap_counts(123, 1, 8, kept, n))
    assert not np.array_equal(c, R.bootstrap_counts(123, 0, 7, kept, n))
    assert np.array_equal(c, R.bootstrap_counts(123, 1, 7, kept, n))


def test_oracle_matches_sklearn_trees_on_fresh_data():
    tree = pytest.importorskip("sklearn.tree")
    rng = np.random.default_rng(5)
    for trial in range(30):
        n, d = int(rng.choice([7, 40, 200])), int(rng.choice([1, 4, 9]))
        kind = trial % 3
        if kind == 0:
            X = rng.standard_normal((n, d)).astype(np.float32)
        elif kind == 1:
            X = rng.integers(0, 3, (n, d)).astype(np.float32)
        else:
            X = (rng.random((n, d)) < 0.3).astype(np.float32)
        y = rng.standard_normal(n).astype(np.float32)
        w = np.bincount(rng.integers(0, n, n), minlength=n)
        t = R.grow_tree(X, y, w)
        sk = tree.DecisionTreeRegressor(random_state=trial).fit(X, y.astype(np.float64), sample_weight=w.astype(np.float64))
        rows = np.nonzero(w > 0)[0]
        assert partition(R.apply(t, X), rows) == partition(sk.apply(X), rows)
        np.testing.assert_allclose(R.tree_predict(t, X)[rows], sk.predict(X)[rows], rtol=1e-12, atol=1e-12)
