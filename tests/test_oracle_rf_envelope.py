"""The level-synchronous forest oracle (rf_oracle.grow_tree_level) and the vectorised predict reference
(rf_oracle.predict_fast) against their readable definitions and against the reference's forests across the envelope of
forest.cu (tests/golden/ref_rf_envelope.npz, tests/golden/make_ref_rf_envelope.py):
  - grow_tree_level is grow_tree bit for bit, node for node, on every ref_rf.npz variant and on random trees over sizes,
    column kinds, signed zeros, cut spacings at FEATURE_THRESHOLD, weights and targets that stress the split search;
  - grown from the reference's bootstrap counts at n = 8192, 5000 and 2048 (width up to 1024), it splits the in-bag rows
    into the reference's leaves;
  - predict_fast is predict byte for byte, and the reference's RF.predict on the fixture's held-out rows (T = 129, 1024,
    NaN candidates);
  - its wall time at n = 8192, width 4096 (one tree), which the device tests pay for their largest case."""
import functools
import hashlib
import os
import time
import zlib

import numpy as np
import pytest

from oracle import rf_oracle as R
from tests.test_oracle_rf import VARIANTS, same_partitions, variant

# name: (n training rows, held-out rows, num_cont, num_uniqs, n_estimators, kind)
ENVELOPE = {
    "ties_n8192_w64_t2": (8192, 64, 64, [], 2, "ties"),
    "mixed_n5000_w51_t2": (5000, 64, 8, [3, 40], 2, "num"),
    "num_n2048_w1024_t1": (2048, 64, 1024, [], 1, "num"),
    "pred_n50_w3_t129": (50, 300, 3, [], 129, "num"),
    "pred_n50_w3_t1024": (50, 300, 3, [], 1024, "num"),
    "nancand_n50_w3_t20": (50, 64, 3, [], 20, "nan_candidates"),
}
LARGE = [k for k, v in ENVELOPE.items() if v[0] > 1000]


def envelope_inputs(name):
    """(Xc float32 [n + m, num_cont], Xe int64 [n + m, num_enum] or None, y float32 [n + m]) of an ENVELOPE variant:
    Gaussian columns (kind 'ties': the last one integer-valued in 0 .. 5), categories uniform, y = sin(first four
    columns + categories / 2) + noise; kind 'nan_candidates': held-out row r has NaN in column 0 (r % 4 == 1), in the
    other columns (r % 4 == 2) or in all of them (r % 4 == 3)."""
    n, m, dc, uniqs, _, kind = ENVELOPE[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    Xc = rng.standard_normal((n + m, dc)).astype(np.float32)
    if kind == "ties":
        Xc[:, -1] = rng.integers(0, 6, n + m)
    Xe = np.stack([rng.integers(0, u, n + m) for u in uniqs], 1) if uniqs else None
    base = Xc[:, :4].astype(np.float64).sum(1) + (0.5 * Xe.sum(1) if uniqs else 0.0)
    y = (np.sin(base) + 0.1 * rng.standard_normal(n + m)).astype(np.float32)
    if kind == "nan_candidates":
        r = np.arange(n, n + m)
        Xc[r[r % 4 == 1], 0] = np.nan
        Xc[r[r % 4 == 2], 1:] = np.nan
        Xc[r[r % 4 == 3], :] = np.nan
    return Xc, Xe, y


def inputs_digest(Xc, Xe, y) -> str:
    h = hashlib.sha256()
    for a in (Xc, Xe, y):
        if a is not None:
            h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


@functools.lru_cache(maxsize=None)
def _gold():
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "ref_rf_envelope.npz"))


def env_variant(name):
    """An ENVELOPE variant with the reference's forest: training / held-out inputs, tree inputs X, trees, counts, apply,
    RF.predict's (mean, var) on the held-out rows and RF.noise."""
    G = _gold()
    p = name + "/"
    g = {k[len(p):]: G[k] for k in G.files if k.startswith(p)}
    n, m, dc, uniqs, T, _ = ENVELOPE[name]
    Xc, Xe, y = envelope_inputs(name)
    assert inputs_digest(Xc, Xe, y) == str(g["digest"]), "inputs no longer regenerate as recorded"
    g.update(uniqs=list(uniqs), T=T, y=y[:n], Xc=Xc[:n], Xc_test=Xc[n:],
             Xe=Xe[:n] if uniqs else np.zeros((n, 0), np.int64), Xe_test=Xe[n:] if uniqs else np.zeros((m, 0), np.int64))
    g["X"] = R.tree_inputs(g["Xc"], g["Xe"], g["uniqs"])
    g["X_test"] = R.tree_inputs(g["Xc_test"], g["Xe_test"], g["uniqs"])
    g["trees"] = [{k: g[k][t, :g["ncount"][t]] for k in ("feature", "threshold", "left", "right", "value",
                                                          "missing_go_to_left")} for t in range(T)]
    return g


def assert_same_tree(a, b, what=""):
    assert len(a["feature"]) == len(b["feature"]), what
    for k in ("feature", "left", "right", "missing_go_to_left"):
        assert np.array_equal(a[k], b[k]), (what, k)
    for k in ("threshold", "value"):
        assert a[k].tobytes() == b[k].tobytes(), (what, k)


def test_fixture_records_the_reference():
    G = _gold()
    assert str(G["sklearn_version"]) == "1.9.0"
    assert [str(v) for v in G["variants"]] == list(ENVELOPE)
    assert G["inf_raises"].tolist() == [True, True]          # RF.predict refuses +inf and -inf candidates


@pytest.mark.parametrize("name", VARIANTS)
def test_level_equals_grow_tree_on_fixture(name):
    g = variant(name)
    y = g["y"].reshape(-1)
    a, na = R.fit(g["X"], y, g["counts"])
    b, nb = R.fit(g["X"], y, g["counts"], grow=R.grow_tree_level)
    for t, (ta, tb) in enumerate(zip(a, b)):
        assert_same_tree(ta, tb, t)
    assert na.tobytes() == nb.tobytes()


def _random_case(rng, n, d):
    """(X, y, w) of one random tree: a column kind, a target kind and a weight kind drawn from rng."""
    kind = int(rng.integers(0, 6))
    if kind == 0:                                    # Gaussian
        X = rng.standard_normal((n, d))
    elif kind == 1:                                  # integer-valued, heavy ties
        X = rng.integers(0, 4, (n, d))
    elif kind == 2:                                  # 0/1
        X = rng.random((n, d)) < 0.3
    elif kind == 3:                                  # mixed numeric, integer and 0/1 columns
        X = np.stack([[rng.standard_normal, lambda k: rng.integers(-2, 3, k), lambda k: rng.random(k) < 0.5][c % 3](n)
                      for c in range(d)], 1)
    elif kind == 4:                                  # zeros of both signs among a few values
        X = rng.choice(np.array([-0.0, 0.0, 1.0, -1.5], np.float32), (n, d))
    else:                                            # spacings just below and above FEATURE_THRESHOLD near 0
        steps = rng.choice(np.array([0.9e-7, 1.0e-7, 1.1e-7, 2e-7, 0.0]), (n, d))
        X = np.cumsum(steps, axis=0)[rng.permutation(n)] - 1e-6
    X = np.asarray(X, dtype=np.float32)
    ykind = int(rng.integers(0, 4))
    if ykind == 0:
        y = np.full(n, 0.25, np.float32)             # constant: the root is a leaf
    elif ykind == 1:
        y = (4.0 ** rng.permutation(min(n, 60)))[np.arange(n) % min(n, 60)].astype(np.float32)   # geometric, as 'chain'
    else:
        y = rng.standard_normal(n).astype(np.float32)
    wkind = int(rng.integers(0, 6))
    w = np.bincount(rng.integers(0, n, n), minlength=n)
    if wkind == 1:
        w = np.zeros(n, np.int64)
        w[rng.integers(0, n)] = 1                   # one-hot
    elif wkind == 2:
        w = w * int(rng.choice([1000, 1 << 20, (1 << 31) - 1])) // max(1, w.max())   # huge
    elif wkind == 3:
        w = np.zeros(n, np.int64)                   # all zero: the root's value is NaN
    elif wkind == 4:
        w = (rng.random(n) < 0.5).astype(np.int64)
    return X, y, w


@pytest.mark.parametrize("block", range(8))
def test_level_equals_grow_tree_random(block):
    """8 blocks x 30 trees: n in {1, 2, 7, 40, 300, 1500}, widths 1 .. 40 (1 .. 6 at n = 1500)."""
    rng = np.random.default_rng(1000 + block)
    for trial in range(30):
        n = int(rng.choice([1, 2, 7, 40, 300, 1500], p=[0.1, 0.1, 0.2, 0.3, 0.25, 0.05]))
        d = int(rng.integers(1, 7 if n == 1500 else 41))
        X, y, w = _random_case(rng, n, d)
        with np.errstate(divide="ignore", invalid="ignore"):
            a = R.grow_tree(X, y, w)
        b = R.grow_tree_level(X, y, w)
        assert_same_tree(a, b, (block, trial, n, d))


def test_level_edge_cases():
    """Every row cut exactly at FEATURE_THRESHOLD apart (no valid cut) and just above it; -0 / +0 in one column; the
    chain corner (y = 4^i on one feature, depth n - 1)."""
    n = 64
    y = np.random.default_rng(0).standard_normal(n).astype(np.float32)
    w = np.ones(n, np.int64)
    for step in (1e-7, 1.0000001e-7, 1.2e-7):
        X = (np.arange(n) * step).astype(np.float32)[:, None]
        assert_same_tree(R.grow_tree(X, y, w), R.grow_tree_level(X, y, w), step)
    X = np.where(np.arange(n) % 2, np.float32(-0.0), np.float32(0.0))[:, None].astype(np.float32)
    X[::7] = 1.0
    assert_same_tree(R.grow_tree(X, y, w), R.grow_tree_level(X, y, w), "signed zeros")
    X = np.arange(n, dtype=np.float32)[:, None]
    yc = (4.0 ** np.arange(n)).astype(np.float32)
    t = R.grow_tree_level(X, yc, w)
    assert_same_tree(R.grow_tree(X, yc, w), t, "chain")
    assert t["feature"].size == 2 * n - 1


def test_missing_go_to_left_rule_is_sklearns():
    """sklearn (trained without NaN) sends NaN to the child with more distinct in-bag rows, ties right: the rule
    grow_tree records, checked on every internal node of fresh sklearn trees through apply."""
    tree = pytest.importorskip("sklearn.tree")
    rng = np.random.default_rng(9)
    seen = set()
    for trial in range(20):
        n, d = int(rng.choice([7, 40, 200])), int(rng.choice([1, 3]))
        X = rng.integers(0, 3, (n, d)).astype(np.float32) if trial % 2 else rng.standard_normal((n, d)).astype(np.float32)
        y = rng.standard_normal(n)
        w = np.bincount(rng.integers(0, n, n), minlength=n)
        t = tree.DecisionTreeRegressor(random_state=trial).fit(X, y, sample_weight=w.astype(np.float64)).tree_
        rows = np.nonzero(w > 0)[0]
        reach = np.zeros(t.node_count, np.int64)
        for r in rows:                                          # distinct in-bag rows through each node
            k = 0
            while True:
                reach[k] += 1
                if t.children_left[k] < 0:
                    break
                k = t.children_left[k] if X[r, t.feature[k]] <= t.threshold[k] else t.children_right[k]
        inner = np.nonzero(t.children_left >= 0)[0]
        nl, nr = reach[t.children_left[inner]], reach[t.children_right[inner]]
        assert np.array_equal(t.missing_go_to_left[inner].astype(bool), nl > nr), trial
        seen.update(zip((nl > nr).tolist(), (nl == nr).tolist()))
    assert {(True, False), (False, False), (False, True)} <= seen          # left, right, and ties going right


@pytest.mark.parametrize("name", LARGE)
def test_level_reproduces_reference_partitions(name):
    g = env_variant(name)
    t0 = time.perf_counter()
    trees, _ = R.fit(g["X"], g["y"], g["counts"], grow=R.grow_tree_level)
    print(f"{name}: grow_tree_level {time.perf_counter() - t0:.1f} s for {len(trees)} trees")
    same_partitions(trees, g["X"], g["y"], g["counts"], g["apply"], g["trees"])


@pytest.mark.parametrize("name", VARIANTS)
def test_predict_fast_is_predict(name):
    g = variant(name)
    nz = g["noise"].astype(np.float32)[0]
    m1, v1 = R.predict(g["trees"], g["X_test"], nz)
    m2, v2 = R.predict_fast(g["trees"], g["X_test"], nz)
    assert m1.tobytes() == m2.tobytes() and v1.tobytes() == v2.tobytes()
    assert m2.tobytes() == g["mean"].reshape(-1).astype(np.float32).tobytes()
    assert v2.tobytes() == g["var"].reshape(-1).astype(np.float32).tobytes()


@pytest.mark.parametrize("name", list(ENVELOPE))
def test_predict_fast_is_the_reference(name):
    g = env_variant(name)
    mean, var = R.predict_fast(g["trees"], g["X_test"], g["noise"].astype(np.float32)[0])
    assert mean.tobytes() == g["mean"].astype(np.float32).tobytes()
    assert var.tobytes() == g["var"].astype(np.float32).tobytes()
    if ENVELOPE[name][5] == "nan_candidates":
        assert np.isnan(g["X_test"]).any(axis=1).sum() == 3 * g["X_test"].shape[0] // 4
        assert np.isfinite(mean).all()


def test_level_oracle_time_at_the_largest_envelope():
    """One tree at n = 8192, width 4096: the device tests grow this with grow_tree_level, so its wall time is their
    largest oracle cost.  Every in-bag row lands in a leaf, and each leaf's value is the weighted mean of its rows."""
    n, d = 8192, 4096
    rng = np.random.default_rng(4096)
    X = rng.standard_normal((n, d)).astype(np.float32)
    y = np.sin(X[:, :4].sum(1)).astype(np.float32)
    w = np.bincount(rng.integers(0, n, n), minlength=n)
    t0 = time.perf_counter()
    t = R.grow_tree_level(X, y, w)
    dt = time.perf_counter() - t0
    print(f"grow_tree_level n = {n}, width {d}: {dt:.1f} s on {os.cpu_count()} host cores, {t['feature'].size} nodes")
    rows = np.nonzero(w > 0)[0]
    leaves = R.apply(t, X[rows])
    assert np.all(t["feature"][leaves] < 0)
    ref = np.bincount(leaves, w[rows] * y[rows].astype(np.float64), t["value"].size) / \
        np.maximum(np.bincount(leaves, w[rows].astype(np.float64), t["value"].size), 1)
    np.testing.assert_allclose(t["value"][leaves], ref[leaves], rtol=1e-12, atol=1e-12)
    assert dt < 600
