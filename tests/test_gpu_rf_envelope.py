"""hb_rf_fit / hb_rf_predict / hb_rf_load across the envelope of forest.cu, against the level-synchronous fp64 oracle
(rf_oracle.grow_tree_level, bit for bit with grow_tree), the vectorised predict reference (rf_oracle.predict_fast, the
reference's own expressions) and the reference's forests (tests/golden/ref_rf_envelope.npz):
  - fit node for node, NaN routing flags and est_noise included: n at and around the bitonic sort's powers of two and
    its 48 KiB shared-memory edge x widths below, at and above the 8 warps; width 4096 at n = 8192 (numeric, and
    mixed with one-hot blocks of 1 and 2048 categories); the Philox draws at n = 8192; 32 outputs with NaN targets;
    more trees than grow slots; the fixture's large variants against the reference's partitions;
  - est_noise at kept-row counts on numpy's pairwise-sum branch edges;
  - predict byte for byte for T and m at the pairwise-sum and block edges, multi-output forests, the fixture's T = 129
    and T = 1024 forests and its NaN candidates; thresholds between floats, on floats, at +-0 and beyond +-FLT_MAX
    against candidates on RD32(t), one ulp above, on t, at +-0, +-inf and NaN; draws at B = 3, odd m.
Each large case prints its oracle time."""
import ctypes as C
import time

import numpy as np
import pytest
import torch

from hebo_b200 import RF, _lib
from hebo_b200.forest import forest_trees
from oracle import rf_oracle as R
from oracle import rng_oracle
from tests.test_gpu_rf import _raw_fit, assert_same_forest, rd32
from tests.test_oracle_rf import same_partitions
from tests.test_oracle_rf_envelope import ENVELOPE, LARGE, env_variant

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _oracle_fit(X, y, counts, label):
    t0 = time.perf_counter()
    out = R.fit(X, y, counts, grow=R.grow_tree_level)
    print(f"{label}: oracle {time.perf_counter() - t0:.1f} s")
    return out


def _fit_numeric(X, y, counts):
    m = RF(X.shape[1], 0, 1, n_estimators=counts.shape[0])
    m.fit(torch.from_numpy(X), None, torch.from_numpy(y)[:, None], counts=counts)
    return m


def _counts(rng, T, n):
    return np.stack([np.bincount(rng.integers(0, n, n), minlength=n) for _ in range(T)]).astype(np.int32)


@pytest.mark.parametrize("n", [1023, 1024, 1025, 4096, 4097, 8192])
@pytest.mark.parametrize("width", [1, 7, 8, 9, 64])
def test_fit_node_for_node(n, width):
    rng = np.random.default_rng(n * 100 + width)
    X = rng.standard_normal((n, width)).astype(np.float32)
    X[:, ::3] = np.round(X[:, ::3] * 2)                      # every third column integer-valued: ties in the sort
    y = (np.sin(X.sum(1)) + 0.1 * rng.standard_normal(n)).astype(np.float32)
    counts = _counts(rng, 1, n)
    m = _fit_numeric(X, y, counts)
    ref, nz = _oracle_fit(X, y, counts, f"n {n} width {width}")
    assert_same_forest(m.trees(), ref)
    assert m.noise.numpy().tobytes() == np.float32(nz).tobytes()


@pytest.mark.parametrize("mixed", [False, True])
def test_fit_width_4096(mixed):
    """n = 8192 at width 4096, node for node: numeric, or 1024 numeric columns and one-hot blocks of 1, 2048 and 1023."""
    n = 8192
    rng = np.random.default_rng(4096 + mixed)
    uniqs = [1, 2048, 1023] if mixed else []
    dc = 4096 - sum(uniqs)
    Xc = rng.standard_normal((n, dc)).astype(np.float32)
    Xe = np.stack([rng.integers(0, u, n) for u in uniqs], 1) if mixed else None
    y = (np.sin(Xc[:, :4].sum(1)) + (0.3 * (Xe[:, 1] % 7) if mixed else 0)).astype(np.float32)
    counts = _counts(rng, 1, n)
    m = RF(dc, len(uniqs), 1, n_estimators=1, **({"num_uniqs": uniqs} if mixed else {}))
    m.fit(torch.from_numpy(Xc), torch.from_numpy(Xe) if mixed else None, torch.from_numpy(y)[:, None], counts=counts)
    X = R.tree_inputs(Xc, Xe, uniqs)
    ref, nz = _oracle_fit(X, y, counts, f"n 8192 width 4096 mixed={mixed}")
    assert_same_forest(m.trees(), ref)
    assert m.noise.numpy().tobytes() == np.float32(nz).tobytes()


def test_fit_philox_draws_at_8192():
    n = 8192
    rng = np.random.default_rng(81)
    X = rng.standard_normal((n, 8)).astype(np.float32)
    y = np.sin(X.sum(1)).astype(np.float32)
    y[::97] = np.nan
    m = RF(8, 0, 1, n_estimators=2)
    torch.manual_seed(3)
    m.fit(torch.from_numpy(X), None, torch.from_numpy(y)[:, None])
    kept = np.nonzero(np.isfinite(y))[0]
    counts = np.stack([R.bootstrap_counts(m.seed, 0, t, kept, n) for t in range(2)])
    ref, nz = _oracle_fit(X, y, counts, "philox n 8192")
    assert_same_forest(m.trees(), ref)
    assert m.noise.numpy().tobytes() == np.float32(nz).tobytes()


def test_fit_32_outputs_with_nan_targets():
    n, d, T, B = 300, 5, 2, 32
    rng = np.random.default_rng(32)
    X = rng.standard_normal((n, d)).astype(np.float32)
    Y = (np.sin(X @ rng.standard_normal((d, B))) + 0.1 * rng.standard_normal((n, B))).astype(np.float32)
    Y[rng.random((n, B)) < 0.05] = np.nan
    counts = np.stack([_counts(rng, T, n) for _ in range(B)])
    trees, noise = _raw_fit(torch.from_numpy(X).to(DEV), torch.from_numpy(Y).to(DEV).contiguous(), _lib.RfSpec(d, 0, None),
                            T, counts, 5)
    for b in range(B):
        ref, nz = R.fit(X, Y[:, b], counts[b], grow=R.grow_tree_level)
        assert_same_forest(trees[b * T:(b + 1) * T], ref)
        assert noise[b].numpy().tobytes() == np.float32(nz).tobytes()


def test_fit_reuses_grow_slots():
    """B T = 400 trees > 264 slots at n = 1024: trees 0, 263, 264, 265 and 399 node for node, and each output bit for bit
    with its own single-output fit."""
    n, d, T, B = 1024, 3, 200, 2
    rng = np.random.default_rng(400)
    X = rng.standard_normal((n, d)).astype(np.float32)
    Y = np.sin(X @ rng.standard_normal((d, B))).astype(np.float32)
    counts = np.stack([_counts(rng, T, n) for _ in range(B)])
    Xd, Yd, spec = torch.from_numpy(X).to(DEV), torch.from_numpy(Y).to(DEV).contiguous(), _lib.RfSpec(d, 0, None)
    trees, noise = _raw_fit(Xd, Yd, spec, T, counts, 7)
    for q in (0, 263, 264, 265, 399):
        b, t = divmod(q, T)
        assert_same_forest([trees[q]], [R.grow_tree_level(X, Y[:, b], counts[b, t])])
    for b in range(B):
        single, sn = _raw_fit(Xd, Yd[:, b:b + 1].contiguous(), spec, T, counts[b:b + 1].copy(), 7)
        assert_same_forest(single, trees[b * T:(b + 1) * T])
        assert sn[0].numpy().tobytes() == noise[b].numpy().tobytes()


@pytest.mark.parametrize("name", LARGE)
def test_fit_reproduces_reference_partitions(name):
    g = env_variant(name)
    m = RF(g["Xc"].shape[1], len(g["uniqs"]), 1, n_estimators=g["T"], **({"num_uniqs": g["uniqs"]} if g["uniqs"] else {}))
    m.fit(torch.from_numpy(g["Xc"]), torch.from_numpy(g["Xe"]) if g["uniqs"] else None, torch.from_numpy(g["y"])[:, None],
          counts=g["counts"])
    same_partitions(m.trees(), g["X"], g["y"], g["counts"], g["apply"], g["trees"])


@pytest.mark.parametrize("nkept", [1, 7, 8, 127, 128, 129, 1024, 1025, 8192])
def test_noise_pairwise_edges(nkept):
    n = 8192
    rng = np.random.default_rng(nkept)
    X = rng.standard_normal((n, 2)).astype(np.float32)
    y = np.full(n, np.nan, np.float32)
    rows = rng.choice(n, nkept, replace=False)
    y[rows] = rng.standard_normal(nkept) * 10.0 ** rng.uniform(-3, 3, nkept)
    counts = _counts(rng, 1, n)
    m = _fit_numeric(X, y, counts)
    keep = np.isfinite(y)
    assert m.noise.numpy().tobytes() == R.noise(m.trees(), X[keep], y[keep]).tobytes()
    assert_same_forest(m.trees(), R.fit(X, y, counts, grow=R.grow_tree_level)[0])


def _random_tree(rng, d, depth):
    """A random tree in sklearn's layout (depth-first numbering), thresholds from N(0, 1) in fp64, missing_go_to_left
    random on every node (a flag on a leaf must not make it internal)."""
    feat, thr, left, right, val, nanl = [], [], [], [], [], []

    def node(level):
        k = len(feat)
        for lst, v in ((feat, -2), (thr, -2.0), (left, -1), (right, -1), (val, float(rng.standard_normal())),
                       (nanl, int(rng.integers(0, 2)))):
            lst.append(v)
        if level < depth and rng.random() < 0.85:
            feat[k], thr[k], nanl[k] = int(rng.integers(0, d)), float(rng.standard_normal()), int(rng.integers(0, 2))
            left[k] = node(level + 1)
            right[k] = node(level + 1)
        return k
    node(0)
    return dict(feature=np.array(feat, np.int32), threshold=np.array(thr), left=np.array(left, np.int32),
                right=np.array(right, np.int32), value=np.array(val), missing_go_to_left=np.array(nanl, np.int32))


@pytest.mark.parametrize("T", [1, 7, 8, 9, 127, 128, 129, 135, 136, 255, 256, 257, 1023, 1024])
def test_predict_loaded_forest(T):
    rng = np.random.default_rng(T)
    d = 4
    trees = [_random_tree(rng, d, 6) for _ in range(T)]
    Xall = rng.standard_normal((20000, d)).astype(np.float32)
    Xall[::53, 1] = np.nan
    noise = np.float32(0.0123)
    mean, var = R.predict_fast(trees, Xall, noise)
    model = RF(d, 0, 1, n_estimators=T)
    model.load_trees(trees, float(noise))
    for m in (1, 127, 128, 129, 20000):
        py, ps2 = model.predict(torch.from_numpy(Xall[:m]))
        assert py.numpy().reshape(-1).tobytes() == mean[:m].tobytes(), m
        assert ps2.numpy().reshape(-1).tobytes() == var[:m].tobytes(), m


def _predict_raw(forest, X, B, T, noise, n_samples=0, seed=0, counter=0):
    m = X.shape[0]
    Xd = torch.from_numpy(X).to(DEV).contiguous()
    mean = torch.empty(m, B, device=DEV)
    var = torch.empty(m, B, device=DEV)
    samp = torch.empty(max(n_samples, 1), m, B, device=DEV)
    spec = _lib.RfSpec(X.shape[1], 0, None)
    _lib.check(_lib.lib().hb_rf_predict(_lib.ptr(Xd), None, m, C.byref(spec), _lib.ptr(forest), B, T, _lib.ptr(noise),
                                        _lib.ptr(mean), _lib.ptr(var), n_samples, seed, counter, _lib.ptr(samp),
                                        _lib.stream_ptr()), "hb_rf_predict")
    return mean.cpu().numpy(), var.cpu().numpy(), samp.cpu().numpy()


def _fit_forest(B, T, n, d, seed):
    """(device forest, device noise, X, Y) of a B-output fit from the device's Philox draws."""
    lib = _lib.lib()
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(np.float32)
    Y = np.sin(X @ rng.standard_normal((d, B))).astype(np.float32)
    spec = _lib.RfSpec(d, 0, None)
    ws_bytes = int(lib.hb_rf_fit_workspace_bytes(n, C.byref(spec), B, T))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    forest = torch.empty(int(lib.hb_rf_forest_bytes(C.byref(spec), 2 * n - 1, B, T)), dtype=torch.uint8, device=DEV)
    noise = torch.empty(B, dtype=torch.float32, device=DEV)
    Xd, Yd = torch.from_numpy(X).to(DEV), torch.from_numpy(Y).to(DEV).contiguous()
    _lib.check(lib.hb_rf_fit(_lib.ptr(Xd), None, _lib.ptr(Yd), n, C.byref(spec), B, T, None, seed, _lib.ptr(forest),
                             _lib.ptr(noise), _lib.ptr(ws), ws_bytes, _lib.stream_ptr()), "hb_rf_fit")
    return forest, noise, X, Y


@pytest.mark.parametrize("B", [3, 32])
def test_predict_multi_output(B):
    T = 9
    forest, noise, X, _ = _fit_forest(B, T, 200, 4, B)
    trees = forest_trees(forest)
    Xs = np.random.default_rng(1).standard_normal((300, 4)).astype(np.float32)
    Xs[::11, 2] = np.nan
    mean, var, _ = _predict_raw(forest, Xs, B, T, noise)
    nz = noise.cpu().numpy()
    for b in range(B):
        rm, rv = R.predict_fast(trees[b * T:(b + 1) * T], Xs, nz[b])
        assert mean[:, b].tobytes() == rm.tobytes() and var[:, b].tobytes() == rv.tobytes(), b


@pytest.mark.parametrize("name", [k for k in ENVELOPE if k not in LARGE])
def test_predict_fixture_is_the_reference(name):
    g = env_variant(name)
    m = RF(3, 0, 1, n_estimators=g["T"])
    m.load_trees(g["trees"], float(g["noise"][0]))
    mean, var = m.predict(torch.from_numpy(g["Xc_test"]), None)
    assert mean.numpy().reshape(-1).tobytes() == g["mean"].astype(np.float32).tobytes()
    assert var.numpy().reshape(-1).tobytes() == g["var"].astype(np.float32).tobytes()


def test_thresholds_and_non_finite_candidates():
    f32 = np.float32
    ths = [0.1, 1.0 / 3.0, -0.7, 0.5, 1.0, -2.0, 0.0, -0.0, 1e300, -1e300, 3.4028235677973366e38, float(np.finfo(f32).max)]
    trees = []
    for i, th in enumerate(ths):
        for nl in (0, 1):
            trees.append(dict(feature=np.array([0, -2, -2], np.int32), threshold=np.array([th, -2.0, -2.0]),
                              left=np.array([1, -1, -1], np.int32), right=np.array([2, -1, -1], np.int32),
                              value=np.array([0.0, 1.0, 2.0]), missing_go_to_left=np.array([nl, 0, 0], np.int32)))
    inf = f32(np.inf)
    for tree in trees:
        th = tree["threshold"][0]
        r = rd32(th)
        cands = np.array([r, np.nextafter(r, inf), f32(th), f32(0.0), f32(-0.0), inf, -inf, f32(np.nan),
                          np.nextafter(r, -inf), np.finfo(f32).max, -np.finfo(f32).max], np.float32)
        m = RF(1, 0, 1, n_estimators=1)
        m.load_trees([tree], 0.0)
        mean, _, _ = m._predict_dev(torch.from_numpy(cands[:, None]).to(DEV), None)
        want = tree["value"][R.apply(tree, cands[:, None])].astype(np.float32)
        assert mean.cpu().numpy().reshape(-1).tobytes() == want.tobytes(), (th, tree["missing_go_to_left"][0])
        assert want[7] == (1.0 if tree["missing_go_to_left"][0] else 2.0)          # NaN follows the flag
        assert want[5] == (1.0 if th >= np.inf else 2.0) and want[6] == 1.0          # +inf right, -inf left


def test_draws_b3_odd_m():
    B, T, m, S = 3, 5, 257, 5
    forest, noise, _, _ = _fit_forest(B, T, 120, 3, 11)
    Xs = np.random.default_rng(2).standard_normal((m, 3)).astype(np.float32)
    mean, var, samp = _predict_raw(forest, Xs, B, T, noise, n_samples=S, seed=4321, counter=9)
    q = np.arange(S * m * B)
    z0, z1, r0, r1 = rng_oracle.normals(4321, q >> 1, 9)
    z, r = np.where(q & 1, z1, z0), np.where(q & 1, r1, r0)
    py, ps = np.tile(mean.reshape(-1), S), np.tile(np.sqrt(var.reshape(-1)), S)
    want = py + ps * z
    err = np.abs(samp.reshape(-1) - want)
    assert np.all(err <= ps * r + 4 * np.spacing(np.abs(want).astype(np.float32)))
