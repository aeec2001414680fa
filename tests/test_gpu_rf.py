"""hb_rf_fit / hb_rf_predict / hb_rf_load and hebo_b200.RF on the device:
  - the reference's own sklearn trees loaded with hb_rf_load score held-out rows bit for bit like RF.predict;
  - the device fit from the reference's bootstrap counts splits every tree's in-bag rows into the reference's leaves;
  - the device forest equals the fp64 oracle (oracle/rf_oracle.py) bit for bit, node for node, with est_noise, on every
    fixture variant and at the envelope's corners;
  - the Philox bootstrap equals its restatement, a fit is bit-identical run to run, and B outputs in one launch equal B
    single fits;
  - draws and NaN rows; the reference's test_acq.py cases over hebo_b200.RF, and the device scorers against acq.eval."""
import ctypes as C

import numpy as np
import pytest
import torch

from hebo_b200 import RF, MOMeanSigmaLCB, _lib
from hebo_b200.acq import LCB, MACE, GeneralAcq, Mean, NoisyAcq, Sigma, ga_score, general_score
from hebo_b200.forest import forest_trees
from oracle import rf_oracle as R
from oracle import rng_oracle
from tests.test_oracle_rf import VARIANTS, partition, same_partitions, variant

pytestmark = pytest.mark.gpu
DEV = "cuda"


def model_of(g, T=None):
    uniqs = g["uniqs"]
    conf = dict(n_estimators=int(g["T"]) if T is None else T)
    if uniqs:
        conf["num_uniqs"] = uniqs
    return RF(g["Xc"].shape[1], len(uniqs), 1, **conf)


def inputs(g, test=False):
    s = "_test" if test else ""
    Xc = torch.from_numpy(g["Xc" + s]) if g["Xc"].shape[1] else None
    Xe = torch.from_numpy(g["Xe" + s]) if g["uniqs"] else None
    return Xc, Xe


def rd32(th):
    f = np.float32(th)
    return np.nextafter(f, np.float32(-np.inf)) if float(f) > th else f


def assert_same_forest(dev_trees, ref_trees):
    assert len(dev_trees) == len(ref_trees)
    for t, (a, b) in enumerate(zip(dev_trees, ref_trees)):
        for k in ("feature", "left", "right"):
            assert np.array_equal(a[k], b[k]), (t, k)
        for k in ("threshold", "value"):
            assert a[k].tobytes() == b[k].tobytes(), (t, k)
        inner = a["feature"] >= 0
        assert all(a["thr32"][i] == rd32(a["threshold"][i]) for i in np.nonzero(inner)[0])


@pytest.mark.parametrize("name", VARIANTS)
def test_load_predict_is_the_reference(name):
    g = variant(name)
    m = model_of(g)
    m.load_trees(g["trees"], float(g["noise"][0]))
    mean, var = m.predict(*inputs(g, test=True))
    assert mean.numpy().tobytes() == g["mean"].astype(np.float32).tobytes()
    assert var.numpy().tobytes() == g["var"].astype(np.float32).tobytes()


@pytest.mark.parametrize("name", VARIANTS)
def test_fit_matches_reference_partitions_and_oracle(name):
    g = variant(name)
    m = model_of(g)
    Xc, Xe = inputs(g)
    y = g["y"].reshape(-1)
    m.fit(Xc, Xe, torch.from_numpy(g["y"]), counts=g["counts"])
    trees = m.trees()
    same_partitions(trees, g["X"], y, g["counts"], g["apply"], g["trees"])
    ref_trees, ref_noise = R.fit(g["X"], y, g["counts"])
    assert_same_forest(trees, ref_trees)
    assert m.noise.numpy().tobytes() == np.float32(ref_noise).tobytes()


def _corner(kind):
    rng = np.random.default_rng(7)
    n, d, T = 40, 3, 4
    if kind == "n1":
        n = 1
    X = rng.standard_normal((n, d)).astype(np.float32)
    y = rng.standard_normal(n).astype(np.float32)
    if kind == "y_equal":
        y[:] = 0.25
    elif kind == "x_constant":
        X[:] = 1.5
    elif kind == "chain":                  # y = 4^i on one feature: every split peels off the largest row
        n, d = 64, 1
        X = np.arange(n, dtype=np.float32)[:, None]
        y = (4.0 ** np.arange(n)).astype(np.float32)
    elif kind == "t1":
        T = 1
    elif kind == "t1024":
        n, d, T = 12, 2, 1024
        X, y = X[:n, :d], y[:n]
    counts = np.stack([np.bincount(rng.integers(0, n, n), minlength=n) for _ in range(T)]).astype(np.int32)
    if kind == "chain":
        counts[:] = 1
    return X, y, counts


@pytest.mark.parametrize("kind", ["n1", "y_equal", "x_constant", "chain", "t1", "t1024"])
def test_fit_equals_oracle_at_corners(kind):
    X, y, counts = _corner(kind)
    T = counts.shape[0]
    m = RF(X.shape[1], 0, 1, n_estimators=T)
    m.fit(torch.from_numpy(X), None, torch.from_numpy(y)[:, None], counts=counts)
    ref_trees, ref_noise = R.fit(X, y, counts)
    assert_same_forest(m.trees(), ref_trees)
    assert m.noise.numpy().tobytes() == np.float32(ref_noise).tobytes()
    if kind == "chain":
        assert len(ref_trees[0]["feature"]) == 2 * X.shape[0] - 1          # depth n - 1


def test_fit_largest_envelope():
    """n = 8192 rows, width 4096 (numeric and one-hot columns): the fit is bit-identical run to run, every in-bag row
    lands in a leaf, and each leaf's value is the weighted mean of its in-bag rows up to fp64 rounding (the Python oracle
    is too slow to grow this tree node for node)."""
    n, dc, uniqs = 8192, 4096 - 96, [32, 64]
    g = torch.Generator().manual_seed(3)
    Xc = torch.rand(n, dc, generator=g)
    Xe = torch.stack([torch.randint(0, u, (n,), generator=g) for u in uniqs], 1)
    y = (Xc[:, :4].sum(1, keepdim=True) + Xe[:, :1].float() * 0.1).sin()
    m = RF(dc, 2, 1, n_estimators=1, num_uniqs=uniqs)
    torch.manual_seed(0)
    m.fit(Xc, Xe, y)
    first = m.trees()
    torch.manual_seed(0)
    m.fit(Xc, Xe, y)
    assert_same_forest(m.trees(), first)
    t = first[0]
    X = R.tree_inputs(Xc.numpy(), Xe.numpy(), uniqs)
    w = R.bootstrap_counts(m.seed, 0, 0, np.arange(n), n)
    rows = np.nonzero(w > 0)[0]
    leaves = R.apply(t, X[rows])
    assert np.all(t["feature"][leaves] < 0)
    yy = y.numpy().reshape(-1).astype(np.float64)[rows]
    ww = w[rows].astype(np.float64)
    ref = np.bincount(leaves, ww * yy, minlength=t["value"].size) / np.maximum(np.bincount(leaves, ww, minlength=t["value"].size), 1)
    np.testing.assert_allclose(t["value"][leaves], ref[leaves], rtol=1e-12, atol=1e-12)


def test_philox_bootstrap_and_determinism():
    g = variant("nan_n50_w3_t20")
    m = model_of(g)
    Xc, Xe = inputs(g)
    torch.manual_seed(11)
    m.fit(Xc, Xe, torch.from_numpy(g["y"]))
    first = m.trees()
    y = g["y"].reshape(-1)
    kept = np.nonzero(np.isfinite(y))[0]
    counts = np.stack([R.bootstrap_counts(m.seed, 0, t, kept, y.size) for t in range(int(g["T"]))])
    ref_trees, ref_noise = R.fit(g["X"], y, counts)
    assert_same_forest(m.trees(), ref_trees)
    assert m.noise.numpy().tobytes() == np.float32(ref_noise).tobytes()
    torch.manual_seed(11)
    m.fit(Xc, Xe, torch.from_numpy(g["y"]))
    assert_same_forest(m.trees(), first)


def _raw_fit(Xc, Y, spec, T, counts, seed):
    lib = _lib.lib()
    n, B = Y.shape
    ws_bytes = int(lib.hb_rf_fit_workspace_bytes(n, C.byref(spec), B, T))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    forest = torch.empty(int(lib.hb_rf_forest_bytes(C.byref(spec), 2 * n - 1, B, T)), dtype=torch.uint8, device=DEV)
    noise = torch.empty(B, dtype=torch.float32, device=DEV)
    cd = None if counts is None else torch.from_numpy(counts).to(DEV).contiguous()
    _lib.check(lib.hb_rf_fit(_lib.ptr(Xc), None, _lib.ptr(Y), n, C.byref(spec), B, T, _lib.ptr(cd), seed, _lib.ptr(forest),
                             _lib.ptr(noise), _lib.ptr(ws), ws_bytes, _lib.stream_ptr()), "hb_rf_fit")
    return forest_trees(forest), noise.cpu()


@pytest.mark.parametrize("given_counts", [True, False])
def test_batched_outputs_equal_single_fits(given_counts):
    rng = np.random.default_rng(2)
    n, d, T, B = 60, 3, 5, 3
    Xc = torch.from_numpy(rng.standard_normal((n, d)).astype(np.float32)).to(DEV)
    Y = rng.standard_normal((n, B)).astype(np.float32)
    Y[3, 0] = np.nan
    Y[10, 1] = np.inf
    Y[[20, 21], 2] = np.nan
    counts = np.stack([np.stack([np.bincount(rng.integers(0, n, n), minlength=n) for _ in range(T)]) for _ in range(B)])
    counts = counts.astype(np.int32)
    spec = _lib.RfSpec(d, 0, None)
    Yd = torch.from_numpy(Y).to(DEV).contiguous()
    trees, noise = _raw_fit(Xc, Yd, spec, T, counts if given_counts else None, 99)
    for b in range(B):
        y = Y[:, b]
        kept = np.nonzero(np.isfinite(y))[0]
        cb = counts[b] if given_counts else np.stack([R.bootstrap_counts(99, b, t, kept, n) for t in range(T)])
        ref_trees, ref_noise = R.fit(Xc.cpu().numpy(), y, cb)
        assert_same_forest(trees[b * T:(b + 1) * T], ref_trees)
        assert noise[b].numpy().tobytes() == np.float32(ref_noise).tobytes()
        if given_counts:
            single, sn = _raw_fit(Xc, Yd[:, b:b + 1].contiguous(), spec, T, counts[b:b + 1].copy(), 99)
            assert_same_forest(single, trees[b * T:(b + 1) * T])
            assert sn[0] == noise[b]


def _fitted_mixed():
    g = variant("mixed_n300_w12_t20")
    m = model_of(g)
    torch.manual_seed(4)
    m.fit(*inputs(g), torch.from_numpy(g["y"]))
    return g, m


def test_draws_and_nan_rows():
    g, m = _fitted_mixed()
    Xc, Xe = inputs(g, test=True)
    xs, xe = Xc.to(DEV), Xe.to(DEV).int()
    mean, var, samp = m._predict_dev(xs, xe, n_samples=3, seed=1234, counter=5)
    py, ps = mean.cpu().numpy().reshape(-1), np.sqrt(var.cpu().numpy().reshape(-1))
    q = np.arange(3 * py.size)
    z0, z1, r0, r1 = rng_oracle.normals(1234, q >> 1, 5)
    z, r = np.where(q & 1, z1, z0), np.where(q & 1, r1, r0)
    want = np.tile(py, 3) + np.tile(ps, 3) * z
    err = np.abs(samp.cpu().numpy().reshape(-1) - want)
    assert np.all(err <= np.tile(ps, 3) * r + 4 * np.spacing(np.abs(want).astype(np.float32)))
    torch.manual_seed(0)
    s1 = m.sample_y(Xc, Xe, n_samples=2)
    torch.manual_seed(0)
    assert torch.equal(s1, m.sample_y(Xc, Xe, n_samples=2)) and s1.shape == (2, Xc.shape[0], 1)
    bad = xe.clone()
    bad[1, 0] = 3
    bad[4, 1] = -1
    mb, vb, _ = m._predict_dev(xs, bad)
    rows = torch.isnan(mb.reshape(-1)) & torch.isnan(vb.reshape(-1))
    assert rows.cpu().tolist() == [i in (1, 4) for i in range(xs.shape[0])]
    assert torch.equal(mb[~rows], mean[~rows])


def test_reference_acq_cases():
    """HEBO/test/test_acq.py over hebo_b200.RF: X ~ N(0, 1) [10, 1], y = X."""
    torch.manual_seed(0)
    X = torch.randn(10, 1)
    model = RF(1, 0, 1)
    model.fit(X, None, X)
    for cls in (Mean, Sigma, LCB):
        acq = cls(model, best_y=0.)
        v = acq(X, None)
        assert acq.num_obj == 1 and acq.num_constr == 0 and v.shape[1] == 1
    for acq, shape in ((MOMeanSigmaLCB(model, best_y=0.), (2, 1)), (MACE(model, best_y=0.), (3, 0)),
                       (GeneralAcq(model, 1, 0), (1, 0)), (NoisyAcq(model, 1, 0), (1, 0))):
        v = acq(X, None)
        assert torch.isfinite(v).all() and (acq.num_obj, acq.num_constr) == shape


def test_device_scorers_agree_with_eval():
    g, m = _fitted_mixed()
    Xc, Xe = inputs(g, test=True)
    xs, xe = Xc.to(DEV), Xe.to(DEV).int()
    for cls in (Mean, Sigma, LCB):
        acq = cls(m, best_y=0.)
        f = ga_score(acq)(xs, xe, 0)
        np.testing.assert_allclose(f.cpu().numpy(), acq(Xc, Xe)[:, 0].numpy(), rtol=1e-6, atol=1e-7)
    acq = GeneralAcq(m, 1, 0, use_noise=False)
    Fo = general_score(acq, seed=3)(xs, xe, 0)
    np.testing.assert_array_equal(Fo.cpu().numpy(), acq(Xc, Xe).cpu().numpy())
    acq = MOMeanSigmaLCB(m, best_y=0.)
    Fo, cv = general_score(acq, seed=3)(xs, xe, 0)
    host = acq(Xc, Xe)
    np.testing.assert_array_equal(Fo[:, 1].cpu().numpy(), host[:, 1].numpy())
    assert Fo.shape == (xs.shape[0], 2) and cv.shape == (xs.shape[0],)
    acq = NoisyAcq(m, 1, 0)
    f0, f1 = ga_score(acq, seed=7)(xs, xe, 0), ga_score(acq, seed=7)(xs, xe, 1)
    _, _, samp = m._predict_dev(xs, xe, n_samples=1, seed=7, counter=1)
    assert torch.equal(f1, samp.reshape(-1)) and not torch.equal(f0, f1)
    acq = MACE(m, best_y=float(np.nanmin(g["y"])))
    torch.manual_seed(5)
    a = acq.eval(Xc, Xe)
    torch.manual_seed(5)
    b = acq._eval_any_model(Xc, Xe, float(acq.tau))
    assert torch.equal(a, b)
