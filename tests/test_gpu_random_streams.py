"""The device random streams and the NSGA-II init and mating kernels against oracle/rng_oracle.py: an exact restatement
of Philox4x32-10 (pinned by known answers, tests/test_rng_oracle.py), of the uniform conversion and of every consumer's
counter layout, fp64 Box-Muller, and fp64 SBX / polynomial mutation with a running error bound.

Exposures with no tolerance:
  * hb_general_acq_epilogue with mu = 0, var = 1, noise_sd = 1, kappa = c_kappa = 0 and xi = NULL writes Fo = z exactly
    (py = 0 + 1 z, ps = 1, Fo = py - 0 ps), so its output is the Philox + Box-Muller stream of (seed, counter) itself;
  * hb_nsga2_init with lb = 0, ub = 1 on Real columns writes u itself (0 + 1 u, either contracted or not).
hb_mace_epilogue and hb_sample_y_batch are then tied bit for bit to the first one through their xi / z inputs; the fused
posterior is tied to hb_mace_epilogue by test_gpu_posterior_mace.py::test_mace_tail_equals_the_epilogue_and_row_ranges.

Blocks shared across entry points: under one seed, the MACE epilogue's rows [128 c, 128 c + 128) and hb_sample_y_batch's
counter c use the same Philox blocks (both are stream 0, row (c << 7) + t).  No caller passes the same seed to both.

The u = 1 edge: a word >= 0xFFFFFF80 converts to u = 1.0f exactly (probability 2^-25).  The seeds below were found by a
search with the host restatement (rng_oracle.find_seeds-style scans over seeds); each test asserts on the host that its
seed really reaches the edge, then that the kernel gives what the restatement says."""
import json

import numpy as np
import pytest
import torch

from hebo_b200 import _lib
from oracle import rng_oracle as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
NAN = float("nan")

# ---- seeds that reach the edges (host-checked in each test)
SEED_Z0 = (120, 5, 300784)          # (seed, counter, row): u0 = 1 in general-acq pair `row` -> z0 = z1 = 0
SEED_BIGZ = (38, 541125)            # (seed, row): word 0 < 2^10 in MACE row `row` (stream 0), z2 > 3.5
SEED_PARENT = (21385, 1, 360)       # (seed, gen, t) at P = 1000: parent word 0 -> u = 1 -> pa = P - 1
SEED_CAT = (1273, 710, 3)           # (seed, p, column) at P = 1000, D = 8: init word -> u = 1 -> category ub
SEED_SBX = (119282, 1, 853)         # (seed, gen, column) at P = 2, D = 1000: uu = 1 with alpha = 2 -> child on a bound


def _report(**kw):
    print(json.dumps(kw))


def _f(a, dtype=torch.float32):
    return torch.as_tensor(np.asarray(a), dtype=dtype).to(DEV).contiguous()


# ---------------------------------------------------------------------------------------------------------------- draws
def acq_draws(m, K, seed, counter):
    """Fo [m, K] of hb_general_acq_epilogue at mu = 0, var = 1, noise_sd = 1, kappa = 0: the draws z themselves."""
    lib = _lib.lib()
    mu, var = torch.zeros(K, m, device=DEV), torch.ones(K, m, device=DEV)
    sd = torch.ones(K, device=DEV)
    Fo = torch.empty(m, K, device=DEV)
    _lib.check(lib.hb_general_acq_epilogue(_lib.ptr(mu), _lib.ptr(var), m, K, 0, 0.0, 0.0, _lib.ptr(sd), None, int(seed),
                                           int(counter), _lib.ptr(Fo), None, None, _lib.stream_ptr()), "general_acq")
    torch.cuda.synchronize()
    return Fo


def ref_flat(n, seed, counter):
    """(z, r): the restated draws of general-acq elements q = 0 .. n-1 (pair q >> 1, half q & 1) and their bounds."""
    pairs = np.arange((n + 1) // 2, dtype=np.uint64)
    z0, z1, r0, r1 = R.normals(seed, pairs, counter)
    z = np.stack([z0, z1], 1).reshape(-1)[:n]
    r = np.stack([r0, r1], 1).reshape(-1)[:n]
    return z, r


@pytest.mark.parametrize("m,K,seed,counter", [(1 << 19, 2, 7, 3), (1 << 18, 3, 7, 4), (4097, 5, 2 ** 40 + 3, 2 ** 33 + 1),
                                              (1, 1, 0, 0), (3, 1, 11, 0)])
def test_general_acq_draws_are_the_restated_box_muller(m, K, seed, counter):
    """Each z within the Box-Muller error bound of the fp64 value at the restated uniforms; pairs, halves and `counter`
    as the layout says (q = r K + b, pair q >> 1, half q & 1, stream = counter)."""
    Fo = acq_draws(m, K, seed, counter).cpu().double().numpy().reshape(-1)
    z, r = ref_flat(m * K, seed, counter)
    err = np.abs(Fo - z)
    zero = r == 0
    assert np.array_equal(Fo[zero], z[zero])
    c = float((err[~zero] / r[~zero]).max()) if (~zero).any() else 0.0
    worst = int(np.argmax(np.where(zero, 0, err / np.where(zero, 1, r))))
    _report(case="general_acq_draws", m=m, K=K, seed=seed, counter=counter, c_needed=c, worst_q=worst,
            worst_z=float(z[worst]), worst_err=float(err[worst]))
    assert c <= 1.0, c
    # a different counter or seed is a different, restated stream
    other = acq_draws(m, K, seed, counter + 1).cpu().double().numpy().reshape(-1)
    z2, r2 = ref_flat(m * K, seed, counter + 1)
    assert np.all(np.abs(other - z2) <= r2) and (m * K < 4 or not np.array_equal(other, Fo))
    other = acq_draws(m, K, seed + 1, counter).cpu().double().numpy().reshape(-1)
    z3, r3 = ref_flat(m * K, seed + 1, counter)
    assert np.all(np.abs(other - z3) <= r3) and (m * K < 4 or not np.array_equal(other, Fo))


def test_u0_equal_to_one_gives_zero_draws():
    seed, counter, row = SEED_Z0
    w0, _ = R.normal_words(seed, np.array([row], dtype=np.uint64), counter)
    assert int(w0[0]) >= R.U1_WORD and R.uniform(w0)[0] == np.float32(1.0)
    K = 2
    Fo = acq_draws(row + 1, K, seed, counter).cpu()
    assert float(Fo[row, 0]) == 0.0 and float(Fo[row, 1]) == 0.0       # logf(1) = 0: z0 = z1 = 0 exactly
    z, r = ref_flat((row + 1) * K, seed, counter)
    assert z[2 * row] == 0.0 and z[2 * row + 1] == 0.0


def test_mace_epilogue_draws_equal_the_general_acq_rows():
    """hb_mace_epilogue(xi = NULL, seed) equals hb_mace_epilogue(xi1, xi2) bit for bit, with (xi1, xi2) the general-acq
    draws of elements 2r, 2r + 1 at counter 0, i.e. philox_normal2(seed, r).  Row SEED_BIGZ[1] has the largest |z| class
    (word < 2^10) and lands on -logPI's asymptotic branch."""
    lib = _lib.lib()
    seed, big = SEED_BIGZ
    m = 1 << 20
    w0, w1 = R.normal_words(seed, np.array([big], dtype=np.uint64))
    assert int(w0[0]) < 1024
    zb = R.box_muller(R.uniform(w0), R.uniform(w1))
    assert zb[1][0] > 3.5
    Fo = acq_draws(m, 2, seed, 0)
    xi1, xi2 = Fo[:, 0].contiguous(), Fo[:, 1].contiguous()
    mu, var = torch.full((m,), 3.0, device=DEV), torch.ones(m, device=DEV)
    noise_var, tau, kappa, eps = 0.5, 0.0, 1.0, 0.0
    F0, F1 = torch.empty(m, 3, device=DEV), torch.empty(m, 3, device=DEV)
    _lib.check(lib.hb_mace_epilogue(_lib.ptr(mu), _lib.ptr(var), m, noise_var, tau, kappa, eps, None, None, seed, _lib.ptr(F0),
                                    _lib.stream_ptr()), "mace")
    _lib.check(lib.hb_mace_epilogue(_lib.ptr(mu), _lib.ptr(var), m, noise_var, tau, kappa, eps, _lib.ptr(xi1), _lib.ptr(xi2), 0,
                                    _lib.ptr(F1), _lib.stream_ptr()), "mace")
    torch.cuda.synchronize()
    assert torch.equal(F0.view(torch.int32), F1.view(torch.int32))
    # the big-z row: zz = (tau - eps - py - noise z2) / ps < -6, the asymptotic branch
    zz = -3.0 - np.sqrt(2.0) * np.sqrt(noise_var) * float(xi2[big])
    assert zz < -6.0 and bool(torch.isfinite(F0[big]).all())
    _report(case="mace_epilogue", rows=m, big_row=big, z2=float(xi2[big]), zz=zz, logPI_col=float(F0[big, 2]))


@pytest.mark.parametrize("m", [1, 7, 256])
@pytest.mark.parametrize("counter", [0, 3])
def test_sample_y_batch_draws_equal_the_general_acq_rows(m, counter):
    """hb_sample_y_batch(z = NULL, seed, counter) equals the same call given z = general-acq elements
    [256 counter, 256 counter + m) at stream 0, bit for bit."""
    from tests.util import fit_model
    gp, X, Xe, y = fit_model("rng_streams", 48, 3, seed=3, epochs=5)
    g = torch.Generator().manual_seed(m + counter)
    Xs = (torch.rand(m, 3, generator=g) * 2 - 1).to(DEV)
    seed = 9
    flat = acq_draws(128 * (counter + 1), 2, seed, 0).reshape(-1)
    z = flat[256 * counter: 256 * counter + m].contiguous()
    f_null = gp.sample_y_batch(Xs, None, seed, counter)
    f_z = gp.sample_y_batch(Xs, None, seed, counter, z=z)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(f_null).all())
    assert torch.equal(f_null.view(torch.int32), f_z.view(torch.int32))


# ---------------------------------------------------------------------------------------------------------------- init
def run_init(P, D, d, kind, lb, ub, fixed, init, seed):
    lib = _lib.lib()
    X = torch.full((P, D), NAN, device=DEV)
    Xc = torch.full((P, max(d, 1)), NAN, device=DEV)
    Xe = torch.full((P, max(D - d, 1)), -7, dtype=torch.int32, device=DEV)
    k, l, u, fx = _f(kind, torch.int32), _f(lb), _f(ub), _f(fixed)
    it = None if init is None else _f(init)
    n_init = 0 if init is None else init.shape[0]
    _lib.check(lib.hb_nsga2_init(_lib.ptr(X), P, D, d, _lib.ptr(k), _lib.ptr(l), _lib.ptr(u), _lib.ptr(fx), _lib.ptr(it), n_init,
                                 int(seed), _lib.ptr(Xc) if d else None, _lib.ptr(Xe) if D > d else None, _lib.stream_ptr()), "init")
    torch.cuda.synchronize()
    X = X.cpu().numpy()
    if d:
        assert np.array_equal(Xc.cpu().numpy()[:, :d], X[:, :d])
    if D > d:
        assert np.array_equal(Xe.cpu().numpy()[:, :D - d], np.rint(X[:, d:]).astype(np.int32))
    return X


@pytest.mark.parametrize("P,D", [(1, 1), (2, 2), (3, 3), (16384, 5), (1, 4097), (33, 4099), (100, 6), (257, 7)])
def test_init_writes_the_restated_uniforms(P, D):
    """lb = 0, ub = 1, Real columns: X is u itself, bit for bit (philox4 and the conversion)."""
    seed = 1234567 + P + D
    X = run_init(P, D, D, np.zeros(D, np.int32), np.zeros(D), np.ones(D), np.full(D, NAN), None, seed)
    A, B = R.init_reference(P, D, np.zeros(D, np.int32), np.zeros(D), np.ones(D), np.full(D, NAN), None, seed)
    assert np.array_equal(A, B)
    assert np.array_equal(X.view(np.uint32), A.view(np.uint32))


def _box():
    """kinds, lb, ub, fixed of a mixed space: negative and asymmetric boxes, lb == ub, an Integer range of width 1, a
    fixed column, a wide Choice"""
    kind = np.array([0, 0, 0, 0, 1, 1, 1, 0, 2, 2, 2, 1], np.int32)
    lb = np.array([-1.0, -7.5, -1e3, 2.0, -3.0, 2.0, 0.0, 0.0, 0.0, 0.0, 0.0, 4.0], np.float32)
    ub = np.array([1.0, 0.25, 1e-2, 2.0, 9.0, 3.0, 1e6, 1.0, 4.0, 1.0, 999.0, 4.0], np.float32)
    fixed = np.full(12, NAN, np.float32)
    fixed[7] = 0.625
    return kind, lb, ub, fixed, 8


@pytest.mark.parametrize("P,seed", [(1, 5), (300, 6), (4099, 7)])
def test_init_general_bounds_types_initial_rows_and_fixed_columns(P, seed):
    kind, lb, ub, fixed, d = _box()
    D = kind.size
    init = np.array([[5.0, -9.0, 0.3, 1.0, 2.6, 2.5, -1.0, 0.1, 3.0, 7.0, 12.4, 4.0],
                     [-0.5, 0.0, -1e3, 2.0, 9.0, 3.0, 1e6, 0.9, 0.0, 0.0, 999.0, 4.0]], np.float32)[:P]
    X = run_init(P, D, d, kind, lb, ub, fixed, init, seed)
    A, B = R.init_reference(P, D, kind, lb, ub, fixed, init, seed)
    ok = (X == A) | (X == B)
    assert ok.all(), np.argwhere(~ok)[:5]
    # initial rows are prepended and repaired; the fixed column overrides them too
    assert X[0, 0] == 1.0 and X[0, 1] == -7.5 and X[0, 4] == 3.0 and X[0, 5] == 2.0 and X[0, 7] == 0.625 and X[0, 9] == 1.0
    assert (X[:, 7] == 0.625).all() and (X[:, 3] == 2.0).all() and (X[:, 11] == 4.0).all()
    _report(case="init_general", P=P, fused_differs=int((A != B).sum()), matched_plain=int((X == A).sum()),
            matched_fused=int((X == B).sum()))


def test_init_u_equal_to_one_gives_the_top_category():
    seed, p, col = SEED_CAT
    P, D = 1000, 8
    w = R.block(seed, p, R.MASK, col - col % 4, 1)[col % 4]
    assert int(w) >= R.U1_WORD
    kind = np.array([0, 1, 2, 2, 0, 1, 2, 0], np.int32)
    lb = np.array([0, 0, 0, 0, -1, -2, 1, 3], np.float32)
    ub = np.array([1, 5, 2, 4, 1, 2, 6, 4], np.float32)
    X = run_init(P, D, 2, kind, lb, ub, np.full(D, NAN), None, seed)
    A, B = R.init_reference(P, D, kind, lb, ub, np.full(D, NAN), None, seed)
    assert ((X == A) | (X == B)).all()
    assert X[p, col] == 4.0          # floorf(0 + 5 * 1) = 5 = ub + 1, repaired to ub


# ---------------------------------------------------------------------------------------------------------------- mating
def run_mate(X, d, kind, lb, ub, fixed, seed, gen):
    lib = _lib.lib()
    P, D = X.shape
    Xd = _f(X)
    C = torch.full((P, D), NAN, device=DEV)
    Cc = torch.full((P, max(d, 1)), NAN, device=DEV)
    Ce = torch.full((P, max(D - d, 1)), -7, dtype=torch.int32, device=DEV)
    k, l, u, fx = _f(kind, torch.int32), _f(lb), _f(ub), _f(fixed)
    _lib.check(lib.hb_nsga2_mate(_lib.ptr(Xd), P, D, d, _lib.ptr(k), _lib.ptr(l), _lib.ptr(u), _lib.ptr(fx), int(seed), int(gen),
                                 _lib.ptr(C), _lib.ptr(Cc) if d else None, _lib.ptr(Ce) if D > d else None, _lib.stream_ptr()), "mate")
    torch.cuda.synchronize()
    C = C.cpu().numpy()
    if d:
        assert np.array_equal(Cc.cpu().numpy()[:, :d], C[:, :d])
    if D > d:
        assert np.array_equal(Ce.cpu().numpy()[:, :D - d], np.rint(C[:, d:]).astype(np.int32))
    return C


def population(P, kind, lb, ub, seed):
    """P distinct, identifiable rows in the box: Real values spread over the box (with rows on a bound), Integer and
    Choice values drawn uniformly; rows 1 and 2 equal row 0 (equal parents) when P > 8."""
    rng = np.random.default_rng(seed)
    D = kind.size
    X = (lb + (ub - lb) * rng.random((P, D))).astype(np.float32)
    X = np.where(kind != 0, np.floor(lb + (ub - lb + 1) * rng.random((P, D))), X)
    X = np.minimum(np.maximum(X, lb), ub).astype(np.float32)
    if P > 8:
        X[3] = lb
        X[4] = ub
        X[1] = X[0]
        X[2] = X[0]
    return X


def check_mate(X, d, kind, lb, ub, fixed, seed, gen, what):
    C = run_mate(X, d, kind, lb, ub, fixed, seed, gen)
    ref = R.mate_reference(X, kind, lb, ub, fixed, seed, gen)
    C64 = C.astype(np.float64)
    ok = (C64 >= ref["lo"]) & (C64 <= ref["hi"])
    bad = np.argwhere(~ok)
    assert ok.all(), (what, bad[:5].tolist(), [(C64[i, j], ref["lo"][i, j], ref["hi"][i, j], ref["mid"][i, j], ref["rad"][i, j])
                                               for i, j in bad[:5]])
    real = (kind == 0)[None, :] & (ref["rad"] > 0) & ~ref["straddle"] & np.isnan(fixed)[None, :]
    ratio = np.where(real, np.abs(C64 - ref["mid"]) / np.where(real, ref["rad"], 1.0), 0.0)
    _report(case=what, P=X.shape[0], D=X.shape[1], seed=seed, gen=gen, c_needed=float(ratio.max()) if ratio.size else 0.0,
            bounded=int(real.sum()), straddled=int(ref["straddle"].sum()), sbx=int(ref["sbx"].sum()),
            pm=int(ref["pm1"].sum() + ref["pm2"].sum()), exact=int((ref["lo"] == ref["hi"]).sum()))
    return C, ref


MATE_CASES = [(1, 5, 3, [1]), (7, 1, 12, [1, 4]), (2, 12, 4, [1, 2]), (3, 12, 5, [1]), (100, 12, 6, [1, 2, 7]), (101, 12, 8, [1]),
              (16384, 12, 9, [1]), (5, 300, 10, [1]), (4, 4096, 11, [3])]


@pytest.mark.parametrize("P,D,seed,gens", MATE_CASES)
def test_mate_equals_the_fp64_operators(P, D, seed, gens):
    """Parents, pairing, swaps, mutation decisions and Choice columns exact; Real / Integer columns within the running
    bound of the fp64 SBX / PM (either side where the interval straddles a clamp or a rint half-integer)."""
    kind0, lb0, ub0, fixed0, _ = _box()
    reps = -(-D // kind0.size)
    kind, lb, ub, fixed = (np.tile(a, reps)[:D] for a in (kind0, lb0, ub0, fixed0))
    order = np.argsort(kind == 2, kind="stable")            # numeric columns first, then the categorical ones
    kind, lb, ub, fixed = kind[order], lb[order], ub[order], fixed[order]
    d = int((kind != 2).sum())
    X = population(P, kind, lb, ub, seed)
    for gen in gens:
        check_mate(X, d, kind, lb, ub, fixed, seed, gen, f"mate P{P} D{D}")
    if len(gens) > 1:
        a = run_mate(X, d, kind, lb, ub, fixed, seed, gens[0])
        b = run_mate(X, d, kind, lb, ub, fixed, seed + 1, gens[0])
        assert not np.array_equal(a, b) or P * D < 4


def test_mate_u_equal_to_one_gives_parent_p_minus_1():
    seed, gen, t = SEED_PARENT
    P = 1000
    w = R.block(seed, t, gen, 0xFFFFFFF0, 2)[0]
    assert int(w) >= R.U1_WORD
    D = 40                                           # pm_prob = 1 / 40: most Choice columns keep a parent's value
    kind = np.array([0, 1] + [2] * (D - 2), np.int32)
    lb, ub = np.zeros(D, np.float32), np.array([1, 50] + [1e6] * (D - 2), np.float32)
    X = population(P, kind, lb, ub, 17)
    X[:, 2:] = np.arange(P)[:, None]                 # identifiable rows
    C, ref = check_mate(X, 2, kind, lb, ub, np.full(D, NAN, np.float32), seed, gen, "mate_parent_edge")
    assert ref["pa"][t] == P - 1
    for row, mut in ((2 * t, ref["mut1"][t]), (2 * t + 1, ref["mut2"][t])):
        for k in range(2, D):
            if not mut[k]:
                assert C[row, k] in (float(P - 1), float(ref["pb"][t]))
    assert (C[2 * t:2 * t + 2, 2:] == P - 1).any()


def test_mate_singular_sbx_clamps_the_child_to_its_bound():
    """uu = 1 with alpha = fl(2 - beta^-16) = 2: 2 - uu alpha = 0 -> 1 / 1e-30 -> beta_q ~ 75, both children leave the box
    and are clamped to lb and ub."""
    seed, gen, col = SEED_SBX
    P, D = 2, 1000
    v = R.block(seed, 0, gen, col, 3)
    assert int(v[1]) >= R.U1_WORD and R.uniform(v[0]) < np.float32(0.5)
    kind, lb, ub = np.zeros(D, np.int32), np.zeros(D, np.float32), np.ones(D, np.float32)
    X = np.stack([np.full(D, 0.45, np.float32), np.full(D, 0.55, np.float32)])
    C, ref = check_mate(X, D, kind, lb, ub, np.full(D, NAN, np.float32), seed, gen, "mate_sbx_edge")
    assert ref["do_pair"][0] and ref["pa"][0] != ref["pb"][0] and ref["sbx"][0, col]
    assert not ref["pm1"][0, col] and not ref["pm2"][0, col]
    assert sorted([C[0, col], C[1, col]]) == [0.0, 1.0]
