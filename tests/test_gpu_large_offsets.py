"""Candidate-side kernels at batch offsets past 2^31 elements, and the Pareto filter and front exchange at the sizes the
sharded scoring runs them with.

Every scoring entry point computes a candidate's row from that row alone, so a window of rows scored inside one large
call must equal, bit for bit, the same rows scored in a small call on a fresh contiguous copy.  The windows are the first
rows whose element offset passes 2^31 and whose byte offset passes 2^32 in every array of the call that is large enough,
the last rows (the last full tile and the partial one) and a few random rows.  Inputs are random on the device so that
every row differs; for each window row past a boundary the test also checks that its output differs from that of the row
its offset folded mod 2^31 reads (a 31-bit mask of the index: an in-bounds stand-in for a truncated int32 offset, which
would point outside the buffer), so a row read from the wrong place cannot pass.

The Pareto filter at 2^28 rows of 8 objectives has a planted answer: filler rows on a totally ordered diagonal and a few
mutually non-dominated rows below zero at offsets past 2^31 elements.  The smaller Pareto and merge cases are checked
against an exact dominance count.

Each case frees its tensors before the next, prints its time and peak device memory, and is skipped, naming the GiB it
needs, only when the shared device lacks that memory."""
import time

import numpy as np
import pytest
import torch

import hebo_b200
from hebo_b200 import _lib
from hebo_b200.pareto import front_merge, front_pack, front_read, pareto_front, pareto_front_device
from tests.test_dist import merge_fn_torch
from tests.test_gpu_nsga_large import _count_dominators
from tests.util import seeded_problem

pytestmark = pytest.mark.gpu

GiB = 1 << 30
E31 = 1 << 31            # elements
B32 = 1 << 32            # bytes


@pytest.fixture
def case(request):
    """Frees the cache, checks free memory (case.need(gib)), and prints the case's time and peak memory at the end."""
    import gc
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()

    class Case:
        def need(self, gib):
            free, _ = torch.cuda.mem_get_info()
            if free < (gib + 2) * GiB:
                pytest.skip(f"needs {gib} GiB of device memory (+2 GiB margin), {free / GiB:.1f} GiB free")
    c = Case()
    t0 = time.perf_counter()
    yield c
    torch.cuda.synchronize()
    print(f"\n[{request.node.name}] {time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / GiB:.2f} GiB")
    gc.collect()
    torch.cuda.empty_cache()


def _first_row_past(limit_elems, width):
    """First row whose elements reach offset `limit_elems` in a row-major array of `width` elements per row (the row that
    straddles the boundary when it is not row-aligned)."""
    return limit_elems // width


def windows(m, widths, tile=128, seed=0, extra=()):
    """Rows to rescore: around the 2^31-element and 2^32-byte offsets of each fp32 / int32 array width, the last full tile,
    the partial last tile, a few random rows.  Returns (sorted unique rows as an int64 device tensor, rows past 2^31)."""
    rows, past = set(), set()
    for w in widths:
        for lim in (E31, B32 // 4):
            if m * w > lim:
                r = _first_row_past(lim, w)
                rows.update(x for x in range(r - 2, r + 3) if 0 <= x < m)
                if lim == E31:
                    past.update(x for x in range(r + 1, r + 3) if x < m)
    full_end = (m // tile) * tile
    rows.update(range(max(0, full_end - tile), m))
    rows.update(int(x) for x in np.random.RandomState(seed).randint(0, m, 4))
    rows.update(extra)
    return torch.tensor(sorted(rows), dtype=torch.int64, device="cuda"), sorted(past)


def wrap_row(r, width, fold=E31):
    """The row an element offset of row r folded mod `fold` reads: mod 2^31 is what a 31-bit mask of the index reads.  A
    truncated int32 offset itself would be r * width - 2^32, a negative address outside the buffer; the folded row is the
    in-bounds proxy for it, so the check below shows that any wrong row would be noticed, not that a fault would be."""
    return ((r * width) % fold) // width


def assert_rows_equal(big, small, rows, what):
    got = big[rows]
    same = (got == small) | (torch.isnan(got) & torch.isnan(small))
    if not bool(same.all()):
        bad = rows[~same.reshape(same.shape[0], -1).all(1)]
        raise AssertionError(f"{what}: rows {bad[:8].tolist()} of the large call differ from the small call")


def assert_sensitive(out, past, width, what, fold=E31):
    """The output of each row past the boundary differs from the output of the row its offset folded mod `fold` reads."""
    assert past, what
    for r in past:
        w = wrap_row(r, width, fold)
        assert w != r and not torch.equal(out[r], out[w]), (what, r, w)


def _rand(shape, gen, lo=-1.0, hi=1.0):
    x = torch.empty(shape, dtype=torch.float32, device="cuda")
    x.uniform_(lo, hi, generator=gen)
    return x


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ======================================================================== GP posterior: hb_posterior_mace_ex, _grad_ex
@pytest.fixture(scope="module")
def gp1024():
    n, d = 96, 1024
    X, y = seeded_problem(n, d, 31)
    np.random.seed(0)
    torch.manual_seed(0)
    gp = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=3, noise_lb=8e-4, pred_likeli=False, langevin=False)
    gp.fit(X, None, y)
    return gp, X.cuda()


def _near_training_rows(X, m, seed):
    """Candidates [m, d] at random training rows plus a small random step: in 1024 dimensions a uniform candidate is far
    from every training row and its posterior is the prior's, the same for every row."""
    g = _gen(seed)
    Xs = X[torch.randint(0, X.shape[0], (m,), generator=g, device="cuda")]
    for r0 in range(0, m, 1 << 18):           # the step in slices: no second [m, d] buffer
        Xs[r0:r0 + (1 << 18)].add_(_rand(Xs[r0:r0 + (1 << 18)].shape, g, -0.05, 0.05))
    return Xs


@pytest.mark.parametrize("tensor_cores", [True, False])
def test_posterior_mace_rows_past_2_31_elements(gp1024, case, tensor_cores):
    """hb_posterior_mace_ex over Xs [2^21 + 131, 1024] (2^31 + 134 144 elements): F, mu and var of every window row equal a
    small call on a copy of those rows (the MACE draws xi1 / xi2 travel with their rows)."""
    (gp, X), d = gp1024, 1024
    m = (1 << 21) + 131
    case.need(9)
    gp.tensor_cores = tensor_cores
    try:
        g = _gen(1)
        Xs = _near_training_rows(X, m, 1)
        xi1, xi2 = torch.randn(m, generator=g, device="cuda"), torch.randn(m, generator=g, device="cuda")
        tau, kappa = -0.5, 2.0
        F, mu, var = gp.predict_mace(Xs, tau, kappa, 1e-4, xi1, xi2, return_mu_var=True)
        rows, past = windows(m, [d])
        Fs, mus, vars_ = gp.predict_mace(Xs[rows].contiguous(), tau, kappa, 1e-4, xi1[rows], xi2[rows], return_mu_var=True)
        for big, small, what in ((F, Fs, "F"), (mu, mus, "mu"), (var, vars_, "var")):
            assert_rows_equal(big, small, rows, what)
        assert_sensitive(mu, past, d, "mu")
        assert_sensitive(F, past, d, "F")
        assert bool(torch.isfinite(F).all())
        del Xs, xi1, xi2, F, mu, var
    finally:
        gp.tensor_cores = True


def test_posterior_grad_rows_past_2_31_elements(gp1024, case):
    """hb_posterior_grad_ex over Xs, dmu, dvar [2^21 + 131, 1024]: mu, var and both gradient rows of every window equal a
    small call, so the 64-bit row offsets of the loads and of the dmu / dvar stores are locked in."""
    (gp, X), d = gp1024, 1024
    m = (1 << 21) + 131
    case.need(25)
    gp._grad_xe = None
    Xs = _near_training_rows(X, m, 2)
    mu, var, dmu, dvar = gp._posterior_grad(Xs, gp._x_mul, gp._x_add)
    rows, past = windows(m, [d])
    mus, vars_, dmus, dvars = gp._posterior_grad(Xs[rows].contiguous(), gp._x_mul, gp._x_add)
    for big, small, what in ((mu, mus, "mu"), (var, vars_, "var"), (dmu, dmus, "dmu"), (dvar, dvars, "dvar")):
        assert_rows_equal(big, small, rows, what)
    assert_sensitive(dmu, past, d, "dmu")
    assert_sensitive(dvar, past, d, "dvar")
    del Xs, mu, var, dmu, dvar


def test_posterior_kstar_panel_past_2_31_elements(case):
    """hb_posterior_mace_ex with n = NP = 4096 and m_chunk = 2^19 + 128: the K* panel of one chunk (m_chunk x NP floats)
    passes 2^31 elements inside the kernels.  Two chunks, the second one partial."""
    lib = _lib.lib()
    n, d = 4096, 4
    mc = (1 << 19) + 128
    m = mc + 131
    need = int(lib.hb_posterior_workspace_bytes(n, d, mc))
    case.need(need / GiB + 1)
    X, y = seeded_problem(n, d, 41)
    np.random.seed(0)
    torch.manual_seed(0)
    gp = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=2, noise_lb=8e-4, pred_likeli=False, langevin=False, m_chunk=mc)
    gp.fit(X, None, y)
    assert int(lib.hb_padded_n(n)) == 4096 and mc * 4096 > E31
    g = _gen(16)
    Xs = _rand((m, d), g, -1.0, 1.0)
    xi1, xi2 = torch.randn(m, generator=g, device="cuda"), torch.randn(m, generator=g, device="cuda")
    F, mu, var = gp.predict_mace(Xs, -0.5, 2.0, 1e-4, xi1, xi2, return_mu_var=True)
    rows, past = windows(mc, [4096], extra=range(m - 140, m))
    Fs, mus, vars_ = gp.predict_mace(Xs[rows].contiguous(), -0.5, 2.0, 1e-4, xi1[rows], xi2[rows], return_mu_var=True)
    for big, small, what in ((F, Fs, "F"), (mu, mus, "mu"), (var, vars_, "var")):
        assert_rows_equal(big, small, rows, what)
    assert_sensitive(mu, past, 4096, "mu")
    assert_sensitive(var, past, 4096, "var")
    del Xs, xi1, xi2, F, mu, var, gp


def test_mixed_posterior_rows_past_2_31_elements(case):
    """hb_posterior_mace_ex of a mixed model over Xs [2^22 + 131, 512] fp32 and Xe_s [2^22 + 131, 512] int32: both the
    numeric and the category loads pass 2^31 elements."""
    m, d, e = (1 << 22) + 131, 512, 512
    case.need(17)
    nu = [3] * e
    X, y = seeded_problem(64, d, 43)
    Xe = torch.from_numpy(np.random.RandomState(43).randint(0, 3, (64, e))).to(torch.int32)
    np.random.seed(0)
    torch.manual_seed(0)
    gp = hebo_b200.GP(d, e, 1, num_uniqs=nu, lr=0.01, num_epochs=2, noise_lb=8e-4, pred_likeli=False, langevin=False)
    gp.fit(X, Xe, y)
    g = _gen(17)
    pick = torch.randint(0, 64, (m,), generator=g, device="cuda")
    Xs = _near_training_rows(X.cuda(), m, 17)
    Xes = Xe.cuda()[pick]
    flip = torch.randint(0, e, (m,), generator=g, device="cuda")        # one category per row moved: every row differs
    Xes[torch.arange(m, device="cuda"), flip] = (Xes[torch.arange(m, device="cuda"), flip] + 1) % 3
    del pick, flip
    xi1, xi2 = torch.randn(m, generator=g, device="cuda"), torch.randn(m, generator=g, device="cuda")
    F, mu, var = gp.predict_mace(Xs, -0.5, 2.0, 1e-4, xi1, xi2, return_mu_var=True, Xe=Xes)
    rows, past = windows(m, [d, e])
    Fs, mus, vars_ = gp.predict_mace(Xs[rows].contiguous(), -0.5, 2.0, 1e-4, xi1[rows], xi2[rows], return_mu_var=True,
                                     Xe=Xes[rows].contiguous())
    for big, small, what in ((F, Fs, "F"), (mu, mus, "mu"), (var, vars_, "var")):
        assert_rows_equal(big, small, rows, what)
    assert_sensitive(mu, past, d, "mu")
    del Xs, Xes, xi1, xi2, F, mu, var, gp


# ======================================================================== epilogues
def test_acq1_epilogue_row_index_past_2_31(case):
    """hb_acq1_epilogue (LCB) at m = 2^31 + 300: the row index itself passes int32."""
    lib = _lib.lib()
    m = E31 + 300
    case.need(25)
    g = _gen(3)
    mu = torch.randn(m, generator=g, device="cuda")
    var = _rand((m,), g, 0.01, 2.0)
    f = torch.empty(m, device="cuda")

    def run(a, b, out):
        _lib.check(lib.hb_acq1_epilogue(_lib.ptr(a), _lib.ptr(b), a.numel(), _lib.HB_ACQ1_LCB, 2.5, 0.0, _lib.ptr(out),
                                        _lib.stream_ptr()), "hb_acq1_epilogue")
    run(mu, var, f)
    rows, past = windows(m, [1])
    fs = torch.empty(rows.numel(), device="cuda")
    run(mu[rows].contiguous(), var[rows].contiguous(), fs)
    assert_rows_equal(f, fs, rows, "f")
    assert_sensitive(f, past, 1, "f")
    del mu, var, f


def test_mace_epilogue_rows_past_2_31_elements(case):
    """hb_mace_epilogue with explicit xi1 / xi2 at m = ceil(2^31 / 3) + 300: F [m, 3] passes 2^31 elements."""
    lib = _lib.lib()
    m = -(-E31 // 3) + 300
    case.need(20)
    g = _gen(4)
    mu = torch.randn(m, generator=g, device="cuda")
    var = _rand((m,), g, 0.01, 2.0)
    xi1, xi2 = torch.randn(m, generator=g, device="cuda"), torch.randn(m, generator=g, device="cuda")
    F = torch.empty(m, 3, device="cuda")

    def run(a, b, x1, x2, out):
        _lib.check(lib.hb_mace_epilogue(_lib.ptr(a), _lib.ptr(b), a.numel(), 1e-3, -0.3, 2.0, 1e-4, _lib.ptr(x1), _lib.ptr(x2),
                                        0, _lib.ptr(out), _lib.stream_ptr()), "hb_mace_epilogue")
    run(mu, var, xi1, xi2, F)
    rows, past = windows(m, [3, 1])
    Fs = torch.empty(rows.numel(), 3, device="cuda")
    run(mu[rows].contiguous(), var[rows].contiguous(), xi1[rows].contiguous(), xi2[rows].contiguous(), Fs)
    assert_rows_equal(F, Fs, rows, "F")
    assert_sensitive(F, past, 3, "F")
    del mu, var, xi1, xi2, F


def test_general_acq_epilogue_past_2_31_elements(case):
    """hb_general_acq_epilogue with K = 16 + 16 outputs over mu / var [32, 2^26 + 300] (output-major: the last output's
    rows pass 2^31 elements) and explicit draws xi [m, 32] (past 2^31 from row 2^26); Fo, Fc and cv of the window rows
    equal a small call on the same rows' mu / var columns and draws."""
    lib = _lib.lib()
    no, nc = 16, 16
    K = no + nc
    m = (1 << 26) + 300
    case.need(34)
    g = _gen(18)
    mu = torch.randn(K, m, generator=g, device="cuda")
    var = _rand((K, m), g, 0.01, 2.0)
    xi = torch.randn(m, K, generator=g, device="cuda")
    noise_sd = _rand((K,), g, 0.05, 0.5)

    def run(a, b, x):
        k = a.shape[1]
        Fo = torch.empty(k, no, device="cuda")
        Fc = torch.empty(k, nc, device="cuda")
        cv = torch.empty(k, device="cuda")
        _lib.check(lib.hb_general_acq_epilogue(_lib.ptr(a), _lib.ptr(b), k, no, nc, 2.0, 1.5, _lib.ptr(noise_sd), _lib.ptr(x),
                                               0, 0, _lib.ptr(Fo), _lib.ptr(Fc), _lib.ptr(cv), _lib.stream_ptr()),
                   "hb_general_acq_epilogue")
        return Fo, Fc, cv
    Fo, Fc, cv = run(mu, var, xi)
    r_mu = E31 - (K - 1) * m                    # first row whose last-output element passes 2^31
    r_mu_b = B32 // 4 - (K // 2 - 1) * m        # first row whose output-15 element passes 2^32 bytes
    rows, past = windows(m, [K], extra=[x for r in (r_mu, max(0, r_mu_b)) for x in range(r - 2, r + 3)])
    Fos, Fcs, cvs = run(mu[:, rows].contiguous(), var[:, rows].contiguous(), xi[rows].contiguous())
    assert_rows_equal(Fo, Fos, rows, "Fo")
    assert_rows_equal(Fc, Fcs, rows, "Fc")
    assert_rows_equal(cv, cvs, rows, "cv")
    assert_sensitive(Fo, past, K, "Fo")
    assert_sensitive(Fc[:, nc - 1], [r_mu + 1, r_mu + 2], 1, "Fc", fold=E31 - (K - 1) * m)
    del mu, var, xi, Fo, Fc, cv


def test_mo_lcb_epilogue_past_2_31_elements(case):
    """hb_mo_lcb_epilogue over F [2^30 + 300, 2] with explicit draws xi [m]."""
    lib = _lib.lib()
    m = (1 << 30) + 300
    case.need(25)
    g = _gen(19)
    mu = torch.randn(m, generator=g, device="cuda")
    var = _rand((m,), g, 0.01, 2.0)
    xi = torch.randn(m, generator=g, device="cuda")

    def run(a, b, x):
        k = a.numel()
        F = torch.empty(k, 2, device="cuda")
        G = torch.empty(k, device="cuda")
        _lib.check(lib.hb_mo_lcb_epilogue(_lib.ptr(a), _lib.ptr(b), k, 0.1, 0.2, 2.0, _lib.ptr(x), 0, 0, _lib.ptr(F),
                                          _lib.ptr(G), _lib.stream_ptr()), "hb_mo_lcb_epilogue")
        return F, G
    F, G = run(mu, var, xi)
    rows, past = windows(m, [2, 1])
    Fs, Gs = run(mu[rows].contiguous(), var[rows].contiguous(), xi[rows].contiguous())
    assert_rows_equal(F, Fs, rows, "F")
    assert_rows_equal(G, Gs, rows, "G")
    assert_sensitive(F, past, 2, "F")
    del mu, var, xi, F, G


# ======================================================================== deep ensemble, random forest, embedding
def test_de_predict_rows_past_2_31_elements(case):
    """hb_de_predict over Xs [2^23 + 131, 256]: the row loads of de_load_inputs pass 2^31 elements."""
    m, d = (1 << 23) + 131, 256
    case.need(9)
    torch.manual_seed(5)
    X, y = seeded_problem(64, d, 5)
    model = hebo_b200.DeepEnsemble(d, 0, 1, num_ensembles=4, num_epochs=3, num_hiddens=32, batch_size=16)
    model.fit(X, None, y)
    Xs = _rand((m, d), _gen(5), -1.2, 1.2)
    mu, var = model._predict_dev(Xs, None)
    rows, past = windows(m, [d])
    mus, vars_ = model._predict_dev(Xs[rows].contiguous(), None)
    assert_rows_equal(mu, mus, rows, "mu")
    assert_rows_equal(var, vars_, rows, "var")
    assert_sensitive(mu, past, d, "mu")
    del Xs, mu, var


def test_rf_predict_rows_past_2_31_elements(case):
    """hb_rf_predict over Xc [2^23 + 131, 256]: mean and variance of the window rows equal a small call."""
    m, d = (1 << 23) + 131, 256
    case.need(9)
    torch.manual_seed(6)
    X, y = seeded_problem(400, d, 6)
    model = hebo_b200.RF(d, 0, 1, n_estimators=16)
    model.fit(X, None, y)
    Xs = _rand((m, d), _gen(6), -1.0, 1.0)
    mean, var, _ = model._predict_dev(Xs, None)
    rows, past = windows(m, [d])
    means, vars_, _ = model._predict_dev(Xs[rows].contiguous(), None)
    assert_rows_equal(mean, means, rows, "mean")
    assert_rows_equal(var, vars_, rows, "var")
    assert_sensitive(mean, past, d, "mean")
    del Xs, mean, var


def test_de_predict_grad_rows_past_2_31_elements(case):
    """hb_de_predict_grad with O = 8 outputs over dc = 128 inputs: dmu / dvar [2^21 + 131, 8, 128] pass 2^31 elements."""
    m, d, O = (1 << 21) + 131, 128, 8
    case.need(19)
    torch.manual_seed(20)
    X, _ = seeded_problem(64, d, 20)
    y = torch.randn(64, O, generator=torch.Generator().manual_seed(20))
    model = hebo_b200.DeepEnsemble(d, 0, O, num_ensembles=2, num_epochs=3, num_hiddens=16, batch_size=16)
    model.fit(X, None, y)
    Xs = _rand((m, d), _gen(20), -1.2, 1.2)
    mu, var, dmu, dvar = model._predict_dev(Xs, None, grad=True)
    rows, past = windows(m, [O * d, d, O])
    mus, vars_, dmus, dvars = model._predict_dev(Xs[rows].contiguous(), None, grad=True)
    for big, small, what in ((mu, mus, "mu"), (var, vars_, "var"), (dmu, dmus, "dmu"), (dvar, dvars, "dvar")):
        assert_rows_equal(big, small, rows, what)
    assert_sensitive(dmu, [r for r in past if r * O * d >= E31], O * d, "dmu")
    del Xs, mu, var, dmu, dvar


def test_de_predict_at_the_largest_admitted_batch(case):
    """hb_de_predict at m = 2^31 - 16 (the largest batch it admits, 2^31 - DE_TM), one input, one output, one member of
    four hidden units: the row index itself comes within one tile of 2^31 and the byte offsets pass 2^32."""
    m = E31 - 16
    case.need(25)
    torch.manual_seed(21)
    X, y = seeded_problem(64, 1, 21)
    model = hebo_b200.DeepEnsemble(1, 0, 1, num_ensembles=1, num_epochs=3, num_hiddens=4, batch_size=16)
    model.fit(X, None, y)
    Xs = _rand((m, 1), _gen(21), -1.0, 1.0)
    mu, var = model._predict_dev(Xs, None)
    rows, _ = windows(m, [1], tile=16)
    past = list(range((1 << 30) + 1, (1 << 30) + 3)) + [m - 2, m - 1]
    mus, vars_ = model._predict_dev(Xs[rows].contiguous(), None)
    assert_rows_equal(mu, mus, rows, "mu")
    assert_rows_equal(var, vars_, rows, "var")
    assert_sensitive(mu, past, 1, "mu", fold=1 << 30)
    del Xs, mu, var


@pytest.mark.parametrize("kind", ["fe", "gumbel"])
def test_feature_selection_predict_rows_past_2_31_elements(case, kind):
    """hb_fe_predict / hb_gumbel_predict over Xs [2^23 + 131, 256] under one (seed, counter): the selection is drawn once
    per call and shared by every row, so the window rows equal a small call under the same key."""
    m, d = (1 << 23) + 131, 256
    case.need(9)
    torch.manual_seed(22)
    X, y = seeded_problem(64, d, 22)
    conf = dict(num_ensembles=2, num_epochs=2, num_hiddens=16, batch_size=8)
    model = (hebo_b200.FeDeepEnsemble(d, 0, 1, **conf) if kind == "fe"
             else hebo_b200.GumbelDeepEnsemble(d, 0, 1, reduced_dim=32, **conf))
    model.fit(X, None, y)
    Xs = _rand((m, d), _gen(22), -1.2, 1.2)
    mu, var = model._predict_dev(Xs, None, seed=1234, counter=5)
    rows, past = windows(m, [d])
    mus, vars_ = model._predict_dev(Xs[rows].contiguous(), None, seed=1234, counter=5)
    assert_rows_equal(mu, mus, rows, "mu")
    assert_rows_equal(var, vars_, rows, "var")
    assert_sensitive(mu, past, d, "mu")
    del Xs, mu, var


def test_de_predict_batch_samples_past_2_31_elements(case):
    """hb_de_predict_batch of B = 4 ensembles of 8 outputs (32 output rows) over 2^24 + 131 candidates with 4 samples and
    explicit draws: y_samp [4, m, 32] passes 2^31 elements in its last sample plane.  mu / var [32, m] and the samples of
    the window rows equal a small call on the same rows and draws."""
    from hebo_b200.ensemble import EnsembleBatch
    m, d, O, S = (1 << 24) + 131, 8, 8, 4
    K = 4 * O
    case.need(22)
    torch.manual_seed(23)
    X, _ = seeded_problem(64, d, 23)
    models = []
    for b in range(4):
        y = torch.randn(64, O, generator=torch.Generator().manual_seed(23 + b))
        mdl = hebo_b200.DeepEnsemble(d, 0, O, num_ensembles=2, num_epochs=2, num_hiddens=16, batch_size=16)
        mdl.fit(X, None, y)
        models.append(mdl)
    eb = EnsembleBatch(models)
    g = _gen(23)
    Xs = _rand((m, d), g, -1.2, 1.2)
    xi = torch.randn(S, m, K, generator=g, device="cuda")
    mu, var, samp = eb.predict(Xs, None, n_samples=S, xi=xi)
    q31 = E31 // K                               # flat sample row (s m + r) whose elements reach 2^31
    q32 = B32 // 4 // K
    extra = [q - (q // m) * m for q0 in (q31, q32) for q in range(q0 - 2, q0 + 3)]
    rows, _ = windows(m, [K], extra=extra)
    mus, vars_, samps = eb.predict(Xs[rows].contiguous(), None, n_samples=S, xi=xi[:, rows].contiguous())
    assert_rows_equal(mu.t(), mus.t(), rows, "mu")
    assert_rows_equal(var.t(), vars_.t(), rows, "var")
    for s_ in range(S):
        assert_rows_equal(samp[s_], samps[s_], rows, f"y_samp[{s_}]")
    flat = samp.view(S * m, K)
    assert_sensitive(flat, [q31 + 1, q31 + 2], K, "y_samp")
    del Xs, xi, mu, var, samp


def test_rf_predict_at_m_2_31_with_one_input(case):
    """hb_rf_predict at m = 2^31 with one input column: the row count itself is 2^31 and the byte offsets of Xc, mean and
    var pass 2^32."""
    m = E31
    case.need(25)
    torch.manual_seed(24)
    X, y = seeded_problem(400, 1, 24)
    model = hebo_b200.RF(1, 0, 1, n_estimators=8)
    model.fit(X, None, y)
    Xs = _rand((m, 1), _gen(24), -1.0, 1.0)
    mean, var, _ = model._predict_dev(Xs, None)
    rows, _ = windows(m, [1])
    past = list(range((1 << 30) + 1, (1 << 30) + 3)) + [m - 2, m - 1]
    means, vars_, _ = model._predict_dev(Xs[rows].contiguous(), None)
    assert_rows_equal(mean, means, rows, "mean")
    assert_rows_equal(var, vars_, rows, "var")
    assert_sensitive(mean, past, 1, "mean", fold=1 << 30)
    del Xs, mean, var


def test_embed_violation_rows_past_2_31_elements(case):
    """hb_embed_violation over Y [2^27 + 131, 16]."""
    from hebo_b200.embedding import embed_violation
    m, e, D = (1 << 27) + 131, 16, 40
    case.need(10)
    g = _gen(7)
    Y = _rand((m, e), g, -1.0, 1.0)
    B = torch.randn(e, D, generator=g, device="cuda") * 0.3
    G = embed_violation(Y, B)
    rows, past = windows(m, [e])
    Gs = embed_violation(Y[rows].contiguous(), B)
    assert_rows_equal(G, Gs, rows, "G")
    assert_sensitive(G, past, e, "G")
    assert bool((G > 0).float().mean() > 0.1)          # the violation is not zero everywhere
    del Y, G


# ======================================================================== Pareto filter
def _planted_rows(K):
    """K-column rows below zero, mutually non-dominated: cyclic shifts of (-1, -2, ..., -K)."""
    v = -(1.0 + torch.arange(K, dtype=torch.float32))
    return torch.stack([torch.roll(v, j) for j in range(min(K, 5))])


def test_pareto_front_k8_planted_rows_past_2_31_elements(case):
    """hb_pareto_front_k, K = 8, over F [2^28 + 4099, 8] on the sampled path.  Filler rows are (1 + t) in every column with
    random t (the sample front is one filler row, and the ~m / 4096 fillers below it survive stage 2 all over the batch);
    five mutually non-dominated rows below zero, one exact duplicate of one of them and some NaN rows are planted past 2^31
    elements.  The front is exactly the planted rows and the duplicate, in ascending order."""
    K = 8
    m = (1 << 28) + 4099
    case.need(12)
    g = _gen(8)
    t = torch.empty(m, device="cuda")
    t.uniform_(0.0, 1.0, generator=g)
    F = (1.0 + t)[:, None].expand(m, K).contiguous()
    del t
    base = E31 // K
    planted = [base + 1, base + 700, base + 2049, base + 4000, m - 1]
    dup = base + 3000
    P = _planted_rows(K).cuda()
    F[torch.tensor(planted, device="cuda")] = P
    F[dup] = P[2]
    for r in (5, base - 3, base + 2, base + 2050, m - 2):
        F[r, r % K] = float("nan")
    idx = pareto_front(F)
    assert idx.tolist() == sorted(planted + [dup])
    for r in planted:
        assert not torch.equal(F[r], F[wrap_row(r, K)])
    del F, idx


def _simplex(m, K, gen):
    x = -torch.log(torch.rand(m, K, generator=gen, device="cuda").clamp_min(1e-12))
    return (x / x.sum(1, keepdim=True)).contiguous()


def _strided_rows(m, ns=4096):
    """Rows of the stratified sample the filter takes when m > 4096 (strided_row of pareto.cu)."""
    stride = m // ns
    a = np.arange(ns, dtype=np.uint64)
    h = ((a * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) >> np.uint64(11)
    return (a.astype(np.int64) * stride + (h % np.uint64(stride)).astype(np.int64)) if stride > 1 else a.astype(np.int64)


def _front_oracle(F):
    """Ascending rows of F with no NaN and no dominator (exact count over all rows; a NaN row never dominates)."""
    ok = ~torch.isnan(F).any(1)
    cnt = _count_dominators(F[ok], F)
    return torch.nonzero(ok & (cnt == 0)).reshape(-1)


def _nan_strided_sample():
    F = torch.randn(5 * 4096 + 77, 2, generator=_gen(9), device="cuda")     # stride 5, every sampled row NaN
    F[torch.from_numpy(_strided_rows(F.shape[0])).cuda(), 0] = float("nan")
    return F


PARETO_CASES = {
    "prefix_sample": lambda: torch.randn(4097, 3, generator=_gen(9), device="cuda"),     # stride 1: the sample is a prefix
    "unsampled_tail": lambda: torch.cat([torch.randn(3 * 4096, 4, generator=_gen(9), device="cuda"),     # rows past
                                         torch.randn(1000, 4, generator=_gen(10), device="cuda") - 1.0]),  # 4096 * stride
    "all_front": lambda: _simplex((1 << 17) + 5, 3, _gen(9)),                            # every row is on the front
    "nan_sample": lambda: torch.cat([torch.full((4096, 3), float("nan"), device="cuda"),  # stride 1, every sampled row NaN
                                     torch.randn(3000, 3, generator=_gen(9), device="cuda")]),
    "nan_strided_sample": _nan_strided_sample,
}


def _sample_front_size(m):
    """Rows of the sample front the last hb_pareto_front_k call left in its workspace (nS of carve_pareto in pareto.cu:
    flags, block counts, survivors, sample front, then nS)."""
    from hebo_b200 import pareto as P
    ws = P._ws_cache[(torch.cuda.current_device(), "front")]
    up = lambda v: -(-v // 256) * 256
    mb = up(m)
    off = mb + up(-(-m // 256) * 4 + 4) + mb * 4 + up(4096 * 4)
    return int(ws[off:off + 4].view(torch.int32).item())


@pytest.mark.parametrize("name", sorted(PARETO_CASES))
def test_pareto_sampled_path_matches_the_dominance_count(case, name):
    F = PARETO_CASES[name]()
    idx = pareto_front(F)
    ref = _front_oracle(F)
    assert torch.equal(idx, ref), (name, idx.numel(), ref.numel())
    if name == "all_front":
        assert idx.numel() == F.shape[0]
    if name.startswith("nan"):
        # the NaN rows are exactly the restated sample, and the kernel's sample front came out empty: the restatement is
        # the kernel's sample and the case reaches stage 2 with nothing to filter against
        sample = torch.from_numpy(_strided_rows(F.shape[0])).cuda()
        assert bool(torch.isnan(F[sample]).any(1).all()) and int(torch.isnan(F).any(1).sum()) == sample.numel()
        assert _sample_front_size(F.shape[0]) == 0
    else:
        assert _sample_front_size(F.shape[0]) > 0


# ======================================================================== front exchange
CAP = 4096


def _rank_buffer(F, off, capacity=CAP, with_stats=True):
    m = F.shape[0]
    g = _gen(off % 1000 + 11)
    mu = torch.randn(m, generator=g, device="cuda") if with_stats else None
    var = _rand((m,), g, 0.1, 1.0) if with_stats else None
    idx, cnt = pareto_front_device(F)
    return front_pack(F, mu, var, idx, cnt, off, capacity)


def _merge_ref_check(bufs, world, capacity=CAP):
    all_buf = torch.stack(bufs).contiguous()
    out = front_merge(all_buf, world, capacity)
    ref = merge_fn_torch(all_buf.cpu(), world, capacity)
    assert torch.equal(out.cpu(), ref)
    return all_buf, out


def _unpacked_front_ids(all_buf, world, capacity=CAP):
    """Global ids of the dominance oracle's front of the rows the ranks packed (each rank's rows under its count)."""
    host = all_buf.cpu()
    F, gid = [], []
    for r in range(world):
        k = min(int(host[r, 0, 0]), capacity)
        body = host[r, 1:k + 1]
        F.append(body[:, :3])
        gid.append(body[:, 5].to(torch.int64) + (body[:, 6].to(torch.int64) << 24))
    F, gid = torch.cat(F).cuda(), torch.cat(gid)
    return gid[_front_oracle(F).cpu()] if F.shape[0] else gid


def test_front_merge_at_bench_size_on_the_sampled_path(case):
    """hb_front_merge at world = 8, capacity = 4096 (R = 32 768 rows, the sampled path): the buffer equals the host
    restatement bit for bit and its ids are the dominance oracle's front of the packed rows.  Each rank's front is a few
    hundred random rows plus, on rank 3, a full 4096-row simplex front."""
    world = 8
    g = _gen(12)
    bufs = []
    for r in range(world):
        if r == 3:
            F = _simplex(CAP, 3, g) - 3.0
        else:
            F = torch.randn(100000, 3, generator=g, device="cuda")
            F[:, 2] = 0.5 * F[:, 0] + 0.5 * F[:, 2]
        bufs.append(_rank_buffer(F, r * 100000 + (1 << 33)))
    assert int(bufs[3][0, 0]) == CAP
    all_buf, out = _merge_ref_check(bufs, world)
    gid, Ff, _ = front_read(out)
    assert gid.numel() > 0
    assert torch.equal(gid, _unpacked_front_ids(all_buf, world))


def test_front_merge_mixed_full_partial_and_empty_ranks(case):
    """Full, partial and empty ranks: bit for bit with the host restatement, the oracle's ids, and the same front as the
    merge of the non-empty ranks alone.  Every rank empty merges to count 0."""
    world = 8
    g = _gen(13)
    bufs = []
    for r in range(world):
        if r in (1, 4, 6):                              # empty: every objective of the shard is NaN
            F = torch.full((5000, 3), float("nan"), device="cuda")
        elif r == 2:
            F = _simplex(CAP, 3, g) * 4.0 - 2.0          # full
        else:
            F = torch.randn(20000, 3, generator=g, device="cuda")
        bufs.append(_rank_buffer(F, r * 20000))
    assert [int(b[0, 0]) for b in bufs].count(0) == 3
    all_buf, out = _merge_ref_check(bufs, world)
    gid, Ff, extra = front_read(out)
    assert gid.numel() > 0 and torch.equal(gid, _unpacked_front_ids(all_buf, world))
    keep = [0, 2, 3, 5, 7]
    _, out5 = _merge_ref_check([bufs[r] for r in keep], len(keep))
    for a, b in zip(front_read(out), front_read(out5)):
        assert torch.equal(a, b)
    empty = [bufs[r] for r in (1, 4, 6)] * 2 + [bufs[1], bufs[4]]
    _, out0 = _merge_ref_check(empty, world)
    assert int(out0[0, 0]) == 0 and int(out0[0, 1]) == 0
    assert front_read(out0)[0].numel() == 0


def test_front_merge_reports_a_rank_at_overflow(case):
    """A rank whose local front exceeds the capacity sets the overflow flag; the merge carries it and front_read raises."""
    world = 8
    g = _gen(14)
    bufs = [_rank_buffer(torch.randn(20000, 3, generator=g, device="cuda"), r * 20000) for r in range(world - 1)]
    bufs.append(_rank_buffer(_simplex(CAP + 500, 3, g), (world - 1) * 20000))
    assert int(bufs[-1][0, 0]) == CAP + 500 and float(bufs[-1][0, 1]) == 1.0
    _, out = _merge_ref_check(bufs, world)
    assert float(out[0, 1]) == 1.0
    with pytest.raises(RuntimeError):
        front_read(out)


def test_front_pack_ids_round_trip_up_to_2_48(case):
    """hb_front_pack ids up to 2^48 - 1 (row_offset = 2^48 - 2^31, row 2^31 - 1 of F [2^31, 3], 24 GiB) come back exactly
    through front_read, with the F of their rows; the largest row_offset plus one is refused."""
    m = E31
    case.need(25)
    F = torch.empty(m, 3, device="cuda")
    rows = torch.tensor([0, 1, (1 << 24) - 1, 1 << 24, (1 << 30) + 7, E31 - 2, E31 - 1], dtype=torch.int32, device="cuda")
    F[rows.long()] = torch.randn(rows.numel(), 3, generator=_gen(15), device="cuda")
    cnt = torch.tensor([rows.numel()], dtype=torch.int32, device="cuda")
    top = (1 << 48) - E31
    for off in (0, (1 << 24) - 1, (1 << 40) + 12345, top):
        gid, Ff, _ = front_read(front_pack(F, None, None, rows, cnt, off, 64))
        assert gid.tolist() == [off + int(r) for r in rows.tolist()], off
        assert torch.equal(Ff, F[rows.long()].cpu()), off
    assert gid[-1].item() == (1 << 48) - 1
    with pytest.raises(_lib.HeboB200Error):
        front_pack(F, None, None, rows, cnt, top + 1, 64)
    del F
