"""Matern-1/2 (gpytorch MaternKernel(nu=0.5)), CPU only: the fp64 oracle's Matern-1/2 -- its closed-form MLL gradient
against autograd on data with exact duplicate rows, the committed fixture -- the host's kernel mapping and the ABI's
kernel-id checks."""
import ctypes
import os

import numpy as np
import pytest
import torch

from hebo_b200 import _lib
from oracle import emb_oracle as E
from oracle import gp_oracle as O
from tests import test_posterior_grad_host as PG
from tests import test_posterior_mace_host as PM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAD_IDS = (-1, 3, 5, 6, 7)


def _with_duplicates(X, k=6):
    """X with its last k rows replaced by copies of its first k (r^2 = 0 off the diagonal)."""
    X = X.clone()
    X[-k:] = X[:k]
    return X


def _close(ga, gc):
    return float((ga - gc).abs().max()) < 1e-10 * max(1.0, float(ga.abs().max()))


def test_kernel_value_and_radial_factor():
    r2 = torch.tensor([0.0, 1e-31, 1e-30, 0.25, 4.0], dtype=torch.float64)
    k = O.kernel_from_sqdist(r2, "matern12")
    assert float(k[0]) == float(torch.exp(torch.tensor(-1e-15, dtype=torch.float64)))
    assert torch.allclose(k[3:], torch.exp(-r2[3:].sqrt()), rtol=0, atol=1e-16)
    h = O.KERNELS["matern12"].h(r2)
    assert float(h[0]) == 0.0 and float(h[1]) == 0.0                       # below the clamp: no gradient
    assert torch.allclose(h[2:], torch.exp(-r2[2:].sqrt()) / r2[2:].sqrt(), rtol=1e-15, atol=0)


@pytest.mark.parametrize("hetero", [False, True], ids=["ard", "noise_diag"])
def test_closed_form_gradient_matches_autograd_with_duplicates(hetero):
    X, y = O.synthetic_problem("ackley", 48, 4, 5)
    X = _with_duplicates(X)
    f = O.make_fitted(X, y, kind="matern12", rng=np.random.RandomState(0))
    g = torch.Generator().manual_seed(1)
    hp = O.Hypers.unpack(f.hp.pack() + 0.3 * torch.randn(7, generator=g, dtype=torch.float64), 8e-4)
    nd = 1e-2 * (1 + (f.Xt ** 2).sum(1)) if hetero else None
    l1, g1 = O.neg_mll_autograd(f.Xt, f._yt, hp, "matern12", noise_diag=nd)
    l2, g2, _ = O.neg_mll_closed_form(f.Xt, f._yt, hp, "matern12", noise_diag=nd, block=7)
    assert torch.isfinite(g1).all() and torch.isfinite(g2).all()
    assert abs(float(l1 - l2)) < 1e-12
    assert _close(g1, g2)
    assert float(g1[3:].abs().min()) > 1e-8                                 # every lengthscale receives gradient


def test_mixed_and_shared_lengthscale_closed_form_matches_autograd_with_duplicates():
    """Matern-1/2 (numeric, ARD or one shared lengthscale) x Matern-3/2 (embedding): every parameter group."""
    from tests.test_oracle_emb import problem
    Xt, Xe, yt, nu = problem(n=50, d=3)
    Xt, Xe = _with_duplicates(Xt), _with_duplicates(Xe)
    g = torch.Generator().manual_seed(5)
    base = E.init_emb_hypers(Xt, Xe, yt, nu, seed=2)
    shared = E.EmbHypers(base.raw_noise, base.tables, base.mean, base.raw_os, torch.zeros(1, dtype=torch.float64),
                         base.raw_ls_e)
    numeric_shared = E.EmbHypers(base.raw_noise, [], base.mean, base.raw_os, torch.zeros(1, dtype=torch.float64),
                                 base.raw_ls_e)
    for hp, Xe_ in ((base, Xe), (shared, Xe), (numeric_shared, Xe[:, :0])):
        hp = hp.like(hp.pack() + 0.3 * torch.randn(hp.pack().numel(), generator=g, dtype=torch.float64))
        la, ga = E.neg_mll_emb_autograd(Xt, Xe_, yt, hp, kind="matern12")
        lc, gc = E.neg_mll_emb_closed_form(Xt, Xe_, yt, hp, kind="matern12")
        assert torch.isfinite(ga).all() and abs(float(la - lc)) < 1e-12 and _close(ga, gc)


def test_learned_warp_autograd_is_finite_with_duplicates():
    """The warp oracle differentiates by autograd; duplicate rows (r^2 = 0 pairs) give finite exponent gradients."""
    from oracle import warp_oracle as WO
    X, y = O.synthetic_problem("hartmann6", 40, 6, 3)
    Xt = _with_duplicates(X)
    yt = (y - y.mean()) / y.std()
    d = Xt.shape[1]
    g = torch.Generator().manual_seed(2)
    vec = torch.cat([torch.tensor([-4.0]), 0.3 * torch.randn(2 * d, generator=g, dtype=torch.float64),
                     torch.tensor([0.0, 0.5]), torch.full((d,), 0.3)]).double()
    loss, grad = WO.neg_mll_autograd(Xt, yt, vec, kind="matern12")
    assert torch.isfinite(loss) and torch.isfinite(grad).all() and float(grad[1:1 + 2 * d].abs().max()) > 0


def test_the_fixture_is_a_matern12_model_with_duplicate_rows():
    """tests/golden/gp_matern12.npz, which test_oracle.py and test_gpu_parity.py check as one of their GP cases."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "gp_matern12.npz"))
    assert str(g["kind"]) == "matern12"
    X = g["X"]
    assert any((X[i] == X[j]).all() for i in range(X.shape[0]) for j in range(i))


def test_host_maps_nu_one_half_and_the_kernel_key():
    import hebo_b200

    class Matern:
        nu = 0.5

    class Scale:
        base_kernel = Matern()
    assert _lib.KERNEL_IDS["matern12"] == O.KERNELS["matern12"].id == 4
    assert hebo_b200.GP(2, 0, 1, kern=Scale()).kernel == "matern12"
    assert hebo_b200.GP(2, 0, 1, kern=Matern()).kern_id == 4
    assert hebo_b200.GP(3, 0, 1, kernel="matern12").kern_id == 4
    with pytest.raises(ValueError):
        hebo_b200.GP(3, 0, 1, kernel="matern05")


def test_header_defines_the_id():
    with open(os.path.join(ROOT, "include", "hebo_b200.h")) as fh:
        defs = dict(line.split()[1:3] for line in fh if line.startswith("#define HB_KERN_"))
    assert {k: int(v) for k, v in defs.items()} == {"HB_KERN_MATERN32": 0, "HB_KERN_MATERN52": 1, "HB_KERN_RBF": 2,
                                                     "HB_KERN_MATERN12": 4}
    assert sorted(_lib.KERNEL_IDS.values()) == [0, 1, 2, 4]
    assert {k: v.id for k, v in O.KERNELS.items()} == _lib.KERNEL_IDS


def test_entry_points_reject_every_id_that_is_not_a_kernel(lib):
    """Fake device pointers: each call must fail its argument checks before any launch.  Ids 0-2 and 4 pass these checks
    and are run on real buffers by tests/test_gpu_matern12.py."""
    bad = _lib.HB_ERR_INVALID
    p = ctypes.c_void_p(16)
    n, d = 300, 2
    fit_ws = int(lib.hb_fit_workspace_bytes(n, d))
    smp_ws = int(lib.hb_sample_workspace_bytes(n, d, None, 8))
    st = (ctypes.c_int32 * 1)()
    for kern in BAD_IDS:
        assert PM._call(lib, kern=kern) == bad, kern
        assert PG._call(lib, kern=kern) == bad, kern
        assert lib.hb_fit_ex(p, None, p, n, d, None, p, kern, None, 8e-4, 0.01, 0.01, 2, None, None, p, fit_ws, None) == bad
        assert lib.hb_fit(p, p, n, d, p, kern, None, 8e-4, 0.01, 0.01, 2, None, None, p, fit_ws, None) == bad
        assert lib.hb_fit_multi_ex(p, None, p, n, d, None, 2, p, kern, None, 8e-4, 0.01, 0.01, 2, None, None, st, p,
                                   2 * fit_ws, None) == bad
        assert lib.hb_factorize_ex(p, None, p, n, d, None, p, kern, None, 8e-4, None, p, fit_ws, None) == bad
        assert lib.hb_factorize(p, p, n, d, p, kern, None, 8e-4, None, p, fit_ws, None) == bad
        assert lib.hb_mll_fwd_bwd(p, None, p, n, d, None, p, kern, None, 8e-4, 0.01, 0.0, p, p, p, p, fit_ws, None) == bad
        assert lib.hb_sample_y(p, None, 8, n, d, None, None, None, p, p, p, p, p, p, p, kern, 0.0, 1.0, 0, p, 4, p, None,
                               p, smp_ws, None) == bad
        assert lib.hb_sample_y_batch(p, None, 8, n, d, None, None, None, p, p, p, p, p, p, kern, 0.0, 1.0, 0, None, 1, 0,
                                     p, p, p, p, smp_ws, None) == bad


@pytest.fixture(scope="module")
def lib():
    if not _lib.available():
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()
