"""Matern-1/2 (k = e^-r, gpytorch MaternKernel(nu=0.5)) through every device path, element by element against fp64.

The checks are those the other kernels pass, run on Matern-1/2 models through the helpers of the test modules that define
them: the Gram per element (test_gpu_fit_state.py 1.), the loss and gradient of the tensor-core epoch and of
hb_mll_fwd_bwd (test_gpu_fit_epoch.py), the fixture's trajectory, posterior, MACE and front (test_gpu_parity.py), the
batched multi-output fit (test_gpu_multitask.py), the prediction state (test_gpu_fit_state.py 3.), mu and sigma^2 of
hb_posterior_mace_ex on both contraction paths (test_gpu_posterior_mace.py), the input gradients
(test_gpu_posterior_grad.py) and the joint samplers' Cholesky roots (test_gpu_sample_root.py).  Those modules bound the
error of kern_eval through tests/util.py kernel_parts and eps_k; for Matern-1/2, with t = r the exponent of fast_exp:
    k = e^-t,  h = e^-t / t (0 below the clamp r^2 < 1e-30),  rate of t in the features 1,
    eps_k = k (E_EX2 + 1.25 t) + t e^-t (E_RSQ + 1.5):
ex2's 2 ulp and the rounded argument t log2 e as for the other kernels, and the radius r = c rsqrt(c) (E_RSQ and one
rounding) moves k by |dk/dt| t = t e^-t times its relative error.  `matern12_bounds` installs the two for the duration
of a test.

Duplicate rows are everywhere: rows that repeat training rows among the candidates, training sets with repeated rows,
integer design spaces.  h is singular at r = 0; the device takes h = 0 there as autograd through gpytorch's clamp does, so
a candidate equal to a training row has finite gradients to which that row contributes nothing."""
import json
import math

import numpy as np
import pytest
import torch

import hebo_b200
from hebo_b200 import _lib
from oracle import emb_oracle as E
from oracle import gp_oracle as O
from oracle import warp_oracle as W
from tests import test_gpu_fit_epoch as FE
from tests import test_gpu_fit_state as FS
from tests import test_gpu_multitask as MT
from tests import test_gpu_parity as GP_
from tests import test_gpu_posterior_grad as PG
from tests import test_gpu_posterior_mace as PM
from tests import test_gpu_sample_root as SR
from tests import test_gpu_warp as GW
from tests import matern12_oracle as M
from tests import util

pytestmark = pytest.mark.gpu

KIND = "matern12"
DEV = util.DEV


# ---------------------------------------------------------------------------------------------------------------- bounds
COINCIDENT = 2.0 ** -20


def kernel_parts(r2, kind):
    """tests/util.py kernel_parts with Matern-1/2: k, h (dk/dr^2 = -h / 2), |exponent of fast_exp| and its rate.  h = 0
    for r^2 < COINCIDENT as well as below the clamp: the own-state references scale the candidate in fp64 from the fp32 row
    the kernel receives, so a candidate equal to a training row lands within the fp32 roundings of the scaling (the MinMax
    shift's absolute u |x_add| / l among them) of that row's fp32 feature vector, where the device, scaling both the same
    way in fp32, has r = 0.  At the kink of e^-r that pair has h = 0 on the device and e^-r / r with an arbitrary direction
    dz / r in fp64.  Those roundings stay below r = 2^-10 here; distinct candidates are at least 0.01 / l from the data."""
    if kind != KIND:
        return util.kernel_parts(r2, kind)
    t = r2.clamp_min(1e-30).sqrt()
    h = torch.where(r2 < COINCIDENT, torch.zeros_like(r2), M.matern12_h(r2))
    return torch.exp(-t), h, t, torch.ones_like(t)


_EPS_K = FS.eps_k


def eps_k(r2, kind):
    """test_gpu_fit_state.py eps_k with Matern-1/2 (module docstring)."""
    if kind != KIND:
        return _EPS_K(r2, kind)
    k, _, t, _ = kernel_parts(r2, kind)
    return k * (FS.E_EX2 + 1.25 * t) + t * torch.exp(-t) * (FS.E_RSQ + 1.5) + FS.FLUSH


@pytest.fixture(autouse=True)
def _matern12_oracle(monkeypatch):
    """The fp64 oracle with Matern-1/2 (tests/matern12_oracle.py) for every test of this module."""
    M.install(monkeypatch)


@pytest.fixture
def matern12_bounds(monkeypatch):
    for mod in (FS, PM, PG):
        monkeypatch.setattr(mod, "kernel_parts", kernel_parts)
    monkeypatch.setattr(FS, "eps_k", eps_k)


def model(key, n, d=4, **conf):
    """util.fit_model of a Matern-1/2 model (cached under its own key)."""
    return util.fit_model((KIND, key), n, d, seed=conf.pop("seed", 7), kernel=KIND, **conf)


VARIANTS = {
    "numeric": dict(pred_likeli=False),
    "numeric_pl": dict(),
    "no_ard": dict(ard_kernel=False),
    "mixed": dict(d=3, num_uniqs=(3, 5), pred_likeli=False),
    "mixed_no_ard": dict(d=3, num_uniqs=(3, 5), ard_kernel=False),
    "hetero": dict(pred_likeli=False, noise_diag="hetero"),
    "warp": dict(warp=True),
    "fixed_warp": dict(warp_a="fixed"),
}


def variant(name):
    return model(("variant", name), 300, **VARIANTS[name])


# ---------------------------------------------------------------------------------------------------------------- Gram
@pytest.mark.parametrize("n,d", FS.GRAM_SHAPES)
def test_gram_per_element(n, d):
    """hb_gram against k64 of the kernel's own fp32 features (test_gpu_fit_state.py docstring 1.): kern_eval within
    u eps_k and K_ABS, the Gram within its bound, the diagonal bit for bit, the pad exact, duplicate rows K_ij = s."""
    Xt, ls, nd = FS.gram_inputs(n, d, seed=1000 * d + n + 12)
    NP = Xt.shape[1]
    inv = (np.float32(1.0) / ls.numpy().astype(np.float32)).astype(np.float32)
    Z = (Xt[:, :n].cpu() * torch.from_numpy(inv)[:, None]).to(DEV)
    r2, r2h = FS.sqdist64(Z.double()), FS.sqdist32_emulated(Z)
    kk, kh = kernel_parts(r2, KIND)[0], kernel_parts(r2h, KIND)[0]
    tril = torch.ones(n, n, dtype=torch.bool, device=DEV).tril()
    offd = tril & ~torch.eye(n, dtype=torch.bool, device=DEV)
    i = torch.arange(NP, device=DEV)
    pad = ((i[:, None] >= n) | (i[None, :] >= n)) & (i[:, None] >= i[None, :])
    eye = torch.eye(NP, device=DEV)
    _, h, _, _ = kernel_parts(r2, KIND)
    bound = 0.5 * h * (d + 2) * FS.U * r2 + FS.U * eps_k(r2, KIND)
    worst_abs = c_eval = c_gram = 0.0
    for cf in (dict(s=1.0, sn2=1e-3, jitter=0.0, nd=None), dict(s=2.7, sn2=0.013, jitter=1e-5, nd=nd),
               dict(s=0.31, sn2=8e-4, jitter=1e-4, nd=None)):
        hyp = torch.tensor([cf["sn2"], 0.0, cf["s"]] + ls.tolist(), dtype=torch.float32, device=DEV)
        s = float(hyp[2])
        K = FS.gram(Xt, n, hyp, KIND, cf["nd"], cf["jitter"])
        Kd = K[:n, :n].double()
        s32, sn32, j32 = (torch.tensor(v, dtype=torch.float32, device=DEV) for v in (s, float(hyp[0]), cf["jitter"]))
        dg = (s32 + sn32) + j32
        dg = dg + cf["nd"] if cf["nd"] is not None else dg.expand(n)
        assert torch.equal(K.diagonal()[:n], dg), cf
        assert torch.equal(K[pad], eye[pad]), (cf, "pad")
        if n >= 5:
            assert float(K[2, 1]) == s and float(K[n - 1, 0]) == s, (cf, "duplicates")
        c_gram = max(c_gram, FS._ratio((Kd - s * kk).abs()[offd], s * bound[offd] + FS.U * Kd.abs()[offd]))
        if cf["s"] == 1.0:
            e_ev = (Kd - kh).abs()[offd]
            c_eval = max(c_eval, FS._ratio(e_ev, FS.U * eps_k(r2h, KIND)[offd]))
            worst_abs = max(worst_abs, float(e_ev.max()) if e_ev.numel() else 0.0)
    rep = dict(case=f"gram-{KIND}-n{n}-d{d}", NP=NP, c_needed=dict(gram=c_gram, kern_eval=c_eval),
               kern_eval_max_abs_err=worst_abs, k_abs_claim=FS.K_ABS)
    FS._report(rep)
    assert worst_abs <= FS.K_ABS, rep


def test_gram_and_mll_grad_reject_ids_that_are_not_kernels():
    """hb_gram and hb_mll_grad dispatch on kern at launch: ids 3 and 5-7 launch nothing and give HB_ERR_INVALID."""
    lib = _lib.lib()
    n, d = 200, 3
    Xt, ls, _ = FS.gram_inputs(n, d, seed=5)
    NP = Xt.shape[1]
    hyp = torch.tensor([1e-3, 0.0, 1.0] + ls.tolist(), dtype=torch.float32, device=DEV)
    K = torch.full((NP, NP), float("nan"), device=DEV)
    buf = torch.zeros(NP * NP + 4 * NP, device=DEV)
    scal = torch.zeros(2, dtype=torch.float64, device=DEV)
    for kern in (3, 5, 6, 7):
        assert lib.hb_gram(FS._p(Xt), n, d, FS._p(hyp), kern, None, 0.0, FS._p(K), _lib.stream_ptr()) == _lib.HB_ERR_INVALID
        assert lib.hb_mll_grad(FS._p(Xt), n, d, FS._p(hyp), FS._p(hyp), kern, FS._p(buf), FS._p(buf), FS._p(scal), 0.01,
                               FS._p(buf), FS._p(buf), FS._p(buf), _lib.stream_ptr()) == _lib.HB_ERR_INVALID
    torch.cuda.synchronize()
    assert bool(torch.isnan(K).all())


# ---------------------------------------------------------------------------------------------------------------- MLL
def _duplicate_rows(m, k=16):
    """m with its last k observations (features, categories and targets) replaced by repeats of its first k."""
    n = m.n
    XtT, y = m.XtT.clone(), m.y.clone()
    XtT[:, n - k:n] = XtT[:, :k]
    y[n - k:n] = y[:k]
    Xe = None
    if m.Xe is not None:
        Xe = m.Xe.clone()
        Xe[n - k:n] = Xe[:k]
    return FE.Model(XtT, y, m.raw, n, m.kern, Xe, m.spec, m.noise_guess, m.H, m.De, m.owner)


def _ref(name, m, raw, dtype, noise_diag=None):
    """fp64 / fp32 (loss, gradient) of the oracles at raw: the closed forms, autograd for the learned warp."""
    Xt, y = m.Xt64().to(dtype), m.y64().to(dtype)
    if name == "learned_warp":
        loss, g = W.neg_mll_autograd(Xt, y, raw.to(dtype), FE.NOISE_LB, KIND, m.noise_guess)
        return float(loss), g.double()
    if name in ("numeric", "hard"):
        hp = O.Hypers.unpack(raw.to(dtype), FE.NOISE_LB)
        nd = None if noise_diag is None else noise_diag.to(dtype).cpu()
        loss, g, _ = O.neg_mll_closed_form(Xt, y, hp, KIND, m.noise_guess, nd)
        return float(loss), g.double()
    Xe = m.Xe.long().cpu() if m.Xe is not None else torch.zeros(m.n, 0, dtype=torch.long)
    hp = util.emb_hypers(m.owner, raw)
    hp = E.EmbHypers(*(v.to(dtype) if torch.is_tensor(v) else [t.to(dtype) for t in v] if isinstance(v, list) else v
                       for v in (hp.raw_noise, hp.tables, hp.mean, hp.raw_os, hp.raw_ls, hp.raw_ls_e, hp.noise_lb)))
    loss, g = E.neg_mll_emb_closed_form(Xt, Xe, y, hp, m.noise_guess, kind=KIND)
    return float(loss), g.double()


def _check_both(what, m, raw, name, noise_diag=None):
    """hb_mll_fwd_bwd and (without noise_diag, which hb_fit_ex takes only through GP) the tensor-core epoch, hb_fit_ex at
    lr = 0, against the fp64 oracle with test_gpu_fit_epoch.py's tolerance."""
    ref64, ref32 = _ref(name, m, raw, torch.float64, noise_diag), _ref(name, m, raw, torch.float32, noise_diag)
    simt = _mll_fwd_bwd(m, raw, noise_diag)
    FE.check(what + " hb_mll_fwd_bwd", simt, ref64, ref32, simt)
    if noise_diag is None:
        FE.check(what + " tensor-core epoch", FE.tc_at(m, raw), ref64, ref32, simt)


def _mll_fwd_bwd(m, raw, noise_diag):
    lib = _lib.lib()
    wsb = int(lib.hb_fit_workspace_bytes_ex(m.n, m.d, m.spec))
    ws = torch.zeros(wsb, dtype=torch.uint8, device=DEV)
    r = raw.float().to(DEV).contiguous()
    grad = torch.full((m.P,), float("nan"), device=DEV)
    loss = torch.full((1,), float("nan"), device=DEV)
    info = torch.full((1,), -7, dtype=torch.int32, device=DEV)
    _lib.check(lib.hb_mll_fwd_bwd(_lib.ptr(m.XtT), _lib.ptr(m.Xe), _lib.ptr(m.y), m.n, m.d, m.spec, _lib.ptr(r), m.kern,
                                  _lib.ptr(noise_diag), FE.NOISE_LB, m.noise_guess, 0.0, _lib.ptr(grad), _lib.ptr(loss),
                                  _lib.ptr(info), _lib.ptr(ws), wsb, _lib.stream_ptr()), "hb_mll_fwd_bwd")
    torch.cuda.synchronize()
    assert int(info.item()) == 0
    return float(loss.item()), grad.cpu()


@pytest.mark.parametrize("n,d", [(300, 5), (2150, 6)])
def test_numeric_loss_gradient_against_fp64(n, d):
    """ARD, at the initial hypers and at small noise with halved lengthscales, with and without duplicate rows;
    noise_diag through hb_mll_fwd_bwd."""
    base = FE.numeric_model(n, d, 900 + n, KIND)
    assert base.kern == 4
    for label, m in (("distinct", base), ("duplicates", _duplicate_rows(base))):
        for name, raw in (("numeric", m.raw), ("hard", FE.hard_raw(m.raw, d))):
            _check_both(f"{KIND} n={n} d={d} {label} {name}", m, raw, name)
    nd = (1e-2 * (1 + torch.rand(n, generator=torch.Generator().manual_seed(n)))).float().to(DEV)
    _check_both(f"{KIND} n={n} d={d} noise_diag", _duplicate_rows(base), base.raw, "numeric", noise_diag=nd)


@pytest.mark.parametrize("name,conf", [("mixed", {"num_uniqs": [4, 3]}), ("learned_warp", {"warp": True}),
                                       ("shared_lengthscale", {"ard_kernel": False}),
                                       ("mixed_shared", {"num_uniqs": [5], "ard_kernel": False})])
def test_model_family_loss_gradient_against_fp64(name, conf):
    m = FE.gp_model(2150 if name == "mixed" else 600, 4, 31, kernel=KIND, **conf)
    for label, mm in (("distinct", m), ("duplicates", _duplicate_rows(m))):
        _check_both(f"{KIND} {name} {label}", mm, mm.raw, name)


def test_deterministic_rmsprop_trajectory():
    """60 epochs without the Langevin term on data with repeated observations: the device fit ends where the fp64 oracle's
    RMSprop does (the smoke() criterion), loss by loss."""
    n, d = 300, 6
    X, y = O.synthetic_problem("ackley", n, d, 42)
    X, y = X.float().double(), y.clone()
    X[n - 20:], y[n - 20:] = X[:20], y[:20]
    yt = torch.from_numpy(O.hebo_y_transform(y.numpy())).float()
    np.random.seed(0)
    gp = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=60, noise_lb=8e-4, pred_likeli=False, langevin=False, kernel=KIND)
    gp.fit(X.float(), None, yt.reshape(-1, 1))
    Xt64 = gp.xscaler.scale_.double() * X + gp.xscaler.min_.double()
    yt64 = (yt.double().reshape(-1) - float(gp.yscaler.mean[0])) / float(gp.yscaler.std[0])
    hp, losses = O.fit_psgld(Xt64, yt64, O.Hypers.unpack(gp.raw_init.double(), 8e-4), KIND, lr=0.01, num_epochs=60,
                             record=True)
    dr = float((hp.pack() - gp.raw.double()).abs().max())
    dl = float(np.abs(gp.losses - np.array(losses)).max())
    print(json.dumps(dict(case=f"{KIND}-rmsprop", raw_diff=dr, loss_diff=dl)))
    assert dr < 1e-3 and dl <= 2e-4 * max(1.0, float(np.abs(losses).max()))


def test_learned_warp_loss_gradient_trajectory_posterior():
    """test_gpu_warp.py's check on a Matern-1/2 model: loss and gradient against autograd, the posterior, the input
    gradients chained through the warp and 30 deterministic epochs against the oracle's."""
    GW.test_learned_warp_loss_gradient_trajectory_posterior(260, 5, KIND)


def test_fixture_trajectory_posterior_mace_front():
    """tests/golden/gp_matern12.npz (12 duplicate rows): loss and gradient, the 100-epoch fit with the fixture's Langevin
    draws, mu, sigma^2, MACE, the front and argmin mu / argmax sigma over it."""
    GP_.test_golden_loss_gradient_fit_posterior_mace_front(KIND)


@pytest.mark.parametrize("d,e,n,B", [(4, [], 260, 3), (3, [4, 3], 250, 2), (4, [], 230, 2)],
                         ids=["numeric", "mixed", "learned_warp"])
def test_batched_fit_equals_per_output_fits(d, e, n, B):
    conf = {"kernel": KIND}
    if e:
        conf["num_uniqs"] = e
    if n == 230:
        conf["warp"] = True
    mt, singles, X, Xe, batched = MT._fit_both(d, e, n, B, conf, 30)
    assert batched and all(g.kern_id == 4 for g in mt.models)
    MT._assert_equal_models(mt, singles, X, Xe)


# ---------------------------------------------------------------------------------------------------------------- state
@pytest.mark.parametrize("name", list(VARIANTS))
def test_state_model_variants(name, matern12_bounds):
    gp, X, Xe, y = variant(name)
    FS.refactor(gp)
    FS.check_state(f"state-{KIND}-{name}", gp, X, Xe, y)


# (n = 5, where L is within 5 % of diagonal and the refinement bound of test_gpu_fit_state.py has R = 0, is left to the
# kernel-independent stage checks there)
@pytest.mark.parametrize("n", [129, 513, 1100, 4097])
def test_state_shapes(n, matern12_bounds):
    gp, X, Xe, y = model(("shape", n), n, 8, seed=n)
    FS.refactor(gp)
    FS.check_state(f"state-{KIND}-n{n}", gp, X, Xe, y)


# ---------------------------------------------------------------------------------------------------------------- posterior
@pytest.mark.parametrize("n", [5, 129, 513, 4224])
def test_posterior_across_kstar_groups(n, matern12_bounds):
    """Both contraction paths against the own-state closed form and the fp64 GP; the first candidates are training rows."""
    gp, X, Xe, y = model(("shape", n), n, 8, seed=n)
    Xs, Xse, dups = util.candidates(gp, X, Xe, 300 if n == 4224 else 129, seed=n + 1)
    PM.check_case(f"{KIND}-shape-n{n}", gp, X, Xe, y, Xs, Xse, dups)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("m,m_chunk", [(1, None), (129, 129), (513, 128), (2049, 1000), (40000, 32768)])
def test_posterior_across_bands_and_chunks(m, m_chunk, matern12_bounds):
    gp, X, Xe, y = model(("shape", 513), 513, 8, seed=513)
    Xs, Xse, dups = util.candidates(gp, X, Xe, m, seed=m + 3)
    PM.check_case(f"{KIND}-bands-m{m}", gp, X, Xe, y, Xs, Xse, dups, m_chunk=m_chunk)
    torch.cuda.empty_cache()


def test_posterior_next_to_training_rows(matern12_bounds):
    """Rows 0.01 from training rows: variance mostly cancelled, the rows the precision guard re-contracts."""
    gp, X, Xe, y = model(("shape", 513), 513, 8, seed=513)
    Xs, Xse, dups = util.candidates(gp, X, Xe, 1500, seed=44, near=True)
    PM.guard_stats(True)
    PM.check_case(f"{KIND}-near", gp, X, Xe, y, Xs, Xse, dups)
    rows, flagged = PM.guard_stats(True)
    print(json.dumps(dict(case=f"{KIND}-near", rows=rows, guard_flagged=flagged)))


@pytest.mark.parametrize("name", list(VARIANTS))
def test_posterior_model_variants(name, matern12_bounds):
    gp, X, Xe, y = variant(name)
    Xs, Xse, dups = util.candidates(gp, X, Xe, 200, seed=200)
    PM.check_case(f"{KIND}-{name}", gp, X, Xe, y, Xs, Xse, dups)


# ---------------------------------------------------------------------------------------------------------------- gradients
# n = 100 for the one-tile case: at n = 5 the 10-epoch fit leaves lengthscales near 0.03, most candidates sit 50 lengthscales
# from the data and dvar ~ 1e-43 is an fp32 subnormal, below what the bound of test_gpu_posterior_grad.py resolves
@pytest.mark.parametrize("n", [100, 129, 513, 4224])
def test_gradients_across_kstar_groups(n, matern12_bounds):
    gp, X, Xe, y = model(("shape", n), n, 8, seed=n)
    Xs, Xse, dups = util.candidates(gp, X, Xe, 300 if n == 4224 else 129, seed=n + 1)
    PG.check_case(f"{KIND}-shape-n{n}", gp, X, Xe, y, Xs, Xse, dups)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", list(VARIANTS))
def test_gradients_model_variants(name, matern12_bounds):
    """With a warp, GP.predict's gradient path warps the candidates in torch in front of the kernel, which rounds
    differently from the fit's fused warp: a training row is then a few ulp from its own feature vector, on the kink of
    e^-r, where the derivative is one-sided.  Those rows (and their repeats) are moved 1e-3 off the training rows."""
    gp, X, Xe, y = variant(name)
    Xs, Xse, dups = util.candidates(gp, X, Xe, 200, seed=200)
    if gp.warp_mode:
        Xs = Xs.clone()
        Xs[:5] += 1e-3
        for s_, t_ in dups:
            Xs[t_] = Xs[s_]
    PG.check_case(f"{KIND}-{name}", gp, X, Xe, y, Xs, Xse, dups)


def test_gradients_at_every_training_row(matern12_bounds):
    """Candidates equal to training rows, each repeated: the gradients are finite, duplicates give identical rows, and they
    match fp64 autograd, where the clamp gives the coinciding training row h = 0 (it contributes nothing)."""
    gp, X, Xe, y = model(("shape", 129), 129, 8, seed=129)
    Xs = torch.cat([X, X[:40]]).to(DEV).contiguous()
    dups = [(k, 129 + k) for k in range(40)]
    got, _, rep = PG.check_case(f"{KIND}-training-rows", gp, X, Xe, y, Xs, None, dups)
    assert all(bool(torch.isfinite(t).all()) for t in got)


# ---------------------------------------------------------------------------------------------------------------- samplers
def _sr_model(key, n, d=4, **conf):
    return SR._fit((KIND, key), n, d, seed=conf.pop("seed", 7), kernel=KIND, **conf)


@pytest.mark.parametrize("n,m", [(129, 1), (129, 257), (700, 512), (700, 1000), (4097, 257)])
def test_sample_y_root(n, m):
    gp, X, Xe = _sr_model(("shape", n), n, 8, seed=n)
    Xs, Xse = SR.candidates(gp, m, seed=m)
    SR.check_sample_y_case(f"{KIND}-n{n}-m{m}", gp, X, Xe, Xs, Xse)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name,conf", [("mixed", dict(d=3, num_uniqs=(3, 5))), ("warp", dict(warp=True)),
                                       ("no_ard", dict(ard_kernel=False)), ("pl_off", dict(pred_likeli=False))])
def test_sample_y_root_model_variants(name, conf):
    gp, X, Xe = _sr_model(("variant", name), 300, **conf)
    Xs, Xse = SR.candidates(gp, 300, seed=300, dup=(3, 250))
    SR.check_sample_y_case(f"{KIND}-{name}", gp, X, Xe, Xs, Xse)


@pytest.mark.parametrize("kind,m", [("numeric", 1), ("numeric", 129), ("numeric", 256), ("mixed", 33), ("mixed", 255)])
def test_sample_y_batch_root(kind, m):
    """The one-CTA root of hb_sample_y_batch: the backward-error and fp64 checks of hb_sample_y."""
    gp, X, Xe = _sr_model(("shape", 129), 129, 8, seed=129) if kind == "numeric" else \
        _sr_model(("variant", "mixed"), 300, d=3, num_uniqs=(3, 5))
    Xs, Xse = SR.candidates(gp, m, seed=1000 + m)
    F, jit, st = SR.sample_y_batch_root(gp, Xs, Xse)
    assert st == _lib.HB_OK
    assert bool((F.triu(1) == 0).all()) and bool((F.diagonal() > 0).all()) and bool(torch.isfinite(F).all())
    ref = SR.own_state_reference(gp, Xs, Xse)
    ratio, RRt, _ = SR.backward_ratio(F, ref, jit, gp.NP, SR.round_up(m, SR.GT))
    tm = SR.true_model(gp, X, Xe)
    Cm, _ = SR.true_posterior(gp, tm, Xs, Xse)
    rep = dict(case=f"{KIND}-batch-{kind}-m{m}", n=gp.n, m=m, jitter=jit, c_needed=ratio)
    rep.update(SR.fp64_errors(RRt, jit, Cm, float(tm["hyp"][2])))
    print(json.dumps(rep))
    assert ratio <= SR.C_MAX, rep
    assert rep["sigma_err_regular"] <= 1e-4 and rep["sigma_err_cancelled"] <= 2e-4 and rep["corr_err"] <= 2e-4, rep


# ---------------------------------------------------------------------------------------------------------------- optimisers
def test_hebo_loop_with_the_kernel_key_and_the_reference_injection():
    """HEBO(model_config={'kernel': 'matern12'}) on Branin, and the reference's own way to pick a kernel -- a gpytorch
    kernel object in model_config['kern'] with base_kernel.nu = 0.5 -- on an integer space (duplicate suggestions).
    On an H100 one of the integer loop's 50-epoch pSGLD fits ran a lengthscale off to softplus(-80) (the Langevin step is
    scaled by the inverse running RMS of its gradient) and gave up as the reference does (gp.py:120-126: random
    predictions for that step); the loop has to complete either way."""
    from hebo_b200.suggest import HEBO

    def f(X):
        return torch.from_numpy(O.branin(X.double().numpy()))
    torch.manual_seed(0)
    np.random.seed(0)
    opt = HEBO(lb=[-5.0, 0.0], ub=[10.0, 15.0], scramble_seed=3, n_candidates=4096,
               model_config={"lr": 0.01, "num_epochs": 100, "noise_lb": 8e-4, "pred_likeli": False, "kernel": KIND})
    for _ in range(12):
        X = opt.suggest(2)
        assert X.shape == (2, 2) and bool(((X >= opt.lb) & (X <= opt.ub)).all())
        opt.observe(X, f(X).numpy())
    assert opt.X.shape[0] == 24 and math.isfinite(opt.best_y)
    assert opt.best_y < 3.0, opt.best_y

    class Matern:
        nu = 0.5

    class Scale:
        base_kernel = Matern()
    space = [{"name": f"i{k}", "type": "int", "lb": -3, "ub": 3} for k in range(3)]
    opt = HEBO(space, scramble_seed=1, model_config={"lr": 0.01, "num_epochs": 50, "noise_lb": 8e-4, "kern": Scale()})
    import pandas as pd
    for _ in range(8):
        rec = opt.suggest(n_suggestions=2)
        assert isinstance(rec, pd.DataFrame) and rec.shape == (2, 3)
        opt.observe(rec, (rec.values.astype(float) ** 2).sum(1, keepdims=True) + 0.1)
    assert hebo_b200.GP(3, 0, 1, **opt.model_config).kernel == KIND
    assert opt.best_y <= 2.1
