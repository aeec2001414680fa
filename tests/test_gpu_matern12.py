"""Matern-1/2 (k = e^-r, gpytorch MaternKernel(nu=0.5)) through every device path, element by element against fp64.

The checks are those the other kernels pass, run on Matern-1/2 models through the helpers of the test modules that define
them: the loss and gradient of the tensor-core epoch and of hb_mll_fwd_bwd (test_gpu_fit_epoch.py), the prediction state
(test_gpu_fit_state.py 3.), mu and sigma^2 of hb_posterior_mace_ex on both contraction paths (test_gpu_posterior_mace.py),
the input gradients (test_gpu_posterior_grad.py) and the joint samplers' Cholesky roots (test_gpu_sample_root.py).  The
Gram, the fixture, the learned warp and the batched fit run Matern-1/2 among the other kernels in their own modules.
The error bounds of kern_eval for Matern-1/2 are those of tests/util.py kernel_parts and test_gpu_fit_state.py eps_k.

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
from oracle import gp_oracle as O
from tests import test_gpu_fit_epoch as FE
from tests import test_gpu_fit_state as FS
from tests import test_gpu_posterior_grad as PG
from tests import test_gpu_posterior_mace as PM
from tests import test_gpu_sample_root as SR
from tests import util

pytestmark = pytest.mark.gpu

KIND = "matern12"
DEV = util.DEV


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


# ---------------------------------------------------------------------------------------------------------------- ids
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


def _check_both(what, m, raw, name, noise_diag=None):
    """hb_mll_fwd_bwd and (without noise_diag, which hb_fit_ex takes only through GP) the tensor-core epoch, hb_fit_ex at
    lr = 0, against the fp64 oracle with test_gpu_fit_epoch.py's tolerance: the closed forms, autograd for the learned
    warp."""
    if name in ("numeric", "hard"):
        ref64, ref32 = (FE.ref_numeric(m, raw, KIND, dt, noise_diag) for dt in (torch.float64, torch.float32))
    else:
        ref64, ref32 = (FE._family_ref(name, m, raw, dt, KIND) for dt in (torch.float64, torch.float32))
    simt = FE.simt_at(m, raw, noise_diag)
    FE.check(what + " hb_mll_fwd_bwd", simt, ref64, ref32, simt)
    if noise_diag is None:
        FE.check(what + " tensor-core epoch", FE.tc_at(m, raw), ref64, ref32, simt)


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


# ---------------------------------------------------------------------------------------------------------------- state
@pytest.mark.parametrize("name", list(VARIANTS))
def test_state_model_variants(name):
    gp, X, Xe, y = variant(name)
    FS.refactor(gp)
    FS.check_state(f"state-{KIND}-{name}", gp, X, Xe, y)


# (n = 5, where L is within 5 % of diagonal and the refinement bound of test_gpu_fit_state.py has R = 0, is left to the
# kernel-independent stage checks there)
@pytest.mark.parametrize("n", [129, 513, 1100, 4097])
def test_state_shapes(n):
    gp, X, Xe, y = model(("shape", n), n, 8, seed=n)
    FS.refactor(gp)
    FS.check_state(f"state-{KIND}-n{n}", gp, X, Xe, y)


# ---------------------------------------------------------------------------------------------------------------- posterior
@pytest.mark.parametrize("n", [5, 129, 513, 4224])
def test_posterior_across_kstar_groups(n):
    """Both contraction paths against the own-state closed form and the fp64 GP; the first candidates are training rows."""
    gp, X, Xe, y = model(("shape", n), n, 8, seed=n)
    Xs, Xse, dups = util.candidates(gp, X, Xe, 300 if n == 4224 else 129, seed=n + 1)
    PM.check_case(f"{KIND}-shape-n{n}", gp, X, Xe, y, Xs, Xse, dups)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("m,m_chunk", [(1, None), (129, 129), (513, 128), (2049, 1000), (40000, 32768)])
def test_posterior_across_bands_and_chunks(m, m_chunk):
    gp, X, Xe, y = model(("shape", 513), 513, 8, seed=513)
    Xs, Xse, dups = util.candidates(gp, X, Xe, m, seed=m + 3)
    PM.check_case(f"{KIND}-bands-m{m}", gp, X, Xe, y, Xs, Xse, dups, m_chunk=m_chunk)
    torch.cuda.empty_cache()


def test_posterior_next_to_training_rows():
    """Rows 0.01 from training rows: variance mostly cancelled, the rows the precision guard re-contracts."""
    gp, X, Xe, y = model(("shape", 513), 513, 8, seed=513)
    Xs, Xse, dups = util.candidates(gp, X, Xe, 1500, seed=44, near=True)
    PM.guard_stats(True)
    PM.check_case(f"{KIND}-near", gp, X, Xe, y, Xs, Xse, dups)
    rows, flagged = PM.guard_stats(True)
    print(json.dumps(dict(case=f"{KIND}-near", rows=rows, guard_flagged=flagged)))


@pytest.mark.parametrize("name", list(VARIANTS))
def test_posterior_model_variants(name):
    gp, X, Xe, y = variant(name)
    Xs, Xse, dups = util.candidates(gp, X, Xe, 200, seed=200)
    PM.check_case(f"{KIND}-{name}", gp, X, Xe, y, Xs, Xse, dups)


# ---------------------------------------------------------------------------------------------------------------- gradients
# n = 100 for the one-tile case: at n = 5 the 10-epoch fit leaves lengthscales near 0.03, most candidates sit 50 lengthscales
# from the data and dvar ~ 1e-43 is an fp32 subnormal, below what the bound of test_gpu_posterior_grad.py resolves
@pytest.mark.parametrize("n", [100, 129, 513, 4224])
def test_gradients_across_kstar_groups(n):
    gp, X, Xe, y = model(("shape", n), n, 8, seed=n)
    Xs, Xse, dups = util.candidates(gp, X, Xe, 300 if n == 4224 else 129, seed=n + 1)
    PG.check_case(f"{KIND}-shape-n{n}", gp, X, Xe, y, Xs, Xse, dups)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", list(VARIANTS))
def test_gradients_model_variants(name):
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


def test_gradients_at_every_training_row():
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
