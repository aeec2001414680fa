"""The learned Kumaraswamy input warp across its whole exponent range [WARP_LO, WARP_HI] = [0.01, 10] (common.cuh).

Models: numeric d = 10 with every exponent value of tests/test_warp_envelope_host.py on some dimension (a_k = TARGETS[k],
b_k = TARGETS[(3 k + shift) % 10], a different shift per kernel), for Matern-3/2, Matern-5/2, RBF and Matern-1/2, plus one
mixed (warp + two categorical columns) and one shared-lengthscale model.  The training columns hold -1 and 1 exactly (so
MinMax is the identity and x_t = x in fp32), rows on the clamp (u = eps, 1 - eps and one ulp inside each) and rows 1e-4 and
1e-3 from each end in u.  The exponents are set through raw values (raw = -30 gives 0.01, raw = +30 gives 10 exactly).

  a. Zt of hb_fit_state_ex (scale_zt_kernel: kumar_warp(x) fl(1 / l)) per element against oracle/warp_oracle.py
     kumar_warp_f32 (the same operations in fp32) and against fp64, both within 2 u W / l, W of tests/util.py warp_error
     (CUDA expf / logf / expm1f are within 2 ulp, not correctly rounded, so the restatement is not a byte match).
  b. Loss and every gradient entry, the 2 d exponents included, of hb_mll_fwd_bwd (GP.evaluate_loss) and of the
     tensor-core epoch (hb_fit_ex, one epoch at lr = 0) against fp64 warp_oracle.neg_mll_autograd, with
     test_gpu_fit_epoch.py's bound max(1e-4 max(|g64|, 0.1), 2 |g32 - g64|); the fp32 floor g32 is autograd of the stable
     restatement warp_stable (autograd of the pow form gives -inf / NaN at the upper clamp for a <= 0.031).  Every value
     must be finite.  The fp64 references clamp u to the fp32 bounds the kernels compare with (warp_oracle.U32):
     fp32(1 - 1e-6) = 1 - 1.0133e-6 moves w by up to 4e-4 at a, b <= 0.1, far above an fp32 error.
  c. The posterior (the candidate side is warped in the K* load stage) at x = +-1 exactly, one ulp inside, on and next to
     the clamp, and outside the box, on the tensor and SIMT paths, under test_gpu_posterior_mace.py check_case.  Its fp64
     GP (tests/util.py true_model) clamps at 1 - 1e-6 in fp64, so these models move each b up the grid until that clamp
     moves w by less than 1e-5 (every a stays; b = 0.5 remains with a <= 0.1, b <= 0.1 does not).
  d. GP.predict's input gradients (the warp chained in torch by hebo_b200.scalers.kumaraswamy_warp) against fp64
     autograd: finite wherever fp64's are, exactly 0 on coordinates outside the clamp, and per element
     |g - g64| <= 1e-3 J64 max |g64_w| + 2^-100 max |g64_w|: test_gpu_warp.py's 1e-3 of the largest gradient, taken in the
     warped coordinates (g64_w, the fp64 gradient with respect to w) and carried to x by that element's fp64 warp
     derivative J64 = dw/dx.  dw/dx reaches 1e4 near the clamp at a = 0.01, so one bound over all x would let small
     derivatives go unchecked or fail on rounding of the large ones; 2^-100 covers a J that underflows in fp32.  The fp64
     side starts from u = fl((x + 1) / 2) as the fp32 chain forms it: near x = 1, x + 1 rounds by up to 6e-8, 3 % of
     1 - u there, and dw/dx depends on 1 - u.  Matern-1/2 leaves out rows on a training row in warped space (no gradient
     at the kink of e^-r).
  e. hb_sample_y's root at a = 0.02, b = 0.5 in every dimension (test_gpu_sample_root.py check_sample_y_case).
  f. A learned-warp fit started at raw_a = -6 (a = 0.035) for 30 epochs without Langevin noise: every loss finite, the
     device loop equal bit for bit to its epochs composed on the host (test_gpu_fit_loop.py), and the GP fit tracking
     fp64 warp_oracle.fit_psgld within test_gpu_warp.py's tolerance.  A fixed warp_a = 0.02 fit is finite and never
     steps its frozen exponent slots."""
import math

import numpy as np
import pytest
import torch

import hebo_b200
from hebo_b200 import _lib
from oracle import warp_oracle as W
from tests.test_gpu_fit_epoch import Model, run_fit
from tests.test_gpu_fit_loop import Prob, check_loop, same_bits
from tests.test_gpu_posterior_mace import check_case
from tests.test_gpu_sample_root import check_sample_y_case
from tests.test_warp_envelope_host import TARGETS, raw_for
from tests.util import COINCIDENT, DEV, warp_error

pytestmark = pytest.mark.gpu

F32 = np.float32
U = 2.0 ** -24
D = len(TARGETS)
N = 300
CASES = {   # name -> (GP conf, shift of the b pairing)
    "matern32": (dict(kernel="matern32"), 1),
    "matern52": (dict(kernel="matern52"), 3),
    "rbf": (dict(kernel="rbf"), 7),
    "matern12": (dict(kernel="matern12"), 9),
    "mixed": (dict(num_uniqs=[3, 5]), 5),
    "shared_ls": (dict(ard_kernel=False), 2),
}
NUMERIC = ["matern32", "matern52", "rbf", "matern12"]


def edge_values():
    """x on the clamp (u = eps, 1 - eps in fp32), one ulp inside each, and 1e-4, 1e-3 from each end in u."""
    lo, hi = (F32(2 * v - 1) for v in W.U32)
    inside = lambda v: np.nextafter(v, F32(0))
    return np.array([lo, inside(lo), -1 + 2e-4, -1 + 2e-3, hi, inside(hi), 1 - 2e-4, 1 - 2e-3], F32)


def data(n, d, seed, num_uniqs=()):
    g = torch.Generator().manual_seed(seed)
    X = torch.rand(n, d, generator=g) * 2 - 1
    X[0], X[1] = -1.0, 1.0
    for j, v in enumerate(edge_values()):
        X[2 + j] = float(v)
    w = torch.randn(d, generator=g) / math.sqrt(d)
    y = torch.sin(3 * (X @ w)) + 0.5 * X[:, 0] ** 2 + 0.05 * torch.randn(n, generator=g)
    Xe = None
    if num_uniqs:
        Xe = torch.stack([torch.randint(u, (n,), generator=g) for u in num_uniqs], 1)
        y = y + 0.4 * Xe[:, 0].float()
    return X, Xe, y.reshape(-1, 1)


def clamp_shift(a, b):
    """|w(1)| moved by the fp64 clamp 1 - 1e-6 against the fp32 one (warp_oracle.U32) at exponents a, b."""
    one, a, b = torch.ones(1, dtype=torch.float64), torch.tensor([a], dtype=torch.float64), torch.tensor([b], dtype=torch.float64)
    return float((W.warp(one, a, b) - W.warp32(one, a, b)).abs())


def exponent_raws(shift, posterior=False):
    """posterior: each b moved up the grid until the fp64 GP's clamp moves w by less than 1e-5 (docstring c.)."""
    ia = np.arange(D)
    ib = (3 * ia + shift) % D
    ra = np.array([raw_for(TARGETS[i]) for i in ia], F32)
    if posterior:
        ib = [next(k for k in range(j, D) if clamp_shift(TARGETS[i], TARGETS[k]) < 1e-5) for i, j in zip(ia, ib)]
    rb = np.array([raw_for(TARGETS[j]) for j in ib], F32)
    return torch.from_numpy(ra), torch.from_numpy(rb)


_MODELS = {}


def warp_model(name, posterior=False):
    """(gp, X, Xe, y) at the grid exponents; gp's state is factorised there (GP.set_hypers)."""
    key = (name, posterior)
    if key in _MODELS:
        return _MODELS[key]
    conf, shift = CASES[name]
    conf = dict(conf)
    nu = conf.pop("num_uniqs", [])
    X, Xe, y = data(N, D, 11 + shift, nu)
    np.random.seed(0)
    torch.manual_seed(0)
    gp = hebo_b200.GP(D, len(nu), 1, lr=0.01, num_epochs=0, noise_lb=8e-4, pred_likeli=False, warp=True,
                      **(dict(num_uniqs=nu) if nu else {}), **conf)
    gp.fit(X, Xe, y)
    assert torch.equal(gp._x_mul.cpu(), torch.ones(D)) and torch.equal(gp._x_add.cpu(), torch.zeros(D))
    raw = gp.raw_init.clone()
    lay = gp._param_layout()
    ra, rb = exponent_raws(shift, posterior)
    raw[lay["wa"]:lay["wa"] + D], raw[lay["wb"]:lay["wb"] + D] = ra, rb
    gp.set_hypers(raw)
    assert not gp._fit_failed
    _MODELS[key] = (gp, X, Xe, y)
    return _MODELS[key]


def hyp_parts(gp, hyp):
    h = gp._h_wa
    return hyp[3:3 + D], hyp[h:h + D], hyp[h + D:h + 2 * D]


# ---------------------------------------------------------------------------------------------------------------- a. Zt
@pytest.mark.parametrize("name", list(CASES))
def test_zt_against_the_restatement_and_fp64(name):
    gp, X, _, _ = warp_model(name)
    ls, a, b = (t.cpu() for t in hyp_parts(gp, gp.hyp_dev))
    assert float(a.min()) == float(F32(0.01)) and float(a.max()) == float(F32(10.0))
    Zt = gp.Zt_dev[:D, :gp.n].t().cpu()
    x = gp._XtT[:, :gp.n].t().cpu()
    il = torch.from_numpy((F32(1.0) / ls.numpy()).astype(F32))
    w32, _, _ = W.kumar_warp_f32(x, a[None], b[None])
    z32 = w32 * il
    x64 = x.double()
    z64 = W.warp32(x64, a.double()[None], b.double()[None]) * il.double()
    B = warp_error(torch.zeros_like(x64), x64, a.double()[None], b.double()[None]) * il.double() + 2 * z64.abs()
    assert bool(torch.isfinite(Zt).all())
    r32 = float(((Zt.double() - z32.double()).abs() / (U * B)).max())
    r64 = float(((Zt.double() - z64).abs() / (U * B)).max())
    print(f"{name}: Zt bit-equal to the restatement {float((Zt == z32).double().mean()):.3f}, "
          f"error / (u bound) restatement {r32:.3f} fp64 {r64:.3f}")
    assert r32 <= 2.0 and r64 <= 2.0, (r32, r64)


# ---------------------------------------------------------------------------------------------------------------- b. loss, gradient
def expanded(gp, raw):
    """The raw vector in warp_oracle's numeric-ARD layout (a shared lengthscale repeated d times)."""
    lay = gp._param_layout()
    if gp.ard_kernel:
        return raw
    return torch.cat([raw[:lay["ls"]], raw[lay["ls"]].repeat(D)])


def folded(gp, g):
    """A gradient in warp_oracle's layout folded back to gp's (a shared lengthscale's gradient sums the d copies)."""
    lay = gp._param_layout()
    if gp.ard_kernel:
        return g
    return torch.cat([g[:lay["ls"]], g[lay["ls"]:].sum().reshape(1)])


@pytest.mark.parametrize("name", NUMERIC + ["shared_ls"])
def test_loss_and_gradient_against_fp64(name):
    gp, X, _, y = warp_model(name)
    raw = gp.raw.clone()
    Xt = gp._XtT[:, :gp.n].t().cpu().double()
    yt = gp._y_dev.cpu().double()
    vec = expanded(gp, raw).double()
    kw = dict(noise_lb=gp.noise_lb, kind=gp.kernel, noise_guess=gp.noise_guess)
    l64, g64 = W.neg_mll_autograd(Xt, yt, vec, warp_fn=W.warp32, **kw)
    l32, g32 = W.neg_mll_autograd(Xt.float(), yt.float(), vec.float(), warp_fn=W.warp_stable, **kw)
    l64, g64, l32, g32 = float(l64), folded(gp, g64), float(l32), folded(gp, g32.double())
    assert math.isfinite(l32) and bool(torch.isfinite(g32).all())
    tol_l = max(1e-4 * max(1.0, abs(l64)), 2 * abs(l32 - l64))
    tol_g = max(1e-4 * max(float(g64.abs().max()), 0.1), 2 * float((g32 - g64).abs().max()))
    m = Model(gp._XtT, gp._y_dev, raw, gp.n, gp.kern_id, None, gp._spec_ptr(), gp.noise_guess, 3 + 3 * D, 0, gp)
    tc = run_fit(m)
    assert torch.equal(tc["raw"], raw)
    for what, loss, g in (("hb_mll_fwd_bwd", *gp.evaluate_loss(return_grad=True)),
                          ("tensor-core epoch", float(tc["losses"][0]), tc["grad"])):
        assert math.isfinite(loss) and bool(torch.isfinite(g).all()), (what, loss, g)
        eg = float((g.double() - g64).abs().max())
        print(f"{name} {what}: loss err {abs(loss - l64):.2e} (tol {tol_l:.2e}), grad err {eg:.2e} (tol {tol_g:.2e}, "
              f"fp32 floor {float((g32 - g64).abs().max()):.2e}), exponent grad max {float(g64[1:1 + 2 * D].abs().max()):.2e}")
        assert abs(loss - l64) <= tol_l, (what, loss, l64)
        assert eg <= tol_g, (what, eg, int((g.double() - g64).abs().argmax()))


# ---------------------------------------------------------------------------------------------------------------- c. posterior
def box_candidates(m, seed):
    """Rows at x = -1 and 1 exactly, one ulp inside, on and next to the clamp, outside the box, and random rows."""
    g = torch.Generator().manual_seed(seed)
    rows = [np.full(D, v, F32) for v in (-1.0, 1.0, np.nextafter(F32(-1), F32(0)), np.nextafter(F32(1), F32(0)), -1.3, 1.3,
                                          -1.0 - 2 ** -20, 1.0 + 2 ** -20)]
    rows += [np.full(D, v, F32) for v in edge_values()]
    Xs = torch.rand(m, D, generator=g) * 2.6 - 1.3
    Xs[:len(rows)] = torch.from_numpy(np.stack(rows))
    Xs[len(rows):2 * len(rows)] = torch.from_numpy(np.stack(rows))[torch.randperm(len(rows), generator=g)]
    mix = torch.rand(m, D, generator=g) < 0.5                      # rows mixing the edges with interior coordinates
    Xs[2 * len(rows):] = torch.where(mix[2 * len(rows):], Xs[torch.randint(len(rows), (m - 2 * len(rows),), generator=g)],
                                     Xs[2 * len(rows):])
    return Xs


@pytest.mark.parametrize("name", list(CASES))
def test_posterior_at_the_box_edges(name):
    gp, X, Xe, y = warp_model(name, posterior=True)
    m = 300
    Xs = box_candidates(m, 3).to(DEV).contiguous()
    Xse = None
    if gp.num_enum:
        g = torch.Generator().manual_seed(4)
        Xse = torch.stack([torch.randint(u, (m,), generator=g) for u in gp.num_uniqs], 1).to(DEV, torch.int32).contiguous()
    check_case(f"warp envelope {name}", gp, X, Xe, y, Xs, Xse)


# ---------------------------------------------------------------------------------------------------------------- d. input gradients
@pytest.mark.parametrize("name", NUMERIC)
def test_input_gradients_against_fp64(name):
    gp, X, _, y = warp_model(name, posterior=True)
    Xs = box_candidates(120, 5)
    xg = Xs.clone().requires_grad_(True)
    pm, pv = gp.predict(xg, None)
    (pm.sum() + pv.sum()).backward()
    Xt = gp._XtT[:, :gp.n].t().cpu().double()
    yt = gp._y_dev.cpu().double()
    x64 = 2.0 * ((Xs + 1.0) * 0.5).double() - 1.0      # u as the fp32 chain forms it (x + 1 rounds near x = 1)
    a, b = (W.exponents(gp.raw.double()[1 + k * D:1 + (k + 1) * D]) for k in (0, 1))
    xo = x64.clone().requires_grad_(True)
    wo = W.warp32(xo, a[None], b[None])
    (J64,) = torch.autograd.grad(wo.sum(), xo)
    wo = wo.detach().requires_grad_(True)
    Wt = W.warp32(Xt, a[None], b[None])               # both sides warped here; predict's own warp is the identity
    mo, vo = W.predict(Wt, yt, gp.raw.double(), wo, noise_lb=gp.noise_lb, kind=gp.kernel, warp_fn=lambda X, a, b: X)
    ys, ym = gp._y_std, gp._y_mean
    ((mo * ys + ym).sum() + (vo * ys ** 2).sum()).backward()
    gw64 = wo.grad
    g, g64 = xg.grad.double(), J64 * gw64
    if gp.kernel == "matern12":
        # e^-r has no gradient at r = 0: leave out rows whose warped features coincide with a training row's (the
        # clamped ones outside the box among them), as tests/util.py kernel_parts does
        ls = gp.hyp[3:3 + D].double()
        r2 = torch.cdist(wo.detach() / ls, Wt / ls).pow(2).min(1).values
        keep = r2 >= COINCIDENT
        assert bool(keep.any()) and not bool(keep.all())
        g, g64, J64, gw64, x64 = g[keep], g64[keep], J64[keep], gw64[keep], x64[keep]
    assert bool(torch.isfinite(g64).all()) and bool(torch.isfinite(g).all())
    h = (x64 + 1) * 0.5
    out = (h < W.U32[0]) | (h > W.U32[1])
    assert bool(out.any()) and bool((g[out] == 0).all()) and bool((J64[out] == 0).all())
    scale = float(gw64.abs().max())
    ratio = ((g - g64).abs() / (1e-3 * J64.abs() * scale + 2.0 ** -100 * scale)).max()
    print(f"{name}: input gradient err / bound {float(ratio):.3f}, largest dw/dx {float(J64.abs().max()):.2e}, "
          f"largest gradient {float(g64.abs().max()):.2e}")
    assert float(ratio) <= 1.0


# ---------------------------------------------------------------------------------------------------------------- e. sampler
def test_sample_y_root_at_small_exponents():
    X, Xe, y = data(N, 4, 21)
    np.random.seed(0)
    torch.manual_seed(0)
    gp = hebo_b200.GP(4, 0, 1, lr=0.01, num_epochs=0, noise_lb=8e-4, pred_likeli=True, warp=True)
    gp.fit(X, None, y)
    raw = gp.raw_init.clone()
    lay = gp._param_layout()
    raw[lay["wa"]:lay["wa"] + 4], raw[lay["wb"]:lay["wb"] + 4] = float(raw_for(0.02)), float(raw_for(0.5))
    gp.set_hypers(raw)
    assert not gp._fit_failed
    g = torch.Generator().manual_seed(6)
    Xs = torch.rand(300, 4, generator=g) * 2.4 - 1.2
    Xs[:8] = torch.from_numpy(np.repeat(edge_values()[:, None], 4, 1))
    Xs[8:10] = torch.tensor([-1.0, 1.0])[:, None]
    check_sample_y_case("warp a 0.02 b 0.5", gp, X, None, Xs.to(DEV).contiguous(), None)


# ---------------------------------------------------------------------------------------------------------------- f. fit
def fit_data(d=3, n=200):
    X, _, y = data(n, d, 31)
    return X * 1.5 + 0.2, y                        # raw scale; MinMax maps it to [-1, 1]


def test_learned_warp_fit_from_small_exponents():
    d, E = 3, 30
    X, y = fit_data(d)
    np.random.seed(0)
    torch.manual_seed(0)
    gp0 = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=0, noise_lb=8e-4, pred_likeli=False, warp=True)
    gp0.fit(X, None, y)
    lay = gp0._param_layout()
    raw0 = gp0.raw_init.clone()
    raw0[lay["wa"]:lay["wa"] + d] = -6.0
    a0 = W.exponents(raw0[lay["wa"]:lay["wa"] + d].double())
    assert bool(((a0 - 0.035).abs() < 1e-3).all())
    # the device loop against its epochs composed on the host, bit for bit
    p = Prob(gp0, raw0)
    st, raw, losses = check_loop(p, E, None, "learned warp from raw_a = -6", raw0=raw0.numpy().astype(F32))
    assert st == _lib.HB_OK and np.isfinite(losses).all() and np.isfinite(raw).all()
    # GP.fit against the fp64 fit
    gp = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=E, noise_lb=8e-4, pred_likeli=False, warp=True, langevin=False,
                      init_raw=raw0.clone())
    gp.fit(X, None, y)
    assert not gp._fit_failed and np.isfinite(gp.losses).all()
    Xt = gp._XtT[:, :gp.n].t().cpu().double()
    yt = gp._y_dev.cpu().double()
    vec1, losses64 = W.fit_psgld(Xt, yt, raw0.double(), lr=0.01, num_epochs=E, record=True, warp_fn=W.warp32)
    dl = float(np.abs(gp.losses - np.array(losses64)).max())
    dr = float((gp.raw.double() - vec1).abs().max())
    print(f"fit from raw_a = -6: loss diff {dl:.2e}, raw diff {dr:.2e}, a now {W.exponents(vec1[1:1 + d]).tolist()}")
    assert dl <= 2e-4 * max(1.0, np.abs(losses64).max()) and dr <= 2e-3


def test_fixed_small_warp_fit_is_finite_and_frozen():
    d, E = 3, 20
    X, y = fit_data(d)
    np.random.seed(0)
    torch.manual_seed(0)
    gp = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=E, noise_lb=8e-4, pred_likeli=False, warp_a=[0.02] * d,
                      warp_b=[0.5, 1.0, 3.0])
    gp.fit(X, None, y)
    assert not gp._fit_failed and np.isfinite(gp.losses).all() and bool(torch.isfinite(gp.raw).all())
    full = gp._expand_raw(gp.raw_init)
    lay = gp._param_layout()
    assert same_bits(gp._raw_dev.cpu().numpy()[lay["wa"]:lay["wa"] + 2 * d], full.numpy()[lay["wa"]:lay["wa"] + 2 * d])
    assert not torch.equal(gp.raw, gp.raw_init)
    h = gp._h_wa
    assert torch.allclose(gp.hyp[h:h + d], torch.full((d,), 0.02), rtol=1e-5)
    loss, grad = gp.evaluate_loss(return_grad=True)
    assert math.isfinite(loss) and bool(torch.isfinite(grad).all())
