"""The device fit loop (hb_fit_multi_ex, api.cu) against its own epoch composed on the host, bit for bit, and the two leaf
kernels it is made of -- the hyper-parameter transform and the pSGLD step -- per element against fp64.

1. Transform.  Numeric ARD through hb_transform_hypers; shared lengthscale, mixed, learned and fixed warp read back from
   hb_factorize_ex -> hb_fit_state_ex.  Against transform64 (tests/test_fit_loop_host.py), with CUDA's documented
   errors expf <= 2 ulp, log1pf <= 1 ulp and u = 2^-24, ulp the fp32 ulp at the fp64 value:
   - softplus, u <= 20: expf gives e(1 + d1), |d1| <= 4u (2 ulp <= 4u relative); log1p(e(1 + d1)) = log1p(e) +
     e d1 / (1 + e) and e / ((1 + e) log1p(e)) <= 1, so with the log1pf rounding the relative error is <= 6u < 6 ulp.
     Where exp(u) is subnormal (u < -87.3) log1pf returns its argument and the error is 2 + 1 ulp of 2^-149.
     + noise_lb rounds once more: K_SOFTPLUS = 7 ulp.
   - warp: sigmoid = 1 / (1 + expf(-u)): 4u for expf, u for the sum, u for the division; 9.99 is (WARP_HI - WARP_LO)
     rounded to fp32, then the product and the sum (contracted or not) round once or twice more, and w >= WARP_LO
     dominates 9.99 sigmoid: K_WARP = 9 ulp.
   Bitwise: the mean (the identity), the u > 20 branch (softplus returns u), +-inf and NaN propagation, and every slot
   of a shared lengthscale (all equal).
2. Step.  hb_psgld_step bit for bit with psgld_step_fp32 over four chained steps, sq carried, at the grid edges P = 1,
   127, 128, 129, 4099, with and without xi and at lr = 0, with g = 0 on sq = 0, subnormal g, |g| on either side of
   2^64 (g g overflows above it: avg = inf, no step), NaN g; the finite elements within the fp64 bound of test_fit_loop_host.py.
3. The loop.  hb_fit_ex(raw_k, E = 1, lr = 0, langevin = NULL) yields the loss at raw_k after the loop's own jitter
   ladder (losses[0]) and the gradient of the successful attempt (hb_fit_state_ex.grad; the final factorisation does
   not touch it).  The host composes raw_{k+1} = psgld_step_fp32(raw_k, grad_k, sq_k, lr, 0.99, 1e-8, 1/n, xi_k),
   xi_k = langevin[k] once k + 1 > E // 10, frozen warp slots left alone, and no step (sq unchanged) on an epoch whose
   loss is +inf (given up, or hopeless).  hb_fit_ex(raw_0, E, lr = 0.03, langevin) must give the same losses, raw and
   status, bit for bit.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from hebo_b200 import GP, _lib
from tests.test_fit_loop_host import (psgld_step64, psgld_step_fp32, raw_layout, sq_bound, step_bound,
                                      transform64, ulp32)

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
F32 = np.float32
LR, ALPHA, EPS = F32(0.03), F32(0.99), F32(1e-8)
K_SOFTPLUS, K_WARP = 7.0, 9.0


def same_bits(a, b):
    """Equal as fp32 bit patterns, every NaN taken as equal."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and np.array_equal(a.view(np.uint32)[~nan],
                                                                                       b.view(np.uint32)[~nan])


# ================================================================ 1. transform
SWEEP = np.array([-200.0, -104.0, -103.9, -100.0, -88.0, -87.0, -20.0, -1e-3, 0.0, -0.0, 1e-3, 1.0, 19.99999, 20.0,
                  float(np.nextafter(F32(20), F32(np.inf))), 40.0, np.inf, -np.inf, np.nan], F32)
NOISE_LB = F32(1e-5)


def _check_hyp(hyp, raw, d, T, e, ard, warp, what):
    lay = raw_layout(d, T, e, ard, warp)
    ref = transform64(raw, d, NOISE_LB, T, e, ard, warp)
    hyp = np.asarray(hyp, F32)
    h64 = hyp.astype(np.float64)
    k = np.full(lay["H"], K_SOFTPLUS)
    if warp:
        k[-2 * d:] = K_WARP
    fin = np.isfinite(ref)
    with np.errstate(invalid="ignore"):
        err = np.abs(h64 - ref)
    assert (err[fin] <= (k * ulp32(ref))[fin]).all(), (what, hyp, ref)
    assert np.array_equal(np.isnan(hyp), np.isnan(ref)) and np.array_equal(hyp[~fin & ~np.isnan(ref)], ref[~fin & ~np.isnan(ref)]), what
    # bitwise: the mean, the u > 20 branch, +-inf, and the shared lengthscale
    assert same_bits(hyp[1], F32(raw[lay["mean"]])), what
    slots = [(0, lay["noise"]), (2, lay["os"])] + [(3 + j, lay["ls"] + (j if ard else 0)) for j in range(d)]
    if e:
        slots.append((3 + d, lay["le"]))
    for h, r in slots:
        u = F32(raw[r])
        if u > 20:
            want = (u + NOISE_LB).astype(F32) if h == 0 else u
            assert same_bits(hyp[h], want), (what, h)
        elif u == -np.inf:
            assert same_bits(hyp[h], NOISE_LB if h == 0 else F32(0.0)), (what, h)
    if not ard:
        assert len(set(hyp[3:3 + d].view(np.uint32).tolist())) == 1, what
    return float(np.max(np.where(fin, err / (k * ulp32(ref)), 0.0)))


def test_transform_numeric_ard_per_element():
    """hb_transform_hypers with every raw slot set to one sweep value, and with the sweep spread over d = 19 lengthscales."""
    lib = _lib.lib()
    worst = 0.0
    d = len(SWEEP)
    rows = [np.full(3 + d, v, F32) for v in SWEEP]
    rows.append(np.concatenate([[SWEEP[0], 0.25, SWEEP[-3]], SWEEP]).astype(F32))
    for raw in rows:
        r = torch.from_numpy(raw).to(dev)
        hyp = torch.empty(3 + d, device=dev)
        _lib.check(lib.hb_transform_hypers(_lib.ptr(r), d, float(NOISE_LB), _lib.ptr(hyp), _lib.stream_ptr()), "transform")
        torch.cuda.synchronize()
        worst = max(worst, _check_hyp(hyp.cpu().numpy(), raw, d, 0, 0, True, 0, f"raw {raw[:4]}"))
    print(f"largest error / bound {worst:.3f}")


FAMILIES = {   # name -> (GP conf, d, num_uniqs, ard, warp)
    "shared_ls": (dict(ard_kernel=False), 3, (), False, 0),
    "mixed": (dict(num_uniqs=[3, 4]), 2, (3, 4), True, 0),
    "learned_warp": (dict(warp=True), 3, (), True, 1),
    "fixed_warp": (dict(warp_a=[0.5, 2.0, 1.5], warp_b=[1.5, 0.7, 3.0]), 3, (), True, 2),
}


class Prob:
    """Everything hb_fit_ex / hb_factorize_ex take besides raw: a GP's device inputs after _prepare_fit."""

    def __init__(self, gp, raw0):
        self.gp, self.XtT, self.Xe, self.y = gp, gp._XtT, gp._Xe_dev, gp._y_dev
        self.n, self.d, self.spec, self.kern = gp.n, gp.d, gp._spec_ptr(), gp.kern_id
        self.noise_lb, self.noise_guess = float(gp.noise_lb), float(gp.noise_guess)
        self.raw0 = raw0.detach().cpu().numpy().astype(F32)
        self.P = self.raw0.size
        lay = gp._param_layout()
        self.frozen = np.zeros(self.P, bool)
        if gp.warp_mode == 2:
            self.frozen[lay["wa"]:lay["wa"] + lay["n_w"]] = True
        self.wsb = int(_lib.lib().hb_fit_workspace_bytes_ex(self.n, self.d, self.spec))


def make_prob(n, d, seed=3, num_uniqs=(), kernel="matern32", langevin=True, epochs=10, **conf):
    g = torch.Generator().manual_seed(seed)
    X = torch.rand(n, d, generator=g) * 4 - 2
    y = (torch.sin(1.5 * X[:, :1]) + 0.3 * X.sum(1, keepdim=True) ** 2).float()
    Xe = None
    if num_uniqs:
        Xe = torch.stack([torch.randint(u, (n,), generator=g) for u in num_uniqs], 1)
        y = y + 0.5 * Xe[:, :1].float()
    torch.manual_seed(seed)
    np.random.seed(seed)
    extra = dict(num_uniqs=list(num_uniqs)) if num_uniqs else {}
    gp = GP(d, len(num_uniqs), 1, num_epochs=epochs, kernel=kernel, noise_lb=1e-5, langevin=langevin, device="cuda",
            **extra, **conf)
    raw0, _ = gp._prepare_fit(X, Xe, y)
    return Prob(gp, raw0)


def family_prob(name, n=120, **kw):
    conf, d, uniqs, _, _ = FAMILIES[name]
    conf = dict(conf)
    conf.pop("num_uniqs", None)
    return make_prob(n, d, num_uniqs=uniqs, **conf, **kw)


@pytest.mark.parametrize("name", sorted(FAMILIES))
def test_transform_model_families_per_element(name):
    """hyp as hb_factorize_ex leaves it, every raw slot (tables excepted) set to one sweep value at a time."""
    lib = _lib.lib()
    conf, d, uniqs, ard, warp = FAMILIES[name]
    p = family_prob(name, n=40)
    lay = raw_layout(d, p.gp.T, len(uniqs), ard, warp)
    worst = 0.0
    for v in SWEEP:
        raw = p.raw0.copy()
        keep = np.zeros(p.P, bool)
        keep[lay["tab"]:lay["tab"] + p.gp.T] = True
        raw[~keep] = v
        r = torch.from_numpy(raw).to(dev)
        ws = torch.empty(p.wsb, dtype=torch.uint8, device=dev)
        jit = C.c_float(-1.0)
        st = lib.hb_factorize_ex(_lib.ptr(p.XtT), _lib.ptr(p.Xe), _lib.ptr(p.y), p.n, p.d, p.spec, _lib.ptr(r), p.kern, None,
                                 float(NOISE_LB), C.byref(jit), _lib.ptr(ws), p.wsb, _lib.stream_ptr())
        torch.cuda.synchronize()
        assert st in (_lib.HB_OK, _lib.HB_ERR_NOT_PD), st
        fs = _lib.FitState()
        _lib.check(lib.hb_fit_state_ex(_lib.ptr(ws), p.n, p.d, p.spec, C.byref(fs)), "state")
        hyp = ws[fs.hyp - ws.data_ptr():][:4 * lay["H"]].view(torch.float32).cpu().numpy()
        worst = max(worst, _check_hyp(hyp, raw, d, p.gp.T, len(uniqs), ard, warp, f"{name} raw {v}"))
    print(f"{name}: largest error / bound {worst:.3f}")


# ================================================================ 2. step
def _device_step(raw, g, sq, lr, factor, xi):
    lib = _lib.lib()
    r, gd, s = (torch.from_numpy(np.ascontiguousarray(t, F32)).to(dev) for t in (raw, g, sq))
    x = None if xi is None else torch.from_numpy(np.ascontiguousarray(xi, F32)).to(dev)
    _lib.check(lib.hb_psgld_step(_lib.ptr(r), _lib.ptr(gd), _lib.ptr(s), raw.size, float(lr), float(ALPHA), float(EPS),
                                 float(factor), _lib.ptr(x), _lib.stream_ptr()), "hb_psgld_step")
    torch.cuda.synchronize()
    return r.cpu().numpy(), s.cpu().numpy()


EDGE_G = np.array([0.0, 1e-41, -1.4e-45, 3e-39, 1.8e19, -1.9e19, 1e30, np.nan], F32)   # g = 0 first, on sq = 0


@pytest.mark.parametrize("mode", ["plain", "langevin", "lr0"])
@pytest.mark.parametrize("P", [1, 127, 128, 129, 4099])
def test_psgld_step_bitwise_and_fp64(P, mode):
    rng = np.random.default_rng(P)
    raw = rng.normal(size=P).astype(F32)
    sq = np.zeros(P, F32)
    lr = F32(0.0) if mode == "lr0" else LR
    factor = F32(1.0) / F32(100)
    k = min(P, EDGE_G.size)
    worst = 0.0
    for step in range(4):
        g = (rng.normal(size=P) * 10.0 ** rng.uniform(-5, 3, P)).astype(F32)
        g[:k] = EDGE_G[:k]
        if step == 0 and P > k:
            g[k] = 0.0                                   # and g = 0 on sq = 0 away from the edge block
        xi = rng.normal(size=P).astype(F32) if mode == "langevin" else None
        xd, sd = _device_step(raw, g, sq, lr, factor, xi)
        xh, sh = psgld_step_fp32(raw, g, sq, lr, ALPHA, EPS, factor, xi)
        assert same_bits(xd, xh) and same_bits(sd, sh), (P, mode, step, np.flatnonzero(xd.view(np.uint32) != xh.view(np.uint32))[:8])
        if step == 0 and mode == "langevin":             # g = 0, sq = 0: avg = eps, the Langevin term is ~1414 f xi
            assert abs(float(xd[0] - raw[0]) - math.sqrt(2 * float(lr) / float(EPS)) * float(factor) * float(xi[0])) < 1e-3 * 1414 * abs(float(xi[0])) + 1e-4
        fin = np.isfinite(g) & (np.abs(g.astype(np.float64)) < 2.0 ** 64) & np.isfinite(sq)
        with np.errstate(all="ignore"):
            x64, v64, S, L, avg = psgld_step64(raw, g, sq, lr, ALPHA, EPS, factor, xi)
        fin &= np.isfinite(x64) & np.isfinite(v64)
        e = np.abs(xd.astype(np.float64) - x64)[fin] / step_bound(x64, S, L, avg)[fin]
        assert (e <= 1.0).all(), (P, mode, step, float(e.max()))
        with np.errstate(invalid="ignore"):
            assert (np.abs(sd.astype(np.float64) - v64)[fin] <= sq_bound(v64)[fin]).all()
        if e.size:
            worst = max(worst, float(e.max()))
        if lr == 0:
            ok = np.isfinite(g) & ~np.isinf(sd)
            assert same_bits(xd[ok], raw[ok])
        raw, sq = xd, sd
    big = np.abs(EDGE_G[:k].astype(np.float64)) > 2.0 ** 64
    assert np.isinf(sq[:k][big]).all()
    print(f"P {P} {mode}: largest error / bound {worst:.3f}")


# ================================================================ 3. the loop against its composition
def run_fit(p, raws, E, lr, lang=None, Y=None):
    """hb_fit_multi_ex over B = len(raws) outputs: (status[B], raw[B, P], losses[B, E], ws)."""
    lib = _lib.lib()
    B = len(raws)
    Y = p.y.reshape(1, -1) if Y is None else Y
    wsb = int(lib.hb_fit_multi_workspace_bytes(p.n, p.d, p.spec, B))
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    r = torch.from_numpy(np.ascontiguousarray(np.stack(raws), F32)).to(dev)
    lg = None if lang is None else torch.from_numpy(np.ascontiguousarray(lang, F32)).to(dev)
    losses = (C.c_float * max(1, B * E))()
    status = (C.c_int32 * B)()
    _lib.check(lib.hb_fit_multi_ex(_lib.ptr(p.XtT), _lib.ptr(p.Xe), _lib.ptr(Y.contiguous()), p.n, p.d, p.spec, B, _lib.ptr(r),
                                   p.kern, None, p.noise_lb, p.noise_guess, float(lr), E, _lib.ptr(lg), losses, status,
                                   _lib.ptr(ws), wsb, _lib.stream_ptr()), "hb_fit_multi_ex")
    torch.cuda.synchronize()
    return list(status), r.cpu().numpy(), np.array(losses[:B * E], F32).reshape(B, E), ws


def one_epoch(p, raw, y=None):
    """(loss, grad) of the loop's epoch at raw: hb_fit_ex with E = 1, lr = 0 and no Langevin draws."""
    lib = _lib.lib()
    _, _, losses, ws = run_fit(p, [raw], 1, 0.0, None, None if y is None else y.reshape(1, -1))
    fs = _lib.FitState()
    _lib.check(lib.hb_fit_state_ex(_lib.ptr(ws), p.n, p.d, p.spec, C.byref(fs)), "state")
    grad = ws[fs.grad - ws.data_ptr():][:4 * p.P].view(torch.float32).cpu().numpy().copy()
    return F32(losses[0, 0]), grad


def compose(p, raw0, E, lang, y=None):
    """The fit composed on the host from single epochs: (status, raw, losses)."""
    raw, sq = raw0.astype(F32).copy(), np.zeros(p.P, F32)
    factor, pre = F32(1.0) / F32(p.n), E // 10
    losses = np.empty(E, F32)
    for k in range(E):
        loss, grad = one_epoch(p, raw, y)
        losses[k] = loss
        if loss == np.inf:                     # given up or hopeless: no step, sq unchanged
            continue
        xi = lang[k] if lang is not None and k + 1 > pre else None
        x, v = psgld_step_fp32(raw, grad, sq, LR, ALPHA, EPS, factor, xi)
        live = ~p.frozen
        raw[live], sq[live] = x[live], v[live]
    st, _, _, _ = run_fit(p, [raw], 0, 0.0, None, None if y is None else y.reshape(1, -1))
    return st[0], raw, losses


def assert_same_fit(got, want, what):
    (st, raw, losses), (st_c, raw_c, losses_c) = got, want
    bad = np.flatnonzero(losses.view(np.uint32) != losses_c.view(np.uint32))
    with np.errstate(invalid="ignore"):
        dr = float(np.nanmax(np.abs(raw.astype(np.float64) - raw_c))) if raw.size else 0.0
    assert bad.size == 0 and same_bits(raw, raw_c) and st == st_c, \
        (f"{what}: first epoch whose loss differs {bad[:1].tolist()} (loop {losses[bad[:1]]}, composed {losses_c[bad[:1]]}), "
         f"largest raw difference {dr:.3g}, status {st} vs {st_c}")


def check_loop(p, E, lang, what, raw0=None):
    raw0 = p.raw0 if raw0 is None else raw0
    st, raw, losses, _ = run_fit(p, [raw0], E, LR, lang)
    want = compose(p, raw0, E, lang)
    assert_same_fit((st[0], raw[0], losses[0]), want, what)
    return st[0], raw[0], losses[0]


def _lang(p, E, seed):
    """[E, P] N(0, 1) draws, frozen warp slots included: the loop must not step those whatever the draws hold (their
    gradient is 0, so a draw of 0 there would hide a step)."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(E, p.P, generator=g).numpy().astype(F32)


@pytest.mark.parametrize("langevin", [False, True])
@pytest.mark.parametrize("n", [100, 333])
def test_loop_equals_composition_matern32(n, langevin):
    """E = 1, 4 (no graph), 5 (the first capture), 16, 17 (FIT_BATCH edges), 40 (pretrain 4)."""
    p = make_prob(n, 3, seed=n)
    for E in (1, 4, 5, 16, 17, 40):
        lang = _lang(p, E, 11 * E) if langevin else None
        st, raw, losses = check_loop(p, E, lang, f"n {n} E {E} langevin {langevin}")
        assert st == _lib.HB_OK and np.isfinite(losses).all()
        assert not np.array_equal(raw, p.raw0)


@pytest.mark.parametrize("kernel", ["matern12", "rbf"])
def test_loop_equals_composition_other_kernels(kernel):
    p = make_prob(150, 2, seed=4, kernel=kernel)
    check_loop(p, 17, _lang(p, 17, 5), kernel)


@pytest.mark.parametrize("name", sorted(FAMILIES))
def test_loop_equals_composition_model_families(name):
    p = family_prob(name, n=120)
    E = 17
    st, raw, losses = check_loop(p, E, _lang(p, E, 6), name)
    assert st == _lib.HB_OK and np.isfinite(losses).all()
    if p.frozen.any():
        assert same_bits(raw[p.frozen], p.raw0[p.frozen])
        assert not np.array_equal(raw[~p.frozen], p.raw0[~p.frozen])


class AbiProb:
    """40 points repeated three times (the Gram is singular without noise), 2 numeric dims, raw noise -40 and
    noise_lb = 1e-12 for the laddering output: the inputs of test_gpu_multitask.py's batched-fit checks."""

    def __init__(self, B):
        lib = _lib.lib()
        g = torch.Generator().manual_seed(5)
        X = torch.randn(40, 2, generator=g)
        X = torch.cat([X, X, X], 0)
        self.n, self.d = X.shape
        NP = int(lib.hb_padded_n(self.n))
        Xs = (X - X.min(0).values) / (X.max(0).values - X.min(0).values) * 2 - 1
        XtT = torch.zeros(self.d, NP)
        XtT[:, :self.n] = Xs.t()
        Y = torch.stack([torch.sin(2 * X[:, 0] + b) + 0.1 * X[:, 1] for b in range(B)])
        Y = (Y - Y.mean(1, keepdim=True)) / Y.std(1, keepdim=True)
        self.XtT, self.Y = XtT.to(dev), Y.float().to(dev).contiguous()
        self.y, self.Xe, self.spec, self.kern = self.Y[0].contiguous(), None, None, 0
        self.noise_lb, self.noise_guess, self.P = 1e-12, 0.01, 5
        self.frozen = np.zeros(self.P, bool)
        self.raw0 = np.array([-2.0, 0.0, 0.5, 0.5, 0.5], F32)


# raw noise -40, outputscale softplus(3) ~ 3.05, lengthscales softplus(6) ~ 6: the Gram of the repeated rows is
# singular to fp32 rounding, and about half the epochs of the 33-epoch fit below need jitter
LADDER_RAW = np.array([-40.0, 0.0, 3.0, 6.0, 6.0], F32)


def _ladder_epochs(p, raw, y):
    """Launches of the loop's epoch at raw beyond those of the final factorisation: more than the minimum means the
    epoch went through the jitter ladder."""
    lib = _lib.lib()
    lib.hb_launch_count(1)
    run_fit(p, [raw], 1, 0.0, None, y.reshape(1, -1))
    a = int(lib.hb_launch_count(1))
    run_fit(p, [raw], 0, 0.0, None, y.reshape(1, -1))
    return a - int(lib.hb_launch_count(1))


def test_loop_equals_composition_through_the_jitter_ladder():
    """E = 33 with Langevin draws: some epochs factorise at jitter 0, some need the ladder, each ladder epoch followed by
    the ramp 1, 2, 4, ... of replay batches."""
    p = AbiProb(1)
    raw0 = LADDER_RAW.copy()
    E = 33
    lang = _lang(p, E, 9)
    st, raw, losses, _ = run_fit(p, [raw0], E, LR, lang)
    want = compose(p, raw0, E, lang)
    assert_same_fit((st[0], raw[0], losses[0]), want, "ladder")
    # replay the composition's raw_k to see which epochs laddered
    r, sq, counts = raw0.copy(), np.zeros(p.P, F32), []
    for k in range(E):
        counts.append(_ladder_epochs(p, r, p.y))
        loss, grad = one_epoch(p, r)
        if loss != np.inf:
            r, sq = psgld_step_fp32(r, grad, sq, LR, ALPHA, EPS, F32(1.0) / F32(p.n), lang[k] if k + 1 > E // 10 else None)
    print("launches per epoch:", counts)
    assert min(counts) < max(counts) and np.isfinite(losses).all()


@pytest.mark.parametrize("case", ["hopeless", "give_up_subnormal_ls"])
def test_loop_gives_up_from_epoch_zero(case):
    """E = 6 from a raw at which no epoch can train: every loss +inf, raw unchanged, HB_ERR_NOT_PD.
    hopeless: lengthscale raw -200 (softplus 0, status -1 in the first epoch); give_up_subnormal_ls: lengthscale raw -100
    (softplus ~ 3.7e-44 > 0 passes the hopeless guard, but 1 / l overflows, so the whole jitter ladder fails in every
    epoch: a give-up that repeats for the rest of the fit because raw does not move)."""
    p = make_prob(60, 2, seed=8)
    raw0 = p.raw0.copy()
    lay = p.gp._param_layout()
    raw0[lay["ls"]] = -200.0 if case == "hopeless" else -100.0
    E = 6
    st, raw, losses = check_loop(p, E, _lang(p, E, 2), case, raw0)
    assert st == _lib.HB_ERR_NOT_PD and (losses == np.inf).all() and same_bits(raw, raw0)


def test_batched_loop_equals_each_outputs_composition():
    """hb_fit_multi_ex with B = 3, output 1 the laddering model: each output equals its own composition, so outputs that
    drift out of lockstep are never stepped past num_epochs nor take another output's Langevin row."""
    B, E = 3, 33
    p = AbiProb(B)
    raws = np.stack([p.raw0] * B)
    raws[1] = LADDER_RAW
    g = torch.Generator().manual_seed(9)
    lang = torch.randn(B, E, p.P, generator=g).numpy().astype(F32)
    st, raw, losses, _ = run_fit(p, list(raws), E, LR, lang.reshape(B * E, p.P), p.Y)
    for b in range(B):
        want = compose(p, raws[b], E, lang[b], p.Y[b].contiguous())
        assert_same_fit((st[b], raw[b], losses[b]), want, f"output {b}")
