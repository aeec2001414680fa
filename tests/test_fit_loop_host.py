"""Host restatements of the pSGLD step (common.cuh psgld_update) and of the hyper-parameter transform
(pairwise.cu transform_hypers_kernel), checked here without a GPU; tests/test_gpu_fit_loop.py checks the device against
them.

u = 2^-24 is the fp32 unit roundoff.  Every fp32 operation, subnormal results included, gives
fl(x op y) = (x op y)(1 + d) + e with |d| <= u, |e| <= 2^-150 (e = 0 for + and -).

The step (a = rms_alpha, c = 1 - a exact for a in [1/2, 1]):
    v = s a + c (g g),  avg = sqrt(v) + eps,  x1 = r + ((-lr) g) / avg,  x = x1 + (f sqrt((2 lr) / avg)) xi.
From fp32 inputs, with S = lr g / avg and L = f sqrt(2 lr / avg) xi in exact arithmetic:
  - v: two non-negative terms, three roundings: |v^ - v| <= 3u v (1 + O(u)) + 3 2^-150.
  - avg: sqrt halves the relative error of v and rounds once, + eps rounds once (eps > 0); the absolute error of v
    moves sqrt(v) by at most sqrt(3 2^-150) < 2^-74 < 2^-47 eps:  |avg^ / avg - 1| <= 3.5u + 2^-47 < 3.6u.
  - S: the relative error of avg, the product, the division: 5.6u, and 2^-150 / avg where (-lr) g underflows; L: 1/avg inside the square root (3.6u), the division
    (u), halved by sqrt (2.3u), its rounding, the products by f and xi: 5.3u.  Both < 6u, plus 2^-150 per product.
  - the two sums round once each: u |x1| + u |x|.
so  |x^ - x| <= B = 6u (|S| + |L|) + u (|x1| + |x|) + 2^-150 / avg + 4 2^-150,  |v^ - v| <= 3.5u v + 3 2^-150  (the O(u^2) terms sit
inside the 6u and 3.5u).  Where g g overflows fp32 (|g| > 2^64 ~ 1.8e19) the fp32 step is 0 by construction (avg = inf)
while the fp64 step is lr / sqrt(c): those elements are compared bit for bit only.

The transform (torch.nn.functional.softplus with threshold 20, gpytorch Positive / GreaterThan, KumarWarp):
  softplus(u) = u if u > 20 else log1p(exp(u));  hyp = (softplus(raw_noise) + noise_lb, raw_mean, softplus(raw_os),
  softplus(raw_ls[...]), softplus(raw_le), WARP_LO + (WARP_HI - WARP_LO) sigmoid(raw_w[...])).
"""
import math

import numpy as np
import pytest
import torch

from oracle import gp_oracle as O

F32 = np.float32
U = 2.0 ** -24
TINY = 2.0 ** -150
WARP_LO, WARP_HI = float(F32(0.01)), float(F32(10.0))   # common.cuh WARP_LO / WARP_HI as the fp32 values they are
WARP_SPAN = float(F32(WARP_HI - WARP_LO))                 # (WARP_HI - WARP_LO), folded to fp32 by the compiler


def psgld_step_fp32(raw, grad, sq, lr, a, eps, factor, xi=None):
    """psgld_update of common.cuh in numpy float32, line by line, each operation rounded on its own: returns (raw, sq)."""
    f = F32
    raw, g, sq = np.asarray(raw, f), np.asarray(grad, f), np.asarray(sq, f)
    lr, a, eps, factor = f(lr), f(a), f(eps), f(factor)
    with np.errstate(over="ignore", under="ignore", invalid="ignore", divide="ignore"):
        v = f(sq * a) + f(f(f(1.0) - a) * f(g * g))
        v = v.astype(f)
        avg = (np.sqrt(v).astype(f) + eps).astype(f)
        x = (raw + ((f(-lr) * g).astype(f) / avg).astype(f)).astype(f)
        if xi is not None:
            t = (factor * np.sqrt((f(f(2.0) * lr) / avg).astype(f)).astype(f)).astype(f)
            x = (x + (t * np.asarray(xi, f)).astype(f)).astype(f)
    return x.astype(f), v


def psgld_step64(raw, grad, sq, lr, a, eps, factor, xi=None):
    """oracle.gp_oracle.psgld_step on float64 copies: (raw, sq, S, L, avg) with the exact step S and Langevin term L."""
    r, g, s = (torch.as_tensor(np.asarray(t, np.float64)) for t in (raw, grad, sq))
    st = O.PSGLDState(s.clone())
    x = O.psgld_step(r, g, st, float(lr), float(factor), -1 if xi is not None else 10 ** 9,
                     None if xi is None else torch.as_tensor(np.asarray(xi, np.float64)), alpha=float(a), eps=float(eps))
    avg = st.square_avg.sqrt() + float(eps)
    S = float(lr) * g / avg
    L = torch.zeros_like(S) if xi is None else float(factor) * torch.sqrt(2 * float(lr) / avg) * torch.as_tensor(np.asarray(xi, np.float64))
    return x.numpy(), st.square_avg.numpy(), S.numpy(), L.numpy(), avg.numpy()


def step_bound(x64, S, L, avg, k=6.0):
    """B of the module docstring, per element."""
    x1 = x64 - L
    return k * U * (np.abs(S) + np.abs(L)) + U * (np.abs(x1) + np.abs(x64)) + TINY / avg + 4 * TINY


def sq_bound(v64):
    return 3.5 * U * np.abs(v64) + 3 * TINY


def ulp_dist(a, b):
    """|a - b| in fp32 ulps (ordered integer distance), per element."""
    def key(t):
        i = np.asarray(t, F32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(key(a) - key(b))


# ---------------------------------------------------------------- the transform
def softplus64(u):
    u = np.asarray(u, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        return np.where(u > 20.0, u, np.log1p(np.exp(np.minimum(u, 20.0))))


def sigmoid64(u):
    u = np.asarray(u, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        return 1.0 / (1.0 + np.exp(-u))


def raw_layout(d, T=0, e=0, ard=True, warp=0):
    """Index ranges of the raw vector, restated from ModelSpec (kernels.h) for (d, T table entries, e enum columns)."""
    n_ls = 0 if d == 0 else (d if ard else 1)
    W = 2 * d if warp else 0
    return dict(noise=0, tab=1, wa=1 + T, wb=1 + T + d, n_w=W, mean=1 + T + W, os=2 + T + W, ls=3 + T + W, n_ls=n_ls,
                le=3 + T + W + n_ls, P=3 + T + W + n_ls + (1 if e > 0 else 0), H=3 + d + (1 if e > 0 else 0) + W)


def transform64(raw, d, noise_lb, T=0, e=0, ard=True, warp=0):
    """hyp[H] of transform_hypers_kernel in fp64 as a function of raw (the fp32 noise_lb is added exactly)."""
    lay = raw_layout(d, T, e, ard, warp)
    r = np.asarray(raw, np.float64)
    hyp = np.empty(lay["H"])
    hyp[0] = softplus64(r[lay["noise"]]) + float(F32(noise_lb))
    hyp[1] = r[lay["mean"]]
    hyp[2] = softplus64(r[lay["os"]])
    for k in range(d):
        hyp[3 + k] = softplus64(r[lay["ls"] + (k if ard else 0)])
    h = 3 + d
    if e > 0:
        hyp[h] = softplus64(r[lay["le"]])
        h += 1
    if warp:
        hyp[h:h + 2 * d] = WARP_LO + WARP_SPAN * sigmoid64(r[lay["wa"]:lay["wa"] + 2 * d])
    return hyp


def ulp32(x):
    """The fp32 ulp at the fp64 value x: 2^(e - 23) for |x| in [2^e, 2^(e+1)), 2^-149 below 2^-126."""
    a = np.abs(np.asarray(x, np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        ex = np.floor(np.log2(np.where(a > 0, a, 1.0)))
    return np.where(a >= 2.0 ** -126, 2.0 ** (np.maximum(ex, -126) - 23), 2.0 ** -149)


# ---------------------------------------------------------------- tests
def _step_inputs(P, seed):
    rng = np.random.default_rng(seed)
    raw = rng.normal(size=P).astype(F32)
    g = (rng.normal(size=P) * 10.0 ** rng.uniform(-6, 4, P)).astype(F32)
    xi = rng.normal(size=P).astype(F32)
    return raw, g, xi


@pytest.mark.parametrize("langevin", [False, True])
def test_fp32_step_is_within_the_fp64_bound_over_many_steps(langevin):
    """200 chained steps of 4096 parameters (gradients over ten decades, g = 0 and subnormal g included), the sq state
    carried in fp32; each step from the fp32 state against the fp64 oracle step from the same state."""
    P, lr, a, eps, factor = 4096, F32(0.03), F32(0.99), F32(1e-8), F32(1.0) / F32(333)
    raw, _, _ = _step_inputs(P, 0)
    sq = np.zeros(P, F32)
    worst = 0.0
    for k in range(200):
        _, g, xi = _step_inputs(P, 100 + k)
        g[:4] = [0.0, 1e-41, -1e-45, 3e-39]
        x32, v32 = psgld_step_fp32(raw, g, sq, lr, a, eps, factor, xi if langevin else None)
        x64, v64, S, L, avg = psgld_step64(raw, g, sq, lr, a, eps, factor, xi if langevin else None)
        e = np.abs(x32.astype(np.float64) - x64) / step_bound(x64, S, L, avg)
        assert (e <= 1.0).all(), (k, int(e.argmax()), float(e.max()))
        assert (np.abs(v32.astype(np.float64) - v64) <= sq_bound(v64)).all(), k
        worst = max(worst, float(e.max()))
        raw, sq = x32, v32
    print(f"largest error / bound: {worst:.3f}")


def test_fp32_step_edges():
    """g = 0 with sq = 0: avg = eps and the Langevin term is f sqrt(2 lr / eps) xi ~ 1414 f xi (lr = 0.01); g g
    overflowing: avg = inf, no step; NaN g: NaN; lr = 0: raw unchanged."""
    lr, a, eps = F32(0.01), F32(0.99), F32(1e-8)
    raw = np.array([0.5, 0.5, 0.5, 0.5, -2.0], F32)
    g = np.array([0.0, 1.9e19, -4e20, np.nan, 1.0], F32)
    x, v = psgld_step_fp32(raw, g, np.zeros(5, F32), lr, a, eps, F32(1.0), np.ones(5, F32))
    assert abs(float(x[0]) - 0.5 - math.sqrt(2 * 0.01 / 1e-8)) < 1e-3 * 1414
    assert np.isinf(v[1]) and np.isinf(v[2]) and x[1] == raw[1] and x[2] == raw[2]
    assert np.isnan(x[3]) and np.isnan(v[3])
    x0, _ = psgld_step_fp32(raw, np.array([0.0, 2e19, -1e-45, 1.0, -3.0], F32), np.zeros(5, F32), F32(0.0), a, eps, F32(1.0))
    assert np.array_equal(x0.view(np.uint32), raw.view(np.uint32))


def test_fp32_step_against_torch_rmsprop_and_sgld():
    """One step of torch.optim.RMSprop (single tensor) followed by the Langevin term of sgld.py:64-70 in fp32 on this
    CPU.  torch differs from the device in ways it does not specify (its CPU addcmul is fused, `2 * lr / avg` is
    avg.reciprocal() * 0.06, and 1 - alpha is rounded from the fp64 constant rather than formed in fp32), so only the bound each of them has against its own exact step is asserted:
    10u for torch (three more roundings of constants than the device has), 6u for the restatement.  The ulp distance
    between the two is printed."""
    P, lr, alpha, eps, n = 4096, 0.03, 0.99, 1e-8, 333
    raw, g, xi = _step_inputs(P, 7)
    sq = (np.abs(_step_inputs(P, 8)[1]) ** 2 * 0.5).astype(F32)
    p = torch.nn.Parameter(torch.from_numpy(raw.copy()))
    p.grad = torch.from_numpy(g.copy())
    opt = torch.optim.RMSprop([p], lr=lr, alpha=alpha, eps=eps, foreach=False)
    opt.state[p]["step"] = torch.tensor(0.0)
    opt.state[p]["square_avg"] = torch.from_numpy(sq.copy())
    opt.step()
    with torch.no_grad():
        avg = opt.state[p]["square_avg"].sqrt().add_(eps)
        noise_var = 2 * lr / avg
        p.add_((1.0 / n) * noise_var.sqrt() * torch.from_numpy(xi))
    xt, vt = p.detach().numpy(), opt.state[p]["square_avg"].numpy()
    x64, v64, S, L, avg = psgld_step64(raw, g, sq, lr, alpha, eps, 1.0 / n, xi)
    assert (np.abs(xt.astype(np.float64) - x64) <= step_bound(x64, S, L, avg, k=10.0)).all()
    assert (np.abs(vt.astype(np.float64) - v64) <= 3 * sq_bound(v64)).all()
    x32, v32 = psgld_step_fp32(raw, g, sq, F32(lr), F32(alpha), F32(eps), F32(1.0) / F32(n), xi)
    d = ulp_dist(x32, xt)
    print(f"restatement vs torch: raw max {int(d.max())} ulp, {int((d > 0).sum())} of {P} differ; "
          f"sq max {int(ulp_dist(v32, vt).max())} ulp")


SPECS = {   # name -> (GP conf, d, e, T, ard, warp)
    "numeric": (dict(), 3, (), True, 0),
    "shared_ls": (dict(ard_kernel=False), 3, (), False, 0),
    "mixed": (dict(num_uniqs=[3, 4]), 2, (3, 4), True, 0),
    "mixed_shared": (dict(num_uniqs=[5], ard_kernel=False), 2, (5,), False, 0),
    "learned_warp": (dict(warp=True), 3, (), True, 1),
    "fixed_warp": (dict(warp_a=[0.5, 2.0, 1.0], warp_b=[1.5, 0.7, 3.0]), 3, (), True, 2),
    "warp_mixed": (dict(num_uniqs=[3], warp=True), 2, (3,), True, 1),
}


@pytest.mark.parametrize("name", sorted(SPECS))
def test_transform_layout_matches_the_model(name):
    """raw_layout (the restatement's reading of ModelSpec) is GP._param_layout for every model family, and transform64
    reads each hyper-parameter from its own raw slot: a raw vector of distinct values maps to the expected ones."""
    from hebo_b200 import GP
    conf, d, uniqs, ard, warp = SPECS[name]
    gp = GP(d, len(uniqs), 1, **conf)
    T = gp.T
    lay = raw_layout(d, T, len(uniqs), ard, warp)
    ref = gp._param_layout()
    assert {k: lay[k] for k in ref} == ref
    assert lay["P"] == 3 + T + lay["n_w"] + lay["n_ls"] + (1 if uniqs else 0)
    raw = 21.0 + np.arange(lay["P"], dtype=np.float64)     # > 20: softplus is the identity
    hyp = transform64(raw, d, 0.0, T, len(uniqs), ard, warp)
    assert hyp[0] == raw[0] and hyp[1] == raw[lay["mean"]] and hyp[2] == raw[lay["os"]]
    for k in range(d):
        assert hyp[3 + k] == raw[lay["ls"] + (k if ard else 0)]
    if uniqs:
        assert hyp[3 + d] == raw[lay["le"]]
    if warp:
        w = raw[lay["wa"]:lay["wa"] + 2 * d]
        assert np.array_equal(hyp[-2 * d:], WARP_LO + WARP_SPAN * sigmoid64(w))


def test_transform64_edges():
    u = np.array([-np.inf, -200.0, 0.0, 20.0, np.nextafter(F32(20), F32(np.inf)), 40.0, np.inf, np.nan])
    s = softplus64(u)
    assert s[0] == 0.0 and s[1] == math.log1p(math.exp(-200.0)) and s[2] == math.log(2.0)
    assert s[3] == math.log1p(math.exp(20.0)) and s[4] == float(u[4]) and s[5] == 40.0 and s[6] == np.inf and np.isnan(s[7])
    sg = sigmoid64(np.array([-np.inf, np.inf, np.nan]))
    assert sg[0] == 0.0 and sg[1] == 1.0 and np.isnan(sg[2])
    assert ulp32(1.0) == 2.0 ** -23 and ulp32(1.5) == 2.0 ** -23 and ulp32(1e-40) == 2.0 ** -149 and ulp32(0.0) == 2.0 ** -149
