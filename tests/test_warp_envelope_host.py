"""The Kumaraswamy input warp over its whole exponent range [WARP_LO, WARP_HI] = [0.01, 10] (common.cuh), on the host.

oracle/warp_oracle.py kumar_warp_f32 restates kumar_warp operation by operation in fp32 (w, dw/da, dw/db); it is checked
here against the fp64 derivatives of the warp (warp_derivatives64, autograd of the reference's pow form) at exponents
reached through raw values as the fit reaches them -- a, b = 0.01 + 9.99 sigmoid(raw) in fp32, raw = -30 giving 0.01
and raw = +30 giving 10 exactly -- and at inputs on the clamp, one ulp inside it, 1e-4 and 1e-3 (in u) from each end and
in the interior.

Bound, per element, in units of u = 2^-24: |w32 - w64| <= 2 u W with W of tests/util.py warp_error, and
|d32 - d64| <= 2 u E + 2^-100 for both exponent derivatives with E of tests/util.py warp_derivs (the errors of log u,
a log u, log(1 - u^a), u^a and the powers carried term by term; 2^-100 covers products whose factors underflow in fp32).
Every derivative must be finite where fp64's is.  1 - u^a has to be formed as -expm1(a log u) for that: at the upper
clamp a log u is about -1e-6 a, and exp of it rounds to 1 in fp32 once a <= 0.031, so the textbook 1 - u^a is 0 there,
log(1 - u^a) = -inf and dw/db = -2 p log(1 - u^a) = 0 (-inf) = NaN.  The last test shows that this is what the pow form
does in fp32."""
import numpy as np
import pytest
import torch

from hebo_b200.scalers import kumaraswamy_warp
from oracle import warp_oracle as W
from tests.util import warp_derivs, warp_error

F32 = np.float32
U = 2.0 ** -24
FLOOR = 2.0 ** -100
TARGETS = [0.01, 0.02, 0.031, 0.045, 0.1, 0.5, 1.0, 2.0, 9.9, 10.0]
EXACT = {0.01: -30.0, 10.0: 30.0}          # fp32 sigmoid saturates: 0.01 + 9.99 * 9.4e-14 and 0.01 + 9.99 * 1 round to these


def exponent32(raw):
    """a = WARP_LO + (WARP_HI - WARP_LO) sigmoid(raw), every operation rounded to fp32."""
    r = torch.as_tensor(raw, dtype=torch.float32)
    return torch.tensor(F32(0.01), dtype=torch.float32) + torch.tensor(F32(9.99)) * (1.0 / (1.0 + torch.exp(-r)))


def raw_for(target):
    """The fp32 raw value whose exponent32 is nearest `target` (exactly `target` for 0.01, 1 and 10)."""
    if target in EXACT:
        return F32(EXACT[target])
    r = F32(np.log((target - 0.01) / (10.0 - target)))
    best = r
    for _ in range(64):
        for s in (np.inf, -np.inf):
            c = np.nextafter(r, F32(s), dtype=F32)
            if abs(float(exponent32(c)) - target) < abs(float(exponent32(best)) - target):
                best = c
        if best == r:
            break
        r = best
    return r


def grid_exponents():
    return torch.stack([exponent32(raw_for(t)) for t in TARGETS])


def grid_inputs():
    """Scaled inputs x in [-1, 1] (fp32) and beyond: the clamp, one ulp inside it, 1e-4 and 1e-3 from each end in u."""
    lo, hi = W.U32
    x_lo, x_hi = F32(2 * lo - 1), F32(2 * hi - 1)
    pts = [-1.5, -1.0, x_lo, np.nextafter(x_lo, F32(0)), np.nextafter(np.nextafter(x_lo, F32(0)), F32(0)),
           -1 + 2e-4, -1 + 2e-3, 1 - 2e-3, 1 - 2e-4, np.nextafter(x_hi, F32(0)), x_hi, np.nextafter(F32(1), F32(0)), 1.0,
           1.5, *np.linspace(-0.9, 0.9, 7)]
    return torch.tensor(np.array(pts, dtype=F32))


def test_grid_reaches_the_bounds_through_raw():
    a = grid_exponents()
    assert float(a[0]) == float(F32(0.01)) and float(a[-1]) == float(F32(10.0)) and float(a[TARGETS.index(1.0)]) == 1.0
    assert torch.allclose(a.double(), torch.tensor(TARGETS, dtype=torch.float64), rtol=1e-6)


def _grid():
    e = grid_exponents()
    x = grid_inputs()
    X, A, B = torch.meshgrid(x, e, e, indexing="ij")
    return X.reshape(-1), A.reshape(-1), B.reshape(-1)


def test_restatement_against_fp64_over_the_grid():
    x, a, b = _grid()
    w, da, db = W.kumar_warp_f32(x, a, b)
    w64, da64, db64 = W.warp_derivatives64(x, a, b)
    x64, a64, b64 = x.double(), a.double(), b.double()
    for name, g, r in (("w", w, w64), ("da", da, da64), ("db", db, db64)):
        fin = torch.isfinite(r)
        assert bool(fin.all()), name                              # fp64 is finite on the whole grid
        bad = fin & ~torch.isfinite(g)
        assert not bool(bad.any()), (name, x[bad][:4], a[bad][:4], b[bad][:4])
    Ww = warp_error(torch.zeros_like(x64), x64, a64, b64)
    da_m, db_m, Ea, Eb = warp_derivs(x64, a64, b64)
    assert torch.allclose(da_m, da64, rtol=1e-6, atol=1e-300) and torch.allclose(db_m, db64, rtol=1e-6, atol=1e-300)
    worst = {}
    for name, g, r, B in (("w", w, w64, Ww), ("da", da, da64, Ea), ("db", db, db64, Eb)):
        err = (g.double() - r).abs()
        ratio = err / (U * B + FLOOR)
        worst[name] = float(ratio.max())
        k = int(ratio.argmax())
        assert worst[name] <= 2.0, (name, worst[name], float(x[k]), float(a[k]), float(b[k]), float(g[k]), float(r[k]))
    print("largest error / (u bound):", worst)


@pytest.mark.parametrize("a", [0.01, 0.02, 0.031])
def test_upper_clamp_keeps_its_value_and_exponent_derivatives(a):
    """At x = 1 (u = 1 - eps) and small a: 1 - u^a ~ 1e-6 a, w well below 1 for b < 1, db finite and nonzero."""
    x = torch.tensor([1.0])
    A = exponent32(raw_for(a)).reshape(1)
    for b in (0.01, 0.5, 1.0, 3.0):
        B = exponent32(raw_for(b)).reshape(1)
        w, da, db = W.kumar_warp_f32(x, A, B)
        w64, da64, db64 = W.warp_derivatives64(x, A, B)
        assert bool(torch.isfinite(da).all() and torch.isfinite(db).all()), (a, b)
        assert abs(float(w) - float(w64)) <= 4 * U, (a, b, float(w), float(w64))
        assert float(db64) != 0 and abs(float(db) - float(db64)) <= 1e-4 * abs(float(db64)), (a, b, float(db), float(db64))


def test_host_warp_is_the_restatement_and_differentiable_in_x():
    """hebo_b200.scalers.kumaraswamy_warp (the input-gradient path's warp and the fixed-warp median heuristic) forms the
    warp the kernels form, and its x-gradient is finite everywhere, 0 outside the clamp, and within 1e-4 of fp64's
    wherever fp64's is above the fp32 range (taken at u = fl((x + 1) / 2), the u the fp32 chain differentiates at).  torch
    differentiates expm1 as expm1 + 1, which rounds to 0 once u^a < 2^-24 (a = 10 below u = 0.19); the warp takes that
    derivative through exp instead."""
    x, a, b = _grid()
    w, _, _ = W.kumar_warp_f32(x, a, b)
    xg = x.clone().requires_grad_(True)
    wh = kumaraswamy_warp(xg, a, b)
    assert torch.equal(wh.detach(), w)
    (g,) = torch.autograd.grad(wh.sum(), xg)
    assert bool(torch.isfinite(g).all())
    lo, hi = W.U32
    h = (x + 1) * 0.5
    assert bool((g[(h < lo) | (h > hi)] == 0).all())
    xr = (2.0 * h.double() - 1.0).requires_grad_(True)
    (g64,) = torch.autograd.grad(W.warp32(xr, a.double(), b.double()).sum(), xr)
    big = g64.abs() > 1e-30
    assert float(((g.double() - g64).abs() / g64.abs())[big].max()) <= 1e-4


def test_pow_form_loses_the_upper_clamp_in_fp32():
    """Why the restatement (and the kernel) do not use 1 - u ** a: in fp32 at the upper clamp with a = 0.02 it gives
    w = 1 and d/db = NaN (0 * -inf) where fp64 gives a finite value."""
    x = torch.tensor([1.0])
    A, B = exponent32(raw_for(0.02)).reshape(1), exponent32(raw_for(0.5)).reshape(1)
    u = torch.clamp((x + 1) * 0.5, *W.U32)
    t = torch.exp(A * torch.log(u))
    assert float(t) == 1.0
    lom = torch.log1p(-t)
    p = torch.exp(B * lom)
    assert float(lom) == -np.inf and bool(torch.isnan(-2 * p * lom).all())
    _, _, db64 = W.warp_derivatives64(x, A, B)
    assert bool(torch.isfinite(db64).all())
