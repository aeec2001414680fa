"""The GP prediction state -- Gram, Cholesky factor, refined L^-1, alpha, quadratic form, log-det, scaled features --
element by element against fp64 references.

Every posterior, gradient and sampler call reads what hb_factorize_ex leaves in the fit workspace: transform ->
[embedding gather, warp] -> gram_kernel -> chol_block64_kernel through the jitter ladder -> launch_tri_inverse ->
launch_linv_refine (one Newton step) -> fp16 split -> launch_solve_logdet -> scale_zt.  u = 2^-24, u64 = 2^-53; |A| is
the element-wise absolute value and |A||B| an fp64 matrix product of absolute values.  Each case prints the c it needs
(max |error| / bound) and requires c <= C_MAX.

1. hb_gram (numeric ARD features, all four kernels), n = 5 ... 4097 (NP up to 4224) and d = 1 ... 300 across the
   32-wide feature chunks:
   - the kernel function itself: with s = 1, K_ij against k64(r^_ij^2), where r^^2 is the fp32 squared distance exactly
     as accum_sqdist forms it (df = fl(z_i - z_j), r2 = fma(df, df, r2) in feature order, emulated in fp64 with a
     rounding to fp32 per step) on the kernel's own fp32 features z = fl(Xt fl(1 / l)) (stage4).  Bound u eps_k:
       RBF        eps_k = k (E_EX2 + 1.25 t)
       Matern-1/2 eps_k = k (E_EX2 + 1.25 t) + t e^-t (E_RSQ + 1.5)
       Matern-3/2 eps_k = k (E_EX2 + 1.25 t + 2) + t^2 e^-t (E_RSQ + 2.5)
       Matern-5/2 eps_k = k (E_EX2 + 1.25 t + 3.5) + t (t + t^2 / 3) e^-t (E_RSQ + 2.5)
     with t the exponent of fast_exp (kernel_parts).  E_EX2 = 4: ex2.approx.ftz.f32 is accurate to 2 ulp of its result
     (PTX ISA), at most 2^-22 relative; the argument fl(x fl(log2 e)) carries 1.22 u relative (constant and product
     rounding), i.e. 1.22 |x| u relative on exp(x), taken as 1.25 t.  E_RSQ = 2^-22.9 / u: rsqrt.approx.f32 (PTX ISA); r =
     c q and a r add one rounding each and a = fl(sqrt 3 | sqrt 5) half of one, so the exponent a r carries
     (E_RSQ + 2.5) u relative, which moves k by |dk/dt| t (E_RSQ + 2.5) u: t^2 e^-t for Matern-3/2, and for Matern-5/2,
     whose r^2 term does not go through the radius, (t + t^2 / 3) e^-t t.  Matern-1/2 has t = r and no constant a: the
     radius (E_RSQ and one rounding) moves k by |dk/dt| t = t e^-t times its relative error.  The last terms of the k
     factor are the roundings of 1 + a r, (5/3) r^2, their sum and the product with the exponential.  Plus 2^-102
     (results below 2^-126 flush to zero).  The largest |K - k64(r^^2)| is also checked against K_ABS = 3e-7, the absolute accuracy
     common.cuh states for k (largest measured 2.4e-7, Matern-5/2 near k ~ 1).
   - the Gram: |K - s k64(r^2)| <= s (h (d + 2) u r^2 / 2 + u eps_k) + u |K|, r^2 in fp64 from the same fp32 features:
     the direct-difference sum has non-negative terms, so its relative error is at most (d + 2) u (d accumulations, the
     squared rounding of each difference), which moves k by |dk/dr^2| = h / 2 times it (kernel_parts); u |K| is the
     rounding of s k.
   - the diagonal bit for bit: fl(fl(fl(s + sigma^2) + jitter) + noise_diag_i), with and without noise_diag, jitter 0
     and not; the pad block exactly the identity and pad off-diagonal entries exactly 0 (the pad columns of Xt hold NaN);
     rows that duplicate another give K_ij = s exactly.  Only lower tiles are written, so only the lower triangle is
     compared.

2. The SIMT stages on their own, on Gram matrices (d = 2, Matern-3/2) at NP = 128 ... 4224, n = NP and n = NP - 37 (an
   identity pad block): sigma^2 = 8e-4 at lengthscale 0.5 (well conditioned) and sigma^2 = 1e-6 at lengthscale 1.0
   (raised tenfold until the fp32 Cholesky succeeds; the sigma^2 used and cond_1(L) are printed).  Lambda = L^-1 in fp64
   of the fp32 factor L.
   - hb_tri_inverse: |X - Lambda| <= c u sqrt(NP) |Lambda||L||X|, and the right residual X L - I = (X - Lambda) L within
     c u sqrt(NP) |Lambda||L||X||L|; the strict upper triangle is exactly 0.  NP = 384, 640, 1152, 2176, 4224 end a
     doubling level in a partial pair.  The row-wise form |X L - I| <= c u sqrt(NP) |X||L| holds for the base blocks'
     substitution but not for the doubling, which forms an off-diagonal block as -B^-1 (C A^-1): its right residual is
     B^-1 C (I - A^-1 A) plus the products' roundings, of size u |X||L||X||L|.  That c grows with cond(L) (about 6 at
     cond_1(L) = 1e4, over 100 after the jitter ladder), so it is printed, not asserted.
   - hb_kinv on every element of the lower 128-tiles: |Kinv - (X^T X)64| <= c u sqrt(NP) |X|^T|X|; upper tiles are not
     written.
   - hb_solve_logdet: r = fl32(y - c) (gemv_rows_kernel subtracts in fp32); v = X r and alpha64 = X^T v in fp64 on the
     device's X.  The kernels accumulate products of fp32 numbers (exact in fp64) in fp64, so with S = |X|^T |X||r|:
     |alpha - alpha64| <= u |alpha64| + 4 NP u64 S (the final rounding; NP u64 S for each GEMV of the device and of the
     reference); alpha pad entries exactly 0; |scal[0] - |v|^2| <= 4 NP u64 sum_i |v_i| (|X||r|)_i + n u64 |v|^2 and
     |scal[1] - 2 sum log L_ii| <= 4 n u64 (sum |log L_ii| + 1).  The bounds of scal are in units of u64, about 1e-12
     relative at these sizes.

3. The state of hb_factorize_ex, read through hb_fit_state_ex (GP.*_dev), for every model variant and feature width
   of tests/util.py, numeric models at n = 5 ... 4097, sigma^2 at noise_lb = 1e-6, and outputscale 1e3:
   (a)  |L L^T - Khat64| <= B_gram + c u sqrt(NP) |L||L|^T on the lower triangle, Khat64 built in fp64 on the state's
        own features (Zt_dev, embedding rows included) with the state's hyp, noise_diag and jitter: B_gram is the Gram
        bound of 1. per factor (numeric with d, the embedding Matern-3/2 with De) plus 2 u |K| for the two products, and
        3 u |Khat_ii| on the diagonal.  Every pad entry of L is exact (identity block).
   (a') numeric rows of Zt of non-warped models are fl(Xt fl(1 / l)) bit for bit; embedding rows the gathered
        fl(table fl(1 / l_e)) and tab_s = fl(tables fl(1 / l_e)) bit for bit; warped rows within W u / l + 2 u |z| of
        the fp64 warp, W the step-by-step fp32 error of kumar_warp (tests/util.py warp_error).
   (b)  X0 = hb_tri_inverse(L_dev), the kernel and input factorize runs it on (the upper part of L is never read).  The
        two refinement kernels: |X - (X0 + X0 R)64| <= u |X| + c u sqrt(NP) |X0||R|, R = fl32((I - L X0)64), and the
        result: |X - Lambda| <= u |X| + c u sqrt(NP) |X0||R| + |E0 L E0|, E0 = X0 - Lambda (exact Newton gives
        Lambda - E0 L E0; the rounding of R is one more u |X0||R|, inside c).  The largest ulp distance of X from
        fl32(Lambda) is printed.
   (c)  alpha and scal against the device's X as in 2., then alpha against the exact alpha_L = Lambda^T Lambda r of the
        fp32 factor, with the bound X's measured error E = X - Lambda implies:
        u |alpha| + 4 NP u64 S + |E|^T |X r| + |Lambda|^T |E||r|.
   (d)  against the fp64 GP (tests/util.py true_model): alpha and |L^-1 k| on eight kernel columns within
        max(1e-4, 2 F), F the error of torch's fp32 Cholesky and triangular solve on the same K (relative to the largest
        fp64 value); an fp32 factorisation that fails counts as F = inf.

4. After the jitter ladder: triplicated rows at sigma^2 ~ 1e-12, n = 600 (across a 512-column outer block of the
   Cholesky).  jitter_used is a rung 1e-6 10^k of the fp32 ladder, (a) - (c) hold against Khat64 + jitter I, and the
   rung below (jitter / 10, or 0 at 1e-6) really fails: hb_gram + hb_cholesky there report info > 0.

The fp64 references run on the device in torch float64; they are references, not the code under test."""
import ctypes as C
import json
import math

import numpy as np
import pytest
import torch

from hebo_b200 import _lib
from tests.util import (DEV, VARIANTS, WIDTHS, fit_model, gather_emb, kernel_parts, reset_hypers, true_model, warp_error)

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
U64 = 2.0 ** -53
C_MAX = 8.0
K_ABS = 3e-7                    # absolute accuracy of k stated in common.cuh
E_EX2 = 4.0                     # ex2.approx.ftz.f32: 2 ulp = 2^-22 relative, in units of u
E_RSQ = 2.0 ** -22.9 / U        # rsqrt.approx.f32: 2^-22.9 relative
FLUSH = 2.0 ** -102             # u FLUSH = 2^-126
GT = 128
F64 = torch.float64


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _ratio(err, B):
    """max err / B, an exact match counting 0 wherever B is 0 (B >= 0)."""
    if err.numel() == 0:
        return 0.0
    return float(torch.where(err == 0, torch.zeros_like(err), err / B).max())


def _excess(err, B0, B1):
    """The c of  err <= B0 + c B1:  max (err - B0)+ / B1."""
    if err.numel() == 0:
        return 0.0
    ex = (err - B0).clamp_min(0)
    return float(torch.where(ex == 0, torch.zeros_like(ex), ex / B1).max())


def _report(rep):
    print(json.dumps(rep))
    worst = max(rep["c_needed"].values())
    assert worst <= C_MAX, rep


# ---------------------------------------------------------------------------------------------------------------- kernel
def eps_k(r2, kind):
    """u eps_k / u: the error of kern_eval<KERN> at the fp32 r2 it receives, unit outputscale (docstring 1.)."""
    k, _, t, _ = kernel_parts(r2, kind)
    if kind == "rbf":
        return k * (E_EX2 + 1.25 * t) + FLUSH
    e = torch.exp(-t)
    if kind == "matern12":
        return k * (E_EX2 + 1.25 * t) + t * e * (E_RSQ + 1.5) + FLUSH
    if kind == "matern32":
        return k * (E_EX2 + 1.25 * t + 2) + t * t * e * (E_RSQ + 2.5) + FLUSH
    return k * (E_EX2 + 1.25 * t + 3.5) + t * (t + t * t / 3) * e * (E_RSQ + 2.5) + FLUSH


def gram_bound(r2, w, kind):
    """Absolute bound on |k32 - k64(r2)| of one unit-outputscale factor whose fp32 r2 sums w squared differences."""
    _, h, _, _ = kernel_parts(r2, kind)
    return 0.5 * h * (w + 2) * U * r2 + U * eps_k(r2, kind)


def sqdist64(Z):
    """fp64 direct-difference squared distances between the columns of Z [w, n] (fp64)."""
    n = Z.shape[1]
    out = torch.zeros(n, n, dtype=F64, device=DEV)
    for k in range(Z.shape[0]):
        out += (Z[k][:, None] - Z[k][None, :]) ** 2
    return out


def sqdist32_emulated(Z):
    """accum_sqdist's fp32 r2: df = fl(z_i - z_j), r2 = fma(df, df, r2) in feature order.  df^2 is exact in fp64, so
    the fma is r2 + df^2 rounded once to fp32 (a second rounding in fp64 first only matters on exact fp32 ties)."""
    Z = Z.float()
    n = Z.shape[1]
    out = torch.zeros(n, n, dtype=torch.float32, device=DEV)
    for k in range(Z.shape[0]):
        z = Z[k].double()
        df = (z[:, None] - z[None, :]).float().double()
        out = (out.double() + df * df).float()
    return out.double()


def k64(r2, kind):
    return kernel_parts(r2, kind)[0]


# ---------------------------------------------------------------------------------------------------------------- C ABI
def gram(Xt, n, hyp, kind, noise_diag=None, jitter=0.0):
    """hb_gram into a NaN-filled [NP, NP] matrix."""
    NP = Xt.shape[1]
    K = torch.full((NP, NP), float("nan"), device=DEV)
    st = _lib.lib().hb_gram(_p(Xt), n, Xt.shape[0], _p(hyp), _lib.KERNEL_IDS[kind], _p(noise_diag), float(jitter), _p(K),
                            _lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == _lib.HB_OK, st
    return K


def cholesky(K):
    """hb_cholesky in place; returns info."""
    NP = K.shape[0]
    ws = torch.empty(GT * GT, device=DEV)
    info = torch.zeros(1, dtype=torch.int32, device=DEV)
    st = _lib.lib().hb_cholesky(_p(K), NP, _p(ws), _p(info), _lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == _lib.HB_OK, st
    return int(info.item())


def tri_inverse(L):
    NP = L.shape[0]
    X = torch.full((NP, NP), float("nan"), device=DEV)
    tmp = torch.full((NP, NP), float("nan"), device=DEV)
    st = _lib.lib().hb_tri_inverse(_p(L), NP, _p(X), _p(tmp), _lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == _lib.HB_OK, st
    return X


def kinv(X):
    NP = X.shape[0]
    K = torch.full((NP, NP), float("nan"), device=DEV)
    st = _lib.lib().hb_kinv(_p(X), NP, _p(K), _lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == _lib.HB_OK, st
    return K


def solve_logdet(L, X, y, n, hyp):
    NP = L.shape[0]
    alpha = torch.full((NP,), float("nan"), device=DEV)
    scal = torch.full((2,), float("nan"), dtype=F64, device=DEV)
    ws = torch.full(((1 + NP // 64) * NP,), float("nan"), dtype=F64, device=DEV)
    st = _lib.lib().hb_solve_logdet(_p(L), _p(X), _p(y), n, NP, _p(hyp), _p(alpha), _p(scal), _p(ws), _lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == _lib.HB_OK, st
    return alpha, scal


# ---------------------------------------------------------------------------------------------------------------- checks
def lower_tiles(NP):
    i = torch.arange(NP, device=DEV)
    return (i[:, None] // GT) >= (i[None, :] // GT)


def check_tri_inverse(L, X):
    """c of the forward error and the right residual of X = hb_tri_inverse(L); strict upper exactly 0.  Returns
    (Lambda, L64, X64, c dict)."""
    NP = L.shape[0]
    L64 = L.double().tril()
    X64 = X.double()
    assert bool((X.triu(1) == 0).all()), "strict upper triangle of L^-1 not zero"
    I = torch.eye(NP, dtype=F64, device=DEV)
    Lam = torch.linalg.solve_triangular(L64, I, upper=False)
    sq = math.sqrt(NP)
    La, Xa, Lama = L64.abs(), X64.abs(), Lam.abs()
    P = Lama @ La @ Xa
    fwd = _ratio((X64 - Lam).abs(), U * sq * P)
    res = (X64 @ L64 - I).abs()
    info = dict(resid_c_of_XL=_ratio(res, U * sq * (Xa @ La)))
    return Lam, L64, X64, dict(tri_inverse_fwd=fwd, tri_inverse_resid=_ratio(res, U * sq * (P @ La))), info


def check_kinv(X64, Kinv):
    NP = X64.shape[0]
    low = lower_tiles(NP)
    assert bool(torch.isnan(Kinv[~low]).all()), "hb_kinv wrote an upper tile"
    ref = X64.t() @ X64
    B = U * math.sqrt(NP) * (X64.abs().t() @ X64.abs())
    return _ratio((Kinv.double() - ref).abs()[low], B[low])


def check_solve(L64, X64, y, c, n, alpha, scal):
    """c of alpha and scal against the closed form on the device's X (docstring 2.).  y [>= n] fp32, c fp32 scalar tensor."""
    NP = X64.shape[0]
    r = torch.zeros(NP, dtype=F64, device=DEV)
    r[:n] = (y[:n] - c).double()                       # fp32 subtraction, as gemv_rows_kernel
    v = X64 @ r
    a64 = X64.t() @ v
    Xr = X64.abs() @ r.abs()
    S = X64.abs().t() @ Xr
    assert bool((alpha[n:] == 0).all()), "alpha pad entries not zero"
    ca = _ratio((alpha[:n].double() - a64[:n]).abs(), U * a64[:n].abs() + 4 * NP * U64 * S[:n])
    q = (v[:n] * v[:n]).sum()
    Bq = 4 * NP * U64 * (v[:n].abs() * Xr[:n]).sum() + n * U64 * q
    lg = torch.log(L64.diagonal()[:n])
    ld = 2 * lg.sum()
    Bld = 4 * n * U64 * (lg.abs().sum() + 1)
    cq = float((scal[0] - q).abs() / Bq)
    cl = float((scal[1] - ld).abs() / Bld)
    rel = dict(quad_rel_err=float((scal[0] - q).abs() / q), logdet_abs_err=float((scal[1] - ld).abs()))
    return dict(alpha=ca, quad=cq, logdet=cl), v, r, S, rel


# ---------------------------------------------------------------------------------------------------------------- 1. Gram
GRAM_SHAPES = [(n, 33) for n in (5, 127, 128, 129, 511, 513, 4097)] + [(513, d) for d in (1, 31, 32, 300)]


def gram_inputs(n, d, seed):
    """Xt [d, NP] in [-1, 1] with NaN pad columns, rows 2 and n - 1 duplicating rows 1 and 0; lengthscales around
    0.6 sqrt(d) (r^2 ~ 1 between random rows, down to 0 between close ones)."""
    g = torch.Generator().manual_seed(seed)
    NP = int(_lib.lib().hb_padded_n(n))
    Xt = torch.full((d, NP), float("nan"))
    Xt[:, :n] = torch.rand(d, n, generator=g) * 2 - 1
    if n >= 5:
        Xt[:, 2] = Xt[:, 1]
        Xt[:, n - 1] = Xt[:, 0]
    ls = (torch.rand(d, generator=g) * 0.8 + 0.3) * math.sqrt(d)
    nd = (1e-3 * (1 + torch.rand(n, generator=g))).float()
    return Xt.float().to(DEV).contiguous(), ls.float(), nd.to(DEV)


@pytest.mark.parametrize("n,d", GRAM_SHAPES)
def test_gram_per_element(n, d):
    """hb_gram for the four kernels against k64 of the kernel's own fp32 features (docstring 1.)."""
    Xt, ls, nd = gram_inputs(n, d, seed=1000 * d + n)
    NP = Xt.shape[1]
    inv = (np.float32(1.0) / ls.numpy().astype(np.float32)).astype(np.float32)          # fl(1 / l), IEEE
    Z = (Xt[:, :n].cpu() * torch.from_numpy(inv)[:, None]).to(DEV)                       # fl(Xt fl(1 / l))
    r2 = sqdist64(Z.double())
    r2h = sqdist32_emulated(Z)
    tril = torch.ones(n, n, dtype=torch.bool, device=DEV).tril()
    offd = tril & ~torch.eye(n, dtype=torch.bool, device=DEV)
    i = torch.arange(NP, device=DEV)
    pad = ((i[:, None] >= n) | (i[None, :] >= n)) & (i[:, None] >= i[None, :])
    eye = torch.eye(NP, device=DEV)
    configs = [dict(s=1.0, sn2=1e-3, jitter=0.0, nd=None), dict(s=2.7, sn2=0.013, jitter=1e-5, nd=nd),
               dict(s=0.31, sn2=8e-4, jitter=1e-4, nd=None)]
    for kind in ("matern32", "matern52", "rbf", "matern12"):
        kk = k64(r2, kind)
        kh = k64(r2h, kind)
        worst_abs = 0.0
        c_eval = c_gram = 0.0
        for cf in configs:
            hyp = torch.tensor([cf["sn2"], 0.0, cf["s"]] + ls.tolist(), dtype=torch.float32, device=DEV)
            s = float(hyp[2])
            K = gram(Xt, n, hyp, kind, cf["nd"], cf["jitter"])
            Kd = K[:n, :n].double()
            # diagonal bit for bit, pad exact, duplicates = s
            s32, sn32, j32 = (torch.tensor(v, dtype=torch.float32, device=DEV) for v in (s, float(hyp[0]), cf["jitter"]))
            dg = (s32 + sn32) + j32
            dg = dg + cf["nd"] if cf["nd"] is not None else dg.expand(n)
            assert torch.equal(K.diagonal()[:n], dg), (kind, cf)
            assert torch.equal(K[pad], eye[pad]), (kind, cf, "pad")
            if n >= 5:
                assert float(K[2, 1]) == s and float(K[n - 1, 0]) == s, (kind, cf, "duplicates")
            err = (Kd - s * kk).abs()[offd]
            B = s * gram_bound(r2, d, kind)[offd] + U * Kd.abs()[offd]
            c_gram = max(c_gram, _ratio(err, B))
            if cf["s"] == 1.0:
                e_ev = (Kd - kh).abs()[offd]
                c_eval = max(c_eval, _ratio(e_ev, U * eps_k(r2h, kind)[offd]))
                worst_abs = max(worst_abs, float(e_ev.max()) if e_ev.numel() else 0.0)
        rep = dict(case=f"gram-{kind}-n{n}-d{d}", NP=NP, c_needed=dict(gram=c_gram, kern_eval=c_eval),
                   kern_eval_max_abs_err=worst_abs, k_abs_claim=K_ABS)
        _report(rep)
        assert worst_abs <= K_ABS, rep
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------- 2. stages
STAGE_NP = [128, 256, 384, 640, 1152, 2176, 4224]


def spd_factor(n, NP, cond, seed):
    """A Gram matrix (d = 2, Matern-3/2) through hb_gram + hb_cholesky; the ill-conditioned setting raises sigma^2
    tenfold from 1e-6 until the fp32 factorisation succeeds.  Returns (L [NP, NP] lower, hyp, sigma^2 used)."""
    g = torch.Generator().manual_seed(seed)
    Xt = torch.full((2, NP), float("nan"))
    Xt[:, :n] = torch.rand(2, n, generator=g) * 2 - 1
    Xt = Xt.to(DEV).contiguous()
    ls, sn2 = (0.5, 8e-4) if cond == "well" else (1.0, 1e-6)
    while True:
        hyp = torch.tensor([sn2, 0.3, 1.0, ls, ls], dtype=torch.float32, device=DEV)
        K = gram(Xt, n, hyp, "matern32")
        if cholesky(K) == 0:
            return K.tril(), hyp, sn2
        assert cond == "ill" and sn2 < 1e-2, (n, NP, cond, sn2)
        sn2 *= 10


def cond1(L64, Lam):
    return float(torch.linalg.matrix_norm(L64, ord=1) * torch.linalg.matrix_norm(Lam, ord=1))


@pytest.mark.parametrize("cond", ["well", "ill"])
@pytest.mark.parametrize("NP", STAGE_NP)
def test_simt_stages(NP, cond):
    """hb_tri_inverse, hb_kinv and hb_solve_logdet on their own (docstring 2.), n = NP and n = NP - 37."""
    for n in (NP, NP - 37):
        L, hyp, sn2 = spd_factor(n, NP, cond, seed=NP + (cond == "ill"))
        X = tri_inverse(L)
        Lam, L64, X64, c, info = check_tri_inverse(L, X)
        if n < NP:
            assert torch.equal(X[n:, n:], torch.eye(NP - n, device=DEV)) and bool((X[n:, :n] == 0).all())
        c["kinv"] = check_kinv(X64, kinv(X))
        y = torch.randn(n, generator=torch.Generator().manual_seed(n)).float().to(DEV)
        alpha, scal = solve_logdet(L, X, y, n, hyp)
        cs, _, _, _, rel = check_solve(L64, X64, y, hyp[1], n, alpha, scal)
        c.update(cs)
        _report(dict(case=f"stages-{cond}-NP{NP}-n{n}", sigma2=sn2, cond1_L=cond1(L64, Lam), c_needed=c, **info, **rel))
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------- 3. state
def khat64(gp, jitter):
    """Khat in fp64 on the state's own fp32 features, and the Gram bound B_gram (docstring 3.(a))."""
    n, d, De = gp.n, gp.d, gp.De
    hyp = gp.hyp_dev.double()
    sn2, s = float(hyp[0]), float(hyp[2])
    Z = gp.Zt_dev[:, :n].double()
    K = torch.full((n, n), s, dtype=F64, device=DEV)
    B = torch.zeros(n, n, dtype=F64, device=DEV)
    kn, bn = torch.ones_like(K), torch.zeros_like(K)
    if d:
        r2 = sqdist64(Z[:d])
        kn, bn = k64(r2, gp.kernel), gram_bound(r2, d, gp.kernel)
        del r2
    ke, be = torch.ones_like(K), torch.zeros_like(K)
    if De:
        r2e = sqdist64(Z[d:])
        ke, be = k64(r2e, "matern32"), gram_bound(r2e, De, "matern32")
        del r2e
    K = K * kn * ke
    B = s * (bn * ke + kn * be) + 2 * U * K.abs()
    diag = sn2 + jitter + (torch.as_tensor(gp.noise_diag).double().to(DEV) if gp.noise_diag is not None else 0.0)
    K.diagonal().fill_(s)
    K.diagonal().add_(diag)
    B.diagonal().copy_(3 * U * K.diagonal().abs())
    return K, B


def check_features(gp, rep):
    """(a') Zt and tab_s against their definitions."""
    n, d = gp.n, gp.d
    hyp = gp.hyp_dev
    if d:
        Zn = gp.Zt_dev[:d, :n]
        inv = torch.from_numpy((np.float32(1.0) / hyp[3:3 + d].cpu().numpy()).astype(np.float32)).to(DEV)
        Xt = gp._XtT[:, :n]
        if not gp.warp_mode:
            assert torch.equal(Zn, Xt * inv[:, None]), "numeric rows of Zt differ from fl(Xt fl(1/l))"
        else:
            from oracle import gp_oracle as O
            a = hyp[gp._h_wa:gp._h_wa + d].double()
            b = hyp[gp._h_wa + d:gp._h_wa + 2 * d].double()
            x = Xt.double().t()
            ls = hyp[3:3 + d].double()
            z64 = O.kumaraswamy_warp(x, a, b) / ls
            W = warp_error(x, x, a, b) / ls
            err = (Zn.double().t() - z64).abs()
            rep["c_needed"]["warp_rows"] = _ratio(err, U * (W + 2 * z64.abs()))
    if gp.num_enum:
        T = gp.T
        tables = gp._raw_dev[1:1 + T]
        inv_e = torch.tensor(np.float32(1.0) / np.float32(float(hyp[3 + d])), device=DEV)
        tab_s = tables * inv_e
        assert torch.equal(gp.tab_s_dev[:T], tab_s), "tab_s differs from fl(tables fl(1/l_e))"
        E = gather_emb(gp, gp._Xe_dev, tab_s).t()
        assert torch.equal(gp.Zt_dev[d:, :n], E), "embedding rows of Zt differ from the gathered scaled tables"


def check_state(name, gp, X, Xe, y, fp64=True):
    """3.(a) - (d) on the state the last factorisation left (docstring)."""
    n, NP = gp.n, gp.NP
    jitter = float(gp.jitter_used)
    rep = dict(case=name, n=n, NP=NP, d=gp.d, De=gp.De, jitter_used=jitter, c_needed={})
    check_features(gp, rep)
    # (a) L L^T against Khat64
    L = gp.L_dev.tril()
    L64 = L.double()
    i = torch.arange(NP, device=DEV)
    padrows = (i[:, None] >= n) & (i[:, None] >= i[None, :])
    assert torch.equal(L[padrows], torch.eye(NP, device=DEV)[padrows]), "pad of L is not the identity block"
    Kh, Bg = khat64(gp, jitter)
    Ln = L64[:n, :n]
    low = torch.ones(n, n, dtype=torch.bool, device=DEV).tril()
    err = (Ln @ Ln.t() - Kh).abs()[low]
    LL = (Ln.abs() @ Ln.abs().t())[low]
    rep["c_needed"]["LLt"] = _excess(err, Bg[low], U * math.sqrt(NP) * LL)
    del Kh, Bg, err, LL
    # (b) the refinement
    X0 = tri_inverse(gp.L_dev)
    Xd = gp.Linv_dev
    Lam, _, X064, cb, info = check_tri_inverse(L, X0)
    rep["c_needed"].update(cb)
    rep.update(info)
    X64 = Xd.double()
    assert bool((Xd.triu(1) == 0).all()), "strict upper triangle of the refined L^-1 not zero"
    I = torch.eye(NP, dtype=F64, device=DEV)
    R = (I - L64 @ X064).tril().float().double()
    Xref = X064 + X064 @ R
    B1 = U * math.sqrt(NP) * (X064.abs() @ R.abs())
    rep["c_needed"]["refine"] = _excess((X64 - Xref).abs(), U * X64.abs(), B1)
    E0 = X064 - Lam
    newton = (E0 @ L64 @ E0).abs()
    rep["c_needed"]["refined_vs_exact"] = _excess((X64 - Lam).abs(), U * X64.abs() + newton, B1)
    bits = lambda t: (lambda b: torch.where(b >= 0, b, -(b & 0x7FFFFFFF)))(t.contiguous().view(torch.int32).long())
    rep["max_ulp_refined"] = int((bits(Xd) - bits(Lam.float())).abs().max())
    rep["max_ulp_unrefined"] = int((bits(X0) - bits(Lam.float())).abs().max())
    rep["max_E0"] = float(E0.abs().max())
    rep["cond1_L"] = cond1(L64, Lam)
    del Xref, B1, R, newton, E0
    # (c) alpha / scal on the device's X, then against the exact alpha of the fp32 factor
    cs, v, r, S, rel = check_solve(L64, X64, gp._y_dev, gp.hyp_dev[1], n, gp.alpha_dev, gp.scal_dev)
    rep["c_needed"].update(cs)
    rep.update(rel)
    aL = Lam.t() @ (Lam @ r)
    E = (X64 - Lam).abs()
    Ba = U * aL.abs() + 4 * NP * U64 * S + E.t() @ v.abs() + Lam.abs().t() @ (E @ r.abs())
    rep["c_needed"]["alpha_vs_exact_L"] = _ratio((gp.alpha_dev.double() - aL).abs()[:n], Ba[:n])
    del E, Lam
    # (d) against the fp64 GP, with torch's fp32 solve on the same K as the evidence
    if fp64:
        tm = true_model(gp, X, Xe, y)
        K64 = tm["L"] @ tm["L"].t()
        K32 = K64.float()
        L32, info = torch.linalg.cholesky_ex(K32)
        ok32 = int(info) == 0
        rr = (y.double().reshape(-1).to(DEV) - float(gp.yscaler.mean[0])) / float(gp.yscaler.std[0]) - tm["c"]
        a64 = tm["alpha"]
        scale = float(a64.abs().max())
        e_dev = float((gp.alpha_dev[:n].double() - a64).abs().max()) / scale
        e_32 = float((torch.cholesky_solve(rr.float().reshape(-1, 1), L32).reshape(-1).double() - a64).abs().max()) / scale \
            if ok32 else math.inf
        cols = torch.linspace(0, n - 1, min(8, n), device=DEV).long()
        Kc = K64[:, cols].clone()
        Kc[cols, torch.arange(cols.numel(), device=DEV)] -= float(tm["hyp"][0])        # the noiseless kernel column
        if gp.noise_diag is not None:
            Kc[cols, torch.arange(cols.numel(), device=DEV)] -= torch.as_tensor(gp.noise_diag).double().to(DEV)[cols]
        v64 = torch.linalg.solve_triangular(tm["L"], Kc, upper=False).norm(dim=0)
        vdev = (X64[:n, :n] @ Kc.float().double()).norm(dim=0)
        e_vdev = float(((vdev - v64).abs() / v64.max()).max())
        e_v32 = float(((torch.linalg.solve_triangular(L32, Kc.float(), upper=False).double().norm(dim=0) - v64).abs()
                       / v64.max()).max()) if ok32 else math.inf
        rep.update(alpha_err=e_dev, alpha_fp32_reference_err=e_32, vnorm_err=e_vdev, vnorm_fp32_reference_err=e_v32)
        print(json.dumps(rep))
        assert e_dev <= max(1e-4, 2 * e_32), rep
        assert e_vdev <= max(1e-4, 2 * e_v32), rep
        del K64, K32, L32
    _report(rep)
    torch.cuda.empty_cache()
    return rep


def refactor(gp):
    """set_hypers at the fitted raw vector: the same state, with jitter_used recorded."""
    gp.set_hypers(gp.raw.clone())
    assert not gp._fit_failed


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_state_model_variants(variant):
    gp, X, Xe, y = fit_model(("variant", variant), 300, seed=7, **VARIANTS[variant])
    refactor(gp)
    check_state(f"state-{variant}", gp, X, Xe, y)


@pytest.mark.parametrize("width", list(WIDTHS))
def test_state_feature_widths(width):
    gp, X, Xe, y = fit_model(("width", width), 300, seed=11, **WIDTHS[width])
    refactor(gp)
    check_state(f"state-width-{width}", gp, X, Xe, y)


@pytest.mark.parametrize("n", [5, 129, 513, 1100, 2150, 4097])
def test_state_shapes(n):
    """Numeric Matern-3/2 models, d = 8 (the posterior tests' shape models), NP = 128 ... 4224."""
    gp, X, Xe, y = fit_model(("shape", n), n, 8, seed=n)
    refactor(gp)
    check_state(f"state-n{n}", gp, X, Xe, y)


@pytest.mark.parametrize("case", ["tiny-noise", "outputscale-1e3"])
def test_state_extremes(case):
    """sigma^2 at noise_lb = 1e-6 with lengthscales 0.4 (n = 513, NP = 640: a partial doubling pair), and outputscale 1e3."""
    if case == "tiny-noise":
        gp, X, Xe, y = fit_model(("fit-state", case), 513, 4, pred_likeli=False, epochs=2, noise_lb=1e-6, seed=3)
        reset_hypers(gp, noise=-30.0, ls=0.4)
    else:
        gp, X, Xe, y = fit_model(("fit-state", case), 300, 4, seed=21)
        reset_hypers(gp, os=1e3)
    check_state(f"state-{case}", gp, X, Xe, y)


# ---------------------------------------------------------------------------------------------------------------- 4. jitter
def test_state_after_the_jitter_ladder():
    """Triplicated rows at sigma^2 ~ 1e-12: the fp32 Khat fails at jitter 0 (docstring 4.)."""
    import hebo_b200
    g = torch.Generator().manual_seed(17)
    X = torch.randn(200, 2, generator=g)
    X = torch.cat([X, X, X], 0)
    y = torch.sin(X[:, :1])
    raw = torch.tensor([-40.0, 0.0, 0.5, 0.5, 0.5])
    gp = hebo_b200.GP(2, 0, 1, num_epochs=0, noise_lb=1e-12, init_raw=raw, pred_likeli=False)
    gp.fit(X, None, y)
    gp.set_hypers(raw)
    assert not gp._fit_failed and gp.n == 600 and gp.NP == 640
    ladder, j = [], np.float32(0.0)
    while j <= np.float32(1e3):
        j = np.float32(1e-6) if j == 0 else np.float32(j * np.float32(10.0))
        ladder.append(j)
    jit = np.float32(gp.jitter_used)
    assert jit in ladder, jit
    below = 0.0 if jit == ladder[0] else float(ladder[ladder.index(jit) - 1])
    K = gram(gp._XtT, gp.n, gp.hyp_dev, gp.kernel, None, below)
    info = cholesky(K)
    print(json.dumps(dict(case="jitter-ladder", jitter_used=float(jit), rung_below=below, info_below=info)))
    assert info > 0, "the rung below jitter_used factorises"
    check_state("state-jitter", gp, X, None, y, fp64=False)
