"""hb_posterior_grad_ex -- the differentiable GP.predict -- element by element against two fp64 references.

The chain under test is kstar_kernel<KERN, 0, EMB> (K* rows and the K* alpha partials, one per 512-column group),
rows_gemm_kernel<0> (V = K* Linv^T), rows_gemm_kernel<1> (W = V Linv) and post_grad_kernel<KERN, EMB>, run chunk by
chunk.  Every element of mu, var [m] and dmu, dvar [m, d] is checked:

  (a) against the closed form of posterior_grad.cu's header evaluated in fp64 on the GP's OWN fp32 state (Zt, alpha,
      Linv, hyp, tab_s), with the candidate features scaled in fp64 from the fp32 rows the kernel receives.  The accuracy
      of the fit drops out, so this isolates the kernel arithmetic:
          z*_k = (x_mul_k x_k + x_add_k) / l_k,  dz_ik = z*_k - z_ik,  r_i^2 = |dz_i|^2,  k*_i = s k(r_i^2) [k_e(r_e,i^2)]
          h_i with dk/dr^2 = -h/2 (times the embedding factor k_e), jac_k = x_mul_k / l_k,
          v = Linv k*,  w = Linv^T v,  mu~ = c + k*.alpha,  var~ = s - |v|^2 (+ sigma_n^2 with pred_likeli),
          dmu_k  =        y_std   sum_i alpha_i (-s h_i dz_ik) jac_k,
          dvar_k = -2     y_std^2 sum_i w_i     (-s h_i dz_ik) jac_k   (0 where a variance floor clamps),
      and |g - g64| <= c u B elementwise, u = 2^-24, with the probabilistic (square-root growth) rounding model
          B^mu_k  =   y_std   |jac_k| sqrt(n)  sum_i |alpha_i| s h^_i (|dz_ik| + |z*_k| + |z_ik|)
          B^var_k = 2 y_std^2 |jac_k| sqrt(NP) sum_i w^_i     s h^_i (|dz_ik| + |z*_k| + |z_ik|)
          B^mu    =   y_std (sqrt(n) sum_i |alpha_i| k^*_i + |c|) + |mu|
          B^var   =   y_std^2 (s (+ sigma_n^2) + sqrt(NP) |v| | |Linv| k^* |)
      where, term by term:
        - |dz_ik| + |z*_k| + |z_ik|: the fp32 candidate feature is rounded two or three times (scale, shift, 1 / l),
          an error of a few u |z*_k|; the difference adds u |dz_ik|; |z_ik| covers |z*_k| <= |dz_ik| + |z_ik| when the
          candidate sits far from the data;
        - h^_i = h_i (2 + |t_i| + g_i) and k^_i = k_i (2 + |t_i| + g_i): fast_exp (ex2.approx of t log2 e) is accurate to
          about (2 + |t|) u at exponent t (-a r for the Matern kernels, -r^2 / 2 for the RBF), and the rounding of r^2
          moves t by g_i u with g_i = a (|z*| + |z_i|) (rate r_i for the RBF); the embedding factor k_e of a mixed
          model carries the same terms for its own features (a = sqrt 3); s h^_i and s k^_i also get 2^-102 added,
          because fast_exp flushes results below u 2^-102 = 2^-126 to zero;
        - sqrt(n), sqrt(NP): the fp32 sums over the training points (the gradient sums, the K* alpha partials, |v|^2)
          and the two GEMMs over the NP padded columns;
        - w^ = |Linv|^T (|Linv| k^*): the rounding of V = K* Linv^T and of W = V Linv propagated to w;
        - |mu| and s: the final scaling by y_std (+ y_mean) and the O(s) kernel values.
      max |g - g64| / (u B) -- the c a case needs -- is printed for every case; c <= C_MAX is required.
  (b) against the fp64 GP at the same hyper-parameters (training features, K + sigma_n^2 I [+ noise_diag], Cholesky and
      alpha refactorised in fp64; a warp through oracle/gp_oracle.py's kumaraswamy_warp), differentiated by autograd
      through mu.sum() and var.sum() separately -- every row depends only on its own x, so these are the exact
      per-element Jacobians.  Per row r:  |g_r - g64_r|_inf <= 1e-4 max(|g64_r|_inf, 1e-2 max_r |g64_r|_inf);  mu within
      1e-4 max(|mu|, y_std) and sigma within 1e-4 relative (2e-4 on rows whose variance has cancelled below 0.02 s, the
      criteria of test_gpu_fullsize.py).  On those cancelled rows dvar is held to 1e-4 of the case's largest dvar row;
      reference (a) still checks them tightly.  Where the fit's own fp32 state is the limit, the same closed form run in
      fp32 on that state is the evidence: its largest error under the same scaling, F, is printed next to the GPU's,
      and the criterion is max(1e-4, 2 F), as in test_gpu_parity.py, but never above 2e-2; the rows above 1e-4 are
      counted.  Random rows in hundreds of dimensions are uncorrelated with the data and have no gradient to speak of,
      so the wide models are probed next to their training rows.

The GPU values reach (b) through GP.predict with requires_grad (a learned or fixed warp chained in torch in front of the
kernel, as GP._predict_autograd does) and reach (a) through the C ABI.  Structure: sentinels past m and m d stay
untouched, repeated calls and every m_chunk give the same bytes, duplicate rows give identical rows, and GP.predict's
mu with requires_grad equals plain GP.predict's mu bit for bit.

The fp64 references run on the device in torch float64; they are references, not the code under test."""
import ctypes as C
import json
import math

import numpy as np
import pytest
import torch

from hebo_b200 import _lib
from hebo_b200.scalers import kumaraswamy_warp
from oracle import gp_oracle as O
from tests.util import (DEV, RATE, VARIANTS, WIDTHS, candidates, features64, fit_model, gather_emb, kernel_parts, kmat64,
                        true_model)

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C_MAX = 6.0             # the c of reference (a); the cases below need at most 1.7 on an H100
CANCEL = 0.02           # sigma^2 / s below which the variance is cancellation residue (test_gpu_fullsize.py)
EPS32 = float(np.finfo(np.float32).eps)
SENTINEL = -777.25
TAIL = 257
FLUSH = 2.0 ** -102     # u FLUSH = 2^-126: fast_exp flushes results below it to zero


# ---------------------------------------------------------------------------------------------------------------- models
def shape_model(n):
    """Numeric Matern-3/2 model, d = 8, with pred_likeli (the default of GP)."""
    return fit_model(("shape", n), n, 8, seed=n)


def kernel_inputs(gp, Xs):
    """(Xin, x_mul, x_add) as GP._predict_autograd hands them to the kernel: with a warp, Xin = the warped MinMax-scaled
    rows and x_mul = 1, x_add = 0."""
    if gp.warp_mode:
        d, h = gp.d, gp._h_wa
        Xin = kumaraswamy_warp(Xs * gp._x_mul + gp._x_add, gp.hyp_dev[h:h + d], gp.hyp_dev[h + d:h + 2 * d])
        return Xin.contiguous(), torch.ones_like(gp._x_mul), torch.zeros_like(gp._x_add)
    return Xs, gp._x_mul, gp._x_add


# ---------------------------------------------------------------------------------------------------------------- C ABI
def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def call_grad(gp, Xin, Xe, x_mul, x_add, m_chunk=None, y_std=None, null_spec=False):
    """(mu, var, dmu, dvar) of one hb_posterior_grad_ex call; the workspace starts out as NaN, and sentinels past m and
    m d must survive."""
    lib = _lib.lib()
    m, d = Xin.shape[0], gp.d
    mc = m if m_chunk is None else m_chunk
    ws = torch.full((int(lib.hb_posterior_workspace_bytes(gp.n, d, mc)) // 4,), float("nan"), device=DEV)
    outs = [torch.full((k + TAIL,), SENTINEL, device=DEV) for k in (m, m, m * d, m * d)]
    mu, var, dmu, dvar = outs
    ys = gp._y_std if y_std is None else y_std
    if null_spec:
        st = lib.hb_posterior_grad(_ptr(Xin), m, gp.n, d, _ptr(x_mul), _ptr(x_add), _ptr(gp.Zt_dev), _ptr(gp.alpha_dev),
                                   _ptr(gp.Linv_dev), _ptr(gp.hyp_dev), gp.kern_id, gp._y_mean, float(ys), int(bool(gp.pred_likeli)),
                                   _ptr(mu), _ptr(var), _ptr(dmu), _ptr(dvar), _ptr(ws), ws.numel() * 4, mc, _lib.stream_ptr())
    else:
        st = lib.hb_posterior_grad_ex(_ptr(Xin), _ptr(Xe), m, gp.n, d, C.byref(gp._spec_nowarp),
                                      _ptr(gp._emb_meta_dev) if gp.num_enum else None, _ptr(gp.tab_s_dev) if gp.num_enum else None,
                                      _ptr(x_mul), _ptr(x_add), _ptr(gp.Zt_dev), _ptr(gp.alpha_dev), _ptr(gp.Linv_dev),
                                      _ptr(gp.hyp_dev), gp.kern_id, gp._y_mean, float(ys), int(bool(gp.pred_likeli)), _ptr(mu),
                                      _ptr(var), _ptr(dmu), _ptr(dvar), _ptr(ws), ws.numel() * 4, mc, _lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == _lib.HB_OK, st
    for t in outs:
        assert bool((t[-TAIL:] == SENTINEL).all()), "hb_posterior_grad_ex wrote past its outputs"
    return mu[:m], var[:m], dmu[:m * d].view(m, d), dvar[:m * d].view(m, d)


def gp_path(gp, Xs, Xe):
    """GP.predict with requires_grad: (mu, var, d mu.sum() / dx, d var.sum() / dx); also checks that the two forward
    calls agree bit for bit and that, without a warp, mu equals plain GP.predict's."""
    xa = Xs.clone().requires_grad_(True)
    mu, var = gp.predict(xa, Xe)
    mu.sum().backward()
    xb = Xs.clone().requires_grad_(True)
    mu2, var2 = gp.predict(xb, Xe)
    var2.sum().backward()
    assert torch.equal(mu, mu2) and torch.equal(var, var2)
    if not gp.warp_mode:       # (a warp runs in torch in front of the gradient path, fused into K* in plain predict)
        with torch.no_grad():
            mu_p, _ = gp.predict(Xs, Xe)
        assert torch.equal(mu.detach(), mu_p), "GP.predict's mu depends on requires_grad"
    return mu.detach().reshape(-1), var.detach().reshape(-1), xa.grad, xb.grad


# ---------------------------------------------------------------------------------------------------------------- (a) own state
def own_state(gp, Xin, Xe, x_mul, x_add, y_std=None, dtype=torch.float64, bounds=True):
    """The closed form of the module docstring on the GP's own fp32 state, in `dtype`, with the bounds B in fp64."""
    dt = dtype
    n, d, NP = gp.n, gp.d, gp.NP
    ys = float(gp._y_std if y_std is None else y_std)
    hyp = gp.hyp_dev.to(dt)
    sn2, c, s = hyp[0], hyp[1], hyp[2]
    pl = sn2 if gp.pred_likeli else torch.zeros((), dtype=dt, device=DEV)
    ls = hyp[3:3 + d]
    jac = x_mul.to(dt) / ls
    zc = (x_mul.to(dt) * Xin.to(dt) + x_add.to(dt)) / ls
    Zn = gp.Zt_dev[:d, :n].to(dt).t()
    emb = gp.num_enum > 0
    if emb:
        zce = gather_emb(gp, Xe, gp.tab_s_dev.to(dt))
        Ze = gp.Zt_dev[d:, :n].to(dt).t()
    L = gp.Linv_dev[:n, :n].to(dt).tril()
    alpha = gp.alpha_dev[:n].to(dt)
    m = Xin.shape[0]
    out = {k: [] for k in ("mu", "var", "dmu", "dvar", "raw_var", "Bmu", "Bvar", "Bdmu", "Bdvar")}
    blk = max(1, (1 << 24) // (n * (d + gp.De)))
    for r0 in range(0, m, blk):
        z = zc[r0:r0 + blk]
        Dz = z[:, None, :] - Zn[None]
        r2 = (Dz * Dz).sum(-1)
        k, h, t, rate = kernel_parts(r2, gp.kernel)
        zn = z.norm(dim=1)[:, None] + Zn.norm(dim=1)[None]
        grow = 2 + t + rate * zn
        if emb:
            ze = zce[r0:r0 + blk]
            De = ze[:, None, :] - Ze[None]
            ke, _, te, _ = kernel_parts((De * De).sum(-1), "matern32")
            keh = ke * (2 + te + math.sqrt(3.0) * (ze.norm(dim=1)[:, None] + Ze.norm(dim=1)[None]))
        else:
            ke = keh = torch.ones_like(k)
        ks = s * k * ke
        H = s * h * ke
        V = ks @ L.t()
        W = V @ L
        mu_t = ks @ alpha + c
        raw_var = s - (V * V).sum(1) + pl
        dmu = ys * jac * torch.einsum("bn,bnd->bd", -alpha[None] * H, Dz)
        dvr = (ys * ys) * jac * torch.einsum("bn,bnd->bd", 2.0 * W * H, Dz)     # -2 sum_i w_i (-s h_i dz_ik)
        ps2_raw = raw_var.clamp_min(1e-6) * (ys * ys)
        live = (raw_var > 1e-6) & (ps2_raw > EPS32)
        out["mu"].append(mu_t * ys + gp._y_mean)
        out["var"].append(ps2_raw.clamp_min(EPS32))
        out["dmu"].append(dmu)
        out["dvar"].append(torch.where(live[:, None], dvr, torch.zeros_like(dvr)))
        out["raw_var"].append(raw_var)
        if bounds:
            Hh = (s * h * grow + FLUSH) * keh
            khat = (s * k * grow + FLUSH) * keh
            T = Dz.abs() + z.abs()[:, None, :] + Zn.abs()[None]
            La = L.abs()
            Lk = khat @ La.t()
            what = Lk @ La
            out["Bdmu"].append(ys * jac.abs() * math.sqrt(n) * torch.einsum("bn,bnd->bd", alpha.abs()[None] * Hh, T))
            out["Bdvar"].append(2 * ys * ys * jac.abs() * math.sqrt(NP) * torch.einsum("bn,bnd->bd", what * Hh, T))
            out["Bmu"].append(ys * (math.sqrt(n) * (khat @ alpha.abs()) + c.abs()) + (mu_t * ys + gp._y_mean).abs())
            out["Bvar"].append(ys * ys * (s + pl + math.sqrt(NP) * V.norm(dim=1) * Lk.norm(dim=1)))
    return {k: torch.cat(v) for k, v in out.items() if v}


def _ratio(got, ref, B):
    """max |got - ref| / (u B), an exact match counting 0 wherever B is 0."""
    err = (got - ref).abs()
    return float(torch.where(err == 0, torch.zeros_like(err), err / (U * B)).max())


def check_own_state(name, gp, Xin, Xe, x_mul, x_add, got, y_std=None):
    """Reference (a): the c each output needs; asserts c <= C_MAX.  dvar rows whose floor decision is within the
    bound of the variance are left out (either side of the floor is right there)."""
    ref = own_state(gp, Xin, Xe, x_mul, x_add, y_std)
    mu, var, dmu, dvar = (t.double() for t in got)
    ys = float(gp._y_std if y_std is None else y_std)
    vb = ref["Bvar"] / (ys * ys)
    amb = ((ref["raw_var"] - 1e-6).abs() <= 4 * C_MAX * U * vb) | \
          ((ref["raw_var"].clamp_min(1e-6) * ys * ys - EPS32).abs() <= 4 * C_MAX * U * ref["Bvar"])
    c = dict(mu=_ratio(mu, ref["mu"], ref["Bmu"]), var=_ratio(var, ref["var"], ref["Bvar"]),
             dmu=_ratio(dmu, ref["dmu"], ref["Bdmu"]),
             dvar=_ratio(dvar[~amb], ref["dvar"][~amb], ref["Bdvar"][~amb]) if bool((~amb).any()) else 0.0)
    rep = dict(case=name, ref="own_state", n=gp.n, NP=gp.NP, m=Xin.shape[0], d=gp.d, De=gp.De, c_needed=c,
               c_max_case=max(c.values()), ambiguous_rows=int(amb.sum()))
    print(json.dumps(rep))
    assert max(c.values()) <= C_MAX, rep
    return ref


# ---------------------------------------------------------------------------------------------------------------- (b) fp64 GP
def oracle_grad(gp, tm, Xs, Xe):
    """fp64 (mu, var, raw variance, dmu, dvar) of the candidates in original y units, by autograd."""
    hyp = tm["hyp"]
    s, sn2 = float(hyp[2]), float(hyp[0])
    X = Xs.double().clone().requires_grad_(True)
    Zc = features64(gp, X, Xe, hyp, tm["tables"])
    Ks = kmat64(gp, Zc, tm["Zt"], s)
    mu_t = tm["c"] + Ks @ tm["alpha"]
    Vt = torch.linalg.solve_triangular(tm["L"], Ks.t(), upper=False)
    raw = s - (Vt * Vt).sum(0) + (sn2 if gp.pred_likeli else 0.0)
    ys, ym = gp._y_std, gp._y_mean
    mu = mu_t * ys + ym
    var = (raw.clamp_min(1e-6) * ys * ys).clamp_min(EPS32)
    (gmu,) = torch.autograd.grad(mu.sum(), X, retain_graph=True)
    (gvar,) = torch.autograd.grad(var.sum(), X)
    return mu.detach(), var.detach(), raw.detach(), gmu, gvar


def check_fp64(name, gp, tm, Xs, Xe, got, g32):
    """Reference (b), per row; g32 = the fp32 closed form's (dmu, dvar) on the same state, the evidence for rows where
    the fit's fp32 state limits the result."""
    mu64, var64, raw64, gmu64, gvar64 = oracle_grad(gp, tm, Xs, Xe)
    mu, var, dmu, dvar = (t.double() for t in got)
    ys, s = gp._y_std, float(tm["hyp"][2])
    emu = ((mu - mu64).abs() / mu64.abs().clamp_min(ys))
    esg = (var.sqrt() - var64.sqrt()).abs() / var64.sqrt()
    canc = raw64 < CANCEL * s
    rep = dict(case=name, ref="fp64", m=Xs.shape[0], mu_err=float(emu.max()),
               sigma_err_regular=float(esg[~canc].max()) if bool((~canc).any()) else 0.0,
               sigma_err_cancelled=float(esg[canc].max()) if bool(canc.any()) else 0.0, rows_cancelled=int(canc.sum()))
    assert rep["mu_err"] <= 1e-4 and rep["sigma_err_regular"] <= 1e-4 and rep["sigma_err_cancelled"] <= 2e-4, rep
    for what, g, g64, e32 in (("dmu", dmu, gmu64, g32[0]), ("dvar", dvar, gvar64, g32[1])):
        err = (g - g64).abs().amax(1)
        nrm = g64.abs().amax(1)
        top = float(nrm.max())
        scale = torch.maximum(nrm, torch.full_like(nrm, 1e-2 * top))
        if what == "dvar":
            scale = torch.where(canc, torch.full_like(scale, top), scale)
        rel = err / scale
        floor32 = float(((e32.double() - g64).abs().amax(1) / scale).max())
        crit = max(1e-4, min(2 * floor32, 2e-2))
        rep[f"{what}_row_err"] = float(rel.max())
        rep[f"{what}_fp32_reference_err"] = floor32
        rep[f"{what}_rows_over_1e-4"] = int((rel > 1e-4).sum())
        bad = rel > crit
        assert not bool(bad.any()), (name, what, rep, torch.nonzero(bad)[:5].tolist())
    print(json.dumps(rep))
    return rep


def fp32_evidence(gp, Xs, Xe):
    """The closed form in fp32 on the GP's state, chained through the warp Jacobian in fp64 (gradients w.r.t. the raw
    rows, like reference (b))."""
    Xin, x_mul, x_add = kernel_inputs(gp, Xs)
    r = own_state(gp, Xin, Xe, x_mul, x_add, dtype=torch.float32, bounds=False)
    J = torch.ones(Xs.shape, dtype=torch.float64, device=DEV)
    if gp.warp_mode:
        X = Xs.double().clone().requires_grad_(True)
        d, h = gp.d, gp._h_wa
        hyp = gp.hyp_dev.double()
        w = O.kumaraswamy_warp(gp._x_mul.double() * X + gp._x_add.double(), hyp[h:h + d], hyp[h + d:h + 2 * d])
        (J,) = torch.autograd.grad(w.sum(), X)
    return r["dmu"].double() * J, r["dvar"].double() * J


# ---------------------------------------------------------------------------------------------------------------- one case
def check_case(name, gp, X, Xe_train, y, Xs, Xse, dups=(), fp64=True):
    """ABI against (a); GP.predict with requires_grad against (b); duplicates; the warp clamp's exact zeros."""
    Xin, x_mul, x_add = kernel_inputs(gp, Xs)
    got = call_grad(gp, Xin, Xse, x_mul, x_add)
    for t in got:
        assert bool(torch.isfinite(t).all())
    for s_, t_ in dups:
        for t in got:
            assert torch.equal(t[s_], t[t_]), ("duplicate rows differ", s_, t_)
    ref = check_own_state(name, gp, Xin, Xse, x_mul, x_add, got)
    mu_g, var_g, gmu, gvar = gp_path(gp, Xs, Xse)
    if not gp.warp_mode:       # the same kernel chain on the same rows: the same bytes whatever the chunking
        assert torch.equal(mu_g, got[0]) and torch.equal(var_g, got[1])
        assert torch.equal(gmu, got[2]) and torch.equal(gvar, got[3])
    else:                      # rows outside the box: the warp's clamp has exactly zero gradient
        t = Xs * gp._x_mul + gp._x_add
        out = (t < -1.0001) | (t > 1.0001)
        assert bool(out.any())
        assert bool((gmu[out] == 0).all()) and bool((gvar[out] == 0).all())
    rep = None
    if fp64:
        rep = check_fp64(name, gp, true_model(gp, X, Xe_train, y), Xs, Xse, (mu_g, var_g, gmu, gvar), fp32_evidence(gp, Xs, Xse))
    return got, ref, rep


# ---------------------------------------------------------------------------------------------------------------- tests
SHAPE_N = [5, 127, 128, 129, 511, 512, 513, 1100, 4224]


@pytest.mark.parametrize("n", SHAPE_N)
def test_gradients_across_kstar_groups(n):
    """NP = 128 ... 4224: one to nine 512-column K* groups (ncg = 2 from n = 513), the 128-wide GEMM tiles either side of
    n, m = 129 rows (two row tiles) and m = 300 at the largest n."""
    gp, X, Xe, y = shape_model(n)
    Xs, Xse, dups = candidates(gp, X, Xe, 300 if n == 4224 else 129, seed=n + 1)
    check_case(f"shape-n{n}", gp, X, Xe, y, Xs, Xse, dups)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("m", [1, 129, 1024, 1025, 2500])
def test_gradients_through_gp_chunks(m):
    """GP._posterior_grad chunks at 1024 rows: m = 1025 and 2500 run two and three chunks (the Xs + c0 d offsets of K*,
    the global row of post_grad_kernel and the reuse of the workspace), at ncg = 2."""
    gp, X, Xe, y = shape_model(513)
    Xs, Xse, dups = candidates(gp, X, Xe, m, seed=m + 7)
    check_case(f"gp-chunks-m{m}", gp, X, Xe, y, Xs, Xse, dups)
    torch.cuda.empty_cache()


def variant_model(name):
    conf = dict(VARIANTS[name])
    return fit_model(("variant", name), 300, seed=7, **conf)


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_gradients_model_variants(variant):
    """Each kernel with pred_likeli on and off, mixed models (the EMB instance) with one, two and six categorical columns,
    ard_kernel=False, heteroscedastic noise, learned and fixed warps (chained in torch in front of the kernel)."""
    gp, X, Xe, y = variant_model(variant)
    if variant == "wide_embeddings":
        assert gp.De == 300
    Xs, Xse, dups = candidates(gp, X, Xe, 200, seed=200, near=variant == "wide_embeddings")
    check_case(variant, gp, X, Xe, y, Xs, Xse, dups)


@pytest.mark.parametrize("width", list(WIDTHS))
def test_gradients_feature_widths(width):
    """d = 1, 33 (across kstar_kernel's 32-wide feature chunk), 300, and d + De = 4096; from d = 300 on, random rows
    are uncorrelated with the data, so the rows there sit next to training rows."""
    conf = dict(WIDTHS[width])
    gp, X, Xe, y = fit_model(("width", width), 300, seed=11, **conf)
    Xs, Xse, dups = candidates(gp, X, Xe, 64 if width == 4096 else 100, seed=width, near=width >= 300)
    check_case(f"width-{width}", gp, X, Xe, y, Xs, Xse, dups)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("kind", ["numeric", "mixed"])
def test_m_chunk_gives_the_same_bytes(kind):
    """Every row is computed on its own, so any m_chunk -- 1, 7, 128, 129, 1000 against one chunk of 1300 rows -- gives
    the same bytes, and so does a second call.  The numeric model's NULL-spec entry hb_posterior_grad equals _ex."""
    gp, X, Xe, y = shape_model(1100) if kind == "numeric" else variant_model("mixed_e2")
    Xs, Xse, _ = candidates(gp, X, Xe, 1300, seed=77)
    Xin, x_mul, x_add = kernel_inputs(gp, Xs)
    one = call_grad(gp, Xin, Xse, x_mul, x_add)
    for mc in (None, 1, 7, 128, 129, 1000):
        got = call_grad(gp, Xin, Xse, x_mul, x_add, m_chunk=mc)
        for a, b in zip(one, got):
            assert torch.equal(a, b), mc
    if kind == "numeric":
        for a, b in zip(one, call_grad(gp, Xin, Xse, x_mul, x_add, m_chunk=129, null_spec=True)):
            assert torch.equal(a, b)
    check_own_state(f"m_chunk-{kind}", gp, Xin, Xse, x_mul, x_add, one)


def test_variance_floor_zeroes_dvar():
    """Rows within 1e-6 (raw units) of training rows, at a noise of 1e-9 and short lengthscales: the variance is under
    gpytorch's 1e-6 floor, so var is the floor exactly and dvar is exactly 0, while dmu is still checked.  Random rows of
    the same batch stay live."""
    gp, X, Xe, y = fit_model("floor", 129, 4, pred_likeli=False, epochs=2, noise_lb=1e-9)
    raw = gp.raw.clone()
    raw[0] = -30.0                                               # sigma_n^2 = noise_lb + softplus(-30)
    raw[3:3 + gp.d] = float(O.inv_softplus(torch.tensor(0.05, dtype=torch.float64)))
    gp.set_hypers(raw)
    assert not gp._fit_failed
    g = torch.Generator().manual_seed(3)
    near = X[:40] + 1e-6 * (torch.rand(40, gp.d, generator=g) * 2 - 1)
    far = torch.rand(40, gp.d, generator=g) * 2 - 1
    Xs = torch.cat([near, far]).float().to(DEV).contiguous()
    got, ref, _ = check_case("variance-floor", gp, X, Xe, y, Xs, None)
    dead = ref["raw_var"] < 0.5e-6
    assert int(dead.sum()) >= 30 and int((~dead).sum()) >= 30, int(dead.sum())
    ys2 = np.float32(gp._y_std) * np.float32(gp._y_std)
    floor = float(max(np.float32(1e-6) * ys2, np.float32(EPS32)))
    assert bool((got[3][dead] == 0).all()) and bool((got[1][dead] == floor).all())
    assert bool((got[2][dead] != 0).any())
    assert bool((got[3][~dead] != 0).any())


def test_flt_epsilon_floor_zeroes_dvar():
    """A y_std so small that y_std^2 var~ crosses FLT_EPSILON inside the batch: var = FLT_EPSILON and dvar = 0 exactly on
    the rows under it, the live rows checked against reference (a) at that y_std."""
    gp, X, Xe, y = shape_model(129)
    s = float(gp.hyp[2])
    ys = math.sqrt(2 * EPS32 / s)
    Xs, Xse, _ = candidates(gp, X, Xe, 129, seed=5)
    Xin, x_mul, x_add = kernel_inputs(gp, Xs)
    got = call_grad(gp, Xin, Xse, x_mul, x_add, y_std=ys)
    ref = check_own_state("flt-epsilon-floor", gp, Xin, Xse, x_mul, x_add, got, y_std=ys)
    ps2 = ref["raw_var"].clamp_min(1e-6) * ys * ys
    dead, live = ps2 < 0.9 * EPS32, ps2 > 1.1 * EPS32
    assert int(dead.sum()) >= 5 and int(live.sum()) >= 5, (int(dead.sum()), int(live.sum()))
    assert bool((got[3][dead] == 0).all()) and bool((got[1][dead] == EPS32).all())
    assert bool((got[3][live] != 0).any())
