"""hb_posterior_mace_ex -- GP.predict and every MACE / GA / NSGA-II score -- element by element against two fp64 references.

The chain under test runs chunk by chunk: kstar_kernel<KERN, SPLIT, EMB> (K* rows with the input warp fused into the
feature load, and the K* alpha partials), then the contraction |v|^2 = |Linv k*|^2, either on the tensor cores
(vnorm_h16_kernel: two-level fp16 operands, 4-CTA clusters over a band-major schedule, the precision guard
guard_kernel + vnorm_fix_kernel re-contracting rows with s - |v|^2 < 0.12 s on the FP32 pipe) or on the FP32 SIMT pipe
(vnorm_kernel, Linv_hi = Linv_lo = NULL), then mace_kernel (floors, un-scaling, MACE).  Every element of mu and var [m]
is checked on both paths:

  (a) against the closed form in fp64 on the GP's OWN fp32 state (Zt, alpha, Linv, hyp, tab_s), with the candidate
      features scaled -- and warped -- in fp64 from the fp32 rows the kernel receives:
          z*_k = w_k(x_mul_k x_k + x_add_k) / l_k,  r_i^2 = |z* - z_i|^2,  k*_i = s k(r_i^2) [k_e(r_e,i^2)],  v = Linv k*,
          mu = y_std (c + k*.alpha) + y_mean,  var = max(max(s - |v|^2 (+ sigma_n^2), 1e-6) y_std^2, FLT_EPSILON),
      and |g - g64| <= c u B elementwise, u = 2^-24, with
          B^mu  = y_std (sqrt(n) sum_i |alpha_i| k^_i + |c|) + |mu|
          B^var = y_std^2 (s (+ sigma_n^2) + sqrt(NP) |v| | |Linv| k^ |)                         (SIMT path)
          B^var = y_std^2 (s (+ sigma_n^2) + 10 |v| | |Linv| k^ | + sqrt(NP / 128) |v|^2)         (guarded rows)
          B^var = SIMT B^var + y_std^2 2 sum_c |v_c| T_c                                          (tensor path, unguarded)
          T_c   = (3 S + 2 q_c) (|Linv| |k*|)_c + 2^-20 max|Linv| |k*|_1 + 2^-11 s |Linv_c|_1
      where, term by term:
        - k^_i = s k_i (2 + |t_i| + g_i) (+ 2^-102) [x the same for k_e]: fast_exp (ex2.approx) is accurate to about
          (2 + |t|) u at exponent t; the rounding of the features moves t by g_i u with g_i = a (|z*| + |z_i| + |W / l|)
          (rate a: sqrt 3 / sqrt 5 for the Matern kernels, r_i for the RBF).  W_k is the fp32 error of the fused warp
          in units of u, propagated step by step through kumar_warp (common.cuh): the relative error of
          u = (x_t + 1) / 2 (the scaling's two roundings and the shift; 1 where the clamp is active), then
          log u (+ 2 |log u| + 1), x = a log u (a x that + |x|, absolute), log(1 - u^a) = log(-expm1(x))
          (u^a / (1 - u^a) x that + 2 |log(1 - u^a)| + 3), p = (1 - u^a)^b (b x that + |b log(1 - u^a)| + 2, relative) and
          2 (1 - p) - 1
          (2 p x that + 2 |1 - p| + |w|); 0 without a warp;
        - sqrt(n), sqrt(NP): the fp32 sums over the training points (the K* alpha partials) and over the NP padded
          columns of the SIMT contraction (square-root growth, as in test_gpu_posterior_grad.py); |mu| and s: the final
          scaling by y_std (+ y_mean) and s - |v|^2;
        - guarded rows: exact fp32 K* rows and fp32 Linv, fp32 partials of 16 products summed in fp64 per tile (2 x
          (1 + 4) |v| | |Linv| k^ |), then one fp32 value per 128-column tile summed in fp32 (sqrt(NP / 128) |v|^2);
        - tensor path: S = 2^-22 / u = 4 for each of the three operand errors of the split (h0 + h1 / 2048 represents each
          operand to 2^-22 relative, and h1 h1 is dropped); q_c = min(128 (J + 1), NP) / 16 accumulate steps of the
          wgmma K = 16 MMAs over column c's k range (c in column tile J), each a truncation of up to one ulp (2 u) of the
          accumulator, so the growth is LINEAR in q_c; the 2^-20 and 2^-11 terms are the fp16 subnormal floors of the
          split (absolute 2^-45 max|Linv| on Linv, 2^-36 s on K*).
      Rows the guard may or may not flag (|s - |v|^2 - 0.12 s| within the bound) get the larger of the two bounds.
      max |g - g64| / (u B) -- the c a case needs -- is printed for every case and path; c <= C_MAX is required.
  (b) against the fp64 GP refactorised at the same hyper-parameters (tests/util.py true_model), per row: mu within
      1e-4 max(|mu|, y_std) and sigma within 1e-4 relative (2e-4 on rows whose variance has cancelled below 0.02 s).
      Where the fit's own fp32 state is the limit, the same closed form run in fp32 on that state is the evidence: its
      largest error F is printed next to the GPU's and the criterion is max(1e-4, 2 F), never above 2e-2.

Invariants: m_chunk leaves every byte of mu, var and F unchanged on both paths, and so does a second call; mu is the
same on both paths (the same fp32 K* feeds both); F equals hb_mace_epilogue on the call's own mu and var, with
noise_var = fl(sigma_n^2 fl(y_std^2)) as mace_kernel forms it; rng_offset makes calls over row ranges draw what one
call draws; GP.predict (device rows and a pinned host batch larger than a chunk) equals the ABI call bit for bit.
The L^-1 operand split is compared with its definition bit for bit.

The fp64 references run on the device in torch float64; they are references, not the code under test."""
import ctypes as C
import json
import math

import numpy as np
import pytest
import torch

from hebo_b200 import _lib
from oracle import gp_oracle as O
from tests.util import (DEV, VARIANTS, WIDTHS, candidates, features64, fit_model, gather_emb, kernel_parts, kmat64,
                        true_model, warp_error)
from tests.util import reset_hypers as _set

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C_MAX = 8.0             # the c of reference (a)
CANCEL = 0.02           # sigma^2 / s below which the variance is cancellation residue (test_gpu_fullsize.py)
EPS32 = float(np.finfo(np.float32).eps)
SENTINEL = -777.25
TAIL = 257
FLUSH = 2.0 ** -102     # u FLUSH = 2^-126: fast_exp flushes results below it to zero
SPLIT = 2.0 ** -22 / U  # operand representation error of the two-level fp16 split, in units of u
THETA = 0.12            # GUARD_THETA of posterior.cu
KSTEP = 16              # products per wgmma f16 accumulate step
CT = 128                # column tile of the contractions
PATHS = ("tensor", "simt")


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _off(t, row0, w=1):
    return None if t is None else C.c_void_p(t.data_ptr() + row0 * w * 4)


def shape_model(n):
    """Numeric Matern-3/2 model, d = 8, with pred_likeli (the default of GP); the same models as the gradient test."""
    return fit_model(("shape", n), n, 8, seed=n)


def variant_model(name):
    return fit_model(("variant", name), 300, seed=7, **VARIANTS[name])


# ---------------------------------------------------------------------------------------------------------------- C ABI
def abi(gp, Xs, Xe, rows, row0, path, F, mu, var, m_chunk, y_std=None, xi=None, seed=0, tau=0.3, kappa=2.0, eps=1e-4,
        null_spec=False, ws=None):
    """One hb_posterior_mace_ex call over rows [row0, row0 + rows) of Xs / Xe / xi, writing F / mu / var at the same
    offsets (rng_offset = row0, as GP._posterior does)."""
    lib = _lib.lib()
    if ws is None:
        ws = torch.full((int(lib.hb_posterior_workspace_bytes(gp.n, gp.d, m_chunk)) // 4,), float("nan"), device=DEV)
    hi, lo = (gp.Linv_hi_dev, gp.Linv_lo_dev) if path == "tensor" else (None, None)
    ys = float(gp._y_std if y_std is None else y_std)
    xi1, xi2 = (None, None) if xi is None else xi
    if null_spec:
        st = lib.hb_posterior_mace(_off(Xs, row0, gp.d), rows, gp.n, gp.d, _ptr(gp._x_mul), _ptr(gp._x_add), _ptr(gp.Zt_dev),
                                   _ptr(gp.alpha_dev), _ptr(gp.Linv_dev), _ptr(hi), _ptr(lo), _ptr(gp.hyp_dev), gp.kern_id,
                                   gp._y_mean, ys, int(bool(gp.pred_likeli)), tau, kappa, eps, _off(xi1, row0), _off(xi2, row0),
                                   seed, _off(F, row0, 3), _off(mu, row0), _off(var, row0), _ptr(ws), ws.numel() * 4, m_chunk,
                                   _lib.stream_ptr())
        assert row0 == 0
    else:
        st = lib.hb_posterior_mace_ex(_off(Xs, row0, gp.d) if gp.d else None, _off(Xe, row0, gp.num_enum), rows, row0, gp.n,
                                      gp.d, C.byref(gp._spec), _ptr(gp._emb_meta_dev) if gp.num_enum else None,
                                      _ptr(gp.tab_s_dev) if gp.num_enum else None, _ptr(gp._x_mul), _ptr(gp._x_add),
                                      _ptr(gp.Zt_dev), _ptr(gp.alpha_dev), _ptr(gp.Linv_dev), _ptr(hi), _ptr(lo),
                                      _ptr(gp.hyp_dev), gp.kern_id, gp._y_mean, ys, int(bool(gp.pred_likeli)), tau, kappa,
                                      eps, _off(xi1, row0), _off(xi2, row0), seed, _off(F, row0, 3), _off(mu, row0),
                                      _off(var, row0), _ptr(ws), ws.numel() * 4, m_chunk, _lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == _lib.HB_OK, st


def call_mace(gp, Xs, Xe, path, m_chunk=None, y_std=None, xi=None, seed=0, null_spec=False, want_F=True):
    """(F [m, 3], mu, var) of one call over all rows; the workspace starts out as NaN, and sentinels past m (mu, var)
    and past 3 m (F) must survive."""
    m = Xs.shape[0] if gp.d else Xe.shape[0]
    outs = [torch.full((k + TAIL,), SENTINEL, device=DEV) for k in (3 * m, m, m)]
    F, mu, var = outs
    abi(gp, Xs, Xe, m, 0, path, F if want_F else None, mu, var, m if m_chunk is None else m_chunk, y_std=y_std, xi=xi,
        seed=seed, null_spec=null_spec)
    for t in outs:
        assert bool((t[-TAIL:] == SENTINEL).all()), "hb_posterior_mace_ex wrote past its outputs"
    return F[:3 * m].view(m, 3), mu[:m], var[:m]


def guard_stats(reset):
    v = (C.c_uint64 * 2)()
    assert _lib.lib().hb_guard_stats(v, int(reset)) == _lib.HB_OK
    return int(v[0]), int(v[1])


# ---------------------------------------------------------------------------------------------------------------- (a) own state
def own_state(gp, Xs, Xe, y_std=None, dtype=torch.float64, bounds=True):
    """The closed form of the module docstring on the GP's own fp32 state, in `dtype`, with the bounds B in fp64."""
    dt = dtype
    n, d, NP = gp.n, gp.d, gp.NP
    ys = float(gp._y_std if y_std is None else y_std)
    hyp = gp.hyp_dev.to(dt)
    sn2, c, s = hyp[0], hyp[1], hyp[2]
    pl = sn2 if gp.pred_likeli else torch.zeros((), dtype=dt, device=DEV)
    m = (Xs if d else Xe).shape[0]
    if d:
        ls = hyp[3:3 + d]
        px = gp._x_mul.to(dt) * Xs.to(dt)
        xt = px + gp._x_add.to(dt)
        Wl = torch.zeros(m, dtype=torch.float64, device=DEV)
        if gp.warp_mode:
            a, b = hyp[gp._h_wa:gp._h_wa + d], hyp[gp._h_wa + d:gp._h_wa + 2 * d]
            if bounds:
                Wl = (warp_error(px.double(), xt.double(), a.double(), b.double()) / ls.double()).norm(dim=1)
            xt = O.kumaraswamy_warp(xt, a, b)
        zc = xt / ls
    else:
        zc = torch.zeros(m, 0, dtype=dt, device=DEV)
        Wl = torch.zeros(m, dtype=torch.float64, device=DEV)
    Zn = gp.Zt_dev[:d, :n].to(dt).t()
    emb = gp.num_enum > 0
    if emb:
        zce = gather_emb(gp, Xe, gp.tab_s_dev.to(dt))
        Ze = gp.Zt_dev[d:, :n].to(dt).t()
    L = gp.Linv_dev[:n, :n].to(dt).tril()
    alpha = gp.alpha_dev[:n].to(dt)
    out = {k: [] for k in ("mu", "var", "raw_var", "vsq", "Bmu", "Bsimt", "Bguard", "Btc")}
    if bounds:
        La = L.abs().double()
        Lrow1 = La.sum(1)                                               # |Linv_c|_1
        Lmax = float(gp.Linv_dev.abs().max())
        col = torch.arange(n, device=DEV)
        q = (torch.clamp((col // CT + 1) * CT, max=NP) // KSTEP).double()      # accumulate steps of column c
        nt = NP // CT
    blk = max(1, (1 << 24) // (n * max(1, d + gp.De)))
    for r0 in range(0, m, blk):
        z = zc[r0:r0 + blk]
        Dz = z[:, None, :] - Zn[None]
        r2 = (Dz * Dz).sum(-1)
        k, _, t, rate = kernel_parts(r2, gp.kernel)
        if emb:
            ze = zce[r0:r0 + blk]
            De = ze[:, None, :] - Ze[None]
            ke, _, te, _ = kernel_parts((De * De).sum(-1), "matern32")
        else:
            ke = torch.ones_like(k)
        ks = s * k * ke
        V = ks @ L.t()
        vsq = (V * V).sum(1)
        mu_t = ks @ alpha + c
        raw_var = s - vsq + pl
        out["mu"].append(mu_t * ys + gp._y_mean)
        out["var"].append((raw_var.clamp_min(1e-6) * (ys * ys)).clamp_min(EPS32))
        out["raw_var"].append(raw_var)
        out["vsq"].append(vsq)
        if bounds:
            zn = z.norm(dim=1)[:, None] + Zn.norm(dim=1)[None] + Wl[r0:r0 + blk, None]
            grow = 2 + t + rate * zn
            if emb:
                keh = ke * (2 + te + math.sqrt(3.0) * (ze.norm(dim=1)[:, None] + Ze.norm(dim=1)[None]))
            else:
                keh = ke
            khat = (s * k * grow + FLUSH) * keh
            Lk = khat @ La.t()
            Lk0 = ks.abs() @ La.t()
            vn, Lkn = V.norm(dim=1), Lk.norm(dim=1)
            base = ys * ys * (s + pl)
            out["Bmu"].append(ys * (math.sqrt(n) * (khat @ alpha.abs()) + c.abs()) + (mu_t * ys + gp._y_mean).abs())
            simt = base + ys * ys * math.sqrt(NP) * vn * Lkn
            out["Bsimt"].append(simt)
            out["Bguard"].append(base + ys * ys * (10 * vn * Lkn + math.sqrt(nt) * vsq))
            T = (3 * SPLIT + 2 * q)[None] * Lk0 + 2.0 ** -20 * Lmax * ks.abs().sum(1, keepdim=True) + 2.0 ** -11 * s * Lrow1[None]
            out["Btc"].append(simt + ys * ys * 2 * (V.abs() * T).sum(1))
    return {k: torch.cat(v) for k, v in out.items() if v}


def _ratio(got, ref, B):
    """max |got - ref| / (u B), an exact match counting 0 wherever B is 0."""
    if got.numel() == 0:
        return 0.0
    err = (got - ref).abs()
    return float(torch.where(err == 0, torch.zeros_like(err), err / (U * B)).max())


def check_own_state(name, gp, Xs, Xe, got, path, y_std=None, ref=None):
    """Reference (a) for one path: the c each output needs; asserts c <= C_MAX."""
    ref = own_state(gp, Xs, Xe, y_std) if ref is None else ref
    F, mu, var = got
    ys = float(gp._y_std if y_std is None else y_std)
    s = float(gp.hyp[2])
    rep = dict(case=name, path=path, ref="own_state", n=gp.n, NP=gp.NP, m=mu.shape[0], d=gp.d, De=gp.De)
    if path == "simt":
        Bv = ref["Bsimt"]
    else:
        # the device flags on its own |v|^2: rows within the tensor bound of the threshold may go either way
        gap = (s - ref["vsq"]) - THETA * s
        margin = C_MAX * U * ref["Btc"] / (ys * ys)
        flag, keep = gap < -margin, gap > margin
        Bv = torch.where(flag, ref["Bguard"], torch.where(keep, ref["Btc"], torch.maximum(ref["Btc"], ref["Bguard"])))
        rep.update(rows_guarded=int(flag.sum()), rows_either=int((~flag & ~keep).sum()))
    c = dict(mu=_ratio(mu.double(), ref["mu"], ref["Bmu"]), var=_ratio(var.double(), ref["var"], Bv))
    rep.update(c_needed=c, c_max_case=max(c.values()))
    print(json.dumps(rep))
    assert max(c.values()) <= C_MAX, rep
    return ref


# ---------------------------------------------------------------------------------------------------------------- (b) fp64 GP
def oracle(gp, tm, Xs, Xe):
    """fp64 (mu, var, raw variance) of the candidates in original y units."""
    hyp = tm["hyp"]
    s, sn2 = float(hyp[2]), float(hyp[0])
    Zc = features64(gp, Xs.double() if gp.d else None, Xe, hyp, tm["tables"])
    Ks = kmat64(gp, Zc, tm["Zt"], s)
    mu_t = tm["c"] + Ks @ tm["alpha"]
    Vt = torch.linalg.solve_triangular(tm["L"], Ks.t(), upper=False)
    raw = s - (Vt * Vt).sum(0) + (sn2 if gp.pred_likeli else 0.0)
    ys, ym = gp._y_std, gp._y_mean
    return mu_t * ys + ym, (raw.clamp_min(1e-6) * ys * ys).clamp_min(EPS32), raw


def check_fp64(name, gp, X, Xe_train, y, Xs, Xe, got, path, rho=None):
    """Reference (b), per row, with the fp32 closed form on the same state as the evidence where the fit's fp32 state is
    the limit.  rho: own-state (s - |v|^2) / s of the rows, to report the worst sigma error for 0.12 <= rho <= 0.2."""
    tm = true_model(gp, X, Xe_train, y)
    mu64, var64, raw64 = oracle(gp, tm, Xs, Xe)
    r32 = own_state(gp, Xs, Xe, dtype=torch.float32, bounds=False)
    _, mu, var = (t.double() for t in got)
    ys, s = gp._y_std, float(tm["hyp"][2])
    canc = raw64 < CANCEL * s

    def errs(mu_, var_):
        emu = (mu_ - mu64).abs() / mu64.abs().clamp_min(ys)
        esg = (var_.sqrt() - var64.sqrt()).abs() / var64.sqrt()
        return emu, esg
    emu, esg = errs(mu, var)
    fmu, fsg = errs(r32["mu"].double(), r32["var"].double())
    worst = lambda e, k: float(e[k].max()) if bool(k.any()) else 0.0
    crit = lambda base, f: max(base, min(2 * f, 2e-2))
    rep = dict(case=name, path=path, ref="fp64", m=int(mu.shape[0]), mu_err=float(emu.max()), mu_fp32_reference_err=float(fmu.max()),
               sigma_err_regular=worst(esg, ~canc), sigma_fp32_reference_err_regular=worst(fsg, ~canc),
               sigma_err_cancelled=worst(esg, canc), sigma_fp32_reference_err_cancelled=worst(fsg, canc),
               rows_cancelled=int(canc.sum()), rows_over_1e4=int(((emu > 1e-4) | (esg > 1e-4)).sum()))
    if rho is not None:
        band = (rho >= THETA) & (rho <= 0.2)
        rep.update(sigma_err_rho_0p12_0p2=worst(esg, band), rows_rho_0p12_0p2=int(band.sum()), NP=gp.NP)
    print(json.dumps(rep))
    assert rep["mu_err"] <= crit(1e-4, rep["mu_fp32_reference_err"]), rep
    assert rep["sigma_err_regular"] <= crit(1e-4, rep["sigma_fp32_reference_err_regular"]), rep
    assert rep["sigma_err_cancelled"] <= crit(2e-4, rep["sigma_fp32_reference_err_cancelled"]), rep
    return rep


# ---------------------------------------------------------------------------------------------------------------- one case
def check_case(name, gp, X, Xe_train, y, Xs, Xse, dups=(), fp64=True, m_chunk=None, rho=None):
    """Both paths through the ABI against (a) and (b); mu equal on both paths; duplicates; GP.predict equal to the ABI."""
    ref = own_state(gp, Xs, Xse)
    got = {}
    for path in PATHS:
        got[path] = call_mace(gp, Xs, Xse, path, m_chunk=m_chunk)
        for t in got[path]:
            assert bool(torch.isfinite(t).all())
        for s_, t_ in dups:        # (F differs: every row draws its own normals)
            for t in got[path][1:]:
                assert torch.equal(t[s_], t[t_]), ("duplicate rows differ", path, s_, t_)
        check_own_state(name, gp, Xs, Xse, got[path], path, ref=ref)
        if fp64:
            check_fp64(name, gp, X, Xe_train, y, Xs, Xse, got[path], path, rho=rho)
    assert torch.equal(got["tensor"][1], got["simt"][1]), "mu depends on the contraction path"
    # GP.predict: the same kernels on the same rows, so the same bytes whatever its chunking
    tc = gp.tensor_cores
    try:
        for path in PATHS:
            gp.tensor_cores = path == "tensor"
            mu_g, var_g = gp.predict(Xs if gp.d else None, Xse)
            assert torch.equal(mu_g.reshape(-1), got[path][1]) and torch.equal(var_g.reshape(-1), got[path][2]), path
    finally:
        gp.tensor_cores = tc
    return got, ref


# ---------------------------------------------------------------------------------------------------------------- tests
SHAPE_N = [5, 127, 128, 129, 511, 512, 513, 1100, 4224]


@pytest.mark.parametrize("n", SHAPE_N)
def test_posterior_across_kstar_groups_and_column_tiles(n):
    """NP = 128 ... 4224: one to nine 512-column K* groups, the 128-column tiles either side of n, m = 129 rows (two bands, padded to one 4-band cluster) and m = 300 at the largest n."""
    gp, X, Xe, y = shape_model(n)
    Xs, Xse, dups = candidates(gp, X, Xe, 300 if n == 4224 else 129, seed=n + 1)
    check_case(f"shape-n{n}", gp, X, Xe, y, Xs, Xse, dups)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("m", [1, 127, 128, 129, 257, 385, 512, 513, 2049, 4100])
def test_posterior_across_bands_clusters_and_chunks(m):
    """One chunk of m rows at n = 513: 1 ... 33 bands of 128 rows, band counts = 1, 2, 3 (mod 4) so that the last cluster
    runs padding bands, chunks of more than 16 bands (the schedule's band-major body), mc_pad_max = round_up(m, 512)."""
    gp, X, Xe, y = shape_model(513)
    Xs, Xse, dups = candidates(gp, X, Xe, m, seed=m + 3)
    check_case(f"bands-m{m}", gp, X, Xe, y, Xs, Xse, dups, m_chunk=m)
    torch.cuda.empty_cache()


def test_posterior_through_gp_predict_chunks():
    """m = 70 001 through GP.predict with the default m_chunk = 32 768: three chunks, the last one partial; both paths
    against both references, and a pinned host batch (uploaded chunk by chunk under the scoring) equals the device call."""
    gp, X, Xe, y = shape_model(513)
    assert gp.m_chunk == 32768
    Xs, Xse, dups = candidates(gp, X, Xe, 70001, seed=70001)
    got, _ = check_case("gp-chunks-m70001", gp, X, Xe, y, Xs, Xse, dups, m_chunk=32768)
    host = Xs.cpu().pin_memory()
    mu_h, var_h = gp.predict(host)
    assert torch.equal(mu_h.reshape(-1), got["tensor"][1].cpu()) and torch.equal(var_h.reshape(-1), got["tensor"][2].cpu())
    xi1, xi2 = torch.randn(70001, 1), torch.randn(70001, 1)
    F_h = gp.predict_mace(host, 0.3, 2.0, 1e-4, xi1=xi1, xi2=xi2)
    F_d = call_mace(gp, Xs, Xse, "tensor", m_chunk=32768, xi=(xi1.reshape(-1).to(DEV), xi2.reshape(-1).to(DEV)))[0]
    assert torch.equal(F_h, F_d.cpu())
    torch.cuda.empty_cache()


@pytest.mark.parametrize("kind", ["numeric", "mixed"])
def test_m_chunk_gives_the_same_bytes(kind):
    """Every row is computed on its own, so any m_chunk -- 1, 7, 128, 129, 511, 512, 513, 1000 against one chunk of 1300
    rows -- gives the same mu, var and F on both paths, and so does a second call.  The numeric model's NULL-spec entry
    hb_posterior_mace equals _ex."""
    gp, X, Xe, y = shape_model(1100) if kind == "numeric" else variant_model("mixed_e2")
    Xs, Xse, _ = candidates(gp, X, Xe, 1300, seed=77)
    for path in PATHS:
        one = call_mace(gp, Xs, Xse, path, seed=5)
        for mc in (None, 1, 7, 128, 129, 511, 512, 513, 1000):
            got = call_mace(gp, Xs, Xse, path, m_chunk=mc, seed=5)
            for a, b in zip(one, got):
                assert torch.equal(a, b), (path, mc)
        if kind == "numeric":
            for a, b in zip(one, call_mace(gp, Xs, Xse, path, m_chunk=129, seed=5, null_spec=True)):
                assert torch.equal(a, b), path
        check_own_state(f"m_chunk-{kind}", gp, Xs, Xse, one, path)


@pytest.mark.parametrize("draws", ["xi", "philox"])
def test_mace_tail_equals_the_epilogue_and_row_ranges(draws):
    """F of the fused call equals hb_mace_epilogue on the call's own mu and var, with noise_var formed in fp32 as
    mace_kernel forms it; calls over row ranges with matching rng_offset and pointer offsets give one call's F."""
    gp, X, Xe, y = shape_model(1100)
    m = 1300
    Xs, Xse, _ = candidates(gp, X, Xe, m, seed=91)
    g = torch.Generator().manual_seed(9)
    xi = (torch.randn(m, generator=g).to(DEV), torch.randn(m, generator=g).to(DEV)) if draws == "xi" else None
    tau, kappa, eps, seed = 0.3, 2.0, 1e-4, 1234
    sn2, ys = np.float32(gp.hyp[0]), np.float32(gp._y_std)
    noise_var = float(np.float32(sn2 * np.float32(ys * ys)))
    lib = _lib.lib()
    for path in PATHS:
        F, mu, var = call_mace(gp, Xs, Xse, path, m_chunk=512, xi=xi, seed=seed)
        F2 = torch.full((3 * m,), SENTINEL, device=DEV)
        xi1, xi2 = (None, None) if xi is None else xi
        assert lib.hb_mace_epilogue(_ptr(mu), _ptr(var), m, noise_var, tau, kappa, eps, _ptr(xi1), _ptr(xi2), seed, _ptr(F2),
                                    _lib.stream_ptr()) == _lib.HB_OK
        torch.cuda.synchronize()
        assert torch.equal(F.reshape(-1), F2), path
        parts = torch.full((3 * m + TAIL,), SENTINEL, device=DEV)
        mp, vp = (torch.full((m + TAIL,), SENTINEL, device=DEV) for _ in range(2))
        for r0, r1 in ((0, 1), (1, 300), (300, 777), (777, m)):
            abi(gp, Xs, Xse, r1 - r0, r0, path, parts, mp, vp, 256, xi=xi, seed=seed)
        assert torch.equal(parts[:3 * m], F.reshape(-1)) and torch.equal(mp[:m], mu) and torch.equal(vp[:m], var), path
        assert bool((parts[3 * m:] == SENTINEL).all()) and bool((mp[m:] == SENTINEL).all())
    if xi is not None:      # GP.predict_mace with the same draws: the same bytes
        F_gp = gp.predict_mace(Xs, tau, kappa, eps, xi1=xi[0].cpu(), xi2=xi[1].cpu(), seed=seed, device_out=True)
        assert torch.equal(F_gp, call_mace(gp, Xs, Xse, "tensor", xi=xi, seed=seed)[0])


# ---------------------------------------------------------------------------------------------------------------- the guard
RHO = (0.05, 0.10, 0.115, 0.125, 0.14, 0.2, 0.3)
PER_RHO = 64


def own_rho(gp, Xs):
    r = own_state(gp, Xs, None, bounds=False)
    s = float(gp.hyp[2])
    return (s - r["vsq"]) / s


def rho_rows(gp, X, seed):
    """PER_RHO rows at each rho in RHO, by fp64 bisection of the own-state rho along segments from a training row
    (rho < 0.04) to a row far enough away (3 units, doubled until rho > 0.35).  Returns the fp32 rows, their target and their own rho."""
    g = torch.Generator().manual_seed(seed)
    cand = X[:2000].to(DEV)
    r0 = own_rho(gp, cand.float().contiguous())
    starts = cand[r0 < 0.04]
    need = len(RHO) * PER_RHO
    assert starts.shape[0] >= 64, "too few training rows with a small variance"
    a = starts[torch.arange(need) % starts.shape[0]].double()
    dirn = torch.randn(need, gp.d, generator=g, dtype=torch.float64).to(DEV)
    dirn = dirn / dirn.norm(dim=1, keepdim=True)
    R = torch.full((need, 1), 3.0, dtype=torch.float64, device=DEV)
    for _ in range(6):
        R = torch.where((own_rho(gp, (a + R * dirn).contiguous()) > 0.35)[:, None], R, 2 * R)
    b = a + R * dirn
    assert bool((own_rho(gp, b.contiguous()) > 0.35).all())
    target = torch.tensor(RHO, dtype=torch.float64, device=DEV).repeat_interleave(PER_RHO)
    lo, hi = torch.zeros(need, 1, dtype=torch.float64, device=DEV), torch.ones(need, 1, dtype=torch.float64, device=DEV)
    for _ in range(30):
        mid = (lo + hi) / 2
        below = (own_rho(gp, (a + mid * (b - a)).contiguous()) < target)[:, None]
        lo, hi = torch.where(below, mid, lo), torch.where(below, hi, mid)
    Xs = (a + (lo + hi) / 2 * (b - a)).float().contiguous()
    rho = own_rho(gp, Xs)
    assert float((rho - target).abs().max()) < 2e-3
    return Xs, target, rho


@pytest.mark.parametrize("n", [1100, 4224])
def test_guard_threshold_band(n):
    """Rows placed at rho = 0.05 ... 0.3 around the guard threshold 0.12, 64 each: every row meets (a) and (b) on both
    paths (the worst sigma error for 0.12 <= rho <= 0.2 is printed), and hb_guard_stats counts m rows seen and flags
    every row at rho <= 0.10, none at rho >= 0.14, and either way at 0.115 / 0.125.  A batch of rho = 0.05 rows is
    flagged entirely, one of rho >= 0.2 rows not at all."""
    gp, X, Xe, y = shape_model(n)
    Xs, target, rho = rho_rows(gp, X, seed=n)
    m = Xs.shape[0]
    check_case(f"guard-n{n}", gp, X, Xe, y, Xs, None, rho=rho)
    guard_stats(reset=True)
    call_mace(gp, Xs, None, "tensor")
    seen, flagged = guard_stats(reset=True)
    must = int((target <= 0.10).sum())
    either = int(((target == 0.115) | (target == 0.125)).sum())
    print(json.dumps(dict(case=f"guard-n{n}", NP=gp.NP, rows=m, flagged=flagged, rows_rho_le_0p10=must,
                          rows_rho_0p115_0p125=either)))
    assert seen == m
    assert 0 <= flagged - must <= either, (flagged, must, either)
    for sel, want in ((target == 0.05, "all"), (target >= 0.2, "none")):
        rows = Xs[sel].contiguous()
        guard_stats(reset=True)
        call_mace(gp, rows, None, "tensor")
        seen, flagged = guard_stats(reset=True)
        assert seen == rows.shape[0] and flagged == (seen if want == "all" else 0), (want, seen, flagged)
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------- operand split
def check_operand_split(gp):
    """Linv_hi / Linv_lo hold h0 = rn_fp16(Linv 2^k), h1 = rn_fp16((Linv 2^k - h0) 2048) and the scale 2^k after h1, with
    max |Linv| 2^k in [512, 1024).  torch's fp32 -> fp16 conversion rounds to nearest even, as __float2half_rn does."""
    NP = gp.NP
    Li = gp.Linv_dev
    sc = float(gp.Linv_lo_dev.reshape(-1)[NP * NP // 2])
    k = math.log2(sc)
    assert k == round(k), sc
    top = float(Li.abs().max()) * sc
    assert 512 <= top < 1024, (top, sc)
    x = Li * sc
    h0 = x.half()
    h1 = ((x - h0.float()) * 2048).half()
    got0 = gp.Linv_hi_dev.reshape(-1).view(torch.float16)[:NP * NP].view(NP, NP)
    got1 = gp.Linv_lo_dev.reshape(-1).view(torch.float16)[:NP * NP].view(NP, NP)
    assert torch.equal(got0.view(torch.int16), h0.view(torch.int16)), "h0 differs from rn_fp16(Linv 2^k)"
    assert torch.equal(got1.view(torch.int16), h1.view(torch.int16)), "h1 differs from rn_fp16((Linv 2^k - h0) 2048)"


# ---------------------------------------------------------------------------------------------------------------- extremes
@pytest.mark.parametrize("outputscale", [1e-3, 1e3])
def test_outputscale_extremes(outputscale):
    """s = 1e-3 and 1e3 move the K* operand scale 2^k far from 1."""
    gp, X, Xe, y = fit_model(("os", outputscale), 300, 4, seed=21)
    _set(gp, os=outputscale)
    assert abs(float(gp.hyp[2]) / outputscale - 1) < 1e-3
    check_operand_split(gp)
    Xs, Xse, dups = candidates(gp, X, Xe, 300, seed=22)
    check_case(f"outputscale-{outputscale:g}", gp, X, Xe, y, Xs, Xse, dups)


def test_tiny_noise_large_linv():
    """sigma_n^2 at noise_lb = 1e-6 with lengthscales 0.4 and no pred_likeli: a large, ill-conditioned Linv.  Random rows
    (the variance of rows on the data sits at the 1e-6 floor there, below what fp32 resolves) meet (a) and (b)."""
    gp, X, Xe, y = fit_model("tiny-noise", 129, 4, pred_likeli=False, epochs=2, noise_lb=1e-6, seed=3)
    _set(gp, noise=-30.0, ls=0.4)
    check_operand_split(gp)
    Xs = (torch.rand(200, gp.d, generator=torch.Generator().manual_seed(4)) * 2 - 1).float().to(DEV).contiguous()
    check_case("tiny-noise", gp, X, Xe, y, Xs, None)
    print(json.dumps(dict(case="tiny-noise", max_abs_linv=float(gp.Linv_dev.abs().max()))))


def test_variance_floor():
    """Rows within 1e-6 (raw units) of training rows, at a noise of 1e-9 and lengthscales 0.05, no pred_likeli: the
    variance is under gpytorch's 1e-6 floor, so var is the floor exactly on both paths; random rows of the same batch
    stay live; every row meets (a) and (b)."""
    gp, X, Xe, y = fit_model("mace-floor", 129, 4, pred_likeli=False, epochs=2, noise_lb=1e-9, seed=3)
    _set(gp, noise=-30.0, ls=0.05)
    check_operand_split(gp)
    g = torch.Generator().manual_seed(3)
    near = X[:40] + 1e-6 * (torch.rand(40, gp.d, generator=g) * 2 - 1)
    far = torch.rand(40, gp.d, generator=g) * 2 - 1
    Xs = torch.cat([near, far]).float().to(DEV).contiguous()
    got, ref = check_case("variance-floor", gp, X, Xe, y, Xs, None)
    dead = ref["raw_var"] < 0.5e-6
    assert int(dead.sum()) >= 30 and int((~dead).sum()) >= 30, int(dead.sum())
    ys2 = np.float32(gp._y_std) * np.float32(gp._y_std)
    floor = float(max(np.float32(1e-6) * ys2, np.float32(EPS32)))
    for path in PATHS:
        assert bool((got[path][2][dead] == floor).all()), path


def test_flt_epsilon_floor():
    """A y_std so small that y_std^2 var~ crosses FLT_EPSILON inside one batch: var = FLT_EPSILON exactly on the rows
    under it, the others checked against reference (a) at that y_std, on both paths."""
    gp, X, Xe, y = shape_model(129)
    s = float(gp.hyp[2])
    ys = math.sqrt(2 * EPS32 / s)
    Xs, Xse, _ = candidates(gp, X, Xe, 129, seed=5)
    ref = own_state(gp, Xs, Xse, y_std=ys)
    ps2 = ref["raw_var"].clamp_min(1e-6) * ys * ys
    dead, live = ps2 < 0.9 * EPS32, ps2 > 1.1 * EPS32
    assert int(dead.sum()) >= 5 and int(live.sum()) >= 5, (int(dead.sum()), int(live.sum()))
    for path in PATHS:
        got = call_mace(gp, Xs, Xse, path, y_std=ys)
        check_own_state("flt-epsilon-floor", gp, Xs, Xse, got, path, y_std=ys, ref=ref)
        assert bool((got[2][dead] == EPS32).all()), path


# ---------------------------------------------------------------------------------------------------------------- variants
@pytest.mark.parametrize("variant", list(VARIANTS) + ["categorical_only"])
def test_posterior_model_variants(variant):
    """Each kernel with pred_likeli on and off, mixed models with one, two and six categorical columns, ard_kernel=False,
    heteroscedastic noise, learned and fixed warps (fused into the K* load here), and a categorical-only model (d = 0)."""
    if variant == "categorical_only":
        gp, X, Xe, y = fit_model(("variant", variant), 300, 0, num_uniqs=(4, 6), seed=7)
    else:
        gp, X, Xe, y = variant_model(variant)
    if variant == "wide_embeddings":
        assert gp.De == 300
    Xs, Xse, dups = candidates(gp, X, Xe, 200, seed=200, near=variant == "wide_embeddings")
    check_case(variant, gp, X, Xe, y, Xs, Xse, dups)


@pytest.mark.parametrize("width", list(WIDTHS))
def test_posterior_feature_widths(width):
    """d = 1, 33 (across kstar_kernel's 32-wide feature chunk), 300, and d + De = 4096; from d = 300 on, random rows are
    uncorrelated with the data, so the rows there sit next to training rows."""
    gp, X, Xe, y = fit_model(("width", width), 300, seed=11, **WIDTHS[width])
    Xs, Xse, dups = candidates(gp, X, Xe, 64 if width == 4096 else 100, seed=width, near=width >= 300)
    check_case(f"width-{width}", gp, X, Xe, y, Xs, Xse, dups)
    torch.cuda.empty_cache()


def test_operand_split_of_every_model():
    """Every model this session has fitted (the shapes, variants, widths and extremes of both posterior tests)."""
    from tests.util import _MODELS
    seen = 0
    for key, (gp, *_rest) in list(_MODELS.items()):
        check_operand_split(gp)
        seen += 1
    if seen == 0:
        check_operand_split(shape_model(513)[0])
