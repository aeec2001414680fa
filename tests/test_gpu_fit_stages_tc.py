"""The tensor-core stages of the fit epoch, one at a time, and the MLL gradient contraction on its own, element by element
against fp64.

Every pSGLD epoch runs transform -> gram -> Cholesky with its outer update on the tensor cores -> triangular inverse
(128 x 128 diagonal blocks on the FP32 pipe, doubling levels on the tensor cores) -> alpha / log-det -> K^-1 = U U^T on the
tensor cores -> gradient contraction.  hb_cholesky_tc, hb_tri_inverse_tc and hb_kinv_tc run those launchers one stage at a
time.  u = 2^-24; |A| is the element-wise absolute value and |A||B| an fp64 product of absolute values.  Each case prints
the c it needs (max |error| / bound) and requires c <= C_MAX.

a. The stage chain is the fit's epoch: hb_gram -> hb_cholesky_tc -> hb_tri_inverse_tc -> hb_solve_logdet -> hb_kinv_tc ->
   hb_mll_grad gives, bit for bit, the losses[0] and state grad of hb_fit_ex with one epoch at lr = 0.  So (b) - (d)
   check what the fit runs.  NP = 640, 2176, 4224.

Bound model of the 3xTF32 GEMMs (b - d).  Each fp32 operand x is split into hi = rn_tf32(x) and lo = x - hi, and the
product is accumulated as hi*hi' + hi*lo' + lo*hi' by three wgmma instructions per 8-wide k-step.  Taken as given, not
re-derived here:
   - hi + lo, as the tensor cores read it (lo truncated to tf32), represents x within 2^-23 = 2u relative.  A CPU emulation
     of the split (1e6 normal samples, K = 2048 dot products) found the same worst case for a truncated and a rounded lo,
     with no bias;
   - the dropped lo*lo' term is at most 2^-24 = u relative;
   - so one product carries at most 2u + 2u + u = 5u relative;
   - accumulation: ASSUMED one truncated fp32 ulp (2u relative to the running sum, which is at most sum |a||b|) per wgmma
     instruction.  This rests on published measurements of earlier tensor-core generations (products exact, alignment to
     the largest exponent, round toward zero); it has not been measured on the H100 here.  It is linear in K, not
     u sqrt(K): a round-to-nearest accumulation lands well inside it (c << 1), and c near or above 1 means the
     accumulation is worse than this model.
   u_tc(K) = (5 + 0.75 K) u.  The 0.75 K counts the instructions tcgemm.cu issues: mma3 runs hi*hi', hi*lo' and lo*hi' as
   three wgmma instructions on the same fp32 accumulator, each of which adds its 8 products and writes a rounded fp32
   result, so every 8-wide k-step rounds the running sum three times.  A model of one truncation per k-step,
   (5 + 0.25 K) u, undercounts that structure: no 3xTF32 GEMM built from three accumulating instructions can meet it in
   general.  Each case also prints its c under that model (c_one_ulp_per_k_step); there hb_kinv_tc reaches 1.1
   (NP = 2176 and 4224 at cond_1(L) ~ 1e6 - 1e7, and the RBF epoch below), and every other stage stays below 0.16.

b. hb_cholesky_tc: the backward error |L L^T - A|, A the fp32 Gram matrix in fp64, on the lower triangle within
   c (u_tc(NP) + NP u) |L||L|^T: the outer updates go through the tensor cores (k-range 512 per outer block, at most NP in
   all), the in-block work and the subtractions through the FP32 pipe (gamma_NP <= NP u).  The same c is printed for
   hb_cholesky on the same A.  Every pad entry (identity block) is exact.  NP = 640, 1152, 2176, 4224 (one, two, four and
   eight 512-column outer blocks) with n = NP and n = NP - 37 (a short last panel); Matern-3/2 and RBF Gram matrices, well
   conditioned (sigma^2 = 8e-4, lengthscale 0.5) and ill conditioned (sigma^2 raised tenfold from 1e-6 until the fp32
   factorisation succeeds; sigma^2 and cond_1(L) printed).  info reports the leading minor (LAPACK) on a matrix built to
   fail at a column past the first outer block, as hb_cholesky does.

c. hb_tri_inverse_tc on the device's own fp32 L from (b), Lambda = L^-1 in fp64: |X - Lambda| <= c u_tc(NP)
   |Lambda||L||X|; the strict upper triangle exactly 0; the 128 x 128 diagonal blocks (triinv_base2_kernel, FP32 pipe)
   to the SIMT accuracy of test_gpu_fit_state.py part 2 against the inverse of L's diagonal block:
   c u sqrt(128) |inv(L_bb)||L_bb||X_bb|.  NP = 384, 640, 1152, 2176, 4224 end doubling levels in partial pairs and switch
   the output tile width between 128 and 256.

d. hb_kinv_tc on every element of the lower 128-tiles against (X^T X)64, X the device's L^-1 from (c): |Kinv - (X^T X)64|
   <= c u_tc(NP) |X|^T|X|.  This also checks that the transposed split U the inverse leaves is X^T.  A NaN-filled output
   stays NaN outside the output tiles' boxes (columns >= min(NP, round_up(r0 + 128, 256)) of tile row r0); the upper
   tiles inside a box hold K^-1 within the same bound.

e. The gradient contraction (mll_grad_kernel + mll_finish_kernel) on its own, for numeric models of all four kernels,
   with ARD (hb_mll_grad on its own inputs) and a shared lengthscale (hb_mll_fwd_bwd, the only entry that takes one).
   After hb_mll_fwd_bwd, K^-1 = hb_kinv(state Linv) and alpha, hyp, scal from the state; for ARD models hb_mll_grad on
   them first reproduces the fused gradient bit for bit, so these are the contraction's inputs.  z = fl(Xt fl(1 / l)).
   W = alpha alpha^T - K^-1 in fp64 (K^-1 read from its lower tiles, the diagonal tiles in full), r^2 in fp64 from z.
   Per lengthscale k the device sums terms t_ij = w W_ij s h(r_ij) dz_ijk^2 (w = 2 below the diagonal tiles):
     |S_k - S64_k| <= u (83 sum |t_ij| + sum |w W s| dz^2 dh_ij)
   83 = 64 (fma chain over a thread's 8 x 8 pairs) + 5 (warp butterfly) + 8 (the warps, in order) + 6 (W, the products
   with s and h, the difference and its square); the per-block partials are summed in fp64.  dh/u bounds the error of
   h as kern_eval_grad forms it from the fp32 r^2: |h| (E_EX2 + 1.25 t + 4 + (t + 1)(E_RSQ + 2.5) + (d + 2)(1 + t)),
   with E_EX2, E_RSQ and t as in test_gpu_fit_state.py part 1 ((d + 2) u is the relative error of the fp32 r^2, and
   |dh/dr^2| r^2 <= |h| (1 + t) for all four kernels).  The outputscale sum w W k and the trace of W take the same
   accumulation bound with the error of k (u eps_k of test_gpu_fit_state.py plus |h| / 2 (d + 2) u r^2).  The fp64
   finish scales these, and the result is rounded once (u |g|).  The loss against the fp64 loss of the same scal:
   u |l| + 1e-12.  Cases: n = 5, 127, 129, 2150, 4097; d = 1, 31, 32, 33, 300 (the 32-feature chunk edges); exactly
   duplicated rows and near-duplicates with r^2 on either side of Matern-1/2's 1e-30 clamp.

   Model families (hb_mll_fwd_bwd with their spec; Zt read from the state): noise_diag; mixed models, with and without
   numeric features -- the embedding lengthscale (sum w W s k1 h2 r_e^2, the Matern-3/2 embedding factor's errors
   carried like h's) and every table entry, (1 / (n l_e)) sum over its category's rows of sum_j W s k1 h2 (E_iq - E_jq),
   accumulated 8 in-thread + 4 butterfly levels + NP / 128 tiles in fp32 (plus the same 6 roundings), then in fp64; and
   learned warps, whose exponent sweeps sum G dz (dZa_i - dZa_j) with dZa, dZb in fp64 from the fp32 x, a, b: their fp32
   error is carried term by term from the absolute errors of log u and log(1 - u^a) and the relative errors of u^a and
   the powers, as tests/util.py warp_error derives them.

The fp64 references run on the device in torch float64; they are references, not the code under test."""
import ctypes as C
import json
import math

import numpy as np
import pytest
import torch

from hebo_b200 import _lib
from oracle import gp_oracle as O
from tests.test_gpu_fit_epoch import NOISE_LB, numeric_model, run_fit
from tests.test_gpu_fit_state import E_EX2, E_RSQ, FLUSH, GT, U, _ratio, cholesky, cond1, eps_k, gram, lower_tiles
from tests.util import DEV, kernel_parts, warp_derivs

pytestmark = pytest.mark.gpu

# Largest c measured on an H100 80GB HBM3 (700 W): hb_cholesky_tc 0.086 (hb_cholesky on the same A: <= 0.0065 at
# NP = 4224), hb_tri_inverse_tc 0.054, its diagonal blocks 0.50, hb_kinv_tc 0.37; gradient contraction 0.90 and loss
# 0.88 (worst-case forms of e.).  C_MAX = 1 is the bound itself: about 2.7x the largest tensor-core stage c.
C_MAX = 1.0
F64 = torch.float64


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def u_tc(K):
    return (5.0 + 0.75 * K) * U


def to_issue_model(c, K, extra=0.0):
    """The same error measured against the one-ulp-per-k-step accumulation model, (5 + 0.25 K) u (+ extra u)."""
    return c * (5.0 + 0.75 * K + extra) / (5.0 + 0.25 * K + extra)


def _report(rep):
    print(json.dumps(rep))
    worst = max(rep["c_needed"].values())
    assert worst <= C_MAX, rep


# ---------------------------------------------------------------------------------------------------------------- C ABI
class TcWs:
    """A tensor-core workspace of hb_tc_workspace_bytes(NP) bytes, NaN-filled."""

    def __init__(self, NP):
        self.bytes = int(_lib.lib().hb_tc_workspace_bytes(NP))
        assert self.bytes > 0
        self.buf = torch.full((self.bytes // 4,), float("nan"), device=DEV)

    @property
    def ptr(self):
        return _p(self.buf)


def cholesky_tc(A, ws):
    """hb_cholesky_tc in place; returns info."""
    NP = A.shape[0]
    cws = torch.empty(GT * GT, device=DEV)
    info = torch.zeros(1, dtype=torch.int32, device=DEV)
    st = _lib.lib().hb_cholesky_tc(_p(A), NP, _p(cws), _p(info), ws.ptr, ws.bytes, _lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == _lib.HB_OK, st
    return int(info.item())


def tri_inverse_tc(L, ws):
    NP = L.shape[0]
    X = torch.full((NP, NP), float("nan"), device=DEV)
    st = _lib.lib().hb_tri_inverse_tc(_p(L), NP, _p(X), ws.ptr, ws.bytes, _lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == _lib.HB_OK, st
    return X


def kinv_tc(NP, ws):
    K = torch.full((NP, NP), float("nan"), device=DEV)
    st = _lib.lib().hb_kinv_tc(NP, _p(K), ws.ptr, ws.bytes, _lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == _lib.HB_OK, st
    return K


# ---------------------------------------------------------------------------------------------------------------- a. chain
def stage_chain(m, ws_fill=float("nan")):
    """The epoch composed of the single-stage entry points; returns (loss, grad, K = A, L, Linv, Kinv, hyp)."""
    lib, st = _lib.lib(), _lib.stream_ptr()
    n, d, NP = m.n, m.d, m.NP
    f32 = dict(dtype=torch.float32, device=DEV)
    raw = m.raw.float().to(DEV).contiguous()
    hyp = torch.empty(d + 3, **f32)
    _lib.check(lib.hb_transform_hypers(_p(raw), d, NOISE_LB, _p(hyp), st), "transform")
    K = torch.full((NP, NP), ws_fill, **f32)
    _lib.check(lib.hb_gram(_p(m.XtT), n, d, _p(hyp), m.kern, None, 0.0, _p(K), st), "gram")
    A = K.clone()
    ws = TcWs(NP)
    info = cholesky_tc(K, ws)
    assert info == 0
    Linv = tri_inverse_tc(K, ws)
    sws = torch.full(((1 + NP // 64) * NP,), float("nan"), dtype=F64, device=DEV)
    alpha = torch.full((NP,), float("nan"), **f32)
    scal = torch.full((2,), float("nan"), dtype=F64, device=DEV)
    _lib.check(lib.hb_solve_logdet(_p(K), _p(Linv), _p(m.y), n, NP, _p(hyp), _p(alpha), _p(scal), _p(sws), st), "solve")
    Kinv = kinv_tc(NP, ws)
    gws = torch.full((int(lib.hb_fit_workspace_bytes(n, d)),), 0xFF, dtype=torch.uint8, device=DEV)
    grad = torch.full((m.P,), float("nan"), **f32)
    loss = torch.full((1,), float("nan"), **f32)
    _lib.check(lib.hb_mll_grad(_p(m.XtT), n, d, _p(raw), _p(hyp), m.kern, _p(Kinv), _p(alpha), _p(scal), m.noise_guess,
                               _p(grad), _p(loss), _p(gws), st), "mll_grad")
    torch.cuda.synchronize()
    return dict(loss=loss.cpu(), grad=grad.cpu(), A=A, L=K, Linv=Linv, Kinv=Kinv, hyp=hyp, alpha=alpha, scal=scal)


@pytest.mark.parametrize("n", [600, 2150, 4100])
def test_stage_chain_equals_the_fit_epoch_bitwise(n):
    m = numeric_model(n, 8, 900 + n)
    fit = run_fit(m)
    ch = stage_chain(m)
    assert torch.equal(ch["loss"], fit["losses"][:1]), (ch["loss"], fit["losses"][:1])
    assert torch.equal(ch["grad"], fit["grad"]), (ch["grad"], fit["grad"])


# ---------------------------------------------------------------------------------------------------------------- b. Cholesky
def gram_matrix(n, NP, kind, cond, seed):
    """A fp32 Gram matrix (d = 2) from hb_gram, and sigma^2: the ill-conditioned setting raises sigma^2 tenfold from 1e-6
    until both fp32 factorisations succeed."""
    g = torch.Generator().manual_seed(seed)
    Xt = torch.full((2, NP), float("nan"))
    Xt[:, :n] = torch.rand(2, n, generator=g) * 2 - 1
    Xt = Xt.to(DEV).contiguous()
    ls, sn2 = (0.5, 8e-4) if cond == "well" else (1.0, 1e-6)
    while True:
        hyp = torch.tensor([sn2, 0.3, 1.0, ls, ls], dtype=torch.float32, device=DEV)
        A = gram(Xt, n, hyp, kind)
        Ls, Lt = A.clone(), A.clone()
        if cholesky(Ls) == 0 and cholesky_tc(Lt, TcWs(NP)) == 0:
            return A, Ls, Lt, sn2
        assert cond == "ill" and sn2 < 1e-2, (n, NP, kind, cond, sn2)
        sn2 *= 10


def chol_c(A, L, n):
    NP = A.shape[0]
    L64 = L.double().tril()
    A64 = A.double()
    low = torch.ones(NP, NP, dtype=torch.bool, device=DEV).tril()
    err = (L64 @ L64.t() - A64).abs()[low]
    B = ((u_tc(NP) + NP * U) * (L64.abs() @ L64.abs().t()))[low]
    i = torch.arange(NP, device=DEV)
    pad = (i[:, None] >= n) & (i[:, None] >= i[None, :])
    assert torch.equal(L.tril()[pad], torch.eye(NP, device=DEV)[pad]), "pad of L is not the identity block"
    return _ratio(err, B)


CHOL_NP = [640, 1152, 2176, 4224]


@pytest.mark.parametrize("cond", ["well", "ill"])
@pytest.mark.parametrize("kind", ["matern32", "rbf"])
@pytest.mark.parametrize("NP", CHOL_NP)
def test_cholesky_tc_backward_error(NP, kind, cond):
    for n in (NP, NP - 37):
        A, Ls, Lt, sn2 = gram_matrix(n, NP, kind, cond, seed=NP + 7 * n + (cond == "ill"))
        c_tc, c_simt = chol_c(A, Lt, n), chol_c(A, Ls, n)
        L64 = Lt.double().tril()
        Lam = torch.linalg.solve_triangular(L64, torch.eye(NP, dtype=F64, device=DEV), upper=False)
        _report(dict(case=f"chol-{kind}-{cond}-NP{NP}-n{n}", sigma2=sn2, cond1_L=cond1(L64, Lam), c_simt=c_simt,
                     c_needed=dict(cholesky_tc=c_tc), c_one_ulp_per_k_step=to_issue_model(c_tc, NP, NP)))
    torch.cuda.empty_cache()


def test_cholesky_tc_reports_leading_minor_like_lapack():
    NP = 1152
    g = torch.Generator().manual_seed(3)
    B = torch.randn(NP, NP, generator=g, dtype=F64)
    A = (B @ B.t() / NP + torch.eye(NP, dtype=F64)).float().to(DEV)
    ws = TcWs(NP)
    assert cholesky_tc(A.clone(), ws) == 0
    for bad in (600, 1000, NP - 1):   # past the first outer block; in the second and the last
        A_bad = A.clone()
        A_bad[bad, bad] = -1.0
        _, info_ref = torch.linalg.cholesky_ex(A_bad.double().cpu())
        A_s = A_bad.clone()
        assert cholesky_tc(A_bad, ws) == cholesky(A_s) == int(info_ref.item()) == bad + 1, bad


# ---------------------------------------------------------------------------------------------------------------- c, d
def check_tri_inverse_tc(L, X):
    NP = L.shape[0]
    L64 = L.double().tril()
    X64 = X.double()
    assert bool((X.triu(1) == 0).all()), "strict upper triangle of L^-1 not zero"
    Lam = torch.linalg.solve_triangular(L64, torch.eye(NP, dtype=F64, device=DEV), upper=False)
    c_fwd = _ratio((X64 - Lam).abs(), u_tc(NP) * (Lam.abs() @ L64.abs() @ X64.abs()))
    c_diag = 0.0
    for b in range(0, NP, GT):
        Lb, Xb = L64[b:b + GT, b:b + GT], X64[b:b + GT, b:b + GT]
        Lamb = torch.linalg.solve_triangular(Lb, torch.eye(GT, dtype=F64, device=DEV), upper=False)
        c_diag = max(c_diag, _ratio((Xb - Lamb).abs(), U * math.sqrt(GT) * (Lamb.abs() @ Lb.abs() @ Xb.abs())))
    return Lam, X64, dict(tri_inverse_tc=c_fwd, base_blocks=c_diag)


def kinv_written(NP):
    """Entries hb_kinv_tc writes: columns < min(NP, round_up(r0 + 128, 256)) of tile row r0."""
    i = torch.arange(NP, device=DEV)
    r0 = i // GT * GT
    lim = ((r0 + GT + 255) // 256 * 256).clamp_max(NP)
    return i[None, :] < lim[:, None]


def check_kinv_tc(X64, Kinv):
    NP = X64.shape[0]
    wr = kinv_written(NP)
    assert bool(torch.isnan(Kinv[~wr]).all()), "hb_kinv_tc wrote outside its output tiles"
    assert bool(lower_tiles(NP)[~wr].logical_not().all())
    ref = X64.t() @ X64
    B = u_tc(NP) * (X64.abs().t() @ X64.abs())
    return _ratio((Kinv.double() - ref).abs()[wr], B[wr])


@pytest.mark.parametrize("cond", ["well", "ill"])
@pytest.mark.parametrize("NP", [384, 640, 1152, 2176, 4224])
def test_tri_inverse_tc_and_kinv_tc(NP, cond):
    for n in (NP, NP - 37):
        _, _, L, sn2 = gram_matrix(n, NP, "matern32", cond, seed=3 * NP + n)
        ws = TcWs(NP)
        X = tri_inverse_tc(L.tril(), ws)
        if n < NP:
            assert torch.equal(X[n:, n:], torch.eye(NP - n, device=DEV)) and bool((X[n:, :n] == 0).all())
        Lam, X64, c = check_tri_inverse_tc(L, X)
        c["kinv_tc"] = check_kinv_tc(X64, kinv_tc(NP, ws))
        _report(dict(case=f"triinv-kinv-{cond}-NP{NP}-n{n}", sigma2=sn2, cond1_L=cond1(L.double().tril(), Lam), c_needed=c,
                     c_one_ulp_per_k_step=dict(tri_inverse_tc=to_issue_model(c["tri_inverse_tc"], NP),
                                               kinv_tc=to_issue_model(c["kinv_tc"], NP))))
    torch.cuda.empty_cache()


def test_rbf_epoch_stages():
    """The stages of the RBF epoch of test_gpu_fit_epoch.py::test_kernel_loss_gradient_against_fp64 (n = 2150, d = 6, init
    hypers): the c of each tensor-core stage on the fit's own A, cond_1(L), and how far the device's K^-1 moves the
    gradient: the contraction of (e.) in fp64 once with the device's K^-1 and once with the exact Lambda^T Lambda of its
    fp32 L, against the epoch's whole error from the fp64 closed form."""
    from tests.test_gpu_fit_epoch import ref_numeric
    m = numeric_model(2150, 6, 41, "rbf")
    ch = stage_chain(m)
    n, NP = m.n, m.NP
    c = dict(cholesky_tc=chol_c(ch["A"], ch["L"], n))
    Lam, X64, ci = check_tri_inverse_tc(ch["L"].tril(), ch["Linv"])
    c.update(ci)
    c["kinv_tc"] = check_kinv_tc(X64, ch["Kinv"])
    L64 = ch["L"].double().tril()
    Kinv64 = Lam.t() @ Lam
    low = lower_tiles(NP)
    rel = dict(kinv_rel_err=float((ch["Kinv"].double() - Kinv64).abs()[low].max() / Kinv64.abs().max()),
               linv_rel_err=float((X64 - Lam).abs().max() / Lam.abs().max()))
    fam = Family(m.XtT, m.y, m.raw, n, m.d, "rbf", noise_guess=m.noise_guess)
    st = dict(hyp=ch["hyp"], alpha=ch["alpha"], scal=ch["scal"])
    g_dev_kinv = contraction_ref(fam, st, ch["Kinv"])[0]
    g_exact_kinv = contraction_ref(fam, st, Kinv64)[0]
    _, g_true = ref_numeric(m, m.raw, "rbf", torch.float64)
    grad_err = float((ch["grad"].double() - g_true).abs().max())
    kinv_move = float((g_dev_kinv - g_exact_kinv).abs().max().cpu())
    # the device's K^-1 accounts for most of the epoch's gradient error (measured 3.3e-5 of 3.7e-5 on an H100)
    assert kinv_move >= 0.5 * grad_err, (kinv_move, grad_err)
    _report(dict(case="rbf-epoch-n2150-d6", cond1_L=cond1(L64, Lam), c_needed=c,
                 c_one_ulp_per_k_step=dict(cholesky_tc=to_issue_model(c["cholesky_tc"], NP, NP),
                                           tri_inverse_tc=to_issue_model(c["tri_inverse_tc"], NP),
                                           kinv_tc=to_issue_model(c["kinv_tc"], NP)),
                 epoch_grad_err=grad_err, grad_move_from_device_kinv=kinv_move, **rel))


# ---------------------------------------------------------------------------------------------------------------- e. gradient
ACC = 83.0


def h_err(r2, kind, d):
    """dh / u of kern_eval_grad at the fp32 r^2 (docstring e.)."""
    _, _, t, _ = kernel_parts(r2, kind)
    h = O.KERNELS[kind].h(r2).abs()
    return h * (E_EX2 + 1.25 * t + 4 + (t + 1) * (E_RSQ + 2.5) + (d + 2) * (1 + t)) + FLUSH


def k_err(r2, kind, d):
    """dk / u of kern_eval(_grad) at the fp32 r^2 (docstring e.)."""
    _, hh, _, _ = kernel_parts(r2, kind)
    return eps_k(r2, kind) + 0.5 * hh.abs() * (d + 2) * r2


class Family:
    """A model as the C ABI takes it, with the parameter layout of kernels.h ModelSpec."""

    def __init__(self, XtT, y, raw, n, d, kind, spec=None, ard=True, Xe=None, num_uniqs=(), emb_sizes=(), warp=0,
                 noise_diag=None, noise_guess=0.01):
        self.XtT, self.y, self.raw, self.n, self.d, self.kind = XtT, y, raw, n, d, kind
        self.spec, self.ard, self.Xe, self.warp, self.noise_diag, self.noise_guess = spec, ard, Xe, warp, noise_diag, noise_guess
        self.num_uniqs, self.emb_sizes = list(num_uniqs), list(emb_sizes)
        self.e, self.De = len(self.num_uniqs), sum(self.emb_sizes)
        self.T = sum(u * q for u, q in zip(self.num_uniqs, self.emb_sizes))
        self.NP = XtT.shape[1]
        nw = 2 * d if warp else 0
        self.n_ls = d if ard else 1
        self.i_wa, self.i_mean, self.i_os, self.i_ls = 1 + self.T, 1 + self.T + nw, 2 + self.T + nw, 3 + self.T + nw
        self.i_le = self.i_ls + self.n_ls
        self.H = 3 + d + (1 if self.e else 0) + nw
        self.h_wa = 3 + d + (1 if self.e else 0)
        assert raw.numel() == self.i_le + (1 if self.e else 0)


def fwd_bwd(m):
    """hb_mll_fwd_bwd (FP32 SIMT) and copies of the fit state it leaves: hyp, Linv, alpha, scal, Zt."""
    lib = _lib.lib()
    n, d, NP = m.n, m.d, m.NP
    wsb = int(lib.hb_fit_workspace_bytes_ex(n, d, m.spec))
    ws = torch.zeros(wsb, dtype=torch.uint8, device=DEV)
    r = m.raw.float().to(DEV).contiguous()
    grad = torch.full((r.numel(),), float("nan"), device=DEV)
    loss = torch.full((1,), float("nan"), device=DEV)
    info = torch.full((1,), -7, dtype=torch.int32, device=DEV)
    _lib.check(lib.hb_mll_fwd_bwd(_p(m.XtT), _p(m.Xe), _p(m.y), n, d, m.spec, _p(r), _lib.KERNEL_IDS[m.kind],
                                  _p(m.noise_diag), NOISE_LB, m.noise_guess, 0.0, _p(grad), _p(loss), _p(info), _p(ws), wsb,
                                  _lib.stream_ptr()), "hb_mll_fwd_bwd")
    torch.cuda.synchronize()
    assert int(info.item()) == 0
    fs = _lib.FitState()
    _lib.check(lib.hb_fit_state_ex(_p(ws), n, d, m.spec, C.byref(fs)), "state")

    def view(p, cnt, dt=torch.float32):
        off = p - ws.data_ptr()
        return ws[off:off + cnt * torch.empty((), dtype=dt).element_size()].view(dt).clone()
    st = dict(hyp=view(fs.hyp, m.H), Linv=view(fs.Linv, NP * NP).view(NP, NP), alpha=view(fs.alpha, NP),
              scal=view(fs.scal, 2, F64), Zt=view(fs.Zt, (d + m.De) * NP).view(d + m.De, NP))
    return grad, loss, st, r


def sqd(Z):
    out = torch.zeros(Z.shape[1], Z.shape[1], dtype=F64, device=DEV)
    for k in range(Z.shape[0]):
        out += (Z[k][:, None] - Z[k][None, :]) ** 2
    return out


def contraction_ref(m, st, Kinv):
    """fp64 gradient and loss of the contraction on the device's own inputs, the per-entry bound (docstring e.) and the
    fp64 numeric r^2."""
    n, d, NP, kind = m.n, m.d, m.NP, m.kind
    hyp = st["hyp"].double()
    sn2, s = float(hyp[0]), float(hyp[2])
    ls32 = st["hyp"][3:3 + d]
    inv = torch.from_numpy((np.float32(1.0) / ls32.cpu().numpy()).astype(np.float32)).to(DEV)
    if m.warp:
        Z = st["Zt"][:d, :n].double()                                 # warp(x) / l as scale_zt_kernel left it
    else:
        Z = (m.XtT[:, :n] * inv[:, None]).double()                    # fl(Xt fl(1 / l)), exact in fp64
    a = st["alpha"][:n].double()
    T = torch.arange(NP, device=DEV) // GT
    Km = Kinv.double()
    Kf = torch.where(T[:, None] >= T[None, :], Km, Km.t())[:n, :n]   # the lower tiles; diagonal tiles in full
    Wm = a[:, None] * a[None, :] - Kf
    ti = T[:n]
    w = torch.where(ti[:, None] > ti[None, :], 2.0, torch.where(ti[:, None] == ti[None, :], 1.0, 0.0)).to(F64)
    r2 = sqd(Z)
    k1, h1 = O.KERNELS[kind].k(r2), O.KERNELS[kind].h(r2)
    dk1, dh1 = U * k_err(r2, kind, d), U * h_err(r2, kind, d)
    one = torch.ones_like(r2)
    k2, h2, dk2, dh2, r2e = one, one, 0 * one, 0 * one, 0 * one
    if m.e:
        E = st["Zt"][d:d + m.De, :n].double()                          # gathered table rows / l_e
        r2e = sqd(E)
        k2, h2 = O.KERNELS["matern32"].k(r2e), O.KERNELS["matern32"].h(r2e)
        dk2, dh2 = U * k_err(r2e, "matern32", m.De), U * h_err(r2e, "matern32", m.De)
    wW = w * Wm
    aWs = (wW * s).abs()
    f = h1 * k2                                                       # the numeric radial factor
    df = dh1 * k2.abs() + h1.abs() * dk2 + U * f.abs()
    G = wW * s * f
    P = m.raw.numel()
    r64 = m.raw.double().to(DEV)
    sig = lambda x: 1.0 / (1.0 + torch.exp(-x))
    inv_n = -1.0 / n
    g = torch.zeros(P, dtype=F64, device=DEV)
    Bg = torch.zeros(P, dtype=F64, device=DEV)
    S, BS = torch.zeros(d, dtype=F64, device=DEV), torch.zeros(d, dtype=F64, device=DEV)
    for k in range(d):
        dz2 = (Z[k][:, None] - Z[k][None, :]) ** 2
        S[k] = (G * dz2).sum()
        BS[k] = U * ACC * (G * dz2).abs().sum() + (aWs * dz2 * df).sum()
    l = hyp[3:3 + d]
    gl, bl = 0.5 * S / l, 0.5 * BS / l
    if d and m.ard:
        g[m.i_ls:m.i_ls + d] = gl * sig(r64[m.i_ls:m.i_ls + d]) * inv_n
        Bg[m.i_ls:m.i_ls + d] = bl * sig(r64[m.i_ls:m.i_ls + d]) * abs(inv_n)
    elif d:
        g[m.i_ls] = gl.sum() * sig(r64[m.i_ls]) * inv_n
        Bg[m.i_ls] = bl.sum() * sig(r64[m.i_ls]) * abs(inv_n)
    if m.warp:   # d K / d a_k: -s h dz_k (dZa_i - dZa_j); chained through a = lo + (hi - lo) sigmoid(raw)
        x = m.XtT[:, :n].double()
        A_, B_ = hyp[m.h_wa:m.h_wa + d, None], hyp[m.h_wa + d:m.h_wa + 2 * d, None]
        dza, dzb, Ea, Eb = warp_derivs(x, A_, B_, inv.double()[:, None])
        for which, (dZ, Ed) in enumerate(((dza, Ea), (dzb, Eb))):
            for k in range(d):
                dz = Z[k][:, None] - Z[k][None, :]
                dd = dZ[k][:, None] - dZ[k][None, :]
                tk = G * dz * dd
                acc = tk.sum()
                bk = U * ACC * tk.abs().sum() + (aWs * (dz * dd).abs() * df).sum() + \
                    U * ((G * dz).abs() * (Ed[k][:, None] + Ed[k][None, :])).sum()
                sg = sig(r64[m.i_wa + which * d + k])
                chain = (10.0 - 0.01) * sg * (1 - sg)
                idx = m.i_wa + which * d + k
                if m.warp == 2:
                    g[idx], Bg[idx] = 0.0, 0.0
                else:
                    g[idx] = -0.5 * acc * chain * inv_n
                    Bg[idx] = 0.5 * bk * chain * abs(inv_n)
    mu0 = math.log(float(np.float32(m.noise_guess)))   # the finish takes noise_guess as a float
    kk = k1 * k2
    dkk = dk1 * k2.abs() + k1.abs() * dk2 + U * kk.abs()
    sum_wk = (wW * kk).sum()
    B_wk = U * ACC * (wW * kk).abs().sum() + (wW.abs() * dkk).sum()
    tr = Wm.diagonal().sum()
    B_tr = U * ACC * Wm.diagonal().abs().sum()
    g_s = 0.5 * sum_wk + (-0.5 / s - 0.5)
    g_n = 0.5 * tr + (-1.0 / sn2 - (math.log(sn2) - mu0) / (0.25 * sn2))
    g[0] = g_n * sig(r64[0]) * inv_n
    Bg[0] = 0.5 * B_tr * sig(r64[0]) * abs(inv_n)
    g[m.i_mean] = a.sum() * inv_n
    Bg[m.i_mean] = 1e-12 * (a.abs().sum() / n)
    g[m.i_os] = g_s * sig(r64[m.i_os]) * inv_n
    Bg[m.i_os] = 0.5 * B_wk * sig(r64[m.i_os]) * abs(inv_n)
    if m.e:
        le = float(hyp[3 + d])
        fe = k1 * h2 * r2e
        dfe = (dk1 * h2.abs() + k1.abs() * dh2 + (m.De + 2) * U * (k1 * h2).abs()) * r2e + 2 * U * fe.abs()
        te = wW * s * fe
        g[m.i_le] = 0.5 * te.sum() / le * sig(r64[m.i_le]) * inv_n
        Bg[m.i_le] = 0.5 * (U * ACC * te.abs().sum() + (aWs * dfe).sum()) / le * sig(r64[m.i_le]) * abs(inv_n)
        # table entries: (1 / (n l_e)) sum over the rows of category u of sum_j G2_ij (E_iq - E_jq), G2 = W s k1 h2
        nt = NP // GT
        acc_e = 8 + 4 + nt + 6
        Wf = Wm * s
        f2 = k1 * h2
        df2 = dk1 * h2.abs() + k1.abs() * dh2 + U * f2.abs()
        G2 = Wf * f2
        R = torch.zeros(m.De, n, dtype=F64, device=DEV)
        BR = torch.zeros(m.De, n, dtype=F64, device=DEV)
        for q in range(m.De):
            dE = E[q][:, None] - E[q][None, :]
            R[q] = (G2 * dE).sum(1)
            BR[q] = U * acc_e * (G2 * dE).abs().sum(1) + (Wf.abs() * dE.abs() * df2).sum(1)
        Xe = m.Xe.long()
        t, q0 = 0, 0
        for c, (nu, es) in enumerate(zip(m.num_uniqs, m.emb_sizes)):
            for u_ in range(nu):
                rows = Xe[:, c] == u_
                for q in range(es):
                    g[1 + t] = R[q0 + q][rows].sum() / (n * le)
                    Bg[1 + t] = BR[q0 + q][rows].sum() / (n * le)
                    t += 1
            q0 += es
    Bg += U * g.abs()
    quad, logdet = float(st["scal"][0]), float(st["scal"][1])
    data = -0.5 * (quad + logdet + n * math.log(2 * math.pi))
    lp_os = 0.5 * math.log(0.5) - 0.5 * math.log(math.pi) - 0.5 * math.log(s) - 0.5 * s
    lp_n = -math.log(sn2 * 0.5 * math.sqrt(2 * math.pi)) - (math.log(sn2) - mu0) ** 2 / 0.5
    loss = -(data + lp_os + lp_n) / n
    return g, Bg, loss, r2


def contraction_problem(n, d, seed, kind, dup, ard=True, noise_diag=False):
    """A numeric model.  dup: rows 2 and n - 1 duplicate rows 1 and 0, and (ARD) feature 0 of rows 3 and 5 lies two ulps
    and one ulp above that of rows 4 and 6 (their other features equal), at lengthscale 2^26: the scaling is exact, so
    the pairs' r^2 are 2^-98 ~ 3.2e-30 and 2^-100 ~ 7.9e-31, either side of Matern-1/2's 1e-30 clamp."""
    g = torch.Generator().manual_seed(seed)
    X = torch.rand(n, d, generator=g, dtype=F64) * 2 - 1
    if dup:
        X[2], X[n - 1], X[3], X[5] = X[1], X[0], X[4], X[6]
    y = torch.sin(3 * X[:, 0]) + 0.3 * X[:, -1] ** 2 + 0.05 * torch.randn(n, generator=g, dtype=F64)
    y = (y - y.mean()) / y.std() if n > 1 else y
    NP = int(_lib.lib().hb_padded_n(n))
    XtT = torch.zeros(d, NP, dtype=torch.float32)
    XtT[:, :n] = X.t().float()
    hp = O.init_hypers(X, y, NOISE_LB, rng=np.random.RandomState(seed))
    raw = hp.pack().float()
    if dup and ard:
        v = torch.tensor(0.75)
        XtT[0, 4] = XtT[0, 6] = v
        XtT[0, 5] = torch.nextafter(v, torch.tensor(2.0))
        XtT[0, 3] = torch.nextafter(XtT[0, 5], torch.tensor(2.0))
        raw[3] = 2.0 ** 26                                            # softplus_f(u) = u above 20: l = 2^26 exactly
    spec = None
    if not ard:
        sp = _lib.ModelSpec(0, 0, None, None, 0)
        spec = (sp, C.byref(sp))
        raw = torch.cat([raw[:3], raw[3:3 + d].mean().reshape(1)])
    nd = None
    if noise_diag:
        nd = (1e-2 * (1 + (X.double() ** 2).sum(1) / d)).float().to(DEV)
    m = Family(XtT.to(DEV).contiguous(), y.float().to(DEV).contiguous(), raw, n, d, kind,
               spec=None if spec is None else spec[1], ard=ard, noise_diag=nd)
    m._keep = spec
    return m


def family_problem(name, kind):
    """Mixed, warped and mixed-warped models set up through hebo_b200.GP."""
    conf = {"mixed": dict(d=4, num_uniqs=[4, 3]), "warp": dict(d=4, warp=True),
            "warp_mixed": dict(d=3, num_uniqs=[3, 5], warp=True),
            "mixed_only": dict(d=0, num_uniqs=[6, 2])}[name]
    import hebo_b200
    n, d = 700, conf.pop("d")
    g = torch.Generator().manual_seed(11 + len(name))
    X = torch.rand(n, max(d, 1), generator=g) * 3 - 1
    nu = conf.get("num_uniqs", [])
    Xe = torch.stack([torch.randint(0, u, (n,), generator=g) for u in nu], 1) if nu else None
    X[2], X[n - 1] = X[1], X[0]                                        # exact duplicates
    if Xe is not None:
        Xe[2], Xe[n - 1] = Xe[1], Xe[0]
    y = torch.sin(2 * X[:, 0]) + 0.3 * X[:, -1] ** 2 + 0.05 * torch.randn(n, generator=g)
    if nu:
        y = y + 0.4 * torch.cos(Xe[:, 0].float() * 1.3)
    np.random.seed(3)
    torch.manual_seed(3)
    gp = hebo_b200.GP(d, len(nu), 1, kernel=kind, lr=0.01, num_epochs=0, noise_lb=NOISE_LB, pred_likeli=False, **conf)
    gp.fit(X if d else None, Xe, y.reshape(-1, 1))
    raw = gp._expand_raw(gp.raw_init.clone())
    es = list(gp.emb_sizes) if nu else []
    m = Family(gp._XtT if d else torch.zeros(0, gp.NP, device=DEV), gp._y_dev, raw, gp.n, d, kind, spec=gp._spec_ptr(),
               ard=True, Xe=gp._Xe_dev, num_uniqs=nu, emb_sizes=es, warp=1 if gp.warp_mode else 0,
               noise_guess=gp.noise_guess)
    m._keep = gp
    return m


def check_contraction(m, case):
    lib = _lib.lib()
    grad, loss, st, r = fwd_bwd(m)
    NP = m.NP
    Kinv = torch.full((NP, NP), float("nan"), device=DEV)
    _lib.check(lib.hb_kinv(_p(st["Linv"]), NP, _p(Kinv), _lib.stream_ptr()), "kinv")
    if m.spec is None and m.noise_diag is None:   # hb_kinv of the state's Linv is the K^-1 the fused call contracted
        g2 = torch.full_like(grad, float("nan"))
        l2 = torch.full_like(loss, float("nan"))
        gws = torch.zeros(int(lib.hb_fit_workspace_bytes(m.n, m.d)), dtype=torch.uint8, device=DEV)
        _lib.check(lib.hb_mll_grad(_p(m.XtT), m.n, m.d, _p(r), _p(st["hyp"]), _lib.KERNEL_IDS[m.kind], _p(Kinv),
                                   _p(st["alpha"]), _p(st["scal"]), m.noise_guess, _p(g2), _p(l2), _p(gws),
                                   _lib.stream_ptr()), "mll_grad")
        torch.cuda.synchronize()
        assert torch.equal(g2, grad) and torch.equal(l2, loss)
    g64, Bg, l64, r2 = contraction_ref(m, st, Kinv)
    err = (grad.double() - g64).abs()
    worst = int(torch.where(err == 0, torch.zeros_like(err), err / Bg).argmax())
    c = dict(gradient=_ratio(err, Bg), loss=abs(float(loss) - l64) / (U * abs(l64) + 1e-12))
    rep = dict(case=case, c_needed=c, max_abs_err=float(err.max()), max_abs_grad=float(g64.abs().max()),
               worst_entry=worst, worst_entry_grad=float(g64[worst]), worst_entry_err=float(err[worst]),
               worst_entry_bound=float(Bg[worst]))
    return rep, r2, st


CONTRACTION = ([(n, 5) for n in (5, 127, 129, 2150, 4097)] + [(513, d) for d in (1, 31, 32, 33, 300)])


@pytest.mark.parametrize("ard", [True, False], ids=["ard", "shared_ls"])
@pytest.mark.parametrize("kind", ["matern32", "matern52", "rbf", "matern12"])
@pytest.mark.parametrize("n,d", CONTRACTION, ids=[f"n{n}_d{d}" for n, d in CONTRACTION])
def test_gradient_contraction_against_fp64(n, d, kind, ard):
    dup = d == 5 and n >= 8
    m = contraction_problem(n, d, seed=31 * n + d, kind=kind, dup=dup, ard=ard)
    rep, r2, st = check_contraction(m, f"contraction-{kind}-{'ard' if ard else 'shared'}-n{n}-d{d}")
    if not ard:
        assert bool((st["hyp"][3:3 + d] == st["hyp"][3]).all())
    if dup and ard:
        r34, r56 = float(r2[3, 4]), float(r2[5, 6])
        rep["near_duplicate_r2"] = [r34, r56]
        assert 0.0 < r56 < 1e-30 < r34, (r34, r56)
    _report(rep)


@pytest.mark.parametrize("kind", ["matern32", "matern12"])
@pytest.mark.parametrize("name", ["noise_diag", "mixed", "mixed_only", "warp", "warp_mixed"])
def test_gradient_contraction_model_families(name, kind):
    """Heteroscedastic noise_diag, mixed models (table entries through emb_scatter_kernel and the embedding lengthscale,
    with and without numeric features) and learned warps (the exponent sweeps on fp64 dZa / dZb)."""
    if name == "noise_diag":
        m = contraction_problem(700, 5, seed=5, kind=kind, dup=True, noise_diag=True)
    else:
        m = family_problem(name, kind)
    rep, _, _ = check_contraction(m, f"contraction-{name}-{kind}")
    _report(rep)
