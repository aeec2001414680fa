"""The GP fit and prediction state past NP = 4224, up to fp32 training matrices larger than 4 GiB, against fp64.

Every per-element check of test_gpu_fit_state.py, test_gpu_fit_epoch.py and test_gpu_posterior_mace.py stops at NP = 4224,
while nothing in the library limits n.  Above that size the doubling levels of launch_tri_inverse, the block-column DAGs of
chol_block64_kernel, the tile-pair decodes of gram_kernel / mll_grad_kernel / linv_resid_kernel / kinv_kernel and the
3xTF32 tile tables take shapes no smaller case reaches, and above NP ~ 32 768 one fp32 [NP, NP] array spans more than
2^32 bytes and each fp16 half of the L^-1 split more than 2^31 bytes.  The workspace is about 44 NP^2 bytes (carve_fit:
L, L^-1, tmp and the tensor-core buffers), 47.9 GB at NP = 32 896.  The module calls the C ABI directly on one workspace
per case: hb_factorize_ex, hb_fit_state_ex, hb_tri_inverse, hb_posterior_mace_ex on both contraction paths, hb_fit_ex
(one epoch at lr = 0: the 3xTF32 loss and gradient) and hb_mll_fwd_bwd (the FP32 SIMT loss and gradient).

1. Dense problems (numeric ARD, inputs in [-1, 1]^d, the oracle's initial hyper-parameters): n = 8192 (NP = 8192, no pad)
   and n = 16 511 (NP = 16 512, one pad row) with Matern-3/2, n = 8319 (NP = 8320 = 2^13 + 128, one pad row: the last
   doubling level of the inverse holds a lone 128-row block) with RBF.
   - The prediction state through test_gpu_fit_state.check_state, unchanged: L L^T against Khat64 on the state's own
     features, hb_tri_inverse and the Newton refinement against the exact inverse of the fp32 factor, alpha and scal
     against fp64 on the same state, the pad, and the operand split bit for bit (test_gpu_posterior_mace).
   - mu and sigma^2 of hb_posterior_mace_ex on both paths against the own-state closed form of
     test_gpu_posterior_mace.own_state with its bounds, for 2048 candidates: 512 training rows, 512 rows 1e-3 from one,
     1024 random rows; the precision guard must flag some rows.
   - The loss and gradient of the 3xTF32 epoch (hb_fit_ex) and of hb_mll_fwd_bwd against the fp64 closed form under the
     bound of test_gpu_fit_epoch.py: |l - l64| <= max(1e-4 max(1, |l64|), 2 |l32 - l64|), |g - g64|_inf <= max(1e-4
     max(|g64|_inf, 0.1), 2 |g32 - g64|_inf), l32 / g32 the same closed form in fp32.  The 3xTF32 RBF gradient exceeds
     it (an expected failure, explained at RBF_TC), as it does at n = 2150 in test_gpu_fit_epoch.py.

2. Clustered problems, NP = 32 768 (n = NP) and NP = 32 896 (n = NP - 1), Matern-3/2, d = 2: clusters of 1000 rows (the
   last one shorter, and none aligned to the 128-row tiles) on a grid with 80 lengthscales between centres and rows within
   3 lengthscales of their centre per coordinate, so two rows of different clusters are at least 74 lengthscales apart.
   There fast_exp's exponent is below -126 and flushes to 0, so every cross-cluster entry of the fp32 Khat is exactly 0:
   Khat is block diagonal, and every stage keeps the off-block entries exactly 0 because every product there has a zero
   factor (the Cholesky updates, the inverse levels, the Newton step, K^-1 and the 3xTF32 splits).
   - Exact zeros: every off-cluster element of L (lower triangle), of hb_tri_inverse's X0, of the refined L^-1 and of
     both fp16 halves of its split is exactly 0, scanned in row chunks.  A truncated offset or a misplaced tile write
     lands a non-zero there.
   - Every cluster per element (check_block): the checks of check_state (a) - (c) on the diagonal block, with the bounds
     of the dense case at the matrix's NP (the sums run over NP columns; the zero terms add no rounding, so the bounds
     hold with room).  The clusters holding the rows where a byte offset crosses 2^31 and 2^32 in an fp32 array and 2^31
     in an fp16 array are printed.
   - Each cluster's log-det against fp64: the factor's 2 sum log L_ii against log det Khat64 of the cluster, within
     sum |Khat64^-1| o |L L^T - Khat64| (the first-order change tr(Khat^-1 dK) of log det under the measured backward error
     dK; c <= C_MAX leaves room for the second order) plus 64 n u64 (sum |log L_ii| + 1) for the fp64 evaluations.
   - The totals: scal (quadratic form and log-det) against the sums of the clusters' fp64 values with the bounds of
     check_state (c) summed, the log-det against the sum of the clusters' fp64 log det Khat64, and the loss and gradient
     of hb_fit_ex and hb_mll_fwd_bwd against the closed form summed over the clusters (every cross-cluster term of the
     gradient has a factor k or dk/dr^2 that is 0) under the dense bound.
   - Posterior: rows on, next to and among the training rows of the clusters that straddle the byte boundaries against the
     cluster-local own-state closed form (the other clusters' K* entries are exactly 0), and rows far from every cluster,
     whose K* row is exactly 0: mu is the constant mean and sigma^2 the outputscale (plus sigma_n^2 with pred_likeli)
     exactly, at y_mean = 0 and y_std = 1.  Both paths.

3. Each case checks the device memory it needs (workspaces from hb_fit_workspace_bytes_ex and hb_posterior_workspace_bytes
   plus the references' buffers) against torch.cuda.mem_get_info() and skips, printing both, when the device lacks it;
   it frees its buffers and prints its wall time and torch.cuda.max_memory_allocated().

The fp64 references run on the device in torch float64; they are references, not the code under test."""
import ctypes as C
import gc
import json
import math
import time

import pytest
import torch

from hebo_b200 import _lib
from oracle import gp_oracle as O
from tests.test_gpu_fit_epoch import NOISE_GUESS, NOISE_LB, Model, numeric_model
from tests.test_gpu_fit_state import (C_MAX, F64, U, U64, _excess, _ratio, check_state, gram_bound, k64, sqdist64,
                                      tri_inverse)
from tests.test_gpu_posterior_mace import check_operand_split, check_own_state, guard_stats, own_state

pytestmark = pytest.mark.gpu

GiB = 1 << 30
CLUSTER = 1000
LS = 0.05                       # lengthscale of the clustered problems
SPACING = 80 * LS               # centre to centre
SPREAD = 3 * LS                 # per coordinate, about the centre


@pytest.fixture
def case(request):
    """Frees the cache, checks free memory (case.need(bytes, what)), prints the case's time and peak memory at the end."""
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()

    class Case:
        def need(self, nbytes, what):
            free, _ = torch.cuda.mem_get_info()
            if free < nbytes + 2 * GiB:
                pytest.skip(f"needs {nbytes / GiB:.1f} GiB ({what}) + 2 GiB margin, {free / GiB:.1f} GiB free")
            print(f"\n[{request.node.name}] needs {nbytes / GiB:.1f} GiB ({what}), {free / GiB:.1f} GiB free")
    c = Case()
    t0 = time.perf_counter()
    yield c
    torch.cuda.synchronize()
    print(f"\n[{request.node.name}] {time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / GiB:.2f} GiB")
    gc.collect()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------- C ABI
def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class State:
    """The prediction state hb_factorize_ex left in workspace `ws`, as views of it, under the attribute names the checkers
    of test_gpu_fit_state.py and test_gpu_posterior_mace.py read from a GP."""

    def __init__(self, m, kind, ws, jitter, pred_likeli=True, y_mean=0.0, y_std=1.0):
        fs = _lib.FitState()
        _lib.check(_lib.lib().hb_fit_state_ex(_p(ws), m.n, m.d, None, C.byref(fs)), "hb_fit_state_ex")

        def view(p, cnt, dt=torch.float32):
            off = p - ws.data_ptr()
            return ws[off:off + cnt * torch.empty((), dtype=dt).element_size()].view(dt)
        n, d, NP = m.n, m.d, m.NP
        self.n, self.d, self.NP, self.De, self.num_enum, self.warp_mode, self.noise_diag = n, d, NP, 0, 0, 0, None
        self.kernel, self.kern_id, self.jitter_used, self.pred_likeli = kind, _lib.KERNEL_IDS[kind], jitter, pred_likeli
        self._y_mean, self._y_std = float(y_mean), float(y_std)
        self._XtT, self._y_dev = m.XtT, m.y
        self._x_mul = torch.ones(d, device="cuda")
        self._x_add = torch.zeros(d, device="cuda")
        self.hyp_dev = view(fs.hyp, 3 + d)
        self.hyp = self.hyp_dev.cpu()
        self.L_dev = view(fs.L, NP * NP).view(NP, NP)
        self.Linv_dev = view(fs.Linv, NP * NP).view(NP, NP)
        self.Linv_hi_dev = view(fs.Linv_hi, NP * NP // 2)
        self.Linv_lo_dev = view(fs.Linv_lo, NP * NP // 2 + 1)       # the split's scale follows h1
        self.alpha_dev = view(fs.alpha, NP)
        self.scal_dev = view(fs.scal, 2, F64)
        self.Zt_dev = view(fs.Zt, d * NP).view(d, NP)


class Block:
    """Rows [a, b) of a clustered state as a model of its own, for own_state: their features, alpha and diagonal block of
    L^-1; NP stays the matrix's (the contractions sum over all NP columns, of which only the cluster's are non-zero)."""

    def __init__(self, st, a, b):
        for k in ("d", "NP", "De", "num_enum", "warp_mode", "kernel", "pred_likeli", "_y_mean", "_y_std", "_x_mul", "_x_add",
                  "hyp_dev", "hyp"):
            setattr(self, k, getattr(st, k))
        self.n = b - a
        self.Zt_dev = st.Zt_dev[:, a:b].contiguous()
        self.alpha_dev = st.alpha_dev[a:b].contiguous()
        self.Linv_dev = st.Linv_dev[a:b, a:b].contiguous()


def workspace_bytes(m):
    return int(_lib.lib().hb_fit_workspace_bytes_ex(m.n, m.d, None))


def factorize(m, raw, ws):
    jit = C.c_float(-1.0)
    st = _lib.lib().hb_factorize_ex(_p(m.XtT), None, _p(m.y), m.n, m.d, None, _p(raw.float().cuda().contiguous()), m.kern,
                                    None, NOISE_LB, C.byref(jit), _p(ws), ws.numel(), _lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == _lib.HB_OK, st
    return float(jit.value)


def tc_loss_grad(m, raw, ws):
    """hb_fit_ex, one epoch at lr = 0 without Langevin draws: the 3xTF32 loss and gradient at raw (raw stays put)."""
    r = raw.float().cuda().contiguous().clone()
    losses = (C.c_float * 1)()
    st = _lib.lib().hb_fit_ex(_p(m.XtT), None, _p(m.y), m.n, m.d, None, _p(r), m.kern, None, NOISE_LB, m.noise_guess, 0.0, 1,
                              None, losses, _p(ws), ws.numel(), _lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == _lib.HB_OK, st
    assert torch.equal(r.cpu(), raw.float().cpu())
    fs = _lib.FitState()
    _lib.check(_lib.lib().hb_fit_state_ex(_p(ws), m.n, m.d, None, C.byref(fs)), "hb_fit_state_ex")
    off = fs.grad - ws.data_ptr()
    return float(losses[0]), ws[off:off + 4 * m.P].view(torch.float32).double().cpu()


def simt_loss_grad(m, raw, ws):
    grad = torch.full((m.P,), float("nan"), device="cuda")
    loss = torch.full((1,), float("nan"), device="cuda")
    info = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().hb_mll_fwd_bwd(_p(m.XtT), None, _p(m.y), m.n, m.d, None, _p(raw.float().cuda().contiguous()), m.kern,
                                         None, NOISE_LB, m.noise_guess, 0.0, _p(grad), _p(loss), _p(info), _p(ws), ws.numel(),
                                         _lib.stream_ptr()), "hb_mll_fwd_bwd")
    torch.cuda.synchronize()
    assert int(info.item()) == 0
    return float(loss.item()), grad.double().cpu()


def posterior(st, Xs, path):
    """(mu, var) of hb_posterior_mace_ex over all rows of Xs in one chunk; NaN-filled workspace and outputs."""
    lib = _lib.lib()
    m = Xs.shape[0]
    wsb = int(lib.hb_posterior_workspace_bytes(st.n, st.d, m))
    ws = torch.full((wsb // 4,), float("nan"), device="cuda")
    mu, var = (torch.full((m,), float("nan"), device="cuda") for _ in range(2))
    hi, lo = (st.Linv_hi_dev, st.Linv_lo_dev) if path == "tensor" else (None, None)
    s = lib.hb_posterior_mace_ex(_p(Xs), None, m, 0, st.n, st.d, None, None, None, _p(st._x_mul), _p(st._x_add), _p(st.Zt_dev),
                                 _p(st.alpha_dev), _p(st.Linv_dev), _p(hi), _p(lo), _p(st.hyp_dev), st.kern_id, st._y_mean,
                                 st._y_std, int(st.pred_likeli), 0.3, 2.0, 1e-4, None, None, 0, None, _p(mu), _p(var), _p(ws),
                                 wsb, m, _lib.stream_ptr())
    torch.cuda.synchronize()
    assert s == _lib.HB_OK, s
    return mu, var


def posterior_bytes(m, rows):
    return int(_lib.lib().hb_posterior_workspace_bytes(m.n, m.d, rows))


# ---------------------------------------------------------------------------------------------------------------- fp64 MLL
def mll_terms(Z, r, s, sn2, kind, block=256):
    """The data terms of oracle.gp_oracle.neg_mll_closed_form on the device of Z [n, d] = Xt / l, r = y - c: quadratic
    form, log-det, and the sums the gradient is assembled from (tr(W dK/dtheta) before the chain rule), in Z's dtype.
    Returns None when the Cholesky fails in that dtype."""
    n, d = Z.shape
    dt, dev = Z.dtype, Z.device
    kern = O.KERNELS[kind]
    r2 = torch.empty(n, n, dtype=dt, device=dev)
    for i0 in range(0, n, block):
        r2[i0:i0 + block] = ((Z[i0:i0 + block, None, :] - Z[None]) ** 2).sum(-1)
    k = kern.k(r2)
    Kh = s * k
    Kh.diagonal().add_(sn2)
    L, info = torch.linalg.cholesky_ex(Kh)
    del Kh
    if int(info) != 0:
        return None
    logdet = 2.0 * torch.log(L.diagonal()).sum()
    Linv = torch.linalg.solve_triangular(L, torch.eye(n, dtype=dt, device=dev), upper=False)
    del L
    W = -(Linv.t() @ Linv)
    del Linv
    alpha = -(W @ r)
    quad = r @ alpha
    W += torch.outer(alpha, alpha)
    gs = 0.5 * (W * k).sum()
    del k
    gn = 0.5 * W.diagonal().sum()
    G = W * kern.h(r2) * s
    del W, r2
    gls = torch.zeros(d, dtype=dt, device=dev)
    for i0 in range(0, n, block):
        gls += torch.einsum("ij,ijk->k", G[i0:i0 + block], (Z[i0:i0 + block, None, :] - Z[None]) ** 2)
    return dict(n=n, quad=quad, logdet=logdet, gls=gls, gs=gs, gn=gn, gc=alpha.sum())


def mll_sum(parts):
    out = dict(parts[0])
    for p in parts[1:]:
        for k in out:
            out[k] = out[k] + p[k]
    return out


def mll_assemble(T, raw, noise_guess=NOISE_GUESS, noise_lb=NOISE_LB):
    """Loss and gradient of neg_mll_closed_form from (summed) data terms T: priors, chain rule, 1 / n (same dtype)."""
    dt = T["quad"].dtype
    hp = O.Hypers.unpack(raw.to(T["quad"].device).to(dt), noise_lb)
    s, sn2, ls, n = hp.outputscale, hp.noise, hp.lengthscale, T["n"]
    sig0, mu0 = 0.5, math.log(noise_guess)
    g_ls = 0.5 * T["gls"] / ls
    g_s = T["gs"] + (-0.5 / s - 0.5)
    g_n = T["gn"] + (-1.0 / sn2 - (torch.log(sn2) - mu0) / (sig0 ** 2 * sn2))
    sg = torch.sigmoid
    grad = torch.cat([(g_n * sg(hp.raw_noise)).reshape(1), T["gc"].reshape(1), (g_s * sg(hp.raw_os)).reshape(1),
                      g_ls * sg(hp.raw_ls)]) * (-1.0 / n)
    data = -0.5 * (T["quad"] + T["logdet"] + n * math.log(2.0 * math.pi))
    lp_os = 0.5 * math.log(0.5) - math.lgamma(0.5) - 0.5 * torch.log(s) - 0.5 * s
    lp_n = -torch.log(sn2 * sig0 * math.sqrt(2.0 * math.pi)) - (torch.log(sn2) - mu0) ** 2 / (2 * sig0 ** 2)
    return float(-(data + lp_os + lp_n) / n), grad.double().cpu()


def mll_reference(m, raw, kind, dtype, rows=None):
    """(loss, grad) of the closed form in `dtype` on the device, summed over the row ranges `rows` (the whole set when
    None); (inf, None) when the Cholesky fails in that dtype."""
    hp = O.Hypers.unpack(raw.to(dtype).to(m.XtT.device), NOISE_LB)
    X = m.XtT[:, :m.n].t().to(dtype)
    ls, r = hp.lengthscale, m.y[:m.n].to(dtype) - hp.mean
    s, sn2 = hp.outputscale, hp.noise
    parts = []
    for a, b in (rows or [(0, m.n)]):
        t = mll_terms(X[a:b] / ls, r[a:b], s, sn2, kind)
        if t is None:
            return math.inf, None
        parts.append(t)
    return mll_assemble(mll_sum(parts), raw)


def check_mll(what, got, ref64, ref32):
    """test_gpu_fit_epoch.check's bound for one path."""
    (l, g), (l64, g64), (l32, g32) = got, ref64, ref32
    gmax = float(g64.abs().max())
    el, ef = abs(l - l64), abs(l32 - l64)
    eg = float((g - g64).abs().max())
    egf = math.inf if g32 is None else float((g32 - g64).abs().max())
    rep = dict(case=what, loss_err=el, loss_fp32_err=ef, grad_err=eg, grad_fp32_err=egf, grad_inf=gmax)
    print(json.dumps(rep))
    assert el <= max(1e-4 * max(1.0, abs(l64)), 2 * ef), rep
    assert eg <= max(1e-4 * max(gmax, 0.1), 2 * egf), rep


# ---------------------------------------------------------------------------------------------------------------- 1. dense
DENSE = [(8192, 8, "matern32"), (8319, 6, "rbf"), (16511, 8, "matern32")]


def dense_candidates(m, seed):
    """512 training rows, 512 training rows moved by 1e-3 per coordinate, 1024 rows in [-1.2, 1.2]^d."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    X = m.XtT[:, :m.n].t()
    idx = torch.randperm(m.n, generator=g, device="cuda")[:1024]
    near = X[idx[512:]] + 1e-3 * (torch.rand(512, m.d, generator=g, device="cuda") * 2 - 1)
    rand = torch.rand(1024, m.d, generator=g, device="cuda") * 2.4 - 1.2
    return torch.cat([X[idx[:512]], near, rand]).contiguous()


@pytest.mark.parametrize("n,d,kind", DENSE, ids=[f"n{n}_{k}" for n, d, k in DENSE])
def test_dense_state_and_posterior_against_fp64(case, n, d, kind):
    m = numeric_model(n, d, 900 + n, kind)
    NP = m.NP
    assert NP == _lib.lib().hb_padded_n(n) and NP > 4224
    wsb = workspace_bytes(m)
    case.need(wsb + posterior_bytes(m, 2048) + 12 * 8 * NP * NP,
              f"workspace {wsb / GiB:.1f} GiB + posterior workspace + twelve fp64 [NP, NP] references")
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    jit = factorize(m, m.raw, ws)
    st = State(m, kind, ws, jit, pred_likeli=True, y_mean=-0.2, y_std=1.3)
    check_state(f"dense-{kind}-n{n}-NP{NP}", st, None, None, None, fp64=False)
    check_operand_split(st)
    # posterior, both paths
    Xs = dense_candidates(m, n)
    ref = own_state(st, Xs, None)
    got = {}
    for path in ("tensor", "simt"):
        guard_stats(reset=True)
        got[path] = posterior(st, Xs, path)
        seen, flagged = guard_stats(reset=True)
        print(json.dumps(dict(case=f"dense-{kind}-n{n}", path=path, rows=seen, guard_flagged=flagged)))
        if path == "tensor":
            assert seen == Xs.shape[0] and flagged > 0, (seen, flagged)
        check_own_state(f"dense-{kind}-n{n}-NP{NP}", st, Xs, None, (None,) + got[path], path, ref=ref)
    assert torch.equal(got["tensor"][0], got["simt"][0]), "mu depends on the contraction path"


RBF_TC = pytest.mark.xfail(strict=True, reason=(
    "3xTF32 epoch outside the bound for RBF at n = 8319, d = 6, init hypers (H100): gradient error 3.9e-4 of |g|inf 0.20 "
    "against 6.0e-5 on the FP32 SIMT path and an fp32 floor of 1.3e-4; the loss (1.8e-5 against a floor of 8.2e-5) and "
    "every state, split and posterior check of this model pass.  The finding of "
    "test_gpu_fit_epoch.py::test_kernel_loss_gradient_against_fp64[rbf] at n = 2150, grown with n: the tensor-core "
    "K^-1 = U U^T carries one truncation per wgmma instruction, and the RBF gradient contracts it with W"))
DENSE_MLL = [pytest.param(n, d, kind, path, marks=RBF_TC if (kind, path) == ("rbf", "3xtf32") else (),
                          id=f"n{n}_{kind}_{path}") for n, d, kind in DENSE for path in ("simt", "3xtf32")]


@pytest.mark.parametrize("n,d,kind,path", DENSE_MLL)
def test_dense_loss_gradient_against_fp64(case, n, d, kind, path):
    """hb_mll_fwd_bwd (simt) or one hb_fit_ex epoch at lr = 0 (3xtf32) on the dense problems, against the fp64 closed
    form under test_gpu_fit_epoch.py's bound."""
    m = numeric_model(n, d, 900 + n, kind)
    wsb = workspace_bytes(m)
    case.need(max(wsb, 6 * 8 * m.NP * m.NP), f"workspace {wsb / GiB:.1f} GiB, then six fp64 [NP, NP] references")
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    got = (simt_loss_grad if path == "simt" else tc_loss_grad)(m, m.raw, ws)
    del ws
    gc.collect()
    torch.cuda.empty_cache()
    check_mll(f"dense-{kind}-n{n}-NP{m.NP} {path}", got, mll_reference(m, m.raw, kind, F64),
              mll_reference(m, m.raw, kind, torch.float32))


# ---------------------------------------------------------------------------------------------------------------- 2. clusters
def cluster_ids(n, NP, size=CLUSTER, device="cuda"):
    """Cluster of every index: i // size for training rows, a distinct negative id for each pad row (its identity block)."""
    i = torch.arange(NP, device=device)
    return torch.where(i < n, i // size, -1 - i)


def cluster_ranges(n, size=CLUSTER):
    return [(a, min(a + size, n)) for a in range(0, n, size)]


def centres(nc, device="cuda"):
    side = math.ceil(math.sqrt(nc))
    c = torch.arange(nc, device=device)
    g = torch.stack([c % side, c // side], 1).double() - (side - 1) / 2
    return g * SPACING


def clustered_model(n, seed, kind="matern32"):
    """d = 2 rows around a grid of centres (module docstring 2.), targets a smooth function of the offset from the
    centre plus noise, and raw hyper-parameters s = 1, sigma_n^2 = 0.01, c = 0.1, l = LS."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    NP = int(_lib.lib().hb_padded_n(n))
    ctr = centres(len(cluster_ranges(n)))
    cid = torch.arange(n, device="cuda") // CLUSTER
    off = (torch.rand(n, 2, generator=g, device="cuda", dtype=F64) * 2 - 1) * SPREAD
    X = (ctr[cid] + off).float()
    XtT = torch.zeros(2, NP, device="cuda")
    XtT[:, :n] = X.t()
    y = torch.sin(off[:, 0] / LS) + 0.5 * torch.cos(0.7 * off[:, 1] / LS) + 0.1 * torch.randn(n, generator=g, device="cuda",
                                                                                               dtype=F64)
    inv = lambda v: float(O.inv_softplus(torch.tensor(v, dtype=F64)))
    raw = torch.tensor([inv(0.01 - NOISE_LB), 0.1, inv(1.0), inv(LS), inv(LS)])
    return Model(XtT, y.float().contiguous(), raw, n, _lib.KERNEL_IDS[kind])


def off_cluster_nonzeros(M, cid, lower=False, chunk_bytes=1 << 28):
    """(count, first (row, col)) of non-zero elements of M [NP, NP] (fp32 or fp16) whose row and column lie in
    different clusters (lower triangle only with `lower`), scanned in row chunks on M's device."""
    NP = M.shape[0]
    rows = max(1, chunk_bytes // (4 * NP))
    cols = torch.arange(NP, device=M.device)
    count, first = 0, None
    for r0 in range(0, NP, rows):
        r1 = min(NP, r0 + rows)
        bad = (M[r0:r1].float() != 0) & (cid[r0:r1, None] != cid[None, :])
        if lower:
            bad &= cols[None, :] <= torch.arange(r0, r1, device=M.device)[:, None]
        k = int(bad.sum())
        if k and first is None:
            i = int(bad.reshape(-1).nonzero()[0])
            first = (r0 + i // NP, i % NP)
        count += k
    return count, first


def khat_block(Z, hyp, kind, jitter=0.0):
    """Khat64 and its Gram bound on the fp32 features Z [d, nb] of one cluster (test_gpu_fit_state.khat64, numeric only)."""
    hyp = hyp.double()
    sn2, s = float(hyp[0]), float(hyp[2])
    r2 = sqdist64(Z.double()) if Z.is_cuda else _sqdist64_any(Z.double())
    K = s * k64(r2, kind)
    B = s * gram_bound(r2, Z.shape[0], kind) + 2 * U * K.abs()
    K.diagonal().fill_(s + sn2 + jitter)
    B.diagonal().copy_(3 * U * K.diagonal().abs())
    return K, B


def _sqdist64_any(Z):
    return ((Z[:, :, None] - Z[:, None, :]) ** 2).sum(0)


def check_block(L, X0, X, Kh, Bg, r, alpha, NP):
    """check_state (a) - (c) on one diagonal block: L, X0 (hb_tri_inverse), X (the refined L^-1) [nb, nb] fp32, Khat64
    and its Gram bound, r = fl32(y - c) and alpha [nb]; sqrt(NP) and NP of the whole matrix.  Returns (c dict, sums for
    the totals)."""
    nb = L.shape[0]
    dev = L.device
    sq = math.sqrt(NP)
    c = {}
    L64 = L.double().tril()
    low = torch.ones(nb, nb, dtype=torch.bool, device=dev).tril()
    LLt = L64 @ L64.t()
    c["LLt"] = _excess((LLt - Kh).abs()[low], Bg[low], U * sq * (L64.abs() @ L64.abs().t())[low])
    assert bool((X0.triu(1) == 0).all()) and bool((X.triu(1) == 0).all()), "strict upper triangle of L^-1 not zero"
    I = torch.eye(nb, dtype=F64, device=dev)
    Lam = torch.linalg.solve_triangular(L64, I, upper=False)
    X064, X64 = X0.double(), X.double()
    P = Lam.abs() @ L64.abs() @ X064.abs()
    c["tri_inverse_fwd"] = _ratio((X064 - Lam).abs(), U * sq * P)
    c["tri_inverse_resid"] = _ratio((X064 @ L64 - I).abs(), U * sq * (P @ L64.abs()))
    R = (I - L64 @ X064).tril().float().double()
    B1 = U * sq * (X064.abs() @ R.abs())
    c["refine"] = _excess((X64 - (X064 + X064 @ R)).abs(), U * X64.abs(), B1)
    E0 = X064 - Lam
    c["refined_vs_exact"] = _excess((X64 - Lam).abs(), U * X64.abs() + (E0 @ L64 @ E0).abs(), B1)
    r = r.double()
    v = X64 @ r
    a64 = X64.t() @ v
    Xr = X64.abs() @ r.abs()
    S = X64.abs().t() @ Xr
    al = alpha.double()
    c["alpha"] = _ratio((al - a64).abs(), U * a64.abs() + 4 * NP * U64 * S)
    aL = Lam.t() @ (Lam @ r)
    E = (X64 - Lam).abs()
    c["alpha_vs_exact_L"] = _ratio((al - aL).abs(), U * aL.abs() + 4 * NP * U64 * S + E.t() @ v.abs()
                                   + Lam.abs().t() @ (E @ r.abs()))
    lg = torch.log(L64.diagonal())
    ld = 2 * lg.sum()
    Lt = torch.linalg.cholesky(Kh)
    ld64 = 2 * torch.log(Lt.diagonal()).sum()
    Bld64 = float((torch.cholesky_inverse(Lt).abs() * (LLt - Kh).abs()).sum()) + 64 * nb * U64 * (float(lg.abs().sum()) + 1)
    c["logdet_vs_fp64"] = float((ld - ld64).abs()) / Bld64
    sums = dict(q=float((v * v).sum()), Bq=4 * NP * U64 * float((v.abs() * Xr).sum()), ld=float(ld),
                lgabs=float(lg.abs().sum()), ld64=float(ld64), Bld64=Bld64)
    return c, sums


def check_totals(scal, sums, n, NP):
    """scal against the sums over the clusters with the bounds of check_state (c) summed; the log-det also against the
    clusters' fp64 log det Khat64."""
    q = sum(s["q"] for s in sums)
    Bq = sum(s["Bq"] for s in sums) + n * U64 * q
    ld = sum(s["ld"] for s in sums)
    Bld = 4 * n * U64 * (sum(s["lgabs"] for s in sums) + 1)
    ld64 = sum(s["ld64"] for s in sums)
    scal = [float(x) for x in scal]
    return dict(quad=abs(scal[0] - q) / Bq, logdet=abs(scal[1] - ld) / Bld,
                logdet_total_vs_fp64=abs(scal[1] - ld64) / (sum(s["Bld64"] for s in sums) + Bld))


def boundary_rows(NP):
    """{what: first row whose elements reach that byte offset} for the offsets an [NP, NP] array actually crosses."""
    out = {}
    for what, esize, lim in (("fp32_2^31", 4, 1 << 31), ("fp32_2^32", 4, 1 << 32), ("fp16_2^31", 2, 1 << 31)):
        e = lim // esize
        if NP * NP > e:
            out[what] = e // NP
    return out


CLUSTERED = [32768, 32895]


@pytest.mark.parametrize("n", CLUSTERED, ids=[f"n{n}" for n in CLUSTERED])
def test_clustered_state_past_4gib_per_matrix(case, n):
    kind = "matern32"
    m = clustered_model(n, seed=n)
    NP, lib = m.NP, _lib.lib()
    ranges = cluster_ranges(n)
    wsb = workspace_bytes(m)
    rows_post = 2048
    case.need(wsb + posterior_bytes(m, rows_post) + 5 * 4 * NP * NP,
              f"workspace {wsb / GiB:.1f} GiB + posterior workspace + five fp32 [NP, NP] buffers")
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    jit = factorize(m, m.raw, ws)
    assert jit == 0.0
    st = State(m, kind, ws, jit, pred_likeli=True)
    cid = cluster_ids(n, NP)
    bnd = boundary_rows(NP)
    rep = dict(case=f"clustered-n{n}-NP{NP}", clusters=len(ranges), workspace_bytes=wsb,
               boundary_clusters={k: int(r // CLUSTER) for k, r in bnd.items()})
    # exact zeros: L, the split, then X0 and the refined L^-1
    zeros = dict(L=off_cluster_nonzeros(st.L_dev, cid, lower=True),
                 Linv=off_cluster_nonzeros(st.Linv_dev, cid),
                 Linv_hi=off_cluster_nonzeros(st.Linv_hi_dev.view(torch.float16)[:NP * NP].view(NP, NP), cid),
                 Linv_lo=off_cluster_nonzeros(st.Linv_lo_dev[:NP * NP // 2].view(torch.float16).view(NP, NP), cid))
    check_operand_split(st)
    gc.collect()
    torch.cuda.empty_cache()
    X0 = tri_inverse(st.L_dev)
    zeros["X0"] = off_cluster_nonzeros(X0, cid)
    rep["off_cluster_nonzeros"] = zeros
    assert all(v[0] == 0 for v in zeros.values()), rep
    # every cluster per element
    hyp = st.hyp_dev
    r = (m.y[:n] - hyp[1]).float()
    worst, sums, per = {}, [], {}
    for ci, (a, b) in enumerate(ranges):
        Kh, Bg = khat_block(st.Zt_dev[:, a:b], hyp, kind)
        c, s = check_block(st.L_dev[a:b, a:b], X0[a:b, a:b], st.Linv_dev[a:b, a:b], Kh, Bg, r[a:b], st.alpha_dev[a:b], NP)
        sums.append(s)
        for k, v in c.items():
            worst[k] = max(worst.get(k, 0.0), v)
        if ci in rep["boundary_clusters"].values() or ci == len(ranges) - 1:
            per[ci] = c
    del X0
    gc.collect()
    torch.cuda.empty_cache()
    assert bool((st.alpha_dev[n:] == 0).all()), "alpha pad entries not zero"
    worst.update(check_totals(st.scal_dev.cpu(), sums, n, NP))
    rep.update(c_needed=worst, boundary_and_last_clusters=per)
    print(json.dumps(rep))
    assert max(worst.values()) <= C_MAX, rep
    # posterior: rows inside the clusters at the byte boundaries and the last cluster, and rows far from every cluster
    check_clustered_posterior(st, m, rep["boundary_clusters"], ranges, rows_post)
    del st
    gc.collect()
    torch.cuda.empty_cache()
    # loss and gradient totals
    tc = tc_loss_grad(m, m.raw, ws)
    simt = simt_loss_grad(m, m.raw, ws)
    del ws
    gc.collect()
    torch.cuda.empty_cache()
    r64 = mll_reference(m, m.raw, kind, F64, ranges)
    r32 = mll_reference(m, m.raw, kind, torch.float32, ranges)
    check_mll(f"clustered-n{n}-NP{NP} simt", simt, r64, r32)
    check_mll(f"clustered-n{n}-NP{NP} 3xtf32", tc, r64, r32)


def check_clustered_posterior(st, m, boundary_clusters, ranges, rows):
    g = torch.Generator(device="cuda").manual_seed(m.n + 5)
    pick = sorted(set(boundary_clusters.values()) | {len(ranges) - 1})
    per = (rows - 256) // len(pick)
    X = m.XtT[:, :m.n].t()
    ctr = centres(len(ranges)).float()
    blocks, sel = [], []
    for ci in pick:
        a, b = ranges[ci]
        idx = a + torch.randperm(b - a, generator=g, device="cuda")[:per // 2]
        k = per // 4
        near = X[idx[k:]] + 0.1 * LS * (torch.rand(idx.numel() - k, 2, generator=g, device="cuda") * 2 - 1)
        box = ctr[ci] + (torch.rand(per - idx.numel(), 2, generator=g, device="cuda") * 2 - 1) * 1.2 * SPREAD
        blocks.append(torch.cat([X[idx[:k]], near, box]))
        sel.append((ci, a, b))
    lo, hi = ctr.min(0).values, ctr.max(0).values
    far = hi + SPACING + torch.rand(256, 2, generator=g, device="cuda") * SPACING      # >= 77 lengthscales from any row
    far[::2] = lo - SPACING - torch.rand(128, 2, generator=g, device="cuda") * SPACING
    Xs = torch.cat(blocks + [far]).contiguous()
    hyp = st.hyp.float()
    for pl in (True, False):
        st.pred_likeli = pl
        got = {path: posterior(st, Xs, path) for path in ("tensor", "simt")}
        assert torch.equal(got["tensor"][0], got["simt"][0]), "mu depends on the contraction path"
        vfar = (hyp[2] + hyp[0]) if pl else hyp[2]
        for path, (mu, var) in got.items():
            f0 = Xs.shape[0] - 256
            assert bool((mu[f0:] == float(hyp[1])).all()), (path, pl, "mu of rows far from every cluster")
            assert bool((var[f0:] == float(vfar)).all()), (path, pl, "var of rows far from every cluster")
            r0 = 0
            for (ci, a, b), blk in zip(sel, blocks):
                loc = Block(st, a, b)
                part = (None, mu[r0:r0 + blk.shape[0]], var[r0:r0 + blk.shape[0]])
                check_own_state(f"clustered-n{m.n}-cluster{ci}-pl{int(pl)}", loc, blk.contiguous(), None, part, path)
                r0 += blk.shape[0]
    st.pred_likeli = True
