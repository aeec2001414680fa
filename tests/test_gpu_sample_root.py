"""The joint posterior samplers hb_sample_y (GP.sample_y) and hb_sample_y_batch (GP.sample_y_batch) read out exactly and
checked against fp64, and hb_cholesky beyond one outer block.

Identity draws make the samplers deterministic matrix outputs.  With y_mean = 0, y_std = 1, alpha = 0 and the mean
constant hyp[1] = 0 -- alpha and hyp[1] feed only the mean: the K* alpha partials of kstar_kernel and the constant of
sample_apply_kernel / sample_batch_kernel -- the mean of every row is an exact 0.  Then z = I_m makes
sample_apply_kernel write out[j][i] = R[i][j] for i >= j bit for bit: one fmaf term is R[i][j] * 1, every other term
adds an exact +-0, and the scalings are by 1 and + 0.  hb_sample_y_batch with z = e_j gives column j of the root of the
distinct rows in the same way.  The root R is then checked three ways:

  1. against the GP's own fp32 state promoted to fp64 (Zt, Linv, hyp; candidate features scaled in fp64 from the raw
     rows), so that the accuracy of the fit drops out:  C' = K** - V V^T (+ sigma_n^2 I with pred_likeli), V = K* Linv^T,
     and the backward error  E = |R R^T - C' - jitter I| <= c u B  elementwise, u = 2^-24, with the probabilistic
     (square-root growth) rounding model
         B_ij = sqrt(NP) (w_i |v_j| + |v_i| w_j + |v_i| |v_j|) + sqrt(mp) (|R| |R|^T)_ij + s',
     |v_i| = ||V_i||, w_i = || |K*_i| |Linv|^T ||, s' = s (+ sigma_n^2 with pred_likeli): the rounding of V, of the
     rank-n update, of the Cholesky and of the O(s) kernel values.  max(E / (u B)) -- the c a case needs -- is printed
     for every case; c = 4 is required (on an H100 the cases below need at most 1.4).  The s' term assumes O(u)
     relative kernel values; candidate features of large norm (|z| >> r) round by more than that in fp32, so a model
     with very short lengthscales needs a larger c without being wrong;
  2. against the true fp64 posterior at the same hyper-parameters (training features, factorisation and solves in fp64):
     sqrt of the variance within 1e-4 relative (2e-4 on rows whose variance has cancelled below 0.02 s, the criteria of
     test_gpu_fullsize.py), the correlations of R R^T - jitter I within 2e-4 on the other rows, and the mean of a z = 0
     draw within 1e-4 max(|mu|, y_std);
  3. structurally: a positive diagonal, exact zeros above it, nothing written past the [m, m] output.

The fp64 references run on the device in torch float64; they are references, not the code under test."""
import ctypes as C
import json
import math

import numpy as np
import pytest
import torch

from hebo_b200 import GP, _lib
from oracle import gp_oracle as O
from tests.util import seeded_problem

DEV = torch.device("cuda")
U = 2.0 ** -24
C_MAX = 4.0             # the c of the backward-error bound
CANCEL = 0.02           # sigma^2 / s below which the variance is cancellation residue (test_gpu_fullsize.py)
SENTINEL = -777.25
TAIL = 4099             # sentinel floats past the m x m output
GT = 128                # row tile of the covariance stages; hb_sample_y pads m to 2 GT


def round_up(x, k):
    return -(-x // k) * k


# ---------------------------------------------------------------------------------------------------------------- models
_MODELS = {}


def _fit(key, n, d, num_uniqs=(), pred_likeli=True, seed=5, epochs=10, **conf):
    if key in _MODELS:
        return _MODELS[key]
    X, y = seeded_problem(n, max(d, 1), seed)
    X = X if d else None
    g = torch.Generator().manual_seed(seed + 100)
    Xe = None
    if num_uniqs:
        Xe = torch.stack([torch.randint(u, (n,), generator=g) for u in num_uniqs], 1)
        y = y + 0.4 * Xe[:, :1].float() - 0.2 * Xe[:, -1:].float()
    torch.manual_seed(seed)
    np.random.seed(seed)
    extra = dict(num_uniqs=list(num_uniqs)) if num_uniqs else {}
    gp = GP(d, len(num_uniqs), 1, lr=0.01, num_epochs=epochs, noise_lb=8e-4, pred_likeli=pred_likeli, **extra, **conf)
    gp.fit(X, Xe, y)
    assert not gp._fit_failed
    _MODELS[key] = (gp, X, Xe)
    return _MODELS[key]


def shape_model(n):
    """Numeric Matern-3/2 model, d = 8, with pred_likeli (the default of GP) for the shape sweep."""
    return _fit(("shape", n), n, 8, seed=n)


VARIANTS = {
    "matern32": dict(d=4, pred_likeli=False),
    "matern52": dict(d=4, kernel="matern52", pred_likeli=False),
    "rbf": dict(d=4, kernel="rbf"),
    "mixed": dict(d=3, num_uniqs=(3, 5)),
    "cat_only": dict(d=0, num_uniqs=(4, 6)),
    "warp": dict(d=4, warp=True),
    "no_ard": dict(d=4, ard_kernel=False),
    "hetero": dict(d=4, pred_likeli=False, noise_diag="hetero"),
    # d + De = 4096 = HB_MAX_FEATURES.  Without Langevin noise: with most lengthscale gradients vanishing at this width,
    # the noise random-walks some lengthscales to ~1e-14 and leaves every row uncorrelated with every other.
    "max_features": dict(d=4000, num_uniqs=(5,), emb_sizes=[96], langevin=False),
}


def variant_model(name):
    conf = dict(VARIANTS[name])
    n = 300
    if conf.get("noise_diag") == "hetero":
        X, _ = seeded_problem(n, conf["d"], 7)
        conf["noise_diag"] = (1e-2 * (1 + (X.double() ** 2).sum(1) / conf["d"])).float()
    return _fit(("variant", name), n, seed=7, epochs=10 if conf["d"] < 100 else 3, **conf)


def candidates(gp, m, seed, dup=None, near=None):
    """m rows in [-1.2, 1.2]^d (some outside the training box) with random categories; dup = (src, at) copies rows;
    near = (X, Xe): training rows moved by 0.01 in every numeric column, with their categories."""
    g = torch.Generator().manual_seed(seed)
    Xs = (torch.rand(m, gp.d, generator=g) * 2.4 - 1.2) if gp.d else None
    Xe = torch.stack([torch.randint(u, (m,), generator=g) for u in gp.num_uniqs], 1) if gp.num_enum else None
    if near is not None:
        idx = torch.randint(near[0].shape[0], (m,), generator=g)
        Xs = near[0][idx] + 0.01 * (torch.rand(m, gp.d, generator=g) * 2 - 1)
        Xe = None if near[1] is None else near[1][idx]
    if dup is not None:
        src, at = dup
        if Xs is not None:
            Xs[at] = Xs[src]
        if Xe is not None:
            Xe[at] = Xe[src]
    return (None if Xs is None else Xs.to(DEV).contiguous(),
            None if Xe is None else Xe.to(DEV, torch.int32).contiguous())


# ---------------------------------------------------------------------------------------------------------------- C ABI
def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def call_sample_y(gp, Xs, Xe, z, n_samples, out, hyp_dev, hyp_host, alpha, y_mean, y_std):
    lib = _lib.lib()
    m = (Xs if Xs is not None else Xe).shape[0]
    ws = torch.empty(int(lib.hb_sample_workspace_bytes(gp.n, gp.d, gp._spec_ptr(), m)), dtype=torch.uint8, device=DEV)
    jit = C.c_float(-1.0)
    st = lib.hb_sample_y(_ptr(Xs), _ptr(Xe), m, gp.n, gp.d, gp._spec_ptr(), _ptr(gp._emb_meta_dev) if gp.num_enum else None,
                         _ptr(gp.tab_s_dev) if gp.num_enum else None, _ptr(gp._x_mul), _ptr(gp._x_add), _ptr(gp.Zt_dev),
                         _ptr(alpha), _ptr(gp.Linv_dev), _ptr(hyp_dev), C.c_void_p(hyp_host.data_ptr()), gp.kern_id,
                         float(y_mean), float(y_std), int(bool(gp.pred_likeli)), _ptr(z), int(n_samples), _ptr(out),
                         C.byref(jit), _ptr(ws), ws.numel(), _lib.stream_ptr())
    torch.cuda.synchronize()
    return st, jit.value


def call_sample_y_batch(gp, Xs, Xe, z, f, hyp_dev, alpha, y_mean, y_std, jitter, status, ws):
    lib = _lib.lib()
    m = f.numel()
    return lib.hb_sample_y_batch(_ptr(Xs), _ptr(Xe), m, gp.n, gp.d, gp._spec_ptr(), _ptr(gp._emb_meta_dev) if gp.num_enum else None,
                                 _ptr(gp.tab_s_dev) if gp.num_enum else None, _ptr(gp._x_mul), _ptr(gp._x_add), _ptr(gp.Zt_dev),
                                 _ptr(alpha), _ptr(gp.Linv_dev), _ptr(hyp_dev), gp.kern_id, float(y_mean), float(y_std),
                                 int(bool(gp.pred_likeli)), _ptr(z), 0, 0, _ptr(f), _ptr(jitter), _ptr(status), _ptr(ws),
                                 ws.numel(), _lib.stream_ptr())


def zero_mean_state(gp):
    """hyp with the mean constant 0 (device and host copies) and an all-zero alpha: every row's mean is an exact 0."""
    hyp_dev = gp.hyp_dev.clone()
    hyp_dev[1] = 0.0
    hyp_host = gp.hyp.clone().contiguous()
    hyp_host[1] = 0.0
    return hyp_dev, hyp_host, torch.zeros(gp.NP, device=DEV)


def sample_y_root(gp, Xs, Xe):
    """(R [m, m] fp32, jitter) of hb_sample_y read out with z = I_m; checks the structure of the output on the way."""
    m = (Xs if Xs is not None else Xe).shape[0]
    hyp_dev, hyp_host, alpha = zero_mean_state(gp)
    z = torch.eye(m, device=DEV)
    out = torch.full((m * m + TAIL,), SENTINEL, device=DEV)
    st, jit = call_sample_y(gp, Xs, Xe, z, m, out, hyp_dev, hyp_host, alpha, 0.0, 1.0)
    assert st == _lib.HB_OK, st
    assert bool((out[m * m:] == SENTINEL).all()), "hb_sample_y wrote past out[n_samples, m]"
    R = out[:m * m].view(m, m).t()                      # out[s][i] = R[i][s]
    del z, out
    assert bool((R.triu(1) == 0).all()), "nonzero entries above the diagonal of the root"
    assert bool((R.diagonal() > 0).all()) and bool(torch.isfinite(R).all())
    return R, jit


def sample_y_batch_root(gp, Xs, Xe, hyp_dev=None):
    """(F [m, m], jitter, status): column j = f of hb_sample_y_batch with z = e_j (the root of the distinct rows)."""
    m = (Xs if Xs is not None else Xe).shape[0]
    hd, _, alpha = zero_mean_state(gp)
    hyp_dev = hd if hyp_dev is None else hyp_dev
    ws = torch.empty(gp.sample_batch_workspace_bytes(m), dtype=torch.uint8, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    jits = torch.empty(m, device=DEV)
    F = torch.empty(m, m, device=DEV)
    eye = torch.eye(m, device=DEV)
    for j in range(m):
        f = torch.empty(m, device=DEV)
        assert call_sample_y_batch(gp, Xs, Xe, eye[j].contiguous(), f, hyp_dev, alpha, 0.0, 1.0, jits[j:j + 1], status, ws) == _lib.HB_OK
        F[:, j] = f
    torch.cuda.synchronize()
    assert bool((jits == jits[0]).all())
    return F, float(jits[0]), int(status.item())


# ---------------------------------------------------------------------------------------------------------------- fp64 references
def _gather_emb(gp, Xe, flat):
    """Embedding features of the rows Xe [m, e] from flat [T] tables laid out column by column, row-major."""
    out, off = [], 0
    for c, (u, e) in enumerate(zip(gp.num_uniqs, gp.emb_sizes)):
        idx = off + Xe[:, c:c + 1].long() * e + torch.arange(e, device=DEV)
        out.append(flat[idx])
        off += u * e
    return torch.cat(out, 1)


def _numeric(gp, X, hyp):
    xt = gp._x_mul.double() * X.double() + gp._x_add.double()
    if gp.warp_mode:
        d, h = gp.d, gp._h_wa
        xt = O.kumaraswamy_warp(xt, hyp[h:h + d], hyp[h + d:h + 2 * d])
    return xt / hyp[3:3 + gp.d]


def features(gp, Xs, Xe, hyp, tables):
    """[m, d + De] fp64 scaled features: numeric columns through the MinMax scale, the warp and 1 / l, embedding columns
    gathered from `tables` (already divided by the embedding lengthscale)."""
    parts = []
    if gp.d:
        parts.append(_numeric(gp, Xs, hyp))
    if gp.num_enum:
        parts.append(_gather_emb(gp, Xe, tables))
    return torch.cat(parts, 1)


def kmat(gp, A, B, s):
    """s k(A, B) in fp64 by direct differences (row blocks keep the difference tensor near 2^26 elements)."""
    d = gp.d
    out = torch.empty(A.shape[0], B.shape[0], dtype=torch.float64, device=DEV)
    blk = max(1, (1 << 26) // max(1, B.shape[0] * A.shape[1]))
    for i0 in range(0, A.shape[0], blk):
        a = A[i0:i0 + blk]
        k = torch.ones(a.shape[0], B.shape[0], dtype=torch.float64, device=DEV)
        if d:
            k = O.kernel_from_sqdist(((a[:, None, :d] - B[None, :, :d]) ** 2).sum(-1), gp.kernel)
        if gp.num_enum:
            k = k * O.kernel_from_sqdist(((a[:, None, d:] - B[None, :, d:]) ** 2).sum(-1), "matern32")
        out[i0:i0 + blk] = s * k
    return out


def own_state_reference(gp, Xs, Xe):
    """C' of the GP's own fp32 state in fp64, and the per-row norms of the backward-error bound."""
    hyp = gp.hyp.double().to(DEV)
    sn2, s = float(hyp[0]), float(hyp[2])
    tab = gp.tab_s_dev.double() if gp.num_enum else None
    Zc = features(gp, Xs, Xe, hyp, tab)
    Zt = gp.Zt_dev[:, :gp.n].double().t()
    Ks = kmat(gp, Zc, Zt, s)
    Linv = gp.Linv_dev[:gp.n, :gp.n].double().tril()
    V = Ks @ Linv.t()
    w = (Ks.abs() @ Linv.abs().t()).norm(dim=1)
    Cp = kmat(gp, Zc, Zc, s) - V @ V.t()
    pl = sn2 if gp.pred_likeli else 0.0
    Cp.diagonal().add_(pl)
    return dict(Cp=Cp, w=w, vn=V.norm(dim=1), s=s + pl, Ks=Ks, znorm=float(Zc.norm(dim=1).max()))


def backward_ratio(R, ref, jitter, NP, mp):
    """max over the lower triangle of E / (u B), and the matrices the jitter check reads."""
    R64 = R.double()
    RRt = R64 @ R64.t()
    B = R64.abs() @ R64.abs().t()
    B.mul_(math.sqrt(mp)).add_(ref["s"])
    w, vn = ref["w"], ref["vn"]
    B.add_(math.sqrt(NP) * (w[:, None] * vn[None] + vn[:, None] * w[None] + vn[:, None] * vn[None]))
    E = RRt - ref["Cp"]
    E.diagonal().sub_(jitter)
    ratio = float((E.abs() / (U * B)).tril().max())
    return ratio, RRt, B


_TRUE = {}


def true_model(gp, X, Xe):
    """The fp64 GP at the hyper-parameters of `gp` (training features, K + sigma_n^2 I [+ noise_diag], Cholesky, alpha)."""
    key = id(gp)
    if key in _TRUE:
        return _TRUE[key]
    hyp = gp.hyp.double().to(DEV)
    tables = None
    if gp.num_enum:
        lay = gp._param_layout()
        tables = gp.raw[lay["tab"]:lay["tab"] + gp.T].double().to(DEV) / hyp[3 + gp.d]
    Xd = None if X is None or gp.d == 0 else X.to(DEV)
    Xed = None if Xe is None else Xe.to(DEV)
    Zt = features(gp, Xd, Xed, hyp, tables)
    K = kmat(gp, Zt, Zt, float(hyp[2]))
    K.diagonal().add_(float(hyp[0]))
    if gp.noise_diag is not None:
        K.diagonal().add_(torch.as_tensor(gp.noise_diag).double().to(DEV))
    L = torch.linalg.cholesky(K)
    c = float(hyp[1])
    yt = gp._y_dev.double()
    alpha = torch.cholesky_solve((yt - c).reshape(-1, 1), L).reshape(-1)
    _TRUE[key] = dict(Zt=Zt, L=L, alpha=alpha, hyp=hyp, tables=tables, c=c)
    return _TRUE[key]


def true_posterior(gp, tm, Xs, Xe):
    """(C, mu) of the fp64 predictive distribution of the candidates, standardised units."""
    hyp = tm["hyp"]
    s, sn2 = float(hyp[2]), float(hyp[0])
    Zc = features(gp, Xs, Xe, hyp, tm["tables"])
    Ks = kmat(gp, Zc, tm["Zt"], s)
    Vt = torch.linalg.solve_triangular(tm["L"], Ks.t(), upper=False)
    Cm = kmat(gp, Zc, Zc, s) - Vt.t() @ Vt
    if gp.pred_likeli:
        Cm.diagonal().add_(sn2)
    return Cm, tm["c"] + Ks @ tm["alpha"]


def fp64_errors(RRt, jitter, Cm, s):
    """sqrt-variance errors (regular / cancelled rows) and the largest correlation error over the regular rows."""
    Ch = RRt.clone()
    Ch.diagonal().sub_(jitter)
    v, vh = Cm.diagonal().clamp_min(0), Ch.diagonal().clamp_min(0)
    esg = (vh.sqrt() - v.sqrt()).abs() / v.sqrt()
    reg = v >= CANCEL * s
    ecor = 0.0
    if int(reg.sum()) > 1:
        sd, sdh = v[reg].sqrt(), vh[reg].sqrt()
        cor = Cm[reg][:, reg] / (sd[:, None] * sd[None])
        corh = Ch[reg][:, reg] / (sdh[:, None] * sdh[None])
        ecor = float((cor - corh).abs().max())
    return dict(sigma_err_regular=float(esg[reg].max()) if bool(reg.any()) else 0.0,
                sigma_err_cancelled=float(esg[~reg].max()) if bool((~reg).any()) else 0.0,
                rows_cancelled=int((~reg).sum()), corr_err=ecor)


def check_sample_y_case(name, gp, X, Xe_train, Xs, Xe, fp64=True):
    m = (Xs if Xs is not None else Xe).shape[0]
    R, jit = sample_y_root(gp, Xs, Xe)
    ref = own_state_reference(gp, Xs, Xe)
    ratio, RRt, B = backward_ratio(R, ref, jit, gp.NP, round_up(m, 2 * GT))
    rep = dict(case=name, n=gp.n, m=m, NP=gp.NP, jitter=jit, c_needed=ratio, feature_norm_max=ref["znorm"])
    out = dict(R=R, RRt=RRt, B=B, ref=ref, jitter=jit, rep=rep)
    if fp64:
        tm = true_model(gp, X, Xe_train)
        Cm, mu = true_posterior(gp, tm, Xs, Xe)
        rep.update(fp64_errors(RRt, jit, Cm, float(tm["hyp"][2])))
        rep.update(mean_errors(gp, Xs, Xe, mu, ref["Ks"], Cm, float(tm["hyp"][2])))
    print(json.dumps(rep))
    assert ratio <= C_MAX, rep
    if fp64:
        assert rep["sigma_err_regular"] <= 1e-4 and rep["sigma_err_cancelled"] <= 2e-4 and rep["corr_err"] <= 2e-4, rep
        assert rep["mu_err"] <= 1e-4 and rep["mu_vs_predict"] <= 1.0, rep
    return out


def mean_errors(gp, Xs, Xe, mu64, Ks64, Cm, s):
    """A z = 0 draw with the real alpha, hyp, y_mean and y_std is mu: against the fp64 mean (1e-4 max(|mu|, y_std)) and
    against GP.predict's mu.  Both add the same fp32 K* alpha partials (kstar_kernel), but in another order: the sampler
    starts from the constant c, the posterior adds c last.  The two fp32 sums of ncg + 1 terms then differ by at most
    2 (ncg + 1) u (|c| + sum |partials|) <= 2 (ncg + 1) u (|c| + |K*| |alpha|) (fp64, plus one u of slack per term), and
    the final scaling adds one rounding each: bound = y_std (2 (ncg + 2) u S) + 2 u |mu|.  mu_vs_predict is the ratio
    to that bound.  GP.predict's own sigma errors on the same rows are reported next to the sampler's (predict_*)."""
    m = (Xs if Xs is not None else Xe).shape[0]
    out = torch.full((m + TAIL,), SENTINEL, device=DEV)
    st, _ = call_sample_y(gp, Xs, Xe, torch.zeros(m, device=DEV), 1, out, gp.hyp_dev, gp.hyp.contiguous(), gp.alpha_dev,
                          gp._y_mean, gp._y_std)
    assert st == _lib.HB_OK and bool((out[m:] == SENTINEL).all())
    mu = out[:m].double()
    ys, ym = gp._y_std, gp._y_mean
    mu_true = mu64 * ys + ym
    emu = float(((mu - mu_true).abs() / mu_true.abs().clamp_min(ys)).max())
    mu_p, var_p = gp.predict(None if Xs is None else Xs, Xe)
    mu_p = mu_p.reshape(-1).to(DEV).double()
    v = Cm.diagonal().clamp_min(0)
    esg = (var_p.reshape(-1).to(DEV).double().sqrt() / ys - v.sqrt()).abs() / v.sqrt()
    reg = v >= CANCEL * s
    ncg = -(-gp.NP // 512)
    S = abs(float(gp.hyp[1])) + Ks64.abs() @ gp.alpha_dev[:gp.n].double().abs()
    bound = ys * 2 * (ncg + 2) * U * S + 2 * U * mu.abs()
    return dict(mu_err=emu, mu_vs_predict=float(((mu - mu_p).abs() / bound).max()),
                mu_equal_predict=bool(torch.equal(mu, mu_p)),
                predict_sigma_err_regular=float(esg[reg].max()) if bool(reg.any()) else 0.0,
                predict_sigma_err_cancelled=float(esg[~reg].max()) if bool((~reg).any()) else 0.0)


# ---------------------------------------------------------------------------------------------------------------- 1-3: hb_sample_y
M_LIST = [1, 2, 127, 128, 129, 255, 256, 257, 511, 512, 513, 767, 768, 769, 1000, 4097, 8192]
SHAPES = [(129, m) for m in M_LIST] + [(700, m) for m in M_LIST] + [(4097, m) for m in (1, 257, 8192)] + \
         [(5, m) for m in (1, 257)] + [(128, m) for m in (129, 769)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,m", SHAPES, ids=[f"n{n}-m{m}" for n, m in SHAPES])
def test_sample_y_root_across_tile_edges(n, m):
    """Every 256-row tile edge of the candidate pad, the 512-wide outer Cholesky blocks (mp = 768 -> two), the m = 8192
    cap (16 outer blocks) and NP = 4224; the root against the GP's own fp32 state and against the fp64 posterior."""
    gp, X, Xe = shape_model(n)
    Xs, Xse = candidates(gp, m, seed=m)
    check_sample_y_case(f"n{n}-m{m}", gp, X, Xe, Xs, Xse)
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_sample_y_root_model_variants(variant):
    """Each kernel, pred_likeli both ways, mixed and categorical-only inputs, a learned warp, ard_kernel=False,
    heteroscedastic noise and d + De = HB_MAX_FEATURES (the 32-wide feature chunks of the candidate Gram), at m = 300
    (three row tiles, two 256-row pads)."""
    gp, X, Xe = variant_model(variant)
    # in 4000 dimensions random rows are uncorrelated with everything: take them next to the training rows instead
    Xs, Xse = candidates(gp, 300, seed=300, near=(X, Xe) if variant == "max_features" else None)
    check_sample_y_case(variant, gp, X, Xe, Xs, Xse)
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_sample_y_keeps_duplicates_and_reports_its_jitter():
    """Exact duplicate candidates stay in hb_sample_y's covariance, which is then singular but for the jitter: for a
    duplicate pair (a, b), (R R^T)_aa - (R R^T)_ab = jitter_used within the backward-error bound of the two entries."""
    gp, X, Xe = shape_model(129)
    src = torch.tensor([3, 0, 7, 130, 250, 251, 12, 290])                  # within a tile, across 128 / 256 edges
    at = torch.tensor([5, 9, 140, 131, 260, 270, 299, 298])
    Xs, Xse = candidates(gp, 300, seed=31, dup=(src, at))
    o = check_sample_y_case("duplicates", gp, X, Xe, Xs, Xse, fp64=False)
    _check_duplicate_jitter(o, src, at)


@pytest.mark.gpu
def test_sample_y_ladder_rung_above_the_first():
    """The ladder case of test_gpu_noisy.py: rows 1e-7 apart far from the data at outputscale 1e3 are numerically
    singular past a jitter of 1e-6; the rung hb_sample_y reports is the one in R R^T."""
    gp, X, Xe = _fit("ladder", 300, 3, pred_likeli=False, epochs=20)
    raw = gp.raw.clone()
    raw[2] = 1000.0                                                          # softplus(1000) = 1000: the outputscale
    gp.set_hypers(raw)
    m = 64
    Xs = (X.max(0).values + 0.5).repeat(m, 1)
    Xs[:, 0] = 0.1 + torch.arange(m, dtype=torch.float64) * 1e-7
    assert torch.unique(Xs, dim=0).shape[0] == m
    o = check_sample_y_case("ladder", gp, X, Xe, Xs.to(DEV).contiguous(), None, fp64=False)
    assert o["jitter"] > 1e-6
    # what the neighbouring rungs would need (the sqrt(mp) |R| |R|^T term of B, ~ 16 s u here, is wider than one rung)
    d0 = o["RRt"].diagonal() - o["ref"]["Cp"].diagonal()
    alt = [float(((d0 - j).abs() / (U * o["B"].diagonal())).max()) for j in (o["jitter"] / 10, o["jitter"] * 10)]
    print(json.dumps(dict(case="ladder-neighbours", jitter=o["jitter"], c_needed_at_neighbour_rungs=alt)))
    _MODELS.pop("ladder")


def _check_duplicate_jitter(o, src, at):
    RRt, B, Cp, jit = o["RRt"], o["B"], o["ref"]["Cp"], o["jitter"]
    worst = 0.0
    for a, b in zip(src.tolist(), at.tolist()):
        i, j = max(a, b), min(a, b)
        diff = float(RRt[i, i] - RRt[i, j]) - float(Cp[i, i] - Cp[i, j])
        tol = C_MAX * U * float(B[i, i] + B[i, j])
        worst = max(worst, abs(diff - jit) / tol)
        assert abs(diff - jit) <= tol, (a, b, diff, jit, tol)
    print(json.dumps(dict(case="duplicate_jitter", jitter=jit, worst_over_tol=worst)))


# ---------------------------------------------------------------------------------------------------------------- 4: hb_sample_y_batch
BATCH_M = [1, 2, 31, 32, 33, 127, 128, 129, 255, 256]
BATCH = [("numeric", m) for m in BATCH_M] + [("mixed", m) for m in BATCH_M]


def batch_model(kind):
    return shape_model(129) if kind == "numeric" else variant_model("mixed")


@pytest.mark.gpu
@pytest.mark.parametrize("kind,m", BATCH, ids=[f"{k}-m{m}" for k, m in BATCH])
def test_sample_y_batch_root(kind, m):
    """The one-CTA root of hb_sample_y_batch over distinct rows: same backward-error and fp64 checks as hb_sample_y."""
    gp, X, Xe = batch_model(kind)
    Xs, Xse = candidates(gp, m, seed=1000 + m)
    F, jit, st = sample_y_batch_root(gp, Xs, Xse)
    assert st == _lib.HB_OK
    assert bool((F.triu(1) == 0).all()) and bool((F.diagonal() > 0).all()) and bool(torch.isfinite(F).all())
    ref = own_state_reference(gp, Xs, Xse)
    ratio, RRt, _ = backward_ratio(F, ref, jit, gp.NP, round_up(m, GT))
    tm = true_model(gp, X, Xe)
    Cm, _ = true_posterior(gp, tm, Xs, Xse)
    rep = dict(case=f"batch-{kind}-m{m}", n=gp.n, m=m, jitter=jit, c_needed=ratio)
    rep.update(fp64_errors(RRt, jit, Cm, float(tm["hyp"][2])))
    print(json.dumps(rep))
    assert ratio <= C_MAX, rep
    assert rep["sigma_err_regular"] <= 1e-4 and rep["sigma_err_cancelled"] <= 2e-4 and rep["corr_err"] <= 2e-4, rep


@pytest.mark.gpu
def test_sample_y_batch_duplicates_leave_the_root_of_the_distinct_rows():
    """With duplicates in the batch, the distinct rows' root is the root of the de-duplicated batch bit for bit, a
    duplicate row is +inf under every draw, and a draw on a duplicate row's z moves nothing."""
    gp, _, _ = variant_model("mixed")
    k = 40
    src = torch.tensor([3, 0, 7, 3, 39, 12, 5, 0, 21, 30])
    at = torch.tensor([5, 9, 14, 20, 41, 44, 45, 47, 48, 49])
    order = torch.full((k + len(src),), -1, dtype=torch.long)
    order[at] = src
    order[order < 0] = torch.arange(k)
    Xs, Xse = candidates(gp, k, seed=9)
    Bs, Bse = Xs[order.to(DEV)].contiguous(), Xse[order.to(DEV)].contiguous()
    first = torch.tensor([int((order[:i] == order[i]).sum()) == 0 for i in range(len(order))])
    F, jit, st = sample_y_batch_root(gp, Bs, Bse)
    Fd, jd, std = sample_y_batch_root(gp, Bs[first.to(DEV)].contiguous(), Bse[first.to(DEV)].contiguous())
    assert st == std == _lib.HB_OK and jit == jd
    fi = first.to(DEV)
    assert bool(torch.isinf(F[~fi]).all()) and bool((F[~fi] > 0).all())
    assert torch.equal(F[fi][:, fi], Fd)
    assert bool((F[fi][:, ~fi] == 0).all())


def last_rung():
    """The last jitter the fp32 ladder 1e-6, x10 per failure, tries before it exceeds 10."""
    j = np.float32(1e-6)
    while np.float32(j * np.float32(10.0)) <= np.float32(10.0):
        j = np.float32(j * np.float32(10.0))
    return float(j)


@pytest.mark.gpu
def test_sample_y_batch_give_up_reports_the_last_rung():
    """A NaN lengthscale makes every rung fail: status = HB_ERR_NOT_PD, f = NaN in every row, and the jitter is the last
    rung tried, as include/hebo_b200.h documents.  hb_sample_y gives up on the same input."""
    gp, _, _ = shape_model(129)
    m = 40
    Xs, _ = candidates(gp, m, seed=4)
    hyp_nan = gp.hyp_dev.clone()
    hyp_nan[3] = float("nan")
    ws = torch.empty(gp.sample_batch_workspace_bytes(m), dtype=torch.uint8, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    jit = torch.zeros(1, device=DEV)
    f = torch.zeros(m, device=DEV)
    assert call_sample_y_batch(gp, Xs, None, torch.randn(m, device=DEV), f, hyp_nan, gp.alpha_dev, gp._y_mean, gp._y_std,
                               jit, status, ws) == _lib.HB_OK
    torch.cuda.synchronize()
    assert int(status.item()) == _lib.HB_ERR_NOT_PD
    assert bool(torch.isnan(f).all())
    assert float(jit.item()) == last_rung() and 9.0 < last_rung() <= 10.0, float(jit.item())
    hyp_host = gp.hyp.clone().contiguous()
    hyp_host[3] = float("nan")
    out = torch.zeros(m, device=DEV)
    st, _ = call_sample_y(gp, Xs, None, torch.randn(m, device=DEV), 1, out, hyp_nan, hyp_host, gp.alpha_dev, gp._y_mean, gp._y_std)
    assert st == _lib.HB_ERR_NOT_PD


# ---------------------------------------------------------------------------------------------------------------- 5: hb_cholesky
def spd(NP):
    g = torch.Generator(device=DEV).manual_seed(NP)
    B = torch.randn(NP, 64, generator=g, dtype=torch.float64, device=DEV)
    A64 = B @ B.t() / 64 + torch.diag(torch.rand(NP, generator=g, dtype=torch.float64, device=DEV) + 0.5)
    return A64.float()


def cholesky(A):
    lib = _lib.lib()
    ws = torch.empty(128 * 128, device=DEV)
    info = torch.zeros(1, dtype=torch.int32, device=DEV)
    _lib.check(lib.hb_cholesky(_ptr(A), A.shape[0], _ptr(ws), _ptr(info), _lib.stream_ptr()), "hb_cholesky")
    return int(info.item())


@pytest.mark.gpu
@pytest.mark.parametrize("NP", [2176, 4224, 8192])
def test_cholesky_backward_error_beyond_one_block(NP):
    """|L L^T - A| <= c u sqrt(NP) (|L| |L|^T) on the lower triangle, with several 512-wide outer blocks."""
    A = spd(NP)
    A0 = A.double()
    assert cholesky(A) == 0
    L = A.double().tril()
    ratio = float(((L @ L.t() - A0).abs() / (U * math.sqrt(NP) * (L.abs() @ L.abs().t()))).tril().max())
    print(json.dumps(dict(case=f"cholesky-NP{NP}", c_needed=ratio)))
    assert ratio <= C_MAX, ratio


@pytest.mark.gpu
@pytest.mark.parametrize("NP", [2176, 4224, 8192])
def test_cholesky_info_at_block_edges(NP):
    """A negative pivot at row j gives info = j + 1 (LAPACK), at the last column of an outer block, the first of the
    next, row 4096 and the last row.  The leading minors up to j are sections of an SPD matrix and the pivot of row j is
    -1 - |L[j, :j]|^2 < 0, so LAPACK's info is j + 1 by definition.  (torch.linalg.cholesky_ex on the device reports 513
    for j = 511 on this matrix, so it is not used as the reference.)"""
    A = spd(NP)
    for j in (511, 512, 4096, NP - 1):
        if j >= NP:
            continue
        Ab = A.clone()
        Ab[j, j] = -1.0
        assert cholesky(Ab) == j + 1, j


# ---------------------------------------------------------------------------------------------------------------- 6: arguments
@pytest.fixture(scope="module")
def lib():
    if not _lib.available():
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


def test_sample_y_rejects_bad_arguments(lib):
    bad = _lib.HB_ERR_INVALID
    p = C.c_void_p(16)               # never dereferenced: every call below must fail its argument checks first
    n, d = 300, 2
    need = int(lib.hb_sample_workspace_bytes(n, d, None, 100))
    assert need > 0

    def call(m=100, n_samples=3, hyp_host=p, ws_bytes=need):
        return lib.hb_sample_y(p, None, m, n, d, None, None, None, p, p, p, p, p, p, hyp_host, 0, 0.0, 1.0, 0, p, n_samples, p,
                               None, p, ws_bytes, None)
    assert call(m=0) == bad
    assert call(m=8193, ws_bytes=int(lib.hb_sample_workspace_bytes(n, d, None, 8193))) == bad
    assert call(n_samples=0) == bad
    assert call(hyp_host=None) == bad
    assert call(ws_bytes=need - 1) == bad
    assert call(ws_bytes=-1) == bad
