"""Shared helpers for the test-suite (test infrastructure; may import oracle/)."""
from __future__ import annotations

import contextlib
import copy
import math
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# Absolute error budget on Phi(z) in the REFERENCE's own fp32 path: ATen's vectorised CPU erf is the
# Abramowitz-Stegun 7.1.26 polynomial (|err| <= 1.5e-7 on erf => 7.5e-8 on Phi) and 0.5*(1+erf) is
# quantised to 2^-25 ~ 3e-8.  -log PI and -log EI inherit delta/Phi and delta*|z|/(Phi z + phi): for
# z < -4 the reference's columns 1-2 are approximation noise, so parity there is defined through this
# budget, not through 1e-4 (DESIGN.md "MACE tail").
PHI_BUDGET = 1.6e-7


def load_golden(name: str):
    return np.load(os.path.join(GOLDEN, name), allow_pickle=False)


def mace_tolerance(mu, var, noise_var, tau, eps, xi2, rtol=1e-4):
    """Per-row absolute tolerances (col0, col1, col2) for MACE objectives given the reference's fp32
    error budget; rows whose tolerance exceeds 0.05 are flagged ill-conditioned (second return)."""
    mu = np.asarray(mu, dtype=np.float64).reshape(-1)
    sd = np.sqrt(np.asarray(var, dtype=np.float64).reshape(-1)).clip(1.1920929e-07)
    xi2 = np.asarray(xi2, dtype=np.float64).reshape(-1)
    noise = math.sqrt(2.0) * math.sqrt(noise_var)
    z = (tau - eps - mu - noise * xi2) / sd
    Phi = 0.5 * (1 + np.vectorize(math.erf)(z / math.sqrt(2.0)))
    phi = np.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)
    ei_n = Phi * z + phi
    with np.errstate(divide="ignore", invalid="ignore"):
        t_pi = PHI_BUDGET / np.maximum(Phi, 1e-300)
        t_ei = PHI_BUDGET * (np.abs(z) + 1) / np.maximum(np.abs(ei_n), 1e-300)
    ill = (t_pi > 0.05) | (t_ei > 0.05) | (z < -5.9)
    return z, t_ei, t_pi, ill


def assert_mace_close(F, F_ref, mu, var, noise_var, tau, eps, xi2, rtol=1e-4, what=""):
    F = np.asarray(F, dtype=np.float64)
    F_ref = np.asarray(F_ref, dtype=np.float64)
    z, t_ei, t_pi, ill = mace_tolerance(mu, var, noise_var, tau, eps, xi2)
    ok = ~ill
    scale = rtol * (1.0 + np.abs(F_ref))
    assert np.all(np.abs(F[:, 0] - F_ref[:, 0]) <= scale[:, 0] + 1e-6), f"{what}: LCB column mismatch"
    d1 = np.abs(F[ok, 1] - F_ref[ok, 1])
    d2 = np.abs(F[ok, 2] - F_ref[ok, 2])
    assert np.all(d1 <= scale[ok, 1] + 2 * t_ei[ok]), f"{what}: -logEI mismatch max {d1.max()}"
    assert np.all(d2 <= scale[ok, 2] + 2 * t_pi[ok]), f"{what}: -logPI mismatch max {d2.max()}"
    # deep-tail rows (z < -6.5) are on the log-approximation branch in every implementation: exact formulas again
    deep = z < -6.5
    if deep.any():
        assert np.all(np.abs(F[deep, 1:] - F_ref[deep, 1:]) <= rtol * (1 + np.abs(F_ref[deep, 1:]))), \
            f"{what}: approximation-branch mismatch"
    return int(ok.sum()), int(ill.sum())


def seeded_problem(n, d, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    X = torch.rand(n, d, generator=g, dtype=torch.float64) * 2 - 1
    w = torch.randn(d, generator=g, dtype=torch.float64) / math.sqrt(d)
    y = torch.sin(3 * (X @ w)) + 0.5 * (X[:, 0] ** 2) + 0.05 * torch.randn(n, generator=g, dtype=torch.float64)
    return X.to(dtype), y.to(dtype).reshape(-1, 1)


def scaled_xy(gp, X, y):
    """fp64 training rows through the fitted GP's MinMax scaler and y through its standardisation."""
    Xt64 = gp.xscaler.scale_.double() * X.double() + gp.xscaler.min_.double()
    yt64 = (y.double().reshape(-1) - float(gp.yscaler.mean[0])) / float(gp.yscaler.std[0])
    return Xt64, yt64


def emb_hypers(gp, raw):
    """oracle/emb_oracle.py EmbHypers of a GP's raw vector (fp64): noise, tables, mean, outputscale, lengthscales."""
    from oracle import emb_oracle as E
    raw = raw.double()
    lay = gp._param_layout()
    tabs, o = [], lay["tab"]
    for u, e in zip(gp.num_uniqs, gp.emb_sizes):
        tabs.append(raw[o:o + u * e].reshape(u, e))
        o += u * e
    rle = raw[lay["le"]] if gp.num_enum else torch.zeros((), dtype=torch.float64)
    return E.EmbHypers(raw[0], tabs, raw[lay["mean"]], raw[lay["os"]], raw[lay["ls"]:lay["ls"] + lay["n_ls"]], rle, gp.noise_lb)


def oracle_posterior(X, yt, raw, kind, Xs, dtype, warp=None, noise_diag=None, pred_likeli=False, noise_lb=8e-4):
    """Oracle predict() (mu, var in y units, flattened float64 numpy) in `dtype` at raw hypers `raw`.

    With dtype=float32 this is the reference's own precision (torch CPU fp32: Cholesky + triangular solve), i.e. the
    NOISE FLOOR the fp32 reference itself has against exact arithmetic -- SURVEY section 8d asks for it to be reported
    next to the GPU error; the sigma criterion is max(1e-4, 2 x floor)."""
    from oracle import gp_oracle as O
    X = torch.as_tensor(X)
    sc, mn = O.minmax_fit(X.numpy().astype(np.float32))
    ym, ys = O.standard_fit(np.asarray(yt, dtype=np.float32).reshape(-1, 1))
    sc_t, mn_t = torch.from_numpy(sc).to(dtype), torch.from_numpy(mn).to(dtype)
    Xt = sc_t * X.to(dtype) + mn_t
    Xm = sc_t * torch.as_tensor(Xs).to(dtype) + mn_t
    if warp is not None:
        a, b = (torch.as_tensor(w).to(dtype) for w in warp)
        Xt, Xm = O.kumaraswamy_warp(Xt, a, b), O.kumaraswamy_warp(Xm, a, b)
    d = X.shape[1]
    hp = O.Hypers.unpack(torch.as_tensor(raw).to(dtype), noise_lb)
    nd = None if noise_diag is None else torch.as_tensor(noise_diag).to(dtype)
    f = O.FittedGP(Xt, hp, kind, torch.ones(d, dtype=dtype), torch.zeros(d, dtype=dtype), float(ym[0]), float(ys[0]),
                   pred_likeli=pred_likeli, noise_diag=nd)
    f._yt = (torch.as_tensor(yt).to(dtype).reshape(-1) - float(ym[0])) / float(ys[0])
    O.refactor(f)
    mu, var = O.predict(f, Xm)
    return mu.double().numpy().reshape(-1), var.double().numpy().reshape(-1), float(ys[0])


def mu_sigma_errors(mu, var, mu_ref, var_ref, y_std):
    mu, var = np.asarray(mu, np.float64).reshape(-1), np.asarray(var, np.float64).reshape(-1)
    emu = np.abs(mu - mu_ref) / np.maximum(np.abs(mu_ref), y_std)
    esg = np.abs(np.sqrt(var) - np.sqrt(var_ref)) / np.sqrt(var_ref)
    return float(emu.max()), float(esg.max())


# ----------------------------------------------------------------------------------------------------------------
# Parity at the sizes BASELINE.json publishes (configs C2-C5 at FULL n, plus the dense low-d regime where the
# tensor path's precision guard fires).  The fp64 oracle is rebuilt on the GPU box's host cores (n = 4096: fp64
# Cholesky + triangular solve for ~2400 candidates, a few seconds), at the hypers the CUDA fit ended on.
FULLSIZE_CASES = {
    # name: objective, n, d, kernel, q, (#Sobol, #near-training, #exact-training candidates), extras
    "c5_shard_n4096_d32": dict(fn="hartmann6", n=4096, d=32, kind="matern32", q=8, m=(2048, 256, 64), seed=1240),
    "c3_warp_n2048_d32": dict(fn="hartmann6", n=2048, d=32, kind="matern32", q=8, m=(2048, 256, 64), seed=1241, warp=True),
    "c4_hetero_n4096_d100": dict(fn="ackley", n=4096, d=100, kind="matern32", q=16, m=(2048, 256, 64), seed=1242, hetero=True),
    "c2_ackley_n512_d8_m4096": dict(fn="ackley", n=512, d=8, kind="matern52", q=8, m=(3776, 256, 64), seed=1243),
    "dense_n4096_d8": dict(fn="ackley", n=4096, d=8, kind="matern32", q=8, m=(2048, 256, 64), seed=1244),
}


def fullsize_inputs(case: str):
    """Seeded (X, y_transformed, candidates, xi1, xi2, conf-extras) of a FULLSIZE_CASES entry."""
    from oracle import gp_oracle as O
    c = FULLSIZE_CASES[case]
    n, d, seed = c["n"], c["d"], c["seed"]
    X, y = O.synthetic_problem(c["fn"], n, d, seed)
    X = X.float()
    yt = torch.from_numpy(O.hebo_y_transform(y.numpy())).float().reshape(-1, 1)
    g = torch.Generator().manual_seed(seed + 1)
    ms, mn, me = c["m"]
    sob = torch.quasirandom.SobolEngine(d, scramble=True, seed=seed).draw(ms).float() * 2 - 1
    sob[: ms // 8] *= 1.3                                                  # some rows leave the training box
    near = X[torch.randperm(n, generator=g)[:mn]] + 1e-3 * torch.randn(mn, d, generator=g)
    exact = X[torch.randperm(n, generator=g)[:me]].clone()
    Xs = torch.cat([sob, near, exact], 0).float()
    m = Xs.shape[0]
    xi1, xi2 = torch.randn(m, 1, generator=g), torch.randn(m, 1, generator=g)
    extra = {}
    if c.get("warp"):
        extra["warp_a"] = (torch.rand(d, generator=g) * 1.5 + 0.5).tolist()
        extra["warp_b"] = (torch.rand(d, generator=g) * 1.5 + 0.5).tolist()
    if c.get("hetero"):
        # BASELINE.md config 4: noise_diag_i = 1e-2 (1 + |x_i|^2 / d), in standardised-y units
        extra["noise_diag"] = (1e-2 * (1 + (X.double() ** 2).sum(1) / d)).float()
    return c, X, yt, Xs, xi1, xi2, extra


def fullsize_oracle(c, gp, X, yt, Xs, xi1, xi2, extra, dtype=torch.float64):
    """Oracle posterior / MACE / front in `dtype` at the hypers and scalers of the fitted CUDA model `gp`."""
    from oracle import gp_oracle as O
    d = X.shape[1]
    sc, mn = gp.xscaler.scale_.to(dtype), gp.xscaler.min_.to(dtype)
    ym, ys = float(gp.yscaler.mean[0]), float(gp.yscaler.std[0])
    Xt, Xm = sc * X.to(dtype) + mn, sc * Xs.to(dtype) + mn
    if "warp_a" in extra:
        a, b = torch.tensor(extra["warp_a"]).float().to(dtype), torch.tensor(extra["warp_b"]).float().to(dtype)
        Xt, Xm = O.kumaraswamy_warp(Xt, a, b), O.kumaraswamy_warp(Xm, a, b)
    nd = extra["noise_diag"].to(dtype) if "noise_diag" in extra else None
    f = O.FittedGP(Xt, O.Hypers.unpack(gp.raw.to(dtype), gp.noise_lb), c["kind"], torch.ones(d, dtype=dtype),
                   torch.zeros(d, dtype=dtype), ym, ys, pred_likeli=bool(gp.pred_likeli), noise_diag=nd)
    f._yt = (yt.to(dtype).reshape(-1) - ym) / ys
    O.refactor(f)
    mu, var = O.predict(f, Xm)
    best = int(torch.argmin(yt.reshape(-1)))
    tau = float(O.predict(f, Xt[best:best + 1])[0])
    kappa = O.kappa_schedule(c["n"], c["q"], d)
    F = O.mace(mu, var, float(f.noise), tau, kappa, 1e-4, xi1, xi2)
    return dict(mu=mu.double().numpy().reshape(-1), var=var.double().numpy().reshape(-1), F=F.double().numpy(), tau=tau,
                kappa=kappa, noise=float(f.noise), y_std=ys, s=float(f.hp.outputscale))


# ----------------------------------------------------------------------------------------------------------------
# Fitted models, candidate rows and the fp64 posterior pieces shared by the per-element posterior tests
# (test_gpu_posterior_grad.py, test_gpu_posterior_mace.py).  Models are cached by key for the whole session; a test
# that changes a model's hypers fits its own key.
DEV = torch.device("cuda")
RATE = {"matern12": 1.0, "matern32": math.sqrt(3.0), "matern52": math.sqrt(5.0)}
COINCIDENT = 2.0 ** -20         # kernel_parts takes Matern-1/2's h as 0 below this r^2
_MODELS = {}


def fit_model(key, n, d, num_uniqs=(), pred_likeli=True, seed=5, epochs=10, **conf):
    """(gp, X, Xe, y) of a GP fitted to seeded_problem(n, d, seed) (plus category effects); d = 0 is categorical-only
    (X = None)."""
    from hebo_b200 import GP
    if key in _MODELS:
        return _MODELS[key]
    X, y = seeded_problem(n, max(d, 1), seed)
    X = X if d else None
    g = torch.Generator().manual_seed(seed + 100)
    Xe = None
    if num_uniqs:
        Xe = torch.stack([torch.randint(u, (n,), generator=g) for u in num_uniqs], 1)
        y = y + 0.4 * Xe[:, :1].float() - 0.2 * Xe[:, -1:].float()
    if conf.get("noise_diag") == "hetero":
        conf["noise_diag"] = (1e-2 * (1 + (X.double() ** 2).sum(1) / d)).float()
    if conf.get("warp_a") == "fixed":
        conf["warp_a"] = (torch.rand(d, generator=g) * 1.5 + 0.5).tolist()
        conf["warp_b"] = (torch.rand(d, generator=g) * 1.5 + 0.5).tolist()
    torch.manual_seed(seed)
    np.random.seed(seed)
    extra = dict(num_uniqs=list(num_uniqs)) if num_uniqs else {}
    conf.setdefault("noise_lb", 8e-4)
    gp = GP(d, len(num_uniqs), 1, lr=0.01, num_epochs=epochs, pred_likeli=pred_likeli, **extra, **conf)
    gp.fit(X, Xe, y)
    assert not gp._fit_failed
    _MODELS[key] = (gp, X, Xe, y)
    return _MODELS[key]


VARIANTS = {
    "matern32": dict(d=4, pred_likeli=False),
    "matern32_pl": dict(d=4),
    "matern52": dict(d=4, kernel="matern52", pred_likeli=False),
    "matern52_pl": dict(d=4, kernel="matern52"),
    "rbf": dict(d=4, kernel="rbf", pred_likeli=False),
    "rbf_pl": dict(d=4, kernel="rbf"),
    "mixed_e1": dict(d=3, num_uniqs=(4,)),
    "mixed_e2": dict(d=3, num_uniqs=(3, 5), pred_likeli=False),
    # De = 6 x 50 = 300.  The wide models are fitted without Langevin noise: with most lengthscale gradients vanishing,
    # the noise of a short fit random-walks lengthscales towards zero (test_gpu_sample_root.py)
    "wide_embeddings": dict(d=8, num_uniqs=(120,) * 6, langevin=False),
    "no_ard": dict(d=4, ard_kernel=False),
    "no_ard_mixed": dict(d=3, num_uniqs=(3, 5), ard_kernel=False),
    "hetero": dict(d=4, pred_likeli=False, noise_diag="hetero"),
    "warp": dict(d=4, warp=True),
    "warp_mixed": dict(d=3, num_uniqs=(3, 5), warp=True),
    "fixed_warp": dict(d=4, warp_a="fixed"),
}

WIDTHS = {1: dict(d=1), 33: dict(d=33), 300: dict(d=300, epochs=3, langevin=False),
          # d + De = 4096 = HB_MAX_FEATURES, fitted without Langevin noise as the wide embeddings above
          4096: dict(d=4000, num_uniqs=(5,), emb_sizes=[96], langevin=False, epochs=3)}


def candidates(gp, X, Xe, m, seed, near=False):
    """m rows in [-1.2, 1.2]^d (outside the training box in places) with random categories; the first rows are exact
    training rows (r^2 = 0; none when m = 1) and the last ones duplicate rows 1, 2, 3.  near: training rows moved by 0.01
    instead.  Returns (Xs [m, d] fp32, Xe int32 or None, [(row, its duplicate)]) on the device."""
    g = torch.Generator().manual_seed(seed)
    Xs = torch.rand(m, gp.d, generator=g) * 2.4 - 1.2
    Xse = torch.stack([torch.randint(u, (m,), generator=g) for u in gp.num_uniqs], 1) if gp.num_enum else None
    n = (X if X is not None else Xe).shape[0]
    if near:
        idx = torch.randint(n, (m,), generator=g)
        Xs = X[idx] + 0.01 * (torch.rand(m, gp.d, generator=g) * 2 - 1)
        Xse = None if Xe is None else Xe[idx].clone()
    k = min(5, m // 2, n)
    if X is not None:
        Xs[:k] = X[:k]
    if Xse is not None:
        Xse[:k] = Xe[:k]
    dups = [(s, m - 4 + j) for j, s in enumerate((1, 2, 3)) if m >= 8]
    for s, t in dups:
        Xs[t] = Xs[s]
        if Xse is not None:
            Xse[t] = Xse[s]
    return (Xs.float().to(DEV).contiguous(), None if Xse is None else Xse.to(DEV, torch.int32).contiguous(), dups)


def gather_emb(gp, Xe, flat):
    """The embedding features of categories Xe [m, e] from the flat tables `flat` (tables / le), [m, De]."""
    out, off = [], 0
    for c, (u, e) in enumerate(zip(gp.num_uniqs, gp.emb_sizes)):
        out.append(flat[off + Xe[:, c:c + 1].long() * e + torch.arange(e, device=flat.device)])
        off += u * e
    return torch.cat(out, 1)


def reset_hypers(gp, **kw):
    """set_hypers on a copy of gp's raw vector: os (outputscale), noise (sigma_n^2 - noise_lb), ls (all lengthscales)."""
    from oracle import gp_oracle as O
    lay = gp._param_layout()
    raw = gp.raw.clone()
    inv = lambda v: float(O.inv_softplus(torch.tensor(v, dtype=torch.float64)))
    if "os" in kw:
        raw[lay["os"]] = inv(kw["os"])
    if "noise" in kw:
        raw[0] = kw["noise"]
    if "ls" in kw:
        raw[lay["ls"]:lay["ls"] + lay["n_ls"]] = inv(kw["ls"])
    gp.set_hypers(raw)
    assert not gp._fit_failed


def warp_error(px, xt, a, b):
    """W: the fp32 error of kumar_warp (common.cuh) at x_t = fl(px + x_add), px = x_mul x, in units of u
    (test_gpu_posterior_mace.py docstring)."""
    eps = 1e-6
    h = (xt + 1) * 0.5
    uu = h.clamp(eps, 1 - eps)
    clamped = (h < eps) | (h > 1 - eps)
    e_u = torch.where(clamped, torch.ones_like(h), (px.abs() + xt.abs() + (xt + 1).abs()) / (2 * uu))
    lu = uu.log()
    e_lu = e_u + 2 * lu.abs() + 1
    e_x = a * e_lu + (a * lu).abs()                  # absolute error of fl(a log u)
    lom = torch.log(-torch.expm1(a * lu))           # log(1 - u^a) = logf(-expm1f(a log u)): the relative error of
    e_lom = torch.exp(a * lu) / -torch.expm1(a * lu) * e_x + 2 * lom.abs() + 3      # 1 - u^a, then logf's 2 |lom|
    p = torch.exp(b * lom)
    e_p = b * e_lom + (b * lom).abs() + 2
    w = 2 * (1 - p) - 1
    return 2 * p * e_p + 2 * (1 - p).abs() + w.abs()


def warp_derivs(x, a, b, il=1.0):
    """fp64 dZa, dZb of scale_zt_kernel (kumar_warp's da, db times fl(1 / l)) from the fp32 x, a, b, and their error in
    units of u, carried term by term from the absolute errors of log u and log(1 - u^a) = log(-expm1(a log u)) and the
    relative errors of u, u^a and the powers (test_gpu_fit_stages_tc.py docstring e.)."""
    from oracle.warp_oracle import U32
    h = (x + 1) * 0.5
    uu = h.clamp(*U32)
    clamped = (h < U32[0]) | (h > U32[1])
    lu = uu.log()
    t = torch.exp(a * lu)
    lom = torch.log(-torch.expm1(a * lu))
    da = 2 * b * torch.exp((b - 1) * lom) * t * lu * il
    db = -2 * torch.exp(b * lom) * lom * il
    e_u = torch.where(clamped, torch.ones_like(h), (x.abs() + (x + 1).abs()) / (2 * uu) + 1)
    e_lu = e_u + 2 * lu.abs() + 1
    e_t = a * e_lu + (a * lu).abs() + 2
    e_lom = t / -torch.expm1(a * lu) * (e_t - 2) + 2 * lom.abs() + 3
    e_q = (b - 1).abs() * e_lom + ((b - 1) * lom).abs() + 2
    e_p = b * e_lom + (b * lom).abs() + 2
    Ea = da.abs() * (e_q + e_t + e_lu / lu.abs().clamp_min(1e-300) + 6)
    Eb = db.abs() * (e_p + e_lom / lom.abs().clamp_min(1e-300) + 4)
    return da, db, Ea, Eb


def kernel_parts(r2, kind):
    """k, h (dk/dr^2 = -h / 2) of the oracle's kernel table, |exponent of fast_exp| and the rate of that exponent in the
    features.

    Matern-1/2's h is 0 for r^2 < COINCIDENT as well as below the oracle's clamp.  This is deliberately not the oracle's
    rule; it covers the own-state references only.  They scale the candidate in fp64 from the fp32 row the kernel
    receives, so a candidate equal to a training row lands within the fp32 roundings of the scaling (the MinMax shift's
    absolute u |x_add| / l among them) of that row's fp32 feature vector, where the device, scaling both the same way in
    fp32, has r = 0.  At the kink of e^-r that pair has h = 0 on the device and e^-r / r with an arbitrary direction
    dz / r in fp64.  Those roundings stay below r = 2^-10 here; distinct candidates are at least 0.01 / l from the
    data."""
    from oracle import gp_oracle as O
    kern = O.KERNELS[kind]
    k, h = kern.k(r2), kern.h(r2)
    if kind == "rbf":
        return k, h, 0.5 * r2, r2.clamp_min(0).sqrt()
    if kind == "matern12":
        h = torch.where(r2 < COINCIDENT, torch.zeros_like(r2), h)
    a = RATE[kind]
    t = a * r2.clamp_min(1e-30).sqrt()
    return k, h, t, torch.full_like(t, a)


def features64(gp, X, Xe, hyp, tables):
    """fp64 features of rows X [m, d] (None when d = 0) / Xe at fp64 hypers: MinMax, [Kumaraswamy warp], 1 / l, then the
    embedding features."""
    from oracle import gp_oracle as O
    parts = []
    if gp.d:
        xt = gp._x_mul.double() * X + gp._x_add.double()
        if gp.warp_mode:
            d, h = gp.d, gp._h_wa
            xt = O.kumaraswamy_warp(xt, hyp[h:h + d], hyp[h + d:h + 2 * d])
        parts.append(xt / hyp[3:3 + gp.d])
    if gp.num_enum:
        parts.append(gather_emb(gp, Xe, tables))
    return torch.cat(parts, 1)


def kmat64(gp, A, B, s):
    """s k(A, B) in fp64 by direct differences, in row blocks; differentiable."""
    from oracle import gp_oracle as O
    d = gp.d
    blk = max(1, (1 << 24) // max(1, B.shape[0] * A.shape[1]))
    rows = []
    for i0 in range(0, A.shape[0], blk):
        a = A[i0:i0 + blk]
        k = O.kernel_from_sqdist(((a[:, None, :d] - B[None, :, :d]) ** 2).sum(-1), gp.kernel)
        if gp.num_enum:
            k = k * O.kernel_from_sqdist(((a[:, None, d:] - B[None, :, d:]) ** 2).sum(-1), "matern32")
        rows.append(s * k)
    return torch.cat(rows)


_TRUE = {}


def true_model(gp, X, Xe, y):
    """The fp64 GP at the hyper-parameters of `gp`: training features, K + sigma_n^2 I [+ noise_diag], Cholesky, alpha.
    Rebuilt whenever gp's raw hypers are a new tensor (GP.set_hypers)."""
    key = id(gp)
    if key in _TRUE and _TRUE[key]["raw"] is gp.raw:
        return _TRUE[key]
    hyp = gp.hyp.double().to(DEV)
    tables = None
    if gp.num_enum:
        tables = torch.cat([t.reshape(-1) for t in emb_hypers(gp, gp.raw).tables]).to(DEV) / hyp[3 + gp.d]
    yt64 = (y.double().reshape(-1) - float(gp.yscaler.mean[0])) / float(gp.yscaler.std[0])
    Zt = features64(gp, None if X is None else X.double().to(DEV), None if Xe is None else Xe.to(DEV), hyp, tables)
    K = kmat64(gp, Zt, Zt, float(hyp[2]))
    K.diagonal().add_(float(hyp[0]))
    if gp.noise_diag is not None:
        K.diagonal().add_(torch.as_tensor(gp.noise_diag).double().to(DEV))
    L = torch.linalg.cholesky(K)
    c = float(hyp[1])
    alpha = torch.cholesky_solve((yt64.to(DEV) - c).reshape(-1, 1), L).reshape(-1)
    _TRUE[key] = dict(Zt=Zt, L=L, alpha=alpha, hyp=hyp, tables=tables, c=c, raw=gp.raw)
    return _TRUE[key]


# ---------------------------------------------------------------------------------------------------- deep ensemble
# The envelope of ensemble.cu at the shapes where its strided loops and leading dimensions matter (the row-float counts
# follow HB_DE_MAX_BATCH_FLOATS of include/hebo_b200.h).  Each case: the net, its data (n rows, the minibatch size) and
# the input generator's category range per column.
DE_CASES = {
    # 1583 floats per row: B = 35 is the largest admitted minibatch; n = 75 drops 5 rows per epoch
    "corner": dict(net=dict(num_cont=256, num_uniqs=[], num_layers=3, num_hiddens=256, num_out=8, rand_prior=True),
                   n=75, batch=35),
    # din = 6 + 5 x 50 = 256 > H: the input delta runs on h_ld = 257; column 0 draws 40 of 120 categories (repeats within a
    # minibatch, rows never drawn)
    "emb-wide": dict(net=dict(num_cont=6, num_uniqs=[120] * 5, num_layers=3, num_hiddens=16, num_out=3), n=70, batch=32,
                     cat_hi=[40, 120, 120, 120, 120]),
    "onehot-wide": dict(net=dict(num_cont=2, num_uniqs=[200, 54], enum_trans="onehot", num_layers=2, num_hiddens=8,
                                 num_out=2), n=70, batch=32),
    "default": dict(net=dict(num_cont=5, num_uniqs=[]), n=70, batch=32, E=5),
    "default-prior": dict(net=dict(num_cont=5, num_uniqs=[], rand_prior=True), n=70, batch=32, E=5),
    # 10 floats per row: B = 5600 is exactly the limit; n = 11 201 drops one row per epoch
    "big-batch": dict(net=dict(num_cont=1, num_uniqs=[], num_layers=1, num_hiddens=1), n=11201, batch=5600),
    # output 5 is NaN on every row, and row i has i % 7 more NaN outputs: 1 ... 7 per row
    "holes": dict(net=dict(num_cont=3, num_uniqs=[4, 7], num_layers=2, num_hiddens=64, num_out=8), n=70, batch=32,
                  holes=True),
    "small-n1": dict(net=dict(num_cont=2, num_uniqs=[3], num_layers=1, num_hiddens=8, num_out=2), n=1, batch=8),
    "small-n8": dict(net=dict(num_cont=2, num_uniqs=[3], num_layers=1, num_hiddens=8, num_out=2), n=8, batch=8),
    "small-n9": dict(net=dict(num_cont=2, num_uniqs=[3], num_layers=1, num_hiddens=8, num_out=2), n=9, batch=8),
}


def de_case(name, seed=0, output_noise=False, m=None):
    """(net kwargs, Xc [n, dc] fp32, Xe [n, ne] int32, y [n, O] fp32) of DE_CASES[name]; m rows instead of n when given
    (candidates for predict)."""
    c = DE_CASES[name]
    kw = dict(c["net"], output_noise=output_noise)
    dc, uniqs, O = kw["num_cont"], kw["num_uniqs"], kw.get("num_out", 1)
    n = c["n"] if m is None else m
    g = np.random.default_rng(seed)
    Xc = g.uniform(-1, 1, (n, dc)).astype(np.float32)
    hi = c.get("cat_hi", uniqs)
    Xe = np.stack([g.integers(0, h, n) for h in hi], 1).astype(np.int32) if uniqs else np.zeros((n, 0), np.int32)
    base = Xc.sum(1, keepdims=True) / max(1, dc) ** 0.5 + (Xe.sum(1, keepdims=True) % 5 if uniqs else 0)
    y = (np.sin(base + np.arange(O)) + 0.1 * g.standard_normal((n, O))).astype(np.float32)
    if c.get("holes") and m is None:
        y[:, 5] = np.nan
        for i in range(n):
            y[i, [k for k in range(O) if k != 5][:i % 7]] = np.nan
    return kw, Xc, Xe, y


U32 = 2.0 ** -24


def gamma32(N):
    return N * U32 / (1 - N * U32)


def de_initial(kw, seed, E=1) -> torch.Tensor:
    """[E, P] BaseNet initial weights of a DE_CASES net (xavier_uniform, zero biases) from torch's generator."""
    from hebo_b200.ensemble import init_params, param_layout
    lay, _ = param_layout(kw["num_cont"], kw["num_uniqs"], kw.get("enum_trans", "embedding"), kw.get("num_layers", 1),
                          kw.get("num_hiddens", 128), kw.get("num_out", 1), kw["output_noise"], kw.get("rand_prior", False))
    torch.manual_seed(seed)
    return torch.stack([init_params(lay) for _ in range(E)])


def de_abs_net(net):
    """A copy of net with |W| and |b| and no forward hooks (a caller's kink hooks must not reach the magnitudes)."""
    a = copy.deepcopy(net)
    for m in a.modules():
        m._forward_hooks.clear()
    with torch.no_grad():
        for p in a.parameters():
            p.abs_()
    return a


def _hidden_linears(net):
    return [m for m in net.hidden if isinstance(m, torch.nn.Linear)]


def de_depth(net):
    """(roundings of the forward chain to the heads, roundings of the backward chain from the heads to the input): a
    dense output is a K-term fmaf chain plus the bias add, ReLU and the prior add."""
    K = [net.din] + [net.H] * (net.L - 1)
    return sum(k + 2 for k in K) + net.H + 3, net.O * 2 + net.H * net.L + 2


def de_kink_units(net64, net32, run):
    """{layer: [B, H] bool} of the hidden units whose fp64 pre-activation z lies within its fp32 error bound of 0, where
    the device's ReLU may decide either way.  The bound is gamma_depth times z computed on |W|, |b| and the absolute
    inputs through the fp64 ReLU masks (a unit that is off by more than its bound is 0 in fp32 too, and adds no error).
    run(net) runs net64 on the rows."""
    lins = _hidden_linears(net64)
    z, xin = {}, []
    hooks = [m.register_forward_hook(lambda m_, i_, o_, l=l: z.__setitem__(l, o_.detach())) for l, m in enumerate(lins)]
    hooks.append(lins[0].register_forward_hook(lambda m_, i_, o_: xin.append(i_[0].detach())))
    try:
        run(net64)
    finally:
        for h in hooks:
            h.remove()
    a = xin[0].abs().numpy()
    depth, out = 0, {}
    for l, lin in enumerate(lins):
        depth += lin.in_features + 2
        zl = z[l].numpy()
        za = a @ lin.weight.detach().abs().numpy().T + lin.bias.detach().abs().numpy()
        out[l] = np.abs(zl) <= gamma32(depth) * za
        a = np.where((zl > 0) | out[l], za, 0.0)
    return out


@contextlib.contextmanager
def de_adopt_masks(net64, kinks, acts32):
    """Within the block, net64's ReLU at each kink unit passes the gradient exactly when the fp32 activation acts32[l]
    is positive (both are BaseNet's derivative there: the pre-activation is 0 within rounding); its value moves by
    less than the unit's bound."""
    def hook(l):
        def f(mod, inp, out):
            k = torch.from_numpy(kinks[l])
            if not bool(k.any()):
                return out
            tiny = torch.tensor(1e-300, dtype=out.dtype)
            s = torch.where(torch.from_numpy(acts32[l] > 0), tiny, -tiny)
            return torch.where(k, s + (out - out.detach()), out)       # value exactly s, derivative 1
        return f
    hooks = [m.register_forward_hook(hook(l)) for l, m in enumerate(_hidden_linears(net64))]
    try:
        yield
    finally:
        for h in hooks:
            h.remove()


def de_step_grad_bound(net64, net32, Xc, Xe, y, rows, l1, n):
    """(fp64 gradient, per-element bound on the fp32 step's error) of one minibatch, output_noise=False.  The bound is
    gamma_N times the same gradient taken on |W|, |x| and the seeds' magnitudes 2 (|t| + |mu|) / cnt (every unit active),
    plus the L1 coefficient's rounding; N is the longest chain of roundings from the inputs to a parameter's gradient."""
    from oracle import ensemble_oracle as EO
    rows = np.asarray(rows)
    xc = torch.from_numpy(Xc[rows]).double()
    xe = torch.from_numpy(Xe[rows]).long() if net32.uniqs else None
    t = torch.from_numpy(y[rows]).double()
    a = de_abs_net(net64)
    _, g64 = EO.step_grad(net64, torch.from_numpy(Xc).double(), torch.from_numpy(Xe).long() if net32.uniqs else None,
                          torch.from_numpy(y).double(), rows, l1, n)
    a.zero_grad()
    mu_a, _ = a(xc.abs(), xe)
    fin = torch.isfinite(t)
    seeds = torch.where(fin, 2 * (t.nan_to_num().abs() + mu_a.detach()) / fin.sum(), torch.zeros_like(t))
    (seeds * mu_a).sum().backward()
    ga = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in a.parameters()])
    f, b = de_depth(net32)
    coef = l1 / (n * net32.O)
    return g64.numpy(), (gamma32(f + b + len(rows) + 6) * ga).numpy() + 4 * U32 * coef + 1e-300


def _heads_and_input_grads(net, xc, xe, O):
    """(mu, z or None, dmu/dxc [B, O, dc], dz/dxc or None) of net at the numeric inputs xc (rows are independent)."""
    xc = xc.detach().clone().requires_grad_(True)
    zs = []
    h = net.sigma2[0].register_forward_hook(lambda m_, i_, o_: zs.append(o_)) if net.output_noise else None
    mu, _ = net(xc, xe)
    if h is not None:
        h.remove()
    heads = [mu] + zs
    grads = [torch.stack([torch.autograd.grad(t[:, o].sum(), xc, retain_graph=True)[0] for o in range(O)], 1) for t in heads]
    return mu.detach(), (zs[0].detach() if zs else None), grads[0], (grads[1] if zs else None)


def de_predict_fp64(net32, params, Xs, Xe, x_mul, x_add, y_mean, y_std):
    """BaseNet's ensemble predict in fp64 on the given rows and per-element bounds on the device's fp32 error:
    ({'mu', 'var', 'dmu', 'dvar'}: (fp64 value, bound)), kink units, hidden units.  Values come from EO.ensemble_predict
    and autograd.  Each bound restates the kernel's error chain: member heads within gamma_f of their |W|, |x| magnitude,
    the member mean and variance sums, softplus and its derivative through expf / log1pf (2 and 1 ulp, CUDA C Programming
    Guide, Mathematical Functions) on the NLL head, and the input-gradient backward within gamma_N of the |W| net's input
    gradient times the seeds' magnitudes and errors.  At kink units the fp64 ReLU takes the fp32 decision (de_adopt_masks)."""
    from oracle import ensemble_oracle as EO
    E, O, dc, noise = params.shape[0], net32.O, net32.dc, net32.noise
    f, b = de_depth(net32)
    f += 2                                                      # x_mul x + x_add
    gf, gN = gamma32(f + E + 4), gamma32(f + b + E + 6)
    xm, xa = torch.from_numpy(x_mul).double(), torch.from_numpy(x_add).double()
    ym, ys = torch.from_numpy(y_mean).double(), torch.from_numpy(y_std).double()
    X64 = torch.from_numpy(Xs).double()
    xe = torch.from_numpy(Xe).long() if net32.uniqs else None
    xc, xc_a = X64 * xm + xa, X64.abs() * xm.abs() + xa.abs()
    nets, kinks, per, stack = [], 0, [], contextlib.ExitStack()
    for e in range(E):
        net = EO.OracleNet(net32.dc, net32.uniqs, "embedding" if net32.emb else "onehot", net32.L, net32.H, O, noise,
                           net32.prior).load_raw(params[e])
        with torch.no_grad():
            k = de_kink_units(net, net32, lambda n_: n_(xc, xe))
        acts32, _, _ = EO.forward32(net32, params[e], EO.load_inputs32(net32, params[e], Xs, Xe, x_mul, x_add))
        kinks += sum(int(v.sum()) for v in k.values())
        a = de_abs_net(net)
        stack.enter_context(de_adopt_masks(net, k, acts32))
        nets.append(net)
        mu, z, gmu, gz = _heads_and_input_grads(net, xc, xe, O)
        mu_a, z_a, gmu_a, gz_a = _heads_and_input_grads(a, xc_a, xe, O)
        per.append((mu, z, mu_a.abs(), None if z is None else z_a.abs(), gmu_a, gz_a))
    with stack:
        X = X64.clone().requires_grad_(True)
        py, ps2 = EO.ensemble_predict(nets, X, xe, xm, xa, ym, ys, noise)
        dmu = torch.stack([torch.autograd.grad(py[:, o].sum(), X, retain_graph=True)[0] for o in range(O)], 1)
        dvar = torch.stack([torch.autograd.grad(ps2[:, o].sum(), X, retain_graph=True)[0] for o in range(O)], 1)
    mean = sum(p_[0] for p_ in per) / E
    mean_a = sum(p_[2] for p_ in per) / E
    e_py = gf * mean_a
    v_b, e_v, d_seed_mu, d_seed_z = 0.0, 0.0, [], []
    for mu, z, mu_a, z_a, _, _ in per:
        d = mu - mean
        e_d = gf * mu_a + e_py + U32 * d.abs()
        v_b = v_b + d * d / E
        e_v = e_v + (2 * d.abs() * e_d + e_d ** 2) / E
        d_seed_mu.append(2 / E * (e_d + gN * d.abs()))          # |error| of the pass-1 mu seed, backward rounding included
        if noise:
            sp = torch.nn.functional.softplus(z)
            sig = torch.sigmoid(z)
            e_z = gf * z_a
            e_s2 = e_z * sig + 8 * U32 * (1e-4 + sp)
            e_v = e_v + (e_s2 + gamma32(E + 2) * (1e-4 + sp)) / E
            d_seed_z.append((e_z * sig * (1 - sig) + 8 * U32 * sig + gN * sig) / E)
    v = ps2.detach() / ys ** 2
    e_v = e_v + gamma32(E + 4) * v
    x_scale = xm.abs()[None, None, :]
    b_dmu = sum(gN / E * p_[4] for p_ in per) * x_scale * ys.abs()[None, :, None]
    b_dvar = sum(s_[:, :, None] * p_[4] for s_, p_ in zip(d_seed_mu, per))
    if noise:
        b_dvar = b_dvar + sum(s_[:, :, None] * p_[5] for s_, p_ in zip(d_seed_z, per))
    b_dvar = b_dvar * x_scale * (ys ** 2)[None, :, None]
    out = {"mu": (py.detach(), gf * (mean_a * ys.abs() + ym.abs())),
           "var": (ps2.detach(), e_v * ys ** 2),
           "dmu": (dmu, b_dmu), "dvar": (dvar, b_dvar)}
    return {k_: (v_.numpy(), b_.numpy() + 1e-300) for k_, (v_, b_) in out.items()}, kinks, Xs.shape[0] * net32.H * net32.L * E


DE_PRED = [("holes", 1), ("holes", 2), ("holes", 32), ("corner", 2), ("emb-wide", 2), ("onehot-wide", 2), ("default-prior", 5)]


def de_predict_case(case, E, output_noise=False):
    """The predict set-up of tests/test_gpu_ensemble_envelope.py: perturbed initial weights (biases away from 0, members
    apart), 4097 candidates, scalers away from the identity."""
    from oracle import ensemble_oracle as EO
    kw, _, _, _ = de_case(case, output_noise=output_noise)
    _, Xs, Xe, _ = de_case(case, seed=21, m=4097)
    net = EO.Net32(**kw)
    g = np.random.default_rng(22)
    params = de_initial(kw, 12, E).numpy()
    params += (0.05 * g.standard_normal(params.shape)).astype(np.float32)
    xm = g.uniform(0.5, 2, net.dc).astype(np.float32)
    xa = g.uniform(-0.5, 0.5, net.dc).astype(np.float32)
    ym = g.standard_normal(net.O).astype(np.float32)
    ys = g.uniform(0.5, 3, net.O).astype(np.float32)
    pick = np.unique(np.r_[0:16, 15:18, 4080:4097, np.random.default_rng(23).integers(0, 4097, 8)])
    return kw, net, params, Xs, Xe, xm, xa, ym, ys, pick


def de_check_against_fp64(got, ref, kinks, units, what):
    """got (mu, var, dmu, dvar) against de_predict_fp64's values and bounds, per element; prints the largest ratio."""
    assert kinks <= units // 20, (kinks, units)
    ratios = []
    for name, g in zip(("mu", "var", "dmu", "dvar"), got):
        v, bnd = ref[name]
        err = np.abs(np.asarray(g, np.float64) - v)
        assert np.all(err <= bnd), f"{what} {name}: {int((err > bnd).sum())} over, worst {float(np.max(err / bnd)):.3g} x bound"
        ratios.append(f"{name} {float(np.max(err / bnd)):.3g}")
    print(f"{what}: error / bound " + ", ".join(ratios) + f"; kink units {kinks} of {units}")
