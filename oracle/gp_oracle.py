"""CPU oracle for the HEBO exact-GP fit + posterior + MACE hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``hebo_b200/`` may import this module;
only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs use it, and only as the checker / CPU baseline.

PARITY UNPINNED at the gpytorch boundary: the arithmetic of this path lives in the
third-party ``gpytorch`` package (``HEBO/requirements.txt:6`` ``gpytorch>=1.4.0``, unpinned,
not vendored in the reference repository), and no reference test holds a
numeric golden vector for it (``HEBO/test/util.py:13-19`` checks shape/finite/positive only).
What *is* pinned: the MACE arithmetic, the scalers and the pSGLD rule are checked against the
reference's real ``acq.py`` / ``scalers.py`` loaded by path (``oracle/ref_loader.py``,
``oracle/make_golden.py``) and against ``torch.optim.RMSprop``; the closed-form MLL gradient is
checked against torch autograd in fp64.

Everything here is plain torch on CPU, dtype-generic (fp64 for parity, fp32 for the CPU
baseline timing, which is what the reference itself computes in).

Semantics followed ("gpytorch ExactGP with Cholesky forced", SURVEY.md section 8a/Appendix A):
  * scaling            HEBO/hebo/models/gp/gp.py:51-71, HEBO/hebo/models/scalers.py:33-90
  * kernel + inits     HEBO/hebo/models/gp/gp_util.py:39-59
  * likelihood/prior   HEBO/hebo/models/gp/gp.py:86-91
  * fit loop           HEBO/hebo/models/gp/gp.py:96-126, HEBO/hebo/models/nn/sgld.py:49-70
  * predict            HEBO/hebo/models/gp/gp.py:137-164
  * noise              HEBO/hebo/models/gp/gp.py:182-184
  * MACE               HEBO/hebo/acquisitions/acq.py:131-171
  * kappa / tau        HEBO/hebo/optimizers/hebo.py:149-162
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Optional, Tuple

import numpy as np
import torch

MIN_VARIANCE_F32 = 1e-6          # gpytorch.settings.min_variance (float) -- MultivariateNormal.variance floor
EPS_F32 = float(torch.finfo(torch.float32).eps)   # gp.py:164 clamp, acq.py:153 clamp


# --------------------------------------------------------------------------- helpers
def softplus(u: torch.Tensor) -> torch.Tensor:
    return torch.nn.functional.softplus(u)


def inv_softplus(v: torch.Tensor) -> torch.Tensor:
    """gpytorch.utils.transforms.inv_softplus: x + log(-expm1(-x))."""
    return v + torch.log(-torch.expm1(-v))


# --------------------------------------------------------------------------- scalers
def minmax_fit(X: np.ndarray, lb: float = -1.0, ub: float = 1.0) -> Tuple[np.ndarray, np.ndarray]:
    """sklearn MinMaxScaler((lb, ub)).fit as used at scalers.py:73-81 (float32 in, float32 out).

    scale_ = (ub - lb) / range, range==0 -> 1 ; min_ = lb - data_min * scale_.
    """
    X = np.asarray(X)
    dmin = X.min(axis=0)
    dmax = X.max(axis=0)
    rng = dmax - dmin
    rng = np.where(rng < 10 * np.finfo(rng.dtype).eps, np.ones_like(rng), rng)
    scale = (ub - lb) / rng
    mn = lb - dmin * scale
    return scale.astype(np.float32), mn.astype(np.float32)


def standard_fit(y: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """sklearn StandardScaler().fit as used at scalers.py:40-51: mean_, sqrt(var_) (ddof=0);
    zero / non-finite std -> 1, non-finite mean -> 0."""
    y = np.asarray(y, dtype=np.float64)
    mean = y.mean(axis=0)
    var = y.var(axis=0)
    std = np.sqrt(var)
    # sklearn _handle_zeros_in_scale: scale < 10*eps -> 1
    std = np.where(std < 10 * np.finfo(np.float64).eps, 1.0, std)
    bad = ~(np.isfinite(mean) & np.isfinite(std))
    mean = np.where(bad, 0.0, mean)
    std = np.where(bad, 1.0, std)
    return mean.astype(np.float32), std.astype(np.float32)


# --------------------------------------------------------------------------- kernel
def scaled_sqdist(Z1: torch.Tensor, Z2: torch.Tensor) -> torch.Tensor:
    """Direct-difference squared distance of already 1/lengthscale-scaled rows."""
    diff = Z1[:, None, :] - Z2[None, :, :]
    return (diff * diff).sum(-1)


def _radius(r2: torch.Tensor) -> torch.Tensor:
    """gpytorch MaternKernel's r = sqrt(clamp_min(r^2, 1e-30)); clamp_min passes no gradient below its bound."""
    return torch.sqrt(torch.clamp_min(r2, 1e-30))


def _matern12(r2):
    return torch.exp(-_radius(r2))


def _matern12_h(r2):
    """e^-r / r is singular at r = 0; autograd through the clamp gives h = 0 below it, so a pair of equal rows
    contributes nothing to any gradient."""
    r = _radius(r2)
    return torch.where(r2 < 1e-30, torch.zeros_like(r2), torch.exp(-r) / r)


def _matern32(r2):
    a, r = math.sqrt(3.0), _radius(r2)
    return (1.0 + a * r) * torch.exp(-a * r)


def _matern32_h(r2):
    a, r = math.sqrt(3.0), _radius(r2)
    return a * a * torch.exp(-a * r)


def _matern52(r2):
    a, r = math.sqrt(5.0), _radius(r2)
    return (1.0 + a * r + (5.0 / 3.0) * r2) * torch.exp(-a * r)


def _matern52_h(r2):
    a, r = math.sqrt(5.0), _radius(r2)
    return (a * a / 3.0) * (1.0 + a * r) * torch.exp(-a * r)


def _rbf(r2):
    return torch.exp(-0.5 * r2)


@dataclass(frozen=True)
class Kernel:
    """One covariance kernel at unit outputscale as a function of the scaled squared distance r^2."""
    id: int                # HB_KERN_* of include/hebo_b200.h
    k: Callable[[torch.Tensor], torch.Tensor]
    h: Callable[[torch.Tensor], torch.Tensor]      # radial factor, dk/dr^2 = -h / 2 (SURVEY Appendix A)


# gpytorch MaternKernel(nu = 0.5, 1.5, 2.5).forward and RBFKernel.  The Matern-3/2 and -5/2 h keep a * a rather than 3:
# the committed fixtures were computed with it.
KERNELS = {
    "matern32": Kernel(0, _matern32, _matern32_h),
    "matern52": Kernel(1, _matern52, _matern52_h),
    "rbf": Kernel(2, _rbf, _rbf),
    "matern12": Kernel(4, _matern12, _matern12_h),
}


def kernel_from_sqdist(r2: torch.Tensor, kind: str) -> torch.Tensor:
    return KERNELS[kind].k(r2)


KERNEL_FORM = "direct"   # "direct": sum((zi-zj)^2), used for parity; "mm": gpytorch's matmul form, used by the
                         # CPU-baseline timing legs of bench.py (what the reference's CPU path actually executes)


def sqdist_mm(Z1: torch.Tensor, Z2: torch.Tensor) -> torch.Tensor:
    """gpytorch.kernels.kernel.sq_dist (recalled from gpytorch 1.x; not vendored): centre on the mean, then
    ||a||^2 + ||b||^2 - 2 a.b as ONE matmul of augmented operands, clamp at 0."""
    adj = Z1.mean(-2, keepdim=True)
    a, b = Z1 - adj, Z2 - adj
    an, bn = a.pow(2).sum(-1, keepdim=True), b.pow(2).sum(-1, keepdim=True)
    a_ = torch.cat([-2.0 * a, an, torch.ones_like(an)], -1)
    b_ = torch.cat([b, torch.ones_like(bn), bn], -1)
    return (a_ @ b_.transpose(-2, -1)).clamp_min(0)


def kernel_matrix(X1: torch.Tensor, X2: torch.Tensor, ls: torch.Tensor, kind: str,
                  block: int = 1024) -> torch.Tensor:
    """k(X1, X2) with ARD lengthscales, unit outputscale; blocked so that m x n x d never exists."""
    Z1 = X1 / ls
    Z2 = X2 / ls
    if KERNEL_FORM == "mm":
        return kernel_from_sqdist(sqdist_mm(Z1, Z2), kind)
    out = torch.empty(X1.shape[0], X2.shape[0], dtype=X1.dtype)
    for i in range(0, X1.shape[0], block):
        for j in range(0, X2.shape[0], block):
            out[i:i + block, j:j + block] = kernel_from_sqdist(
                scaled_sqdist(Z1[i:i + block], Z2[j:j + block]), kind)
    return out


def kumaraswamy_warp(Xt: torch.Tensor, a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Kumaraswamy CDF input warp on MinMax(-1,1)-scaled inputs (config 3; the only definition in the
    reference is HEBO/hebo/models/nn/mono_layers/layers.py:85-117 / gpy_wgp.py:120-128):
    u = clamp((x+1)/2, eps, 1-eps); w = 1 - (1 - u^a)^b ; returned mapped back to [-1, 1]."""
    eps = 1e-6
    u = ((Xt + 1.0) * 0.5).clamp(eps, 1.0 - eps)
    w = 1.0 - (1.0 - u ** a) ** b
    return 2.0 * w - 1.0


# --------------------------------------------------------------------------- hyper-parameters
@dataclass
class Hypers:
    """Raw (unconstrained) parameters in gpytorch registration order (SURVEY Appendix A):
    raw_noise, mean constant, raw_outputscale, raw_lengthscale[d]."""
    raw_noise: torch.Tensor      # scalar
    mean: torch.Tensor           # scalar
    raw_os: torch.Tensor         # scalar
    raw_ls: torch.Tensor         # [d]
    noise_lb: float = 8e-4

    def pack(self) -> torch.Tensor:
        return torch.cat([self.raw_noise.reshape(1), self.mean.reshape(1),
                          self.raw_os.reshape(1), self.raw_ls.reshape(-1)])

    @staticmethod
    def unpack(vec: torch.Tensor, noise_lb: float) -> "Hypers":
        return Hypers(vec[0], vec[1], vec[2], vec[3:], noise_lb)

    @property
    def noise(self):
        return softplus(self.raw_noise) + self.noise_lb

    @property
    def outputscale(self):
        return softplus(self.raw_os)

    @property
    def lengthscale(self):
        return softplus(self.raw_ls)

    def to(self, dtype):
        return Hypers(self.raw_noise.to(dtype), self.mean.to(dtype), self.raw_os.to(dtype),
                      self.raw_ls.to(dtype), self.noise_lb)


def init_lengthscales(Xt: torch.Tensor, max_x: int = 1000, rng: Optional[np.random.RandomState] = None
                      ) -> torch.Tensor:
    """gp_util.py:47-52: per-dim median pairwise |dx| over <= max_x rows (np.random.choice per dim),
    clamp >= 0.02.  torch.pdist(...).median() returns the LOWER median for even counts."""
    n, d = Xt.shape
    out = torch.empty(d, dtype=Xt.dtype)
    for i in range(d):
        if rng is None:
            idx = np.random.choice(n, min(n, max_x), replace=False)
        else:
            idx = rng.choice(n, min(n, max_x), replace=False)
        out[i] = torch.pdist(Xt[idx, i].view(-1, 1)).median().clamp(min=0.02)
    return out


def init_hypers(Xt: torch.Tensor, yt: torch.Tensor, noise_lb: float = 8e-4, ard: bool = True,
                rng: Optional[np.random.RandomState] = None) -> Hypers:
    """gp.py:86-91 + gp_util.py:39-59 initial values (in raw space)."""
    dt = Xt.dtype
    d = Xt.shape[1]
    if ard:
        ls = init_lengthscales(Xt, rng=rng)
    else:
        ls = torch.full((d,), math.log(2.0), dtype=dt)     # gpytorch default raw=0 -> softplus(0)
    os_ = yt[torch.isfinite(yt)].var()                     # unbiased, gp_util.py:58
    noise = torch.tensor(max(1e-2, noise_lb), dtype=dt)    # gp.py:91
    return Hypers(raw_noise=inv_softplus(noise - noise_lb),
                  mean=torch.zeros((), dtype=dt),
                  raw_os=inv_softplus(os_.to(dt)),
                  raw_ls=inv_softplus(ls.to(dt)),
                  noise_lb=noise_lb)


# --------------------------------------------------------------------------- MLL
def neg_mll(Xt: torch.Tensor, yt: torch.Tensor, hp: Hypers, kind: str = "matern32",
            noise_guess: float = 0.01, noise_diag: Optional[torch.Tensor] = None,
            jitter: float = 0.0) -> torch.Tensor:
    """loss = -ExactMarginalLogLikelihood / n including the Gamma(.5,.5) outputscale prior and
    the LogNormal(ln noise_guess, .5) noise prior (gp.py:86-88,102,113; gp_util.py:57).
    Differentiable (autograd) in hp."""
    n = Xt.shape[0]
    s, sn2, ls, c = hp.outputscale, hp.noise, hp.lengthscale, hp.mean
    K = s * kernel_matrix(Xt, Xt, ls, kind)
    diag = sn2 + jitter
    Khat = K + torch.eye(n, dtype=Xt.dtype) * diag
    if noise_diag is not None:
        Khat = Khat + torch.diag(noise_diag)
    L = torch.linalg.cholesky(Khat)
    r = (yt.reshape(-1) - c).reshape(-1, 1)
    v = torch.linalg.solve_triangular(L, r, upper=False)
    quad = (v * v).sum()
    logdet = 2.0 * torch.log(torch.diagonal(L)).sum()
    data = -0.5 * (quad + logdet + n * math.log(2.0 * math.pi))
    lp_os = 0.5 * math.log(0.5) - math.lgamma(0.5) - 0.5 * torch.log(s) - 0.5 * s
    sig0 = 0.5
    mu0 = math.log(noise_guess)
    lp_n = -torch.log(sn2 * sig0 * math.sqrt(2.0 * math.pi)) - (torch.log(sn2) - mu0) ** 2 / (2 * sig0 ** 2)
    return -(data + lp_os + lp_n) / n


def neg_mll_autograd(Xt, yt, hp: Hypers, kind="matern32", noise_guess=0.01, noise_diag=None):
    vec = hp.pack().detach().clone().requires_grad_(True)
    loss = neg_mll(Xt, yt, Hypers.unpack(vec, hp.noise_lb), kind, noise_guess, noise_diag)
    (g,) = torch.autograd.grad(loss, vec)
    return loss.detach(), g


def neg_mll_closed_form(Xt, yt, hp: Hypers, kind="matern32", noise_guess=0.01, noise_diag=None, block: int = 128
                        ) -> Tuple[torch.Tensor, torch.Tensor, dict]:
    """Same loss, gradient by the closed forms of SURVEY Appendix A (what the CUDA path implements):
    alpha = Khat^-1 r ; W = alpha alpha^T - Khat^-1 ; d(data)/dtheta = 1/2 tr(W dKhat/dtheta).

    The pairwise differences are formed ``block`` rows at a time, so memory stays O(n^2 + block n d): the full
    [n, n, d] difference tensor would be 4.6 GB in fp64 at n = 4224, d = 32."""
    n, d = Xt.shape
    dt = Xt.dtype
    s, sn2, ls, c = hp.outputscale, hp.noise, hp.lengthscale, hp.mean
    Z = Xt / ls
    r2 = torch.empty(n, n, dtype=dt)
    for i0 in range(0, n, block):
        r2[i0:i0 + block] = scaled_sqdist(Z[i0:i0 + block], Z)
    k = kernel_from_sqdist(r2, kind)
    Khat = s * k + torch.eye(n, dtype=dt) * sn2
    if noise_diag is not None:
        Khat = Khat + torch.diag(noise_diag)
    L = torch.linalg.cholesky(Khat)
    rvec = (yt.reshape(-1) - c)
    Linv = torch.linalg.solve_triangular(L, torch.eye(n, dtype=dt), upper=False)
    Kinv = Linv.T @ Linv
    alpha = Kinv @ rvec
    quad = rvec @ alpha
    logdet = 2.0 * torch.log(torch.diagonal(L)).sum()
    W = torch.outer(alpha, alpha) - Kinv
    # radial derivative factor  h(r) with dk/dl_k = h * dz_k^2 / l_k   (dz = scaled difference)
    G = W * KERNELS[kind].h(r2) * s                          # [n,n]
    g_ls = torch.zeros(d, dtype=dt)
    for i0 in range(0, n, block):
        dZ2 = (Z[i0:i0 + block, None, :] - Z[None, :, :]) ** 2   # [block,n,d]
        g_ls = g_ls + torch.einsum("ij,ijk->k", G[i0:i0 + block], dZ2)
    g_ls = 0.5 * g_ls / ls
    g_s = 0.5 * (W * k).sum()
    g_n = 0.5 * torch.diagonal(W).sum()
    g_c = alpha.sum()
    # priors (on the transformed values)
    g_s = g_s + (-0.5 / s - 0.5)
    sig0, mu0 = 0.5, math.log(noise_guess)
    g_n = g_n + (-1.0 / sn2 - (torch.log(sn2) - mu0) / (sig0 ** 2 * sn2))
    # chain through softplus, negate, divide by n
    sg = torch.sigmoid
    grad = torch.cat([(g_n * sg(hp.raw_noise)).reshape(1), g_c.reshape(1),
                      (g_s * sg(hp.raw_os)).reshape(1), g_ls * sg(hp.raw_ls)]) * (-1.0 / n)
    data = -0.5 * (quad + logdet + n * math.log(2.0 * math.pi))
    lp_os = 0.5 * math.log(0.5) - math.lgamma(0.5) - 0.5 * torch.log(s) - 0.5 * s
    lp_n = -torch.log(sn2 * sig0 * math.sqrt(2.0 * math.pi)) - (torch.log(sn2) - mu0) ** 2 / (2 * sig0 ** 2)
    loss = -(data + lp_os + lp_n) / n
    aux = dict(K=Khat, L=L, Linv=Linv, Kinv=Kinv, alpha=alpha, quad=quad, logdet=logdet)
    return loss, grad, aux


# --------------------------------------------------------------------------- pSGLD
@dataclass
class PSGLDState:
    square_avg: torch.Tensor
    n_step: int = 0


def psgld_step(vec: torch.Tensor, grad: torch.Tensor, st: PSGLDState, lr: float, factor: float,
               pretrain_step: int, xi: Optional[torch.Tensor], alpha: float = 0.99, eps: float = 1e-8
               ) -> torch.Tensor:
    """sgld.py:49-70 on top of torch.optim.RMSprop (momentum=0, centered=False, weight_decay=0):
    v <- a v + (1-a) g^2 ; p <- p - lr g / (sqrt(v)+eps) ; n_step += 1 ;
    if n_step > pretrain_step: p += factor * sqrt(2 lr / (sqrt(v)+eps)) * xi."""
    st.square_avg = alpha * st.square_avg + (1 - alpha) * grad * grad
    avg = st.square_avg.sqrt() + eps
    vec = vec - lr * grad / avg
    st.n_step += 1
    if st.n_step > pretrain_step and xi is not None:
        vec = vec + factor * torch.sqrt(2 * lr / avg) * xi
    return vec


def fit_psgld(Xt, yt, hp0: Hypers, kind="matern32", lr=0.01, num_epochs=100, noise_guess=0.01,
              noise_diag=None, langevin: Optional[torch.Tensor] = None, closed_form: bool = True,
              record: bool = False):
    """gp.py:96-126 with optimizer='psgld' (the default).  ``langevin`` [num_epochs, P] holds the
    N(0,1) draws the reference takes with torch.randn_like per parameter tensor in registration
    order; None = no Langevin noise (deterministic RMSprop)."""
    n = Xt.shape[0]
    vec = hp0.pack().clone()
    st = PSGLDState(torch.zeros_like(vec))
    losses = []
    for ep in range(num_epochs):
        hp = Hypers.unpack(vec, hp0.noise_lb)
        if closed_form:
            loss, g, _ = neg_mll_closed_form(Xt, yt, hp, kind, noise_guess, noise_diag)
        else:
            loss, g = neg_mll_autograd(Xt, yt, hp, kind, noise_guess, noise_diag)
        xi = None if langevin is None else langevin[ep].to(vec.dtype)
        vec = psgld_step(vec, g, st, lr, 1.0 / n, num_epochs // 10, xi)
        losses.append(float(loss))
    hp = Hypers.unpack(vec, hp0.noise_lb)
    return (hp, losses) if record else hp


def fit_torch_optimizer(Xt, yt, hp0: Hypers, optimizer: str, kind="matern32", lr=0.01, num_epochs=100, noise_guess=0.01,
                        record: bool = False):
    """gp.py:96-126 with optimizer='lbfgs' (torch LBFGS, max_iter=5, strong Wolfe) or any other name (torch Adam): the
    reference's own optimizer objects on the autograd of neg_mll."""
    vec = torch.nn.Parameter(hp0.pack().clone())
    if optimizer.lower() == "lbfgs":
        opt = torch.optim.LBFGS([vec], lr=lr, max_iter=5, line_search_fn="strong_wolfe")
    else:
        opt = torch.optim.Adam([vec], lr=lr)
    losses = []
    for ep in range(num_epochs):
        seen = []

        def closure():
            opt.zero_grad()
            loss = neg_mll(Xt, yt, Hypers.unpack(vec, hp0.noise_lb), kind, noise_guess)
            loss.backward()
            if not seen:
                seen.append(float(loss.detach()))
            return loss
        opt.step(closure)
        losses.append(seen[0])
    hp = Hypers.unpack(vec.detach(), hp0.noise_lb)
    return (hp, losses) if record else hp


# --------------------------------------------------------------------------- posterior
@dataclass
class FittedGP:
    """Everything predict() needs (gp.py:137-164)."""
    Xt: torch.Tensor            # scaled training inputs [n,d]
    hp: Hypers
    kind: str
    x_scale: torch.Tensor       # MinMax scale_ [d]
    x_min: torch.Tensor         # MinMax min_   [d]
    y_mean: float
    y_std: float
    L: torch.Tensor = field(repr=False, default=None)
    alpha: torch.Tensor = field(repr=False, default=None)
    pred_likeli: bool = False
    noise_diag: Optional[torch.Tensor] = None

    @property
    def noise(self) -> torch.Tensor:
        """gp.py:182-184: sigma_n^2 * std_y^2, shape [1]."""
        return (self.hp.noise * self.y_std ** 2).reshape(1)


def make_fitted(Xc_raw: torch.Tensor, y_raw: torch.Tensor, hp: Optional[Hypers] = None, kind="matern32",
                dtype=torch.float64, noise_lb=8e-4, pred_likeli=False, noise_diag=None,
                rng: Optional[np.random.RandomState] = None) -> FittedGP:
    """Scalers (fit in numpy as the reference does, applied in ``dtype``) + factorisation at ``hp``
    (default: the reference initial hypers)."""
    sc, mn = minmax_fit(Xc_raw.numpy().astype(np.float32))
    ym, ys = standard_fit(y_raw.numpy().astype(np.float32).reshape(-1, 1))
    sc_t, mn_t = torch.from_numpy(sc).to(dtype), torch.from_numpy(mn).to(dtype)
    Xt = sc_t * Xc_raw.to(dtype) + mn_t
    yt = (y_raw.to(dtype).reshape(-1) - float(ym[0])) / float(ys[0])
    if hp is None:
        hp = init_hypers(Xt, yt, noise_lb, rng=rng)
    hp = hp.to(dtype)
    f = FittedGP(Xt, hp, kind, sc_t, mn_t, float(ym[0]), float(ys[0]), pred_likeli=pred_likeli,
                 noise_diag=noise_diag)
    f._yt = yt
    refactor(f)
    return f


def refactor(f: FittedGP) -> None:
    n = f.Xt.shape[0]
    K = f.hp.outputscale * kernel_matrix(f.Xt, f.Xt, f.hp.lengthscale, f.kind)
    K = K + torch.eye(n, dtype=K.dtype) * f.hp.noise
    if f.noise_diag is not None:
        K = K + torch.diag(f.noise_diag.to(K.dtype))
    f.L = torch.linalg.cholesky(K)
    r = (f._yt - f.hp.mean).reshape(-1, 1)
    f.alpha = torch.cholesky_solve(r, f.L).reshape(-1)


def predict(f: FittedGP, Xc_raw: torch.Tensor, block: int = 2048) -> Tuple[torch.Tensor, torch.Tensor]:
    """gp.py:137-164.  Returns (mu [m,1], var [m,1]) in original y units."""
    dt = f.Xt.dtype
    Xs = f.x_scale * Xc_raw.to(dt) + f.x_min
    m = Xs.shape[0]
    mu = torch.empty(m, dtype=dt)
    var = torch.empty(m, dtype=dt)
    s = f.hp.outputscale
    for i in range(0, m, block):
        Ks = s * kernel_matrix(Xs[i:i + block], f.Xt, f.hp.lengthscale, f.kind)     # [b,n]
        mu[i:i + block] = f.hp.mean + Ks @ f.alpha
        V = torch.linalg.solve_triangular(f.L, Ks.T, upper=False)                  # [n,b]
        var[i:i + block] = s - (V * V).sum(0)
    if f.pred_likeli:
        var = var + f.hp.noise                            # gp.py:158-159 (GaussianLikelihood adds noise to the covariance)
    var = var.clamp_min(MIN_VARIANCE_F32)                 # gp.py:161 .variance: gpytorch MultivariateNormal.variance floor
    mu = mu * f.y_std + f.y_mean                          # gp.py:162
    var = (var * f.y_std ** 2).clamp_min(EPS_F32)         # gp.py:163-164
    return mu.reshape(-1, 1), var.reshape(-1, 1)


# --------------------------------------------------------------------------- MACE
def mace(mu: torch.Tensor, var: torch.Tensor, noise_var: float, tau: float, kappa: float,
         eps: float, xi1: torch.Tensor, xi2: torch.Tensor) -> torch.Tensor:
    """acq.py:146-171 restated in the dtype of ``mu`` (columns: LCB, -log EI, -log PI)."""
    dt = mu.dtype
    py = mu.reshape(-1)
    ps2 = var.reshape(-1)
    noise = math.sqrt(2.0) * math.sqrt(noise_var)
    ps = ps2.sqrt().clamp(min=EPS_F32)
    lcb = (py + noise * xi1.reshape(-1).to(dt)) - kappa * ps
    z = (tau - eps - py - noise * xi2.reshape(-1).to(dt)) / ps
    log_phi = -0.5 * z * z - 0.5 * math.log(2 * math.pi)
    Phi = 0.5 * (1.0 + torch.erf(z / math.sqrt(2.0)))
    EI = ps * (Phi * z + log_phi.exp())
    logEIapp = ps.log() - 0.5 * z ** 2 - (z ** 2 - 1).log()
    logPIapp = -0.5 * z ** 2 - torch.log(-z) - math.log(math.sqrt(2 * math.pi))
    use_app = ~((z > -6) & torch.isfinite(EI.log()) & torch.isfinite(Phi.log()))
    out = torch.zeros(py.shape[0], 3, dtype=dt)
    out[:, 0] = lcb
    out[:, 1] = torch.where(use_app, -logEIapp, -EI.log())
    out[:, 2] = torch.where(use_app, -logPIapp, -Phi.log())
    return out


def kappa_schedule(n_obs: int, q: int, D: int, upsi: float = 0.5, delta: float = 0.01) -> float:
    """hebo.py:156-160."""
    it = max(1, n_obs // q)
    return float(np.sqrt(upsi * 2 * ((2.0 + D / 2.0) * np.log(it) + np.log(3 * np.pi ** 2 / (3 * delta)))))


# --------------------------------------------------------------------------- Pareto front
def pareto_front(F: np.ndarray) -> np.ndarray:
    """Indices of the non-dominated rows of F (all objectives minimised); a dominates b iff
    all(a <= b) and any(a < b) -- the rank-0 set pymoo's NSGA-II returns as res.X
    (evolution_optimizer.py:141).  O(m * |front|) with an incremental front; exact.
    Rows with a NaN objective are excluded: they can neither dominate nor be dominated, and the selection step
    (hebo.py:182-193) must never receive a candidate whose acquisition value is NaN."""
    F = np.asarray(F)
    m = F.shape[0]
    order = np.lexsort(tuple(F[:, k] for k in range(F.shape[1] - 1, -1, -1)))   # sort by col0, col1, ...
    front: list[int] = []
    FF = np.empty((0, F.shape[1]), dtype=F.dtype)
    for idx in order:
        p = F[idx]
        if np.isnan(p).any():
            continue
        if FF.shape[0]:
            dom = np.all(FF <= p, axis=1) & np.any(FF < p, axis=1)
            if dom.any():
                continue
        front.append(int(idx))
        FF = np.vstack([FF, p[None]])
    return np.sort(np.asarray(front, dtype=np.int64))


def pareto_front_bruteforce(F: np.ndarray) -> np.ndarray:
    F = np.asarray(F)
    keep = []
    for i in range(F.shape[0]):
        if np.isnan(F[i]).any():
            continue
        dom = np.all(F <= F[i], axis=1) & np.any(F < F[i], axis=1)
        if not dom.any():
            keep.append(i)
    return np.asarray(keep, dtype=np.int64)


# --------------------------------------------------------------------------- synthetic objectives
def branin(X: np.ndarray) -> np.ndarray:
    """Branin on x1 in [-5,10], x2 in [0,15] (synthetic_benchmarks.py:22-60 wraps pymoo's)."""
    x1, x2 = X[:, 0], X[:, 1]
    a, b, c, r, s, t = 1.0, 5.1 / (4 * np.pi ** 2), 5 / np.pi, 6.0, 10.0, 1 / (8 * np.pi)
    return a * (x2 - b * x1 ** 2 + c * x1 - r) ** 2 + s * (1 - t) * np.cos(x1) + s


def ackley(X: np.ndarray, a=20.0, b=0.2, c=2 * np.pi) -> np.ndarray:
    d = X.shape[1]
    return (-a * np.exp(-b * np.sqrt((X ** 2).sum(1) / d)) - np.exp(np.cos(c * X).sum(1) / d) + a + np.e)


_H6_A = np.array([[10, 3, 17, 3.5, 1.7, 8], [0.05, 10, 17, 0.1, 8, 14],
                  [3, 3.5, 1.7, 10, 17, 8], [17, 8, 0.05, 10, 0.1, 14]])
_H6_P = 1e-4 * np.array([[1312, 1696, 5569, 124, 8283, 5886], [2329, 4135, 8307, 3736, 1004, 9991],
                         [2348, 1451, 3522, 2883, 3047, 6650], [4047, 8828, 8732, 5743, 1091, 381]])
_H6_ALPHA = np.array([1.0, 1.2, 3.0, 3.2])


def hartmann6(X01: np.ndarray) -> np.ndarray:
    """Hartmann-6 on the first 6 dims of X01 in [0,1]^d (the 'Hartmann6Dummy' embedding,
    synthetic_benchmarks.py:115-117)."""
    x = X01[:, :6]
    inner = (_H6_A[None] * (x[:, None, :] - _H6_P[None]) ** 2).sum(-1)
    return -(_H6_ALPHA[None] * np.exp(-inner)).sum(1)


def synthetic_problem(cfg: str, n: int, d: int, seed: int):
    """Seeded (X in model space U(-1,1)^d, y) per BASELINE.md section 4."""
    g = torch.Generator().manual_seed(seed)
    X = torch.rand(n, d, generator=g, dtype=torch.float64) * 2 - 1
    Xn = X.numpy()
    if cfg == "branin":
        Xp = np.stack([(Xn[:, 0] + 1) * 7.5 - 5, (Xn[:, 1] + 1) * 7.5], 1)
        y = branin(Xp)
    elif cfg == "ackley":
        y = ackley((Xn + 1) * 7.5 - 5)
    elif cfg == "hartmann6":
        y = hartmann6((Xn + 1) * 0.5)
    else:
        raise ValueError(cfg)
    y = y + 0.05 * torch.randn(n, generator=g, dtype=torch.float64).numpy()
    return X, torch.from_numpy(y)


def hebo_y_transform(y: np.ndarray) -> np.ndarray:
    """hebo.py:128-135 (+ fallback 144-147): power-transform of y/std (sklearn, host)."""
    from sklearn.preprocessing import power_transform
    y = np.asarray(y, dtype=np.float64).reshape(-1, 1)
    try:
        if y.min() <= 0:
            t = power_transform(y / y.std(), method="yeo-johnson")
        else:
            t = power_transform(y / y.std(), method="box-cox")
            if t.std() < 0.5:
                t = power_transform(y / y.std(), method="yeo-johnson")
        if t.std() < 0.5:
            raise RuntimeError("Power transformation failed")
        return t.astype(np.float32)
    except Exception:
        return y.astype(np.float32)
