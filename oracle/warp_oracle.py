"""CPU oracle of the exact GP with a LEARNED Kumaraswamy input warp (BASELINE config 3 "input-warped").

TEST INFRASTRUCTURE ONLY (same rules as gp_oracle.py).  The reference's registered torch GP has no input warping; the only
definitions in the tree are the torch layer KumarWarp (HEBO/hebo/models/nn/mono_layers/layers.py:85-117: a, b =
0.01 + 9.99 sigmoid(raw), w(x) = 1 - (1 - clamp(x, eps, 1 - eps)^a)^b, eps = 1e-6) and GPy's InputWarpedGP
(HEBO/hebo/models/gp/gpy_wgp.py:120-128, Xmin = -1, Xmax = 1 on the MinMax-scaled numeric columns).  The model here chains
them the way `hebo_b200.GP(warp=True)` does: x~ in [-1, 1] -> u = (x~ + 1) / 2 -> w(u) -> 2 w - 1 -> ARD kernel.  PARITY
UNPINNED (no reference implementation of this combination exists); gradients come from torch autograd in fp64.

Parameter vector (registration order, include/hebo_b200.h): raw_noise, raw_a[d], raw_b[d], mean, raw_outputscale, raw_ls[d].
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .gp_oracle import PSGLDState, kernel_from_sqdist, psgld_step, softplus

LO, HI, EPS = 0.01, 10.0, 1e-6
# The clamp bounds as fp32 numbers: the kernels and the reference layer on fp32 tensors compare u with these.  fp32(1 - eps)
# = 1 - 1.0133e-6, so log u there is 1.3 % further from 0 than in fp64; at a, b <= 0.1 that moves w by up to 4e-4.
U32 = (float(np.float32(EPS)), float(np.float32(1.0 - EPS)))


def exponents(raw: torch.Tensor) -> torch.Tensor:
    return LO + (HI - LO) * torch.sigmoid(raw)


def warp(Xt: torch.Tensor, a: torch.Tensor, b: torch.Tensor, bounds=(EPS, 1.0 - EPS)) -> torch.Tensor:
    u = ((Xt + 1.0) * 0.5).clamp(*bounds)
    return 2.0 * (1.0 - (1.0 - u ** a) ** b) - 1.0


def warp32(Xt: torch.Tensor, a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """warp at the fp32 clamp bounds U32: the function the kernels evaluate."""
    return warp(Xt, a, b, U32)


def warp_stable(Xt: torch.Tensor, a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """warp32 with 1 - u^a formed as -expm1(a log u), as kumar_warp (common.cuh) forms it.  Differentiable in any dtype:
    fp32 autograd of `warp` cancels 1 - u^a to 0 at the upper clamp once a <= 0.031 and gives d/db = NaN or -0 there."""
    u = ((Xt + 1.0) * 0.5).clamp(*U32)
    return 2.0 * (1.0 - torch.exp(b * torch.log(-torch.expm1(a * torch.log(u))))) - 1.0


def kumar_warp_f32(x: torch.Tensor, a: torch.Tensor, b: torch.Tensor):
    """kumar_warp (common.cuh) operation by operation in fp32: (w, dw/da, dw/db).  Each CUDA expf / logf / expm1f is within
    2 ulp of the correctly rounded value torch's CPU functions give, so this is a restatement up to those ulps, not bytes."""
    f = torch.float32
    x, a, b = x.to(f), a.to(f), b.to(f)
    u = torch.clamp((x + 1.0) * 0.5, *U32)
    lu = torch.log(u)
    lom = torch.log(-torch.expm1(a * lu))
    p = torch.exp(b * lom)
    da = 2.0 * b * torch.exp((b - 1.0) * lom) * torch.exp(a * lu) * lu
    db = -2.0 * p * lom
    return 2.0 * (1.0 - p) - 1.0, da, db


def warp_derivatives64(x: torch.Tensor, a: torch.Tensor, b: torch.Tensor):
    """(w, dw/da, dw/db) of warp32 in fp64 by autograd, element by element (x, a, b broadcast to one shape)."""
    x, a, b = torch.broadcast_tensors(x.double(), a.double(), b.double())
    a, b = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    w = warp32(x, a, b)
    da, db = torch.autograd.grad(w.sum(), (a, b))
    return w.detach(), da, db


def unpack(vec: torch.Tensor, d: int):
    return dict(raw_noise=vec[0], raw_a=vec[1:1 + d], raw_b=vec[1 + d:1 + 2 * d], mean=vec[1 + 2 * d], raw_os=vec[2 + 2 * d],
                raw_ls=vec[3 + 2 * d:3 + 3 * d])


def _kernel(Z1, Z2, kind):
    r2 = ((Z1[:, None, :] - Z2[None, :, :]) ** 2).sum(-1)
    return kernel_from_sqdist(r2, kind)


def neg_mll(Xt, yt, vec, noise_lb=8e-4, kind="matern32", noise_guess=0.01, warp_fn=warp):
    n, d = Xt.shape
    p = unpack(vec, d)
    s, sn2 = softplus(p["raw_os"]), softplus(p["raw_noise"]) + noise_lb
    Z = warp_fn(Xt, exponents(p["raw_a"]), exponents(p["raw_b"])) / softplus(p["raw_ls"])
    K = s * _kernel(Z, Z, kind) + torch.eye(n, dtype=Xt.dtype) * sn2
    L = torch.linalg.cholesky(K)
    v = torch.linalg.solve_triangular(L, (yt.reshape(-1) - p["mean"]).reshape(-1, 1), upper=False)
    data = -0.5 * ((v * v).sum() + 2.0 * torch.log(torch.diagonal(L)).sum() + n * math.log(2.0 * math.pi))
    lp_os = 0.5 * math.log(0.5) - math.lgamma(0.5) - 0.5 * torch.log(s) - 0.5 * s
    sig0, mu0 = 0.5, math.log(noise_guess)
    lp_n = -torch.log(sn2 * sig0 * math.sqrt(2.0 * math.pi)) - (torch.log(sn2) - mu0) ** 2 / (2 * sig0 ** 2)
    return -(data + lp_os + lp_n) / n


def neg_mll_autograd(Xt, yt, vec, noise_lb=8e-4, kind="matern32", noise_guess=0.01, warp_fn=warp):
    v = vec.detach().clone().requires_grad_(True)
    loss = neg_mll(Xt, yt, v, noise_lb, kind, noise_guess, warp_fn)
    (g,) = torch.autograd.grad(loss, v)
    return loss.detach(), g


def fit_psgld(Xt, yt, vec0, lr=0.01, num_epochs=100, noise_lb=8e-4, kind="matern32", langevin=None, frozen=None, record=False,
              warp_fn=warp):
    """gp.py:96-126 (optimizer='psgld') over the packed vector; `frozen`: index range (begin, end) that is never updated."""
    n = Xt.shape[0]
    vec = vec0.clone()
    st = PSGLDState(torch.zeros_like(vec))
    losses = []
    for ep in range(num_epochs):
        loss, g = neg_mll_autograd(Xt, yt, vec, noise_lb, kind, warp_fn=warp_fn)
        if frozen:
            g[frozen[0]:frozen[1]] = 0.0
        xi = None if langevin is None else langevin[ep].to(vec.dtype)
        new = psgld_step(vec, g, st, lr, 1.0 / n, num_epochs // 10, xi)
        if frozen:
            new[frozen[0]:frozen[1]] = vec[frozen[0]:frozen[1]]
        vec = new
        losses.append(float(loss))
    return (vec, losses) if record else vec


def predict(Xt, yt, vec, Xs_t, noise_lb=8e-4, kind="matern32", warp_fn=warp):
    """Posterior mean / variance in the scaled space (variance floored at 1e-6)."""
    n, d = Xt.shape
    p = unpack(vec, d)
    s, sn2 = softplus(p["raw_os"]), softplus(p["raw_noise"]) + noise_lb
    a, b, ls = exponents(p["raw_a"]), exponents(p["raw_b"]), softplus(p["raw_ls"])
    Z, Zs = warp_fn(Xt, a, b) / ls, warp_fn(Xs_t, a, b) / ls
    L = torch.linalg.cholesky(s * _kernel(Z, Z, kind) + torch.eye(n, dtype=Xt.dtype) * sn2)
    Ks = s * _kernel(Zs, Z, kind)
    alpha = torch.cholesky_solve((yt.reshape(-1, 1) - p["mean"]), L).reshape(-1)
    V = torch.linalg.solve_triangular(L, Ks.T, upper=False)
    return p["mean"] + Ks @ alpha, torch.clamp_min(s - (V * V).sum(0), 1e-6)
