"""Matern-1/2 (gpytorch MaternKernel(nu=0.5), k = e^-r) for the fp64 oracle.  TEST INFRASTRUCTURE ONLY.

oracle/ restates Matern-3/2, Matern-5/2 and RBF.  This module adds k = e^-r and its closed-form MLL gradient, and puts
them behind the oracle's own entry points -- `install(monkeypatch)` for one test, `installed()` for a block:
    gp_oracle.kernel_from_sqdist, gp_oracle.neg_mll_closed_form, emb_oracle.kernel_from_sqdist, emb_oracle._phi_kind,
    warp_oracle.kernel_from_sqdist
take kind = 'matern12' and are the oracle's own functions for every other kind.  Everything built on them by name --
neg_mll and its autograd, fit_psgld, make_fitted / refactor / predict, the embedding and warp oracles, and the fp64
helpers of the test modules -- then evaluates Matern-1/2.

Radial factor (dk/dl_k = h dz_k^2 / l_k, SURVEY Appendix A): h = e^-r / r, singular at r = 0.  gpytorch evaluates
r = sqrt(clamp_min(r^2, 1e-30)), and clamp_min passes no gradient below its bound, so h = 0 for r^2 < 1e-30: a pair of
equal rows contributes nothing to any gradient, as autograd through the clamp gives."""
from __future__ import annotations

import math
from contextlib import contextmanager

import torch

from oracle import emb_oracle as E
from oracle import gp_oracle as O
from oracle import warp_oracle as W

KIND = "matern12"
ID = 4                                   # HB_KERN_MATERN12

_kernel_from_sqdist = O.kernel_from_sqdist
_neg_mll_closed_form = O.neg_mll_closed_form
_phi_kind_emb = E._phi_kind


def matern12_h(r2: torch.Tensor) -> torch.Tensor:
    r = torch.sqrt(torch.clamp_min(r2, 1e-30))
    return torch.where(r2 < 1e-30, torch.zeros_like(r2), torch.exp(-r) / r)


def kernel_from_sqdist(r2: torch.Tensor, kind: str) -> torch.Tensor:
    if kind == KIND:
        return torch.exp(-torch.sqrt(torch.clamp_min(r2, 1e-30)))
    return _kernel_from_sqdist(r2, kind)


def _phi_kind(r2: torch.Tensor, kind: str):
    """emb_oracle._phi_kind: (k, h) of the numeric-dims kernel."""
    if kind == KIND:
        return kernel_from_sqdist(r2, kind), matern12_h(r2)
    return _phi_kind_emb(r2, kind)


def neg_mll_closed_form(Xt, yt, hp, kind="matern32", noise_guess=0.01, noise_diag=None, block: int = 128):
    """gp_oracle.neg_mll_closed_form: the loss and the closed-form gradient of SURVEY Appendix A, here with Matern-1/2's h."""
    if kind != KIND:
        return _neg_mll_closed_form(Xt, yt, hp, kind, noise_guess, noise_diag, block)
    n, d = Xt.shape
    dt = Xt.dtype
    s, sn2, ls, c = hp.outputscale, hp.noise, hp.lengthscale, hp.mean
    Z = Xt / ls
    r2 = torch.empty(n, n, dtype=dt)
    for i0 in range(0, n, block):
        r2[i0:i0 + block] = O.scaled_sqdist(Z[i0:i0 + block], Z)
    k = kernel_from_sqdist(r2, kind)
    Khat = s * k + torch.eye(n, dtype=dt) * sn2
    if noise_diag is not None:
        Khat = Khat + torch.diag(noise_diag)
    L = torch.linalg.cholesky(Khat)
    rvec = yt.reshape(-1) - c
    Linv = torch.linalg.solve_triangular(L, torch.eye(n, dtype=dt), upper=False)
    Kinv = Linv.T @ Linv
    alpha = Kinv @ rvec
    quad = rvec @ alpha
    logdet = 2.0 * torch.log(torch.diagonal(L)).sum()
    W_ = torch.outer(alpha, alpha) - Kinv
    G = W_ * matern12_h(r2) * s
    g_ls = torch.zeros(d, dtype=dt)
    for i0 in range(0, n, block):
        dZ2 = (Z[i0:i0 + block, None, :] - Z[None, :, :]) ** 2
        g_ls = g_ls + torch.einsum("ij,ijk->k", G[i0:i0 + block], dZ2)
    g_ls = 0.5 * g_ls / ls
    sig0, mu0 = 0.5, math.log(noise_guess)
    g_s = 0.5 * (W_ * k).sum() + (-0.5 / s - 0.5)
    g_n = 0.5 * torch.diagonal(W_).sum() + (-1.0 / sn2 - (torch.log(sn2) - mu0) / (sig0 ** 2 * sn2))
    sg = torch.sigmoid
    grad = torch.cat([(g_n * sg(hp.raw_noise)).reshape(1), alpha.sum().reshape(1),
                      (g_s * sg(hp.raw_os)).reshape(1), g_ls * sg(hp.raw_ls)]) * (-1.0 / n)
    data = -0.5 * (quad + logdet + n * math.log(2.0 * math.pi))
    lp_os = 0.5 * math.log(0.5) - math.lgamma(0.5) - 0.5 * torch.log(s) - 0.5 * s
    lp_n = -torch.log(sn2 * sig0 * math.sqrt(2.0 * math.pi)) - (torch.log(sn2) - mu0) ** 2 / (2 * sig0 ** 2)
    loss = -(data + lp_os + lp_n) / n
    return loss, grad, dict(K=Khat, L=L, Linv=Linv, Kinv=Kinv, alpha=alpha, quad=quad, logdet=logdet)


PATCHES = ((O, "kernel_from_sqdist", kernel_from_sqdist), (O, "neg_mll_closed_form", neg_mll_closed_form),
           (E, "kernel_from_sqdist", kernel_from_sqdist), (E, "_phi_kind", _phi_kind),
           (W, "kernel_from_sqdist", kernel_from_sqdist))


def install(monkeypatch) -> None:
    for mod, name, fn in PATCHES:
        monkeypatch.setattr(mod, name, fn)


@contextmanager
def installed():
    saved = [getattr(mod, name) for mod, name, _ in PATCHES]
    try:
        for mod, name, fn in PATCHES:
            setattr(mod, name, fn)
        yield
    finally:
        for (mod, name, _), fn in zip(PATCHES, saved):
            setattr(mod, name, fn)
