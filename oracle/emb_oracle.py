"""CPU oracle for the CATEGORICAL (embedding) variant of the exact-GP path -- groundwork for SURVEY.md section 8(f) row 2.

TEST INFRASTRUCTURE ONLY (same rules as gp_oracle.py): the checker of `hebo_b200.GP(num_enum > 0)` and of
`ard_kernel=False` (tests/test_gpu_emb.py); its closed-form gradient is checked against torch autograd
(tests/test_oracle_emb.py) and its embedding lookup against the reference's real EmbTransform loaded by path
(tests/test_oracle_emb.py::test_embedding_lookup_matches_the_reference_module).  PARITY UNPINNED at the gpytorch boundary,
like the rest of the GP core.  Degenerate layouts are covered: no numeric columns (enum-only model), no categorical
columns, and a single shared numeric lengthscale (`raw_ls.numel() == 1`, ard_kernel=False, gp_util.py:45).

Reference semantics restated:
  * HEBO/hebo/models/layers.py:14-34     EmbTransform: one nn.Embedding(num_uniq_i, emb_size_i) per categorical column,
                                         emb_size_i = min(50, 1 + num_uniq_i // 2), outputs concatenated; weights ~ N(0,1)
  * HEBO/hebo/models/gp/gp_util.py:22-37 DummyFeatureExtractor: x_all = cat([Xc, emb(Xe)])
  * HEBO/hebo/models/gp/gp_util.py:39-59 default_kern: ScaleKernel( Matern32(ARD over the numeric dims) *
                                         Matern32(ONE lengthscale over the embedding dims) ), outputscale init var(y)
  * HEBO/hebo/models/gp/gp.py:86-103     the embedding weights are ordinary parameters of the marginal-likelihood
                                         optimisation (pSGLD over likelihood.raw_noise, emb weights, mean, raw_outputscale,
                                         raw lengthscales -- module registration order)

Model:   K_ij = s * phi(r1_ij) * phi(r2_ij) + sn2 * delta_ij,   phi(r) = (1 + sqrt3 r) exp(-sqrt3 r)
         r1^2 = sum_k ((x_ik - x_jk) / l_k)^2,   r2^2 = |e_i - e_j|^2 / le^2,   e_i = cat_c  E_c[xe_ic]
Closed-form gradient (W = alpha alpha^T - Khat^-1, G1 = W * s * phi(r2) * h(r1), G2 = W * s * phi(r1) * h(r2), h = 3 exp(-sqrt3 r)):
         d data / d l_k   = 1/2 sum_ij G1_ij dz_ijk^2 / l_k
         d data / d le    = 1/2 sum_ij G2_ij r2_ij^2 / le
         d data / d e_i   = - sum_j G2_ij (e_i - e_j) / le^2            (then scattered onto the table rows by category)
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Tuple

import torch

from .gp_oracle import KERNELS, PSGLDState, inv_softplus, kernel_from_sqdist, psgld_step, softplus


def default_emb_sizes(num_uniqs: List[int]) -> List[int]:
    return [min(50, 1 + v // 2) for v in num_uniqs]        # layers.py:19


@dataclass
class EmbHypers:
    """All trainable parameters, in the reference's registration order."""
    raw_noise: torch.Tensor          # []
    tables: List[torch.Tensor]       # [num_uniq_c, emb_size_c] per categorical column
    mean: torch.Tensor               # []
    raw_os: torch.Tensor             # []
    raw_ls: torch.Tensor             # [d] numeric ARD lengthscales, [1] when ard_kernel=False, [0] without numeric columns
    raw_ls_e: torch.Tensor           # []  embedding lengthscale (ignored when there are no tables)
    noise_lb: float = 8e-4

    def pack(self) -> torch.Tensor:
        tail = [self.raw_ls_e.reshape(1)] if self.tables else []
        return torch.cat([self.raw_noise.reshape(1)] + [t.reshape(-1) for t in self.tables] +
                         [self.mean.reshape(1), self.raw_os.reshape(1), self.raw_ls.reshape(-1)] + tail)

    def like(self, vec: torch.Tensor) -> "EmbHypers":
        o = 0
        rn = vec[o]; o += 1
        tabs = []
        for t in self.tables:
            tabs.append(vec[o:o + t.numel()].reshape(t.shape)); o += t.numel()
        mean = vec[o]; o += 1
        ros = vec[o]; o += 1
        d = self.raw_ls.numel()
        rls = vec[o:o + d]; o += d
        if self.tables:
            rle = vec[o]; o += 1
        else:
            rle = self.raw_ls_e
        assert o == vec.numel()
        return EmbHypers(rn, tabs, mean, ros, rls, rle, self.noise_lb)

    @property
    def noise(self):
        return softplus(self.raw_noise) + self.noise_lb

    @property
    def outputscale(self):
        return softplus(self.raw_os)


def init_emb_hypers(Xt: torch.Tensor, Xe: torch.Tensor, yt: torch.Tensor, num_uniqs: List[int], noise_lb: float = 8e-4,
                    seed: int = 0) -> EmbHypers:
    """Reference initial values: N(0,1) embedding weights (nn.Embedding), default lengthscales softplus(0) = ln 2
    (the median-heuristic initialisation of the numeric lengthscales, gp_util.py:47-52, is exercised in gp_oracle),
    outputscale var(y), noise max(1e-2, noise_lb)."""
    dt = Xt.dtype
    g = torch.Generator().manual_seed(seed)
    tables = [torch.randn(u, e, generator=g, dtype=dt) for u, e in zip(num_uniqs, default_emb_sizes(num_uniqs))]
    noise = torch.tensor(max(1e-2, noise_lb), dtype=dt)
    return EmbHypers(inv_softplus(noise - noise_lb), tables, torch.zeros((), dtype=dt),
                     inv_softplus(yt[torch.isfinite(yt)].var().to(dt)), torch.zeros(Xt.shape[1], dtype=dt),
                     torch.zeros((), dtype=dt), noise_lb)


def embed(Xe: torch.Tensor, tables: List[torch.Tensor]) -> torch.Tensor:
    if not tables:
        return torch.zeros(Xe.shape[0], 0, dtype=torch.float64)
    return torch.cat([tables[c][Xe[:, c]] for c in range(len(tables))], 1)      # layers.py:33-34


def _phi_kind(r2: torch.Tensor, kind: str) -> Tuple[torch.Tensor, torch.Tensor]:
    """(k, h) of the numeric-dims kernel: k = kernel value, h with  dk / d r^2 = -h / 2  (SURVEY Appendix A)."""
    return kernel_from_sqdist(r2, kind), KERNELS[kind].h(r2)


def _phi(r2: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(phi, h) of the embedding-dims kernel, always Matern-3/2."""
    return _phi_kind(r2, "matern32")


def neg_mll_emb(Xt: torch.Tensor, Xe: torch.Tensor, yt: torch.Tensor, hp: EmbHypers, noise_guess: float = 0.01,
                kind: str = "matern32") -> torch.Tensor:
    """-ExactMarginalLogLikelihood / n with the Gamma(.5,.5) outputscale and LogNormal noise priors (autograd-able)."""
    n = Xt.shape[0]
    s, sn2, c = hp.outputscale, hp.noise, hp.mean
    Z = Xt / softplus(hp.raw_ls)
    E = embed(Xe, hp.tables).to(Xt.dtype) / softplus(hp.raw_ls_e)
    r1 = ((Z[:, None, :] - Z[None, :, :]) ** 2).sum(-1)
    r2 = ((E[:, None, :] - E[None, :, :]) ** 2).sum(-1)
    K = s * _phi_kind(r1, kind)[0] * _phi(r2)[0] + torch.eye(n, dtype=Xt.dtype) * sn2
    L = torch.linalg.cholesky(K)
    r = (yt.reshape(-1) - c).reshape(-1, 1)
    v = torch.linalg.solve_triangular(L, r, upper=False)
    data = -0.5 * ((v * v).sum() + 2.0 * torch.log(torch.diagonal(L)).sum() + n * math.log(2.0 * math.pi))
    lp_os = 0.5 * math.log(0.5) - math.lgamma(0.5) - 0.5 * torch.log(s) - 0.5 * s
    sig0, mu0 = 0.5, math.log(noise_guess)
    lp_n = -torch.log(sn2 * sig0 * math.sqrt(2.0 * math.pi)) - (torch.log(sn2) - mu0) ** 2 / (2 * sig0 ** 2)
    return -(data + lp_os + lp_n) / n


def neg_mll_emb_autograd(Xt, Xe, yt, hp: EmbHypers, noise_guess=0.01, kind="matern32"):
    vec = hp.pack().detach().clone().requires_grad_(True)
    loss = neg_mll_emb(Xt, Xe, yt, hp.like(vec), noise_guess, kind)
    (g,) = torch.autograd.grad(loss, vec)
    return loss.detach(), g


def neg_mll_emb_closed_form(Xt, Xe, yt, hp: EmbHypers, noise_guess=0.01, kind="matern32") -> Tuple[torch.Tensor, torch.Tensor]:
    """Same loss; gradient by the closed forms in the module docstring (what a CUDA implementation would compute:
    one more pairwise contraction per embedding dimension, then a scatter-add by category)."""
    n, d = Xt.shape
    dt = Xt.dtype
    s, sn2, c = hp.outputscale, hp.noise, hp.mean
    ls, le = softplus(hp.raw_ls), softplus(hp.raw_ls_e)
    Z = Xt / ls
    Eraw = embed(Xe, hp.tables).to(dt)
    E = Eraw / le
    r1 = ((Z[:, None, :] - Z[None, :, :]) ** 2).sum(-1)
    r2 = ((E[:, None, :] - E[None, :, :]) ** 2).sum(-1)
    p1, h1 = _phi_kind(r1, kind)
    p2, h2 = _phi(r2)
    k = p1 * p2
    Khat = s * k + torch.eye(n, dtype=dt) * sn2
    L = torch.linalg.cholesky(Khat)
    Linv = torch.linalg.solve_triangular(L, torch.eye(n, dtype=dt), upper=False)
    Kinv = Linv.T @ Linv
    rvec = yt.reshape(-1) - c
    alpha = Kinv @ rvec
    W = torch.outer(alpha, alpha) - Kinv
    G1 = W * s * p2 * h1
    G2 = W * s * p1 * h2
    dZ2 = (Z[:, None, :] - Z[None, :, :]) ** 2
    g_ls = 0.5 * torch.einsum("ij,ijk->k", G1, dZ2) / ls
    if hp.raw_ls.numel() == 1 and d > 1:                                 # ard_kernel=False: one shared lengthscale
        g_ls = g_ls.sum().reshape(1)
    g_le = 0.5 * (G2 * r2).sum() / le
    # d data / d e_i (unscaled embedding rows): 1/2 sum_ij W_ij dK_ij/de_i, both (i,j) and (j,i) contribute
    dE = E[:, None, :] - E[None, :, :]                                   # scaled differences
    g_E = -torch.einsum("ij,ijq->iq", G2, dE) / le                       # [n, De]
    g_tabs, o = [], 0
    for ci, t in enumerate(hp.tables):
        gt = torch.zeros_like(t)
        gt.index_add_(0, Xe[:, ci], g_E[:, o:o + t.shape[1]])
        g_tabs.append(gt)
        o += t.shape[1]
    g_s = 0.5 * (W * k).sum() + (-0.5 / s - 0.5)
    sig0, mu0 = 0.5, math.log(noise_guess)
    g_n = 0.5 * torch.diagonal(W).sum() + (-1.0 / sn2 - (torch.log(sn2) - mu0) / (sig0 ** 2 * sn2))
    g_c = alpha.sum()
    sg = torch.sigmoid
    tail = [(g_le * sg(hp.raw_ls_e)).reshape(1)] if hp.tables else []
    grad = torch.cat([(g_n * sg(hp.raw_noise)).reshape(1)] + [g.reshape(-1) for g in g_tabs] +
                     [g_c.reshape(1), (g_s * sg(hp.raw_os)).reshape(1), g_ls * sg(hp.raw_ls)] + tail) * (-1.0 / n)
    quad = rvec @ alpha
    logdet = 2.0 * torch.log(torch.diagonal(L)).sum()
    data = -0.5 * (quad + logdet + n * math.log(2.0 * math.pi))
    lp_os = 0.5 * math.log(0.5) - math.lgamma(0.5) - 0.5 * torch.log(s) - 0.5 * s
    lp_n = -torch.log(sn2 * sig0 * math.sqrt(2.0 * math.pi)) - (torch.log(sn2) - mu0) ** 2 / (2 * sig0 ** 2)
    return -(data + lp_os + lp_n) / n, grad


def fit_psgld_emb(Xt, Xe, yt, hp0: EmbHypers, lr=0.01, num_epochs=100, noise_guess=0.01, langevin=None, kind="matern32",
                  record=False):
    """The reference's training loop (gp.py:96-126, optimizer='psgld') over the packed parameter vector: RMSprop +
    Langevin noise after the pretrain phase (sgld.py:49-70).  langevin [num_epochs, P] N(0,1) draws or None."""
    n = Xt.shape[0]
    vec = hp0.pack().clone()
    st = PSGLDState(torch.zeros_like(vec))
    losses = []
    for ep in range(num_epochs):
        loss, g = neg_mll_emb_closed_form(Xt, Xe, yt, hp0.like(vec), noise_guess, kind)
        xi = None if langevin is None else langevin[ep].to(vec.dtype)
        vec = psgld_step(vec, g, st, lr, 1.0 / n, num_epochs // 10, xi)
        losses.append(float(loss))
    hp = hp0.like(vec)
    return (hp, losses) if record else hp


def predict_emb(Xt, Xe, yt, hp: EmbHypers, Xs_t, Xs_e, kind="matern32") -> Tuple[torch.Tensor, torch.Tensor]:
    """Posterior mean / variance in the scaled space (gp.py:137-164 without the un-scaling), variance floored at 1e-6."""
    n = Xt.shape[0]
    s, sn2, c = hp.outputscale, hp.noise, hp.mean
    ls, le = softplus(hp.raw_ls), softplus(hp.raw_ls_e)

    def kfun(A, Ae, B, Be):
        r1 = (((A / ls)[:, None, :] - (B / ls)[None, :, :]) ** 2).sum(-1)
        r2 = (((embed(Ae, hp.tables).to(A.dtype) / le)[:, None, :] - (embed(Be, hp.tables).to(A.dtype) / le)[None, :, :]) ** 2).sum(-1)
        return s * _phi_kind(r1, kind)[0] * _phi(r2)[0]
    L = torch.linalg.cholesky(kfun(Xt, Xe, Xt, Xe) + torch.eye(n, dtype=Xt.dtype) * sn2)
    Ks = kfun(Xs_t, Xs_e, Xt, Xe)
    alpha = torch.cholesky_solve((yt.reshape(-1, 1) - c), L).reshape(-1)
    V = torch.linalg.solve_triangular(L, Ks.T, upper=False)
    return c + Ks @ alpha, torch.clamp_min(s - (V * V).sum(0), 1e-6)
