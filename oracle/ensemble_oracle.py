"""fp64 restatement of the deep-ensemble surrogate (HEBO/hebo/models/nn/deep_ensemble.py): BaseNet's forward, the NLL /
MSE data losses, the L1 term, torch's Adam, the ensemble combination, its input gradients (through autograd in fp64),
and the keyed Philox minibatch order of ``hb_de_fit``.

``OracleNet`` has BaseNet's module names and registration order, so its ``named_parameters()`` define the raw layout
independently of hebo_b200.ensemble.param_layout.  Test infrastructure; never imported by hebo_b200/.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn as nn

from oracle import rng_oracle

F64 = torch.float64


class _Emb(nn.Module):
    def __init__(self, num_uniqs):
        super().__init__()
        self.emb = nn.ModuleList([nn.Embedding(u, min(50, 1 + u // 2)) for u in num_uniqs])


class OracleNet(nn.Module):
    """BaseNet (deep_ensemble.py:183-238) in fp64."""

    def __init__(self, num_cont, num_uniqs, enum_trans="embedding", num_layers=1, num_hiddens=128, num_out=1,
                 output_noise=True, rand_prior=False, noise_lb=1e-4):
        super().__init__()
        self.num_cont, self.num_uniqs, self.enum_trans = num_cont, list(num_uniqs), enum_trans
        self.num_out, self.output_noise, self.rand_prior, self.noise_lb = num_out, output_noise, rand_prior, noise_lb
        din = num_cont
        if self.num_uniqs:
            if enum_trans == "embedding":
                self.enum_layer = _Emb(self.num_uniqs)
                din += sum(min(50, 1 + u // 2) for u in self.num_uniqs)
            else:
                din += sum(self.num_uniqs)

        def mlp():
            layers, k = [], din
            for _ in range(num_layers):
                layers += [nn.Linear(k, num_hiddens), nn.ReLU()]
                k = num_hiddens
            return nn.Sequential(*layers)
        self.hidden = mlp()
        self.mu = nn.Linear(num_hiddens, num_out)
        if output_noise:
            self.sigma2 = nn.Sequential(nn.Linear(num_hiddens, num_out), nn.Softplus())
        if rand_prior:
            self.prior_net = mlp()
            self.prior_net.add_module("prior_net_out", nn.Linear(num_hiddens, num_out))
        self.double()

    def load_raw(self, raw):
        raw = torch.as_tensor(raw, dtype=F64).reshape(-1)
        o = 0
        with torch.no_grad():
            for _, p in self.named_parameters():
                p.copy_(raw[o:o + p.numel()].reshape(p.shape))
                o += p.numel()
        assert o == raw.numel()
        return self

    def raw(self) -> torch.Tensor:
        return torch.cat([p.detach().reshape(-1) for p in self.parameters()])

    def xtrans(self, Xc, Xe):
        dt = self.mu.weight.dtype
        parts = [Xc.to(dt)] if self.num_cont > 0 else []
        if self.num_uniqs:
            Xe = torch.as_tensor(Xe).long()
            if self.enum_trans == "embedding":
                parts += [self.enum_layer.emb[i](Xe[:, i]) for i in range(len(self.num_uniqs))]
            else:
                parts += [nn.functional.one_hot(Xe[:, i], u).to(dt) for i, u in enumerate(self.num_uniqs)]
        return torch.cat(parts, 1)

    def forward(self, Xc, Xe):
        """(mu [B, O], sigma2 [B, O] or None)"""
        x = self.xtrans(Xc, Xe)
        prior = 0.0
        if self.rand_prior:
            with torch.no_grad():
                prior = self.prior_net(x).detach()
        h = self.hidden(x)
        mu = self.mu(h) + prior
        return mu, (self.noise_lb + self.sigma2(h)) if self.output_noise else None


def data_loss(net: OracleNet, mu, s2, t):
    mask = torch.isfinite(t)
    if net.output_noise:
        return torch.mean(0.5 * (t[mask] - mu[mask]) ** 2 / s2[mask] + 0.5 * torch.log(s2[mask]))
    return torch.mean((mu[mask] - t[mask]) ** 2)


def step_grad(net: OracleNet, Xc, Xe, y, rows, l1: float, n: int):
    """(data loss, gradient [P]) of one minibatch (deep_ensemble.py:163-171): data loss + l1 sum|p| / (n num_out)."""
    net.zero_grad()
    rows = torch.as_tensor(rows).long()
    mu, s2 = net(Xc[rows] if Xc is not None and net.num_cont > 0 else torch.zeros(len(rows), 0, dtype=F64),
                 Xe[rows] if Xe is not None and net.num_uniqs else None)
    dl = data_loss(net, mu, s2, torch.as_tensor(y, dtype=F64)[rows])
    reg = sum(l1 * p.abs().sum() / (n * net.num_out) for p in net.parameters())
    (dl + reg).backward()
    g = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in net.parameters()])
    return float(dl.detach()), g.detach().clone()


def adam_update(p, g, m, v, step: int, lr: float, b1=0.9, b2=0.999, eps=1e-8):
    """torch.optim.Adam's single-tensor update in fp64 (returns new p, m, v)."""
    m = m + (1 - b1) * (g - m)
    v = v * b2 + (1 - b2) * g * g
    denom = v.sqrt() / math.sqrt(1 - b2 ** step) + eps
    return p - (lr / (1 - b1 ** step)) * m / denom, m, v


def adam_update_f32(p, g, m, v, step: int, lr: float):
    """The fp32 update ``hb_de_fit`` applies, each operation rounded once in IEEE fp32 (torch's single-tensor order:
    lerp of m, v * b2 + (1 - b2) g g, sqrt(v) / sqrt(bc2) + eps, p + (-lr / bc1) m / denom)."""
    f = np.float32
    p, g, m, v = (np.asarray(t, dtype=f) for t in (p, g, m, v))
    m = f(m + f(f(0.1) * f(g - m)))
    v = f(f(v * f(0.999)) + f(f(f(0.001) * g) * g))
    bc1 = 1.0 - 0.9 ** step
    bc2s = math.sqrt(1.0 - 0.999 ** step)
    denom = f(f(np.sqrt(v) / f(bc2s)) + f(1e-8))
    p = f(p + f(f(f(-(lr / bc1)) * m) / denom))
    return p, m, v


def fit(net: OracleNet, Xc, Xe, y, perm, lr: float, l1: float, batch_size: int):
    """fit_one (deep_ensemble.py:151-181) of one member over the given orders perm [epochs, n], Adam in fp64."""
    n = y.shape[0]
    nb, B = (n // batch_size, batch_size) if n > batch_size else (1, n)
    p = net.raw()
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    step, losses = 0, []
    for order in perm:
        el = 0.0
        for b in range(nb):
            step += 1
            dl, g = step_grad(net, Xc, Xe, y, order[b * B:(b + 1) * B], l1, n)
            p, m, v = adam_update(net.raw(), g, m, v, step, lr)
            net.load_raw(p)
            el += dl * B
        losses.append(el / n)
    return losses


def ensemble_predict(nets, Xs, Xe, x_mul, x_add, y_mean, y_std, output_noise=True):
    """DeepEnsemble.predict (deep_ensemble.py:95-106) in fp64 on raw inputs Xs (scaled as x_mul x + x_add)."""
    Xc = Xs.to(F64) * torch.as_tensor(x_mul, dtype=F64) + torch.as_tensor(x_add, dtype=F64) if Xs is not None else None
    if Xc is None:
        Xc = torch.zeros(Xe.shape[0], 0, dtype=F64)
    outs = [net(Xc, Xe) for net in nets]
    mu = torch.stack([o[0] for o in outs])
    py = mu.mean(0)
    if output_noise:
        ps2 = mu.var(0, unbiased=False) + torch.stack([o[1] for o in outs]).mean(0)
    else:
        ps2 = 1e-8 + mu.var(0, unbiased=False)
    ym, ys = torch.as_tensor(y_mean, dtype=F64), torch.as_tensor(y_std, dtype=F64)
    return py * ys + ym, ps2 * ys ** 2


def member_mu(net, Xs, Xe, x_mul, x_add, y_mean, y_std):
    """sample_f's function of one member (deep_ensemble.py:112-115)."""
    Xc = Xs.to(F64) * torch.as_tensor(x_mul, dtype=F64) + torch.as_tensor(x_add, dtype=F64)
    return net(Xc, Xe)[0] * torch.as_tensor(y_std, dtype=F64) + torch.as_tensor(y_mean, dtype=F64)


# ------------------------------------------------------------------------------------------------ minibatch order
def feistel_bits(n: int) -> int:
    h = 1
    while (1 << (2 * h)) < n:
        h += 1
    return h


def perm(seed: int, member: int, epoch: int, n: int) -> np.ndarray:
    """The order of hb_de_fit's epoch `epoch` of member `member`: position i -> row, a 4-round Feistel network on 2h bits
    (round r: word 0 of the Philox block of (half, epoch, member, 0x44450000 + r) under seed) cycle-walked into 0..n-1."""
    h = feistel_bits(n)
    mask = np.uint64((1 << h) - 1)

    def feistel(x):
        L, R = x >> np.uint64(h), x & mask
        for r in range(4):
            w = rng_oracle.block(seed, R, epoch, member, 0x44450000 + r)[0].astype(np.uint64)
            L, R = R, L ^ (w & mask)
        return (L << np.uint64(h)) | R
    x = np.arange(n, dtype=np.uint64)
    x = feistel(x)
    while (x >= n).any():
        bad = x >= n
        x[bad] = feistel(x[bad])
    return x.astype(np.int64)
