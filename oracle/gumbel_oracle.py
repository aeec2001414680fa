"""GumbelDeepEnsemble (models/nn/gumbel_linear.py) restated on top of the deep ensemble's oracle
(oracle/ensemble_oracle.py), which it imports and leaves as it is.

fp64: ``GumbelOracleNet`` is GumbelNet over BaseNet's fp64 restatement: BaseNet over the selected width
(num_cont -> r when num_cont > 0), then ``feature_select.logits`` [r, num_cont] registered last.  ``selection`` builds
W = RelaxedOneHotCategorical(T, logits).rsample() from given uniforms in ExpRelaxedCategorical.rsample's order, and
``gumbel_step_grad`` is one minibatch of GumbelDeepEnsemble.fit_one: data loss + l1 sum|w| / (n O) over the parameters
whose name contains 'weight', differentiated by autograd through W, the softmax and the logits' normalisation.

fp32: ``GumbelNet32`` / ``gumbel_step_grad32`` / ``gumbel_fit32`` restate hb_gumbel_fit operation by operation without
numeric columns and with the MSE head, where every operation is a correctly rounded IEEE one.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from .ensemble_oracle import (F64, Net32, OracleNet, adam_update_f32, backward32, data_loss, forward32, load_inputs32,
                              scatter32)

EPS32 = float(torch.finfo(torch.float32).eps)


class GumbelOracleNet(OracleNet):
    """GumbelNet (gumbel_linear.py:42-61) in fp64."""

    def __init__(self, num_cont, num_uniqs, enum_trans="embedding", num_layers=1, num_hiddens=128, num_out=1,
                 output_noise=True, rand_prior=False, noise_lb=1e-4, reduced_dim=None):
        r = num_cont // 2 + 1 if reduced_dim is None else reduced_dim
        super().__init__(r if num_cont > 0 else 0, num_uniqs, enum_trans, num_layers, num_hiddens, num_out, output_noise,
                         rand_prior, noise_lb)
        self.dx, self.r = num_cont, r
        self.feature_select = nn.Module()       # registered last, so the logits come last, as in GumbelNet
        self.feature_select.logits = nn.Parameter(torch.zeros(r, num_cont, dtype=F64))

    def selection(self, u, T):
        """W [r, num_cont] from uniforms u at temperature T."""
        lg = self.feature_select.logits
        L = lg - lg.logsumexp(-1, keepdim=True)
        g = -torch.log(-torch.log(torch.as_tensor(u, dtype=F64).clamp(EPS32, 1 - EPS32)))
        s = (L + g) / T
        return torch.exp(s - s.logsumexp(-1, keepdim=True))

    def forward_selected(self, Xc, Xe, u, T):
        """(mu, sigma2 or None) of GumbelNet.forward with the selection's uniforms u."""
        if self.dx > 0:
            Xc = Xc.to(F64) @ self.selection(u, T).t()
        return self(Xc, Xe)


def gumbel_step_grad(net: GumbelOracleNet, Xc, Xe, y, rows, u, T, l1: float, n: int):
    """(data loss, gradient [P_gb]) of one minibatch of GumbelDeepEnsemble.fit_one (gumbel_linear.py:83-93) with the
    selection's uniforms u [r, num_cont]."""
    net.zero_grad()
    rows = torch.as_tensor(rows).long()
    xc = Xc[rows] if Xc is not None and net.dx > 0 else torch.zeros(len(rows), 0, dtype=F64)
    xe = Xe[rows] if Xe is not None and net.num_uniqs else None
    mu, s2 = net.forward_selected(xc, xe, u, float(T))
    dl = data_loss(net, mu, s2, torch.as_tensor(y, dtype=F64)[rows])
    loss = dl + sum(l1 * p.abs().sum() / (n * net.num_out) for name, p in net.named_parameters() if "weight" in name)
    loss.backward()
    g = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in net.parameters()])
    return float(dl.detach()), g.detach().clone()


__all__ = ["GumbelOracleNet", "gumbel_step_grad"]


# ---------------------------------------------------------------------------------------------------------- fp32
# hb_gumbel_fit / hb_gumbel_predict restated operation by operation where every operation is a correctly rounded IEEE one:
# no numeric columns (nothing is drawn: the member is a BaseNet over the embedding / one-hot columns) with the MSE head.
# The selection's expf / logf are not correctly rounded and are checked against the fp64 path instead.
f32 = np.float32


class GumbelNet32(Net32):
    """One member of hb_gumbel_fit without numeric columns: Net32's layout, then the empty logits [r, 0]."""

    def __init__(self, num_uniqs, enum_trans="embedding", num_layers=1, num_hiddens=128, num_out=1, rand_prior=False):
        super().__init__(0, num_uniqs, enum_trans, num_layers, num_hiddens, num_out, False, rand_prior)
        self.is_weight = np.zeros(self.P, bool)
        for name, (o, shape) in self.slices.items():
            if "weight" in name:
                self.is_weight[o:o + int(np.prod(shape))] = True


def minibatches(n: int, batch: int):
    """(rows per full step, steps per epoch) without drop_last: B = min(n, batch), ceil(n / B) steps."""
    B = min(n, batch)
    return B, -(-n // B)


def gumbel_step_grad32(net: GumbelNet32, prm, Xe, y, rows, n, l1):
    """One minibatch's total gradient as hb_gumbel_fit forms it: MSE seeds over the finite targets of these rows,
    de_backward (the prior net evaluated, not differentiated), the embedding scatter, L1 over the weights only with the
    prior net's data gradient held at zero."""
    rows = np.asarray(rows)
    xe = np.asarray(Xe)[rows]
    xin = load_inputs32(net, prm, None, xe)
    acts, mu, _ = forward32(net, prm, xin)
    t = f32(y)[rows]
    fin = np.isfinite(t)
    cnt = f32(fin.sum())
    with np.errstate(invalid="ignore"):
        gmu = np.where(fin, (f32(-2.0) * (t - mu)) / cnt, f32(0))
    want_in = net.emb and len(net.uniqs) > 0
    g, dx = backward32(net, prm, xin, acts, gmu, np.zeros_like(gmu), True, 0 if want_in else None)
    if want_in:
        g.update(scatter32(net, dx, xe))
    gd = np.zeros(net.P, f32)
    for name, v in g.items():
        o, _ = net.slices[name]
        gd[o:o + v.size] = v.reshape(-1)
    coef = (f32(1.0) / f32(n * net.O)) * f32(l1)
    sg = np.where(prm > 0, f32(1), np.where(prm < 0, f32(-1), f32(0)))
    return np.where(net.is_weight, gd + coef * sg, gd)


def gumbel_fit32(net: GumbelNet32, prm0, Xe, y, orders, lr: float, l1: float, batch: int):
    """One member of hb_gumbel_fit over orders [epochs, n], the partial last minibatch trained: (params, exp_avg,
    exp_avg_sq, last gradient)."""
    n = y.shape[0]
    B, nb = minibatches(n, batch)
    p = f32(prm0).copy()
    m1, m2, g = (np.zeros(net.P, f32) for _ in range(3))
    step = 0
    for order in orders:
        for b in range(nb):
            step += 1
            g = gumbel_step_grad32(net, p, Xe, y, order[b * B:(b + 1) * B], n, l1)
            p, m1, m2 = adam_update_f32(p, g, m1, m2, step, lr)
    return p, m1, m2, g


__all__ += ["GumbelNet32", "minibatches", "gumbel_step_grad32", "gumbel_fit32"]
