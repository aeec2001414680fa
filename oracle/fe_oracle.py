"""FeDeepEnsemble (models/nn/fe_deep_ensemble.py, fe_layers.py) restated on top of the deep ensemble's oracle
(oracle/ensemble_oracle.py), which it imports and leaves as it is.

fp64: ``FeOracleNet`` is FeNet over BaseNet's fp64 restatement: the gate parameter ``gate`` [din] registered last, the
input row multiplied by the gate's mask before the hidden layers, the prior net built but not evaluated.
``fe_step_grad`` is one minibatch of FeDeepEnsemble.fit_one: data loss + l1 sum|w| / (n O) over the parameters whose
name contains 'weight' + mask_reg mask_norm / (n O) when there are numeric columns, differentiated by autograd.

fp32: ``FeNet32`` / ``fe_fit32`` / ``fe_predict32`` restate hb_fe_fit and hb_fe_predict operation by operation for the
stg gate with the MSE head and mask_reg = 0, where every operation is a correctly rounded IEEE one (the mask penalty's
and the concrete layers' expf / logf are not, and are checked against the fp64 path instead).  The draws are given.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from .ensemble_oracle import (F64, Net32, OracleNet, adam_update_f32, backward32, data_loss, dense32, fma32,
                              load_inputs32, minibatch_rule, scatter32)

f32 = np.float32
KINDS = ("stg", "concrete", "hard_concrete")
EPS32 = float(np.finfo(np.float32).eps)


class FeOracleNet(OracleNet):
    """FeNet (fe_deep_ensemble.py:20-35) in fp64: BaseNet's parameters, then the gate [din] last."""

    def __init__(self, num_cont, num_uniqs, enum_trans="embedding", num_layers=1, num_hiddens=128, num_out=1,
                 output_noise=True, rand_prior=False, noise_lb=1e-4, kind="stg"):
        super().__init__(num_cont, num_uniqs, enum_trans, num_layers, num_hiddens, num_out, output_noise, rand_prior,
                         noise_lb)
        din = num_cont + (sum(min(50, 1 + u // 2) if enum_trans == "embedding" else u for u in self.num_uniqs))
        self.kind, self.din = kind, din
        self.feature_select = nn.Module()       # a sub-module registered last, so its parameter comes last, as in FeNet
        self.feature_select.theta = nn.Parameter(torch.zeros(din, dtype=F64))

    @property
    def gate(self):
        return self.feature_select.theta

    def mask(self, r, T):
        """The gate's mask for raw draws r ([B, din] in training, [din] in eval) at temperature T."""
        th = self.gate
        if self.kind == "stg":
            return (T * r + th + 0.5).clamp(0.0, 1.0)
        u = r.clamp(EPS32, 1 - EPS32)
        y = ((th + torch.log(u / (1 - u))) / T).sigmoid()
        return y if self.kind == "concrete" else (y * 1.2 - 0.1).clamp(0.0, 1.0)

    def mask_norm(self, T):
        if self.kind == "stg":
            return (0.5 * (1 + torch.erf((self.gate + 0.5) / T / np.sqrt(2)))).sum()
        return self.gate.sigmoid().sum()

    def forward_gated(self, Xc, Xe, r, T):
        """(mu, sigma2 or None) of FeNet.forward: no prior net."""
        x = self.xtrans(Xc, Xe) * self.mask(r, T)
        h = self.hidden(x)
        return self.mu(h), (self.noise_lb + self.sigma2(h)) if self.output_noise else None


def fe_step_grad(net: FeOracleNet, Xc, Xe, y, rows, r, T, l1: float, mask_reg: float, n: int):
    """(data loss, gradient [P_fe]) of one minibatch of FeDeepEnsemble.fit_one (fe_deep_ensemble.py:60-72) with the
    training draws r [B, din]."""
    net.zero_grad()
    rows = torch.as_tensor(rows).long()
    xc = Xc[rows] if Xc is not None and net.num_cont > 0 else torch.zeros(len(rows), 0, dtype=F64)
    xe = Xe[rows] if Xe is not None and net.num_uniqs else None
    mu, s2 = net.forward_gated(xc, xe, torch.as_tensor(r, dtype=F64), float(T))
    dl = data_loss(net, mu, s2, torch.as_tensor(y, dtype=F64)[rows])
    N = n * net.num_out
    loss = dl + sum(l1 * p.abs().sum() / N for name, p in net.named_parameters() if "weight" in name)
    if net.num_cont > 0:
        loss = loss + mask_reg * net.mask_norm(float(T)) / N
    loss.backward()
    g = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in net.parameters()])
    return float(dl.detach()), g.detach().clone()


# ---------------------------------------------------------------------------------------------------------- fp32
class FeNet32(Net32):
    """One gated member of hb_fe_fit: Net32's layout, then the gate [din] at gate0 = BaseNet's P."""

    def __init__(self, *a, kind="stg", **kw):
        super().__init__(*a, **kw)
        self.kind = kind
        self.gate0 = self.P
        self.slices["feature_select.mu" if kind == "stg" else "feature_select.logits"] = (self.P, (self.din,))
        self.P += self.din
        self.is_weight = np.zeros(self.P, bool)
        for name, (o, shape) in self.slices.items():
            if "weight" in name:
                self.is_weight[o:o + int(np.prod(shape))] = True


def _forward_noprior32(net, prm, xin):
    prior, net.prior = net.prior, False
    try:
        from .ensemble_oracle import forward32
        return forward32(net, prm, xin)
    finally:
        net.prior = prior


def stg_state32(prm, gate0, r, T):
    """(T r + theta) + 0.5, each operation rounded in fp32."""
    return (f32(T) * f32(r) + prm[gate0:]) + f32(0.5)


def fe_step_grad32(net: FeNet32, prm, Xc, Xe, y, rows, n, l1, r, T):
    """One minibatch's total gradient [P_fe] as hb_fe_fit forms it for the stg gate, MSE, mask_reg = 0: the mask after
    the load, de_backward down to the masked input, the gate column sums over the rows in order through the clamp's
    inclusive pass-through, dx mask into the embedding tables, L1 over the weights only."""
    assert net.kind == "stg" and not net.noise
    rows = np.asarray(rows)
    xc = f32(Xc)[rows] if net.dc else None
    xe = np.asarray(Xe)[rows] if net.uniqs else None
    xraw = load_inputs32(net, prm, xc, xe)
    st = stg_state32(prm, net.gate0, r, T)
    mask = np.minimum(np.maximum(st, f32(0)), f32(1))
    xin = xraw * mask
    acts, mu, _ = _forward_noprior32(net, prm, xin)
    t = f32(y)[rows]
    fin = np.isfinite(t)
    cnt = f32(fin.sum())
    with np.errstate(invalid="ignore"):
        gmu = np.where(fin, (f32(-2.0) * (t - mu)) / cnt, f32(0))
    g, dx = backward32(net, prm, xin, acts, gmu, np.zeros_like(gmu), True, 0)
    acc = np.zeros(net.din, f32)
    for p in range(dx.shape[0]):
        acc = acc + np.where((st[p] >= 0) & (st[p] <= 1), dx[p] * xraw[p], f32(0))
    dx = dx * mask
    if net.emb and net.uniqs:
        g.update(scatter32(net, dx[:, net.dc:], xe))
    gd = np.zeros(net.P, f32)
    for name, v in g.items():
        o, _ = net.slices[name]
        gd[o:o + v.size] = v.reshape(-1)
    gd[net.gate0:] = acc
    coef = (f32(1.0) / f32(n * net.O)) * f32(l1)
    sg = np.where(prm > 0, f32(1), np.where(prm < 0, f32(-1), f32(0)))
    return np.where(net.is_weight, gd + coef * sg, gd)


def fe_fit32(net: FeNet32, prm0, Xc, Xe, y, orders, draws, lr, l1, batch, T):
    """One member of hb_fe_fit over orders [epochs, n] and draws [epochs, nb, B, din]: (params, exp_avg, exp_avg_sq,
    last gradient)."""
    n = y.shape[0]
    B, nb = minibatch_rule(n, batch)
    p = f32(prm0).copy()
    m1, m2, g = (np.zeros(net.P, f32) for _ in range(3))
    step = 0
    for ep, order in enumerate(orders):
        for b in range(nb):
            step += 1
            g = fe_step_grad32(net, p, Xc, Xe, y, order[b * B:(b + 1) * B], n, l1, draws[ep, b], T)
            p, m1, m2 = adam_update_f32(p, g, m1, m2, step, lr)
    return p, m1, m2, g


def fe_predict32(net: FeNet32, params, Xs, Xe, x_mul, x_add, y_mean, y_std, draws, T):
    """hb_fe_predict (member = -1) for the stg gate and the MSE head: member e's inputs times its eval mask
    clamp((T r_e + theta_e) + 0.5, 0, 1), the members combined in order.  (mu, var) [B, O]."""
    assert net.kind == "stg" and not net.noise
    E = params.shape[0]
    mus = []
    for e in range(E):
        st = stg_state32(params[e], net.gate0, draws[e], T)
        gm = np.minimum(np.maximum(st, f32(0)), f32(1))
        xin = load_inputs32(net, params[e], Xs, Xe, x_mul, x_add) * gm
        mus.append(_forward_noprior32(net, params[e], xin)[1])
    ne, ys, ym = f32(E), f32(y_std), f32(y_mean)
    mean = np.zeros_like(mus[0])
    for m in mus:
        mean = mean + m
    mean = mean / ne
    v = np.zeros_like(mean)
    for m in mus:
        d = m - mean
        v = fma32(d, d, v)
    v = f32(1e-8) + v / ne
    return mean * ys + ym, v * (ys * ys)


__all__ = ["FeOracleNet", "fe_step_grad", "FeNet32", "fe_step_grad32", "fe_fit32", "fe_predict32", "KINDS", "dense32"]
