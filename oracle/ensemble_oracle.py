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


# ------------------------------------------------------------------------------------------------ fp32 restatement
# hebo_b200/csrc/ensemble.cu operation by operation, each rounded as the device rounds it: every sum of products is a
# sequential fmaf chain from 0 in the kernel's index order, everything else a single IEEE fp32 operation.  With
# output_noise=False nothing else enters a fit step, predict or the input gradients, so these functions equal the device
# bit for bit.  Arrays are numpy float32; the row-wise stages take only the rows they are given, so a caller may restate
# chosen rows of a large predict.
fma32 = rng_oracle.fma32
f32 = np.float32


class Net32:
    """One member's DeNet: shapes, and the raw-vector slice of every parameter from OracleNet's registration order."""

    def __init__(self, num_cont, num_uniqs, enum_trans="embedding", num_layers=1, num_hiddens=128, num_out=1,
                 output_noise=False, rand_prior=False, noise_lb=1e-4):
        ref = OracleNet(num_cont, num_uniqs, enum_trans, num_layers, num_hiddens, num_out, output_noise, rand_prior, noise_lb)
        self.dc, self.uniqs, self.emb = num_cont, list(num_uniqs), enum_trans == "embedding"
        self.L, self.H, self.O, self.noise, self.prior = num_layers, num_hiddens, num_out, output_noise, rand_prior
        self.widths = [min(50, 1 + u // 2) if self.emb else u for u in self.uniqs]
        self.din = num_cont + sum(self.widths)
        self.slices, o = {}, 0
        for name, p in ref.named_parameters():
            self.slices[name] = (o, tuple(p.shape))
            o += p.numel()
        self.P = o
        self.prior0 = min([s[0] for k, s in self.slices.items() if k.startswith("prior_net")], default=o)

    def view(self, prm, name):
        o, shape = self.slices[name]
        return prm[o:o + int(np.prod(shape))].reshape(shape)


def load_inputs32(net, prm, Xc, Xe, x_mul=None, x_add=None):
    """de_load_inputs: numeric columns (x_mul x + x_add, two roundings, when x_mul is given), then the embedding rows or
    one-hot codes of the categorical columns.  Xc [B, dc] fp32, Xe [B, ne] int."""
    cols = []
    if net.dc:
        x = f32(Xc)
        if x_mul is not None:
            x = f32(x_mul) * x + f32(x_add)
        cols.append(x)
    for c, u in enumerate(net.uniqs):
        cat = np.asarray(Xe)[:, c]
        if net.emb:
            cols.append(net.view(prm, f"enum_layer.emb.{c}.weight")[cat])
        else:
            cols.append((cat[:, None] == np.arange(u)[None, :]).astype(f32))
    return np.concatenate(cols, 1).astype(f32)


def dense32(x, W, b, relu, add=None):
    """de_dense: acc = 0, fmaf over k ascending, + bias, ReLU (v < 0 -> 0), + add."""
    acc = np.zeros((x.shape[0], W.shape[0]), f32)
    for k in range(W.shape[1]):
        acc = fma32(x[:, k:k + 1], W[None, :, k], acc)
    v = acc + b
    if relu:
        v = np.where(v < 0, f32(0), v)
    return v if add is None else v + add


def forward32(net, prm, xin):
    """de_forward: (hidden activations [L][B, H], mu head [B, O] with the prior net's output added, sigma2 head's
    pre-softplus z [B, O] or None)."""
    V = lambda name: net.view(prm, name)
    pri = None
    if net.prior:
        h = xin
        for l in range(net.L):
            h = dense32(h, V(f"prior_net.{2 * l}.weight"), V(f"prior_net.{2 * l}.bias"), True)
        pri = dense32(h, V("prior_net.prior_net_out.weight"), V("prior_net.prior_net_out.bias"), False)
    acts, h = [], xin
    for l in range(net.L):
        h = dense32(h, V(f"hidden.{2 * l}.weight"), V(f"hidden.{2 * l}.bias"), True)
        acts.append(h)
    mu = dense32(h, V("mu.weight"), V("mu.bias"), False, pri)
    z = dense32(h, V("sigma2.0.weight"), V("sigma2.0.bias"), False) if net.noise else None
    return acts, mu, z


def relu_mask32(a, d):
    """The delta d where the layer's output a is positive, else +0."""
    return np.where(a > 0, d, f32(0))


def fma_over_rows32(d, x):
    """sum_p d[p, :, None] x[p, None, :]: one fmaf chain per element over the rows p ascending."""
    acc = np.zeros((d.shape[1], x.shape[1]), f32)
    for p in range(d.shape[0]):
        acc = fma32(d[p][:, None], x[p][None, :], acc)
    return acc


def sum_rows32(d):
    acc = np.zeros(d.shape[1], f32)
    for p in range(d.shape[0]):
        acc = acc + d[p]
    return acc


def backward32(net, prm, xin, acts, dmu, dz, grads, k0=None):
    """de_backward from head seeds dmu, dz [B, O]: ({name: gradient} when grads, else None; the input delta's columns
    k0: of [B, din] when k0 is not None, else None)."""
    V = lambda name: net.view(prm, name)
    aL, g = acts[-1], {} if grads else None
    if grads:
        g["mu.weight"], g["mu.bias"] = fma_over_rows32(dmu, aL), sum_rows32(dmu)
        if net.noise:
            g["sigma2.0.weight"], g["sigma2.0.bias"] = fma_over_rows32(dz, aL), sum_rows32(dz)
    acc = np.zeros_like(aL)
    for o in range(net.O):
        acc = fma32(dmu[:, o:o + 1], V("mu.weight")[None, o], acc)
        if net.noise:
            acc = fma32(dz[:, o:o + 1], V("sigma2.0.weight")[None, o], acc)
    cur = relu_mask32(aL, acc)
    for l in reversed(range(net.L)):
        inp = xin if l == 0 else acts[l - 1]
        W = V(f"hidden.{2 * l}.weight")
        if grads:
            g[f"hidden.{2 * l}.weight"], g[f"hidden.{2 * l}.bias"] = fma_over_rows32(cur, inp), sum_rows32(cur)
        if l > 0 or k0 is not None:
            kb = 0 if l > 0 else k0
            acc = np.zeros((cur.shape[0], W.shape[1] - kb), f32)
            for j in range(net.H):
                acc = fma32(cur[:, j:j + 1], W[None, j, kb:], acc)
            cur = relu_mask32(inp, acc) if l > 0 else acc
    return g, (cur if k0 is not None else None)


def scatter32(net, dx, Xe):
    """The embedding tables' gradients: the input delta dx [B, din - dc] of each row added into the row of its
    category, plain fp32 adds in minibatch-row order from +0 (categories never drawn keep +0)."""
    out = {}
    for c, (u, w) in enumerate(zip(net.uniqs, net.widths)):
        c0 = sum(net.widths[:c])
        tab = np.zeros((u, w), f32)
        for p in range(dx.shape[0]):
            cat = int(Xe[p, c])
            tab[cat] = tab[cat] + dx[p, c0:c0 + w]
        out[f"enum_layer.emb.{c}.weight"] = tab
    return out


def minibatch_rule(n: int, batch: int):
    """(rows per step, steps per epoch): B = min(n, batch); drop_last = n > batch, so the partial minibatch is dropped."""
    return min(n, batch), (n // batch if n > batch else 1)


def step_grad32(net, prm, Xc, Xe, y, rows, n, l1):
    """One minibatch's gradient as hb_de_fit forms it, output_noise=False: MSE seeds -2 (t - mu) / cnt over the finite
    targets, de_backward, the embedding scatter, plus the L1 term (1 / (float)(n O)) l1 sign(p).  The prior net's
    parameters get the L1 term only.  Returns the total gradient [P]."""
    assert not net.noise, "the fp32 restatement covers output_noise=False (the NLL path goes through expf / log1pf / logf)"
    rows = np.asarray(rows)
    xc = f32(Xc)[rows] if net.dc else None
    xe = np.asarray(Xe)[rows] if net.uniqs else None
    xin = load_inputs32(net, prm, xc, xe)
    acts, mu, _ = forward32(net, prm, xin)
    t = f32(y)[rows]
    fin = np.isfinite(t)
    cnt = f32(fin.sum())
    with np.errstate(invalid="ignore"):
        gmu = np.where(fin, (f32(-2.0) * (t - mu)) / cnt, f32(0))
    want_in = net.emb and len(net.uniqs) > 0
    g, dx = backward32(net, prm, xin, acts, gmu, np.zeros_like(gmu), True, net.dc if want_in else None)
    if want_in:
        g.update(scatter32(net, dx, xe))
    gd = np.zeros(net.P, f32)
    for name, v in g.items():
        o, shape = net.slices[name]
        gd[o:o + v.size] = v.reshape(-1)
    coef = (f32(1.0) / f32(n * net.O)) * f32(l1)
    sg = np.where(prm > 0, f32(1), np.where(prm < 0, f32(-1), f32(0)))
    return gd + coef * sg


def fit32(net, prm0, Xc, Xe, y, orders, lr: float, l1: float, batch: int):
    """One member of hb_de_fit over the given orders [epochs, n]: (params, exp_avg, exp_avg_sq, last gradient)."""
    n = y.shape[0]
    B, nb = minibatch_rule(n, batch)
    p = f32(prm0).copy()
    m1, m2, g = (np.zeros(net.P, f32) for _ in range(3))
    step = 0
    for order in orders:
        for b in range(nb):
            step += 1
            g = step_grad32(net, p, Xc, Xe, y, order[b * B:(b + 1) * B], n, l1)
            p, m1, m2 = adam_update_f32(p, g, m1, m2, step, lr)
    return p, m1, m2, g


def predict32(net, params, Xs, Xe, x_mul, x_add, y_mean, y_std, member=-1, grad=False):
    """de_predict_kernel<grad> on the given rows: (mu, var) [B, O] un-scaled, and with grad (dmu, dvar) [B, O, dc].
    params [E, P]; member >= 0 restates that member alone (var 0).  The members combine in the order of params."""
    E = params.shape[0]
    members = [member] if member >= 0 else list(range(E))
    ne = f32(len(members))
    ys, ym = f32(y_std), f32(y_mean)
    state = []
    for e in members:
        xin = load_inputs32(net, params[e], Xs, Xe, x_mul, x_add)
        state.append((params[e], xin) + forward32(net, params[e], xin))
    mus = [s[3] for s in state]
    if member >= 0:
        mean, v = mus[0], np.zeros_like(mus[0])
    else:
        mean = np.zeros_like(mus[0])
        for m in mus:
            mean = mean + m
        mean = mean / ne
        v = np.zeros_like(mean)
        for m in mus:
            d = m - mean
            v = fma32(d, d, v)
        v = f32(1e-8) + v / ne
    out = (mean * ys + ym, v * (ys * ys))
    if not grad:
        return out
    B, O, dc = mean.shape[0], net.O, net.dc
    dmu, dvar = np.zeros((B, O, dc), f32), np.zeros((B, O, dc), f32)
    invE = f32(1.0) / ne
    for prm, xin, acts, mu_e, _ in state:
        for o in range(O):
            for ps, dst in ((0, dmu), (1, dvar)):
                seed = np.zeros((B, O), f32)
                seed[:, o] = invE if ps == 0 else (f32(2.0) * invE) * (mu_e[:, o] - mean[:, o])
                _, dx = backward32(net, prm, xin, acts, seed, np.zeros_like(seed), False, 0)
                sc = ys[o] if ps == 0 else ys[o] * ys[o]
                dst[:, o, :] = dst[:, o, :] + (dx[:, :dc] * f32(x_mul)) * sc
    return out + (dmu, dvar)


def mismatches(got, want) -> int:
    """Elements whose bits differ (NaN equals NaN only with the same bits)."""
    a = np.ascontiguousarray(np.asarray(got, dtype=np.float32)).view(np.uint32)
    b = np.ascontiguousarray(np.asarray(want, dtype=np.float32)).view(np.uint32)
    assert a.shape == b.shape, (a.shape, b.shape)
    return int((a != b).sum())
