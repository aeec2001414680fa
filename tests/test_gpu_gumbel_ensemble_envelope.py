"""hb_gumbel_fit across its envelope: one step's gradient (the logits' included) per element against the fp64 oracle
(oracle/gumbel_oracle.py), Adam's update bit for bit given the device gradient, the envelope corner, and the on-chip
limit of a minibatch rejected before any launch."""
import copy

import numpy as np
import pytest
import torch

from hebo_b200 import DeepEnsemble, GumbelDeepEnsemble, _lib
from oracle import ensemble_oracle as EO
from oracle import gumbel_oracle as GO
from tests.util import U32, gamma32

pytestmark = pytest.mark.gpu


def _one_step(dc, uniqs, r, O, H, L, n, noise, prior=False, seed=0):
    """One device step (n rows, one minibatch) from GumbelNet's initialisation with random logits, given uniforms."""
    g = torch.Generator().manual_seed(seed)
    Xc = torch.rand(n, dc, generator=g) * 2 - 1
    Xe = torch.stack([torch.randint(0, u, (n,), generator=g) for u in uniqs], 1) if uniqs else None
    y = torch.sin(Xc.sum(1, keepdim=True) if dc else Xe.float().sum(1, keepdim=True)).repeat(1, O)
    torch.manual_seed(seed)
    m = GumbelDeepEnsemble(dc, len(uniqs), O, num_ensembles=1, num_epochs=1, batch_size=n, num_hiddens=H, num_layers=L,
                           output_noise=noise, rand_prior=prior, num_uniqs=uniqs, reduced_dim=r)
    init = m.init_member()
    init[m.P - r * dc:] = torch.randn(r * dc, generator=g)          # logits away from zero
    m.params = init.reshape(1, -1).cuda().contiguous()
    u = torch.rand(m.draws_shape(n), generator=g)
    perm = torch.arange(n, dtype=torch.int32).reshape(1, 1, n)
    m.fit(Xc, Xe, y, perm=perm, draws=u, eval_draws=torch.rand(1, r, dc, generator=g))
    torch.cuda.synchronize()
    return m, init, Xc, Xe, y, u


def _w_bound(net, u, T):
    """(W64 [r, dx], per-element bound on |W32 - W64|).  The chain: lse(theta) and lse(s) each carry |value| u plus the
    sum's gamma_(dx) and a few ulps of expf / logf; g = -log(-log u) carries a few ulps of |g| + 1; s = (L + g) / T adds
    one rounding per operation.  z = s - lse(s) then has error dz, and W = exp(z) relative error dz + 2 ulps."""
    with torch.no_grad():
        th = net.feature_select.logits
        lse = th.logsumexp(-1, keepdim=True)
        uu = torch.as_tensor(u, dtype=torch.float64).clamp(GO.EPS32, 1 - GO.EPS32)
        g = -torch.log(-torch.log(uu))
        s = (th - lse + g) / T
        ls = s.logsumexp(-1, keepdim=True)
        W = torch.exp(s - ls)
        K = gamma32(th.shape[1] + 8)
        dlse = (lse.abs() + th.abs().amax(-1, keepdim=True) + 1) * K
        ds = ((th.abs() + lse.abs() + g.abs() + 2) * K + dlse) / T + s.abs() * K
        dz = 2 * ds.amax(-1, keepdim=True) + (ls.abs() + s.abs().amax(-1, keepdim=True) + 1) * K
        return W, W * (dz + 4 * U32)


def _abs_grads(net, W, xs, xe, seed_abs):
    """Sums of absolute terms: the gradient of sum |seed| mu over a copy of the net with |parameters|, |x| and W as a
    leaf, so every product of the forward and backward enters with its magnitude (an upper bound on each dot product's
    sum of |terms|)."""
    a = copy.deepcopy(net)
    with torch.no_grad():
        for p in a.parameters():
            p.abs_()
    Wl = W.clone().requires_grad_(True)
    a.zero_grad()
    mu, _ = a(xs.abs() @ Wl.t() if net.dx else xs, xe)
    (seed_abs * mu).sum().backward()
    return torch.cat([p.grad.reshape(-1) if p.grad is not None else torch.zeros(p.numel(), dtype=torch.float64)
                      for p in a.parameters()]), Wl.grad, mu.detach()


@pytest.mark.parametrize("dc,uniqs,r,O,H,L,n", [
    (5, [], 3, 1, 16, 1, 12), (6, [3, 4], 1, 2, 16, 2, 12), (4, [5], 4, 1, 8, 1, 12), (0, [3, 5], 1, 1, 8, 1, 12),
    (40, [], 21, 2, 32, 1, 12), (256, [], 129, 8, 256, 3, 32)])      # the last: the corner at its largest minibatch
def test_one_step_w_gradient_and_adam(dc, uniqs, r, O, H, L, n):
    """MSE head: the step's W and gradient (the logits' included) per element against fp64 within the bound of their
    fp32 error chains, and Adam's update bit for bit given the device gradient."""
    T = 0.8 ** 0 + 0.1
    m, init, Xc, Xe, y, u = _one_step(dc, uniqs, r, O, H, L, n, False)
    gdev = m.fit_state()[2][0].cpu().double()
    net = GO.GumbelOracleNet(dc, uniqs, "embedding", L, H, O, False, False, reduced_dim=r).load_raw(init)
    xs, xe, ys = m.trans(Xc, Xe, y)
    xs = xs.double()
    _, g64 = GO.gumbel_step_grad(net, xs if dc else None, xe if uniqs else None, ys.double(), np.arange(n), u[0, 0, 0], T,
                                 m.l1, n)
    W64, dW = (_w_bound(net, u[0, 0, 0], T) if dc else (torch.zeros(r, 0, dtype=torch.float64),) * 2)
    if dc:
        E, P = 1, m.P
        Wdev = m.fit_ws.view(torch.float32)[3 * E * P:].view(r, dc).cpu().double()
        assert ((Wdev - W64).abs() <= dW).all(), float(((Wdev - W64).abs() / dW).max())
    # data gradient: chains of at most N terms over |values| (rows, input width, hidden widths, heads), the MSE seeds
    # -2 (t - mu) / cnt carrying the forward's error, and W's relative error through x_sel
    with torch.no_grad():
        mu64, _ = net.forward_selected(xs if dc else torch.zeros(n, 0, dtype=torch.float64), xe, u[0, 0, 0], T)
    epsW = float((dW / W64.clamp_min(1e-300)).max()) if dc else 0.0
    N = n + dc + net.hidden[0].in_features + L * H + O + 8
    rel = 4 * gamma32(N) + 2 * epsW
    _, _, Mabs = _abs_grads(net, W64, xs, xe, torch.ones_like(mu64))
    seed = 2 * ((ys.double() - mu64).abs() + rel * Mabs) / (n * O)          # MSE seeds with the forward's error
    Gabs, GWabs, _ = _abs_grads(net, W64, xs, xe, seed)
    bound = rel * Gabs + 2 * U32 * m.l1 / (n * O)
    lg = slice(m.P - r * dc, m.P)
    # the logits: dW's bound through the softmax backward (W dW, its row sum, / T) and the normalisation term
    if dc:
        dWb, Wb = rel * GWabs, W64
        A, dA = Wb * GWabs, Wb * dWb + Wb * GWabs * epsW
        S1, dS1 = A.sum(1, keepdim=True), dA.sum(1, keepdim=True) + gamma32(dc) * A.sum(1, keepdim=True)
        dl, ddl = (A + Wb * S1) / T, (dA + Wb * dS1 + epsW * Wb * S1) / T
        ddl = ddl + gamma32(4) * dl
        sm = torch.softmax(net.feature_select.logits.detach(), -1)
        S2, dS2 = dl.sum(1, keepdim=True), ddl.sum(1, keepdim=True) + gamma32(dc) * dl.sum(1, keepdim=True)
        bl = ddl + sm * dS2 + (gamma32(dc + 8) + U32) * sm * S2 + gamma32(3) * (dl + sm * S2)
        bound[lg] = bl.reshape(-1)
    err = (gdev - g64).abs()
    assert (err <= bound + 1e-30).all(), float((err / (bound + 1e-30)).max())
    p1, _, _ = EO.adam_update_f32(init.numpy(), gdev.float().numpy(), np.zeros(m.P, np.float32), np.zeros(m.P, np.float32),
                                  1, m.lr)
    assert np.array_equal(m.params[0].cpu().numpy(), p1)


@pytest.mark.parametrize("dc,uniqs,r,E", [(5, [], 3, 3), (6, [3, 4], 1, 2), (40, [4], 21, 5)])
def test_predict_against_fp64(dc, uniqs, r, E):
    """MSE head: predict mu / sigma2 per element against fp64 over given eval uniforms, within the bound of the chain
    (W's relative error, then dot products of |terms| through the net, the member mean and variance, the un-scaling)."""
    torch.manual_seed(4)
    m = GumbelDeepEnsemble(dc, len(uniqs), 1, num_ensembles=E, num_epochs=5, num_hiddens=16, num_uniqs=uniqs,
                           reduced_dim=r, output_noise=False, batch_size=8)
    g = torch.Generator().manual_seed(5)
    Xc = torch.rand(30, dc, generator=g) * 2 - 1
    Xe = torch.stack([torch.randint(0, q, (30,), generator=g) for q in uniqs], 1) if uniqs else None
    m.fit(Xc, Xe, Xc[:, :1] ** 2)
    Xs = torch.rand(37, dc, generator=g) * 2 - 1
    Xes = torch.stack([torch.randint(0, q, (37,), generator=g) for q in uniqs], 1) if uniqs else None
    u = torch.rand(E, r, dc, generator=g)
    py, ps2 = m.predict(Xs, Xes, draws=u)
    T = m.temperature
    xs = m.xscaler.transform(Xs).double()
    mus, dmus = [], []
    for e in range(E):
        net = GO.GumbelOracleNet(dc, uniqs, "embedding", 1, 16, 1, False, False, reduced_dim=r).load_raw(m.params[e].cpu())
        W, dW = _w_bound(net, u[e], T)
        with torch.no_grad():
            mu, _ = net.forward_selected(xs, Xes, u[e], T)
        _, _, Mabs = _abs_grads(net, W, xs, Xes, torch.ones(37, 1, dtype=torch.float64))
        epsW = float((dW / W.clamp_min(1e-300)).max())
        N = dc + net.hidden[0].in_features + 16 + 8
        mus.append(mu)
        dmus.append((2 * gamma32(N) + 2 * epsW + 4 * U32) * Mabs + 4 * U32 * xs.abs().max() * Mabs)
    mus, dmus = torch.stack(mus), torch.stack(dmus)
    mean, dmean = mus.mean(0), dmus.mean(0) + gamma32(E + 1) * mus.abs().mean(0)
    var = 1e-8 + ((mus - mean) ** 2).mean(0)
    dvar = (2 * (mus - mean).abs() * (dmus + dmean)).mean(0) + gamma32(E + 4) * var
    ym, sd = float(m.yscaler.mean), float(m.yscaler.std)
    b_mu = dmean * sd + gamma32(3) * (mean.abs() * sd + abs(ym))
    b_var = dvar * sd * sd + gamma32(3) * var * sd * sd
    assert ((py.double() - (mean * sd + ym)).abs() <= b_mu).all()
    assert ((ps2.double() - var * sd * sd).abs() <= b_var).all()


# ------------------------------------------------------------------------------------------------ bit for bit
def _fit_case(uniqs, trans, prior, n, batch, E=2, epochs=2, seed=0):
    g = torch.Generator().manual_seed(seed)
    Xe = torch.stack([torch.randint(0, q, (n,), generator=g) for q in uniqs], 1)
    y = torch.sin(Xe.float().sum(1, keepdim=True)).repeat(1, 2)
    y[1, 0] = float("nan")
    torch.manual_seed(seed)
    m = GumbelDeepEnsemble(0, len(uniqs), 2, num_ensembles=E, num_epochs=epochs, batch_size=batch, num_hiddens=16,
                           num_layers=2, output_noise=False, rand_prior=prior, num_uniqs=uniqs, enum_trans=trans)
    perm = torch.stack([torch.stack([torch.randperm(n, generator=g) for _ in range(epochs)]) for _ in range(E)]).int()
    m.params = torch.stack([m.init_member() for _ in range(E)]).cuda().contiguous()
    raw0 = m.params.cpu().numpy().copy()
    return m, Xe, y, perm, raw0


@pytest.mark.parametrize("n", [8, 9, 19])          # bs, bs + 1, 2 bs + 3 with bs = 8: the partial last minibatch
@pytest.mark.parametrize("uniqs,trans,prior", [([4, 7], "embedding", True), ([3, 5], "onehot", False)])
def test_fit_without_numeric_columns_equals_the_restatement_bit_for_bit(n, uniqs, trans, prior):
    bs = 8
    m, Xe, y, perm, raw0 = _fit_case(uniqs, trans, prior, n, bs)
    m.fit(None, Xe, y, perm=perm)
    torch.cuda.synchronize()
    net = GO.GumbelNet32(uniqs, trans, 2, 16, 2, rand_prior=prior)
    xe, ys = m.trans(None, Xe, y)[1:]
    m1, m2, g = (t.cpu().numpy() for t in m.fit_state())
    for e in range(2):
        p, a, b, gg = GO.gumbel_fit32(net, raw0[e], xe.numpy(), ys.numpy(), perm[e].numpy(), m.lr, m.l1, bs)
        for what, dv, rv in (("params", m.params[e].cpu().numpy(), p), ("exp_avg", m1[e], a), ("exp_avg_sq", m2[e], b),
                             ("grad", g[e], gg)):
            assert EO.mismatches(dv, rv) == 0, f"member {e} {what}"
    if prior:           # the prior net's biases do not move, its weights take the L1 term
        for name, (o, shape) in net.slices.items():
            sl = slice(o, o + int(np.prod(shape)))
            if name.startswith("prior_net"):
                assert np.array_equal(m.params.cpu().numpy()[:, sl], raw0[:, sl]) == name.endswith("bias")
    # predict of the same members: BaseNet's restated predict with the prior net evaluated
    ym, sd = m.yscaler.mean.numpy(), m.yscaler.std.numpy()
    py, ps2 = m.predict(None, Xe, seed=0)
    rmu, rvar = EO.predict32(net, m.params.cpu().numpy(), None, xe.numpy(), None, None, ym, sd)
    assert EO.mismatches(py.numpy(), rmu) == 0 and EO.mismatches(ps2.numpy(), rvar) == 0


def test_envelope_corner_runs_to_run_identically():
    """num_cont = 256, r = 129, 3 x 256 hidden, 8 outputs, at the largest admitted minibatch and a partial last one; its
    step values are checked against fp64 in test_one_step_w_gradient_and_adam."""
    dc, r, O, H, L = 256, 129, 8, 256, 3
    m = GumbelDeepEnsemble(dc, 0, O, num_ensembles=2, num_epochs=1, num_hiddens=H, num_layers=L, reduced_dim=r)
    B = max(b for b in range(1, 64) if m.batch_floats(b) <= _lib.HB_DE_MAX_BATCH_FLOATS)
    assert B == 32
    g = torch.Generator().manual_seed(1)
    X, y = torch.rand(B + 3, dc, generator=g), torch.randn(B + 3, O, generator=g)
    out = []
    for _ in range(2):
        torch.manual_seed(0)
        m = GumbelDeepEnsemble(dc, 0, O, num_ensembles=2, num_epochs=1, num_hiddens=H, num_layers=L, reduced_dim=r,
                               batch_size=B)
        m.fit(X, None, y)
        out.append(m.params.clone())
    assert torch.equal(out[0], out[1]) and torch.isfinite(out[0]).all()


def test_one_row_over_the_limit_is_rejected_without_a_launch():
    dc, r, O, H, L = 256, 129, 8, 256, 3
    m = GumbelDeepEnsemble(dc, 0, O, num_ensembles=1, num_epochs=1, num_hiddens=H, num_layers=L, reduced_dim=r)
    B = max(b for b in range(1, 64) if m.batch_floats(b) <= _lib.HB_DE_MAX_BATCH_FLOATS)
    X, y = torch.rand(B + 1, dc), torch.randn(B + 1, O)
    m.batch_size = B + 1
    with pytest.raises(NotImplementedError):
        m.fit(X, None, y)
    assert not m.fitted
    lib = _lib.lib()
    P = int(lib.hb_gumbel_num_params(m._spec, r))
    params = torch.zeros(1, P, device="cuda")
    ws = torch.empty(int(lib.hb_gumbel_fit_workspace_bytes(m._spec, r, 1)), dtype=torch.uint8, device="cuda")
    losses = torch.empty(1, 1, device="cuda")
    xd, yd = X.cuda(), y.cuda()
    torch.cuda.synchronize()
    lib.hb_launch_count(1)
    rc = lib.hb_gumbel_fit(_lib.ptr(xd), None, _lib.ptr(yd), B + 1, m._spec, r, 1, _lib.ptr(params), 5e-3, 1e-3, B + 1, 1,
                           None, None, 0, _lib.ptr(losses), _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
    assert rc == _lib.HB_ERR_INVALID and lib.hb_launch_count(0) == 0
    assert not params.any()
    # the plain deep ensemble takes the same shape: 256 numeric columns, 3 x 256, 8 outputs, B + 1 rows
    de = DeepEnsemble(dc, 0, O, num_ensembles=1, num_epochs=1, num_hiddens=H, num_layers=L, batch_size=B + 1)
    assert de.batch_floats(B + 1) <= _lib.HB_DE_MAX_BATCH_FLOATS
    de.fit(X, None, y)
    assert torch.isfinite(de.params).all()
