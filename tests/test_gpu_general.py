"""GeneralAcq / GeneralBO on the device: hb_general_acq_epilogue, hb_nsga2_survive_k, hb_ga_survive_cv, hb_pareto_front_k and
the optimiser contracts of the reference (HEBO/test/test_optimizer.py, test_constrained_multi_objective.py)."""
import os

import numpy as np
import pandas as pd
import pytest
import torch

from hebo_b200 import _lib
from hebo_b200.acq import GeneralAcq, _general_epilogue
from hebo_b200.evolution import DeviceNSGA2, ga_survive_host, survive_host
from hebo_b200.general import GeneralBO, hypervolume
from hebo_b200.pareto import pareto_front
from hebo_b200.space import DesignSpace

pytestmark = pytest.mark.gpu
INF = float("inf")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ref_general_acq.npz")
dev = torch.device("cuda")
t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)


# ------------------------------------------------------------------ survival inputs and references
def case(P, D, k, seed, cons):
    """Ties, duplicate children (of population rows, of earlier children, within 1e-16), NaN / +-inf objectives and a
    constraint with NaN / inf and about half the rows feasible."""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2, 2, (P, D)).astype(np.float32)
    C = rng.uniform(-2, 2, (P, D)).astype(np.float32)
    X[:, D - 1], C[:, D - 1] = np.rint(X[:, D - 1]), np.rint(C[:, D - 1])
    allx = np.concatenate([X, C], 0)
    for i in np.flatnonzero(rng.random(P) < 0.15):
        j = rng.integers(0, P + i)
        C[i] = allx[j] if j < P else C[j - P]
    C[rng.random(P) < 0.03] += np.float32(1e-17)
    F = np.round(rng.normal(size=(P, k)), 1).astype(np.float32)
    FC = np.round(rng.normal(size=(P, k)), 1).astype(np.float32)
    F[:, -1] = np.round(-0.7 * F[:, 0] + 0.1 * rng.normal(size=P), 2)             # a trade-off: several large fronts
    FC[:, -1] = np.round(-0.7 * FC[:, 0] + 0.1 * rng.normal(size=P), 2)
    for a in (F, FC):
        for v in (np.nan, np.inf, -np.inf):
            a[rng.random(a.shape) < 0.01] = v
    G = GC = None
    if cons:
        G = np.round(rng.normal(size=P) - 0.1, 1).astype(np.float32)
        GC = np.round(rng.normal(size=P) - 0.1, 1).astype(np.float32)
        G[rng.random(P) < 0.02], GC[rng.random(P) < 0.02] = np.nan, np.inf
    return X, F, C, FC, G, GC


def _dominators(fa, fb):
    out = torch.zeros(fb.shape[0], dtype=torch.int64, device=fb.device)
    for b0 in range(0, fb.shape[0], 1024):
        me = fb[b0:b0 + 1024]
        acc = torch.zeros(me.shape[0], dtype=torch.int64, device=fb.device)
        for a0 in range(0, fa.shape[0], 4096):
            o = fa[a0:a0 + 4096]
            acc += ((o[None] <= me[:, None]).all(-1) & (o[None] < me[:, None]).any(-1)).sum(1)
        out[b0:b0 + 1024] = acc
    return out


def survive_torch(X, F, C, FC, G=None, GC=None):
    """The rules of survive_host on the device (for populations where the numpy dominance matrix is too large)."""
    P, D = X.shape
    N = 2 * P
    Xa = torch.cat([X, C], 0)
    f = torch.cat([F, FC], 0).clone()
    f = torch.where(torch.isfinite(f), f, torch.full_like(f, INF))
    g = torch.zeros(N, device=dev) if G is None else torch.cat([G, GC]).clone()
    g = torch.where(torch.isfinite(g), g, torch.full_like(g, INF))
    idx = torch.arange(N, device=dev)
    for c0 in range(P, N, 64):
        c1 = min(N, c0 + 64)
        eq = ((Xa[None, :c1] - Xa[c0:c1, None]).abs() <= 1e-16).all(-1) & (idx[None, :c1] < idx[c0:c1, None])
        dup = eq.any(1)
        f[c0:c1][dup] = INF
        if G is not None:
            g[c0:c1][dup] = INF
    feas = g <= 0
    nf = int(feas.sum())
    keep = torch.zeros(N, dtype=torch.bool, device=dev)
    if nf < P:
        keep |= feas
        inf_rows = torch.nonzero(~feas).reshape(-1)
        keep[inf_rows[torch.sort(g[inf_rows], stable=True).indices[:P - nf]]] = True
        return torch.nonzero(keep).reshape(-1), f, g
    rows = torch.nonzero(feas).reshape(-1)
    fr = f[rows]
    ndom = _dominators(fr, fr)
    rank = torch.full((rows.numel(),), -1, dtype=torch.int64, device=dev)
    cum, r = 0, 0
    while True:
        front = torch.nonzero((rank < 0) & (ndom == 0)).reshape(-1)
        rank[front] = r
        if cum + front.numel() >= P:
            break
        cum += front.numel()
        rest = torch.nonzero(rank < 0).reshape(-1)
        ndom[rest] -= _dominators(fr[front], fr[rest])
        r += 1
    keep[rows[(rank >= 0) & (rank < r)]] = True
    members = torch.nonzero(rank == r).reshape(-1)
    m = members.numel()
    fm = fr[members]
    crowd = torch.zeros(m, device=dev)
    ar = torch.arange(m, device=dev)
    for k in range(fm.shape[1]):
        v = fm[:, k]
        order = torch.sort(v, stable=True).indices
        pos = torch.empty_like(order)
        pos[order] = ar
        fmin, fmax = v[order[0]], v[order[-1]]
        ends = (pos == 0) | (pos == m - 1)
        if bool(fmax > fmin) and bool(torch.isfinite(fmax - fmin)):
            crowd = torch.where(ends, crowd, crowd + (v[order[(pos + 1).clamp(max=m - 1)]] - v[order[(pos - 1).clamp(min=0)]]) / (fmax - fmin))
        crowd = torch.where(ends, torch.full_like(crowd, INF), crowd)
    keep[rows[members[torch.sort(crowd, descending=True, stable=True).indices[:P - cum]]]] = True
    return torch.nonzero(keep).reshape(-1), f, g


def run_survive_k(X, F, C, FC, G, GC, d, k, entry="k"):
    lib = _lib.lib()
    P, D = X.shape
    Xn, Fn = torch.full((P, D), -7.0, device=dev), torch.full((P, k), -7.0, device=dev)
    Gn = None if G is None else torch.full((P,), -7.0, device=dev)
    Xcn, Xen = torch.full((P, d), -7.0, device=dev), torch.full((P, D - d), -7, dtype=torch.int32, device=dev)
    pc = lambda x: _lib.ptr(x) if x.numel() else None
    ws_bytes = int(lib.hb_nsga2_workspace_bytes_k(P, D, k))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    p = _lib.ptr
    if entry == "k":
        st = lib.hb_nsga2_survive_k(p(X), p(F), p(G), p(C), p(FC), p(GC), P, D, d, k, p(Xn), p(Fn), p(Gn), pc(Xcn), pc(Xen), p(ws),
                                    ws_bytes, _lib.stream_ptr())
    elif G is None:
        st = lib.hb_nsga2_survive_ex(p(X), p(F), p(C), p(FC), P, D, d, p(Xn), p(Fn), pc(Xcn), pc(Xen), p(ws), ws_bytes,
                                     _lib.stream_ptr())
    else:
        st = lib.hb_nsga2_survive_cv(p(X), p(F), p(G), p(C), p(FC), p(GC), P, D, d, p(Xn), p(Fn), p(Gn), pc(Xcn), pc(Xen), p(ws),
                                     ws_bytes, _lib.stream_ptr())
    _lib.check(st, "survive")
    torch.cuda.synchronize()
    return Xn, Fn, Gn, Xcn, Xen


@pytest.mark.parametrize("cons", [False, True])
@pytest.mark.parametrize("k", [2, 3, 4, 8])
@pytest.mark.parametrize("P", [1, 2, 100, 256, 257, 4096, 16384])
def test_survive_k_equals_the_restatement(P, k, cons):
    D, d = 5, 4
    X, F, C, FC, G, GC = case(P, D, k, 1000 * P + 10 * k + cons, cons)
    out = run_survive_k(*[None if a is None else t(a) for a in (X, F, C, FC, G, GC)], d, k)
    if P <= 257:
        sel, f, g = survive_host(X, F, C, FC, G, GC)
        sel, f, g = t(sel), t(f), t(g)
    else:
        sel, f, g = survive_torch(*[None if a is None else t(a) for a in (X, F, C, FC, G, GC)])
    Xa = torch.cat([t(X), t(C)], 0)
    Xn, Fn, Gn, Xcn, Xen = out
    assert torch.equal(Xn, Xa[sel])
    assert torch.equal(Fn, f[sel])
    assert torch.equal(Xcn, Xa[sel][:, :d]) and torch.equal(Xen, Xa[sel][:, d:].round().to(torch.int32))
    if cons:
        assert torch.equal(Gn, g[sel])


@pytest.mark.parametrize("cons", [False, True])
@pytest.mark.parametrize("P", [100, 257, 4096])
def test_k3_instance_gives_the_bytes_of_the_three_objective_entries(P, cons):
    X, F, C, FC, G, GC = [None if a is None else t(a) for a in case(P, 5, 3, P + 7, cons)]
    a = run_survive_k(X, F, C, FC, G, GC, 4, 3, "k")
    b = run_survive_k(X, F, C, FC, G, GC, 4, 3, "old")
    for u, v in zip(a, b):
        assert (u is None and v is None) or torch.equal(u, v)


def test_host_and_device_restatements_agree():
    X, F, C, FC, G, GC = case(257, 5, 4, 3, True)
    sel, f, g = survive_host(X, F, C, FC, G, GC)
    sel2, f2, g2 = survive_torch(*[t(a) for a in (X, F, C, FC, G, GC)])
    assert torch.equal(t(sel), sel2) and torch.equal(t(f), f2) and torch.equal(t(g), g2)


def run_ga(X, F, C, FC, G, GC, d):
    lib = _lib.lib()
    P, D = X.shape
    Xn, Fn, Gn = torch.full((P, D), -7.0, device=dev), torch.full((P,), -7.0, device=dev), torch.full((P,), -7.0, device=dev)
    Xcn, Xen = torch.full((P, d), -7.0, device=dev), torch.full((P, D - d), -7, dtype=torch.int32, device=dev)
    ws_bytes = int(lib.hb_nsga2_workspace_bytes(P, D))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    p = _lib.ptr
    if G is None:
        st = lib.hb_ga_survive(p(X), p(F), p(C), p(FC), P, D, d, p(Xn), p(Fn), p(Xcn), p(Xen), p(ws), ws_bytes, _lib.stream_ptr())
        Gn = None
    else:
        st = lib.hb_ga_survive_cv(p(X), p(F), p(G), p(C), p(FC), p(GC), P, D, d, p(Xn), p(Fn), p(Gn), p(Xcn), p(Xen), p(ws), ws_bytes,
                                  _lib.stream_ptr())
    _lib.check(st, "ga_survive")
    torch.cuda.synchronize()
    return Xn, Fn, Gn, Xcn, Xen


@pytest.mark.parametrize("P", [1, 2, 100, 256, 257, 4096, 16384])
def test_ga_survive_cv_equals_the_restatement(P):
    X, F, C, FC, G, GC = case(P, 5, 1, P + 11, True)
    F, FC = F[:, 0].copy(), FC[:, 0].copy()
    G[::7] = -G[::7]                                                    # negative constraints count as cv = 0
    Xn, Fn, Gn, Xcn, Xen = run_ga(*[t(a) for a in (X, F, C, FC, G, GC)], 4)
    sel, f, g = ga_survive_host(X, F, C, FC, G, GC)
    Xa = np.concatenate([X, C], 0)
    assert np.array_equal(Xn.cpu().numpy(), Xa[sel]) and np.array_equal(Fn.cpu().numpy(), f[sel])
    assert np.array_equal(Gn.cpu().numpy(), g[sel])


@pytest.mark.parametrize("P", [100, 4096])
def test_ga_survive_cv_with_zero_constraint_gives_the_unconstrained_bytes(P):
    X, F, C, FC, _, _ = case(P, 5, 1, P + 5, False)
    F, FC = np.nan_to_num(F[:, 0], posinf=3.0, neginf=-3.0, nan=2.0), np.nan_to_num(FC[:, 0], posinf=3.0, neginf=-3.0, nan=2.0)
    z = np.zeros(P, np.float32)
    a = run_ga(*[t(v) for v in (X, F, C, FC, z, z)], 4)
    b = run_ga(*[t(v) for v in (X, F, C, FC)], None, None, 4)
    for i in (0, 1, 3, 4):
        assert torch.equal(a[i], b[i])


@pytest.mark.parametrize("k", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("m", [1, 300, 4096, 20000])
def test_pareto_front_k_equals_the_dominance_oracle(m, k):
    rng = np.random.default_rng(m + k)
    F = np.round(rng.normal(size=(m, k)), 1).astype(np.float32)
    F[rng.random(m) < 0.01, 0] = np.nan
    idx = pareto_front(t(F)).cpu().numpy()
    Fg = t(F)
    dom = _dominators(Fg, Fg).cpu().numpy()
    oracle = np.flatnonzero((dom == 0) & ~np.isnan(F).any(1))
    assert np.array_equal(idx, oracle)
    if k == 3:
        lib = _lib.lib()
        ws = torch.empty(int(lib.hb_pareto_workspace_bytes(m)), dtype=torch.uint8, device=dev)
        i3, c3 = torch.empty(m, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
        _lib.check(lib.hb_pareto_front3(_lib.ptr(Fg), m, _lib.ptr(i3), _lib.ptr(c3), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "f3")
        assert np.array_equal(i3[:int(c3)].cpu().numpy(), idx)


# ------------------------------------------------------------------ the epilogue
def fp32_expr(mu, var, no, noise, xi, kappa, c_kappa):
    """The reference's torch expression in IEEE fp32 (numpy: correctly rounded sqrt, no contraction)."""
    f = np.float32
    ps = np.sqrt(var.astype(f))
    ps = np.where(ps < f(np.finfo(f).eps), f(np.finfo(f).eps), ps)
    py = mu.astype(f)
    if noise is not None:
        py = (py + (noise.astype(f)[None, :] * xi.astype(f)).astype(f)).astype(f)
    out = np.empty_like(py)
    out[:, :no] = py[:, :no] - (f(kappa) * ps[:, :no]).astype(f)
    out[:, no:] = py[:, no:] - (f(c_kappa) * ps[:, no:]).astype(f)
    return out


def test_epilogue_and_eval_reproduce_the_reference():
    z = np.load(GOLDEN)
    for ci in range(int(z["n_cases"])):
        p = f"c{ci}_"
        m, no, nc, use_noise, seed = [int(v) for v in z[p + "meta"]]
        kappa, c_kappa = [float(v) for v in z[p + "kappa"]]
        mu, var, noise, xi, ref = z[p + "mu"], z[p + "var"], z[p + "noise"], z[p + "xi"], z[p + "out"]
        noise_sd = z[p + "noise_sd"]                                             # model.noise.sqrt() as the reference computed it
        want = fp32_expr(mu, var, no, noise_sd if use_noise else None, xi, kappa, c_kappa)
        Fo, Fc, cv = _general_epilogue(t(mu.T), t(var.T), no, nc, kappa, c_kappa, t(noise_sd) if use_noise else None,
                                       t(xi) if use_noise else None, want_fc=True, want_cv=True)
        got = torch.cat([Fo, Fc], 1).cpu().numpy()
        assert np.array_equal(got, want), ci                                    # bit for bit with IEEE fp32
        assert np.array_equal(cv.cpu().numpy(), np.maximum(want[:, no:], 0).sum(1, dtype=np.float32)) if nc else True
        # the reference's CPU eval differs only through torch's CPU sqrt (one ulp of ps in some rows), scaled by kappa
        ps = np.maximum(np.sqrt(var), np.finfo(np.float32).eps)
        kap = np.array([kappa] * no + [c_kappa] * nc, np.float32)
        assert (np.abs(got - ref) <= 2 * (kap * np.spacing(ps) + np.spacing(np.abs(got)))).all(), ci

        # eval: the draws of torch's CPU generator in the reference's order, then the same epilogue
        stub = type("Stub", (), dict(num_out=no + nc, noise=torch.from_numpy(noise),
                                     predict=staticmethod(lambda x, xe, mu=mu, var=var: (torch.from_numpy(mu), torch.from_numpy(var)))))()
        torch.manual_seed(seed)
        v = GeneralAcq(stub, no, nc, kappa=kappa, c_kappa=c_kappa, use_noise=bool(use_noise))(torch.zeros(m, 1), None)
        sd = torch.from_numpy(noise).sqrt().numpy()                              # this CPU's sqrt, as eval takes it
        Fo, Fc, _ = _general_epilogue(t(mu.T), t(var.T), no, nc, kappa, c_kappa, t(sd) if use_noise else None,
                                      t(xi) if use_noise else None, want_fc=True)
        assert v.device.type == "cpu" and np.array_equal(v.numpy(), torch.cat([Fo, Fc], 1).cpu().numpy())


def test_dummy_contract():
    class Dummy:                                        # HEBO/test/test_constrained_multi_objective.py
        num_obj, num_constr, num_out = 3, 4, 7
        noise = torch.zeros(7)
        predict = staticmethod(lambda x, _: (torch.zeros(x.shape[0], 7), torch.ones(x.shape[0], 7)))
    acq = GeneralAcq(Dummy(), 3, 4, kappa=3, c_kappa=4, use_noise=True)
    v = acq(torch.randn(10, 3), torch.ones(10, 3).long())
    assert (v[:, :3] + 3).abs().max() < 1e-6 and (v[:, 3:] + 4).abs().max() < 1e-6


def test_philox_draws_replay():
    m, no, nc = 1000, 2, 2
    mu, var = torch.randn(4, m, device=dev), torch.rand(4, m, device=dev)
    sd = torch.full((4,), 0.5, device=dev)
    a = _general_epilogue(mu, var, no, nc, 2.0, 0.5, sd, None, 7, 3, want_fc=True, want_cv=True)
    b = _general_epilogue(mu, var, no, nc, 2.0, 0.5, sd, None, 7, 3, want_fc=True, want_cv=True)
    c = _general_epilogue(mu, var, no, nc, 2.0, 0.5, sd, None, 7, 4, want_fc=True)
    assert all(torch.equal(u, v) for u, v in zip(a, b))
    assert not torch.equal(a[0], c[0])
    z = (torch.cat([a[0], a[1]], 1) - (mu.t() - torch.cat([2.0 * var.t()[:, :2].sqrt(), 0.5 * var.t()[:, 2:].sqrt()], 1))) / 0.5
    assert abs(float(z.mean())) < 0.05 and abs(float(z.std()) - 1) < 0.05     # N(0, 1) draws


# ------------------------------------------------------------------ optimisers (HEBO/test/test_optimizer.py)
def obj(x: pd.DataFrame) -> np.ndarray:
    return x["x0"].values.astype(float).reshape(-1, 1) ** 2


def test_opt_general_gp():
    space = DesignSpace().parse([{"name": "x0", "type": "num", "lb": -3, "ub": 7},
                                 {"name": "x1", "type": "cat", "categories": ["a", "b", "c"]}])
    opt = GeneralBO(space, rand_sample=8, model_name="gp")
    num_suggest = 0
    for i in range(11):
        num_suggest = 8 if opt.support_parallel_opt else 1
        rec = opt.suggest(n_suggestions=num_suggest)
        y = obj(rec)
        if y.shape[0] > 1 and i > 0:
            y[np.argmax(y.reshape(-1))] = np.inf
        opt.observe(rec, y)
        num_suggest += rec.shape[0]
        if num_suggest > 11:
            break


@pytest.mark.parametrize("num_suggest", [1, 4, 50])
def test_general_mo_constrained_opt(num_suggest):
    def f(param: pd.DataFrame) -> np.ndarray:
        x = param[["x0"]].values
        return np.hstack([x ** 2, (x - 3) * 2, -10 - x])
    space = DesignSpace().parse([{"name": "x0", "type": "num", "lb": -1, "ub": 4.0}])
    opt = GeneralBO(space, 2, 1, rand_sample=4)
    opt.evo_pop = 20
    for _ in range(2):
        rec = opt.suggest(num_suggest)
        assert rec.shape[0] == num_suggest
        opt.observe(rec, f(rec))


def test_contextual_opt_general():
    space = DesignSpace().parse([{"name": "x0", "type": "int", "lb": -20, "ub": 20},
                                 {"name": "x1", "type": "int", "lb": -20, "ub": 20}])
    opt = GeneralBO(space, rand_sample=2, model_name="gp")
    assert not opt.support_contextual                    # so the reference's test body does not run for GeneralBO


def test_ref_point_selection_and_one_objective_constrained_ga():
    space = DesignSpace().parse([{"name": "x0", "type": "num", "lb": -1, "ub": 4.0}])
    np.random.seed(3)
    opt = GeneralBO(space, 2, 0, rand_sample=6, evo_pop=30, evo_iters=20, ref_point=np.array([20.0, 10.0]))
    for _ in range(3):
        rec = opt.suggest(3)
        x = rec[["x0"]].values
        opt.observe(rec, np.hstack([x ** 2, (x - 3) * 2]))
        assert rec.shape[0] == 3 and len(set(rec.index)) == 3
    opt1 = GeneralBO(space, 1, 1, rand_sample=5, evo_pop=30, evo_iters=20)
    for _ in range(3):
        rec = opt1.suggest(1)
        x = rec[["x0"]].values
        opt1.observe(rec, np.hstack([(x - 1) ** 2, 0.5 - x]))             # feasible iff x >= 0.5
    assert opt1.best_y.shape[1] == 2


def test_one_objective_constrained_ga_returns_the_best_feasible_row():
    def score(xc, xe, gen):
        x = xc[:, 0]
        return (x - 1.0) ** 2, 0.5 - x                                     # best feasible: x = 1
    evo = DeviceNSGA2(["real"], [-2.0], [2.0], 1, score, pop=50, iters=30, seed=1, constrained=True, num_obj=1)
    xc, _, _ = evo.optimize()
    assert xc.shape == (1, 1) and abs(float(xc[0, 0]) - 1.0) < 0.05

    def infeasible(xc, xe, gen):
        x = xc[:, 0]
        return x, 5.0 - x                                                   # never feasible: least infeasible is x = 2
    xc, _, _ = DeviceNSGA2(["real"], [-2.0], [2.0], 1, infeasible, pop=20, iters=10, seed=2, constrained=True, num_obj=1).optimize()
    assert abs(float(xc[0, 0]) - 2.0) < 0.05


def test_quality_beats_random_sampling():
    """Two objectives and one constraint, 20 evaluations: the feasible front's hypervolume beats uniform random sampling
    with the same budget (fixed seeds)."""
    def f(x):
        x0, x1 = x[:, 0], x[:, 1]
        return np.stack([x0, (1 + x1) * (1 - np.sqrt(np.clip(x0, 0, None) / (1 + x1))), 0.2 - x0 - x1], 1)
    space = DesignSpace().parse([{"name": "x0", "type": "num", "lb": 0, "ub": 1}, {"name": "x1", "type": "num", "lb": 0, "ub": 1}])
    ref = np.array([1.1, 2.1])
    np.random.seed(0)
    torch.manual_seed(0)
    opt = GeneralBO(space, 2, 1, rand_sample=8, evo_pop=50, evo_iters=50)
    while opt.y.shape[0] < 20:
        rec = opt.suggest(4)
        opt.observe(rec, f(rec[["x0", "x1"]].values))
    hv_bo = hypervolume(opt.best_y[:, :2], ref)
    rng = np.random.default_rng(0)
    hv_rand = []
    for _ in range(5):
        y = f(rng.uniform(0, 1, (20, 2)))
        y = y[y[:, 2] <= 0]
        hv_rand.append(hypervolume(y[:, :2], ref))
    assert hv_bo > np.mean(hv_rand), (hv_bo, hv_rand)
