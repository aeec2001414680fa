"""Large-population NSGA-II survival (hebo_b200/csrc/nsga.cu, nsga_survive_large_kernel: 256 < pop <= 16384) against a
restatement of the survival rules written here in torch, chunked on the device:
  * every objective component that is not finite becomes +inf, one component at a time;
  * child i is a duplicate when |o[k] - me[k]| <= 1e-16 (fp32) for every k against any merged row j < i; its three
    objectives become +inf;
  * fast non-dominated sort (all <=, one <), fronts peeled until the cumulative count reaches pop;
  * fp32 crowding on the cut front, k = 0, 1, 2: stable order by f_k (ties by merged index), ends +inf, interior adds
    (f[next] - f[prev]) / (fmax - fmin) when fmax > fmin and fmax - fmin is finite; the `need` largest crowding values
    survive, ties by lower merged index;
  * survivors in ascending merged-row order."""
import numpy as np
import pandas as pd
import pytest
import torch

from hebo_b200 import _lib
from hebo_b200.evolution import DeviceNSGA2, fast_non_dominated_sort
from hebo_b200.suggest import HEBO

pytestmark = pytest.mark.gpu
INF = float("inf")


def _count_dominators(fa, fb):
    """For every row of fb: how many rows of fa dominate it."""
    chunk = max(1024, (1 << 23) // max(1, min(fa.shape[0], 8192)))
    out = torch.zeros(fb.shape[0], dtype=torch.int64, device=fb.device)
    for b0 in range(0, fb.shape[0], chunk):
        me = fb[b0:b0 + chunk]
        acc = torch.zeros(me.shape[0], dtype=torch.int64, device=fb.device)
        for a0 in range(0, fa.shape[0], 8192):
            o = fa[a0:a0 + 8192]
            le = (o[None, :, :] <= me[:, None, :]).all(-1)
            lt = (o[None, :, :] < me[:, None, :]).any(-1)
            acc += (le & lt).sum(1)
        out[b0:b0 + chunk] = acc
    return out


def survive_reference(X, F, C, FC):
    P, D = X.shape
    N = 2 * P
    Xa = torch.cat([X, C], 0)
    f = torch.cat([F, FC], 0).clone()
    f = torch.where(torch.isfinite(f), f, torch.full_like(f, INF))
    # duplicates
    idx = torch.arange(N, device=X.device)
    for c0 in range(P, N, 64):
        c1 = min(N, c0 + 64)
        me = Xa[c0:c1]
        eq = torch.ones(c1 - c0, c1, dtype=torch.bool, device=X.device)
        for k in range(D):
            eq &= (Xa[None, :c1, k] - me[:, None, k]).abs() <= 1e-16
        eq &= idx[None, :c1] < idx[c0:c1, None]
        dup = eq.any(1)
        f[c0:c1][dup] = INF
    # ranks
    ndom = _count_dominators(f, f)
    rank = torch.full((N,), -1, dtype=torch.int64, device=X.device)
    cum, r, rc, need = 0, 0, -1, 0
    while True:
        front = torch.nonzero((rank < 0) & (ndom == 0)).reshape(-1)
        if front.numel() == 0:
            break
        rank[front] = r
        if cum + front.numel() >= P:
            rc, need = r, P - cum
            break
        cum += front.numel()
        rest = torch.nonzero(rank < 0).reshape(-1)
        ndom[rest] -= _count_dominators(f[front], f[rest])
        r += 1
    keep = (rank >= 0) & (rank < rc)
    members = torch.nonzero(rank == rc).reshape(-1)          # ascending merged index
    m = members.numel()
    fm = f[members]
    crowd = torch.zeros(m, dtype=torch.float32, device=X.device)
    ar = torch.arange(m, device=X.device)
    for k in range(3):
        v = fm[:, k]
        order = torch.sort(v, stable=True).indices
        pos = torch.empty_like(order)
        pos[order] = ar
        fmin, fmax = v[order[0]], v[order[-1]]
        prev = v[order[(pos - 1).clamp(min=0)]]
        nxt = v[order[(pos + 1).clamp(max=m - 1)]]
        ends = (pos == 0) | (pos == m - 1)
        ok = bool(fmax > fmin) and bool(torch.isfinite(fmax - fmin))
        if ok:
            crowd = torch.where(ends, crowd, crowd + (nxt - prev) / (fmax - fmin))
        crowd = torch.where(ends, torch.full_like(crowd, INF), crowd)
    chosen = members[torch.sort(crowd, descending=True, stable=True).indices[:need]]
    keep[chosen] = True
    sel = torch.nonzero(keep).reshape(-1)
    return Xa[sel], f[sel]


def run_survive(X, F, C, FC, d, entry="ex"):
    lib = _lib.lib()
    P, D = X.shape
    dev = X.device
    Xn, Fn = torch.full((P, D), -7.0, device=dev), torch.full((P, 3), -7.0, device=dev)
    Xcn, Xen = torch.full((P, d), -7.0, device=dev), torch.full((P, D - d), -7, dtype=torch.int32, device=dev)
    pc = lambda x: _lib.ptr(x) if x.numel() else None
    if entry == "ex":
        ws_bytes = int(lib.hb_nsga2_workspace_bytes(P, D))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        _lib.check(lib.hb_nsga2_survive_ex(_lib.ptr(X), _lib.ptr(F), _lib.ptr(C), _lib.ptr(FC), P, D, d, _lib.ptr(Xn), _lib.ptr(Fn),
                                           pc(Xcn), pc(Xen), _lib.ptr(ws), ws_bytes, _lib.stream_ptr()), "survive_ex")
    else:
        _lib.check(lib.hb_nsga2_survive(_lib.ptr(X), _lib.ptr(F), _lib.ptr(C), _lib.ptr(FC), P, D, d, _lib.ptr(Xn), _lib.ptr(Fn),
                                        pc(Xcn), pc(Xen), _lib.stream_ptr()), "survive")
    torch.cuda.synchronize()
    return Xn, Fn, Xcn, Xen


def assert_matches_reference(X, F, C, FC, d, out):
    Xn, Fn, Xcn, Xen = out
    Xr, Fr = survive_reference(X, F, C, FC)
    assert Xr.shape == Xn.shape
    assert torch.equal(Xn, Xr)
    assert torch.equal(Fn, Fr)
    assert torch.equal(Xcn, Xr[:, :d])
    assert torch.equal(Xen, Xr[:, d:].round().to(torch.int32))


def make_case(P, D, d, seed):
    """Ties, duplicates (child = population row, child = earlier child, near-0 rows within 1e-16), NaN / +-inf objectives
    and a trade-off surface with many fronts."""
    g = torch.Generator().manual_seed(seed)
    X, C = torch.rand(P, D, generator=g), torch.rand(P, D, generator=g)
    X[:, d:] = torch.randint(0, 5, (P, D - d), generator=g).float()
    C[:, d:] = torch.randint(0, 5, (P, D - d), generator=g).float()
    F, FC = torch.randn(P, 3, generator=g), torch.randn(P, 3, generator=g)
    # a noisy trade-off: several large fronts plus many small ones
    F[:, 2] = 0.5 * F[:, 0] - 0.5 * F[:, 1] + 0.05 * torch.randn(P, generator=g)
    FC[:, 2] = 0.5 * FC[:, 0] - 0.5 * FC[:, 1] + 0.1 + 0.05 * torch.randn(P, generator=g)
    F[:, 0] = torch.round(F[:, 0] * 4) / 4                             # ties
    FC[::3, 1] = torch.round(FC[::3, 1] * 2) / 2
    C[3] = X[5]                                                        # child = population row
    C[10] = C[4]                                                       # child = earlier child
    X[7] = 1e-17                                                       # near 0: within 1e-16 -> duplicate
    C[11] = 3e-17
    C[12] = 1e-12                                                      # near 0 but farther than 1e-16: distinct
    X[8] = 0.0
    C[13] = -0.0                                                       # -0 == +0
    C[14] = X[200 % P]
    C[14, 0] = torch.nextafter(C[14, 0], torch.tensor(2.0))            # one ulp away: distinct
    FC[7, 1] = float("nan")
    F[9, 0] = INF
    FC[20, 2] = -INF
    F[15] = float("nan")
    FC[21] = torch.tensor([float("nan"), -INF, INF])
    return [t.cuda() for t in (X, F, C, FC)]


@pytest.mark.parametrize("P", [257, 1000, 4096, 16384])
def test_large_survival_equals_the_restatement(P):
    D, d = 6, 4
    X, F, C, FC = make_case(P, D, d, seed=P)
    assert_matches_reference(X, F, C, FC, d, run_survive(X, F, C, FC, d))


def test_both_sides_of_the_size_switch_agree_at_pop_256():
    P, D, d = 256, 6, 4
    X, F, C, FC = make_case(P, D, d, seed=7)
    a = run_survive(X, F, C, FC, d, "ex")
    b = run_survive(X, F, C, FC, d, "plain")
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    assert_matches_reference(X, F, C, FC, d, a)


def test_totally_ordered_objectives_one_row_per_front():
    P, D, d = 2048, 3, 3
    g = torch.Generator().manual_seed(3)
    X, C = torch.rand(P, D, generator=g), torch.rand(P, D, generator=g)
    t = torch.randperm(2 * P, generator=g).float()
    Fa = torch.stack([t, 2 * t, t - 5], 1)
    F, FC = Fa[:P].contiguous(), Fa[P:].contiguous()
    X, F, C, FC = [v.cuda() for v in (X, F, C, FC)]
    out = run_survive(X, F, C, FC, d)
    assert_matches_reference(X, F, C, FC, d, out)
    keep = torch.nonzero(t < P).reshape(-1).cuda()                       # the P smallest survive
    assert torch.equal(out[0], torch.cat([X, C], 0)[keep])


def test_population_that_cannot_be_filled_with_distinct_rows():
    """Two 3-way categorical columns: 9 distinct rows for 2000 merged rows.  Half the population holds the duplicates an
    earlier generation kept (+inf objectives), so the duplicate children survive as +inf rows."""
    P, D, d = 1000, 2, 0
    g = torch.Generator().manual_seed(4)
    X = torch.randint(0, 3, (P, D), generator=g).float()
    C = torch.randint(0, 3, (P, D), generator=g).float()
    F, FC = torch.randn(P, 3, generator=g), torch.randn(P, 3, generator=g)
    F[P // 2:] = INF
    X, F, C, FC = [v.cuda() for v in (X, F, C, FC)]
    out = run_survive(X, F, C, FC, d)
    assert_matches_reference(X, F, C, FC, d, out)
    assert int(torch.isinf(out[1]).all(1).sum()) > 0


def test_two_calls_are_bitwise_equal():
    P, D, d = 16384, 8, 6
    X, F, C, FC = make_case(P, D, d, seed=11)
    a = run_survive(X, F, C, FC, d)
    b = run_survive(X, F, C, FC, d)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def _toy_score(xc, xe, gen):
    p = xc[:, 1] ** 2 + (xe[:, 0].float() - 2) ** 2
    return torch.stack([xc[:, 0] ** 2 + p, (xc[:, 0] - 1) ** 2 + p, p], 1)


def test_device_nsga2_large_population_finds_the_pareto_set():
    """The toy problem of test_gpu_nsga.py at pop 4096: Pareto set {x0 in [0, 1], x1 = 0, k = 2}.  With thousands of
    members, the row of smallest penalty p stays non-dominated wherever its x0 lies, so a few members of the final
    front may sit outside [0, 1]; nearly all must lie in the Pareto set."""
    def run():
        evo = DeviceNSGA2(["real", "real", "choice"], [-2.0, -2.0, 0.0], [2.0, 2.0, 4.0], 2, _toy_score, pop=4096, iters=40, seed=5)
        xc, xe, F = evo.optimize(initial_suggest=np.array([[1.9, 1.9, 0.0]]))
        return evo, xc, xe, F
    evo, xc, xe, F = run()
    assert evo.n_evals == 4096 * 40 and xc.shape[0] >= 500
    assert bool((xe.reshape(-1) == 2).all())
    inside = (xc[:, 1].abs() < 0.12) & (xc[:, 0] > -0.1) & (xc[:, 0] < 1.1)
    assert float(inside.float().mean()) >= 0.95, float(inside.float().mean())
    assert float(xc[inside, 0].max() - xc[inside, 0].min()) > 0.8
    rank = fast_non_dominated_sort(evo.pop_F.cpu().double().numpy())
    assert (rank == 0).sum() == xc.shape[0]
    evo2, xc2, xe2, F2 = run()
    assert torch.equal(evo.pop_X, evo2.pop_X) and torch.equal(evo.pop_F, evo2.pop_F)
    assert torch.equal(xc, xc2) and torch.equal(xe, xe2) and torch.equal(F, F2)


def _mixed_objective(df: pd.DataFrame) -> np.ndarray:
    pen = {"a": 0.6, "b": 0.0, "c": 1.2}
    return ((np.log10(df["lr"].values.astype(float)) + 2.5) ** 2 + 0.05 * (df["n"].values.astype(float) - 6) ** 2 +
            np.array([pen[c] for c in df["c"]]) + 0.5 * (df["x"].values.astype(float) - 0.5) ** 2).reshape(-1, 1)


def test_bo_loop_with_a_large_nsga2_population_on_a_mixed_space():
    torch.manual_seed(0)
    np.random.seed(0)
    spec = [{"name": "lr", "type": "pow", "lb": 1e-5, "ub": 1e-1}, {"name": "n", "type": "int", "lb": 1, "ub": 10},
            {"name": "c", "type": "cat", "categories": ["a", "b", "c"]}, {"name": "x", "type": "num", "lb": -2, "ub": 2}]
    opt = HEBO(spec, scramble_seed=2, acq_optimizer="nsga2", evo_pop=2048, evo_iters=6)
    for it in range(5):
        rec = opt.suggest(4)
        assert isinstance(rec, pd.DataFrame) and len(rec) == 4 and set(rec["c"]) <= {"a", "b", "c"}
        assert all(float(v).is_integer() and 1 <= v <= 10 for v in rec["n"]) and bool(((rec["x"] >= -2) & (rec["x"] <= 2)).all())
        opt.observe(rec, _mixed_objective(rec))
    assert opt.Xc.shape[0] == 20
    rec = opt.suggest(3, fix_input={"c": "a"})
    assert len(rec) == 3 and set(rec["c"]) == {"a"}
