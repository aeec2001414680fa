"""HEBO_Embedding on the device: hb_embed_violation against an fp64 oracle, MACE_Embedding against hebo_b200.MACE and the
reference's fixture (tests/golden/ref_embedding.npz), hb_nsga2_survive_cv against hb_nsga2_survive_ex and the numpy
restatement (hebo_b200.evolution.survive_host), and the optimiser end to end on a problem too wide for the GP alone."""
import math

import numpy as np
import pytest
import torch

from hebo_b200 import _lib
from hebo_b200.acq import MACE
from hebo_b200.embedding import HEBO_Embedding, MACE_Embedding, embed_violation
from hebo_b200.evolution import survive_host
from hebo_b200.gp import GP

from .test_gpu_nsga_large import make_case, run_survive
from .util import assert_mace_close, load_golden

pytestmark = pytest.mark.gpu


def fp32_projection_bound(Y, B):
    """|fl32(Y B) - Y B| <= gamma_e sum_k |Y_ik B_kj| for an fp32 sum of e products (Higham 3.1), gamma_e = e u / (1 - e u)."""
    e = Y.shape[1]
    u = 2.0 ** -24
    return (e * u / (1 - e * u)) * (np.abs(Y) @ np.abs(B))


def check_against_fp64(Y, B, G):
    """G [m] from the device against the fp64 oracle.  Tolerance per row: 1e-5 max(G, 2^-20 sum_j |p_j|), plus the fp32
    error bound of every coordinate that may sit on the active side of |p| = 1.  Feasibility must agree on every row
    whose coordinates all keep a distance to 1 larger than their bound."""
    Y64, B64 = Y.astype(np.float64), B.astype(np.float64)
    p = Y64 @ B64
    G64 = np.maximum(np.abs(p) - 1.0, 0.0).sum(1)
    delta = fp32_projection_bound(Y64, B64)
    near = np.abs(p) >= 1.0 - delta
    tol = 1e-5 * np.maximum(G64, np.abs(p).sum(1) * 2.0 ** -20) + (delta * near).sum(1)
    err = np.abs(G.astype(np.float64) - G64)
    assert np.all(err <= tol), f"max excess {np.max(err - tol)}"
    clear = (np.abs(np.abs(p) - 1.0) > delta).all(1)
    assert np.array_equal((G > 0)[clear], (G64 > 0)[clear])
    return int(clear.sum())


SHAPES = [(1, 1, 1), (1, 16, 100003), (7, 1, 5), (129, 3, 1), (1000, 8, 10000), (300, 33, 257), (10001, 16, 1000),
          (65, 4096, 130), (131, 17, 4097)]


@pytest.mark.parametrize("m,e,D", SHAPES)
def test_embed_violation_matches_fp64_and_repeats_bit_for_bit(m, e, D):
    g = torch.Generator().manual_seed(m * 7 + e * 13 + D)
    B = torch.randn(e, D, generator=g) / math.sqrt(e)
    Y = (torch.rand(m, e, generator=g) * 2 - 1) * 1.5
    Y[::5] *= 0.05                                    # rows that are feasible or nearly so
    Yd, Bd = Y.cuda(), B.cuda()
    G1 = embed_violation(Yd, Bd)
    G2 = embed_violation(Yd, Bd)
    torch.cuda.synchronize()
    assert torch.equal(G1, G2)
    clear = check_against_fp64(Y.numpy(), B.numpy(), G1.cpu().numpy())
    assert clear >= 1 or m * D > 10 ** 6


def test_nan_coordinates_are_never_feasible():
    """torch.clamp keeps NaN in the reference's column; a NaN in a row of Y, or in a column of B, gives G = NaN."""
    g = torch.Generator().manual_seed(9)
    B = torch.randn(5, 300, generator=g) * 0.01                   # every finite row is feasible
    Y = torch.rand(40, 5, generator=g) * 2 - 1
    Y[7, 2] = float("nan")
    G = embed_violation(Y.cuda(), B.cuda()).cpu()
    assert torch.isnan(G[7]) and bool((G[torch.arange(40) != 7] == 0).all())
    B[3, 211] = float("nan")
    assert bool(torch.isnan(embed_violation(Y.cuda(), B.cuda())).all())
    Y[11, 0] = float("inf")                                       # an infinite coordinate is an infinite violation
    B[3, 211] = 0.0
    G = embed_violation(Y.cuda(), B.cuda()).cpu()
    assert torch.isinf(G[11]) or torch.isnan(G[11])


def test_embed_violation_rejects_bad_arguments():
    lib = _lib.lib()
    p = torch.zeros(16, device="cuda")
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    P, W = _lib.ptr(p), _lib.ptr(ws)
    for m, e, D in [(0, 2, 2), (2, 0, 2), (2, 4097, 2), (2, 2, 0), (-1, 2, 2)]:
        assert lib.hb_embed_violation_workspace_bytes(m, e, D) < 0
        assert lib.hb_embed_violation(P, m, e, P, D, P, W, ws.numel(), None) == _lib.HB_ERR_INVALID
    assert lib.hb_embed_violation(P, 2, 2, P, 2, P, W, 0, None) == _lib.HB_ERR_INVALID      # workspace too small
    assert lib.hb_embed_violation(None, 2, 2, P, 2, P, W, ws.numel(), None) == _lib.HB_ERR_INVALID


class FixedModel:
    """predict() returns fixed (mu, var): the stub model of the reference fixture."""

    def __init__(self, mu, var, noise):
        self.mu, self.var, self._n = mu, var, noise
        self.num_out = 1

    def predict(self, x, xe):
        return self.mu.clone(), self.var.clone()

    @property
    def noise(self):
        return self._n


def test_mace_embedding_against_mace_kernel_and_reference():
    z = load_golden("ref_embedding.npz")
    for ci in range(3):
        x, P, mu, var = (torch.from_numpy(z[f"e{ci}_{k}"]) for k in ("x", "P", "mu", "var"))
        tau, kappa, noise, eps, seed = z[f"e{ci}_par"]
        model = FixedModel(mu, var, torch.tensor([noise], dtype=torch.float32))
        acq = MACE_Embedding(model, best_y=np.float32(tau), proj_matrix=P.numpy(), kappa=float(kappa))
        assert acq.num_obj == 3 and acq.num_constr == 1
        torch.manual_seed(int(seed))
        out = acq.eval(x, None)
        torch.manual_seed(int(seed))
        F3 = MACE(model, best_y=np.float32(tau), kappa=float(kappa)).eval(x, None)
        assert out.shape == (x.shape[0], 4)
        assert torch.equal(out[:, :3], F3)
        check_against_fp64(x.numpy(), P.numpy().astype(np.float32), out[:, 3].numpy())
        F_ref = z[f"e{ci}_F"]
        assert_mace_close(out[:, :3].numpy(), F_ref[:, :3], mu.numpy(), var.numpy(), float(noise), float(tau), float(eps),
                          z[f"e{ci}_xi2"], what=f"case {ci}")
        # the reference's column 3 is an fp32 torch.mm: both sides sit within the fp32 bound of the exact value
        xn, Pn = x.numpy().astype(np.float64), z[f"e{ci}_P"].astype(np.float32).astype(np.float64)
        p = xn @ Pn
        delta = fp32_projection_bound(xn, Pn)
        tol = 2e-5 * np.maximum(F_ref[:, 3], np.abs(p).sum(1) * 2.0 ** -20) + 2 * (delta * (np.abs(p) >= 1 - delta)).sum(1)
        assert np.all(np.abs(out[:, 3].numpy().astype(np.float64) - F_ref[:, 3]) <= tol)


def test_mace_embedding_with_a_fitted_gp_equals_mace():
    g = torch.Generator().manual_seed(0)
    X = torch.rand(40, 4, generator=g) * 2 - 1
    y = (X ** 2).sum(1, keepdim=True) + 0.05 * torch.randn(40, 1, generator=g)
    np.random.seed(0)
    gp = GP(4, 0, 1, num_epochs=20, device="cuda")
    gp.fit(X, None, y)
    P = np.random.randn(4, 3000) / 2
    Xs = (torch.rand(500, 4, generator=g) * 2 - 1).cuda()
    torch.manual_seed(3)
    out = MACE_Embedding(gp, best_y=float(y.min()), proj_matrix=P, kappa=2.0).eval(Xs, None)
    torch.manual_seed(3)
    F3 = MACE(gp, best_y=float(y.min()), kappa=2.0).eval(Xs, None)
    assert torch.equal(out[:, :3], F3)
    assert torch.equal(out[:, 3], embed_violation(Xs, torch.as_tensor(P, dtype=torch.float32).cuda()).to(out.device))


# ---------------------------------------------------------------------------------------------------- survival
def run_survive_cv(X, F, G, C, FC, GC, d):
    lib = _lib.lib()
    P, D = X.shape
    dev = X.device
    Xn, Fn, Gn = torch.full((P, D), -7.0, device=dev), torch.full((P, 3), -7.0, device=dev), torch.full((P,), -7.0, device=dev)
    Xcn, Xen = torch.full((P, d), -7.0, device=dev), torch.full((P, D - d), -7, dtype=torch.int32, device=dev)
    pc = lambda x: _lib.ptr(x) if x.numel() else None
    ws_bytes = int(lib.hb_nsga2_workspace_bytes(P, D))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    _lib.check(lib.hb_nsga2_survive_cv(_lib.ptr(X), _lib.ptr(F), _lib.ptr(G), _lib.ptr(C), _lib.ptr(FC), _lib.ptr(GC), P, D, d,
                                       _lib.ptr(Xn), _lib.ptr(Fn), _lib.ptr(Gn), pc(Xcn), pc(Xen), _lib.ptr(ws), ws_bytes,
                                       _lib.stream_ptr()), "survive_cv")
    torch.cuda.synchronize()
    return Xn, Fn, Gn, Xcn, Xen


@pytest.mark.parametrize("P", [100, 1024, 4096])
def test_zero_constraint_equals_survive_ex(P):
    D, d = 6, 4
    X, F, C, FC = make_case(P, D, d, seed=P + 1)
    z = torch.zeros(P, device="cuda")
    a = run_survive(X, F, C, FC, d)
    b = run_survive_cv(X, F, z, C, FC, z, d)
    for u, v in zip(a, (b[0], b[1], b[3], b[4])):
        assert torch.equal(u, v)
    assert torch.equal(b[2], torch.zeros(P, device="cuda"))


DUP_CHILDREN = (3, 10, 11, 13)     # make_case: children equal to an earlier merged row


def constrained_case(P, n_feas, seed):
    D, d = 6, 4
    X, F, C, FC = make_case(P, D, d, seed=seed)
    rng = np.random.default_rng(seed)
    N = 2 * P
    G = np.abs(np.round(rng.standard_normal(N) * 8)).astype(np.float32) / 4 + 0.25     # infeasible, many ties
    unique = np.setdiff1d(np.arange(N), P + np.array(DUP_CHILDREN))
    G[rng.permutation(unique)[:n_feas]] = -rng.random(n_feas).astype(np.float32)
    infeas = np.flatnonzero(G > 0)
    G[infeas[:3]] = [np.nan, np.inf, -np.inf]
    Gt = torch.from_numpy(G).cuda()
    return X, F, Gt[:P].contiguous(), C, FC, Gt[P:].contiguous(), d


@pytest.mark.parametrize("P", [100, 300, 2048])
@pytest.mark.parametrize("which", ["none", "few", "exactly_pop", "more"])
def test_constrained_survival_equals_the_restatement(P, which):
    n_feas = {"none": 0, "few": 5, "exactly_pop": P, "more": P + P // 2}[which]
    X, F, G, C, FC, GC, d = constrained_case(P, n_feas, seed=P + len(which))
    Xn, Fn, Gn, Xcn, Xen = run_survive_cv(X, F, G, C, FC, GC, d)
    sel, f, g = survive_host(*(t.cpu().numpy() for t in (X, F, C, FC, G, GC)))
    Xa = torch.cat([X, C], 0)
    sel_t = torch.from_numpy(sel).cuda()
    assert sel.size == P
    assert torch.equal(Xn, Xa[sel_t])
    assert torch.equal(Fn, torch.from_numpy(f[sel]).cuda())
    assert torch.equal(Gn, torch.from_numpy(g[sel]).cuda())
    assert torch.equal(Xcn, Xa[sel_t][:, :d]) and torch.equal(Xen, Xa[sel_t][:, d:].round().to(torch.int32))
    nf = int((g <= 0).sum())
    assert nf == min(n_feas, 2 * P) and int((Gn <= 0).sum()) == min(nf, P)


@pytest.mark.parametrize("P", [100, 2048])
def test_non_finite_constraints_and_duplicates_survive_last(P):
    X, F, G, C, FC, GC, d = constrained_case(P, 7, seed=5)
    Ga = torch.cat([G, GC]).cpu().numpy()
    # many rows with a non-finite G, more finite infeasible rows than free slots
    Ga[np.flatnonzero(Ga > 0)[::4]] = np.nan
    Gt = torch.from_numpy(Ga).cuda()
    Xn, Fn, Gn, _, _ = run_survive_cv(X, F, Gt[:P].contiguous(), C, FC, Gt[P:].contiguous(), d)
    g = Gn.cpu().numpy()
    assert np.isfinite(g).all()
    dup_rows = torch.cat([X, C], 0)[[P + i for i in DUP_CHILDREN]]
    for row in dup_rows:
        hits = (Xn == row).all(1).sum().item()
        assert hits <= 1                                  # its earlier twin may survive, the duplicate child never does
    # enough finite, unique infeasible rows for every free slot: the survivors' G is the smallest such values
    _, _, gs = survive_host(*(t.cpu().numpy() for t in (X, F, C, FC)), Ga[:P], Ga[P:])
    finite_inf = np.sort(gs[np.isfinite(gs) & (gs > 0)])
    n_free = P - int((gs <= 0).sum())
    assert finite_inf.size >= n_free and np.array_equal(np.sort(g[g > 0]), finite_inf[:n_free])


# ---------------------------------------------------------------------------------------------------- end to end
D_BIG, I1, I2 = 10000, 17, 4242


def hidden_branin(x_hd: np.ndarray) -> np.ndarray:
    x = np.clip(x_hd, -1.0, 1.0)
    u, v = 7.5 * x[:, I1] + 2.5, 7.5 * x[:, I2] + 7.5      # [-1, 1] -> [-5, 10] x [0, 15]
    a, b, c, r, s, t = 1.0, 5.1 / (4 * np.pi ** 2), 5 / np.pi, 6.0, 10.0, 1 / (8 * np.pi)
    return (a * (v - b * u ** 2 + c * u - r) ** 2 + s * (1 - t) * np.cos(u) + s).reshape(-1, 1)


@pytest.mark.parametrize("acq_optimizer", ["sobol", "nsga2"])
def test_hidden_branin_in_ten_thousand_dimensions(acq_optimizer):
    space = [{"name": f"x{i}", "type": "num", "lb": -1, "ub": 1} for i in range(D_BIG)]
    with pytest.raises(NotImplementedError):
        GP(D_BIG, 0, 1)                                  # too wide for the GP on its own
    wins = []
    for seed in range(5):
        np.random.seed(seed)
        torch.manual_seed(seed)
        rnd = HEBO_Embedding(space, eff_dim=4, device="cuda")
        rs = hidden_branin(rnd.project(rnd.quasi_sample(40)).values).min()
        np.random.seed(seed)
        torch.manual_seed(seed)
        opt = HEBO_Embedding(space, eff_dim=4, acq_optimizer=acq_optimizer, device="cuda")
        for _ in range(40):
            rec = opt.suggest()
            x = opt.project(rec).values
            # the bound is evaluated in fp32: allow the fp32 rounding of a projection that sits on the boundary
            assert np.abs(x).max() <= 1.0 + 1e-5, np.abs(x).max()
            opt.observe(rec, hidden_branin(x))
        wins.append(opt.best_y < rs)
        print(f"{acq_optimizer} seed {seed}: HEBO_Embedding {opt.best_y:.4f}, random {rs:.4f}")
    assert sum(wins) >= 4, wins
