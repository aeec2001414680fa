"""HEBO_Embedding host logic (hebo_b200/embedding.py) and the constrained survival rule, CPU only."""
import itertools

import numpy as np
import pandas as pd
import pytest
import torch

from hebo_b200.embedding import HEBO_Embedding, check_design_space, gen_emb_space, gen_proj_matrix
from hebo_b200.evolution import survive_host
from hebo_b200.space import DesignSpace

from .util import load_golden


def box(D, lo=-1.0, hi=1.0):
    return [{"name": f"x{i}", "type": "num", "lb": lo, "ub": hi} for i in range(D)]


def test_gen_proj_matrix_equals_the_reference():
    z = load_golden("ref_embedding.npz")
    strategies = set()
    for ci in itertools.count():
        if f"proj{ci}" not in z:
            break
        eff, dim, seed = (int(v) for v in z[f"proj{ci}_case"])
        strategy = str(z[f"proj{ci}_strategy"])
        np.random.seed(seed)
        M = gen_proj_matrix(eff, dim, strategy)
        assert np.array_equal(M, z[f"proj{ci}"]), strategy
        strategies.add(strategy)
    assert strategies == {"hesbo", "alebo", "gaussian"}


def test_check_design_space_and_gen_emb_space():
    assert check_design_space(DesignSpace().parse(box(7)))
    assert not check_design_space(DesignSpace().parse(box(3, -1.0, 2.0)))
    assert not check_design_space(DesignSpace().parse(box(3, 0.0, 1.0)))
    assert not check_design_space(DesignSpace().parse(box(2) + [{"name": "n", "type": "int", "lb": -1, "ub": 1}]))
    assert not check_design_space(DesignSpace().parse(box(2) + [{"name": "c", "type": "cat", "categories": ["a", "b"]}]))
    sp = gen_emb_space(5, -2.5)
    assert sp.numeric_names == [f"y{i}" for i in range(5)]
    assert torch.equal(sp.opt_lb, torch.full((5,), -2.5, dtype=torch.float64))
    assert torch.equal(sp.opt_ub, torch.full((5,), 2.5, dtype=torch.float64))
    with pytest.raises(AssertionError):
        HEBO_Embedding(box(4, 0.0, 1.0), eff_dim=2, device="cpu")
    with pytest.raises(NotImplementedError):
        HEBO_Embedding(box(4), model_name="rf", eff_dim=2, device="cpu")


@pytest.mark.parametrize("strategy,eff_dim,D", [("alebo", 4, 500), ("hesbo", 3, 64), ("gaussian", 6, 2000)])
def test_quasi_sample_rows_project_inside_the_box(strategy, eff_dim, D):
    np.random.seed(3)
    h = HEBO_Embedding(box(D), eff_dim=eff_dim, strategy=strategy, device="cpu")
    for n in (1, 37, 250):
        s = h.quasi_sample(n)
        assert isinstance(s, pd.DataFrame) and s.shape == (n, eff_dim) and list(s.columns) == h.eff_space.numeric_names
        x = h.project(s).values
        assert x.shape == (n, D) and np.abs(x).max() <= 1.0
    xc, xe = h.quasi_sample(9, as_opt=True)
    assert xc.shape == (9, eff_dim) and xe.shape == (9, 0)


def test_project_with_and_without_clip():
    np.random.seed(0)
    h = HEBO_Embedding(box(30), eff_dim=3, device="cpu")
    df = pd.DataFrame(np.array([[0.5, -2.0, 1.0], [0.0, 0.0, 0.0]]), columns=h.eff_space.numeric_names)
    x = h.project(df)
    assert list(x.columns) == h.space.numeric_names
    assert np.allclose(x.values, df.values @ h.proj_matrix, rtol=0, atol=1e-15)
    np.random.seed(0)
    hc = HEBO_Embedding(box(30), eff_dim=3, clip=True, device="cpu")
    assert np.array_equal(hc.proj_matrix, h.proj_matrix)
    xc = hc.project(df).values
    assert np.allclose(xc, np.tanh(df.values @ h.proj_matrix), rtol=0, atol=1e-15) and np.abs(xc).max() < 1
    s = hc.quasi_sample(20)                                        # clip: uniform in the embedding box
    assert s.shape == (20, 3) and s.values.min() >= -1 and s.values.max() <= 1


def test_acquisition_optimiser_defaults_to_nsga2():
    assert HEBO_Embedding(box(10), eff_dim=2, device="cpu").mace.acq_optimizer == "nsga2"
    assert HEBO_Embedding(box(10), eff_dim=2, device="cpu", acq_optimizer="sobol").mace.acq_optimizer == "sobol"


def test_parallel_suggestions_need_clip():
    h = HEBO_Embedding(box(10), eff_dim=2, device="cpu")
    with pytest.raises(RuntimeError, match="Parallel optimization is supported only for MACE acquisition"):
        h.suggest(2)
    hc = HEBO_Embedding(box(10), eff_dim=2, clip=True, device="cpu")
    assert len(hc.suggest(3)) == 3                                  # start-up design, no GPU involved
    with pytest.raises(ValueError):
        HEBO_Embedding(box(10), eff_dim=2, device="cpu", n_refine=2)


def test_start_up_design_comes_from_the_embedding_sampler():
    D, eff = 200, 3
    np.random.seed(5)
    h = HEBO_Embedding(box(D), eff_dim=eff, device="cpu")
    assert h.mace.rand_sample == 1 + eff
    w = HEBO_Embedding(box(D), eff_dim=eff, device="cpu")
    w.proj_matrix = h.proj_matrix.copy()
    for it in range(h.mace.rand_sample):
        state = np.random.get_state()
        rec = h.suggest()
        np.random.set_state(state)
        assert np.array_equal(rec.values, w.quasi_sample(1).values)
        assert np.abs(h.project(rec).values).max() <= 1.0
        h.observe(rec, np.array([[float(it)]]))
    assert h.mace.Xc.shape == (h.mace.rand_sample, eff) and h.best_y == 0.0
    assert np.array_equal(h.best_x.values, h.mace.X.iloc[[0]].values)


# ---------------------------------------------------------------------------------------- constrained survival rule
def brute_survivors(F, G, P):
    """The constrained rule stated directly (no duplicates in the inputs): feasible iff G <= 0 (non-finite -> +inf); with
    >= P feasible rows, whole fronts of the feasible rows, the cut front by descending fp32 crowding (ties by index);
    otherwise all feasible rows, then the infeasible ones by (G, index)."""
    N = F.shape[0]
    f = [[np.float32(v) if np.isfinite(v) else np.float32(np.inf) for v in row] for row in F]
    g = [np.float32(v) if np.isfinite(v) else np.float32(np.inf) for v in G]
    feas = [i for i in range(N) if g[i] <= 0]
    if len(feas) < P:
        rest = sorted((i for i in range(N) if not g[i] <= 0), key=lambda i: (g[i], i))
        return sorted(feas + rest[:P - len(feas)])
    dom = lambda a, b: all(x <= y for x, y in zip(f[a], f[b])) and any(x < y for x, y in zip(f[a], f[b]))
    left, keep = set(feas), []
    while len(keep) < P:
        front = sorted(i for i in left if not any(dom(j, i) for j in left if j != i))
        left -= set(front)
        if len(keep) + len(front) <= P:
            keep += front
            continue
        m = len(front)
        crowd = {i: np.float32(0) for i in front}
        for k in range(3):
            order = sorted(front, key=lambda i: (f[i][k], i))
            lo, hi = f[order[0]][k], f[order[-1]][k]
            for p, i in enumerate(order):
                if p == 0 or p == m - 1:
                    crowd[i] = np.float32(np.inf)
                elif hi > lo and np.isfinite(hi - lo):
                    crowd[i] = np.float32(crowd[i] + np.float32(f[order[p + 1]][k] - f[order[p - 1]][k]) / np.float32(hi - lo))
        keep += sorted(front, key=lambda i: (-crowd[i], i))[:P - len(keep)]
    return sorted(keep)


@pytest.mark.parametrize("P,n_feas", [(12, 0), (12, 3), (12, 12), (12, 20), (30, 45), (30, 60), (30, 29)])
def test_constrained_survival_restatement_matches_the_brute_force_rule(P, n_feas):
    rng = np.random.default_rng(P * 100 + n_feas)
    N = 2 * P
    X = rng.random((P, 4)).astype(np.float32)
    C = rng.random((P, 4)).astype(np.float32)
    F = np.round(rng.standard_normal((P, 3)) * 2).astype(np.float32) / 2        # ties
    FC = np.round(rng.standard_normal((P, 3)) * 2).astype(np.float32) / 2
    G = np.abs(np.round(rng.standard_normal(N) * 4).astype(np.float32)) + 0.5     # infeasible, with ties
    G[rng.permutation(N)[:n_feas]] = -rng.random(n_feas).astype(np.float32)
    if n_feas < N:
        G[np.flatnonzero(G > 0)[:2]] = [np.nan, np.inf]
    F[1, 0] = np.nan
    sel, f, g = survive_host(X, F, C, FC, G[:P], G[P:])
    assert sel.tolist() == brute_survivors(np.concatenate([F, FC]), G, P)
    assert sel.size == P and np.isinf(g[~np.isfinite(G)]).all()


def test_restatement_without_g_is_the_zero_g_rule():
    rng = np.random.default_rng(1)
    P = 40
    X, C = rng.random((P, 3)).astype(np.float32), rng.random((P, 3)).astype(np.float32)
    F, FC = rng.standard_normal((P, 3)).astype(np.float32), rng.standard_normal((P, 3)).astype(np.float32)
    a, _, _ = survive_host(X, F, C, FC)
    b, _, _ = survive_host(X, F, C, FC, np.zeros(P, np.float32), np.zeros(P, np.float32))
    assert np.array_equal(a, b) and a.tolist() == brute_survivors(np.concatenate([F, FC]), np.zeros(2 * P), P)
