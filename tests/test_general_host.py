"""Host logic of GeneralBO (hebo_b200/general.py) and the k-objective / constrained host survivals (hebo_b200/evolution.py)."""
import itertools
import os

import numpy as np
import pandas as pd
import pytest

from hebo_b200.evolution import DeviceNSGA2, ga_survive_host, rank_and_crowding_survival, survive_host
from hebo_b200.general import GeneralBO, hypervolume
from hebo_b200.space import DesignSpace

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ref_general_acq.npz")
SPACE = [{"name": "x0", "type": "num", "lb": -1, "ub": 4.0}]


def test_golden_fixture_is_the_fp32_expression():
    """The reference outputs stored in the fixture are the torch expression of acq.py:234-241 on the recorded draws.  They
    differ from the correctly rounded fp32 evaluation only through torch's CPU sqrt, which is off by one ulp in some rows:
    at most one ulp of ps, scaled by kappa, plus the final rounding."""
    z = np.load(GOLDEN)
    f = np.float32
    for ci in range(int(z["n_cases"])):
        p = f"c{ci}_"
        m, no, nc, use_noise, _ = [int(v) for v in z[p + "meta"]]
        kappa, c_kappa = [f(v) for v in z[p + "kappa"]]
        ps = np.sqrt(z[p + "var"])
        ps = np.where(ps < np.finfo(f).eps, np.finfo(f).eps, ps).astype(f)
        noise_sd = z[p + "noise_sd"]                                         # model.noise.sqrt() as the reference computed it
        py = z[p + "mu"] + (noise_sd[None] * z[p + "xi"]).astype(f) if use_noise else z[p + "mu"]
        want = np.concatenate([py[:, :no] - kappa * ps[:, :no], py[:, no:] - c_kappa * ps[:, no:]], 1).astype(f)
        kap = np.array([kappa] * no + [c_kappa] * nc, f)
        tol = 2 * (kap * np.spacing(ps) + np.spacing(np.abs(want)))        # one ulp of ps through two roundings
        assert want.shape == (m, no + nc) and (np.abs(want - z[p + "out"]) <= tol).all()
        assert (want[: m // 10] == z[p + "out"][: m // 10]).all()        # clamped ps = FLT_EPSILON: no sqrt involved


def _box_union_volume(Y, ref):
    """Inclusion-exclusion over the boxes [y, ref]."""
    Y = [y for y in Y if (y < ref).all()]
    vol = 0.0
    for r in range(1, len(Y) + 1):
        for S in itertools.combinations(Y, r):
            vol += (-1) ** (r + 1) * np.prod(ref - np.max(S, 0))
    return vol


def test_hypervolume_closed_forms_and_inclusion_exclusion():
    ref = np.array([4.0, 4.0])
    Y = np.array([[1.0, 3.0], [2.0, 2.0], [3.0, 1.0], [5.0, 0.0], [2.5, 2.5]])
    assert hypervolume(Y, ref) == pytest.approx(3 * 1 + 2 * 1 + 1 * 1)      # staircase; (5, 0) and (2.5, 2.5) add nothing
    assert hypervolume(np.zeros((0, 2)), ref) == 0.0
    rng = np.random.default_rng(0)
    for k in (3, 4):
        for _ in range(5):
            Y = rng.uniform(0, 1, (7, k))
            ref = np.full(k, 0.9)
            assert hypervolume(Y, ref) == pytest.approx(_box_union_volume(Y, ref), rel=1e-12, abs=1e-15)


def test_get_pf_and_best_x_are_the_feasible_front():
    opt = GeneralBO(SPACE, 2, 1)
    rng = np.random.default_rng(1)
    y = np.round(rng.normal(size=(60, 3)), 1)
    X = pd.DataFrame({"x0": rng.uniform(-1, 4, 60)})
    opt.observe(X, y)
    feas = y[:, 2] <= 0
    brute = [i for i in range(60) if feas[i] and not any(feas[j] and (y[j, :2] <= y[i, :2]).all() and (y[j, :2] < y[i, :2]).any()
                                                          for j in range(60))]
    assert np.array_equal(opt.best_y, y[brute])
    assert np.array_equal(opt.best_x["x0"].values, X["x0"].values[brute])


def test_observe_drops_non_finite_rows_and_checks_the_width():
    opt = GeneralBO(SPACE, 2, 0)
    opt.observe(pd.DataFrame({"x0": [0.0, 1.0, 2.0]}), np.array([[1.0, 2.0], [np.nan, 1.0], [3.0, np.inf]]))
    assert opt.y.shape == (1, 2) and opt.X.shape[0] == 1
    with pytest.raises(AssertionError):
        opt.observe(pd.DataFrame({"x0": [0.0]}), np.array([[1.0, 2.0, 3.0]]))


def test_constructor_checks():
    with pytest.raises(NotImplementedError):
        GeneralBO(SPACE, model_name="rf")
    with pytest.raises(AssertionError):
        GeneralBO(SPACE, 2, 0, model_name="gp")
    opt = GeneralBO(SPACE, 2, 1)
    assert opt.rand_sample == 2 and opt.evo_pop == 100 and opt.evo_iters == 200 and opt.kappa == 2.0 and opt.c_kappa == 0.0
    assert not (opt.support_parallel_opt or opt.support_constraint or opt.support_multi_objective or opt.support_contextual)
    with pytest.raises(ValueError):
        DeviceNSGA2(["real"], [0.0], [1.0], 1, None, pop=10, num_obj=9, device="cpu")


class _StubModel:
    def __init__(self, ps2):
        self.ps2 = ps2

    def predict(self, Xc, Xe):
        return np.zeros_like(self.ps2), self.ps2

    def sample_y(self, Xc, Xe, n):
        rng = np.random.default_rng(5)
        return rng.normal(size=(n, self.ps2.shape[0], self.ps2.shape[1])) + 1.0


def _stubbed(opt, front, ps2):
    opt._fit = lambda: _StubModel(ps2)
    opt._optimise = lambda model, kappa, c_kappa: front
    return opt


def test_selection_rules():
    front = pd.DataFrame({"x0": np.linspace(0, 3, 6)})
    ps2 = np.ones((6, 2))
    ps2[4] = 10.0
    opt = GeneralBO(SPACE, 2, 0, rand_sample=1)
    opt.observe(pd.DataFrame({"x0": [0.0]}), np.array([[1.0, 1.0]]))
    _stubbed(opt, front, ps2)
    np.random.seed(0)
    rec = opt.suggest(8)                                                     # top-up: the front plus random rows
    assert rec.shape[0] == 8 and np.array_equal(rec["x0"].values[:6], front["x0"].values)
    np.random.seed(0)
    rec = opt.suggest(3)                                                     # the most uncertain row is always picked
    assert 4 in rec.index and rec.shape[0] == 3
    opt.ref_point = np.array([5.0, 5.0])
    np.random.seed(0)
    rec = opt.suggest(4)                                                     # EHVI, de-duplicated, topped up
    assert rec.shape[0] == 4 and len(set(rec.index)) == 4


def test_start_up_design_and_kappa_schedule():
    opt = GeneralBO(SPACE, 2, 1, rand_sample=3, kappa=None, c_kappa=None)
    rec = opt.suggest(5, fix_input={"x0": 1.5})
    assert (rec["x0"] == 1.5).all() and rec.shape[0] == 5
    k, c = opt._kappas()
    assert k == c and k > 0


def _brute_ga(X, F, C, FC, G, GC):
    P = X.shape[0]
    Xa = np.concatenate([X, C], 0)
    f = np.concatenate([F, FC]).astype(np.float32)
    g = np.concatenate([G, GC]).astype(np.float32)
    f = np.where(np.isfinite(f), f, np.inf)
    g = np.where(np.isfinite(g), np.maximum(g, 0), np.inf)
    for i in range(P, 2 * P):
        if any((np.abs(Xa[j] - Xa[i]) <= 1e-16).all() for j in range(i)):
            f[i] = g[i] = np.inf
    return sorted(range(2 * P), key=lambda i: (g[i], f[i], i))[:P]


def test_ga_survive_host_with_constraint_equals_a_sort():
    rng = np.random.default_rng(2)
    for P in (1, 5, 40):
        X, C = rng.integers(0, 3, (P, 2)).astype(np.float32), rng.integers(0, 3, (P, 2)).astype(np.float32)
        F, FC = np.round(rng.normal(size=P), 1).astype(np.float32), np.round(rng.normal(size=P), 1).astype(np.float32)
        G, GC = np.round(rng.normal(size=P), 1).astype(np.float32), np.round(rng.normal(size=P), 1).astype(np.float32)
        F[::5], GC[::7] = np.nan, np.inf
        sel, _, _ = ga_survive_host(X, F, C, FC, G, GC)
        assert list(sel) == _brute_ga(X, F, C, FC, G, GC)
        sel0, _ = ga_survive_host(X, F, C, FC)
        assert len(sel0) == P


@pytest.mark.parametrize("k", [2, 4, 8])
def test_survive_host_k_equals_rank_and_crowding(k):
    """Distinct rows and continuous objectives (no ties): survive_host over k objectives picks the rows of the plain
    rank-and-crowding restatement."""
    rng = np.random.default_rng(k)
    P = 30
    X, C = rng.uniform(size=(P, 3)).astype(np.float32), rng.uniform(size=(P, 3)).astype(np.float32)
    F, FC = rng.uniform(size=(P, k)).astype(np.float32), rng.uniform(size=(P, k)).astype(np.float32)
    sel, f, _ = survive_host(X, F, C, FC)
    assert f.shape == (2 * P, k)
    want = np.sort(rank_and_crowding_survival(np.concatenate([F, FC]).astype(np.float64), P))
    assert np.array_equal(sel, want)
