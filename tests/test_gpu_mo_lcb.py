"""MOMeanSigmaLCB on the device: hb_mo_lcb_epilogue against the fp32 restatement, MOMeanSigmaLCB.eval against the
reference fixture, the device score of general_score, and HEBO(acq_cls=...) with both acquisition optimisers
(HEBO/test/test_acq.py::test_mo_acq and the acq_cls argument of optimizers/hebo.py)."""
import os

import numpy as np
import pandas as pd
import pytest
import torch

import hebo_b200.acq as A
import hebo_b200.evolution as E
from hebo_b200 import GP, MACE, MOMeanSigmaLCB
from hebo_b200.acq import _general_epilogue, _mo_lcb_epilogue, general_score
from hebo_b200.space import DesignSpace
from hebo_b200.suggest import HEBO
from tests.test_mo_lcb_host import mo_lcb_fp32, same_bits
from tests.util import seeded_problem

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ref_mo_lcb.npz")
dev = torch.device("cuda")
t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
EDGE_VAR = [0.0, 1e-30, 1e-40, 1e-45, 1e-12, 1e30, -1.0, float("nan"), float("inf")]


def epilogue_case(m, seed):
    rng = np.random.default_rng(seed)
    mu = (rng.normal(size=m) * 3).astype(np.float32)
    var = (rng.random(m) * 2).astype(np.float32)
    k = min(m, len(EDGE_VAR))
    var[:k] = np.array(EDGE_VAR, np.float32)[:k]
    if m > k:
        mu[k] = np.nan
    xi = rng.normal(size=m).astype(np.float32)
    return mu, var, xi


@pytest.mark.parametrize("kappa,best_y", [(2.0, 0.0), (3.7, -1.25), (-1.5, 0.6180339887)])
@pytest.mark.parametrize("m", [1, 2, 9, 255, 256, 257, 1000, 4097, 131072, 1000003])
def test_epilogue_is_the_fp32_expression(m, kappa, best_y):
    mu, var, xi = epilogue_case(m, 7 * m + int(10 * abs(kappa)))
    noise_sd = float(np.sqrt(np.float32(0.037)))
    F, G = _mo_lcb_epilogue(t(mu), t(var), noise_sd, best_y, kappa, t(xi))
    want = mo_lcb_fp32(mu[:, None], var[:, None], noise_sd, xi[:, None], kappa, best_y)
    got = torch.cat([F, G[:, None]], 1).cpu().numpy()
    assert same_bits(got, want)
    if m >= 2:
        assert np.signbit(got[0, 1]) and got[0, 1] == 0                     # var = 0: -1 * +0 = -0
        assert -1e-14 < got[1, 1] < 0                                        # tiny var: no FLT_EPSILON clamp
    if m >= 8:
        assert np.isnan(got[6:8, 1:]).all()                                  # negative and NaN var give NaN


def test_philox_draws_replay_and_match_the_general_epilogue():
    m = 100003
    mu, var, _ = epilogue_case(m, 5)
    var = np.abs(np.nan_to_num(var, nan=1.0, posinf=1.0))                    # finite ps, so that 0 * ps = 0 below
    mu = np.nan_to_num(mu)
    sd = 0.25
    a = _mo_lcb_epilogue(t(mu), t(var), sd, 0.3, 2.0, None, 11, 4)
    b = _mo_lcb_epilogue(t(mu), t(var), sd, 0.3, 2.0, None, 11, 4)
    c = _mo_lcb_epilogue(t(mu), t(var), sd, 0.3, 2.0, None, 11, 5)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert not torch.equal(a[0][:, 0], c[0][:, 0])
    Fo, _, _ = _general_epilogue(t(mu)[None], t(var)[None], 1, 0, 0.0, 0.0, torch.full((1,), sd, device=dev), None, 11, 4)
    assert same_bits(a[0][:, 0].cpu().numpy(), Fo[:, 0].cpu().numpy())     # K = 1, kappa = 0: py itself
    z = (a[0][:, 0] - t(mu)) / sd
    assert abs(float(z.mean())) < 0.02 and abs(float(z.std()) - 1) < 0.02


def test_epilogue_graph_capture_replays_bit_for_bit():
    m = 5000
    mu, var, _ = epilogue_case(m, 9)
    mu_d, var_d = t(mu), t(var)
    F0, G0 = _mo_lcb_epilogue(mu_d, var_d, 0.1, 0.5, 2.0, None, 3, 7)
    eager = torch.cat([F0, G0[:, None]], 1)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _mo_lcb_epilogue(mu_d, var_d, 0.1, 0.5, 2.0, None, 3, 7)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        F, G = _mo_lcb_epilogue(mu_d, var_d, 0.1, 0.5, 2.0, None, 3, 7)
    F.fill_(0.0)
    G.fill_(0.0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.cat([F, G[:, None]], 1).cpu().numpy().tobytes() == eager.cpu().numpy().tobytes()


class Stub:
    """A non-GP model: fixed (mu, var) [m, 1] and a float32 noise [1]."""

    def __init__(self, mu, var, noise):
        self.mu, self.var, self.noise, self.num_out = mu, var, noise, 1

    def predict(self, x, xe):
        return self.mu.clone(), self.var.clone()


def test_eval_reproduces_the_reference():
    """eval's draws are the reference's; its ps is the correctly rounded root, which torch's CPU sqrt (and so the
    fixture) misses by one ulp in some rows."""
    z = np.load(GOLDEN)
    for ci in range(int(z["n_cases"])):
        p = f"c{ci}_"
        m, seed = [int(v) for v in z[p + "meta"]]
        kappa, best_y = float(z[p + "kappa"]), float(z[p + "best_y"])
        stub = Stub(torch.from_numpy(z[p + "mu"]), torch.from_numpy(z[p + "var"]), torch.from_numpy(z[p + "noise"]))
        torch.manual_seed(seed)
        v = MOMeanSigmaLCB(stub, best_y=best_y, kappa=kappa)(torch.zeros(m, 1), None)
        assert v.device.type == "cpu" and v.shape == (m, 3)
        v = v.numpy()
        assert same_bits(v, mo_lcb_fp32(z[p + "mu"], z[p + "var"], z[p + "noise_sd"][0], z[p + "xi"], kappa, best_y)), ci
        ref = z[p + "out"]
        assert same_bits(np.isnan(v), np.isnan(ref)) and same_bits(v[:, 0], ref[:, 0])
        ok = ~np.isnan(ref[:, 1])
        ps = -v[ok, 1]
        assert (np.abs(v[ok, 1] - ref[ok, 1]) <= np.spacing(ps)).all(), ci
        ok = ~np.isnan(ref[:, 2])                                            # a NaN mean leaves ps finite
        ps = np.abs(v[ok, 1])
        tol = abs(np.float32(kappa)) * np.spacing(ps) + 2 * np.spacing(np.abs(v[ok, 2]))
        assert (np.abs(v[ok, 2] - ref[ok, 2]) <= tol).all(), ci


def fitted_gp(d=3, e=1, n=60, seed=0):
    X, y = seeded_problem(n, d, seed)
    g = torch.Generator().manual_seed(seed + 1)
    Xe = torch.randint(0, 3, (n, e), generator=g) if e else None
    if e:
        y = y + 0.3 * Xe[:, :1].float()
    gp = GP(d, e, 1, device="cuda", num_epochs=40, num_uniqs=[3] * e if e else None)
    gp.fit(X, Xe, y)
    return gp


def rows(m, d, e, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(m, d, generator=g) * 2 - 1, torch.randint(0, 3, (m, e), generator=g)


@pytest.mark.parametrize("model", ["gp", "stand_in"])
def test_mo_acq(model):
    """HEBO/test/test_acq.py::test_mo_acq over a hebo_b200.GP and over a non-GP model."""
    X = torch.randn(10, 1)
    if model == "gp":
        m = GP(1, 0, 1, device="cuda", num_epochs=20)
        m.fit(X, None, X.clone())
    else:
        m = Stub(X.clone(), torch.full((10, 1), 0.04), torch.tensor([1e-3]))
    acq = MOMeanSigmaLCB(m, best_y=0.)
    v = acq(X, None)
    assert v.shape == (10, 3) and torch.isfinite(v).all()
    assert acq.num_obj == 2 and acq.num_constr == 1


def test_device_score_equals_eval_with_the_same_draws(monkeypatch):
    gp = fitted_gp()
    xc, xe = rows(3000, 3, 1, 4)
    acq = MOMeanSigmaLCB(gp, best_y=np.float32(-0.3), kappa=2.7)
    score = general_score(acq, seed=21)
    F, G = score(xc.to(dev), xe.to(dev), 6)
    # the Philox draws the score took: py of a zero posterior with noise_sd = 1
    zero = torch.zeros(3000, device=dev)
    xi = _mo_lcb_epilogue(zero, zero, 1.0, 0.0, 0.0, None, 21, 6)[0][:, 0].cpu().reshape(-1, 1)
    monkeypatch.setattr(torch, "randn", lambda shape: xi.reshape(shape).clone())
    v = acq.eval(xc, xe)
    assert same_bits(torch.cat([F, G[:, None]], 1).cpu().numpy(), v.numpy())


def test_device_score_does_not_synchronise():
    gp = fitted_gp()
    xc, xe = rows(512, 3, 1, 5)
    xc, xe = xc.to(dev), xe.to(dev, torch.int32)
    score = general_score(MOMeanSigmaLCB(gp, best_y=0.1), seed=1)
    score(xc, xe, 0)                                                         # workspaces allocated
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        F, G = score(xc, xe, 1)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert F.shape == (512, 2) and G.shape == (512,) and F.is_cuda and G.is_cuda


def test_device_score_after_a_failed_fit():
    gp = fitted_gp(e=0)
    gp._fit_failed = True                                                    # predicts N(y_mean, y_std^2)
    xc, _ = rows(300, 3, 0, 6)
    F, G = general_score(MOMeanSigmaLCB(gp, best_y=0.0), seed=2)(xc.to(dev), torch.zeros(300, 0, device=dev), 0)
    _, var = gp.predict(xc)
    assert same_bits(F[:, 1].cpu().numpy(), -np.sqrt(var.reshape(-1).numpy()))


def test_subclass_runs_through_its_own_eval():
    calls = []

    class Mine(MOMeanSigmaLCB):
        def eval(self, x, xe):
            calls.append((x.device.type, xe.dtype))
            v = super().eval(x, xe)
            v[:, 2] = -1.0                                                    # every row feasible
            return v
    gp = fitted_gp()
    xc, xe = rows(200, 3, 1, 7)
    F, G = general_score(Mine(gp, best_y=0.0), seed=3)(xc.to(dev), xe.to(dev), 0)
    assert calls == [("cpu", torch.int64)] and F.is_cuda and torch.equal(G, torch.zeros_like(G))


# ------------------------------------------------------------------ HEBO(acq_cls=...)
def branin_box(X):
    X = torch.as_tensor(X, dtype=torch.float64)
    x1, x2 = X[:, 0], X[:, 1]
    return ((x2 - 5.1 / (4 * np.pi ** 2) * x1 ** 2 + 5 / np.pi * x1 - 6) ** 2 + 10 * (1 - 1 / (8 * np.pi)) * torch.cos(x1) + 10).numpy()


def box_opt(acq_optimizer, **kw):
    np.random.seed(0)
    torch.manual_seed(0)
    opt = HEBO(torch.tensor([-5.0, 0.0]), torch.tensor([10.0, 15.0]), acq_cls=MOMeanSigmaLCB, acq_optimizer=acq_optimizer,
               scramble_seed=1, **kw)
    X = opt.quasi_sample(12)
    opt.observe(X, branin_box(X))
    return opt


def host_feasible_front(F, G):
    F, G = F.astype(np.float64), np.where(np.isfinite(G), G, np.inf)
    feas = np.flatnonzero(G <= 0)
    if feas.size == 0:
        return np.array([int(np.argmin(G))])
    Ff = F[feas]
    dom = [(np.all(Ff <= Ff[i], 1) & np.any(Ff < Ff[i], 1)).any() for i in range(feas.size)]
    return feas[~np.array(dom)]


def record_scores(monkeypatch, change_g=None):
    seen = []

    def wrapped(acq, seed=None):
        inner = general_score(acq, seed)

        def score(xc, xe, gen):
            F, G = inner(xc, xe, gen)
            if change_g is not None:
                G = change_g(G)
            seen.append((xc.clone(), F.clone(), G.clone()))
            return F, G
        return score
    monkeypatch.setattr(A, "general_score", wrapped)
    return seen


def test_sobol_suggestion_is_on_the_feasible_front(monkeypatch):
    opt = box_opt("sobol", n_candidates=3000)
    seen = record_scores(monkeypatch)
    rec = opt.suggest(1)
    (xc, F, G), = seen
    front = host_feasible_front(F.cpu().numpy(), G.cpu().numpy())
    assert (G[front] <= 0).all() and front.size > 1
    cand = xc.cpu()[front]
    assert ((cand == rec).all(1)).any()
    assert opt.last_timing["front"] == front.size


def test_sobol_without_a_feasible_candidate_takes_the_least_infeasible(monkeypatch):
    opt = box_opt("sobol", n_candidates=3000)
    # every row infeasible, the incumbent (row 0, an observation the duplicate check would drop) the most
    change = lambda G: torch.where(torch.arange(G.numel(), device=G.device) == 0, torch.full_like(G, 1e30), G.abs() + 1)
    seen = record_scores(monkeypatch, change)
    rec = opt.suggest(1)
    (xc, F, G), = seen
    assert (G > 0).all()
    assert torch.equal(rec, xc.cpu()[[int(np.argmin(G.cpu().numpy()))]])


def test_nsga2_suggestion_is_on_the_final_feasible_front(monkeypatch):
    runs = []

    class Recorded(E.DeviceNSGA2):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            runs.append(self)
    monkeypatch.setattr(E, "DeviceNSGA2", Recorded)
    opt = box_opt("nsga2", evo_pop=64, evo_iters=30)
    rec = opt.suggest(1)
    evo, = runs
    assert evo.k == 2 and evo.constrained
    front = host_feasible_front(evo.pop_F.cpu().numpy(), evo.pop_G.cpu().numpy())
    assert ((evo.pop_X.cpu()[front] == rec).all(1)).any()


SPACE = [{"name": "x0", "type": "num", "lb": -5, "ub": 10}, {"name": "x1", "type": "num", "lb": 0, "ub": 15},
         {"name": "c", "type": "cat", "categories": ["a", "b", "c"]}]


def branin_mixed(df: pd.DataFrame) -> np.ndarray:
    off = df["c"].map({"a": 0.0, "b": 3.0, "c": 7.0}).values
    return (branin_box(df[["x0", "x1"]].values.astype(np.float64)) + off).reshape(-1, 1)


@pytest.mark.parametrize("acq_optimizer", ["sobol", "nsga2"])
def test_branin_loop_with_a_categorical_column(acq_optimizer):
    np.random.seed(3)
    torch.manual_seed(3)
    space = DesignSpace().parse(SPACE)
    opt = HEBO(space, acq_cls=MOMeanSigmaLCB, acq_optimizer=acq_optimizer, n_candidates=2000, scramble_seed=5)
    for _ in range(20):
        rec = opt.suggest(1)
        assert rec.shape == (1, 3)
        assert (rec["x0"].between(-5, 10) & rec["x1"].between(0, 15) & rec["c"].isin(["a", "b", "c"])).all()
        opt.observe(rec, branin_mixed(rec))
    assert opt.y.shape == (20, 1) and np.isfinite(opt.y).all()


@pytest.mark.parametrize("acq_optimizer", ["sobol", "nsga2"])
def test_user_acquisition_runs_through_its_eval(acq_optimizer):
    calls = []

    class Mine(MOMeanSigmaLCB):
        def eval(self, x, xe):
            calls.append(x.shape[0])
            return super().eval(x, xe)
    np.random.seed(1)
    torch.manual_seed(1)
    opt = HEBO(DesignSpace().parse(SPACE), acq_cls=Mine, acq_optimizer=acq_optimizer, n_candidates=1000, evo_pop=32,
               evo_iters=5)
    for _ in range(6):
        rec = opt.suggest(1)
        opt.observe(rec, branin_mixed(rec))
    assert calls and set(calls) == ({1000} if acq_optimizer == "sobol" else {32})


@pytest.mark.parametrize("acq_optimizer", ["sobol", "nsga2"])
def test_default_is_mace_bit_for_bit(acq_optimizer):
    outs = []
    for kw in ({}, {"acq_cls": MACE}):
        np.random.seed(7)
        torch.manual_seed(7)
        opt = HEBO(DesignSpace().parse(SPACE), acq_optimizer=acq_optimizer, n_candidates=2000, scramble_seed=2, evo_iters=20, **kw)
        got = []
        for _ in range(8):
            rec = opt.suggest(3 if len(got) % 2 else 1)
            got.append(rec)
            opt.observe(rec, branin_mixed(rec))
        outs.append(pd.concat(got, ignore_index=True))
    pd.testing.assert_frame_equal(outs[0], outs[1], check_exact=True)


def test_too_many_objectives_are_rejected():
    class Wide(MOMeanSigmaLCB):
        num_obj = 9

    opt = box_opt("sobol", n_candidates=500)
    opt.acq_cls = Wide
    with pytest.raises(ValueError, match="at most 8"):
        opt.suggest(1)
