"""Single-objective GA and optimisers on the device: hb_ga_survive against ga_survive_host, hb_acq1_epilogue against the
acquisitions' CPU eval, DeviceNSGA2 with a one-column score, and the contracts of the reference's BO / NoMR_BO /
HEBO_VectorContextual tests (test/test_optimizer.py, test/test_nju.py)."""
import numpy as np
import pandas as pd
import pytest
import torch

from hebo_b200 import GP, LCB, AbsEtaDifference, BO, HEBO_VectorContextual, Mean, NoMR_BO, Sigma, _lib
from hebo_b200.acq import SingleObjectiveAcq, ga_score
from hebo_b200.evolution import DeviceNSGA2, ga_survive_host
from hebo_b200.space import DesignSpace

pytestmark = pytest.mark.gpu


def survival_case(P, D, seed):
    """Typed columns (real, integer, a fixed one), NaN / +-inf objectives, ties and duplicate children."""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-3, 3, (P, D)).astype(np.float32)
    C = rng.uniform(-3, 3, (P, D)).astype(np.float32)
    X[:, 1::3], C[:, 1::3] = np.rint(X[:, 1::3]), np.rint(C[:, 1::3])    # integer / choice columns
    if D > 2:
        X[:, 2], C[:, 2] = 0.25, 0.25                                      # a fixed column
    if D == 1:
        X, C = np.rint(X), np.rint(C)                                      # few distinct rows: many duplicates
    src = rng.integers(0, 2 * P, P)
    pick = rng.random(P) < 0.2
    allx = np.concatenate([X, C], 0)
    for i in np.flatnonzero(pick):                                         # copies of earlier merged rows
        j = src[i] % (P + i)
        C[i] = allx[j] if j < P else C[j - P]
    C[rng.random(P) < 0.05] += np.float32(1e-17)                           # within 1e-16: still duplicates
    F = np.round(rng.normal(size=P), 1).astype(np.float32)                 # ties
    FC = np.round(rng.normal(size=P), 1).astype(np.float32)
    for a in (F, FC):
        a[rng.random(P) < 0.05] = np.nan
        a[rng.random(P) < 0.05] = np.inf
        a[rng.random(P) < 0.05] = -np.inf
    return X, F, C, FC


def run_ga_survive(X, F, C, FC, d):
    lib = _lib.lib()
    dev = torch.device("cuda")
    P, D = X.shape
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    Xd, Fd, Cd, FCd = t(X), t(F), t(C), t(FC)
    Xn, Fn = torch.full((P, D), -7.0, device=dev), torch.full((P,), -7.0, device=dev)
    Xcn, Xen = torch.full((P, d), -7.0, device=dev), torch.full((P, D - d), -7, dtype=torch.int32, device=dev)
    ws_bytes = int(lib.hb_nsga2_workspace_bytes(P, D))
    ws = torch.full((ws_bytes,), 0xAB, dtype=torch.uint8, device=dev)
    pc = lambda x: _lib.ptr(x) if x.numel() else None
    _lib.check(lib.hb_ga_survive(_lib.ptr(Xd), _lib.ptr(Fd), _lib.ptr(Cd), _lib.ptr(FCd), P, D, d, _lib.ptr(Xn), _lib.ptr(Fn),
                                 pc(Xcn), pc(Xen), _lib.ptr(ws), ws_bytes, _lib.stream_ptr()), "hb_ga_survive")
    torch.cuda.synchronize()
    return Xn.cpu().numpy(), Fn.cpu().numpy(), Xcn.cpu().numpy(), Xen.cpu().numpy()


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


@pytest.mark.parametrize("D", [1, 5, 40])
@pytest.mark.parametrize("P", [1, 2, 7, 100, 256, 257, 1000, 4096, 16384])
def test_ga_survive_equals_host(P, D):
    X, F, C, FC = survival_case(P, D, 1000 * P + D)
    d = max(0, D - 2)                                                      # the last columns are categorical
    Xn, Fn, Xcn, Xen = run_ga_survive(X, F, C, FC, d)
    idx, f = ga_survive_host(X, F, C, FC)
    allx = np.concatenate([X, C], 0)
    assert np.array_equal(bits(Xn), bits(allx[idx]))
    assert np.array_equal(bits(Fn), bits(f[idx]))
    assert np.array_equal(bits(Xcn), bits(allx[idx][:, :d]))
    assert np.array_equal(Xen, np.rint(allx[idx][:, d:]).astype(np.int32))


def test_ga_survive_is_deterministic():
    X, F, C, FC = survival_case(16384, 5, 3)
    a, b = run_ga_survive(X, F, C, FC, 3), run_ga_survive(X, F, C, FC, 3)
    for u, v in zip(a, b):
        assert u.tobytes() == v.tobytes()


@pytest.fixture(scope="module")
def fitted_gp():
    torch.manual_seed(0)
    np.random.seed(0)
    rng = np.random.default_rng(0)
    n, d = 60, 3
    Xc = torch.FloatTensor(rng.uniform(-2, 2, (n, d)))
    Xe = torch.LongTensor(rng.integers(0, 3, (n, 1)))
    y = torch.FloatTensor(((Xc.numpy() - 0.5) ** 2).sum(1, keepdims=True) + Xe.numpy())
    gp = GP(d, 1, 1, num_uniqs=[3], warp=False, device="cuda")
    gp.fit(Xc, Xe, y)
    return gp


@pytest.mark.parametrize("cls,conf", [(LCB, {"kappa": 2.0}), (LCB, {"kappa": 0.6}), (Mean, {}), (Sigma, {}),
                                      (AbsEtaDifference, {}), (AbsEtaDifference, {"eta": 0.5, "kappa": 1.3})])
def test_acq1_epilogue_equals_cpu_eval(fitted_gp, cls, conf):
    rng = np.random.default_rng(1)
    m = 3000
    xc = torch.FloatTensor(rng.uniform(-3, 3, (m, 3)))
    xc[:50] = torch.FloatTensor(rng.uniform(-2, 2, (50, 3)))
    xe = torch.LongTensor(rng.integers(0, 3, (m, 1)))
    acq = cls(fitted_gp, **conf)
    ref = acq.eval(xc, xe).reshape(-1)
    got = ga_score(acq)(xc.cuda(), xe.cuda().int(), 0).cpu()
    # bit for bit against the same expression in IEEE fp32 (numpy: correctly rounded sqrt, products, differences) on the
    # same mu / var; torch's CPU sqrt goes through MKL VML (< 1 ulp, not always correctly rounded), so the CPU eval itself
    # may differ from that by one ulp in a few rows
    mu, var = (t.reshape(-1).numpy() for t in fitted_gp.predict(xc, xe))
    k, e, s = np.float32(getattr(acq, "kappa", 0.0)), np.float32(getattr(acq, "eta", 0.0)), np.sqrt(var)
    ieee = {LCB: lambda: mu - k * s, Mean: lambda: mu, Sigma: lambda: np.float32(-1) * s,
            AbsEtaDifference: lambda: np.abs(mu - e) - k * s}[cls]()
    assert ieee.dtype == np.float32
    assert np.array_equal(got.numpy().view(np.uint32), ieee.view(np.uint32))
    ulp = np.abs(got.numpy().view(np.int32).astype(np.int64) - ref.numpy().view(np.int32).astype(np.int64))
    assert ulp.max() <= (0 if cls is Mean else 1)


def test_user_acquisition_scores_through_its_eval(fitted_gp):
    class Custom(SingleObjectiveAcq):
        def eval(self, x, xe):
            assert not x.is_cuda and xe.dtype == torch.int64
            py, ps2 = self.model.predict(x, xe)
            return py + 0.5 * ps2
    acq = Custom(fitted_gp)
    xc, xe = torch.rand(64, 3) * 4 - 2, torch.randint(0, 3, (64, 1))
    got = ga_score(acq)(xc.cuda(), xe.cuda().int(), 0)
    assert got.is_cuda and torch.equal(got.cpu(), acq.eval(xc, xe).reshape(-1))


def ga(fitted_gp, iters, seed=5, init=None):
    kinds = ["real", "real", "real", "choice"]
    evo = DeviceNSGA2(kinds, [-3, -3, -3, 0], [3, 3, 3, 2], 3, ga_score(LCB(fitted_gp, kappa=2.0)), pop=64, iters=iters,
                      seed=seed, fixed={2: 0.75})
    return evo, evo.optimize(initial_suggest=init)


def test_ga_properties(fitted_gp):
    init = np.array([[1.0, -1.0, 0.75, 2.0]], np.float32)
    best, f_init = [], None
    for iters in range(1, 13):                       # the Philox streams are keyed by (seed, generation): run k is a prefix
        evo, (xc, xe, f) = ga(fitted_gp, iters, init=init)
        F = evo.pop_F.cpu()
        fin = torch.where(torch.isfinite(F), F, torch.full_like(F, float("inf")))
        assert xc.shape == (1, 3) and xe.shape == (1, 1) and f.shape == (1, 1)
        assert float(f) == float(fin.min())          # the returned row is the minimum of the final population
        k = int(torch.argmin(fin))
        assert torch.equal(xc.cpu()[0], evo.pop_X.cpu()[k, :3]) and bool((xc[:, 2] == 0.75).all())
        if iters > 1:
            assert k == 0                            # survivors are written best first
        else:
            f_init = float(F[0])                     # row 0 of the initial population is initial_suggest
            assert torch.equal(evo.pop_X.cpu()[0], torch.from_numpy(init[0]))
        best.append(float(f))
    assert all(b <= a for a, b in zip(best, best[1:])), best
    assert best[-1] <= f_init


def test_ga_one_column_argument_checks(fitted_gp):
    score = ga_score(LCB(fitted_gp))
    evo = DeviceNSGA2(["real"] * 3 + ["choice"], [-1] * 4, [1, 1, 1, 2], 3, lambda xc, xe, g: (score(xc, xe, g), score(xc, xe, g)),
                      pop=8, iters=2, constrained=True)
    with pytest.raises(ValueError):
        evo.optimize()
    evo = DeviceNSGA2(["real"] * 3 + ["choice"], [-1] * 4, [1, 1, 1, 2], 3, lambda xc, xe, g: score(xc, xe, g).reshape(-1, 1).repeat(1, 2),
                      pop=8, iters=2)
    with pytest.raises(ValueError):
        evo.optimize()


def test_ga_finds_the_bowl_minimum():
    # typed 6-D space: 3 real, 1 integer, 1 choice and one fixed real column; the bowl's minimum is known
    kinds = ["real", "real", "real", "int", "real", "choice"]
    lb, ub = [-5, -5, -5, -10, -1, 0], [5, 5, 5, 10, 1, 4]
    opt = torch.tensor([1.3, -2.2, 0.7, 3.0], device="cuda")

    def bowl(xc, xe, gen):
        return ((xc[:, :4] - opt) ** 2).sum(1) + (xc[:, 4] - 0.2) ** 2 + (xe[:, 0] != 2).float()
    evo = DeviceNSGA2(kinds, lb, ub, 5, bowl, pop=100, iters=100, seed=11, fixed={4: -0.5})
    xc, xe, f = evo.optimize()
    xc, xe = xc.cpu()[0], xe.cpu()[0]
    # tolerance: the real coordinates within 0.05 of the optimum, the integer and choice columns exact
    assert float(xc[4]) == -0.5 and float(xc[3]) == 3.0 and int(xe[0]) == 2
    assert float((xc[:3] - opt[:3].cpu()).abs().max()) < 0.05
    assert float(f) < 0.49 + 3 * 0.05 ** 2               # 0.49 = (-0.5 - 0.2)^2 from the fixed column


# ---- the reference's optimiser tests, with the 'gp' model
def test_opt_bo_gp():                                      # test_optimizer.py::test_opt[bo-gp]
    space = DesignSpace().parse([{"name": "x0", "type": "num", "lb": -3, "ub": 7},
                                 {"name": "x1", "type": "cat", "categories": ["a", "b", "c"]}])
    opt = BO(space, rand_sample=8, model_name="gp")
    for _ in range(11):
        rec = opt.suggest(n_suggestions=1)
        assert rec.shape == (1, 2) and -3 <= float(rec["x0"].iloc[0]) <= 7 and rec["x1"].iloc[0] in ("a", "b", "c")
        opt.observe(rec, rec["x0"].values.astype(float).reshape(-1, 1) ** 2)
    assert opt.y.shape == (11, 1) and opt.last_timing["acq_ms"] > 0


def test_contextual_opt_bo():                              # test_optimizer.py::test_contextual_opt[bo]
    space = DesignSpace().parse([{"name": "x0", "type": "int", "lb": -20, "ub": 20},
                                 {"name": "x1", "type": "int", "lb": -20, "ub": 20}])
    opt = BO(space, rand_sample=2, model_name="gp")
    for _ in range(4):
        context = np.random.randint(40) - 20
        rec = opt.suggest(n_suggestions=1, fix_input={"x0": context})
        assert (rec["x0"] == context).all()
        opt.observe(rec, (rec[["x0", "x1"]].values ** 2).sum(axis=1, keepdims=True))


def test_best_xy_bo():                                     # test_optimizer.py::test_best_xy[bo]
    space = DesignSpace().parse([{"name": "x", "type": "num", "lb": 0, "ub": 1}])
    opt = BO(space, rand_sample=100)
    with pytest.raises(RuntimeError):
        opt.best_x
    with pytest.raises(RuntimeError):
        opt.best_y
    rec = opt.suggest()
    opt.observe(rec, rec["x"].values.reshape(-1, 1))
    assert isinstance(opt.best_x, pd.DataFrame)
    assert isinstance(opt.best_y, float)


def test_nju_opt():                                        # test_nju.py::test_opt, both runs
    space = DesignSpace().parse([{"name": "x0", "type": "num", "lb": -3, "ub": 7},
                                 {"name": "x1", "type": "cat", "categories": ["a", "b", "c"]}])
    obj = lambda x: x["x0"].values.astype(float).reshape(-1, 1) ** 2
    for opt in (NoMR_BO(space), NoMR_BO(space, opt2=BO(space, acq_cls=AbsEtaDifference, acq_conf={"eta": 0.5}))):
        for _ in range(11):
            rec = opt.suggest()
            opt.observe(rec, obj(rec))
        assert opt.opt1.y.shape == (11, 1) and opt.opt2.y.shape == (11, 1)
        assert opt.best_y == float(opt.opt1.y.min())
        assert opt.opt2.last_timing                    # stage two ran its GA


def test_contextual_vector_gp():                           # test_optimizer.py::test_contextual_vector, 'gp' for 'rf'
    space = DesignSpace().parse([{"name": "x", "type": "num", "lb": -1, "ub": 1},
                                 {"name": "c1", "type": "num", "lb": -1, "ub": 1},
                                 {"name": "c2", "type": "int", "lb": -3, "ub": 3},
                                 {"name": "c3", "type": "cat", "categories": ["a", "b", "c"]}])
    context_dict = {"context1": {"c1": 0.5, "c2": 1, "c3": "a"}, "context2": {"c1": 0.3, "c2": -1, "c3": "b"}}
    opt = HEBO_VectorContextual(space, context_dict, rand_sample=10, model_name="gp")
    for i in range(11):
        opt.context = ["context1", "context2"][i % 2]
        rec = opt.suggest(1)
        for k, v in context_dict[opt.context].items():
            assert (rec[k] == v).all() if k != "c1" else np.allclose(rec[k].values.astype(float), v)
        opt.observe(rec, (rec[["x", "c1", "c2"]].values.astype(float) ** 2).sum(axis=1, keepdims=True))
