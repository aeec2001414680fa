"""Single-objective optimisers (hebo_b200/bo.py), the GA survival rule and the new C-ABI argument checks, CPU only."""
import ctypes

import numpy as np
import pandas as pd
import pytest
import torch

from hebo_b200 import _lib
from hebo_b200 import bo as bo_mod
from hebo_b200.bo import BO, HEBO_VectorContextual, NoMR_BO
from hebo_b200.evolution import ga_survive_host
from hebo_b200.space import DesignSpace

INF = np.float32(np.inf)


def brute_force_survivors(X, F, C, FC):
    """The GA survival spelled out with Python scalars: sanitise, duplicates, then sort by (f, merged index)."""
    P = X.shape[0]
    rows = list(np.concatenate([X, C], 0).astype(np.float32))
    f = []
    for v in list(np.asarray(F, np.float32).reshape(-1)) + list(np.asarray(FC, np.float32).reshape(-1)):
        f.append(np.float32(v) if np.isfinite(v) else INF)
    for i in range(P, 2 * P):
        for j in range(i):
            if all(abs(np.float32(a) - np.float32(b)) <= np.float32(1e-16) for a, b in zip(rows[i], rows[j])):
                f[i] = INF
                break
    order = sorted(range(2 * P), key=lambda i: (float(f[i]), i))
    return np.asarray(order[:P]), np.asarray(f, np.float32)


def case(P, D, seed, special=True):
    rng = np.random.default_rng(seed)
    X = rng.integers(-2, 3, (P, D)).astype(np.float32)
    C = rng.integers(-2, 3, (P, D)).astype(np.float32)
    F = rng.integers(-3, 4, P).astype(np.float32)        # many ties
    FC = rng.integers(-3, 4, P).astype(np.float32)
    if special:
        F[rng.random(P) < 0.1] = np.nan
        F[rng.random(P) < 0.1] = np.inf
        FC[rng.random(P) < 0.1] = -np.inf
        FC[rng.random(P) < 0.1] = np.nan
        C[0] = X[P // 2]                                  # duplicate of a population row
        if P > 2:
            C[1] = C[0]                                   # duplicate of a duplicate
            C[2] = X[0] + np.float32(1e-17)               # within 1e-16 (rounds onto X[0] where |X| >= 1e-16)
            X[1, :] = 0.0
            C[P - 1] = np.float32(5e-17)                  # near zero: within 1e-16 of the zero row
            F[1] = -0.0
            FC[P - 1] = 0.0
    return X, F, C, FC


@pytest.mark.parametrize("P,D,seed", [(1, 1, 0), (2, 1, 1), (7, 3, 2), (40, 5, 3), (100, 2, 4), (300, 4, 5)])
def test_ga_survive_host_equals_brute_force(P, D, seed):
    X, F, C, FC = case(P, D, seed)
    idx, f = ga_survive_host(X, F, C, FC)
    ridx, rf = brute_force_survivors(X, F, C, FC)
    assert np.array_equal(idx, ridx)
    assert np.array_equal(f.view(np.uint32), rf.view(np.uint32))
    assert np.all(f[idx][:-1] <= f[idx][1:])              # best first


def test_ga_survive_host_marks_duplicates():
    X = np.array([[0.0, 1.0], [2.0, 3.0]], np.float32)
    C = np.array([[2.0, 3.0], [2.0, 3.0]], np.float32)
    F, FC = np.array([5.0, 6.0], np.float32), np.array([-1.0, -2.0], np.float32)
    idx, f = ga_survive_host(X, F, C, FC)
    assert np.isinf(f[2]) and np.isinf(f[3])              # child 0 equals X[1], child 1 equals child 0
    assert idx.tolist() == [0, 1]
    C2 = np.array([[5e-17, 1.0], [1e-15, 1.0]], np.float32)
    idx, f = ga_survive_host(X, F, C2, FC)
    assert np.isinf(f[2]) and f[3] == -2.0                # 5e-17 is within 1e-16 of 0, 1e-15 is not
    assert idx.tolist() == [3, 0]


@pytest.fixture(scope="module")
def lib():
    if not _lib.available():
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


def test_new_entries_reject_bad_arguments(lib):
    bad = _lib.HB_ERR_INVALID
    p = ctypes.c_void_p(16)          # never dereferenced: every call below must fail its argument checks first
    # NULL pointers
    assert lib.hb_ga_survive(None, p, p, p, 4, 2, 2, p, p, p, None, None, 0, None) == bad
    assert lib.hb_ga_survive(p, p, p, p, 4, 2, 2, None, p, p, None, None, 0, None) == bad
    assert lib.hb_ga_survive(p, p, p, p, 4, 2, 1, p, p, p, None, None, 0, None) == bad          # Xe_next missing, e = 1
    assert lib.hb_acq1_epilogue(None, p, 4, 0, 2.0, 0.0, p, None) == bad
    assert lib.hb_acq1_epilogue(p, p, 4, 0, 2.0, 0.0, None, None) == bad
    # sizes, mode, workspace
    for pop in (0, -1, 16385):
        assert lib.hb_ga_survive(p, p, p, p, pop, 2, 2, p, p, p, None, None, 0, None) == bad
    assert lib.hb_ga_survive(p, p, p, p, 4, 0, 0, p, p, None, None, None, 0, None) == bad
    assert lib.hb_ga_survive(p, p, p, p, 4, 2, 3, p, p, p, p, None, 0, None) == bad
    assert lib.hb_ga_survive(p, p, p, p, 257, 2, 2, p, p, p, None, None, 0, None) == bad         # pop > 256 needs ws
    need = int(lib.hb_nsga2_workspace_bytes(257, 2))
    assert lib.hb_ga_survive(p, p, p, p, 257, 2, 2, p, p, p, None, p, need - 1, None) == bad
    for m in (0, -3):
        assert lib.hb_acq1_epilogue(p, p, m, 0, 2.0, 0.0, p, None) == bad
    for mode in (-1, 4):
        assert lib.hb_acq1_epilogue(p, p, 4, mode, 2.0, 0.0, p, None) == bad


SPACE = [{"name": "x0", "type": "num", "lb": -3, "ub": 7}, {"name": "n", "type": "int", "lb": -5, "ub": 5},
         {"name": "c", "type": "cat", "categories": ["a", "b", "c"]}]


def test_bo_start_up_design():
    space = DesignSpace().parse(SPACE)
    assert BO(space).rand_sample == 4                    # 1 + num_paras
    assert BO(space, rand_sample=1).rand_sample == 2     # max(2, rand_sample)
    assert BO(space, rand_sample=9).rand_sample == 9
    opt = BO(space)
    np.random.seed(3)
    rec = opt.suggest()
    np.random.seed(3)
    ref = space.sample(1)                                # uniform, numpy's global RNG
    pd.testing.assert_frame_equal(rec, ref)
    rec = opt.suggest(fix_input={"n": 2, "c": "b"})
    assert rec["n"].tolist() == [2] and rec["c"].tolist() == ["b"]
    with pytest.raises(AssertionError):
        opt.suggest(2)
    with pytest.raises(NotImplementedError):
        BO(space, model_name="rf")


def test_bo_observe_and_best():
    space = DesignSpace().parse(SPACE)
    opt = BO(space)
    with pytest.raises(RuntimeError):
        opt.best_x
    with pytest.raises(RuntimeError):
        opt.best_y
    X = pd.DataFrame({"x0": [0.5, 1.5, 2.5, 3.5], "n": [1, 2, 3, 4], "c": ["a", "b", "c", "a"]})
    opt.observe(X, np.array([[3.0], [np.nan], [-1.0], [np.inf]]))
    assert opt.y.reshape(-1).tolist() == [3.0, -1.0]
    assert opt.best_y == -1.0
    assert opt.best_x.iloc[0].tolist() == [2.5, 3, "c"]
    with pytest.raises(AssertionError):
        opt.observe(X, np.zeros((4, 2)))


def test_bo_rejects_multi_objective_acquisitions(monkeypatch):
    class StubGP:
        def __init__(self, *a, **k):
            self.num_out = 1

        def fit(self, *a):
            pass

    class ThreeObjectives:
        num_obj, num_constr = 3, 0

        def __init__(self, model, **conf):
            pass

    class Constrained(ThreeObjectives):
        num_obj, num_constr = 1, 1
    monkeypatch.setattr(bo_mod, "GP", StubGP)
    space = DesignSpace().parse(SPACE)
    for cls in (ThreeObjectives, Constrained):
        opt = BO(space, rand_sample=2, acq_cls=cls, acq_conf={})
        opt.observe(pd.DataFrame({"x0": [0.5, 1.5], "n": [1, 2], "c": ["a", "b"]}), np.array([[1.0], [2.0]]))
        with pytest.raises(NotImplementedError):
            opt.suggest()


class Stage:
    def __init__(self, name, ys=()):
        self.name, self.y, self.seen = name, np.asarray(ys, float).reshape(-1, 1), []

    def suggest(self, n, fix_input=None):
        return (self.name, n, fix_input)

    def observe(self, X, y):
        self.seen.append((X, y))
        self.y = np.vstack([self.y, np.asarray(y, float).reshape(-1, 1)])

    @property
    def best_y(self):
        return float(self.y.min())

    @property
    def best_x(self):
        return self.name


def test_nomr_stage_switching():
    space = DesignSpace().parse(SPACE)
    one, two = Stage("one"), Stage("two")
    opt = NoMR_BO(space, eta=0.5, opt1=one, opt2=two)
    assert opt.suggest()[0] == "one"                      # no data
    opt.observe("X0", [[2.0]])
    assert opt.suggest(1, {"c": "a"}) == ("one", 1, {"c": "a"})   # best y above eta
    opt.observe("X1", [[0.5]])
    assert opt.suggest()[0] == "two"                      # best y at eta
    opt.observe("X2", [[-1.0]])
    assert opt.suggest()[0] == "two"                      # below eta
    assert [x for x, _ in one.seen] == [x for x, _ in two.seen] == ["X0", "X1", "X2"]
    with pytest.raises(AssertionError):
        opt.suggest(2)
    # eta = None is +inf: everything after the first observation goes to stage two
    one, two = Stage("one"), Stage("two")
    opt = NoMR_BO(space, opt1=one, opt2=two)
    assert opt.eta == np.inf
    assert opt.suggest()[0] == "one"
    opt.observe("X0", [[1e30]])
    assert opt.suggest()[0] == "two"


def test_nomr_best_of_the_two_stages():
    space = DesignSpace().parse(SPACE)
    opt = NoMR_BO(space, opt1=Stage("one", [3.0, 1.0]), opt2=Stage("two", [2.0]))
    assert opt.best_y == 1.0 and opt.best_x == "one"
    opt = NoMR_BO(space, opt1=Stage("one", [3.0]), opt2=Stage("two", [2.0]))
    assert opt.best_y == 2.0 and opt.best_x == "two"


def test_nomr_default_stages():
    space = DesignSpace().parse(SPACE)
    opt = NoMR_BO(space)
    assert type(opt.opt2) is BO and opt.opt2.acq_conf == {"kappa": 0.6}
    assert type(opt.opt1).__name__ == "HEBO"


def test_vector_contextual_forwards_the_context():
    space = DesignSpace().parse(SPACE)
    ctx = {"one": {"n": 1, "c": "a"}, "two": {"x0": 0.5}}
    opt = HEBO_VectorContextual(space, ctx, rand_sample=3)
    calls = []
    opt.hebo.suggest = lambda n, fix_input=None: calls.append((n, fix_input)) or "rec"
    opt.context = "one"
    assert opt.suggest(4) == "rec"
    opt.context = "two"
    opt.suggest(1)
    assert calls == [(4, {"n": 1, "c": "a"}), (1, {"x0": 0.5})]
    with pytest.raises(NotImplementedError):
        opt.best_x
    with pytest.raises(NotImplementedError):
        opt.best_y
    with pytest.raises(NotImplementedError):
        HEBO_VectorContextual(space, ctx, model_name="rf")


def test_vector_contextual_rejects_unknown_keys():
    space = DesignSpace().parse(SPACE)
    opt = HEBO_VectorContextual(space, {"bad": {"x0": 0.5, "nope": 1}})
    opt.hebo.suggest = lambda n, fix_input=None: "rec"
    opt.context = "bad"
    with pytest.raises(AssertionError):
        opt.suggest(1)
    with pytest.raises(KeyError):
        opt.context = "missing"
        opt.suggest(1)


def test_vector_contextual_random_design_keeps_the_context():
    space = DesignSpace().parse(SPACE)
    opt = HEBO_VectorContextual(space, {"k": {"n": -2, "c": "c"}}, rand_sample=50)
    opt.context = "k"
    rec = opt.suggest(5)
    assert (rec["n"] == -2).all() and (rec["c"] == "c").all()
    assert torch.is_tensor(opt.hebo.Xc)
