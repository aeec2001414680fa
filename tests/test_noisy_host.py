"""NoisyOpt's host logic (hebo_b200/noisy.py) with a stub model and a stub GA, NoisyAcq, and the argument checks of
hb_sample_y_batch, CPU only."""
import ctypes

import numpy as np
import pandas as pd
import pytest
import torch

from hebo_b200 import NoisyAcq, NoisyOpt, _lib
from hebo_b200 import noisy as noisy_mod
from hebo_b200.space import DesignSpace
from hebo_b200.suggest import HEBO

SPACE = [{"name": "x0", "type": "num", "lb": -3, "ub": 7}, {"name": "c", "type": "cat", "categories": ["a", "b", "c"]}]


@pytest.fixture(scope="module")
def lib():
    if not _lib.available():
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


def test_sample_y_batch_rejects_bad_arguments(lib):
    bad = _lib.HB_ERR_INVALID
    p = ctypes.c_void_p(16)          # never dereferenced: every call below must fail its argument checks first
    n, d = 300, 2
    need = int(lib.hb_sample_workspace_bytes(n, d, None, 100))
    assert need > 0

    def call(m=100, ws_bytes=need, **null):
        a = dict(Xs=p, x_mul=p, x_add=p, Zt=p, alpha=p, Linv=p, hyp=p, f=p, jitter=p, status=p, ws=p)
        a.update(null)
        return lib.hb_sample_y_batch(a["Xs"], None, m, n, d, None, None, None, a["x_mul"], a["x_add"], a["Zt"], a["alpha"],
                                     a["Linv"], a["hyp"], 0, 0.0, 1.0, 0, None, 1, 2, a["f"], a["jitter"], a["status"], a["ws"],
                                     ws_bytes, None)
    for name in ("Xs", "x_mul", "x_add", "Zt", "alpha", "Linv", "hyp", "f", "jitter", "status", "ws"):
        assert call(**{name: None}) == bad, name
    for m in (0, -1, 257):
        assert call(m=m, ws_bytes=1 << 40) == bad, m
    assert call(ws_bytes=need - 1) == bad                                  # short workspace
    assert call(ws_bytes=-1) == bad                                        # negative: not a huge unsigned size
    need256 = int(lib.hb_sample_workspace_bytes(n, d, None, 256))
    assert need256 >= need
    u, e = (ctypes.c_int32 * 1)(3), (ctypes.c_int32 * 1)(2)
    spec = _lib.ModelSpec(1, 1, u, e)                                      # a categorical column needs Xe / meta / tables
    assert lib.hb_sample_y_batch(p, None, 4, n, d, ctypes.byref(spec), p, p, p, p, p, p, p, p, 0, 0.0, 1.0, 0, None, 1, 2, p, p,
                                 p, p, 1 << 40, None) == bad


class StubModel:
    num_out = 1

    def __init__(self, *a, **k):
        self.fitted = None

    def fit(self, Xc, Xe, y):
        self.fitted = (Xc, Xe, y)

    def predict(self, Xc, Xe):
        mu = Xc[:, :1].double().clone().float()                # argmin mu = the smallest x0
        var = (Xe[:, :1].float() + 1.0) ** 2                    # argmax sigma = the largest category
        return mu, var

    def sample_y(self, Xc, Xe, n_samples=1):
        return torch.arange(Xc.shape[0], dtype=torch.float32).reshape(1, -1, 1) * 2.0


class StubGA:
    """Returns a fixed final population; records how it was built and called."""
    pop_c = None
    pop_e = None
    calls = []

    def __init__(self, kinds, lb, ub, d, score, pop, iters, seed, device):
        StubGA.calls.append(dict(kinds=kinds, d=d, pop=pop, iters=iters, score=score))

    def optimize(self, initial_suggest=None, return_pop=False):
        StubGA.calls[-1].update(init=initial_suggest, return_pop=return_pop)
        c, e = StubGA.pop_c, StubGA.pop_e
        return c.clone(), e.int().clone(), torch.zeros(c.shape[0], 1)


@pytest.fixture
def stubs(monkeypatch):
    monkeypatch.setattr(noisy_mod, "GP", StubModel)
    monkeypatch.setattr(noisy_mod, "DeviceNSGA2", StubGA)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    StubGA.calls = []
    return StubGA


def observed(opt):
    X = pd.DataFrame({"x0": [0.5, 1.5, -2.0], "c": ["a", "b", "c"]})
    opt.observe(X, np.array([[3.0], [1.0], [2.0]]))
    return X


def test_noisy_acq_counts_and_eval():
    acq = NoisyAcq(StubModel(), 1, 0)
    assert acq.num_obj == 1 and acq.num_constr == 0
    acq2 = NoisyAcq(StubModel(), 2, 1)
    assert acq2.num_obj == 2 and acq2.num_constr == 1
    v = acq(torch.zeros(4, 1), torch.zeros(4, 1, dtype=torch.long))      # model.sample_y(x, xe).reshape(-1, 1)
    assert v.shape == (4, 1) and v.reshape(-1).tolist() == [0.0, 2.0, 4.0, 6.0]
    with pytest.raises(RuntimeError):
        acq2(torch.zeros(4, 1), torch.zeros(4, 1, dtype=torch.long))     # 4 values do not reshape to 3 columns


def test_noisy_start_up_design_and_arguments():
    space = DesignSpace().parse(SPACE)
    opt = NoisyOpt(space, scramble_seed=4)
    assert opt.rand_sample == 3 and NoisyOpt(space, rand_sample=8).rand_sample == 8
    assert NoisyOpt.support_parallel_opt and NoisyOpt.support_combinatorial and NoisyOpt.support_contextual
    rec = opt.suggest(5)
    ref = HEBO(space, scramble_seed=4).quasi_sample(5)                      # the same scrambled Sobol design
    pd.testing.assert_frame_equal(rec, ref)
    with pytest.raises(AssertionError):
        opt.suggest(1, fix_input={"c": "a"})
    with pytest.raises(ValueError):
        NoisyOpt(space, evo_pop=257)
    with pytest.raises(NotImplementedError):
        NoisyOpt(space, model_name="rf")


def test_noisy_suggest_drops_observed_rows_and_fills_the_slots(stubs):
    space = DesignSpace().parse(SPACE)
    opt = NoisyOpt(space, rand_sample=3, scramble_seed=1)
    observed(opt)
    # final population: row 1 repeats observation 1, row 3 repeats row 0; x0 = -2.5 has the smallest mu, category 2 the
    # largest sigma
    stubs.pop_c = torch.tensor([[4.0], [1.5], [-2.5], [4.0], [6.0], [0.0]])
    stubs.pop_e = torch.tensor([[0], [1], [0], [0], [2], [1]])
    np.random.seed(0)
    rec = opt.suggest(3)
    call = stubs.calls[-1]
    assert call["return_pop"] is True and call["pop"] == 100 and call["iters"] == 100
    assert call["init"].tolist() == [[1.5, 1.0]]                          # best_x: the argmin-y observation
    assert opt.model.fitted[2].reshape(-1).tolist() == [3.0, 1.0, 2.0]     # the raw y, no power transform
    assert rec.shape == (3, 2)
    pairs = list(zip(rec["x0"].tolist(), rec["c"].tolist()))
    assert (1.5, "b") not in pairs and len(set(pairs)) == 3                # observation and duplicate dropped
    kept = [(4.0, "a"), (-2.5, "a"), (6.0, "c"), (0.0, "b")]              # survival order, after check_unique
    np.random.seed(0)
    np.random.randint(0, 2 ** 31 - 1)                                      # the GA's seed
    sel = np.random.choice(4, 3, replace=False).tolist()
    if 2 not in sel:
        sel[0] = 2                                                         # argmax sigma into slot 0
    if 1 not in sel:
        sel[1] = 1                                                         # argmin mu into slot 1
    assert pairs == [kept[i] for i in sel]
    for seed in range(20):                                                 # q > 2: argmin mu is always picked
        np.random.seed(seed)
        r = opt.suggest(3)
        assert (-2.5, "a") in list(zip(r["x0"].tolist(), r["c"].tolist()))


def test_noisy_suggest_q_le_2_is_a_plain_random_pick(stubs):
    space = DesignSpace().parse(SPACE)
    opt = NoisyOpt(space, rand_sample=3, scramble_seed=1)
    observed(opt)
    stubs.pop_c = torch.tensor([[4.0], [1.0], [2.0], [3.0]])
    stubs.pop_e = torch.tensor([[0], [0], [0], [0]])
    np.random.seed(7)
    rec = opt.suggest(2)
    np.random.seed(7)
    np.random.randint(0, 2 ** 31 - 1)
    pick = np.random.choice(4, 2, replace=False).tolist()
    assert rec["x0"].tolist() == [[4.0, 1.0, 2.0, 3.0][i] for i in pick]


def test_noisy_suggest_tops_up_with_sobol(stubs):
    space = DesignSpace().parse(SPACE)
    opt = NoisyOpt(space, rand_sample=3, scramble_seed=2)
    observed(opt)
    stubs.pop_c = torch.tensor([[0.5], [0.5], [1.5]])                      # every row repeats an observation
    stubs.pop_e = torch.tensor([[0], [0], [1]])
    np.random.seed(1)
    rec = opt.suggest(4)
    assert rec.shape == (4, 2)
    obs = {(0.5, "a"), (1.5, "b"), (-2.0, "c")}
    pairs = list(zip(rec["x0"].tolist(), rec["c"].tolist()))
    assert not obs & set(pairs) and len(set(pairs)) == 4
    assert ((rec["x0"] >= -3) & (rec["x0"] <= 7)).all()
