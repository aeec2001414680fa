"""hb_de_fit_batch / hb_de_predict_batch and the optimisers that run the deep ensemble through them: the batched fit
against separate hb_de_fit calls and the batched predict against hb_de_predict, bit for bit; the sample_y draws against
torch's expression and the restated Philox stream; MultiTaskModel(base_model_name='deep_ensemble') against its models
fitted one after another; the device scorers against the epilogues run on predict; and the reference's test_opt loop
(HEBO/test/test_optimizer.py) for GeneralBO, NoisyOpt, HEBO_Embedding and HEBO_VectorContextual over the ensemble."""
import ctypes as C

import numpy as np
import pandas as pd
import pytest
import torch

from hebo_b200 import DeepEnsemble, MOMeanSigmaLCB, _lib
from hebo_b200.acq import GeneralAcq, NoisyAcq, _general_epilogue, _mo_lcb_epilogue, _noise_sd, _best_y, ga_score, general_score
from hebo_b200.bo import HEBO_VectorContextual
from hebo_b200.embedding import HEBO_Embedding
from hebo_b200.ensemble import EnsembleBatch, init_params
from hebo_b200.general import GeneralBO
from hebo_b200.gp import MultiTaskModel
from hebo_b200.noisy import NoisyOpt
from hebo_b200.space import DesignSpace
from oracle import rng_oracle as R
from tests.test_gpu_ensemble import INPUTS, VARIANTS, VID

pytestmark = pytest.mark.gpu
DEV = "cuda"
# rows per ensemble with batch_size 16: below the batch (5, 9, 12), not a multiple of it (37, 20, 50, 33), a multiple (64)
NS = [37, 5, 20, 64, 9, 50, 33, 12]


def _model(v, **kw):
    noise, prior, inp, O, L = v
    dc, uniqs, trans = INPUTS[inp]
    conf = dict(num_ensembles=2, num_layers=L, num_hiddens=24, output_noise=noise, rand_prior=prior, enum_trans=trans,
                num_uniqs=uniqs, num_epochs=3, batch_size=16)
    conf.update(kw)
    return DeepEnsemble(dc, len(uniqs), O, **conf)


def _rows(m, n, seed):
    """Scaled training rows of one ensemble: Xc in [-1, 1], Xe in range, y standard-ish with masked entries."""
    g = torch.Generator().manual_seed(seed)
    Xc = torch.rand(n, m.num_cont, generator=g) * 2 - 1
    Xe = torch.stack([torch.randint(0, u, (n,), generator=g) for u in m.num_uniqs], 1) if m.num_enum else torch.zeros(n, 0)
    y = torch.randn(n, m.num_out, generator=g)
    if m.num_out == 2 and n > 3:
        y[1, 0] = float("nan")
        y[3, 1] = float("nan")
    return Xc, Xe.int(), y


def _fit_one(m, xc, xe, y, params, seed):
    lib, E, T = _lib.lib(), m.num_ensembles, int(m.num_epochs)
    need = int(lib.hb_de_fit_workspace_bytes(C.byref(m._spec), E))
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    losses = torch.empty(E, T, device=DEV)
    _lib.check(lib.hb_de_fit(_lib.ptr(xc) if m.num_cont else None, _lib.ptr(xe) if m.num_enum else None, _lib.ptr(y), y.shape[0],
                             C.byref(m._spec), E, _lib.ptr(params), float(m.lr), float(m.l1), int(m.batch_size), T, None, seed,
                             _lib.ptr(losses), _lib.ptr(ws), need, _lib.stream_ptr()), "hb_de_fit")
    return ws, losses


def _fit_batch(m, xc, xe, y, off, params, seeds):
    lib, E, T, B = _lib.lib(), m.num_ensembles, int(m.num_epochs), len(seeds)
    need = int(lib.hb_de_fit_workspace_bytes(C.byref(m._spec), E))
    ws = torch.empty(B * need, dtype=torch.uint8, device=DEV)
    losses = torch.empty(B, E, T, device=DEV)
    st = lib.hb_de_fit_batch(_lib.ptr(xc) if m.num_cont else None, _lib.ptr(xe) if m.num_enum else None, _lib.ptr(y),
                             (C.c_int64 * (B + 1))(*off), B, C.byref(m._spec), E, _lib.ptr(params), float(m.lr), float(m.l1),
                             int(m.batch_size), T, (C.c_uint64 * B)(*seeds), _lib.ptr(losses), _lib.ptr(ws), B * need,
                             _lib.stream_ptr())
    return st, ws, losses


def _check_fit_batch(m, ns, seed0):
    B, E = len(ns), m.num_ensembles
    data = [_rows(m, n, seed0 + b) for b, n in enumerate(ns)]
    off = [0] + np.cumsum(ns).tolist()
    xc, xe, y = (torch.cat([d[i] for d in data]).to(DEV).contiguous() for i in range(3))
    torch.manual_seed(seed0)
    p0 = torch.stack([torch.stack([init_params(m.layout) for _ in range(E)]) for _ in range(B)]).to(DEV).contiguous()
    seeds = [(0x9E3779B97F4A7C15 * (b + 1) + seed0) % 2 ** 64 for b in range(B)]
    params = p0.clone()
    st, ws, losses = _fit_batch(m, xc, xe, y, off, params, seeds)
    _lib.check(st, "hb_de_fit_batch")
    need = ws.numel() // B
    for b in range(B):
        pb = p0[b].clone()
        sl = slice(off[b], off[b + 1])
        ws1, l1 = _fit_one(m, xc[sl].contiguous(), xe[sl].contiguous(), y[sl].contiguous(), pb, seeds[b])
        torch.cuda.synchronize()
        assert torch.equal(params[b], pb), b
        assert torch.equal(ws[b * need:(b + 1) * need].view(torch.float32), ws1.view(torch.float32)), b   # m1, m2, grad
        assert torch.equal(losses[b], l1), b
    assert not torch.equal(params, p0)


@pytest.mark.parametrize("v", VARIANTS, ids=VID)
def test_fit_batch_is_separate_fits(v):
    _check_fit_batch(_model(v), NS[:3], 11)


@pytest.mark.parametrize("ns", [[20], NS], ids=["B1", "B8"])
@pytest.mark.parametrize("v", [VARIANTS[0], VARIANTS[-1]], ids=[VID[0], VID[-1]])
def test_fit_batch_one_and_eight_ensembles(v, ns):
    _check_fit_batch(_model(v), ns, 5)


def test_fit_batch_envelope():
    m = _model(VARIANTS[0])
    xc, xe, y = (t.to(DEV).contiguous() for t in _rows(m, 80, 0))
    st, _, _ = _fit_batch(m, xc, xe, y, list(range(34)), torch.zeros(33, 2, m.P, device=DEV), list(range(33)))
    assert st == _lib.HB_ERR_INVALID                                               # B = 33 > HB_MAX_OUTPUTS
    st, _, _ = _fit_batch(m, xc, xe, y, [0, 10, 10], torch.zeros(2, 2, m.P, device=DEV), [1, 2])
    assert st == _lib.HB_ERR_INVALID                                               # an ensemble without rows
    wide = _model(VARIANTS[0], num_hiddens=256, num_layers=3, batch_size=64)
    assert wide.batch_floats(30) <= _lib.HB_DE_MAX_BATCH_FLOATS < wide.batch_floats(64)
    p = torch.zeros(2, 2, wide.P, device=DEV)
    st, _, _ = _fit_batch(wide, xc, xe, y, [0, 10, 80], p, [1, 2])                 # ensemble 1 takes 64-row minibatches
    assert st == _lib.HB_ERR_INVALID
    st, _, _ = _fit_batch(wide, xc, xe, y, [0, 10, 40], p, [1, 2])                 # 30 rows: within the floats
    assert st == _lib.HB_OK
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------- predict
def _fitted_batch(v, B, seed):
    torch.manual_seed(seed)
    models = []
    for b in range(B):
        m = _model(v)
        m.params = torch.stack([init_params(m.layout) for _ in range(2)]).to(DEV)
        m.params += 0.05 * torch.randn_like(m.params)          # non-zero biases
        Xc, Xe, y = _rows(m, 30, seed + b)
        m.fit(Xc * 3 + b, Xe.long(), y * (b + 1) + b)         # each its own scalers
        models.append(m)
    return models


def _cands(m, n, seed):
    g = torch.Generator().manual_seed(seed)
    xs = (torch.rand(n, m.num_cont, generator=g) * 8 - 2).to(DEV) if m.num_cont else None
    xe = torch.stack([torch.randint(0, u, (n,), generator=g) for u in m.num_uniqs], 1).int().to(DEV) if m.num_enum else None
    return xs, xe


@pytest.mark.parametrize("v", VARIANTS, ids=VID)
def test_predict_batch_is_predict(v):
    models = _fitted_batch(v, 3, 2)
    xs, xe = _cands(models[0], 37, 3)
    mu, var, _ = EnsembleBatch(models).predict(xs, xe)
    O = models[0].num_out
    for b, m in enumerate(models):
        mu1, var1 = m._predict_dev(xs, xe)
        assert torch.equal(mu[b * O:(b + 1) * O], mu1.t()) and torch.equal(var[b * O:(b + 1) * O], var1.t()), b


@pytest.mark.parametrize("B", [1, 8])
def test_predict_batch_draws(B):
    v = (True, True, "mixed", 2, 2)
    models = _fitted_batch(v, B, 4)
    m0, S, m, KO = models[0], 3, 41, 2 * B
    xs, xe = _cands(m0, m, 5)
    batch = EnsembleBatch(models)
    xi = torch.randn(S, m, KO, device=DEV)
    mu, var, samp = batch.predict(xs, xe, n_samples=S, xi=xi)
    assert torch.equal(samp, mu.t() + var.t().sqrt() * xi)          # torch's fp32 expression of BaseModel.sample_y
    seed, counter = 2 ** 40 + 7, 3
    _, _, z_null = batch.predict(xs, xe, n_samples=S, seed=seed, counter=counter)
    # the in-kernel draws: flat element q of y_samp takes half q & 1 of Philox pair q >> 1 under (seed, counter), which
    # is hb_general_acq_epilogue's stream over [S m, KO] (read back at mu = 0, var = 1, noise_sd = 1, kappa = 0)
    zdev = _acq_draws(S * m, KO, seed, counter)
    _, _, z_given = batch.predict(xs, xe, n_samples=S, xi=zdev.reshape(S, m, KO))
    assert torch.equal(z_null, z_given)
    pairs = np.arange((S * m * KO + 1) // 2, dtype=np.uint64)
    z0, z1, r0, r1 = R.normals(seed, pairs, counter)
    z = np.stack([z0, z1], 1).reshape(-1)[:S * m * KO]
    r = np.stack([r0, r1], 1).reshape(-1)[:S * m * KO]
    assert np.all(np.abs(zdev.cpu().double().numpy().reshape(-1) - z) <= r)
    _, _, again = batch.predict(xs, xe, n_samples=S, seed=seed, counter=counter)
    assert torch.equal(again, z_null)
    _, _, other = batch.predict(xs, xe, n_samples=S, seed=seed, counter=counter + 1)
    assert not torch.equal(other, z_null)


def _acq_draws(m, K, seed, counter):
    """[m, K] draws of hb_general_acq_epilogue's stream (seed, counter): its Fo at mu = 0, var = 1, noise_sd = 1, kappa = 0."""
    mu, var, sd = torch.zeros(K, m, device=DEV), torch.ones(K, m, device=DEV), torch.ones(K, device=DEV)
    Fo = torch.empty(m, K, device=DEV)
    _lib.check(_lib.lib().hb_general_acq_epilogue(_lib.ptr(mu), _lib.ptr(var), m, K, 0, 0.0, 0.0, _lib.ptr(sd), None, int(seed),
                                                  int(counter), _lib.ptr(Fo), None, None, _lib.stream_ptr()), "draws")
    return Fo


def test_sample_y_reproducible_and_on_input_device():
    m = _fitted_batch((True, False, "cont", 2, 1), 1, 6)[0]
    xs, _ = _cands(m, 20, 7)
    torch.manual_seed(3)
    a = m.sample_y(xs.cpu(), None, 4)
    torch.manual_seed(3)
    b = m.sample_y(xs, None, 4)
    assert a.device.type == "cpu" and b.is_cuda and tuple(a.shape) == (4, 20, 2) and torch.equal(a, b.cpu())
    assert not torch.equal(a[0], a[1])


# ---------------------------------------------------------------------------------------------------------------- MultiTaskModel
def _mt_data(K, n, seed, dc=3):
    g = torch.Generator().manual_seed(seed)
    Xc = torch.rand(n, dc, generator=g) * 5
    Xe = torch.randint(0, 4, (n, 1), generator=g)
    y = torch.cat([torch.sin(Xc.sum(1, keepdim=True) * (k + 1)) + Xe.float() for k in range(K)], 1)
    for k in range(K):          # every output its own finite rows
        y[torch.arange(k, n, 7 + k), k] = float("nan")
    return Xc, Xe, y


@pytest.mark.parametrize("K", [1, 3])
def test_multitask_ensembles_are_sequential_fits(K):
    conf = dict(num_ensembles=2, num_hiddens=24, num_epochs=5, batch_size=16, num_uniqs=[4], device=DEV)
    Xc, Xe, y = _mt_data(K, 45, 1)
    torch.manual_seed(0)
    mt = MultiTaskModel(3, 1, K, base_model_name="deep_ensemble", **conf)
    mt.fit(Xc, Xe, y)
    torch.manual_seed(0)
    seq = [DeepEnsemble(3, 1, 1, **conf) for _ in range(K)]
    for i, m in enumerate(seq):
        m.fit(Xc, Xe, y[:, [i]])
    Xs, Xse = _mt_data(K, 33, 2)[:2]
    for rnd in range(2):                      # the second round is a warm start from the current weights
        for a, b in zip(mt.models, seq):
            assert torch.equal(a.params, b.params) and torch.equal(a.noise, b.noise) and a.seed == b.seed
            fa, fb = a.fit_state(), b.fit_state()
            assert all(torch.equal(p, q) for p, q in zip(fa, fb)) and torch.equal(a.losses, b.losses)
        py, ps2 = mt.predict(Xs, Xse)
        assert torch.equal(py, torch.cat([b.predict(Xs, Xse)[0] for b in seq], 1))
        assert torch.equal(ps2, torch.cat([b.predict(Xs, Xse)[1] for b in seq], 1))
        assert torch.equal(mt.noise, torch.cat([b.noise for b in seq]))
        if rnd == 0:
            torch.manual_seed(9)
            mt.fit(Xc, Xe, y)
            torch.manual_seed(9)
            for i, m in enumerate(seq):
                m.fit(Xc, Xe, y[:, [i]])


# ---------------------------------------------------------------------------------------------------------------- scorers
def _general_models(K, seed):
    Xc, Xe, y = _mt_data(K, 40, seed)
    conf = dict(num_ensembles=2, num_hiddens=24, num_epochs=5, num_uniqs=[4], device=DEV)
    torch.manual_seed(seed)
    mt = MultiTaskModel(3, 1, K, base_model_name="deep_ensemble", **conf)
    mt.fit(Xc, Xe, y)
    one = DeepEnsemble(3, 1, K, **conf)
    one.fit(Xc, Xe, torch.nan_to_num(y))          # a NaN entry makes its column's noise estimate NaN, as in the reference
    return mt, one


@pytest.mark.parametrize("use_noise", [False, True])
@pytest.mark.parametrize("which", ["multi_task", "one"])
def test_general_score_is_epilogue_on_predict(which, use_noise):
    mt, one = _general_models(3, 4)
    model = mt if which == "multi_task" else one
    acq = GeneralAcq(model, 2, 1, kappa=2.0, c_kappa=0.5, use_noise=use_noise)
    xs, xe = _cands(mt.models[0], 50, 8)
    score = general_score(acq, seed=123)
    for gen in (0, 5):
        Fo, cv = score(xs, xe, gen)
        py, ps2 = model.predict(xs, xe)
        sd = model.noise.reshape(-1).float().sqrt().to(DEV).contiguous() if use_noise else None
        Fo1, _, cv1 = _general_epilogue(py.t().contiguous(), ps2.t().contiguous(), 2, 1, 2.0, 0.5, sd, None, 123, gen,
                                        want_cv=True)
        assert torch.equal(Fo, Fo1) and torch.equal(cv, cv1)


def test_mo_lcb_score_is_epilogue_on_predict():
    _, one = _general_models(1, 5)
    acq = MOMeanSigmaLCB(one, best_y=np.float32(0.3), kappa=2.0)
    xs, xe = _cands(one, 50, 9)
    F, G = general_score(acq, seed=77)(xs, xe, 4)
    py, ps2 = one.predict(xs, xe)
    F1, G1 = _mo_lcb_epilogue(py.reshape(-1).contiguous(), ps2.reshape(-1).contiguous(), _noise_sd(one), _best_y(acq), 2.0,
                              None, 77, 4)
    assert torch.equal(F, F1) and torch.equal(G, G1)


def test_noisy_score_is_sample_on_predict():
    _, one = _general_models(1, 6)
    xs, xe = _cands(one, 300, 10)                       # more rows than the GP's joint sampler takes
    score = ga_score(NoisyAcq(one, 1, 0), seed=55)
    f = score(xs, xe, 7)
    py, ps2 = one.predict(xs, xe)
    zref = _acq_draws(300, 1, 55, 7)
    assert torch.equal(f, (py + ps2.sqrt() * zref).reshape(-1))
    assert not torch.equal(f, score(xs, xe, 8))


# ---------------------------------------------------------------------------------------------------------------- optimisers
SPACE = [{"name": "x0", "type": "num", "lb": -3, "ub": 7}, {"name": "x1", "type": "cat", "categories": ["a", "b", "c"]}]
FAST = {"num_epochs": 100}


def _obj(x: pd.DataFrame) -> np.ndarray:
    return x["x0"].values.astype(float).reshape(-1, 1) ** 2


@pytest.mark.parametrize("make", [
    lambda sp: GeneralBO(sp, rand_sample=8, model_name="deep_ensemble", evo_iters=50),
    lambda sp: GeneralBO(sp, rand_sample=8, model_config={"base_model_name": "deep_ensemble"}, evo_iters=50),
    lambda sp: NoisyOpt(sp, rand_sample=8, model_name="deep_ensemble"),
    lambda sp: NoisyOpt(sp, rand_sample=8, model_name="deep_ensemble", evo_pop=300, evo_iters=20),
], ids=["general", "general-multitask", "noisy", "noisy-pop300"])
def test_opt(make):
    """HEBO/test/test_optimizer.py::test_opt for the deep ensemble."""
    opt = make(DesignSpace().parse(SPACE))
    for _ in range(11):
        rec = opt.suggest(n_suggestions=1)
        opt.observe(rec, _obj(rec))
    assert opt.y.shape[0] == 11 and np.isfinite(opt.y).all()
    assert ((opt.X["x0"] >= -3) & (opt.X["x0"] <= 7)).all()


@pytest.mark.parametrize("ref_point", [None, np.array([60.0, 10.0])], ids=["random", "ehvi"])
@pytest.mark.parametrize("cfg", [dict(model_name="deep_ensemble"), dict(model_config={"base_model_name": "deep_ensemble"})],
                         ids=["one", "multitask"])
def test_general_two_objectives_one_constraint(cfg, ref_point):
    space = DesignSpace().parse([{"name": f"x{i}", "type": "num", "lb": 0, "ub": 1} for i in range(2)])
    nc = 0 if ref_point is not None else 1                 # the EHVI selection takes no constraint (general.py:116)
    opt = GeneralBO(space, 2, nc, rand_sample=5, evo_iters=30, ref_point=ref_point, **cfg)

    def f(x):
        a, b = x["x0"].values, x["x1"].values
        cols = [(a - 0.3) ** 2 + b, (a - 0.7) ** 2 + 1 - b] + ([a + b - 1.2] if nc else [])
        return np.stack(cols, 1)
    for _ in range(8):
        rec = opt.suggest(2)
        assert rec.shape[0] == 2
        opt.observe(rec, f(rec))
    assert opt.y.shape == (16, 2 + nc) and opt.best_y.shape[1] == 2 + nc


def test_embedding_and_contextual_with_the_ensemble():
    box = [{"name": f"x{i}", "type": "num", "lb": -1, "ub": 1} for i in range(6)]
    opt = HEBO_Embedding(box, model_name="deep_ensemble", eff_dim=2, rand_sample=4, evo_iters=20)
    for _ in range(6):
        rec = opt.suggest(1)
        opt.observe(rec, (rec.values ** 2).sum(1, keepdims=True))
    assert opt.mace.y.shape[0] == 6
    ctx = {"one": {"x1": "a"}, "two": {"x1": "b"}}
    cb = HEBO_VectorContextual(SPACE, ctx, model_name="deep_ensemble", rand_sample=3, acq_optimizer="nsga2", evo_iters=20)
    for i in range(5):
        cb.context = "one" if i % 2 == 0 else "two"
        rec = cb.suggest(1)
        assert rec["x1"].iloc[0] == ctx[cb.context]["x1"]
        cb.observe(rec, _obj(rec))
    assert cb.hebo.y.shape[0] == 5
