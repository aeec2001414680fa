"""Host-side checks of the multi-output deep ensemble: constructor gating of the optimisers that take it, MultiTaskModel's
base_model_name dispatch, the argument checks of hb_de_fit_batch / hb_de_predict_batch (no CUDA call is made), and the
row offsets and generator order of fit_ensembles against a plain restatement."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

from hebo_b200 import DeepEnsemble, _lib
from hebo_b200.bo import HEBO_VectorContextual
from hebo_b200.embedding import HEBO_Embedding
from hebo_b200.ensemble import batch_offsets, fit_ensembles, init_params
from hebo_b200.evolution import DeviceNSGA2
from hebo_b200.general import GeneralBO
from hebo_b200.gp import GP, MultiTaskModel
from hebo_b200.noisy import NoisyOpt

SPACE = [{"name": "x0", "type": "num", "lb": -3, "ub": 7}, {"name": "x1", "type": "cat", "categories": ["a", "b", "c"]}]


@pytest.fixture(scope="module")
def lib():
    if not _lib.available():
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


def test_optimisers_accept_the_ensemble():
    for kw in (dict(model_name="deep_ensemble"), dict(model_config={"base_model_name": "deep_ensemble"})):
        opt = GeneralBO(SPACE, 2, 1, **kw)
        assert opt.model_name == kw.get("model_name", "multi_task")
    assert GeneralBO(SPACE, 1, 0, model_name="gp").model_name == "gp"
    with pytest.raises(NotImplementedError):
        GeneralBO(SPACE, 2, 1, model_name="rf")
    with pytest.raises(AssertionError):
        GeneralBO(SPACE, 2, 1, model_name="gp")
    assert NoisyOpt(SPACE, model_name="deep_ensemble").model_name == "deep_ensemble"
    with pytest.raises(NotImplementedError):
        NoisyOpt(SPACE, model_name="rf")
    box = [{"name": f"x{i}", "type": "num", "lb": -1, "ub": 1} for i in range(4)]
    assert HEBO_Embedding(box, model_name="deep_ensemble", eff_dim=2, device="cpu").mace.model_name == "deep_ensemble"
    with pytest.raises(NotImplementedError):
        HEBO_Embedding(box, model_name="rf", eff_dim=2, device="cpu")
    ctx = {"one": {"x1": "a"}}
    assert HEBO_VectorContextual(SPACE, ctx, model_name="deep_ensemble").hebo.model_name == "deep_ensemble"
    assert HEBO_VectorContextual(SPACE, ctx).hebo.model_name == "gp"
    with pytest.raises(NotImplementedError):
        HEBO_VectorContextual(SPACE, ctx, model_name="rf")


def test_noisy_population_cap_is_the_gp_sampler_only():
    with pytest.raises(ValueError):
        NoisyOpt(SPACE, evo_pop=257)
    with pytest.raises(ValueError):
        NoisyOpt(SPACE, model_name="gp", evo_pop=NoisyOpt.MAX_POP + 1)
    assert NoisyOpt(SPACE, model_name="deep_ensemble", evo_pop=257).evo_pop == 257
    assert NoisyOpt(SPACE, model_name="deep_ensemble", evo_pop=DeviceNSGA2.MAX_POP).evo_pop == DeviceNSGA2.MAX_POP
    with pytest.raises(ValueError):
        NoisyOpt(SPACE, model_name="deep_ensemble", evo_pop=DeviceNSGA2.MAX_POP + 1)


def test_base_model_name_dispatch():
    mt = MultiTaskModel(2, 1, 3, num_uniqs=[3], device="cpu")
    assert mt.base_model_name == "gp" and all(type(m) is GP for m in mt.models)
    mt = MultiTaskModel(2, 0, 3, base_model_name="gp", device="cpu")
    assert all(type(m) is GP for m in mt.models)
    mt = MultiTaskModel(2, 1, 3, base_model_name="deep_ensemble", num_uniqs=[3], num_ensembles=4, num_hiddens=16, device="cpu")
    assert len(mt.models) == 3 and all(type(m) is DeepEnsemble for m in mt.models)
    assert all(m.num_out == 1 and m.num_ensembles == 4 and m.num_hiddens == 16 and m.num_uniqs == [3] for m in mt.models)
    assert "base_model_name" not in mt.models[0].conf
    for bad in ("rf", "psgld", "svgp"):
        with pytest.raises(NotImplementedError):
            MultiTaskModel(2, 0, 2, base_model_name=bad, device="cpu")
    with pytest.raises(NotImplementedError):
        MultiTaskModel(2, 0, _lib.HB_MAX_OUTPUTS + 1, base_model_name="deep_ensemble", device="cpu")


def _dummy_args(B=2, off=(0, 10, 25), E=2, batch=32, ws=1 << 40):
    spec = _lib.DeSpec(2, 0, None, _lib.HB_DE_EMBEDDING, 1, 16, 1, 1, 0, 1e-4)
    p = C.c_void_p(256)                     # never dereferenced: the arguments are checked first
    return (p, None, p, (C.c_int64 * len(off))(*off), B, C.byref(spec), E, p, 5e-3, 1e-3, batch, 3,
            (C.c_uint64 * max(1, B))(*range(max(1, B))), p, p, ws, None)


def test_fit_batch_rejects_bad_arguments(lib):
    bad = _lib.HB_ERR_INVALID
    spec = _lib.DeSpec(2, 0, None, _lib.HB_DE_EMBEDDING, 1, 16, 1, 1, 0, 1e-4)
    one = lib.hb_de_fit_workspace_bytes(C.byref(spec), 2)
    off33 = tuple(range(34))
    assert lib.hb_de_fit_batch(*_dummy_args(B=_lib.HB_MAX_OUTPUTS + 1, off=off33)) == bad
    assert lib.hb_de_fit_batch(*_dummy_args(B=0, off=(0,))) == bad
    assert lib.hb_de_fit_batch(*_dummy_args(off=(0, 10, 10))) == bad             # an ensemble without rows
    assert lib.hb_de_fit_batch(*_dummy_args(off=(-1, 10, 20))) == bad
    assert lib.hb_de_fit_batch(*_dummy_args(ws=2 * one - 1)) == bad              # short workspace
    assert lib.hb_de_fit_batch(*_dummy_args(E=_lib.HB_DE_MAX_MEMBERS + 1)) == bad
    # minibatch floats (HB_DE_MAX_BATCH_FLOATS): ensemble 1's minibatch is one row too many
    per_row = (2 | 1) + 3 * (16 | 1) + 5 + 1
    rows = _lib.HB_DE_MAX_BATCH_FLOATS // per_row
    assert lib.hb_de_fit_batch(*_dummy_args(off=(0, 10, 10 + rows + 1), batch=rows + 1)) == bad
    args = list(_dummy_args())
    args[12] = None                                                               # seeds
    assert lib.hb_de_fit_batch(*args) == bad
    args = list(_dummy_args())
    args[3] = None                                                                # off
    assert lib.hb_de_fit_batch(*args) == bad


def test_predict_batch_rejects_bad_arguments(lib):
    bad = _lib.HB_ERR_INVALID
    spec = _lib.DeSpec(2, 0, None, _lib.HB_DE_EMBEDDING, 1, 16, 1, 1, 0, 1e-4)
    p = C.c_void_p(256)

    def call(B=2, E=2, n_samples=0, y_samp=p, var=p, m=10):
        return lib.hb_de_predict_batch(p, None, m, C.byref(spec), B, E, p, p, p, p, p, p, var, n_samples, None, 0, 0, y_samp,
                                       None)
    assert call(B=0) == bad and call(B=_lib.HB_MAX_OUTPUTS + 1) == bad
    assert call(E=0) == bad and call(n_samples=-1) == bad and call(var=None) == bad
    assert call(n_samples=1, y_samp=None) == bad and call(m=-1) == bad
    assert call(m=0) == _lib.HB_OK                                                # nothing to do: no launch


def test_batch_offsets_restated():
    for ns in ([1], [5, 37, 20], [64] * 32, [3, 1, 4, 1, 5, 9, 2, 6]):
        off = batch_offsets(ns)
        ref = [0]
        for n in ns:
            ref.append(ref[-1] + n)
        assert off == ref


class _FakeLib:
    def __init__(self):
        self.calls = []

    def hb_de_fit_workspace_bytes(self, spec, E):
        return 64

    def hb_de_fit_batch(self, xc, xe, y, off, B, spec, E, params, lr, l1, bs, T, seeds, losses, ws, ws_bytes, stream):
        self.calls.append(dict(off=[off[i] for i in range(B + 1)], seeds=[seeds[i] for i in range(B)], B=B, E=E,
                               ws_bytes=ws_bytes, y=C.cast(y, C.c_void_p).value))
        return _lib.HB_OK


@pytest.fixture
def fake(monkeypatch):
    f = _FakeLib()
    monkeypatch.setattr(_lib, "lib", lambda: f)
    monkeypatch.setattr(_lib, "stream_ptr", lambda: None)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(DeepEnsemble, "_finish_fit", lambda self, *a: None)
    return f


def _data(K, n):
    g = torch.Generator().manual_seed(3)
    Xc = torch.rand(n, 2, generator=g)
    y = torch.randn(n, K, generator=g)
    y[torch.arange(0, n, 4), 0] = float("nan")                  # output 0 loses every fourth row
    if K > 2:
        y[torch.arange(1, n, 3), 2] = float("inf")              # output 2 every third
    return Xc, y


@pytest.mark.parametrize("K", [1, 3])
def test_fit_ensembles_rows_and_generator_order(fake, K):
    conf = dict(num_ensembles=3, num_hiddens=8, num_epochs=2, device="cpu")
    Xc, y = _data(K, 23)
    torch.manual_seed(5)
    models = [DeepEnsemble(2, 0, 1, **conf) for _ in range(K)]
    fit_ensembles(models, Xc, None, [y[:, [i]] for i in range(K)])
    # restatement: model b keeps its own finite rows, draws its E initial weight vectors and then its seed
    torch.manual_seed(5)
    ref_params, ref_seeds, ns = [], [], []
    for b in range(K):
        ns.append(int(torch.isfinite(y[:, b]).sum()))
        ref_params.append(torch.stack([init_params(models[b].layout) for _ in range(3)]))
        ref_seeds.append(int(torch.randint(0, 2 ** 62, (1,)).item()))
    call = fake.calls[-1]
    assert call["B"] == K and call["E"] == 3 and call["ws_bytes"] == 64 * K
    assert call["off"] == [0] + np.cumsum(ns).tolist() and call["seeds"] == ref_seeds
    assert [m.seed for m in models] == ref_seeds
    for b, m in enumerate(models):
        assert torch.equal(m.params, ref_params[b])
        assert m.fit_ws.numel() == 64 and tuple(m.losses.shape) == (3, 2)
    # a second fit is a warm start: no weights drawn, one seed per model, and the params slices carried over
    before = [m.params.clone() for m in models]
    torch.manual_seed(8)
    fit_ensembles(models, Xc, None, [y[:, [i]] for i in range(K)])
    torch.manual_seed(8)
    assert fake.calls[-1]["seeds"] == [int(torch.randint(0, 2 ** 62, (1,)).item()) for _ in range(K)]
    assert all(torch.equal(m.params, p) for m, p in zip(models, before))


def test_fit_ensembles_checks_its_envelope(fake):
    models = [DeepEnsemble(2, 0, 1, num_ensembles=1, device="cpu") for _ in range(_lib.HB_MAX_OUTPUTS + 1)]
    Xc, y = _data(1, 10)
    with pytest.raises(NotImplementedError):
        fit_ensembles(models, Xc, None, [y] * len(models))
    wide = MultiTaskModel(2, 0, 2, base_model_name="deep_ensemble", num_layers=3, num_hiddens=256, batch_size=64, device="cpu")
    Xc, y = _data(2, 80)
    with pytest.raises(NotImplementedError):
        wide.fit(Xc, None, y)
    assert not fake.calls
