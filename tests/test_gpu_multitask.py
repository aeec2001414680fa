"""Batched multi-output fit (hb_fit_multi_ex, MultiTaskModel): every output of one batched fit equals a single-output fit of
that output bit for bit -- hypers, losses, the prediction state in its workspace slice and what predict / MACE / sample_y
return -- across the model families; a jitter ladder or give-up of one output leaves the others untouched; the launch chain
of an epoch does not grow with the number of outputs."""
import ctypes as C

import numpy as np
import pytest
import torch

import hebo_b200
from hebo_b200 import _lib
from hebo_b200.gp import MultiTaskModel

pytestmark = pytest.mark.gpu

FAMILIES = {
    # name: (num_cont, n, num_out, conf)
    "matern32": (6, 300, 3, {}),
    "matern32_n1100": (6, 1100, 5, {}),
    "matern52": (4, 260, 2, {"kernel": "matern52"}),
    "rbf": (4, 260, 2, {"kernel": "rbf"}),
    "no_ard": (5, 240, 3, {"ard_kernel": False}),
    "mixed": (3, 250, 3, {"num_uniqs": [4, 3]}),
    "learned_warp": (4, 230, 2, {"warp": True}),
    "fixed_warp": (3, 220, 2, {"warp_a": [0.7, 1.3, 2.0], "warp_b": [1.5, 0.8, 1.1]}),
    "matern12": (4, 260, 3, {"kernel": "matern12"}),
    "matern12_mixed": (3, 250, 2, {"kernel": "matern12", "num_uniqs": [4, 3]}),
    "matern12_learned_warp": (4, 230, 2, {"kernel": "matern12", "warp": True}),
}


def _problem(n, d, e, B, seed):
    g = torch.Generator().manual_seed(seed)
    X = torch.rand(n, d, generator=g) * 3 - 1
    Xe = torch.stack([torch.randint(0, u, (n,), generator=g) for u in e], 1) if e else None
    cols = []
    for b in range(B):
        w = torch.randn(d, generator=g)
        f = torch.sin(X @ w + b) + 0.3 * b * X[:, 0] ** 2
        if e:
            f = f + 0.5 * (Xe[:, 0] == b % e[0]).float()
        cols.append(f + 0.05 * torch.randn(n, generator=g))
    return X, Xe, torch.stack(cols, 1)


def _fit_both(d, e, n, B, conf, epochs, seed=0, Y=None):
    X, Xe, Yp = _problem(n, d, e, B, 100 + seed)
    Y = Yp if Y is None else Y
    cf = dict(conf, num_epochs=epochs, noise_lb=8e-4)
    np.random.seed(seed)
    torch.manual_seed(seed)
    mt = MultiTaskModel(d, len(e), B, **cf)
    batched = mt._batched(Y)
    mt.fit(X, Xe, Y)
    np.random.seed(seed)
    torch.manual_seed(seed)
    singles = [hebo_b200.GP(d, len(e), 1, **cf) for _ in range(B)]
    for b, gp in enumerate(singles):
        gp.fit(X, Xe, Y[:, [b]])
    return mt, singles, X, Xe, batched


def _same(a, b):
    """Same shape, dtype and bytes (NaN-safe, -0.0 != 0.0)."""
    a, b = torch.as_tensor(a).detach().cpu().contiguous(), torch.as_tensor(b).detach().cpu().contiguous()
    return a.shape == b.shape and a.dtype == b.dtype and a.numpy().tobytes() == b.numpy().tobytes()


def _assert_equal_models(mt, singles, X, Xe):
    m = 300
    g = torch.Generator().manual_seed(3)
    Xs = torch.rand(m, X.shape[1], generator=g) * 3 - 1
    Xes = torch.stack([torch.randint(0, u, (m,), generator=g) for u in mt.models[0].num_uniqs], 1) if Xe is not None else None
    for b, (gb, gs) in enumerate(zip(mt.models, singles)):
        assert _same(gb.raw, gs.raw), b
        assert _same(torch.from_numpy(gb.losses), torch.from_numpy(gs.losses)), b
        assert gb._fit_failed == gs._fit_failed
        # the prediction state; L is the lower triangle (the strict upper part of its buffer is never written), the fp16
        # split of L^-1 fills the first half of each of its two buffers plus the scale word (GP.state_tensors)
        half = gb.NP * gb.NP // 2
        assert _same(torch.tril(gb.L_dev), torch.tril(gs.L_dev)), b
        # (the categorical layout view carries one pad word after the layout arrays)
        for x, y in zip(gb.state_tensors(), gs.state_tensors()):
            if x.dtype == torch.int32:
                x, y = x[:-1], y[:-1]
            assert _same(x, y), b
        assert _same(gb.scal_dev, gs.scal_dev) and half > 0
        mu_b, var_b = gb.predict(Xs, Xes)
        mu_s, var_s = gs.predict(Xs, Xes)
        assert _same(mu_b, mu_s) and _same(var_b, var_s), b
        xi1, xi2 = torch.randn(m, 1, generator=g), torch.randn(m, 1, generator=g)
        tau = float(mu_s.min())
        assert _same(gb.predict_mace(Xs, tau, 2.0, 1e-4, xi1, xi2, Xe=Xes), gs.predict_mace(Xs, tau, 2.0, 1e-4, xi1, xi2, Xe=Xes))
        torch.manual_seed(11)
        yb = gb.sample_y(Xs[:20], None if Xes is None else Xes[:20], n_samples=3)
        torch.manual_seed(11)
        ys = gs.sample_y(Xs[:20], None if Xes is None else Xes[:20], n_samples=3)
        assert _same(yb, ys), b
        assert _same(gb.noise, gs.noise)
    mu, var = mt.predict(Xs, Xes)
    assert mu.shape == (m, mt.num_out) and var.shape == (m, mt.num_out)


# 30 epochs: replays of a captured epoch; 3 epochs: too short to capture, every epoch enqueued directly
@pytest.mark.parametrize("family,epochs", [pytest.param(f, 30, id=f) for f in FAMILIES]
                         + [pytest.param(f, 3, id=f"{f}-3epochs") for f in ("matern32", "mixed")])
def test_batched_fit_equals_per_output_fits(family, epochs):
    d, n, B, conf = FAMILIES[family]
    e = conf.get("num_uniqs", [])
    mt, singles, X, Xe, batched = _fit_both(d, e, n, B, conf, epochs)
    assert batched and all(g.kernel == conf.get("kernel", "matern32") for g in mt.models)
    _assert_equal_models(mt, singles, X, Xe)


def test_nan_rows_select_the_path_and_match_per_output_fits():
    d, n, B = 4, 200, 3
    X, _, Y = _problem(n, d, [], B, 7)
    same = Y.clone()
    same[[3, 50, 120]] = float("nan")              # the same rows in every column: one batched fit on the 197 others
    mt, singles, X, _, batched = _fit_both(d, [], n, B, {}, 30, seed=1, Y=same)
    assert batched and mt.models[0].n == n - 3
    _assert_equal_models(mt, singles, X, None)
    diff = Y.clone()
    diff[3, 0] = float("nan")                      # differing rows: each output keeps its own n, the per-output loop
    mt, singles, X, _, batched = _fit_both(d, [], n, B, {}, 30, seed=2, Y=diff)
    assert not batched and mt.models[0].n == n - 1 and mt.models[1].n == n
    _assert_equal_models(mt, singles, X, None)


# ---------------------------------------------------------------------------------------------- through the C ABI
def _abi_inputs(B):
    g = torch.Generator().manual_seed(5)
    X = torch.randn(40, 2, generator=g)
    X = torch.cat([X, X, X], 0)                    # duplicated rows: singular without noise
    n, d = X.shape
    lib = _lib.lib()
    NP = int(lib.hb_padded_n(n))
    Xs = (X - X.min(0).values) / (X.max(0).values - X.min(0).values) * 2 - 1
    XtT = torch.zeros(d, NP, dtype=torch.float32)
    XtT[:, :n] = Xs.t()
    Y = torch.stack([torch.sin(2 * X[:, 0] + b) + 0.1 * X[:, 1] for b in range(B)])
    Y = (Y - Y.mean(1, keepdim=True)) / Y.std(1, keepdim=True)
    raw = torch.tensor([[-2.0, 0.0, 0.5, 0.5, 0.5]]).repeat(B, 1)
    return XtT.cuda(), Y.float().cuda().contiguous(), raw, n, d


def _fit_single(XtT, y, raw, n, d, E, lang=None):
    lib = _lib.lib()
    wsb = int(lib.hb_fit_workspace_bytes(n, d))
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    r = raw.clone().cuda().contiguous()
    losses = (C.c_float * max(1, E))()
    st = lib.hb_fit_ex(_lib.ptr(XtT), None, _lib.ptr(y), n, d, None, _lib.ptr(r), 0, None, 1e-12, 0.01, 0.03, E, _lib.ptr(lang),
                       losses, _lib.ptr(ws), wsb, _lib.stream_ptr())
    torch.cuda.synchronize()
    return st, r.cpu(), np.array(losses[:E], dtype=np.float32), ws


def _fit_multi(XtT, Y, raw, n, d, E, lang=None):
    lib = _lib.lib()
    B = Y.shape[0]
    wsb = int(lib.hb_fit_multi_workspace_bytes(n, d, None, B))
    assert wsb == B * int(lib.hb_fit_workspace_bytes(n, d))
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    r = raw.clone().cuda().contiguous()
    losses = (C.c_float * (B * E))()
    status = (C.c_int32 * B)()
    _lib.check(lib.hb_fit_multi_ex(_lib.ptr(XtT), None, _lib.ptr(Y), n, d, None, B, _lib.ptr(r), 0, None, 1e-12, 0.01, 0.03, E,
                                   _lib.ptr(lang), losses, status, _lib.ptr(ws), wsb, _lib.stream_ptr()), "hb_fit_multi_ex")
    torch.cuda.synchronize()
    return list(status), r.cpu(), np.array(losses[:B * E], dtype=np.float32).reshape(B, E), ws


# (0, -40): ~0 noise on the duplicated rows, the jitter ladder for output 1 only;
# (3, -200): a lengthscale that underflows to 0, a hopeless output (every epoch given up) next to healthy ones;
# E = 12 replays a captured epoch, E = 3 is too short to capture and enqueues every epoch directly
@pytest.mark.parametrize("slot,value,E", [pytest.param(s, v, E, id=f"{s}-{v}" + ("" if E == 12 else f"-E{E}"))
                                          for E in (12, 3) for s, v in [(0, -40.0), (3, -200.0)]])
def test_jitter_ladder_of_one_output_leaves_the_others_alone(slot, value, E):
    B = 3
    XtT, Y, raw, n, d = _abi_inputs(B)
    raw[1, slot] = value
    g = torch.Generator().manual_seed(9)
    lang = torch.randn(B, E, raw.shape[1], generator=g).cuda().contiguous()
    lib = _lib.lib()
    # the first epoch of output 1 is not positive definite at jitter 0
    wsb = int(lib.hb_fit_workspace_bytes(n, d))
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    grad, loss = torch.empty(5, device="cuda"), torch.empty(1, device="cuda")
    info = torch.zeros(1, dtype=torch.int32, device="cuda")
    r1 = raw[1].cuda().contiguous()
    _lib.check(lib.hb_mll_fwd_bwd(_lib.ptr(XtT), None, _lib.ptr(Y[1]), n, d, None, _lib.ptr(r1), 0, None, 1e-12, 0.01, 0.0,
                                  _lib.ptr(grad), _lib.ptr(loss), _lib.ptr(info), _lib.ptr(ws), wsb, _lib.stream_ptr()), "mll")
    if slot == 0:
        assert int(info.item()) != 0
    status, rm, lm, wsm = _fit_multi(XtT, Y, raw, n, d, E, lang)
    stride = wsb
    for b in range(B):
        st, rs, ls, wss = _fit_single(XtT, Y[b].contiguous(), raw[b], n, d, E, lang[b].contiguous())
        assert status[b] == st, b
        assert torch.equal(rm[b], rs), b
        assert np.array_equal(lm[b].view(np.uint32), ls.view(np.uint32)), b
        # the whole slice the prediction state lives in
        fs_m, fs_s = _lib.FitState(), _lib.FitState()
        _lib.check(lib.hb_fit_state(C.c_void_p(wsm.data_ptr() + b * stride), n, d, C.byref(fs_m)), "state")
        _lib.check(lib.hb_fit_state(_lib.ptr(wss), n, d, C.byref(fs_s)), "state")
        NP = int(lib.hb_padded_n(n))
        for name, cnt in (("hyp", 5), ("Linv", NP * NP), ("alpha", NP)):
            a = wsm[getattr(fs_m, name) - wsm.data_ptr():][:cnt * 4]
            s = wss[getattr(fs_s, name) - wss.data_ptr():][:cnt * 4]
            if status[b] == _lib.HB_OK:
                assert torch.equal(a, s), (b, name)
    for b in (0, 2):                               # the well-posed outputs trained normally
        assert np.isfinite(lm[b]).all() and status[b] == _lib.HB_OK
    if slot == 3:
        assert not np.isfinite(lm[1]).any()


def test_launches_per_epoch_do_not_depend_on_the_number_of_outputs():
    lib = _lib.lib()
    per = {}
    for B in (1, 4):
        XtT, Y, raw, n, d = _abi_inputs(B)
        raw[:, 0] = 0.0                            # well-posed: every epoch on the graph, no ladder
        counts = []
        for E in (10, 30):
            lib.hb_launch_count(1)
            _fit_multi(XtT, Y, raw, n, d, E)
            counts.append(int(lib.hb_launch_count(1)))
        per[B] = (counts[1] - counts[0]) / 20
    assert per[1] == per[4] and per[1] > 0
