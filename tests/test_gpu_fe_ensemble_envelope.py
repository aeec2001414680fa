"""hb_fe_fit / hb_fe_predict across the gated envelope of ensemble.cu.

- stg gate, MSE head, mask_reg = 0: bit for bit against the fp32 restatement (oracle/fe_oracle.py), at small shapes and
  at the envelope corner (din = 256, 3 x 256 hidden units, 8 outputs, a prior net, the largest minibatch the gated
  check admits), with draws that put some gate states exactly on both clamp bounds.
- every gate, both heads, the mask penalty on: one step's gradient per element against the fp64 oracle, and Adam's
  update of it bit for bit.  The gate's mask, the penalty and the concrete layers go through expf / logf, which are not
  correctly rounded, so these are checked against fp64 rather than bit for bit.
- one row over the gated minibatch limit is rejected without a launch, and the plain ensemble still takes it."""
import ctypes as C

import numpy as np
import pytest
import torch

from hebo_b200 import _lib
from oracle import ensemble_oracle as EO
from oracle import fe_oracle as FO

pytestmark = pytest.mark.gpu

LR, L1 = 5e-3, 1e-3
KIND = {"stg": _lib.HB_FE_STG, "concrete": _lib.HB_FE_CONCRETE, "hard_concrete": _lib.HB_FE_HARD_CONCRETE}


def _rows_max(kw):
    """The largest minibatch the gated check admits for kw (include/hebo_b200.h)."""
    din = kw["num_cont"] + sum(min(50, 1 + u // 2) if kw.get("enum_trans", "embedding") == "embedding" else u
                               for u in kw["num_uniqs"])
    in_ld, h_ld = din | 1, max(kw["num_hiddens"], din) | 1
    per_row = in_ld + (kw["num_layers"] + 2) * h_ld + 5 * kw["num_out"] + 1 + 2 * in_ld
    return _lib.HB_DE_MAX_BATCH_FLOATS // per_row


CORNER = dict(num_cont=256, num_uniqs=[], num_layers=3, num_hiddens=256, num_out=8, rand_prior=True)
CASES = {
    "mixed-prior": (dict(num_cont=3, num_uniqs=[4, 7], num_layers=1, num_hiddens=16, num_out=2, rand_prior=True), 30, 8),
    "onehot-L2": (dict(num_cont=2, num_uniqs=[3, 5], enum_trans="onehot", num_layers=2, num_hiddens=24, num_out=1), 20, 8),
    "enum-only": (dict(num_cont=0, num_uniqs=[3, 5], num_layers=1, num_hiddens=8, num_out=1), 12, 16),
    "corner": (CORNER, _rows_max(CORNER) + 1, _rows_max(CORNER)),
}


def _spec(kw, noise):
    u = (C.c_int32 * max(1, len(kw["num_uniqs"])))(*kw["num_uniqs"])
    s = _lib.DeSpec(kw["num_cont"], len(kw["num_uniqs"]), u,
                    _lib.HB_DE_ONEHOT if kw.get("enum_trans") == "onehot" else _lib.HB_DE_EMBEDDING, kw["num_layers"],
                    kw["num_hiddens"], kw["num_out"], int(noise), int(kw.get("rand_prior", False)), 1e-4)
    return s, u


def _dev(a, dt=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dt).contiguous() if a is not None and np.size(a) else None


def _data(kw, n, seed):
    g = np.random.default_rng(seed)
    Xc = g.uniform(-1, 1, (n, kw["num_cont"])).astype(np.float32) if kw["num_cont"] else None
    Xe = np.stack([g.integers(0, u, n) for u in kw["num_uniqs"]], 1).astype(np.int32) if kw["num_uniqs"] else None
    y = g.normal(size=(n, kw["num_out"])).astype(np.float32)
    if kw["num_out"] > 1:
        y[1, 0] = np.nan
    return Xc, Xe, y


def _init(net, E, seed, zero_gate_cols=4):
    g = np.random.default_rng(seed)
    raw = (g.normal(size=(E, net.P)) * 0.2).astype(np.float32)
    raw[:, net.gate0:] = (0.01 * g.normal(size=(E, net.din))).astype(np.float32)
    raw[:, net.gate0:net.gate0 + zero_gate_cols] = 0.0        # theta = 0: draws of +-1/2 land exactly on the bounds
    return raw


def _draws(shape, seed, bounds=True):
    r = np.random.default_rng(seed).normal(size=shape).astype(np.float32)
    if bounds:      # with T = 1 and theta = 0: (0.5 + 0) + 0.5 = 1 and (-0.5 + 0) + 0.5 = 0 exactly
        r[..., 0], r[..., 1] = 0.5, -0.5
        r[..., 1::2, 2], r[..., 0::2, 3] = 0.5, -0.5
    return r


def fe_fit(kw, noise, kind, raw0, Xc, Xe, y, perm, draws, batch, epochs, mask_reg=0.0, T=1.0):
    spec, keep = _spec(kw, noise)
    lib = _lib.lib()
    E = raw0.shape[0]
    gate = _lib.FeGate(KIND[kind], T, 1.0, 0.1, 0.99, mask_reg)
    params = _dev(raw0)
    need = int(lib.hb_fe_fit_workspace_bytes(C.byref(spec), E))
    ws = torch.zeros(need, dtype=torch.uint8, device="cuda")
    losses = torch.zeros(E, max(1, epochs), device="cuda")
    # every device operand is held in a local until the launch has finished: a temporary's memory could be handed to
    # the next upload before the kernel reads it
    xc, xe, yd, pd_, dd = _dev(Xc), _dev(Xe, torch.int32), _dev(y), _dev(perm, torch.int32), _dev(draws)
    st = lib.hb_fe_fit(_lib.ptr(xc), _lib.ptr(xe), _lib.ptr(yd), y.shape[0], C.byref(spec), C.byref(gate), E,
                       _lib.ptr(params), LR, L1, batch, epochs, _lib.ptr(pd_), _lib.ptr(dd), 7,
                       _lib.ptr(losses), _lib.ptr(ws), need, _lib.stream_ptr())
    torch.cuda.synchronize()
    w = ws.view(torch.float32).view(3, E, -1).cpu().numpy()
    return st, params.cpu().numpy(), w[0], w[1], w[2]


def _orders(n, E, epochs, seed):
    g = np.random.default_rng(seed)
    return np.stack([np.stack([g.permutation(n) for _ in range(epochs)]) for _ in range(E)]).astype(np.int32)


def assert_bits(got, want, what):
    bad = EO.mismatches(got, want)
    assert bad == 0, f"{what}: {bad} of {np.size(want)} elements differ"


# ------------------------------------------------------------------------------------------------ a. fit, bit for bit
@pytest.mark.parametrize("case", list(CASES))
def test_stg_fit_equals_the_restatement_bit_for_bit(case):
    kw, n, batch = CASES[case]
    E, epochs = 2, 2
    net = FO.FeNet32(kw["num_cont"], kw["num_uniqs"], kw.get("enum_trans", "embedding"), kw["num_layers"],
                     kw["num_hiddens"], kw["num_out"], False, kw.get("rand_prior", False), kind="stg")
    Xc, Xe, y = _data(kw, n, 1)
    raw0 = _init(net, E, 2)
    perm = _orders(n, E, epochs, 3)
    B, nb = EO.minibatch_rule(n, batch)
    draws = _draws((E, epochs, nb, B, net.din), 4)
    st, params, m1, m2, g = fe_fit(kw, False, "stg", raw0, Xc, Xe, y, perm, draws, batch, epochs)
    assert st == _lib.HB_OK
    for e in range(E):
        p, a, b, gg = FO.fe_fit32(net, raw0[e], Xc, Xe, y, perm[e], draws[e], LR, L1, batch, 1.0)
        for what, dv, rv in (("params", params[e], p), ("exp_avg", m1[e], a), ("exp_avg_sq", m2[e], b), ("grad", g[e], gg)):
            assert_bits(dv, rv, f"member {e} {what}")
    # the gate moved, the biases took no L1 term, the prior net's biases did not move at all
    assert not np.array_equal(params[:, net.gate0:], raw0[:, net.gate0:])
    for name, (o, shape) in net.slices.items():
        sl = slice(o, o + int(np.prod(shape)))
        if name.startswith("prior_net") and name.endswith("bias"):
            assert np.array_equal(params[:, sl], raw0[:, sl]) and not g[:, sl].any()


def test_inclusive_clamp_bounds_carry_the_gradient():
    """Gate states exactly on 0 and on 1 pass the gradient (torch.clamp's rule): one step whose draws put states on both
    bounds, with nonzero inputs there, equals the inclusive restatement bit for bit."""
    kw, _, _ = CASES["mixed-prior"]
    n = batch = 8
    net = FO.FeNet32(kw["num_cont"], kw["num_uniqs"], "embedding", 1, kw["num_hiddens"], kw["num_out"], False, True)
    Xc, Xe, y = _data(kw, n, 1)
    raw0 = _init(net, 1, 2)
    perm = _orders(n, 1, 1, 3)
    draws = _draws((1, 1, 1, n, net.din), 4)
    st_, _, _, _, g = fe_fit(kw, False, "stg", raw0, Xc, Xe, y, perm, draws, batch, 1)
    assert st_ == _lib.HB_OK
    rows = perm[0, 0]
    st = FO.stg_state32(raw0[0], net.gate0, draws[0, 0, 0], 1.0)
    xraw = EO.load_inputs32(net, raw0[0], Xc[rows], Xe[rows])
    assert ((st == 0) & (xraw != 0)).any() and ((st == 1) & (xraw != 0)).any()
    assert_bits(g[0], FO.fe_step_grad32(net, raw0[0], Xc, Xe, y, rows, n, L1, draws[0, 0, 0], 1.0), "gradient")


# ------------------------------------------------------------------------------------------------ b. predict
@pytest.mark.parametrize("case,E", [("mixed-prior", 1), ("mixed-prior", 32), ("onehot-L2", 2), ("enum-only", 3),
                                    ("corner", 2)])
def test_stg_predict_equals_the_restatement_bit_for_bit(case, E):
    kw, _, _ = CASES[case]
    net = FO.FeNet32(kw["num_cont"], kw["num_uniqs"], kw.get("enum_trans", "embedding"), kw["num_layers"],
                     kw["num_hiddens"], kw["num_out"], False, kw.get("rand_prior", False), kind="stg")
    m = 37
    Xs, Xe, _ = _data(kw, m, 9)
    params = _init(net, E, 10)
    draws = _draws((E, net.din), 11)
    dc, O = kw["num_cont"], kw["num_out"]
    g = np.random.default_rng(12)
    xm, xa = g.uniform(0.5, 2, dc).astype(np.float32), g.uniform(-1, 1, dc).astype(np.float32)
    ym, ys = g.normal(size=O).astype(np.float32), g.uniform(0.5, 2, O).astype(np.float32)
    spec, keep = _spec(kw, False)
    gate = _lib.FeGate(_lib.HB_FE_STG, 1.0, 1.0, 0.1, 0.99, 0.1)
    mu, var = torch.empty(m, O, device="cuda"), torch.empty(m, O, device="cuda")
    d = [_dev(Xs), _dev(Xe, torch.int32), _dev(params), _dev(xm), _dev(xa), _dev(ym), _dev(ys), _dev(draws)]
    _lib.check(_lib.lib().hb_fe_predict(_lib.ptr(d[0]), _lib.ptr(d[1]), m, C.byref(spec), C.byref(gate), E, _lib.ptr(d[2]),
                                        _lib.ptr(d[3]), _lib.ptr(d[4]), _lib.ptr(d[5]), _lib.ptr(d[6]), -1, _lib.ptr(d[7]), 0,
                                        0, _lib.ptr(mu), _lib.ptr(var), _lib.stream_ptr()), "hb_fe_predict")
    torch.cuda.synchronize()
    rmu, rvar = FO.fe_predict32(net, params, Xs, Xe, xm if dc else None, xa if dc else None, ym, ys, draws, 1.0)
    assert_bits(mu.cpu().numpy(), rmu, "mu")
    assert_bits(var.cpu().numpy(), rvar, "var")


# ------------------------------------------------------------------------------------------------ c. one step vs fp64
STEP = [(k, c, noise) for k in KIND for c in ("mixed-prior", "onehot-L2", "enum-only", "corner") for noise in (False, True)]


@pytest.mark.parametrize("kind,case,noise", STEP, ids=[f"{k}-{c}-{'nll' if z else 'mse'}" for k, c, z in STEP])
def test_step_gradient_matches_fp64_and_adam_is_bit_exact(kind, case, noise):
    kw, n, batch = CASES[case]
    n = min(n, batch)                    # one minibatch of all n rows: the fit is exactly one step
    net32 = FO.FeNet32(kw["num_cont"], kw["num_uniqs"], kw.get("enum_trans", "embedding"), kw["num_layers"],
                       kw["num_hiddens"], kw["num_out"], noise, kw.get("rand_prior", False), kind=kind)
    net64 = FO.FeOracleNet(kw["num_cont"], kw["num_uniqs"], kw.get("enum_trans", "embedding"), kw["num_layers"],
                           kw["num_hiddens"], kw["num_out"], noise, kw.get("rand_prior", False), kind=kind)
    Xc, Xe, y = _data(kw, n, 21)
    raw0 = _init(net32, 1, 22, zero_gate_cols=0)
    perm = _orders(n, 1, 1, 23)
    if kind == "stg":
        draws = _draws((1, 1, 1, n, net32.din), 24, bounds=False)
    else:
        draws = np.random.default_rng(24).uniform(0, 1, (1, 1, 1, n, net32.din)).astype(np.float32)
    T = 1.0 if kind == "stg" else 1.0          # the concrete layers' epoch 0: max(1.0 * 0.99^0, 0.1)
    st, params, m1, m2, g = fe_fit(kw, noise, kind, raw0, Xc, Xe, y, perm, draws, batch, 1, mask_reg=0.1)
    assert st == _lib.HB_OK
    net64.load_raw(raw0[0].astype(np.float64))
    _, g64 = FO.fe_step_grad(net64, torch.from_numpy(Xc).double() if Xc is not None else None,
                             torch.from_numpy(Xe) if Xe is not None else None, torch.from_numpy(y).double(), perm[0, 0],
                             draws[0, 0, 0].astype(np.float64), T, L1, 0.1, n)
    g64 = g64.numpy()
    scale = float(np.abs(g64).max())
    err = np.abs(g[0].astype(np.float64) - g64)
    # fp32 sums of at most max(n, H, din) terms of this scale, and the device's expf / logf
    assert float(err.max()) <= 1e-4 * scale, (float(err.max()), scale)
    gate = slice(net32.gate0, None)
    assert float(np.abs(g[0, gate] - g64[gate]).max()) <= 1e-4 * max(float(np.abs(g64[gate]).max()), 1e-6)
    # the L1 term: weights only (coef sign(w)), and the prior net's biases take nothing
    coef = (np.float32(1.0) / np.float32(n * net32.O)) * np.float32(L1)
    for name, (o, shape) in net32.slices.items():
        sl = slice(o, o + int(np.prod(shape)))
        if name.startswith("prior_net"):
            want = np.where("weight" in name, coef * np.sign(raw0[0, sl]), 0).astype(np.float32)
            assert_bits(g[0, sl], want, name)
    p, a, b = EO.adam_update_f32(raw0[0], g[0], np.zeros(net32.P, np.float32), np.zeros(net32.P, np.float32), 1, LR)
    assert_bits(params[0], p, "params")
    assert_bits(m1[0], a, "exp_avg")
    assert_bits(m2[0], b, "exp_avg_sq")


# ------------------------------------------------------------------------------------------------ d. the gated limit
def test_one_row_over_the_gated_minibatch_is_rejected_and_the_plain_ensemble_still_takes_it():
    kw = CORNER
    Bmax = _rows_max(kw)
    net = FO.FeNet32(kw["num_cont"], [], "embedding", 3, 256, 8, False, True)
    n = Bmax + 2
    Xc, Xe, y = _data(kw, n, 31)
    raw0 = _init(net, 1, 32)
    params0 = raw0.copy()
    st, params, *_ = fe_fit(kw, False, "stg", raw0, Xc, Xe, y, None, None, Bmax + 1, 1)
    assert st == _lib.HB_ERR_INVALID and np.array_equal(params, params0)
    spec, keep = _spec(kw, False)
    de_floats = (Bmax + 1) * (257 + 5 * 257 + 41)
    assert de_floats <= _lib.HB_DE_MAX_BATCH_FLOATS          # the plain ensemble's limit is unchanged
    lib = _lib.lib()
    P = int(lib.hb_de_num_params(C.byref(spec)))
    need = int(lib.hb_de_fit_workspace_bytes(C.byref(spec), 1))
    prm = _dev(raw0[:, :P])
    ws = torch.zeros(need, dtype=torch.uint8, device="cuda")
    losses = torch.zeros(1, 1, device="cuda")
    xc, yd = _dev(Xc), _dev(y)
    st = lib.hb_de_fit(_lib.ptr(xc), None, _lib.ptr(yd), n, C.byref(spec), 1, _lib.ptr(prm), LR, L1, Bmax + 1, 1,
                       None, 7, _lib.ptr(losses), _lib.ptr(ws), need, _lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == _lib.HB_OK and bool(torch.isfinite(prm).all())
