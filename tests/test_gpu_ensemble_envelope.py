"""hb_de_fit / hb_de_predict / hb_de_predict_grad across the envelope of ensemble.cu (tests/util.py DE_CASES: the 3 x 256
corner with 8 outputs and a prior net, inputs wider than the hidden layer, wide embeddings and one-hot codes, the largest
admitted minibatch, NaN targets, tiny n): with output_noise=False bit for bit against the fp32 restatement
(oracle/ensemble_oracle.py), with output_noise=True per element against the fp64 oracle under a rounding bound."""
import ctypes as C

import numpy as np
import pytest
import torch

from hebo_b200 import _lib
from oracle import ensemble_oracle as EO
from tests.util import (DE_CASES, DE_PRED, U32, de_abs_net, de_adopt_masks, de_case, de_check_against_fp64, de_depth,
                        de_initial, de_kink_units, de_predict_case, de_predict_fp64, gamma32)

pytestmark = pytest.mark.gpu

LR, L1 = 5e-3, 1e-3


def _spec(kw):
    u = (C.c_int32 * max(1, len(kw["num_uniqs"])))(*kw["num_uniqs"])
    s = _lib.DeSpec(kw["num_cont"], len(kw["num_uniqs"]), u,
                    _lib.HB_DE_ONEHOT if kw.get("enum_trans") == "onehot" else _lib.HB_DE_EMBEDDING, kw.get("num_layers", 1),
                    kw.get("num_hiddens", 128), kw.get("num_out", 1), int(kw["output_noise"]), int(kw.get("rand_prior", False)),
                    1e-4)
    return s, u


def _dev(a, dt=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dt).contiguous() if a is not None and np.size(a) else None


def de_fit(kw, raw0, Xc, Xe, y, perm, batch, epochs, seed=7):
    """hb_de_fit from raw0 [E, P]: (status, params, exp_avg, exp_avg_sq, last gradient, losses) on the host."""
    spec, keep = _spec(kw)
    lib = _lib.lib()
    E = raw0.shape[0]
    params = raw0.clone().cuda().contiguous()
    need = int(lib.hb_de_fit_workspace_bytes(C.byref(spec), E))
    ws = torch.zeros(need, dtype=torch.uint8, device="cuda")
    losses = torch.zeros(E, max(1, epochs), device="cuda")
    xc, xe, yd = _dev(Xc), _dev(Xe, torch.int32) if kw["num_uniqs"] else None, _dev(y)
    pd_ = None if perm is None else _dev(perm, torch.int32)
    st = lib.hb_de_fit(_lib.ptr(xc), _lib.ptr(xe), _lib.ptr(yd), y.shape[0], C.byref(spec), E, _lib.ptr(params), LR, L1,
                       batch, epochs, _lib.ptr(pd_), seed, _lib.ptr(losses), _lib.ptr(ws), need, _lib.stream_ptr())
    torch.cuda.synchronize()
    w = ws.view(torch.float32).view(3, E, -1).cpu().numpy()
    return st, params.cpu().numpy(), w[0], w[1], w[2], losses.cpu().numpy()


def de_predict(kw, params, Xs, Xe, xm, xa, ym, ys, member=-1, grad=False):
    spec, keep = _spec(kw)
    lib = _lib.lib()
    E, m, O, dc = params.shape[0], Xs.shape[0], kw.get("num_out", 1), kw["num_cont"]
    pd_ = _dev(params)
    xs, xe = _dev(Xs), _dev(Xe, torch.int32) if kw["num_uniqs"] else None
    xm, xa, ym, ys = _dev(xm), _dev(xa), _dev(ym), _dev(ys)
    mu = torch.empty(m, O, device="cuda")
    var = torch.empty(m, O, device="cuda") if member < 0 else None
    if grad:
        dmu, dvar = torch.empty(m, O, dc, device="cuda"), torch.empty(m, O, dc, device="cuda")
        _lib.check(lib.hb_de_predict_grad(_lib.ptr(xs), _lib.ptr(xe), m, C.byref(spec), E, _lib.ptr(pd_), _lib.ptr(xm),
                                          _lib.ptr(xa), _lib.ptr(ym), _lib.ptr(ys), _lib.ptr(mu), _lib.ptr(var), _lib.ptr(dmu),
                                          _lib.ptr(dvar), _lib.stream_ptr()), "hb_de_predict_grad")
        out = (mu, var, dmu, dvar)
    else:
        _lib.check(lib.hb_de_predict(_lib.ptr(xs), _lib.ptr(xe), m, C.byref(spec), E, _lib.ptr(pd_), _lib.ptr(xm), _lib.ptr(xa),
                                     _lib.ptr(ym), _lib.ptr(ys), member, _lib.ptr(mu), _lib.ptr(var), _lib.stream_ptr()),
                   "hb_de_predict")
        out = (mu, var)
    torch.cuda.synchronize()
    return tuple(None if t is None else t.cpu().numpy() for t in out)


def orders(n, E, epochs, seed):
    g = np.random.default_rng(seed)
    return np.stack([np.stack([g.permutation(n) for _ in range(epochs)]) for _ in range(E)]).astype(np.int32)


def assert_bits(got, want, what):
    bad = EO.mismatches(got, want)
    assert bad == 0, f"{what}: {bad} of {np.size(want)} elements differ"


# ------------------------------------------------------------------------------------------------ a. fit, bit for bit
@pytest.mark.parametrize("case", list(DE_CASES))
def test_fit_equals_the_restatement_bit_for_bit(case):
    c = DE_CASES[case]
    kw, Xc, Xe, y = de_case(case)
    E, n, epochs = c.get("E", 2), c["n"], 2
    raw0 = de_initial(kw, 3, E)
    perm = orders(n, E, epochs, 5)
    st, params, m1, m2, g, _ = de_fit(kw, raw0, Xc, Xe, y, perm, c["batch"], epochs)
    assert st == _lib.HB_OK
    net = EO.Net32(**kw)
    for e in range(min(E, 2)):
        p, a, b, gg = EO.fit32(net, raw0[e].numpy(), Xc, Xe, y, perm[e], LR, L1, c["batch"])
        for what, dv, rv in (("params", params[e], p), ("exp_avg", m1[e], a), ("exp_avg_sq", m2[e], b), ("grad", g[e], gg)):
            assert_bits(dv, rv, f"member {e} {what}")
    if net.prior:       # the prior net moves by the L1 term only: its gradient is +-coef or 0
        coef = (np.float32(1.0) / np.float32(n * net.O)) * np.float32(L1)
        assert set(np.unique(np.abs(g[:, net.prior0:]))) <= {np.float32(0), coef}
        assert not np.array_equal(params[:, net.prior0:], raw0[:, net.prior0:].numpy())


# ------------------------------------------------------------------------------------------------ b. members
def test_members_are_independent():
    kw, Xc, Xe, y = de_case("holes")
    E, n, epochs, batch = 32, 70, 2, 16
    raw0 = de_initial(kw, 4, E)
    perm = orders(n, E, epochs, 6)
    _, params, m1, m2, g, losses = de_fit(kw, raw0, Xc, Xe, y, perm, batch, epochs)
    for e in range(E):
        _, p1, a1, b1, g1, l1 = de_fit(kw, raw0[e:e + 1], Xc, Xe, y, perm[e:e + 1], batch, epochs)
        for what, x, x1 in (("params", params, p1), ("exp_avg", m1, a1), ("exp_avg_sq", m2, b1), ("grad", g, g1),
                            ("losses", losses, l1)):
            assert_bits(x[e], x1[0], f"member {e} {what}")
    net = EO.Net32(**kw)
    for e in (0, 31):
        assert_bits(params[e], EO.fit32(net, raw0[e].numpy(), Xc, Xe, y, perm[e], LR, L1, batch)[0], f"member {e}")


# ------------------------------------------------------------------------------------------------ c. the NLL path
def nll_step_bound(net64, net32, Xc, Xe, y, rows, n):
    """(fp64 gradient, bound) of one NLL minibatch.  The seeds' magnitudes and their errors (the device's expf, log1pf
    and logf within 2, 1 and 1 ulp, CUDA C Programming Guide, Mathematical Functions) go through the same |W| backward
    as de_step_grad_bound's."""
    rows = np.asarray(rows)
    xc = torch.from_numpy(Xc[rows]).double()
    xe = torch.from_numpy(Xe[rows]).long() if net32.uniqs else None
    t = torch.from_numpy(y[rows]).double()
    _, g64 = EO.step_grad(net64, torch.from_numpy(Xc).double(), torch.from_numpy(Xe).long() if net32.uniqs else None,
                          torch.from_numpy(y).double(), rows, L1, n)
    with torch.no_grad():
        zs = []
        h = net64.sigma2[0].register_forward_hook(lambda m_, i_, o_: zs.append(o_))
        mu, s2 = net64(xc, xe)
        h.remove()
        z = zs[0]
    a = de_abs_net(net64)
    za = []
    h = a.sigma2[0].register_forward_hook(lambda m_, i_, o_: za.append(o_))
    mu_a, _ = a(xc.abs(), xe)
    h.remove()
    f, b = de_depth(net32)
    gf, gN = gamma32(f), gamma32(f + b + len(rows) + 12)
    fin = torch.isfinite(t)
    cnt = fin.sum()
    tt = t.nan_to_num()
    sig = torch.sigmoid(z)
    e_mu, e_z = gf * mu_a.detach(), gf * za[0].detach()
    e_s2 = e_z * sig + 8 * U32 * s2
    dif = (tt.abs() + mu.abs() + e_mu)
    A, Bq = 0.5 / s2, 0.5 * dif ** 2 / s2 ** 2
    mag_mu = dif / s2 / cnt
    err_mu = (e_mu / s2 + dif * e_s2 / s2 ** 2 + 4 * U32 * dif / s2) / cnt
    e_sig = e_z * sig * (1 - sig) + 8 * U32 * sig
    e_A = A * (e_s2 / s2 + U32)
    e_B = (dif * e_mu) / s2 ** 2 + Bq * (2 * e_s2 / s2 + 4 * U32)
    mag_z = (A + Bq) * sig / cnt
    err_z = ((e_A + e_B) * sig + (A + Bq) * e_sig) / cnt + 4 * U32 * mag_z
    zero = torch.zeros_like(t)
    s_mu = torch.where(fin, gN * mag_mu + err_mu, zero)
    s_z = torch.where(fin, gN * mag_z + err_z, zero)
    a.zero_grad()
    (s_mu * mu_a + s_z * za[0]).sum().backward()
    ga = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in a.parameters()])
    return g64.numpy(), ga.numpy() + 4 * U32 * L1 / (n * net32.O) + 1e-300


@pytest.mark.parametrize("case", list(DE_CASES))
def test_nll_step_gradient_matches_fp64_and_adam_is_bit_exact(case):
    c = DE_CASES[case]
    kw, Xc, Xe, y = de_case(case, output_noise=True)
    B, _ = EO.minibatch_rule(c["n"], c["batch"])
    rows = np.random.default_rng(8).permutation(c["n"])[:B]
    Xc, Xe, y = Xc[rows], Xe[rows], y[rows]            # one minibatch is the whole data: one step
    raw0 = de_initial(kw, 9, 1)
    st, params, m1, m2, g, _ = de_fit(kw, raw0, Xc, Xe, y, orders(B, 1, 1, 0), B, 1)
    assert st == _lib.HB_OK
    net32, net64 = EO.Net32(**kw), EO.OracleNet(**kw).load_raw(raw0[0].double())
    xc, xe = torch.from_numpy(Xc).double(), torch.from_numpy(Xe).long() if net32.uniqs else None
    with torch.no_grad():
        kinks = de_kink_units(net64, net32, lambda net: net(xc, xe))
    acts32, _, _ = EO.forward32(net32, raw0[0].numpy(), EO.load_inputs32(net32, raw0[0].numpy(), Xc, Xe))
    assert sum(int(k.sum()) for k in kinks.values()) <= B * net32.H * net32.L // 20
    with de_adopt_masks(net64, kinks, acts32):
        g64, bound = nll_step_bound(net64, net32, Xc, Xe, y, np.arange(B), B)
    err = np.abs(g[0].astype(np.float64) - g64)
    print(f"{case}: largest NLL gradient error / bound = {float(np.max(err / bound)):.3g}")
    assert np.all(err <= bound), f"{int((err > bound).sum())} over, worst {float(np.max(err / bound)):.3g} x bound"
    z = np.zeros(net32.P, np.float32)
    p, a, b = EO.adam_update_f32(raw0[0].numpy(), g[0], z, z, 1, LR)
    assert_bits(params[0], p, "params")
    assert_bits(m1[0], a, "exp_avg")
    assert_bits(m2[0], b, "exp_avg_sq")


@pytest.mark.parametrize("case", list(DE_CASES))
def test_nll_losses_track_fp64(case):
    c = DE_CASES[case]
    kw, Xc, Xe, y = de_case(case, output_noise=True)
    raw0 = de_initial(kw, 10, 1)
    perm = orders(c["n"], 1, 2, 11)
    *_, losses = de_fit(kw, raw0, Xc, Xe, y, perm, c["batch"], 2)
    net = EO.OracleNet(**kw).load_raw(raw0[0].double())
    ref = EO.fit(net, torch.from_numpy(Xc).double(), torch.from_numpy(Xe).long() if kw["num_uniqs"] else None,
                 torch.from_numpy(y).double(), perm[0], LR, L1, c["batch"])
    print(f"{case}: losses {losses[0]} fp64 {ref}")
    assert np.allclose(losses[0], ref, rtol=2e-4, atol=0)


# ------------------------------------------------------------------------------------------------ d. predict
@pytest.mark.parametrize("case,E", DE_PRED, ids=[f"{c}-E{e}" for c, e in DE_PRED])
def test_predict_and_input_gradients_equal_the_restatement(case, E):
    kw, net, params, Xs, Xe, xm, xa, ym, ys, pick = de_predict_case(case, E)
    full = de_predict(kw, params, Xs, Xe, xm, xa, ym, ys, grad=True)
    want = EO.predict32(net, params, Xs[pick], Xe[pick], xm, xa, ym, ys, grad=True)
    for what, d, w in zip(("mu", "var", "dmu", "dvar"), full, want):
        assert_bits(d[pick], w, what)
    for m in (1, 15, 16, 17):
        part = de_predict(kw, params, Xs[:m], Xe[:m], xm, xa, ym, ys, grad=True)
        for what, d, f in zip(("mu", "var", "dmu", "dvar"), part, full):
            assert_bits(d, f[:m], f"m = {m} {what}")
    for lo, hi in ((37, 1040), (4090, 4097), (5, 6)):
        part = de_predict(kw, params, Xs[lo:hi], Xe[lo:hi], xm, xa, ym, ys, grad=True)
        for what, d, f in zip(("mu", "var", "dmu", "dvar"), part, full):
            assert_bits(d, f[lo:hi], f"rows {lo}:{hi} {what}")
    plain = de_predict(kw, params, Xs, Xe, xm, xa, ym, ys)
    assert_bits(plain[0], full[0], "mu without gradients")
    assert_bits(plain[1], full[1], "var without gradients")
    for member in sorted({0, E - 1}):
        mu, _ = de_predict(kw, params, Xs, Xe, xm, xa, ym, ys, member=member)
        assert_bits(mu[pick], EO.predict32(net, params, Xs[pick], Xe[pick], xm, xa, ym, ys, member=member)[0], f"member {member}")


@pytest.mark.parametrize("case,E", DE_PRED, ids=[f"{c}-E{e}" for c, e in DE_PRED])
def test_nll_predict_and_input_gradients_match_fp64(case, E):
    """output_noise=True: mu, sigma2 (the s2s member buffer, v + sum s2 / E) and both input gradients (the softplus'
    seed on the sigma2 head in pass 1) per element against fp64 autograd, on chosen rows of m = 4097."""
    kw, net, params, Xs, Xe, xm, xa, ym, ys, pick = de_predict_case(case, E, output_noise=True)
    full = de_predict(kw, params, Xs, Xe, xm, xa, ym, ys, grad=True)
    ref, kinks, units = de_predict_fp64(net, params, Xs[pick], Xe[pick], xm, xa, ym, ys)
    de_check_against_fp64([t[pick] for t in full], ref, kinks, units, f"{case} E={E} NLL")
    part = de_predict(kw, params, Xs[37:1040], Xe[37:1040], xm, xa, ym, ys, grad=True)
    for what, d, f in zip(("mu", "var", "dmu", "dvar"), part, full):
        assert_bits(d, f[37:1040], f"rows 37:1040 {what}")


# ------------------------------------------------------------------------------------------------ e. minibatch order
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 16, 17, 64, 65, 4096, 4097])
def test_device_order_equals_the_restated_order(n):
    kw, Xc, Xe, y = de_case("small-n9", seed=n, m=n)
    E, epochs, batch, seed = 32, 3, 8, 0x5EED0000 + n
    raw0 = de_initial(kw, 13, E)
    _, p_dev, *_, l_dev = de_fit(kw, raw0, Xc, Xe, y, None, batch, epochs, seed)
    perm = np.tile(np.arange(n, dtype=np.int32), (E, epochs, 1))
    for e in (0, 31):
        perm[e] = np.stack([EO.perm(seed, e, t, n) for t in range(epochs)])
    _, p_giv, *_, l_giv = de_fit(kw, raw0, Xc, Xe, y, perm, batch, epochs, seed)
    for e in (0, 31):
        assert_bits(p_dev[e], p_giv[e], f"member {e} params")
        assert_bits(l_dev[e], l_giv[e], f"member {e} losses")


# ------------------------------------------------------------------------------------------------ f. ABI edges
@pytest.mark.parametrize("case", ["corner", "big-batch"])
def test_one_row_over_the_largest_minibatch_is_rejected_without_a_launch(case):
    c = DE_CASES[case]
    kw, Xc, Xe, y = de_case(case)
    raw0 = de_initial(kw, 14, 1)
    lib = _lib.lib()
    lib.hb_launch_count(1)
    st, params, *_ = de_fit(kw, raw0, Xc, Xe, y, None, c["batch"] + 1, 1)
    assert st == _lib.HB_ERR_INVALID and lib.hb_launch_count(0) == 0
    assert_bits(params, raw0.numpy(), "params after a rejected call")
    st, params, *_ = de_fit(kw, raw0, Xc, Xe, y, None, c["batch"], 0)
    assert st == _lib.HB_OK and lib.hb_launch_count(0) == 0
    assert_bits(params, raw0.numpy(), "params after num_epochs = 0")
