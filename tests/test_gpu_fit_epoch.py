"""The fit's MLL loss and gradient on the 3xTF32 tensor-core path -- the only path a pSGLD fit trains on -- against the fp64
closed form, read through the C ABI: hb_fit_ex with one epoch, lr = 0 and no Langevin draws leaves raw unchanged, its
losses[0] is the tensor-core loss at raw and the fit state's grad the tensor-core gradient at raw (the final factorisation
does not touch grad).  Covered: every tile-table shape class of the Cholesky outer update, the triangular-inverse doubling
levels and K^-1 = U U^T up to NP = 4224; the model families whose gradient consumes the tensor-core K^-1; batched slices
that start past 2^31 and 2^32 bytes; captured-graph replays; and that no result depends on the pad columns of Xt or on what
the fit workspace held before the call.

Tolerance: the fp32 closed form (the reference's own precision) gives the floor.  loss: |l_tc - l64| <= max(1e-4 max(1,
|l64|), 2 |l32 - l64|); gradient: |g_tc - g64|_inf <= max(1e-4 max(|g64|_inf, 0.1), 2 |g32 - g64|_inf)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import hebo_b200
from hebo_b200 import _lib
from oracle import emb_oracle as E
from oracle import gp_oracle as O
from oracle import warp_oracle as W
from tests.util import emb_hypers, seeded_problem

pytestmark = pytest.mark.gpu

NOISE_LB = 8e-4
NOISE_GUESS = 0.01


def _same(a, b):
    """Same shape, dtype and bytes (NaN-safe, -0.0 != 0.0)."""
    a, b = torch.as_tensor(a).detach().cpu().contiguous(), torch.as_tensor(b).detach().cpu().contiguous()
    return a.shape == b.shape and a.dtype == b.dtype and a.numpy().tobytes() == b.numpy().tobytes()


class Model:
    """Device inputs of one model as the C ABI takes them (XtT [d, NP] with zero pad columns, y [n], raw [P])."""

    def __init__(self, XtT, y, raw, n, kern=0, Xe=None, spec=None, noise_guess=NOISE_GUESS, H=None, De=0, owner=None):
        self.XtT, self.y, self.raw, self.n, self.kern, self.Xe, self.spec = XtT, y, raw, n, kern, Xe, spec
        self.d = XtT.shape[0]
        self.NP = XtT.shape[1]
        self.noise_guess, self.De, self.owner = noise_guess, De, owner
        self.H = 3 + self.d if H is None else H
        self.P = raw.numel()

    def Xt64(self):
        return self.XtT[:, :self.n].t().double().cpu()

    def y64(self):
        return self.y.double().cpu()


def numeric_model(n, d, seed, kind="matern32"):
    """Numeric ARD model built directly: inputs in [-1, 1], standardised targets, raw = O.init_hypers."""
    X, y = seeded_problem(n, d, seed)
    y = y.reshape(-1)
    y = (y - y.mean()) / y.std()
    NP = int(_lib.lib().hb_padded_n(n))
    XtT = torch.zeros(d, NP, dtype=torch.float32)
    XtT[:, :n] = X.t()
    hp = O.init_hypers(X.double(), y.double(), NOISE_LB, rng=np.random.RandomState(seed))
    return Model(XtT.cuda(), y.float().cuda().contiguous(), hp.pack().float(), n, _lib.KERNEL_IDS[kind])


def gp_model(n, d, seed, **conf):
    """A model family set up through hebo_b200.GP (mixed, warped, shared lengthscale): its device inputs and initial raw."""
    g = torch.Generator().manual_seed(seed)
    X = torch.rand(n, d, generator=g) * 3 - 1
    nu = conf.get("num_uniqs", [])
    Xe = torch.stack([torch.randint(0, u, (n,), generator=g) for u in nu], 1) if nu else None
    y = torch.sin(2 * X[:, 0]) + 0.3 * X[:, -1] ** 2 + 0.05 * torch.randn(n, generator=g)
    if nu:
        y = y + 0.4 * torch.cos(Xe[:, 0].float() * 1.3)
    np.random.seed(seed)
    torch.manual_seed(seed)
    gp = hebo_b200.GP(d, len(nu), 1, lr=0.01, num_epochs=0, noise_lb=NOISE_LB, pred_likeli=False, **conf)
    gp.fit(X, Xe, y.reshape(-1, 1))
    H = 3 + d + (1 if nu else 0) + (2 * d if gp.warp_mode else 0)
    return Model(gp._XtT, gp._y_dev, gp._expand_raw(gp.raw_init.clone()), gp.n, gp.kern_id, gp._Xe_dev, gp._spec_ptr(),
                 gp.noise_guess, H, gp.De, gp)


def hard_raw(raw, d):
    """sigma_n^2 = noise_lb + 1e-4 and halved lengthscales (numeric ARD layout)."""
    r = raw.clone().double()
    r[0] = O.inv_softplus(torch.tensor(1e-4, dtype=torch.float64))
    r[3:3 + d] = O.inv_softplus(O.softplus(r[3:3 + d]) / 2)
    return r.float()


# ---------------------------------------------------------------------------------------------- ABI runners
def _ws(nbytes, fill):
    return torch.full((nbytes,), fill, dtype=torch.uint8, device="cuda")


def _state(m, ws, base=0):
    """Copies of the fit state of the workspace slice at byte offset `base`."""
    lib = _lib.lib()
    fs = _lib.FitState()
    _lib.check(lib.hb_fit_state_ex(C.c_void_p(ws.data_ptr() + base), m.n, m.d, m.spec, C.byref(fs)), "hb_fit_state_ex")

    def view(p, cnt, dt=torch.float32):
        off = p - ws.data_ptr()
        nb = cnt * torch.empty((), dtype=dt).element_size()
        return ws[off:off + nb].view(dt).cpu().clone()

    NP = m.NP
    return dict(grad=view(fs.grad, m.P), loss=view(fs.loss, 1), hyp=view(fs.hyp, m.H),
                L=torch.tril(view(fs.L, NP * NP).view(NP, NP)), Linv=torch.tril(view(fs.Linv, NP * NP).view(NP, NP)),
                alpha=view(fs.alpha, NP), scal=view(fs.scal, 2, torch.float64),
                Zt=view(fs.Zt, (m.d + m.De) * NP).view(m.d + m.De, NP)[:, :m.n].clone())


def run_fit(m, raw=None, E=1, lr=0.0, fill=0, XtT=None):
    lib = _lib.lib()
    wsb = int(lib.hb_fit_workspace_bytes_ex(m.n, m.d, m.spec))
    ws = _ws(wsb, fill)
    r = (m.raw if raw is None else raw).float().cuda().contiguous().clone()
    losses = (C.c_float * E)()
    st = lib.hb_fit_ex(_lib.ptr(m.XtT if XtT is None else XtT), _lib.ptr(m.Xe), _lib.ptr(m.y), m.n, m.d, m.spec, _lib.ptr(r),
                       m.kern, None, NOISE_LB, m.noise_guess, lr, E, None, losses, _lib.ptr(ws), wsb, _lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == _lib.HB_OK, st
    return dict(raw=r.cpu(), losses=torch.tensor(np.array(losses[:E], dtype=np.float32)), **_state(m, ws))


def run_multi(m, Y, raws, E=1, lr=0.0, fill=0, XtT=None):
    """hb_fit_multi_ex over the outputs Y [B, n] from raws [B, P]; one result dict per output slice."""
    lib = _lib.lib()
    B = Y.shape[0]
    stride = int(lib.hb_fit_workspace_bytes_ex(m.n, m.d, m.spec))
    wsb = int(lib.hb_fit_multi_workspace_bytes(m.n, m.d, m.spec, B))
    assert wsb == B * stride
    ws = _ws(wsb, fill)
    r = raws.float().cuda().contiguous().clone()
    losses = (C.c_float * (B * E))()
    status = (C.c_int32 * B)()
    _lib.check(lib.hb_fit_multi_ex(_lib.ptr(m.XtT if XtT is None else XtT), _lib.ptr(m.Xe), _lib.ptr(Y), m.n, m.d, m.spec, B,
                                   _lib.ptr(r), m.kern, None, NOISE_LB, m.noise_guess, lr, E, None, losses, status,
                                   _lib.ptr(ws), wsb, _lib.stream_ptr()), "hb_fit_multi_ex")
    torch.cuda.synchronize()
    assert list(status) == [_lib.HB_OK] * B
    L = torch.tensor(np.array(losses[:B * E], dtype=np.float32)).view(B, E)
    out = [dict(raw=r[b].cpu(), losses=L[b].clone(), **_state(m, ws, b * stride)) for b in range(B)]
    return out, stride


def run_simt(m, raw=None, fill=0, XtT=None, noise_diag=None):
    """hb_mll_fwd_bwd: one loss + gradient on the FP32 SIMT path."""
    lib = _lib.lib()
    wsb = int(lib.hb_fit_workspace_bytes_ex(m.n, m.d, m.spec))
    ws = _ws(wsb, fill)
    r = (m.raw if raw is None else raw).float().cuda().contiguous()
    grad = torch.full((m.P,), float("nan"), device="cuda")
    loss = torch.full((1,), float("nan"), device="cuda")
    info = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    _lib.check(lib.hb_mll_fwd_bwd(_lib.ptr(m.XtT if XtT is None else XtT), _lib.ptr(m.Xe), _lib.ptr(m.y), m.n, m.d, m.spec,
                                  _lib.ptr(r), m.kern, _lib.ptr(noise_diag), NOISE_LB, m.noise_guess, 0.0, _lib.ptr(grad),
                                  _lib.ptr(loss), _lib.ptr(info), _lib.ptr(ws), wsb, _lib.stream_ptr()), "hb_mll_fwd_bwd")
    torch.cuda.synchronize()
    assert int(info.item()) == 0
    st = _state(m, ws)
    del st["Zt"]   # the numeric rows of Zt are a product of the factorisation only
    st.update(grad=grad.cpu(), loss=loss.cpu())
    return st


def run_factorize(m, raw=None, fill=0, XtT=None):
    lib = _lib.lib()
    wsb = int(lib.hb_fit_workspace_bytes_ex(m.n, m.d, m.spec))
    ws = _ws(wsb, fill)
    r = (m.raw if raw is None else raw).float().cuda().contiguous()
    jit = C.c_float(-1.0)
    st = lib.hb_factorize_ex(_lib.ptr(m.XtT if XtT is None else XtT), _lib.ptr(m.Xe), _lib.ptr(m.y), m.n, m.d, m.spec,
                             _lib.ptr(r), m.kern, None, NOISE_LB, C.byref(jit), _lib.ptr(ws), wsb, _lib.stream_ptr())
    torch.cuda.synchronize()
    assert st == _lib.HB_OK and jit.value == 0.0
    out = _state(m, ws)
    del out["grad"], out["loss"]   # not part of the prediction state
    return out


# ---------------------------------------------------------------------------------------------- references
def ref_numeric(m, raw, kind, dtype, noise_diag=None):
    hp = O.Hypers.unpack(raw.to(dtype), NOISE_LB)
    nd = None if noise_diag is None else noise_diag.to(dtype).cpu()
    loss, grad, _ = O.neg_mll_closed_form(m.Xt64().to(dtype), m.y64().to(dtype), hp, kind, m.noise_guess, nd)
    return float(loss), grad.double()


def check(what, tc, ref64, ref32, simt):
    (l_tc, g_tc), (l64, g64), (l32, g32), (l_s, g_s) = tc, ref64, ref32, simt
    g_tc, g_s = g_tc.double(), g_s.double()
    gmax = float(g64.abs().max())
    el, es, ef = abs(l_tc - l64), abs(l_s - l64), abs(l32 - l64)
    eg, egs, egf = (float((g - g64).abs().max()) for g in (g_tc, g_s, g32))
    print(f"{what}: loss err tc {el:.2e} simt {es:.2e} fp32 {ef:.2e} | grad err tc {eg:.2e} simt {egs:.2e} fp32 {egf:.2e} "
          f"(|g|inf {gmax:.2e})")
    assert el <= max(1e-4 * max(1.0, abs(l64)), 2 * ef), (what, el, ef)
    assert eg <= max(1e-4 * max(gmax, 0.1), 2 * egf), (what, eg, egf)


def tc_at(m, raw):
    r = run_fit(m, raw)
    assert _same(r["raw"], raw.float())   # lr = 0: the step leaves raw unchanged
    return float(r["losses"][0]), r["grad"]


def simt_at(m, raw, noise_diag=None):
    r = run_simt(m, raw, noise_diag=noise_diag)
    return float(r["loss"][0]), r["grad"]


# ---------------------------------------------------------------------------------------------- a. tile-table shapes
# n -> NP: 100 -> 128 (one tile; the K^-1 tile overhangs NP), 250 -> 256 (one doubling level, bn = 128), 333 -> 384 (short
# last block), 600 -> 640 (first 512-column outer update), 1100 -> 1152 (partial last panel; b = 1024 with s2 = 128),
# 2048 (no pad rows), 2150 -> 2176 (b = 2048 with s2 = 128), 4096 (the BASELINE headline size), 4100 -> 4224 (124 pad
# rows; b = 4096 with s2 = 128)
SHAPES = [(100, 8), (250, 8), (333, 8), (600, 8), (1100, 8), (2048, 8), (2150, 8), (4096, 32), (4100, 32)]


@pytest.mark.parametrize("n,d", SHAPES, ids=[f"n{n}_d{d}" for n, d in SHAPES])
def test_tensor_core_loss_gradient_against_fp64(n, d):
    m = numeric_model(n, d, 700 + n)
    for name, raw in (("init", m.raw), ("hard", hard_raw(m.raw, d))):
        check(f"matern32 n={n} NP={m.NP} d={d} {name}", tc_at(m, raw), ref_numeric(m, raw, "matern32", torch.float64),
              ref_numeric(m, raw, "matern32", torch.float32), simt_at(m, raw))


# ---------------------------------------------------------------------------------------------- b. model families
FAMILIES = {
    "mixed": dict(d=4, conf={"num_uniqs": [4, 3]}),
    "learned_warp": dict(d=4, conf={"warp": True}),
    "shared_lengthscale": dict(d=6, conf={"ard_kernel": False}),
}


def _family_ref(name, m, raw, dtype, kind="matern32"):
    Xt, y = m.Xt64().to(dtype), m.y64().to(dtype)
    if name == "learned_warp":
        loss, g = W.neg_mll_autograd(Xt, y, raw.to(dtype), NOISE_LB, kind, m.noise_guess)
        return float(loss), g.double()
    Xe = m.Xe.long().cpu() if m.Xe is not None else torch.zeros(m.n, 0, dtype=torch.long)
    hp = emb_hypers(m.owner, raw)
    hp = E.EmbHypers(*(v.to(dtype) if torch.is_tensor(v) else [t.to(dtype) for t in v] if isinstance(v, list) else v
                       for v in (hp.raw_noise, hp.tables, hp.mean, hp.raw_os, hp.raw_ls, hp.raw_ls_e, hp.noise_lb)))
    loss, g = E.neg_mll_emb_closed_form(Xt, Xe, y, hp, m.noise_guess, kind=kind)
    return float(loss), g.double()


@pytest.mark.parametrize("name", list(FAMILIES))
def test_model_family_loss_gradient_against_fp64(name):
    f = FAMILIES[name]
    m = gp_model(2150, f["d"], 31, **f["conf"])
    raw = m.raw
    check(f"{name} n=2150 NP={m.NP}", tc_at(m, raw), _family_ref(name, m, raw, torch.float64),
          _family_ref(name, m, raw, torch.float32), simt_at(m, raw))


@pytest.mark.parametrize("kind", ["matern52", pytest.param("rbf", marks=pytest.mark.xfail(strict=True, reason=(
    "3xTF32 epoch outside the bound for RBF at n = 2150, d = 6, init hypers (H100): gradient error 3.7e-5 of |g|inf 0.24 "
    "against 1.6e-6 on the FP32 SIMT path and an fp32 floor of 7.9e-7; loss error 1.3e-5 against 7.4e-7.  "
    "test_gpu_fit_stages_tc.py::test_rbf_epoch_stages (H100): at cond_1(L) = 1.8e4 every tensor-core stage is within its "
    "bound of one truncation per wgmma instruction (Cholesky c = 0.040, inverse 0.028, K^-1 = U U^T 0.37; under one "
    "truncation per 8-wide k-step K^-1 reaches 1.1); K^-1 carries 3.2e-5 relative error (L^-1: 8.7e-6), and contracting "
    "the fp64 W with it instead of the exact inverse of the same fp32 L moves the gradient by 3.3e-5 of the 3.7e-5")))])
def test_kernel_loss_gradient_against_fp64(kind):
    m = numeric_model(2150, 6, 41, kind)
    for name, raw in (("init", m.raw), ("hard", hard_raw(m.raw, 6))):
        check(f"{kind} n=2150 NP={m.NP} {name}", tc_at(m, raw), ref_numeric(m, raw, kind, torch.float64),
              ref_numeric(m, raw, kind, torch.float32), simt_at(m, raw))


# ---------------------------------------------------------------------------------------------- c. slices past 2^32 bytes
def test_batched_slices_past_4gib_match_single_fits():
    n, d = 4096, 8
    m = numeric_model(n, d, 77)
    stride = int(_lib.lib().hb_fit_workspace_bytes(n, d))
    B = (1 << 32) // stride + 2   # smallest B whose last slice starts beyond 2^32 bytes
    assert (B - 1) * stride > (1 << 32) >= (B - 2) * stride and B <= _lib.HB_MAX_OUTPUTS
    print(f"slice {stride / 2 ** 30:.3f} GiB, B = {B}, last slice at {(B - 1) * stride / 2 ** 30:.3f} GiB")
    g = torch.Generator().manual_seed(8)
    Y = torch.stack([m.y.cpu() * (1 + 0.1 * b) + 0.2 * torch.randn(n, generator=g) for b in range(B)])
    Y = ((Y - Y.mean(1, keepdim=True)) / Y.std(1, keepdim=True)).cuda().contiguous()
    raws = torch.stack([m.raw + 0.05 * b * torch.randn(m.P, generator=g) for b in range(B)])
    outs, _ = run_multi(m, Y, raws)
    for b in range(B):
        mb = Model(m.XtT, Y[b].contiguous(), raws[b], n)
        single = run_fit(mb)
        for key in ("raw", "losses", "grad"):
            assert _same(outs[b][key], single[key]), (b, key)
    mb = Model(m.XtT, Y[B - 1].contiguous(), raws[B - 1], n)
    raw = raws[B - 1]
    check(f"slice {B - 1} of {B}", (float(outs[B - 1]["losses"][0]), outs[B - 1]["grad"]),
          ref_numeric(mb, raw, "matern32", torch.float64), ref_numeric(mb, raw, "matern32", torch.float32), simt_at(mb, raw))


# ---------------------------------------------------------------------------------------------- d. replays
def test_replayed_epochs_at_zero_lr_are_bit_identical():
    m = numeric_model(1100, 8, 91)
    one = run_fit(m, E=1)
    many = run_fit(m, E=20)   # one direct epoch, then replays of the captured epoch
    assert _same(many["raw"], m.raw)
    assert all(_same(many["losses"][e], many["losses"][0]) for e in range(20))
    assert _same(many["losses"][0], one["losses"][0]) and _same(many["grad"], one["grad"])


# ---------------------------------------------------------------------------------------------- e. undefined memory
def _e_model(name):
    if name == "numeric":
        return numeric_model(300, 5, 55)
    return gp_model(300, 4, 56, **({"num_uniqs": [4, 3]} if name == "mixed" else {"warp": True}))


def _run_entry(entry, m, fill, XtT):
    if entry == "fit":
        return [run_fit(m, E=6, lr=0.01, fill=fill, XtT=XtT)]
    if entry == "fit_multi":
        Y = torch.stack([m.y, m.y.flip(0)]).contiguous()
        raws = torch.stack([m.raw, m.raw + 0.1])
        return run_multi(m, Y, raws, E=6, lr=0.01, fill=fill, XtT=XtT)[0]
    if entry == "mll_fwd_bwd":
        return [run_simt(m, fill=fill, XtT=XtT)]
    return [run_factorize(m, fill=fill, XtT=XtT)]


POISON = [(pad, fill) for pad in ("0", "nan", "inf", "1e30") for fill in (0x00, 0xFF) if (pad, fill) != ("0", 0x00)]


@pytest.mark.parametrize("pad,fill", POISON, ids=[f"pad_{p}-ws_{f:#04x}" for p, f in POISON])
@pytest.mark.parametrize("entry", ["fit", "fit_multi", "mll_fwd_bwd", "factorize"])
@pytest.mark.parametrize("model", ["numeric", "mixed", "learned_warp"])
def test_results_do_not_depend_on_pad_columns_or_workspace_contents(model, entry, pad, fill):
    m = _e_model(model)
    assert m.NP > m.n
    ref = _run_entry(entry, m, 0x00, m.XtT)
    XtT = m.XtT.clone()
    XtT[:, m.n:] = float(pad)
    got = _run_entry(entry, m, fill, XtT)
    for b, (r, g) in enumerate(zip(ref, got)):
        assert r.keys() == g.keys()
        for key in r:
            assert _same(r[key], g[key]), (b, key)
