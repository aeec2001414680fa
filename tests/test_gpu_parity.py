"""GPU parity tests (run with -m gpu on an H100).  Everything goes through the reference-facing classes,
i.e. through the C ABI of libhebo_b200.so; the oracle is only the checker.

Tolerances (BASELINE.md section 5 / north_star):
    |d mu|    <= 1e-4 * max(|mu|, std_y)          vs the fp64 oracle
    |d sigma| <= 1e-4 * sigma
    loss / gradient 1e-4 scale-relative
    MACE objectives: LCB 1e-4 scale-relative; -logEI / -logPI through the reference's own fp32 error budget
    (tests/util.py PHI_BUDGET); Pareto index set identical to the dominance test on the GPU's F;
    argmin mu / argmax sigma over the golden front identical.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import hebo_b200
from hebo_b200 import _lib
from hebo_b200.pareto import pareto_front
from oracle import gp_oracle as O
from tests.util import assert_mace_close, load_golden, mu_sigma_errors, oracle_posterior, seeded_problem

pytestmark = pytest.mark.gpu

GP_CASES = ["c1_branin", "c2_ackley", "c3_hartmann_warp", "c4_hetero", "rbf", "matern12"]


def _gp_from_golden(g, **extra):
    kind = str(g["kind"])
    conf = dict(kernel=kind, lr=0.01, num_epochs=100, noise_lb=8e-4, pred_likeli=False)
    if g["warp_a"].size:
        conf.update(warp_a=g["warp_a"].astype(np.float32), warp_b=g["warp_b"].astype(np.float32))
    if g["noise_diag"].size:
        conf.update(noise_diag=g["noise_diag"].astype(np.float32))
    conf.update(extra)
    d = g["X"].shape[1]
    return hebo_b200.GP(d, 0, 1, **conf)


def _mu_sigma_ok(mu, var, mu_ref, var_ref, y_std, tol=1e-4):
    mu, var = np.asarray(mu, np.float64).reshape(-1), np.asarray(var, np.float64).reshape(-1)
    emu = np.abs(mu - mu_ref) / np.maximum(np.abs(mu_ref), y_std)
    esg = np.abs(np.sqrt(var) - np.sqrt(var_ref)) / np.sqrt(var_ref)
    return float(emu.max()), float(esg.max())


@pytest.mark.parametrize("case", GP_CASES)
def test_golden_loss_gradient_fit_posterior_mace_front(case):
    g = load_golden(f"gp_{case}.npz")
    X = torch.from_numpy(g["X"])
    y = torch.from_numpy(g["y_transformed"]).reshape(-1, 1)
    d = X.shape[1]
    # ---- loss + gradient at the initial and at the post-fit hypers
    gp = _gp_from_golden(g, num_epochs=0, init_raw=g["raw0"].astype(np.float32))
    gp.fit(X, None, y)
    for which in ("0", "1"):
        gp.set_hypers(torch.from_numpy(g["raw" + which]).float())
        loss, grad = gp.evaluate_loss(return_grad=True)
        assert abs(loss - float(g["loss" + which])) <= 1e-4 * max(1.0, abs(float(g["loss" + which])))
        gref = g["grad" + which]
        # the gradient is a difference of two O(0.5) terms (alpha^T dK alpha vs tr(K^-1 dK), both / 2n): the floor
        # below is 2e-5 of that term scale, i.e. "1e-4 scale-relative" (BASELINE.md section 5)
        assert np.abs(grad.numpy() - gref).max() <= 1e-4 * max(np.abs(gref).max(), 0.1), (case, which)
    # ---- posterior / MACE / front at the post-fit hypers (state from set_hypers(raw1))
    Xs = torch.from_numpy(g["Xs"])
    tau, kappa = float(g["tau"]), float(g["kappa"])
    F, mu, var = gp.predict_mace(Xs, tau, kappa, 1e-4, torch.from_numpy(g["xi1"]), torch.from_numpy(g["xi2"]),
                                 return_mu_var=True)
    emu, esg = _mu_sigma_ok(mu, var, g["mu"], g["var"], float(g["y_std"]))
    # noise floor of the reference's own precision (fp32 oracle vs the fp64 golden) on the same inputs
    warp = (g["warp_a"], g["warp_b"]) if g["warp_a"].size else None
    nd = g["noise_diag"] if g["noise_diag"].size else None
    mu32, var32, _ = oracle_posterior(g["X"], g["y_transformed"], g["raw1"], str(g["kind"]), g["Xs"], torch.float32, warp, nd)
    fmu, fsg = mu_sigma_errors(mu32, var32, g["mu"], g["var"], float(g["y_std"]))
    print(f"{case}: GPU mu/sigma err {emu:.2e}/{esg:.2e}; fp32-reference floor {fmu:.2e}/{fsg:.2e}")
    assert emu <= max(1e-4, 2 * fmu) and esg <= max(1e-4, 2 * fsg), (case, emu, esg, fmu, fsg)
    mu2, var2 = gp.predict(Xs, None)
    assert torch.equal(mu2.reshape(-1), mu) and torch.equal(var2.reshape(-1), var)      # predict == fused path
    assert mu2.shape == (Xs.shape[0], 1) and (var2 > 0).all()
    assert abs(float(gp.noise) - float(g["noise"])) <= 1e-5 * float(g["noise"]) and gp.noise.shape == (1,)
    # (a) epilogue arithmetic alone: fp32 restatement of acq.py:151-171 evaluated on the GPU's own mu / var
    F32 = O.mace(mu, var, float(gp.noise), tau, kappa, 1e-4, torch.from_numpy(g["xi1"]), torch.from_numpy(g["xi2"]))
    assert_mace_close(F.numpy(), F32.numpy(), mu.numpy(), var.numpy(), float(gp.noise), tau, 1e-4, g["xi2"], what=case)
    # (b) end to end against the fp64 golden objectives: -logEI / -logPI ~ z^2/2 amplify the (<= 1e-4) sigma and mu
    #     deviations by up to 2x + 1x, hence 5e-4 here
    assert_mace_close(F.numpy(), g["F"], g["mu"], g["var"], float(g["noise"]), tau, 1e-4, g["xi2"], rtol=5e-4, what=case)
    idx = pareto_front(F.cuda()).cpu().numpy()
    assert np.array_equal(idx, O.pareto_front(F.numpy()))
    front = g["front"]
    assert int(np.argmin(mu.numpy()[front])) == int(g["argmin_mu"])
    assert int(np.argmax(var.numpy()[front])) == int(g["argmax_sigma"])
    # ---- 100-epoch pSGLD fit with the golden Langevin draws ends at the golden hypers
    gpf = _gp_from_golden(g, init_raw=g["raw0"].astype(np.float32), langevin=g["langevin"])
    gpf.fit(X, None, y)
    assert np.abs(gpf.losses - g["losses"]).max() <= 2e-4 * max(1.0, np.abs(g["losses"]).max())
    assert np.abs(gpf.raw.numpy() - g["raw1"]).max() <= 2e-3, np.abs(gpf.raw.numpy() - g["raw1"]).max()


def test_reference_mace_vectors_through_the_epilogue_entry_point():
    """hb_mace_epilogue on the reference's own MACE.eval inputs/outputs (tests/golden/ref_mace.npz)."""
    lib = _lib.lib()
    g = load_golden("ref_mace.npz")
    for ci in range(4):
        mu = torch.from_numpy(g[f"c{ci}_mu"]).reshape(-1).cuda()
        var = torch.from_numpy(g[f"c{ci}_var"]).reshape(-1).cuda()
        xi1 = torch.from_numpy(g[f"c{ci}_xi1"]).reshape(-1).cuda()
        xi2 = torch.from_numpy(g[f"c{ci}_xi2"]).reshape(-1).cuda()
        tau, kappa, noise, eps = g[f"c{ci}_par"]
        F = torch.empty(mu.numel(), 3, device="cuda")
        st = lib.hb_mace_epilogue(_lib.ptr(mu), _lib.ptr(var), mu.numel(), float(noise), float(np.float32(tau)),
                                  float(kappa), float(eps), _lib.ptr(xi1), _lib.ptr(xi2), 0, _lib.ptr(F), _lib.stream_ptr())
        _lib.check(st, "hb_mace_epilogue")
        Fr = g[f"c{ci}_F"]
        assert np.array_equal(np.isnan(F.cpu().numpy()), np.isnan(Fr))
        ok, ill = assert_mace_close(F.cpu().numpy(), Fr, g[f"c{ci}_mu"], g[f"c{ci}_var"], float(noise),
                                    float(np.float32(tau)), float(eps), g[f"c{ci}_xi2"], what=f"ref case {ci}")
        assert ok >= 100


@pytest.mark.parametrize("kind,n,d,m,pred_likeli", [("matern32", 700, 10, 3001, False), ("matern52", 333, 3, 1000, True),
                                                    ("rbf", 1100, 17, 2500, False)])
def test_live_oracle_parity_unaligned_shapes(kind, n, d, m, pred_likeli):
    X, y = seeded_problem(n, d, 11 + n)
    np.random.seed(1)
    gp = hebo_b200.GP(d, 0, 1, kernel=kind, lr=0.01, num_epochs=5, noise_lb=8e-4, pred_likeli=pred_likeli, langevin=False,
                      m_chunk=1024)
    gp.fit(X, None, y)
    Xt64 = gp.xscaler.scale_.double() * X.double() + gp.xscaler.min_.double()
    yt64 = (y.double().reshape(-1) - float(gp.yscaler.mean[0])) / float(gp.yscaler.std[0])
    hp = O.fit_psgld(Xt64, yt64, O.Hypers.unpack(gp.raw_init.double(), 8e-4), kind, lr=0.01, num_epochs=5)
    assert float((hp.pack() - gp.raw.double()).abs().max()) < 1e-4
    f = O.FittedGP(Xt64, O.Hypers.unpack(gp.raw.double(), 8e-4), kind, gp.xscaler.scale_.double(), gp.xscaler.min_.double(),
                   float(gp.yscaler.mean[0]), float(gp.yscaler.std[0]), pred_likeli=pred_likeli)
    f._yt = yt64
    O.refactor(f)
    g = torch.Generator().manual_seed(5)
    Xs = torch.rand(m, d, generator=g) * 2.4 - 1.2
    Xs[:50] = X[:50]                                   # exact training points: the sigma^2 cancellation case
    mu, var = gp.predict(Xs, None)
    mu64, var64 = O.predict(f, Xs.double())
    emu, esg = _mu_sigma_ok(mu, var, mu64.numpy().reshape(-1), var64.numpy().reshape(-1), float(gp.yscaler.std[0]))
    mu32, var32, _ = oracle_posterior(X, y, gp.raw, kind, Xs, torch.float32, pred_likeli=pred_likeli)
    fmu, fsg = mu_sigma_errors(mu32, var32, mu64.numpy().reshape(-1), var64.numpy().reshape(-1), float(gp.yscaler.std[0]))
    print(f"{kind} n={n}: GPU mu/sigma err {emu:.2e}/{esg:.2e}; fp32-reference floor {fmu:.2e}/{fsg:.2e}")
    assert emu <= max(1e-4, 2 * fmu) and esg <= max(1e-4, 2 * fsg), (emu, esg, fmu, fsg)
    # chunking must not change a single bit
    gp.m_chunk = 8192
    mu_b, var_b = gp.predict(Xs, None)
    assert torch.equal(mu, mu_b) and torch.equal(var, var_b)
    # device tensors in -> device tensors out
    mu_d, var_d = gp.predict(Xs.cuda(), None)
    assert mu_d.is_cuda and torch.equal(mu_d.cpu(), mu)


@pytest.mark.parametrize("optimizer,epochs,lr", [("adam", 40, 0.05), ("lbfgs", 8, 0.5)])
def test_fit_with_the_reference_other_optimizers(optimizer, epochs, lr):
    """gp.py:96-101: optimizer='lbfgs' / Adam.  torch's optimizer objects drive the raw vector, every closure is one
    hb_mll_fwd_bwd; compared with the same optimizer on the fp64 oracle's autograd loss."""
    n, d = 150, 4
    X, y = seeded_problem(n, d, 21)
    np.random.seed(3)
    gp = hebo_b200.GP(d, 0, 1, lr=lr, num_epochs=epochs, noise_lb=8e-4, optimizer=optimizer, pred_likeli=False)
    gp.fit(X, None, y)
    Xt64 = gp.xscaler.scale_.double() * X.double() + gp.xscaler.min_.double()
    yt64 = (y.double().reshape(-1) - float(gp.yscaler.mean[0])) / float(gp.yscaler.std[0])
    hp, losses = O.fit_torch_optimizer(Xt64, yt64, O.Hypers.unpack(gp.raw_init.double(), 8e-4), optimizer, "matern32", lr=lr,
                                       num_epochs=epochs, record=True)
    final_gpu = gp.evaluate_loss()
    final_ref = float(O.neg_mll(Xt64, yt64, hp))
    print(f"{optimizer}: loss {gp.losses[0]:.5f} -> {final_gpu:.5f} (oracle {losses[0]:.5f} -> {final_ref:.5f}), "
          f"max |raw diff| {float((hp.pack() - gp.raw.double()).abs().max()):.2e}")
    assert abs(gp.losses[0] - losses[0]) < 1e-4 and final_gpu < gp.losses[0] - 0.05
    if optimizer == "adam":          # smooth deterministic rule: the trajectories agree
        assert np.abs(gp.losses - np.array(losses)).max() < 2e-4
        assert float((hp.pack() - gp.raw.double()).abs().max()) < 2e-3
    else:                            # line-search decisions may differ at fp32 loss resolution; the optimum reached may not
        assert final_gpu < final_ref + 1e-3
    mu, var = gp.predict(X[:20], None)
    assert torch.isfinite(mu).all() and (var > 0).all()


def test_full_size_properties_n4096_d32():
    """BASELINE headline size: size-independent properties instead of an fp64 oracle run."""
    n, d, m = 4096, 32, 10000
    X, y = seeded_problem(n, d, 77)
    np.random.seed(0)
    gp = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=3, noise_lb=8e-4, pred_likeli=False, langevin=False)
    gp.fit(X, None, y)
    assert np.isfinite(gp.losses).all() and gp.losses[-1] < gp.losses[0]
    L = gp.L_dev.tril()
    Linv = gp.Linv_dev
    # L^-1 L = I on a row sample; L L^T reproduces Khat on a sample of entries (via the Gram entry point)
    rows = torch.arange(0, n, 97, device="cuda")
    eye = Linv[rows].double() @ L.double()
    ref = torch.zeros_like(eye)
    ref[torch.arange(rows.numel()), rows] = 1.0
    assert float((eye - ref).abs().max()) < 5e-4
    lib = _lib.lib()
    K = torch.empty(gp.NP, gp.NP, device="cuda")
    _lib.check(lib.hb_gram(_lib.ptr(gp._XtT), n, d, _lib.ptr(gp.hyp_dev), gp.kern_id, None, 0.0, _lib.ptr(K), _lib.stream_ptr()), "gram")
    LLt = (L[rows].double() @ L.double().t())
    Kfull = torch.tril(K) + torch.tril(K, -1).t()
    assert float((LLt - Kfull[rows].double()).abs().max()) < 1e-4 * float(Kfull.abs().max())
    # Khat alpha = y - c
    r = (gp._y_dev - gp.hyp_dev[1]).double()
    resid = Kfull[:n, :n].double() @ gp.alpha_dev[:n].double() - r
    assert float(resid.abs().max()) < 2e-3 * float(r.abs().max())
    # posterior: training points are reproduced within the noise level, variance is positive and below the prior
    mu, var = gp.predict(X[:512], None)
    s = float(gp.hyp[2]) * float(gp.yscaler.std[0]) ** 2
    assert (var > 0).all() and float(var.max()) <= s * (1 + 1e-5)
    assert float((mu - y[:512]).abs().mean()) < 0.5 * float(y.std())
    # determinism: two fused passes over 10k candidates are bit-identical
    g = torch.Generator().manual_seed(1)
    Xs = (torch.rand(m, d, generator=g) * 2 - 1).cuda()
    xi1, xi2 = torch.randn(m, generator=g).cuda(), torch.randn(m, generator=g).cuda()
    F1 = gp.predict_mace(Xs, float(y.min()), 3.0, 1e-4, xi1, xi2)
    F2 = gp.predict_mace(Xs, float(y.min()), 3.0, 1e-4, xi1, xi2)
    assert torch.equal(F1, F2) and torch.isfinite(F1).all()
    idx = pareto_front(F1).cpu().numpy()
    assert np.array_equal(idx, O.pareto_front(F1.cpu().numpy()))


def test_cholesky_reports_leading_minor_like_lapack():
    lib = _lib.lib()
    NP = 256
    g = torch.Generator().manual_seed(0)
    B = torch.randn(NP, NP, generator=g, dtype=torch.float64)
    A = (B @ B.t() / NP + torch.eye(NP, dtype=torch.float64)).float().cuda()
    ws = torch.empty(128 * 128, device="cuda")
    info = torch.zeros(1, dtype=torch.int32, device="cuda")
    A_ok = A.clone()
    _lib.check(lib.hb_cholesky(_lib.ptr(A_ok), NP, _lib.ptr(ws), _lib.ptr(info), _lib.stream_ptr()), "chol")
    assert int(info.item()) == 0
    Lref = torch.linalg.cholesky(A.double().cpu())
    assert float((A_ok.tril().cpu().double() - Lref).abs().max()) < 1e-5
    for bad in (0, 70, 200):
        A_bad = A.clone()
        A_bad[bad, bad] = -1.0
        info.zero_()
        _lib.check(lib.hb_cholesky(_lib.ptr(A_bad), NP, _lib.ptr(ws), _lib.ptr(info), _lib.stream_ptr()), "chol")
        _, info_ref = torch.linalg.cholesky_ex(A_bad.double().cpu())
        assert int(info.item()) == int(info_ref.item()) == bad + 1


def test_not_positive_definite_escalates_jitter_then_falls_back(capsys):
    # duplicated rows + (almost) no noise floor: plain Cholesky fails, the jitter ladder rescues it (gp.py:117-126)
    X = torch.randn(40, 2)
    X = torch.cat([X, X, X], 0)
    y = torch.sin(X[:, :1])
    raw = torch.tensor([-40.0, 0.0, 0.5, 0.5, 0.5])     # softplus(-40) ~ 4e-18 noise, noise_lb = 1e-12
    gp = hebo_b200.GP(2, 0, 1, num_epochs=0, noise_lb=1e-12, init_raw=raw, pred_likeli=False)
    gp.fit(X, None, y)
    gp.set_hypers(raw)
    assert gp.jitter_used > 0 and not gp._fit_failed
    mu, var = gp.predict(X[:5], None)
    assert torch.isfinite(mu).all() and (var > 0).all()


def test_base_model_contract_like_reference_tests():
    """Mirrors HEBO/test/test_base_model.py for the 'gp' id (cont-only, NaN rows, noise, grad, sample_f)."""
    torch.manual_seed(0)
    Xc = torch.randn(50, 1)
    y = Xc + 1e-2 * torch.randn(50, 1)
    model = hebo_b200.GP(1, 0, 1, num_epochs=1)
    model.fit(Xc, None, y)
    with torch.no_grad():
        py, ps2 = model.predict(Xc, None)
    assert py.shape == (50, 1) and torch.isfinite(py).all() and (ps2 > 0).all()
    assert model.noise.shape == torch.Size([1]) and (model.noise >= 0).all()
    with pytest.raises(NotImplementedError):
        model.sample_f()
    y_nan = y.clone()
    y_nan[0] = np.nan
    model.fit(Xc, None, y_nan)                       # test_fit_with_nan
    assert model.n == 49
    py, ps2 = model.predict(Xc, None)
    assert torch.isfinite(py).all() and (ps2 > 0).all()
    X_tst = torch.randn(50, 1, requires_grad=True)   # test_grad
    py, _ = model.predict(X_tst, None)
    py.sum().backward()
    assert X_tst.grad is not None and torch.isfinite(X_tst.grad).all()
    mu_plain, var_plain = model.predict(X_tst.detach(), None)
    assert torch.allclose(mu_plain, py.detach(), rtol=1e-4, atol=1e-5)
    samp = model.sample_y(Xc[:7], None, 3)
    assert samp.shape == (3, 7, 1) and torch.isfinite(samp).all()


def test_verbose_output_format_like_reference_test_gp(capsys):
    X = torch.randn(10, 1)
    y = torch.randn(10, 1)
    model = hebo_b200.GP(1, 0, 1, num_epochs=10, verbose=True, print_every=5)
    model.fit(X, None, y)
    out = capsys.readouterr()
    assert "After" in out.out and "epochs" in out.out and "loss" in out.out and out.err == ""
    assert out.out.count("After") == 3            # epochs 1, 5, 10 (gp.py:127)


def test_mace_class_num_obj_and_device_rng():
    X, y = seeded_problem(300, 4, 9)
    gp = hebo_b200.GP(4, 0, 1, num_epochs=2, pred_likeli=False, noise_lb=8e-4, lr=0.01, rng="device")
    gp.fit(X, None, y)
    acq = hebo_b200.MACE(gp, best_y=np.float32(y.min()), kappa=2.0)
    Xs = torch.rand(2000, 4) * 2 - 1
    F = acq(Xs, None)
    assert F.shape == (2000, 3) and torch.isfinite(F).all() and acq.num_obj == 3 and acq.num_constr == 0
    Fa = gp.predict_mace(Xs, float(y.min()), 2.0, 1e-4, seed=5)
    Fb = gp.predict_mace(Xs, float(y.min()), 2.0, 1e-4, seed=5)
    Fc = gp.predict_mace(Xs, float(y.min()), 2.0, 1e-4, seed=6)
    assert torch.equal(Fa, Fb) and not torch.equal(Fa, Fc)
    # implied Philox normals: LCB - (mu - kappa sigma) = noise * xi1  ->  xi1 ~ N(0,1)
    mu, var = gp.predict(Xs, None)
    xi = (Fa[:, 0] - (mu.reshape(-1) - 2.0 * var.reshape(-1).sqrt())) / (math.sqrt(2.0) * float(gp.noise.sqrt()))
    assert abs(float(xi.mean())) < 0.1 and abs(float(xi.std()) - 1.0) < 0.1
    # host RNG mode consumes torch's generator exactly like acq.py:154-155
    gp.rng = "host"
    torch.manual_seed(3)
    F1 = acq(Xs, None)
    torch.manual_seed(3)
    xi1, xi2 = torch.randn(2000, 1), torch.randn(2000, 1)
    F2 = gp.predict_mace(Xs, float(np.float32(y.min())), 2.0, 1e-4, xi1, xi2)
    assert torch.equal(F1, F2)


@pytest.mark.parametrize("m", [1, 5, 1000, 40000, 300000])
def test_pareto_front_matches_dominance_oracle(m):
    g = torch.Generator().manual_seed(m)
    F = torch.randn(m, 3, generator=g)
    F[:, 1] = 0.6 * F[:, 0] + 0.4 * F[:, 1]
    if m >= 1000:
        F[10:20] = F[0:10]                 # duplicates never dominate each other
        F[30, 1] = float("nan")            # NaN rows never dominate and are excluded from the front
        F[31] = float("inf")
    idx = pareto_front(F.cuda()).cpu().numpy()
    ref = O.pareto_front(F.numpy()) if m > 5000 else O.pareto_front_bruteforce(F.numpy())
    assert np.array_equal(idx, ref)


@pytest.mark.parametrize("world,m,capacity", [(2, 3000, 256), (8, 20000, 512), (4, 500, 8)])
def test_front_pack_and_merge_kernels_match_the_host_protocol(world, m, capacity):
    """hb_front_pack / hb_front_merge (the device side of the multi-GPU front exchange) against the torch restatements the
    gloo tests run (tests/test_dist.py): same buffers bit for bit, overflow flagged, no host sync needed in between."""
    from hebo_b200.pareto import front_merge, front_pack, front_read, pareto_front_device
    from tests.test_dist import front_fn_torch, merge_fn_torch, pack_fn_torch
    g = torch.Generator().manual_seed(m)
    bufs_dev, bufs_ref = [], []
    for r in range(world):
        F = torch.randn(m, 3, generator=g)
        F[:, 2] = 0.5 * F[:, 0] + 0.5 * F[:, 2]
        mu, var = torch.randn(m, generator=g), torch.rand(m, generator=g) + 0.1
        off = r * m + (1 << 25)
        idx, cnt = pareto_front_device(F.cuda())
        bufs_dev.append(front_pack(F.cuda(), mu.cuda(), var.cuda(), idx, cnt, off, capacity))
        bufs_ref.append(pack_fn_torch(F, mu, var, *front_fn_torch(F), off, capacity))
        a, b = bufs_dev[-1].cpu(), bufs_ref[-1]
        sig = 4                                              # sigma column: device sqrtf vs torch CPU sqrt may differ by 1 ulp
        assert torch.equal(a[:, :sig], b[:, :sig]) and torch.equal(a[:, sig + 1:], b[:, sig + 1:])
        assert torch.allclose(a[:, sig], b[:, sig], rtol=2e-7, atol=0)
    out = front_merge(torch.stack(bufs_dev).contiguous(), world, capacity)
    ref = merge_fn_torch(torch.stack([t.cpu() for t in bufs_dev]), world, capacity)     # same inputs, bit for bit
    assert torch.equal(out.cpu(), ref)
    if capacity >= 64:
        gid, Ff, extra = front_read(out)
        assert torch.equal(gid, torch.sort(gid).values) and Ff.shape[0] == int(ref[0, 0])
    else:
        with pytest.raises(RuntimeError):
            front_read(out)


def test_pareto_all_equal_points_all_survive():
    F = torch.ones(300, 3).cuda()
    assert pareto_front(F).numel() == 300


@pytest.mark.parametrize("n,d", [(7, 3), (64, 2), (1000, 5), (2500, 4)])
def test_lengthscale_init_kernel_matches_torch_pdist_median(n, d):
    """hb_median_pdist == torch.pdist(...).median().clamp(min=0.02) per dimension (gp_util.py:47-52), bit for bit."""
    lib = _lib.lib()
    g = torch.Generator().manual_seed(n)
    X = torch.rand(n, d, generator=g) * 2 - 1
    X[:, 0] = torch.round(X[:, 0] * 4) / 4            # ties / zero differences
    NP = int(lib.hb_padded_n(n))
    XtT = torch.zeros(d, NP, device="cuda")
    XtT[:, :n] = X.t().cuda()
    k = min(n, 1000)
    rng = np.random.RandomState(0)
    idx = np.stack([rng.choice(n, k, replace=False) for _ in range(d)]).astype(np.int32)
    idx_dev = torch.from_numpy(idx).cuda()
    out = torch.empty(d, device="cuda")
    _lib.check(lib.hb_median_pdist(_lib.ptr(XtT), n, d, _lib.ptr(idx_dev), k, 0.02, _lib.ptr(out), _lib.stream_ptr()), "median")
    ref = torch.stack([torch.pdist(X[torch.from_numpy(idx[i]).long(), i].view(-1, 1)).median().clamp(min=0.02) for i in range(d)])
    assert torch.equal(out.cpu(), ref)


@pytest.mark.parametrize("NP", [128, 384, 640, 1152])
def test_cholesky_two_level_blocking_shapes(NP):
    """Outer-block boundaries (512) and partial last blocks: factor, compare with LAPACK in fp64."""
    lib = _lib.lib()
    g = torch.Generator().manual_seed(NP)
    B = torch.randn(NP, 64, generator=g, dtype=torch.float64)
    A64 = B @ B.t() / 64 + torch.diag(torch.rand(NP, generator=g, dtype=torch.float64) + 0.5)
    A = A64.float().cuda()
    ws = torch.empty(128 * 128, device="cuda")
    info = torch.zeros(1, dtype=torch.int32, device="cuda")
    _lib.check(lib.hb_cholesky(_lib.ptr(A), NP, _lib.ptr(ws), _lib.ptr(info), _lib.stream_ptr()), "chol")
    assert int(info.item()) == 0
    Lref = torch.linalg.cholesky(A64.float().double())
    err = float((A.tril().cpu().double() - Lref).abs().max() / Lref.abs().max())
    assert err < 2e-6, err


@pytest.mark.parametrize("hetero", [False, True])
@pytest.mark.parametrize("kind", ["matern32", "matern52", "rbf"])
def test_stage_chain_equals_fused_mll_fwd_bwd_bitwise(kind, hetero):
    """The seven single-stage entry points (transform, gram, cholesky, tri_inverse, solve_logdet, kinv, mll_grad) and the
    fused hb_mll_fwd_bwd -- with a NULL spec and with the numeric ARD spec the model passes -- run the same FP32 SIMT kernels
    in the same order: loss and gradient are bit-identical, and GP.evaluate_loss returns exactly those values."""
    lib = _lib.lib()
    n, d = 700, 5
    X, y = seeded_problem(n, d, 17)
    nd = (1e-2 * (1 + (X.double() ** 2).sum(1) / d)).float() if hetero else None
    np.random.seed(0)
    gp = hebo_b200.GP(d, 0, 1, kernel=kind, lr=0.01, num_epochs=3, noise_lb=8e-4, pred_likeli=False, langevin=False,
                      noise_diag=nd)
    gp.fit(X, None, y)
    NP, st, dev = gp.NP, _lib.stream_ptr(), gp.device
    XtT, yd, raw, ndd = _lib.ptr(gp._XtT), _lib.ptr(gp._y_dev), _lib.ptr(gp._raw_dev), _lib.ptr(gp._nd_dev)
    f32 = dict(dtype=torch.float32, device=dev)
    ws_bytes = int(lib.hb_fit_workspace_bytes(n, d))     # holds the solve and gradient workspaces: an upper bound for each
    hyp, alpha, grad, loss = torch.empty(d + 3, **f32), torch.empty(NP, **f32), torch.empty(d + 3, **f32), torch.empty(1, **f32)
    K, Linv, tmp = (torch.empty(NP, NP, **f32) for _ in range(3))
    cholws = torch.empty(128 * 128, **f32)
    scal = torch.empty(2, dtype=torch.float64, device=dev)
    sws, gws = (torch.empty(ws_bytes, dtype=torch.uint8, device=dev) for _ in range(2))
    info = torch.zeros(1, dtype=torch.int32, device=dev)
    _lib.check(lib.hb_transform_hypers(raw, d, float(gp.noise_lb), _lib.ptr(hyp), st), "transform")
    _lib.check(lib.hb_gram(XtT, n, d, _lib.ptr(hyp), gp.kern_id, ndd, 0.0, _lib.ptr(K), st), "gram")
    _lib.check(lib.hb_cholesky(_lib.ptr(K), NP, _lib.ptr(cholws), _lib.ptr(info), st), "cholesky")
    _lib.check(lib.hb_tri_inverse(_lib.ptr(K), NP, _lib.ptr(Linv), _lib.ptr(tmp), st), "tri_inverse")
    _lib.check(lib.hb_solve_logdet(_lib.ptr(K), _lib.ptr(Linv), yd, n, NP, _lib.ptr(hyp), _lib.ptr(alpha), _lib.ptr(scal),
                                   _lib.ptr(sws), st), "solve_logdet")
    _lib.check(lib.hb_kinv(_lib.ptr(Linv), NP, _lib.ptr(tmp), st), "kinv")
    _lib.check(lib.hb_mll_grad(XtT, n, d, raw, _lib.ptr(hyp), gp.kern_id, _lib.ptr(tmp), _lib.ptr(alpha), _lib.ptr(scal),
                               float(gp.noise_guess), _lib.ptr(grad), _lib.ptr(loss), _lib.ptr(gws), st), "mll_grad")
    assert int(info.item()) == 0 and torch.isfinite(grad).all() and torch.isfinite(loss).all()
    for spec in (None, C.byref(gp._spec)):
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        grad2, loss2, info2 = torch.empty_like(grad), torch.empty_like(loss), torch.zeros_like(info)
        _lib.check(lib.hb_mll_fwd_bwd(XtT, None, yd, n, d, spec, raw, gp.kern_id, ndd, float(gp.noise_lb), float(gp.noise_guess),
                                      0.0, _lib.ptr(grad2), _lib.ptr(loss2), _lib.ptr(info2), _lib.ptr(ws), ws_bytes, st),
                   "hb_mll_fwd_bwd")
        assert int(info2.item()) == 0
        assert torch.equal(loss2, loss) and torch.equal(grad2, grad), (kind, hetero, spec is None)
    loss_e, grad_e = gp.evaluate_loss(return_grad=True)
    assert torch.equal(torch.tensor([loss_e], dtype=torch.float32), loss.cpu()) and torch.equal(grad_e, grad.cpu())


def test_tensor_path_guard_recomputes_cancelling_rows_on_fp32():
    """Tensor-core fp16-split path vs the FP32 SIMT path: rows with sigma^2 << s (dense data: heavy cancellation) are
    flagged by the guard and recomputed on the FP32 pipe (fp64 chunk accumulation); the other rows agree to ~1e-5."""
    n, d, m = 700, 3, 3000
    X, y = seeded_problem(n, d, 21)
    np.random.seed(0)
    gp = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=20, noise_lb=8e-4, pred_likeli=False, langevin=False)
    gp.fit(X, None, y)
    g = torch.Generator().manual_seed(2)
    Xs = torch.rand(m, d, generator=g) * 3.0 - 1.5             # inside the data (confident) and outside (prior-like)
    gp.tensor_cores = False
    mu0, v0 = gp.predict(Xs, None)
    gp.tensor_cores = True
    mu1, v1 = gp.predict(Xs, None)
    assert torch.equal(mu0, mu1)
    ratio = (v0 / (float(gp.yscaler.std[0]) ** 2 * float(gp.hyp[2]))).reshape(-1)
    dense, sparse = ratio < 0.10, ratio > 0.15
    assert int(dense.sum()) > 20 and int(sparse.sum()) > 20, (int(dense.sum()), int(sparse.sum()), ratio.quantile(torch.tensor([.01, .1, .5, .9])).tolist())
    rel = ((v1.sqrt() - v0.sqrt()).abs() / v0.sqrt()).reshape(-1)
    # guarded rows: recomputed on the FP32 pipe with fp64 chunk accumulation -- agreement with the plain FP32 SIMT
    # contraction to its own rounding level; unguarded rows: tensor-path bias (<= ~1.3e-5 on ||v||^2 at this size)
    # amplified by at most 1 / (2 * 0.12)
    assert float(rel[dense].max()) < 5e-4, float(rel[dense].max())   # (the plain FP32 running sums are the less accurate side)
    assert float(rel[sparse].max()) < 6e-5, float(rel[sparse].max())
    # and against the fp64 oracle the guarded rows are at least as good as the all-SIMT path
    Xt64 = gp.xscaler.scale_.double() * X.double() + gp.xscaler.min_.double()
    f = O.FittedGP(Xt64, O.Hypers.unpack(gp.raw.double(), 8e-4), "matern32", gp.xscaler.scale_.double(), gp.xscaler.min_.double(),
                   float(gp.yscaler.mean[0]), float(gp.yscaler.std[0]))
    f._yt = (y.double().reshape(-1) - float(gp.yscaler.mean[0])) / float(gp.yscaler.std[0])
    O.refactor(f)
    _, var64 = O.predict(f, Xs.double())
    e0 = ((v0.double().sqrt() - var64.sqrt()).abs() / var64.sqrt()).reshape(-1)
    e1 = ((v1.double().sqrt() - var64.sqrt()).abs() / var64.sqrt()).reshape(-1)
    print(f"guarded rows vs fp64: tensor+guard {float(e1[dense].max()):.2e}, all-SIMT {float(e0[dense].max()):.2e}")
    assert float(e1[dense].max()) <= max(1e-4, 1.05 * float(e0[dense].max()))
    assert float(e1.max()) <= 1e-4, float(e1.max())


def test_bo_loop_on_branin_converges():
    """End-to-end drop-in check on BASELINE config C1's objective: HEBO-style suggest/observe loop (Sobol start-up,
    power transform, CUDA fit, fused MACE scoring, device Pareto front, selection) drives Branin close to its
    optimum 0.3979 within 25 evaluations of batch size 2."""
    from hebo_b200.suggest import HEBO

    def f(X):
        return torch.from_numpy(O.branin(X.double().numpy()))
    torch.manual_seed(0)
    np.random.seed(0)
    opt = HEBO(lb=[-5.0, 0.0], ub=[10.0, 15.0], scramble_seed=3, n_candidates=4096, n_refine=1,
               model_config={"lr": 0.01, "num_epochs": 100, "noise_lb": 8e-4, "pred_likeli": False})
    for it in range(14):
        X = opt.suggest(2)
        assert X.shape == (2, 2) and bool(((X >= opt.lb) & (X <= opt.ub)).all())
        opt.observe(X, f(X).numpy())
    assert opt.X.shape[0] == 28
    assert opt.best_y < 0.3979 + 0.35, opt.best_y      # Sobol alone (28 points) typically sits above 1.0 here
    assert opt.best_x.shape == (1, 2)


def test_empty_and_single_candidate_batches():
    X, y = seeded_problem(150, 4, 2)
    gp = hebo_b200.GP(4, 0, 1, num_epochs=2, pred_likeli=False)
    gp.fit(X, None, y)
    mu, var = gp.predict(torch.zeros(0, 4), None)
    assert mu.shape == (0, 1) and var.shape == (0, 1)
    mu1, var1 = gp.predict(X[:1], None)
    mu5, var5 = gp.predict(X[:5], None)
    assert mu1.shape == (1, 1) and torch.equal(mu1, mu5[:1]) and torch.equal(var1, var5[:1])   # batch composition independent
    F = gp.predict_mace(torch.zeros(0, 4), 0.0, 2.0)
    assert F.shape == (0, 3)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,warp,pred_likeli", [("matern32", False, False), ("matern52", False, True), ("rbf", False, False),
                                                     ("matern32", True, False)])
def test_predict_input_gradients_closed_form_vs_fp64_oracle_autograd(kernel, warp, pred_likeli):
    """support_grad contract (HEBO/test/test_base_model.py:94-108): d mu / d x and d var / d x from the CUDA kernels
    (hb_posterior_grad, closed form) against torch autograd through the fp64 ORACLE's predict (oracle/gp_oracle.py) at the
    same hypers -- 1e-4 of the gradient scale (VERDICT r1: no comparison against a restatement inside the product)."""
    n, d, m = 300, 5, 70
    X, y = seeded_problem(n, d, 31)
    conf = dict(lr=0.01, num_epochs=30, noise_lb=8e-4, pred_likeli=pred_likeli, langevin=False, kernel=kernel)
    wa = wb = None
    if warp:
        g = torch.Generator().manual_seed(3)
        wa, wb = (0.5 + 1.5 * torch.rand(d, generator=g)), (0.5 + 1.5 * torch.rand(d, generator=g))
        conf.update(warp_a=wa.tolist(), warp_b=wb.tolist())
    np.random.seed(0)
    gp = hebo_b200.GP(d, 0, 1, **conf)
    gp.fit(X, None, y)
    g = torch.Generator().manual_seed(4)
    Xs = torch.rand(m, d, generator=g) * 1.6 - 0.8
    Xs[:5] = X[:5]                                         # exact training points
    with torch.no_grad():
        mu0, var0 = gp.predict(Xs.clone(), None)
    wm = torch.randn(m, 1, generator=g)
    wv = torch.randn(m, 1, generator=g)
    xa = Xs.clone().requires_grad_(True)
    mu1, var1 = gp.predict(xa, None)                       # CUDA closed form behind an autograd.Function
    ((wm * mu1).sum() + (wv * var1).sum()).backward()
    # ---- fp64 oracle + autograd
    dt = torch.float64
    sc, mn = gp.xscaler.scale_.to(dt), gp.xscaler.min_.to(dt)
    ym, ys = float(gp.yscaler.mean[0]), float(gp.yscaler.std[0])
    Xt = sc * X.to(dt) + mn
    xb = Xs.to(dt).clone().requires_grad_(True)
    Xm = sc * xb + mn
    if warp:
        Xt, Xm = O.kumaraswamy_warp(Xt, wa.to(dt), wb.to(dt)), O.kumaraswamy_warp(Xm, wa.to(dt), wb.to(dt))
    f = O.FittedGP(Xt, O.Hypers.unpack(gp.raw.to(dt), 8e-4), kernel, torch.ones(d, dtype=dt), torch.zeros(d, dtype=dt), ym, ys,
                   pred_likeli=pred_likeli)
    f._yt = (y.to(dt).reshape(-1) - ym) / ys
    O.refactor(f)
    mu2, var2 = O.predict(f, Xm)
    ((wm.to(dt) * mu2).sum() + (wv.to(dt) * var2).sum()).backward()
    assert mu1.shape == (m, 1) and var1.shape == (m, 1)
    assert torch.allclose(mu1.detach(), mu0, rtol=1e-5, atol=1e-5 * float(y.std()))
    assert torch.allclose(var1.detach(), var0, rtol=2e-4, atol=1e-7)
    emu = float(((mu1.detach().double() - mu2.detach()).abs() / mu2.detach().abs().clamp_min(ys)).max())
    esg_all = ((var1.detach().double().sqrt() - var2.detach().sqrt()).abs() / var2.detach().sqrt()).reshape(-1)
    # rows 0..4 are exact training points (sigma^2 is pure cancellation residue; the gradient path contracts in plain FP32)
    assert emu <= 1e-4 and float(esg_all[5:].max()) <= 1e-4 and float(esg_all[:5].max()) <= 5e-4, (emu, esg_all.max())
    ga, gb = xa.grad.double(), xb.grad
    assert torch.isfinite(ga).all()
    scale = float(gb.abs().max())
    gerr = float((ga - gb).abs().max())
    print(f"{kernel} warp={warp}: input-gradient err {gerr / scale:.2e} of the gradient scale")
    assert gerr <= 1e-4 * scale, (gerr, scale)
    # a finite-difference probe of mu along one coordinate (independent of autograd)
    h = 1e-2
    e0 = torch.zeros(1, d)
    e0[0, 0] = h
    with torch.no_grad():
        mp, _ = gp.predict(Xs[10:11] + e0, None)
        mm, _ = gp.predict(Xs[10:11] - e0, None)
    xc = Xs[10:11].clone().requires_grad_(True)
    gp.predict(xc, None)[0].sum().backward()
    fd = float((mp - mm) / (2 * h))
    assert abs(float(xc.grad[0, 0]) - fd) <= 2e-2 * max(abs(fd), 1e-2)


@pytest.mark.gpu
def test_bo_loop_with_nsga2_acquisition_optimiser():
    """The reference-shaped acquisition optimiser (NSGA-II over the MACE objectives, every generation scored by one fused
    device pass; evolution_optimizer.py:127-160) drives the same loop."""
    from hebo_b200.suggest import HEBO

    def f(X):
        return torch.from_numpy(O.branin(X.double().numpy()))
    torch.manual_seed(0)
    np.random.seed(0)
    opt = HEBO(lb=[-5.0, 0.0], ub=[10.0, 15.0], scramble_seed=3, acq_optimizer="nsga2", evo_pop=50, evo_iters=25,
               model_config={"lr": 0.01, "num_epochs": 100, "noise_lb": 8e-4, "pred_likeli": False})
    for it in range(12):
        X = opt.suggest(2)
        assert X.shape == (2, 2) and bool(((X >= opt.lb) & (X <= opt.ub)).all())
        opt.observe(X, f(X).numpy())
    assert opt.X.shape[0] == 24
    assert opt.best_y < 0.3979 + 0.6, opt.best_y


def test_pinned_host_batch_is_scored_chunkwise_with_identical_results():
    """A pinned host batch larger than one chunk is uploaded chunk by chunk under the scoring (GP._posterior): objectives,
    mu, sigma -- and the in-kernel Philox draws, which are indexed by the global row -- equal the one-call device path."""
    X, y = seeded_problem(400, 6, 13)
    gp = hebo_b200.GP(6, 0, 1, num_epochs=3, pred_likeli=False, noise_lb=8e-4, lr=0.01, rng="device", m_chunk=1024)
    gp.fit(X, None, y)
    g = torch.Generator().manual_seed(1)
    Xs = (torch.rand(5000, 6, generator=g) * 2 - 1).pin_memory()
    Fh, muh, varh = gp.predict_mace(Xs, float(y.min()), 2.0, 1e-4, seed=11, return_mu_var=True, device_out=True)
    Fd, mud, vard = gp.predict_mace(Xs.cuda(), float(y.min()), 2.0, 1e-4, seed=11, return_mu_var=True)
    assert Fh.is_cuda and torch.equal(Fh, Fd) and torch.equal(muh, mud) and torch.equal(varh, vard)
    Fc = gp.predict_mace(Xs, float(y.min()), 2.0, 1e-4, seed=11)          # host in -> host out
    assert not Fc.is_cuda and torch.equal(Fc, Fd.cpu())


@pytest.mark.parametrize("mixed", [False, True])
def test_sample_y_moments_match_the_joint_posterior(mixed):
    """GP.sample_y (gp.py:166-177) through hb_sample_y: with fixed N(0,1) draws the samples are mu + R z with R R^T equal to
    the oracle's joint predictive covariance (checked through the empirical moments of 4000 draws and exactly through the
    mean of antithetic pairs)."""
    n, d, m, S = 300, 3, 40, 4000
    X, y = seeded_problem(n, d, 5)
    torch.manual_seed(0)
    np.random.seed(0)
    if mixed:
        Xe = torch.randint(3, (n, 1))
        y = y + 0.5 * Xe.float()
        gp = hebo_b200.GP(d, 1, 1, num_uniqs=[3], lr=0.01, num_epochs=20, noise_lb=8e-4, pred_likeli=True)
        gp.fit(X, Xe, y)
        Xs, Xse = X[:m] + 0.05, Xe[:m]
    else:
        gp = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=20, noise_lb=8e-4, pred_likeli=False)
        gp.fit(X, None, y)
        Xs, Xse = X[:m] + 0.05, None
    mu, var = gp.predict(Xs, Xse)
    torch.manual_seed(7)
    samp = gp.sample_y(Xs, Xse, S)
    assert samp.shape == (S, m, 1) and torch.isfinite(samp).all()
    sm, sv = samp.mean(0).reshape(-1), samp.var(0).reshape(-1)
    sd = var.reshape(-1).sqrt()
    assert float(((sm - mu.reshape(-1)).abs() / sd).max()) < 5.0 / np.sqrt(S) * 1.5           # mean within ~5 sigma / sqrt(S)
    assert float((sv / (var.reshape(-1) + gp.sample_jitter * gp._y_std ** 2) - 1).abs().max()) < 0.15
    # correlation structure: neighbouring candidates (0.05 apart in some rows of X) are strongly correlated in the joint draw
    if not mixed:
        f = O.FittedGP(gp.xscaler.scale_.double() * X.double() + gp.xscaler.min_.double(), O.Hypers.unpack(gp.raw.double(), 8e-4),
                       "matern32", gp.xscaler.scale_.double(), gp.xscaler.min_.double(), float(gp.yscaler.mean[0]), float(gp.yscaler.std[0]))
        f._yt = (y.double().reshape(-1) - f.y_mean) / f.y_std
        O.refactor(f)
        Z = (f.x_scale * Xs.double() + f.x_min)
        Kss = f.hp.outputscale * O.kernel_matrix(Z, Z, f.hp.lengthscale, "matern32")
        Ks = f.hp.outputscale * O.kernel_matrix(Z, f.Xt, f.hp.lengthscale, "matern32")
        Vo = torch.linalg.solve_triangular(f.L, Ks.T, upper=False)
        cov = (Kss - Vo.T @ Vo) * f.y_std ** 2
        emp = torch.cov(samp.reshape(S, m).double().T)
        scale = float(cov.diag().max())
        assert float((emp - cov).abs().max()) < 0.12 * scale


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs in one process")
def test_two_devices_in_one_process_share_no_state():
    """Per-device lazily built state (kernel attributes, tile tables, schedules, capture streams, pinned status words):
    the same model fitted and scored on cuda:0, then on cuda:1, then on cuda:0 again gives identical bits (the opt-in
    shared-memory attributes are per device: a process-wide `done` flag made the second device's launches fail)."""
    n, d = 700, 6
    X, y = seeded_problem(n, d, 5)
    Xs = torch.rand(3000, d, generator=torch.Generator().manual_seed(2)) * 2 - 1
    out = []
    for dev in ("cuda:0", "cuda:1", "cuda:0"):
        np.random.seed(0)
        torch.manual_seed(0)
        gp = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=12, noise_lb=8e-4, pred_likeli=False, device=dev)
        gp.fit(X, None, y)
        mu, var = gp.predict(Xs, None)
        F = gp.predict_mace(Xs, float(y.min()), 2.0, 1e-4, seed=3)
        out.append((gp.raw.clone(), mu, var, F.cpu()))
    for a, b in ((0, 1), (0, 2)):
        for u, v in zip(out[a], out[b]):
            assert torch.equal(u, v)
