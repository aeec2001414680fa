"""hb_sample_y_batch (GP.sample_y_batch, the device scorer of NoisyAcq) against hb_sample_y and the fp64 oracle, and
NoisyOpt end to end (the reference's test/test_optimizer.py::test_opt[noisy-gp] contract)."""
import numpy as np
import pandas as pd
import pytest
import torch

import hebo_b200
from hebo_b200 import GP, NoisyAcq, NoisyOpt, _lib
from hebo_b200.acq import ga_score
from hebo_b200.space import DesignSpace
from oracle import gp_oracle as O
from tests.util import seeded_problem

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def fitted(mixed, pred_likeli, n=300, d=3):
    X, y = seeded_problem(n, d, 5)
    torch.manual_seed(0)
    np.random.seed(0)
    Xe = None
    if mixed:
        Xe = torch.randint(3, (n, 1))
        y = y + 0.5 * Xe.float()
        gp = GP(d, 1, 1, num_uniqs=[3], lr=0.01, num_epochs=20, noise_lb=8e-4, pred_likeli=pred_likeli)
    else:
        gp = GP(d, 0, 1, lr=0.01, num_epochs=20, noise_lb=8e-4, pred_likeli=pred_likeli)
    gp.fit(X, Xe, y)
    return gp, X, Xe, y


def dev_rows(Xs, Xse):
    return Xs.to(DEV).contiguous(), None if Xse is None else Xse.to(DEV, torch.int32).contiguous()


def reference_draw(gp, Xs, Xse, seed):
    """hb_sample_y on the batch (one sample) and the N(0,1) draws it used."""
    torch.manual_seed(seed)
    ref = gp.sample_y(Xs, Xse, 1).reshape(-1)
    torch.manual_seed(seed)
    z = torch.randn(1, Xs.shape[0]).reshape(-1)
    return ref, z, gp.sample_jitter


def device_draw(gp, Xs, Xse, z=None, seed=0, counter=0):
    xs, xe = dev_rows(Xs, Xse)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    jit = torch.zeros(1, device=DEV)
    f = gp.sample_y_batch(xs, xe, seed, counter, z=None if z is None else z.to(DEV).contiguous(), status=status, jitter=jit)
    torch.cuda.synchronize()
    return f.cpu(), float(jit.item()), int(status.item())


@pytest.mark.parametrize("mixed", [False, True])
@pytest.mark.parametrize("pred_likeli", [False, True])
def test_same_draws_give_the_same_sample(mixed, pred_likeli):
    """With the same z, f equals hb_sample_y's sample up to the rounding of the two fp32 factorisations.  Both factor the
    same fp32 matrix (the covariance stages are shared and give the same bits); the tile-DAG Cholesky and the one-CTA
    right-looking Cholesky only sum in a different order, so R differs by the forward error of an fp32 Cholesky, about
    kappa u relative (u = 6e-8).  The bound is 2e-5 sigma_max (sigma_max: the largest posterior standard deviation of the
    batch): kappa up to ~300 for these well-separated rows; the H100 measured at most 6e-7 sigma_max.  The antithetic mean
    (z and -z) is mu of GP.predict."""
    gp, X, Xe, y = fitted(mixed, pred_likeli)
    m = 100
    g = torch.Generator().manual_seed(3)
    Xs = (torch.rand(m, X.shape[1], generator=g) * 2 - 1)
    Xse = None if Xe is None else torch.randint(3, (m, 1), generator=g)
    ref, z, jref = reference_draw(gp, Xs, Xse, 11)
    f, jit, st = device_draw(gp, Xs, Xse, z)
    assert st == _lib.HB_OK and jit == jref
    mu, var = gp.predict(Xs, Xse)
    mu, sd = mu.reshape(-1), var.reshape(-1).sqrt()
    err = float((f - ref).abs().max())
    print(f"max |f - hb_sample_y| = {err:.3e}, sigma_max = {float(sd.max()):.3e}")
    assert err <= 2e-5 * float(sd.max()), err
    fm, _, _ = device_draw(gp, Xs, Xse, -z)
    anti = 0.5 * (f.double() + fm.double())
    assert float((anti - mu.double()).abs().max()) <= 1e-5 * (1.0 + float(mu.abs().max())) + 1e-4 * float(sd.max())


def test_philox_draws_match_the_joint_posterior():
    """In-kernel draws over 4000 counters at m = 40: empirical mean and covariance against the fp64 oracle's joint
    posterior (the construction and tolerances of test_gpu_parity.py::test_sample_y_moments_match_the_joint_posterior)."""
    n, d, m, S = 300, 3, 40, 4000
    X, y = seeded_problem(n, d, 5)
    torch.manual_seed(0)
    np.random.seed(0)
    gp = GP(d, 0, 1, lr=0.01, num_epochs=20, noise_lb=8e-4, pred_likeli=False)
    gp.fit(X, None, y)
    Xs = X[:m] + 0.05
    mu, var = gp.predict(Xs, None)
    xs, _ = dev_rows(Xs, None)
    status, jit = torch.zeros(1, dtype=torch.int32, device=DEV), torch.zeros(1, device=DEV)
    ws = torch.empty(gp.sample_batch_workspace_bytes(m), dtype=torch.uint8, device=DEV)
    samp = torch.stack([gp.sample_y_batch(xs, None, 1234, c, status=status, jitter=jit, ws=ws) for c in range(S)]).cpu()
    assert int(status.item()) == 0 and torch.isfinite(samp).all()
    sm, sv = samp.mean(0), samp.var(0)
    sd = var.reshape(-1).sqrt()
    assert float(((sm - mu.reshape(-1)).abs() / sd).max()) < 5.0 / np.sqrt(S) * 1.5
    assert float((sv / (var.reshape(-1) + float(jit.item()) * gp._y_std ** 2) - 1).abs().max()) < 0.15
    f = O.FittedGP(gp.xscaler.scale_.double() * X.double() + gp.xscaler.min_.double(), O.Hypers.unpack(gp.raw.double(), 8e-4),
                   "matern32", gp.xscaler.scale_.double(), gp.xscaler.min_.double(), float(gp.yscaler.mean[0]), float(gp.yscaler.std[0]))
    f._yt = (y.double().reshape(-1) - f.y_mean) / f.y_std
    O.refactor(f)
    Z = (f.x_scale * Xs.double() + f.x_min)
    Kss = f.hp.outputscale * O.kernel_matrix(Z, Z, f.hp.lengthscale, "matern32")
    Ks = f.hp.outputscale * O.kernel_matrix(Z, f.Xt, f.hp.lengthscale, "matern32")
    Vo = torch.linalg.solve_triangular(f.L, Ks.T, upper=False)
    cov = (Kss - Vo.T @ Vo) * f.y_std ** 2
    emp = torch.cov(samp.double().T)
    assert float((emp - cov).abs().max()) < 0.12 * float(cov.diag().max())
    # the same (seed, counter) gives the same bits, another counter other draws
    a = gp.sample_y_batch(xs, None, 1234, 17, status=status, jitter=jit, ws=ws)
    b = gp.sample_y_batch(xs, None, 1234, 17, status=status, jitter=jit, ws=ws)
    c = gp.sample_y_batch(xs, None, 1234, 18, status=status, jitter=jit, ws=ws)
    assert torch.equal(a, b) and torch.equal(a.cpu(), samp[17]) and not torch.equal(a, c)


def test_ladder_runs_on_the_device():
    """Rows 1e-7 apart far from the data, with the outputscale raised to 1e3: the covariance is s times a matrix of ones
    up to the fp32 rounding of the kernel values (a few ulps, of either sign), so it is numerically singular well past a
    jitter of 1e-6.  The ladder steps past 1e-6, and the device stops at the jitter hb_sample_y stops at."""
    gp, X, _, _ = fitted(False, False)
    raw = gp.raw.clone()
    raw[2] = 1000.0                                                          # softplus(1000) = 1000: the outputscale
    gp.set_hypers(raw)
    m = 64
    Xs = (X.max(0).values + 0.5).repeat(m, 1)
    Xs[:, 0] = 0.1 + torch.arange(m, dtype=torch.float64) * 1e-7           # fp32 spacing at 0.1 is 7.5e-9: all distinct
    assert torch.unique(Xs, dim=0).shape[0] == m
    ref, z, jref = reference_draw(gp, Xs, None, 5)
    assert jref > 1e-6
    f, jit, st = device_draw(gp, Xs, None, z)
    assert st == _lib.HB_OK and jit == jref and torch.isfinite(f).all()


def test_duplicate_rows_leave_the_covariance():
    """Exact duplicates are +inf, the jitter stays at 1e-6, and the distinct rows get what the de-duplicated batch gives."""
    gp, X, Xe, _ = fitted(True, False)
    g = torch.Generator().manual_seed(9)
    k = 40
    Xs = torch.rand(k, X.shape[1], generator=g) * 2 - 1
    Xse = torch.randint(3, (k, 1), generator=g)
    src = torch.tensor([3, 0, 7, 3, 39, 12, 5, 0, 21, 30])                # copies of earlier rows, one copied twice
    at = torch.tensor([5, 9, 14, 20, 41, 44, 45, 47, 48, 49])              # where they go in the batch of 50
    order = torch.full((k + len(src),), -1, dtype=torch.long)
    order[at] = src
    order[order < 0] = torch.arange(k)
    Bs, Bse = Xs[order], Xse[order]
    z = torch.randn(len(order), generator=g)
    f, jit, st = device_draw(gp, Bs, Bse, z)
    first = torch.tensor([int((order[:i] == order[i]).sum()) == 0 for i in range(len(order))])
    assert st == _lib.HB_OK and jit == np.float32(1e-6)
    assert torch.isinf(f[~first]).all() and (f[~first] > 0).all() and torch.isfinite(f[first]).all()
    fd, jd, _ = device_draw(gp, Bs[first], Bse[first], z[first])
    assert jd == jit and torch.equal(f[first], fd)
    Bs2 = Bs.clone()
    Bs2[at[0], 0] += 1e-6                                                   # no longer a duplicate
    f2, _, _ = device_draw(gp, Bs2, Bse, z)
    assert torch.isfinite(f2[at[0]])


def test_graph_capture_replays_bit_for_bit():
    """One scoring call has no host synchronisation: it is captured in a CUDA graph and the replay equals the eager call."""
    gp, X, Xe, _ = fitted(True, True)
    m = 100
    g = torch.Generator().manual_seed(2)
    xs, xe = dev_rows(torch.rand(m, X.shape[1], generator=g) * 2 - 1, torch.randint(3, (m, 1), generator=g))
    status, jit = torch.zeros(1, dtype=torch.int32, device=DEV), torch.zeros(1, device=DEV)
    ws = torch.empty(gp.sample_batch_workspace_bytes(m), dtype=torch.uint8, device=DEV)
    eager = gp.sample_y_batch(xs, xe, 77, 5, status=status, jitter=jit, ws=ws).clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        gp.sample_y_batch(xs, xe, 77, 5, status=status, jitter=jit, ws=ws)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = gp.sample_y_batch(xs, xe, 77, 5, status=status, jitter=jit, ws=ws)
    out.fill_(0.0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager) and int(status.item()) == 0


def test_ga_score_picks_the_device_sampler():
    gp, X, _, _ = fitted(False, False)
    score = ga_score(NoisyAcq(gp, 1, 0), seed=3)
    assert hasattr(score, "status")
    xs = torch.rand(20, X.shape[1], device=DEV) * 2 - 1
    f = score(xs, torch.empty(20, 0, dtype=torch.int32, device=DEV), 4)
    assert f.is_cuda and f.shape == (20,)
    assert torch.equal(f, gp.sample_y_batch(xs, None, 3, 4))
    assert not hasattr(ga_score(NoisyAcq(gp, 2, 0)), "status")             # two columns: the acquisition's own eval


def obj(x: pd.DataFrame) -> np.ndarray:
    return x["x0"].values.astype(float).reshape(-1, 1) ** 2


def test_opt_noisy_gp_contract():
    """test/test_optimizer.py::test_opt[noisy-gp]: the 1-num + 1-cat space, rand_sample = 8, q = 8, the worst y of each
    later batch replaced by inf; here run past the start-up design."""
    space = DesignSpace().parse([{"name": "x0", "type": "num", "lb": -3, "ub": 7},
                                 {"name": "x1", "type": "cat", "categories": ["a", "b", "c"]}])
    np.random.seed(0)
    torch.manual_seed(0)
    opt = NoisyOpt(space, rand_sample=8, model_name="gp")
    assert opt.support_parallel_opt
    for i in range(3):
        rec = opt.suggest(n_suggestions=8)
        assert rec.shape == (8, 2)
        assert ((rec["x0"] >= -3) & (rec["x0"] <= 7)).all() and rec["x1"].isin(["a", "b", "c"]).all()
        if i > 0:
            seen = set(zip(opt.X["x0"].round(12), opt.X["x1"]))
            assert not seen & set(zip(rec["x0"].round(12), rec["x1"]))
        y = obj(rec)
        if i > 0:
            y[np.argmax(y.reshape(-1))] = np.inf
        opt.observe(rec, y)
    assert opt.y.shape[0] == 22


def test_noisy_opt_improves_on_its_start_up_design():
    def f(df):
        x = df[["x0", "x1"]].values.astype(float)
        return ((x - np.array([0.3, -0.2])) ** 2).sum(1, keepdims=True) + 0.01 * rng.standard_normal((len(df), 1))
    rng = np.random.default_rng(0)
    space = DesignSpace().parse([{"name": "x0", "type": "num", "lb": -1, "ub": 1}, {"name": "x1", "type": "num", "lb": -1, "ub": 1}])
    np.random.seed(1)
    torch.manual_seed(1)
    opt = NoisyOpt(space, rand_sample=8, scramble_seed=0)
    rec = opt.suggest(8)
    opt.observe(rec, f(rec))
    start = opt.best_y
    for _ in range(6):
        rec = opt.suggest(4)
        opt.observe(rec, f(rec))
    assert opt.best_y < start - 0.01, (start, opt.best_y)
    assert opt.last_timing["acq_ms"] > 0
    assert isinstance(hebo_b200.NoisyOpt(space), NoisyOpt)
