"""The checkers of tests/test_gpu_large_training.py on the CPU: on an exact-structure clustered state built in torch fp32
they pass, and they flag one off-cluster element set to 1e-30 and one diagonal-block element of the refined L^-1 moved
just past its bound.  The fp64 MLL reference summed over clusters equals oracle.gp_oracle.neg_mll_closed_form."""
import math

import pytest
import torch

from oracle import gp_oracle as O
from tests.test_gpu_large_training import (C_MAX, U, check_block, check_totals, khat_block, mll_assemble, mll_sum,
                                           mll_terms, off_cluster_nonzeros)

F64 = torch.float64
SIZE, NCL, NP, D, LS = 50, 3, 256, 2, 0.05


def clustered_state():
    """Three clusters of 50 rows (n = 150, NP = 256: pad rows and tiles that straddle clusters), spaced as in the GPU test,
    factorised the way the device does it: fp32 Cholesky and inverse, R = fl32(I - L X0) and X = fl32(X0 + X0 R) from fp64
    products, alpha = fl32(X^T X r) in fp64."""
    g = torch.Generator().manual_seed(3)
    n = SIZE * NCL
    ctr = torch.arange(NCL, dtype=F64)[:, None] * torch.tensor([80 * LS, 0.0], dtype=F64)
    X = (ctr.repeat_interleave(SIZE, 0) + (torch.rand(n, D, generator=g, dtype=F64) * 2 - 1) * 3 * LS).float()
    hyp = torch.tensor([0.01, 0.1, 1.0, LS, LS], dtype=torch.float32)
    Z = X.t() / hyp[3:, None]
    K = torch.zeros(NP, NP, dtype=torch.float32)
    for c in range(NCL):
        a, b = c * SIZE, (c + 1) * SIZE
        K[a:b, a:b] = khat_block(Z[:, a:b], hyp, "matern32")[0].float()
    K[n:, n:] = torch.eye(NP - n)
    L = torch.linalg.cholesky(K)
    X0 = torch.linalg.solve_triangular(L, torch.eye(NP), upper=False)
    R = (torch.eye(NP, dtype=F64) - L.double() @ X0.double()).tril().float().double()
    Xr = (X0.double() + X0.double() @ R).float()
    y = torch.randn(n, generator=g)
    r = torch.zeros(NP)
    r[:n] = y - hyp[1]
    alpha = (Xr.double().t() @ (Xr.double() @ r.double())).float()
    return dict(n=n, Z=Z, hyp=hyp, L=L, X0=X0, X=Xr, r=r, alpha=alpha)


def cids(n):
    i = torch.arange(NP)
    return torch.where(i < n, i // SIZE, -1 - i)


def run_checks(s):
    worst, sums = {}, []
    for c in range(NCL):
        a, b = c * SIZE, (c + 1) * SIZE
        Kh, Bg = khat_block(s["Z"][:, a:b], s["hyp"], "matern32")
        cc, sm = check_block(s["L"][a:b, a:b], s["X0"][a:b, a:b], s["X"][a:b, a:b], Kh, Bg, s["r"][a:b], s["alpha"][a:b], NP)
        sums.append(sm)
        for k, v in cc.items():
            worst[k] = max(worst.get(k, 0.0), v)
    return worst, sums


def test_checkers_pass_an_exact_state_and_flag_one_bad_element():
    s = clustered_state()
    cid = cids(s["n"])
    for M, lower in ((s["L"], True), (s["X0"], False), (s["X"], False), (s["X"].half(), False)):
        assert off_cluster_nonzeros(M, cid, lower=lower, chunk_bytes=4 * NP * 7) == (0, None)
    worst, sums = run_checks(s)
    lg = torch.log(s["L"].double().diagonal()[:s["n"]])
    scal = torch.tensor([float(sum(x["q"] for x in sums)), float(2 * lg.sum())], dtype=F64)
    worst.update(check_totals(scal, sums, s["n"], NP))
    assert max(worst.values()) <= C_MAX, worst
    # one off-cluster element (row 120 is in cluster 2, column 10 in cluster 0)
    bad = s["X"].clone()
    bad[120, 10] = 1e-30
    assert off_cluster_nonzeros(bad, cid, chunk_bytes=4 * NP * 7) == (1, (120, 10))
    L = s["L"].clone()
    L[70, 10] = 1e-30
    assert off_cluster_nonzeros(L, cid, lower=True)[0] == 1
    # one element of a diagonal block of the refined L^-1 moved to the first fp32 value past the bound of `refine`,
    # |X - Xref| <= u |X| + C_MAX B1 (the element of cluster 1's strict lower block with the widest bound in ulps)
    a = SIZE
    X0 = s["X0"][a:a + SIZE, a:a + SIZE].double()
    L64 = s["L"][a:a + SIZE, a:a + SIZE].double().tril()
    R = (torch.eye(SIZE, dtype=F64) - L64 @ X0).tril().float().double()
    Xref = X0 + X0 @ R
    B1 = U * math.sqrt(NP) * (X0.abs() @ R.abs())
    width = torch.where(torch.ones(SIZE, SIZE, dtype=torch.bool).tril(-1), B1 / Xref.abs().clamp_min(1e-30), 0)
    ii, jj = divmod(int(width.argmax()), SIZE)
    over = lambda x: abs(float(x) - float(Xref[ii, jj])) - U * abs(float(x)) > C_MAX * float(B1[ii, jj])
    x = torch.tensor(float(Xref[ii, jj]), dtype=torch.float32)
    while not over(x):
        x = torch.nextafter(x, torch.tensor(math.inf))
    for val, fails in ((torch.nextafter(x, torch.tensor(-math.inf)), False), (x, True)):
        moved = s["X"].clone()
        moved[a + ii, a + jj] = val
        worst2, _ = run_checks(dict(s, X=moved))
        assert (worst2["refine"] > C_MAX) == fails, (float(val), worst2["refine"])


@pytest.mark.parametrize("kind", ["matern32", "rbf"])
def test_mll_reference_summed_over_clusters_equals_the_oracle(kind):
    """On a block-diagonal problem (clusters far apart in fp64 too, so the oracle's cross-cluster k is below 1e-300),
    the per-cluster data terms, summed and assembled, give the oracle's loss and gradient."""
    g = torch.Generator().manual_seed(5)
    n = 90
    ctr = torch.arange(3, dtype=F64).repeat_interleave(30)[:, None] * torch.tensor([200.0, 0.0], dtype=F64)
    X = ctr + torch.rand(n, 2, generator=g, dtype=F64) * 0.5
    y = torch.randn(n, generator=g, dtype=F64)
    raw = torch.tensor([-3.0, 0.1, 0.2, -0.5, 0.3], dtype=F64)
    loss, grad, _ = O.neg_mll_closed_form(X, y, O.Hypers.unpack(raw, 8e-4), kind, 0.01)
    hp = O.Hypers.unpack(raw, 8e-4)
    parts = [mll_terms(X[a:a + 30] / hp.lengthscale, y[a:a + 30] - hp.mean, hp.outputscale, hp.noise, kind)
             for a in (0, 30, 60)]
    l2, g2 = mll_assemble(mll_sum(parts), raw, 0.01, 8e-4)
    assert abs(l2 - float(loss)) <= 1e-12 * max(1.0, abs(float(loss)))
    assert float((g2 - grad).abs().max()) <= 1e-12 * max(1.0, float(grad.abs().max()))
