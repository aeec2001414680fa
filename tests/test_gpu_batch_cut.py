"""Scores of a candidate must not depend on the batch it is scored in.  The posterior variance contraction deals
128-candidate bands to clusters of CTAs and pads a band count that is not a multiple of the cluster size
(hebo_b200/csrc/vnorm_sched.h); the cuts below give odd band counts, a last band that is not full, fewer work units than
clusters and more than one chunk."""
import numpy as np
import pytest
import torch

import hebo_b200
from tests.util import seeded_problem

pytestmark = pytest.mark.gpu


def test_sub_batches_score_bitwise_like_the_whole_batch():
    n, d = 1000, 6
    X, y = seeded_problem(n, d, 5)
    np.random.seed(0)
    gp = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=10, noise_lb=8e-4, pred_likeli=False, langevin=False)
    gp.fit(X, None, y)
    assert gp.tensor_cores and gp.m_chunk == 32768
    # 1 row: one band, 8 units < clusters; 129: two bands, the last holding one row; 384: three bands; 640: five;
    # 32 768 + 128: a full chunk and a one-band chunk
    cuts = [1, 129, 384, 640, 32768 + 128]
    m = sum(cuts)
    g = torch.Generator().manual_seed(6)
    Xs = torch.rand(m, d, generator=g) * 2.4 - 1.2
    xi1, xi2 = torch.randn(m, 1, generator=g), torch.randn(m, 1, generator=g)
    tau, kappa = float(y.min()), 2.0
    F, mu, var = gp.predict_mace(Xs.cuda(), tau, kappa, 1e-4, xi1, xi2, return_mu_var=True)
    assert bool(torch.isfinite(F).all()) and bool((var > 0).all())
    r0 = 0
    for c in cuts:
        Fc, muc, varc = gp.predict_mace(Xs[r0:r0 + c].cuda(), tau, kappa, 1e-4, xi1[r0:r0 + c], xi2[r0:r0 + c],
                                        return_mu_var=True)
        assert torch.equal(Fc, F[r0:r0 + c]), c
        assert torch.equal(muc, mu[r0:r0 + c]), c
        assert torch.equal(varc, var[r0:r0 + c]), c
        r0 += c
