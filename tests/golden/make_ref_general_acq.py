"""Generates tests/golden/ref_general_acq.npz from the reference's own ``GeneralAcq`` (acquisitions/acq.py:192-242).

    HEBO_SRC=<checkout of the HEBO sources> python tests/golden/make_ref_general_acq.py

acq.py is loaded unmodified by path (oracle/ref_loader.py).  The model is a stub with fixed (mu, var) [m, K] and a fixed
noise [K]; per case the script seeds torch's global generator, runs ``GeneralAcq.eval`` and then, from the same seed,
records the N(0, 1) draws eval took (``torch.randn(py.shape)``; predict draws nothing) and ``model.noise.sqrt()`` as
computed there (torch's CPU sqrt is not correctly rounded everywhere and differs between CPUs).  Cases cover several
(num_obj, num_constr), use_noise on and off, and non-default kappa / c_kappa.  Test infrastructure; never imported by
hebo_b200/.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ref_general_acq.npz")

CASES = [  # (m, num_obj, num_constr, use_noise, kappa, c_kappa, seed)
    (200, 2, 1, True, 2.0, 0.0, 0),
    (200, 2, 1, False, 2.0, 0.0, 1),
    (333, 3, 4, True, 3.0, 4.0, 2),
    (64, 1, 2, True, 1.7, 0.5, 3),
    (128, 5, 0, True, 2.5, 0.0, 4),
    (97, 1, 0, False, 0.3, 0.0, 5),
]


class StubModel:
    def __init__(self, mu, var, noise):
        self.mu, self.var, self._noise = mu, var, noise
        self.num_out = mu.shape[1]

    @property
    def noise(self):
        return self._noise.clone()

    def predict(self, x, xe):
        return self.mu.clone(), self.var.clone()


def main():
    ref_loader.load_reference()
    acq_mod = sys.modules["_hebo_ref.acquisitions.acq"]
    out = {}
    for ci, (m, no, nc, use_noise, kappa, c_kappa, seed) in enumerate(CASES):
        K = no + nc
        g = torch.Generator().manual_seed(100 + ci)
        mu = torch.randn(m, K, generator=g) * 3.0
        var = torch.rand(m, K, generator=g) * 2.0
        var[: m // 10] = torch.rand(m // 10, K, generator=g) * 1e-14          # below FLT_EPSILON^2: the clamp is active
        noise = torch.rand(K, generator=g) * 0.1
        model = StubModel(mu, var, noise)
        acq = acq_mod.GeneralAcq(model, no, nc, kappa=kappa, c_kappa=c_kappa, use_noise=use_noise)
        x = torch.zeros(m, 1)
        torch.manual_seed(seed)
        v = acq.eval(x, None)
        torch.manual_seed(seed)
        xi = torch.randn(m, K) if use_noise else torch.zeros(m, K)
        p = f"c{ci}_"
        out[p + "meta"] = np.array([m, no, nc, int(use_noise), seed], np.int64)
        out[p + "kappa"] = np.array([kappa, c_kappa], np.float64)
        out[p + "mu"], out[p + "var"], out[p + "noise"] = mu.numpy(), var.numpy(), noise.numpy()
        out[p + "noise_sd"] = noise.sqrt().numpy()       # the noise term's factor as the reference computed it (torch's CPU sqrt)
        out[p + "xi"], out[p + "out"] = xi.numpy(), v.numpy()
    out["n_cases"] = np.array(len(CASES))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
