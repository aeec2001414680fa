"""Generates tests/golden/ref_mo_lcb.npz from the reference's own ``MOMeanSigmaLCB`` (acquisitions/acq.py:99-129).

    HEBO_SRC=<checkout of the HEBO sources> python tests/golden/make_ref_mo_lcb.py

acq.py is loaded unmodified by path (oracle/ref_loader.py).  The model is a stub with fixed (mu, var) [m, 1] and a fixed
float32 noise [1], as hebo_b200.GP.noise is; per case the script seeds torch's global generator, runs
``MOMeanSigmaLCB.eval`` and then, from the same seed, records the N(0, 1) draws eval took (``torch.randn(py.shape)``;
predict draws nothing) and ``np.sqrt(model.noise)`` as computed there.  Cases cover several kappa (the default 2.0 and
others, one negative), positive, negative and zero best_y, and rows with var = 0, tiny (subnormal included), large,
negative and NaN, and a NaN mean.  Test infrastructure; never imported by hebo_b200/.
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

OUT = os.path.join(ROOT, "tests", "golden", "ref_mo_lcb.npz")

CASES = [  # (m, kappa or None for the default, best_y, noise, seed)
    (200, None, 0.0, 0.05, 0),
    (333, 3.0, 1.25, 0.3, 1),
    (97, 0.7310585, -2.5, 1e-3, 2),
    (256, 2.3, 0.1, 0.0, 3),
    (129, -1.5, -0.0, 2.0, 4),
    (64, 5.123456789, 1e4, 0.07, 5),
]
EDGE_VAR = [0.0, 1e-30, 1e-40, 1e-12, 1e30, -1.0, float("nan")]


class StubModel:
    def __init__(self, mu, var, noise):
        self.mu, self.var, self._noise = mu, var, noise
        self.num_out = 1

    @property
    def noise(self):
        return self._noise.clone()

    def predict(self, x, xe):
        return self.mu.clone(), self.var.clone()


def main():
    ref_loader.load_reference()
    acq_mod = sys.modules["_hebo_ref.acquisitions.acq"]
    out = {}
    for ci, (m, kappa, best_y, noise, seed) in enumerate(CASES):
        g = torch.Generator().manual_seed(200 + ci)
        mu = torch.randn(m, 1, generator=g) * 3.0
        var = torch.rand(m, 1, generator=g) * 2.0
        var[: len(EDGE_VAR), 0] = torch.tensor(EDGE_VAR)
        mu[len(EDGE_VAR), 0] = float("nan")
        noise_t = torch.tensor([noise], dtype=torch.float32)
        model = StubModel(mu, var, noise_t)
        conf = {} if kappa is None else {"kappa": kappa}
        acq = acq_mod.MOMeanSigmaLCB(model, best_y=best_y, **conf)
        x = torch.zeros(m, 1)
        torch.manual_seed(seed)
        v = acq.eval(x, None)
        torch.manual_seed(seed)
        xi = torch.randn(m, 1)
        p = f"c{ci}_"
        out[p + "meta"] = np.array([m, seed], np.int64)
        out[p + "kappa"] = np.array(acq.kappa, np.float64)
        out[p + "best_y"] = np.array(best_y, np.float64)
        out[p + "mu"], out[p + "var"], out[p + "noise"] = mu.numpy(), var.numpy(), noise_t.numpy()
        out[p + "noise_sd"] = np.asarray(np.sqrt(model.noise))      # the noise factor exactly as acq.py:119 computes it
        out[p + "xi"], out[p + "out"] = xi.numpy(), v.numpy()
    out["n_cases"] = np.array(len(CASES))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
