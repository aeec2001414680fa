"""Generates tests/golden/ref_embedding.npz from the reference's own ``optimizers/hebo_embedding.py``.

    HEBO_SRC=<checkout of the HEBO sources> python tests/golden/make_ref_embedding.py

The file is loaded unmodified by path (oracle/ref_loader.py).  Its imports are satisfied by stubs: the ``hebo`` package
tree (design space, model factory and evolution optimiser are never called here), the sibling modules ``.hebo`` and
``.abstract_optimizer``, and ``hebo.acquisitions.acq``, which is the reference's real acq.py, so MACE_Embedding runs the
reference's own MACE.  Recorded:
  * ``gen_proj_matrix`` for "hesbo", "alebo" and Gaussian under fixed numpy seeds;
  * ``MACE_Embedding.eval`` ([m, 4]) on seeded inputs with the fixed-(mu, var) stub model of make_golden.gen_ref_mace,
    together with the N(0, 1) draws it takes from torch's global generator.
Test infrastructure; never imported by hebo_b200/.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ref_embedding.npz")

PROJ_CASES = [("hesbo", 4, 37, 0), ("hesbo", 1, 9, 1), ("alebo", 4, 37, 2), ("alebo", 16, 300, 3), ("gaussian", 3, 50, 4),
              ("gaussian", 8, 129, 5)]
EVAL_CASES = [  # (m, eff_dim, D, strategy, tau, kappa, noise, x range, seed)
    (300, 4, 37, "alebo", -0.5, 2.3, 0.013, 1.5, 10),
    (257, 8, 129, "gaussian", -1.0, 3.1, 1e-3, 0.6, 11),
    (64, 2, 20, "hesbo", 0.2, 2.0, 0.05, 1.2, 12),
]


def load_hebo_embedding():
    ref = ref_loader.load_reference()
    acq = types.ModuleType("hebo.acquisitions.acq")
    for k in ("Acquisition", "MACE", "Mean", "Sigma"):
        setattr(acq, k, getattr(ref, k))
    fake = {"hebo.acquisitions.acq": acq}
    for name, attrs in [("hebo", ()), ("hebo.design_space", ()), ("hebo.design_space.design_space", ("DesignSpace",)),
                        ("hebo.design_space.numeric_param", ("NumericPara",)), ("hebo.models", ()),
                        ("hebo.models.model_factory", ("get_model",)), ("hebo.acquisitions", ()), ("hebo.acq_optimizers", ()),
                        ("hebo.acq_optimizers.evolution_optimizer", ("EvolutionOpt",))]:
        m = types.ModuleType(name)
        m.__path__ = []
        for k in attrs:
            setattr(m, k, type(k, (), {}))
        fake[name] = m
    saved = {k: sys.modules.get(k) for k in fake}
    sys.modules.update(fake)
    try:
        return ref, ref_loader.load_file("_hebo_ref_opt.hebo_embedding", os.path.join("optimizers", "hebo_embedding.py"),
                                         stubs=[("_hebo_ref_opt", ()), ("_hebo_ref_opt.abstract_optimizer", ("AbstractOptimizer",)),
                                                ("_hebo_ref_opt.hebo", ("HEBO",))])
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def main():
    threads = torch.get_num_threads()
    ref, mod = load_hebo_embedding()
    torch.set_num_threads(threads)          # the module pins torch to one thread at import (hebo_embedding.py:26)
    out = {}
    for ci, (strategy, eff, dim, seed) in enumerate(PROJ_CASES):
        np.random.seed(seed)
        out[f"proj{ci}"] = mod.gen_proj_matrix(eff, dim, strategy)
        out[f"proj{ci}_case"] = np.array([eff, dim, seed])
        out[f"proj{ci}_strategy"] = np.array(strategy)

    class Dummy(ref.BaseModel):
        def __init__(self, mu, var, noise):
            super().__init__(1, 0, 1)
            self.mu, self.var, self._n = mu, var, noise

        def fit(self, *a):
            pass

        def predict(self, x, xe):
            return self.mu.clone(), self.var.clone()

        @property
        def noise(self):
            return self._n

    for ci, (m, eff, dim, strategy, tau, kappa, noise, rng, seed) in enumerate(EVAL_CASES):
        np.random.seed(seed)
        P = mod.gen_proj_matrix(eff, dim, strategy)
        g = torch.Generator().manual_seed(seed)
        x = (torch.rand(m, eff, generator=g) * 2 - 1) * rng
        mu = torch.randn(m, 1, generator=g) * 1.5
        var = torch.rand(m, 1, generator=g) ** 4 * 2 + 1e-8
        acq = mod.gen_mace_cls(P)(Dummy(mu, var, torch.tensor([noise])), best_y=np.float32(tau), kappa=kappa)
        torch.manual_seed(2000 + ci)
        F = acq(x, None)
        torch.manual_seed(2000 + ci)
        xi1, xi2 = torch.randn(m, 1), torch.randn(m, 1)
        out.update({f"e{ci}_x": x.numpy(), f"e{ci}_P": P, f"e{ci}_mu": mu.numpy(), f"e{ci}_var": var.numpy(),
                    f"e{ci}_xi1": xi1.numpy(), f"e{ci}_xi2": xi2.numpy(), f"e{ci}_F": F.numpy(),
                    f"e{ci}_par": np.array([tau, kappa, noise, 1e-4, 2000 + ci], dtype=np.float64)})
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, sorted(out)[:4], "...")


if __name__ == "__main__":
    main()
