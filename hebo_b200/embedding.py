"""HEBO in a random low-dimensional embedding (HEBO/hebo/optimizers/hebo_embedding.py) for continuous problems of any
dimension, including those above the GP's HB_MAX_FEATURES.

HEBO runs in an ``eff_dim``-dimensional box ``y``; a point maps to the original box [-1, 1]^D as ``x = y B`` with the
projection matrix ``B [eff_dim, D]`` (HeSBO, ALEBO or Gaussian, ``gen_proj_matrix``).  With ``clip=False`` (the default)
the acquisition is ``MACE_Embedding``: the three MACE objectives plus one constraint, the bound violation

    G(y) = sum_j max(|(y B)_j| - 1, 0)        (hebo_embedding.py:88-89)

computed on the device by ``hb_embed_violation`` without forming ``y B``.  Both acquisition optimisers of
``hebo_b200.HEBO`` then return the feasible front (device NSGA-II survival with ``hb_nsga2_survive_cv``, or the Sobol
batch filtered by ``pareto.feasible_front``).  With ``clip=True`` the acquisition is plain MACE and ``project`` squashes
with tanh.  Suggestions are DataFrames in the embedding space, as in the reference; ``project`` maps them to the
original space.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import pandas as pd
import torch

from . import _lib
from .acq import MACE
from .base import Acquisition
from .space import DesignSpace
from .suggest import HEBO


def gen_emb_space(eff_dim: int, scale: float) -> DesignSpace:
    """hebo_embedding.py:29-37: the box [-|scale|, |scale|]^eff_dim, parameters y0 .. y{eff_dim-1}."""
    scale = abs(scale)
    return DesignSpace().parse([{"name": f"y{i}", "type": "num", "lb": -1 * scale, "ub": scale} for i in range(eff_dim)])


def check_design_space(space: DesignSpace) -> bool:
    """hebo_embedding.py:40-53: numeric parameters only, every range [-1, 1]."""
    if any(p.kind != "num" for p in space.paras.values()):
        return False
    if not (space.opt_lb + torch.ones(space.num_paras)).abs().sum() < 1e-6:
        return False
    if not (space.opt_ub - torch.ones(space.num_paras)).abs().sum() < 1e-6:
        return False
    return True


def gen_proj_matrix(eff_dim: int, dim: int, strategy: str = "alebo") -> np.ndarray:
    """hebo_embedding.py:56-67, drawing from numpy's global RNG in the same order: "hesbo" (one signed 1 per column),
    "alebo" (Gaussian columns normalised to unit length), anything else Gaussian."""
    if strategy == "hesbo":
        matrix = np.zeros((eff_dim, dim))
        for i in range(dim):
            sig = np.random.choice([-1, 1])
            idx = np.random.choice(eff_dim)
            matrix[idx, i] = sig * 1.0
    else:
        matrix = np.random.randn(eff_dim, dim)
        if strategy == "alebo":
            matrix = matrix / np.sqrt((matrix ** 2).sum(axis=0))
    return matrix


def embed_violation(Y: torch.Tensor, B: torch.Tensor) -> torch.Tensor:
    """G [m] = sum_j max(|(Y B)_j| - 1, 0) of Y [m, e] and B [e, D], both on the same CUDA device (hb_embed_violation)."""
    from .pareto import _workspace
    lib = _lib.lib()
    if not (Y.is_cuda and B.is_cuda):
        raise ValueError("embed_violation: Y and B must be CUDA tensors")
    Y = Y.to(torch.float32).contiguous()
    B = B.to(torch.float32).contiguous()
    m, e = Y.shape
    D = B.shape[1]
    if B.shape[0] != e:
        raise ValueError(f"embed_violation: Y has {e} columns, B has {B.shape[0]} rows")
    G = torch.empty(m, dtype=torch.float32, device=Y.device)
    if m == 0:
        return G
    need = int(lib.hb_embed_violation_workspace_bytes(m, e, D))
    if need < 0:
        raise _lib.HeboB200Error(f"hb_embed_violation_workspace_bytes: invalid size (m {m}, e {e}, D {D})")
    ws = _workspace(Y.device, need, "embed")
    with torch.cuda.device(Y.device):
        _lib.check(lib.hb_embed_violation(_lib.ptr(Y), m, e, _lib.ptr(B), D, _lib.ptr(G), _lib.ptr(ws), ws.numel(),
                                          _lib.stream_ptr()), "hb_embed_violation")
    return G


class MACE_Embedding(Acquisition):
    """hebo_embedding.py:71-90: MACE's three objectives plus the bound violation of the projection as one constraint.
    ``proj_matrix`` [eff_dim, D] may be a numpy array or a (CUDA) tensor; it is held on the device once."""

    def __init__(self, model, best_y, proj_matrix, device="cuda", **conf):
        super().__init__(model, **conf)
        self.mace = MACE(model, best_y, **conf)
        self.B = torch.as_tensor(proj_matrix).to(device=device, dtype=torch.float32).contiguous()

    @property
    def num_constr(self):
        return 1

    @property
    def num_obj(self):
        return 3

    def eval(self, x, xe=None):
        """[m, 4]: (LCB, -log EI, -log PI) as hebo_b200.MACE returns them, then the bound violation G."""
        assert xe is None or xe.shape[1] == 0
        F = self.mace.eval(x, xe)
        G = embed_violation(torch.as_tensor(x).to(self.B.device), self.B)
        return torch.cat([F, G.reshape(-1, 1).to(F.device)], 1)


class HEBO_Embedding:
    """hebo_embedding.py:95-167 on this project's HEBO.  ``space``: a DesignSpace (or its list-of-dicts spec) of numeric
    parameters on [-1, 1]; ``hebo_kwargs`` go to ``hebo_b200.HEBO`` (acq_optimizer, n_candidates, device, ...).  The
    acquisition optimiser defaults to the device NSGA-II, as the reference uses its evolutionary optimiser; with
    ``acq_optimizer="sobol"`` and a large eff_dim no candidate of the Sobol batch may be feasible, and the suggestion is
    then the least infeasible candidate, whose projection leaves [-1, 1]^D."""

    support_parallel_opt = True
    support_combinatorial = False
    support_contextual = False

    def __init__(self, space, model_name: str = "gp", eff_dim: int = 1, scale: float = 1, strategy: str = "alebo",
                 clip: bool = False, rand_sample: Optional[int] = None, **hebo_kwargs):
        if model_name not in ("gp", "deep_ensemble"):
            raise NotImplementedError(f"HEBO_Embedding: model_name {model_name!r} is not supported, only 'gp' and "
                                      "'deep_ensemble'")
        self.space = space if isinstance(space, DesignSpace) else DesignSpace().parse(space)
        assert check_design_space(self.space)
        self.scale, self.eff_dim, self.clip = scale, eff_dim, clip
        self.proj_matrix = gen_proj_matrix(eff_dim, self.space.num_paras, strategy)
        self.eff_space = gen_emb_space(eff_dim, scale)
        # the reference always optimises the acquisition with its evolutionary optimiser (hebo.py:165); in 16 embedding
        # dimensions no point of a 10 000-row Sobol batch was feasible (BASELINE §6), so the Sobol path is opt-in
        hebo_kwargs.setdefault("acq_optimizer", "nsga2")
        self.device = hebo_kwargs.get("device", "cuda")
        self._B_dev = None
        constraint = None if clip else (lambda xc: embed_violation(xc, self.B_device))
        self.mace = HEBO(self.eff_space, rand_sample=rand_sample, _constraint=constraint, model_name=model_name, **hebo_kwargs)
        sobol_sample = self.mace.quasi_sample

        def quasi_sample(n, fix_input=None, engine=None, as_opt=False):
            # HEBO draws its Sobol candidate batch through an explicit engine; the start-up design and the top-up use
            # the embedding's sampler, as `self.mace.quasi_sample = self.quasi_sample` does in the reference
            if engine is not None:
                return sobol_sample(n, fix_input, engine, as_opt)
            return self.quasi_sample(n, fix_input, as_opt=as_opt)
        self.mace.quasi_sample = quasi_sample

    @property
    def B_device(self) -> torch.Tensor:
        """The projection matrix as fp32 on the device, uploaded once."""
        if self._B_dev is None:
            self._B_dev = torch.as_tensor(self.proj_matrix, dtype=torch.float32).to(self.device).contiguous()
        return self._B_dev

    def quasi_sample(self, n: int, fix_input=None, factor: float = 16, as_opt: bool = False):
        """hebo_embedding.py:124-145: points of [-1, 1]^D drawn uniformly (numpy's global RNG, the draws of
        ``space.sample(100)``) and mapped back by ``factor (B B^T)^-1 B x``; rows whose projection leaves [-1, 1]^D are
        rejected, and ``factor`` grows by 1/0.8 when a batch is accepted whole (the batch is then discarded) and shrinks by
        0.8 when none of it is.  With ``clip`` the embedding box is sampled uniformly instead."""
        assert fix_input is None
        if self.clip:
            df = self.eff_space.sample(n)
        else:
            B = torch.FloatTensor(self.proj_matrix)
            L = torch.linalg.cholesky(B.mm(B.t()))
            lb, ub = self.space.opt_lb.numpy(), self.space.opt_ub.numpy()
            parts, have = [], 0
            while have < n:
                x_hd = torch.FloatTensor(np.random.uniform(lb[:, None], ub[:, None], (lb.size, 100)))   # [D, 100]
                y = factor * torch.cholesky_solve(B.mm(x_hd), L).t()                                     # [100, eff_dim]
                pj = np.matmul(y.numpy().astype(np.float64), self.proj_matrix)
                ok = (pj.max(axis=1) <= 1.0) & (pj.min(axis=1) >= -1.0)
                if ok.all():
                    factor /= 0.8
                    continue
                if not ok.any():
                    factor *= 0.8
                parts.append(y[torch.from_numpy(ok)])
                have += int(ok.sum())
            df = pd.DataFrame(torch.cat(parts, 0)[:n].numpy(), columns=self.eff_space.numeric_names)
        if as_opt:
            Xc, Xe = self.eff_space.transform(df)
            return Xc, Xe
        return df

    def project(self, df_x_ld: pd.DataFrame) -> pd.DataFrame:
        """hebo_embedding.py:147-152: x = y B (then tanh with ``clip``), as a DataFrame over the original parameters."""
        x = df_x_ld[self.eff_space.numeric_names].values
        x_hd = np.matmul(x, self.proj_matrix)
        if self.clip:
            x_hd = np.tanh(x_hd)
        return pd.DataFrame(x_hd, columns=self.space.numeric_names)

    def suggest(self, n_suggestions: int = 1) -> pd.DataFrame:
        if not self.clip and n_suggestions != 1:   # hebo.py:119-120, reached through acq_cls = MACE_Embedding
            raise RuntimeError("Parallel optimization is supported only for MACE acquisition")
        return self.mace.suggest(n_suggestions)

    def observe(self, X: pd.DataFrame, y) -> None:
        self.mace.observe(X, y)

    @property
    def best_x(self) -> pd.DataFrame:
        return self.mace.best_x

    @property
    def best_y(self) -> float:
        return self.mace.best_y
