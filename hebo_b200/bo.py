"""Single-objective Bayesian optimisers on the device GA: ``BO`` (HEBO/hebo/optimizers/bo.py), ``NoMR_BO``
(optimizers/nomr.py) and ``HEBO_VectorContextual`` (optimizers/hebo_contextual.py).

``BO`` fits one ``hebo_b200.GP`` on the raw y and optimises a single-objective acquisition (``LCB`` with kappa 2 by
default) with the device GA: ``hebo_b200.evolution.DeviceNSGA2`` with a one-column score, pop 100 x 100 generations, as
the reference's EvolutionOpt runs pymoo's MixedVariableGA.  The four acquisitions of ``hebo_b200.acq`` are scored on the
device without a host synchronisation inside a generation; any other single-objective acquisition through its own
``eval`` on CPU tensors (``hebo_b200.acq.ga_score``).  The method names follow ``hebo_b200.HEBO``: ``suggest``,
``observe``, ``best_x``, ``best_y``.
"""
from __future__ import annotations

import time
from typing import Optional

import numpy as np
import pandas as pd
import torch

from .acq import LCB, AbsEtaDifference, ga_score  # noqa: F401  (AbsEtaDifference: nomr.py exports it next to NoMR_BO)
from .ensemble import DeepEnsemble, FeDeepEnsemble, GumbelDeepEnsemble
from .gp import GP
from .space import DesignSpace
from .suggest import HEBO


def _design_space(space) -> DesignSpace:
    return space if isinstance(space, DesignSpace) else DesignSpace().parse(space)


class BO:
    """bo.py:22-109.  ``space``: a DesignSpace (or its list-of-dicts spec).  Suggestions and observations are DataFrames.
    ``acq_cls`` is any single-objective acquisition without constraints (``num_obj == 1``, ``num_constr == 0``), built as
    ``acq_cls(model, **acq_conf)``."""

    support_parallel_opt = False
    support_combinatorial = True
    support_contextual = True

    def __init__(self, space, model_name: str = "gp", rand_sample: Optional[int] = None, acq_cls=None,
                 acq_conf: Optional[dict] = None, pop: int = 100, iters: int = 100, device: str = "cuda"):
        if model_name not in ("gp", "deep_ensemble", "fe_deep_ensemble", "gumbel"):
            raise NotImplementedError(f"BO: model_name {model_name!r} is not supported, only 'gp', 'deep_ensemble', "
                                      "'fe_deep_ensemble' and 'gumbel'")
        self.space = _design_space(space)
        sp = self.space
        self.d, self.e = sp.num_numeric, sp.num_categorical
        self.model_name = model_name
        self.rand_sample = 1 + sp.num_paras if rand_sample is None else max(2, rand_sample)   # bo.py:40-42
        self.acq_cls = LCB if acq_cls is None else acq_cls
        self.acq_conf = {"kappa": 2.0} if acq_conf is None else acq_conf
        self.pop, self.iters, self.device = int(pop), int(iters), device
        self.Xc = torch.zeros(0, self.d)                         # observations in the optimisation space
        self.Xe = torch.zeros(0, self.e, dtype=torch.long)
        self.y = np.zeros((0, 1))
        self.last_timing = {}

    @property
    def X(self) -> pd.DataFrame:
        return self.space.inverse_transform(self.Xc, self.Xe)

    def _fixed_columns(self, fix_input: Optional[dict]) -> dict:
        """{optimisation column index: value} of a fix_input dict."""
        out = {}
        for name, v in (fix_input or {}).items():
            p = self.space.paras[name]
            out[self.space.para_names.index(name)] = float(p.transform(np.array([v], dtype=object if p.is_categorical else None))[0])
        return out

    def suggest(self, n_suggestions: int = 1, fix_input: Optional[dict] = None) -> pd.DataFrame:
        assert n_suggestions == 1
        if self.Xc.shape[0] < self.rand_sample:                    # bo.py:47-53: uniform start-up design
            sample = self.space.sample(n_suggestions)
            for k, v in (fix_input or {}).items():
                sample[k] = v
            return sample
        t0 = time.perf_counter()
        conf = {"warp": False, "device": self.device}              # bo.py:62-69: the GP's own defaults, raw y
        if self.e > 0:
            conf["num_uniqs"] = self.space.num_uniqs
        model = {"gp": GP, "deep_ensemble": DeepEnsemble, "fe_deep_ensemble": FeDeepEnsemble,
                 "gumbel": GumbelDeepEnsemble}[self.model_name](self.d, self.e, 1, **conf)
        model.fit(self.Xc if self.d else None, self.Xe if self.e else None, torch.FloatTensor(self.y))
        acq = self.acq_cls(model, **self.acq_conf)
        if acq.num_obj != 1 or acq.num_constr != 0:
            raise NotImplementedError("BO: only single-objective acquisitions without constraints are supported")
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        from .evolution import DeviceNSGA2
        evo = DeviceNSGA2(self.space.var_kinds, self.space.opt_lb.numpy(), self.space.opt_ub.numpy(), self.d, ga_score(acq),
                          pop=self.pop, iters=self.iters, seed=int(np.random.randint(0, 2 ** 31 - 1)),
                          fixed=self._fixed_columns(fix_input), device=model.device)
        best = int(np.argmin(self.y.reshape(-1)))                  # bo.py:74: initial_suggest = the argmin-y row
        init = torch.cat([self.Xc[[best]], self.Xe[[best]].float()], 1).numpy()
        xc, xe, _ = evo.optimize(initial_suggest=init)
        out = self.space.inverse_transform(xc.cpu(), xe.cpu().long())
        for k, v in (fix_input or {}).items():                     # evolution_optimizer.py:155-157
            out[k] = v
        t2 = time.perf_counter()
        self.last_timing = dict(fit_ms=(t1 - t0) * 1e3, acq_ms=(t2 - t1) * 1e3, total_ms=(t2 - t0) * 1e3)
        self.model = model
        return out

    def observe(self, X: pd.DataFrame, y) -> None:
        """bo.py:77-95: one objective column; rows with a non-finite y are dropped."""
        y = np.asarray(y, dtype=np.float64)
        assert y.shape[1] == 1
        valid = np.isfinite(y.reshape(-1))
        Xc, Xe = self.space.transform(X)
        keep = torch.from_numpy(valid)
        self.Xc = torch.cat([self.Xc, Xc[keep]], 0)
        self.Xe = torch.cat([self.Xe, Xe[keep]], 0)
        self.y = np.vstack([self.y, y[valid].reshape(-1, 1)])

    @property
    def best_x(self) -> pd.DataFrame:
        if self.Xc.shape[0] == 0:
            raise RuntimeError("No data has been observed!")
        i = int(self.y.argmin())
        return self.space.inverse_transform(self.Xc[[i]], self.Xe[[i]])

    @property
    def best_y(self) -> float:
        if self.Xc.shape[0] == 0:
            raise RuntimeError("No data has been observed!")
        return float(self.y.min())


class NoMR_BO:
    """nomr.py:37-93: stage one (``opt1``, default ``HEBO(space)``) until the best observed y reaches ``eta``, then stage
    two (``opt2``, default ``BO(space, acq_conf={"kappa": 0.6})``).  Both stages observe every point.  ``eta = None``
    means +inf, as in the reference: every suggestion after the first observation then comes from stage two."""

    support_parallel_opt = False
    support_combinatorial = True
    support_contextual = False

    def __init__(self, space, eta: Optional[float] = None, opt1=None, opt2=None):
        self.space = _design_space(space)
        self.eta = np.inf if eta is None else eta
        self.opt1 = HEBO(self.space) if opt1 is None else opt1
        self.opt2 = BO(self.space, acq_conf={"kappa": 0.6}) if opt2 is None else opt2

    def observe(self, X: pd.DataFrame, y) -> None:
        self.opt1.observe(X, y)
        self.opt2.observe(X, y)

    def suggest(self, n_suggestions: int = 1, fix_input: Optional[dict] = None) -> pd.DataFrame:
        assert n_suggestions == 1
        y = self.opt1.y
        if y is None or y.shape[0] == 0 or y.min() > self.eta:     # nomr.py:74-80
            return self.opt1.suggest(n_suggestions, fix_input)
        return self.opt2.suggest(n_suggestions, fix_input)

    @property
    def best_x(self) -> pd.DataFrame:
        return self.opt1.best_x if self.opt1.best_y < self.opt2.best_y else self.opt2.best_x

    @property
    def best_y(self) -> float:
        return self.opt1.best_y if self.opt1.best_y < self.opt2.best_y else self.opt2.best_y


class HEBO_VectorContextual:
    """hebo_contextual.py:20-50: HEBO with the named context ``self.context`` of ``context_dict`` ({name: {parameter:
    value}}) passed as ``fix_input`` to every suggestion.  model_name: 'gp' or 'deep_ensemble', passed to HEBO."""

    support_parallel_opt = True
    support_combinatorial = True
    support_contextual = True

    def __init__(self, space, context_dict: dict, model_name: str = "gp", rand_sample: Optional[int] = None, **hebo_kwargs):
        if model_name not in ("gp", "deep_ensemble"):
            raise NotImplementedError(f"HEBO_VectorContextual: model_name {model_name!r} is not supported, only 'gp' and "
                                      "'deep_ensemble'")
        self.hebo = HEBO(_design_space(space), rand_sample=rand_sample, model_name=model_name, **hebo_kwargs)
        self.context_dict = context_dict
        self.context = None

    @property
    def context_vector(self) -> dict:
        fix_input = self.context_dict[self.context]
        for k in fix_input.keys():
            assert k in self.hebo.space.para_names
        return fix_input

    def suggest(self, n: int = 1) -> pd.DataFrame:
        return self.hebo.suggest(n, fix_input=self.context_vector)

    def observe(self, X: pd.DataFrame, y) -> None:
        self.hebo.observe(X, y)

    @property
    def best_x(self) -> pd.DataFrame:
        raise NotImplementedError("Not supported for contextual BO")

    @property
    def best_y(self) -> float:
        raise NotImplementedError("Not supported for contextual BO")
