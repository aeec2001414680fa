"""Multi-objective and constrained Bayesian optimisation: ``GeneralBO`` (HEBO/hebo/optimizers/general.py:23-204).

``GeneralBO`` fits a ``hebo_b200.MultiTaskModel`` (one GP per objective and constraint column, trained in one batched
device fit) on the raw y, scores ``GeneralAcq`` -- the LCB of every output -- with the device GA
(``hebo_b200.evolution.DeviceNSGA2`` with ``num_obj`` objectives and, when there are constraints, the summed constraint
violation as its constraint column), and picks the suggestions from the resulting (feasible) front: at random with the
most uncertain row kept, or by a Monte-Carlo expected hypervolume improvement when ``ref_point`` is given.

Hypervolumes are computed exactly on the host (``hypervolume``), in any number of objectives.  The reference uses pymoo's
``HV`` there; the selection only reads ``argmax`` and ``> 0`` of the improvements, so any exact hypervolume gives its
choice.
"""
from __future__ import annotations

import time
from typing import Optional

import numpy as np
import pandas as pd
import torch

from .acq import GeneralAcq, general_score
from .bo import _design_space
from .gp import GP, MultiTaskModel


def hypervolume(Y: np.ndarray, ref_point) -> float:
    """Exact hypervolume (minimisation) of the region dominated by the rows of Y and bounded by ref_point, in any number
    of objectives.  Only rows that strictly dominate ref_point (every coordinate below it) contribute.  Slices along the
    last objective and recurses on the non-dominated rows of each slab."""
    ref = np.asarray(ref_point, dtype=np.float64).reshape(-1)
    Y = np.asarray(Y, dtype=np.float64).reshape(-1, ref.size)
    Y = Y[(Y < ref).all(1)]
    return _hv(Y, ref)


def _hv(Y: np.ndarray, ref: np.ndarray) -> float:
    if Y.shape[0] == 0:
        return 0.0
    if ref.size == 1:
        return float(ref[0] - Y[:, 0].min())
    Y = Y[np.argsort(Y[:, -1], kind="stable")]
    vol = 0.0
    for i in range(Y.shape[0]):
        hi = Y[i + 1, -1] if i + 1 < Y.shape[0] else ref[-1]
        if hi > Y[i, -1]:
            vol += _hv(_nondominated(Y[:i + 1, :-1]), ref[:-1]) * (hi - Y[i, -1])
    return vol


def _nondominated(Y: np.ndarray) -> np.ndarray:
    le = (Y[:, None, :] <= Y[None, :, :]).all(-1)
    lt = (Y[:, None, :] < Y[None, :, :]).any(-1)
    return Y[~(le & lt).any(0)]


class GeneralBO:
    """general.py:23-204.  ``space``: a DesignSpace (or its list-of-dicts spec).  y has num_obj objective columns
    followed by num_constr constraint columns, all minimised; a row is feasible when every constraint is <= 0.

    model_name: 'multi_task' (the default, ``hebo_b200.MultiTaskModel``) or 'gp' when num_obj + num_constr == 1; any
    other surrogate raises NotImplementedError, and 'gp' with several outputs fails the reference's multi-output assertion.
    ``evo_pop`` / ``evo_iters`` are read when ``suggest`` runs, so they may be changed after construction.  As in the
    reference, ``fix_input`` only applies to the random start-up design: the model stage does not pass it to the GA."""

    support_parallel_opt = False          # AbstractOptimizer defaults: general.py does not override them
    support_constraint = False
    support_multi_objective = False
    support_combinatorial = False
    support_contextual = False

    def __init__(self, space, num_obj: int = 1, num_constr: int = 0, rand_sample: Optional[int] = None,
                 model_name: str = "multi_task", model_config: Optional[dict] = None, kappa: Optional[float] = 2.0,
                 c_kappa: Optional[float] = 0.0, use_noise: bool = False, evo_pop: int = 100, evo_iters: int = 200,
                 ref_point: Optional[np.ndarray] = None, device: str = "cuda"):
        if model_name not in ("multi_task", "gp"):
            raise NotImplementedError(f"GeneralBO: model_name {model_name!r} is not supported, only 'multi_task' and 'gp'")
        if num_obj + num_constr > 1:
            assert model_name == "multi_task", "GeneralBO: several outputs need a multi-output model"   # general.py:63-64
        self.space = _design_space(space)
        self.num_obj, self.num_constr = num_obj, num_constr
        self.rand_sample = 1 + self.space.num_paras if rand_sample is None else rand_sample
        self.model_name = model_name
        self.model_config = model_config if model_config is not None else {}
        self.X = pd.DataFrame(columns=self.space.para_names)
        self.y = np.zeros((0, num_obj + num_constr))
        self.kappa, self.c_kappa, self.use_noise = kappa, c_kappa, use_noise
        self.model = None
        self.evo_pop, self.evo_iters = evo_pop, evo_iters
        self.iter = 0
        self.ref_point = ref_point
        self.device = device
        self.last_timing = {}

    # ------------------------------------------------------------------ model and acquisition stages
    def _fit(self):
        Xc, Xe = self.space.transform(self.X)
        d, e, K = Xc.shape[1], Xe.shape[1], self.num_obj + self.num_constr
        conf = {"device": self.device, **self.model_config}
        if e > 0:
            conf["num_uniqs"] = self.space.num_uniqs
        model = MultiTaskModel(d, e, K, **conf) if self.model_name == "multi_task" else GP(d, e, 1, **conf)
        model.fit(Xc if d else None, Xe if e else None, torch.FloatTensor(self.y))
        torch.cuda.synchronize()
        return model

    def _kappas(self):
        """general.py:88-96: the schedule replaces a kappa / c_kappa of None."""
        upsi, delta = 0.1, 0.01
        sched = lambda: np.sqrt(upsi * 2 * ((2.0 + self.X.shape[1] / 2.0) * np.log(self.iter) + np.log(3 * np.pi ** 2 / (3 * delta))))
        return (sched() if self.kappa is None else self.kappa), (sched() if self.c_kappa is None else self.c_kappa)

    def _optimise(self, model, kappa, c_kappa) -> pd.DataFrame:
        """general.py:97-106: GeneralAcq on the device GA; the (feasible) front as a DataFrame."""
        from .evolution import DeviceNSGA2
        acq = GeneralAcq(model, self.num_obj, self.num_constr, kappa=kappa, c_kappa=c_kappa, use_noise=self.use_noise)
        seed = int(np.random.randint(0, 2 ** 31 - 1))
        sp = self.space
        evo = DeviceNSGA2(sp.var_kinds, sp.opt_lb.numpy(), sp.opt_ub.numpy(), sp.num_numeric, general_score(acq, seed ^ 0x5BD1E995),
                          pop=self.evo_pop, iters=self.evo_iters, seed=seed, device=self.device,
                          constrained=self.num_constr > 0, num_obj=self.num_obj)
        xc, xe, _ = evo.optimize()
        return sp.inverse_transform(xc.cpu(), xe.cpu().long())

    # ------------------------------------------------------------------ public interface
    def suggest(self, n_suggestions: int = 1, fix_input: Optional[dict] = None) -> pd.DataFrame:
        self.iter += 1
        if self.X.shape[0] < self.rand_sample:                       # general.py:67-73
            sample = self.space.sample(n_suggestions)
            for k, v in (fix_input or {}).items():
                sample[k] = v
            return sample
        t0 = time.perf_counter()
        model = self._fit()
        self.model = model
        t1 = time.perf_counter()
        kappa, c_kappa = self._kappas()
        suggest = self._optimise(model, kappa, c_kappa)
        t2 = time.perf_counter()
        out = self._select(model, suggest, n_suggestions)
        t3 = time.perf_counter()
        self.last_timing = dict(fit_ms=(t1 - t0) * 1e3, acq_ms=(t2 - t1) * 1e3, select_ms=(t3 - t2) * 1e3,
                                total_ms=(t3 - t0) * 1e3)
        return out

    def _select(self, model, suggest: pd.DataFrame, n_suggestions: int) -> pd.DataFrame:
        """general.py:107-158: random top-up of a short front; otherwise a random pick that keeps the most uncertain row, or
        with ref_point the Monte-Carlo EHVI choice, de-duplicated and topped up at random."""
        if suggest.shape[0] < n_suggestions:
            rand_samp = self.space.sample(n_suggestions - suggest.shape[0])
            return pd.concat([suggest, rand_samp], axis=0, ignore_index=True)
        if self.ref_point is None:
            with torch.no_grad():
                _, ps2 = model.predict(*self.space.transform(suggest))
                largest_uncert_id = int(np.argmax(np.log(torch.as_tensor(ps2).cpu().numpy()).sum(axis=1)))
            select_id = np.random.choice(suggest.shape[0], n_suggestions, replace=False).tolist()
            if largest_uncert_id not in select_id:
                select_id[0] = largest_uncert_id
            return suggest.iloc[select_id]
        assert self.num_obj > 1
        assert self.num_constr == 0
        n_mc = 10
        ref = np.asarray(self.ref_point, dtype=np.float64).reshape(-1)
        with torch.no_grad():
            y_samp = torch.as_tensor(model.sample_y(*self.space.transform(suggest), n_mc)).cpu().numpy()
        y_curr = self.get_pf(self.y).copy()
        select_id = []
        for _ in range(n_suggestions):
            base_hv = hypervolume(y_curr, ref)
            ehvi = []
            for j in range(suggest.shape[0]):
                samp = y_samp[:, j]
                hvi = sum(hypervolume(np.vstack([y_curr, samp[[k]]]), ref) - base_hv for k in range(n_mc))
                ehvi.append(hvi / n_mc)
            best_id = int(np.argmax(ehvi)) if max(ehvi) > 0 else np.random.choice(suggest.shape[0])
            y_curr = np.vstack([y_curr, y_samp[:, best_id].min(axis=0, keepdims=True)])
            select_id.append(best_id)
        select_id = list(set(select_id))
        if len(select_id) < n_suggestions:
            candidate_id = [i for i in range(suggest.shape[0]) if i not in select_id]
            select_id += np.random.choice(candidate_id, n_suggestions - len(select_id), replace=False).tolist()
        return suggest.iloc[select_id]

    def observe(self, X: pd.DataFrame, y) -> None:
        self.observe_new_data(X, y)

    def observe_new_data(self, X: pd.DataFrame, y) -> None:
        """general.py:160-178: rows with any non-finite value are dropped; y must have num_obj + num_constr columns."""
        y = np.asarray(y, dtype=np.float64).reshape(len(X), -1)
        assert y.shape[1] == self.num_obj + self.num_constr
        valid = np.isfinite(y).all(axis=1)
        self.X = pd.concat([self.X, X.iloc[valid]], axis=0, ignore_index=True)
        self.y = np.vstack([self.y, y[valid]])

    def get_pf(self, y: np.ndarray, return_optimal: bool = False):
        """general.py:183-195: the feasible rows of y that no feasible row dominates in the objectives (equal rows are both
        kept).  return_optimal=True: that mask over the FEASIBLE rows, as the reference returns it."""
        y = np.asarray(y, dtype=np.float64)
        feasible = (y[:, self.num_obj:] <= 0).all(axis=1)
        y = y[feasible].copy()
        yo = y[:, :self.num_obj]
        le = (yo[:, None, :] <= yo[None, :, :]).all(-1)
        lt = (yo[:, None, :] < yo[None, :, :]).any(-1)
        optimal = ~(le & lt).any(0)
        return optimal if return_optimal else y[optimal].copy()

    @property
    def best_x(self) -> pd.DataFrame:
        """The observed rows in the feasible front.  The reference indexes X with get_pf's mask over the feasible rows
        only, which selects the wrong rows (or fails) once any row is infeasible; here the mask is taken over all rows."""
        feasible = (self.y[:, self.num_obj:] <= 0).all(axis=1)
        rows = np.flatnonzero(feasible)[self.get_pf(self.y, return_optimal=True)]
        return self.X.iloc[rows].copy()

    @property
    def best_y(self) -> np.ndarray:
        return self.get_pf(self.y)
