"""HEBO.suggest / observe on the CUDA path (SURVEY rows a1-a3, a14-a18, f1).

Mirrors the control flow of HEBO/hebo/optimizers/hebo.py:119-229 -- Sobol start-up, y power transform with the raw-y
refit fallback, GP fit, tau = mu(best_x), kappa schedule, MACE, Pareto set, duplicate check, Sobol top-up, random pick of q
with the argmax-sigma / argmin-mu slots -- over a typed design space (``hebo_b200.space.DesignSpace``: num / int / pow /
pow_int / int_exponent / step_int / bool / cat, the reference's eight parameter types).  The acquisition optimiser is
either ONE big-batch device pass (default: m scrambled-Sobol candidates + the incumbent -> fused posterior+MACE -> device
non-dominated filter) or -- ``acq_optimizer="nsga2"`` -- a device-resident NSGA-II of the reference's shape
(``hebo_b200.evolution.DeviceNSGA2``: pop 100 x 100 generations, typed variables, every generation scored by one fused call,
no per-generation host round trip; evolution_optimizer.py:107-160).
The acquisition is MACE unless ``acq_cls`` names another class (hebo.py:35-61,162), which is built per suggest as
``acq_cls(model, best_y=py_best, kappa=kappa)``, scored by ``hebo_b200.acq.general_score`` and optimised over its own
objective and constraint columns; such a class takes one suggestion per call, as in the reference.

Two front ends:  ``HEBO(space)`` with a DesignSpace (or its list-of-dicts spec) speaks pandas DataFrames like the reference;
``HEBO(lb, ub)`` is the continuous-box shorthand that speaks tensors.  With a real HEBO install use
``hebo_b200.register()`` and HEBO's own optimiser classes instead.
"""
from __future__ import annotations

import time
from typing import Optional

import numpy as np
import pandas as pd
import torch
from torch.quasirandom import SobolEngine

from . import _lib
from .acq import MACE
from .ensemble import DeepEnsemble, FeDeepEnsemble, GumbelDeepEnsemble
from .gp import GP
from .pareto import feasible_front, pareto_front
from .space import DesignSpace, box_space


def hebo_y_transform(y: np.ndarray, strict: bool = False) -> torch.Tensor:
    """hebo.py:128-135: power transform of y / std (sklearn, host).  strict=False folds in the fallback of hebo.py:144-147
    (raw y when the transform fails); strict=True raises instead, for callers that implement the fallback themselves."""
    from sklearn.preprocessing import power_transform
    y = np.asarray(y, dtype=np.float64).reshape(-1, 1)
    try:
        if y.min() <= 0:
            t = torch.FloatTensor(power_transform(y / y.std(), method="yeo-johnson"))
        else:
            t = torch.FloatTensor(power_transform(y / y.std(), method="box-cox"))
            if t.std() < 0.5:
                t = torch.FloatTensor(power_transform(y / y.std(), method="yeo-johnson"))
        if t.std() < 0.5:
            raise RuntimeError("Power transformation failed")
        return t
    except Exception:
        if strict:
            raise
        return torch.FloatTensor(y).clone()


def kappa_schedule(n_obs: int, q: int, D: int) -> float:
    """hebo.py:156-160."""
    it = max(1, n_obs // q)
    upsi, delta = 0.5, 0.01
    return float(np.sqrt(upsi * 2 * ((2.0 + D / 2.0) * np.log(it) + np.log(3 * np.pi ** 2 / (3 * delta)))))


class HEBO:
    def __init__(self, space=None, ub=None, model_config: Optional[dict] = None, rand_sample: Optional[int] = None,
                 scramble_seed: Optional[int] = None, n_candidates: int = 10000, device: str = "cuda",
                 n_refine: int = 0, refine_sigma: float = 0.05, acq_optimizer: str = "sobol", evo_pop: int = 100,
                 evo_iters: int = 100, lb=None, _constraint=None, model_name: str = "gp", acq_cls=MACE):
        if model_name not in ("gp", "deep_ensemble", "fe_deep_ensemble", "gumbel"):
            raise NotImplementedError(f"HEBO: model_name {model_name!r} is not supported, only 'gp', 'deep_ensemble', "
                                      "'fe_deep_ensemble' and 'gumbel'")
        if acq_cls is not MACE and (n_refine or _constraint is not None):
            raise ValueError("n_refine and the embedding constraint are defined for the MACE front only; an acq_cls other "
                             "than MACE takes neither")
        if lb is not None:
            space = lb
        if ub is not None:                                   # HEBO(lb, ub): continuous box, tensors in / out
            self.space, self.tensor_api = box_space(space, ub), True
        else:
            self.space = space if isinstance(space, DesignSpace) else DesignSpace().parse(space)
            self.tensor_api = False
        sp = self.space
        self.d, self.e, self.D = sp.num_numeric, sp.num_categorical, sp.num_paras
        self.lb, self.ub = sp.opt_lb.float(), sp.opt_ub.float()                        # optimisation space, all columns
        self.int_cols = torch.tensor([sp.paras[n].integer_after_transform for n in sp.numeric_names], dtype=torch.bool)
        self.Xc = torch.zeros(0, self.d)                                               # observations, optimisation space
        self.Xe = torch.zeros(0, self.e, dtype=torch.long)
        self.y = np.zeros((0, 1))
        self.rand_sample = 1 + self.D if rand_sample is None else max(2, rand_sample)   # hebo.py:57
        assert acq_optimizer in ("sobol", "nsga2")
        self.acq_optimizer, self.evo_pop, self.evo_iters = acq_optimizer, evo_pop, evo_iters
        self.sobol = SobolEngine(self.D, scramble=True, seed=scramble_seed)
        self.cand_sobol = SobolEngine(self.D, scramble=True, seed=None if scramble_seed is None else scramble_seed + 1)
        self.n_candidates = n_candidates
        # optional evolutionary refinement of the Sobol front (numeric columns): n_refine rounds of Gaussian mutation around
        # the current front, rescored and merged on the device
        self.n_refine = int(n_refine)
        self.refine_sigma = float(refine_sigma)
        self.device = device
        # constraint hook (hebo_b200.embedding.HEBO_Embedding): Xc [m, d] on the device -> G [m], feasible iff G <= 0.  Both
        # acquisition optimisers then return the feasible front (pareto.feasible_front); there is no constrained refinement
        self._constraint = _constraint
        if _constraint is not None and self.n_refine:
            raise ValueError("n_refine is not supported together with a constraint")
        self._model_config = model_config
        self.model_name = model_name
        # the acquisition of hebo.py:162, built as acq_cls(model, best_y=py_best, kappa=kappa) in every suggest.  MACE keeps
        # the fused posterior + MACE path; any other class is scored by hebo_b200.acq.general_score
        self.acq_cls = acq_cls
        self.last_timing = {}

    # ------------------------------------------------------------------ config / data
    @property
    def model_config(self):
        if self._model_config is not None:
            cfg = dict(self._model_config)
        elif self.model_name == "gp":
            cfg = {"lr": 0.01, "num_epochs": 100, "verbose": False, "noise_lb": 8e-4, "pred_likeli": False}     # hebo.py:80-87
        else:
            cfg = {}                                                                                        # hebo.py:94-95
        if self.e > 0:
            cfg["num_uniqs"] = self.space.num_uniqs                                                         # hebo.py:99-100
        return cfg

    @property
    def X(self):
        """Observed inputs: a tensor [n, d] (box front end) or a DataFrame (typed space)."""
        return self.Xc if self.tensor_api else self.space.inverse_transform(self.Xc, self.Xe)

    def _to_opt(self, X):
        if self.tensor_api:
            Xc = torch.as_tensor(X, dtype=torch.float32).reshape(-1, self.d)
            return Xc, torch.zeros(Xc.shape[0], 0, dtype=torch.long)
        return self.space.transform(X)

    def _from_opt(self, Xc, Xe):
        return Xc.clone() if self.tensor_api else self.space.inverse_transform(Xc, Xe)

    def _fixed_columns(self, fix_input: Optional[dict]) -> dict:
        """{optimisation column index: value} of a fix_input dict (evolution_optimizer.py:97-101, hebo.py:70-72)."""
        out = {}
        for name, v in (fix_input or {}).items():
            col = self.space.para_names.index(name)
            out[col] = float(self.space.paras[name].transform(np.array([v], dtype=object if self.space.paras[name].is_categorical else None))[0])
        return out

    def quasi_sample(self, n, fix_input: Optional[dict] = None, engine=None, as_opt: bool = False):
        """hebo.py:63-75: scrambled Sobol in the optimisation box, integer-valued columns rounded."""
        samp = (engine or self.sobol).draw(n) * (self.ub - self.lb) + self.lb
        for col, v in self._fixed_columns(fix_input).items():
            samp[:, col] = v
        Xc = samp[:, :self.d].clone()
        Xc[:, self.int_cols] = Xc[:, self.int_cols].round()
        Xe = samp[:, self.d:].round().long()
        return (Xc, Xe) if as_opt else self._from_opt(Xc, Xe)

    def observe(self, X, y):
        y = np.asarray(y, dtype=np.float64).reshape(-1, 1)
        valid = torch.from_numpy(np.isfinite(y.reshape(-1)))               # hebo.py:211-215
        Xc, Xe = self._to_opt(X)
        self.Xc = torch.cat([self.Xc, Xc[valid]], 0)
        self.Xe = torch.cat([self.Xe, Xe[valid]], 0)
        self.y = np.vstack([self.y, y[valid.numpy()]])

    @property
    def best_x(self):
        if self.Xc.shape[0] == 0:
            raise RuntimeError("No data has been observed!")
        i = int(self.y.argmin())
        return self._from_opt(self.Xc[[i]], self.Xe[[i]])

    @property
    def best_y(self):
        if self.Xc.shape[0] == 0:
            raise RuntimeError("No data has been observed!")
        return float(self.y.min())

    def get_best_id(self, fix_input: Optional[dict] = None) -> int:
        """hebo.py:103-117: the incumbent among the rows that agree with fix_input (if any)."""
        y = self.y.reshape(-1).copy()
        rows = torch.cat([self.Xc, self.Xe.float()], 1)
        for col, v in self._fixed_columns(fix_input).items():
            y[((rows[:, col] - v).abs() > np.finfo(float).eps).numpy()] = np.inf
        return int(np.argmin(y)) if np.isfinite(y).any() else int(np.argmin(self.y.reshape(-1)))

    def _unique_mask(self, Xc: torch.Tensor, Xe: torch.Tensor) -> torch.Tensor:
        """hebo.py:196-197 check_unique: drop rows equal to an observed row or to an earlier row of the batch."""
        allx = torch.cat([torch.cat([self.Xc, self.Xe.float()], 1), torch.cat([Xc, Xe.float()], 1)], 0).numpy()
        _, first = np.unique(allx, axis=0, return_index=True)
        keep = np.zeros(allx.shape[0], dtype=bool)
        keep[first] = True
        return torch.from_numpy(keep[self.Xc.shape[0]:])

    # ------------------------------------------------------------------ suggest
    def _fit(self):
        """hebo.py:127-147: power-transformed y, and on ANY failure (transform or fit) a refit on the raw y."""
        cls = {"gp": GP, "deep_ensemble": DeepEnsemble, "fe_deep_ensemble": FeDeepEnsemble,
               "gumbel": GumbelDeepEnsemble}[self.model_name]

        def build(y):
            model = cls(self.d, self.e, 1, device=self.device, **self.model_config)
            model.fit(self.Xc if self.d else None, self.Xe if self.e else None, y)
            return model
        try:
            return build(hebo_y_transform(self.y, strict=True))
        except Exception:
            return build(torch.FloatTensor(self.y).clone())

    def _acq_front(self, model, py_best, kappa, bxc, bxe, fix_input, fixed, candidates, mark):
        """hebo.py:162-165 with an acquisition other than MACE: acq_cls(model, best_y=py_best, kappa=kappa), optimised by
        DeviceNSGA2 with its objective count and constraint (evolution_optimizer.py:72-105), or scored on the Sobol batch
        with the incumbent prepended.  Returns the (feasible) front (cand_c, cand_e) with its posterior mean and variance."""
        from .acq import general_score
        acq = self.acq_cls(model, best_y=py_best.numpy().squeeze(), kappa=kappa)
        if acq.num_obj > _lib.HB_MAX_OBJ:
            raise ValueError(f"HEBO: an acquisition with {acq.num_obj} objectives; at most {_lib.HB_MAX_OBJ} are supported")
        dev, constrained = model.device, acq.num_constr > 0
        seed = int(np.random.randint(0, 2 ** 31 - 1))
        score = general_score(acq, seed ^ 0x5BD1E995)
        if self.acq_optimizer == "nsga2" and candidates is None:
            from .evolution import DeviceNSGA2
            evo = DeviceNSGA2(self.space.var_kinds, self.lb.numpy(), self.ub.numpy(), self.d, score, pop=self.evo_pop,
                              iters=self.evo_iters, seed=seed, fixed=fixed, device=dev, constrained=constrained,
                              num_obj=acq.num_obj)
            cand_c, cand_e, _ = evo.optimize(initial_suggest=torch.cat([bxc, bxe.float()], 1).numpy())
            cand_e = cand_e.long()                                   # res.X is already the (feasible) rank-0 set
            mark("candidates_ms")
        else:
            if candidates is None:
                cc, ce = self.quasi_sample(self.n_candidates - 1, fix_input, self.cand_sobol, as_opt=True)
                cand_c, cand_e = torch.cat([bxc, cc], 0), torch.cat([bxe, ce], 0)
            else:
                cand_c, cand_e = self._to_opt(candidates)
            cand_c = cand_c.to(dev, torch.float32, non_blocking=True)
            cand_e = cand_e.to(dev, non_blocking=True)
            mark("candidates_ms")
            F, G = (score(cand_c, cand_e, 0), None) if not constrained else score(cand_c, cand_e, 0)
            idx = pareto_front(F) if G is None else feasible_front(F, G)
            cand_c, cand_e = cand_c[idx], cand_e[idx]
        with torch.no_grad():
            mu, var = model.predict(cand_c if self.d else None, cand_e if self.e else None)
        mark("posterior_ms")
        return cand_c, cand_e, mu.reshape(-1), var.reshape(-1)

    def suggest(self, n_suggestions: int = 1, fix_input: Optional[dict] = None, candidates=None):
        if self.acq_cls is not MACE and n_suggestions != 1:                 # hebo.py:120-121
            raise RuntimeError("Parallel optimization is supported only for MACE acquisition")
        if self.Xc.shape[0] < self.rand_sample:
            return self.quasi_sample(n_suggestions, fix_input)
        t0 = time.perf_counter()
        model = self._fit()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        marks = {}
        last = [t1]

        def mark(name):
            torch.cuda.synchronize()
            now = time.perf_counter()
            marks[name] = (now - last[0]) * 1e3
            last[0] = now
        dev = model.device
        best_id = self.get_best_id(fix_input)
        bxc, bxe = self.Xc[[best_id]], self.Xe[[best_id]]
        py_best, _ = model.predict(bxc if self.d else None, bxe if self.e else None)                  # hebo.py:152
        kappa = kappa_schedule(self.Xc.shape[0], n_suggestions, self.D)
        fixed = self._fixed_columns(fix_input)
        if self.acq_cls is not MACE:
            mark("predict_best_ms")
            cand_c, cand_e, mu, var = self._acq_front(model, py_best, kappa, bxc, bxe, fix_input, fixed, candidates, mark)
            idx = torch.arange(cand_c.shape[0], device=dev)
        else:
            acq = MACE(model, best_y=py_best.numpy().squeeze(), kappa=kappa)
            tau = float(np.asarray(acq.tau).reshape(-1)[0])
            mark("predict_best_ms")

            def score(xc, xe, seed=0):
                return model.predict_mace(xc if self.d else None, tau, kappa, acq.eps, seed=seed, return_mu_var=True,
                                          Xe=xe if self.e else None, device_out=True)
            cons = self._constraint
            if self.acq_optimizer == "nsga2" and candidates is None:
                from .evolution import DeviceNSGA2
                if cons is None:
                    evo_score = lambda xc, xe, gen: score(xc, xe, gen)[0]
                else:
                    evo_score = lambda xc, xe, gen: (score(xc, xe, gen)[0], cons(xc))
                evo = DeviceNSGA2(self.space.var_kinds, self.lb.numpy(), self.ub.numpy(), self.d, evo_score, pop=self.evo_pop,
                                  iters=self.evo_iters, seed=int(np.random.randint(0, 2 ** 31 - 1)), fixed=fixed, device=dev,
                                  constrained=cons is not None)
                cand_c, cand_e, _ = evo.optimize(initial_suggest=torch.cat([bxc, bxe.float()], 1).numpy())
                cand_e = cand_e.long()
                mark("candidates_ms")
                F, mu, var = score(cand_c, cand_e.int())
                mark("posterior_mace_ms")
                idx = torch.arange(cand_c.shape[0], device=dev)          # res.X is already the rank-0 set
            else:
                if candidates is None:
                    cc, ce = self.quasi_sample(self.n_candidates - 1, fix_input, self.cand_sobol, as_opt=True)
                    cand_c, cand_e = torch.cat([bxc, cc], 0), torch.cat([bxe, ce], 0)
                else:
                    cand_c, cand_e = self._to_opt(candidates)
                cand_c = cand_c.to(dev, torch.float32, non_blocking=True)
                cand_e = cand_e.to(dev, non_blocking=True)
                mark("candidates_ms")
                F, mu, var = score(cand_c, cand_e)
                mark("posterior_mace_ms")
                idx = pareto_front(F) if cons is None else feasible_front(F, cons(cand_c))
        for _ in range(self.n_refine if self.d else 0):
            pc, pe = cand_c[idx], cand_e[idx]
            reps = max(1, (self.n_candidates // 4) // max(1, pc.shape[0]))
            lbd, ubd = self.lb[:self.d].to(dev), self.ub[:self.d].to(dev)
            kc = pc.repeat(reps, 1)
            kc = kc + self.refine_sigma * (ubd - lbd) * torch.randn(kc.shape, device=dev)
            kc = torch.minimum(torch.maximum(kc, lbd), ubd)
            ic = self.int_cols.to(dev)
            kc[:, ic] = kc[:, ic].round()
            for col, v in fixed.items():
                if col < self.d:
                    kc[:, col] = v
            ke = pe.repeat(reps, 1)
            Fk, muk, vark = score(kc, ke)
            cand_c, cand_e = torch.cat([pc, kc], 0), torch.cat([pe, ke], 0)
            F = torch.cat([F[idx], Fk], 0)
            mu, var = torch.cat([mu[idx], muk]), torch.cat([var[idx], vark])
            idx = pareto_front(F)
        mark("front_ms")
        rec_c, rec_e = cand_c[idx].cpu(), cand_e[idx].cpu().long()
        mu_f, sig_f = mu[idx].cpu(), var[idx].sqrt().cpu()
        keep = self._unique_mask(rec_c, rec_e)
        rec_c, rec_e, mu_f, sig_f = rec_c[keep], rec_e[keep], mu_f[keep], sig_f[keep]

        def append(xc, xe):
            nonlocal rec_c, rec_e, mu_f, sig_f
            if xc.shape[0] == 0:
                return
            m2, v2 = model.predict(xc if self.d else None, xe if self.e else None)
            rec_c, rec_e = torch.cat([rec_c, xc], 0), torch.cat([rec_e, xe], 0)
            mu_f, sig_f = torch.cat([mu_f, m2.reshape(-1)]), torch.cat([sig_f, v2.reshape(-1).sqrt()])
        cnt = 0
        while rec_c.shape[0] < n_suggestions:                              # hebo.py:169-180 Sobol top-up
            xc, xe = self.quasi_sample(n_suggestions - rec_c.shape[0], fix_input, as_opt=True)
            allc, alle = torch.cat([rec_c, xc], 0), torch.cat([rec_e, xe], 0)
            ok = self._unique_mask(allc, alle)[rec_c.shape[0]:]            # unique w.r.t. the observations AND the current rec
            append(xc[ok], xe[ok])
            cnt += 1
            if cnt > 3:       # "sometimes the design space is so small that duplicated sampling is unavoidable"
                break
        if rec_c.shape[0] < n_suggestions:
            append(*self.quasi_sample(n_suggestions - rec_c.shape[0], fix_input, as_opt=True))
        select_id = np.random.choice(rec_c.shape[0], n_suggestions, replace=False).tolist()   # hebo.py:182
        best_pred_id = int(torch.argmin(mu_f))
        best_unce_id = int(torch.argmax(sig_f))
        if best_unce_id not in select_id and n_suggestions > 2:
            select_id[0] = best_unce_id
        if best_pred_id not in select_id and n_suggestions > 2:
            select_id[1] = best_pred_id
        out = self._from_opt(rec_c[select_id], rec_e[select_id])
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        mark("select_ms")
        self.last_timing = dict(fit_ms=(t1 - t0) * 1e3, score_ms=(t2 - t1) * 1e3, total_ms=(t2 - t0) * 1e3,
                                front=int(idx.numel()), **marks)
        self.model = model
        return out
