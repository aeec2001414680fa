"""``NoisyOpt`` (HEBO/hebo/optimizers/noisy_opt.py): HEBO's batch selection over the final population of a single-objective
GA whose acquisition is one joint posterior draw per generation (``hebo_b200.acq.NoisyAcq``, acq.py:173-190).

The model (a GP, or with ``model_name='deep_ensemble'`` a ``hebo_b200.DeepEnsemble``) is fitted on the raw y.  The device
GA (``hebo_b200.evolution.DeviceNSGA2`` with a one-column score, pop 100 x 100 generations) scores every generation on the
device.  Over the GP: ``hb_sample_y_batch``, one correlated draw over the batch, with the jitter ladder on the device and
duplicate rows left out of the joint covariance (they are +inf, which the GA survival gives a duplicate child anyway); the
status word of the ladder is read once, after the GA.  Over the deep ensemble: ``hb_de_predict_batch`` with one independent
draw per row, as the reference's ``BaseModel.sample_y`` draws them.  The generation loop never synchronises with the
host.  Suggestions follow noisy_opt.py:59-89: the final population in survival order, rows equal to an observation
dropped, a Sobol top-up, then a random pick of q with the argmax-sigma / argmin-mu rows forced into slots 0 / 1 when
q > 2.
"""
from __future__ import annotations

import time
from typing import Optional

import numpy as np
import torch

from . import _lib
from .acq import NoisyAcq, ga_score
from .ensemble import DeepEnsemble
from .evolution import DeviceNSGA2
from .gp import GP
from .suggest import HEBO


class NoisyOpt(HEBO):
    """noisy_opt.py:27-89.  ``space``: a DesignSpace (or its list-of-dicts spec); DataFrames in and out.  model_name:
    'gp' or 'deep_ensemble'.  With 'gp', ``evo_pop`` <= 256: the GP sampler draws at most 256 rows jointly; the deep
    ensemble's draws are independent, so it takes any population the device GA takes (DeviceNSGA2.MAX_POP)."""

    support_parallel_opt = True
    support_combinatorial = True
    support_contextual = True
    MAX_POP = 256

    def __init__(self, space, model_name: str = "gp", rand_sample: Optional[int] = None, model_config: Optional[dict] = None,
                 scramble_seed: Optional[int] = None, evo_pop: int = 100, evo_iters: int = 100, device: str = "cuda"):
        if model_name not in ("gp", "deep_ensemble"):
            raise NotImplementedError(f"NoisyOpt: model_name {model_name!r} is not supported, only 'gp' and 'deep_ensemble'")
        max_pop = self.MAX_POP if model_name == "gp" else DeviceNSGA2.MAX_POP
        if not 2 <= int(evo_pop) <= max_pop:
            raise ValueError(f"NoisyOpt: evo_pop must lie in [2, {max_pop}], got {evo_pop}")
        super().__init__(space, model_config=model_config, rand_sample=rand_sample, scramble_seed=scramble_seed, device=device,
                         acq_optimizer="nsga2", evo_pop=int(evo_pop), evo_iters=int(evo_iters), model_name=model_name)
        self.acq_cls = NoisyAcq

    def suggest(self, n_suggestions: int = 1, fix_input: Optional[dict] = None):
        assert fix_input is None
        if self.Xc.shape[0] < self.rand_sample:                    # noisy_opt.py:41-43: Sobol start-up design
            return self.quasi_sample(n_suggestions)
        t0 = time.perf_counter()
        model = (GP if self.model_name == "gp" else DeepEnsemble)(self.d, self.e, 1, device=self.device, **self.model_config)
        model.fit(self.Xc if self.d else None, self.Xe if self.e else None, torch.FloatTensor(self.y).clone())   # raw y
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        best_id = self.get_best_id()
        acq = self.acq_cls(model, 1, 0)
        score = ga_score(acq)
        evo = DeviceNSGA2(self.space.var_kinds, self.lb.numpy(), self.ub.numpy(), self.d, score, pop=self.evo_pop,
                          iters=self.evo_iters, seed=int(np.random.randint(0, 2 ** 31 - 1)), device=self.device)
        init = torch.cat([self.Xc[[best_id]], self.Xe[[best_id]].float()], 1).numpy()
        rec_c, rec_e, _ = evo.optimize(initial_suggest=init, return_pop=True)
        status = getattr(score, "status", None)
        if status is not None:
            _lib.check(int(status.item()), "hb_sample_y_batch")    # a give-up raises what GP.sample_y raises
        rec_c, rec_e = rec_c.cpu(), rec_e.cpu().long()
        keep = self._unique_mask(rec_c, rec_e)                     # noisy_opt.py:60 check_unique
        rec_c, rec_e = rec_c[keep], rec_e[keep]
        cnt = 0
        while rec_c.shape[0] < n_suggestions:                      # noisy_opt.py:62-73 Sobol top-up
            xc, xe = self.quasi_sample(n_suggestions - rec_c.shape[0], as_opt=True)
            ok = self._unique_mask(xc, xe)
            rec_c, rec_e = torch.cat([rec_c, xc[ok]], 0), torch.cat([rec_e, xe[ok]], 0)
            cnt += 1
            if cnt > 3:       # "sometimes the design space is so small that duplicated sampling is unavoidable"
                break
        if rec_c.shape[0] < n_suggestions:
            xc, xe = self.quasi_sample(n_suggestions - rec_c.shape[0], as_opt=True)
            rec_c, rec_e = torch.cat([rec_c, xc], 0), torch.cat([rec_e, xe], 0)
        select_id = np.random.choice(rec_c.shape[0], n_suggestions, replace=False).tolist()   # noisy_opt.py:75
        with torch.no_grad():
            py, ps2 = model.predict(rec_c if self.d else None, rec_e if self.e else None)      # noisy_opt.py:77-83
        best_pred_id = int(torch.argmin(py.reshape(-1)))
        best_unce_id = int(torch.argmax(ps2.reshape(-1).sqrt()))
        if best_unce_id not in select_id and n_suggestions > 2:
            select_id[0] = best_unce_id
        if best_pred_id not in select_id and n_suggestions > 2:
            select_id[1] = best_pred_id
        out = self._from_opt(rec_c[select_id], rec_e[select_id])
        t2 = time.perf_counter()
        self.last_timing = dict(fit_ms=(t1 - t0) * 1e3, acq_ms=(t2 - t1) * 1e3, total_ms=(t2 - t0) * 1e3)
        self.model = model
        return out
