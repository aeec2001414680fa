"""Acquisitions behind HEBO's ``Acquisition`` plugin surface (HEBO/hebo/acquisitions/acq.py:17-39).

``MACE`` is the drop-in for the reference's MACE (acq.py:131-171): with a ``hebo_b200.GP`` model the
predict + (LCB, -logEI, -logPI) arithmetic is ONE fused C-ABI call (``GP.predict_mace``); with any other
``BaseModel`` that model's ``predict`` output is pushed through the same CUDA epilogue (``hb_mace_epilogue``), so the
class stays a valid general-purpose acquisition.  ``Mean`` / ``Sigma`` / ``LCB`` mirror acq.py:55-82 and
``AbsEtaDifference`` nomr.py:25-34.

The single-objective GA (``hebo_b200.evolution.DeviceNSGA2`` with a one-column score, as ``hebo_b200.BO`` runs it) scores
its offspring through ``ga_score``: ``LCB``, ``Mean``, ``Sigma`` and ``AbsEtaDifference`` over a ``hebo_b200.GP`` are one
posterior call with F = NULL plus one ``hb_acq1_epilogue`` on the device: the ``eval`` expression in IEEE fp32 on the same
mu / var (torch's CPU sqrt, used by ``eval``, may differ from the correctly rounded one by one ulp).  Any other single-objective acquisition -- another model, or a user's own class, including a subclass of these
four -- is scored through its own ``eval`` on CPU tensors, once per generation, as the reference's EvolutionOpt does.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from .base import Acquisition
from .gp import GP


class SingleObjectiveAcq(Acquisition):
    def __init__(self, model, **conf):
        super().__init__(model, **conf)

    @property
    def num_obj(self):
        return 1

    @property
    def num_constr(self):
        return 0


class LCB(SingleObjectiveAcq):
    def __init__(self, model, **conf):
        super().__init__(model, **conf)
        self.kappa = conf.get("kappa", 3.0)
        assert model.num_out == 1

    def eval(self, x, xe):
        py, ps2 = self.model.predict(x, xe)
        return py - self.kappa * ps2.sqrt()


class Mean(SingleObjectiveAcq):
    def __init__(self, model, **conf):
        super().__init__(model, **conf)
        assert model.num_out == 1

    def eval(self, x, xe):
        py, _ = self.model.predict(x, xe)
        return py


class Sigma(SingleObjectiveAcq):
    def __init__(self, model, **conf):
        super().__init__(model, **conf)
        assert model.num_out == 1

    def eval(self, x, xe):
        _, ps2 = self.model.predict(x, xe)
        return -1 * ps2.sqrt()


class AbsEtaDifference(SingleObjectiveAcq):
    """nomr.py:25-34: |mu - eta| - kappa sigma, the stage-two acquisition a NoMR_BO may be given."""

    def __init__(self, model, kappa=3.0, eta=0.7, **conf):
        super().__init__(model, **conf)
        self.kappa = kappa
        self.eta = eta
        assert model.num_out == 1

    def eval(self, x, xe):
        py, ps2 = self.model.predict(x, xe)
        return torch.abs(py - self.eta) - self.kappa * ps2.sqrt()


# exact classes whose eval hb_acq1_epilogue restates; a subclass may override eval, so it takes the host path
_ACQ1_MODES = {LCB: _lib.HB_ACQ1_LCB, Mean: _lib.HB_ACQ1_MEAN, Sigma: _lib.HB_ACQ1_SIGMA,
               AbsEtaDifference: _lib.HB_ACQ1_ABS_ETA}


def ga_score(acq):
    """score(xc, xe, gen) -> f [m] fp32 on the device for DeviceNSGA2, of a single-objective acquisition.  xc [m, d] fp32
    and xe [m, e] int32 are device tensors.  With a hebo_b200.GP and one of the four acquisitions above: predict on the
    device (hb_posterior_mace_ex with F = NULL) and hb_acq1_epilogue, no host synchronisation.  Otherwise: acq.eval on CPU
    tensors (xe as int64, like the reference's BOProblem), its first column copied back to the device."""
    mode = _ACQ1_MODES.get(type(acq))
    if mode is not None and isinstance(acq.model, GP):
        kappa = float(getattr(acq, "kappa", 0.0))
        eta = float(getattr(acq, "eta", 0.0))

        def device_score(xc, xe, gen):
            with torch.no_grad():
                mu, var = acq.model.predict(xc, xe)
            mu, var = mu.reshape(-1), var.reshape(-1)
            f = torch.empty_like(mu)
            if f.numel():
                with torch.cuda.device(f.device):
                    _lib.check(_lib.lib().hb_acq1_epilogue(_lib.ptr(mu), _lib.ptr(var), f.numel(), mode, kappa, eta, _lib.ptr(f),
                                                           _lib.stream_ptr()), "hb_acq1_epilogue")
            return f
        return device_score

    def host_score(xc, xe, gen):
        with torch.no_grad():
            v = acq(xc.cpu(), xe.cpu().long())
        return torch.as_tensor(v).reshape(xc.shape[0], -1)[:, 0].to(xc.device, torch.float32).contiguous()
    return host_score


class MACE(Acquisition):
    def __init__(self, model, best_y, **conf):
        super().__init__(model, **conf)
        self.kappa = conf.get("kappa", 2.0)
        self.eps = conf.get("eps", 1e-4)
        self.tau = best_y

    @property
    def num_constr(self):
        return 0

    @property
    def num_obj(self):
        return 3

    def eval(self, x, xe=None):
        """minimize (lcb, -log EI, -log PI) -- the column order of acq.py:166-170."""
        tau = float(np.asarray(self.tau).reshape(-1)[0])
        with torch.no_grad():
            if isinstance(self.model, GP):     # predict + MACE fused in ONE C-ABI call (a failed fit degrades inside it, gp.py:152-154)
                return self.model.predict_mace(x, tau, float(self.kappa), float(self.eps), Xe=xe)
            return self._eval_any_model(x, xe, tau)

    def _eval_any_model(self, x, xe, tau):
        """Any other BaseModel (e.g. the RF stand-in of HEBO/test/test_acq.py:18-21): its predict() output goes through the
        same CUDA epilogue (hb_mace_epilogue), with the two N(0,1) draws of acq.py:154-155 taken from torch's CPU generator
        in the reference's order."""
        py, ps2 = self.model.predict(x, xe)
        m = py.shape[0]
        xi1, xi2 = torch.randn(py.shape), torch.randn(py.shape)
        dev = torch.device("cuda")
        up = lambda t: t.reshape(-1).to(dev, torch.float32).contiguous()
        mu_d, var_d, z1, z2 = up(py), up(ps2), up(xi1), up(xi2)
        F = torch.empty(m, 3, dtype=torch.float32, device=dev)
        if m:
            with torch.cuda.device(dev):
                _lib.check(_lib.lib().hb_mace_epilogue(_lib.ptr(mu_d), _lib.ptr(var_d), m, float(self.model.noise.reshape(-1)[0]), tau,
                                                       float(self.kappa), float(self.eps), _lib.ptr(z1), _lib.ptr(z2), 0, _lib.ptr(F),
                                                       _lib.stream_ptr()), "hb_mace_epilogue")
        return F.cpu()


FusedMACE = MACE
