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

``GeneralAcq`` (acq.py:192-242) is the LCB of every objective and constraint of a multi-output model, for ``GeneralBO``.
Its ``eval`` runs on any model through ``hb_general_acq_epilogue``; ``general_score`` scores it for the device GA, over GPs
and over deep ensembles.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from .base import Acquisition
from .ensemble import DeepEnsemble, EnsembleBatch, FeatureSelectionEnsemble
from .forest import RF
from .gp import GP, MultiTaskModel


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


class NoisyAcq(Acquisition):
    """acq.py:173-190: the acquisition is one joint posterior draw over the whole batch, ``model.sample_y(x, xe)``, which
    is the CPU-tensor path for any model.  The device GA scores it through ``ga_score``."""

    def __init__(self, model, num_obj, num_constr):
        super().__init__(model)
        self._num_obj = num_obj
        self._num_constr = num_constr

    @property
    def num_obj(self):
        return self._num_obj

    @property
    def num_constr(self):
        return self._num_constr

    def eval(self, x, xe):
        with torch.no_grad():
            return self.model.sample_y(x, xe).reshape(-1, self.num_obj + self.num_constr)


# exact classes whose eval hb_acq1_epilogue restates; a subclass may override eval, so it takes the host path
_ACQ1_MODES = {LCB: _lib.HB_ACQ1_LCB, Mean: _lib.HB_ACQ1_MEAN, Sigma: _lib.HB_ACQ1_SIGMA,
               AbsEtaDifference: _lib.HB_ACQ1_ABS_ETA}


def _noisy_device_score(model, seed: int):
    """score(xc, xe, gen) of NoisyAcq over a fitted hebo_b200.GP: one hb_sample_y_batch per generation with counter = gen,
    so every generation draws fresh N(0,1) values from the same seed.  The workspace is allocated at the first batch and
    reused.  ``score.status`` is the device word a give-up of the jitter ladder sets to HB_ERR_NOT_PD; nothing in the
    generation loop reads it."""
    state = {}

    def score(xc, xe, gen):
        m = xc.shape[0] if model.d > 0 else xe.shape[0]
        ws = state.get(m)
        if ws is None:
            ws = state[m] = torch.empty(model.sample_batch_workspace_bytes(m), dtype=torch.uint8, device=model.device)
        return model.sample_y_batch(xc if model.d > 0 else None, xe if model.num_enum else None, seed, gen,
                                    status=score.status, jitter=score.jitter, ws=ws)
    score.status = torch.zeros(1, dtype=torch.int32, device=model.device)
    score.jitter = torch.zeros(1, dtype=torch.float32, device=model.device)
    return score


def _noisy_ensemble_score(model, seed: int):
    """score(xc, xe, gen) of NoisyAcq over a fitted single-output DeepEnsemble: one hb_de_predict_batch per generation
    with one independent draw per row (BaseModel.sample_y), keyed by (seed, counter = gen)."""
    batch = EnsembleBatch([model])

    def score(xc, xe, gen):
        _, _, samp = batch.predict(xc if model.num_cont > 0 else None, xe if model.num_enum > 0 else None, n_samples=1,
                                   seed=seed, counter=gen)
        return samp.reshape(-1)
    return score


def _noisy_forest_score(model, seed: int):
    """score(xc, xe, gen) of NoisyAcq over a fitted RF: one hb_rf_predict per generation with one independent draw per row
    (BaseModel.sample_y), keyed by (seed, counter = gen)."""
    def score(xc, xe, gen):
        _, _, samp = model._predict_dev(xc if model.num_cont > 0 else None, xe if model.num_enum > 0 else None, n_samples=1,
                                        seed=seed, counter=gen)
        return samp.reshape(-1)
    return score


def ga_score(acq, seed=None):
    """score(xc, xe, gen) -> f [m] fp32 on the device for DeviceNSGA2, of a single-objective acquisition.  xc [m, d] fp32
    and xe [m, e] int32 are device tensors.  With a hebo_b200.GP and one of the four acquisitions above: predict on the
    device (hb_posterior_mace_ex with F = NULL) and hb_acq1_epilogue, no host synchronisation.  With a NoisyAcq of one
    objective and no constraint over a fitted hebo_b200.GP: one joint draw per generation on the device
    (``GP.sample_y_batch``, counter = the generation, ``seed`` drawn from numpy's global generator when None; batches of at
    most 256 rows); over a fitted single-output DeepEnsemble: one hb_de_predict_batch per generation with one
    independent draw per row (counter = the generation, any batch size); over a fitted RF: one hb_rf_predict per generation
    with the same draw layout.  The four acquisitions above over an RF score on the device as over a GP.  Otherwise: acq.eval on CPU tensors (xe as int64,
    like the reference's BOProblem), its first column copied back to the device."""
    if type(acq) is NoisyAcq and acq.num_obj == 1 and acq.num_constr == 0:
        if isinstance(acq.model, GP) and not acq.model._fit_failed:
            return _noisy_device_score(acq.model, int(np.random.randint(0, 2 ** 31 - 1)) if seed is None else int(seed))
        if _batchable(acq.model) and acq.model.fitted and acq.model.num_out == 1:
            return _noisy_ensemble_score(acq.model, int(np.random.randint(0, 2 ** 31 - 1)) if seed is None else int(seed))
        if isinstance(acq.model, RF) and acq.model.fitted:
            return _noisy_forest_score(acq.model, int(np.random.randint(0, 2 ** 31 - 1)) if seed is None else int(seed))
    mode = _ACQ1_MODES.get(type(acq))
    if mode is not None and isinstance(acq.model, (GP, DeepEnsemble, RF)):
        kappa = float(getattr(acq, "kappa", 0.0))
        eta = float(getattr(acq, "eta", 0.0))
        fe = isinstance(acq.model, FeatureSelectionEnsemble)     # fresh draws per generation: (fe_seed, gen)
        fe_seed = (int(np.random.randint(0, 2 ** 31 - 1)) if seed is None else int(seed)) if fe else 0

        def device_score(xc, xe, gen):
            with torch.no_grad():
                mu, var = acq.model.predict(xc, xe, seed=fe_seed, counter=gen) if fe else acq.model.predict(xc, xe)
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


class GeneralAcq(Acquisition):
    """acq.py:192-242: minimise (py - kappa ps) of the num_obj objectives subject to (py - c_kappa ps) <= 0 of the
    num_constr constraints, ps = sqrt(ps2) clamped at FLT_EPSILON, with py + noise^0.5 xi when use_noise.  ``eval`` takes
    the N(0,1) draws from torch's CPU generator as ``torch.randn(py.shape)``, like the reference, and runs the arithmetic in
    the CUDA epilogue ``hb_general_acq_epilogue`` (correctly rounded fp32: torch's CPU sqrt may differ by one ulp).
    Returns [m, num_obj + num_constr] on the input's device."""

    def __init__(self, model, num_obj, num_constr, **conf):
        super().__init__(model, **conf)
        self._num_obj = num_obj
        self._num_constr = num_constr
        self.kappa = conf.get("kappa", 2.0)
        self.c_kappa = conf.get("c_kappa", 0.)
        self.use_noise = conf.get("use_noise", True)
        assert self.model.num_out == self.num_obj + self.num_constr
        assert self.num_obj >= 1

    @property
    def num_obj(self):
        return self._num_obj

    @property
    def num_constr(self):
        return self._num_constr

    def eval(self, x, xe):
        with torch.no_grad():
            py, ps2 = self.model.predict(x, xe)
            xi = torch.randn(py.shape) if self.use_noise else None
            dev = torch.device("cuda")
            mu = torch.as_tensor(py).to(dev, torch.float32).t().contiguous()        # [K, m], output-major
            var = torch.as_tensor(ps2).to(dev, torch.float32).t().contiguous()
            noise_sd = self.model.noise.reshape(-1).float().sqrt().to(dev).contiguous() if self.use_noise else None
            xi = None if xi is None else xi.to(dev, torch.float32).contiguous()
            Fo, Fc, _ = _general_epilogue(mu, var, self.num_obj, self.num_constr, self.kappa, self.c_kappa, noise_sd, xi,
                                          want_fc=True)
            out = torch.cat([Fo, Fc], 1)
        probe = x if torch.is_tensor(x) else xe
        return out.to(probe.device if torch.is_tensor(probe) else "cpu")


def _general_epilogue(mu, var, num_obj, num_constr, kappa, c_kappa, noise_sd, xi, seed=0, counter=0, want_fc=False,
                      want_cv=False):
    """(Fo [m, num_obj], Fc [m, num_constr] or None, cv [m] or None) of hb_general_acq_epilogue over mu / var [K, m]."""
    m, dev = mu.shape[1], mu.device
    Fo = torch.empty(m, num_obj, dtype=torch.float32, device=dev)
    Fc = torch.empty(m, num_constr, dtype=torch.float32, device=dev) if want_fc else None
    cv = torch.empty(m, dtype=torch.float32, device=dev) if want_cv else None
    if m:
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().hb_general_acq_epilogue(_lib.ptr(mu), _lib.ptr(var), m, num_obj, num_constr, float(kappa),
                                                          float(c_kappa), _lib.ptr(noise_sd), _lib.ptr(xi), int(seed), int(counter),
                                                          _lib.ptr(Fo), _lib.ptr(Fc) if num_constr else None, _lib.ptr(cv),
                                                          _lib.stream_ptr()), "hb_general_acq_epilogue")
    return Fo, Fc, cv


class MOMeanSigmaLCB(Acquisition):
    """acq.py:99-129: minimise (py, -ps) subject to (py - kappa ps) - best_y <= 0, with py = mu + sqrt(model.noise) xi and
    ps = sqrt(ps2) (no clamp), the acquisition ``HEBO(acq_cls=MOMeanSigmaLCB)`` optimises.  ``eval`` works over any
    single-output model: it takes the N(0, 1) draws from torch's CPU generator as ``torch.randn(py.shape)``, like the
    reference, and runs the arithmetic in the CUDA epilogue ``hb_mo_lcb_epilogue`` (correctly rounded fp32: torch's CPU
    sqrt may differ by one ulp).  Returns [m, 3] on the input's device.  ``general_score`` scores it on the device."""

    def __init__(self, model, best_y, **conf):
        super().__init__(model, **conf)
        self.best_y = best_y
        self.kappa = conf.get("kappa", 2.0)
        assert self.model.num_out == 1

    @property
    def num_obj(self):
        return 2

    @property
    def num_constr(self):
        return 1

    def eval(self, x, xe):
        with torch.no_grad():
            py, ps2 = self.model.predict(x, xe)
            xi = torch.randn(py.shape)
            dev = torch.device("cuda")
            up = lambda v: torch.as_tensor(v).reshape(-1).to(dev, torch.float32).contiguous()
            F, G = _mo_lcb_epilogue(up(py), up(ps2), _noise_sd(self.model), _best_y(self), float(self.kappa), up(xi))
            out = torch.cat([F, G[:, None]], 1)
        probe = x if torch.is_tensor(x) else xe
        return out.to(probe.device if torch.is_tensor(probe) else "cpu")


def _noise_sd(model) -> float:
    """np.sqrt(model.noise) as acq.py:119 takes it: a float32 noise gives its correctly rounded fp32 square root."""
    return float(np.sqrt(np.asarray(model.noise)).reshape(-1)[0])


def _best_y(acq) -> float:
    return float(np.asarray(acq.best_y, dtype=np.float32).reshape(-1)[0])


def _mo_lcb_epilogue(mu, var, noise_sd, best_y, kappa, xi, seed=0, counter=0):
    """(F [m, 2], G [m]) of hb_mo_lcb_epilogue over mu / var [m]."""
    m, dev = mu.shape[0], mu.device
    F = torch.empty(m, 2, dtype=torch.float32, device=dev)
    G = torch.empty(m, dtype=torch.float32, device=dev)
    if m:
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().hb_mo_lcb_epilogue(_lib.ptr(mu), _lib.ptr(var), m, noise_sd, best_y, kappa, _lib.ptr(xi),
                                                     int(seed), int(counter), _lib.ptr(F), _lib.ptr(G), _lib.stream_ptr()),
                       "hb_mo_lcb_epilogue")
    return F, G


def general_score(acq, seed=None):
    """score(xc, xe, gen) of a multi-objective or constrained acquisition for DeviceNSGA2(num_obj=acq.num_obj,
    constrained=acq.num_constr > 0): Fo [m, num_obj] fp32 on the device, and with constraints (Fo, cv [m]), cv the summed
    positive parts of the constraint columns.  A GeneralAcq over a hebo_b200.MultiTaskModel of GPs, or one GP: one
    posterior call per output with F = NULL, writing row b of [K, m] buffers, then hb_general_acq_epilogue with Philox
    draws keyed by (seed, gen).  A MOMeanSigmaLCB over a hebo_b200.GP: one posterior call with F = NULL, then
    hb_mo_lcb_epilogue with Philox draws keyed by (seed, gen), its G being the one constraint column.  With deep
    ensembles -- a GeneralAcq over one multi-output DeepEnsemble or a MultiTaskModel of them, a MOMeanSigmaLCB over one
    DeepEnsemble -- the posterior is one hb_de_predict_batch (GeneralAcq, writing [K, m] directly) or hb_de_predict
    (MOMeanSigmaLCB) call, followed by the same epilogue; with an RF, one hb_rf_predict call and the same epilogues.  None of these synchronises with the host inside a generation;
    an output whose GP fit failed predicts N(y_mean, y_std^2) as GP.predict does.  ``seed`` is drawn from numpy's global
    generator when None.  Any other acquisition or model, including subclasses of these two: acq.eval on CPU tensors (xe as
    int64), once per generation."""
    no, nc = acq.num_obj, acq.num_constr
    model = acq.model
    if type(acq) is MOMeanSigmaLCB and isinstance(model, (GP, DeepEnsemble, RF)):
        return _mo_lcb_device_score(acq, seed)
    if type(acq) is GeneralAcq and _ensembles_of(model) is not None:
        return _general_ensemble_score(acq, _ensembles_of(model), seed)
    if type(acq) is GeneralAcq and isinstance(model, RF):
        return _general_forest_score(acq, seed)
    gps = None
    if isinstance(model, GP):
        gps = [model]
    elif isinstance(model, MultiTaskModel) and all(isinstance(g, GP) for g in model.models):
        gps = model.models
    if type(acq) is not GeneralAcq or gps is None:
        def host_score(xc, xe, gen):
            with torch.no_grad():
                v = torch.as_tensor(acq(xc.cpu(), xe.cpu().long())).reshape(xc.shape[0], no + nc).to(xc.device, torch.float32)
            Fo = v[:, :no].contiguous()
            if nc == 0:
                return Fo
            c = v[:, no:]
            return Fo, torch.where(torch.isnan(c), c, c.clamp_min(0)).sum(1).contiguous()
        return host_score
    seed = int(np.random.randint(0, 2 ** 31 - 1)) if seed is None else int(seed)
    dev = gps[0].device
    noise_sd = model.noise.reshape(-1).float().sqrt().to(dev).contiguous() if acq.use_noise else None
    kappa, c_kappa = float(acq.kappa), float(acq.c_kappa)

    def device_score(xc, xe, gen):
        m = xc.shape[0]
        mu = torch.empty(no + nc, m, dtype=torch.float32, device=dev)
        var = torch.empty_like(mu)
        with torch.no_grad():
            for b, gp in enumerate(gps):
                gp._posterior(gp._to_dev(xc), False, Xe_dev=gp._xe_dev(xe, m), out=(mu[b], var[b]))
        Fo, _, cv = _general_epilogue(mu, var, no, nc, kappa, c_kappa, noise_sd, None, seed, gen, want_cv=nc > 0)
        return (Fo, cv) if nc else Fo
    return device_score


def _ensembles_of(model):
    """The DeepEnsembles behind a GeneralAcq's model as hb_de_predict_batch operands (one multi-output ensemble, or every
    output's single-output ensemble of a MultiTaskModel), or None."""
    if _batchable(model):
        return [model]
    if isinstance(model, MultiTaskModel) and all(_batchable(m) for m in model.models):
        return model.models
    return None


def _batchable(model) -> bool:
    """A DeepEnsemble that hb_de_predict_batch scores: not a FeatureSelectionEnsemble, whose selection layer only its
    own predict entry point applies."""
    return isinstance(model, DeepEnsemble) and not isinstance(model, FeatureSelectionEnsemble)


def _general_ensemble_score(acq, models, seed=None):
    seed = int(np.random.randint(0, 2 ** 31 - 1)) if seed is None else int(seed)
    no, nc, m0 = acq.num_obj, acq.num_constr, models[0]
    batch = EnsembleBatch(models)
    noise_sd = acq.model.noise.reshape(-1).float().sqrt().to(m0.device).contiguous() if acq.use_noise else None
    kappa, c_kappa = float(acq.kappa), float(acq.c_kappa)

    def device_score(xc, xe, gen):
        mu, var, _ = batch.predict(xc if m0.num_cont > 0 else None, xe if m0.num_enum > 0 else None)
        Fo, _, cv = _general_epilogue(mu, var, no, nc, kappa, c_kappa, noise_sd, None, seed, gen, want_cv=nc > 0)
        return (Fo, cv) if nc else Fo
    return device_score


def _general_forest_score(acq, seed=None):
    seed = int(np.random.randint(0, 2 ** 31 - 1)) if seed is None else int(seed)
    no, nc, model = acq.num_obj, acq.num_constr, acq.model
    noise_sd = model.noise.reshape(-1).float().sqrt().to(model.device).contiguous() if acq.use_noise else None
    kappa, c_kappa = float(acq.kappa), float(acq.c_kappa)

    def device_score(xc, xe, gen):
        mu, var, _ = model._predict_dev(xc if model.num_cont > 0 else None, xe if model.num_enum > 0 else None)
        Fo, _, cv = _general_epilogue(mu.reshape(1, -1), var.reshape(1, -1), no, nc, kappa, c_kappa, noise_sd, None, seed, gen,
                                      want_cv=nc > 0)
        return (Fo, cv) if nc else Fo
    return device_score


def _mo_lcb_device_score(acq, seed=None):
    seed = int(np.random.randint(0, 2 ** 31 - 1)) if seed is None else int(seed)
    model = acq.model
    noise_sd, best_y, kappa = _noise_sd(model), _best_y(acq), float(acq.kappa)

    def device_score(xc, xe, gen):
        m = xc.shape[0]
        with torch.no_grad():
            if isinstance(model, GP):
                _, mu, var = model._posterior(model._to_dev(xc), False, Xe_dev=model._xe_dev(xe, m))
            else:
                mu, var = model._predict_dev(xc if model.num_cont > 0 else None, xe if model.num_enum > 0 else None)[:2]
                mu, var = mu.reshape(-1), var.reshape(-1)
        return _mo_lcb_epilogue(mu, var, noise_sd, best_y, kappa, None, seed, gen)
    return device_score


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
            if isinstance(self.model, RF):     # predict + hb_mace_epilogue, draws as acq.py:154-155
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
