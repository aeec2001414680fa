"""Deep-ensemble surrogate behind HEBO's ``BaseModel`` plugin surface.

Drop-in for ``hebo.models.nn.deep_ensemble.DeepEnsemble`` (HEBO/hebo/models/nn/deep_ensemble.py:29-181): the same
constructor keys and defaults, the same ``fit / predict / noise / sample_f`` contract with CPU tensors in and out, but the
whole fit of every member runs in one launch of ``hb_de_fit`` and prediction in ``hb_de_predict`` /
``hb_de_predict_grad`` (hebo_b200/csrc/ensemble.cu); nothing falls back to torch.

Initial weights are drawn on the host from torch's global CPU generator in BaseNet's registration order and shapes
(xavier_uniform_ with the ReLU gain for every weight, embedding tables included; zero biases) and uploaded once.  The
minibatch order of each member's epochs is a keyed Philox bijection on the device, seeded from the same generator.

Deliberate deviation: the reference calls ``torch.seed()`` at the start of every ``fit_one`` (:152), which makes each fit
irreproducible and reseeds the caller's global generator.  This port does not reseed, so a fit is reproducible under
``torch.manual_seed``.

Extra conf key: ``device`` (default 'cuda').
"""
from __future__ import annotations

import ctypes as C
from importlib import import_module

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .base import BaseModel
from .scalers import MinMaxScaler, StandardScaler


def param_layout(num_cont, num_uniqs, enum_trans, num_layers, num_hiddens, num_out, output_noise, rand_prior):
    """[(state_dict name, shape)] of one BaseNet in registration order (deep_ensemble.py:183-221); the flat raw vector of
    hb_de_fit is their concatenation."""
    out = []
    din = num_cont
    if num_uniqs:
        if enum_trans == "embedding":
            for c, u in enumerate(num_uniqs):
                w = min(50, 1 + u // 2)
                out.append((f"enum_layer.emb.{c}.weight", (u, w)))
                din += w
        else:
            din += sum(num_uniqs)

    def mlp(prefix):
        k = din
        for l in range(num_layers):
            out.append((f"{prefix}.{2 * l}.weight", (num_hiddens, k)))
            out.append((f"{prefix}.{2 * l}.bias", (num_hiddens,)))
            k = num_hiddens
    mlp("hidden")
    out += [("mu.weight", (num_out, num_hiddens)), ("mu.bias", (num_out,))]
    if output_noise:
        out += [("sigma2.0.weight", (num_out, num_hiddens)), ("sigma2.0.bias", (num_out,))]
    if rand_prior:
        mlp("prior_net")
        out += [("prior_net.prior_net_out.weight", (num_out, num_hiddens)), ("prior_net.prior_net_out.bias", (num_out,))]
    return out, din


def init_params(layout) -> torch.Tensor:
    """BaseNet's initialisation (:217-221) from torch's global CPU generator, in registration order; a feature gate's
    parameter (FeNet's feature_select, last) is 0.01 randn (fe_layers.py:26, 82)."""
    parts = []
    for name, shape in layout:
        t = torch.empty(shape)
        if name.startswith("feature_select."):
            t = 0.01 * torch.randn(shape)
        elif "bias" in name:
            nn.init.zeros_(t)
        else:
            nn.init.xavier_uniform_(t, gain=nn.init.calculate_gain("relu"))
        parts.append(t.reshape(-1))
    return torch.cat(parts)


def state_dict_to_raw(sd, layout) -> torch.Tensor:
    return torch.cat([sd[name].detach().float().reshape(-1) for name, _ in layout])


def raw_to_state_dict(raw: torch.Tensor, layout) -> dict:
    out, o = {}, 0
    for name, shape in layout:
        k = int(np.prod(shape))
        out[name] = raw[o:o + k].reshape(shape).clone()
        o += k
    return out


def _reference_net(module: str, name: str):
    """Class `name` of an installed HEBO's hebo.models.nn.`module`, or None."""
    try:  # pragma: no cover - depends on the environment
        return getattr(import_module(f"hebo.models.nn.{module}"), name)
    except Exception:
        return None


def _is_basenet(cls, ref_basenet) -> bool:
    """basenet_cls names the stock network: the installed reference's BaseNet itself when HEBO is importable; without it,
    a class named BaseNet defined in a module named deep_ensemble (the reference file loaded some other way).  A subclass
    or a look-alike elsewhere is not trained as BaseNet: it raises."""
    if ref_basenet is not None:
        return cls is ref_basenet
    return getattr(cls, "__name__", "") == "BaseNet" and str(getattr(cls, "__module__", "")).rsplit(".", 1)[-1] == "deep_ensemble"


def _check_categories(Xe, num_uniqs) -> None:
    """nn.Embedding / F.one_hot raise on a category outside 0 .. num_uniq - 1 (layers.py:34, 50); so does this model."""
    Xe = torch.as_tensor(Xe)
    if Xe.numel() == 0:
        return
    hi = torch.as_tensor(num_uniqs, dtype=torch.int64, device=Xe.device)
    if bool((Xe.long() < 0).any()) or bool((Xe.long() >= hi).any()):
        raise IndexError("categorical index out of range")


def _check_perm(perm, E: int, T: int, n: int) -> None:
    """A caller-given minibatch order must be [E, T, n] with every row a permutation of 0 .. n - 1: hb_de_fit indexes the
    training rows with it unchecked."""
    p = torch.as_tensor(perm)
    if tuple(p.shape) != (E, T, n):
        raise ValueError(f"perm must be [num_ensembles, num_epochs, n] = [{E}, {T}, {n}], got {list(p.shape)}")
    if p.numel() and not bool((torch.sort(p.reshape(-1, n).long(), dim=1).values == torch.arange(n, device=p.device)).all()):
        raise ValueError("every row of perm must be a permutation of 0 .. n - 1")


class _PredictWithGrad(torch.autograd.Function):
    """DeepEnsemble.predict as an autograd node over ``hb_de_predict_grad``."""

    @staticmethod
    def forward(ctx, Xs, model, xe):
        mu, var, dmu, dvar = model._predict_dev(Xs, xe, grad=True)
        ctx.save_for_backward(dmu, dvar)
        return mu, var

    @staticmethod
    def backward(ctx, gmu, gvar):
        dmu, dvar = ctx.saved_tensors          # [m, O, d]
        return (gmu.unsqueeze(2) * dmu + gvar.unsqueeze(2) * dvar).sum(1), None, None


class DeepEnsemble(BaseModel):
    support_ts = True
    support_grad = True
    support_multi_output = True
    support_warm_start = True

    def __init__(self, num_cont, num_enum, num_out, **conf):
        super().__init__(num_cont, num_enum, num_out, **conf)
        self.conf = conf
        # deep_ensemble.py:36-51 (keys and defaults)
        self.bootstrap = self.conf.setdefault("bootstrap", False)        # accepted, unused (as in the reference)
        self.rand_prior = self.conf.setdefault("rand_prior", False)
        self.output_noise = self.conf.setdefault("output_noise", True)
        self.num_ensembles = self.conf.setdefault("num_ensembles", 5)
        self.num_process = self.conf.setdefault("num_processes", 1)      # accepted; one launch trains every member
        self.num_epochs = self.conf.setdefault("num_epochs", 500)
        self.print_every = self.conf.setdefault("print_every", 50)
        self.num_layers = self.conf.setdefault("num_layers", 1)
        self.num_hiddens = self.conf.setdefault("num_hiddens", 128)
        self.l1 = self.conf.setdefault("l1", 1e-3)
        self.batch_size = self.conf.setdefault("batch_size", 32)
        self.lr = self.conf.setdefault("lr", 5e-3)
        self.adv_eps = self.conf.setdefault("adv_eps", 0.)              # accepted, unused (as in the reference)
        self.verbose = self.conf.setdefault("verbose", False)
        ref_basenet = _reference_net("deep_ensemble", "BaseNet")
        self.basenet_cls = self.conf.setdefault("basenet_cls", ref_basenet)
        assert self.num_ensembles > 0
        if self.basenet_cls is not None and not _is_basenet(self.basenet_cls, ref_basenet):
            raise NotImplementedError("DeepEnsemble: only BaseNet members are supported (basenet_cls)")
        act = self.conf.get("act", None)
        if act is not None and type(act) is not nn.ReLU:
            raise NotImplementedError("DeepEnsemble: only the nn.ReLU activation is supported (act)")
        # BaseNet's own keys (:189-205)
        self.noise_lb = float(self.conf.get("noise_lb", 1e-4))
        self.enum_trans = self.conf.get("enum_trans", "embedding") if num_enum > 0 else "embedding"
        if self.enum_trans not in ("embedding", "onehot"):
            raise RuntimeError(f"Unknown enum processing type {self.enum_trans}, can only be [embedding|onehot]")
        self.num_uniqs = [int(u) for u in self.conf["num_uniqs"]] if num_enum > 0 else []
        self.device = torch.device(self.conf.get("device", "cuda"))
        self.layout, self.din = param_layout(num_cont, self.num_uniqs, self.enum_trans, self.num_layers, self.num_hiddens,
                                             num_out, self.output_noise, self.rand_prior)
        self._check_envelope()
        self._c_uniqs = (C.c_int32 * max(1, num_enum))(*self.num_uniqs)
        self._spec = _lib.DeSpec(num_cont, num_enum, self._c_uniqs,
                                 _lib.HB_DE_EMBEDDING if self.enum_trans == "embedding" else _lib.HB_DE_ONEHOT,
                                 self.num_layers, self.num_hiddens, num_out, int(bool(self.output_noise)),
                                 int(bool(self.rand_prior)), self.noise_lb)
        self.P = sum(int(np.prod(s)) for _, s in self.layout)
        self.xscaler = MinMaxScaler((-1, 1))
        self.yscaler = StandardScaler()
        self.loss_name = "NLL" if self.output_noise else "MSE"
        self.params = None          # [E, P] device tensor once fitted (the reference's self.models)
        self.sample_idx = 0
        self.noise_est = torch.zeros(self.num_out)
        self.losses = None

    def _check_envelope(self):
        L = _lib
        for what, v, lim in (("num_layers", self.num_layers, L.HB_DE_MAX_LAYERS), ("num_hiddens", self.num_hiddens, L.HB_DE_MAX_HIDDEN),
                             ("num_out", self.num_out, L.HB_DE_MAX_OUT),
                             ("input width (num_cont + embedding / one-hot width)", self.din, L.HB_DE_MAX_IN),
                             ("num_ensembles", self.num_ensembles, L.HB_DE_MAX_MEMBERS)):
            if v > lim:
                raise NotImplementedError(f"DeepEnsemble: {what} = {v} exceeds the limit of {lim}")
        if self.num_layers < 1 or self.num_hiddens < 1:
            raise NotImplementedError("DeepEnsemble: num_layers and num_hiddens must be at least 1")

    def batch_floats(self, rows: int) -> int:
        """Shared-memory floats a fit minibatch of `rows` rows needs (HB_DE_MAX_BATCH_FLOATS of include/hebo_b200.h)."""
        h_ld = max(self.num_hiddens, self.din) | 1
        return rows * ((self.din | 1) + (self.num_layers + 2) * h_ld + 5 * self.num_out + 1)

    @property
    def fitted(self):
        return self.params is not None

    @property
    def noise(self) -> torch.Tensor:
        return self.noise_est

    # ------------------------------------------------------------------ scaling (deep_ensemble.py:118-138)
    def fit_scaler(self, Xc, Xe, y):
        if Xc is not None and Xc.shape[1] > 0:
            self.xscaler.fit(Xc)
        self.yscaler.fit(y)

    def trans(self, Xc, Xe, y=None):
        if Xc is not None and Xc.shape[1] > 0:
            Xc_t = self.xscaler.transform(Xc)
        else:
            Xc_t = torch.zeros(Xe.shape[0], 0)
        Xe_t = torch.zeros(Xc.shape[0], 0).long() if Xe is None else Xe.long()
        if y is not None:
            return Xc_t, Xe_t, self.yscaler.transform(y)
        return Xc_t, Xe_t

    # ------------------------------------------------------------------ fit (deep_ensemble.py:71-93, 151-181)
    def fit(self, Xc_, Xe_, y_, perm=None):
        """perm: optional [E, num_epochs, n] int32 minibatch order of each member's epochs over the filtered rows (tests);
        otherwise the device's Philox order under a seed drawn from torch's generator."""
        Xc, Xe, y, valid = self._prepare_fit(Xc_, Xe_, y_, perm)
        self._fit_dev(Xc, Xe, y, perm, self.seed)
        self._finish_fit(Xc_, Xe_, y_, valid)

    def _prepare_fit(self, Xc_, Xe_, y_, perm=None):
        """fit's host side up to the launch: the row filter, the scalers (first fit only), the initial weights (first fit
        only) and then the seed, both from torch's generator.  Returns the filtered, scaled (Xc, Xe, y) and the row mask."""
        y_ = torch.as_tensor(y_).float()
        if self.num_enum > 0:
            _check_categories(Xe_, self.num_uniqs)
        valid = torch.isfinite(y_).any(dim=1)
        Xc = Xc_[valid] if Xc_ is not None else None
        Xe = Xe_[valid] if Xe_ is not None else None
        y = y_[valid]
        if not self.yscaler.fitted:             # the first fit only: `if self.models is None: self.fit_scaler(...)`
            self.fit_scaler(Xc, Xe, y)
        Xc, Xe, y = self.trans(Xc, Xe, y)
        n, E, dev = y.shape[0], self.num_ensembles, self.device
        if perm is not None:
            _check_perm(perm, E, int(self.num_epochs), n)
        rows = min(n, int(self.batch_size))
        if self.batch_floats(rows) > _lib.HB_DE_MAX_BATCH_FLOATS:
            raise NotImplementedError(
                f"DeepEnsemble: a minibatch of {rows} rows needs {self.batch_floats(rows)} floats of on-chip buffers, over "
                f"the limit of {_lib.HB_DE_MAX_BATCH_FLOATS} (HB_DE_MAX_BATCH_FLOATS); use a smaller batch_size")
        if self.params is None:
            self.params = torch.stack([self.init_member() for _ in range(E)]).to(dev).contiguous()
        self.seed = int(torch.randint(0, 2 ** 62, (1,)).item())     # the Philox key of this fit's minibatch order
        return Xc, Xe, y, valid

    def init_member(self) -> torch.Tensor:
        """One member's initial raw parameters [P] from torch's global generator."""
        return init_params(self.layout)

    def _finish_fit(self, Xc_, Xe_, y_, valid, **predict_kw):
        """fit's host side after the launch: the noise estimate on the kept rows (deep_ensemble.py:89-93); predict_kw
        goes to that predict."""
        self.sample_idx = 0
        with torch.no_grad():
            py, _ = self.predict(Xc_, Xe_, **predict_kw)
            err = (py - torch.as_tensor(y_).float())[valid]
            self.noise_est = (err ** 2).mean(dim=0).detach().clone()

    def _print_losses(self):
        L = self.losses.cpu()
        for i in range(self.num_ensembles):
            for ep in range(0, int(self.num_epochs), self.print_every):
                print("Epoch %d, %s loss = %g" % (ep, self.loss_name, float(L[i, ep])), flush=True)

    def _fit_dev(self, Xc, Xe, y, perm, seed):
        lib, dev, E = _lib.lib(), self.device, self.num_ensembles
        n, T = y.shape[0], int(self.num_epochs)
        xc = Xc.to(dev, torch.float32).contiguous() if self.num_cont > 0 else None
        xe = Xe.to(dev, torch.int32).contiguous() if self.num_enum > 0 else None
        yd = y.to(dev, torch.float32).contiguous()
        pd_ = None if perm is None else torch.as_tensor(perm).to(dev, torch.int32).contiguous()
        need = int(lib.hb_de_fit_workspace_bytes(C.byref(self._spec), E))
        self.fit_ws = torch.empty(need, dtype=torch.uint8, device=dev)
        losses = torch.empty(E, max(1, T), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.hb_de_fit(_lib.ptr(xc), _lib.ptr(xe), _lib.ptr(yd), n, C.byref(self._spec), E, _lib.ptr(self.params),
                                     float(self.lr), float(self.l1), int(self.batch_size), T, _lib.ptr(pd_), seed & (2 ** 64 - 1),
                                     _lib.ptr(losses), _lib.ptr(self.fit_ws), need, _lib.stream_ptr()), "hb_de_fit")
        self.losses = losses[:, :T]
        if self.verbose:
            self._print_losses()

    def fit_state(self):
        """Views of the fit workspace: Adam's exp_avg, exp_avg_sq and the last step's gradient, each [E, P]."""
        E, P = self.num_ensembles, self.P
        return tuple(self.fit_ws.view(torch.float32)[:3 * E * P].view(3, E, P))

    # ------------------------------------------------------------------ predict (deep_ensemble.py:95-116)
    def _scal_dev(self):
        dev = self.device
        if self.num_cont > 0:
            xm, xa = self.xscaler.scale_.to(dev).contiguous(), self.xscaler.min_.to(dev).contiguous()
        else:
            xm = xa = None
        return xm, xa, self.yscaler.mean.to(dev).contiguous(), self.yscaler.std.to(dev).contiguous()

    def _inputs(self, Xc, Xe):
        dev = self.device
        m = (Xc if (Xc is not None and self.num_cont > 0) else Xe).shape[0]
        xe = None
        if self.num_enum > 0:
            Xe = torch.as_tensor(Xe)
            if not Xe.is_cuda:          # device categories are not read back (a GA batch is in range by construction);
                _check_categories(Xe, self.num_uniqs)      # the kernels turn an out-of-range one into a NaN row
            xe = Xe.to(dev, torch.int32).contiguous()
        xs = torch.as_tensor(Xc).detach().to(dev, torch.float32).contiguous() if self.num_cont > 0 else None
        return xs, xe, m

    def _predict_dev(self, Xs, xe, grad=False, member=-1):
        lib, dev = _lib.lib(), self.device
        assert self.fitted, "fit() first"
        m = (Xs if Xs is not None else xe).shape[0]
        xm, xa, ym, ys = self._scal_dev()
        mu = torch.empty(m, self.num_out, dtype=torch.float32, device=dev)
        var = torch.empty(m, self.num_out, dtype=torch.float32, device=dev) if member < 0 else None
        with torch.cuda.device(dev):
            if grad:
                dmu = torch.empty(m, self.num_out, self.num_cont, dtype=torch.float32, device=dev)
                dvar = torch.empty_like(dmu)
                _lib.check(lib.hb_de_predict_grad(_lib.ptr(Xs), _lib.ptr(xe), m, C.byref(self._spec), self.num_ensembles,
                                                  _lib.ptr(self.params), _lib.ptr(xm), _lib.ptr(xa), _lib.ptr(ym), _lib.ptr(ys),
                                                  _lib.ptr(mu), _lib.ptr(var), _lib.ptr(dmu), _lib.ptr(dvar),
                                                  _lib.stream_ptr()), "hb_de_predict_grad")
                return mu, var, dmu, dvar
            _lib.check(lib.hb_de_predict(_lib.ptr(Xs), _lib.ptr(xe), m, C.byref(self._spec), self.num_ensembles,
                                         _lib.ptr(self.params), _lib.ptr(xm), _lib.ptr(xa), _lib.ptr(ym), _lib.ptr(ys),
                                         int(member), _lib.ptr(mu), _lib.ptr(var), _lib.stream_ptr()), "hb_de_predict")
        return mu, var

    def predict(self, Xc, Xe=None):
        """(py, ps2) [m, num_out]: CPU tensors for CPU inputs, device tensors for device inputs; an input with
        requires_grad goes through the input-gradient kernel."""
        probe = Xc if (Xc is not None and self.num_cont > 0) else Xe
        on_cpu = not (torch.is_tensor(probe) and probe.is_cuda)
        xs, xe, m = self._inputs(Xc, Xe)
        if torch.is_tensor(Xc) and Xc.requires_grad and self.num_cont > 0:
            mu, var = _PredictWithGrad.apply(Xc.to(self.device, torch.float32).contiguous(), self, xe)
            return mu.to(Xc.device), var.to(Xc.device)
        mu, var = self._predict_dev(xs, xe)
        return (mu.cpu(), var.cpu()) if on_cpu else (mu, var)

    def sample_y(self, Xc, Xe=None, n_samples: int = 1):
        """BaseModel.sample_y (base_model.py:78-84): py + sqrt(ps2) * N(0, 1), independent draws, [n_samples, m, num_out].
        One hb_de_predict_batch launch with in-kernel Philox draws keyed by a seed from torch's global generator, so the
        result is reproducible under torch.manual_seed (the reference draws torch.randn on the host).  CPU tensors for CPU
        inputs."""
        probe = Xc if (Xc is not None and self.num_cont > 0) else Xe
        on_cpu = not (torch.is_tensor(probe) and probe.is_cuda)
        xs, xe, _ = self._inputs(Xc, Xe)
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        _, _, samp = EnsembleBatch([self]).predict(xs, xe, n_samples=n_samples, seed=seed)
        return samp.cpu() if on_cpu else samp

    def predict_mace(self, Xc, tau: float, kappa: float, eps: float = 1e-4, xi1=None, xi2=None, seed: int = 0,
                     return_mu_var: bool = False, Xe=None, device_out: bool = False):
        """predict + MACE.eval (acq.py:146-171) through ``hb_mace_epilogue``: F [m, 3] = (LCB, -logEI, -logPI), on the
        input's device (device_out=True: on the GPU for host inputs too).  Single-output models."""
        assert self.num_out == 1, "MACE needs a single-output model"
        probe = Xc if (Xc is not None and self.num_cont > 0) else Xe
        on_cpu = not (torch.is_tensor(probe) and probe.is_cuda) and not device_out
        xs, xe, m = self._inputs(Xc, Xe)
        if xi1 is None:
            xi1 = torch.randn(m, 1)          # acq.py:154-155
            xi2 = torch.randn(m, 1)
        dev = self.device
        xi1 = torch.as_tensor(xi1).reshape(-1).to(dev, torch.float32).contiguous()
        xi2 = torch.as_tensor(xi2).reshape(-1).to(dev, torch.float32).contiguous()
        mu, var = self._predict_dev(xs, xe)
        mu, var = mu.reshape(-1), var.reshape(-1)
        F = torch.empty(m, 3, dtype=torch.float32, device=dev)
        if m:
            with torch.cuda.device(dev):
                _lib.check(_lib.lib().hb_mace_epilogue(_lib.ptr(mu), _lib.ptr(var), m, float(self.noise[0]), float(tau),
                                                       float(kappa), float(eps), _lib.ptr(xi1), _lib.ptr(xi2), int(seed),
                                                       _lib.ptr(F), _lib.stream_ptr()), "hb_mace_epilogue")
        if on_cpu:
            F, mu, var = F.cpu(), mu.cpu(), var.cpu()
        return (F, mu, var) if return_mu_var else F

    def sample_f(self):
        assert self.fitted
        idx = self.sample_idx
        self.sample_idx = (self.sample_idx + 1) % self.num_ensembles

        def f(Xc, Xe):
            probe = Xc if (Xc is not None and self.num_cont > 0) else Xe
            on_cpu = not (torch.is_tensor(probe) and probe.is_cuda)
            xs, xe, _ = self._inputs(Xc, Xe)
            mu, _ = self._predict_dev(xs, xe, member=idx)
            return mu.cpu() if on_cpu else mu
        return f

    def state_dicts(self):
        """One BaseNet state_dict per member, from the device parameters."""
        raw = self.params.cpu()
        return [raw_to_state_dict(raw[i], self.layout) for i in range(self.num_ensembles)]


def _stacked_params(models) -> torch.Tensor:
    """[B, E, P] device parameters of B ensembles: the common tensor when their params are consecutive slices of one
    (as fit_ensembles leaves them), otherwise a stacked copy."""
    base = models[0].params
    step = base.numel() * base.element_size()
    if all(m.params.is_contiguous() and m.params.data_ptr() == base.data_ptr() + b * step for b, m in enumerate(models)):
        return torch.as_strided(base, (len(models),) + tuple(base.shape), (base.numel(), base.shape[1], 1))
    return torch.stack([m.params for m in models]).contiguous()


class EnsembleBatch:
    """B fitted DeepEnsembles of one spec (one multi-output ensemble, or the single-output ensembles of a MultiTaskModel)
    as one ``hb_de_predict_batch`` operand.  The stacked parameters and scalers are taken when it is built."""

    def __init__(self, models):
        m0 = models[0]
        assert all(m.fitted for m in models), "fit() first"
        for m in models:
            if isinstance(m, FeatureSelectionEnsemble):
                raise TypeError(f"EnsembleBatch: a {type(m).__name__} predicts through {m._C_PREDICT}, which applies its "
                                "selection layer")
        self.models, self.spec, self.E, self.device = models, m0._spec, m0.num_ensembles, m0.device
        self.num_cont, self.num_out = m0.num_cont, len(models) * m0.num_out
        self.params = _stacked_params(models)
        sc = [m._scal_dev() for m in models]
        self.xm = torch.stack([t[0] for t in sc]).contiguous() if self.num_cont > 0 else None
        self.xa = torch.stack([t[1] for t in sc]).contiguous() if self.num_cont > 0 else None
        self.ym = torch.stack([t[2] for t in sc]).contiguous()
        self.ys = torch.stack([t[3] for t in sc]).contiguous()

    def predict(self, xs, xe, n_samples: int = 0, xi=None, seed: int = 0, counter: int = 0):
        """(mu, var) [B num_out, m] output-major, and y_samp [n_samples, m, B num_out] (None when n_samples = 0), from
        device inputs xs [m, num_cont] fp32 (None without numeric columns) and xe [m, num_enum] int32."""
        m = (xs if xs is not None else xe).shape[0]
        dev, K = self.device, self.num_out
        mu = torch.empty(K, m, dtype=torch.float32, device=dev)
        var = torch.empty_like(mu)
        samp = torch.empty(n_samples, m, K, dtype=torch.float32, device=dev) if n_samples > 0 else None
        xi = None if xi is None else torch.as_tensor(xi).to(dev, torch.float32).contiguous()
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().hb_de_predict_batch(
                _lib.ptr(xs), _lib.ptr(xe), m, C.byref(self.spec), len(self.models), self.E, _lib.ptr(self.params),
                _lib.ptr(self.xm), _lib.ptr(self.xa), _lib.ptr(self.ym), _lib.ptr(self.ys), _lib.ptr(mu), _lib.ptr(var),
                int(n_samples), _lib.ptr(xi), int(seed) & (2 ** 64 - 1), int(counter), _lib.ptr(samp), _lib.stream_ptr()),
                "hb_de_predict_batch")
        return mu, var, samp


def batch_offsets(ns) -> list:
    """off [B + 1] of hb_de_fit_batch: ensemble b's rows are off[b] .. off[b + 1] - 1 of the concatenation."""
    return [0] + np.cumsum(np.asarray(ns, dtype=np.int64)).tolist()


def fit_ensembles(models, Xc, Xe, ys) -> None:
    """model.fit(Xc, Xe, ys[b]) for every model b of B DeepEnsembles with one spec, in ONE hb_de_fit_batch launch.  The
    host side runs model by model in the order the sequential loop draws from torch's generator (model b: its initial
    weights on its first fit, then its seed), so every model ends bit-identical to its own fit.  Each model keeps its own
    row filter and scalers; afterwards its params, fit workspace and losses are slices of the batch's tensors."""
    m0 = models[0]
    B, E, T, dev = len(models), m0.num_ensembles, int(m0.num_epochs), m0.device
    if B > _lib.HB_MAX_OUTPUTS:
        raise NotImplementedError(f"fit_ensembles: {B} ensembles exceed the limit of {_lib.HB_MAX_OUTPUTS} (HB_MAX_OUTPUTS)")
    preps = [m._prepare_fit(Xc, Xe, y) for m, y in zip(models, ys)]
    off = batch_offsets([p[2].shape[0] for p in preps])
    xc = torch.cat([p[0] for p in preps]).to(dev, torch.float32).contiguous() if m0.num_cont > 0 else None
    xe = torch.cat([p[1] for p in preps]).to(dev, torch.int32).contiguous() if m0.num_enum > 0 else None
    yd = torch.cat([p[2] for p in preps]).to(dev, torch.float32).contiguous()
    params = torch.stack([m.params for m in models]).contiguous()
    lib = _lib.lib()
    need = int(lib.hb_de_fit_workspace_bytes(C.byref(m0._spec), E))
    ws = torch.empty(B * need, dtype=torch.uint8, device=dev)
    losses = torch.empty(B, E, max(1, T), dtype=torch.float32, device=dev)
    c_off = (C.c_int64 * (B + 1))(*off)
    c_seed = (C.c_uint64 * B)(*[m.seed & (2 ** 64 - 1) for m in models])
    with torch.cuda.device(dev):
        _lib.check(lib.hb_de_fit_batch(_lib.ptr(xc), _lib.ptr(xe), _lib.ptr(yd), c_off, B, C.byref(m0._spec), E,
                                       _lib.ptr(params), float(m0.lr), float(m0.l1), int(m0.batch_size), T, c_seed,
                                       _lib.ptr(losses), _lib.ptr(ws), B * need, _lib.stream_ptr()), "hb_de_fit_batch")
    for b, m in enumerate(models):
        m.params, m.fit_ws, m.losses = params[b], ws[b * need:(b + 1) * need], losses[b, :, :T]
        if m.verbose:
            m._print_losses()
        m._finish_fit(Xc, Xe, ys[b], preps[b][3])


class FeatureSelectionEnsemble(DeepEnsemble):
    """The host side shared by FeDeepEnsemble and GumbelDeepEnsemble: a DeepEnsemble whose members pass their inputs
    through a random selection layer, after BaseNet's parameters, before the first hidden layer.  A subclass names its C
    entry points (_C_FIT, _C_FIT_WS, _C_PREDICT), the variant arguments they take after the spec (_layout_args,
    _fit_args, _predict_args, the last with predict's workspace tensor or None) and what a fit of T epochs leaves for
    predict (_trained_epochs).

    The selection is random in predict too (the reference redraws it on every forward): each call draws afresh from a
    Philox key taken from torch's global generator, or from the given ``seed`` / ``counter``, so a call is reproducible
    under ``torch.manual_seed``.  No input gradients (``support_grad = False``).  Like DeepEnsemble, the fit does not call
    ``torch.seed()``, a deliberate deviation that keeps it reproducible under ``torch.manual_seed``."""
    support_grad = False

    def fit(self, Xc_, Xe_, y_, perm=None, draws=None, eval_draws=None):
        """perm: as DeepEnsemble.fit.  draws: optional training draws (``draws_shape``); otherwise Philox draws on the
        device.  eval_draws: optional draws of the noise estimate's predict (``eval_draws_shape``; tests replaying the
        reference's own draws)."""
        Xc, Xe, y, valid = self._prepare_fit(Xc_, Xe_, y_, perm)
        if draws is not None:
            draws = torch.as_tensor(draws, dtype=torch.float32)
            if tuple(draws.shape) != self.draws_shape(y.shape[0]):
                raise ValueError(f"draws must be {list(self.draws_shape(y.shape[0]))}, got {list(draws.shape)}")
        self._fit_dev(Xc, Xe, y, perm, self.seed, draws)
        self._finish_fit(Xc_, Xe_, y_, valid, draws=eval_draws)

    def _fit_dev(self, Xc, Xe, y, perm, seed, draws=None):
        lib, dev, E = _lib.lib(), self.device, self.num_ensembles
        n, T = y.shape[0], int(self.num_epochs)
        xc = Xc.to(dev, torch.float32).contiguous() if self.num_cont > 0 else None
        xe = Xe.to(dev, torch.int32).contiguous() if self.num_enum > 0 else None
        yd = y.to(dev, torch.float32).contiguous()
        pd_ = None if perm is None else torch.as_tensor(perm).to(dev, torch.int32).contiguous()
        dd = None if draws is None else draws.to(dev, torch.float32).contiguous()
        need = int(getattr(lib, self._C_FIT_WS)(C.byref(self._spec), *self._layout_args(), E))
        self.fit_ws = torch.empty(need, dtype=torch.uint8, device=dev)
        losses = torch.empty(E, max(1, T), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(getattr(lib, self._C_FIT)(_lib.ptr(xc), _lib.ptr(xe), _lib.ptr(yd), n, C.byref(self._spec),
                                                 *self._fit_args(), E, _lib.ptr(self.params), float(self.lr), float(self.l1),
                                                 int(self.batch_size), T, _lib.ptr(pd_), _lib.ptr(dd), seed & (2 ** 64 - 1),
                                                 _lib.ptr(losses), _lib.ptr(self.fit_ws), need, _lib.stream_ptr()),
                       self._C_FIT)
        self.losses = losses[:, :T]
        if T > 0:
            self._trained_epochs(T)
        if self.verbose:
            self._print_losses()

    def _predict_dev(self, Xs, xe, grad=False, member=-1, draws=None, seed=None, counter=0):
        if grad:
            raise NotImplementedError(f"{type(self).__name__}: no input gradients (support_grad = False)")
        lib, dev = _lib.lib(), self.device
        assert self.fitted, "fit() first"
        m = (Xs if Xs is not None else xe).shape[0]
        xm, xa, ym, ys = self._scal_dev()
        mu = torch.empty(m, self.num_out, dtype=torch.float32, device=dev)
        var = torch.empty(m, self.num_out, dtype=torch.float32, device=dev) if member < 0 else None
        if draws is not None:
            draws = torch.as_tensor(draws).to(dev, torch.float32).contiguous()
            if tuple(draws.shape) != self.eval_draws_shape():
                raise ValueError(f"eval draws must be {list(self.eval_draws_shape())}, got {list(draws.shape)}")
        elif seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        head, ws = self._predict_args()
        tail = () if ws is None else (_lib.ptr(ws), ws.numel() * ws.element_size())
        with torch.cuda.device(dev):
            _lib.check(getattr(lib, self._C_PREDICT)(_lib.ptr(Xs), _lib.ptr(xe), m, C.byref(self._spec), *head,
                                                     self.num_ensembles, _lib.ptr(self.params), _lib.ptr(xm), _lib.ptr(xa),
                                                     _lib.ptr(ym), _lib.ptr(ys), int(member), _lib.ptr(draws),
                                                     int(seed or 0) & (2 ** 64 - 1), int(counter) & (2 ** 64 - 1),
                                                     _lib.ptr(mu), _lib.ptr(var), *tail, _lib.stream_ptr()),
                       self._C_PREDICT)
        return mu, var

    def predict(self, Xc, Xe=None, draws=None, seed=None, counter=0):
        """(py, ps2) [m, num_out] under a fresh selection: CPU tensors for CPU inputs, device tensors for device inputs.
        draws (``eval_draws_shape``): the selection's raw draws (tests); otherwise Philox keyed by (seed, counter), seed
        from torch's generator when None."""
        probe = Xc if (Xc is not None and self.num_cont > 0) else Xe
        on_cpu = not (torch.is_tensor(probe) and probe.is_cuda)
        xs, xe, _ = self._inputs(Xc, Xe)
        mu, var = self._predict_dev(xs, xe, draws=draws, seed=seed, counter=counter)
        return (mu.cpu(), var.cpu()) if on_cpu else (mu, var)

    def sample_y(self, Xc, Xe=None, n_samples: int = 1):
        """BaseModel.sample_y (base_model.py:78-84): one predict, then py + sqrt(ps2) * torch.randn per sample."""
        py, ps2 = self.predict(Xc, Xe)
        ps = ps2.sqrt()
        samp = torch.zeros(n_samples, py.shape[0], self.num_out, device=py.device)
        for i in range(n_samples):
            samp[i] = py + ps * torch.randn(py.shape).to(py.device)
        return samp


_FE_KINDS = {"stg": _lib.HB_FE_STG, "concrete": _lib.HB_FE_CONCRETE, "hard_concrete": _lib.HB_FE_HARD_CONCRETE}
_FE_DEFAULT_T = {"stg": 1.0, "concrete": 0.1, "hard_concrete": 0.1}      # the layers' constructor defaults


def fe_epoch_temperature(start_temp: float, end_temp: float, anneal_base: float, epoch: int) -> float:
    """The concrete layers' temperature of an epoch as fe_deep_ensemble.py:59-60 rounds it: the product in double, then
    torch.tensor (fp32) clamped below at end_temp."""
    return float(np.float32(max(start_temp * anneal_base ** epoch, end_temp)))


class FeDeepEnsemble(FeatureSelectionEnsemble):
    """Drop-in for ``hebo.models.nn.fe_deep_ensemble.FeDeepEnsemble``: a DeepEnsemble whose members gate their input
    columns with a learned feature-selection layer (``fe_layer``: 'stg' (default), 'concrete' or 'hard_concrete') before
    the first hidden layer, so irrelevant inputs can be switched off.  The fit runs in one ``hb_fe_fit`` launch and
    prediction in ``hb_fe_predict`` (hebo_b200/csrc/ensemble.cu, the deep ensemble's kernels with the gate compiled in).

    Extra conf keys and defaults: fe_layer 'stg', temperature None (the layer's own: 1.0 for stg, 0.1 otherwise),
    mask_reg 0.1, start_temp 1.0, end_temp 0.1, anneal_base 0.99.  A member's parameters are FeNet's state_dict in
    registration order: BaseNet's, then ``feature_select.mu`` (stg) or ``feature_select.logits`` [din] last.  The L1 term
    covers weights only, the mask penalty applies when there are numeric columns, and the random prior net (rand_prior)
    is built but not evaluated, all as the reference does.  Predict draws fresh eval masks on every call."""
    _C_FIT, _C_FIT_WS, _C_PREDICT = "hb_fe_fit", "hb_fe_fit_workspace_bytes", "hb_fe_predict"

    def __init__(self, num_cont, num_enum, num_out, **conf):
        fe_layer = conf.get("fe_layer", "stg")
        if fe_layer not in _FE_KINDS:
            raise KeyError(f"FeDeepEnsemble: unknown fe_layer {fe_layer!r}, can only be [stg|concrete|hard_concrete]")
        conf.pop("basenet_cls", None)
        super().__init__(num_cont, num_enum, num_out, **conf)
        self.basenet_cls = _reference_net("fe_deep_ensemble", "FeNet")
        self.conf["basenet_cls"] = self.basenet_cls
        self.fe_layer = fe_layer
        self.temperature = self.conf.get("temperature")
        self.mask_reg = self.conf.get("mask_reg", 0.1)
        self.end_temp = self.conf.get("end_temp", 0.1)
        self.start_temp = self.conf.get("start_temp", 1.0)
        self.anneal_base = self.conf.get("anneal_base", 0.99)
        t = self.temperature if self.temperature else _FE_DEFAULT_T[fe_layer]      # FeNet: `if self.temperature:`
        self.gate_temperature = float(np.float32(t))        # stg's T throughout; the concrete layers' until a fit
        self.layout = self.layout + [("feature_select.mu" if fe_layer == "stg" else "feature_select.logits", (self.din,))]
        self.P += self.din

    def batch_floats(self, rows: int) -> int:
        """On-chip floats of a gated minibatch: the deep ensemble's plus the unmasked inputs and gate states."""
        return super().batch_floats(rows) + 2 * rows * (self.din | 1)

    def _gate(self):
        return _lib.FeGate(_FE_KINDS[self.fe_layer], self.gate_temperature, float(self.start_temp), float(self.end_temp),
                           float(self.anneal_base), float(self.mask_reg))

    def draws_shape(self, n: int):
        """Shape of fit's explicit training draws for n kept rows: [E, num_epochs, minibatches, rows, din]; N(0, 1) for
        stg, U(0, 1) for the concrete layers."""
        bs = int(self.batch_size)
        return (self.num_ensembles, int(self.num_epochs), n // bs if n > bs else 1, min(n, bs), self.din)

    def eval_draws_shape(self):
        """Shape of predict's explicit draws: one per member and input column, [E, din]."""
        return (self.num_ensembles, self.din)

    def _layout_args(self):
        return ()

    def _fit_args(self):
        return (C.byref(self._gate()),)

    def _predict_args(self):
        return (C.byref(self._gate()),), None

    def _trained_epochs(self, T: int):
        if self.fe_layer != "stg":       # predict uses the last epoch's temperature
            self.gate_temperature = fe_epoch_temperature(self.start_temp, self.end_temp, self.anneal_base, T - 1)


def gumbel_epoch_temperature(epoch: int) -> float:
    """GumbelDeepEnsemble.fit_one's temperature of an epoch (gumbel_linear.py:81), a double that torch uses as fp32(T)."""
    return float(np.float32(0.8 ** epoch + 0.1))


class GumbelDeepEnsemble(FeatureSelectionEnsemble):
    """Drop-in for ``hebo.models.nn.gumbel_linear.GumbelDeepEnsemble``: a DeepEnsemble whose members map their numeric
    columns to ``reduced_dim`` learned soft selections of them (a Gumbel-softmax selection layer, one draw of its
    [reduced_dim, num_cont] matrix per forward) before the first hidden layer.  The fit runs in one ``hb_gumbel_fit``
    launch and prediction in ``hb_gumbel_predict`` (hebo_b200/csrc/ensemble.cu, the deep ensemble's kernels with the
    selection layer compiled in).

    Extra conf key and default: reduced_dim = num_cont // 2 + 1.  A member's parameters are GumbelNet's state_dict in
    order: BaseNet's over the selected width, then ``feature_select.logits`` [reduced_dim, num_cont] last.  The hidden
    layers (rebuilt by GumbelNet when num_cont > 0) keep torch's default nn.Linear initialisation, the logits start at
    zero.  Every epoch's minibatches cover all rows (no drop_last); the L1 term covers weights only; the temperature is
    0.8**epoch + 0.1.  The random prior net (rand_prior) needs reduced_dim == num_cont or no numeric columns.  Predict
    draws one matrix per member on every call, at the last trained epoch's temperature."""
    _C_FIT, _C_FIT_WS, _C_PREDICT = "hb_gumbel_fit", "hb_gumbel_fit_workspace_bytes", "hb_gumbel_predict"

    def __init__(self, num_cont, num_enum, num_out, **conf):
        conf.pop("basenet_cls", None)
        self.reduced_dim = int(conf.setdefault("reduced_dim", num_cont // 2 + 1))
        if self.reduced_dim < 1:
            raise NotImplementedError("GumbelDeepEnsemble: reduced_dim must be at least 1")
        if conf.get("rand_prior", False) and num_cont > 0 and self.reduced_dim != num_cont:
            raise NotImplementedError("GumbelDeepEnsemble: rand_prior needs reduced_dim == num_cont (the prior net keeps the "
                                      "unselected input width, so the reference fails in forward)")
        if num_cont > _lib.HB_DE_MAX_IN:
            raise NotImplementedError(f"GumbelDeepEnsemble: num_cont = {num_cont} exceeds the limit of {_lib.HB_DE_MAX_IN}")
        super().__init__(num_cont, num_enum, num_out, **conf)
        self.basenet_cls = _reference_net("gumbel_linear", "GumbelNet")
        self.conf["basenet_cls"] = self.basenet_cls
        self.temperature = 0.1          # GumbelSelectionLayer's default until a fit sets the last epoch's

    def _check_envelope(self):
        """GumbelNet's layout replaces BaseNet's here, before DeepEnsemble's envelope check and parameter count read it:
        BaseNet's over the selected width (num_cont -> reduced_dim when num_cont > 0), then the logits."""
        sel = self.reduced_dim if self.num_cont > 0 else 0
        lay, self.din = param_layout(sel, self.num_uniqs, self.enum_trans, self.num_layers, self.num_hiddens, self.num_out,
                                     self.output_noise, self.rand_prior)
        self.layout = lay + [("feature_select.logits", (self.reduced_dim, self.num_cont))]
        super()._check_envelope()

    def batch_floats(self, rows: int) -> int:
        """On-chip floats of a minibatch: the deep ensemble's over the selected width plus the numeric rows."""
        return super().batch_floats(rows) + (rows * (self.num_cont | 1) if self.num_cont > 0 else 0)

    def draws_shape(self, n: int):
        """Shape of fit's explicit training uniforms for n kept rows: [E, num_epochs, ceil(n / batch), r, num_cont]."""
        bs = min(n, int(self.batch_size))
        return (self.num_ensembles, int(self.num_epochs), -(-n // bs), self.reduced_dim, self.num_cont)

    def eval_draws_shape(self):
        """Shape of predict's explicit uniforms: one matrix per member, [E, reduced_dim, num_cont]."""
        return (self.num_ensembles, self.reduced_dim, self.num_cont)

    def init_member(self) -> torch.Tensor:
        """GumbelNet's initialisation from torch's global generator: BaseNet's (xavier with the ReLU gain, zero biases) over
        its own layout; with numeric columns the hidden layers are then rebuilt with nn.Linear's default initialisation
        (kaiming-uniform weights, U(+-1/sqrt(fan_in)) biases), and the logits are zeros."""
        full, _ = param_layout(self.num_cont, self.num_uniqs, self.enum_trans, self.num_layers, self.num_hiddens,
                               self.num_out, self.output_noise, self.rand_prior)
        base = raw_to_state_dict(init_params(full), full)
        if self.num_cont > 0:
            k = self.din
            for l in range(self.num_layers):
                lin = nn.Linear(k, self.num_hiddens)
                base[f"hidden.{2 * l}.weight"], base[f"hidden.{2 * l}.bias"] = lin.weight.detach(), lin.bias.detach()
                k = self.num_hiddens
        base["feature_select.logits"] = torch.zeros(self.reduced_dim, self.num_cont)
        return state_dict_to_raw(base, self.layout)

    def _layout_args(self):
        return (self.reduced_dim,)

    def _fit_args(self):
        return (self.reduced_dim,)

    def _predict_args(self):
        """reduced_dim and the temperature, and the workspace of each member's W [E, reduced_dim, num_cont]."""
        ws = torch.empty(max(1, self.num_ensembles * self.reduced_dim * self.num_cont), dtype=torch.float32,
                         device=self.device)
        return (self.reduced_dim, float(self.temperature)), ws

    def _trained_epochs(self, T: int):
        self.temperature = gumbel_epoch_temperature(T - 1)      # predict uses the last trained epoch's temperature
