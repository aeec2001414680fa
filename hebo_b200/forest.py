"""Random-forest surrogate behind HEBO's ``BaseModel`` plugin surface.

Drop-in for ``hebo.models.rf.rf.RF`` (HEBO/hebo/models/rf/rf.py:19-56): the same constructor key (``n_estimators``,
default 100; HEBO's own default config passes 20) and the same ``fit / predict / noise`` contract with CPU tensors in and
out, but every tree is grown on the device in one ``hb_rf_fit`` call and candidates are scored through the whole forest by
``hb_rf_predict`` (hebo_b200/csrc/forest.cu); nothing falls back to sklearn.

The trees are exact CART on bootstrap weights, as sklearn's ``RandomForestRegressor`` with the defaults the reference
uses.  Where sklearn breaks ties at random, the device takes the highest proxy, then the lowest feature, then the lowest
cut; this changes no in-bag partition, only where out-of-bag inputs fall.  ``predict`` reproduces the reference's fp32
outputs bit for bit for the same trees (sklearn's sequential tree sum for the mean, numpy's pairwise sums for np.var).

Candidates: a NaN is scored as sklearn scores it, going at each node to the child with more distinct training rows
(``tree_.missing_go_to_left``).  Host candidates with +-inf raise ``ValueError``, as sklearn's input validation does.
Device candidates are not read back (the GA scorers keep them on the device) and are not checked: there +inf goes right
and -inf goes left at every node, the decisions of the threshold comparison.

Deliberate deviation: the reference is unseeded (``RandomForestRegressor`` without ``random_state``).  This port draws its
bootstrap key from torch's global generator, so a fit is reproducible under ``torch.manual_seed``.

Extra conf key: ``device`` (default 'cuda').
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .base import BaseModel
from .ensemble import _check_categories


class RF(BaseModel):
    support_ts = False
    support_grad = False
    support_multi_output = False
    support_warm_start = False

    def __init__(self, num_cont, num_enum, num_out, **conf):
        if num_out != 1:
            raise NotImplementedError("RF: single-output only (the reference's BaseModel asserts num_out == 1)")
        super().__init__(num_cont, num_enum, num_out, **conf)
        self.n_estimators = int(self.conf.get("n_estimators", 100))          # rf.py:22
        self.num_uniqs = [int(u) for u in self.conf["num_uniqs"]] if num_enum > 0 else []
        self.width = num_cont + sum(self.num_uniqs)
        if not 1 <= self.n_estimators <= _lib.HB_RF_MAX_TREES:
            raise NotImplementedError(f"RF: n_estimators = {self.n_estimators} is outside 1 .. {_lib.HB_RF_MAX_TREES}")
        if self.width > _lib.HB_RF_MAX_WIDTH:
            raise NotImplementedError(f"RF: input width (num_cont + sum(num_uniqs)) = {self.width} exceeds the limit of "
                                      f"{_lib.HB_RF_MAX_WIDTH}")
        self.device = torch.device(self.conf.get("device", "cuda"))
        self._c_uniqs = (C.c_int32 * max(1, num_enum))(*self.num_uniqs)
        self._spec = _lib.RfSpec(num_cont, num_enum, self._c_uniqs)
        self.est_noise = torch.zeros(self.num_out)
        self.forest = None          # device bytes of hb_rf_forest_bytes(spec, 2 n - 1, 1, T) once fitted
        self.n = 0
        self.seed = None

    @property
    def fitted(self) -> bool:
        return self.forest is not None

    @property
    def noise(self) -> torch.Tensor:
        return self.est_noise

    # ------------------------------------------------------------------ fit (rf.py:37-43)
    def fit(self, Xc, Xe, y, counts=None):
        """counts: optional [1, T, n] (or [T, n]) int bootstrap counts over the given rows (tests); otherwise the device's
        Philox draws under a seed from torch's generator.  Rows with non-finite y weigh 0 (filter_nan, rf.py:38)."""
        y = torch.as_tensor(y).float().reshape(-1, 1)
        n = y.shape[0]
        if self.num_cont > 0:
            assert torch.isfinite(torch.as_tensor(Xc)).all()                # util.py:19
        if self.num_enum > 0:
            _check_categories(Xe, self.num_uniqs)
        assert torch.isfinite(y).any(), "No valid data in the dataset"       # util.py:21
        if n > _lib.HB_RF_MAX_ROWS:
            raise NotImplementedError(f"RF: {n} training rows exceed the limit of {_lib.HB_RF_MAX_ROWS}")
        T, dev, lib = self.n_estimators, self.device, _lib.lib()
        xc, xe, _ = self._inputs(Xc, Xe)
        cd = None
        if counts is not None:
            cd = torch.as_tensor(counts).reshape(1, T, n).to(dev, torch.int32).contiguous()
        self.seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        ws_bytes = int(lib.hb_rf_fit_workspace_bytes(n, C.byref(self._spec), 1, T))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        forest = torch.empty(int(lib.hb_rf_forest_bytes(C.byref(self._spec), 2 * n - 1, 1, T)), dtype=torch.uint8, device=dev)
        noise = torch.empty(1, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.hb_rf_fit(_lib.ptr(xc), _lib.ptr(xe), _lib.ptr(y.to(dev).contiguous()), n, C.byref(self._spec), 1,
                                     T, _lib.ptr(cd), self.seed, _lib.ptr(forest), _lib.ptr(noise), _lib.ptr(ws), ws_bytes,
                                     _lib.stream_ptr()), "hb_rf_fit")
        self.forest, self.n, self._noise_dev = forest, n, noise
        self.est_noise = noise.cpu()

    def load_trees(self, trees, noise: float = 0.0):
        """Take a fitted forest from sklearn-layout trees (``tree_.children_left / children_right / feature / threshold``,
        ``value`` and optionally ``missing_go_to_left`` of each tree, as dicts of arrays; without it NaN goes right), for
        scoring trees grown elsewhere."""
        T = len(trees)
        assert T == self.n_estimators, "one tree per estimator"
        cap = max(int(np.asarray(t["feature"]).size) for t in trees)
        dev = self.device

        def stack(key, dt, fill):
            a = np.full((T, cap), fill, dtype=dt)
            for i, t in enumerate(trees):
                v = np.asarray(t.get(key, fill)).reshape(-1)
                a[i, :v.size] = v
            return torch.from_numpy(a).to(dev).contiguous()
        L, R, Fe = stack("left", np.int32, -1), stack("right", np.int32, -1), stack("feature", np.int32, -2)
        Th, V = stack("threshold", np.float64, -2.0), stack("value", np.float64, 0.0)
        nan_left = (stack("missing_go_to_left", np.int32, 0) != 0) & (L >= 0)
        Fe = torch.where(nan_left, Fe | _lib.HB_RF_NAN_LEFT, Fe)          # hb_rf_load reads the flag from the feature
        cnt = torch.tensor([int(np.asarray(t["feature"]).size) for t in trees], dtype=torch.int32, device=dev)
        lib = _lib.lib()
        forest = torch.empty(int(lib.hb_rf_forest_bytes(C.byref(self._spec), cap, 1, T)), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.hb_rf_load(_lib.ptr(L), _lib.ptr(R), _lib.ptr(Fe), _lib.ptr(Th), _lib.ptr(V), _lib.ptr(cnt),
                                      C.byref(self._spec), T, cap, _lib.ptr(forest), _lib.stream_ptr()), "hb_rf_load")
        self.forest = forest
        self.est_noise = torch.tensor([noise], dtype=torch.float32)
        self._noise_dev = self.est_noise.to(dev)

    def trees(self):
        """The fitted forest as sklearn-layout dicts (feature, threshold, left, right, value), one per tree."""
        return forest_trees(self.forest)

    # ------------------------------------------------------------------ predict (rf.py:49-56)
    def _inputs(self, Xc, Xe):
        dev = self.device
        m = (Xc if (Xc is not None and self.num_cont > 0) else Xe).shape[0]
        xe = None
        if self.num_enum > 0:
            Xe = torch.as_tensor(Xe)
            if not Xe.is_cuda:          # device categories are not read back; the kernel turns an out-of-range one into NaN
                _check_categories(Xe, self.num_uniqs)
            xe = Xe.to(dev, torch.int32).contiguous()
        xs = None
        if self.num_cont > 0:
            Xc = torch.as_tensor(Xc).detach()
            if not Xc.is_cuda and torch.isinf(Xc).any():          # sklearn's check_array(..., allow-nan)
                raise ValueError("RF: input contains infinity")
            xs = Xc.to(dev, torch.float32).contiguous()
        return xs, xe, m

    def _predict_dev(self, xs, xe, n_samples: int = 0, seed: int = 0, counter: int = 0):
        """(mean [m, 1], var [m, 1], samples [n_samples, m, 1] or None) on the device from device inputs."""
        assert self.fitted, "fit() first"
        dev = self.device
        m = (xs if xs is not None else xe).shape[0]
        mean = torch.empty(m, 1, dtype=torch.float32, device=dev)
        var = torch.empty_like(mean)
        samp = torch.empty(n_samples, m, 1, dtype=torch.float32, device=dev) if n_samples > 0 else None
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().hb_rf_predict(_lib.ptr(xs), _lib.ptr(xe), m, C.byref(self._spec), _lib.ptr(self.forest), 1,
                                                self.n_estimators, _lib.ptr(self._noise_dev), _lib.ptr(mean), _lib.ptr(var),
                                                int(n_samples), int(seed) & (2 ** 64 - 1), int(counter), _lib.ptr(samp),
                                                _lib.stream_ptr()), "hb_rf_predict")
        return mean, var, samp

    def _on_cpu(self, Xc, Xe) -> bool:
        probe = Xc if (Xc is not None and self.num_cont > 0) else Xe
        return not (torch.is_tensor(probe) and probe.is_cuda)

    def predict(self, Xc, Xe=None):
        """(py, ps2) [m, 1]: CPU tensors for CPU inputs, device tensors for device inputs."""
        xs, xe, _ = self._inputs(Xc, Xe)
        mean, var, _ = self._predict_dev(xs, xe)
        return (mean.cpu(), var.cpu()) if self._on_cpu(Xc, Xe) else (mean, var)

    def sample_y(self, Xc, Xe=None, n_samples: int = 1):
        """BaseModel.sample_y (base_model.py:78-84): py + sqrt(ps2) N(0, 1), [n_samples, m, 1], drawn in the predict launch
        under a key from torch's global generator (reproducible under torch.manual_seed)."""
        xs, xe, _ = self._inputs(Xc, Xe)
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        _, _, samp = self._predict_dev(xs, xe, n_samples=n_samples, seed=seed)
        return samp.cpu() if self._on_cpu(Xc, Xe) else samp

    def predict_mace(self, Xc, tau: float, kappa: float, eps: float = 1e-4, xi1=None, xi2=None, seed: int = 0,
                     return_mu_var: bool = False, Xe=None, device_out: bool = False):
        """predict + MACE.eval (acq.py:146-171) through ``hb_mace_epilogue``: F [m, 3] = (LCB, -logEI, -logPI), on the
        input's device (device_out=True: on the GPU for host inputs too)."""
        on_cpu = self._on_cpu(Xc, Xe) and not device_out
        xs, xe, m = self._inputs(Xc, Xe)
        if xi1 is None:
            xi1 = torch.randn(m, 1)          # acq.py:154-155
            xi2 = torch.randn(m, 1)
        dev = self.device
        xi1 = torch.as_tensor(xi1).reshape(-1).to(dev, torch.float32).contiguous()
        xi2 = torch.as_tensor(xi2).reshape(-1).to(dev, torch.float32).contiguous()
        mu, var, _ = self._predict_dev(xs, xe)
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


def forest_trees(f: torch.Tensor) -> list:
    """The trees of a device forest (include/hebo_b200.h) as sklearn-layout dicts: feature (-2 at a leaf), threshold (-2 at
    a leaf), left / right (-1 at a leaf), value, missing_go_to_left (0 / 1), and thr32 (the fp32 threshold the traversal
    compares), tree b T + t at index b T + t."""
    h = f[:32].cpu().view(torch.int32).numpy()
    cap, B, T, woh, ne = (int(v) for v in h[:5])
    align = lambda b: (b + 255) // 256 * 256
    o = 256 + align(4 * (ne + woh))
    cnt = f[o:o + 4 * B * T].cpu().view(torch.int32).numpy()
    o += align(4 * B * T)
    nn = B * T * cap
    nodes = f[o:o + 16 * nn].cpu().view(torch.int32).numpy().reshape(B * T, cap, 4)
    o += align(16 * nn)
    thr = f[o:o + 8 * nn].cpu().view(torch.float64).numpy().reshape(B * T, cap)
    o += align(8 * nn)
    val = f[o:o + 8 * nn].cpu().view(torch.float64).numpy().reshape(B * T, cap)
    out = []
    for t in range(B * T):
        k = int(cnt[t])
        nd = nodes[t, :k]
        leaf = nd[:, 0] < 0
        feature = np.where(leaf, nd[:, 0], nd[:, 0] & (_lib.HB_RF_NAN_LEFT - 1)).astype(np.int32)
        out.append(dict(feature=feature, threshold=thr[t, :k].copy(), left=np.where(leaf, -1, nd[:, 2]),
                        right=np.where(leaf, -1, nd[:, 3]), value=val[t, :k].copy(),
                        missing_go_to_left=np.where(leaf, 0, (nd[:, 0] & _lib.HB_RF_NAN_LEFT) != 0).astype(np.int32),
                        thr32=nd[:, 1].view(np.float32).copy()))
    return out
