"""Host-side scalers and NaN filter with the reference's semantics.

MinMaxScaler / StandardScaler mirror TorchMinMaxScaler / TorchStandardScaler
(HEBO/hebo/models/scalers.py:33-90), which fit with sklearn on the numpy view of the tensor and apply in
torch: the fit statistics below are sklearn's formulas (`_handle_zeros_in_scale` included), without the
sklearn dependency.  filter_nan mirrors HEBO/hebo/models/util.py:18-30.
"""
from __future__ import annotations

import numpy as np
import torch


class MinMaxScaler:
    def __init__(self, range=(0, 1)):
        self.range_lb = float(range[0])
        self.range_ub = float(range[1])
        assert self.range_ub > self.range_lb
        self.scale_ = None
        self.min_ = None
        self.fitted = False

    def fit(self, x: torch.Tensor):
        assert x.dim() == 2
        X = x.detach().cpu().numpy()
        dmin, dmax = np.nanmin(X, axis=0), np.nanmax(X, axis=0)
        rng = dmax - dmin
        rng = np.where(rng < 10 * np.finfo(rng.dtype).eps, np.ones_like(rng), rng)   # sklearn _handle_zeros_in_scale
        scale = (self.range_ub - self.range_lb) / rng
        self.scale_ = torch.FloatTensor(np.asarray(scale, dtype=np.float32))
        self.min_ = torch.FloatTensor(np.asarray(self.range_lb - dmin * scale, dtype=np.float32))
        self.fitted = True
        return self

    def transform(self, x: torch.Tensor) -> torch.Tensor:
        return self.scale_.to(x.device) * x + self.min_.to(x.device)

    __call__ = transform

    def inverse_transform(self, x: torch.Tensor) -> torch.Tensor:
        return (x - self.min_.to(x.device)) / self.scale_.to(x.device)


class StandardScaler:
    def __init__(self):
        self.mean = None
        self.std = None
        self.fitted = False

    def fit(self, x: torch.Tensor):
        assert x.dim() == 2
        X = x.detach().cpu().numpy().astype(np.float64)
        mean = np.nanmean(X, axis=0) if np.isfinite(X).any() else np.zeros(X.shape[1])
        var = np.nanvar(X, axis=0) if np.isfinite(X).any() else np.ones(X.shape[1])
        std = np.sqrt(var)
        std = np.where(std < 10 * np.finfo(np.float64).eps, 1.0, std)                 # sklearn _handle_zeros_in_scale
        self.mean = torch.FloatTensor(mean.astype(np.float32)).view(-1)
        self.std = torch.FloatTensor(std.astype(np.float32)).view(-1)
        invalid = ~(torch.isfinite(self.mean) & torch.isfinite(self.std))
        self.mean[invalid] = 0.0
        self.std[invalid] = 1.0
        self.fitted = True
        return self

    def transform(self, x: torch.Tensor) -> torch.Tensor:
        return (x - self.mean.to(x.device)) / self.std.to(x.device)

    __call__ = transform

    def inverse_transform(self, x: torch.Tensor) -> torch.Tensor:
        return x * self.std.to(x.device) + self.mean.to(x.device)


def filter_nan(x, xe, y, keep_rule="any"):
    assert x is None or torch.isfinite(x).all()
    assert xe is None or torch.isfinite(xe).all()
    assert torch.isfinite(y).any(), "No valid data in the dataset"
    if keep_rule == "any":
        valid = torch.isfinite(y).any(dim=1)
    else:
        valid = torch.isfinite(y).all(dim=1)
    return (x[valid] if x is not None else None, xe[valid] if xe is not None else None, y[valid])


def kumaraswamy_warp(Xt: torch.Tensor, a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Kumaraswamy-CDF input warp on MinMax(-1,1)-scaled inputs (BASELINE config 3); the reference's only
    definitions are KumarWarp (HEBO/hebo/models/nn/mono_layers/layers.py:85-117) and GPy's InputWarpedGP
    (HEBO/hebo/models/gp/gpy_wgp.py:120-128): u in [eps, 1-eps], w = 1 - (1 - u^a)^b, mapped back to [-1,1].
    1 - u^a is formed as -expm1(a log u) as kumar_warp (common.cuh) forms it: 1 - u ** a cancels to 0 in fp32 at the
    upper clamp once a <= 0.031."""
    eps = 1e-6
    u = ((Xt + 1.0) * 0.5).clamp(eps, 1.0 - eps)
    x = a * torch.log(u)
    # the value is -expm1(x); its derivative is taken through -exp(x) (t.detach() - t adds exactly 0): torch
    # differentiates expm1 as expm1(x) + 1, which rounds to 0 in fp32 once e^x < 2^-24 (a = 10 below u = 0.19)
    t = torch.exp(x)
    om = -torch.expm1(x).detach() + (t.detach() - t) if torch.is_grad_enabled() and x.requires_grad else -torch.expm1(x)
    return 2.0 * (1.0 - torch.exp(b * torch.log(om))) - 1.0
