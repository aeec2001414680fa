"""Load the reference's real source files (HEBO's ``acq.py`` / ``scalers.py`` / ``base_model.py`` and a few layers) by
path.

TEST INFRASTRUCTURE ONLY: used by ``oracle/make_golden.py`` to regenerate the committed fixtures under tests/golden/ from
a checkout of the HEBO sources, given as ``HEBO_SRC=<directory that contains hebo/>``.  Nothing else (tests, smoke(),
bench.py) reads the reference; the tests compare against the stored vectors.

``import hebo`` itself needs pymoo / gpytorch (evolution_optimizer.py:14, gp.py:14); the files below import only
torch/numpy/sklearn/pandas and load unmodified under stub parent packages.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

REF_ROOT = os.path.join(os.environ.get("HEBO_SRC", ""), "hebo")


def available() -> bool:
    return bool(os.environ.get("HEBO_SRC")) and os.path.isfile(os.path.join(REF_ROOT, "acquisitions", "acq.py"))


def load_file(modname: str, relpath: str, stubs=()):
    """Load one reference source file unmodified under stub parents: stubs = [(module name, attribute names)]"""
    saved = {}
    for name, attrs in stubs:
        saved[name] = sys.modules.get(name)
        m = types.ModuleType(name)
        m.__path__ = []
        for k in attrs:
            setattr(m, k, type(k, (), {}))
        sys.modules[name] = m
    try:
        spec = importlib.util.spec_from_file_location(modname, os.path.join(REF_ROOT, relpath))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[modname] = mod
        spec.loader.exec_module(mod)
        return mod
    finally:
        for name, old in saved.items():
            if old is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = old


def _load(modname: str, relpath: str):
    if modname in sys.modules:
        return sys.modules[modname]
    spec = importlib.util.spec_from_file_location(modname, os.path.join(REF_ROOT, relpath))
    mod = importlib.util.module_from_spec(spec)
    sys.modules[modname] = mod
    spec.loader.exec_module(mod)
    return mod


def load_reference():
    """Returns a namespace with the reference's MACE, Mean, Sigma, BaseModel, scalers."""
    if not available():
        raise RuntimeError("set HEBO_SRC to a checkout of the HEBO sources")
    for pkg in ("_hebo_ref", "_hebo_ref.models", "_hebo_ref.acquisitions"):
        if pkg not in sys.modules:
            m = types.ModuleType(pkg)
            m.__path__ = []          # mark as package so relative imports resolve
            sys.modules[pkg] = m
    scalers = _load("_hebo_ref.models.scalers", "models/scalers.py")
    base_model = _load("_hebo_ref.models.base_model", "models/base_model.py")
    acq = _load("_hebo_ref.acquisitions.acq", "acquisitions/acq.py")
    ns = types.SimpleNamespace(MACE=acq.MACE, Mean=acq.Mean, Sigma=acq.Sigma, LCB=acq.LCB,
                               Acquisition=acq.Acquisition, BaseModel=base_model.BaseModel,
                               TorchMinMaxScaler=scalers.TorchMinMaxScaler,
                               TorchStandardScaler=scalers.TorchStandardScaler)
    return ns
