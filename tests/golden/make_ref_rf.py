"""Generates tests/golden/ref_rf.npz from the reference's own ``RF`` (models/rf/rf.py) over sklearn.

    HEBO_SRC=<checkout of the HEBO sources> python tests/golden/make_ref_rf.py

rf.py, layers.py, base_model.py and util.py are loaded unmodified by path (oracle/ref_loader.py); util.py's
``disjoint_set`` import (used only by get_random_graph) is stubbed, and networkx too when it is not installed.  Per variant
(input kinds numeric / mixed / categorical-only / integer-valued numeric; n in {10, 50, 300}; width in {1, 3, 12};
n_estimators in {1, 20, 100}; the HEBO/test/test_acq.py setup X ~ N(0, 1) [10, 1], y = X; a NaN-y row) it records:
  - the data (Xc, Xe, y) and held-out rows;
  - each tree's bootstrap counts over the training rows, recovered with sklearn's own _generate_sample_indices from the
    tree's random_state (checked against tree_.weighted_n_node_samples[0] == n_kept);
  - each tree's arrays (children_left / right, feature, threshold, value, missing_go_to_left) and tree.apply on the
    training rows (ref_rf.npz was generated before missing_go_to_left was recorded; its held-out rows have no NaN);
  - RF.predict (mean, var) on the held-out rows, and RF.noise.
The sklearn version is stored with them.  Test infrastructure; never imported by hebo_b200/.
"""
from __future__ import annotations

import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ref_rf.npz")
M_TEST = 64
# name: (kind, n, num_cont, num_uniqs, n_estimators)
VARIANTS = {
    "num_n10_w1_t1": ("num", 10, 1, [], 1),
    "num_n50_w3_t20": ("num", 50, 3, [], 20),
    "num_n300_w12_t100": ("num", 300, 12, [], 100),
    "mixed_n50_w3_t20": ("num", 50, 1, [2], 20),
    "mixed_n300_w12_t20": ("num", 300, 4, [3, 5], 20),
    "cat_n50_w3_t20": ("num", 50, 0, [3], 20),
    "cat_n300_w12_t100": ("num", 300, 0, [4, 8], 100),
    "int_n10_w1_t20": ("int", 10, 1, [], 20),
    "int_n50_w3_t20": ("int", 50, 3, [], 20),
    "int_n300_w12_t20": ("int", 300, 12, [], 20),
    "test_acq": ("acq", 10, 1, [], 100),
    "nan_n50_w3_t20": ("nan", 50, 3, [], 20),
}


def load_rf():
    ref_loader.load_reference()                     # _hebo_ref.models.{scalers, base_model}
    ref_loader._load("_hebo_ref.models.layers", "models/layers.py")
    stubs = [("disjoint_set", ["DisjointSet"])]
    if importlib.util.find_spec("networkx") is None:
        stubs.append(("networkx", []))
    ref_loader.load_file("_hebo_ref.models.util", "models/util.py", stubs=stubs)
    import types
    if "_hebo_ref.models.rf" not in sys.modules:
        m = types.ModuleType("_hebo_ref.models.rf")
        m.__path__ = []
        sys.modules["_hebo_ref.models.rf"] = m
    return ref_loader._load("_hebo_ref.models.rf.rf", "models/rf/rf.py")


def record_forest(model, keep, Xtr):
    """(counts [T, n], tree arrays [T, cap], apply [T, n], node counts [T]) of a fitted reference RF: each tree's
    bootstrap counts over the n training rows (keep: the rows filter_nan kept), recovered with sklearn's own
    _generate_sample_indices from the tree's random_state and checked against tree_.weighted_n_node_samples[0]."""
    from sklearn.ensemble._forest import _generate_sample_indices
    kept = np.nonzero(keep)[0]
    n, T = keep.size, len(model.rf.estimators_)
    cap = max(e.tree_.node_count for e in model.rf.estimators_)
    counts = np.zeros((T, n), dtype=np.int32)
    arrs = {k: np.zeros((T, cap), dtype=dt) for k, dt in
            (("left", np.int32), ("right", np.int32), ("feature", np.int32), ("threshold", np.float64), ("value", np.float64),
             ("missing_go_to_left", np.int32))}
    apply = np.zeros((T, n), dtype=np.int32)
    ncount = np.zeros(T, dtype=np.int32)
    for t, est in enumerate(model.rf.estimators_):
        idx = _generate_sample_indices(est.random_state, kept.size, kept.size, None)
        c = np.bincount(idx, minlength=kept.size)
        assert est.tree_.weighted_n_node_samples[0] == kept.size
        counts[t, kept] = c
        k = est.tree_.node_count
        ncount[t] = k
        arrs["left"][t, :k] = est.tree_.children_left
        arrs["right"][t, :k] = est.tree_.children_right
        arrs["feature"][t, :k] = est.tree_.feature
        arrs["threshold"][t, :k] = est.tree_.threshold
        arrs["value"][t, :k] = est.tree_.value.reshape(-1)
        arrs["missing_go_to_left"][t, :k] = est.tree_.missing_go_to_left
        apply[t] = est.apply(Xtr.astype(np.float32))
    return counts, arrs, apply, ncount


def data(kind, n, dc, uniqs, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "acq":
        X = torch.randn(n + M_TEST, 1, generator=g)
        return X, None, X.clone()
    Xc = torch.randn(n + M_TEST, dc, generator=g)
    if kind == "int":
        Xc = torch.randint(0, 4, (n + M_TEST, dc), generator=g).float()
    Xe = torch.stack([torch.randint(0, u, (n + M_TEST,), generator=g) for u in uniqs], 1) if uniqs else None
    base = Xc.sum(1, keepdim=True) + (Xe.float().sum(1, keepdim=True) if uniqs else 0)
    y = torch.sin(base) + 0.1 * torch.randn(n + M_TEST, 1, generator=g)
    if kind == "nan":
        y[7] = float("nan")
    return Xc, Xe, y


def main():
    import sklearn
    rf_mod = load_rf()
    out = {"sklearn_version": np.array(sklearn.__version__), "variants": np.array(list(VARIANTS))}
    for vi, (name, (kind, n, dc, uniqs, T)) in enumerate(VARIANTS.items()):
        Xc, Xe, y = data(kind, n, dc, uniqs, 100 + vi)
        tr = slice(0, n)
        te = slice(n, n + M_TEST)
        conf = {"n_estimators": T}
        if uniqs:
            conf["num_uniqs"] = list(uniqs)
        model = rf_mod.RF(dc, len(uniqs), 1, **conf)
        Xc_tr = Xc[tr] if dc > 0 else None
        Xe_tr = Xe[tr] if uniqs else None
        model.fit(Xc_tr if dc > 0 else torch.zeros(n, 0), Xe_tr, y[tr])
        mean, var = model.predict(Xc[te] if dc > 0 else torch.zeros(M_TEST, 0), Xe[te] if uniqs else None)
        keep = torch.isfinite(y[tr]).all(1).numpy()
        Xtr = model.xtrans(Xc_tr if dc > 0 else torch.zeros(n, 0), Xe_tr)
        counts, arrs, apply, ncount = record_forest(model, keep, Xtr)
        p = name + "/"
        out.update({p + "Xc": (Xc[tr] if dc > 0 else torch.zeros(n, 0)).numpy(), p + "y": y[tr].numpy(),
                    p + "Xc_test": (Xc[te] if dc > 0 else torch.zeros(M_TEST, 0)).numpy(),
                    p + "Xe": (Xe[tr] if uniqs else torch.zeros(n, 0).long()).numpy(),
                    p + "Xe_test": (Xe[te] if uniqs else torch.zeros(M_TEST, 0).long()).numpy(),
                    p + "uniqs": np.array(uniqs, dtype=np.int32), p + "T": np.array(T), p + "counts": counts,
                    p + "ncount": ncount, p + "apply": apply, p + "mean": mean.numpy(), p + "var": var.numpy(),
                    p + "noise": model.noise.numpy()})
        out.update({p + k: v for k, v in arrs.items()})
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, "sklearn", sklearn.__version__)


if __name__ == "__main__":
    main()
