"""Generates tests/golden/ref_rf_envelope.npz from the reference's own ``RF`` (models/rf/rf.py) over sklearn.

    HEBO_SRC=<checkout of the HEBO sources> python tests/golden/make_ref_rf_envelope.py

The reference is loaded as make_ref_rf.py loads it, and each tree's bootstrap counts are recovered the same way
(make_ref_rf.record_forest).  The inputs of every variant come from tests/test_oracle_rf_envelope.py's
envelope_inputs (numpy's PCG64 under a fixed seed), so only their SHA-256 is stored, not the megabytes of rows.  sklearn's
bootstrap draws come from numpy's global generator, seeded per variant, so the file regenerates byte for byte under the
recorded sklearn version.  Variants (ENVELOPE in the test module):
  - large-n partitions: n = 8192 at width 64 (Gaussian columns and an integer-valued column with heavy ties), T = 2;
    n = 5000 mixed (8 numeric columns, num_uniqs = [3, 40]), T = 2; n = 2048 at width 1024, T = 1;
  - predict at T = 129 and T = 1024 (n = 50, width 3, 300 held-out rows);
  - held-out rows with NaN in one or more numeric columns, scored through RF.predict.
Per variant: the trees, the bootstrap counts, tree.apply on the training rows, RF.predict (mean, var) on the held-out
rows and RF.noise.  Also whether RF.predict raises ValueError on a +inf and on a -inf candidate.
Test infrastructure; never imported by hebo_b200/.
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from make_ref_rf import load_rf, record_forest  # noqa: E402
from tests.test_oracle_rf_envelope import ENVELOPE, envelope_inputs, inputs_digest  # noqa: E402

OUT = os.path.join(HERE, "ref_rf_envelope.npz")


def main():
    import sklearn
    rf_mod = load_rf()
    out = {"sklearn_version": np.array(sklearn.__version__), "variants": np.array(list(ENVELOPE))}
    model = None
    for vi, (name, (n, m, dc, uniqs, T, _)) in enumerate(ENVELOPE.items()):
        Xc, Xe, y = envelope_inputs(name)
        conf = {"n_estimators": T}
        if uniqs:
            conf["num_uniqs"] = list(uniqs)
        model = rf_mod.RF(dc, len(uniqs), 1, **conf)
        tc = lambda a, s: torch.from_numpy(a[s]) if a is not None else None
        tr, te = slice(0, n), slice(n, n + m)
        np.random.seed(1000 + vi)                      # RandomForestRegressor() draws from numpy's global generator
        model.fit(tc(Xc, tr), tc(Xe, tr), torch.from_numpy(y[tr]).reshape(-1, 1))
        mean, var = model.predict(tc(Xc, te), tc(Xe, te))
        Xtr = model.xtrans(tc(Xc, tr), tc(Xe, tr))
        counts, arrs, apply, ncount = record_forest(model, np.isfinite(y[tr]), Xtr)
        p = name + "/"
        out.update({p + "digest": np.array(inputs_digest(Xc, Xe, y)), p + "counts": counts, p + "ncount": ncount,
                    p + "apply": apply, p + "mean": mean.numpy().reshape(-1), p + "var": var.numpy().reshape(-1),
                    p + "noise": model.noise.numpy()})
        out.update({p + k: v for k, v in arrs.items()})
    # sklearn validates candidates with allow-nan: NaN is scored, +-inf is refused
    x = torch.zeros(1, model.num_cont)
    raises = []
    for v in (np.inf, -np.inf):
        x[0, 0] = float(v)
        try:
            model.predict(x, torch.zeros(1, model.num_enum).long() if model.num_enum else None)
            raises.append(False)
        except ValueError:
            raises.append(True)
    out["inf_raises"] = np.array(raises)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, "sklearn", sklearn.__version__, f"{os.path.getsize(OUT) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
