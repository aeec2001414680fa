"""Gumbel feature-selection deep ensemble on the device: fit ms for n in {50, 200, 1000} x d in {8, 32, 128} beside the
plain and fe deep ensembles, timed alternately (per repetition each model is fitted once in turn), predict candidates/s,
and HEBO(model_name='gumbel').suggest() fit and acquisition ms from its last_timing marks.  Prints and writes JSON with the card name and power limit (--out DIR).  Default ensemble conf (5 members,
500 epochs, batch 32, 128 hidden units), so the sizes are the ones HEBO users run."""
import argparse
import json
import os
import subprocess
import time

import numpy as np
import torch

from hebo_b200 import DeepEnsemble, FeDeepEnsemble, GumbelDeepEnsemble
from hebo_b200.space import DesignSpace
from hebo_b200.suggest import HEBO


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception:
        return "unknown"


MODELS = (("deep_ensemble", DeepEnsemble), ("fe_deep_ensemble", FeDeepEnsemble), ("gumbel", GumbelDeepEnsemble))


def _fit_once(cls, X, y):
    m = cls(X.shape[1], 0, 1)
    torch.cuda.synchronize()
    t = time.perf_counter()
    m.fit(X, None, y)
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    torch.manual_seed(0)
    res = {"card": _card(), "fit": [], "predict": [], "suggest": []}
    for n in (50, 200, 1000):
        for d in (8, 32, 128):
            X = torch.rand(n, d) * 2 - 1
            y = (X[:, :2] ** 2).sum(1, keepdim=True)
            row = {"n": n, "d": d}
            for _, cls in MODELS:      # warm-up
                _fit_once(cls, X, y)
            ts = {name: [] for name, _ in MODELS}
            for _ in range(a.reps):
                for name, cls in MODELS:
                    t, m = _fit_once(cls, X, y)
                    ts[name].append(t)
            for name, _ in MODELS:
                row[name + "_ms"] = float(np.median(ts[name]))
            res["fit"].append(row)
            print(json.dumps(row), flush=True)
            if n == 200:
                for mc in (10000, 131072):
                    Xs = (torch.rand(mc, d) * 2 - 1).cuda()
                    m.predict(Xs, None, seed=0, counter=0)
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    for c in range(10):
                        m.predict(Xs, None, seed=0, counter=c)
                    torch.cuda.synchronize()
                    rate = 10 * mc / (time.perf_counter() - t)
                    res["predict"].append({"d": d, "m": mc, "candidates_per_s": rate})
                    print(json.dumps(res["predict"][-1]), flush=True)
    sp = DesignSpace().parse([{"name": f"x{i}", "type": "num", "lb": -1, "ub": 1} for i in range(8)])
    for opt in ("sobol", "nsga2"):
        h = HEBO(sp, model_name="gumbel", rand_sample=10, acq_optimizer=opt)
        X0 = h.suggest(10)
        h.observe(X0, (X0.values ** 2).sum(1, keepdims=True))
        h.suggest(1)
        fit, acq = [], []
        for _ in range(a.reps):
            h.suggest(1)
            fit.append(h.last_timing["fit_ms"])
            acq.append(h.last_timing["score_ms"])
        res["suggest"].append({"acq_optimizer": opt, "fit_ms": float(np.median(fit)), "acq_ms": float(np.median(acq))})
        print(json.dumps(res["suggest"][-1]), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_gumbel_ensemble.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
