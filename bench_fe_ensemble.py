"""Feature-selecting deep ensemble (FeDeepEnsemble) on the device: fit, predict and HEBO.suggest, beside the plain deep
ensemble at the same shapes.

    python bench_fe_ensemble.py --out DIR [--ns 50,200,1000] [--ds 8,32,128] [--reps 2]

Fit: the default config (5 members, 128 hidden units, 500 epochs, batch 32) for n x d numeric columns, for each gate
(stg, concrete, hard_concrete) and for DeepEnsemble, timed alternately: per repetition every model is fitted once in turn,
after one warm-up fit of each.  A host clock around calls that end in a device synchronisation; the median is reported.
Predict: candidates/s of predict on device tensors at m = 131 072 (d = 32, CUDA events, 20 calls), both models.
HEBO.suggest (d = 8, n = 50): fit and acquisition ms from its last_timing marks, both models.
The reference's CPU fit is not timed here.  Writes DIR/bench_fe_ensemble.json with the card name and power limit read in
the same run.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_nsga import gpu_info  # noqa: E402
from hebo_b200 import DeepEnsemble, FeDeepEnsemble  # noqa: E402
from hebo_b200.suggest import HEBO  # noqa: E402

MODELS = {"deep_ensemble": (DeepEnsemble, {}), "stg": (FeDeepEnsemble, {"fe_layer": "stg"}),
          "concrete": (FeDeepEnsemble, {"fe_layer": "concrete"}),
          "hard_concrete": (FeDeepEnsemble, {"fe_layer": "hard_concrete"})}


def problem(n, d, seed=0):
    """Only the first two of the d columns matter: the regime the gate is for."""
    g = torch.Generator().manual_seed(seed)
    Xc = torch.rand(n, d, generator=g)
    y = torch.sin(3 * Xc[:, :2]).sum(1, keepdim=True) + 0.05 * torch.randn(n, 1, generator=g)
    return Xc, y


def fit_once(name, n, d):
    cls, conf = MODELS[name]
    Xc, y = problem(n, d)
    torch.manual_seed(0)
    m = cls(d, 0, 1, **conf)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    m.fit(Xc, None, y)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, m


def predict_rate(m, d, M=131072, calls=20):
    xs = torch.rand(M, d, device="cuda")
    m.predict(xs, None)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        m.predict(xs, None)
    b.record()
    torch.cuda.synchronize()
    return M * calls / (a.elapsed_time(b) / 1e3)


def suggest_ms(model_name, reps=3):
    """Median fit and acquisition ms of HEBO.suggest, from the marks it records in last_timing."""
    torch.manual_seed(0)
    opt = HEBO(torch.zeros(8), torch.ones(8), model_name=model_name, scramble_seed=0)
    Xc, y = problem(50, 8, seed=1)
    opt.observe(Xc, y)
    fit, acq = [], []
    for _ in range(reps):
        opt.suggest(1)
        fit.append(opt.last_timing["fit_ms"])
        acq.append(opt.last_timing["score_ms"])
    return statistics.median(fit), statistics.median(acq)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--ns", default="50,200,1000")
    ap.add_argument("--ds", default="8,32,128")
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    res = {"gpu": gpu_info(), "fit_ms": [], "predict_cands_per_s": {}, "suggest_ms": {}}
    for n in (int(v) for v in a.ns.split(",")):
        for d in (int(v) for v in a.ds.split(",")):
            for name in MODELS:
                fit_once(name, n, d)
            times = {name: [] for name in MODELS}
            for _ in range(a.reps):
                for name in MODELS:
                    times[name].append(fit_once(name, n, d)[0])
            row = {"n": n, "d": d, **{name: statistics.median(t) for name, t in times.items()}}
            res["fit_ms"].append(row)
            print(json.dumps(row), flush=True)
    for name in MODELS:
        _, m = fit_once(name, 200, 32)
        res["predict_cands_per_s"][name] = predict_rate(m, 32)
    for model_name in ("deep_ensemble", "fe_deep_ensemble"):
        res["suggest_ms"][model_name] = dict(zip(("fit", "acq"), suggest_ms(model_name)))
    print(json.dumps({k: res[k] for k in ("gpu", "predict_cands_per_s", "suggest_ms")}), flush=True)
    with open(os.path.join(a.out, "bench_fe_ensemble.json"), "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
