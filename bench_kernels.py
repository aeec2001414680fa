"""The four GP kernels side by side on bench.py's synthetic problem (Hartmann-6 embedded in d dims, n = 4096).

For each kernel (Matern-1/2, Matern-3/2, Matern-5/2, RBF) and d in {32, 100}:
  fit_ms          the 100-epoch device fit without the Langevin term (deterministic RMSprop), host clock around
                  synchronised work;
  cand_per_s      fused posterior + MACE over 131 072 scrambled-Sobol candidates (GP.predict_mace, device rows, Philox
                  draws), CUDA events around 5 calls after 2 warm-up calls;
  guard_flagged_frac  candidate rows the precision guard re-contracted on the FP32 pipe, over those timed calls.
The kernels alternate inside every repetition (the starting kernel rotates), and each number is the median of --reps
repetitions.  A separate torch.profiler run (one 10-epoch fit and 3 scoring calls per configuration) gives the mean device
time per launch of kstar_kernel, gram_kernel and mll_grad_kernel.  The card's name and power limit are read in the same
process.  Writes bench_kernels.json under --out and prints it as one JSON line."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import candidates, synth  # noqa: E402

KERNELS = ["matern12", "matern32", "matern52", "rbf"]
PROFILED = ("kstar_kernel", "gram_kernel", "mll_grad_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (v.strip() for v in q.stdout.strip().split(","))
    return dict(name=name, power_limit=power, sm_clock_max=clock)


def setup(kernel, n, d, epochs):
    import hebo_b200
    from hebo_b200.suggest import hebo_y_transform
    X, y = synth(n, d, 1234 + 5)
    yt = hebo_y_transform(y)
    np.random.seed(0)
    torch.manual_seed(0)
    gp = hebo_b200.GP(d, 0, 1, lr=0.01, num_epochs=epochs, noise_lb=8e-4, pred_likeli=False, kernel=kernel,
                      langevin=False, rng="device")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    gp.fit(X, None, yt)
    torch.cuda.synchronize()
    assert not gp._fit_failed, kernel
    return gp, (time.perf_counter() - t0) * 1e3, float(yt.min())


def score(gp, Xs, tau):
    return gp.predict_mace(Xs, tau, 2.0, 1e-4, None, None, seed=7, return_mu_var=True, device_out=True)


def measure(kernel, n, d, m, epochs, Xs):
    import ctypes as C
    from hebo_b200 import _lib
    lib = _lib.lib()
    gp, fit_ms, tau = setup(kernel, n, d, epochs)
    for _ in range(2):
        score(gp, Xs, tau)
    torch.cuda.synchronize()
    g = (C.c_uint64 * 2)()
    lib.hb_guard_stats(g, 1)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(5)]
    for a, b in ev:
        a.record()
        score(gp, Xs, tau)
        b.record()
    torch.cuda.synchronize()
    ms = statistics.mean(a.elapsed_time(b) for a, b in ev)
    lib.hb_guard_stats(g, 1)
    out = dict(fit_ms=fit_ms, score_ms=ms, cand_per_s=m / (ms * 1e-3), guard_flagged_frac=(g[1] / g[0]) if g[0] else 0.0)
    del gp
    torch.cuda.empty_cache()
    return out


def profile(kernel, n, d, Xs):
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        gp, _, tau = setup(kernel, n, d, 10)
        for _ in range(3):
            score(gp, Xs, tau)
        torch.cuda.synchronize()
    out = {}
    for name in PROFILED:
        ev = [e for e in p.key_averages() if f"hb::{name}<" in e.key]       # every <KERN, ...> instance of that kernel
        cnt = sum(e.count for e in ev)
        out[name] = dict(us_per_launch=sum(e.device_time_total for e in ev) / cnt, launches=cnt) if cnt else None
    del gp
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for bench_kernels.json")
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--dims", default="32,100")
    ap.add_argument("--m", type=int, default=131072)
    ap.add_argument("--epochs", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_kernels.py measures on a CUDA device"
    os.makedirs(args.out, exist_ok=True)
    dims = [int(v) for v in args.dims.split(",")]
    res = {d: {k: [] for k in KERNELS} for d in dims}
    for rep in range(args.reps):
        for d in dims:
            Xs = candidates(args.m, d, 1000).cuda()
            order = KERNELS[rep % len(KERNELS):] + KERNELS[:rep % len(KERNELS)]
            for k in order:
                res[d][k].append(measure(k, args.n, d, args.m, args.epochs, Xs))
    prof = {d: {k: profile(k, args.n, d, candidates(args.m, d, 1000).cuda()) for k in KERNELS} for d in dims}
    table = {}
    for d in dims:
        for k in KERNELS:
            runs = res[d][k]
            table[f"{k}_d{d}"] = dict({key: statistics.median(r[key] for r in runs) for key in runs[0]},
                                      runs=runs, profiler=prof[d][k])
    line = dict(card=card(), n=args.n, m=args.m, epochs=args.epochs, reps=args.reps, langevin=False,
                torch=torch.__version__, results=table)
    with open(os.path.join(args.out, "bench_kernels.json"), "w") as fh:
        json.dump(line, fh, indent=1)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
