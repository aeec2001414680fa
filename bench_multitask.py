"""Batched multi-output fit against the per-output loop (MultiTaskModel).

    python bench_multitask.py --out DIR [--outs 1,2,4,8] [--ns 256,1024,4096] [--reps 3]

For every (num_out, n): d = 32, Matern-3/2, 100 pSGLD epochs on bench.py's synthetic inputs (one Hartmann-6 / Ackley target
per output, shifted so that the outputs differ).  The Langevin term is off so that every output runs all 100 epochs (with
most lengthscale gradients vanishing, pSGLD's noise can random-walk a fit into an early give-up, sgld.py:64-70, which would
time fewer epochs).  Per shape, after one warm-up fit of each path, the batched fit (one hb_fit_multi_ex call) and the
loop (one single-output GP.fit per output) are timed alternately, --reps times each, with a host clock around calls that end in a
device synchronisation; the JSON reports median, min and max.  Every timed pair is checked bit for bit: the raw hypers and
losses of the batched fit equal those of the loop.  launches_per_epoch = kernel launches of a fit / 100 (hb_launch_count;
the final per-output factorisation included).  Writes DIR/bench_multitask.json with the card name and power limit read in
the same run.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import KERNEL, synth  # noqa: E402
from bench_nsga import gpu_info  # noqa: E402
from hebo_b200 import _lib  # noqa: E402
from hebo_b200.gp import MultiTaskModel  # noqa: E402

D, EPOCHS = 32, 100


def problem(n, B):
    X, y0 = synth(n, D, 1234 + n)
    _, y1 = synth(n, D, 1234 + n, fn="ackley")
    y0, y1 = torch.as_tensor(y0).reshape(-1), torch.as_tensor(y1).reshape(-1)
    cols = [(y0 if b % 2 == 0 else y1) + 0.1 * b * X[:, b % D] for b in range(B)]
    return X.float(), torch.stack(cols, 1).float()


def fit(X, Y, batched):
    B = Y.shape[1]
    np.random.seed(0)
    torch.manual_seed(0)
    mt = MultiTaskModel(D, 0, B, kernel=KERNEL, num_epochs=EPOCHS, langevin=False)
    torch.cuda.synchronize()
    lib = _lib.lib()
    lib.hb_launch_count(1)
    t0 = time.perf_counter()
    if batched:
        mt._fit_batched(X, None, Y)
    else:
        for i in range(B):
            mt.models[i].fit(X, None, Y[:, [i]])
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    launches = int(lib.hb_launch_count(1))
    return ms, launches, mt


def same(a, b):
    return all(np.asarray(x.raw).tobytes() == np.asarray(y.raw).tobytes() and x.losses.tobytes() == y.losses.tobytes()
               for x, y in zip(a.models, b.models))


def stats(v):
    return {"median_ms": round(statistics.median(v), 3), "min_ms": round(min(v), 3), "max_ms": round(max(v), 3)}


def bench_shape(n, B, reps):
    X, Y = problem(n, B)
    fit(X, Y, True)
    fit(X, Y, False)
    tb, tl = [], []
    equal = True
    for _ in range(reps):
        ms_b, lb, mb = fit(X, Y, True)
        ms_l, ll, ml = fit(X, Y, False)
        tb.append(ms_b)
        tl.append(ms_l)
        equal = equal and same(mb, ml)
    row = {"n": n, "num_out": B, "batched": stats(tb), "loop": stats(tl),
           "speedup_median": round(statistics.median(tl) / statistics.median(tb), 3),
           "launches_per_epoch": {"batched": lb / EPOCHS, "loop": ll / EPOCHS}, "bitwise_equal": equal,
           "epochs_run": [int(np.isfinite(m.losses).sum()) for m in mb.models]}
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--outs", default="1,2,4,8")
    ap.add_argument("--ns", default="256,1024,4096")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_multitask.py needs a GPU"
    info = gpu_info()
    rows = []
    for n in [int(v) for v in args.ns.split(",")]:
        for B in [int(v) for v in args.outs.split(",")]:
            rows.append(bench_shape(n, B, args.reps))
            print(json.dumps(rows[-1]), flush=True)
    res = {"metric": "100-epoch multi-output fit ms, batched vs per-output loop", "gpu": info, "d": D, "kernel": KERNEL,
           "epochs": EPOCHS, "reps": args.reps, "rows": rows}
    line = json.dumps(res)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_multitask.json"), "w") as fh:
            fh.write(line + "\n")
    print(line)
    bad = [(r["n"], r["num_out"]) for r in rows if not r["bitwise_equal"]]
    assert not bad, f"batched fit differs from the per-output loop at (n, num_out) = {bad}"


if __name__ == "__main__":
    main()
