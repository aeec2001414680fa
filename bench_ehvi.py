"""GeneralBO's Monte-Carlo EHVI selection (ref_point) on the device (hb_ehvi) against the host loop over hypervolume.

    python bench_ehvi.py --out DIR [--ks 2,3,4,5] [--ns 10,30,100] [--m 100] [--n-mc 10] [--reps 3] [--host-budget 20]

Round: one selection round (base_hv and the m EHVI values) for a K-objective front of n mutually non-dominated rows
(points of a simplex) and n_mc x m draws scattered around it, as GeneralBO._select feeds it: the draws already on the
device, the front on the host.  Device: expected_hvi, host clock around a call that ends with the result on the host, after
one warm-up call, median of --reps.  Host: the _select loop over general.hypervolume, run between the device repetitions.
The host time of 2 columns is measured first; a round whose extrapolated time exceeds --host-budget seconds is not run
and reported as "not run" with that estimate.  Every compared column must give byte-identical EHVI and the same argmax.
Suggest: GeneralBO(K = 2 and 3, ref_point, 30 observations of a DTLZ2-like problem).suggest(q) for q in {1, 8}: the
fit / acq / select split of suggest() on the device path, then, on the same GA front and the same draws, the selection
stage on the device against the host loop (same rows chosen under the same np.random seed).
Writes DIR/bench_ehvi.json with the card name and power limit read in the same run.  Needs a GPU.
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

from bench_nsga import gpu_info  # noqa: E402
from hebo_b200.general import GeneralBO, expected_hvi, hypervolume  # noqa: E402
from hebo_b200.space import DesignSpace  # noqa: E402


def host_columns(front, samp, ref, cols):
    base = hypervolume(front, ref)
    n_mc = samp.shape[0]
    out = []
    for j in cols:
        s = samp[:, j]
        out.append(sum(hypervolume(np.vstack([front, s[[k]]]), ref) - base for k in range(n_mc)) / n_mc)
    return np.array(out, dtype=np.float64)


def simplex(rng, rows, K, shift):
    x = rng.random((rows, K))
    return x / x.sum(1, keepdims=True) * 2 - shift


def bench_round(K, n, m, n_mc, reps, budget):
    rng = np.random.default_rng(1000 * K + n)
    front, ref = simplex(rng, n, K, 0.5), np.ones(K)
    samp = (simplex(rng, n_mc * m, K, 0.55).reshape(n_mc, m, K) + 0.02 * rng.normal(size=(n_mc, m, K))).astype(np.float32)
    samp_dev = torch.from_numpy(samp).cuda()

    def dev():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _, e = expected_hvi(front, samp_dev, ref)
        return (time.perf_counter() - t0) * 1e3, e

    dev()
    times = []
    half = reps // 2
    for _ in range(half):
        times.append(dev()[0])
    t0 = time.perf_counter()
    probe = host_columns(front, samp, ref, [0, 1])
    est_s = (time.perf_counter() - t0) * m / 2
    host_ms, host = None, None
    if est_s <= budget:
        t0 = time.perf_counter()
        host = host_columns(front, samp, ref, range(m))
        host_ms = (time.perf_counter() - t0) * 1e3
    for _ in range(reps - half):
        t, ehvi = dev()
        times.append(t)
    cols = list(range(m)) if host is not None else [0, 1]
    ref_vals = host if host is not None else probe
    same = ehvi[cols].tobytes() == ref_vals.tobytes()
    same_pick = host is None or int(np.argmax(ehvi)) == int(np.argmax(host))
    row = {"K": K, "front_rows": n, "m": m, "n_mc": n_mc, "device_ms": round(statistics.median(times), 3),
           "host_ms": round(host_ms, 1) if host_ms is not None else "not run",
           "host_estimate_s": round(est_s, 1), "compared_columns": len(cols), "identical": bool(same and same_pick)}
    if host_ms is not None:
        row["speedup"] = round(host_ms / row["device_ms"], 1)
    print(json.dumps(row), flush=True)
    return row


class _FixedDraws:
    def __init__(self, draws):
        self.draws = draws

    def sample_y(self, Xc, Xe, n):
        return self.draws


def bench_suggest(K, q):
    space = DesignSpace().parse([{"name": f"x{i}", "type": "num", "lb": 0, "ub": 1} for i in range(4)])

    def f(X):
        x = X[[f"x{i}" for i in range(4)]].values
        g = ((x[:, K - 1:] - 0.5) ** 2).sum(1)
        th = x[:, :K - 1] * np.pi / 2
        cols = []
        for i in range(K):
            v = (1 + g) * np.prod(np.cos(th[:, :K - 1 - i]), axis=1)
            if i > 0:
                v = v * np.sin(th[:, K - 1 - i])
            cols.append(v)
        return np.stack(cols, 1)

    np.random.seed(K)
    torch.manual_seed(K)
    opt = GeneralBO(space, K, 0, rand_sample=1, ref_point=np.full(K, 2.5))
    X = space.sample(30)
    opt.observe(X, f(X))
    opt.suggest(q)                                                  # warm-up
    np.random.seed(q)
    opt.suggest(q)
    timing = {k: round(v, 1) for k, v in opt.last_timing.items()}
    model = opt._fit()
    front = opt._optimise(model, *opt._kappas())
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        draws = torch.as_tensor(model.sample_y(*space.transform(front), 10))
    torch.cuda.synchronize()
    draw_ms = (time.perf_counter() - t0) * 1e3
    sel, picks = {}, {}
    for device in ("cuda", "cpu"):
        opt.device = device
        np.random.seed(q)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        picks[device] = list(opt._select(_FixedDraws(draws), front, q).index)
        sel[device] = round((time.perf_counter() - t0) * 1e3, 1)
    opt.device = "cuda"
    row = {"K": K, "q": q, "front_rows": int(front.shape[0]), "observed_front_rows": int(opt.get_pf(opt.y).shape[0]),
           "suggest_ms": timing, "draws_ms": round(draw_ms, 1), "select_device_ms": sel["cuda"], "select_host_ms": sel["cpu"],
           "identical": picks["cuda"] == picks["cpu"]}
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="2,3,4,5")
    ap.add_argument("--ns", default="10,30,100")
    ap.add_argument("--m", type=int, default=100)
    ap.add_argument("--n-mc", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-budget", type=float, default=20.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ehvi.py needs a GPU"
    ints = lambda s: [int(v) for v in s.split(",")]
    rounds = [bench_round(K, n, args.m, args.n_mc, args.reps, args.host_budget) for K in ints(args.ks) for n in ints(args.ns)]
    suggest = [bench_suggest(K, q) for K in (2, 3) for q in (1, 8)]
    res = {"metric": "EHVI selection round and GeneralBO.suggest(ref_point)", "gpu": gpu_info(), "rounds": rounds,
           "suggest": suggest, "all_identical": all(r["identical"] for r in rounds + suggest)}
    line = json.dumps(res)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_ehvi.json"), "w") as fh:
            fh.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
