"""bench_highdim.py -- the fit and the scoring step at high feature counts (d up to HB_MAX_FEATURES = 4096) on one GPU.

    python bench_highdim.py --out DIR [--dims 32,100,...] [--n 4096] [--m 131072] [--steps 3]
    python bench_highdim.py --dump-outputs DIR      # results only (d = 32, 100 and a mixed model with d + De = 200)

Writes DIR/bench_highdim.json (and prints it as one JSON line) with the card name and power limit read from nvidia-smi in
the same run.  Per d, at n = 4096, Matern-3/2, bench.py's synthetic problem (Hartmann-6 embedded in d dims):
  fit_ms         the 100-epoch fit (host clock around a synchronised call, after a 2-epoch warm-up fit), without the
                 Langevin term: with most lengthscale gradients vanishing at high d, pSGLD's noise random-walks those
                 parameters until the fit gives up early (sgld.py:64-70), which would time fewer epochs
  cands_per_s    posterior + MACE + device front over m scrambled-Sobol candidates (CUDA events, mean over --steps)
  kernels_ms     kstar_kernel / vnorm_h16_kernel per scoring step, mll_grad_kernel / mll_finish_kernel per MLL
                 forward + backward, from a separate torch.profiler run
  kstar_tflops   n (3 d + 8) flop per candidate (the direct-difference distance, kernel and mean) over the kstar_kernel
                 time, against the 67 TFLOP/s FP32 figure of NVIDIA's H100 SXM data sheet (700 W card)
and suggest() ms at (n, d) = (1024, 1024), q = 8, 100 epochs without the Langevin term.  --dump-outputs writes what the
fits and the scoring computed as .npy, so that two builds can be compared bit for bit.  Nothing is written outside DIR; it needs a GPU and fails without one.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import KERNEL, Q, candidates, synth  # noqa: E402
from bench_nsga import gpu_info  # noqa: E402

DIMS = [32, 100, 128, 256, 512, 1024, 2048, 4096]
FP32_PEAK = 67.0   # TFLOP/s, H100 SXM data sheet
CAP = 4096


def fitted_gp(n, d, seed, epochs=100, num_uniqs=None, langevin=True):
    import hebo_b200
    from hebo_b200.suggest import hebo_y_transform
    X, y = synth(n, d, seed)
    yt = hebo_y_transform(y)
    Xe = None
    conf = dict(lr=0.01, num_epochs=epochs, noise_lb=8e-4, pred_likeli=False, kernel=KERNEL, rng="device", langevin=langevin)
    if num_uniqs:
        g = torch.Generator().manual_seed(seed + 1)
        Xe = torch.stack([torch.randint(0, u, (n,), generator=g) for u in num_uniqs], 1)
        yt = yt + 0.3 * torch.cos(Xe.float() * 1.7).sum(1, keepdim=True)
        conf["num_uniqs"] = list(num_uniqs)
    np.random.seed(0)
    torch.manual_seed(0)
    gp = hebo_b200.GP(d, len(num_uniqs or []), 1, **conf)
    gp.fit(X, Xe, yt)
    return gp, X, yt


def score_step(gp, Xs, tau, kappa, Xe=None):
    from hebo_b200 import dist as hdist
    if Xe is None:
        return hdist.sharded_score_front(gp, Xs, 0, tau, kappa, 1e-4, seed=7, capacity=CAP)
    return gp.predict_mace(Xs, tau, kappa, 1e-4, None, None, seed=7, return_mu_var=True, Xe=Xe)


def dump_outputs(dirname, n, m):
    """Fit and score d = 32, d = 100 and a mixed model (100 numeric columns, two categoricals of 100 choices: De = 100)."""
    os.makedirs(dirname, exist_ok=True)
    for name, d, nu in [("d32", 32, None), ("d100", 100, None), ("mixed_d100_De100", 100, [100, 100])]:
        gp, X, yt = fitted_gp(n, d, 4321 + d, num_uniqs=nu)
        Xs = candidates(m, d, 99).cuda()
        Xe = None
        if nu:
            g = torch.Generator().manual_seed(5)
            Xe = torch.stack([torch.randint(0, u, (m,), generator=g) for u in nu], 1).cuda()
        F, mu, var = gp.predict_mace(Xs, float(yt.min()), 2.0, 1e-4, None, None, seed=7, return_mu_var=True, Xe=Xe)
        out = dict(raw=gp.raw, losses=torch.as_tensor(np.asarray(gp.losses)), F=F, mu=mu, var=var)
        for k, v in out.items():
            np.save(os.path.join(dirname, f"{name}_{k}.npy"), v.detach().cpu().numpy())
        print(f"dumped {name}", flush=True)


def kernel_times(prof, names):
    out = {k: 0.0 for k in names}
    events = prof.key_averages()
    for e in events:
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0.0)
        for k in names:
            if k in e.key:
                out[k] += t / 1e3     # us -> ms
    if not all(out.values()):
        print("profiled kernels:", sorted({e.key[:80] for e in events}), file=sys.stderr)
    return out


def bench_dim(n, d, m, steps):
    from hebo_b200.suggest import kappa_schedule
    fitted_gp(n, d, 1234 + d, epochs=2)                  # warm-up: workspaces, lazily built per-device state
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    gp, X, yt = fitted_gp(n, d, 1234 + d, langevin=False)
    torch.cuda.synchronize()
    fit_ms = (time.perf_counter() - t0) * 1e3
    fit_epochs = int(np.isfinite(np.asarray(gp.losses)).sum())
    tau, kappa = float(yt.min()), kappa_schedule(n, Q, d)
    Xs = candidates(m, d, 1000).cuda()
    score_step(gp, Xs, tau, kappa)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        score_step(gp, Xs, tau, kappa)
    b.record()
    torch.cuda.synchronize()
    step_ms = a.elapsed_time(b) / steps
    # separate profiled run: one scoring step and one MLL forward + backward
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        score_step(gp, Xs, tau, kappa)
        torch.cuda.synchronize()
    ks = kernel_times(prof, ["kstar_kernel", "vnorm_h16_kernel"])
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gp.evaluate_loss(return_grad=True)
        torch.cuda.synchronize()
    ks.update(kernel_times(prof, ["mll_grad_kernel", "mll_finish_kernel", "gram_kernel"]))
    kstar_flop = float(n) * (3 * d + 8) * m
    tflops = kstar_flop / (ks["kstar_kernel"] / 1e3) / 1e12 if ks["kstar_kernel"] > 0 else None
    r = {"d": d, "n": n, "m": m, "fit_ms": fit_ms, "fit_epochs_completed": fit_epochs, "score_ms_per_step": step_ms,
         "cands_per_s": m / (step_ms / 1e3),
         "kernels_ms": {k: round(v, 4) for k, v in ks.items()}, "kstar_tflops": tflops,
         "kstar_frac_of_fp32_peak": (tflops / FP32_PEAK) if tflops else None,
         "kstar_share_of_step": ks["kstar_kernel"] / step_ms if step_ms > 0 else None}
    del gp, Xs
    torch.cuda.empty_cache()
    return r


def bench_suggest(n, d):
    from hebo_b200.suggest import HEBO
    # rand_sample: HEBO's default (1 + d random suggestions before the first fit) exceeds n here
    opt = HEBO(-torch.ones(d), torch.ones(d), device="cuda", scramble_seed=1, rand_sample=64,
               model_config={"lr": 0.01, "num_epochs": 100, "noise_lb": 8e-4, "pred_likeli": False, "langevin": False})
    X, y = synth(n, d, 77)
    opt.observe(X, y)
    ts = []
    for _ in range(3):
        np.random.seed(0)
        opt.suggest(Q)
        ts.append(dict(opt.last_timing))
    best = min(ts[1:], key=lambda r: r["total_ms"])       # the first call pays workspace allocation
    return {"n": n, "d": d, "q": Q, "total_ms": best["total_ms"], "fit_ms": best["fit_ms"], "score_ms": best["score_ms"],
            "fit_epochs_completed": int(np.isfinite(np.asarray(opt.model.losses)).sum()),
            "all_total_ms": [round(r["total_ms"], 2) for r in ts]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--dims", default=",".join(map(str, DIMS)))
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--m", type=int, default=131072)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_highdim.py needs a GPU"
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, args.n, args.m)
        return
    info = gpu_info()
    rows = []
    for d in [int(v) for v in args.dims.split(",")]:
        rows.append(bench_dim(args.n, d, args.m, args.steps))
        print(json.dumps(rows[-1]), flush=True)
    res = {"metric": "fit ms / candidates per s / K* FLOP/s vs feature count", "gpu": info, "kernel": KERNEL,
           "fp32_peak_tflops": FP32_PEAK, "peak_source": "H100 SXM data sheet (FP32, 700 W card)", "dims": rows,
           "suggest": bench_suggest(1024, 1024)}
    line = json.dumps(res)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_highdim.json"), "w") as fh:
            fh.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
