"""Deep-ensemble surrogate on the device: fit, predict, HEBO.suggest and one BO GA generation.

    python bench_deep_ensemble.py --out DIR [--ns 50,200,1000] [--ds 8,32] [--reps 3] [--cpu-epochs 5]

Fit: 5 members, 500 epochs, batch 32, for n x d x {default, rand_prior, num_layers=2, the envelope corner (3 x 256 hidden
units, rand_prior)}; d numeric columns plus one categorical column of 5 categories.  After one warm-up fit per shape, --reps
fits are timed with a host clock around calls that end in a device synchronisation; us_per_step = fit time / (500 epochs x
steps per epoch), one step advancing every member.  The CPU arm is the oracle's restatement of fit_one (oracle/
ensemble_oracle.py, torch on the host, fp32 here) for --cpu-epochs epochs of ONE member, scaled to 5 x 500 epochs: the
same arithmetic the reference runs per member, without its DataLoader.
Predict: candidates/s of DeepEnsemble.predict on device tensors at m = 10^4 and 131 072 (CUDA events, 20 calls).
HEBO.suggest (d = 8, n = 50): fit and acquisition ms for the Sobol batch and the NSGA-II optimiser.  BO: one GA
generation (pop 100) over ga_score (LCB) split into mate / score / survive with CUDA events around each call, the calls
DeviceNSGA2.optimize makes for a one-column score, over 100 generations.
Writes DIR/bench_deep_ensemble.json with the card name and power limit read in the same run.  Needs a GPU.
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
from hebo_b200 import DeepEnsemble, _lib  # noqa: E402
from oracle import ensemble_oracle as EO  # noqa: E402

CONFIGS = {"default": {}, "rand_prior": {"rand_prior": True}, "num_layers=2": {"num_layers": 2},
           "corner": {"num_layers": 3, "num_hiddens": 256, "rand_prior": True}}


def problem(n, d, seed=0):
    g = torch.Generator().manual_seed(seed)
    Xc = torch.rand(n, d, generator=g)
    Xe = torch.randint(0, 5, (n, 1), generator=g)
    y = (torch.sin(3 * Xc).sum(1, keepdim=True) + 0.3 * Xe.float() + 0.05 * torch.randn(n, 1, generator=g))
    return Xc, Xe, y


def fit_once(n, d, conf):
    Xc, Xe, y = problem(n, d)
    torch.manual_seed(0)
    m = DeepEnsemble(d, 1, 1, num_uniqs=[5], **conf)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    m.fit(Xc, Xe, y)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def cpu_fit_ms(n, d, conf, epochs):
    Xc, Xe, y = problem(n, d)
    m = DeepEnsemble(d, 1, 1, num_uniqs=[5], **conf)
    net = EO.OracleNet(d, [5], "embedding", m.num_layers, m.num_hiddens, 1, True, m.rand_prior).float()
    EO_F = torch.float32
    xs = ((Xc - Xc.min(0).values) / (Xc.max(0).values - Xc.min(0).values) * 2 - 1).to(EO_F)
    ys = ((y - y.mean()) / y.std()).to(EO_F)
    opt = torch.optim.Adam(net.parameters(), lr=m.lr)
    nb, B = (n // 32, 32) if n > 32 else (1, n)
    t0 = time.perf_counter()
    for _ in range(epochs):
        order = torch.randperm(n)
        for b in range(nb):
            rows = order[b * B:(b + 1) * B]
            mu, s2 = net(xs[rows], Xe[rows])
            loss = torch.mean(0.5 * (ys[rows] - mu) ** 2 / s2 + 0.5 * torch.log(s2))
            loss = loss + sum(m.l1 * p.abs().sum() / n for p in net.parameters())
            opt.zero_grad()
            loss.backward()
            opt.step()
    return (time.perf_counter() - t0) * 1e3 / epochs * 500 * 5


def bench_fit(ns, ds, reps, cpu_epochs):
    rows = []
    for name, conf in CONFIGS.items():
        for d in ds:
            for n in ns:
                fit_once(n, d, conf)
                t = [fit_once(n, d, conf) for _ in range(reps)]
                steps = 500 * (n // 32 if n > 32 else 1)
                med = statistics.median(t)
                row = {"config": name, "n": n, "d": d, "fit_ms_median": round(med, 3), "fit_ms_min": round(min(t), 3),
                       "fit_ms_max": round(max(t), 3), "steps": steps, "us_per_step": round(med * 1e3 / steps, 3)}
                if cpu_epochs > 0:
                    row["cpu_torch_fit_ms_est"] = round(cpu_fit_ms(n, d, conf, cpu_epochs), 1)
                rows.append(row)
                print(json.dumps(row), flush=True)
    return rows


def bench_predict():
    Xc, Xe, y = problem(200, 8)
    torch.manual_seed(0)
    m = DeepEnsemble(8, 1, 1, num_uniqs=[5])
    m.fit(Xc, Xe, y)
    out = []
    for mm in (10 ** 4, 131072):
        xs = torch.rand(mm, 8, device="cuda")
        xe = torch.randint(0, 5, (mm, 1), device="cuda")
        for _ in range(3):
            m.predict(xs, xe)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(20):
            m.predict(xs, xe)
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / 20
        out.append({"m": mm, "ms": round(ms, 4), "candidates_per_s": round(mm / ms * 1e3)})
        print(json.dumps(out[-1]), flush=True)
    return out


def bench_suggest(reps):
    from hebo_b200.suggest import HEBO
    res = {}
    for acq_opt in ("sobol", "nsga2"):
        fit, acq = [], []
        for r in range(reps + 1):
            torch.manual_seed(r)
            np.random.seed(r)
            opt = HEBO(torch.zeros(8), torch.ones(8), model_name="deep_ensemble", scramble_seed=r, acq_optimizer=acq_opt)
            X = torch.rand(50, 8, generator=torch.Generator().manual_seed(r))
            opt.observe(X, (torch.sin(3 * X).sum(1)).numpy().reshape(-1, 1))
            opt.suggest(1)
            if r:
                fit.append(opt.last_timing["fit_ms"])
                acq.append(opt.last_timing["score_ms"])
        res[acq_opt] = {"fit_ms_median": round(statistics.median(fit), 3), "acq_ms_median": round(statistics.median(acq), 3)}
        print(json.dumps({acq_opt: res[acq_opt]}), flush=True)
    return res


def bench_ga_generation():
    from hebo_b200.acq import LCB, ga_score
    from hebo_b200.evolution import DeviceNSGA2
    from hebo_b200.space import DesignSpace
    sp = DesignSpace().parse([{"name": f"x{i}", "type": "num", "lb": 0, "ub": 1} for i in range(8)])
    Xc, _, y = problem(50, 8)
    torch.manual_seed(0)
    m = DeepEnsemble(8, 0, 1)
    m.fit(Xc, None, y)
    score = ga_score(LCB(m, kappa=2.0))
    evo = DeviceNSGA2(sp.var_kinds, sp.opt_lb.numpy(), sp.opt_ub.numpy(), 8, score, pop=100, iters=100, seed=0, device=m.device)
    evo.optimize()                        # warm-up of every launch below
    # one generation as DeviceNSGA2.optimize runs it for a one-column score: mate, score the children, survive
    lib, P, D, d, st = _lib.lib(), evo.pop, evo.D, evo.d, _lib.stream_ptr
    pc = lambda x: _lib.ptr(x) if x.numel() else None
    X, Xc, Xe = evo._bufs()
    Xn, Xcn, Xen = evo._bufs()
    C, Cc, Ce = evo._bufs()
    ws_bytes = int(lib.hb_nsga2_workspace_bytes_k(P, D, 3))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=m.device)
    _lib.check(lib.hb_nsga2_init(_lib.ptr(X), P, D, d, _lib.ptr(evo.kind), _lib.ptr(evo.lb), _lib.ptr(evo.ub), _lib.ptr(evo.fixed),
                                 None, 0, evo.seed, pc(Xc), pc(Xe), st()), "hb_nsga2_init")
    F = score(Xc, Xe, 0)
    Fn = torch.empty_like(F)
    ev = {k: [] for k in ("mate", "score", "survive")}

    def rec(name, fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        ev[name].append((e0, e1))
        return out
    G = 100
    for gen in range(1, G + 1):
        rec("mate", lambda: _lib.check(lib.hb_nsga2_mate(_lib.ptr(X), P, D, d, _lib.ptr(evo.kind), _lib.ptr(evo.lb), _lib.ptr(evo.ub),
                                                         _lib.ptr(evo.fixed), evo.seed, gen, _lib.ptr(C), pc(Cc), pc(Ce), st()), "mate"))
        FC = rec("score", lambda: score(Cc, Ce, gen))
        rec("survive", lambda: _lib.check(lib.hb_ga_survive(_lib.ptr(X), _lib.ptr(F), _lib.ptr(C), _lib.ptr(FC), P, D, d, _lib.ptr(Xn),
                                                            _lib.ptr(Fn), pc(Xcn), pc(Xen), _lib.ptr(ws), ws_bytes, st()), "survive"))
        X, Xn, Xc, Xcn, Xe, Xen, F, Fn = Xn, X, Xcn, Xc, Xen, Xe, Fn, F
    torch.cuda.synchronize()
    out = {k: round(sum(a.elapsed_time(b) for a, b in v) / G, 4) for k, v in ev.items()}
    return {"generations": G, **{f"{k}_ms_per_gen": v for k, v in out.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ns", default="50,200,1000")
    ap.add_argument("--ds", default="8,32")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-epochs", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_deep_ensemble.py needs a GPU"
    res = {"metric": "deep-ensemble fit / predict / suggest", "gpu": gpu_info(), "members": 5, "epochs": 500,
           "fit": bench_fit([int(v) for v in args.ns.split(",")], [int(v) for v in args.ds.split(",")], args.reps,
                            args.cpu_epochs),
           "predict": bench_predict(), "suggest": bench_suggest(args.reps), "ga_generation_ms": bench_ga_generation()}
    line = json.dumps(res)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_deep_ensemble.json"), "w") as fh:
            fh.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
