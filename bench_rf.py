"""Random-forest surrogate on the device: fit, predict, one GA generation, and HEBO(model_name='rf') when installed.

    python bench_rf.py --out DIR [--ns 50,200,1000,4096] [--ds 8,32,256] [--ts 20,100] [--reps 3]

Fit: RF.fit for n x d x T (d numeric columns), after one warm-up fit per shape, --reps fits timed with a host clock around
calls that end in a device synchronisation.  Next to it, the reference's own arithmetic on the host: sklearn's
RandomForestRegressor(n_estimators=T) (n_jobs=None, one core, as rf.py builds it) plus the in-sample predict of the noise
estimate, when sklearn is importable and n d T <= 4096 * 32 * 100 (larger shapes take minutes per fit on one core).
Predict: candidates/s of RF.predict on device tensors at m = 10^4, 131 072 and 10^6 (n = 1000, d = 32, T = 20; CUDA events,
10 calls), and the reference's predict (forest mean + np.var over the per-tree predictions) on the host at m = 131 072.
GA: one generation (pop 100) over ga_score (LCB) split into mate / score / survive with CUDA events around each call.
HEBO: the installed reference's HEBO(model_name='rf').suggest through register(override_rf=True), if hebo imports.
Writes DIR/bench_rf.json with the card name and power limit read in the same run.  Needs a GPU.
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
from hebo_b200 import RF, _lib  # noqa: E402

SKLEARN_MAX_WORK = 4096 * 32 * 100


def problem(n, d, seed=0):
    g = torch.Generator().manual_seed(seed)
    Xc = torch.rand(n, d, generator=g)
    y = torch.sin(3 * Xc[:, :8]).sum(1, keepdim=True) + 0.05 * torch.randn(n, 1, generator=g)
    return Xc, y


def fit_ms(n, d, T):
    Xc, y = problem(n, d)
    m = RF(d, 0, 1, n_estimators=T)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    m.fit(Xc, None, y)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def sklearn_fit_ms(n, d, T):
    from sklearn.ensemble import RandomForestRegressor
    Xc, y = problem(n, d)
    X, yy = Xc.numpy(), y.numpy().reshape(-1)
    t0 = time.perf_counter()
    rf = RandomForestRegressor(n_estimators=T).fit(X, yy)
    np.mean((rf.predict(X) - yy) ** 2)
    return (time.perf_counter() - t0) * 1e3


def bench_fit(ns, ds, ts, reps):
    try:
        import sklearn  # noqa: F401
        have_sk = True
    except Exception:
        have_sk = False
    rows = []
    for n in ns:
        for d in ds:
            for T in ts:
                fit_ms(n, d, T)
                dev = [fit_ms(n, d, T) for _ in range(reps)]
                row = {"n": n, "d": d, "T": T, "device_ms_median": round(statistics.median(dev), 3)}
                if have_sk and n * d * T <= SKLEARN_MAX_WORK:
                    row["sklearn_ms"] = round(sklearn_fit_ms(n, d, T), 1)
                    row["speedup"] = round(row["sklearn_ms"] / row["device_ms_median"], 1)
                rows.append(row)
                print(json.dumps(row), flush=True)
    return {"rows": rows, "host_cores": os.cpu_count(), "sklearn_cores_used": 1 if have_sk else None}


def bench_predict():
    n, d, T = 1000, 32, 20
    Xc, y = problem(n, d)
    torch.manual_seed(0)
    m = RF(d, 0, 1, n_estimators=T)
    m.fit(Xc, None, y)
    res = {"n": n, "d": d, "T": T}
    for M in (10_000, 131_072, 1_000_000):
        xs = torch.rand(M, d, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
        m.predict(xs)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            m.predict(xs)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        res[f"m={M}"] = {"ms": round(ms, 4), "candidates_per_s": round(M / ms * 1e3)}
        print(json.dumps({f"predict m={M}": res[f"m={M}"]}), flush=True)
    try:
        from sklearn.ensemble import RandomForestRegressor
        rf = RandomForestRegressor(n_estimators=T).fit(Xc.numpy(), y.numpy().reshape(-1))
        X = np.random.default_rng(1).random((131_072, d)).astype(np.float32)
        t0 = time.perf_counter()
        rf.predict(X)
        np.var(np.stack([e.predict(X) for e in rf.estimators_], 1), axis=1)
        res["sklearn_m=131072_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    except ImportError:
        pass
    return res


def bench_ga_generation():
    from hebo_b200.acq import LCB, ga_score
    from hebo_b200.evolution import DeviceNSGA2
    from hebo_b200.space import DesignSpace
    sp = DesignSpace().parse([{"name": f"x{i}", "type": "num", "lb": 0, "ub": 1} for i in range(8)])
    Xc, y = problem(1000, 8)
    torch.manual_seed(0)
    m = RF(8, 0, 1, n_estimators=20)
    m.fit(Xc, None, y)
    score = ga_score(LCB(m, kappa=2.0))
    evo = DeviceNSGA2(sp.var_kinds, sp.opt_lb.numpy(), sp.opt_ub.numpy(), 8, score, pop=100, iters=100, seed=0, device=m.device)
    evo.optimize()                        # warm-up of every launch below
    lib, P, D, d, st = _lib.lib(), evo.pop, evo.D, evo.d, _lib.stream_ptr
    pc = lambda x: _lib.ptr(x) if x.numel() else None
    X, Xc_, Xe = evo._bufs()
    Xn, Xcn, Xen = evo._bufs()
    C, Cc, Ce = evo._bufs()
    ws_bytes = int(lib.hb_nsga2_workspace_bytes_k(P, D, 3))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=m.device)
    _lib.check(lib.hb_nsga2_init(_lib.ptr(X), P, D, d, _lib.ptr(evo.kind), _lib.ptr(evo.lb), _lib.ptr(evo.ub), _lib.ptr(evo.fixed),
                                 None, 0, evo.seed, pc(Xc_), pc(Xe), st()), "hb_nsga2_init")
    F = score(Xc_, Xe, 0)
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
        X, Xn, Xc_, Xcn, Xe, Xen, F, Fn = Xn, X, Xcn, Xc_, Xen, Xe, Fn, F
    torch.cuda.synchronize()
    out = {k: round(sum(a.elapsed_time(b) for a, b in v) / G, 4) for k, v in ev.items()}
    return {"n": 1000, "T": 20, "pop": P, "generations": G, **{f"{k}_ms_per_gen": v for k, v in out.items()}}


def bench_hebo(reps):
    try:
        from hebo.design_space.design_space import DesignSpace
        from hebo.optimizers.hebo import HEBO
    except Exception:
        return "hebo not installed"
    from hebo_b200 import register
    register(override_rf=True)
    sp = DesignSpace().parse([{"name": f"x{i}", "type": "num", "lb": 0, "ub": 1} for i in range(8)])
    times = []
    for r in range(reps + 1):
        opt = HEBO(sp, model_name="rf", rand_sample=4)
        X = opt.quasi_sample(50)
        opt.observe(X, np.sin(3 * X.values).sum(1, keepdims=True))
        t0 = time.perf_counter()
        opt.suggest(1)
        if r:
            times.append((time.perf_counter() - t0) * 1e3)
    return {"suggest_ms_median": round(statistics.median(times), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ns", default="50,200,1000,4096")
    ap.add_argument("--ds", default="8,32,256")
    ap.add_argument("--ts", default="20,100")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_rf.py needs a GPU"
    ints = lambda s: [int(v) for v in s.split(",")]
    res = {"metric": "random-forest fit / predict / GA generation", "gpu": gpu_info(),
           "fit": bench_fit(ints(args.ns), ints(args.ds), ints(args.ts), args.reps), "predict": bench_predict(),
           "ga_generation_ms": bench_ga_generation(), "hebo_rf": bench_hebo(args.reps)}
    line = json.dumps(res)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_rf.json"), "w") as fh:
            fh.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
