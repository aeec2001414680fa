"""bench_bo.py -- the single-objective GA and BO.suggest() on one GPU.

    python bench_bo.py --out DIR [--reps-floor 5]

Writes DIR/bench_bo.json with the card name and power limit read from nvidia-smi in the same run, and:
  survival    hb_ga_survive against hb_nsga2_survive_ex at the same pop (D = 16, random inputs, no duplicates), at pop
              100, 1024, 4096 and 16 384, timed alternately (5 rounds of CUDA-event means, the median of each);
  generation  one GA generation at pop 100 split into mate (hb_nsga2_mate), score (GP predict + hb_acq1_epilogue, LCB)
              and survive (hb_ga_survive), CUDA events around each step, mean over 100 generations, for n in {200, 1000}
              observations x d in {8, 32};
  suggest     BO.suggest() (pop 100 x 100 generations) for n in {50, 200, 1000} x d in {2, 8, 32}: last_timing fit_ms /
              acq_ms / total_ms, median of 3 calls after one warm-up call.
Nothing is written outside DIR; it needs a GPU and fails without one.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import pandas as pd
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_nsga import event_ms, gpu_info  # noqa: E402


def objective(x: np.ndarray) -> np.ndarray:
    return ((x - 0.3) ** 2).sum(1, keepdims=True) + 0.1 * np.sin(5 * x).sum(1, keepdims=True)


def bench_survival(reps_floor):
    from hebo_b200 import _lib
    lib, p = _lib.lib(), _lib.ptr
    out = []
    for P in (100, 1024, 4096, 16384):
        D = 16
        g = torch.Generator(device="cuda").manual_seed(P)
        X, C = torch.rand(P, D, device="cuda", generator=g), torch.rand(P, D, device="cuda", generator=g)
        F, FC = torch.randn(P, 3, device="cuda", generator=g), torch.randn(P, 3, device="cuda", generator=g)
        f, fc = F[:, 0].contiguous(), FC[:, 0].contiguous()
        Xn, Fn, fn, Xcn = torch.empty_like(X), torch.empty_like(F), torch.empty_like(f), torch.empty_like(X)
        ws_bytes = int(lib.hb_nsga2_workspace_bytes(P, D))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")

        def ex():
            _lib.check(lib.hb_nsga2_survive_ex(p(X), p(F), p(C), p(FC), P, D, D, p(Xn), p(Fn), p(Xcn), None, p(ws), ws_bytes,
                                               _lib.stream_ptr()), "hb_nsga2_survive_ex")

        def ga():
            _lib.check(lib.hb_ga_survive(p(X), p(f), p(C), p(fc), P, D, D, p(Xn), p(fn), p(Xcn), None, p(ws), ws_bytes,
                                         _lib.stream_ptr()), "hb_ga_survive")
        reps = max(reps_floor, 50 if P < 16384 else 10)
        t_ex, t_ga = [], []
        for _ in range(5):
            t_ga.append(event_ms(ga, reps))
            t_ex.append(event_ms(ex, reps))
        r = dict(pop=P, D=D, ga_ms=float(np.median(t_ga)), nsga_ex_ms=float(np.median(t_ex)), ga_all=t_ga, nsga_ex_all=t_ex)
        out.append(r)
        print(f"survival pop={P}: ga {r['ga_ms']:.4f} ms, nsga2 ex {r['nsga_ex_ms']:.4f} ms")
    return out


def fitted(n, d, seed):
    from hebo_b200 import GP
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (n, d))
    y = objective(X)
    model = GP(d, 0, 1, warp=False, device="cuda")
    model.fit(torch.FloatTensor(X), None, torch.FloatTensor(y))
    return model


def bench_generation():
    from hebo_b200 import LCB, _lib
    from hebo_b200.acq import ga_score
    lib, p = _lib.lib(), _lib.ptr
    out = []
    P, gens = 100, 100
    for n in (200, 1000):
        for d in (8, 32):
            score = ga_score(LCB(fitted(n, d, n + d), kappa=2.0))
            kind = torch.zeros(d, dtype=torch.int32, device="cuda")
            lb, ub = -torch.ones(d, device="cuda"), torch.ones(d, device="cuda")
            fixed = torch.full((d,), float("nan"), device="cuda")
            X, Xc = torch.empty(P, d, device="cuda"), torch.empty(P, d, device="cuda")
            Xn, Xcn, C, Cc = (torch.empty(P, d, device="cuda") for _ in range(4))
            fn = torch.empty(P, device="cuda")
            ws_bytes = int(lib.hb_nsga2_workspace_bytes(P, d))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
            st = _lib.stream_ptr
            _lib.check(lib.hb_nsga2_init(p(X), P, d, d, p(kind), p(lb), p(ub), p(fixed), None, 0, 7, p(Xc), None, st()), "init")
            f = score(Xc, None, 0)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            t = np.zeros(3)
            for gen in range(1, gens + 1):
                ev[0].record()
                _lib.check(lib.hb_nsga2_mate(p(X), P, d, d, p(kind), p(lb), p(ub), p(fixed), 7, gen, p(C), p(Cc), None, st()), "mate")
                ev[1].record()
                fc = score(Cc, torch.empty(P, 0, dtype=torch.int32, device="cuda"), gen)
                ev[2].record()
                _lib.check(lib.hb_ga_survive(p(X), p(f), p(C), p(fc), P, d, d, p(Xn), p(fn), p(Xcn), None, p(ws), ws_bytes, st()),
                           "ga_survive")
                ev[3].record()
                torch.cuda.synchronize()
                t += [ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[2].elapsed_time(ev[3])]
                X, Xn, Xc, Xcn = Xn, X, Xcn, Xc
                f, fn = fn, f
            t /= gens
            r = dict(pop=P, n=n, d=d, mate_ms=float(t[0]), score_ms=float(t[1]), survive_ms=float(t[2]), gens=gens)
            out.append(r)
            print(f"generation n={n} d={d}: mate {t[0]:.4f} ms, score {t[1]:.4f} ms, survive {t[2]:.4f} ms")
    return out


def bench_suggest():
    from hebo_b200 import BO
    out = []
    for n in (50, 200, 1000):
        for d in (2, 8, 32):
            np.random.seed(0)
            torch.manual_seed(0)
            space = [{"name": f"x{i}", "type": "num", "lb": -1, "ub": 1} for i in range(d)]
            opt = BO(space, device="cuda")
            X = pd.DataFrame(np.random.uniform(-1, 1, (n, d)), columns=[f"x{i}" for i in range(d)])
            opt.observe(X, objective(X.values))
            opt.suggest()
            runs = []
            for _ in range(3):
                opt.suggest()
                runs.append(dict(opt.last_timing))
            med = {k: float(np.median([r[k] for r in runs])) for k in ("fit_ms", "acq_ms", "total_ms")}
            out.append(dict(n=n, d=d, **med, runs=runs))
            print(f"suggest n={n} d={d}: fit {med['fit_ms']:.1f} ms, acq {med['acq_ms']:.1f} ms, total {med['total_ms']:.1f} ms")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps-floor", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bo.py needs a CUDA device")
    import __graft_entry__  # noqa: F401  (puts the repository on sys.path)
    res = dict(gpu=gpu_info(), survival=bench_survival(a.reps_floor), generation=bench_generation(), suggest=bench_suggest())
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_bo.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(dict(gpu=res["gpu"]), indent=None))


if __name__ == "__main__":
    main()
