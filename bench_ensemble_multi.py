"""Deep ensembles behind the multi-output optimisers: the batched MultiTaskModel fit, one GA generation of GeneralBO and
NoisyOpt, and their suggest() timings.

    python bench_ensemble_multi.py --out DIR [--ks 1,2,4,8] [--ns 50,200,1000] [--reps 2]

Fit: MultiTaskModel(base_model_name='deep_ensemble') of K default ensembles (5 members, 500 epochs, batch 32, 1 x 128
hidden units) on n rows of d = 8 numeric columns, one hb_de_fit_batch launch of 5 K CTAs, against the per-output loop
(K DeepEnsemble.fit calls, each one hb_de_fit launch of 5 CTAs).  After one warm-up of each, --reps rounds time the two
alternately with a host clock around calls that end in a device synchronisation, and every round checks the two give
the same parameters bit for bit.  Output k has its own finite rows (every (7 + k)-th target is NaN).
GA generation (pop 100, 50 generations): mate, score the children and survive, each closed by a device synchronisation
and timed with a host clock, the calls DeviceNSGA2.optimize makes.  GeneralBO: GeneralAcq over a MultiTaskModel of K = 3
ensembles (2 objectives, 1 constraint), scored by one hb_de_predict_batch + hb_general_acq_epilogue, against acq.eval on
CPU tensors once per generation (the path a GeneralAcq takes over a model the device scorer does not know).  NoisyOpt:
NoisyAcq over one ensemble, scored by one hb_de_predict_batch with one draw per row, against acq.eval on CPU tensors with
BaseModel.sample_y's host draws.
suggest(): GeneralBO (K = 3, both model forms) and NoisyOpt over the ensemble after 30 observations, fit_ms / acq_ms of
last_timing, medians over --reps runs after a warm-up.
Writes DIR/bench_ensemble_multi.json with the card name and power limit read in the same run.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import pandas as pd
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_nsga import gpu_info  # noqa: E402
from hebo_b200 import DeepEnsemble, _lib  # noqa: E402
from hebo_b200.acq import GeneralAcq, NoisyAcq, ga_score, general_score  # noqa: E402
from hebo_b200.base import BaseModel  # noqa: E402
from hebo_b200.evolution import DeviceNSGA2  # noqa: E402
from hebo_b200.gp import MultiTaskModel  # noqa: E402
from hebo_b200.space import DesignSpace  # noqa: E402

D = 8


def problem(n, K, seed=0):
    g = torch.Generator().manual_seed(seed)
    Xc = torch.rand(n, D, generator=g)
    y = torch.cat([torch.sin(3 * Xc * (k + 1)).sum(1, keepdim=True) + 0.05 * torch.randn(n, 1, generator=g) for k in range(K)], 1)
    for k in range(K):
        y[torch.arange(k, n, 7 + k), k] = float("nan")
    return Xc, y


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def fit_batched(Xc, y, K):
    torch.manual_seed(0)
    mt = MultiTaskModel(D, 0, K, base_model_name="deep_ensemble")
    t, _ = timed(lambda: mt.fit(Xc, None, y))
    return t, [m.params.clone() for m in mt.models]


def fit_loop(Xc, y, K):
    torch.manual_seed(0)
    models = [DeepEnsemble(D, 0, 1) for _ in range(K)]

    def run():
        for k, m in enumerate(models):
            m.fit(Xc, None, y[:, [k]])
    t, _ = timed(run)
    return t, [m.params.clone() for m in models]


def bench_fit(ks, ns, reps):
    rows = []
    for n in ns:
        for K in ks:
            Xc, y = problem(n, K)
            fit_batched(Xc, y, K)
            fit_loop(Xc, y, K)
            tb, tl, same = [], [], True
            for _ in range(reps):
                a, pa = fit_batched(Xc, y, K)
                b, pb = fit_loop(Xc, y, K)
                tb.append(a)
                tl.append(b)
                same &= all(torch.equal(p, q) for p, q in zip(pa, pb))
            row = {"K": K, "n": n, "d": D, "ctas": 5 * K, "batched_ms_median": round(statistics.median(tb), 2),
                   "loop_ms_median": round(statistics.median(tl), 2), "batched_ms": [round(v, 2) for v in tb],
                   "loop_ms": [round(v, 2) for v in tl], "speedup": round(statistics.median(tl) / statistics.median(tb), 2),
                   "bit_identical": bool(same)}
            rows.append(row)
            print(json.dumps(row), flush=True)
    return rows


class HostGeneralAcq(GeneralAcq):
    """A subclass: general_score scores it through eval on CPU tensors."""


class HostNoisyAcq(NoisyAcq):
    """NoisyAcq.eval with BaseModel.sample_y's host draws (predict, then torch.randn on the CPU)."""

    def eval(self, x, xe):
        with torch.no_grad():
            return BaseModel.sample_y(self.model, x, xe).reshape(-1, 1)


def ga_generation(score, num_obj, constrained, G=50, pop=100):
    sp = DesignSpace().parse([{"name": f"x{i}", "type": "num", "lb": 0, "ub": 1} for i in range(D)])
    evo = DeviceNSGA2(sp.var_kinds, sp.opt_lb.numpy(), sp.opt_ub.numpy(), D, score, pop=pop, iters=3, seed=0,
                      constrained=constrained, num_obj=num_obj if num_obj > 1 else None)
    lib, P, Dd, d, st = _lib.lib(), evo.pop, evo.D, evo.d, _lib.stream_ptr
    pc = lambda x: _lib.ptr(x) if x.numel() else None
    X, Xc, Xe = evo._bufs()
    Xn, Xcn, Xen = evo._bufs()
    C, Cc, Ce = evo._bufs()
    k = num_obj if num_obj >= 2 else 3
    ws_bytes = int(lib.hb_nsga2_workspace_bytes_k(P, Dd, k))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    _lib.check(lib.hb_nsga2_init(_lib.ptr(X), P, Dd, d, _lib.ptr(evo.kind), _lib.ptr(evo.lb), _lib.ptr(evo.ub), _lib.ptr(evo.fixed),
                                 None, 0, evo.seed, pc(Xc), pc(Xe), st()), "hb_nsga2_init")
    F, Gc = evo._scored(Xc, Xe, 0)
    Fn = torch.empty_like(F)
    Gn = None if Gc is None else torch.empty_like(Gc)
    t = {"mate": [], "score": [], "survive": []}
    for gen in range(1, G + 1):
        a, _ = timed(lambda: _lib.check(lib.hb_nsga2_mate(_lib.ptr(X), P, Dd, d, _lib.ptr(evo.kind), _lib.ptr(evo.lb), _lib.ptr(evo.ub),
                                                          _lib.ptr(evo.fixed), evo.seed, gen, _lib.ptr(C), pc(Cc), pc(Ce), st()), "mate"))
        b, (FC, GC) = timed(lambda: evo._scored(Cc, Ce, gen))
        if num_obj == 1:
            c, _ = timed(lambda: _lib.check(lib.hb_ga_survive(_lib.ptr(X), _lib.ptr(F), _lib.ptr(C), _lib.ptr(FC), P, Dd, d, _lib.ptr(Xn),
                                                              _lib.ptr(Fn), pc(Xcn), pc(Xen), _lib.ptr(ws), ws_bytes, st()), "survive"))
        else:
            c, _ = timed(lambda: _lib.check(lib.hb_nsga2_survive_k(_lib.ptr(X), _lib.ptr(F), _lib.ptr(Gc), _lib.ptr(C), _lib.ptr(FC),
                                                                   _lib.ptr(GC), P, Dd, d, k, _lib.ptr(Xn), _lib.ptr(Fn), _lib.ptr(Gn),
                                                                   pc(Xcn), pc(Xen), _lib.ptr(ws), ws_bytes, st()), "survive"))
            Gc, Gn = Gn, Gc
        t["mate"].append(a)
        t["score"].append(b)
        t["survive"].append(c)
        X, Xn, Xc, Xcn, Xe, Xen, F, Fn = Xn, X, Xcn, Xc, Xen, Xe, Fn, F
    return {f"{k}_ms_median": round(statistics.median(v), 4) for k, v in t.items()}


def bench_generation():
    out = {}
    Xc, y = problem(50, 3)
    torch.manual_seed(0)
    mt = MultiTaskModel(D, 0, 3, base_model_name="deep_ensemble")
    mt.fit(Xc, None, y)
    for name, cls in (("device", GeneralAcq), ("host", HostGeneralAcq)):
        acq = cls(mt, 2, 1, kappa=2.0, c_kappa=0.0, use_noise=True)
        ga_generation(general_score(acq, 1), 2, True, G=3)                 # warm-up
        out[f"general_K3_{name}"] = ga_generation(general_score(acq, 1), 2, True)
        print(json.dumps({f"general_K3_{name}": out[f"general_K3_{name}"]}), flush=True)
    torch.manual_seed(0)
    one = DeepEnsemble(D, 0, 1)
    one.fit(Xc, None, y[:, [0]])
    for name, cls in (("device", NoisyAcq), ("host", HostNoisyAcq)):
        score = ga_score(cls(one, 1, 0), 1)
        ga_generation(score, 1, False, G=3)
        out[f"noisy_{name}"] = ga_generation(score, 1, False)
        print(json.dumps({f"noisy_{name}": out[f"noisy_{name}"]}), flush=True)
    return out


def bench_suggest(reps):
    from hebo_b200.general import GeneralBO
    from hebo_b200.noisy import NoisyOpt
    space = [{"name": f"x{i}", "type": "num", "lb": 0, "ub": 1} for i in range(D)]
    makers = {"general_deep_ensemble": lambda: GeneralBO(space, 2, 1, model_name="deep_ensemble"),
              "general_multitask_deep_ensemble": lambda: GeneralBO(space, 2, 1, model_config={"base_model_name": "deep_ensemble"}),
              "noisy_deep_ensemble": lambda: NoisyOpt(space, model_name="deep_ensemble")}
    res = {}
    for name, make in makers.items():
        fit, acq = [], []
        for r in range(reps + 1):
            torch.manual_seed(r)
            np.random.seed(r)
            opt = make()
            X = pd.DataFrame(np.random.RandomState(r).rand(30, D), columns=[f"x{i}" for i in range(D)])
            v = X.values
            y = np.stack([np.sin(3 * v).sum(1), np.cos(3 * v).sum(1), v.sum(1) - 4], 1)
            opt.observe(X, y if name.startswith("general") else y[:, :1])
            opt.suggest(1)
            if r:
                fit.append(opt.last_timing["fit_ms"])
                acq.append(opt.last_timing["acq_ms"])
        res[name] = {"fit_ms_median": round(statistics.median(fit), 2), "acq_ms_median": round(statistics.median(acq), 2)}
        print(json.dumps({name: res[name]}), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,2,4,8")
    ap.add_argument("--ns", default="50,200,1000")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ensemble_multi.py needs a GPU"
    res = {"metric": "multi-output deep ensembles: batched fit, GA generation, suggest", "gpu": gpu_info(), "members": 5,
           "epochs": 500, "fit": bench_fit([int(v) for v in args.ks.split(",")], [int(v) for v in args.ns.split(",")], args.reps),
           "ga_generation": bench_generation(), "suggest": bench_suggest(args.reps)}
    line = json.dumps(res)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_ensemble_multi.json"), "w") as fh:
            fh.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
