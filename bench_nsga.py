"""bench_nsga.py -- device NSGA-II at large populations (hebo_b200/csrc/nsga.cu) on one GPU.

    python bench_nsga.py --out DIR [--reps 20] [--budget 327680]

Writes DIR/bench_nsga.json with the card name and power limit read from nvidia-smi in the same run, and:
  survival     hb_nsga2_survive_ex kernel time (CUDA events, mean over --reps launches after warm-up) at pop 100 ... 16384,
               D = 32, on (a) the MACE objectives of seeded Sobol candidates under a GP fitted at bench.py's n = 4096,
               d = 32 and (b) a totally ordered set (one row per front, the worst case), with the fronts peeled;
  generation   mate / scoring / survival time per generation at pop 100 and 16384 with that GP;
  suggest      suggest().last_timing, acq_optimizer "nsga2" at evo_pop 100 and 16384 (100 generations) and the default
               Sobol path;
  quality      Sobol mega-batch of B candidates vs NSGA-II pop 100 x B/100 generations vs pop 16384 x B/16384
               generations on the same GP; every final front re-scored once with xi1 = xi2 = 0; per-objective minima and
               the coverage C(A, B) = fraction of B's front weakly dominated by a row of A.
Nothing is written outside DIR; it needs a GPU and fails without one.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import DIM, KERNEL, N_OBS, Q, candidates, synth  # noqa: E402

POPS = [100, 256, 1024, 4096, 16384]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def fronts_to_cut(F, P):
    """Fronts peeled until the cumulative count reaches P (the cut front included), same sanitising as the kernel
    (duplicates are not removed here: the bench inputs have none)."""
    f = torch.where(torch.isfinite(F), F, torch.full_like(F, float("inf")))
    N = f.shape[0]
    dom = torch.empty(N, N, dtype=torch.bool, device=f.device)           # dom[j, i]: j dominates i
    for a in range(0, N, 2048):
        o = f[a:a + 2048]
        dom[a:a + 2048] = (o[:, None, :] <= f[None, :, :]).all(-1) & (o[:, None, :] < f[None, :, :]).any(-1)
    ndom = dom.sum(0)
    ranked = torch.zeros(N, dtype=torch.bool, device=f.device)
    cum, r = 0, 0
    while True:
        front = (~ranked) & (ndom == 0)
        c = int(front.sum())
        r += 1
        if c == 0 or cum + c >= P:
            return r
        cum += c
        ranked |= front
        ndom -= dom[front].sum(0)


class Survive:
    def __init__(self, lib, _lib, X, F, C, FC):
        self.lib, self._lib = lib, _lib
        self.X, self.F, self.C, self.FC = X, F, C, FC
        P, D = X.shape
        self.P, self.D = P, D
        self.Xn, self.Fn, self.Xcn = torch.empty_like(X), torch.empty_like(F), torch.empty_like(X)
        self.Xen = torch.empty(P, 0, dtype=torch.int32, device=X.device)
        self.ws_bytes = int(lib.hb_nsga2_workspace_bytes(P, D))
        self.ws = torch.empty(self.ws_bytes, dtype=torch.uint8, device=X.device)

    def __call__(self):
        p = self._lib.ptr
        self._lib.check(self.lib.hb_nsga2_survive_ex(p(self.X), p(self.F), p(self.C), p(self.FC), self.P, self.D, self.D, p(self.Xn),
                                                     p(self.Fn), p(self.Xcn), None, p(self.ws), self.ws_bytes,
                                                     self._lib.stream_ptr()), "hb_nsga2_survive_ex")


def event_ms(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def coverage(A, B):
    """Fraction of B's rows weakly dominated (all <=) by some row of A."""
    hit = torch.zeros(B.shape[0], dtype=torch.bool, device=B.device)
    for a in range(0, A.shape[0], 1024):
        hit |= (A[a:a + 1024, None, :] <= B[None, :, :]).all(-1).any(0)
    return float(hit.float().mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--budget", type=int, default=16384 * 20)
    ap.add_argument("--skip", default="", help="comma list of sections to skip: survival,generation,suggest,quality")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_nsga.py needs a GPU"
    skip = set(filter(None, args.skip.split(",")))
    os.makedirs(args.out, exist_ok=True)
    import hebo_b200
    from hebo_b200 import _lib
    from hebo_b200.evolution import DeviceNSGA2
    from hebo_b200.pareto import pareto_front
    from hebo_b200.suggest import HEBO, hebo_y_transform, kappa_schedule
    lib = _lib.lib()
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info(), "D": DIM, "n_obs": N_OBS}

    X, y = synth(N_OBS, DIM, 1234 + 5)
    yt = hebo_y_transform(y)
    np.random.seed(0)
    torch.manual_seed(0)
    gp = hebo_b200.GP(DIM, 0, 1, lr=0.01, num_epochs=100, noise_lb=8e-4, pred_likeli=False, kernel=KERNEL, device=str(dev), rng="device")
    gp.fit(X, None, yt)
    tau, kappa = float(yt.min()), kappa_schedule(N_OBS, Q, DIM)

    def score(x, seed=0, xi=None):
        return gp.predict_mace(x, tau, kappa, 1e-4, xi, xi, seed=seed, return_mu_var=True, device_out=True)[0].contiguous()

    # ---- 1. survival kernel time
    if "survival" not in skip:
        rows = []
        for P in POPS:
            Xa = candidates(2 * P, DIM, 77).to(dev)
            sets = {"mace": score(Xa, seed=3)}
            t = torch.randperm(2 * P, generator=torch.Generator().manual_seed(P)).float().to(dev)
            sets["totally_ordered"] = torch.stack([t, 2 * t, t - 5], 1).contiguous()
            for name, Fa in sets.items():
                s = Survive(lib, _lib, Xa[:P].contiguous(), Fa[:P].contiguous(), Xa[P:].contiguous(), Fa[P:].contiguous())
                s()
                torch.cuda.synchronize()
                ms = event_ms(s, args.reps if not (name == "totally_ordered" and P >= 4096) else max(3, args.reps // 4))
                fr = fronts_to_cut(Fa, P)
                rows.append({"pop": P, "objectives": name, "kernel": "single-CTA" if P <= 256 else "multi-CTA",
                             "fronts_peeled": fr, "ms": round(ms, 4), "us_per_front": round(1e3 * ms / fr, 3)})
                print(json.dumps(rows[-1]), flush=True)
        res["survival"] = rows

    def make_evo(pop, iters, seed=5):
        return DeviceNSGA2(["real"] * DIM, -np.ones(DIM), np.ones(DIM), DIM, lambda xc, xe, gen: score(xc, seed=gen),
                           pop=pop, iters=iters, seed=seed, device=dev)

    # ---- 2. per-generation breakdown (events around each stage of a generation loop written out here)
    if "generation" not in skip:
        rows = []
        for P in (100, 16384):
            evo = make_evo(P, 2)
            evo.optimize()
            Xp = evo.pop_X.contiguous()
            Fp = evo.pop_F.contiguous()
            kind = evo.kind
            lb, ub, fixed = evo.lb, evo.ub, evo.fixed
            C = torch.empty_like(Xp)
            Cc = torch.empty_like(Xp)
            Ce = torch.empty(P, 0, dtype=torch.int32, device=dev)
            p = _lib.ptr

            def mate(gen=[1]):
                gen[0] += 1
                _lib.check(lib.hb_nsga2_mate(p(Xp), P, DIM, DIM, p(kind), p(lb), p(ub), p(fixed), 5, gen[0], p(C), p(Cc), None,
                                             _lib.stream_ptr()), "mate")
            mate()
            FC = score(Cc)
            s = Survive(lib, _lib, Xp, Fp, C, FC)
            reps = 50
            row = {"pop": P, "mate_ms": event_ms(mate, reps), "score_ms": event_ms(lambda: score(Cc), reps),
                   "survive_ms": event_ms(s, reps)}
            row = {k: (round(v, 4) if isinstance(v, float) else v) for k, v in row.items()}
            rows.append(row)
            print(json.dumps(row), flush=True)
        res["generation"] = rows

    # ---- 3. suggest() time
    if "suggest" not in skip:
        rows = []
        for opt_name, pop in (("sobol", None), ("nsga2", 100), ("nsga2", 16384)):
            kw = {} if pop is None else {"acq_optimizer": "nsga2", "evo_pop": pop, "evo_iters": 100}
            opt = HEBO(-torch.ones(DIM), torch.ones(DIM), n_candidates=10000, device=str(dev), scramble_seed=1, **kw)
            opt.observe(X, y)
            ts = []
            for _ in range(3):
                np.random.seed(0)
                opt.suggest(Q)
                ts.append(dict(opt.last_timing))
            best = min(ts[1:], key=lambda r: r["total_ms"])
            row = {"acq_optimizer": opt_name, "evo_pop": pop, "evo_iters": None if pop is None else 100,
                   "last_timing": {k: (round(v, 2) if isinstance(v, float) else v) for k, v in best.items()},
                   "all_total_ms": [round(r["total_ms"], 2) for r in ts]}
            rows.append(row)
            print(json.dumps(row), flush=True)
        res["suggest"] = rows

    # ---- 4. quality at equal evaluation budget
    if "quality" not in skip:
        B = args.budget
        fronts = {}
        t0 = time.perf_counter()
        Xs = candidates(B, DIM, 4242).to(dev)
        Fs = score(Xs, seed=1)
        fronts["sobol"] = Xs[pareto_front(Fs)]
        timing = {"sobol": time.perf_counter() - t0}
        for P in (100, 16384):
            t0 = time.perf_counter()
            evo = make_evo(P, max(1, B // P), seed=9)
            xc, _, _ = evo.optimize()
            torch.cuda.synchronize()
            timing[f"nsga2_pop{P}"] = time.perf_counter() - t0
            fronts[f"nsga2_pop{P}"] = xc
        F0 = {}
        for k, xf in fronts.items():
            z = torch.zeros(xf.shape[0], device=dev)
            F0[k] = score(xf.contiguous(), xi=z)
        q = {"budget": B, "generations": {"nsga2_pop100": max(1, B // 100), "nsga2_pop16384": max(1, B // 16384)},
             "wall_s": {k: round(v, 3) for k, v in timing.items()},
             "front_size": {k: int(v.shape[0]) for k, v in F0.items()},
             "min_objectives": {k: [float(x) for x in v.min(0).values] for k, v in F0.items()},
             "coverage": {f"C({a},{b})": round(coverage(F0[a], F0[b]), 4) for a in F0 for b in F0 if a != b}}
        res["quality"] = q
        print(json.dumps(q), flush=True)

    with open(os.path.join(args.out, "bench_nsga.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps({"gpu": res["gpu"]}))


if __name__ == "__main__":
    main()
