"""bench_noisy.py -- the device scorer of NoisyAcq (hb_sample_y_batch), the GA it drives and NoisyOpt.suggest() on one GPU.

    python bench_noisy.py --out DIR [--reps 50]

Writes DIR/bench_noisy.json with the card name and power limit read from nvidia-smi in the same run, and:
  scorer      one hb_sample_y_batch call at m = 100 rows for n in {200, 1000, 4096} observations x d in {8, 32}: time per
              call (CUDA events over --reps calls, median of 3 rounds), and its split by kernel from torch.profiler over 20
              calls in a separate pass: K* (kstar_kernel), V (rows_gemm_kernel), K** + cov (cand_features_kernel, gram_kernel,
              cov_update_kernel, the K* memset) and the new kernel (sample_batch_kernel); V's FP32 rate from 2 m n_pad^2
              flop (n_pad: n rounded up to 128);
  generation  one GA generation at pop 100 split into mate / score / survive (CUDA events around each step, mean over 100
              generations) for n in {200, 1000} x d in {8, 32}; then the whole 100-generation GA (DeviceNSGA2.optimize)
              scored by hb_sample_y_batch and by GP.sample_y per generation (the host-synchronised path), the two timed
              alternately, 3 rounds each, medians;
  suggest     NoisyOpt.suggest(8) for n in {200, 1000} x d in {8, 32}: last_timing fit_ms / acq_ms, median of 3 calls after one
              warm-up call.
Nothing is written outside DIR; it needs a GPU and fails without one.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import pandas as pd
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_nsga import event_ms, gpu_info  # noqa: E402

STAGES = {"kstar": "K*", "rows_gemm": "V", "cand_features": "K**+cov", "gram_kernel": "K**+cov", "cov_update": "K**+cov",
          "Memset": "K**+cov", "sample_batch": "sample_batch"}


def objective(x: np.ndarray) -> np.ndarray:
    return ((x - 0.3) ** 2).sum(1, keepdims=True) + 0.1 * np.sin(5 * x).sum(1, keepdims=True)


def fitted(n, d, seed):
    from hebo_b200 import GP
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (n, d))
    model = GP(d, 0, 1, warp=False, device="cuda")
    model.fit(torch.FloatTensor(X), None, torch.FloatTensor(objective(X)))
    return model


def stage_split(call, calls=20):
    from torch.profiler import ProfilerActivity, profile
    call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            call()
        torch.cuda.synchronize()
    ms = {v: 0.0 for v in STAGES.values()}
    for ev in prof.key_averages():
        for key, stage in STAGES.items():
            if key in ev.key:
                ms[stage] += ev.device_time_total / 1e3 / calls
                break
    return ms


def bench_scorer(reps):
    out = []
    m = 100
    for n in (200, 1000, 4096):
        for d in (8, 32):
            gp = fitted(n, d, n + d)
            xs = torch.rand(m, d, device="cuda") * 2 - 1
            ws = torch.empty(gp.sample_batch_workspace_bytes(m), dtype=torch.uint8, device="cuda")
            status, jit = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(1, device="cuda")
            ctr = [0]

            def call():
                ctr[0] += 1
                gp.sample_y_batch(xs, None, 7, ctr[0], status=status, jitter=jit, ws=ws)
            total = float(np.median([event_ms(call, reps) for _ in range(3)]))
            split = stage_split(call)
            n_pad = -(-n // 128) * 128
            r = dict(n=n, d=d, m=m, call_ms=total, stages_ms=split, v_tflops=2 * m * n_pad ** 2 / (split["V"] * 1e-3) / 1e12,
                     status=int(status.item()))
            out.append(r)
            print(f"scorer n={n} d={d}: {total:.4f} ms/call; " + ", ".join(f"{k} {v:.4f}" for k, v in split.items())
                  + f" ms; V {r['v_tflops']:.2f} TFLOP/s")
    return out


def ga_pieces(d):
    from hebo_b200 import _lib
    lib, p, st = _lib.lib(), _lib.ptr, _lib.stream_ptr
    P = 100
    kind = torch.zeros(d, dtype=torch.int32, device="cuda")
    lb, ub = -torch.ones(d, device="cuda"), torch.ones(d, device="cuda")
    fixed = torch.full((d,), float("nan"), device="cuda")
    ws_bytes = int(lib.hb_nsga2_workspace_bytes(P, d))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    return lib, p, st, P, kind, lb, ub, fixed, ws, ws_bytes


def bench_generation():
    from hebo_b200 import NoisyAcq, _lib
    from hebo_b200.acq import ga_score
    from hebo_b200.evolution import DeviceNSGA2
    out = []
    gens = 100
    for n in (200, 1000):
        for d in (8, 32):
            gp = fitted(n, d, n + d)
            score = ga_score(NoisyAcq(gp, 1, 0), seed=5)
            lib, p, st, P, kind, lb, ub, fixed, ws, ws_bytes = ga_pieces(d)
            X, Xc, Xn, Xcn, C, Cc = (torch.empty(P, d, device="cuda") for _ in range(6))
            fn = torch.empty(P, device="cuda")
            noe = torch.empty(P, 0, dtype=torch.int32, device="cuda")
            _lib.check(lib.hb_nsga2_init(p(X), P, d, d, p(kind), p(lb), p(ub), p(fixed), None, 0, 7, p(Xc), None, st()), "init")
            f = score(Xc, noe, 0)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            t = np.zeros(3)
            for gen in range(1, gens + 1):
                ev[0].record()
                _lib.check(lib.hb_nsga2_mate(p(X), P, d, d, p(kind), p(lb), p(ub), p(fixed), 7, gen, p(C), p(Cc), None, st()), "mate")
                ev[1].record()
                fc = score(Cc, noe, gen)
                ev[2].record()
                _lib.check(lib.hb_ga_survive(p(X), p(f), p(C), p(fc), P, d, d, p(Xn), p(fn), p(Xcn), None, p(ws), ws_bytes, st()),
                           "ga_survive")
                ev[3].record()
                torch.cuda.synchronize()
                t += [ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[2].elapsed_time(ev[3])]
                X, Xn, Xc, Xcn = Xn, X, Xcn, Xc
                f, fn = fn, f
            t /= gens

            def host_score(xc, xe, gen):
                return gp.sample_y(xc, None, 1).reshape(-1).to("cuda")

            def run_ga(sc):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                evo = DeviceNSGA2(["real"] * d, -np.ones(d), np.ones(d), d, sc, pop=P, iters=gens, seed=3)
                evo.optimize(return_pop=True)
                torch.cuda.synchronize()
                return (time.perf_counter() - t0) * 1e3
            run_ga(ga_score(NoisyAcq(gp, 1, 0), seed=5))
            run_ga(host_score)
            dev_ms, host_ms = [], []
            for _ in range(3):
                dev_ms.append(run_ga(ga_score(NoisyAcq(gp, 1, 0), seed=5)))
                host_ms.append(run_ga(host_score))
            r = dict(pop=P, n=n, d=d, gens=gens, mate_ms=float(t[0]), score_ms=float(t[1]), survive_ms=float(t[2]),
                     ga_device_ms=float(np.median(dev_ms)), ga_host_sample_y_ms=float(np.median(host_ms)), ga_device_all=dev_ms,
                     ga_host_all=host_ms, status=int(score.status.item()))
            out.append(r)
            print(f"generation n={n} d={d}: mate {t[0]:.4f} ms, score {t[1]:.4f} ms, survive {t[2]:.4f} ms; "
                  f"GA device {r['ga_device_ms']:.1f} ms, GA via GP.sample_y {r['ga_host_sample_y_ms']:.1f} ms")
    return out


def bench_suggest():
    from hebo_b200 import NoisyOpt
    out = []
    for n in (200, 1000):
        for d in (8, 32):
            np.random.seed(0)
            torch.manual_seed(0)
            space = [{"name": f"x{i}", "type": "num", "lb": -1, "ub": 1} for i in range(d)]
            opt = NoisyOpt(space, device="cuda")
            X = pd.DataFrame(np.random.uniform(-1, 1, (n, d)), columns=[f"x{i}" for i in range(d)])
            opt.observe(X, objective(X.values))
            opt.suggest(8)
            runs = []
            for _ in range(3):
                opt.suggest(8)
                runs.append(dict(opt.last_timing))
            med = {k: float(np.median([r[k] for r in runs])) for k in ("fit_ms", "acq_ms", "total_ms")}
            out.append(dict(n=n, d=d, q=8, **med, runs=runs))
            print(f"suggest n={n} d={d}: fit {med['fit_ms']:.1f} ms, acq {med['acq_ms']:.1f} ms, total {med['total_ms']:.1f} ms")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_noisy.py needs a CUDA device")
    import __graft_entry__  # noqa: F401  (puts the repository on sys.path)
    res = dict(gpu=gpu_info(), scorer=bench_scorer(a.reps), generation=bench_generation(), suggest=bench_suggest())
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_noisy.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(dict(gpu=res["gpu"]), indent=None))


if __name__ == "__main__":
    main()
