"""bench_embedding.py -- HEBO_Embedding on one GPU: the bound-violation kernel, the constrained NSGA-II survival, and
suggest().

    python bench_embedding.py --out DIR [--reps-floor 5]

Writes DIR/bench_embedding.json with the card name and power limit read from nvidia-smi in the same run, and:
  violation   hb_embed_violation time (CUDA events, mean over repeated launches after warm-up; both launches of a call),
              achieved FLOP/s over the algorithmic 2 m e D flop, and that rate over the data-sheet FP32 peak of the H100
              SXM (67 TFLOP/s), at e in {8, 16, 32} x D in {1e3, 1e4, 1e5} x m in {10 000, 131 072};
  survival    hb_nsga2_survive_cv against hb_nsga2_survive_ex on the same all-feasible inputs (G = 0), D = 16, at pop 100,
              1024 and 4096, timed alternately (5 rounds, the median of each);
  suggest     HEBO_Embedding.suggest() at D = 10 000, eff_dim = 16, 200 observations, both acquisition optimisers:
              last_timing fit_ms / score_ms / total_ms, median of 3 calls after one warm-up call.
Nothing is written outside DIR; it needs a GPU and fails without one.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_nsga import event_ms, gpu_info  # noqa: E402

FP32_PEAK = 67e12      # H100 SXM data sheet, dense FP32, at up to 700 W


def bench_violation(reps_floor):
    from hebo_b200.embedding import embed_violation
    out = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for e in (8, 16, 32):
        for D in (1000, 10000, 100000):
            B = torch.randn(e, D, device="cuda", generator=g) / e ** 0.5
            for m in (10000, 131072):
                Y = torch.rand(m, e, device="cuda", generator=g) * 2 - 1
                flop = 2.0 * m * e * D
                reps = max(reps_floor, min(200, int(4e12 / flop)))
                ms = event_ms(lambda: embed_violation(Y, B), reps)
                rate = flop / (ms * 1e-3)
                out.append(dict(m=m, e=e, D=D, ms=ms, reps=reps, tflops=rate / 1e12, fp32_peak_share=rate / FP32_PEAK))
                print(f"violation m={m} e={e} D={D}: {ms:.3f} ms, {rate / 1e12:.1f} TFLOP/s ({100 * rate / FP32_PEAK:.0f}% of peak)")
    return out


def bench_survival(reps_floor):
    from hebo_b200 import _lib
    lib, p = _lib.lib(), _lib.ptr
    out = []
    for P in (100, 1024, 4096):
        D = 16
        g = torch.Generator(device="cuda").manual_seed(P)
        X, C = torch.rand(P, D, device="cuda", generator=g), torch.rand(P, D, device="cuda", generator=g)
        F, FC = torch.randn(P, 3, device="cuda", generator=g), torch.randn(P, 3, device="cuda", generator=g)
        z = torch.zeros(P, device="cuda")
        Xn, Fn, Gn, Xcn = torch.empty_like(X), torch.empty_like(F), torch.empty_like(z), torch.empty_like(X)
        ws_bytes = int(lib.hb_nsga2_workspace_bytes(P, D))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")

        def ex():
            _lib.check(lib.hb_nsga2_survive_ex(p(X), p(F), p(C), p(FC), P, D, D, p(Xn), p(Fn), p(Xcn), None, p(ws), ws_bytes,
                                               _lib.stream_ptr()), "hb_nsga2_survive_ex")

        def cv():
            _lib.check(lib.hb_nsga2_survive_cv(p(X), p(F), p(z), p(C), p(FC), p(z), P, D, D, p(Xn), p(Fn), p(Gn), p(Xcn), None,
                                               p(ws), ws_bytes, _lib.stream_ptr()), "hb_nsga2_survive_cv")
        reps = max(reps_floor, 50)
        t_ex, t_cv = [], []
        for _ in range(5):
            t_ex.append(event_ms(ex, reps))
            t_cv.append(event_ms(cv, reps))
        r = dict(pop=P, ex_ms=float(np.median(t_ex)), cv_ms=float(np.median(t_cv)), ex_all=t_ex, cv_all=t_cv)
        out.append(r)
        print(f"survival pop={P}: ex {r['ex_ms']:.4f} ms, cv {r['cv_ms']:.4f} ms")
    return out


def bench_suggest():
    from hebo_b200.embedding import HEBO_Embedding
    D, eff, n_obs = 10000, 16, 200
    space = [{"name": f"x{i}", "type": "num", "lb": -1, "ub": 1} for i in range(D)]
    out = {}
    for acq_optimizer in ("sobol", "nsga2"):
        np.random.seed(0)
        torch.manual_seed(0)
        h = HEBO_Embedding(space, eff_dim=eff, acq_optimizer=acq_optimizer, device="cuda")
        X = h.quasi_sample(n_obs)
        x = h.project(X).values
        h.observe(X, ((x[:, :20] - 0.3) ** 2).sum(1, keepdims=True) + 0.1 * np.sin(7 * x[:, 20:40]).sum(1, keepdims=True))
        h.suggest()
        runs = []
        for _ in range(3):
            h.suggest()
            runs.append(dict(h.mace.last_timing))
        med = {k: float(np.median([r[k] for r in runs])) for k in ("fit_ms", "score_ms", "total_ms")}
        out[acq_optimizer] = dict(**med, front=runs[-1]["front"], runs=runs)
        print(f"suggest {acq_optimizer}: fit {med['fit_ms']:.1f} ms, score {med['score_ms']:.1f} ms, total {med['total_ms']:.1f} ms")
    return dict(D=D, eff_dim=eff, n_obs=n_obs, **out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps-floor", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_embedding.py needs a CUDA device")
    import __graft_entry__  # noqa: F401  (puts the repository on sys.path)
    res = dict(gpu=gpu_info(), violation=bench_violation(a.reps_floor), survival=bench_survival(a.reps_floor),
               suggest=bench_suggest())
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_embedding.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(dict(gpu=res["gpu"]), indent=None))


if __name__ == "__main__":
    main()
