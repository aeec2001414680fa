"""Measures MOMeanSigmaLCB on the device and HEBO.suggest() with its acquisition classes.

    python bench_acq.py --out DIR

Writes DIR/bench_acq.json with the card name and power limit read from nvidia-smi in the same run, and:
  * epilogue: hb_mo_lcb_epilogue (Philox draws) at m = 10^4, 131 072 and 10^6 rows, time per launch (launches replayed
    from a CUDA graph; the time of one eager call from Python is recorded beside it) and bytes/s against the 3.35 TB/s
    HBM3 figure of the H100 SXM data sheet; the traffic is 8 B in (mu, var) and 12 B out (F [m, 2], G) per row;
  * generation: one NSGA-II generation at pop 100 for n = 200 / 1000 observations and d = 8 / 32, split into mate /
    posterior / epilogue / hb_nsga2_survive_k (K = 2 with the G column), CUDA events around each stage, medians;
  * suggest: HEBO.suggest() fit and acquisition ms for acq_cls = MACE / MOMeanSigmaLCB with the Sobol and the NSGA-II
    acquisition optimisers, at the same sizes (medians of three suggests after one warm-up).
"""
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

HBM_BYTES_PER_S = 3.35e12


def bench_epilogue():
    from hebo_b200 import _lib
    lib, p = _lib.lib(), _lib.ptr
    out = []
    for m in (10 ** 4, 131072, 10 ** 6):
        mu, var = torch.randn(m, device="cuda"), torch.rand(m, device="cuda")
        F, G = torch.empty(m, 2, device="cuda"), torch.empty(m, device="cuda")

        def run():
            _lib.check(lib.hb_mo_lcb_epilogue(p(mu), p(var), m, 0.1, 0.0, 2.0, None, 1, 2, p(F), p(G), _lib.stream_ptr()),
                       "hb_mo_lcb_epilogue")
        reps = 2000 if m < 10 ** 6 else 500
        eager = float(np.median([event_ms(run, reps) for _ in range(5)]))
        # one call from Python costs more host time than a small launch takes on the device, so the kernel is timed as
        # `burst` launches back to back in one CUDA graph
        burst = 100
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            run()
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(burst):
                run()
        runs = [event_ms(graph.replay, 20) / burst for _ in range(5)]
        ms = float(np.median(runs))
        nbytes = 20 * m
        rate = nbytes / (ms * 1e-3)
        out.append(dict(m=m, ms=ms, bytes=nbytes, bytes_per_s=rate, share_of_hbm=rate / HBM_BYTES_PER_S, runs=runs,
                        eager_call_ms=eager))
        print(f"epilogue m={m}: {ms * 1e3:.2f} us in a graph, {rate / 1e9:.1f} GB/s ({100 * rate / HBM_BYTES_PER_S:.1f}% of "
              f"3.35 TB/s); {eager * 1e3:.2f} us per eager call")
    return out


def fitted(n, d, seed):
    import hebo_b200
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (n, d)).astype(np.float32)
    y = (np.sin(3 * X[:, :1]) + (X ** 2).sum(1, keepdims=True) / d).astype(np.float32)
    gp = hebo_b200.GP(d, 0, 1, device="cuda")
    gp.fit(torch.from_numpy(X), None, torch.from_numpy(y))
    torch.cuda.synchronize()
    return gp, X, y


def bench_generation():
    from hebo_b200 import _lib
    from hebo_b200.acq import MOMeanSigmaLCB, _mo_lcb_epilogue, _noise_sd
    lib, p = _lib.lib(), _lib.ptr
    out = []
    P, K = 100, 2
    for n in (200, 1000):
        for d in (8, 32):
            gp, _, y = fitted(n, d, n + d)
            acq = MOMeanSigmaLCB(gp, best_y=float(y.min()), kappa=2.0)
            sd = _noise_sd(gp)
            kind = torch.zeros(d, dtype=torch.int32, device="cuda")
            lb, ub = -torch.ones(d, device="cuda"), torch.ones(d, device="cuda")
            fixed = torch.full((d,), float("nan"), device="cuda")
            X = torch.rand(P, d, device="cuda") * 2 - 1
            Cb, Cc = torch.empty(P, d, device="cuda"), torch.empty(P, d, device="cuda")
            Xn, Xcn = torch.empty_like(X), torch.empty_like(X)
            mu, var = torch.empty(P, device="cuda"), torch.empty(P, device="cuda")
            F, G = _mo_lcb_epilogue(*gp._posterior(X, False)[1:], sd, float(y.min()), 2.0, None, 1, 0)
            FC, GC = torch.empty_like(F), torch.empty_like(G)
            Fn, Gn = torch.empty_like(F), torch.empty_like(G)
            ws_bytes = int(lib.hb_nsga2_workspace_bytes_k(P, d, 3))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")

            def mate():
                _lib.check(lib.hb_nsga2_mate(p(X), P, d, d, p(kind), p(lb), p(ub), p(fixed), 1, 1, p(Cb), p(Cc), None,
                                             _lib.stream_ptr()), "mate")

            def post():
                gp._posterior(Cc, False, out=(mu, var))

            def epi():
                _lib.check(lib.hb_mo_lcb_epilogue(p(mu), p(var), P, sd, float(acq.best_y), 2.0, None, 1, 1, p(FC), p(GC),
                                                  _lib.stream_ptr()), "hb_mo_lcb_epilogue")

            def surv():
                _lib.check(lib.hb_nsga2_survive_k(p(X), p(F), p(G), p(Cb), p(FC), p(GC), P, d, d, K, p(Xn), p(Fn), p(Gn), p(Xcn),
                                                  None, p(ws), ws_bytes, _lib.stream_ptr()), "survive_k")
            mate()
            post()
            epi()
            t = {k: [] for k in ("mate", "posterior", "epilogue", "survive")}
            for _ in range(5):
                t["mate"].append(event_ms(mate, 50))
                t["posterior"].append(event_ms(post, 50))
                t["epilogue"].append(event_ms(epi, 50))
                t["survive"].append(event_ms(surv, 50))
            med = {k + "_ms": float(np.median(v)) for k, v in t.items()}
            med["generation_ms"] = sum(med.values())
            out.append(dict(n=n, d=d, pop=P, **med))
            print(f"generation n={n} d={d}: " + ", ".join(f"{k} {v:.4f}" for k, v in med.items()))
    return out


def bench_suggest():
    from hebo_b200 import MACE, MOMeanSigmaLCB
    from hebo_b200.suggest import HEBO
    out = []
    for n in (200, 1000):
        for d in (8, 32):
            _, X, y = fitted(n, d, n + d)
            for acq_cls in (MACE, MOMeanSigmaLCB):
                for acq_optimizer in ("sobol", "nsga2"):
                    np.random.seed(0)
                    torch.manual_seed(0)
                    opt = HEBO(-torch.ones(d), torch.ones(d), acq_cls=acq_cls, acq_optimizer=acq_optimizer, scramble_seed=0)
                    opt.observe(torch.from_numpy(X), y)
                    opt.suggest(1)
                    runs = []
                    for _ in range(3):
                        opt.suggest(1)
                        runs.append(dict(opt.last_timing))
                    med = {k: float(np.median([r[k] for r in runs])) for k in ("fit_ms", "score_ms", "total_ms")}
                    out.append(dict(n=n, d=d, acq_cls=acq_cls.__name__, acq_optimizer=acq_optimizer, **med, runs=runs))
                    print(f"suggest n={n} d={d} {acq_cls.__name__} {acq_optimizer}: "
                          + ", ".join(f"{k} {v:.1f}" for k, v in med.items()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_acq.py needs a CUDA device")
    import __graft_entry__  # noqa: F401  (puts the repository on sys.path)
    res = dict(gpu=gpu_info(), epilogue=bench_epilogue(), generation=bench_generation(), suggest=bench_suggest())
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_acq.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(dict(gpu=res["gpu"]), indent=None))


if __name__ == "__main__":
    main()
