"""Measures the GeneralBO path on the device.

    python bench_general.py --out DIR [--reps-floor 5]

Writes DIR/bench_general.json with the card name and power limit read from nvidia-smi in the same run, and:
  * survival: hb_nsga2_survive_k at pop 100 / 1024 / 4096 / 16 384 and k = 2, 3, 4, 8 objectives, timed alternately with
    hb_nsga2_survive_ex (k = 3) on the same rows; hb_ga_survive_cv alternately with hb_ga_survive;
  * generation: one GA generation at pop 100 for n = 200 / 1000 observations, K = 2 / 3 / 5 outputs, d = 8, split into
    mate / K posterior calls / epilogue / survive (CUDA events around each stage, medians over repetitions);
  * suggest: GeneralBO.suggest() split into fit / acquisition / selection ms, with and without ref_point.
"""
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


def bench_survival(reps_floor):
    from hebo_b200 import _lib
    lib, p = _lib.lib(), _lib.ptr
    out = []
    for P in (100, 1024, 4096, 16384):
        D = 16
        g = torch.Generator(device="cuda").manual_seed(P)
        X, C = torch.rand(P, D, device="cuda", generator=g), torch.rand(P, D, device="cuda", generator=g)
        G, GC = torch.randn(P, device="cuda", generator=g), torch.randn(P, device="cuda", generator=g)
        Xn, Xcn, Gn = torch.empty_like(X), torch.empty_like(X), torch.empty_like(G)
        reps = max(reps_floor, 50 if P < 16384 else 10)
        for k in (2, 3, 4, 8):
            F, FC = torch.randn(P, k, device="cuda", generator=g), torch.randn(P, k, device="cuda", generator=g)
            Fn = torch.empty_like(F)
            ws_bytes = int(lib.hb_nsga2_workspace_bytes_k(P, D, max(k, 3)))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
            F3, FC3 = F[:, :1].repeat(1, 3).contiguous(), FC[:, :1].repeat(1, 3).contiguous()
            F3[:, :min(k, 3)], FC3[:, :min(k, 3)] = F[:, :3], FC[:, :3]
            Fn3 = torch.empty_like(F3)

            def sk():
                _lib.check(lib.hb_nsga2_survive_k(p(X), p(F), None, p(C), p(FC), None, P, D, D, k, p(Xn), p(Fn), None, p(Xcn), None,
                                                  p(ws), ws_bytes, _lib.stream_ptr()), "hb_nsga2_survive_k")

            def ex():
                _lib.check(lib.hb_nsga2_survive_ex(p(X), p(F3), p(C), p(FC3), P, D, D, p(Xn), p(Fn3), p(Xcn), None, p(ws), ws_bytes,
                                                   _lib.stream_ptr()), "hb_nsga2_survive_ex")
            t_k, t_ex = [], []
            for _ in range(5):
                t_k.append(event_ms(sk, reps))
                t_ex.append(event_ms(ex, reps))
            r = dict(pop=P, D=D, k=k, survive_k_ms=float(np.median(t_k)), survive_ex_k3_ms=float(np.median(t_ex)), k_all=t_k, ex_all=t_ex)
            out.append(r)
            print(f"survival pop={P} k={k}: survive_k {r['survive_k_ms']:.4f} ms, survive_ex (k=3) {r['survive_ex_k3_ms']:.4f} ms")
        f, fc, fn = G.clone(), GC.clone(), torch.empty_like(G)
        ws_bytes = int(lib.hb_nsga2_workspace_bytes(P, D))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")

        def ga():
            _lib.check(lib.hb_ga_survive(p(X), p(f), p(C), p(fc), P, D, D, p(Xn), p(fn), p(Xcn), None, p(ws), ws_bytes,
                                         _lib.stream_ptr()), "hb_ga_survive")

        def gacv():
            _lib.check(lib.hb_ga_survive_cv(p(X), p(f), p(G), p(C), p(fc), p(GC), P, D, D, p(Xn), p(fn), p(Gn), p(Xcn), None, p(ws),
                                            ws_bytes, _lib.stream_ptr()), "hb_ga_survive_cv")
        t_ga, t_cv = [], []
        for _ in range(5):
            t_ga.append(event_ms(ga, reps))
            t_cv.append(event_ms(gacv, reps))
        r = dict(pop=P, D=D, ga_ms=float(np.median(t_ga)), ga_cv_ms=float(np.median(t_cv)), ga_all=t_ga, ga_cv_all=t_cv)
        out.append(r)
        print(f"survival pop={P}: ga {r['ga_ms']:.4f} ms, ga_cv {r['ga_cv_ms']:.4f} ms")
    return out


def bench_generation():
    """One generation of the GeneralBO GA at pop 100 (d = 8, one constraint among the K outputs), stage by stage."""
    import hebo_b200
    from hebo_b200 import _lib
    from hebo_b200.acq import GeneralAcq, general_score
    lib, p = _lib.lib(), _lib.ptr
    out = []
    P, d = 100, 8
    for n in (200, 1000):
        for K in (2, 3, 5):
            rng = np.random.default_rng(n + K)
            Xo = torch.from_numpy(rng.uniform(-1, 1, (n, d)).astype(np.float32))
            Y = torch.from_numpy(rng.normal(size=(n, K)).astype(np.float32))
            model = hebo_b200.MultiTaskModel(d, 0, K, device="cuda")
            model.fit(Xo, None, Y)
            acq = GeneralAcq(model, K - 1, 1, kappa=2.0, c_kappa=0.0, use_noise=True)
            score = general_score(acq, 1)
            kind = torch.zeros(d, dtype=torch.int32, device="cuda")
            lb, ub = -torch.ones(d, device="cuda"), torch.ones(d, device="cuda")
            fixed = torch.full((d,), float("nan"), device="cuda")
            X, Xc = torch.rand(P, d, device="cuda") * 2 - 1, torch.empty(P, d, device="cuda")
            Cb, Cc = torch.empty(P, d, device="cuda"), torch.empty(P, d, device="cuda")
            Xn, Xcn = torch.empty_like(X), torch.empty_like(X)
            F, Gv = score(X, None, 0)
            FC, GC = score(X, None, 1)
            Fn, Gn = torch.empty_like(F), torch.empty_like(Gv)
            ws_bytes = int(lib.hb_nsga2_workspace_bytes_k(P, d, max(K - 1, 3)))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
            mu, var = torch.empty(K, P, device="cuda"), torch.empty(K, P, device="cuda")

            def mate():
                _lib.check(lib.hb_nsga2_mate(p(X), P, d, d, p(kind), p(lb), p(ub), p(fixed), 1, 1, p(Cb), p(Cc), None,
                                             _lib.stream_ptr()), "mate")

            def post():
                for b, gp in enumerate(model.models):
                    gp._posterior(Cc, False, out=(mu[b], var[b]))

            def epi():
                score(Cc, None, 2)

            def surv():
                if K - 1 >= 2:
                    _lib.check(lib.hb_nsga2_survive_k(p(X), p(F), p(Gv), p(Cb), p(FC), p(GC), P, d, d, K - 1, p(Xn), p(Fn), p(Gn), p(Xcn),
                                                      None, p(ws), ws_bytes, _lib.stream_ptr()), "survive_k")
                else:
                    _lib.check(lib.hb_ga_survive_cv(p(X), p(F), p(Gv), p(Cb), p(FC), p(GC), P, d, d, p(Xn), p(Fn), p(Gn), p(Xcn), None,
                                                    p(ws), ws_bytes, _lib.stream_ptr()), "ga_survive_cv")
            mate()
            t = {k: [] for k in ("mate", "posterior_K", "score_total", "survive")}
            for _ in range(5):
                t["mate"].append(event_ms(mate, 50))
                t["posterior_K"].append(event_ms(post, 50))
                t["score_total"].append(event_ms(epi, 50))
                t["survive"].append(event_ms(surv, 50))
            med = {k + "_ms": float(np.median(v)) for k, v in t.items()}
            med["epilogue_ms"] = med["score_total_ms"] - med["posterior_K_ms"]
            out.append(dict(n=n, K=K, d=d, pop=P, **med))
            print(f"generation n={n} K={K}: " + ", ".join(f"{k} {v:.4f}" for k, v in med.items()))
    return out


def bench_suggest():
    import hebo_b200
    out = []
    d = 8
    space = [{"name": f"x{i}", "type": "num", "lb": -1, "ub": 1} for i in range(d)]
    for n in (200, 1000):
        for ref in (None, np.array([3.0, 3.0])):
            np.random.seed(0)
            nc = 1 if ref is None else 0                  # the EHVI selection takes unconstrained problems only
            opt = hebo_b200.GeneralBO(space, 2, nc, ref_point=ref, evo_pop=100, evo_iters=200)
            X = pd.DataFrame(np.random.uniform(-1, 1, (n, d)), columns=[f"x{i}" for i in range(d)])
            x = X.values
            y = np.stack([(x ** 2).sum(1), ((x - 0.5) ** 2).sum(1), x[:, 0] - 0.5], 1)
            opt.observe(X, y[:, :2 + nc])
            opt.suggest(4)
            runs = []
            for _ in range(3):
                opt.suggest(4)
                runs.append(dict(opt.last_timing))
            med = {k: float(np.median([r[k] for r in runs])) for k in ("fit_ms", "acq_ms", "select_ms", "total_ms")}
            out.append(dict(n=n, d=d, ref_point=ref is not None, **med, runs=runs))
            print(f"suggest n={n} ref_point={ref is not None}: " + ", ".join(f"{k} {v:.1f}" for k, v in med.items()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps-floor", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_general.py needs a CUDA device")
    import __graft_entry__  # noqa: F401  (puts the repository on sys.path)
    res = dict(gpu=gpu_info(), survival=bench_survival(a.reps_floor), generation=bench_generation(), suggest=bench_suggest())
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_general.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(dict(gpu=res["gpu"]), indent=None))


if __name__ == "__main__":
    main()
