"""NSGA-II acquisition optimiser for box-bounded continuous spaces (tensor/array form).

The reference optimises the MACE objectives with pymoo's NSGA-II (HEBO/hebo/acq_optimizers/evolution_optimizer.py:107-160:
pop 100, `iters` generations of 100 offspring, MixedVariableMating = random parent selection + SBX crossover +
polynomial mutation, duplicate elimination, rank-and-crowding survival; the result is the non-dominated part of the
final population).  pymoo is a third-party dependency that is not installed here, so this is a restatement of the
published algorithm (Deb et al. 2002) with pymoo 0.6 operator defaults as recalled in SURVEY.md Appendix C
(SBX eta=15, pair probability 0.9, per-variable 0.5; PM eta=20, per-variable min(0.5, 1/d)); parity with pymoo's random
stream is neither possible nor claimed.  The bookkeeping (200 x 3 objective values per generation) runs vectorised on the
host like pymoo's; every generation's offspring are scored in ONE call of `acq_fn` (the fused posterior+MACE pass on the
device), which replaces the per-individual marshalling of evolution_optimizer.py:84-105.

`hebo_b200.suggest.HEBO(acq_optimizer="nsga2")` runs the DEVICE version below (`DeviceNSGA2`: population, mating, typed
repair, duplicate elimination and rank-and-crowding survival in CUDA kernels, hebo_b200/csrc/nsga.cu; no per-generation
host round trip); the numpy functions in this file restate the same operators on the host and serve as the checker of
those kernels (tests/test_evolution.py, tests/test_gpu_nsga.py).  The default optimiser of suggest() is the one-pass Sobol
mega-batch.  With a one-objective score `DeviceNSGA2` is the single-objective GA of the reference (pymoo's
MixedVariableGA, evolution_optimizer.py:123-124,132-133): the same mating, the fitness survival of `hb_ga_survive`
(restated by `ga_survive_host`); `hebo_b200.BO` runs it.
"""
from __future__ import annotations

from typing import Callable, Optional

import numpy as np


def dominance_matrix(F: np.ndarray) -> np.ndarray:
    """D[i, j] = True iff row i dominates row j (all <=, one <), minimisation."""
    le = (F[:, None, :] <= F[None, :, :]).all(-1)
    lt = (F[:, None, :] < F[None, :, :]).any(-1)
    return le & lt


def fast_non_dominated_sort(F: np.ndarray) -> np.ndarray:
    """Front index (0 = non-dominated) of every row."""
    n = F.shape[0]
    D = dominance_matrix(F)
    n_dom = D.sum(0).astype(np.int64)          # how many rows dominate j
    rank = np.full(n, -1, dtype=np.int64)
    current = np.flatnonzero(n_dom == 0)
    r = 0
    while current.size:
        rank[current] = r
        n_dom[current] = -1                    # never selected again
        n_dom -= D[current].sum(0)             # remove their dominance (entries already at -1 only go lower)
        current = np.flatnonzero(n_dom == 0)
        r += 1
    return rank


def crowding_distance(F: np.ndarray) -> np.ndarray:
    """Crowding distance inside ONE front (boundary points get +inf)."""
    n, m = F.shape
    if n <= 2:
        return np.full(n, np.inf)
    dist = np.zeros(n)
    for k in range(m):
        order = np.argsort(F[:, k], kind="stable")
        f = F[order, k]
        span = f[-1] - f[0]
        d = np.zeros(n)
        d[0] = d[-1] = np.inf
        if span > 0:
            d[1:-1] = (f[2:] - f[:-2]) / span
        dist[order] += d
    return dist


def rank_and_crowding_survival(F: np.ndarray, n_survive: int) -> np.ndarray:
    """Indices of the survivors: whole fronts in rank order, the last one truncated by descending crowding distance."""
    rank = fast_non_dominated_sort(F)
    keep = []
    for r in range(rank.max() + 1):
        front = np.flatnonzero(rank == r)
        if len(keep) + front.size <= n_survive:
            keep.extend(front.tolist())
        else:
            cd = crowding_distance(F[front])
            order = np.argsort(-cd, kind="stable")
            keep.extend(front[order[: n_survive - len(keep)]].tolist())
        if len(keep) >= n_survive:
            break
    return np.asarray(keep, dtype=np.int64)


def ga_survive_host(X: np.ndarray, F: np.ndarray, C: np.ndarray, FC: np.ndarray):
    """numpy restatement of hb_ga_survive in fp32: a non-finite f becomes +inf, a duplicate child (the predicate of
    survive_host) gets +inf, and the P merged rows first in ascending (f, merged index) order survive in that order.
    Returns the merged indices of the survivors in output order (best first) and the sanitised f [2P]."""
    P = X.shape[0]
    Xa = np.concatenate([X, C], 0).astype(np.float32)
    f = np.concatenate([np.asarray(F).reshape(-1), np.asarray(FC).reshape(-1)]).astype(np.float32)
    f = np.where(np.isfinite(f), f, np.float32(np.inf))
    # rows the predicate calls equal share a key (0 for |v| < 2^-20, else the bit pattern: the fp32 spacing above 2^-20
    # exceeds 1e-16), so each child is tested against the earlier rows of its key only -- the exact predicate, in O(N D)
    key = np.where(np.abs(Xa) < np.float32(2.0 ** -20), np.uint32(0), Xa.view(np.uint32))
    earlier = {}
    for i in range(2 * P):
        rows = earlier.setdefault(key[i].tobytes(), [])
        if i >= P and rows and (np.abs(Xa[rows] - Xa[i]) <= np.float32(1e-16)).all(1).any():
            f[i] = np.inf
        rows.append(i)
    order = np.lexsort((np.arange(2 * P), f))          # primary f, ties by the lower merged index
    return order[:P], f


def survive_host(X: np.ndarray, F: np.ndarray, C: np.ndarray, FC: np.ndarray, G: Optional[np.ndarray] = None,
                 GC: Optional[np.ndarray] = None):
    """numpy restatement of the device survival (hb_nsga2_survive_ex, and hb_nsga2_survive_cv when G / GC are given),
    fp32 like the kernels so that the survivors agree bit for bit: sanitising, duplicate children, the constraint rule,
    ranks, fp32 crowding of the cut front (see the rules in hebo_b200/csrc/nsga.cu).  Returns the merged indices of the
    survivors in ascending order, and the sanitised objectives [2P, 3] and constraint [2P] of the merged rows."""
    P = X.shape[0]
    Xa = np.concatenate([X, C], 0).astype(np.float32)
    f = np.concatenate([F, FC], 0).astype(np.float32)
    f = np.where(np.isfinite(f), f, np.float32(np.inf))
    cons = G is not None
    g = np.zeros(2 * P, np.float32) if not cons else np.concatenate([G, GC]).astype(np.float32).reshape(-1)
    g = np.where(np.isfinite(g), g, np.float32(np.inf))
    for i in range(P, 2 * P):
        if (np.abs(Xa[:i] - Xa[i]) <= np.float32(1e-16)).all(1).any():
            f[i] = np.inf
            if cons:
                g[i] = np.inf
    feas = g <= 0
    nf = int(feas.sum())
    keep = np.zeros(2 * P, bool)
    if nf < P:
        keep |= feas
        inf_rows = np.flatnonzero(~feas)
        keep[inf_rows[np.argsort(g[inf_rows], kind="stable")[:P - nf]]] = True
        return np.flatnonzero(keep), f, g
    rows = np.flatnonzero(feas)
    fr = f[rows]
    rank = fast_non_dominated_sort(fr)
    cum = 0
    for r in range(rank.max() + 1):
        members = np.flatnonzero(rank == r)
        if cum + members.size < P:
            keep[rows[members]] = True
            cum += members.size
            continue
        fm, m = fr[members], members.size
        crowd = np.zeros(m, np.float32)
        for k in range(3):
            v = fm[:, k]
            order = np.argsort(v, kind="stable")
            pos = np.empty(m, np.int64)
            pos[order] = np.arange(m)
            fmin, fmax = v[order[0]], v[order[-1]]
            ends = (pos == 0) | (pos == m - 1)
            if fmax > fmin and np.isfinite(fmax - fmin):
                with np.errstate(invalid="ignore", over="ignore"):
                    step = (v[order[np.minimum(pos + 1, m - 1)]] - v[order[np.maximum(pos - 1, 0)]]) / (fmax - fmin)
                crowd = np.where(ends, crowd, crowd + step).astype(np.float32)
            crowd = np.where(ends, np.float32(np.inf), crowd).astype(np.float32)
        keep[rows[members[np.argsort(-crowd, kind="stable")[:P - cum]]]] = True
        break
    return np.flatnonzero(keep), f, g


class EvolutionOpt:
    def __init__(self, lb, ub, acq_fn: Callable[[np.ndarray], np.ndarray], pop: int = 100, iters: int = 100,
                 seed: Optional[int] = None, sbx_eta: float = 15.0, sbx_prob: float = 0.9, sbx_prob_var: float = 0.5,
                 pm_eta: float = 20.0, pm_prob_var: Optional[float] = None):
        self.lb = np.asarray(lb, dtype=np.float64).reshape(-1)
        self.ub = np.asarray(ub, dtype=np.float64).reshape(-1)
        assert self.lb.shape == self.ub.shape and (self.ub > self.lb).all()
        self.d = self.lb.size
        self.acq_fn = acq_fn
        self.pop, self.iters = int(pop), int(iters)
        self.rng = np.random.default_rng(seed)
        self.sbx_eta, self.sbx_prob, self.sbx_prob_var = sbx_eta, sbx_prob, sbx_prob_var
        self.pm_eta = pm_eta
        self.pm_prob_var = min(0.5, 1.0 / self.d) if pm_prob_var is None else pm_prob_var
        self.n_evals = 0

    # ------------------------------------------------------------------ variation operators
    def _sbx(self, P1: np.ndarray, P2: np.ndarray):
        """Simulated binary crossover with bounds (Deb & Agrawal); returns two children per parent pair."""
        rng, eta = self.rng, self.sbx_eta
        n, d = P1.shape
        lo, hi = self.lb[None, :], self.ub[None, :]
        y1, y2 = np.minimum(P1, P2), np.maximum(P1, P2)
        diff = y2 - y1
        do = (rng.random((n, 1)) < self.sbx_prob) & (rng.random((n, d)) < self.sbx_prob_var) & (diff > 1e-14)
        safe = np.where(diff > 1e-14, diff, 1.0)
        u = rng.random((n, d))

        def betaq(beta):
            alpha = 2.0 - np.power(beta, -(eta + 1.0))
            inner = np.where(u <= 1.0 / alpha, u * alpha, 1.0 / np.maximum(2.0 - u * alpha, 1e-300))
            return np.power(inner, 1.0 / (eta + 1.0))
        c1 = 0.5 * ((y1 + y2) - betaq(1.0 + 2.0 * (y1 - lo) / safe) * diff)
        c2 = 0.5 * ((y1 + y2) + betaq(1.0 + 2.0 * (hi - y2) / safe) * diff)
        swap = rng.random((n, d)) < 0.5
        c1, c2 = np.where(swap, c2, c1), np.where(swap, c1, c2)
        C1 = np.where(do, c1, P1)
        C2 = np.where(do, c2, P2)
        return np.clip(C1, lo, hi), np.clip(C2, lo, hi)

    def _pm(self, X: np.ndarray) -> np.ndarray:
        """Polynomial mutation (Deb & Goyal)."""
        rng, eta = self.rng, self.pm_eta
        lo, hi = self.lb[None, :], self.ub[None, :]
        span = hi - lo
        do = rng.random(X.shape) < self.pm_prob_var
        u = rng.random(X.shape)
        d1, d2 = (X - lo) / span, (hi - X) / span
        mp = 1.0 / (eta + 1.0)
        low = np.power(2.0 * u + (1.0 - 2.0 * u) * np.power(1.0 - d1, eta + 1.0), mp) - 1.0
        high = 1.0 - np.power(2.0 * (1.0 - u) + 2.0 * (u - 0.5) * np.power(1.0 - d2, eta + 1.0), mp)
        dq = np.where(u < 0.5, low, high)
        return np.clip(np.where(do, X + dq * span, X), lo, hi)

    def _offspring(self, X: np.ndarray, n_off: int) -> np.ndarray:
        """Random mating until n_off non-duplicate children exist (a bounded number of rounds, like pymoo's infill)."""
        kids = np.zeros((0, self.d))
        for _ in range(10):
            need = n_off - kids.shape[0]
            if need <= 0:
                break
            n_pairs = (need + 1) // 2
            a = self.rng.integers(0, X.shape[0], n_pairs)
            b = self.rng.integers(0, X.shape[0], n_pairs)
            c1, c2 = self._sbx(X[a], X[b])
            new = self._pm(np.concatenate([c1, c2], 0))
            # duplicate elimination against the population, the accepted children and inside the new batch
            ref = np.concatenate([X, kids], 0)
            dup = (np.abs(new[:, None, :] - ref[None, :, :]).max(-1) <= 1e-16).any(1)
            _, first = np.unique(new.round(16), axis=0, return_index=True)
            uniq = np.zeros(new.shape[0], dtype=bool)
            uniq[first] = True
            kids = np.concatenate([kids, new[~dup & uniq]], 0)
        return kids[:n_off]

    # ------------------------------------------------------------------ main loop
    def _eval(self, X: np.ndarray) -> np.ndarray:
        F = np.asarray(self.acq_fn(X.astype(np.float32)), dtype=np.float64).reshape(X.shape[0], -1)
        self.n_evals += X.shape[0]
        return np.where(np.isfinite(F), F, np.inf)

    def optimize(self, initial_suggest: Optional[np.ndarray] = None, return_pop: bool = False) -> np.ndarray:
        X = self.lb + (self.ub - self.lb) * self.rng.random((self.pop, self.d))      # evolution_optimizer.py:44-55 (uniform)
        if initial_suggest is not None:
            init = np.clip(np.asarray(initial_suggest, dtype=np.float64).reshape(-1, self.d), self.lb, self.ub)
            X = np.concatenate([init, X], 0)[: self.pop]                              # :56-57 prepend + truncate
        F = self._eval(X)
        for _ in range(self.iters - 1):                                               # ('n_gen', iters): gen 1 = the initial pop
            kids = self._offspring(X, self.pop)
            if kids.shape[0] == 0:
                break
            Fk = self._eval(kids)
            Xa, Fa = np.concatenate([X, kids], 0), np.concatenate([F, Fk], 0)
            keep = rank_and_crowding_survival(Fa, self.pop)
            X, F = Xa[keep], Fa[keep]
        self.pop_X, self.pop_F = X, F
        if return_pop:
            return X
        nd = fast_non_dominated_sort(F) == 0                                          # res.X: non-dominated members
        return X[nd]


class DeviceNSGA2:
    """The evolutionary acquisition optimiser with the population resident on the GPU (include/hebo_b200.h "device
    NSGA-II"): NSGA-II over the MACE objectives, or the single-objective GA -- as in the reference, the algorithm follows
    from the number of objectives (evolution_optimizer.py:123-124,132-133).

    kinds [D]: 'real' | 'int' | 'choice' per optimisation column (numeric columns first, then the categorical ones:
    evolution_optimizer.py:26-41); lb / ub [D]; fixed: {column index: value} (fix_input, :97-101).  `score(Xc, Xe, gen)`
    returns the objectives of a batch as a device tensor: F [pop, 3] (the fused posterior + MACE call; rank-and-crowding
    survival, hb_nsga2_survive_ex) or one column, F [pop] or [pop, 1] (e.g. hebo_b200.acq.ga_score; fitness survival,
    hb_ga_survive, and the result is the best row).  Any other column count raises ValueError.  2 <= pop <= 16384:
    survival runs in one CTA up to pop 256 and in a cooperative multi-CTA kernel above, with the same results.

    constrained=True: `score` returns (F [pop, 3], G [pop]) with one constraint column (feasible iff G <= 0, the pymoo
    constraint of evolution_optimizer.py:82,105); survival is hb_nsga2_survive_cv and the result is the feasible front
    (hebo_b200.pareto.feasible_front).  The generation loop still never synchronises with the host.  There is no
    constrained single-objective GA: constrained=True with a one-column score raises ValueError."""

    KIND = {"real": 0, "int": 1, "choice": 2}
    MAX_POP = 16384                                 # hb_nsga2_survive_ex: single CTA up to 256, cooperative multi-CTA above

    def __init__(self, kinds, lb, ub, num_numeric: int, score: Callable, pop: int = 100, iters: int = 100,
                 seed: Optional[int] = None, fixed: Optional[dict] = None, device="cuda", constrained: bool = False):
        import torch
        self.torch = torch
        self.D, self.d, self.pop, self.iters = len(kinds), int(num_numeric), int(pop), int(iters)
        if not 2 <= self.pop <= self.MAX_POP:
            raise ValueError(f"DeviceNSGA2: pop must lie in [2, {self.MAX_POP}], got {self.pop}")
        dev = torch.device(device)
        self.dev = dev
        self.kind = torch.tensor([self.KIND[k] for k in kinds], dtype=torch.int32, device=dev)
        self.lb = torch.as_tensor(np.asarray(lb, dtype=np.float32)).to(dev)
        self.ub = torch.as_tensor(np.asarray(ub, dtype=np.float32)).to(dev)
        fx = np.full(self.D, np.nan, dtype=np.float32)
        for k, v in (fixed or {}).items():
            fx[k] = v
        self.fixed = torch.from_numpy(fx).to(dev)
        self.score = score
        self.constrained = bool(constrained)
        self.seed = int(np.random.randint(0, 2 ** 31 - 1)) if seed is None else int(seed)
        self.n_evals = 0
        self.num_obj = None            # set by the first scored batch: 1 (GA) or 3 (NSGA-II)

    def _bufs(self):
        t, dev, P, D, d = self.torch, self.dev, self.pop, self.D, self.d
        return (t.empty(P, D, device=dev), t.empty(P, max(d, 1), device=dev)[:, :d].contiguous() if d else t.empty(P, 0, device=dev),
                t.empty(P, D - d, dtype=t.int32, device=dev))

    def optimize(self, initial_suggest=None, return_pop: bool = False):
        """Returns (Xc [K, d] fp32, Xe [K, e] int32, F [K, 3]) of the non-dominated members of the final population
        (res.X of evolution_optimizer.py:141-149), all on the device; with constraints, of its feasible front.  With a
        one-column score: (Xc [1, d], Xe [1, e], F [1, 1]) of the best member (the first minimum of the sanitised f, which
        after a survival is row 0), res.X of a single-objective run.  return_pop=True with a one-column score: the whole
        final population (Xc [pop, d], Xe [pop, e], F [pop, 1]) in survival order, ascending (sanitised f, row), as res.pop
        of evolution_optimizer.py:148-151; after a survival that is the population's own order."""
        from . import _lib
        from .pareto import feasible_front, pareto_front
        t, lib, P, D, d = self.torch, _lib.lib(), self.pop, self.D, self.d
        st = _lib.stream_ptr
        X, Xc, Xe = self._bufs()
        Xn, Xcn, Xen = self._bufs()
        C, Cc, Ce = self._bufs()
        init = None if initial_suggest is None else t.as_tensor(np.asarray(initial_suggest, dtype=np.float32).reshape(-1, D)).to(self.dev)
        n_init = 0 if init is None else min(init.shape[0], P)
        pc = lambda x: _lib.ptr(x) if x.numel() else None
        ws_bytes = int(lib.hb_nsga2_workspace_bytes(P, D))
        if ws_bytes < 0:
            raise _lib.HeboB200Error(f"hb_nsga2_workspace_bytes: invalid size (pop {P}, D {D})")
        ws = t.empty(ws_bytes, dtype=t.uint8, device=self.dev)       # survival workspace, reused by every generation
        with t.cuda.device(self.dev):
            _lib.check(lib.hb_nsga2_init(_lib.ptr(X), P, D, d, _lib.ptr(self.kind), _lib.ptr(self.lb), _lib.ptr(self.ub), _lib.ptr(self.fixed),
                                         _lib.ptr(init), n_init, self.seed, pc(Xc), pc(Xe), st()), "hb_nsga2_init")
            F, G = self._scored(Xc, Xe, 0)
            Fn = t.empty_like(F)
            Gn = None if G is None else t.empty_like(G)
            self.n_evals = P
            for gen in range(1, self.iters):                       # ('n_gen', iters): generation 1 is the initial population
                _lib.check(lib.hb_nsga2_mate(_lib.ptr(X), P, D, d, _lib.ptr(self.kind), _lib.ptr(self.lb), _lib.ptr(self.ub),
                                             _lib.ptr(self.fixed), self.seed, gen, _lib.ptr(C), pc(Cc), pc(Ce), st()), "hb_nsga2_mate")
                FC, GC = self._scored(Cc, Ce, gen)
                if self.num_obj == 1:
                    _lib.check(lib.hb_ga_survive(_lib.ptr(X), _lib.ptr(F), _lib.ptr(C), _lib.ptr(FC), P, D, d, _lib.ptr(Xn), _lib.ptr(Fn),
                                                 pc(Xcn), pc(Xen), _lib.ptr(ws), ws_bytes, st()), "hb_ga_survive")
                elif G is None:
                    _lib.check(lib.hb_nsga2_survive_ex(_lib.ptr(X), _lib.ptr(F), _lib.ptr(C), _lib.ptr(FC), P, D, d, _lib.ptr(Xn),
                                                       _lib.ptr(Fn), pc(Xcn), pc(Xen), _lib.ptr(ws), ws_bytes, st()), "hb_nsga2_survive_ex")
                else:
                    _lib.check(lib.hb_nsga2_survive_cv(_lib.ptr(X), _lib.ptr(F), _lib.ptr(G), _lib.ptr(C), _lib.ptr(FC), _lib.ptr(GC), P, D,
                                                       d, _lib.ptr(Xn), _lib.ptr(Fn), _lib.ptr(Gn), pc(Xcn), pc(Xen), _lib.ptr(ws),
                                                       ws_bytes, st()), "hb_nsga2_survive_cv")
                    G, Gn = Gn, G
                X, Xn, Xc, Xcn, Xe, Xen, F, Fn = Xn, X, Xcn, Xc, Xen, Xe, Fn, F
                self.n_evals += P
        self.pop_X, self.pop_F, self.pop_G = X, F, G
        if return_pop and self.num_obj != 1:
            raise ValueError("DeviceNSGA2: return_pop=True needs a one-column score")
        if self.num_obj == 1:
            f = t.where(t.isfinite(F), F, t.full_like(F, float("inf")))
            if return_pop:
                idx = t.sort(f, stable=True).indices
                return Xc[idx], Xe[idx], F[idx].reshape(-1, 1)
            idx = t.argmin(f).reshape(1)
            return Xc[idx], Xe[idx], F[idx].reshape(1, 1)
        idx = pareto_front(F) if G is None else feasible_front(F, G)
        return Xc[idx], Xe[idx], F[idx]

    def _scored(self, Xc, Xe, gen):
        """(F [n, 3] or [n], G [n] or None) of a batch, contiguous fp32 on the device."""
        out = self.score(Xc, Xe, gen)
        F, G = out if self.constrained else (out, None)
        F = F.reshape(self.pop, -1)
        if F.shape[1] not in (1, 3):
            raise ValueError(f"DeviceNSGA2: the score must have 1 or 3 columns, got {F.shape[1]}")
        if F.shape[1] == 1 and self.constrained:
            raise ValueError("DeviceNSGA2: constrained=True needs the 3 MACE columns; a one-column score has no constrained GA")
        self.num_obj = F.shape[1]
        F = F.reshape(-1) if self.num_obj == 1 else F
        G = None if G is None else G.reshape(-1).to(self.torch.float32)
        return F.to(self.torch.float32).contiguous(), None if G is None else G.contiguous()
