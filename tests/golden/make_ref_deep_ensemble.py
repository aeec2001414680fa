"""Generates tests/golden/ref_deep_ensemble.npz from the reference's own ``DeepEnsemble`` (models/nn/deep_ensemble.py).

    HEBO_SRC=<checkout of the HEBO sources> python tests/golden/make_ref_deep_ensemble.py

deep_ensemble.py, layers.py, scalers.py, base_model.py and util.py are loaded unmodified by path (oracle/ref_loader.py);
util.py's ``disjoint_set`` import (used only by get_random_graph) is stubbed, and networkx too when it is not installed.
Per variant (NLL / MSE x prior off / on x {numeric only, mixed with embeddings, categorical only, one-hot} x num_out in
{1, 2 with a NaN entry and a NaN row} x num_layers in {1, 2}; 2 members of 8 hidden units, batch 8, n = 30):
  - the data, and the scaled rows fit_one received (recorded by wrapping fit_one);
  - each member's initial state_dict, recorded through the reference's own ``basenet_cls`` key by a subclass of BaseNet;
  - the minibatch order its DataLoader used, recorded by wrapping torch.randperm, with torch.seed patched to a fixed seed;
  - the parameters after the first Adam step (recorded by wrapping torch.optim.Adam.step) and after 3 epochs of fit_one;
  - predict, noise and sample_f of the fitted ensemble on held-out rows, with the scalers' statistics.
It also stores the train and held-out RMSE of default 500-epoch fits (5 members, 128 hidden units) over three seeds at the
shapes of HEBO/test/test_base_model.py (X ~ N(0, 1) [50, 1], y = X^2 + 0.01 N(0, 1)).  Test infrastructure; never imported
by hebo_b200/.
"""
from __future__ import annotations

import importlib.util
import itertools
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ref_deep_ensemble.npz")
INPUTS = [(3, [], "embedding"), (2, [4, 7], "embedding"), (0, [3, 5], "embedding"), (2, [3, 5], "onehot")]
N, H, E, BATCH, EPOCHS, M_TEST = 30, 8, 2, 8, 3, 24


def load_deep_ensemble():
    ref_loader.load_reference()                     # _hebo_ref.models.{scalers, base_model}
    if "_hebo_ref.models.nn" not in sys.modules:
        m = types.ModuleType("_hebo_ref.models.nn")
        m.__path__ = []
        sys.modules["_hebo_ref.models.nn"] = m
    ref_loader._load("_hebo_ref.models.layers", "models/layers.py")
    stubs = [("disjoint_set", ["DisjointSet"])]
    if importlib.util.find_spec("networkx") is None:
        stubs.append(("networkx", []))
    ref_loader.load_file("_hebo_ref.models.util", "models/util.py", stubs=stubs)
    return ref_loader._load("_hebo_ref.models.nn.deep_ensemble", "models/nn/deep_ensemble.py")


def data(dc, uniqs, O, n, seed):
    g = torch.Generator().manual_seed(seed)
    Xc = torch.rand(n, dc, generator=g) * 4 - 1
    Xe = torch.stack([torch.randint(0, u, (n,), generator=g) for u in uniqs], 1) if uniqs else torch.zeros(n, 0).long()
    base = Xc.sum(1, keepdim=True) + (Xe.float().sum(1, keepdim=True) if uniqs else 0)
    y = torch.cat([torch.sin(base + k) for k in range(O)], 1) + 0.05 * torch.randn(n, O, generator=g)
    if O == 2:
        y[1, 0] = float("nan")
        y[4, :] = float("nan")
    return Xc, Xe, y


class Recorder:
    """Patches torch.seed (fixed reseed per call), torch.randperm (records every order) and torch.optim.Adam.step
    (records the parameters after each optimiser's first step) while active."""

    def __init__(self, base_seed):
        self.base_seed, self.calls, self.orders, self.first_step = base_seed, 0, [], []

    def __enter__(self):
        self._seed, self._randperm, self._step = torch.seed, torch.randperm, torch.optim.Adam.step
        rec = self

        def seed():
            s = rec.base_seed + rec.calls
            rec.calls += 1
            torch.manual_seed(s)
            return s

        def randperm(*a, **kw):
            p = rec._randperm(*a, **kw)
            rec.orders.append(p.clone())
            return p

        def step(opt, *a, **kw):
            out = rec._step(opt, *a, **kw)
            if not getattr(opt, "_recorded", False):
                opt._recorded = True
                rec.first_step.append(torch.cat([p.detach().reshape(-1).clone() for g in opt.param_groups for p in g["params"]]))
            return out
        torch.seed, torch.randperm, torch.optim.Adam.step = seed, randperm, step
        return self

    def __exit__(self, *exc):
        torch.seed, torch.randperm, torch.optim.Adam.step = self._seed, self._randperm, self._step


def flat(sd):
    return torch.cat([t.detach().reshape(-1).float() for t in sd.values()]).numpy()


def main():
    de = load_deep_ensemble()
    inits = []

    class RecordingNet(de.BaseNet):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            inits.append(flat(self.state_dict()))

    out = {}
    variants = list(itertools.product([1, 0], [0, 1], range(len(INPUTS)), [1, 2], [1, 2]))
    for vi, (noise, prior, inp, O, L) in enumerate(variants):
        dc, uniqs, trans = INPUTS[inp]
        Xc, Xe, y = data(dc, uniqs, O, N, 100 + vi)
        Xs, Xes, _ = data(dc, uniqs, O, M_TEST, 500 + vi)
        conf = dict(num_ensembles=E, num_epochs=EPOCHS, batch_size=BATCH, num_hiddens=H, num_layers=L, output_noise=bool(noise),
                    rand_prior=bool(prior), basenet_cls=RecordingNet)
        if uniqs:
            conf.update(num_uniqs=uniqs, enum_trans=trans)
        model = de.DeepEnsemble(dc, len(uniqs), O, **conf)
        seen = []
        fit_one = model.fit_one

        def recording_fit_one(Xc_, Xe_, y_, idx, **kw):
            seen.append((Xc_.clone(), Xe_.clone(), y_.clone()))
            return fit_one(Xc_, Xe_, y_, idx, **kw)
        model.fit_one = recording_fit_one
        inits.clear()
        with Recorder(1000 * vi) as rec:
            model.fit(Xc if dc else None, Xe if uniqs else None, y)
        xc_in, xe_in = (Xs if dc else None), (Xes if uniqs else None)
        with torch.no_grad():
            py, ps2 = model.predict(xc_in, xe_in)
            f = [model.sample_f()(xc_in, xe_in) for _ in range(E)]
        p = f"v{vi}_"
        out[p + "cfg"] = np.array([noise, prior, inp, O, L], dtype=np.int64)
        out[p + "Xc"], out[p + "Xe"], out[p + "y"] = Xc.numpy(), Xe.numpy(), y.numpy()
        out[p + "Xs"], out[p + "Xes"] = Xs.numpy(), Xes.numpy()
        out[p + "xs_fit"], out[p + "xe_fit"], out[p + "ys_fit"] = (seen[0][0].numpy(), seen[0][1].numpy(), seen[0][2].numpy())
        out[p + "init"] = np.stack(inits)
        # RandomSampler draws randperm(n) once per epoch and then randperm(n)[:n % n] for the (empty) remainder: every
        # second recorded order is the one the epoch used; the members run one after another
        assert len(rec.orders) == 2 * E * EPOCHS
        out[p + "order"] = torch.stack(rec.orders[0::2]).reshape(E, EPOCHS, -1).numpy()
        out[p + "step1"] = torch.stack(rec.first_step).numpy()
        out[p + "epoch3"] = np.stack([flat(mdl.state_dict()) for mdl in model.models])
        out[p + "py"], out[p + "ps2"], out[p + "noise"] = py.numpy(), ps2.numpy(), model.noise.numpy()
        out[p + "sample_f"] = torch.stack(f).numpy()
        sc = model.xscaler
        out[p + "x_scale"] = sc.scale_.numpy() if dc else np.zeros(0, np.float32)
        out[p + "x_min"] = sc.min_.numpy() if dc else np.zeros(0, np.float32)
        out[p + "y_mean"] = model.yscaler.mean.reshape(-1).float().numpy()
        out[p + "y_std"] = model.yscaler.std.reshape(-1).float().numpy()
        print(vi, noise, prior, INPUTS[inp], O, L, flush=True)
    out["num_variants"] = np.array(len(variants))
    # default 500-epoch fits at test_base_model.py's shapes
    rm = []
    for s in range(3):
        g = torch.Generator().manual_seed(7000 + s)
        X = torch.randn(50, 1, generator=g)
        y = X ** 2 + 0.01 * torch.randn(50, 1, generator=g)
        Xt = torch.randn(200, 1, generator=g).clamp(-1.8, 1.8)
        model = de.DeepEnsemble(1, 0, 1)
        with Recorder(9000 + 100 * s):
            model.fit(X, None, y)
        with torch.no_grad():
            rtr = float(((model.predict(X, None)[0] - y) ** 2).mean().sqrt())
            rte = float(((model.predict(Xt, None)[0] - Xt ** 2) ** 2).mean().sqrt())
        out[f"rmse_X{s}"], out[f"rmse_y{s}"], out[f"rmse_Xt{s}"] = X.numpy(), y.numpy(), Xt.numpy()
        rm.append((rtr, rte))
        print("rmse", s, rtr, rte, flush=True)
    out["rmse_ref"] = np.array(rm)          # [seed, (train, held-out)]
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
