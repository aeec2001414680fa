"""Generates tests/golden/ref_fe_deep_ensemble.npz from the reference's own ``FeDeepEnsemble``
(models/nn/fe_deep_ensemble.py, fe_layers.py).

    HEBO_SRC=<checkout of the HEBO sources> python tests/golden/make_ref_fe_deep_ensemble.py

The reference files are loaded unmodified by path, as make_ref_deep_ensemble.py loads deep_ensemble.py.  Per variant
(fe_layer in {stg, concrete, hard_concrete} x NLL / MSE x {numeric only, mixed with embeddings, one-hot, categorical only}
x num_out in {1, 2 with a NaN entry and a NaN row}; the random prior net on in half of them; 2 members of 8 hidden units,
batch 8, n = 30, 3 epochs) it records:
  - the data, the scaled rows fit_one received, and each member's initial FeNet state_dict;
  - the minibatch order of every epoch (torch.randperm, with torch.seed patched to a fixed seed per call);
  - every gate draw, by wrapping torch.randn / torch.rand inside the gate layers' get_mask: the training draws
    [E, epochs, steps, B, din], then the eval draws [E, din] of the noise estimate's predict and of a held-out predict;
  - the temperature each training forward used;
  - the parameters after the first Adam step and after 3 epochs, and predict / noise on held-out rows.
Test infrastructure; never imported by hebo_b200/.
"""
from __future__ import annotations

import importlib.util
import itertools
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402

OUT = os.path.join(HERE, "ref_fe_deep_ensemble.npz")
LAYERS = ["stg", "concrete", "hard_concrete"]
INPUTS = [(3, [], "embedding"), (2, [4, 7], "embedding"), (2, [3, 5], "onehot"), (0, [3, 5], "embedding")]
N, H, E, BATCH, EPOCHS, M_TEST = 30, 8, 2, 8, 3, 24


def _de_generator():
    spec = importlib.util.spec_from_file_location("_make_ref_de", os.path.join(HERE, "make_ref_deep_ensemble.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_fe(gen):
    gen.load_deep_ensemble()
    fl = ref_loader._load("_hebo_ref.models.nn.fe_layers", "models/nn/fe_layers.py")
    fe = ref_loader._load("_hebo_ref.models.nn.fe_deep_ensemble", "models/nn/fe_deep_ensemble.py")
    return fl, fe


class GateDraws:
    """Records every torch.randn / torch.rand call a gate's get_mask makes, with the layer's mode and temperature."""

    def __init__(self, fl):
        self.fl, self.rec = fl, []

    def __enter__(self):
        rec = self.rec
        self._orig = {c: c.get_mask for c in (self.fl.StochasticGate, self.fl.ConcreteLayer)}

        def wrap(orig):
            def get_mask(layer, x):
                rn, ru = torch.randn, torch.rand

                def randn(*a, **kw):
                    t = rn(*a, **kw)
                    rec.append((layer.training, float(layer.temperature), t.clone()))
                    return t

                def rand(*a, **kw):
                    t = ru(*a, **kw)
                    rec.append((layer.training, float(layer.temperature), t.clone()))
                    return t
                torch.randn, torch.rand = randn, rand
                try:
                    return orig(layer, x)
                finally:
                    torch.randn, torch.rand = rn, ru
            return get_mask
        for c, f in self._orig.items():
            c.get_mask = wrap(f)
        return self

    def __exit__(self, *exc):
        for c, f in self._orig.items():
            c.get_mask = f


def flat(sd):
    return torch.cat([t.detach().reshape(-1).float() for t in sd.values()]).numpy()


def main():
    gen = _de_generator()
    fl, fe = load_fe(gen)
    inits = []

    class RecordingNet(fe.FeNet):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            inits.append(flat(self.state_dict()))

    out = {}
    variants = list(itertools.product(range(len(LAYERS)), [1, 0], range(len(INPUTS)), [1, 2]))
    for vi, (li, noise, inp, O) in enumerate(variants):
        dc, uniqs, trans = INPUTS[inp]
        prior = (inp + O) % 2
        Xc, Xe, y = gen.data(dc, uniqs, O, N, 300 + vi)
        Xs, Xes, _ = gen.data(dc, uniqs, O, M_TEST, 700 + vi)
        conf = dict(num_ensembles=E, num_epochs=EPOCHS, batch_size=BATCH, num_hiddens=H, num_layers=1,
                    output_noise=bool(noise), rand_prior=bool(prior), fe_layer=LAYERS[li])
        if uniqs:
            conf.update(num_uniqs=uniqs, enum_trans=trans)
        model = fe.FeDeepEnsemble(dc, len(uniqs), O, **conf)
        model.basenet_cls = RecordingNet
        seen = []
        fit_one = model.fit_one

        def recording_fit_one(Xc_, Xe_, y_, idx, **kw):
            seen.append((Xc_.clone(), Xe_.clone(), y_.clone()))
            return fit_one(Xc_, Xe_, y_, idx, **kw)
        model.fit_one = recording_fit_one
        inits.clear()
        xc_in, xe_in = (Xs if dc else None), (Xes if uniqs else None)
        with gen.Recorder(5000 + 1000 * vi) as rec, GateDraws(fl) as gd:
            model.fit(Xc if dc else None, Xe if uniqs else None, y)
            with torch.no_grad():
                py, ps2 = model.predict(xc_in, xe_in)
        n = seen[0][2].shape[0]
        nb = n // BATCH if n > BATCH else 1
        B = min(n, BATCH)
        train = [r for r in gd.rec if r[0]]
        ev = [r for r in gd.rec if not r[0]]
        assert len(train) == E * EPOCHS * nb and len(ev) == 2 * E, (len(train), len(ev))
        p = f"v{vi}_"
        out[p + "cfg"] = np.array([li, noise, inp, O, prior], dtype=np.int64)
        out[p + "Xc"], out[p + "Xe"], out[p + "y"] = Xc.numpy(), Xe.numpy(), y.numpy()
        out[p + "Xs"], out[p + "Xes"] = Xs.numpy(), Xes.numpy()
        out[p + "xs_fit"], out[p + "xe_fit"], out[p + "ys_fit"] = (seen[0][0].numpy(), seen[0][1].numpy(), seen[0][2].numpy())
        out[p + "init"] = np.stack(inits)
        assert len(rec.orders) == 2 * E * EPOCHS
        out[p + "order"] = torch.stack(rec.orders[0::2]).reshape(E, EPOCHS, -1).numpy()
        out[p + "draws"] = torch.stack([r[2] for r in train]).reshape(E, EPOCHS, nb, B, -1).numpy()
        out[p + "temps"] = np.array([r[1] for r in train], dtype=np.float32).reshape(E, EPOCHS, nb)
        out[p + "noise_draws"] = torch.stack([r[2] for r in ev[:E]]).numpy()
        out[p + "pred_draws"] = torch.stack([r[2] for r in ev[E:]]).numpy()
        out[p + "eval_temp"] = np.array([ev[-1][1]], dtype=np.float32)
        out[p + "step1"] = torch.stack(rec.first_step).numpy()
        out[p + "epoch3"] = np.stack([flat(mdl.state_dict()) for mdl in model.models])
        out[p + "py"], out[p + "ps2"], out[p + "noise"] = py.numpy(), ps2.numpy(), model.noise.numpy()
        sc = model.xscaler
        out[p + "x_scale"] = sc.scale_.numpy() if dc else np.zeros(0, np.float32)
        out[p + "x_min"] = sc.min_.numpy() if dc else np.zeros(0, np.float32)
        out[p + "y_mean"] = model.yscaler.mean.reshape(-1).float().numpy()
        out[p + "y_std"] = model.yscaler.std.reshape(-1).float().numpy()
        print(vi, LAYERS[li], noise, INPUTS[inp], O, prior, flush=True)
    out["num_variants"] = np.array(len(variants))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
