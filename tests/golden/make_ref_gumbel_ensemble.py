"""Generates tests/golden/ref_gumbel_ensemble.npz from the reference's own ``GumbelDeepEnsemble``
(models/nn/gumbel_linear.py).

    HEBO_SRC=<checkout of the HEBO sources> python tests/golden/make_ref_gumbel_ensemble.py

The reference files are loaded unmodified by path, as make_ref_fe_deep_ensemble.py loads fe_deep_ensemble.py.  Per variant
(NLL / MSE x {numeric only, mixed with embeddings, one-hot, categorical only} x num_out in {1, 2 with a NaN entry and a NaN
row} x reduced_dim in {default, 1, num_cont with the random prior net}; n = 32 (a multiple of the batch of 8) or 30 (not);
2 members of 8 hidden units, 3 epochs) it records:
  - the data, the scaled rows fit_one received, and each member's initial GumbelNet state_dict;
  - the minibatch order of every epoch (torch.randperm, with torch.seed patched to a fixed seed per call);
  - every uniform the selection layer drew, by wrapping torch.rand inside GumbelSelectionLayer.forward: the training
    draws [E, epochs, steps, r, num_cont], then the eval draws [E, r, num_cont] of the noise estimate's predict and of a
    held-out predict;
  - the temperature each forward used;
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

OUT = os.path.join(HERE, "ref_gumbel_ensemble.npz")
INPUTS = [(3, [], "embedding"), (2, [4, 7], "embedding"), (2, [3, 5], "onehot"), (0, [3, 5], "embedding")]
RMODES = ["default", "one", "full_prior"]
H, E, BATCH, EPOCHS, M_TEST = 8, 2, 8, 3, 24


def _de_generator():
    spec = importlib.util.spec_from_file_location("_make_ref_de", os.path.join(HERE, "make_ref_deep_ensemble.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_gumbel(gen):
    gen.load_deep_ensemble()
    return ref_loader._load("_hebo_ref.models.nn.gumbel_linear", "models/nn/gumbel_linear.py")


class SelectionDraws:
    """Records every torch.rand call GumbelSelectionLayer.forward makes, with the layer's mode and temperature."""

    def __init__(self, gl):
        self.cls, self.rec = gl.GumbelSelectionLayer, []

    def __enter__(self):
        rec, orig = self.rec, self.cls.forward
        self._orig = orig

        def forward(layer, x):
            ru = torch.rand

            def rand(*a, **kw):
                t = ru(*a, **kw)
                rec.append((layer.training, float(layer.temperature), t.clone()))
                return t
            torch.rand = rand
            try:
                return orig(layer, x)
            finally:
                torch.rand = ru
        self.cls.forward = forward
        return self

    def __exit__(self, *exc):
        self.cls.forward = self._orig


def main():
    gen = _de_generator()
    gl = load_gumbel(gen)
    inits = []

    class RecordingNet(gl.GumbelNet):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            inits.append(gen.flat(self.state_dict()))

    out = {}
    variants = list(itertools.product([1, 0], range(len(INPUTS)), [1, 2], range(len(RMODES))))
    for vi, (noise, inp, O, rm) in enumerate(variants):
        dc, uniqs, trans = INPUTS[inp]
        N = 32 if vi % 2 else 30
        Xc, Xe, y = gen.data(dc, uniqs, O, N, 900 + vi)
        Xs, Xes, _ = gen.data(dc, uniqs, O, M_TEST, 1300 + vi)
        conf = dict(num_ensembles=E, num_epochs=EPOCHS, batch_size=BATCH, num_hiddens=H, num_layers=1,
                    output_noise=bool(noise), rand_prior=RMODES[rm] == "full_prior")
        if RMODES[rm] == "one":
            conf["reduced_dim"] = 1
        elif RMODES[rm] == "full_prior" and dc > 0:
            conf["reduced_dim"] = dc
        if uniqs:
            conf.update(num_uniqs=uniqs, enum_trans=trans)
        model = gl.GumbelDeepEnsemble(dc, len(uniqs), O, **conf)
        model.basenet_cls = RecordingNet
        seen = []
        fit_one = model.fit_one

        def recording_fit_one(Xc_, Xe_, y_, idx, **kw):
            seen.append((Xc_.clone(), Xe_.clone(), y_.clone()))
            return fit_one(Xc_, Xe_, y_, idx, **kw)
        model.fit_one = recording_fit_one
        inits.clear()
        xc_in, xe_in = (Xs if dc else None), (Xes if uniqs else None)
        with gen.Recorder(7000 + 1000 * vi) as rec, SelectionDraws(gl) as sd:
            model.fit(Xc if dc else None, Xe if uniqs else None, y)
            with torch.no_grad():
                py, ps2 = model.predict(xc_in, xe_in)
        n = seen[0][2].shape[0]
        nb = -(-n // BATCH)
        r = int(conf.get("reduced_dim", dc // 2 + 1))
        train = [t for t in sd.rec if t[0]]
        ev = [t for t in sd.rec if not t[0]]
        p = f"v{vi}_"
        if dc:
            assert len(train) == E * EPOCHS * nb and len(ev) == 2 * E, (len(train), len(ev))
            out[p + "draws"] = torch.stack([t[2] for t in train]).reshape(E, EPOCHS, nb, r, dc).numpy()
            out[p + "temps"] = np.array([t[1] for t in train], dtype=np.float64).reshape(E, EPOCHS, nb)
            out[p + "noise_draws"] = torch.stack([t[2] for t in ev[:E]]).numpy()
            out[p + "pred_draws"] = torch.stack([t[2] for t in ev[E:]]).numpy()
            out[p + "eval_temp"] = np.array([ev[-1][1]], dtype=np.float64)
        else:
            assert not sd.rec
            out[p + "draws"] = np.zeros((E, EPOCHS, nb, r, 0), np.float32)
            out[p + "temps"] = np.array([0.8 ** ep + 0.1 for ep in range(EPOCHS) for _ in range(nb)] * E).reshape(E, EPOCHS, nb)
            out[p + "noise_draws"] = out[p + "pred_draws"] = np.zeros((E, r, 0), np.float32)
            out[p + "eval_temp"] = np.array([0.8 ** (EPOCHS - 1) + 0.1])
        out[p + "cfg"] = np.array([noise, inp, O, rm, r, int(conf["rand_prior"]), N], dtype=np.int64)
        out[p + "Xc"], out[p + "Xe"], out[p + "y"] = Xc.numpy(), Xe.numpy(), y.numpy()
        out[p + "Xs"], out[p + "Xes"] = Xs.numpy(), Xes.numpy()
        out[p + "xs_fit"], out[p + "xe_fit"], out[p + "ys_fit"] = (seen[0][0].numpy(), seen[0][1].numpy(), seen[0][2].numpy())
        out[p + "init"] = np.stack(inits)
        assert len(rec.orders) == 2 * E * EPOCHS
        out[p + "order"] = torch.stack(rec.orders[0::2]).reshape(E, EPOCHS, -1).numpy()
        out[p + "step1"] = torch.stack(rec.first_step).numpy()
        out[p + "epoch3"] = np.stack([gen.flat(mdl.state_dict()) for mdl in model.models])
        out[p + "py"], out[p + "ps2"], out[p + "noise"] = py.numpy(), ps2.numpy(), model.noise.numpy()
        sc = model.xscaler
        out[p + "x_scale"] = sc.scale_.numpy() if dc else np.zeros(0, np.float32)
        out[p + "x_min"] = sc.min_.numpy() if dc else np.zeros(0, np.float32)
        out[p + "y_mean"] = model.yscaler.mean.reshape(-1).float().numpy()
        out[p + "y_std"] = model.yscaler.std.reshape(-1).float().numpy()
        print(vi, noise, INPUTS[inp], O, RMODES[rm], r, N, flush=True)
    out["num_variants"] = np.array(len(variants))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
