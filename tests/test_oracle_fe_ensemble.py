"""The gated-ensemble oracle (oracle/fe_oracle.py) against the reference's own FeDeepEnsemble fits
(tests/golden/ref_fe_deep_ensemble.npz): the fp64 step of fit_one from the reference's initial weights, first
minibatch and draws reproduces the parameters the reference reached after its first Adam step, for every gate; and the
fp32 restatement of hb_fe_fit's step tracks the fp64 gradient."""
import numpy as np
import pytest
import torch

from oracle import ensemble_oracle as EO
from oracle import fe_oracle as FO
from tests.util import load_golden

REF = load_golden("ref_fe_deep_ensemble.npz")
INPUTS = [(3, [], "embedding"), (2, [4, 7], "embedding"), (2, [3, 5], "onehot"), (0, [3, 5], "embedding")]
LR, L1, MASK_REG, BATCH = 5e-3, 1e-3, 0.1, 8


def _net(p, cls=FO.FeOracleNet, **kw):
    li, noise, inp, O, prior = (int(v) for v in REF[p + "cfg"])
    dc, uniqs, trans = INPUTS[inp]
    return cls(dc, uniqs, trans, 1, 8, O, bool(noise), bool(prior), kind=FO.KINDS[li], **kw), dc, uniqs


def _first_batch(p, e):
    xs = torch.from_numpy(REF[p + "xs_fit"]).double()
    xe = torch.from_numpy(REF[p + "xe_fit"])
    ys = torch.from_numpy(REF[p + "ys_fit"]).double()
    rows = REF[p + "order"][e, 0, :BATCH]
    return xs, xe, ys, rows, REF[p + "draws"][e, 0, 0], float(REF[p + "temps"][e, 0, 0])


@pytest.mark.parametrize("vi", range(int(REF["num_variants"])))
def test_fp64_first_step_reproduces_the_reference(vi):
    p = f"v{vi}_"
    for e in range(2):
        net, dc, uniqs = _net(p)
        net.load_raw(REF[p + "init"][e])
        xs, xe, ys, rows, r, T = _first_batch(p, e)
        _, g = FO.fe_step_grad(net, xs if dc else None, xe if uniqs else None, ys, rows, r, T, L1, MASK_REG, ys.shape[0])
        p0 = torch.from_numpy(REF[p + "init"][e]).double()
        p1, _, _ = EO.adam_update(p0, g, torch.zeros_like(g), torch.zeros_like(g), 1, LR)
        ref = torch.from_numpy(REF[p + "step1"][e]).double()
        d = (p1 - ref).abs()
        # a first Adam step moves every parameter with a gradient by lr sign(g): fp32 and fp64 gradients agree on every
        # sign except where the gradient is within rounding of zero
        assert float(d.max()) <= 2 * LR
        assert float((d > 1e-6).double().mean()) <= 0.01, float(d.max())
        gate = slice(net.raw().numel() - net.din, None)
        assert float(d[gate].max()) <= 1e-6, d[gate]          # the gate's step: data term through the mask + penalty


@pytest.mark.parametrize("vi", [vi for vi in range(int(REF["num_variants"]))
                                if int(REF[f"v{vi}_cfg"][0]) == 0 and int(REF[f"v{vi}_cfg"][1]) == 0])
def test_fp32_restatement_tracks_fp64(vi):
    """fe_step_grad32 (stg, MSE, mask_reg = 0) against fe_step_grad per element."""
    p = f"v{vi}_"
    net64, dc, uniqs = _net(p)
    net32, _, _ = _net(p, cls=FO.FeNet32)
    raw = REF[p + "init"][0]
    net64.load_raw(raw)
    xs, xe, ys, rows, r, T = _first_batch(p, 0)
    n = ys.shape[0]
    _, g64 = FO.fe_step_grad(net64, xs if dc else None, xe if uniqs else None, ys, rows, r, T, L1, 0.0, n)
    g32 = FO.fe_step_grad32(net32, np.float32(raw), xs.float().numpy() if dc else None, xe.numpy() if uniqs else None,
                            ys.float().numpy(), rows, n, L1, r, T)
    scale = float(g64.abs().max())
    assert np.allclose(g32, g64.numpy(), rtol=1e-4, atol=1e-5 * scale)
    # the prior net's biases take no gradient at all; biases and the gate take no L1 term
    for name, (o, shape) in net32.slices.items():
        if name.startswith("prior_net") and name.endswith("bias"):
            assert not g32[o:o + int(np.prod(shape))].any()
