"""The fp64 GumbelDeepEnsemble oracle (oracle/gumbel_oracle.py) against the reference's own first Adam step
(tests/golden/ref_gumbel_ensemble.npz, make_ref_gumbel_ensemble.py)."""
import pytest
import torch

from oracle import ensemble_oracle as EO
from oracle import gumbel_oracle as GO
from tests.util import load_golden

REF = load_golden("ref_gumbel_ensemble.npz")
INPUTS = [(3, [], "embedding"), (2, [4, 7], "embedding"), (2, [3, 5], "onehot"), (0, [3, 5], "embedding")]
LR, L1, BATCH = 5e-3, 1e-3, 8


def _net(p):
    noise, inp, O, rm, r, prior, N = (int(v) for v in REF[p + "cfg"])
    dc, uniqs, trans = INPUTS[inp]
    return GO.GumbelOracleNet(dc, uniqs, trans, 1, 8, O, bool(noise), bool(prior), reduced_dim=r), dc, uniqs


@pytest.mark.parametrize("vi", range(int(REF["num_variants"])))
def test_fp64_first_step_reproduces_the_reference(vi):
    p = f"v{vi}_"
    for e in range(2):
        net, dc, uniqs = _net(p)
        net.load_raw(REF[p + "init"][e])
        xs = torch.from_numpy(REF[p + "xs_fit"]).double()
        xe = torch.from_numpy(REF[p + "xe_fit"])
        ys = torch.from_numpy(REF[p + "ys_fit"]).double()
        rows = REF[p + "order"][e, 0, :BATCH]
        _, g = GO.gumbel_step_grad(net, xs if dc else None, xe if uniqs else None, ys, rows, REF[p + "draws"][e, 0, 0],
                                   float(REF[p + "temps"][e, 0, 0]), L1, ys.shape[0])
        p0 = torch.from_numpy(REF[p + "init"][e]).double()
        p1, _, _ = EO.adam_update(p0, g, torch.zeros_like(g), torch.zeros_like(g), 1, LR)
        d = (p1 - torch.from_numpy(REF[p + "step1"][e]).double()).abs()
        # a first Adam step moves every parameter with a gradient by lr sign(g): fp32 and fp64 gradients agree on every
        # sign except where the gradient is within rounding of zero (the logits' gradients sum to zero over each row)
        assert float(d.max()) <= 2 * LR
        assert float((d > 1e-6).double().mean()) <= 0.02, float(d.max())
