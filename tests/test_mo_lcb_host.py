"""Host side of MOMeanSigmaLCB (hebo_b200/acq.py) and of HEBO's acq_cls / model_name arguments (hebo_b200/suggest.py): the
reference fixture against the fp32 expression, the constructor contract, and the argument checks.  No GPU needed."""
import os

import numpy as np
import pytest
import torch

from hebo_b200 import MACE, MOMeanSigmaLCB
from hebo_b200.suggest import HEBO

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ref_mo_lcb.npz")
SPACE = [{"name": "x0", "type": "num", "lb": -1, "ub": 4.0}, {"name": "x1", "type": "cat", "categories": ["a", "b"]}]


def mo_lcb_fp32(mu, var, noise_sd, xi, kappa, best_y, ps=None):
    """acq.py:116-128 in IEEE fp32, each operation rounded: [m, 3] = (py, -1 * ps, (py - kappa ps) - best_y).  ps defaults
    to the correctly rounded sqrt(var)."""
    f = np.float32
    with np.errstate(invalid="ignore"):
        py = (mu + (f(noise_sd) * xi).astype(f)).astype(f)
        ps = np.sqrt(var).astype(f) if ps is None else ps
        g = ((py - (f(kappa) * ps).astype(f)).astype(f) - f(best_y)).astype(f)
    return np.concatenate([py, -ps, g], 1)


def same_bits(a, b):
    """Equal as fp32 bit patterns, with every NaN taken as equal (the sign and payload of a NaN are not specified)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and np.array_equal(a.view(np.uint32)[~nan], b.view(np.uint32)[~nan])


def test_fixture_is_the_fp32_expression():
    """The reference outputs stored in the fixture are the fp32 expression on the recorded draws, bit for bit, once ps is
    the one the reference took.  That ps is -1 * column 1 exactly; torch's CPU sqrt is off the correctly rounded root by
    one ulp in some rows, and by no more."""
    z = np.load(GOLDEN)
    assert int(z["n_cases"]) >= 6
    kappas, best = set(), set()
    for ci in range(int(z["n_cases"])):
        p = f"c{ci}_"
        m, _ = [int(v) for v in z[p + "meta"]]
        kappa, best_y = float(z[p + "kappa"]), float(z[p + "best_y"])
        noise_sd = z[p + "noise_sd"]
        assert noise_sd.dtype == np.float32 and noise_sd.tobytes() == np.sqrt(z[p + "noise"]).tobytes()
        ps_ref = -z[p + "out"][:, 1:2]
        want = mo_lcb_fp32(z[p + "mu"], z[p + "var"], noise_sd[0], z[p + "xi"], kappa, best_y, ps=ps_ref)
        assert want.shape == (m, 3) and same_bits(want, z[p + "out"]), ci
        with np.errstate(invalid="ignore"):
            ps = np.sqrt(z[p + "var"])
        assert same_bits(np.isnan(ps), np.isnan(ps_ref))
        ok = ~np.isnan(ps)
        assert (np.abs(ps[ok] - ps_ref[ok]) <= np.spacing(ps[ok])).all(), ci
        kappas.add(kappa)
        best.add(np.sign(best_y))
        var = z[p + "var"][:, 0]
        assert (var == 0).any() and ((var > 0) & (var < 1e-38)).any() and (var > 1e29).any() and np.isnan(var).any()
        assert np.signbit(z[p + "out"][var == 0, 1]).all()                     # -1 * +0 is -0
        assert np.isnan(z[p + "mu"]).any()
    assert 2.0 in kappas and len(kappas) >= 4 and min(kappas) < 0
    assert best == {-1.0, 0.0, 1.0}


class _Model:
    def __init__(self, num_out=1):
        self.num_out = num_out
        self.noise = torch.full((num_out,), 0.01)


def test_constructor_contract():
    acq = MOMeanSigmaLCB(_Model(), best_y=0.5)
    assert acq.num_obj == 2 and acq.num_constr == 1 and acq.kappa == 2.0 and acq.best_y == 0.5
    assert MOMeanSigmaLCB(_Model(), best_y=0.0, kappa=3.5).kappa == 3.5
    with pytest.raises(AssertionError):
        MOMeanSigmaLCB(_Model(2), best_y=0.0)


def test_hebo_rejects_parallel_suggestions_without_mace():
    opt = HEBO(SPACE, acq_cls=MOMeanSigmaLCB)
    with pytest.raises(RuntimeError, match="Parallel optimization is supported only for MACE acquisition"):
        opt.suggest(2)                                                        # in the start-up phase too (hebo.py:120-121)
    assert opt.suggest(1).shape == (1, 2)
    assert HEBO(SPACE, acq_cls=MACE).suggest(3).shape == (3, 2)


def test_hebo_model_name_and_mace_only_options():
    assert HEBO(SPACE, model_name="gp").model_name == "gp"
    for name in ("rf", "gpy", "svgp"):
        with pytest.raises(NotImplementedError, match="only 'gp'"):
            HEBO(SPACE, model_name=name)
    with pytest.raises(ValueError):
        HEBO(SPACE, n_refine=2, acq_cls=MOMeanSigmaLCB)
    with pytest.raises(ValueError):
        HEBO(SPACE, acq_cls=MOMeanSigmaLCB, _constraint=lambda xc: xc[:, 0])
    assert HEBO(SPACE, n_refine=2).acq_cls is MACE                          # MACE keeps both
