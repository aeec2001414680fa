"""The fp32 restatement of hebo_b200/csrc/ensemble.cu (oracle/ensemble_oracle.py, output_noise=False) on the host:
fma32 against exact rationals; the restated fit step against BaseNet's fp64 gradient per element at every shape of
tests/util.py DE_CASES, so the restatement computes BaseNet's mathematics and not only the kernel's; and the comparators
of tests/test_gpu_ensemble_envelope.py against deliberately broken restatements, each of which they must catch."""
import numpy as np
import pytest
import torch

from oracle import ensemble_oracle as EO
from oracle import rng_oracle as R
from tests.util import (DE_CASES, DE_PRED, de_adopt_masks, de_case, de_check_against_fp64, de_initial, de_kink_units,
                        de_predict_case, de_predict_fp64, de_step_grad_bound)

L1, LR = 1e-3, 5e-3


def test_fma32_matches_exact_rationals():
    g = np.random.default_rng(3)
    n = 2000
    cases = {
        "random": (g.standard_normal(n), g.standard_normal(n), g.standard_normal(n) * 10.0 ** g.integers(-8, 8, n)),
        # c = -(a b rounded to fp32) plus a few ulps: the sum cancels to the product's rounding error
        "cancelling": None,
        "subnormal": (g.standard_normal(n) * 1e-20, g.standard_normal(n) * 1e-20, g.standard_normal(n) * 1e-39),
        "overflow": (g.uniform(1, 2, n) * 1.8e19, g.uniform(1, 2, n) * 1.8e19, -g.uniform(0, 1, n) * 3e38),
    }
    a, b = (g.standard_normal(n).astype(np.float32) for _ in range(2))
    c = -(a * b) + (g.integers(-3, 4, n) * np.spacing(a * b)).astype(np.float32)
    cases["cancelling"] = (a, b, c)
    for name, (a, b, c) in cases.items():
        a, b, c = (np.asarray(t, dtype=np.float32) for t in (a, b, c))
        got = EO.fma32(a, b, c)
        want = np.array([R.fma32_exact(x, y, z) for x, y, z in zip(a, b, c)], dtype=np.float32)
        assert EO.mismatches(got, want) == 0, name
        if name == "subnormal":
            assert (np.abs(want) < np.finfo(np.float32).tiny).sum() > n // 4
        if name == "overflow":
            assert np.isinf(want).sum() > n // 10 and np.isfinite(want).sum() > n // 10


def initial(kw, seed, E=1) -> np.ndarray:
    return de_initial(kw, seed, E).numpy()


def step_against_fp64(case, raw=None, seed=2):
    """(restated gradient, fp64 gradient, bound, kink units, hidden units) of one minibatch of the case."""
    kw, Xc, Xe, y = de_case(case)
    n, batch = DE_CASES[case]["n"], DE_CASES[case]["batch"]
    net32, net64 = EO.Net32(**kw), EO.OracleNet(**kw)
    raw = initial(kw, 1)[0] if raw is None else raw
    net64.load_raw(raw)
    B, _ = EO.minibatch_rule(n, batch)
    rows = np.random.default_rng(seed).permutation(n)[:B]
    xc = torch.from_numpy(Xc[rows]).double()
    xe = torch.from_numpy(Xe[rows]).long() if net32.uniqs else None
    with torch.no_grad():
        kinks = de_kink_units(net64, net32, lambda net: net(xc, xe))
    acts32, _, _ = EO.forward32(net32, raw, EO.load_inputs32(net32, raw, Xc[rows], Xe[rows]))
    g32 = EO.step_grad32(net32, raw, Xc, Xe, y, rows, n, L1)
    with de_adopt_masks(net64, kinks, acts32):
        g64, bound = de_step_grad_bound(net64, net32, Xc, Xe, y, rows, L1, n)
    return g32, g64, bound, sum(int(k.sum()) for k in kinks.values()), B * net32.H * net32.L


@pytest.mark.parametrize("case", list(DE_CASES))
def test_restated_step_matches_fp64_per_element(case):
    g32, g64, bound, kinks, units = step_against_fp64(case)
    assert kinks <= units // 20, (kinks, units)            # most units keep a distance to 0 beyond their bound
    err = np.abs(g32.astype(np.float64) - g64)
    assert np.all(err <= bound), f"{int((err > bound).sum())} elements over, worst {float(np.max(err / bound)):.3g} x bound"
    coef = L1 / (DE_CASES[case]["n"] * EO.Net32(**de_case(case)[0]).O)
    data = np.abs(g64) > 10 * coef                          # elements the data gradient dominates, not the L1 term
    assert data.sum() > 0
    print(f"{case}: step gradient error / bound {float(np.max(err / bound)):.3g}, "
          f"where the data term dominates {float(np.max(err[data] / bound[data])):.3g}; kink units {kinks} of {units}")


@pytest.mark.parametrize("case,E", DE_PRED, ids=[f"{c}-E{e}" for c, e in DE_PRED])
def test_restated_predict_matches_fp64_per_element(case, E):
    kw, net, params, Xs, Xe, xm, xa, ym, ys, pick = de_predict_case(case, E)
    got = EO.predict32(net, params, Xs[pick], Xe[pick], xm, xa, ym, ys, grad=True)
    ref, kinks, units = de_predict_fp64(net, params, Xs[pick], Xe[pick], xm, xa, ym, ys)
    de_check_against_fp64(got, ref, kinks, units, f"{case} E={E}")


# ------------------------------------------------------------------------------------------------ teeth
def _fit_outputs(case="holes", E=1):
    kw, Xc, Xe, y = de_case(case)
    c = DE_CASES[case]
    net = EO.Net32(**kw)
    n = c["n"]
    order = np.random.default_rng(4).permutation(n)[None]
    return np.concatenate(EO.fit32(net, initial(kw, 1)[0], Xc, Xe, y, order, LR, L1, c["batch"]))


def _predict_outputs(case="default"):
    kw, Xc, Xe, y = de_case(case, m=17)
    net = EO.Net32(**kw)
    params = initial(kw, 1, E=DE_CASES[case]["E"])
    xm, xa = np.full(net.dc, 0.7, np.float32), np.full(net.dc, 0.1, np.float32)
    return params, lambda p: np.concatenate([a.reshape(-1) for a in EO.predict32(net, p, Xc, Xe, xm, xa, np.float32([0.3]),
                                                                                  np.float32([1.7]), grad=True)])


def _drop_last_k(mp):
    dense = EO.dense32
    mp.setattr(EO, "dense32", lambda x, W, b, relu, add=None: dense(x[:, :-1], W[:, :-1], b, relu, add))


def _wrong_ld(mp):
    dense = EO.dense32

    def bad(x, W, b, relu, add=None):          # rows read with a leading dimension one too long: row p drifts p columns
        B, K = x.shape
        idx = np.minimum(np.arange(B)[:, None] * (K + 1) + np.arange(K)[None, :], B * K - 1)
        return dense(x.reshape(-1)[idx], W, b, relu, add)
    mp.setattr(EO, "dense32", bad)


def _skip_one_mask(mp):
    mask = EO.relu_mask32

    def bad(a, d):                             # hidden unit 0 passes its delta whether or not it is active
        r = mask(a, d)
        r[:, 0] = d[:, 0]
        return r
    mp.setattr(EO, "relu_mask32", bad)


def _category_plus_one(mp):
    scatter = EO.scatter32
    mp.setattr(EO, "scatter32", lambda net, dx, Xe: scatter(net, dx, (Xe + 1) % np.asarray(net.uniqs)))


def _keep_partial(mp):
    mp.setattr(EO, "minibatch_rule", lambda n, batch: (min(n, batch), -(-n // batch)))


STEP_MUTATIONS = {"last-k-term-dropped": _drop_last_k, "wrong-leading-dimension": _wrong_ld,
                  "one-relu-mask-skipped": _skip_one_mask, "embedding-row-to-category+1": _category_plus_one}


@pytest.mark.parametrize("name", list(STEP_MUTATIONS))
def test_mutated_step_is_caught(name, monkeypatch):
    """The GPU file compares the device bit for bit with the restatement; a broken restatement must differ from the
    sound one in some bit of a 1-epoch fit, and its step gradient must leave the fp64 bound."""
    good = _fit_outputs()
    g32, g64, bound, _, _ = step_against_fp64("holes")
    assert np.all(np.abs(g32 - g64) <= bound)
    with monkeypatch.context() as mp:
        STEP_MUTATIONS[name](mp)
        bad = _fit_outputs()
        b32, _, _, _, _ = step_against_fp64("holes")
    assert EO.mismatches(bad, good) > 0
    assert np.any(np.abs(b32 - g64) > bound)


def test_partial_minibatch_kept_is_caught(monkeypatch):
    good = _fit_outputs()
    with monkeypatch.context() as mp:
        _keep_partial(mp)
        bad = _fit_outputs()
    assert EO.mismatches(bad, good) > 0


def test_members_combined_in_reverse_order_are_caught():
    params, run = _predict_outputs()
    assert EO.mismatches(run(params[::-1].copy()), run(params)) > 0
