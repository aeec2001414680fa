"""Parity at the sizes BASELINE.json publishes (VERDICT r1 item 1): mu / sigma / MACE objectives / Pareto front /
argmin-mu / argmax-sigma of the CUDA path against the fp64 oracle rebuilt on the GPU box's host cores, for
    C5 shard shape  n=4096 d=32  (2048 Sobol + 256 near-training + 64 exact-training candidates)
    C3              n=2048 d=32  Kumaraswamy-warped inputs
    C4              n=4096 d=100 heteroscedastic noise_diag
    C2              n=512  d=8   m=4096, Matern-5/2 (full size)
    dense regime    n=4096 d=8   (sigma^2 << s on most rows: the tensor path's precision guard fires)

Criteria (north_star): |d mu| <= 1e-4 max(|mu|, std_y), |d sigma| <= 1e-4 sigma against the fp64 oracle -- plain 1e-4, no
widening by the fp32 floor.  The one exception is written out: rows whose variance has cancelled to sigma^2 < 0.02 s
(candidates ON or within 1e-3 of a training point, where sigma^2 is the residue of s - |L^-1 k*|^2 and inherits the
rounding of the fp32 Cholesky factor itself, ~50 eps s at n = 4096; the reference's own fp32 path, torch CPU potrf + trsm, is
6e-5 .. 8e-5 off the fp64 value on the same rows): hard cap 2e-4, with the fp32-reference error on those rows printed next to
ours.  Every case's numbers are printed, and appended to the file HEBO_PARITY_LOG names when that variable is set."""
import json
import os

import numpy as np
import pytest
import torch

import hebo_b200
from hebo_b200.pareto import pareto_front
from oracle import gp_oracle as O
from tests.util import FULLSIZE_CASES, assert_mace_close, fullsize_inputs, fullsize_oracle

pytestmark = pytest.mark.gpu

CANCEL = 0.02       # sigma^2 / s below which the variance is pure cancellation residue


def _errs(mu, var, ref):
    mu, var = np.asarray(mu, np.float64).reshape(-1), np.asarray(var, np.float64).reshape(-1)
    emu = np.abs(mu - ref["mu"]) / np.maximum(np.abs(ref["mu"]), ref["y_std"])
    esg = np.abs(np.sqrt(var) - np.sqrt(ref["var"])) / np.sqrt(ref["var"])
    return emu, esg


@pytest.mark.parametrize("case", list(FULLSIZE_CASES))
def test_fullsize_parity_vs_fp64_oracle(case):
    c, X, yt, Xs, xi1, xi2, extra = fullsize_inputs(case)
    n, d = c["n"], c["d"]
    np.random.seed(0)
    torch.manual_seed(0)
    gp = hebo_b200.GP(d, 0, 1, kernel=c["kind"], lr=0.01, num_epochs=100, noise_lb=8e-4, pred_likeli=False, **extra)
    gp.fit(X, None, yt)
    assert not gp._fit_failed and np.isfinite(gp.losses).all()
    ref = fullsize_oracle(c, gp, X, yt, Xs, xi1, xi2, extra, torch.float64)
    ref32 = fullsize_oracle(c, gp, X, yt, Xs, xi1, xi2, extra, torch.float32)     # the reference's own precision
    tau, kappa = float(np.float32(ref["tau"])), ref["kappa"]
    F, mu, var = gp.predict_mace(Xs, tau, kappa, 1e-4, xi1, xi2, return_mu_var=True)
    emu, esg = _errs(mu, var, ref)
    fmu, fsg = _errs(ref32["mu"], ref32["var"], ref)
    ratio = ref["var"] / (ref["s"] * ref["y_std"] ** 2)          # sigma^2 / s per row
    reg, can = ratio >= CANCEL, ratio < CANCEL
    rep = dict(case=case, n=n, d=d, m=int(Xs.shape[0]), mu_err=float(emu.max()), sigma_err=float(esg.max()),
               sigma_err_regular=float(esg[reg].max()) if reg.any() else 0.0,
               sigma_err_cancelled=float(esg[can].max()) if can.any() else 0.0, rows_cancelled=int(can.sum()),
               fp32_ref_mu_err=float(fmu.max()), fp32_ref_sigma_err_regular=float(fsg[reg].max()) if reg.any() else 0.0,
               fp32_ref_sigma_err_cancelled=float(fsg[can].max()) if can.any() else 0.0,
               ratio_quantiles=[float(q) for q in np.quantile(ratio, [0.0, 0.01, 0.1, 0.5, 0.9])],
               jitter_used=float(getattr(gp, "jitter_used", 0.0) or 0.0))
    # ---- objectives, front, selections
    mace_err = None
    try:
        assert_mace_close(F.numpy(), ref["F"], ref["mu"], ref["var"], ref["noise"], tau, 1e-4, xi2.numpy(), rtol=5e-4, what=case)
    except AssertionError as e:
        mace_err = str(e)
    rep["mace_ok"] = mace_err is None
    idx = pareto_front(F.cuda()).cpu().numpy()
    assert np.array_equal(idx, O.pareto_front(F.numpy())), "device front != dominance test on the device's own F"
    front64 = O.pareto_front(ref["F"])
    rep["front_size"], rep["front_size_oracle"] = int(idx.size), int(front64.size)
    rep["front_equal"] = bool(np.array_equal(idx, front64))
    rep["front_jaccard"] = float(np.intersect1d(idx, front64).size / max(1, np.union1d(idx, front64).size))
    am, ax = int(np.argmin(mu.numpy()[front64])), int(np.argmax(var.numpy()[front64]))
    rep["argmin_mu_equal"] = am == int(np.argmin(ref["mu"][front64]))
    rep["argmax_sigma_equal"] = ax == int(np.argmax(ref["var"][front64]))
    print(json.dumps(rep))
    log = os.environ.get("HEBO_PARITY_LOG")
    if log:
        with open(log, "a") as fh:
            fh.write(json.dumps(rep) + "\n")
    assert mace_err is None, mace_err
    assert rep["mu_err"] <= 1e-4, rep
    assert rep["sigma_err_regular"] <= 1e-4, rep
    assert rep["sigma_err_cancelled"] <= 2e-4, rep
    assert rep["argmin_mu_equal"] and rep["argmax_sigma_equal"], rep
    assert rep["front_jaccard"] >= 0.9, rep
