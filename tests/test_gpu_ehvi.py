"""hb_ehvi (hypervolume.cu): one Monte-Carlo EHVI round of GeneralBO's ref_point selection on the device, byte for byte
against the host's exact hypervolume (general.hypervolume) and the host loop of GeneralBO._select."""
import numpy as np
import pytest
import torch

import hebo_b200.general as general
from hebo_b200.general import GeneralBO, expected_hvi, hypervolume
from hebo_b200.space import DesignSpace

pytestmark = pytest.mark.gpu
INF, NAN = float("inf"), float("nan")


def host_round(front, samp, ref):
    """The host loop of GeneralBO._select for one round."""
    base = hypervolume(front, ref)
    n_mc, m, _ = samp.shape
    ehvi = []
    for j in range(m):
        s = samp[:, j]
        hvi = sum(hypervolume(np.vstack([front, s[[k]]]), ref) - base for k in range(n_mc))
        ehvi.append(hvi / n_mc)
    return base, np.array(ehvi, dtype=np.float64)


def assert_same(front, samp, ref, cols=None):
    base, ehvi = expected_hvi(front, samp, ref)
    if cols is not None:
        samp, ehvi = samp[:, cols], ehvi[cols]
    hbase, hehvi = host_round(front, samp, ref)
    assert np.float64(base).tobytes() == np.float64(hbase).tobytes(), (base, hbase)
    assert ehvi.dtype == np.float64 and ehvi.tobytes() == hehvi.tobytes(), np.flatnonzero(ehvi != hehvi)
    return ehvi


def trade_off(rng, n, K, scale=2.0, shift=0.5):
    """n points of a K-objective trade-off (a simplex), all below ref = 1."""
    x = rng.random((n, K))
    return x / x.sum(1, keepdims=True) * scale - shift


FRONT_ROWS = {2: 40, 3: 25, 4: 12, 5: 8, 6: 6, 7: 5, 8: 4}


@pytest.mark.parametrize("K", range(2, 9))
def test_every_number_of_objectives(K):
    rng = np.random.default_rng(K)
    front = trade_off(rng, FRONT_ROWS[K], K)
    samp = trade_off(rng, 10 * 12, K, shift=0.6).reshape(10, 12, K) + 0.05 * rng.normal(size=(10, 12, K))
    ehvi = assert_same(front, samp, np.ones(K))
    assert (ehvi > 0).any()


def edge_case(name, K, rng):
    ref = np.ones(K)
    front = trade_off(rng, 12, K)
    samp = trade_off(rng, 10 * 8, K, shift=0.6).reshape(10, 8, K)
    if name == "empty_front":
        front = np.zeros((0, K))
    elif name == "rows_on_or_above_ref":
        front[0, 0] = 1.0                      # on ref: not strictly below, dropped
        front[1, -1] = 1.5                     # above ref in one coordinate
        front[2] = [NAN] + [0.0] * (K - 1)     # NaN rows drop out too
        samp[0, :4, 0] = 1.0
        samp[1, :4, -1] = 3.0
    elif name == "duplicates_and_last_column_ties":
        front = np.round(front, 1)
        front[3] = front[2]
        front[5, -1] = front[4, -1]
        samp = np.round(samp, 1)
        samp[:, :4] = front[None, 2:6]         # samples equal to front rows
        samp[:, 4:, -1] = front[6, -1]         # samples tying the front's last column
    elif name == "dominated_samples":
        # a front row, or one worse in every coordinate but the last: no new slice, so the HVI is exactly 0 (a sample
        # dominated in general position splits a slice and moves the host's sum by rounding)
        samp = np.broadcast_to(front[rng.integers(0, 12, 8)], (10, 8, K)).copy()
        samp[::2, :, :-1] += 0.1
    elif name == "samples_dominating_the_front":
        samp = front.min(0) - 0.5 - 0.1 * rng.random((10, 8, K))
    elif name == "nan_and_inf_samples":
        samp[0, 0, 0], samp[1, 1, -1], samp[2, 2, 0], samp[3, 3, -1] = NAN, INF, -INF, -INF
        samp[4, 4] = -INF
        samp[:, 5, 0] = NAN
        samp[5, 6, 1] = -0.0
    elif name == "fp32_samples":
        samp = samp.astype(np.float32)
    return front, samp, ref


EDGES = ["empty_front", "rows_on_or_above_ref", "duplicates_and_last_column_ties", "dominated_samples",
         "samples_dominating_the_front", "nan_and_inf_samples", "fp32_samples"]


@pytest.mark.parametrize("name", EDGES)
@pytest.mark.parametrize("K", [2, 3, 4])
def test_edge_cases(K, name):
    front, samp, ref = edge_case(name, K, np.random.default_rng(100 + K))
    ehvi = assert_same(front, samp, ref)
    if name == "dominated_samples":
        assert (ehvi == 0).all()
    if name == "samples_dominating_the_front":
        assert (ehvi > 0).all()
    if name == "empty_front":
        assert expected_hvi(front, samp, ref)[0] == 0.0


@pytest.mark.parametrize("n", [31, 32, 33, 255, 256, 257])
def test_front_sizes_at_warp_and_block_edges(n):
    rng = np.random.default_rng(n)
    front = trade_off(rng, n, 2)
    samp = trade_off(rng, 10 * 24, 2, shift=0.55).reshape(10, 24, 2)
    assert_same(front, samp, np.ones(2))


def test_front_read_from_global_memory():
    """n K 8 bytes beyond the shared-memory staging size (rows above ref still count there); 40 rows stay below ref."""
    rng = np.random.default_rng(9)
    front = np.vstack([trade_off(rng, 40, 2), 2.0 + rng.random((1100, 2))])
    front = front[rng.permutation(front.shape[0])]
    samp = trade_off(rng, 10 * 24, 2, shift=0.55).reshape(10, 24, 2)
    assert_same(front, samp, np.ones(2))


def test_ga_sized_candidate_set():
    """m = 16 384 (the GA's largest population): more items than resident threads; 320 columns are checked on the host."""
    rng = np.random.default_rng(16384)
    m = 16384
    front = trade_off(rng, 20, 2)
    samp = (trade_off(rng, 10 * m, 2, shift=0.55).reshape(10, m, 2)).astype(np.float32)
    cols = np.unique(np.concatenate([np.arange(64), rng.integers(0, m, 192), np.arange(m - 64, m)]))
    assert_same(front, samp, np.ones(2), cols)


class _FixedDraws:
    def __init__(self, draws):
        self.draws = draws

    def sample_y(self, Xc, Xe, n):
        return self.draws


@pytest.mark.parametrize("base", ["gp", "deep_ensemble"])
@pytest.mark.parametrize("K", [2, 3, 4])
def test_select_chooses_the_host_rows(K, base, monkeypatch):
    """GeneralBO._select with ref_point: the device rounds and the host loop pick the same rows under np.random.seed, on
    draws of a fitted MultiTaskModel taken once and fed to both."""
    space = DesignSpace().parse([{"name": f"x{i}", "type": "num", "lb": 0, "ub": 1} for i in range(2)])
    opt = GeneralBO(space, K, 0, rand_sample=1, model_config={"base_model_name": base}, ref_point=np.full(K, 2.0))
    np.random.seed(K)
    torch.manual_seed(K)
    X = space.sample(12)
    x = X[["x0", "x1"]].values
    centres = np.linspace(0, 1, K)
    opt.observe(X, np.stack([(x[:, 0] - c) ** 2 + (x[:, 1] - 1 + c) ** 2 for c in centres], 1))
    model = opt._fit()
    suggest = space.sample(16)
    with torch.no_grad():
        draws = torch.as_tensor(model.sample_y(*space.transform(suggest), 10))
    calls = []
    host_hv = general.hypervolume
    monkeypatch.setattr(general, "hypervolume", lambda Y, r: calls.append(1) or host_hv(Y, r))
    for q in (1, 4, 8):
        picks = {}
        for device in ("cuda", "cpu"):
            opt.device = device
            calls.clear()
            np.random.seed(q)
            picks[device] = list(opt._select(_FixedDraws(draws), suggest, q).index)
            assert (len(calls) == 0) == (device == "cuda")
        assert picks["cuda"] == picks["cpu"], (q, picks)
        assert len(set(picks["cuda"])) == q
