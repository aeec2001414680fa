"""oracle/rng_oracle.py on its own, CPU only: the Philox4x32-10 restatement against known answers, the uniform
conversion's edge, the exact FMA, and the counter layouts of one suggest(), which must not reuse a Philox block inside
any one entry point."""
import numpy as np
import pytest

from oracle import rng_oracle as R


@pytest.mark.parametrize("counter,key,out", R.KAT)
def test_philox_known_answers(counter, key, out):
    got = R.philox4x32_10(*counter, *key)
    assert [int(x) for x in got] == list(out)
    # vectorised: the same block at every position of an array of counters
    arr = [np.full(5, c, dtype=np.uint64) for c in counter]
    got = R.philox4x32_10(*arr, *key)
    assert all((g == o).all() for g, o in zip(got, out))


def test_seed_is_the_key_low_word_first():
    seed = 0x299F31D0A4093822
    c = (0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344)
    assert [int(x) for x in R.block(seed, *c)] == list(R.KAT[2][2])


def test_uniform_conversion_and_its_u_equal_to_one_edge():
    c = np.array([0, 1, 2 ** 24 - 1, 2 ** 24, 2 ** 31, R.U1_WORD - 1, R.U1_WORD, 0xFFFFFFFF], dtype=np.uint32)
    u = R.uniform(c)
    assert u.dtype == np.float32
    assert u[0] == np.float32(2.0 ** -33) and u[1] == np.float32(1.5 * 2.0 ** -32)
    assert u[-3] < 1.0 and u[-2] == 1.0 and u[-1] == 1.0     # (float)c rounds up to 2^32 from 0xFFFFFF80 on
    assert (u > 0).all() and (np.diff(u.astype(np.float64)) >= 0).all()
    # exactly ((float)c + 0.5f) * 2^-32 with one rounding each: compare with an independent rational evaluation
    from fractions import Fraction
    for ci, ui in zip(c.tolist(), u.tolist()):
        f = float(np.float32(float(ci)))                    # float(int) is exact here; fp32 rounds to nearest even
        s = float(np.float32(Fraction(f) + Fraction(1, 2)))
        assert ui == s * 2.0 ** -32


def test_fma32_is_correctly_rounded():
    rng = np.random.default_rng(1)
    n = 4000
    a = rng.standard_normal(n).astype(np.float32)
    b = rng.random(n).astype(np.float32)
    c = (rng.standard_normal(n) * rng.choice([1e-9, 1.0, 1e9], n)).astype(np.float32)
    # half-way cases: a b + c exactly between two fp32 values, plus or minus a tail below fp64 precision of the sum
    a[:4] = np.float32(1 + 2 ** -23)
    b[:4] = np.float32(1 + 2 ** -23)
    c[:4] = np.float32([1.0, -1.0, 2.0 ** 30, -(2.0 ** 30)])
    f = R.fma32(a, b, c)
    assert all(R.fma32_exact(x, y, z) == r for x, y, z, r in zip(a, b, c, f))


def test_box_muller_bound_is_zero_at_u0_equal_to_one_and_positive_elsewhere():
    z0, z1, r0, r1 = R.box_muller(np.float32([1.0, 0.5, 2.0 ** -33]), np.float32([0.25, 0.125, 0.5]))
    assert z0[0] == 0 and z1[0] == 0 and r0[0] == 0 and r1[0] == 0
    assert z0[2] < -6.7 and abs(z1[2]) < 1e-15                    # sincospif(1) = (0, -1): the exact zero of the sine
    assert (r0[1:] > 0).all() and (r0[1:] < 1e-5 * np.abs(z0[1:]) + 1e-300).all()


def _dup(*layouts):
    """Blocks used more than once among the counters of the given layouts (each a 4-tuple of broadcastable arrays)."""
    a = np.concatenate([np.stack([w.reshape(-1) for w in np.broadcast_arrays(*[np.asarray(x, dtype=np.uint64) for x in c])], 1)
                        for c in layouts]).astype(np.uint32)
    return a.shape[0] - np.unique(np.ascontiguousarray(a).view(np.dtype((np.void, 16))).reshape(-1)).shape[0]


def test_counter_layouts_of_one_suggest_do_not_reuse_a_block():
    """Per entry point and seed, over one suggest(): every Philox block is used once.  Sizes: populations up to 16384, up
    to 4096 + 3 columns at init, generations 1 .. 100, batches of up to 256 rows, candidate ranges with offsets."""
    L = R.LAYOUTS
    # hb_nsga2_init: one call
    for P, D in ((16384, 7), (64, 4099)):
        p, k = np.meshgrid(np.arange(P, dtype=np.uint64), np.arange(0, D, 4, dtype=np.uint64), indexing="ij")
        assert _dup(L["nsga_init"](p, k)) == 0
    # hb_nsga2_mate: generations 1 .. 100 of one run, parent and column blocks together (and apart from init: word 3)
    P, D, G = 100, 300, 100
    t, g, k = np.meshgrid(np.arange((P + 1) // 2, dtype=np.uint64), np.arange(1, G + 1, dtype=np.uint64),
                          np.arange(D, dtype=np.uint64), indexing="ij")
    assert _dup(L["nsga_parents"](t[:, :, 0], g[:, :, 0]), L["nsga_col_v"](t, g, k), L["nsga_col_w"](t, g, k)) == 0
    big = L["nsga_parents"](np.arange(8192, dtype=np.uint64), np.uint64(1))
    assert _dup(big) == 0
    # hb_general_acq_epilogue: m rows x K outputs per generation, counter = generation
    m, K = 2000, 5
    q, c = np.meshgrid(np.arange(0, m * K, 2, dtype=np.uint64), np.arange(1, G + 1, dtype=np.uint64), indexing="ij")
    assert _dup(L["general_acq"](q, c)) == 0
    # hb_sample_y_batch: pairs t < 128 of batches of up to 256 rows, counter = generation
    tt, c = np.meshgrid(np.arange(128, dtype=np.uint64), np.arange(1, G + 1, dtype=np.uint64), indexing="ij")
    assert _dup(L["sample_y_batch"](tt, c)) == 0
    # MACE rows of a candidate set scored in row ranges [row_offset, row_offset + mc) at rng_offset = 0: rows once each
    ranges = [(0, 4096), (4096, 8192), (8192, 10000)]
    r = np.concatenate([np.arange(a, b, dtype=np.uint64) for a, b in ranges])
    assert _dup(L["posterior"](np.uint64(0), r)) == 0 and _dup(L["mace"](r)) == 0
