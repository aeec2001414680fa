"""Host restatement of the device random streams and of the NSGA-II init and mating operators.

TEST INFRASTRUCTURE ONLY: a checker, not code under test.  It restates, in numpy:

  * Philox4x32-10 (philox4x32_10, hebo_b200/csrc/common.cuh), vectorised over arrays of counters, pinned by the
    known-answer vectors KAT below;
  * the uniform conversion u = ((float)c + 0.5f) * 2^-32 in numpy float32.  uint32 -> float64 is exact and float64 ->
    float32 rounds to nearest even, as cvt.rn.f32.u32 does; the add is one fp32 rounding and the scaling is exact, so the
    result equals the device's bit for bit.  A word c >= 0xFFFFFF80 gives u = 1 exactly;
  * the counter layout of every consumer (LAYOUTS);
  * Box-Muller in fp64 from the exact fp32 uniforms, with a bound on the device's fp32 error;
  * the init kernel (nsga_init_kernel) exactly, and the mating kernel (nsga_mate_kernel: parent draw, SBX with bounds,
    Deb & Agrawal eta = 15, polynomial mutation, Deb & Goyal eta = 20, Choice crossover and resampling) in fp64 with a
    running error bound, following the kernel's branch structure and taking its own uniforms.

Error bounds.  Each value is carried as a midpoint m and a radius r with |device - m| <= r to first order.  An fp32
operation the device rounds correctly adds u |x| (u = 2^-24); powf, logf and sincospif add E ulp <= 2 E u |x|, with E from
the CUDA C++ Programming Guide's table of single-precision maximum ulp errors (ULP below; sqrtf and division are correctly
rounded as this library is built, without -use_fast_math).  The radius of an input reaches the output through the step's
partial derivative; for the monotone steps (powf, 1 / x, the clamps, rint) the derivative is taken over the whole interval
m +- r, i.e. the step maps the two endpoints.  For a small radius that is the first-order term; near uu * alpha = 2, where
SBX's beta_q = (1 / (2 - uu alpha))^(1/16) turns singular and a fixed ulp tolerance is wrong in both directions, it stays a
bound.  A product adds |a| r_b + |b| r_a + r_a r_b.  An FMA the compiler may contract is covered by the bound of the
separate product and sum.
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

MASK = 0xFFFFFFFF
M0, M1 = 0xD2511F53, 0xCD9E8D57          # Philox4x32 round multipliers
W0, W1 = 0x9E3779B9, 0xBB67AE85          # Weyl key increments

# counter (4 words) / key (2 words) -> block, computed with cuRAND's curand_Philox4x32_10 (curand_philox4x32_x.h) in a
# host build; they agree with Random123's published known-answer test for philox4x32_10
KAT = [
    ((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000),
     (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF), (0xFFFFFFFF, 0xFFFFFFFF),
     (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]

U = 2.0 ** -24                            # fp32 unit roundoff
ULP = dict(powf=4, logf=1, sincospif=1)   # CUDA C++ Programming Guide, single-precision maximum ulp error (full range)
TINY = 2.0 ** -149                        # the ulp of the fp32 subnormals
U1_WORD = 0xFFFFFF80                      # words >= this convert to u = 1.0f

# Counter layouts (word 0, 1, 2, 3); every generator takes `seed` as the 64-bit key (k0 = low, k1 = high word).
#   philox_normal2(seed, row, stream): (row_lo, row_hi, stream_lo, stream_hi) -> z0, z1 from words 0, 1
#   Box-Muller row of each consumer (row, stream):
#     MACE epilogue (hb_mace_epilogue)        (r, 0)
#     fused posterior (hb_posterior_mace_ex)  (rng_offset + r, 0)
#     hb_general_acq_epilogue                 (q >> 1, counter), q = r K + b; element q takes half q & 1
#     hb_sample_y_batch                       ((counter << 7) + t, 0); batch rows 2t, 2t + 1
#   nsga init (hb_nsga2_init):                (p, 0xFFFFFFFF, k, 1), k = 0, 4, 8, ...; column k + j takes word j
#   nsga mate parents (hb_nsga2_mate):        (t, gen, 0xFFFFFFF0, 2); words: pa, pb, do_pair, unused
#   nsga mate column k:                       (t, gen, k, 3) -> v, (t, gen, k, 4) -> w
LAYOUTS = {
    "mace": lambda r: (r & MASK, r >> 32, 0, 0),
    "posterior": lambda rng_offset, r: ((rng_offset + r) & MASK, (rng_offset + r) >> 32, 0, 0),
    "general_acq": lambda q, counter: ((q >> 1) & MASK, (q >> 1) >> 32, counter & MASK, counter >> 32),
    "sample_y_batch": lambda t, counter: (((counter << 7) + t) & MASK, ((counter << 7) + t) >> 32, 0, 0),
    "nsga_init": lambda p, k: (p, MASK, k, 1),
    "nsga_parents": lambda t, gen: (t, gen & MASK, 0xFFFFFFF0, 2),
    "nsga_col_v": lambda t, gen, k: (t, gen & MASK, k, 3),
    "nsga_col_w": lambda t, gen, k: (t, gen & MASK, k, 4),
}


# ---------------------------------------------------------------------------------------------------------------- Philox
def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """The Philox4x32-10 block of counters (c0, c1, c2, c3) under keys (k0, k1): arrays (broadcast) of uint32 words in,
    four uint32 arrays out."""
    c = [np.asarray(x, dtype=np.uint64) & MASK for x in (c0, c1, c2, c3)]
    c = list(np.broadcast_arrays(*c))
    k0 = np.asarray(k0, dtype=np.uint64) & MASK
    k1 = np.asarray(k1, dtype=np.uint64) & MASK
    m0, m1, mask = np.uint64(M0), np.uint64(M1), np.uint64(MASK)
    for _ in range(10):
        p0, p1 = m0 * c[0], m1 * c[2]                 # exact: 32 x 32 -> 64 bits
        hi0, lo0 = p0 >> np.uint64(32), p0 & mask
        hi1, lo1 = p1 >> np.uint64(32), p1 & mask
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0 = (k0 + np.uint64(W0)) & mask
        k1 = (k1 + np.uint64(W1)) & mask
    return tuple(x.astype(np.uint32) for x in c)


def block(seed: int, c0, c1, c2, c3):
    """philox4x32_10 keyed by a 64-bit seed, as the device keys it."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    return philox4x32_10(c0, c1, c2, c3, seed & MASK, seed >> 32)


def uniform(c) -> np.ndarray:
    """((float)c + 0.5f) * 2^-32 in fp32, bit for bit (module docstring)."""
    f = np.asarray(c, dtype=np.uint32).astype(np.float64).astype(np.float32)
    return (f + np.float32(0.5)) * np.float32(2.0 ** -32)


def normal_words(seed: int, row, stream=0):
    """Words 0, 1 of philox_normal2(seed, row, stream)."""
    row = np.asarray(row, dtype=np.uint64)
    stream = np.asarray(stream, dtype=np.uint64)
    w = block(seed, row & np.uint64(MASK), row >> np.uint64(32), stream & np.uint64(MASK), stream >> np.uint64(32))
    return w[0], w[1]


# ---------------------------------------------------------------------------------------------------------------- Box-Muller
def _sincospi64(x):
    """(sin(pi x), cos(pi x)) in fp64 for fp32 x in [0, 2], with the argument reduced exactly (so that the zeros of
    sincospif at x = 0.5, 1, 1.5 are zeros here too)."""
    x = np.asarray(x, dtype=np.float64)
    n = np.rint(2.0 * x)                       # quadrant: x = n / 2 + r, |r| <= 1 / 4, exact in fp64
    r = x - 0.5 * n
    s, c = np.sin(math.pi * r), np.cos(math.pi * r)
    q = n.astype(np.int64) % 4
    sn = np.choose(q, [s, c, -s, -c])
    cs = np.choose(q, [c, -s, -c, s])
    return sn, cs


def box_muller(u0, u1):
    """(z0, z1, r0, r1): the fp64 Box-Muller pair at the fp32 uniforms (u0, u1) and the radii that bound the device's fp32
    evaluation rad = sqrtf(-2 logf(u0)), sincospif(2 u1), z0 = rad cos, z1 = rad sin."""
    u0 = np.asarray(u0, dtype=np.float32).astype(np.float64)
    u1 = np.asarray(u1, dtype=np.float32).astype(np.float64)
    L = np.log(u0)
    eL = 2 * ULP["logf"] * U * np.abs(L)                       # logf; -2 L is exact
    t = -2.0 * L
    rad = np.sqrt(t)
    with np.errstate(divide="ignore", invalid="ignore"):
        e_rad = np.where(rad > 0, 2.0 * eL / (2.0 * rad), 0.0) + U * rad   # d sqrt(t) / dt = 1 / (2 sqrt t); sqrtf
    sn, cs = _sincospi64(2.0 * u1)                              # 2 u1 is exact
    e_sc = 2 * ULP["sincospif"] * U
    z0, z1 = rad * cs, rad * sn
    r0 = np.abs(cs) * e_rad + rad * e_sc * np.abs(cs) + U * np.abs(z0)
    r1 = np.abs(sn) * e_rad + rad * e_sc * np.abs(sn) + U * np.abs(z1)
    return z0, z1, r0, r1


def normals(seed: int, row, stream=0):
    """(z0, z1, r0, r1) of philox_normal2(seed, row, stream) in fp64, with the device error radii."""
    w0, w1 = normal_words(seed, row, stream)
    return box_muller(uniform(w0), uniform(w1))


# ---------------------------------------------------------------------------------------------------------------- fp32 helpers
def f32(x):
    return np.asarray(x, dtype=np.float32)


def fma32(a, b, c) -> np.ndarray:
    """fmaf(a, b, c): a b + c rounded once to fp32.  a b is exact in fp64; the sum's fp64 rounding error e (two-sum) only
    matters when the fp64 sum lies exactly half-way between two fp32 values, and then e decides the side."""
    a, b, c = (np.asarray(x, dtype=np.float32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(np.float32)
    rd = r.astype(np.float64)
    other = np.nextafter(r, np.where(s > rd, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    tie = (rd != s) & (s == 0.5 * (rd + other.astype(np.float64))) & (e != 0)
    if tie.any():
        up = e > 0
        hi, lo = np.maximum(r, other), np.minimum(r, other)
        r = np.where(tie, np.where(up, hi, lo), r)
    return r.astype(np.float32)


F32_OVERFLOW = Fraction(float(np.finfo(np.float32).max)) + Fraction(2) ** 103     # half an ulp above the largest float


def fma32_exact(a: float, b: float, c: float) -> np.float32:
    """fmaf(a, b, c) by rational arithmetic, for checking fma32."""
    v = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    if abs(v) >= F32_OVERFLOW:                # ties to even round the midpoint above the largest float up to inf
        return np.float32(np.inf if v > 0 else -np.inf)
    lo = np.float32(float(v))                 # float(Fraction) rounds correctly to fp64; step to the fp32 neighbours
    cands = [x for x in (np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))) if np.isfinite(x)]
    best = min(cands, key=lambda x: (abs(Fraction(float(x)) - v), int(np.float32(x).view(np.uint32)) & 1))
    return np.float32(best)


# ---------------------------------------------------------------------------------------------------------------- init
def init_reference(P, D, kind, lb, ub, fixed, init, seed):
    """(A, B): the two candidate results of hb_nsga2_init, X [P, D] fp32.  A evaluates lb + (ub - lb) u with a separate
    product and sum, B with one FMA (the compiler may contract either expression); they agree almost everywhere.
    kind / lb / ub / fixed [D], init [n_init, D] or None."""
    kind, lb, ub, fixed = np.asarray(kind), f32(lb), f32(ub), f32(fixed)
    n_init = 0 if init is None else init.shape[0]
    p = np.arange(P, dtype=np.uint64)[:, None]
    kk = np.arange(0, D, 4, dtype=np.uint64)[None, :]
    words = block(seed, p, MASK, kk, 1)
    u = np.stack([uniform(w) for w in words], 2).reshape(P, -1)[:, :D]          # column k + j <- word j of block k
    w = ub - lb
    outs = []
    for fused in (False, True):
        v = fma32(w, u, lb) if fused else (lb + w * u).astype(np.float32)
        n = (ub - lb) + np.float32(1.0)
        cat = np.floor(fma32(n, u, lb) if fused else (lb + n * u).astype(np.float32))
        v = np.where(kind == 2, cat, v).astype(np.float32)
        if n_init:
            v[:n_init] = f32(init)[:n_init]
        outs.append(repair(v, kind, lb, ub, fixed))
    return outs[0], outs[1]


def repair(v, kind, lb, ub, fixed):
    """repair (nsga.cu) in fp32: fixed value, else rint for Integer / Choice, then the clamp to [lb, ub]."""
    v = np.where(kind != 0, np.rint(v), v).astype(np.float32)
    v = np.minimum(np.maximum(v, lb), ub)
    return np.where(np.isnan(fixed), v, fixed).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------- intervals
class Iv:
    """Midpoint m / radius r arrays (fp64): |device - m| <= r."""

    def __init__(self, m, r=0.0):
        self.m = np.asarray(m, dtype=np.float64)
        self.r = np.broadcast_to(np.asarray(r, dtype=np.float64), self.m.shape).copy()

    @property
    def lo(self):
        return self.m - self.r

    @property
    def hi(self):
        return self.m + self.r

    @staticmethod
    def span(lo, hi, err=0.0):
        lo, hi = np.minimum(lo, hi), np.maximum(lo, hi)
        return Iv(0.5 * (lo + hi), 0.5 * (hi - lo) + err)

    def __add__(self, o):
        o = _iv(o)
        m = self.m + o.m
        return Iv(m, self.r + o.r + U * (np.abs(m) + self.r + o.r))

    def __sub__(self, o):
        o = _iv(o)
        m = self.m - o.m
        return Iv(m, self.r + o.r + U * (np.abs(m) + self.r + o.r))

    def __mul__(self, o):
        o = _iv(o)
        m = self.m * o.m
        r = np.abs(self.m) * o.r + np.abs(o.m) * self.r + self.r * o.r
        return Iv(m, r + U * (np.abs(m) + r))

    def scale(self, s):
        """times a power of two: exact"""
        return Iv(self.m * s, self.r * abs(s))

    def mono(self, f, ulps):
        """an increasing or decreasing step f over the interval, plus `ulps` ulp of the device function (0.5: correctly
        rounded)"""
        a, b = f(self.lo), f(self.hi)
        mag = np.maximum(np.abs(a), np.abs(b))
        return Iv.span(a, b, 2 * ulps * U * mag + 2 * ulps * TINY)

    def clamp(self, lo, hi):
        return Iv.span(np.clip(self.lo, lo, hi), np.clip(self.hi, lo, hi))


def _iv(x):
    return x if isinstance(x, Iv) else Iv(x)


def where(c, a, b):
    a, b = _iv(a), _iv(b)
    return Iv(np.where(c, a.m, b.m), np.where(c, a.r, b.r))


def union(a, b):
    return Iv.span(np.minimum(a.lo, b.lo), np.maximum(a.hi, b.hi))


def _div(a: Iv, b: Iv) -> Iv:
    """a / b for b > 0 on its interval, correctly rounded"""
    q = [a.lo / b.lo, a.lo / b.hi, a.hi / b.lo, a.hi / b.hi]
    lo, hi = np.minimum.reduce(q), np.maximum.reduce(q)
    return Iv.span(lo, hi, U * np.maximum(np.abs(lo), np.abs(hi)))


def _pow(x: Iv, y: float) -> Iv:
    """powf(x, y) for x >= 0 (monotone in x), 4 ulp"""
    with np.errstate(divide="ignore", over="ignore"):
        return x.mono(lambda t: np.power(np.maximum(t, 0.0), y), ULP["powf"])


# ---------------------------------------------------------------------------------------------------------------- mating
SBX_ETA, SBX_PROB, SBX_VAR, PM_ETA = 15.0, np.float32(0.9), np.float32(0.5), 20.0
SBX_EX = float(np.float32(1.0) / np.float32(SBX_ETA + 1.0))     # 1 / 16
PM_MP = float(np.float32(1.0) / np.float32(PM_ETA + 1.0))       # fl(1 / 21): the fp32 constant the kernel uses
DEN_FLOOR = float(np.float32(1e-30))


def pm_prob(D: int) -> np.float32:
    return np.minimum(np.float32(0.5), np.float32(1.0) / np.float32(D))


def mate_draws(seed, gen, P, D):
    """The mating kernel's uniforms: parents u [T, 4] and per column v, w [T, D, 4], T = ceil(P / 2) matings."""
    T = (P + 1) // 2
    t = np.arange(T, dtype=np.uint64)
    up = np.stack([uniform(x) for x in block(seed, t, gen & MASK, 0xFFFFFFF0, 2)], 1)
    tt, kk = t[:, None], np.arange(D, dtype=np.uint64)[None, :]
    v = np.stack([uniform(x) for x in block(seed, tt, gen & MASK, kk, 3)], 2)
    w = np.stack([uniform(x) for x in block(seed, tt, gen & MASK, kk, 4)], 2)
    return up, v, w


def mate_reference(X, kind, lb, ub, fixed, seed, gen):
    """The expected hb_nsga2_mate output for population X [P, D] fp32.

    Returns a dict:
      pa, pb, do_pair [T]      the parent draw (exact);
      swap, mut1, mut2 [T, D]  Choice swap and resample decisions, sbx [T, D] (SBX applied), pm1, pm2 (PM applied);
      lo, hi [P, D]            the accepted range of every child element: exact (lo == hi) for copied values, fixed and
                               Choice columns (Choice: the two contraction variants may give lo < hi), otherwise the
                               image of the fp64 reference +- its radius under the kernel's clamps and rint;
      mid, rad [P, D]          the fp64 reference and its radius before the final repair (0 where exact);
      straddle [P, D]          the interval crossed a clamp or a rint half-integer (either side accepted)."""
    X = f32(X)
    P, D = X.shape
    kind, lb, ub, fixed = np.asarray(kind), f32(lb), f32(ub), f32(fixed)
    up, v, w = mate_draws(seed, gen, P, D)
    T = up.shape[0]
    Pf = np.float32(P)
    pa = np.minimum((up[:, 0] * Pf).astype(np.float32).astype(np.int64), P - 1)
    pb = np.minimum((up[:, 1] * Pf).astype(np.float32).astype(np.int64), P - 1)
    do_pair = up[:, 2] < SBX_PROB
    A, B = X[pa], X[pb]
    lo, hi = np.broadcast_to(lb, (T, D)), np.broadcast_to(ub, (T, D))
    pmp = pm_prob(D)
    dp = do_pair[:, None]

    # ---- Choice: uniform crossover, random resampling (floorf of lo + (hi - lo + 1) u, product and sum or one FMA)
    swap = dp & (v[..., 0] < np.float32(0.5))
    c1, c2 = np.where(swap, B, A), np.where(swap, A, B)
    n = (ub - lb) + np.float32(1.0)
    mut1, mut2 = v[..., 1] < pmp, w[..., 1] < pmp
    r1 = [np.floor((lb + n * v[..., 2]).astype(np.float32)), np.floor(fma32(n, v[..., 2], lb))]
    r2 = [np.floor((lb + n * w[..., 2]).astype(np.float32)), np.floor(fma32(n, w[..., 2], lb))]
    ch1 = [np.where(mut1, r, c1) for r in r1]
    ch2 = [np.where(mut2, r, c2) for r in r2]

    # ---- Real / Integer: SBX with bounds
    y1, y2 = np.minimum(A, B), np.maximum(A, B)
    diff32 = (y2 - y1).astype(np.float32)
    sbx = dp & (v[..., 0] < SBX_VAR) & (diff32 > np.float32(1e-14))
    with np.errstate(all="ignore"):
        y1i, y2i = Iv(y1), Iv(y2)
        diff = y2i - y1i
        s = y1i + y2i
        uu = v[..., 1].astype(np.float64)

        def betaq(beta: Iv) -> Iv:
            alpha = Iv(2.0) - _pow(beta, -(SBX_ETA + 1.0))
            x = alpha * uu
            # the device tests uu <= fl(1 / alpha); near uu alpha = 1 it may take either branch (they meet with equal
            # slope there), so an interval that reaches 1 takes the union of both
            near = (x.lo * (1 - 4 * U) <= 1.0) & (x.hi * (1 + 4 * U) >= 1.0)
            den = Iv(2.0) - x               # fmaxf(den, 1e-30f), then 1 / den, from the endpoints
            q_hi, q_lo = 1.0 / np.maximum(den.lo, DEN_FLOOR), 1.0 / np.maximum(den.hi, DEN_FLOOR)
            b2 = Iv.span(q_lo, q_hi, U * q_hi)
            inner = where(x.m <= 1.0, x, b2)
            inner = where(near, union(x, b2), inner)
            return _pow(inner, SBX_EX)

        beta_lo = Iv(1.0) + _div((y1i - lo).scale(2.0), diff)
        beta_hi = Iv(1.0) + _div((Iv(hi) - y2i).scale(2.0), diff)
        a = (s - betaq(beta_lo) * diff).scale(0.5)
        b = (s + betaq(beta_hi) * diff).scale(0.5)
        sw = v[..., 2] < np.float32(0.5)
        a, b = where(sw, b, a), where(sw, a, b)
        x1 = where(sbx, a, Iv(A))
        x2 = where(sbx, b, Iv(B))

        # ---- polynomial mutation
        span32 = (ub - lb).astype(np.float32)
        spn = Iv(hi) - Iv(lo)
        live = np.broadcast_to(span32 > 0, (T, D))

        def pm(x: Iv, um) -> Iv:
            um = um.astype(np.float64)
            d1 = _div(x - lo, spn)
            d2 = _div(Iv(hi) - x, spn)
            q1 = _pow(Iv(1.0) - d1, PM_ETA + 1.0)
            q2 = _pow(Iv(1.0) - d2, PM_ETA + 1.0)
            in1 = Iv(2.0 * um) + Iv(1.0 - 2.0 * um) * q1          # 2 um and 1 - 2 um: exact for um < 1/2
            in2 = Iv(2.0 * (1.0 - um)) + q2 * (2.0 * (um - 0.5))    # 2 (1 - um), 2 (um - 1/2): exact for um >= 1/2
            dq = where(um < 0.5, _pow(in1, PM_MP) - 1.0, Iv(1.0) - _pow(in2, PM_MP))
            return x + dq * spn

        pm1 = live & (v[..., 3] < pmp)
        pm2 = live & (w[..., 3] < pmp)
        x1 = where(live, x1.clamp(lo, hi), x1)
        x2 = where(live, x2.clamp(lo, hi), x2)
        x1 = where(pm1, pm(x1, w[..., 0]), x1)
        x2 = where(pm2, pm(x2, w[..., 1]), x2)

    # ---- repair and the children rows 2t, 2t + 1
    out = {k: np.zeros((P, D)) for k in ("lo", "hi", "mid", "rad")}
    out["straddle"] = np.zeros((P, D), dtype=bool)
    rows1, rows2 = np.arange(T) * 2, np.arange(T) * 2 + 1
    for rows, x, ch in ((rows1, x1, ch1), (rows2, x2, ch2)):
        keep = rows < P
        rows = rows[keep]
        slack = 1e-6 * x.r + 1e-300 * (x.r > 0)          # the reference's own fp64 rounding
        xlo, xhi = x.lo - slack, x.hi + slack
        xlo = np.where(x.r > 0, xlo, x.m)
        xhi = np.where(x.r > 0, xhi, x.m)
        rep = lambda t: np.clip(np.where(kind != 0, np.rint(t), t), lb, ub)
        elo, ehi = rep(xlo), rep(xhi)
        strad = (x.r > 0) & (((kind != 0) & (np.rint(xlo) != np.rint(xhi))) | ((xlo < lb) & (xhi >= lb)) |
                             ((xlo <= ub) & (xhi > ub)))
        clo = np.minimum(rep(ch[0]), rep(ch[1]))
        chi = np.maximum(rep(ch[0]), rep(ch[1]))
        elo = np.where(kind == 2, clo, elo)
        ehi = np.where(kind == 2, chi, ehi)
        fx = ~np.isnan(fixed)
        elo = np.where(fx, fixed, elo)
        ehi = np.where(fx, fixed, ehi)
        out["lo"][rows], out["hi"][rows] = elo[keep], ehi[keep]
        out["mid"][rows], out["rad"][rows] = x.m[keep], np.where(kind == 2, 0.0, x.r)[keep]
        out["straddle"][rows] = (strad & (kind != 2) & ~fx)[keep]
    out.update(pa=pa, pb=pb, do_pair=do_pair, swap=swap, mut1=mut1, mut2=mut2, sbx=sbx, pm1=pm1, pm2=pm2)
    return out


# ---------------------------------------------------------------------------------------------------------------- searches
def find_seeds(counter, word: int, pred, start: int = 0, count: int = 1, batch: int = 1 << 22, limit: int = 1 << 30):
    """Seeds s >= start (ascending) whose block at `counter` (4 words) has word `word` satisfying pred (vectorised over
    seeds): the offline search behind the hard-coded edge seeds of the tests."""
    found = []
    c = counter
    for s0 in range(start, start + limit, batch):
        s = np.arange(s0, s0 + batch, dtype=np.uint64)
        w = block_keys(s, *c)[word]
        hit = np.nonzero(pred(w))[0]
        found.extend(int(s[i]) for i in hit[: count - len(found)])
        if len(found) >= count:
            return found
    return found


def block_keys(seeds, c0, c1, c2, c3):
    seeds = np.asarray(seeds, dtype=np.uint64)
    return philox4x32_10(c0, c1, c2, c3, seeds & np.uint64(MASK), seeds >> np.uint64(32))
