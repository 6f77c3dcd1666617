"""The quantiser / dequantiser at their rounding edges: a plain numpy statement of the arithmetic every stored value
passes through, emulations of the subtly wrong variants a kernel could compute instead, and the witness set
(tests/golden/quant_edges.npz, made by tests/golden/make_quant_edges.py) that tells them apart.

Spec (cachegen_encoder.py:40-61 / cachegen_decoder.py:24-35 of the reference, fp32 ops each rounded):

    sym = rint_half_even( fl32( fl32(x * fl32(MAX / m)) + MAX ) ),   NaN / out of range -> 0
    out = RNE_to_half( fl32( fl32( fl32(sym - MAX) / MAX ) * m ) )

MAX = bins // 2 - 1 (1..15), m = the row's absolute maximum in the input half type.  Every operand below is an
np.float32 array or scalar, so nothing is promoted to float64.

Used by tests/test_quant_edges_cpu.py, tests/test_gpu_quant_edges.py and the fixture generator."""
from __future__ import annotations

import os
from fractions import Fraction

import numpy as np

from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "quant_edges.npz")

DTYPES = (O.DT_BF16, O.DT_FP16)
DT_NAME = ("bf16", "fp16")
MAXES = tuple(range(1, 16))
F32_TINY = np.float32(2.0 ** -126)

# the variants a kernel could compute instead of the spec; a pair (x, m) is a witness of a variant when the variant's
# symbol (quantiser variants) or decoded bits (dequantiser variants, after the spec symbol) differ from the spec's
QUANT_MUTANTS = ("fma", "rcp", "divmul", "half_away", "ftz_in", "ftz_prod")
DEQUANT_MUTANTS = ("ftz_deq_bf16", "ftz_deq_fp16", "trunc_bf16", "trunc_fp16")
MUTANTS = QUANT_MUTANTS + DEQUANT_MUTANTS
MUTANT_DOC = {
    "fma": "x * f + MAX contracted into one fused multiply-add (one rounding)",
    "rcp": "factor MAX * fl(1 / m) instead of fl(MAX / m)",
    "divmul": "fl(fl(x / m) * MAX) instead of fl(x * fl(MAX / m))",
    "half_away": "round half away from zero instead of half to even",
    "ftz_in": "subnormal fp32 inputs (x, m) flushed to zero",
    "ftz_prod": "subnormal fp32 results of the quantiser (factor, product, sum) flushed to zero",
    "ftz_deq_bf16": "subnormal dequantised fp32 value (and maximum) flushed to zero, bf16 output",
    "ftz_deq_fp16": "subnormal dequantised fp32 value (and maximum) flushed to zero, fp16 output",
    "trunc_bf16": "fp32 -> bf16 output conversion truncates instead of rounding to nearest even",
    "trunc_fp16": "fp32 -> fp16 output conversion truncates instead of rounding to nearest even",
}
# kinds of fixture pairs (bit mask: a pair can be several)
K_TIE, K_TIE_NB, K_WITNESS, K_SPECIAL, K_RANDOM = 1, 2, 4, 8, 16
WITNESS_CAP = 256      # witnesses stored per (dtype, MAX, mutant); the scan count records how many exist
RANDOM_PER_MAX = 1500
SEED = 20261016


# ------------------------------------------------------------------------------------------------ conversions
def to_f32(bits, dtype: int) -> np.ndarray:
    b = np.asarray(bits, np.uint16)
    if dtype == O.DT_BF16:
        return (b.astype(np.uint32) << 16).view(np.float32)
    return b.view(np.float16).astype(np.float32)


def from_f32(v, dtype: int) -> np.ndarray:
    """RNE, subnormals kept, NaN stays NaN"""
    v = np.asarray(v, np.float32)
    if dtype == O.DT_BF16:
        return O.f32_to_bf16_bits(v.reshape(-1)).reshape(v.shape)
    with np.errstate(over="ignore", invalid="ignore"):
        return v.astype(np.float16).view(np.uint16)


def flush(v: np.ndarray) -> np.ndarray:
    v = np.asarray(v, np.float32)
    return np.where(np.abs(v) < F32_TINY, np.copysign(np.float32(0), v), v).astype(np.float32)


def is_nan_bits(bits, dtype: int) -> np.ndarray:
    a = np.asarray(bits, np.uint16) & 0x7FFF
    return a > (0x7F80 if dtype == O.DT_BF16 else 0x7C00)


# ------------------------------------------------------------------------------------------------ spec
def _symbols(v: np.ndarray, MAX: int) -> np.ndarray:
    with np.errstate(invalid="ignore"):
        r = np.rint(v)
        ok = np.isfinite(r) & (r >= 0) & (r <= 2 * MAX)
    return np.where(ok, r, 0).astype(np.uint8)


def spec_quant(x_bits, m_bits, MAX: int, dtype: int) -> np.ndarray:
    """uint8 symbols of x (half bits) in rows whose maximum is m (half bits, broadcast against x)"""
    x, m, M = to_f32(x_bits, dtype), to_f32(m_bits, dtype), np.float32(MAX)
    with np.errstate(all="ignore"):
        f = M / m
        v = x * f + M              # two numpy float32 ops: each rounded, never fused
    return _symbols(v, MAX)


def spec_dequant_f32(sym, m_bits, MAX: int, max_dtype: int) -> np.ndarray:
    m, M = to_f32(m_bits, max_dtype), np.float32(MAX)
    with np.errstate(all="ignore"):
        a = np.asarray(sym).astype(np.float32) - M
        b = a / M
        return b * m


def spec_dequant(sym, m_bits, MAX: int, max_dtype: int, out_dtype: int) -> np.ndarray:
    """output half bits of symbols `sym` in rows whose stored maximum is m (bits of max_dtype)"""
    return from_f32(spec_dequant_f32(sym, m_bits, MAX, max_dtype), out_dtype)


def spec_absmax(row_bits) -> np.ndarray:
    """the row maxima as stored in a container: integer max of the magnitude bits over the last axis (for a row with a
    NaN, any NaN is accepted in its place: compare with eq_nan)"""
    return (np.asarray(row_bits, np.uint16) & 0x7FFF).max(axis=-1).astype(np.uint16)


def eq_nan(a, b, dtype: int) -> np.ndarray:
    """element-wise bit equality with every NaN equal to every NaN"""
    a, b = np.asarray(a, np.uint16), np.asarray(b, np.uint16)
    return (a == b) | (is_nan_bits(a, dtype) & is_nan_bits(b, dtype))


# ------------------------------------------------------------------------------------------------ mutants
def _fma_f32(p64: np.ndarray, M: float) -> np.ndarray:
    """fl32(p + M) with ONE rounding, p exact in float64: TwoSum gives the exact error of the float64 sum, which decides
    the direction wherever that sum sits exactly on a float32 midpoint (the only place double rounding can go wrong)"""
    s = p64 + M
    bp = s - M
    e = (p64 - bp) + (M - (s - bp))
    r = s.astype(np.float32)
    u = s.view(np.uint64)
    mid = ((u & np.uint64((1 << 29) - 1)) == np.uint64(1 << 28)) & (e != 0)
    if mid.any():
        i = np.flatnonzero(mid)
        r64 = r[i].astype(np.float64)
        up = (e[i] > 0) & (r64 < s[i])
        dn = (e[i] < 0) & (r64 > s[i])
        r[i[up]] = np.nextafter(r[i[up]], np.float32(np.inf))
        r[i[dn]] = np.nextafter(r[i[dn]], np.float32(-np.inf))
    return r


def trunc_half(v: np.ndarray, dtype: int) -> np.ndarray:
    """fp32 -> half by truncation (round toward zero); NaN stays NaN"""
    v = np.asarray(v, np.float32)
    if dtype == O.DT_BF16:
        r = (v.view(np.uint32) >> 16).astype(np.uint16)
        nan = np.isnan(v)
        r[nan] = from_f32(v[nan], dtype)
        return r
    with np.errstate(over="ignore", invalid="ignore"):
        h = v.astype(np.float16)
        over = np.abs(h.astype(np.float32)) > np.abs(v)
    h[over] = np.nextafter(h[over], np.float16(0))
    return h.view(np.uint16)


def mutant_quant(name: str, x_bits, m_bits, MAX: int, dtype: int) -> np.ndarray:
    x, m, M = to_f32(x_bits, dtype), to_f32(m_bits, dtype), np.float32(MAX)
    with np.errstate(all="ignore"):
        if name == "fma":
            f = M / m
            x, f = np.broadcast_arrays(x, f)
            fin = np.isfinite(f) & np.isfinite(x)
            v = (x * f + M).astype(np.float32)
            v[fin] = _fma_f32(x[fin].astype(np.float64) * f[fin].astype(np.float64), float(MAX))
        elif name == "rcp":
            v = x * (M * (np.float32(1) / m)) + M
        elif name == "divmul":
            v = (x / m) * M + M
        elif name == "half_away":
            v = (x * (M / m) + M).astype(np.float64)
            v = np.copysign(np.floor(np.abs(v) + 0.5), v)
        elif name == "ftz_in":
            v = flush(x) * (M / flush(m)) + M
        elif name == "ftz_prod":
            v = flush(flush(x * flush(M / m)) + M)
        else:
            raise ValueError(name)
    return _symbols(v, MAX)


def mutant_dequant(name: str, sym, m_bits, MAX: int, max_dtype: int) -> np.ndarray:
    """output bits of a dequantiser variant (the output dtype is part of the name)"""
    kind, out = name.rsplit("_", 1)
    out_dt = O.DT_BF16 if out == "bf16" else O.DT_FP16
    if kind == "ftz_deq":
        m, M = flush(to_f32(m_bits, max_dtype)), np.float32(MAX)
        with np.errstate(all="ignore"):
            v = flush(((np.asarray(sym).astype(np.float32) - M) / M) * m)
        return from_f32(v, out_dt)
    if kind == "trunc":
        return trunc_half(spec_dequant_f32(sym, m_bits, MAX, max_dtype), out_dt)
    raise ValueError(name)


def mutant_differs(name: str, x_bits, m_bits, MAX: int, dtype: int) -> np.ndarray:
    """bool per pair: the variant's result differs from the spec's"""
    if name in QUANT_MUTANTS:
        return mutant_quant(name, x_bits, m_bits, MAX, dtype) != spec_quant(x_bits, m_bits, MAX, dtype)
    out_dt = O.DT_BF16 if name.endswith("bf16") else O.DT_FP16
    sym = spec_quant(x_bits, m_bits, MAX, dtype)
    return ~eq_nan(mutant_dequant(name, sym, m_bits, MAX, dtype), spec_dequant(sym, m_bits, MAX, dtype, out_dt), out_dt)


# ------------------------------------------------------------------------------------------------ float64 check
def exact_round(x_bits, m_bits, MAX: int, dtype: int):
    """round_half_even(x * MAX / m + MAX) of the true real value (m finite and nonzero), and whether that value lies
    within 8 fp32 ulps of a half-integer (where the fp32 spec may legitimately round the other way).  float64 is
    within 2^-49 relative of the true value; the pairs closer than that to a half-integer are redone in Fraction."""
    x = to_f32(x_bits, dtype).astype(np.float64)
    m = to_f32(m_bits, dtype).astype(np.float64)
    t = x * MAX / m + MAX
    frac = t - np.floor(t)
    near = np.abs(frac - 0.5) <= np.abs(t) * 2.0 ** -45 + 2.0 ** -60
    r = np.rint(t)
    for i in np.flatnonzero(near):
        q = Fraction(float(x[i])) * MAX / Fraction(float(m[i])) + MAX
        fl = q.numerator // q.denominator
        d = q - fl
        r[i] = fl + (1 if d > Fraction(1, 2) or (d == Fraction(1, 2) and fl % 2) else 0)
    close = np.abs(frac - 0.5) <= 8 * np.abs(t) * 2.0 ** -23 + 2.0 ** -40
    return r, close


# ------------------------------------------------------------------------------------------------ the scan
def finite_max_bits(dtype: int) -> int:
    return 0x7F7F if dtype == O.DT_BF16 else 0x7BFF


def ladder(dtype: int) -> np.ndarray:
    """row maxima of the exhaustive scan: bf16 every normal exponent with mantissas 0x00/0x01/0x40/0x7f (1016); fp16
    every normal exponent with 34 mantissas from 0 to 0x3ff (1020)"""
    if dtype == O.DT_BF16:
        e, mant, sh = np.arange(1, 255), np.array([0x00, 0x01, 0x40, 0x7F]), 7
    else:
        e, sh = np.arange(1, 31), 10
        mant = np.unique(np.concatenate([np.linspace(0, 0x3FF, 32).astype(int), [1, 0x200]]))
    return ((e[:, None] << sh) | mant[None, :]).ravel().astype(np.uint16)


def pairs_of(m_list) -> tuple:
    """every (x, m) with |x| <= m (both signs) for the given finite maxima"""
    m_list = np.asarray(m_list, np.int64)
    n = m_list + 1
    mm = np.repeat(m_list, 2 * n)
    xs = np.concatenate([np.concatenate([np.arange(k + 1), np.arange(k + 1) | 0x8000]) for k in m_list]) \
        if m_list.size else np.zeros(0, np.int64)
    return xs.astype(np.uint16), mm.astype(np.uint16)


def scan_block(dtype: int, MAX: int, m_list):
    """ties (fp32 v == k + 0.5) and per-mutant witnesses among every |x| <= m pair of the maxima m_list:
    (x, m) of the ties, {mutant: (x, m)} of the witnesses"""
    X, Mb = pairs_of(m_list)
    x, m, M = to_f32(X, dtype), to_f32(Mb, dtype), np.float32(MAX)
    with np.errstate(all="ignore"):
        v = x * (M / m) + M
        tie = (v - np.floor(v)) == np.float32(0.5)
    wit = {}
    spec = _symbols(v, MAX)
    for name in QUANT_MUTANTS:
        if name == "ftz_in" and dtype == O.DT_FP16:
            d = np.zeros(X.size, bool)                 # fp16 values are normal fp32 numbers
        else:
            d = mutant_quant(name, X, Mb, MAX, dtype) != spec
        wit[name] = (X[d], Mb[d])
    for name in DEQUANT_MUTANTS:
        out_dt = O.DT_BF16 if name.endswith("bf16") else O.DT_FP16
        d = ~eq_nan(mutant_dequant(name, spec, Mb, MAX, dtype), spec_dequant(spec, Mb, MAX, dtype, out_dt), out_dt)
        wit[name] = (X[d], Mb[d])
    return (X[tie], Mb[tie]), wit


def blocks(ms, budget=3_000_000):
    """split a list of maxima into blocks of at most ~budget pairs"""
    out, cur, n = [], [], 0
    for k in ms:
        cur.append(int(k))
        n += 2 * (int(k) + 1)
        if n >= budget:
            out.append(cur)
            cur, n = [], 0
    if cur:
        out.append(cur)
    return out


def cap_pick(n: int, cap: int = WITNESS_CAP) -> np.ndarray:
    """indices of the stored witnesses among n found ones: all, or `cap` spread evenly"""
    if n <= cap:
        return np.arange(n)
    return np.unique(np.linspace(0, n - 1, cap).round().astype(np.int64))


def tie_neighbours(x, m):
    """the +-1 ulp neighbours (in magnitude, same sign) of the tie x that still satisfy |x| <= m"""
    x, m = np.asarray(x, np.int64), np.asarray(m, np.int64)
    a, s = x & 0x7FFF, x & 0x8000
    up = a + 1 <= m
    dn = a >= 1
    xs = np.concatenate([(s | (a + 1))[up], (s | (a - 1))[dn]])
    ms = np.concatenate([m[up], m[dn]])
    return xs.astype(np.uint16), ms.astype(np.uint16)


# ------------------------------------------------------------------------------------------------ special classes
def smallest_finite_factor_max(dtype: int, MAX: int) -> int:
    """bits of the smallest positive maximum whose factor MAX / m is finite"""
    b = np.arange(1, finite_max_bits(dtype) + 1, dtype=np.uint16)
    with np.errstate(all="ignore"):
        f = np.float32(MAX) / to_f32(b, dtype)
    return int(b[np.isfinite(f)][0])


def random_pairs(dtype: int, MAX: int, n: int = RANDOM_PER_MAX):
    """a seeded sample of |x| <= m pairs, m uniform over the finite nonzero bit patterns"""
    rng = np.random.default_rng([SEED, dtype, MAX])
    m = rng.integers(1, finite_max_bits(dtype) + 1, size=n)
    x = rng.integers(0, m + 1) | (rng.integers(0, 2, size=n) << 15)
    return x.astype(np.uint16), m.astype(np.uint16)


def special_pairs(dtype: int, MAX: int):
    rng = np.random.default_rng([SEED, 1, dtype, MAX])
    xs, ms = [], []

    def nan_max(m):
        return bool(is_nan_bits(m, dtype))

    def add(x, m):
        x = np.atleast_1d(np.asarray(x, np.int64))
        if not nan_max(m):
            x = x[(x & 0x7FFF) <= m]                            # a row's values never exceed its maximum
        xs.append(x)
        ms.append(np.full(x.size, int(m), np.int64))

    def below(m, k):
        """+-m, +-0, +-1 ulp and k random values of magnitude <= m"""
        a = rng.integers(0, m + 1, size=k)
        base = np.unique(np.concatenate([[0, m, max(m - 1, 0), min(1, m)], a]))
        return np.concatenate([base, base | 0x8000])

    lad = ladder(dtype)
    for m in lad[np.linspace(0, lad.size - 1, 64).astype(int)]:
        add([m, m | 0x8000, 0, 0x8000], m)                       # x = +-m, +-0
    add([0x8000], 0)                                            # a -0-only row (maximum +0: factor inf)
    add([0x0000, 0x8000], 0)
    top = finite_max_bits(dtype)
    add(below(top, 200), top)                                   # bf16 3.39e38 / fp16 65504
    mf = smallest_finite_factor_max(dtype, MAX)
    for m in (mf - 1, mf, mf + 1, mf + 2):                      # either side of MAX / m overflowing
        if m >= 1:
            add(pairs_of([m])[0], m)
    if dtype == O.DT_BF16:
        sub = np.arange(0x01, 0x80)
        for m in (mf, mf + 1, mf + 3):                          # subnormal x, smallest maxima with a finite factor
            add(np.concatenate([sub, sub | 0x8000]), m)
        for m in sub:                                           # subnormal maxima
            add(below(int(m), 2), m)
    else:
        for m in np.unique(np.concatenate([[1, 2, 3, 0x3FF, 0x200], rng.integers(1, 0x400, size=40)])):
            add(below(int(m), 6), m)                            # fp16 subnormal maxima
    inf = 0x7F80 if dtype == O.DT_BF16 else 0x7C00
    fin = rng.integers(0, top + 1, size=30)
    add(np.concatenate([[inf, inf | 0x8000, 0, 0x8000, top, top | 0x8000], fin, fin | 0x8000]), inf)
    nans = (0x7FC0, 0x7F81, 0x7FFF, 0x7FA5) if dtype == O.DT_BF16 else (0x7E00, 0x7C01, 0x7FFF, 0x7D55)
    for p in nans:                                              # NaN maxima, several payloads
        add(np.concatenate([[p, p | 0x8000, inf, inf | 0x8000, 0, 0x8000], fin[:10], fin[:10] | 0x8000]), p)
    return np.concatenate(xs).astype(np.uint16), np.concatenate(ms).astype(np.uint16)


# ------------------------------------------------------------------------------------------------ fixture
def load():
    return np.load(FIXTURE)


def fixture_pairs(fx, dtype: int, MAX: int = None):
    """(x, m, MAX, kind, mut) arrays of one dtype's pairs, optionally of one MAX"""
    p = DT_NAME[dtype]
    x, m, mx, kind, mut = (fx[f"{p}/{k}"] for k in ("x", "m", "max", "kind", "mut"))
    if MAX is not None:
        s = mx == MAX
        x, m, mx, kind, mut = x[s], m[s], mx[s], kind[s], mut[s]
    return x, m, mx, kind, mut


# ------------------------------------------------------------------------------------------------ row packing
def row_positions(C: int) -> list:
    """channel positions a row's maximum cycles through: first, last, inside the last (partial) 8-wide vector, inside
    the last (partial) 128-channel tile, and one in the middle"""
    last_vec = ((C - 1) // 8) * 8
    last_tile = ((C - 1) // 128) * 128
    return sorted({0, C - 1, last_vec + (C - 1 - last_vec) // 2, last_tile + (C - 1 - last_tile) // 3, C // 2})


def pack_rows(x, m, C: int, dtype: int, start: int = 0):
    """rows [R, C] (half bits) holding every pair: each row has one maximum m at a position that cycles through
    row_positions(C); its other channels take that m's test values (cycled to fill the row).  The maximum's slot
    holds a test value of magnitude m if there is one (so a -0-only or a -m row stays one), else +m.  Returns the rows
    and their maxima bits."""
    x, m = np.asarray(x, np.uint16), np.asarray(m, np.uint16)
    pos = row_positions(C)
    rows, maxes = [], []
    order = np.argsort(m, kind="stable")
    um, first = np.unique(m[order], return_index=True)
    bounds = list(first) + [m.size]
    r = start
    for i, mb in enumerate(um):
        vals = x[order[bounds[i]: bounds[i + 1]]]
        nan = is_nan_bits(mb, dtype)
        if not nan:
            assert ((vals & 0x7FFF) <= mb).all(), "a test value exceeds its row maximum"
        else:
            assert (~is_nan_bits(vals, dtype) | ((vals & 0x7FFF) == mb)).all()
        tops = vals[(vals & 0x7FFF) == mb]
        rest = vals
        per = C - 1
        nrows = max(1, -(-rest.size // per))
        need = nrows * per
        fill = np.resize(rest, need).reshape(nrows, per)
        for k in range(nrows):
            p = pos[r % len(pos)]
            row = np.empty(C, np.uint16)
            row[:p] = fill[k, :p]
            row[p + 1:] = fill[k, p:]
            row[p] = tops[k % tops.size] if tops.size else mb
            rows.append(row)
            maxes.append(mb)
            r += 1
    return np.stack(rows), np.array(maxes, np.uint16)


def plane_maxes(L: int = 15):
    """MAX of the key and value planes of layer l for key bins 4, 6, ..., 32 and value bins in the reverse order"""
    kb = np.arange(4, 4 + 2 * L, 2, dtype=np.float32)
    vb = kb[::-1].copy()
    return kb, vb, [int(b) // 2 - 1 for b in kb], [int(b) // 2 - 1 for b in vb]


def assemble(rows_by_max: dict, L: int = 15, T: int = None):
    """KV bits [L, 2, T, C] whose key plane l holds the rows of MAX l + 1 and value plane l those of MAX 15 - l (key bins
    4..32, value bins reversed); planes with fewer rows repeat theirs.  Returns (bits, kb, vb)."""
    kb, vb, mk, mv = plane_maxes(L)
    T = T or max(r.shape[0] for r in rows_by_max.values())
    C = next(iter(rows_by_max.values())).shape[1]
    bits = np.empty((L, 2, T, C), np.uint16)
    for l in range(L):
        for kv, M in ((0, mk[l]), (1, mv[l])):
            rws = rows_by_max[M]
            bits[l, kv] = rws[np.arange(T) % rws.shape[0]]
    return bits, kb, vb
