"""The CDF normaliser (a7) and the version-3 stream header at their edges: a plain numpy statement of the arithmetic that
turns a stream's symbol histogram into its 16-bit CDF, an exact restatement in fractions.Fraction, emulations of the
subtly wrong variants a kernel could compute instead, and the deterministic search for the histograms that tell them
apart (stored, with the reference's own CDF rows, in tests/golden/cdf_edges.npz by tests/golden/make_cdf_edges.py).

Spec, from the reference's op chain (cachegen_encoder.py:185-196 process_batch, :95-126 _convert_to_int_and_normalize;
torch-CPU semantics), counts n[0..32] over t tokens:

    p_i    = fl32( fl32(n_i) / fl32(t) )
    cum_i  = p_0 + ... + p_{i-1}        accumulated sequentially in float64 (torch's cumsum of a float32 tensor),
    img_i  = fl32(cum_i)                stored per step; the image never feeds back into the sum
    cdf_i  = int16( rint_half_even( fl32(img_i * 65504) ) + i ),   cdf_0 = 0

The float64 running sum is exact here (at most 32 fp32 terms between 2^-11 and 1 fit 53 bits), so a sum in another order
differs only when it is carried in float32.  No intermediate is subnormal (the smallest is 1 / 1030), so a flush-to-zero
variant is not reachable and is left out.

Used by tests/test_cdf_edges_cpu.py, tests/test_gpu_cdf_edges.py and the fixture generator."""
from __future__ import annotations

import os
from fractions import Fraction

import numpy as np

import quant_edges as Q

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "cdf_edges.npz")

LP = 33
F32_SCALE = np.float32(65504.0)           # 2^16 - (Lp - 1)
TOP_SYMBOL = 30                           # 2 * MAX of a 32-bin plane: the highest symbol a stream can hold
BIG_T = (257, 300, 511, 512, 700, 1030)   # chunk sizes past one group: cdf_kernel's domain (fl32(n / t) beyond the table)

# what a kernel could compute instead of the spec; each has the spec's signature (counts, t)
VARIANTS = ("f32sum", "f32sum_rev", "f32sum_pair", "int_prefix", "p_double", "rcp", "mul_double", "no_image",
            "half_away", "trunc", "fma")
VARIANT_DOC = {
    "f32sum": "running sum carried in float32",
    "f32sum_rev": "float32 sum of each prefix taken from its last term down to its first",
    "f32sum_pair": "float32 sum of each prefix as a balanced tree",
    "int_prefix": "fl32(N_i / t) of the integer prefix count N_i: the sum rounded to fp32 only at the end",
    "p_double": "p_i = n_i / t in float64, never rounded to fp32 before the sum",
    "rcp": "p_i = n_i * fl32(1 / t) instead of fl32(n_i / t)",
    "mul_double": "img * 65504 in float64, rounded once by rint",
    "no_image": "the float64 sum times 65504 in float64: no fp32 image, one rounding",
    "half_away": "round half away from zero instead of half to even",
    "trunc": "truncate instead of round",
    "fma": "fma(img, 65504, i): the multiply and the + i rounded to fp32 once",
}
# kinds of fixture rows
K_TIE, K_TIE_NB, K_WITNESS, K_DIRECTED = 1, 2, 4, 8
# search domains
D_TWO, D_THREE, D_MANY, D_BIG = 0, 1, 2, 3
DOMAINS = ("two-part t<=256", "three-part t<=256", "many-symbol t<=256", "t>256")
WITNESS_T = 6          # distinct t kept per (variant, domain), spread over the t that have a witness
WITNESS_PER_T = 3      # rows kept per such t


# ------------------------------------------------------------------------------------------------ spec and variants
def wrap16(v) -> np.ndarray:
    return (np.asarray(v, np.int64) & 0xFFFF).astype(np.uint16).view(np.int16)


def _tree(a: np.ndarray) -> np.ndarray:
    w = a.shape[-1]
    if w == 0:
        return np.zeros(a.shape[:-1], np.float32)
    if w == 1:
        return a[..., 0]
    return _tree(a[..., : w // 2]) + _tree(a[..., w // 2:])


def _images(name: str, c: np.ndarray, t) -> np.ndarray:
    """cdf_f[0..W]: the value the scale multiplies, float32 (float64 for no_image)"""
    W = c.shape[-1]
    tf, td = np.asarray(t, np.float32), np.asarray(t, np.float64)
    if tf.ndim:
        tf, td = tf[..., None], td[..., None]
    n32 = c.astype(np.float32)
    p = n32 * (np.float32(1) / tf) if name == "rcp" else n32 / tf
    assert p.dtype == np.float32
    img = np.zeros(c.shape[:-1] + (W + 1,), np.float64 if name == "no_image" else np.float32)
    if name == "f32sum":
        s = np.zeros(c.shape[:-1], np.float32)
        for i in range(W):
            s = s + p[..., i]
            img[..., i + 1] = s
    elif name == "f32sum_rev":
        for i in range(1, W + 1):
            s = np.zeros(c.shape[:-1], np.float32)
            for k in range(i - 1, -1, -1):
                s = s + p[..., k]
            img[..., i] = s
    elif name == "f32sum_pair":
        for i in range(1, W + 1):
            img[..., i] = _tree(p[..., :i])
    elif name == "int_prefix":
        img[..., 1:] = np.cumsum(c.astype(np.int64), axis=-1).astype(np.float32) / tf
    elif name == "p_double":
        img[..., 1:] = np.cumsum(c.astype(np.float64) / td, axis=-1).astype(np.float32)
    elif name == "no_image":
        img[..., 1:] = np.cumsum(p.astype(np.float64), axis=-1)
    else:
        cum = np.zeros(c.shape[:-1], np.float64)
        for i in range(W):
            cum = cum + p[..., i].astype(np.float64)
            img[..., i + 1] = cum.astype(np.float32)
    return img


def cdf_values(name: str, counts, t, idx=None) -> np.ndarray:
    """int64 [..., W + 1] unwrapped CDF entries of `name` ("spec" or one of VARIANTS).  counts [..., W] are the counts of
    consecutive absorbing steps; idx [W + 1] the entry index added to each (default 0..W: W = 32 symbols in place);
    t a scalar or one value per row."""
    c = np.asarray(counts)
    idx = np.arange(c.shape[-1] + 1) if idx is None else np.asarray(idx)
    img = _images(name, c, t)
    if name in ("mul_double", "no_image"):
        r = np.rint(img.astype(np.float64) * 65504.0)
    elif name == "fma":
        # the exact product (24 x 16 bits) plus i is exact in float64: one rounding to fp32
        return np.rint((img.astype(np.float64) * 65504.0 + idx).astype(np.float32)).astype(np.int64)
    else:
        v = img * F32_SCALE
        assert v.dtype == np.float32
        if name == "half_away":
            r = np.floor(v.astype(np.float64) + 0.5)
        elif name == "trunc":
            r = np.floor(v)
        else:
            r = np.rint(v)
    return r.astype(np.int64) + idx


def spec_cdf(counts, t) -> np.ndarray:
    """counts [..., 33] over t tokens -> int16 [..., 33], the reference's CDF tensor"""
    return wrap16(cdf_values("spec", _steps(counts), t))


def _steps(counts) -> np.ndarray:
    """the 32 counts that entries 0..32 absorb (entry i sums the symbols below i; the count of symbol 32 is never used)"""
    c = np.asarray(counts)
    assert c.shape[-1] == LP
    return c[..., :LP - 1]


def variant_cdf(name: str, counts, t) -> np.ndarray:
    return wrap16(cdf_values(name, _steps(counts), t))


def tie_entries(counts, t):
    """(tie, odd) bool [..., W + 1]: fl32(img_i * 65504) lies exactly on k + 0.5; odd: k is odd (the tie rounds up)"""
    v = _images("spec", np.asarray(counts), t) * F32_SCALE
    fl = np.floor(v)
    tie = (v - fl) == np.float32(0.5)
    return tie, tie & (np.mod(fl, 2) == 1)


def variant_tags(counts, t) -> np.ndarray:
    """uint32 per row: bit k set <=> VARIANTS[k] differs from the spec somewhere in the row"""
    spec = cdf_values("spec", _steps(counts), t)
    tags = np.zeros(spec.shape[:-1], np.uint32)
    for k, name in enumerate(VARIANTS):
        tags |= (cdf_values(name, _steps(counts), t) != spec).any(axis=-1).astype(np.uint32) << np.uint32(k)
    return tags


# ------------------------------------------------------------------------------------------------ the exact form
def _rne_f32(q: Fraction) -> Fraction:
    """q >= 0 rounded to the nearest float32 (half to even); normal range only"""
    if q == 0:
        return q
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if Fraction(2) ** e > q:
        e -= 1
    assert Fraction(2) ** e <= q < Fraction(2) ** (e + 1) and -126 <= e <= 127
    ulp = Fraction(2) ** (e - 23)
    m = q / ulp
    fl = m.numerator // m.denominator
    d = m - fl
    if d > Fraction(1, 2) or (d == Fraction(1, 2) and fl % 2):
        fl += 1
    return fl * ulp


def fraction_cdf(counts_row, t: int):
    """the spec evaluated in exact rationals, every rounding spelled out: (unwrapped entries [33], indices of the exact
    ties).  Nothing here can round except _rne_f32."""
    cum, out, ties = Fraction(0), [], []
    assert len(counts_row) == LP
    for i, n in enumerate(counts_row):
        v = _rne_f32(_rne_f32(cum) * 65504)
        fl = v.numerator // v.denominator
        d = v - fl
        if d == Fraction(1, 2):
            ties.append(i)
        out.append(fl + (1 if d > Fraction(1, 2) or (d == Fraction(1, 2) and fl % 2) else 0) + i)
        cum += _rne_f32(Fraction(int(n), int(t)))
    return out, ties


# ------------------------------------------------------------------------------------------------ placing parts
def place(parts, pattern: int) -> np.ndarray:
    """a histogram [33] whose nonzero counts are `parts`, in order, at symbols chosen by the pattern: 0 the first
    symbols, 1 the last ones of a 32-bin plane (.., 29, 30), 2 spread evenly from 0 to an even top symbol that cycles
    with the number of parts, 3 adjacent in the middle.  Positions matter only through + i and through what the header
    and the lanes' common skip mask see."""
    parts = [int(x) for x in parts]
    K = len(parts)
    assert 1 <= K <= TOP_SYMBOL + 1 and all(x > 0 for x in parts)
    if pattern % 4 == 0:
        pos = np.arange(K)
    elif pattern % 4 == 1:
        pos = np.arange(TOP_SYMBOL + 1 - K, TOP_SYMBOL + 1)
    elif pattern % 4 == 2:
        lo = K - 1 + ((K - 1) & 1)
        lo = max(lo, 2)
        tops = list(range(lo, TOP_SYMBOL + 1, 2)) or [TOP_SYMBOL]
        top = tops[(pattern // 4 + K) % len(tops)]
        pos = np.round(np.linspace(0, top, K)).astype(int) if K > 1 else np.array([top])
    else:
        start = max(0, (TOP_SYMBOL + 1 - K) // 2)
        pos = np.arange(start, start + K)
    assert np.unique(pos).size == K and pos.max() <= TOP_SYMBOL
    row = np.zeros(LP, np.uint16)
    row[pos] = parts
    return row


# ------------------------------------------------------------------------------------------------ the search
class _Collector:
    """per variant: how many witnesses a domain's search met, and a bounded, evenly spread choice of them"""

    def __init__(self):
        self.found = np.zeros(len(VARIANTS), np.int64)
        self.ties = 0
        self.cand = {k: {} for k in range(len(VARIANTS))}     # variant -> {t: [parts, ...]}
        self.rows, self.ts, self.kinds = [], [], []

    def witnesses(self, k: int, t: int, parts: np.ndarray):
        """parts [M, K]: every witness of variant k at this t, in search order"""
        self.found[k] += parts.shape[0]
        if parts.shape[0]:
            sel = np.unique(np.linspace(0, parts.shape[0] - 1, WITNESS_PER_T).round().astype(int))
            self.cand[k].setdefault(int(t), []).extend(parts[sel].tolist())

    def add(self, row, t, kind):
        self.rows.append(np.asarray(row, np.uint16))
        self.ts.append(int(t))
        self.kinds.append(kind)

    def finish(self):
        n = 0
        for k in range(len(VARIANTS)):
            ts = sorted(self.cand[k])
            keep = [ts[i] for i in np.unique(np.linspace(0, len(ts) - 1, WITNESS_T).round().astype(int))] if ts else []
            for t in keep:
                for parts in self.cand[k][t][:WITNESS_PER_T]:
                    parts = [x for x in parts if x > 0]
                    # + i matters to the fused multiply-add alone: its witnesses stay where the search saw them
                    self.add(place(parts, 0 if VARIANTS[k] == "fma" else n), t, K_WITNESS)
                    n += 1
        rows = np.stack(self.rows) if self.rows else np.zeros((0, LP), np.uint16)
        return rows, np.array(self.ts, np.int32), np.array(self.kinds, np.uint8), self.found, self.ties


def _scan(col: _Collector, parts: np.ndarray, t: int):
    """parts [M, K] (zero parts allowed: they absorb nothing) at token count t: count and collect the witnesses of every
    variant (entries taken where the first-symbols placement puts them); returns the tie masks"""
    idx = np.arange(parts.shape[1] + 1)
    spec = cdf_values("spec", parts, t, idx)
    for k, name in enumerate(VARIANTS):
        d = (cdf_values(name, parts, t, idx) != spec).any(axis=-1)
        col.witnesses(k, t, parts[d])
    return tie_entries(parts, t)


def search_two(ts=range(1, 257)):
    """every histogram (n, t - n), 0 <= n < t (n = 0: a lone symbol): all exact ties are kept with their n +- 1
    neighbours, at three placements in turn"""
    col = _Collector()
    k = 0
    for t in ts:
        n = np.arange(0, t)
        parts = np.stack([n, t - n], axis=1)
        tie, odd = _scan(col, parts, t)
        for i in np.flatnonzero(tie.any(axis=1)):
            col.ties += 1
            col.add(place([x for x in parts[i] if x], k), t, K_TIE)
            for j in (i - 1, i + 1):
                if 0 < j < t:
                    col.add(place(parts[j], k), t, K_TIE_NB)
            k += 1
    return col.finish()


def _three_parts(t: int) -> np.ndarray:
    a = np.arange(1, t - 1)
    reps = t - 1 - a
    A = np.repeat(a, reps)
    B = np.concatenate([np.arange(1, r + 1) for r in reps]) if a.size else np.zeros(0, np.int64)
    return np.stack([A, B, t - A - B], axis=1)


def search_three(ts=range(3, 257), tie_cap=2):
    """every composition a + b + c = t into positive parts; of the ties, those at the second prefix (a + b) that the
    first prefix does not already show, at most tie_cap per t"""
    col = _Collector()
    k = 0
    for t in ts:
        parts = _three_parts(t)
        tie, odd = _scan(col, parts, t)
        col.ties += int(tie.any(axis=1).sum())
        second = np.flatnonzero(tie[:, 2] & ~tie[:, 1])
        for i in second[np.unique(np.linspace(0, second.size - 1, tie_cap).round().astype(int))] if second.size else []:
            col.add(place(parts[i], k), t, K_TIE)
            k += 1
    return col.finish()


def many_symbol_parts(t: int) -> np.ndarray:
    """directed many-symbol histograms of t tokens, as rows of 31 parts (zero padded): K near-equal counts, one heavy
    symbol (first, middle, last) among 1s, and arithmetic ramps (ascending, descending), for every K that fits"""
    out = []
    for K in range(2, min(t, TOP_SYMBOL + 1) + 1):
        out.append([t // K + (1 if i < t % K else 0) for i in range(K)])
        out.append(out[-1][::-1])
        heavy = t - (K - 1)
        for at in sorted({0, K // 2, K - 1}):
            out.append([heavy if i == at else 1 for i in range(K)])
        if K * (K + 1) // 2 <= t:
            ramp = list(range(1, K + 1))
            ramp[-1] += t - K * (K + 1) // 2
            out.append(ramp)
            out.append(ramp[::-1])
    a = np.zeros((len(out), TOP_SYMBOL + 1), np.int64)
    for i, r in enumerate(out):
        a[i, :len(r)] = r
    return a


def search_many(ts=range(2, 257)):
    """the directed many-symbol family at every t <= 256; kept beside the witnesses: 30 and 31 symbols at t = 256, counts
    of 255 and 256, and every tie row of t = 255 / 256 with the most symbols"""
    col = _Collector()
    for t in ts:
        parts = many_symbol_parts(t)
        if parts.shape[0] == 0:
            continue
        tie, odd = _scan(col, parts, t)
        col.ties += int(tie.any(axis=1).sum())
        if t in (255, 256):
            nz = (parts > 0).sum(axis=1)
            for i in np.flatnonzero(nz >= 30)[:6]:
                col.add(place([x for x in parts[i] if x], 0), t, K_DIRECTED)
            best = np.flatnonzero(tie.any(axis=1))
            for i in best[np.argsort(-nz[best], kind="stable")][:4]:
                col.add(place([x for x in parts[i] if x], 2), t, K_TIE)
    for t, parts in ((256, [256]), (256, [255, 1]), (256, [1, 255]), (255, [255]), (255, [254, 1]), (1, [1]), (2, [1, 1]),
                     (2, [2]), (3, [1, 1, 1]), (17, [16, 1]), (17, [1] * 17)):
        for pat in (0, 1, 2):
            col.add(place(parts, pat), t, K_DIRECTED)
    return col.finish()


def search_big(ts=BIG_T):
    """chunks of more than one group: every two-part histogram, every three-part composition and the many-symbol family
    at each t (counts up to t); ties as in the smaller domains"""
    col = _Collector()
    k = 0
    for t in ts:
        n = np.arange(0, t)
        two = np.stack([n, t - n], axis=1)
        tie, odd = _scan(col, two, t)
        hit = np.flatnonzero(tie.any(axis=1))
        col.ties += hit.size
        for i in hit[np.unique(np.linspace(0, hit.size - 1, 6).round().astype(int))] if hit.size else []:
            col.add(place([x for x in two[i] if x], k), t, K_TIE)
            k += 1
        _scan(col, _three_parts(t), t)
        _scan(col, many_symbol_parts(t), t)
        for parts in ([t], [t - 1, 1], [1, t - 1], [t - 30] + [1] * 30):
            col.add(place(parts, k), t, K_DIRECTED)
            k += 1
    return col.finish()


SEARCHES = (search_two, search_three, search_many, search_big)


def build_rows():
    """the whole witness set: counts uint16 [N, 33], t int32 [N], kind, domain, the variant tags of every row, and per
    (domain, variant) the number of witnesses the search met (0 = the variant is equivalent to the spec there)"""
    rows, ts, kinds, doms, found, ties = [], [], [], [], [], []
    for d, fn in enumerate(SEARCHES):
        r, t, k, f, n = fn()
        rows.append(r)
        ts.append(t)
        kinds.append(k)
        doms.append(np.full(t.size, d, np.uint8))
        found.append(f)
        ties.append(n)
    counts, t = np.concatenate(rows), np.concatenate(ts)
    assert (counts.sum(axis=1) == t).all() and (counts[:, TOP_SYMBOL + 1:] == 0).all()
    tags = np.zeros(t.size, np.uint32)
    for tv in np.unique(t):
        s = t == tv
        tags[s] = variant_tags(counts[s], int(tv))
    return dict(counts=counts, t=t, kind=np.concatenate(kinds), domain=np.concatenate(doms), tags=tags,
                found=np.stack(found), ties=np.array(ties, np.int64), variants=np.array(VARIANTS))


def load():
    return np.load(FIXTURE)


# ------------------------------------------------------------------------------------------------ driving a kernel
def header_len(mask: int, nb: int) -> int:
    """bytes of a version-3 stream header: the mask, one count per used symbol but the last, padded to even"""
    nz = bin(int(mask)).count("1")
    h = (nb + 7) // 8 + max(nz - 1, 0)
    return h + (h & 1)


def mask_of(counts_row) -> int:
    return int(sum(1 << i for i in np.flatnonzero(np.asarray(counts_row)[:32])))


def column(counts_row, rng=None) -> np.ndarray:
    """a symbol column with the given histogram: ascending, or shuffled by rng"""
    col = np.repeat(np.arange(LP, dtype=np.uint8), np.asarray(counts_row, np.int64))
    return col if rng is None else rng.permutation(col)


def kv_for_symbols(sym, plane_max, dt: int) -> np.ndarray:
    """half bits [P, t, C] that quantise to exactly sym [P, t, C]: x = s - MAX, which is exact in bf16 and fp16 and needs
    no rounding when every (plane, token) row's maximum is MAX (factor 1) -- the caller keeps one channel per plane at
    symbol 0 (x = -MAX) on every token to pin it"""
    sym = np.asarray(sym)
    M = np.asarray(plane_max, np.int64)[:, None, None]
    assert (sym <= 2 * M).all() and (sym.min(axis=2) == 0).all(), "a row lacks its pinned maximum or exceeds 2 MAX"
    return Q.from_f32((sym.astype(np.int64) - M).astype(np.float32), dt)


# ------------------------------------------------------------------------------------------------ header layouts
# Tiles built lane by lane (one stream per lane, 32 lanes per warp, 128 per tile), so that the per-warp decisions of the
# header code are the test's to choose: which of the two header readers decode_kernel takes (aligned word loads when 8 or
# more active lanes have headers longer than 8 bytes, byte loads otherwise), where a header crosses from the 16-byte
# side record into the temp row (8 versus 10 bytes), and which symbols every lane of a warp skips.  Channel 0 of every
# plane is the lone-symbol stream that pins the row maxima (kv_for_symbols).
WARP, TILE, LONG_HDR, WORD_READER_LANES = 32, 128, 8, 8


def long_nz(nb: int) -> int:
    """the fewest used symbols that make a header longer than LONG_HDR bytes (may exceed what the plane can hold)"""
    return next(nz for nz in range(1, 40) if header_len((1 << nz) - 1, nb) > LONG_HDR)


def lane_histogram(nb: int, nz: int, t: int, style: int, rng) -> np.ndarray:
    """a histogram of t tokens over nz symbols of a plane of nb symbols (symbols 0 .. nb - 2): the first nz, the last nz or
    a random subset; every count 1 but one"""
    nz = max(1, min(nz, nb - 1, t))
    if style % 3 == 0:
        syms = np.arange(nz)
    elif style % 3 == 1:
        syms = np.arange(nb - 1 - nz, nb - 1)
    else:
        syms = np.sort(rng.choice(nb - 1, nz, replace=False))
    row = np.zeros(LP, np.uint16)
    row[syms] = 1
    row[syms[int(rng.integers(0, nz))]] += t - nz
    return row


def _pin(hist, t):
    hist[:, 0] = 0
    hist[:, 0, 0] = t
    return hist


def layout_sweep(nbs, C: int, t: int, rng) -> np.ndarray:
    """lane c of every plane uses 1 + (c - 1) mod (nb - 1) symbols: every header length of every nb, side by side"""
    hist = np.zeros((len(nbs), C, LP), np.uint16)
    for p, nb in enumerate(nbs):
        for c in range(1, C):
            hist[p, c] = lane_histogram(nb, 1 + (c - 1) % (nb - 1), t, c + p, rng)
    return _pin(hist, t)


def layout_threshold(nbs, C: int, t: int, rng) -> np.ndarray:
    """warp w of plane p has 7, 8, 9, 0, all or 1 lanes with long headers (in turn), at its first lanes, its last lanes
    or scattered: neighbouring warps of a tile sit on different sides of the reader threshold"""
    hist = np.zeros((len(nbs), C, LP), np.uint16)
    for p, nb in enumerate(nbs):
        ln = long_nz(nb)
        for w0 in range(0, C, WARP):
            lanes = np.arange(max(w0, 1), min(w0 + WARP, C))
            k = min((7, 8, 9, 0, WARP, 1)[(w0 // WARP + p) % 6], lanes.size) if ln <= min(nb - 1, t) else 0
            where = (p // 2 + w0 // WARP) % 3
            chosen = lanes[:k] if where == 0 else lanes[lanes.size - k:] if where == 1 else rng.choice(lanes, k, replace=False)
            for c in lanes:
                if c in chosen:
                    nz = int(rng.integers(ln, min(nb - 1, t) + 1))
                else:
                    nz = int(rng.integers(1, max(2, min(ln, nb, t + 1))))
                hist[p, c] = lane_histogram(nb, nz, t, c, rng)
    return _pin(hist, t)


def layout_seam(nbs, C: int, t: int, rng) -> np.ndarray:
    """headers of 8, 10 and 12 bytes next to each other: even warps all of them (word reader), odd warps mostly short
    headers with fewer than 8 long ones among them (byte reader)"""
    hist = np.zeros((len(nbs), C, LP), np.uint16)
    for p, nb in enumerate(nbs):
        mb = (nb + 7) // 8
        want = [h - mb + 1 for h in (8, 8, 10, 10, 12, 12)]        # used symbols giving 8, 10, 12 bytes (odd ones pad)
        want = [w - (i & 1) for i, w in enumerate(want)]
        for c in range(1, C):
            w = c // WARP
            nz = want[c % 6] if (w % 2 == 0 or c % WARP in (3, 4, 5, 17, 18, 30)) else want[c % 2]
            hist[p, c] = lane_histogram(nb, nz, t, c + p, rng)
    return _pin(hist, t)


def layout_wany(nbs, C: int, t: int, rng) -> np.ndarray:
    """what the warp's common symbol mask sees: every lane uses symbols 0 and 1; symbol 2 only the odd warps (so a warp
    that skips it sits next to one that does not); one lane of a warp alone uses symbol 3; one lane alone the top symbol
    nb - 2"""
    hist = np.zeros((len(nbs), C, LP), np.uint16)
    for p, nb in enumerate(nbs):
        for c in range(1, C):
            w, lane = c // WARP, c % WARP
            syms = [0, 1] if t >= 2 else [0]
            if w % 2 == 1 and nb - 2 >= 2:
                syms.append(2)
            if lane == (5 + p) % WARP and nb - 2 >= 3:
                syms.append(3)
            if lane == (9 + 2 * p) % WARP:
                syms.append(nb - 2)
            syms = sorted(set(syms))[:t]
            hist[p, c, syms] = 1
            hist[p, c, syms[int(rng.integers(0, len(syms)))]] += t - len(syms)
    return _pin(hist, t)


def layout_counts(nbs, C: int, t: int, rng) -> np.ndarray:
    """count bytes at their ends: (t - 1, 1) and (1, t - 1) -- at t = 256 the stored bytes 255 and 1, the implied last
    counts 1 and 255 -- and lone symbols (the implied 256), on low, high and mixed symbols"""
    hist = np.zeros((len(nbs), C, LP), np.uint16)
    for p, nb in enumerate(nbs):
        for c in range(1, C):
            a, b = sorted(rng.choice(nb - 1, 2, replace=False).tolist())
            kind = c % 3 if t >= 2 else 2
            if kind == 0:
                hist[p, c, [a, b]] = (t - 1, 1)
            elif kind == 1:
                hist[p, c, [a, b]] = (1, t - 1)
            else:
                hist[p, c, (a, b, nb - 2)[c % 3]] = t
    return _pin(hist, t)


LAYOUTS = dict(sweep=layout_sweep, threshold=layout_threshold, seam=layout_seam, wany=layout_wany, counts=layout_counts)


def masks_of(hist) -> np.ndarray:
    return ((np.asarray(hist)[..., :32] > 0).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=-1).astype(np.uint32)


def header_lens(hist, nbs) -> np.ndarray:
    m = masks_of(hist)
    return np.array([[header_len(int(m[p, c]), nbs[p]) for c in range(m.shape[1])] for p in range(m.shape[0])])


def warp_readers(hist, nbs, window=None) -> np.ndarray:
    """[P, warps] int8: the reader each warp of each plane takes when the lanes of `window` = (c0, c1) are active: 1 word
    loads, 0 byte loads, -1 no active lane"""
    hl = header_lens(hist, nbs)
    P, C = hl.shape
    c0, c1 = window or (0, C)
    out = np.full((P, -(-C // WARP)), -1, np.int8)
    for w in range(out.shape[1]):
        a, b = max(w * WARP, c0), min((w + 1) * WARP, C, c1)
        if a < b:
            out[:, w] = (hl[:, a:b] > LONG_HDR).sum(axis=1) >= WORD_READER_LANES
    return out


class Coverage:
    """what a set of layouts reaches, computed from the prescribed histograms alone (add), plus the stream phases, which
    need the streams' lengths (add_phases)"""

    def __init__(self):
        self.readers, self.long_counts, self.ts = set(), set(), set()
        self.hl = {}                      # nb -> header lengths seen
        self.reader_hl = set()            # (reader, nb > 16, header length) over active lanes
        self.seam, self.wany, self.partial, self.counts, self.phases = set(), set(), set(), set(), set()
        self.window_flips = 0

    def add(self, hist, t, nbs, window=None):
        hist = np.asarray(hist)
        P, C = hist.shape[:2]
        c0, c1 = window or (0, C)
        hl, m = header_lens(hist, nbs), masks_of(hist)
        rd, whole = warp_readers(hist, nbs, window), warp_readers(hist, nbs)
        self.ts.add(int(t))
        for p, nb in enumerate(nbs):
            self.hl.setdefault(nb, set()).update(hl[p, c0:c1].tolist())
            stored = hist[p, c0:c1, :32].astype(np.int64)
            for c in range(stored.shape[0]):
                nzs = np.flatnonzero(stored[c])
                self.counts.update(("byte", int(v)) for v in stored[c, nzs[:-1]] if v in (1, 255))
                if int(stored[c, nzs[-1]]) in (1, 255, 256):
                    self.counts.add(("implied", int(stored[c, nzs[-1]])))
            wanys = {}
            for w in range(rd.shape[1]):
                a, b = max(w * WARP, c0), min((w + 1) * WARP, C, c1)
                if a >= b:
                    continue
                name = ("byte", "word")[rd[p, w]]
                self.readers.add(name)
                self.long_counts.add(int((hl[p, a:b] > LONG_HDR).sum()))
                self.reader_hl.update((name, nb > 16, int(h)) for h in hl[p, a:b])
                if {8, 10, 12} <= set(hl[p, a:b].tolist()):
                    self.seam.add(name)
                if window and whole[p, w] == 1 and rd[p, w] == 0:
                    self.window_flips += 1
                live = min((w + 1) * WARP, C) - w * WARP
                if live < WARP:
                    self.partial.add(("warp", live))
                if C - (w * WARP // TILE) * TILE <= TILE // 2:
                    self.partial.add(("tile", "half-empty"))
                bits = (m[p, a:b, None] >> np.arange(32, dtype=np.uint32)) & 1
                uses = bits.sum(axis=0)
                wanys[w] = uses > 0
                if b - a > 1 and (uses[:nb - 2] == 1).any():
                    self.wany.add("a symbol used by one lane of a warp")
                if b - a > 1 and uses[nb - 2] == 1:
                    self.wany.add("the top symbol used by one lane of a warp")
                if b - a > 1 and (uses[:nb - 1] == 0).any():
                    self.wany.add("a warp skips symbols")
                if w - 1 in wanys and w * WARP // TILE == (w - 1) * WARP // TILE and (wanys[w] & ~wanys[w - 1]).any():
                    self.wany.add("a symbol no lane of a warp uses, used in the next warp of the tile")

    def add_phases(self, hist, nbs, half, window=None):
        """half: the container's half-lengths [P, C]; streams lie back to back from a 16-byte aligned payload start"""
        hl, rd = header_lens(hist, nbs), warp_readers(hist, nbs, window)
        P, C = hl.shape
        c0, c1 = window or (0, C)
        start = np.concatenate([[0], np.cumsum(2 * np.asarray(half, np.int64).ravel())[:-1]]).reshape(P, C)
        for p in range(P):
            for c in range(c0, c1):
                if hl[p, c] > LONG_HDR:
                    self.phases.add((("byte", "word")[rd[p, c // WARP]], int(start[p, c] % 4)))

    def missing(self) -> list:
        out = []
        out += [f"reader {r}" for r in ("byte", "word") if r not in self.readers]
        out += [f"{k} long-header lanes in a warp" for k in (0, 7, 8, 9, 32) if k not in self.long_counts]
        for nb in range(4, 33, 2):
            mb = (nb + 7) // 8
            full = set(range(mb + (mb & 1), mb + nb - 2 + ((mb + nb) & 1) + 1, 2))
            out += [f"nb {nb}: header of {h} bytes" for h in sorted(full - self.hl.get(nb, set()))]
        for h in range(4, 35, 2):
            if ("word", True, h) not in self.reader_hl:
                out.append(f"word reader, nb > 16, header of {h} bytes")
        for h in range(2, 17, 2):
            if ("word", False, h) not in self.reader_hl:
                out.append(f"word reader, nb <= 16, header of {h} bytes")
        for h in (2, 4, 6, 8, 10, 12, 16, 34):
            if not any(("byte", wide, h) in self.reader_hl for wide in (False, True)):
                out.append(f"byte reader, header of {h} bytes")
        out += [f"8 / 10 / 12-byte headers in one warp, {r} reader" for r in ("byte", "word") if r not in self.seam]
        out += [w for w in ("a symbol used by one lane of a warp", "the top symbol used by one lane of a warp",
                            "a warp skips symbols", "a symbol no lane of a warp uses, used in the next warp of the tile")
                if w not in self.wany]
        out += [f"{p}" for p in (("warp", 3), ("tile", "half-empty")) if p not in self.partial]
        out += [f"count {c}" for c in (("byte", 1), ("byte", 255), ("implied", 1), ("implied", 255), ("implied", 256))
                if c not in self.counts]
        out += [f"t = {t}" for t in (1, 2, 3, 17, 255, 256) if t not in self.ts]
        out += [f"long header at phase {ph}, {r} reader" for r in ("byte", "word") for ph in (0, 2)
                if self.phases and (r, ph) not in self.phases]
        return out

    def report(self) -> str:
        return (f"readers {sorted(self.readers)}; long-header lanes per warp {sorted(self.long_counts)}; header lengths "
                f"per nb { {nb: sorted(v) for nb, v in sorted(self.hl.items())} }; word reader lengths "
                f"{sorted(h for r, _, h in self.reader_hl if r == 'word')[0]}..{max(h for r, _, h in self.reader_hl if r == 'word')}"
                f"; 8/10/12 seam under {sorted(self.seam)}; common-mask cases {sorted(self.wany)}; partial {sorted(self.partial, key=str)}"
                f"; counts {sorted(self.counts)}; t {sorted(self.ts)}; phases {sorted(self.phases)}; windows that flip a "
                f"warp from the word to the byte reader {self.window_flips}")


def layout_cases():
    """(name, t, H, D, window heads or None) of every layout tile the GPU suite runs; C = H * D"""
    return [("sweep", 256, 1, 128, None), ("sweep", 255, 3, 33, None), ("sweep", 17, 1, 64, None),
             ("threshold", 256, 1, 576, None), ("threshold", 256, 3, 33, None), ("threshold", 255, 2, 96, None),
             ("seam", 256, 2, 128, None), ("seam", 17, 3, 33, None),
             ("wany", 256, 1, 128, None), ("wany", 3, 3, 33, None), ("wany", 2, 1, 64, None), ("wany", 1, 1, 40, None),
             ("counts", 256, 1, 128, None), ("counts", 255, 1, 40, None), ("counts", 2, 1, 40, None),
             ("window", 256, 3, 40, (1, 1))]


def layout_window(nbs, C: int, t: int, rng, D: int = 40) -> np.ndarray:
    """for a decode of head 1 alone (channels D .. 2 D - 1, D = 40): warp 1 (channels 32 .. 63) has 8 long-header lanes
    of which one sits at channel 32 .. D - 1, outside the window -- the whole warp takes the word reader, the window's
    active lanes the byte reader; warp 2 has 9 with two outside on the far side"""
    hist = layout_wany(nbs, C, t, rng)
    for p, nb in enumerate(nbs):
        ln = long_nz(nb)
        if ln > nb - 1:
            continue
        for c in [WARP + 2] + list(range(D + 1, D + 8)) + list(range(2 * WARP, 2 * WARP + 7)) + [2 * D, 2 * D + 3]:
            hist[p, c] = lane_histogram(nb, int(rng.integers(ln, nb)), t, c, rng)
    return hist


LAYOUTS["window"] = layout_window
