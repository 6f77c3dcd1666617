"""The arithmetic coder (container version 1) at its carry, pending-run, renormalisation and row-bound edges: an
independent statement of the bitstream in plain Python integers, traces of every coded and decoded symbol, kernel-shaped
models of EncState2 (enc_symbol2, enc_append, enc_ripple, enc_finish2) and DecState2 (dec_init2, dec_symbol2) in
wrapping 32-bit arithmetic that can be told to make one plausible mistake each (MUTANTS), and the seeded search for
producible streams that reach each edge and tell each mutant from the spec (stored in tests/golden/ac_edges.npz by
tests/golden/make_ac_edges.py).

Every CDF row comes from cdf_edges.spec_cdf, so every stream is one the product can produce: a chunk of g <= 256 tokens
coded under its own histogram, or a group of a longer chunk coded under the chunk-wide CDF.

Format (DESIGN.md 3.2 step 4 and 3.4), one stream of g symbols under c[0..32] (c[32] := 65536):
    encoder  low = 0, high = 2^32 - 1, pending = 0.  Per symbol s: span = high - low + 1,
             high = low + (span c[s + 1] >> 16) - 1, low = low + (span c[s] >> 16); then, one bit at a time:
               high < 2^31: emit 0 and `pending` 1s;  low >= 2^31: emit 1 and `pending` 0s, subtract 2^31 from both;
               2^30 <= low and high < 3 2^30: pending += 1, subtract 2^30 from both;  otherwise stop;
               low = 2 low, high = 2 high + 1.
             termination: pending += 1, emit (low < 2^30 ? 0 : 1) and the pending run, zero pad to a byte.
    bits     MSB first
    decoder  value = the first 32 bits (zeros past the end); per symbol s = max{s : low + (span c[s] >> 16) <= value},
             then the encoder's interval update and the same shifts, which pull the next stream bit into value.

What the search settled about the edges one might ask for (numbers from search(); tests/test_ac_edges_cpu.py keeps
them true):
  * the largest shift count found is k = 17, not 18.  The new interval is >= floor(span / 2^16) >= 2^14 wide, so k = 18
    needs a width-1 symbol, a new interval of exactly 2^14 and an absolute low that is a multiple of 2^14 -- chance
    about 1e-9 per width-1 step.  A used symbol gets width 1 first in a chunk of WIDTH1_T = 65505 tokens (every count
    moves the scaled CDF by n 65504 / T >= 1 below that); there k is 15, 16 or 17.  The own-CDF streams and the chunks
    of up to 1030 tokens reach k = 11 at most;
  * the longest own-CDF stream is 159 bytes, the bound (own_bound_bits) 1269.95 bits = 159 bytes, the row 160;
  * long pending runs (31, 32, 33, > 64 bits) do not turn up at random: run_column builds them by decoding a value
    that has a long run of equal bits behind a random prefix;
  * two mutants are equivalent to the spec on every producible stream (EQUIVALENT), with the reason.

Used by tests/test_ac_edges_cpu.py, tests/test_gpu_ac_edges.py and the fixture generator."""
from __future__ import annotations

import math
import os

import numpy as np

import cdf_edges as E
import rans_edges as R

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "ac_edges.npz")

M32 = 0xFFFFFFFF
HALF, Q1, Q3 = 1 << 31, 1 << 30, 3 << 30
G = 256
ROW_WORDS_OWN = 40          # TEMPW_FUSED: words per own-CDF stream row in encode_kernel
ROW_WORDS_SPLIT = 132       # TEMPW_SPLIT: words per chunk-wide-CDF group row
BIG_T = (257, 300, 700, 1030)


# ------------------------------------------------------------------------------------------------ the row bound
def own_bound_bits(t: int = G, K: int = 31) -> float:
    """an upper bound on the bits of an own-CDF stream of t tokens over K symbols, every term counted:
      * the ideal cost under the rounded CDF.  Each entry is rint(fl32(F) 65504) + i, off the exact F 65504 by at most
        0.5 + 0.01 (fl32 of the double sum, the float multiply), and the + i gives every symbol one slot more, so a
        symbol of count n has width w >= n 65504 / t - 0.02 and costs <= log2(65536 / w) bits per token.  The sum over
        the histogram is Schur-concave in the counts (each term is concave in n), so the most even histogram of t
        tokens over K symbols is the worst;
      * the truncation of every step: the new span is >= span w / 2^16 - 1 with span > 2^30, so a step costs at most
        -log2(1 - 2^16 / (2^30 w)) bits more than its ideal;
      * termination: the renormalised final interval is wider than 2^30, so the k shifts of the whole stream are below
        the cost above, and termination adds 2 bits (the final bit and the run behind it).
    Byte padding is the caller's ceil(bits / 8)."""
    K = min(K, t)
    cnt = [t // K + (1 if k < t % K else 0) for k in range(K)]
    ideal = sum(n * math.log2(65536.0 / (n * 65504.0 / t - 0.02)) for n in cnt if n)
    wmin = 65504.0 / t - 0.02
    trunc = t * -math.log2(1.0 - 65536.0 / (2.0 ** 30 * wmin))
    return ideal + trunc + 2.0


def split_bound_bits(g: int = G) -> float:
    """the same for a group under a chunk-wide CDF: every width is >= 1, so <= 16 bits per token, plus truncation
    (new span >= 2^14 - 1 for width 1) and termination"""
    return g * (16.0 - math.log2(1.0 - 2.0 ** -14)) + 2.0


# ------------------------------------------------------------------------------------------------ the spec
def _bounds(cdf_row, s):
    start, freq = R.table(cdf_row)
    return start[s], start[s] + freq[s]


def encode(cdf_row, symbols, trace=None, term=None) -> bytes:
    """the stream of `symbols`.  trace: a list that receives per symbol (i, s, c_lo, c_hi, n, m, k, pending after,
    [(run length, first run bit's position, run bit)] resolved by this symbol's shifts).  term: a dict that receives the
    termination's run and the bit count before padding."""
    start, freq = R.table(cdf_row)
    low, high, pend, bits = 0, M32, 0, []

    def emit(b):
        nonlocal pend
        runs = []
        bits.append(b)
        if pend:
            runs.append((pend, len(bits), 1 - b))
            bits.extend([1 - b] * pend)
            pend = 0
        return runs

    for i, s in enumerate(symbols):
        s = int(s)
        span = high - low + 1
        high = low + ((span * (start[s] + freq[s])) >> 16) - 1
        low = low + ((span * start[s]) >> 16)
        n = m = 0
        runs = []
        while True:
            if high < HALF:
                runs += emit(0)
                n += 1
            elif low >= HALF:
                runs += emit(1)
                low, high, n = low - HALF, high - HALF, n + 1
            elif low >= Q1 and high < Q3:
                pend, low, high, m = pend + 1, low - Q1, high - Q1, m + 1
            else:
                break
            low, high = 2 * low, 2 * high + 1
        if trace is not None:
            trace.append((i, s, start[s], start[s] + freq[s], n, m, n + m, pend, runs))
    pend += 1
    runs = emit(0 if low < Q1 else 1)
    if term is not None:
        term.update(runs=runs, nbits=len(bits))
    bits += [0] * (-len(bits) % 8)
    return bytes(int("".join(map(str, bits[k:k + 8])), 2) for k in range(0, len(bits), 8))


def decode(cdf_row, data: bytes, g: int, tail: bytes = b""):
    """symbols uint8 [g]: the format's decoder, by the book.  Bits past the stream come from `tail`, then zeros."""
    start, freq = R.table(cdf_row)
    src = bytes(data) + bytes(tail)
    nbits = 8 * len(src)

    def bit(k):
        return (src[k >> 3] >> (7 - (k & 7))) & 1 if k < nbits else 0
    value = sum(bit(k) << (31 - k) for k in range(32))
    pos, low, high = 32, 0, M32
    out = np.zeros(g, np.uint8)
    for i in range(g):
        span = high - low + 1
        s = max(k for k in range(32) if low + ((span * start[k]) >> 16) <= value)
        out[i] = s
        high = low + ((span * (start[s] + freq[s])) >> 16) - 1
        low = low + ((span * start[s]) >> 16)
        assert low <= value <= high
        while True:
            if high < HALF:
                pass
            elif low >= HALF:
                low, high, value = low - HALF, high - HALF, value - HALF
            elif low >= Q1 and high < Q3:
                low, high, value = low - Q1, high - Q1, value - Q1
            else:
                break
            low, high, value = 2 * low, 2 * high + 1, 2 * value + bit(pos)
            pos += 1
    return out


# ------------------------------------------------------------------------------------------------ the kernels' shape
ENC_MUTANTS = ("no_carry", "ripple_once", "ripple_not_word0", "finish_no_over", "finish_no_carry", "shl_wrap",
               "rng_no_ones", "e3_minus_one", "phi_no_chi", "plo_no_clo")
DEC_MUTANTS = ("walk_up_only", "walk_down_only", "no_force31", "span0_as_max", "skip_ignored", "refill_gt32",
               "check_gt", "renorm_phi_as_is")
MUTANTS = ENC_MUTANTS + DEC_MUTANTS
MUTANT_DOC = {
    "no_carry": "the carry out of x + plo is dropped (add.cc without addc)",
    "ripple_once": "enc_ripple adds the carry to one row word and stops",
    "ripple_not_word0": "enc_ripple stops before word 0 of the row",
    "finish_no_over": "enc_finish2 ignores a carry that rippled through the whole tail",
    "finish_no_carry": "enc_finish2 drops the carry out of x + 2^30",
    "shl_wrap": "shl_clamp wraps its count mod 32 instead of clamping (only the carry bit above nb is cut)",
    "rng_no_ones": "rng = (h << k) - x: the shifted-in low bits of high are zeros instead of ones",
    "e3_minus_one": "the E3 run is counted one short when there is one",
    "phi_no_chi": "phi = (r c_hi) >> 16 without the + c_hi term",
    "plo_no_clo": "plo = (r c_lo) >> 16 without the + c_lo term",
    "walk_up_only": "the slow path only walks upward",
    "walk_down_only": "the slow path only walks downward",
    "no_force31": "a guess of s = 31 is not forced into the slow path",
    "span0_as_max": "span = 0 (2^32) taken as 2^32 - 1 in the exact products",
    "skip_ignored": "dec_init2 ignores the leading bytes of the first word that belong to the previous stream",
    "refill_gt32": "the window moves on when pos > 32 instead of pos >= 32",
    "check_gt": "the exactness check lets off == phi through ((off - plo) > (phi - plo) sends to the slow path)",
    "renorm_phi_as_is": "the renormalisation uses the search's umulhi(span, e[s + 1]) also for s = 31",
}
EQUIVALENT = {
    "no_force31": "no stream codes symbol 31 (symbols are <= 30), and a guess of 31 has off < (span c[31]) >> 16, which "
                  "the exactness check already sends to the slow path",
    "renorm_phi_as_is": "the same: phi for s = 31 only matters when the decoded symbol is 31, which no stream codes",
}


def bfind(x: int) -> int:
    return x.bit_length() - 1 if x else M32


def funnel_l(lo: int, hi: int, n: int) -> int:
    """upper 32 bits of (hi:lo) << (n mod 32), as __funnelshift_l"""
    n &= 31
    return ((hi << n) | (lo >> (32 - n))) & M32 if n else hi


def funnel_r(lo: int, hi: int, n: int) -> int:
    n &= 31
    return ((lo >> n) | (hi << (32 - n))) & M32 if n else lo


def shl_clamp(x: int, n: int, mut=None) -> int:
    if mut == "shl_wrap":
        return (x << (n & 31)) & M32
    return 0 if n >= 32 else (x << n) & M32


class Enc2:
    """EncState2 with its row.  Records per step (k, carry, flushed, ripple: (words, reached word 0, over at flush)) and
    per termination (carry, w at that moment, nb, over)."""

    def __init__(self, cap: int, mut=None, guard: int = 0):
        self.x, self.rng, self.lo, self.m, self.w = 0, M32, 0, 0xFFFFFFE0, 0
        self.cap, self.mut = cap, mut
        self.row = [0] * (cap + 2 * guard)
        self.base = guard
        self.steps, self.term = [], None
        self._rip = None

    def _ripple(self, w, capm1, over):
        words, ok = 0, True
        while True:
            w -= 1
            q = self.base + (w if w < capm1 else capm1)
            v = self.row[q] + over
            self.row[q] = v & M32
            over = 1 if v > M32 else 0
            words += 1
            if self.mut == "ripple_once":
                break
            if over == 0 or w == (1 if self.mut == "ripple_not_word0" else 0):
                break
        self._rip = (words, w == 0)

    def _append(self, x, k, capm1):
        hi = funnel_l(self.lo, 0, k)
        lo = funnel_l(x, self.lo, k)
        m = (self.m + k) & M32
        word = funnel_r(lo, hi, m)
        flush = m < (1 << 31)
        if flush:
            self.row[self.base + (self.w if self.w < capm1 else capm1)] = word
        over = funnel_r(hi, 0, m)
        self._rip = None
        if over:
            self._ripple(self.w, capm1, over)
        self.lo = lo & ~shl_clamp(M32, m, self.mut) & M32
        self.w += 1 if flush else 0
        self.m = m | 0xFFFFFFE0
        return flush, over

    def symbol(self, c_lo, width):
        r, c_hi = self.rng, c_lo + width
        plo = ((r * c_lo + (0 if self.mut == "plo_no_clo" else c_lo)) >> 16) & M32
        phi = ((r * c_hi + (0 if self.mut == "phi_no_chi" else c_hi)) >> 16) & M32
        h = (self.x + phi - 1) & M32
        x = self.x + plo
        carry = x >> 32
        x &= M32
        if self.mut != "no_carry":
            self.lo = (self.lo + carry) & M32
        p = bfind((x ^ h) | 1)
        f = (~x | h) & ((1 << p) - 1)
        k = (30 - bfind(f)) & M32
        if self.mut == "e3_minus_one" and k > 31 - p:
            k -= 1
        self.x = (x << k) & M32
        fill = ((h << k) & M32) if self.mut == "rng_no_ones" else funnel_l(M32, h, k)
        self.rng = (fill - self.x) & M32
        flush, over = self._append(x, k, self.cap - 1)
        self.steps.append((k, carry, flush, self._rip))

    def finish(self) -> int:
        capm1 = self.cap - 1
        x = (self.x + Q1) & M32
        carry = 1 if x < Q1 else 0
        w0 = self.w
        if self.mut != "finish_no_carry":
            self.lo = (self.lo + carry) & M32
        flush, over_at_flush = self._append(x, 2, capm1)
        rip = self._rip
        nb = self.m & 31
        over = self.lo >> nb
        if over and self.mut != "finish_no_over":
            if self.w:
                self._ripple(self.w, capm1, over)
                rip = self._rip
            self.lo &= ~(M32 << nb) & M32
        full = self.w
        if nb:
            self.row[self.base + (self.w if self.w < capm1 else capm1)] = (self.lo << (32 - nb)) & M32
            self.w += 1
        self.term = dict(carry=carry, w=w0, nb=nb, over=over, flush=flush, ripple=rip)
        return 4 * full + ((nb + 7) >> 3)

    def bytes(self, n: int) -> bytes:
        b = b"".join(v.to_bytes(4, "big") for v in self.row[self.base:self.base + self.cap])
        return b[:n]


def encode_as_kernel(cdf_row, symbols, mut=None, cap=None):
    """(bytes, Enc2): enc_symbol2 on every symbol, then enc_finish2, into a row of `cap` words (default: room enough)"""
    start, freq = R.table(cdf_row)
    e = Enc2(cap if cap is not None else len(symbols) // 2 + 4, mut)
    for s in symbols:
        e.symbol(start[int(s)], freq[int(s)])
    n = e.finish()
    return e.bytes(n), e


# the decoder's key: what dec_key_approx returns; the model takes it as an input
def key_exact(off: int, span: int) -> int:
    return min(M32, (off << 32) // (span or 1 << 32))


def key_host(off: int, span: int) -> int:
    """the host branch of dec_key_approx: float32 division"""
    if span == 0:
        return 0
    q = np.float32(np.float32(off) / np.float32(span)) * np.float32(4294967296.0)
    return M32 if q >= np.float32(4294967040.0) else int(q)


def key_device_like(off: int, span: int) -> int:
    """the device branch with a correctly rounded reciprocal: span = 0 gives rcp = inf, off * inf = inf (0 * inf =
    NaN, which converts to 0), and the conversion saturates"""
    if span == 0:
        return M32 if off else 0
    rc = np.float32(np.float32(1.0) / np.float32(span))
    q = np.float32(np.float32(off) * np.float32(rc * np.float32(4294967296.0)))
    return M32 if q >= np.float32(4294967296.0) else int(q)


def dec_table(cdf_row):
    u = [int(v) & 0xFFFF for v in np.asarray(cdf_row).reshape(-1)]
    return [(u[i] << 16) if i < 32 else M32 for i in range(33)]


def decode_as_kernel(cdf_row, data: bytes, g: int, skip: int = 0, nsteps: int = 5, key=key_host, mut=None, trace=None,
                     before: bytes = b"\x5a\x5a\x5a", after: bytes = b"\xa5" * 16):
    """dec_init2 + dec_symbol2 over the stream placed `skip` bytes into an aligned word (foreign bytes on both sides).
    trace receives per symbol (span, off, pos, s, guess, slow, walk) with walk = (+/- steps) and per refill the pos
    it moved at.  Returns the symbols."""
    e = dec_table(cdf_row)
    buf = before[:skip] + bytes(data) + after
    buf += bytes(-len(buf) % 4)
    nw = len(buf) // 4
    words = [int.from_bytes(buf[4 * i:4 * i + 4], "big") for i in range(nw)]
    idx = 0

    def next_be():
        nonlocal idx
        v = words[idx] if idx < nw else 0xA5A5A5A5
        idx += 1
        return v
    st = dict(x=0, span=0)
    cur, nxt = next_be(), next_be()
    pos = 0 if mut == "skip_ignored" else 8 * skip
    off = funnel_l(nxt, cur, pos)
    pos += 32
    if (pos > 32) if mut == "refill_gt32" else (pos >= 32):
        cur, nxt, pos = nxt, next_be(), pos - 32
    x, span = 0, 0
    top = (1 << nsteps) - 1
    out = np.zeros(g, np.uint8)

    def exact(s):
        r = (M32 - 1) if (mut == "span0_as_max" and span == 0) else (span - 1) & M32
        c0 = e[s] >> 16
        c1 = 0x10000 if s >= 31 else e[s + 1] >> 16
        return ((r * c0 + c0) >> 16) & M32, ((r * c1 + c1) >> 16) & M32

    for i in range(g):
        cnt = key(off, span) & M32
        a = 0
        step = 1 << (nsteps - 1)
        while step:
            if e[a + step] <= cnt:
                a += step
            step >>= 1
        s = guess = a
        plo = (span * e[s]) >> 32
        phi = (span * e[s + 1]) >> 32
        if mut == "span0_as_max" and span == 0:
            plo, phi = (M32 * e[s]) >> 32, (M32 * e[s + 1]) >> 32
        bad = ((off - plo) & M32) > ((phi - plo) & M32) if mut == "check_gt" else ((off - plo) & M32) >= ((phi - plo) & M32)
        slow = bad or (nsteps == 5 and s == 31 and mut != "no_force31")
        walk = 0
        if slow:
            plo, phi = exact(s)
            if mut == "renorm_phi_as_is" and s == 31:
                phi = (span * e[32]) >> 32
            while mut != "walk_up_only" and off < plo and s > 0:
                s -= 1
                walk -= 1
                plo, phi = exact(s)
            while mut != "walk_down_only" and s < top and ((off - plo) & M32) >= ((phi - plo) & M32):
                s += 1
                walk += 1
                plo, phi = exact(s)
        out[i] = s
        rec = [span, off, pos, s, guess, slow, walk, None]
        if i < g - 1:
            xx = (x + plo) & M32
            h = (x + phi - 1) & M32
            p = bfind((xx ^ h) | 1)
            f = (~xx | h) & ((1 << p) - 1)
            k = (30 - bfind(f)) & M32
            t = funnel_l(nxt, cur, pos)
            off = funnel_l(t, (off - plo) & M32, k)
            pos += k
            x = (xx << k) & M32
            span = ((phi - plo) << k) & M32
            if (pos > 32) if mut == "refill_gt32" else (pos >= 32):
                rec[7] = pos
                cur, nxt, pos = nxt, next_be(), pos - 32
        if trace is not None:
            trace.append(tuple(rec))
    return out


KEYS = {"host": key_host, "device-like": key_device_like, "exact": key_exact, "zero": lambda o, s: 0,
        "ones": lambda o, s: M32, "exact + 2^16": lambda o, s: min(M32, key_exact(o, s) + 65536),
        "exact - 2^16": lambda o, s: max(0, key_exact(o, s) - 65536)}


def kills(cdf_row, col, nsteps: int = 5) -> int:
    """bit k set <=> MUTANTS[k] gives other bytes (encoder) or other symbols (decoder, any skip, host or device-like
    key, or a key guessed all-zero / all-ones)"""
    col = np.asarray(col, np.uint8)
    want = encode(cdf_row, col)
    out = 0
    for k, name in enumerate(MUTANTS):
        if name in ENC_MUTANTS:
            bad = encode_as_kernel(cdf_row, col, name)[0] != want
        else:
            bad = False
            for skip in (0, 1, 2, 3):
                for kn in ("host", "device-like", "zero", "ones"):
                    if not bad:
                        bad = not np.array_equal(decode_as_kernel(cdf_row, want, col.size, skip, nsteps, KEYS[kn], name), col)
        out |= int(bad) << k
    return out


# ------------------------------------------------------------------------------------------------ what a stream reaches
def stream_items(cdf_row, col, plane: str, own: bool, data: bytes = None) -> set:
    """coverage items of one stream, from the spec's trace, the encoder model's record and the decoder model's trace
    (host-branch key and the device-like key, skip 0..3).  plane: 'wide' (5-step search) or 'narrow' (4-step)."""
    col = np.asarray(col, np.uint8)
    g = col.size
    tr, term = [], {}
    want = encode(cdf_row, col, tr, term)
    got, enc = encode_as_kernel(cdf_row, col)
    assert got == want
    it = set()
    for (i, s, c_lo, c_hi, n, m, k, pend, runs) in tr:
        it.add(f"k = {k}" if k <= 1 else "k >= 16" if k >= 16 else "k 2..15")
        for (ln, bp, b) in runs:
            _run_items(it, ln, bp)
    for (ln, bp, b) in term["runs"]:
        _run_items(it, ln, bp)
    it.add(f"k = {max(t[6] for t in tr)} (largest in the stream)")
    for (k, carry, flush, rip) in enc.steps:
        if carry:
            it.add("carry out of x + plo")
        if rip:
            words, w0 = rip
            it.add("carry through the whole accumulator")
            it.add("carry into 1 row word" if words == 1 else "carry into >= 2 row words")
            if w0:
                it.add("carry into word 0")
    if enc.steps[-1][2]:
        it.add("flush on the last symbol")
    tm = enc.term
    if tm["carry"]:
        it.add(f"carry at termination, st.w {'= 0' if tm['w'] == 0 else '> 0'}")
    if tm["ripple"]:
        it.add("carry at termination ripples into the row")
    nb = tm["nb"]
    it.add(f"{nb} bits left at termination" if nb in (0, 30, 31) else "1..7 bits left at termination" if nb <= 7 else
           "8..29 bits left at termination")
    it.add(f"stream length = {len(want) % 4} mod 4")
    # decoder
    for kn in ("host", "device-like"):
        for skip in range(4):
            dt = []
            dec = decode_as_kernel(cdf_row, want, g, skip, 5 if plane == "wide" else 4, KEYS[kn], trace=dt)
            assert np.array_equal(dec, col)
            for j, (span, off, pos, s, guess, slow, walk, rf) in enumerate(dt):
                if span == 0 and j == 1:
                    it.add("span = 2^32 after the first symbol")
                if slow and walk < 0:
                    it.add("slow path from a guess too high")
                if slow and walk > 0:
                    it.add("slow path from a guess too low")
                if abs(walk) > 1:
                    it.add("slow-path walk of more than one step")
                if guess == 31 and slow:
                    it.add("guess s = 31 forced into the slow path")
                if plane == "narrow" and s == 14:
                    it.add("symbol 14 in the 4-step search")
                if rf == 32:
                    it.add("refill exactly at pos = 32")
            if skip == 0:
                break
    if own:
        it.add(f"own-CDF, t = {g}" if g in (1, 2, 255, 256) else "own-CDF, other t")
    else:
        words = -(-len(want) // 4)
        if words > ROW_WORDS_OWN:
            it.add("a chunk-wide-CDF group longer than an own-CDF row (40 words)")
    return it


def _run_items(it, ln, bp):
    if ln in (31, 32, 33):
        it.add(f"pending run of {ln} bits")
    if ln > 64:
        it.add("pending run of > 64 bits")
    if bp // 32 != (bp + ln - 1) // 32:
        it.add("pending run straddling a flushed word")


class Coverage:
    def __init__(self):
        self.items = set()

    def add(self, items):
        self.items |= set(items)

    @staticmethod
    def wanted(kmax: int) -> list:
        w = ["carry out of x + plo", "carry through the whole accumulator", "carry into 1 row word",
             "carry into >= 2 row words", "carry into word 0", "carry at termination, st.w = 0",
             "carry at termination, st.w > 0", "carry at termination ripples into the row"]
        w += [f"pending run of {n} bits" for n in (31, 32, 33)]
        w += ["pending run of > 64 bits", "pending run straddling a flushed word"]
        w += ["k = 0", "k = 1", "k 2..15", "k >= 16", f"k = {kmax} (largest in the stream)", "flush on the last symbol"]
        w += [f"{n} bits left at termination" for n in (0, 30, 31)] + ["1..7 bits left at termination"]
        w += [f"stream length = {r} mod 4" for r in range(4)]
        w += ["span = 2^32 after the first symbol", "slow path from a guess too high", "slow path from a guess too low",
              "slow-path walk of more than one step", "guess s = 31 forced into the slow path",
              "symbol 14 in the 4-step search", "refill exactly at pos = 32"]
        w += [f"own-CDF, t = {t}" for t in (1, 2, 255, 256)]
        w += ["a chunk-wide-CDF group longer than an own-CDF row (40 words)"]
        return w

    def missing(self, kmax: int) -> list:
        return [w for w in self.wanted(kmax) if w not in self.items]


# ------------------------------------------------------------------------------------------------ naming a failure
def first_bad_step(cdf_row, col, got: bytes) -> str:
    """where a stream that should be encode(cdf_row, col) went wrong: the first differing bit, and the coding step whose
    shifts emitted it (bits leave the encoder in coding order; a carry changes bits already out, so the step named is the
    one that emitted the first wrong bit or a later one whose carry rippled back into it)"""
    tr, term = [], {}
    want = encode(cdf_row, col, tr, term)
    if bytes(got) == want:
        return "stream equals the spec's"
    a = "".join(f"{b:08b}" for b in want)
    b = "".join(f"{v:08b}" for v in bytes(got))
    k = next((j for j in range(min(len(a), len(b))) if a[j] != b[j]), min(len(a), len(b)))
    # bits emitted (final or pending) after each step: the spec's bits are final once emitted, pending ones are counted
    done, step = 0, len(tr)
    for j, t in enumerate(tr):
        done += t[6]
        if done > k:
            step = j
            break
    s = tr[step] if step < len(tr) else None
    return (f"{len(got)} bytes, spec {len(want)}; first differing bit {k} (got {b[k] if k < len(b) else None}, spec "
            f"{a[k] if k < len(a) else None}): shifted out by coding step {step} of {len(tr)}"
            + (f" (token {s[0]}, symbol {s[1]}, interval [{s[2]}, {s[3]}), n = {s[4]}, m = {s[5]}, pending {s[7]})"
               if s else " (termination)"))


# ------------------------------------------------------------------------------------------------ the search
WIDTH1_T = 65505            # the smallest chunk in which a used symbol can get CDF width 1 (min_width_t)


def width1_prefixes(T: int) -> np.ndarray:
    """the prefix counts P for which a chunk of T tokens -- P of symbol 0, one of symbol 1, the rest symbol 2 -- gives
    symbol 1 width 1 under its chunk-wide CDF"""
    P = np.arange(0, T - 1)
    h = np.zeros((P.size, 33), np.uint32)
    h[:, 0], h[:, 1], h[:, 2] = P, 1, T - 1 - P
    c = E.spec_cdf(h, T).view(np.uint16).astype(np.int64)
    return P[c[:, 2] - c[:, 1] == 1]


def min_width_t() -> int:
    """every count n >= 1 moves the scaled CDF by n 65504 / T >= 1 when T <= 65504, so a width of 1 (the + i alone)
    needs T > 65504; this finds the first T at which the rounding lets it happen"""
    T = 65504
    while not width1_prefixes(T).size:
        T += 1
    return T


def longest_own_stream(rng, top: int = 30, t: int = G, tries: int = 64):
    """the 31 symbols as even as t tokens allow (the cost bound's worst histogram), in the order of `tries` shuffles
    that gives the longest stream (order moves only the truncation and the termination)"""
    K = top + 1
    cnt = np.full(K, t // K)
    cnt[K - t % K:] += 1
    base = np.repeat(np.arange(K), cnt).astype(np.uint8)
    best = None
    for _ in range(tries):
        col = rng.permutation(base)
        n = len(encode(R.own_cdf(col), col))
        if best is None or n > best[0]:
            best = (n, col)
    return best[1]


def foreign_columns(T: int, rng, top: int = 30, n: int = 4) -> np.ndarray:
    """columns [n, T] of a chunk of T > 256 tokens: one common symbol, with the chunk's rare symbols crowded into a
    few groups (long streams, pending runs under small widths) -- rans_edges.foreign_columns"""
    return R.foreign_columns(T, rng, top, n)


def wide_column(rng, kwant: int = 17, tries: int = 4000) -> np.ndarray:
    """a chunk of WIDTH1_T tokens whose lone symbol 1 has width 1 and is coded with k = kwant shifts: group 0 is a random
    run of symbols 0 and 2 ending in the lone symbol (the state in front of it decides k), the other groups hold the
    remaining 0s, then the 2s"""
    T = WIDTH1_T
    P = int(width1_prefixes(T)[0])
    h = np.zeros(33, np.uint32)
    h[0], h[1], h[2] = P, 1, T - 1 - P
    cdf = E.spec_cdf(h, T)
    for _ in range(tries):
        n = int(rng.integers(1, G))
        head = rng.choice(np.array([0, 2], np.uint8), n)
        tr = []
        encode(cdf, np.concatenate([head, [1]]).astype(np.uint8), tr)
        if tr[-1][6] == kwant and (head == 0).sum() <= P:
            rest0 = P - int((head == 0).sum())
            col = np.concatenate([head, [1], np.zeros(rest0, np.uint8),
                                  np.full(T - n - 1 - rest0, 2, np.uint8)]).astype(np.uint8)
            assert np.array_equal(np.bincount(col, minlength=33)[:3], h[:3])
            return col
    raise RuntimeError("no order reached k = %d" % kwant)


RUN_T = 1030


def run_column(rng, L: int, carry: bool, at: int = 40, T: int = RUN_T):
    """a chunk of T tokens whose group 0 codes a value with a long pending run: the chunk's histogram is fixed first
    (31 symbols, as even as T allows), group 0 is the decode of the bits  random(at) . (1 0^L | 0 1^L) . random  under
    that chunk-wide CDF -- every interval around such a value straddles the dyadic point in front of the run, so the
    encoder counts about L pending bits there, resolved by a carry (1 0^L) or not (0 1^L) -- and the other groups hold
    the rest of the histogram, shuffled"""
    H = np.zeros(33, np.int64)
    H[:31] = T // 31
    H[:T % 31] += 1
    cdf = E.spec_cdf(H.astype(np.uint32), T)
    bits = list(rng.integers(0, 2, at)) + ([1] + [0] * L if carry else [0] + [1] * L) + list(rng.integers(0, 2, 4096))
    data = bytes(int("".join(map(str, bits[k:k + 8])), 2) for k in range(0, len(bits) - 7, 8))
    head = decode(cdf, data, G)
    rest = H - np.bincount(head, minlength=33)
    if (rest < 0).any():
        return None
    col = np.concatenate([head, rng.permutation(np.repeat(np.arange(33), rest))]).astype(np.uint8)
    assert np.array_equal(E.spec_cdf(np.bincount(col, minlength=33).astype(np.uint32), T), cdf)
    return col


def run_columns(rng) -> np.ndarray:
    """columns of RUN_T tokens that reach pending runs of 31, 32, 33 and more than 64 bits, and carries that ripple
    into two or more row words"""
    want = {"pending run of 31 bits", "pending run of 32 bits", "pending run of 33 bits", "pending run of > 64 bits",
            "carry into >= 2 row words"}
    have, cols = set(), []
    for L in [29, 30, 31, 32, 33, 34, 70, 100] * 8:
        for carry in (True, False):
            col = run_column(rng, L, carry, int(rng.integers(8, 200)))
            if col is None:
                continue
            cdf, _ = chunk_streams(col)
            it = stream_items(cdf, col[:G], "wide", False) & want
            if it - have:
                have |= it
                cols.append(col)
        if have == want:
            break
    return np.stack(cols)


def search(seed: int = 20261017, budget: int = 300, verbose=print):
    """the fixture: own-CDF columns (sym [N, 256], g [N], wide [N]) chosen greedily so that every own-CDF item of
    Coverage.wanted() and every mutant that can be killed has a witness; the longest own-CDF stream found; the
    chunk-wide-CDF columns of every T in BIG_T and of the width-1 chunk (big_wide, T = min_width_t())"""
    rng = np.random.default_rng(seed)
    have, killed, rows = set(), 0, []
    killable = sum(1 << k for k, m in enumerate(MUTANTS) if m not in EQUIVALENT)

    def consider(col, wide, force=False):
        nonlocal have, killed
        col = np.asarray(col, np.uint8)
        cdf = R.own_cdf(col)
        items = stream_items(cdf, col, "wide" if wide else "narrow", True)
        new = items - have
        kl = 0
        if (killed & killable) != killable and (new or force or len(rows) % 5 == 0):
            kl = kills(cdf, col, 5 if wide else 4)
        if new or (kl & ~killed & killable) or force:
            have |= items
            killed |= kl
            rows.append((col, wide))
            return True
        return False

    longest = longest_own_stream(rng)
    consider(longest, True, force=True)
    for t in (1, 2, 3, 4, 5, 255, 256):
        for wide in (True, False):
            top = 30 if wide else 14
            consider(np.full(t, top, np.uint8), wide)
            if t >= 2:
                col = np.zeros(t, np.uint8)
                col[t // 2] = top
                consider(col, wide)
    # span = 2^32 after the first symbol: a power-of-two width at an aligned start (count 8 of 256 at symbol 0)
    for wide in (True, False):
        top = 30 if wide else 14
        col = np.concatenate([np.zeros(8, np.uint8), rng.integers(1, top + 1, 248).astype(np.uint8)])
        consider(np.concatenate([col[:1], rng.permutation(col[1:])]), wide)
    for wide in (True, False):
        top = 30 if wide else 14
        for t in (256, 255, 128, 64, 17, 8, 5, 3):
            for col in R._hist_columns(rng, t, top, budget if t >= 255 else budget // 6):
                consider(col, wide)
            verbose(f"  {'wide' if wide else 'narrow'} t = {t}: {len(rows)} rows, {len(have)} items, killed {killed:#x}")
    sym = np.zeros((len(rows), G), np.uint8)
    g = np.zeros(len(rows), np.int16)
    for k, (col, wide) in enumerate(rows):
        sym[k, :col.size], g[k] = col, col.size
    out = dict(sym=sym, g=g, wide=np.array([w for _, w in rows], np.uint8),
               longest=np.int32(len(encode(R.own_cdf(longest), longest))), mutants=np.array(MUTANTS))
    frng = np.random.default_rng(seed + 1)
    for T in BIG_T:
        out[f"big_{T}"] = foreign_columns(T, frng)
    out["big_wide"] = np.stack([wide_column(frng, k) for k in (17, 16, 15)])
    out["big_runs"] = run_columns(frng)
    return out


def load():
    return np.load(FIXTURE)


def own_rows(fx):
    return R.own_rows(fx)


def big_columns(fx):
    """(T, columns [n, T]) of every chunk-wide-CDF set of the fixture"""
    out = [(T, fx[f"big_{T}"]) for T in BIG_T]
    out.append((int(fx["big_wide"].shape[1]), fx["big_wide"]))
    out.append((RUN_T, fx["big_runs"]))
    return out


def chunk_streams(col):
    """(cdf row, [(tok0, g) ...]) of a chunk column of more than 256 tokens under the chunk-wide CDF"""
    return R.foreign_groups(col)


# ------------------------------------------------------------------------------------------------ the device harness
ACSIM_SRC = os.path.join(HERE, "devsim", "acsim.cu")
ACSIM_LIB = os.path.join(HERE, "devsim", "libacsim.so")


def build_acsim(force: bool = False) -> str:
    """tests/devsim/acsim.cu compiled with the product's flags.  An in-tree library newer than its sources is used as it
    is; otherwise it is compiled next to its source, or -- when the tree is read-only -- into the temporary directory
    under a name that carries a hash of the sources, so that a stale library is never loaded and nothing is written
    into a tree that may not be written."""
    import hashlib
    import subprocess
    import tempfile
    import __graft_entry__ as g
    deps = [ACSIM_SRC, os.path.join(g.CSRC, "ac_core.cuh")]
    if not force and not g._stale(ACSIM_LIB, deps):
        return ACSIM_LIB
    out = ACSIM_LIB
    if not os.access(os.path.dirname(ACSIM_LIB), os.W_OK):
        h = hashlib.sha256(b"".join(open(d, "rb").read() for d in deps)).hexdigest()[:16]
        out = os.path.join(tempfile.gettempdir(), f"lmcache_b200_acsim_{os.getuid()}_{h}.so")
        if os.path.exists(out) and not force:
            return out
    tmp = f"{out}.{os.getpid()}.tmp"
    subprocess.check_call([g.NVCC] + g.NVCC_FLAGS + ["-o", tmp, ACSIM_SRC])
    os.replace(tmp, out)
    return out
