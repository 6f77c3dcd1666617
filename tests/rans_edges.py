"""The rANS coder (DESIGN.md 3.7) at its arithmetic and window edges: an independent statement of the stream format in
plain Python integers, traces of every coded and decoded symbol, kernel-shaped models of the encode step (rans_put) and
the decode loop (rans_decode_stream) that can be told to make one plausible mistake each (MUTANTS), and the seeded
search for the streams -- a histogram AND an order, since for rANS the order is the input -- that reach each edge and
tell each mutant from the spec (stored in tests/golden/rans_edges.npz by tests/golden/make_rans_edges.py).

Every CDF row comes from cdf_edges.spec_cdf, so every stream is one the product can produce: an own-CDF stream (a chunk
of g <= 256 tokens coded under its own histogram) or a group of a longer chunk coded under the chunk-wide CDF.

Format, one stream of g symbols under c[0..32] (c[32] := 65536), start(s) = c[s], f(s) = c[s + 1] - c[s]:
    encoder  x = 2^16; for i = g - 1 .. 0: if (x >> 16) >= f: push x & 0xffff, x >>= 16;  x = ((x / f) << 16) + x % f + start
    bytes    LE32(x), then the pushed halfwords in reverse push order, LE16 each
    decoder  x = LE32; for i = 0 .. g - 1: slot = x & 0xffff; s = max{s: c[s] <= slot}; x = f (x >> 16) + slot - start;
             if x < 2^16: x = (x << 16) | next LE16;  x == 2^16 at the end
The push in front of symbol i is the pull behind symbol i, and the remainder x % f is slot - start: remainder 0 and
f - 1 are the two ends of the decoder's search interval.

What the search settled about the edges one might ask for:
  * a dividend of the form 2^k - 1, k >= 24, cannot occur: without a push x = (q << 16) + r + start with
    r + start <= c[s + 1] - 1 <= 65534 for s <= 30, with one x < 2^16.  The steps where float(x) rounds up under
    round-to-nearest (where RZ and RN part) are common and are what the coverage asks for instead;
  * the longest stream-header a stream can have is 34 bytes (31 used symbols), not the 36 the row reserves;
  * a push on EVERY symbol of a 256-token group needs f = 1 for symbols with 8 tokens each, a chunk of a million tokens,
    and the first coded symbol never pushes (x = 2^16), so no pull follows the last decoded symbol.  An own-CDF step gains
    at most 8 bits, so own-CDF streams never push on neighbouring symbols.  What is reachable and asked for: groups
    under a chunk-wide CDF that outgrow the 96 halfwords of an own-CDF row, pushes on four consecutive symbols (symbols
    seen once in 8192 tokens, f = 9, 12.8 bits each) and a pull behind the last symbol but one;
  * two mutants are equivalent to the spec on every producible stream (EQUIVALENT), with the reason.

Used by tests/test_rans_edges_cpu.py, tests/test_gpu_rans_edges.py and the fixture generator."""
from __future__ import annotations

import os

import numpy as np

import cdf_edges as E

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "rans_edges.npz")

M32 = 0xFFFFFFFF
LOW = 1 << 16
G = 256                    # tokens per coder group
ROW_HALFWORDS = 96         # capacity of an own-CDF stream's row in encode_kernel
PROVEN_MAX_HALFWORDS = 95  # DESIGN.md 3.7
LONG_T = 8192              # the long chunk: a symbol seen once has f = 9 under its CDF
BIG_T = E.BIG_T + (LONG_T,)
BIAS = np.float32(0.99999952316284179688)

# ------------------------------------------------------------------------------------------------ mutants
ENC_MUTANTS = ("no_bias", "rn_convert", "no_fixup", "fixup_gt", "push_gt", "m65535")
DEC_MUTANTS = ("dec_lt", "no_or", "pull_le", "never_move", "move_wrong_half", "freq_hi")
MUTANTS = ENC_MUTANTS + DEC_MUTANTS
MUTANT_DOC = {
    "no_bias": "quotient estimate without the factor that biases it low: it can be q + 1, which the fix-up cannot repair",
    "rn_convert": "float(x) rounded to nearest instead of towards zero",
    "no_fixup": "no fix-up when the estimate is one short",
    "fixup_gt": "fix-up on r > f instead of r >= f",
    "push_gt": "the state sheds a halfword on (x >> 16) > f instead of >= f",
    "m65535": "q * m with m = 65535 - f",
    "dec_lt": "decoder search compares entry < key instead of entry <= key",
    "no_or": "decoder key (x << 16) without the | 0xffff",
    "pull_le": "decoder pulls a halfword on x <= 2^16 instead of x < 2^16",
    "never_move": "the halfword selector toggles but the two-word window never moves on",
    "move_wrong_half": "the window moves on after the LOWER half was taken",
    "freq_hi": "freq taken as entry >> 16 (the start) instead of entry & 0xffff",
}
EQUIVALENT = {
    "rn_convert": "RN raises float(x) by < 2^-24 relative, the bias lowers the estimate by 2^-21: the estimate stays at or "
                  "below the quotient, so only WHICH steps take the fix-up changes, never a state",
    "dec_lt": "entry == key needs freq == 0xffff, and no CDF row gives a symbol more than 65505 slots",
}


# ------------------------------------------------------------------------------------------------ tables
def table(cdf_row):
    """(start[32], freq[32]) as Python ints from an int16 / uint16 CDF row [33]; c[32] := 65536"""
    u = [int(v) & 0xFFFF for v in np.asarray(cdf_row).reshape(-1)]
    assert len(u) == 33
    u[32] = 65536
    return u[:32], [u[i + 1] - u[i] for i in range(32)]


def own_cdf(col) -> np.ndarray:
    """the CDF row an own-CDF stream of these symbols is coded under"""
    col = np.asarray(col)
    return E.spec_cdf(np.bincount(col, minlength=33).astype(np.uint16), col.size)


# ------------------------------------------------------------------------------------------------ the spec
def encode(cdf_row, symbols, trace=None) -> bytes:
    """the stream of `symbols` (coded last first).  trace: a list that receives, per coded symbol in coding order,
    (i, s, x_before, pushed, f, start, q, r, x_after)"""
    start, freq = table(cdf_row)
    x, pushed = LOW, []
    for i in range(len(symbols) - 1, -1, -1):
        s = int(symbols[i])
        f, st, xb = freq[s], start[s], x
        p = (x >> 16) >= f
        if p:
            pushed.append(x & 0xFFFF)
            x >>= 16
        q, r = divmod(x, f)
        x = (q << 16) + r + st
        assert x <= M32
        if trace is not None:
            trace.append((i, s, xb, p, f, st, q, r, x))
    return x.to_bytes(4, "little") + b"".join(h.to_bytes(2, "little") for h in reversed(pushed))


def decode(cdf_row, data: bytes, g: int):
    """(symbols uint8 [g], final state): the format's decoder, by the book"""
    start, freq = table(cdf_row)
    x, pos = int.from_bytes(data[:4], "little"), 4
    out = np.zeros(g, np.uint8)
    for i in range(g):
        slot = x & 0xFFFF
        s = max(k for k in range(32) if start[k] <= slot)
        out[i] = s
        x = freq[s] * (x >> 16) + slot - start[s]
        if x < LOW:
            x = (x << 16) | int.from_bytes(data[pos:pos + 2], "little")
            pos += 2
    assert pos == len(data) or x != LOW
    return out, x


# ------------------------------------------------------------------------------------------------ the kernels' shape
def _f32_rz(x: int) -> np.float32:
    v = np.float32(x)
    return np.nextafter(v, np.float32(0)) if float(v) > x else v


def estimate(x: int, f: int, bump: int = 0, mut=None) -> int:
    """float32 model of rans_put's quotient estimate; bump: the reciprocal 1 ulp below / at / above the rounded 1 / f"""
    rc = np.float32(1) / np.float32(f)
    if bump:
        rc = np.nextafter(rc, np.float32(np.inf if bump > 0 else 0))
    fx = np.float32(x) if mut == "rn_convert" else _f32_rz(x)
    c = rc if mut == "no_bias" else np.float32(rc * BIAS)
    return int(np.floor(np.float32(fx * c)))


def classify(x: int, f: int) -> str:
    """'taken' / 'not taken' when the fix-up is certain whatever the reciprocal's last bit, else 'depends'"""
    q = x // f
    est = {estimate(x, f, b) for b in (-1, 0, 1)}
    assert est <= {q, q - 1}, (x, f, est)
    return "taken" if est == {q - 1} else "not taken" if est == {q} else "depends"


def encode_as_kernel(cdf_row, symbols, mut=None) -> bytes:
    """rans_put step by step in wrapping 32-bit arithmetic, with the float32 estimate; mut: one of ENC_MUTANTS"""
    start, freq = table(cdf_row)
    x, pushed = LOW, []
    for i in range(len(symbols) - 1, -1, -1):
        s = int(symbols[i])
        f, st = freq[s], start[s]
        xh = x >> 16
        if (xh > f) if mut == "push_gt" else (xh >= f):
            pushed.append(x & 0xFFFF)
            x = xh
        q = estimate(x, f, 0, mut) & M32
        m = (65535 if mut == "m65535" else 65536) - f
        a = (q * m + x) & M32
        r = (a - (q << 16)) & M32
        x = (a + st) & M32
        if mut != "no_fixup" and ((r > f) if mut == "fixup_gt" else (r >= f)):
            x = (x + m) & M32
    return x.to_bytes(4, "little") + b"".join(h.to_bytes(2, "little") for h in reversed(pushed))


def decode_as_kernel(cdf_row, data: bytes, g: int, odd: int = 0, mut=None, nsteps: int = 5, trace=None,
                     before: bytes = b"\x5a\x5a", after: bytes = b"\xa5" * 16):
    """rans_decode_stream: the stream starts `odd` halfwords into an aligned word (foreign bytes on both sides), a
    two-word window with one word of look-ahead, the packed table, a fixed-depth search.  trace receives per symbol
    (slot, leaf, pulled, window_moved).  Returns (symbols, final state)."""
    start, freq = table(cdf_row)
    pk = [(start[i] << 16) | (freq[i] & 0xFFFF) for i in range(32)]
    buf = before * odd + bytes(data) + after
    buf += bytes(-len(buf) % 4)

    def word(i):
        return int.from_bytes(buf[4 * i:4 * i + 4], "little")
    w0, w1 = word(0), word(1)
    x = (((w1 << 32) | w0) >> (16 * odd)) & M32
    cur, nxt, idx, hi = w1, word(2), 3, bool(odd)
    out = np.zeros(g, np.uint8)
    for i in range(g):
        key = ((x << 16) & M32) | (0 if mut == "no_or" else 0xFFFF)
        s, step = 0, 1 << (nsteps - 1)
        while step:
            e = pk[s + step]
            if (e < key) if mut == "dec_lt" else (e <= key):
                s += step
            step >>= 1
        e = pk[s]
        out[i] = s
        fr = (e >> 16) if mut == "freq_hi" else (e & 0xFFFF)
        x = (fr * (x >> 16) + (((key - e) & M32) >> 16)) & M32
        pulled = (x <= LOW) if mut == "pull_le" else (x < LOW)
        moved = False
        if pulled:
            x = ((x << 16) & M32) | ((cur >> 16) if hi else (cur & 0xFFFF))
            moved = False if mut == "never_move" else (not hi) if mut == "move_wrong_half" else hi
            hi = not hi
            if moved:
                cur, nxt, idx = nxt, word(idx), idx + 1
        if trace is not None:
            trace.append((key >> 16, s, pulled, moved))
    return out, x


def kills(cdf_row, col, nsteps: int = 5) -> int:
    """bit k set <=> MUTANTS[k] gives other bytes (encoder) or other symbols / final state (decoder, either phase)"""
    col = np.asarray(col, np.uint8)
    want = encode(cdf_row, col)
    out = 0
    for k, name in enumerate(MUTANTS):
        if name in ENC_MUTANTS:
            bad = encode_as_kernel(cdf_row, col, name) != want
        else:
            bad = False
            for odd in (0, 1):
                got, xf = decode_as_kernel(cdf_row, want, col.size, odd, name, nsteps)
                bad = bad or xf != LOW or not np.array_equal(got, col)
        out |= int(bad) << k
    return out


# ------------------------------------------------------------------------------------------------ what a stream reaches
def max_run(flags) -> int:
    best = run = 0
    for v in flags:
        run = run + 1 if v else 0
        best = max(best, run)
    return best


def stream_items(tr, g: int, plane: str, own: bool, model: bool = False) -> set:
    """coverage items of one stream from its encode trace.  plane: 'wide' (32-entry plane, 5-step search) or 'narrow'
    (16-entry plane, 4-step search).  model: also classify every step's fix-up with the float32 model (slow)."""
    it = set()
    pushed = [False] * g
    for (i, s, xb, p, f, st, q, r, xa) in tr:
        pushed[i] = p
        xd = xb >> 16 if p else xb
        xh = xb >> 16
        if r == 0:
            it.add(f"remainder 0, symbol {s}, {plane} plane")
        if r == f - 1:
            it.add(f"remainder f - 1, symbol {s}, {plane} plane")
        if xh == f:
            it.add("x >> 16 == f (push)")
        if xh == f - 1:
            it.add("x >> 16 == f - 1 (no push)")
        if q == 1:
            it.add("q = 1")
        if q >= 65000:
            it.add("q >= 65000")
        if xd >= 1 << 31:
            it.add("dividend >= 2^31")
        if float(np.float32(xd)) > xd:
            it.add("float(x) rounds up under RN")
        if not own and f < 16:
            it.add("f < 16 under a chunk-wide CDF")
        if own and g in (1, 2, 255, 256):
            lo, hi = own_f_range(g)
            if f == lo:
                it.add(f"smallest f of t = {g}")
            if f == hi:
                it.add(f"largest f of t = {g}")
        if r == 0:
            it.add("fix-up certainly taken")           # estimate < q whatever the reciprocal's last bit
        elif model:
            c = classify(xd, f)
            if c != "depends":
                it.add("fix-up certainly " + c)
    n = sum(pushed)
    full = 4 * (g // 4)
    for i in range(g):
        if pushed[i]:
            it.add(f"pull at position {i % 4} of the four-symbol trip" if i < full else "pull in the tail loop")
    assert not pushed[g - 1]                    # the first coded symbol meets x = 2^16: a push would need f = 1
    if g >= 2 and pushed[g - 2]:
        it.add("pull behind the last symbol but one")
    if max_run(pushed) >= 4:
        it.add("pulls on four consecutive symbols")
    if own:
        it.add(f"gt = {g}")
    else:
        if n > ROW_HALFWORDS:
            it.add("a chunk-wide-CDF group longer than an own-CDF row (96 halfwords)")
        if g < G:
            it.add(f"partial last group, gt mod 4 = {g % 4}")
    return it


def own_f_range(t: int):
    """(smallest, largest) f an own-CDF stream of t tokens can have: a symbol seen once among two, and a lone symbol"""
    lone = np.zeros(33, np.uint16)
    lone[0] = t
    hi = table(E.spec_cdf(lone, t))[1][0]
    if t == 1:
        return hi, hi
    two = np.zeros(33, np.uint16)
    two[0], two[1] = 1, t - 1
    return table(E.spec_cdf(two, t))[1][0], hi


class Coverage:
    """what the streams a test really coded reach: stream_items of every trace, plus what depends on where the stream
    lies in the payload (phase: its first rANS byte at 0 or 2 mod 4) and on its neighbours"""

    def __init__(self, longest: int):
        self.items, self.longest = set(), int(longest)

    def add(self, items, halfwords: int, phase: int, own: bool, header: int = 0, neighbours=()):
        self.items |= set(items)
        if own:
            n = "the most" if halfwords == self.longest else str(halfwords) if halfwords <= 3 else None
            if n:
                self.items.add(f"{n} halfwords, stream at {phase} mod 4")
            if halfwords == self.longest and header == 34:
                self.items.add("the longest stream behind the longest header (34 bytes)")
            if halfwords == self.longest and len(neighbours) == 2 and all(v == 4 for v in neighbours):
                self.items.add("the longest stream between 4-byte streams")

    @staticmethod
    def wanted() -> list:
        w = [f"remainder {e}, symbol {s}, {pl} plane" for e in ("0", "f - 1")
             for pl, top in (("wide", 31), ("narrow", 15)) for s in range(top)]
        w += ["x >> 16 == f (push)", "x >> 16 == f - 1 (no push)", "q = 1", "q >= 65000", "dividend >= 2^31",
              "float(x) rounds up under RN", "f < 16 under a chunk-wide CDF", "fix-up certainly taken",
              "fix-up certainly not taken"]
        w += [f"{e} f of t = {t}" for e in ("smallest", "largest") for t in (1, 2, 255, 256)]
        w += [f"{n} halfwords, stream at {ph} mod 4" for n in ("0", "1", "2", "3", "the most") for ph in (0, 2)]
        w += [f"pull at position {k} of the four-symbol trip" for k in range(4)]
        w += ["pull in the tail loop", "pull behind the last symbol but one", "pulls on four consecutive symbols"]
        w += [f"gt = {g}" for g in (1, 2, 3, 4, 5, 253, 254, 255, 256)]
        w += [f"partial last group, gt mod 4 = {k}" for k in range(4)]
        w += ["a chunk-wide-CDF group longer than an own-CDF row (96 halfwords)",
              "the longest stream behind the longest header (34 bytes)", "the longest stream between 4-byte streams"]
        return w

    def missing(self) -> list:
        return [w for w in self.wanted() if w not in self.items]


# ------------------------------------------------------------------------------------------------ naming a failure
def first_bad_step(cdf_row, col, got: bytes) -> str:
    """where a stream that should be encode(cdf_row, col) went wrong.  Halfwords leave the encoder in coding order and
    lie in the stream back to front, so the stream is compared from its END: the first halfword that differs names the
    push it came from, and the faulty step lies between the push before it and that one."""
    tr = []
    want = encode(cdf_row, col, tr)
    if got == want:
        return "stream equals the spec's"
    hw = lambda b: [int.from_bytes(b[k:k + 2], "little") for k in range(len(b) - 2, 2, -2)]    # coding order
    a, b = hw(want), hw(bytes(got))
    k = next((j for j in range(min(len(a), len(b))) if a[j] != b[j]), min(len(a), len(b)))
    pushes = [n for n, stp in enumerate(tr) if stp[3]]
    lo = pushes[k - 1] if k else 0
    hi = pushes[k] if k < len(pushes) else len(tr) - 1
    i, s, xb, p, f, st, q, r, xa = tr[lo]
    return (f"{len(got)} bytes, spec {len(want)}; halfword {k} in coding order differs (got "
            f"{b[k] if k < len(b) else None}, spec {a[k] if k < len(a) else 'the final state'}): the first wrong step is "
            f"among coding steps {lo}..{hi} (tokens {tr[lo][0]} down to {tr[hi][0]}); step {lo}: token {i} symbol {s} "
            f"x = {xb:#x} pushed = {p} f = {f} start = {st} q = {q} r = {r} -> x = {xa:#x}; final state got "
            f"{int.from_bytes(bytes(got[:4]), 'little'):#x}, spec {int.from_bytes(want[:4], 'little'):#x}")


# ------------------------------------------------------------------------------------------------ the search
def _hist_columns(rng, t: int, top: int, n: int):
    """n random columns of t tokens over symbols 0..top: even, skewed and random histograms; shuffled, sorted into runs,
    or with the rare symbols together"""
    for k in range(n):
        K = int(rng.integers(1, min(t, top + 1) + 1)) if k % 3 else min(t, top + 1)
        syms = np.sort(rng.choice(top + 1, K, replace=False))
        style = k % 4
        if style == 0:
            cnt = np.full(K, t // K)
            cnt[: t % K] += 1
        elif style == 1:
            cnt = np.ones(K, np.int64)
            cnt[int(rng.integers(0, K))] += t - K
        else:
            cnt = 1 + rng.multinomial(t - K, rng.dirichlet(np.full(K, 0.6)))
        col = np.repeat(syms, cnt).astype(np.uint8)
        order = (k // 4) % 3
        if order == 0:
            col = rng.permutation(col)
        elif order == 1 and K > 1:
            col = np.concatenate([rng.permutation(col[col != syms[np.argmax(cnt)]]), col[col == syms[np.argmax(cnt)]]])
            if k % 8 >= 4:
                col = col[::-1].copy()
        yield col


def longest_own_stream(top: int = 30, t: int = G):
    """directed search for the longest own-CDF stream: top + 1 symbols as even as t tokens allow, the order chosen
    greedily back to front -- at every step the symbol still owed whose step gains the most over its ideal
    log2(65536 / f) bits (a small quotient and a high start round the state up the most).  Returns the column."""
    K = top + 1
    cnt = np.full(K, t // K)
    cnt[K - t % K:] += 1                                      # the high symbols (large start) get the extra tokens
    hist = np.zeros(33, np.uint16)
    hist[:K] = cnt
    start, freq = table(E.spec_cdf(hist, t))
    left, x, rev = cnt.tolist(), LOW, []
    for _ in range(t):
        best = None
        for s in range(K):
            if not left[s]:
                continue
            xx = x >> 16 if (x >> 16) >= freq[s] else x
            xn = ((xx // freq[s]) << 16) + xx % freq[s] + start[s]
            gain = np.log2(xn / xx) - np.log2(65536 / freq[s])
            if best is None or gain > best[0]:
                best = (gain, s, xn)
        rev.append(best[1])
        left[best[1]] -= 1
        x = best[2]
    return np.array(rev[::-1], np.uint8)


def foreign_columns(T: int, rng, top: int = 30, n: int = 6) -> np.ndarray:
    """columns [n, T] of a chunk of T > 256 tokens: one common symbol everywhere except in a few groups, which hold the
    chunk's rare symbols -- every one of them (count 1 or a handful each) or runs of a few.  Under the chunk-wide CDF a
    rare symbol costs up to 13 bits, so those groups are long streams with pushes on consecutive symbols."""
    cols = np.zeros((n, T), np.uint8)
    ngroups = -(-T // G)
    for k in range(n):
        common = int(rng.integers(0, top + 1))
        col = np.full(T, common, np.uint8)
        rare = np.array([s for s in range(top + 1) if s != common])
        for gi in rng.choice(ngroups, size=min(ngroups, 1 + k % 3), replace=False):
            a, b = gi * G, min(T, gi * G + G)
            if k % 2 == 0:
                col[a:b] = rng.choice(rare, b - a)                         # every token of the group is rare
            else:
                pos = a + rng.choice(b - a, size=max(1, (b - a) // 3), replace=False)
                col[pos] = rng.choice(rare[1:7], pos.size)
        if k == n - 2:
            col[:] = common                                                # every rare symbol once, side by side, at
            col[G - rare.size - 1:G - 1] = rng.permutation(rare)           # the end of the first group
        if k == n - 1:
            col[T - 1] = rare[0]                                           # the last token of the chunk alone is rare
        cols[k] = col
    return cols


def search(seed: int = 20240607, budget: int = 800, verbose=print):
    """the fixture: own-CDF columns (symbols [N, 256], g [N], plane [N]: 1 wide, 0 narrow) chosen greedily so that every
    own-CDF item of Coverage.wanted() and every mutant that can be killed has a witness, the longest stream found, and the
    chunk-wide-CDF columns of every T in BIG_T"""
    rng = np.random.default_rng(seed)
    wanted = set(Coverage.wanted())
    have, killed, rows = set(), 0, []
    killable = sum(1 << k for k, m in enumerate(MUTANTS) if m not in EQUIVALENT)

    def consider(col, wide, force=False):
        nonlocal have, killed
        plane = "wide" if wide else "narrow"
        tr = []
        cdf = own_cdf(col)
        data = encode(cdf, col, tr)
        n = (len(data) - 4) // 2
        items = stream_items(tr, col.size, plane, True) & wanted
        new = items - have
        kl = 0
        if n <= 3 and f"{n} halfwords" not in have:
            new.add(f"{n} halfwords")
        if (killed & killable) != killable and (new or len(rows) % 7 == 0 or force):
            kl = kills(cdf, col, 5 if wide else 4)
        if new or (kl & ~killed & killable) or force:
            if "fix-up certainly not taken" not in have:
                new |= stream_items(tr, col.size, plane, True, model=True) & wanted
            have |= new | items
            killed |= kl
            rows.append((col, wide))
            return True
        return False

    longest = longest_own_stream()
    consider(longest, True, force=True)
    best = (len(encode(own_cdf(longest), longest)) - 4) // 2
    # directed: the token counts and f extremes, short streams
    for t in (1, 2, 3, 4, 5, 253, 254, 255, 256):
        for wide in (True, False):
            top = 30 if wide else 14
            consider(np.full(t, top, np.uint8), wide, force=t in (1, 2, 255, 256))       # lone symbol: largest f
            if t >= 2:
                col = np.full(t, 0, np.uint8)
                col[t // 2] = top                                                        # seen once: smallest f
                consider(col, wide, force=t in (2, 255, 256))
    for wide in (True, False):
        top = 30 if wide else 14
        for t in (256, 255, 64, 17, 254, 253, 8, 6, 5, 4, 3):
            for col in _hist_columns(rng, t, top, budget if t >= 253 else budget // 8):
                consider(col, wide)
            verbose(f"  {'wide' if wide else 'narrow'} t = {t}: {len(rows)} rows, "
                    f"{len([w for w in wanted if w in have])} items, mutants killed {killed:#x}")
    sym = np.zeros((len(rows), G), np.uint8)
    g = np.zeros(len(rows), np.int16)
    for k, (col, wide) in enumerate(rows):
        sym[k, :col.size], g[k] = col, col.size
    out = dict(sym=sym, g=g, wide=np.array([w for _, w in rows], np.uint8), longest=np.int32(best),
               mutants=np.array(MUTANTS))
    out.update(foreign_set(seed))
    return out


def foreign_set(seed: int) -> dict:
    rng = np.random.default_rng(seed + 1)
    return {f"big_{T}": foreign_columns(T, rng) for T in BIG_T}


def load():
    return np.load(FIXTURE)


def own_rows(fx):
    """(column, wide) of every own-CDF fixture row"""
    return [(fx["sym"][k, :int(fx["g"][k])], bool(fx["wide"][k])) for k in range(fx["g"].size)]


def foreign_groups(col):
    """(cdf row, [(tok0, g) ...]) of a chunk column of more than 256 tokens: its groups under the chunk-wide CDF"""
    col = np.asarray(col)
    T = col.size
    return E.spec_cdf(np.bincount(col, minlength=33).astype(np.uint32), T), [(a, min(G, T - a)) for a in range(0, T, G)]


# ------------------------------------------------------------------------------------------------ the device sweep
DEVSIM_SRC = os.path.join(HERE, "devsim", "devsim.cu")
DEVSIM_LIB = os.path.join(HERE, "devsim", "libdevsim.so")


def build_devsim(force: bool = False) -> str:
    """compile tests/devsim/devsim.cu with the product's flags when it is missing or older than its sources.  Without a
    compiler an up-to-date or travelled library is used as it is; with neither, this raises."""
    import shutil
    import subprocess
    import __graft_entry__ as g
    deps = [DEVSIM_SRC, os.path.join(g.CSRC, "ac_core.cuh")]
    have_nvcc = os.path.exists(g.NVCC) or shutil.which(g.NVCC) is not None
    if have_nvcc and (force or g._stale(DEVSIM_LIB, deps)):
        subprocess.check_call([g.NVCC] + g.NVCC_FLAGS + ["-o", DEVSIM_LIB, DEVSIM_SRC])
    if not os.path.exists(DEVSIM_LIB):
        raise RuntimeError("tests/devsim/libdevsim.so is missing and there is no nvcc to build it")
    return DEVSIM_LIB


# ------------------------------------------------------------------------------------------------ driving the kernels
def plane_kind(plane_max: int) -> str:
    """decode_kernel searches 4 steps on planes of MAX <= 7 (symbols 0..14) and 5 steps on the others"""
    return "narrow" if plane_max <= 7 else "wide"


def own_tile(fx, t: int, plane_max) -> np.ndarray:
    """sym uint8 [P, t, C] of one chunk of t <= 256 tokens: channel 0 of every plane is symbol 0 throughout (it pins the
    row maxima, and is a 4-byte stream); the other channels of plane p hold the fixture's columns of t tokens whose top
    symbol the plane can hold, in fixture order, repeated to fill.  At t = 256 the longest stream is channel 1 and an
    all-zero column channel 2: a long stream between two 4-byte ones."""
    cols = [col for col, _ in own_rows(fx) if col.size == t]
    if t == G:
        cols.insert(1, np.zeros(G, np.uint8))
    C = 1 + len(cols)
    sym = np.zeros((len(plane_max), t, C), np.uint8)
    for p, M in enumerate(plane_max):
        fit = [c for c in cols if c.max() <= 2 * M]
        for c in range(1, C):
            if fit:
                sym[p, :, c] = fit[(c - 1) % len(fit)]
    return sym


def big_tile(fx, T: int, plane_max) -> np.ndarray:
    """sym uint8 [P, T, C] of one chunk of T > 256 tokens: the fixture's columns, clipped to each plane's top symbol"""
    cols = fx[f"big_{T}"]
    sym = np.zeros((len(plane_max), T, 1 + cols.shape[0]), np.uint8)
    for p, M in enumerate(plane_max):
        sym[p, :, 1:] = np.minimum(cols, 2 * M).T
    return sym


class Expect:
    """the spec's streams for tiles of prescribed symbols, cached by (CDF row, column), and the coverage they amount to"""

    def __init__(self, longest: int):
        self.cov = Coverage(longest)
        self._cache = {}

    def stream(self, cdf_row, col, kind: str, own: bool):
        key = (cdf_row.tobytes(), col.tobytes(), kind, own)
        if key not in self._cache:
            tr = []
            data = encode(cdf_row, col, tr)
            self._cache[key] = (data, stream_items(tr, col.size, kind, own, model=own and len(data) < 60))
        return self._cache[key]

    def group(self, sym, cdfs, plane_max, tok0: int, g: int, own: bool, hdr=None):
        """streams [P][C] of tokens [tok0, tok0 + g) under cdfs [P, C, 33], recorded in the coverage as they lie in a
        payload: back to back in (plane, channel) order, each behind its version-3 header of hdr[p][c] bytes if given"""
        P, _, C = sym.shape
        out, off = [], 0
        for p in range(P):
            kind = plane_kind(int(plane_max[p]))
            row = [self.stream(cdfs[p, c], np.ascontiguousarray(sym[p, tok0:tok0 + g, c]), kind, own) for c in range(C)]
            for c, (data, items) in enumerate(row):
                h = int(hdr[p][c]) if hdr is not None else 0
                nb = () if hdr is not None or not 0 < c < C - 1 else (len(row[c - 1][0]), len(row[c + 1][0]))
                self.cov.add(items, (len(data) - 4) // 2, (off + h) % 4, own, h, nb)
                off += h + len(data)
            out.append([d for d, _ in row])
        return out


def own_cdfs(sym) -> np.ndarray:
    """int16 [P, C, 33]: the CDF row of every column of sym [P, t, C]"""
    P, t, C = sym.shape
    hist = np.zeros((P, C, 33), np.uint32)
    for p in range(P):
        for c in range(C):
            hist[p, c] = np.bincount(sym[p, :, c], minlength=33)
    return E.spec_cdf(hist, t), hist


def own_ts(fx) -> list:
    return sorted({int(g) for g in fx["g"]})


def plan_coverage(fx, plane_max, nbs) -> Coverage:
    """everything the GPU suite's tiles reach, computed from the spec alone (the GPU suite asserts that the product's
    bytes ARE the spec's, so this is what it ran)"""
    ex = Expect(int(fx["longest"]))
    for t in own_ts(fx):
        sym = own_tile(fx, t, plane_max)
        cdfs, hist = own_cdfs(sym)
        ex.group(sym, cdfs, plane_max, 0, t, True)
        ex.group(sym, cdfs, plane_max, 0, t, True, E.header_lens(hist, nbs))
    for T in BIG_T:
        sym = big_tile(fx, T, plane_max)
        cdfs, _ = own_cdfs(sym)
        for a in range(0, T, G):
            ex.group(sym, cdfs, plane_max, a, min(G, T - a), False)
    return ex.cov
