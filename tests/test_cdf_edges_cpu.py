"""CPU: the CDF-normaliser witness set (tests/golden/cdf_edges.npz, CDF rows made by the reference's own functions)
against the numpy spec and its exact Fraction form (tests/cdf_edges.py), the CPU oracle, the product's host shim and
the host build of CdfAccum / CdfAccum2 (tests/hostsim); proof that every emulated variant of the arithmetic is caught
where the search found it can be; the whole search regenerated equal to the committed set; and the version-3 stream
header (hdr_write_host / hdr_len) against the oracle's packer at every header length that exists."""
import ctypes
import os

import numpy as np
import pytest

from oracle import oracle as O

import cdf_edges as E

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def fx():
    return {k: v for k, v in E.load().items()}


@pytest.fixture(scope="module")
def sim():
    S = ctypes.CDLL(os.path.join(HERE, "hostsim", "libhostsim.so"))
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    S.sim_cdf.argtypes = [vp, i32, vp]
    S.sim_cdf_skip.argtypes = [vp, i32, ctypes.c_uint32, vp]
    S.sim_hdr_write.argtypes = [vp, i32, vp]
    S.sim_hdr_len.argtypes = [ctypes.c_uint32, i32]
    return S


def _P(a):
    return ctypes.c_void_p(a.ctypes.data)


def _row(fx, i, got=None):
    """names a fixture row: its histogram, t, and the first entry where `got` leaves the reference's CDF row"""
    c, t = fx["counts"][i], int(fx["t"][i])
    s = f"row {i} ({E.DOMAINS[fx['domain'][i]]}), t = {t}, histogram {{symbol: count}} = " \
        f"{ {int(k): int(c[k]) for k in np.flatnonzero(c)} }"
    if got is not None:
        want = fx["cdf"][i]
        e = int(np.flatnonzero(np.asarray(got) != want)[0])
        s += f": cdf[{e}] = {int(np.asarray(got)[e]) & 0xFFFF}, the reference has {int(want[e]) & 0xFFFF}"
    return s


def _assert_rows(fx, got, what):
    bad = np.flatnonzero((got != fx["cdf"]).any(axis=1))
    assert bad.size == 0, f"{what} != reference CDF on {bad.size} rows; first: {_row(fx, bad[0], got[bad[0]])}"


def _by_t(fx, fn):
    """fn(counts [n, 33] of one t, t) -> [n, 33], applied per token count"""
    out = np.zeros(fx["cdf"].shape, np.int16)
    for t in np.unique(fx["t"]):
        s = fx["t"] == t
        out[s] = fn(fx["counts"][s], int(t))
    return out


def test_fixture_shape(fx):
    assert list(fx["variants"]) == list(E.VARIANTS) and fx["found"].shape == (len(E.DOMAINS), len(E.VARIANTS))
    assert fx["counts"].shape[0] < 5000 and os.path.getsize(E.FIXTURE) < 1 << 20
    assert (fx["counts"].sum(axis=1) == fx["t"]).all() and (fx["counts"][:, E.TOP_SYMBOL + 1:] == 0).all()
    t = fx["t"]
    assert set(E.BIG_T) <= set(t.tolist()) and {1, 2, 3, 17, 255, 256} <= set(t.tolist())
    assert (fx["counts"] == 256).any() and (fx["counts"] == 255).any() and (fx["counts"] == 1030).any()
    nz = (fx["counts"] > 0).sum(axis=1)
    assert nz.max() == 31 and nz.min() == 1
    for d in range(len(E.DOMAINS)):
        assert fx["ties"][d] > 0 and ((fx["kind"] == E.K_TIE) & (fx["domain"] == d)).any(), E.DOMAINS[d]


def test_spec_and_fraction_form_equal_the_reference(fx):
    """reference-made rows == spec_cdf == the spec in exact rationals, on every row; the exact form finds a tie exactly
    where the fp32 product sits on k + 0.5, ties go both ways (up to an even value, down to one), and every row stored as
    a tie has one"""
    _assert_rows(fx, _by_t(fx, E.spec_cdf), "spec_cdf")
    up = down = 0
    for i in range(fx["t"].size):
        c, t = fx["counts"][i], int(fx["t"][i])
        vals, ties = E.fraction_cdf(c.tolist(), t)
        assert vals[0] == 0 and vals[32] == 65536, _row(fx, i)
        assert np.array_equal(E.wrap16(vals), fx["cdf"][i]), "exact form: " + _row(fx, i, E.wrap16(vals))
        tie, odd = E.tie_entries(c[:32], t)
        assert np.flatnonzero(tie).tolist() == ties, _row(fx, i)
        assert bool(ties) or fx["kind"][i] != E.K_TIE, _row(fx, i)
        up += int(odd.sum())
        down += int((tie & ~odd).sum())
    assert up > 50 and down > 50, (up, down)


def test_oracle_equals_the_reference(fx):
    _assert_rows(fx, _by_t(fx, lambda c, t: O.cdf_from_counts(c.astype(np.uint32), t)), "oracle cdf_from_counts")

    def from_symbols(c, t):
        sym = np.stack([E.column(r) for r in c], axis=1).astype(np.int8)[None]          # [1, t, n]
        assert np.array_equal(O.counts(sym)[0], c)
        return O.cdf(sym)[0]
    _assert_rows(fx, _by_t(fx, from_symbols), "oracle cdf (symbols in)")


def test_host_shim_equals_the_reference(fx):
    from lmcache_b200.storage_backend.serde.cachegen_basics import cdf_from_counts
    _assert_rows(fx, _by_t(fx, cdf_from_counts), "host shim cdf_from_counts")


def test_hostsim_cdf_accumulators_equal_the_reference(fx, sim):
    """CdfAccum (sim_cdf: what cdf_kernel runs, any t) on every row; CdfAccum2 (sim_cdf_skip: the fused encoder and the
    decoder, t <= 256) skipping nothing, every unused symbol, and random subsets of them -- what the warp's common mask
    amounts to for one lane among 32"""
    rng = np.random.default_rng(11)
    out = np.zeros(33, np.uint16)
    for i in range(fx["t"].size):
        c, t = np.ascontiguousarray(fx["counts"][i].astype(np.uint32)), int(fx["t"][i])
        sim.sim_cdf(_P(c), t, _P(out))
        assert np.array_equal(out.view(np.int16), fx["cdf"][i]), "CdfAccum: " + _row(fx, i, out.view(np.int16))
        unused = int(sum(1 << int(k) for k in np.flatnonzero(c[:32] == 0)))
        for skip in [0, unused] + [unused & int(rng.integers(0, 1 << 32)) for _ in range(3)]:
            sim.sim_cdf_skip(_P(c), t, skip, _P(out))
            assert np.array_equal(out.view(np.int16), fx["cdf"][i]), \
                f"CdfAccum2 skipping {skip:#010x}: " + _row(fx, i, out.view(np.int16))


def test_every_variant_is_caught(fx):
    """the stored tags are what the variants do now; every stored witness disagrees with the reference-made row; in every
    domain where the search met a witness of a variant one is stored, and where it met none the variant equals the
    reference on every stored row of the domain.  What the search settled: a float32 running sum in any order cannot be
    told from the double one by histograms of two or three symbols at t <= 256, but many-symbol histograms at t <= 256 do
    tell it apart, so the default path has witnesses of every variant."""
    vi = {n: k for k, n in enumerate(E.VARIANTS)}
    differs = np.zeros((len(E.VARIANTS), fx["t"].size), bool)
    for k, name in enumerate(E.VARIANTS):
        differs[k] = (_by_t(fx, lambda c, t: E.variant_cdf(name, c, t)) != fx["cdf"]).any(axis=1)
        assert np.array_equal(differs[k], ((fx["tags"] >> k) & 1).astype(bool)), name
    for d, dom in enumerate(E.DOMAINS):
        s = fx["domain"] == d
        for k, name in enumerate(E.VARIANTS):
            if fx["found"][d, k] > 0:
                assert differs[k][s].any(), f"variant {name} ({E.VARIANT_DOC[name]}) not caught in domain {dom}"
            else:
                assert not differs[k][s].any(), (name, dom)
    found = fx["found"]
    for name in ("f32sum", "f32sum_rev", "f32sum_pair"):
        assert found[E.D_TWO, vi[name]] == 0 and found[E.D_THREE, vi[name]] == 0
        assert found[E.D_MANY, vi[name]] > 0 and found[E.D_BIG, vi[name]] > 0
    small = fx["t"] <= 256
    for k, name in enumerate(E.VARIANTS):
        assert differs[k][small].any() and differs[k][~small].any(), name
    # round-half-away is wrong on some ties, not all; truncation on most rows
    tie = fx["kind"] == E.K_TIE
    assert differs[vi["half_away"]][tie].any() and not differs[vi["half_away"]][tie].all()


def test_regenerated_search_equals_fixture(fx):
    """the whole deterministic search, run again: the same rows, kinds, witness and tie counts as the committed set, so
    the generator and the fixture cannot drift"""
    out = E.build_rows()
    for k in ("counts", "t", "kind", "domain", "tags", "found", "ties"):
        assert np.array_equal(out[k], fx[k]), k


def test_structure_of_every_row(fx):
    """c[0] = 0, c[32] = 65536 (wraps to 0), strictly increasing, every symbol keeps a slot (freq >= 1), and a symbol's
    share of the 65504 free slots is its share of the tokens to within one slot per preceding rounding"""
    u = fx["cdf"].view(np.uint16).astype(np.int64)
    assert (u[:, 0] == 0).all() and (u[:, 32] == 0).all()
    u[:, 32] = 65536
    freq = np.diff(u, axis=1)
    assert (freq >= 1).all()
    exact = fx["counts"][:, :32].astype(np.float64) / fx["t"][:, None] * 65504 + 1
    assert (np.abs(freq - exact) <= 1.01).all()


@pytest.mark.parametrize("nb", range(4, 33, 2))
def test_stream_header_every_length(sim, nb):
    """hdr_write_host / hdr_len (ac_core.cuh) against the oracle's packer and parser for every number of used symbols
    1 .. nb - 1 of the plane, at the first, last and random symbol subsets, with count bytes of 1 and 255 and the implied
    last count 1, 255 and 256"""
    rng = np.random.default_rng(nb)
    lengths = set()
    for nz in range(1, nb):
        subsets = [np.arange(nz), np.arange(nb - 1 - nz, nb - 1), np.sort(rng.choice(nb - 1, nz, replace=False))]
        for j, syms in enumerate(subsets):
            for last in (1, 255, 256):
                cnt = np.zeros(33, np.uint32)
                cnt[syms] = 1
                cnt[syms[-1]] = last
                if nz > 1 and j == 2:
                    cnt[syms[0]] = 255 if last == 1 else 1 + int(rng.integers(0, 200))
                t = int(cnt.sum())
                if t > 256 or (nz > 1 and last == 256):
                    continue
                out = np.full(48, 0xEE, np.uint8)
                n = sim.sim_hdr_write(_P(cnt), nb, _P(out))
                mask = E.mask_of(cnt)
                assert n == sim.sim_hdr_len(mask, nb) == E.header_len(mask, nb) and n % 2 == 0 and n <= 36
                assert (out[n:] == 0xEE).all()
                pl, half = O.v3_pack(cnt.reshape(1, 1, 33), [nb], np.array([[4]], np.int32), np.zeros(4, np.uint8))
                assert bytes(out[:n]) == pl[:n].tobytes() and int(half[0, 0]) * 2 == n + 4, (nb, nz, syms)
                back, ln, _ = O.v3_unpack(pl, half, [nb], t)
                assert np.array_equal(back[0, 0], cnt) and int(ln[0, 0]) == 4
                lengths.add(n)
    mb = (nb + 7) // 8
    assert lengths == set(range(mb + (mb & 1), mb + nb - 2 + ((mb + nb) & 1) + 1, 2)), sorted(lengths)


def test_kv_for_symbols_quantises_to_the_prescribed_symbols():
    """the inputs the GPU tests build: x = s - MAX with every row's maximum pinned to MAX quantise to s exactly, on every
    MAX and in both dtypes, by the oracle's quantiser; the stored maxima are MAX"""
    import quant_edges as Q
    L = 15
    kb, vb, mk, mv = Q.plane_maxes(L)
    pmax = np.array(mk + mv)
    rng = np.random.default_rng(3)
    t, C = 9, 20
    sym = np.stack([rng.integers(0, 2 * M + 1, size=(t, C)) for M in pmax]).astype(np.uint8)
    sym[:, :, 0] = 0
    sym[:, 0, 1] = 2 * pmax
    for dt in (0, 1):
        planes = E.kv_for_symbols(sym, pmax, dt)
        kv = np.ascontiguousarray(planes.reshape(2, L, t, C).transpose(1, 0, 2, 3))
        got, maxes = O.quantize(kv, dt, kb, vb)
        assert np.array_equal(got.view(np.uint8), sym)
        assert np.array_equal(maxes.reshape(2 * L, t), np.broadcast_to(Q.from_f32(pmax.astype(np.float32), dt)[:, None],
                                                                      (2 * L, t)))
