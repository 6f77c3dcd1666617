"""CPU: the quantiser / dequantiser witness set (tests/golden/quant_edges.npz) against the spec of tests/quant_edges.py,
the CPU oracle and the host build of the kernels' arithmetic (tests/hostsim); proof that every emulated variant of the
arithmetic the set claims to catch is caught; the spec itself against a float64 / Fraction computation; and a
regenerated slice of the set equal to the committed one."""
import ctypes
import os

import numpy as np
import pytest

from oracle import oracle as O

import quant_edges as Q

HERE = os.path.dirname(os.path.abspath(__file__))
C = 37          # packed row width for the CPU checks: a partial 8-wide vector


@pytest.fixture(scope="module")
def fx():
    return Q.load()


@pytest.fixture(scope="module")
def sim():
    S = ctypes.CDLL(os.path.join(HERE, "hostsim", "libhostsim.so"))
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    S.sim_quant_row.argtypes = [vp, i32, i32, ctypes.c_uint16, ctypes.c_float, vp]
    S.sim_dequant_row.argtypes = [vp, i32, ctypes.c_uint16, i32, ctypes.c_float, i32, vp]
    return S


def _P(a):
    return ctypes.c_void_p(a.ctypes.data)


def _bins(MAX):
    return np.array([2 * (MAX + 1)], np.float32)


def test_fixture_shape(fx):
    """every (dtype, MAX) has ties, specials and random pairs; stored witnesses per variant are the scan's, capped"""
    assert list(fx["mutants"]) == list(Q.MUTANTS)
    for dt in Q.DTYPES:
        x, m, mx, kind, mut = Q.fixture_pairs(fx, dt)
        scan = fx[f"{Q.DT_NAME[dt]}/scan_count"]
        ties = fx[f"{Q.DT_NAME[dt]}/ties"]
        for M in Q.MAXES:
            s = mx == M
            assert ties[M - 1] > 0 and int(((kind[s] & Q.K_TIE) != 0).sum()) == ties[M - 1], (dt, M)
            assert ((kind[s] & Q.K_SPECIAL) != 0).any() and ((kind[s] & Q.K_RANDOM) != 0).any()
            for bit, name in enumerate(Q.MUTANTS):
                n = int(((mut[s] >> bit) & 1).sum())
                assert n == Q.cap_pick(int(scan[M - 1, bit])).size, (dt, M, name)
        fin = ~Q.is_nan_bits(m, dt)
        assert ((x[fin] & 0x7FFF) <= m[fin]).all(), "a pair's |x| exceeds its maximum"


@pytest.mark.parametrize("dt", Q.DTYPES, ids=Q.DT_NAME)
def test_spec_equals_oracle_and_hostsim(fx, sim, dt):
    """the fixture's pairs, packed into rows: spec_absmax / spec_quant / spec_dequant == the oracle's quantize and
    dequantize (both output dtypes) == the host build of quant_factor / quant_symbol / dequant_lut / dequant_value; the
    only latitude is NaN against NaN in the maxima and values of NaN-maximum rows"""
    for M in Q.MAXES:
        x, m, _, _, _ = Q.fixture_pairs(fx, dt, M)
        rows, rmax = Q.pack_rows(x, m, C, dt)
        assert np.array_equal(Q.spec_absmax(rows), rmax) or Q.eq_nan(Q.spec_absmax(rows), rmax, dt).all()
        want = Q.spec_quant(rows, rmax[:, None], M, dt)
        # the pairs themselves: each one's spec symbol is the one its packed row holds at its value
        assert np.array_equal(Q.spec_quant(x, m, M, dt)[:8], Q.spec_quant(x[:8], m[:8], M, dt))
        kv = np.ascontiguousarray(np.stack([rows, rows])[None])            # [1, 2, R, C]
        sym, maxes = O.quantize(kv, dt, _bins(M), _bins(M))
        assert Q.eq_nan(maxes[0, 0], rmax, dt).all() and Q.eq_nan(maxes[1, 0], rmax, dt).all()
        bad = np.argwhere(sym[0].view(np.uint8) != want)
        assert bad.size == 0, (f"oracle quantize != spec, MAX {M} dt {dt}: first x={rows[tuple(bad[0])]:#06x} "
                               f"m={rmax[bad[0][0]]:#06x}")
        assert np.array_equal(sym[1].view(np.uint8), want)
        for out_dt in Q.DTYPES:
            dq = O.dequantize(sym.view(np.uint8), maxes, dt, _bins(M), _bins(M), out_dt)
            wd = Q.spec_dequant(want, maxes[0, 0][:, None], M, dt, out_dt)
            assert Q.eq_nan(dq[0, 0], wd, out_dt).all(), (M, dt, out_dt)
            assert Q.eq_nan(dq[0, 1], wd, out_dt).all()
        got = np.zeros(C, np.uint8)
        dq = np.zeros(C, np.uint16)
        for r in range(rows.shape[0]):
            row = np.ascontiguousarray(rows[r])
            sim.sim_quant_row(_P(row), dt, C, int(rmax[r]), float(M), _P(got))
            assert np.array_equal(got, want[r]), (M, dt, r, hex(int(rmax[r])))
            for out_dt in Q.DTYPES:
                sim.sim_dequant_row(_P(got), C, int(rmax[r]), dt, float(M), out_dt, _P(dq))
                assert Q.eq_nan(dq, Q.spec_dequant(want[r], rmax[r], M, dt, out_dt), out_dt).all(), (M, dt, r, out_dt)


@pytest.mark.parametrize("dt", Q.DTYPES, ids=Q.DT_NAME)
def test_every_variant_is_caught(fx, dt):
    """every emulated variant disagrees with the spec on the fixture wherever the exhaustive scan found a witness, and
    every stored witness of a variant is one"""
    scan = fx[f"{Q.DT_NAME[dt]}/scan_count"]
    caught = 0
    for M in Q.MAXES:
        x, m, _, _, mut = Q.fixture_pairs(fx, dt, M)
        for bit, name in enumerate(Q.MUTANTS):
            d = Q.mutant_differs(name, x, m, M, dt)
            if scan[M - 1, bit] > 0:
                assert d.any(), f"variant {name} not caught at MAX {M} ({Q.DT_NAME[dt]})"
                caught += 1
            mine = ((mut >> bit) & 1).astype(bool)
            assert d[mine].all(), (name, M, dt)
    assert caught >= 4 * len(Q.MAXES)


def test_scan_found_what_the_variants_should_break(fx):
    """sanity of the scan: round-half-away is wrong on some exact ties of every MAX but not on all of them;
    FMA contraction differs at some MAX; truncating conversions differ for every MAX >= 3 and output dtype; a flush of
    bf16 subnormal inputs is seen, fp16 inputs are never subnormal in fp32"""
    mi = {n: i for i, n in enumerate(Q.MUTANTS)}
    for dt in Q.DTYPES:
        scan = fx[f"{Q.DT_NAME[dt]}/scan_count"]
        ties = fx[f"{Q.DT_NAME[dt]}/ties"]
        assert (scan[:, mi["half_away"]] > 0).all() and (scan[:, mi["half_away"]] < ties).all()
        assert scan[:, mi["fma"]].sum() > 0
        # MAX 1 and 2 decode to exact multiples of m in the input dtype, which no conversion rounds
        assert (scan[2:, mi["trunc_bf16"]] > 0).all() and (scan[2:, mi["trunc_fp16"]] > 0).all()
        assert (scan[:, mi["ftz_in"]] > 0).all() == (dt == O.DT_BF16)


@pytest.mark.parametrize("dt", Q.DTYPES, ids=Q.DT_NAME)
def test_spec_against_float64(fx, dt):
    """the fp32 spec symbol is within one of round(x * MAX / m + MAX) computed exactly, and equal to it except within a
    few fp32 ulps of a half-integer"""
    for M in Q.MAXES:
        x, m, _, _, _ = Q.fixture_pairs(fx, dt, M)
        xf, mf = Q.to_f32(x, dt), Q.to_f32(m, dt)
        with np.errstate(all="ignore"):
            ok = np.isfinite(xf) & np.isfinite(mf) & (mf > 0) & np.isfinite(np.float32(M) / mf)
        x, m = x[ok], m[ok]
        spec = Q.spec_quant(x, m, M, dt).astype(np.float64)
        r, close = Q.exact_round(x, m, M, dt)
        assert (np.abs(spec - r) <= 1).all(), M
        bad = np.flatnonzero((spec != r) & ~close)
        assert bad.size == 0, (M, dt, hex(int(x[bad[0]])), hex(int(m[bad[0]])))
        tie = (Q.fixture_pairs(fx, dt, M)[3][ok] & Q.K_TIE) != 0
        assert close[tie].all()


@pytest.mark.parametrize("dt", Q.DTYPES, ids=Q.DT_NAME)
def test_regenerated_slice_equals_fixture(fx, dt):
    """a random slice of the set, regenerated from quant_edges: ties and uncapped witnesses of 6 ladder maxima at 3 MAX
    values, every special pair and the random sample are in the committed fixture exactly as they are made now"""
    rng = np.random.default_rng(7 + dt)
    scan = fx[f"{Q.DT_NAME[dt]}/scan_count"]
    for M in rng.choice(Q.MAXES, 3, replace=False):
        M = int(M)
        x, m, _, kind, mut = Q.fixture_pairs(fx, dt, M)
        key = (m.astype(np.int64) << 16) | x
        ms = np.sort(rng.choice(Q.ladder(dt), 6, replace=False))
        (tx, tm), wit = Q.scan_block(dt, M, ms)
        inm = np.isin(m, ms)
        assert np.array_equal(np.sort((tm.astype(np.int64) << 16) | tx), np.sort(key[inm & ((kind & Q.K_TIE) != 0)]))
        for bit, name in enumerate(Q.MUTANTS):
            if scan[M - 1, bit] <= Q.WITNESS_CAP:
                wk = (wit[name][1].astype(np.int64) << 16) | wit[name][0]
                assert np.array_equal(np.sort(wk), np.sort(key[inm & (((mut >> bit) & 1) != 0)])), (name, M)
        for sx, sm, k in (Q.special_pairs(dt, M) + (Q.K_SPECIAL,), Q.random_pairs(dt, M) + (Q.K_RANDOM,)):
            sk = np.unique((sm.astype(np.int64) << 16) | sx)
            assert np.array_equal(sk, np.sort(key[(kind & k) != 0])), (k, M)


def test_readback_maximum_gives_symbol_minus_max():
    """fl(fl(fl(sym - MAX) / MAX) * MAX) == sym - MAX exactly for every symbol and MAX, in both half dtypes: a row whose
    stored maximum is rewritten to MAX decodes to its symbols (the GPU tests read symbols back that way)"""
    for M in Q.MAXES:
        sym = np.arange(2 * M + 1)
        for dt in Q.DTYPES:
            mb = Q.from_f32(np.float32(M), dt)
            for out_dt in Q.DTYPES:
                got = Q.to_f32(Q.spec_dequant(sym, mb, M, dt, out_dt), out_dt)
                assert np.array_equal(got, (sym - M).astype(np.float32)), (M, dt, out_dt)


def test_pack_rows_places_the_maximum_everywhere():
    """the cycled maximum positions include the first and last channel and one inside the last partial 8-wide vector
    and 128-channel tile; every packed row's maximum is its pair's m and every pair lands in a row"""
    assert {0, 98} <= set(Q.row_positions(99)) and any(96 <= p < 98 for p in Q.row_positions(99))
    assert any(128 <= p < 199 for p in Q.row_positions(200))
    x, m = Q.random_pairs(O.DT_BF16, 7, 400)
    for Cw in (99, 128, 37):
        rows, rmax = Q.pack_rows(x, m, Cw, O.DT_BF16)
        assert np.array_equal(Q.spec_absmax(rows), rmax)
        got = set(zip(rows.ravel().tolist(), np.repeat(rmax, Cw).tolist()))
        assert set(zip(x.tolist(), m.tolist())) <= got
