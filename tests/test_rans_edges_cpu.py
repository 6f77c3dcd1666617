"""CPU: the rANS edge set (tests/golden/rans_edges.npz) against the plain-Python statement of the stream format
(tests/rans_edges.py), the CPU oracle and the host build of ac_core.cuh; the kernel-shaped models of rans_put and
rans_decode_stream against that statement; proof that every mutant of those models that CAN be told from the spec is
told apart by a stored stream (the mutation check), that the set still reaches every own-CDF edge it was searched for,
and that a reduced search finds such streams again.  Also cross-compiles the device sweep (tests/devsim) so that a
compile error in it shows without a GPU."""
import ctypes
import os

import numpy as np
import pytest

from oracle import oracle as O

import rans_edges as R

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def fx():
    return {k: v for k, v in R.load().items()}


@pytest.fixture(scope="module")
def sim():
    S = ctypes.CDLL(os.path.join(HERE, "hostsim", "libhostsim.so"))
    vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    S.sim_rans_encode_stream.restype = i64
    S.sim_rans_encode_stream.argtypes = [vp, vp, i64, i32, vp, i64]
    S.sim_rans_decode_stream.restype = ctypes.c_uint32
    S.sim_rans_decode_stream.argtypes = [vp, vp, i64, i32, vp, i64, i32, i32]
    return S


def _P(a):
    return ctypes.c_void_p(a.ctypes.data)


def _streams(fx):
    """(name, cdf row, column, wide, own) of every stream of the set: the own-CDF rows, and every group of every
    chunk-wide-CDF column"""
    for k, (col, wide) in enumerate(R.own_rows(fx)):
        yield f"own row {k} (g = {col.size}, {'wide' if wide else 'narrow'})", R.own_cdf(col), col, wide, True
    for T in R.BIG_T:
        for n, col in enumerate(fx[f"big_{T}"]):
            cdf, groups = R.foreign_groups(col)
            for a, g in groups:
                if T == R.LONG_T and (col[a:a + g] == col[a]).all() and a not in (0, T - g):
                    continue                                    # the long chunk's many one-symbol groups: two are enough
                yield f"T = {T} column {n} group at token {a} (g = {g})", cdf, col[a:a + g], True, False


@pytest.fixture(scope="module")
def streams(fx):
    return list(_streams(fx))


def test_fixture_shape(fx):
    assert list(fx["mutants"]) == list(R.MUTANTS) and set(R.EQUIVALENT) < set(R.MUTANTS)
    assert fx["g"].size < 400 and os.path.getsize(R.FIXTURE) < 1 << 19
    for col, wide in R.own_rows(fx):
        assert 1 <= col.size <= 256 and col.max() <= (30 if wide else 14)
    assert set(R.BIG_T) == {int(k[4:]) for k in fx if k.startswith("big_")}


def test_spec_oracle_hostsim_and_kernel_models_agree(streams, sim):
    """spec encode == oracle == host build of rans_enc_symbol == the model of rans_put, byte for byte; spec decode, the
    host build of rans_dec_symbol and the model of rans_decode_stream invert it from both halfword phases, with the 4-
    and the 5-step search, back to state 2^16"""
    for name, cdf, col, wide, own in streams:
        g = col.size
        want = R.encode(cdf, col)
        sym = np.ascontiguousarray(col.astype(np.int8).reshape(1, g, 1))
        bs, ln = O.encode_group(cdf.reshape(1, 1, 33), sym, 0, g, O.CODER_RANS)
        assert bs.tobytes() == want and int(ln[0, 0]) == len(want), f"oracle != spec: {name}: " + R.first_bad_step(cdf, col, bs.tobytes())
        back = np.zeros((1, g, 1), np.uint8)
        O.decode_group(cdf.reshape(1, 1, 33), bs, ln, back, 0, g, O.CODER_RANS)
        assert np.array_equal(back[0, :, 0], col), name
        cd = np.ascontiguousarray(cdf).view(np.uint16)
        out = np.zeros(2 * g + 64, np.uint8)
        n = sim.sim_rans_encode_stream(_P(cd), _P(sym), 1, g, _P(out), out.size)
        assert out[:n].tobytes() == want, f"hostsim != spec: {name}: " + R.first_bad_step(cdf, col, out[:n].tobytes())
        assert R.encode_as_kernel(cdf, col) == want, f"model of rans_put != spec: {name}"
        got, xf = R.decode(cdf, want, g)
        assert xf == R.LOW and np.array_equal(got, col), name
        for odd in (0, 1):
            for nsteps in (5, 4) if col.max() <= 14 else (5,):
                got, xf = R.decode_as_kernel(cdf, want, g, odd, None, nsteps)
                assert xf == R.LOW and np.array_equal(got, col), (name, odd, nsteps)
                buf = np.concatenate([np.full(2 * odd, 0x5A, np.uint8), np.frombuffer(want, np.uint8), np.full(8, 0xA5, np.uint8)])
                dec = np.zeros(g, np.uint8)
                xf = sim.sim_rans_decode_stream(_P(cd), ctypes.c_void_p(buf.ctypes.data + 2 * odd), len(want), g, _P(dec), 1, odd, nsteps)
                assert xf == R.LOW and np.array_equal(dec, col), f"hostsim decode: {name} phase {odd} {nsteps}-step"


def test_every_killable_mutant_is_killed(streams):
    """the mutation check.  Each mutant is one plausible slip in a rewrite of rans_put or rans_decode_stream; a stored
    stream must give other bytes (encoder) or other symbols / final state (decoder) under it.  The two mutants listed as
    equivalent must survive EVERY stream of the set -- if one dies, its reason is wrong."""
    killed = 0
    per = {m: 0 for m in R.MUTANTS}
    for name, cdf, col, wide, own in streams:
        if not own and col.size == R.G and killed == sum(1 << k for k, m in enumerate(R.MUTANTS) if m not in R.EQUIVALENT):
            continue                                            # the long groups are slow and add nothing once all died
        k = R.kills(cdf, col, 5 if wide else 4)
        killed |= k
        for b, m in enumerate(R.MUTANTS):
            per[m] += (k >> b) & 1
    print("\nstreams that kill each mutant: " + ", ".join(f"{m} {n}" for m, n in per.items()))
    for b, m in enumerate(R.MUTANTS):
        if m in R.EQUIVALENT:
            assert not (killed >> b) & 1, f"mutant {m} was listed as equivalent ({R.EQUIVALENT[m]}) but a stream tells it apart"
        else:
            assert (killed >> b) & 1, f"mutant {m} ({R.MUTANT_DOC[m]}) survives every stream of the set"


def test_the_set_reaches_every_edge(fx, streams):
    """coverage computed from the traces of the stored streams: everything that does not depend on where a stream lies in
    a payload (that part is the GPU test's, which lays the streams out)"""
    cov = R.Coverage(int(fx["longest"]))
    longest = 0
    for name, cdf, col, wide, own in streams:
        tr = []
        data = R.encode(cdf, col, tr)
        n = (len(data) - 4) // 2
        cov.add(R.stream_items(tr, col.size, "wide" if wide else "narrow", own, model=own and n < 40), n, 0, own)
        if own:
            longest = max(longest, n)
            assert n <= R.PROVEN_MAX_HALFWORDS < R.ROW_HALFWORDS, name
        else:
            assert n <= col.size, name                          # at most one halfword per symbol
    layout = ("stream at", "the longest stream")
    missing = [m for m in cov.missing() if not m.startswith(layout[1]) and layout[0] not in m]
    assert not missing, f"the stored streams no longer reach: {missing}"
    assert longest == int(fx["longest"])
    print(f"\nlongest own-CDF stream found: {longest} halfwords; proven bound {R.PROVEN_MAX_HALFWORDS}, row {R.ROW_HALFWORDS}")


def test_reduced_search_refinds_a_sample(fx):
    """the directed longest-stream search gives the stored column again, and a small random search still meets both ends of
    a search interval, both sides of the push threshold and a witness of every killable mutant"""
    col = R.longest_own_stream()
    assert np.array_equal(col, R.own_rows(fx)[0][0])
    rng = np.random.default_rng(5)
    items, killed = set(), 0
    for k, col in enumerate(R._hist_columns(rng, 256, 30, 160)):
        tr = []
        cdf = R.own_cdf(col)
        R.encode(cdf, col, tr)
        items |= R.stream_items(tr, 256, "wide", True)
        if k % 8 == 0:
            killed |= R.kills(cdf, col)
    assert any(i.startswith("remainder 0") for i in items) and any(i.startswith("remainder f - 1") for i in items)
    assert "x >> 16 == f - 1 (no push)" in items or "x >> 16 == f (push)" in items
    for b, m in enumerate(R.MUTANTS):
        if m not in R.EQUIVALENT and m not in ("no_bias", "fixup_gt", "push_gt"):      # these need an exact hit: the big search
            assert (killed >> b) & 1, m


def test_first_bad_step_names_the_step():
    """a stream damaged the way a wrong encode step damages it is traced to the push behind that step"""
    col = R.longest_own_stream()
    cdf = R.own_cdf(col)
    tr = []
    want = R.encode(cdf, col, tr)
    assert R.first_bad_step(cdf, col, want) == "stream equals the spec's"
    for mut in ("no_fixup", "m65535"):
        msg = R.first_bad_step(cdf, col, R.encode_as_kernel(cdf, col, mut))
        assert "the first wrong step is among coding steps 0.." in msg and "q = " in msg, msg


def test_float_model_classifies_the_fixup():
    """the model that labels steps: remainder 0 always takes the fix-up, a remainder in the middle of a large f never"""
    assert R.classify(40000 * 2115, 2115) == "taken"
    assert R.classify(40000 * 2115 + 1000, 2115) == "not taken"
    for x, f in ((65536, 1), (2 ** 32 - 1, 65535), (65535 * 65505 + 65504, 65505)):
        assert R.classify(x, f) in ("taken", "not taken", "depends")


def test_device_sweep_compiles():
    """tests/devsim/devsim.cu (the exhaustive sweep of rans_put, run by the GPU suite) cross-compiles for sm_90a"""
    assert os.path.exists(R.build_devsim(force=True))


def test_the_gpu_tiles_reach_every_edge(fx):
    """the tiles tests/test_gpu_rans_edges.py lays out (rans_edges.own_tile / big_tile on planes of MAX 1..15), traced by
    the spec: every item of Coverage.wanted(), the ones that depend on a stream's place in the payload included"""
    import quant_edges as Q
    _, _, mk, mv = Q.plane_maxes(15)
    pmax = np.array(mk + mv)
    cov = R.plan_coverage(fx, pmax, [2 * (int(m) + 1) for m in pmax])
    assert not cov.missing(), cov.missing()
