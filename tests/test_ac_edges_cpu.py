"""CPU: the arithmetic-coder edge set (tests/golden/ac_edges.npz) against the plain-Python statement of the container-
version-1 bitstream (tests/ac_edges.py), the CPU oracle and the host build of ac_core.cuh; the kernel-shaped models of
EncState2 / DecState2 against that statement, the decoder model under keys guessed too low, too high and at random; the
mutation check; coverage of the stored set; the row bound; a reduced search; and the device harness cross-compiles."""
import ctypes
import os

import numpy as np
import pytest

from oracle import oracle as O

import ac_edges as A
import rans_edges as R

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def fx():
    return {k: v for k, v in A.load().items()}


@pytest.fixture(scope="module")
def sim():
    S = ctypes.CDLL(os.path.join(HERE, "hostsim", "libhostsim.so"))
    vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    S.sim_encode_stream.restype = i64
    S.sim_encode_stream.argtypes = [vp, vp, i64, i32, vp, i64]
    S.sim_encode_stream2.restype = i64
    S.sim_encode_stream2.argtypes = [vp, vp, i64, i32, vp, i64]
    S.sim_decode_stream2.argtypes = [vp, vp, i64, i32, vp, i64, i32, i32]
    return S


def _P(a):
    return ctypes.c_void_p(a.ctypes.data)


def _streams(fx):
    """(name, cdf row, column, wide, own) of every distinct stream of the set"""
    for k, (col, wide) in enumerate(A.own_rows(fx)):
        yield f"own row {k} (g = {col.size}, {'wide' if wide else 'narrow'})", R.own_cdf(col), col, wide, True
    seen = set()
    for T, cols in A.big_columns(fx):
        for n, col in enumerate(cols):
            cdf, groups = A.chunk_streams(col)
            for a, g in groups:
                key = (cdf.tobytes(), col[a:a + g].tobytes())
                if key not in seen:
                    seen.add(key)
                    yield f"T = {T} column {n} group at token {a} (g = {g})", cdf, col[a:a + g], True, False


@pytest.fixture(scope="module")
def streams(fx):
    return list(_streams(fx))


def test_fixture_shape(fx):
    assert list(fx["mutants"]) == list(A.MUTANTS) and set(A.EQUIVALENT) < set(A.MUTANTS) and len(A.MUTANTS) >= 10
    assert fx["g"].size < 200 and os.path.getsize(A.FIXTURE) < 1 << 18
    for col, wide in A.own_rows(fx):
        assert 1 <= col.size <= 256 and col.max() <= (30 if wide else 14)
    assert int(fx["big_wide"].shape[1]) == A.WIDTH1_T


def test_spec_oracle_hostsim_and_kernel_models_agree(streams, sim):
    """spec encode == oracle == host enc_symbol (sim_encode_stream) == host enc_symbol2 (sim_encode_stream2) == the model
    of EncState2, byte for byte; the spec decoder, the host dec_symbol2 at every skip and both depths and the model of
    DecState2 with the host and device-like keys invert it"""
    for name, cdf, col, wide, own in streams:
        g = col.size
        want = A.encode(cdf, col)
        sym = np.ascontiguousarray(col.astype(np.int8).reshape(1, g, 1))
        bs, ln = O.encode_group(cdf.reshape(1, 1, 33), sym, 0, g, O.CODER_AC)
        assert bs.tobytes() == want and int(ln[0, 0]) == len(want), f"oracle != spec: {name}: " + A.first_bad_step(cdf, col, bs.tobytes())
        back = np.zeros((1, g, 1), np.uint8)
        O.decode_group(cdf.reshape(1, 1, 33), bs, ln, back, 0, g, O.CODER_AC)
        assert np.array_equal(back[0, :, 0], col), name
        cd = np.ascontiguousarray(cdf).view(np.uint16)
        for fn in (sim.sim_encode_stream, sim.sim_encode_stream2):
            out = np.zeros(2 * g + 64, np.uint8)
            n = fn(_P(cd), _P(sym), 1, g, _P(out), out.size)
            assert out[:n].tobytes() == want, f"hostsim != spec: {name}: " + A.first_bad_step(cdf, col, out[:n].tobytes())
        assert A.encode_as_kernel(cdf, col)[0] == want, f"model of EncState2 != spec: {name}"
        assert np.array_equal(A.decode(cdf, want, g), col), name
        for skip in range(4):
            buf = np.concatenate([np.full(skip, 0x5A, np.uint8), np.frombuffer(want, np.uint8)])
            for nsteps in (5, 4) if col.max() <= 14 else (5,):
                dec = np.zeros(g, np.uint8)
                sim.sim_decode_stream2(_P(cd), ctypes.c_void_p(buf.ctypes.data + skip), len(want), g, _P(dec), 1, skip, nsteps)
                assert np.array_equal(dec, col), f"hostsim decode: {name} skip {skip} {nsteps}-step"
                for kn in ("host", "device-like"):
                    assert np.array_equal(A.decode_as_kernel(cdf, want, g, skip, nsteps, A.KEYS[kn]), col), (name, skip, kn)


def test_decoder_walk_is_exact_for_any_guess(streams):
    """dec_symbol2's slow path finds the symbol whatever the key: exact, all zeros, all ones, 2^16 too high or too low,
    or random -- on the own-CDF streams and one group per chunk-wide set"""
    rng = np.random.default_rng(7)
    keys = dict(A.KEYS)
    keys["random"] = lambda o, s: int(rng.integers(0, 1 << 32))
    for name, cdf, col, wide, own in streams[:: 3]:
        want = A.encode(cdf, col)
        for kn, kf in keys.items():
            assert np.array_equal(A.decode_as_kernel(cdf, want, col.size, 1, 5, kf), col), (name, kn)


def test_trailing_bytes_cannot_change_a_decode(streams):
    """the termination emits the final bit and its run, so every continuation of the stream lies inside the final
    interval: the spec decoder and the model of DecState2 give the same symbols with 0x00, 0xFF or random bytes after
    the stream"""
    rng = np.random.default_rng(11)
    for name, cdf, col, wide, own in streams[:: 2]:
        want = A.encode(cdf, col)
        for tail in (b"\x00" * 16, b"\xff" * 16, rng.integers(0, 256, 16).astype(np.uint8).tobytes()):
            assert np.array_equal(A.decode(cdf, want, col.size, tail), col), name
            for skip in (0, 3):
                assert np.array_equal(A.decode_as_kernel(cdf, want, col.size, skip, 5, A.key_device_like, after=tail), col), name


def test_every_killable_mutant_is_killed(streams):
    """the mutation check: each mutant is one plausible slip in a rewrite of enc_symbol2 / enc_append / enc_ripple /
    enc_finish2 or dec_init2 / dec_symbol2; a stored stream must tell it apart.  The mutants listed as equivalent must
    survive every stream -- if one dies, its reason is wrong."""
    killed = 0
    killable = sum(1 << k for k, m in enumerate(A.MUTANTS) if m not in A.EQUIVALENT)
    for name, cdf, col, wide, own in streams:
        killed |= A.kills(cdf, col, 5 if wide else 4)
    for b, m in enumerate(A.MUTANTS):
        if m in A.EQUIVALENT:
            assert not (killed >> b) & 1, f"mutant {m} was listed as equivalent ({A.EQUIVALENT[m]}) but a stream tells it apart"
        else:
            assert (killed >> b) & 1, f"mutant {m} ({A.MUTANT_DOC[m]}) survives every stream of the set"
    assert killed == killable


def test_the_set_reaches_every_edge_and_fits_its_rows(fx, streams):
    """coverage computed from the traces of the stored streams; the longest own-CDF stream is the stored one and fits the
    stated bound, which fits the 160-byte row; every chunk-wide group fits the bound of 16 bits per token and its row"""
    cov = A.Coverage()
    longest_own = longest_split = 0
    bound_own = int(np.ceil(A.own_bound_bits() / 8))
    bound_split = int(np.ceil(A.split_bound_bits() / 8))
    assert bound_own <= 4 * A.ROW_WORDS_OWN and bound_split <= 4 * A.ROW_WORDS_SPLIT
    for name, cdf, col, wide, own in streams:
        n = len(A.encode(cdf, col))
        cov.add(A.stream_items(cdf, col, "wide" if wide else "narrow", own))
        if own:
            longest_own = max(longest_own, n)
            assert n <= int(np.ceil(A.own_bound_bits(col.size) / 8)), name
        else:
            longest_split = max(longest_split, n)
            assert n <= bound_split, name
    assert longest_own == int(fx["longest"]) <= bound_own
    assert not cov.missing(17), f"the stored streams no longer reach: {cov.missing(17)}"
    assert not any(i.startswith("k = 18") for i in cov.items)
    print(f"\nlongest own-CDF v1 stream: {longest_own} bytes (bound {A.own_bound_bits():.2f} bits = {bound_own} bytes, row "
          f"{4 * A.ROW_WORDS_OWN}); longest chunk-wide group: {longest_split} bytes (bound {bound_split}, row "
          f"{4 * A.ROW_WORDS_SPLIT}); largest k 17")


def test_width1_threshold():
    """a used symbol gets CDF width 1 first in a chunk of 65505 tokens, and width 1 is what k = 17 needs"""
    assert A.width1_prefixes(A.WIDTH1_T).size and not A.width1_prefixes(A.WIDTH1_T - 1).size


def test_reduced_search_refinds_a_sample():
    """a small seeded search meets carries, runs across a flushed word, the slow path from both sides, every stream
    length mod 4 and the decoder's refill at pos = 32; the pending-run construction still reaches its runs"""
    rng = np.random.default_rng(5)
    items = set()
    for col in R._hist_columns(rng, 256, 30, 24):
        items |= A.stream_items(R.own_cdf(col), col, "wide", True)
    for w in ("carry out of x + plo", "pending run straddling a flushed word", "refill exactly at pos = 32",
              "slow path from a guess too low", "slow path from a guess too high"):
        assert w in items, w
    col = A.run_column(np.random.default_rng(1), 70, True)
    cdf, _ = A.chunk_streams(col)
    assert "pending run of > 64 bits" in A.stream_items(cdf, col[:A.G], "wide", False)


def test_first_bad_step_names_the_step():
    col = np.random.default_rng(2).integers(0, 31, 256).astype(np.uint8)
    cdf = R.own_cdf(col)
    assert A.first_bad_step(cdf, col, A.encode(cdf, col)) == "stream equals the spec's"
    msg = A.first_bad_step(cdf, col, A.encode_as_kernel(cdf, col, "phi_no_chi")[0])
    assert "coding step" in msg, msg


def test_clamp_model():
    """the model of the clamped row: a stream longer than its row stores only inside the row and reports w > cap"""
    col = np.random.default_rng(3).integers(0, 31, 256).astype(np.uint8)
    cdf = R.own_cdf(col)
    for cap in (1, 2, 3):
        e = A.Enc2(cap, guard=2)
        e.row = [0xDEADBEEF] * len(e.row)
        start, freq = R.table(cdf)
        for s in col:
            e.symbol(start[int(s)], freq[int(s)])
        e.finish()
        assert e.w > cap and e.row[:2] == [0xDEADBEEF] * 2 and e.row[-2:] == [0xDEADBEEF] * 2


def test_device_harness_compiles():
    """tests/devsim/acsim.cu (the arithmetic coder's device harness) cross-compiles for sm_90a"""
    assert os.path.exists(A.build_acsim(force=True))
