"""GPU: the arithmetic coder (container version 1) the kernels run, driven to the streams of tests/golden/ac_edges.npz.

Every kernel is driven as in test_gpu_rans_edges.py: channel 0 of every plane is symbol 0 on every token, so each
(plane, token) row's maximum is MAX, the factor is 1 and x = s - MAX quantises to s exactly; every other channel's symbol
sequence is a column of the set.

* the device harness (tests/devsim/acsim.cu): enc_symbol2 / enc_finish2 and dec_init2 / dec_symbol2<4|5> on the set's streams
  with their per-step state against the Python models; a row of 1..3 words between guard words; the decoder sweep over
  spans and the ends of every symbol's interval, with the key error and the slow-path rate;
* own-CDF tiles (every token count of the set), bf16 and fp16, blob and paged sources: coder 0 must give the spec's bytes
  (ac_edges.encode) stream for stream, a mismatch names plane, channel, lane and coding step; chunks of 257 ... 65505
  tokens (FUSED = false under the chunk-wide CDF; the largest carries a width-1 symbol coded with k = 17);
* every container decodes through decode_chunks, plan + decode_layers, vllm / huggingface / paged destinations and one
  decode_plan_heads window to s - MAX with status 0, and with every byte outside the decoded layer's planes replaced by
  0x00 or 0xFF;
* coverage computed from the compared streams' traces is asserted complete."""
import ctypes

import numpy as np
import pytest
import torch

import ac_edges as A
import cdf_edges as E
import quant_edges as Q
import rans_edges as R
from test_gpu_cdf_edges import ALL_COMBOS, _decode_all, _sections, _want_bits
from test_gpu_layer_split import _Dest, _decode, _encode_chunks, _source
from test_gpu_layer_split import _s
from test_gpu_quant_edges import _planes, _tensor, _unplanes

pytestmark = pytest.mark.gpu
L = 15
KB, VB, MK, MV = Q.plane_maxes(L)
PLANE_MAX = np.array(MK + MV)
NBS = [2 * (int(m) + 1) for m in PLANE_MAX]


@pytest.fixture(scope="module")
def fx():
    return {k: v for k, v in A.load().items()}


class _Expect:
    """the spec's streams, cached by (CDF row, column), and the coverage of every stream compared"""

    def __init__(self):
        self.cov = A.Coverage()
        self._c = {}

    def stream(self, cdf, col, kind, own):
        key = (cdf.tobytes(), col.tobytes(), kind, own)
        if key not in self._c:
            self._c[key] = A.encode(cdf, col)
            self.cov.add(A.stream_items(cdf, col, kind, own, self._c[key]))
        return self._c[key]


@pytest.fixture(scope="module")
def expect():
    return _Expect()


def _check_v1(raw, sym, cdfs, expect, own, what):
    """version-1 container: CDF rows, lengths and every stream of every group are the spec's"""
    hd, lo, a = _sections(raw)
    P, T, C = sym.shape
    assert hd.version == 1, what
    cdf = a[lo.off_cdf: lo.off_cdf + P * C * 33 * 2].view(np.int16).reshape(P, C, 33)
    assert np.array_equal(cdf, cdfs), f"{what}: CDF rows"
    lengths = a[lo.off_lengths: lo.off_lengths + hd.ngroups * P * C * 4].view(np.int32).reshape(hd.ngroups, P, C)
    off = lo.off_payload
    for k in range(hd.ngroups):
        t0, g = k * A.G, min(A.G, T - k * A.G)
        for p in range(P):
            kind = R.plane_kind(int(PLANE_MAX[p]))
            for c in range(C):
                col = np.ascontiguousarray(sym[p, t0:t0 + g, c])
                want = expect.stream(cdfs[p, c], col, kind, own)
                n = int(lengths[k, p, c])
                got = bytes(a[off: off + n])
                if got != want:
                    raise AssertionError(f"{what}: stream != spec at plane {p} (MAX {int(PLANE_MAX[p])}), channel {c} "
                                         f"(lane {c % 32} of warp {c // 32}), group {k} (tokens {t0}..{t0 + g - 1}): "
                                         + A.first_bad_step(cdfs[p, c], col, got))
                off += n
    assert off == hd.total_bytes, what


def _encode(fx, sym, dt, kind, rng):
    C = sym.shape[2]
    x = _tensor(_unplanes(E.kv_for_symbols(sym, PLANE_MAX, dt)), dt, 1, C)
    raw, = _encode_chunks(_source(kind, x, rng), 0, 1, sym.shape[1], sym.shape[1], KB, VB, 0)
    return raw


def _trailing(raw, sym, hist, dt, rng, what):
    """decode layer l alone (plan + decode_layers) with every payload byte outside planes l and L + l set to 0x00 or
    0xFF: the values of that layer must not change"""
    hd, lo, a = _sections(raw)
    P, T, C = sym.shape
    lengths = a[lo.off_lengths: lo.off_lengths + hd.ngroups * P * C * 4].view(np.int32).reshape(hd.ngroups, P, C)
    starts = lo.off_payload + np.concatenate([[0], np.cumsum(lengths.reshape(-1))])[:-1].reshape(hd.ngroups, P, C)
    for l in (0, 7, L - 1):
        for fill in (0x00, 0xFF):
            b = np.full(len(raw), fill, np.uint8)
            b[:lo.off_payload] = a[:lo.off_payload]
            for k in range(hd.ngroups):
                for p in (l, L + l):
                    s0, s1 = int(starts[k, p, 0]), int(starts[k, p, C - 1] + lengths[k, p, C - 1])
                    b[s0:s1] = a[s0:s1]
            dest = _Dest("vllm", L, 1, C, T, 0, 3, rng)
            assert _decode([b.tobytes()], 0, dest, [dest.tok0], KB, VB, dt, parts=[(l, l + 1)]) == [0], what
            got = _planes(dest.bits())
            want = _want_bits(sym, PLANE_MAX, 0)
            for p in (l, L + l):
                assert np.array_equal(got[p], want[p]), f"{what}: layer {l}, bytes after the plane set to {fill:#04x}"


# ------------------------------------------------------------------------------------------------ 1. device harness
def _lib():
    lib = ctypes.CDLL(A.build_acsim())
    vp, i32, u32, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32, ctypes.c_int64
    lib.devsim_ac_encode.argtypes = [vp, vp, i32, i32, u32, vp, vp, vp]
    lib.devsim_ac_decode.argtypes = [vp, vp, i64, vp, i32, i32, i32, vp]
    lib.devsim_ac_clamp.argtypes = [vp, vp, i32, u32, u32, vp, vp]
    lib.devsim_ac_sweep.argtypes = [vp, i32, vp, i32, i32, vp]
    return lib


def _P(a):
    return ctypes.c_void_p(a.ctypes.data)


def _harness_streams(fx):
    out = [(R.own_cdf(col), col, wide) for col, wide in A.own_rows(fx)]
    for T, cols in A.big_columns(fx):
        for col in cols:
            cdf, _ = A.chunk_streams(col)
            out.append((cdf, col[:A.G], True))
    return out


def test_device_steps_match_the_models(fx):
    """enc_symbol2 / enc_finish2 and dec_init2 / dec_symbol2 compiled for the device, per step, against the models;
    every stream decoded alone at skips 0..3 with 0x00 or 0xFF behind it"""
    lib = _lib()
    for cdf, col, wide in _harness_streams(fx):
        g = col.size
        cd = np.ascontiguousarray(cdf).view(np.uint16).reshape(1, 33)
        cap = g // 2 + 4
        steps = np.zeros((1, g + 1, 5), np.uint32)
        rows = np.zeros((1, cap), np.uint32)
        lens = np.zeros(1, np.uint32)
        assert lib.devsim_ac_encode(_P(cd), _P(np.ascontiguousarray(col)), g, 1, cap, _P(steps), _P(rows), _P(lens)) == 0
        want, enc = A.encode_as_kernel(cdf, col)
        model = A.Enc2(cap)
        start, freq = R.table(cdf)
        for i, s in enumerate(col):
            model.symbol(start[int(s)], freq[int(s)])
            st = (model.x, model.rng, model.lo, model.m, model.w)
            assert tuple(int(v) for v in steps[0, i]) == st, f"enc_symbol2 step {i}: device {steps[0, i]}, model {st}"
        assert int(lens[0]) == len(want) and rows[0].astype(">u4").tobytes()[:len(want)] == want
        for nsteps in (5, 4) if col.max() <= 14 else (5,):
            for fill in (0x00, 0xFF):
                n = 4
                buf = np.full(n * (len(want) + 40) + 64, fill, np.uint8)
                starts = np.zeros(n, np.uint32)
                for skip in range(n):
                    o = skip * (len(want) + 40) // 4 * 4 + skip
                    starts[skip] = o
                    buf[o:o + len(want)] = np.frombuffer(want, np.uint8)
                st = np.zeros((n, g, 5), np.uint32)
                cds = np.ascontiguousarray(np.repeat(cd, n, 0))
                assert lib.devsim_ac_decode(_P(cds), _P(buf), buf.size, _P(starts), g, n, nsteps, _P(st)) == 0
                for skip in range(n):
                    assert np.array_equal(st[skip, :, 3], col), f"device decode, skip {skip}, {nsteps}-step, fill {fill}"
                tr = []
                A.decode_as_kernel(cdf, want, g, 0, nsteps, lambda o, s: 0, trace=tr, after=bytes([fill]) * 64)
                dev = [(int(a), int(b), int(c)) for a, b, c in st[0, :, :3]]
                assert dev == [(t[0], t[1], t[2]) for t in tr], "decoder (span, off, pos) != model"


def test_clamp_harness(fx):
    """the longest stream of the set into rows of 1..3 words between guard words: nothing outside the row changes and
    w > cap is reported"""
    lib = _lib()
    col, _ = A.own_rows(fx)[0]
    cd = np.ascontiguousarray(R.own_cdf(col)).view(np.uint16)
    for cap in (1, 2, 3):
        guard = 4
        buf = np.full(cap + 2 * guard, 0xC0FFEE11, np.uint32)
        res = np.zeros(2, np.uint32)
        assert lib.devsim_ac_clamp(_P(cd), _P(np.ascontiguousarray(col)), col.size, cap, guard, _P(buf), _P(res)) == 0
        assert (buf[:guard] == 0xC0FFEE11).all() and (buf[guard + cap:] == 0xC0FFEE11).all(), f"cap {cap}: guard written"
        assert int(res[1]) > cap, f"cap {cap}: w = {int(res[1])} not reported past the row"


def test_decoder_sweep(fx):
    """a sample, not a proof: every CDF row of the set at spans just above 2^30, around 2^31, up to 2^32, powers of two
    +- 1 and 200 seeded spans, at both ends of every symbol's off interval and +- 1: dec_symbol2 == the exact rule"""
    lib = _lib()
    rows = np.stack([np.ascontiguousarray(c).view(np.uint16) for c, _, _ in _harness_streams(fx)])
    rows = np.unique(rows, axis=0)
    rng = np.random.default_rng(31)
    spans = [2 ** 30 + 1, 2 ** 30 + 2, 2 ** 30 + 3, 2 ** 31 - 1, 2 ** 31, 2 ** 31 + 1, 3 * 2 ** 30, 2 ** 32 - 1, 0]
    spans += [int(v) for v in rng.integers(2 ** 30 + 1, 2 ** 32, 200)]
    sp = np.array(spans, np.uint32)
    for nsteps in (5, 4):
        tally = np.zeros(7, np.uint64)
        assert lib.devsim_ac_sweep(_P(rows), rows.shape[0], _P(sp), sp.size, nsteps, _P(tally)) == 0
        checks, wrong, slow = (int(v) for v in tally[:3])
        print(f"\ndecoder sweep ({nsteps}-step) on {torch.cuda.get_device_name(0)}: {checks} offsets, {wrong} wrong, slow "
              f"path {slow} ({100.0 * slow / checks:.3f} %); key count off by <= -2: {int(tally[3])}, -1: {int(tally[4])}, "
              f"+1: {int(tally[5])}, >= +2: {int(tally[6])}")
        assert checks > 10000 and wrong == 0


# ------------------------------------------------------------------------------------------------ 2. own-CDF tiles
@pytest.mark.parametrize("dt", [0, 1], ids=["bf16", "fp16"])
def test_own_cdf_tiles(fx, expect, dt, monkeypatch):
    for k, t in enumerate(R.own_ts(fx)):
        rng = np.random.default_rng(100 * dt + t)
        sym = R.own_tile(fx, t, PLANE_MAX)
        cdfs, hist = R.own_cdfs(sym)
        what = f"own-CDF tile t = {t}, dtype {dt}"
        raw = _encode(fx, sym, dt, "blob", rng)
        _check_v1(raw, sym, cdfs, expect, True, what)
        if t == 256 or k % 2 == dt:
            assert _encode(fx, sym, dt, "paged", rng) == raw, f"{what}: paged source != blob source"
        combos = ALL_COMBOS[::2] if t == 256 else [ALL_COMBOS[(k + dt) % len(ALL_COMBOS)]]
        _decode_all([raw], 0, sym, hist, NBS, 1, sym.shape[2], dt, rng, monkeypatch, combos, f"{what}, coder 0", t)
        if t == 256:
            _trailing(raw, sym, hist, dt, rng, what)


def test_heads_window(fx):
    """b200kv_decode_plan_heads over head 1 of the t = 256 tile split into two heads"""
    t, dt = 256, 0
    rng = np.random.default_rng(9)
    sym = R.own_tile(fx, t, PLANE_MAX)
    if sym.shape[2] % 2:
        sym = np.concatenate([sym, sym[:, :, -1:]], axis=2)
    D = sym.shape[2] // 2
    x = _tensor(_unplanes(E.kv_for_symbols(sym, PLANE_MAX, dt)), dt, 2, D)
    raw, = _encode_chunks(_source("blob", x, rng), 0, 1, t, t, KB, VB, 0)
    dest = _Dest("vllm", L, 2, D, t, dt, 0, rng)
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import parse_header
    lib = N.lib()
    total = ((len(raw) + 15) & ~15) + N.READ_SLACK
    host = np.zeros(total, np.uint8)
    host[:len(raw)] = np.frombuffer(raw, np.uint8)
    buf = torch.from_numpy(host).cuda()
    v = dest.view
    wsb = N.check(lib.b200kv_decode_workspace_bytes(v.L, 2, v.D, t, 1), "decode_workspace_bytes")
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    status = torch.full((1,), 0x5555, dtype=torch.int32, device="cuda")
    plan = N.DecodePlan()
    N.check(lib.b200kv_decode_plan_heads(buf.data_ptr(), total, N.i64_array([0]), N.i64_array([len(raw)]),
                                         N.i32_array([int(parse_header(raw).ntokens)]), N.i64_array([0]), 1, dt, 0,
                                         ctypes.byref(v.desc), N.float_array(KB), N.float_array(VB), status.data_ptr(),
                                         ws.data_ptr(), wsb, ctypes.byref(plan), _s(), 2, N.i32_array([1]),
                                         N.i32_array([1]), N.i32_array([1])), "decode_plan_heads")
    N.check(lib.b200kv_decode_layers(ctypes.byref(plan), 0, v.L, _s()), "decode_layers")
    torch.cuda.synchronize()
    assert status.cpu().tolist() == [0], "window status"
    got = dest.tokens()[:, :, :, 1:2].cpu().contiguous().view(torch.int16).numpy().view(np.uint16)
    want = Q.from_f32((sym[:, :, D:].astype(np.int64) - PLANE_MAX[:, None, None]).astype(np.float32), dt)
    assert np.array_equal(_planes(got.reshape(L, 2, t, D)), want), "decode_plan_heads window"


# ------------------------------------------------------------------------------------------------ 3. chunk-wide CDF
def _big_sets(fx):
    return [(T, cols) for T, cols in A.big_columns(fx)]


@pytest.mark.parametrize("which", range(6))
def test_chunk_wide_cdf_groups(fx, expect, which, monkeypatch):
    T, cols = _big_sets(fx)[which]
    dt = which % 2
    rng = np.random.default_rng(T)
    sym = np.zeros((2 * L, T, 1 + cols.shape[0]), np.uint8)
    for p, M in enumerate(PLANE_MAX):
        sym[p, :, 1:] = np.minimum(cols, 2 * M).T
    cdfs, hist = R.own_cdfs(sym)
    raw = _encode(fx, sym, dt, "blob" if which % 3 else "paged", rng)
    _check_v1(raw, sym, cdfs, expect, False, f"T = {T}")
    combos = [ALL_COMBOS[(which + 5 * k) % len(ALL_COMBOS)] for k in range(2 if T < 4096 else 1)]
    _decode_all([raw], 0, sym, hist, NBS, 1, sym.shape[2], dt, rng, monkeypatch, combos, f"T = {T}, coder 0", T)


# ------------------------------------------------------------------------------------------------ 4. coverage
def test_coverage_is_complete(fx, expect):
    missing = expect.cov.missing(17)
    assert not missing, f"the tiles no longer reach: {missing}"
    assert not any(i.startswith("k = 18") for i in expect.cov.items)
    print(f"\nv1 edges reached: {len(expect.cov.items)} items; longest own-CDF stream {int(fx['longest'])} bytes")
