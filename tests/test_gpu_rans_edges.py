"""GPU: the rANS encode step and decode loop the kernels run, driven to prescribed symbol ORDERS.

Every kernel is driven as in test_gpu_cdf_edges.py: channel 0 of every plane is symbol 0 on every token, so each
(plane, token) row's maximum is MAX, the factor is 1 and x = s - MAX quantises to s exactly; every other channel's symbol
sequence is a column of tests/golden/rans_edges.npz -- streams that reach remainder 0 and f - 1 on every search leaf of
both table depths, both sides of the push threshold, the smallest and largest quotients and frequencies, 0 to 3 and the
most halfwords at both phases, a pull on every position of the decode loop's unrolled trip and in its tail, and the
longest stream a directed search found, between 4-byte neighbours and behind a 34-byte header.

* the exhaustive sweep: rans_put (tests/devsim, the function the encode kernels inline) at both ends of every quotient
  bucket of every freq, 8.6e9 steps, against integer division: zero wrong states;
* own-CDF tiles (every token count of the set): coder 1 (version 2), coder 2 (version 3), a latent descriptor
  (version 4), the layer-split encode and a paged source must give the plain-Python spec's bytes (rans_edges.encode)
  stream for stream; a mismatch names the plane, channel, lane and the coding step.  Coder 0 rides along against the
  oracle.  Every container decodes through decode_chunks, plan + decode_layers, both table layouts, vllm / huggingface /
  paged destinations, both dtypes and one decode_plan_heads window to s - MAX bit for bit with status 0;
* chunks of 257 .. 8192 tokens: encode_kernel<FUSED = false> walks each group backwards in batches of four under the
  chunk-wide CDF, where a rare symbol costs up to 13 bits: groups longer than an own-CDF row, f < 16, partial last
  groups of every length mod 4;
* what the tiles reached is computed from the spec's traces of the very streams compared (rans_edges.Coverage) and
  asserted complete."""
import ctypes
import time
import types

import numpy as np
import pytest
import torch

from oracle import oracle as O

import cdf_edges as E
import quant_edges as Q
import rans_edges as R
from test_gpu_cdf_edges import ALL_COMBOS, _check_values, _decode_all, _sections
from test_gpu_layer_split import _Dest, _containers, _decode, _encode_chunks, _encode_layers, _rand_partition, _s, _source
from test_gpu_quant_edges import _decode_heads, _planes, _tensor, _unplanes

pytestmark = pytest.mark.gpu
TDT = (torch.bfloat16, torch.float16)
L = 15
KB, VB, MK, MV = Q.plane_maxes(L)
PLANE_MAX = np.array(MK + MV)
NBS = [2 * (int(m) + 1) for m in PLANE_MAX]


def _N():
    from lmcache_b200 import _native as N
    return N


@pytest.fixture(scope="module")
def fx():
    return {k: v for k, v in R.load().items()}


@pytest.fixture(scope="module")
def expect(fx):
    return R.Expect(int(fx["longest"]))


def _where(p, c, tok0, g, pmax=PLANE_MAX):
    return (f"plane {p} (MAX {int(pmax[p])}, {R.plane_kind(int(pmax[p]))}), channel {c} (lane {c % 32} of warp {c // 32}), "
            f"tokens {tok0}..{tok0 + g - 1}")


def _compare_streams(payload, lengths, want, sym, cdfs, tok0, g, what, pmax=PLANE_MAX):
    """payload bytes + lengths [P, C] of one group against the spec's streams want[p][c]; names the first wrong stream
    and the coding step it went wrong at"""
    off = 0
    for p in range(len(want)):
        for c, w in enumerate(want[p]):
            n = int(lengths[p, c])
            got = bytes(payload[off: off + n])
            if got != w:
                raise AssertionError(f"{what}: stream != spec at {_where(p, c, tok0, g, pmax)}: "
                                     + R.first_bad_step(cdfs[p, c], sym[p, tok0:tok0 + g, c], got))
            off += n
    return off


def _check_v2(raw, sym, cdfs, want_groups, what):
    """version-2 container: CDF rows, lengths and payload are the spec's, group by group"""
    hd, lo, a = _sections(raw)
    P, T, C = sym.shape
    cdf = a[lo.off_cdf: lo.off_cdf + P * C * 33 * 2].view(np.int16).reshape(P, C, 33)
    assert np.array_equal(cdf, cdfs), f"{what}: CDF rows"
    G_ = hd.ngroups
    lengths = a[lo.off_lengths: lo.off_lengths + G_ * P * C * 4].view(np.int32).reshape(G_, P, C)
    off = lo.off_payload
    for k, want in enumerate(want_groups):
        g = min(R.G, T - k * R.G)
        off += _compare_streams(a[off:], lengths[k], want, sym, cdfs, k * R.G, g, f"{what}, group {k}")
    assert off == hd.total_bytes, what


def _check_v3(raw, sym, cdfs, hist, want, nbs, what, pmax=PLANE_MAX):
    """version-3 / 4 container: every stream's rANS bytes behind its header are the spec's; the whole payload is the
    oracle's packing of them"""
    hd, lo, a = _sections(raw)
    P, t, C = sym.shape
    half = a[lo.off_lengths: lo.off_lengths + P * C].reshape(P, C)
    cnt, ln, rans = O.v3_unpack(a[lo.off_payload: hd.total_bytes], half, nbs, t)
    assert np.array_equal(cnt, hist), f"{what}: stream header counts"
    _compare_streams(rans, ln, want, sym, cdfs, 0, t, what, pmax)
    lens = np.array([[len(w) for w in row] for row in want], np.int32)
    pl, half_o = O.v3_pack(hist, nbs, lens, np.frombuffer(b"".join(b"".join(row) for row in want), np.uint8))
    assert np.array_equal(half, half_o) and bytes(a[lo.off_payload: hd.total_bytes]) == pl.tobytes(), f"{what}: packing"


def _oracle_equal(raw, sym, cdfs, T, coder, what):
    """coder 0: the arithmetic coder's payload against the oracle's, group by group"""
    hd, lo, a = _sections(raw)
    P, _, C = sym.shape
    lengths = a[lo.off_lengths: lo.off_lengths + hd.ngroups * P * C * 4].view(np.int32).reshape(hd.ngroups, P, C)
    off = lo.off_payload
    for k in range(hd.ngroups):
        g = min(R.G, T - k * R.G)
        bs, ln = O.encode_group(cdfs, sym.view(np.int8), k * R.G, g, coder)
        assert np.array_equal(lengths[k], ln) and bytes(a[off: off + bs.size]) == bs.tobytes(), f"{what}, group {k}"
        off += bs.size


# ------------------------------------------------------------------------------------------------ 1. the sweep
def test_rans_put_exhaustive_sweep():
    """every (f, q), both ends of the bucket, plus the push branch on the states below 2^16"""
    lib = ctypes.CDLL(R.build_devsim())
    lib.devsim_rans_sweep.argtypes = [ctypes.c_void_p]
    out = (ctypes.c_ulonglong * 12)()
    rc = lib.devsim_rans_sweep(ctypes.cast(out, ctypes.c_void_p))
    assert rc == 0, f"CUDA error {rc}"
    steps, bad, fix, pushes = (int(out[k]) for k in range(4))
    name = torch.cuda.get_device_name(0)
    print(f"\nrans_put sweep on {name}: {steps} steps ({pushes} behind a push), {bad} wrong, {fix} of the "
          f"{steps - pushes} plain steps took the fix-up ({100.0 * fix / (steps - pushes):.3f} %), kernel {int(out[11])} us")
    assert bad == 0, (f"{bad} wrong states; first: f = {int(out[4])}, q = {int(out[5])}, case {int(out[6])} "
                      f"(0: x = q f, 1: x = q f + f - 1, 2 / 3: behind a push), x = {int(out[7]):#x}, estimate "
                      f"{int(out[10])}, state {int(out[8]):#x}, want {int(out[9]):#x}")
    assert steps - pushes == 2 * 65535 * 65535 and pushes > 2 * 600000
    assert 0 < fix < steps


# ------------------------------------------------------------------------------------------------ 2. own-CDF tiles
@pytest.mark.parametrize("dt", [0, 1], ids=["bf16", "fp16"])
def test_own_cdf_tiles(fx, expect, dt, monkeypatch):
    """every token count of the set; t = 256 and the odd-indexed or even-indexed others per dtype take every path"""
    N = _N()
    for k, t in enumerate(R.own_ts(fx)):
        full = t == 256 or k % 2 == dt
        rng = np.random.default_rng(100 * dt + t)
        sym = R.own_tile(fx, t, PLANE_MAX)
        C = sym.shape[2]
        cdfs, hist = R.own_cdfs(sym)
        what = f"own-CDF tile t = {t}, dtype {dt}"
        x = _tensor(_unplanes(E.kv_for_symbols(sym, PLANE_MAX, dt)), dt, 1, C)
        view = _source("blob", x, rng)
        want = expect.group(sym, cdfs, PLANE_MAX, 0, t, True)
        expect.group(sym, cdfs, PLANE_MAX, 0, t, True, E.header_lens(hist, NBS))
        raw2, = _encode_chunks(view, 0, 1, t, t, KB, VB, N.CODER_RANS)
        _check_v2(raw2, sym, cdfs, [want], f"{what}, coder 1")
        raw3, = _encode_chunks(view, 0, 1, t, t, KB, VB, N.CODER_RANS_COMPACT)
        _check_v3(raw3, sym, cdfs, hist, want, NBS, f"{what}, coder 2")
        combos = ALL_COMBOS if full else [ALL_COMBOS[k % len(ALL_COMBOS)]]
        _decode_all([raw3], N.CODER_RANS_COMPACT, sym, hist, NBS, 1, C, dt, rng, monkeypatch, combos, f"{what}, coder 2", t)
        _decode_all([raw2], N.CODER_RANS, sym, hist, NBS, 1, C, dt, rng, monkeypatch, combos[:4], f"{what}, coder 1", t)
        if full:
            raw0, = _encode_chunks(view, 0, 1, t, t, KB, VB, 0)
            _oracle_equal(raw0, sym, cdfs, t, O.CODER_AC, f"{what}, coder 0")
            _decode_all([raw0], 0, sym, hist, NBS, 1, C, dt, rng, monkeypatch, combos[:2], f"{what}, coder 0", t)
            assert _containers(_encode_layers(view, 0, 1, t, t, KB, VB, _rand_partition(rng, L))) == [raw3], \
                f"{what}: layer-split encode != encode_chunks"
            assert _encode_chunks(_source("paged", x, rng), 0, 1, t, t, KB, VB, N.CODER_RANS_COMPACT) == [raw3], \
                f"{what}: paged source != blob source"
            assert _encode_chunks(_source("paged", x, rng), 0, 1, t, t, KB, VB, N.CODER_RANS) == [raw2], \
                f"{what}: paged source != blob source, coder 1"


@pytest.mark.parametrize("dt", [0, 1], ids=["bf16", "fp16"])
def test_own_cdf_tiles_latent(fx, expect, dt):
    """a latent (version-4) descriptor: the key planes of the t = 256, 255 and 5 tiles as 15 latent layers"""
    from lmcache_b200.codec import KvView
    N = _N()
    lib = N.lib()
    pmax, nbs = PLANE_MAX[:L], NBS[:L]
    for t in (256, 255, 5):
        sym = np.ascontiguousarray(R.own_tile(fx, t, PLANE_MAX)[:L])
        D = sym.shape[2]
        cdfs, hist = R.own_cdfs(sym)
        want = expect.group(sym, cdfs, pmax, 0, t, True)
        x = torch.from_numpy(np.ascontiguousarray(E.kv_for_symbols(sym, pmax, dt)).view(np.int16)).view(TDT[dt]).cuda()
        view = KvView.from_blob(x, "vllm")
        assert view.latent
        stride = (N.container_layout(L, 1, D, t, N.CODER_LATENT).max_total_bytes + 15) & ~15
        out = torch.empty(stride, dtype=torch.uint8, device="cuda")
        sizes = torch.zeros(1, dtype=torch.int64, device="cuda")
        wsb = N.check(lib.b200kv_encode_workspace_bytes(L, 1, D, t, 1, N.CODER_LATENT), "encode_workspace_bytes")
        ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
        N.check(lib.b200kv_encode_chunks(ctypes.byref(view.desc), 0, 1, t, t, N.float_array(KB), N.float_array(VB),
                                         N.CODER_RANS_COMPACT, out.data_ptr(), stride, sizes.data_ptr(), ws.data_ptr(),
                                         wsb, _s()), "encode_chunks")
        torch.cuda.synchronize()
        raw = bytes(out.cpu().numpy()[: int(sizes.cpu()[0])])
        assert raw[4] == 4
        _check_v3(raw, sym, cdfs, hist, want, nbs, f"latent t = {t}", pmax)
        for out_dt in (0, 1):
            dst = torch.full((L, t, D), 3.0, dtype=TDT[out_dt], device="cuda")
            dest = types.SimpleNamespace(view=KvView.from_blob(dst, "vllm"))
            assert _decode([raw], N.CODER_LATENT, dest, [0], KB, VB, dt) == [0], f"latent t = {t}: status"
            got = dst.cpu().view(torch.int16).numpy().view(np.uint16)
            _check_values(got, sym, pmax, hist, nbs, out_dt, f"latent t = {t} dtype {out_dt}")


def test_heads_window(fx, monkeypatch):
    """b200kv_decode_plan_heads over head 1 of the t = 256 tile split into two heads: that slice of the whole decode"""
    N = _N()
    t, dt = 256, 0
    rng = np.random.default_rng(9)
    sym = R.own_tile(fx, t, PLANE_MAX)
    if sym.shape[2] % 2:
        sym = np.concatenate([sym, sym[:, :, -1:]], axis=2)
    D = sym.shape[2] // 2
    x = _tensor(_unplanes(E.kv_for_symbols(sym, PLANE_MAX, dt)), dt, 2, D)
    raw3, = _encode_chunks(_source("blob", x, rng), 0, 1, t, t, KB, VB, N.CODER_RANS_COMPACT)
    for table in ("rows", "transposed"):
        monkeypatch.setenv("B200KV_DECODE_TABLE", table)
        dest = _Dest("vllm", L, 2, D, t, dt, 0, rng)
        assert _decode_heads([raw3], dest, 2, 1, 1, 1, dt, 1) == [0], f"window status, table {table}"
        got = dest.tokens()[:, :, :, 1:2].cpu().contiguous().view(torch.int16).numpy().view(np.uint16)
        want = Q.from_f32((sym[:, :, D:].astype(np.int64) - PLANE_MAX[:, None, None]).astype(np.float32), dt)
        assert np.array_equal(_planes(got.reshape(L, 2, t, D)), want), f"decode_plan_heads window, table {table}"
        assert bool((dest.tokens()[:, :, :, 0] == 3.0).all()), "decode_plan_heads wrote outside its head window"


# ------------------------------------------------------------------------------------------------ 3. chunk-wide CDF
@pytest.mark.parametrize("T", R.BIG_T)
def test_chunk_wide_cdf_groups(fx, expect, T, monkeypatch):
    """chunks of more than 256 tokens: coder 1's groups are the spec's streams under the chunk-wide CDF; coder 0 the
    oracle's; both decode to s - MAX with status 0"""
    N = _N()
    dt = T % 2
    rng = np.random.default_rng(T)
    sym = R.big_tile(fx, T, PLANE_MAX)
    C = sym.shape[2]
    cdfs, hist = R.own_cdfs(sym)
    x = _tensor(_unplanes(E.kv_for_symbols(sym, PLANE_MAX, dt)), dt, 1, C)
    view = _source("blob" if T % 3 else "paged", x, rng)
    want = [expect.group(sym, cdfs, PLANE_MAX, a, min(R.G, T - a), False) for a in range(0, T, R.G)]
    raw, = _encode_chunks(view, 0, 1, T, T, KB, VB, N.CODER_RANS)
    _check_v2(raw, sym, cdfs, want, f"T = {T}, coder 1")
    combos = [ALL_COMBOS[(T + 7 * k) % len(ALL_COMBOS)] for k in range(4)]
    _decode_all([raw], N.CODER_RANS, sym, hist, NBS, 1, C, dt, rng, monkeypatch, combos, f"T = {T}, coder 1", T)
    if T != R.LONG_T:
        raw0, = _encode_chunks(view, 0, 1, T, T, KB, VB, 0)
        _oracle_equal(raw0, sym, cdfs, T, O.CODER_AC, f"T = {T}, coder 0")
        _decode_all([raw0], 0, sym, hist, NBS, 1, C, dt, rng, monkeypatch, combos[:1], f"T = {T}, coder 0", T)


# ------------------------------------------------------------------------------------------------ 4. coverage
def test_coverage_is_complete(fx, expect):
    """runs last in the module: what the streams compared above reached"""
    missing = expect.cov.missing()
    assert not missing, f"the tiles no longer reach: {missing}"
    print(f"\nrANS edges reached: {len(expect.cov.items)} items; longest own-CDF stream {int(fx['longest'])} halfwords "
          f"(proven bound {R.PROVEN_MAX_HALFWORDS})")
