"""GPU: the CDF normaliser and the version-3 stream header at their edges, on every encode and decode path.

Every kernel is driven to PRESCRIBED histograms: each (plane, token) row holds its plane's MAX exactly (channel 0 is
symbol 0, x = -MAX, on every token), so the factor is 1 and x = s - MAX quantises to symbol s with no rounding; every
other channel's symbol column is the test's to choose, and a decoded value is s - MAX exactly in both output dtypes.
15 layers with key bins 4, 6, ..., 32 and value bins reversed put every nb on a key and on a value plane.

* witness tiles: the histograms of tests/golden/cdf_edges.npz (exact ties both ways, their neighbours, the rows where a
  float32 running sum, another summation order, n * fl32(1 / t), a double multiply, round-half-away, truncation or an
  FMA differ from the reference) at every token count of the set.  Coders 1 and 0: the stored CDF rows == the
  reference-made rows (encode_kernel's CdfAccum2 at t <= 256, cdf_kernel's CdfAccum at 257 .. 1030 tokens).  Coder 2 and
  a latent descriptor: the stream headers hold the prescribed counts, payload and half-lengths are the oracle's packing
  of the oracle's rANS streams under the reference-made CDF; the layer-split encoder and a paged source give the same
  bytes.  Every container decodes (decode_chunks, plan + decode_layers, both table layouts, vllm / huggingface / paged
  destinations, both dtypes) to s - MAX bit for bit with status 0 on every chunk: a rebuilt table that is one off in a
  used entry cannot bring the rANS state back to 2^16.
* header layouts (cdf_edges.LAYOUTS): tiles built lane by lane so that warps fall on both sides of the decoder's
  reader threshold, headers of 8 / 10 / 12 bytes sit side by side, warps skip different symbols, count bytes are 1 and
  255, warps and tiles are partial, and a decode_plan_heads window flips a warp's reader.  What was reached is computed
  from the histograms (cdf_edges.Coverage) and asserted complete."""
import ctypes
import types

import numpy as np
import pytest
import torch

from oracle import oracle as O

import cdf_edges as E
import quant_edges as Q
from test_gpu_layer_split import _Dest, _containers, _decode, _encode_chunks, _encode_layers, _rand_partition, _s, _source
from test_gpu_quant_edges import _decode_heads, _planes, _tensor, _unplanes

pytestmark = pytest.mark.gpu
TDT = (torch.bfloat16, torch.float16)
L = 15
KB, VB, MK, MV = Q.plane_maxes(L)
PLANE_MAX = np.array(MK + MV)            # MAX of plane kv * L + l
NBS = [2 * (int(m) + 1) for m in PLANE_MAX]
FULL_T = (1, 2, 3, 17, 37, 64, 255, 256)  # token counts whose witness tiles take every path; the others rotate


def _N():
    from lmcache_b200 import _native as N
    return N


@pytest.fixture(scope="module")
def fx():
    return {k: v for k, v in E.load().items()}


@pytest.fixture(scope="module")
def coverage():
    return E.Coverage()


def _where(hist, nbs, p, c, window=None):
    nb = nbs[p]
    rd = E.warp_readers(hist[p:p + 1], [nb], window)[0, c // E.WARP]
    used = {int(k): int(hist[p, c, k]) for k in np.flatnonzero(hist[p, c])}
    return (f"plane {p} (nb {nb}), channel {c} (lane {c % E.WARP} of warp {c // E.WARP}), header "
            f"{E.header_len(E.mask_of(hist[p, c]), nb)} bytes, {('byte', 'word', 'no')[rd]} reader, histogram {used}")


def _symbols(hist, t, rng):
    """sym uint8 [P, t, C]: column (p, c) has histogram hist[p, c], in a shuffled order"""
    P, C = hist.shape[:2]
    sym = np.empty((P, t, C), np.uint8)
    for p in range(P):
        for c in range(C):
            sym[p, :, c] = E.column(hist[p, c], rng)
    return sym


def _sections(raw):
    from lmcache_b200.codec import container_layout_of, parse_header
    hd = parse_header(raw)
    return hd, container_layout_of(hd), np.frombuffer(raw, np.uint8)


def _check_cdf_rows(raw, hist, want_cdf, nbs, what):
    hd, lo, a = _sections(raw)
    P, C = hist.shape[:2]
    cdf = a[lo.off_cdf: lo.off_cdf + P * C * 33 * 2].view(np.int16).reshape(P, C, 33)
    bad = np.argwhere(cdf != want_cdf)
    if bad.size:
        p, c, e = (int(v) for v in bad[0])
        raise AssertionError(f"{what}: CDF row != reference, {np.unique(bad[:, :2], axis=0).shape[0]} streams; first: "
                             f"{_where(hist, nbs, p, c)}, t = {hd.ntokens}: cdf[{e}] = {int(cdf[p, c, e]) & 0xFFFF}, "
                             f"reference {int(want_cdf[p, c, e]) & 0xFFFF}")


def _oracle_v3(hist, want_cdf, sym, nbs, t):
    """(payload, half-lengths) the oracle packs for these symbols under the given CDF rows"""
    bs, ln = O.encode_group(want_cdf, sym.view(np.int8), 0, t, O.CODER_RANS)
    return O.v3_pack(hist.astype(np.uint32), nbs, ln, bs)


def _check_v3(raw, hist, want_cdf, sym, nbs, t, what):
    """the stream headers hold the prescribed counts; half-lengths and payload are the oracle's; returns half"""
    hd, lo, a = _sections(raw)
    P, C = hist.shape[:2]
    assert hd.ntokens == t and hd.nb == list(nbs), what
    half = a[lo.off_lengths: lo.off_lengths + P * C].reshape(P, C)
    cnt, _, _ = O.v3_unpack(a[lo.off_payload: hd.total_bytes], half, nbs, t)
    bad = np.argwhere((cnt != hist).any(axis=2))
    assert bad.size == 0, (f"{what}: stream header counts != prescribed; first: {_where(hist, nbs, *bad[0])}, got "
                           f"{ {int(k): int(cnt[tuple(bad[0])][k]) for k in np.flatnonzero(cnt[tuple(bad[0])])} }")
    pl, half_o = _oracle_v3(hist, want_cdf, sym, nbs, t)
    bad = np.argwhere(half != half_o)
    assert bad.size == 0, f"{what}: stream length != oracle's; first: {_where(hist, nbs, *bad[0])}"
    assert bytes(a[lo.off_payload: hd.total_bytes]) == pl.tobytes(), f"{what}: payload != oracle's packing"
    return half


def _want_bits(sym, pmax, out_dt):
    return Q.from_f32((sym.astype(np.int64) - np.asarray(pmax)[:, None, None]).astype(np.float32), out_dt)


def _check_values(got, sym, pmax, hist, nbs, out_dt, what, window=None):
    want = _want_bits(sym, pmax, out_dt)
    bad = np.argwhere(got != want)
    if bad.size:
        p, tok, c = (int(v) for v in bad[0])
        raise AssertionError(f"{what}: decoded value != s - MAX at {bad.shape[0]} places; first: token {tok}, "
                             f"{_where(hist, nbs, p, c, window)}: want symbol {int(sym[p, tok, c])}, got value bits "
                             f"{int(got[p, tok, c]):#06x}")


def _decode_all(raws, coder, sym, hist, nbs, H, D, dt, rng, monkeypatch, combos, what, dst_step):
    """decode the containers (consecutive chunks) by each (destination kind, output dtype, table layout, split) of combos"""
    T = sym.shape[1]
    for kind, out_dt, table, split in combos:
        monkeypatch.setenv("B200KV_DECODE_TABLE", table)
        dest = _Dest(kind, L, H, D, T, out_dt, 3, rng)
        parts = _rand_partition(rng, L) if split else None
        st = _decode(raws, coder, dest, [dest.tok0 + j * dst_step for j in range(len(raws))], KB, VB, dt, parts=parts)
        w = f"{what}, {kind} dtype {out_dt} table {table} parts {parts}"
        assert st == [0] * len(raws), f"{w}: decode status {st}"
        _check_values(_planes(dest.bits()), sym, PLANE_MAX, hist, nbs, out_dt, w)
        assert dest.rest_untouched(), w
    monkeypatch.delenv("B200KV_DECODE_TABLE")


ALL_COMBOS = [(k, o, tb, sp) for k, o in (("vllm", 0), ("hf", 1), ("paged", 0)) for tb in ("rows", "transposed")
              for sp in (False, True)]


def _run_tile(hist, want_cdf, t, H, D, dt, rng, monkeypatch, full, what, coverage=None, k=0):
    """one chunk of t <= 256 tokens whose stream (p, c) has histogram hist[p, c]: every encode path and decode path when
    `full`, else coder 2 and coder 1 with one decode each (the k-th combination)"""
    N = _N()
    C = H * D
    sym = _symbols(hist, t, rng)
    x = _tensor(_unplanes(E.kv_for_symbols(sym, PLANE_MAX, dt)), dt, H, D)
    view = _source("blob", x, rng)
    combos = ALL_COMBOS if full else [ALL_COMBOS[k % len(ALL_COMBOS)]]
    # coder 2 (version 3): headers, lengths, payload
    raw3, = _encode_chunks(view, 0, 1, t, t, KB, VB, N.CODER_RANS_COMPACT)
    half = _check_v3(raw3, hist, want_cdf, sym, NBS, t, f"{what}, coder 2")
    if coverage is not None:
        coverage.add(hist, t, NBS)
        coverage.add_phases(hist, NBS, half)
    _decode_all([raw3], N.CODER_RANS_COMPACT, sym, hist, NBS, H, D, dt, rng, monkeypatch, combos, f"{what}, coder 2", t)
    # coders 1 and 0 (the fused kernel stores the CDF rows)
    for coder in ((1, 0) if full else (1,)):
        raw, = _encode_chunks(view, 0, 1, t, t, KB, VB, coder)
        _check_cdf_rows(raw, hist, want_cdf, NBS, f"{what}, coder {coder}")
        _decode_all([raw], coder, sym, hist, NBS, H, D, dt, rng, monkeypatch, combos[:2], f"{what}, coder {coder}", t)
    if full:
        assert _containers(_encode_layers(view, 0, 1, t, t, KB, VB, _rand_partition(rng, L))) == [raw3], \
            f"{what}: layer-split encode != encode_chunks"
        assert _encode_chunks(_source("paged", x, rng), 0, 1, t, t, KB, VB, N.CODER_RANS_COMPACT) == [raw3], \
            f"{what}: paged source != blob source"
    return sym, raw3


def _witness_tile(fx, t):
    """(hist [2L, C, 33], reference CDF rows [2L, C, 33]) holding every fixture row of t tokens on every plane that can
    hold its top symbol (planes cycle through the rows that fit them); channel 0 pins the row maxima"""
    rows = np.flatnonzero(fx["t"] == t)
    top = np.array([int(np.flatnonzero(fx["counts"][i])[-1]) for i in rows])
    C = 1 + rows.size
    hist = np.zeros((2 * L, C, 33), np.uint16)
    cdf = np.zeros((2 * L, C, 33), np.int16)
    lone = np.zeros(33, np.uint16)
    lone[0] = t
    for p in range(2 * L):
        fit = rows[top <= 2 * PLANE_MAX[p]]
        pick = fit[(np.arange(C - 1) + p) % fit.size] if fit.size else None
        hist[p, 0], cdf[p, 0] = lone, E.spec_cdf(lone, t)
        for c in range(1, C):
            if pick is None:
                hist[p, c], cdf[p, c] = hist[p, 0], cdf[p, 0]
            else:
                hist[p, c], cdf[p, c] = fx["counts"][pick[c - 1]], fx["cdf"][pick[c - 1]]
    return hist, cdf


# ------------------------------------------------------------------------------------------------ 1. witness tiles
@pytest.mark.parametrize("dt", [0, 1], ids=["bf16", "fp16"])
def test_witness_tiles_one_group(fx, dt, monkeypatch):
    """every token count <= 256 of the witness set: the t of FULL_T on every path, the others on coder 2 + coder 1 with
    the decode combination rotating.  bf16 takes the even-indexed token counts and fp16 the odd ones, FULL_T both."""
    ts = [int(t) for t in np.unique(fx["t"]) if t <= 256]
    assert set(FULL_T) <= set(ts)
    seen = 0
    for k, t in enumerate(ts):
        full = t in FULL_T
        if not full and k % 2 != dt:
            continue
        rng = np.random.default_rng(1000 * dt + t)
        hist, cdf = _witness_tile(fx, t)
        _run_tile(hist, cdf, t, 1, hist.shape[1], dt, rng, monkeypatch, full, f"witness tile t = {t}", k=k)
        seen += 1
    assert seen >= len(ts) // 2


@pytest.mark.parametrize("dt", [0, 1], ids=["bf16", "fp16"])
def test_witness_tiles_latent(fx, dt):
    """a latent (version-4) descriptor: the key planes of the t = 256, 255 and 37 witness tiles as 15 latent layers"""
    from lmcache_b200.codec import KvView
    N = _N()
    lib = N.lib()
    pmax, nbs = PLANE_MAX[:L], NBS[:L]
    for t in (256, 255, 37):
        rng = np.random.default_rng(t + dt)
        hist, cdf = (a[:L] for a in _witness_tile(fx, t))
        D = hist.shape[1]
        sym = _symbols(hist, t, rng)
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
        _check_v3(raw, hist, cdf, sym, nbs, t, f"latent t = {t}")
        for out_dt in (0, 1):
            dst = torch.full((L, t, D), 3.0, dtype=TDT[out_dt], device="cuda")
            dest = types.SimpleNamespace(view=KvView.from_blob(dst, "vllm"))
            assert _decode([raw], N.CODER_LATENT, dest, [0], KB, VB, dt) == [0], f"latent t = {t}: status"
            got = dst.cpu().view(torch.int16).numpy().view(np.uint16)
            _check_values(got, sym, pmax, hist, nbs, out_dt, f"latent t = {t} dtype {out_dt}")


@pytest.mark.parametrize("t", E.BIG_T)
def test_witness_tiles_chunk_wide_cdf(fx, t, monkeypatch):
    """chunks of 257 .. 1030 tokens (two to five groups, one chunk-wide CDF from cdf_kernel, fl32(n / t) with n and t
    past 256): coders 1 and 0 store the reference-made rows and decode to s - MAX with status 0"""
    dt = t % 2
    rng = np.random.default_rng(t)
    hist, cdf = _witness_tile(fx, t)
    H, D = 1, hist.shape[1]
    sym = _symbols(hist, t, rng)
    x = _tensor(_unplanes(E.kv_for_symbols(sym, PLANE_MAX, dt)), dt, H, D)
    view = _source("blob" if t % 3 else "paged", x, rng)
    for coder in (1, 0):
        raw, = _encode_chunks(view, 0, 1, t, t, KB, VB, coder)
        assert _sections(raw)[0].ngroups == -(-t // 256)
        _check_cdf_rows(raw, hist, cdf, NBS, f"t = {t}, coder {coder}")
        combos = [ALL_COMBOS[(t + 5 * coder) % len(ALL_COMBOS)], ALL_COMBOS[(t + 5 * coder + 7) % len(ALL_COMBOS)]]
        _decode_all([raw], coder, sym, hist, NBS, H, D, dt, rng, monkeypatch, combos, f"t = {t}, coder {coder}", t)


# ------------------------------------------------------------------------------------------------ 2. header layouts
def test_header_layouts(coverage, monkeypatch):
    """every layout tile of cdf_edges.layout_cases() on every encode and decode path; the window case also through
    b200kv_decode_plan_heads over head 1 alone, whose result must be that slice of the whole decode, status 0"""
    for i, (name, t, H, D, win) in enumerate(E.layout_cases()):
        rng = np.random.default_rng(50 + i)
        dt = i % 2
        C = H * D
        hist = E.LAYOUTS[name](NBS, C, t, rng)
        cdf = E.spec_cdf(hist, t)
        what = f"layout {name} t = {t} C = {H} x {D}"
        sym, raw3 = _run_tile(hist, cdf, t, H, D, dt, rng, monkeypatch, True, what, coverage)
        if win:
            h0, k = win
            window = (h0 * D, (h0 + k) * D)
            coverage.add(hist, t, NBS, window)
            half = _sections(raw3)
            half = half[2][half[1].off_lengths: half[1].off_lengths + 2 * L * C].reshape(2 * L, C)
            coverage.add_phases(hist, NBS, half, window)
            dest = _Dest("vllm", L, k + 1, D, t, dt, 0, rng)
            assert _decode_heads([raw3], dest, H, h0, 1, k, dt, 1) == [0], f"{what}: window status"
            got = dest.tokens()[:, :, :, 1:1 + k].cpu().contiguous().view(torch.int16).numpy().view(np.uint16)
            whole = _want_bits(sym, PLANE_MAX, dt)            # outside the window: not decoded, not compared
            whole[:, :, window[0]:window[1]] = _planes(got.reshape(L, 2, t, k * D))
            _check_values(whole, sym, PLANE_MAX, hist, NBS, dt, f"{what}: decode_plan_heads window", window)
            assert bool((dest.tokens()[:, :, :, 0] == 3.0).all()), "decode_plan_heads wrote outside its head window"
    missing = coverage.missing()
    print("\nheader layouts reached: " + coverage.report())
    assert not missing, f"the header layouts no longer reach: {missing}"
    assert coverage.window_flips > 0 and coverage.phases, "no window flipped a warp's reader / no phases recorded"
