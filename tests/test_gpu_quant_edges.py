"""GPU: the quantiser and dequantiser at their rounding edges, on every encode and decode path, held to the numpy spec of
tests/quant_edges.py bit for bit.

15 layers with key bins 4, 6, ..., 32 and value bins in the reverse order put every MAX 1..15 on a key and on a value
plane.  The inputs are the witness set tests/golden/quant_edges.npz (exact ties and their neighbours, the pairs where
FMA contraction, a reciprocal factor, (x / m) * MAX, round-half-away, flush-to-zero or truncating half conversions
differ from the spec, subnormal / overflowing / infinite / NaN maxima) packed into rows whose maximum sits at the first,
last, last-partial-vector and last-partial-tile channel.

* encode: b200kv_encode_chunks coder 2 (256-token chunks, ragged last), coders 0 / 1 (512- and 700-token chunks),
  b200kv_encode_layers in a random layer partition, a latent (version-4) descriptor; vllm blob with D = 128 (vector
  absmax), H x D = 3 x 33 (scalar absmax, partial tiles), a paged cache with a random slot map.  Per container: maxima ==
  spec_absmax; symbols read back by the CPU oracle (independent of the GPU decoder) == spec_quant; per-stream counts or
  CDF rows == those of the spec symbols; layer-split and paged-source containers byte-identical to encode_chunks'.
* decode: decode_chunks into vllm bf16, huggingface fp16 and a paged cache, both rANS table layouts, plan + decode_layers
  in a partition, a decode_plan_heads window: values == spec_dequant bit for bit (NaN == NaN, -0.0 kept), status 0.
* every (symbol, MAX, maximum bit pattern, output dtype): rows emitting all 2 MAX + 1 symbols, the maxima section
  rewritten to all 65536 patterns of the max dtype, decoded into both output dtypes.
* the quantiser over every finite x of each dtype against the ladder of row maxima (quant_edges.ladder), on the default
  path (coder 2, 256 tokens); symbols read back by rewriting each row's maximum to MAX (value = sym - MAX exactly).
  To stay inside about a minute the ladder is split by index modulo 15 over the layers, so each maximum is swept at
  two MAX values (its layer's key and value planes) rather than all fifteen; the witness set covers every MAX."""
import ctypes
import types

import numpy as np
import pytest
import torch

import quant_edges as Q
from test_gpu_layer_split import _Dest, _containers, _decode, _encode_chunks, _encode_layers, _rand_partition, _s, _source

pytestmark = pytest.mark.gpu
TDT = (torch.bfloat16, torch.float16)
L = 15
KB, VB, MK, MV = Q.plane_maxes(L)
PLANE_MAX = np.array(MK + MV)            # MAX of plane kv * L + l


def _N():
    from lmcache_b200 import _native as N
    return N


@pytest.fixture(scope="module")
def fx():
    return Q.load()


def _planes(bits):
    """[L, 2, t, C] -> [2L, t, C] in container plane order (keys, then values)"""
    return np.ascontiguousarray(bits.transpose(1, 0, 2, 3).reshape(-1, bits.shape[2], bits.shape[3]))


def _unplanes(p, L_=L):
    return np.ascontiguousarray(p.reshape(2, L_, p.shape[1], p.shape[2]).transpose(1, 0, 2, 3))


def _witness_bits(fx, dt, C, ragged=True):
    rows = {M: Q.pack_rows(*Q.fixture_pairs(fx, dt, M)[:2], C, dt)[0] for M in Q.MAXES}
    T = max(r.shape[0] for r in rows.values())
    if ragged and T % 256 == 0:
        T += 17
    return Q.assemble(rows, L, T)[0]


def _tensor(bits, dt, H, D):
    L_, two, T, C = bits.shape
    return torch.from_numpy(np.ascontiguousarray(bits).view(np.int16)).view(TDT[dt]).reshape(L_, two, T, H, D).cuda()


def _where(planes, idx, maxes, pmax, what):
    p, t, c = (int(i) for i in idx)
    kind = ("key" if p < len(pmax) // 2 else "value") if len(pmax) == 2 * L else "latent"
    return (f"{what}: MAX {pmax[p]} ({kind} plane {p}), token {t} channel {c}: x={int(planes[p, t, c]):#06x} "
            f"m={int(maxes[p, t]):#06x}")


def _spec_syms(planes, maxes, pmax, dt):
    return np.stack([Q.spec_quant(planes[p], maxes[p][:, None], int(pmax[p]), dt) for p in range(planes.shape[0])])


def _check_container(raw, planes, dt, kb, vb, pmax):
    """maxima == spec_absmax, symbols read back by the oracle == spec_quant, per-stream counts / CDF rows == the spec
    symbols'.  planes: the chunk's input [P, t, C].  Returns the stored maxima [P, t]."""
    from oracle import oracle as O
    from lmcache_b200.codec import container_layout_of, parse_header
    hd = parse_header(raw)
    P, t, C = planes.shape
    assert hd.ntokens == t and hd.H * hd.D == C and hd.max_dtype == dt
    lo = container_layout_of(hd)
    a = np.frombuffer(raw, np.uint8)
    maxes = a[lo.off_maxes: lo.off_maxes + 2 * P * t].view(np.uint16).reshape(P, t)
    ok = Q.eq_nan(maxes, Q.spec_absmax(planes), dt)
    assert ok.all(), f"maxima section != spec_absmax at plane / token {np.argwhere(~ok)[0]}"
    want = _spec_syms(planes, maxes, pmax, dt)
    got = np.zeros((P, t, C), np.uint8)
    if hd.version >= 3:
        nb = [2 * (int(b) // 2) for b in (list(kb[:hd.L]) + (list(vb[:hd.L]) if P == 2 * hd.L else []))]
        half = a[lo.off_lengths: lo.off_lengths + P * C].reshape(P, C)
        cnt, ln, rans = O.v3_unpack(a[lo.off_payload: hd.total_bytes], half, nb, t)
        O.decode_group(O.cdf_from_counts(cnt, t), rans, ln, got, 0, t, O.CODER_RANS)
        tables = ("stream histograms", cnt, O.counts(want.view(np.int8)))
    else:
        cdf = a[lo.off_cdf: lo.off_cdf + P * C * 33 * 2].view(np.int16).reshape(P, C, 33)
        tables = ("CDF rows", cdf, O.cdf(want.view(np.int8)))
        G = hd.ngroups
        lengths = a[lo.off_lengths: lo.off_lengths + G * P * C * 4].view(np.int32).reshape(G, P, C)
        off = lo.off_payload
        for g in range(G):
            n = int(lengths[g].sum())
            O.decode_group(cdf, a[off: off + n], lengths[g], got, g * 256, min(256, t - g * 256), hd.version - 1)
            off += n
    bad = np.argwhere(got != want)
    assert bad.size == 0, (_where(planes, bad[0], maxes, pmax, f"symbol != spec_quant ({bad.shape[0]} of them)") +
                           f": want {int(want[tuple(bad[0])])} got {int(got[tuple(bad[0])])}")
    assert np.array_equal(tables[1], tables[2]), f"{tables[0]} != those of the spec symbols"
    return maxes


def _want_values(planes, maxes, pmax, dt, out_dt):
    sym = _spec_syms(planes, maxes, pmax, dt)
    return np.stack([Q.spec_dequant(sym[p], maxes[p][:, None], int(pmax[p]), dt, out_dt) for p in range(sym.shape[0])])


def _check_values(got_planes, planes, maxes, pmax, dt, out_dt, what):
    want = _want_values(planes, maxes, pmax, dt, out_dt)
    ok = Q.eq_nan(got_planes, want, out_dt)
    if not ok.all():
        i = tuple(np.argwhere(~ok)[0])
        raise AssertionError(_where(planes, i, maxes, pmax, f"{what}: decoded value != spec_dequant "
                                                         f"({int((~ok).sum())} of them)") +
                             f": want {int(want[i]):#06x} got {int(got_planes[i]):#06x}")


def _chunks(T, cs):
    n = (T + cs - 1) // cs
    return n, T - (n - 1) * cs


def _dtok(n, cs, base=0):
    return [base + j * cs for j in range(n)]


# ------------------------------------------------------------------------------------------------ 1. witness set
@pytest.mark.parametrize("dt", [0, 1], ids=["bf16", "fp16"])
@pytest.mark.parametrize("H,D", [(1, 128), (3, 33)])
def test_witness_encode_decode_every_path(fx, dt, H, D, monkeypatch):
    N = _N()
    rng = np.random.default_rng(100 * dt + D)
    C = H * D
    bits = _witness_bits(fx, dt, C)
    T = bits.shape[2]
    x = _tensor(bits, dt, H, D)
    view = _source("blob", x, rng)
    planes = _planes(bits)

    # coder 2 at 256 tokens, ragged last chunk
    n, last = _chunks(T, 256)
    raws = _encode_chunks(view, 0, n, 256, last, KB, VB, N.CODER_RANS_COMPACT)
    maxes = np.concatenate([_check_container(r, planes[:, j * 256: j * 256 + (256 if j < n - 1 else last)], dt, KB, VB,
                                             PLANE_MAX) for j, r in enumerate(raws)], axis=1)
    # the layer-split encoder and a paged source: the same bytes
    assert _containers(_encode_layers(view, 0, n, 256, last, KB, VB, _rand_partition(rng, L))) == raws
    assert _encode_chunks(_source("paged", x, rng), 0, n, 256, last, KB, VB, N.CODER_RANS_COMPACT) == raws

    # decode: vllm bf16, huggingface fp16, paged (random dtype); both table layouts; whole and layer-split
    for i, (kind, out_dt) in enumerate((("vllm", 0), ("hf", 1), ("paged", int(rng.integers(0, 2))))):
        for table in ("rows", "transposed"):
            monkeypatch.setenv("B200KV_DECODE_TABLE", table)
            parts = None if (i + (table == "rows")) % 2 else _rand_partition(rng, L)
            dest = _Dest(kind, L, H, D, T, out_dt, 3, rng)
            st = _decode(raws, N.CODER_RANS_COMPACT, dest, _dtok(n, 256, dest.tok0), KB, VB, dt, parts=parts)
            assert st == [0] * n
            _check_values(_planes(dest.bits()), planes, maxes, PLANE_MAX, dt, out_dt, f"{kind} {table} parts={parts}")
            assert dest.rest_untouched()
    monkeypatch.delenv("B200KV_DECODE_TABLE")

    # a decode_plan_heads window: source heads [h0, h0 + k) into a destination of k + 1 heads from head 1
    h0, k = (1, 2) if H == 3 else (0, 1)
    dest = _Dest("vllm", L, k + 1, D, T, dt, 0, rng)
    status = _decode_heads(raws, dest, H, h0, 1, k, dt, n)
    assert status == [0] * n
    got = dest.tokens()[:, :, :, 1:1 + k].cpu()
    got = got.contiguous().view(torch.int16).numpy().view(np.uint16).reshape(L, 2, T, k * D)
    sl = np.ascontiguousarray(bits.reshape(L, 2, T, H, D)[:, :, :, h0:h0 + k].reshape(L, 2, T, k * D))
    wv = _want_values(planes, maxes, PLANE_MAX, dt, dt).reshape(2 * L, T, H, D)[:, :, h0:h0 + k].reshape(2 * L, T, -1)
    ok = Q.eq_nan(_planes(got), wv, dt)
    assert ok.all(), _where(_planes(sl), np.argwhere(~ok)[0], maxes, PLANE_MAX, "decode_plan_heads window")
    assert bool((dest.tokens()[:, :, :, 0] == 3.0).all()), "decode_plan_heads wrote outside its head window"

    # coders 0 and 1: 512- and 700-token chunks (multi-group, the split cdf_kernel + checked quant_symbol path)
    for coder in (0, 1):
        for cs in (512, 700):
            n2, last2 = _chunks(T, cs)
            raws2 = _encode_chunks(view, 0, n2, cs, last2, KB, VB, coder)
            mx2 = np.concatenate([_check_container(r, planes[:, j * cs: j * cs + (cs if j < n2 - 1 else last2)], dt, KB,
                                                   VB, PLANE_MAX) for j, r in enumerate(raws2)], axis=1)
            assert np.array_equal(mx2, maxes)
            if cs == 700:
                dest = _Dest("vllm", L, H, D, T, 1 - dt, 0, rng)
                assert _decode(raws2, coder, dest, _dtok(n2, cs), KB, VB, dt) == [0] * n2
                _check_values(_planes(dest.bits()), planes, maxes, PLANE_MAX, dt, 1 - dt, f"coder {coder}")


def _decode_heads(raws, dest, src_H, h0, d0, k, max_dtype, n):
    """b200kv_decode_plan_heads + decode_layers over all layers: heads [h0, h0 + k) of every container -> dest heads from
    d0 on.  Returns the status words."""
    from lmcache_b200.codec import parse_header
    N = _N()
    lib = N.lib()
    offs, o = [], 0
    for r in raws:
        offs.append(o)
        o = (o + len(r) + 15) & ~15
    total = o + N.READ_SLACK
    host = np.zeros(total, np.uint8)
    for r, off in zip(raws, offs):
        host[off: off + len(r)] = np.frombuffer(r, np.uint8)
    buf = torch.from_numpy(host).cuda()
    ntok = [int(parse_header(r).ntokens) for r in raws]
    v = dest.view
    wsb = N.check(lib.b200kv_decode_workspace_bytes(v.L, src_H, v.D, max(ntok), n), "decode_workspace_bytes")
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    status = torch.full((n,), 0x5555, dtype=torch.int32, device="cuda")
    plan = N.DecodePlan()
    N.check(lib.b200kv_decode_plan_heads(buf.data_ptr(), total, N.i64_array(offs), N.i64_array([len(r) for r in raws]),
                                         N.i32_array(ntok), N.i64_array(_dtok(n, 256)), n, max_dtype,
                                         N.CODER_RANS_COMPACT, ctypes.byref(v.desc), N.float_array(KB),
                                         N.float_array(VB), status.data_ptr(), ws.data_ptr(), wsb, ctypes.byref(plan),
                                         _s(), src_H, N.i32_array([h0] * n), N.i32_array([d0] * n),
                                         N.i32_array([k] * n)), "decode_plan_heads")
    N.check(lib.b200kv_decode_layers(ctypes.byref(plan), 0, v.L, _s()), "decode_layers")
    torch.cuda.synchronize()
    return status.cpu().tolist()


@pytest.mark.parametrize("dt", [0, 1], ids=["bf16", "fp16"])
def test_witness_latent(fx, dt):
    """a latent (version-4) descriptor: the key planes' witness rows as 15 latent layers with key bins 4..32"""
    from lmcache_b200.codec import KvView
    N = _N()
    D = 40
    bits = np.ascontiguousarray(_witness_bits(fx, dt, D)[:, 0])              # [L, T, D]
    T = bits.shape[1]
    x = torch.from_numpy(bits.view(np.int16)).view(TDT[dt]).cuda()
    view = KvView.from_blob(x, "vllm")
    assert view.latent
    n, last = _chunks(T, 256)
    lib = N.lib()
    stride = (N.container_layout(L, 1, D, 256, N.CODER_LATENT).max_total_bytes + 15) & ~15
    out = torch.empty(n * stride, dtype=torch.uint8, device="cuda")
    sizes = torch.zeros(n, dtype=torch.int64, device="cuda")
    wsb = N.check(lib.b200kv_encode_workspace_bytes(L, 1, D, 256, n, N.CODER_LATENT), "encode_workspace_bytes")
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    N.check(lib.b200kv_encode_chunks(ctypes.byref(view.desc), 0, n, 256, last, N.float_array(KB), N.float_array(VB),
                                     N.CODER_RANS_COMPACT, out.data_ptr(), stride, sizes.data_ptr(), ws.data_ptr(), wsb,
                                     _s()), "encode_chunks")
    torch.cuda.synchronize()
    buf, sz = out.cpu().numpy(), sizes.cpu().tolist()
    raws = [bytes(buf[j * stride: j * stride + sz[j]]) for j in range(n)]
    assert all(r[4] == 4 for r in raws)
    pmax = np.array(MK)
    maxes = np.concatenate([_check_container(r, bits[:, j * 256: j * 256 + (256 if j < n - 1 else last)], dt, KB, VB,
                                             pmax) for j, r in enumerate(raws)], axis=1)
    for out_dt in (0, 1):
        dst = torch.full((L, T, D), 3.0, dtype=TDT[out_dt], device="cuda")

        dest = types.SimpleNamespace(view=KvView.from_blob(dst, "vllm"))
        assert _decode(raws, N.CODER_LATENT, dest, _dtok(n, 256), KB, VB, dt) == [0] * n
        got = dst.cpu().view(torch.int16).numpy().view(np.uint16)
        _check_values(got, bits, maxes, pmax, dt, out_dt, "latent")


# ------------------------------------------------------------------------------------------------ 2. every maximum
@pytest.mark.parametrize("dt", [0, 1], ids=["bf16", "fp16"])
def test_dequantiser_every_maximum_bit_pattern(dt):
    """rows emitting all 2 MAX + 1 symbols on every plane, the maxima section rewritten to all 65536 bit patterns of the
    max dtype (subnormal, infinite and NaN maxima included), decoded into both output dtypes == spec_dequant"""
    from lmcache_b200.codec import container_layout_of, parse_header
    N = _N()
    C, T = 32, 65536
    sym = np.stack([np.arange(C) % (2 * M + 1) for M in PLANE_MAX])                     # [2L, C]
    vals = (sym - PLANE_MAX[:, None]).astype(np.float32)                                 # row maximum = MAX: f = 1
    row = Q.from_f32(vals, dt)
    planes = np.ascontiguousarray(np.broadcast_to(row[:, None, :], (2 * L, T, C)))
    x = _tensor(_unplanes(planes), dt, 1, C)
    view = _source("blob", x, None)
    n = T // 256
    raws = _encode_chunks(view, 0, n, 256, 256, KB, VB, N.CODER_RANS_COMPACT)
    del x
    pats = np.arange(65536, dtype=np.uint16)
    new = []
    for j, r in enumerate(raws):
        lo = container_layout_of(parse_header(r))
        b = bytearray(r)
        a = np.frombuffer(b, np.uint8)
        mx = a[lo.off_maxes: lo.off_maxes + 2 * L * 256 * 2].view(np.uint16).reshape(2 * L, 256)
        assert np.array_equal(mx, np.broadcast_to(Q.from_f32(PLANE_MAX.astype(np.float32), dt)[:, None], mx.shape))
        mx[:] = pats[j * 256: (j + 1) * 256][None, :]
        new.append(bytes(b))
    for out_dt in (0, 1):
        dest = _Dest("vllm", L, 1, C, T, out_dt, 0, None)
        assert _decode(new, N.CODER_RANS_COMPACT, dest, _dtok(n, 256), KB, VB, dt) == [0] * n
        got = _planes(dest.bits())
        del dest
        for p in range(2 * L):
            want = Q.spec_dequant(sym[p][None, :], pats[:, None], int(PLANE_MAX[p]), dt, out_dt)
            ok = Q.eq_nan(got[p], want, out_dt)
            if not ok.all():
                t, c = np.argwhere(~ok)[0]
                raise AssertionError(f"MAX {PLANE_MAX[p]} sym {sym[p, c]} m={t:#06x} out dtype {out_dt}: want "
                                     f"{int(want[t, c]):#06x} got {int(got[p, t, c]):#06x} ({int((~ok).sum())} wrong)")


# ------------------------------------------------------------------------------------------------ 3. quantiser sweep
@pytest.mark.parametrize("dt", [0, 1], ids=["bf16", "fp16"])
def test_quantiser_sweep_every_finite_x(dt):
    """every finite x of the dtype (both signs) against each ladder maximum m >= |x|, on coder 2 / 256 tokens: maxima
    == spec_absmax, symbols (read back through the GPU decoder with every row maximum rewritten to MAX) == spec_quant.
    Ladder entry i sits on layer i mod 15, i.e. is swept at MAX (i mod 15) + 1 on the key plane and 15 - (i mod 15) on
    the value plane."""
    from lmcache_b200.codec import container_layout_of, parse_header
    N = _N()
    H, D = 1, 128
    C = H * D
    lad = Q.ladder(dt)
    rows, rmax = {}, {}
    for l in range(L):
        xs, ms = Q.pairs_of(lad[l::L])
        rows[l], rmax[l] = Q.pack_rows(xs, ms, C, dt, start=l)
    T = max(r.shape[0] for r in rows.values())
    T += (-T) % 256
    bits = np.empty((L, 2, T, C), np.uint16)
    for l in range(L):
        idx = np.arange(T) % rows[l].shape[0]
        bits[l, 0] = bits[l, 1] = rows[l][idx]
    planes = _planes(bits)
    view_x = _tensor(bits, dt, H, D)
    n = T // 256
    raws = _encode_chunks(_source("blob", view_x, None), 0, n, 256, 256, KB, VB, N.CODER_RANS_COMPACT)
    del view_x
    maxes = np.empty((2 * L, T), np.uint16)
    mb = Q.from_f32(PLANE_MAX.astype(np.float32), dt)
    new = []
    for j, r in enumerate(raws):
        lo = container_layout_of(parse_header(r))
        b = bytearray(r)
        mx = np.frombuffer(b, np.uint8)[lo.off_maxes: lo.off_maxes + 2 * L * 256 * 2].view(np.uint16).reshape(2 * L, 256)
        maxes[:, j * 256: (j + 1) * 256] = mx
        mx[:] = mb[:, None]
        new.append(bytes(b))
    assert np.array_equal(maxes, Q.spec_absmax(planes)), "maxima section != spec_absmax"
    dest = _Dest("vllm", L, H, D, T, 0, 0, None)
    assert _decode(new, N.CODER_RANS_COMPACT, dest, _dtok(n, 256), KB, VB, dt) == [0] * n
    got = _planes(dest.bits())
    del dest
    for p in range(2 * L):
        M = int(PLANE_MAX[p])
        want = Q.spec_dequant(Q.spec_quant(planes[p], maxes[p][:, None], M, dt), mb[p], M, dt, 0)
        bad = np.argwhere(got[p] != want)
        if bad.size:
            t, c = bad[0]
            gs = int(Q.to_f32(got[p, t, c], 0)) + M
            raise AssertionError(_where(planes, (p, t, c), maxes, PLANE_MAX, f"quantiser sweep ({bad.shape[0]} wrong)") +
                                 f": want sym {int(Q.to_f32(want[t, c], 0)) + M} got {gs}")
