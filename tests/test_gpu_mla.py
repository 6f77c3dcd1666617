"""GPU: latent KV caches (multi-head latent attention, DeepSeek-V2/V3) -- one plane per layer through the codec and the
mover, into and out of container version 4.

* encode (b200kv_encode_chunks) byte-equal to the oracle's version-4 container, decode bit-equal to the oracle's values,
  for L in {1, 27, 61, 128}, D in {20, 576}, bf16 / fp16, blob / tuple / paged sources, ragged last chunk; the rows
  of a paged destination that no token maps to are untouched.
* the version-4 streams, maxima and half-lengths are the K-plane parts of version 3's encode of (latent, latent).
* layer-wise encode splits byte-identical to encode_chunks; split decodes bit-identical to a whole decode.
* pack / unpack round trips, plane offsets on the device, and every refusal of the ABI (nothing written)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle as O

import mla_ref

pytestmark = pytest.mark.gpu

MODEL = "deepseek-ai/DeepSeek-V3"


def _N():
    from lmcache_b200 import _native as N
    return N


def _s():
    return torch.cuda.current_stream().cuda_stream


def _cfg(L):
    return dict(key_first_layers=min(3, L), key_second_layers=min(20, L), key_third_layers=L, key_first_bins=32,
                key_second_bins=16, key_third_bins=8, value_first_layers=2, value_first_bins=32, value_second_bins=16)


def _codec(L):
    from lmcache_b200.codec import CacheGenCodec
    return CacheGenCodec(MODEL, cachegen_config=_cfg(L))


def _latent(L, T, D, dt, seed):
    """uint16 bits [L, T, D] of the given dtype and the CUDA tensor holding them"""
    bits = O.synth_kv_bits(L, T, D, seed=seed)[:, 0]
    if dt == torch.float16:
        bits = O.bf16_bits_to_f32(bits).astype(np.float16).view(np.uint16)
    bits = np.ascontiguousarray(bits)
    return bits, torch.from_numpy(bits.view(np.int16)).view(dt).cuda()


SENT = -12345


class _Src:
    """the latent KV as one of the view kinds, over storage that has rows / channels no token maps to"""

    def __init__(self, kind, L, T, D, dt, seed=0, x=None):
        from lmcache_b200.codec import KvView
        g = torch.Generator().manual_seed(seed)
        self.kind, self.T, self.D = kind, T, D
        fill = torch.tensor(SENT, dtype=torch.int16).view(dt).item()
        if kind == "blob":           # strided: every token row is D + 8 wide
            self.store = torch.full((L, T, D + 8), fill, dtype=dt, device="cuda")
            self.x = self.store[..., :D]
            self.view = lambda: KvView.from_blob(self.x, "vllm")
        elif kind == "tuple":
            self.store = torch.full((L, T + 5, D), fill, dtype=dt, device="cuda")
            self.x = self.store[:, 3:T + 3]
            self.view = lambda: KvView.from_tuple([self.x[l] for l in range(L)], "vllm")
        else:                        # vLLM's paged MLA cache [num_blocks, 64, D], shuffled slots
            nblk = (T + 63) // 64 + 2
            self.store = torch.full((L, nblk, 64, D), fill, dtype=dt, device="cuda")
            self.slots = torch.randperm(nblk * 64, generator=g)[:T].cuda()
            self.view = lambda: KvView.from_paged([self.store[l] for l in range(L)], self.slots)
        if x is not None:
            self.write(x)

    def write(self, x):
        if self.kind == "paged":
            flat = self.store.view(self.store.shape[0], -1, self.D)
            flat[:, self.slots] = x
        else:
            self.x.copy_(x)

    def read(self):
        if self.kind == "paged":
            return self.store.view(self.store.shape[0], -1, self.D)[:, self.slots]
        return self.x

    def untouched_outside(self):
        """every element no token maps to still holds the sentinel"""
        s = self.store.view(torch.int16)
        if self.kind == "blob":
            return bool((s[..., self.D:] == SENT).all())
        if self.kind == "tuple":
            return bool((s[:, :3] == SENT).all() and (s[:, self.T + 3:] == SENT).all())
        flat = s.view(s.shape[0], -1, self.D)
        mask = torch.ones(flat.shape[1], dtype=torch.bool, device="cuda")
        mask[self.slots] = False
        return bool((flat[:, mask] == SENT).all())


def _bits(t):
    return t.contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


SHAPES = [(1, 576, 256, 5), (27, 20, 64, 37), (61, 576, 256, 19), (128, 20, 256, 3)]


@pytest.mark.parametrize("kind", ["blob", "tuple", "paged"])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("L,D,cs,rag", SHAPES, ids=[f"L{s[0]}-D{s[1]}" for s in SHAPES])
def test_encode_decode_vs_oracle(L, D, cs, rag, dt, kind):
    N = _N()
    T = cs + rag
    bits, x = _latent(L, T, D, dt, seed=L + D)
    dtc = N.DT_BF16 if dt == torch.bfloat16 else N.DT_FP16
    codec = _codec(L)
    kb = np.array(codec.config.key_bins_list(), np.float32)
    src = _Src(kind, L, T, D, dt, seed=1, x=x)
    batch = codec.encode(src.view(), 0, T, cs)
    assert batch.coder == N.CODER_LATENT and len(batch.sizes) == 2
    starts, ntoks, want_vals = [0, cs], [cs, rag], []
    for j, (a, t) in enumerate(zip(starts, ntoks)):
        want, _, enc = mla_ref.v4_container(bits[:, a:a + t], dtc, kb, 1, D)
        got = batch.container(j).cpu().numpy().tobytes()
        assert got == want, f"chunk {j}: version-4 container differs from the oracle's"
        want_vals.append(mla_ref.decode_latent(enc, dtc, kb, dtc))
    dst = _Src(kind, L, T, D, dt, seed=2)
    codec.decode_device_batch(batch, ntoks, dst.view(), starts)
    torch.cuda.synchronize()
    assert np.array_equal(_bits(dst.read()), np.concatenate(want_vals, axis=1))
    assert dst.untouched_outside()
    assert codec.decode_status() == [0, 0]
    # the host path (parse_header + upload) decodes the same
    dst2 = _Src(kind, L, T, D, dt, seed=2)
    codec.decode([batch.container(j).cpu().numpy().tobytes() for j in range(2)], dst2.view(), starts)
    torch.cuda.synchronize()
    assert torch.equal(dst2.read().view(torch.int16), dst.read().view(torch.int16))


@pytest.mark.parametrize("L,D,t", [(27, 576, 256), (61, 20, 77)])
def test_v4_is_the_key_half_of_v3_of_the_pair(L, D, t):
    from lmcache_b200.codec import KvView, parse_header, plane_offsets
    N = _N()
    _, x = _latent(L, t, D, torch.bfloat16, seed=5)
    codec = _codec(L)
    raw4 = codec.encode_to_host(KvView.from_blob(x, "vllm"), 0, t, t)[0]
    xh = x.unsqueeze(2)                                       # [L, t, 1, D]: one head of D channels
    raw3 = codec.encode_to_host(KvView.from_tuple([(xh[l], xh[l]) for l in range(L)], "vllm"), 0, t, t)[0]
    h4, h3 = parse_header(raw4), parse_header(raw3)
    assert (h4.version, h3.version) == (4, 3) and h4.nb == h3.nb[:L]
    lo4 = N.container_layout(L, 1, D, t, N.CODER_LATENT)
    lo3 = N.container_layout(L, 1, D, t, N.CODER_RANS_COMPACT)
    assert raw4[lo4.off_maxes:lo4.off_maxes + L * t * 2] == raw3[lo3.off_maxes:lo3.off_maxes + L * t * 2]
    assert raw4[lo4.off_lengths:lo4.off_lengths + L * D] == raw3[lo3.off_lengths:lo3.off_lengths + L * D]
    p3 = plane_offsets(raw3)
    assert raw4[lo4.off_payload:] == raw3[lo3.off_payload:p3[L]]
    assert len(raw4) - lo4.off_payload == p3[L] - lo3.off_payload
    assert len(raw4) < 0.55 * len(raw3)


@pytest.mark.parametrize("L,D,calls", [(61, 576, [(0, 1), (1, 30), (30, 60), (60, 61)]),
                                       (27, 20, [(5, 27), (0, 5)])])
def test_layer_split_encode_and_decode(L, D, calls):
    from lmcache_b200.codec import KvView
    N = _N()
    lib = N.lib()
    cs, T = 64, 64 * 3 + 11
    n, last = 4, 11
    _, x = _latent(L, T, D, torch.bfloat16, seed=9)
    codec = _codec(L)
    view = KvView.from_blob(x, "vllm")
    whole = codec.encode(view, 0, T, cs)
    want = [whole.container(j).cpu().numpy().tobytes() for j in range(n)]
    lo = N.container_layout(L, 1, D, cs, N.CODER_LATENT)
    stride = (lo.off_payload + 15) & ~15
    arena_bytes = n * (lo.max_total_bytes - lo.off_payload + 16 * L)
    arena = torch.zeros(arena_bytes, dtype=torch.uint8, device="cuda")
    fixed = torch.zeros(n * stride, dtype=torch.uint8, device="cuda")
    seg = torch.full((n * L * 2,), -7, dtype=torch.int64, device="cuda")
    sizes = torch.zeros(n, dtype=torch.int64, device="cuda")
    ml = max(b - a for a, b in calls)
    wsb = N.check(lib.b200kv_encode_layers_workspace_bytes(L, 1, D, cs, n, ml), "ws")
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    plan = N.EncodePlan()
    N.check(lib.b200kv_encode_layers_plan(ctypes.byref(view.desc), 0, n, cs, last, codec._kb, codec._vb,
                                          N.CODER_RANS_COMPACT, arena.data_ptr(), arena_bytes, fixed.data_ptr(), stride,
                                          seg.data_ptr(), sizes.data_ptr(), ml, ws.data_ptr(), wsb, ctypes.byref(plan),
                                          _s()), "encode_layers_plan")
    for a, b in calls:
        N.check(lib.b200kv_encode_layers(ctypes.byref(plan), a, b, _s()), "encode_layers")
    N.check(lib.b200kv_encode_layers_finish(ctypes.byref(plan), _s()), "encode_layers_finish")
    torch.cuda.synchronize()
    ar, fx, sg = arena.cpu().numpy(), fixed.cpu().numpy(), seg.cpu().numpy().reshape(n, L, 2)
    for j in range(n):
        offp = N.container_layout(L, 1, D, cs if j < n - 1 else last, N.CODER_LATENT).off_payload
        got = fx[j * stride: j * stride + offp].tobytes() + b"".join(ar[o:o + m].tobytes() for o, m in sg[j])
        assert int(sizes[j]) == len(got) and got == want[j], f"chunk {j}"
    # decode: one plan, layers in pieces == the whole decode
    ref = torch.empty_like(x)
    codec.decode_device_batch(whole, [cs] * 3 + [last], KvView.from_blob(ref, "vllm"), [0, cs, 2 * cs, 3 * cs])
    out = torch.full_like(x, 7.0)
    dv = KvView.from_blob(out, "vllm")
    s = torch.cuda.current_stream()
    plan_d, ws_d = codec.decode_plan(whole.buf.data_ptr(), whole.buf.numel(), [j * whole.stride for j in range(n)],
                                     whole.sizes, [cs] * 3 + [last], dv, [0, cs, 2 * cs, 3 * cs], whole.max_dtype,
                                     whole.coder, s)
    for a, b in sorted(calls, key=lambda c: -c[0]):
        codec.decode_layers(plan_d, a, b, s)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16))


@pytest.mark.parametrize("kind", ["blob", "tuple", "paged"])
def test_pack_unpack_round_trip(kind):
    N = _N()
    L, D, T, cs = 61, 576, 300, 128
    _, x = _latent(L, T, D, torch.bfloat16, seed=3)
    src = _Src(kind, L, T, D, torch.bfloat16, seed=4, x=x)
    buf, blobs = src.view().pack_chunks(0, cs)
    assert [tuple(b.shape) for b in blobs] == [(L, 128, D), (L, 128, D), (L, 44, D)]
    for j, b in enumerate(blobs):
        assert torch.equal(b.view(torch.int16), x[:, j * cs: j * cs + b.shape[1]].contiguous().view(torch.int16))
    dst = _Src(kind, L, T, D, torch.bfloat16, seed=4)
    N.check(N.lib().b200kv_unpack_chunks(buf.data_ptr(), L * cs * D * 2, 3, cs, 44, 0, ctypes.byref(dst.view().desc), 0,
                                         _s()), "unpack_chunks")
    torch.cuda.synchronize()
    assert torch.equal(dst.read().view(torch.int16), x.view(torch.int16)) and dst.untouched_outside()


def test_device_plane_offsets_on_v4():
    from lmcache_b200.codec import KvView, PinnedBuffer, plane_offsets
    N = _N()
    L, D, T, cs = 61, 576, 512, 256
    _, x = _latent(L, T, D, torch.bfloat16, seed=6)
    codec = _codec(L)
    b = codec.encode(KvView.from_blob(x, "vllm"), 0, T, cs)
    pin = PinnedBuffer(2 * 8 * (N.MAX_PLANES + 1))
    N.check(N.lib().b200kv_plane_offsets_device(b.buf.data_ptr(), b.stride, 2, pin.dev_ptr, _s()), "plane_offsets_device")
    torch.cuda.synchronize()
    po = np.frombuffer(pin.view(), np.int64).reshape(2, N.MAX_PLANES + 1)
    for j in range(2):
        want = plane_offsets(b.container(j).cpu().numpy().tobytes())
        assert np.array_equal(po[j, :L + 1], want) and (po[j, L + 1:] == 0).all()
    pin.close()


def test_refusals_write_nothing():
    from lmcache_b200.codec import KvView
    N = _N()
    lib = N.lib()
    L, D, t = 4, 576, 32
    _, x = _latent(L, t, D, torch.bfloat16, seed=8)
    codec = _codec(L)
    lat = KvView.from_blob(x, "vllm")
    pair_kv = torch.stack([x, x], 1).unsqueeze(3).contiguous()          # [L, 2, t, 1, D]
    pair = KvView.from_blob(pair_kv, "vllm")
    out = torch.full((1 << 20,), 0x5A, dtype=torch.uint8, device="cuda")
    sizes = torch.zeros(1, dtype=torch.int64, device="cuda")
    ws = torch.empty(1 << 24, dtype=torch.uint8, device="cuda")
    for coder in (N.CODER_AC, N.CODER_RANS):                               # a latent KV has version 4 only
        assert lib.b200kv_encode_chunks(ctypes.byref(lat.desc), 0, 1, t, t, codec._kb, codec._vb, coder, out.data_ptr(),
                                        1 << 19, sizes.data_ptr(), ws.data_ptr(), ws.numel(), _s()) < 0
    torch.cuda.synchronize()
    assert bool((out == 0x5A).all())
    v4 = codec.encode(lat, 0, t, t)
    v3 = codec.encode(pair, 0, t, t)
    raw4, raw3 = v4.container(0).cpu().numpy().tobytes(), v3.container(0).cpu().numpy().tobytes()
    dl = torch.full_like(x, 3.0)
    dp = torch.full_like(pair_kv, 3.0)
    lat_d, pair_d = KvView.from_blob(dl, "vllm"), KvView.from_blob(dp, "vllm")

    def dec(batch, dst, coder):
        return lib.b200kv_decode_chunks(batch.buf.data_ptr(), batch.buf.numel(), N.i64_array([0]),
                                        N.i64_array(batch.sizes), N.i32_array([t]), N.i64_array([0]), 1, N.DT_BF16, coder,
                                        ctypes.byref(dst.desc), codec._kb, codec._vb, None, ws.data_ptr(), ws.numel(),
                                        _s())
    assert dec(v3, lat_d, N.CODER_RANS_COMPACT) < 0                        # version 3 into a latent destination
    assert dec(v4, pair_d, N.CODER_LATENT) < 0                             # version 4 into a (K, V) destination
    assert dec(v4, lat_d, N.CODER_RANS_COMPACT) < 0                        # coder and destination disagree
    assert dec(v4, lat_d, N.CODER_RANS | N.KV_LATENT) < 0
    plan = N.DecodePlan()
    one = N.i32_array([1])
    zero = N.i32_array([0])
    assert lib.b200kv_decode_plan_heads(v4.buf.data_ptr(), v4.buf.numel(), N.i64_array([0]), N.i64_array(v4.sizes),
                                        N.i32_array([t]), N.i64_array([0]), 1, N.DT_BF16, N.CODER_LATENT,
                                        ctypes.byref(lat_d.desc), codec._kb, codec._vb, None, ws.data_ptr(), ws.numel(),
                                        ctypes.byref(plan), _s(), 1, zero, zero, one) < 0
    with pytest.raises(ValueError):
        codec.decode([raw3], lat_d, [0])
    with pytest.raises(ValueError):
        codec.decode([raw4], pair_d, [0])
    torch.cuda.synchronize()
    assert bool((dl == 3.0).all()) and bool((dp == 3.0).all())
    # the accepted pairing decodes
    assert dec(v4, lat_d, N.CODER_LATENT) == 0
    torch.cuda.synchronize()
    assert not bool((dl == 3.0).all())


def test_version_mismatch_is_flagged_on_the_device():
    """b200kv_decode_chunks cannot read headers before it returns, so it trusts the coder; the decode flags a container
    whose header names another version (status bit 2) and the caller drops it as a miss"""
    from lmcache_b200.codec import KvView, PinnedBuffer
    N = _N()
    lib = N.lib()
    L, D, t = 4, 576, 32
    _, x = _latent(L, t, D, torch.bfloat16, seed=12)
    codec = _codec(L)
    v4 = codec.encode(KvView.from_blob(x, "vllm"), 0, t, t)
    pair_kv = torch.stack([x, x], 1).unsqueeze(3).contiguous()
    v3 = codec.encode(KvView.from_blob(pair_kv, "vllm"), 0, t, t)
    assert max(v4.sizes) <= codec.max_container_bytes(L, 1, D, t, latent=True) < codec.max_container_bytes(L, 1, D, t)
    ws = torch.empty(1 << 24, dtype=torch.uint8, device="cuda")
    st = PinnedBuffer(4096)

    def status(batch, dst, coder):
        N.check(lib.b200kv_decode_chunks(batch.buf.data_ptr(), batch.buf.numel(), N.i64_array([0]),
                                         N.i64_array(batch.sizes), N.i32_array([t]), N.i64_array([0]), 1, N.DT_BF16,
                                         coder, ctypes.byref(dst.desc), codec._kb, codec._vb, st.dev_ptr, ws.data_ptr(),
                                         ws.numel(), _s()), "decode_chunks")
        torch.cuda.synchronize()
        return int(np.frombuffer(st.view(0, 4), np.uint32)[0])
    lat_d = KvView.from_blob(torch.empty_like(x), "vllm")
    pair_d = KvView.from_blob(torch.empty_like(pair_kv), "vllm")
    assert status(v4, lat_d, N.CODER_LATENT) == 0
    assert status(v3, pair_d, N.CODER_RANS_COMPACT) == 0
    assert status(v3, lat_d, N.CODER_LATENT) & 4                 # version 3 handed over as version 4
    assert status(v4, pair_d, N.CODER_RANS_COMPACT) & 4          # version 4 handed over as version 3
    st.close()
