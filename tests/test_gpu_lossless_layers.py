"""GPU: the per-layer lossless decode (b200kv_lossless_decode_plan / b200kv_lossless_decode_layers) and the stream
offsets of lossless containers (b200kv_lossless_plane_offsets{,_device}).

Every set of layer calls that covers the layers once writes what b200kv_lossless_decode writes, status words included,
for bf16 and fp16, (K, V) and latent KV, blob / huggingface / tuple / paged destinations and 1 to 4096 tokens.  Before
each call every container byte the call may not read is overwritten with a fill pattern, and so is the destination
outside the call's layers: the call's layers are still exact and the rest of the destination is untouched.  The plan
runs while only [0, off_raw) of the containers has been uploaded."""
import ctypes

import numpy as np
import pytest
import torch

import lossless_ref as R

pytestmark = pytest.mark.gpu
SPLITS = {"one": lambda L: [(0, L)], "per_layer": lambda L: [(l, l + 1) for l in range(L)],
          "uneven": lambda L: [(0, L - 2), (L - 2, L - 1), (L - 1, L)], "reverse": lambda L: [(l, l + 1) for l in reversed(range(L))]}


def _np(x):
    return x.contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def _kv(shape, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, device="cuda", generator=g) * torch.exp(2 * torch.randn(shape[-1], device="cuda", generator=g))
    return x.to(dtype)


class Dest:
    """A destination of one kind, with access to the rows of each plane (keys of layer l: plane l, values: L + l)"""

    def __init__(self, kind, L, T, H, D, dtype):
        from lmcache_b200.codec import KvView
        self.kind, self.L = kind, L
        fill = lambda shape: torch.zeros(shape, dtype=torch.int16, device="cuda").view(dtype)   # noqa: E731
        if kind == "vllm":
            self.t = fill((L, 2, T, H, D))
            self.planes = [self.t[l, k] for k in range(2) for l in range(L)]
            self.view = lambda: KvView.from_blob(self.t, "vllm")
        elif kind == "huggingface":
            self.t = fill((L, 2, H, T, D))
            self.planes = [self.t[l, k] for k in range(2) for l in range(L)]
            self.view = lambda: KvView.from_blob(self.t, "huggingface")
        elif kind == "tuple":
            self.t = [(fill((T, H, D)), fill((T, H, D))) for _ in range(L)]
            self.planes = [self.t[l][k] for k in range(2) for l in range(L)]
            self.view = lambda: KvView.from_tuple(self.t, "vllm")
        elif kind == "paged":
            self.slots = torch.randperm(T + 40, generator=torch.Generator().manual_seed(T))[:T].cuda()
            nb = (T + 40 + 15) // 16
            self.t = [(fill((nb, 16, H, D)), fill((nb, 16, H, D))) for _ in range(L)]
            self.planes = [self.t[l][k] for k in range(2) for l in range(L)]
            self.view = lambda: KvView.from_paged(self.t, self.slots)
        else:                                   # latent [L, T, D]
            self.t = fill((L, T, D))
            self.planes = [self.t[l] for l in range(L)]
            self.view = lambda: KvView.from_blob(self.t, "vllm")

    def layer_planes(self, lb, le):
        ppl = len(self.planes) // self.L
        return [k * self.L + l for k in range(ppl) for l in range(lb, le)]

    def snapshot(self):
        """the rows a decode writes, per plane, as [T, C] (a paged cache's mapped slots only)"""
        out = []
        for p in self.planes:
            a = _np(p)
            if self.kind == "huggingface":
                a = a.transpose(1, 0, 2)
            a = a.reshape(-1, a.shape[-2] * a.shape[-1]) if self.kind != "latent" else a
            out.append(a[self.slots.cpu().numpy()] if self.kind == "paged" else a)
        return out


def _case(kind, dtype, t, seed=0):
    """(containers as host bytes, destination token offsets, L, H, D, T, source planes as numpy [P][T][C])"""
    from lmcache_b200.codec import KvView, LosslessCodec
    latent = kind == "latent"
    L, H, D = (4, 1, 576) if latent else (4, 2, 64)
    t2 = max(1, t // 3 + 1)                  # a ragged last chunk
    T = t + t2
    codec = LosslessCodec()
    if latent:
        src = _kv((L, T, D), dtype, seed + t)
        conts = codec.encode_to_host(KvView.from_blob(src, "vllm"), 0, T, t)
        planes = _np(src).reshape(L, T, D)
    else:
        src = _kv((L, 2, T, H, D), dtype, seed + t)
        conts = codec.encode_to_host(KvView.from_blob(src, "vllm"), 0, T, t)
        planes = R.planes_of_blob(_np(src))
    assert [R.parse_header(c)["ntokens"] for c in conts] == [t, t2]
    return conts, [0, t], L, H, D, T, planes, latent


def _upload(host: np.ndarray, dev: torch.Tensor, stream):
    from lmcache_b200 import _native as N
    N.check(N.lib().b200kv_copy_async(ctypes.c_void_p(dev.data_ptr()), ctypes.c_void_p(host.ctypes.data), host.size,
                                      stream.cuda_stream), "copy")


def _pack(conts):
    from lmcache_b200 import _native as N
    offs, o = [], 0
    for c in conts:
        offs.append(o)
        o += (len(c) + 15) & ~15
    buf = np.zeros(o + N.READ_SLACK, np.uint8)
    for c, off in zip(conts, offs):
        buf[off:off + len(c)] = np.frombuffer(c, np.uint8)
    return buf, offs


def _allowed(conts, offs, nbytes, planes, latent):
    """mask of the buffer bytes a call over `planes` may read (None: the plan's [0, off_raw) of every container)"""
    from lmcache_b200.codec import lossless_plane_offsets
    m = np.zeros(nbytes, bool)
    for c, off in zip(conts, offs):
        hd = R.parse_header(c)
        P = hd["L"] if latent else 2 * hd["L"]
        C, t = hd["H"] * hd["D"], hd["ntokens"]
        lo = R.layout(P, C, t)
        po = lossless_plane_offsets(bytearray(c))
        if planes is None:
            m[off:off + lo["off_raw"]] = True
            continue
        m[off:off + lo["off_freq"]] = True
        m[off + lo["off_lens"]:off + lo["off_raw"]] = True
        for p in planes:
            m[off + lo["off_freq"] + 512 * p:off + lo["off_freq"] + 512 * (p + 1)] = True
            m[off + lo["off_raw"] + p * t * C:off + lo["off_raw"] + (p + 1) * t * C] = True
            m[off + po[p]:off + po[p + 1]] = True
    return m


def _whole(conts, offs, dst_tok, dest, dtype_code):
    """b200kv_lossless_decode of the containers into `dest`: (plane snapshots, status words)"""
    from lmcache_b200.codec import LosslessCodec
    codec = LosslessCodec()
    buf, _ = _pack(conts)
    dev = torch.from_numpy(buf).cuda()
    hds = [R.parse_header(c) for c in conts]
    view = dest.view()
    coder = codec.coder_for(max(h["ntokens"] for h in hds), view.latent)
    codec.decode_raw(dev.data_ptr(), dev.numel(), offs, [len(c) for c in conts], [h["ntokens"] for h in hds], view,
                     dst_tok, dtype_code, coder)
    torch.cuda.synchronize()
    return dest.snapshot(), codec.decode_status()


def _split(conts, offs, dst_tok, dest, dtype_code, ranges, poison=True):
    """plan (with only [0, off_raw) uploaded) + one decode_layers call per range, each after poisoning every container
    byte the call may not read and the destination outside its layers; checks that poisoned rows stay untouched.
    Returns (plane snapshots after each call, status words)."""
    from lmcache_b200.codec import LosslessCodec, PinnedBuffer
    codec = LosslessCodec()
    buf, _ = _pack(conts)
    hds = [R.parse_header(c) for c in conts]
    view = dest.view()
    s = torch.cuda.Stream()
    dev = torch.empty(buf.size, dtype=torch.uint8, device="cuda")
    fill = np.full(buf.size, 0xA5, np.uint8)
    plan_mask = _allowed(conts, offs, buf.size, None, view.latent)
    staged = np.where(plan_mask, buf, fill) if poison else buf
    status = PinnedBuffer(64)
    with torch.cuda.stream(s):
        _upload(staged, dev, s)
        coder = codec.coder_for(max(h["ntokens"] for h in hds), view.latent)
        plan, ws = codec.decode_plan(dev.data_ptr(), dev.numel(), offs, [len(c) for c in conts],
                                     [h["ntokens"] for h in hds], view, dst_tok, dtype_code, coder, s, status.dev_ptr)
    shots = []
    for i, (lb, le) in enumerate(ranges):
        mine = dest.layer_planes(lb, le)
        s.synchronize()
        if poison:
            m = _allowed(conts, offs, buf.size, mine, view.latent)
            staged = np.where(m, buf, np.uint8(0x5A + 37 * i))
            for p, t in enumerate(dest.planes):
                if p not in mine:
                    t.view(torch.int16).fill_(-1000 - i)
            torch.cuda.synchronize()
            with torch.cuda.stream(s):
                _upload(staged, dev, s)
        codec.decode_layers(plan, lb, le, s)
        s.synchronize()
        snap = dest.snapshot()
        if poison:
            for p, a in enumerate(snap):
                if p not in mine:
                    assert (a.view(np.int16) == -1000 - i).all(), f"call {i} wrote plane {p} outside layers [{lb}, {le})"
        shots.append((mine, snap))
    words = list((ctypes.c_uint32 * len(conts)).from_address(status.host_ptr))
    del ws
    return shots, words


@pytest.mark.parametrize("t", [1, 7, 256, 4096])
@pytest.mark.parametrize("kind", ["vllm", "huggingface", "tuple", "paged", "latent"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_layer_calls_equal_the_whole_decode(kind, dtype, t):
    conts, dst_tok, L, H, D, T, planes, latent = _case(kind, dtype, t)
    _, offs = _pack(conts)
    code = 0 if dtype == torch.bfloat16 else 1
    want, want_status = _whole(conts, offs, dst_tok, Dest(kind, L, T, H, D, dtype), code)
    assert want_status == [0, 0]
    for p in range(len(want)):                       # the whole decode gives back the source
        assert np.array_equal(want[p], planes[p]), p
    for name, f in SPLITS.items():
        ranges = f(L)
        shots, words = _split(conts, offs, dst_tok, Dest(kind, L, T, H, D, dtype), code, ranges)
        assert words == want_status, name
        for mine, snap in shots:
            for p in mine:
                assert np.array_equal(snap[p], want[p]), f"{name}: plane {p}"


def _damage(conts, what):
    """a copy of container 0 with one section damaged"""
    c = bytearray(conts[0])
    hd = R.parse_header(c)
    P = 2 * hd["L"]
    lo = R.layout(P, hd["H"] * hd["D"], hd["ntokens"])
    if what == "freq":
        c[lo["off_freq"] + 512 * 1 + 2 * 0x7F] ^= 0x01               # plane 1's row no longer sums to 4096
    elif what == "lens":
        c[lo["off_lens"] + 2 * 3] ^= 0x02                             # one length of plane 0
    elif what == "stream":
        c[lo["off_payload"] + 40] ^= 0xFF
    elif what == "header":
        c[16:20] = (hd["D"] + 1).to_bytes(4, "little")               # D: the header is not the one the call names
    return [bytes(c)] + conts[1:]


@pytest.mark.parametrize("what", ["freq", "lens", "stream", "header"])
def test_damage_sets_the_status_bits_of_the_whole_decode(what):
    conts, dst_tok, L, H, D, T, _, _ = _case("vllm", torch.bfloat16, 256, seed=9)
    bad = _damage(conts, what)
    _, offs = _pack(bad)
    want, want_status = _whole(bad, offs, dst_tok, Dest("vllm", L, T, H, D, torch.bfloat16), 0)
    assert want_status[0] != 0 and want_status[1] == 0
    for name in ("one", "per_layer", "reverse"):
        shots, words = _split(bad, offs, dst_tok, Dest("vllm", L, T, H, D, torch.bfloat16), 0, SPLITS[name](L),
                              poison=False)
        assert words == want_status, (what, name)
        for mine, snap in shots:
            for p in mine:
                assert np.array_equal(snap[p], want[p])


@pytest.mark.parametrize("latent", [False, True])
def test_host_and_device_plane_offsets_agree(latent):
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView, LosslessCodec, PinnedBuffer, lossless_plane_offsets
    codec = LosslessCodec()
    L, T, cs = 4, 700, 256
    src = _kv((L, T, 576), torch.float16, 3) if latent else _kv((L, 2, T, 4, 64), torch.float16, 3)
    batch = codec.encode(KvView.from_blob(src, "vllm"), 0, T, cs)
    n = len(batch.sizes)
    rows = PinnedBuffer(8 * (N.MAX_PLANES + 1) * (n + 1))
    # one more row: a CacheGen-looking header (version 3) gets -1
    buf = torch.zeros((n + 1) * batch.stride, dtype=torch.uint8, device="cuda")
    buf[:n * batch.stride] = batch.buf[:n * batch.stride]
    buf[n * batch.stride:n * batch.stride + 64] = batch.buf[:64]
    buf[n * batch.stride + 4] = 3
    N.check(N.lib().b200kv_lossless_plane_offsets_device(buf.data_ptr(), batch.stride, n + 1, rows.dev_ptr,
                                                         torch.cuda.current_stream().cuda_stream), "offsets")
    torch.cuda.synchronize()
    got = np.frombuffer(rows.view(), np.int64, count=(n + 1) * (N.MAX_PLANES + 1)).reshape(n + 1, -1)
    P = L if latent else 2 * L
    for j in range(n):
        host = lossless_plane_offsets(bytearray(batch.container(j).cpu().numpy().tobytes()))
        assert np.array_equal(got[j, :P + 1], host) and (got[j, P + 1:] == 0).all()
        assert host[-1] == batch.sizes[j]
    assert got[n, 0] == -1
