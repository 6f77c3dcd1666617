"""GPU: decoding another tensor-parallel layout's lossless containers (versions 5) into this rank's KV heads.

Kernel: b200kv_lossless_decode_plan_heads (through LosslessCodec.decode_raw_heads / decode_plan_heads) over seeded
random shapes, dtypes, destinations and layer splits: the windowed decode is the input KV's head slice bit for bit, the
slice of a whole b200kv_lossless_decode and the slice of tests/lossless_ref.decode; bytes outside the windows keep a
sentinel; refused arguments write nothing; a damaged stream sets a status bit inside the window and none outside it.
Engine: lossless stores of one layout retrieved by engines of another through an in-process lm:// server."""
import ctypes
import random

import numpy as np
import pytest
import torch

import lossless_ref as R

pytestmark = pytest.mark.gpu
MODEL = "mistralai/Mistral-7B-Instruct-v0.2"
SENT = -21555                      # sentinel int16 pattern of destination bytes nobody may write


def _i16(t):
    return t.contiguous().view(torch.int16)


def _codec():
    from lmcache_b200.codec import LosslessCodec
    return LosslessCodec()


def _encode(codec, kv, chunk):
    """containers of blob kv [L,2,T,H,D] (vllm) in chunks: (device buffer, offsets, totals, ntokens, max_dtype, coder)"""
    from lmcache_b200.codec import KvView
    T = kv.shape[2]
    b = codec.encode(KvView.from_blob(kv, "vllm"), 0, T, chunk)
    buf = b.buf.clone()
    offs = [j * b.stride for j in range(len(b.sizes))]
    ntok = [min(chunk, T - j * chunk) for j in range(len(b.sizes))]
    return buf, offs, list(b.sizes), ntok, b.max_dtype, b.coder


def _full_decode(codec, enc, kv_shape, dtype):
    from lmcache_b200.codec import KvView
    buf, offs, tot, ntok, md, cd = enc
    out = torch.empty(kv_shape, dtype=dtype, device="cuda")
    codec.decode_raw(buf.data_ptr(), buf.numel(), offs, tot, ntok, KvView.from_blob(out, "vllm"),
                     [sum(ntok[:j]) for j in range(len(offs))], md, cd)
    assert codec.decode_status() == [0] * len(offs)
    return out


def _kv(shape, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, device="cuda", generator=g) * torch.exp(2 * torch.randn(shape[-1], device="cuda", generator=g))
    return x.to(dtype)


class _Dst:
    """A destination of H heads and T tokens in one of three layouts, filled with the sentinel; dense() reads it back as
    [L,2,T,H,D], untouched() says whether every paged slot outside the token rows is still the sentinel."""

    def __init__(self, kind, L, T, H, D, dtype, rng):
        from lmcache_b200.codec import KvView
        self.kind, self.T = kind, T
        if kind == "paged":
            self.nslots = T + 37
            perm = list(range(self.nslots))
            rng.shuffle(perm)
            self.slots = torch.tensor(perm[:T], dtype=torch.int64, device="cuda")
            self.caches = [tuple(torch.full((self.nslots, H, D), SENT, dtype=torch.int16, device="cuda").view(dtype)
                                 for _ in range(2)) for _ in range(L)]
            self.view = KvView.from_paged(self.caches, self.slots)
        else:
            shape = (L, 2, T, H, D) if kind == "vllm" else (L, 2, H, T, D)
            self.blob = torch.full(shape, SENT, dtype=torch.int16, device="cuda").view(dtype)
            self.view = KvView.from_blob(self.blob, kind)

    def dense(self):
        if self.kind == "vllm":
            return self.blob
        if self.kind == "huggingface":
            return self.blob.permute(0, 1, 3, 2, 4)
        return torch.stack([torch.stack([k[self.slots], v[self.slots]]) for k, v in self.caches])

    def untouched(self):
        if self.kind != "paged":
            return True
        rest = torch.ones(self.nslots, dtype=torch.bool, device="cuda")
        rest[self.slots] = False
        return all(bool((c.view(torch.int16)[rest] == SENT).all()) for kv in self.caches for c in kv)


def _layer_splits(L, rng):
    cuts = sorted(rng.sample(range(1, L), rng.randint(0, L - 1))) if L > 1 else []
    return list(zip([0] + cuts, cuts + [L]))


def _decode_windows(codec, enc, dst, toks, Hs, src0, dst0, nh, L, rng, use_plan):
    """decode_raw_heads, or decode_plan_heads + decode_layers over a random split of the layers; the status words"""
    buf, offs, tot, ntok, md, cd = enc
    n = len(offs)
    if not use_plan:
        codec.decode_raw_heads(buf.data_ptr(), buf.numel(), offs, tot, ntok, dst.view, toks, md, cd, Hs, src0, dst0, nh)
        return codec.decode_status()
    stream = torch.cuda.current_stream()
    st = torch.full((n,), 99, dtype=torch.int32, device="cuda")
    plan, ws = codec.decode_plan_heads(buf.data_ptr(), buf.numel(), offs, tot, ntok, dst.view, toks, md, cd, Hs, src0,
                                       dst0, nh, stream, st.data_ptr())
    for a, b in _layer_splits(L, rng):
        codec.decode_layers(plan, a, b, stream)
    torch.cuda.synchronize()
    del ws
    return st.tolist()


# ---------------------------------------------------------------------------------------------- kernel
CHUNKS = [1, 7, 64, 256, 1000, 4096]


@pytest.mark.parametrize("case", range(36))
def test_windowed_decode_is_the_head_slice_of_the_input(case):
    rng = random.Random(2000 + case)
    Hs = [1, 2, 4, 8, 32][case % 5]
    D = [64, 128][(case // 5) % 2]                                    # D = 64: windows start and end mid-tile
    dtype = [torch.bfloat16, torch.float16][(case // 2) % 2]
    kind = ["vllm", "huggingface", "paged"][(case // 6) % 3]
    chunk = CHUNKS[case % len(CHUNKS)]
    big = chunk * Hs * D >= (1 << 20)
    L = 1 if big else rng.choice([1, 2, 3])
    nch = rng.randint(1, 2 if big else 3)
    T = chunk * (nch - 1) + rng.randint(1, chunk)                    # a ragged last chunk
    codec = _codec()
    kv = _kv((L, 2, T, Hs, D), dtype, case)
    enc = _encode(codec, kv, chunk)
    n = len(enc[1])
    ntok = enc[3]
    full = _full_decode(codec, enc, kv.shape, dtype)
    assert torch.equal(_i16(full), _i16(kv))
    # per chunk a random window, landing at a random head of a destination with more heads
    src0 = [rng.randrange(Hs) for _ in range(n)]
    nh = [rng.randint(1, Hs - s) for s in src0]
    Hd = max(nh) + rng.randint(0, 3)
    dst0 = [rng.randint(0, Hd - k) for k in nh]
    dst = _Dst(kind, L, T, Hd, D, dtype, rng)
    want = torch.full((L, 2, T, Hd, D), SENT, dtype=torch.int16, device="cuda")
    toks = [j * chunk for j in range(n)]
    for j in range(n):
        a = toks[j]
        want[:, :, a:a + ntok[j], dst0[j]:dst0[j] + nh[j]] = _i16(kv[:, :, a:a + ntok[j], src0[j]:src0[j] + nh[j]])
        ws = _i16(full[:, :, a:a + ntok[j], src0[j]:src0[j] + nh[j]])
        assert torch.equal(want[:, :, a:a + ntok[j], dst0[j]:dst0[j] + nh[j]], ws)
    status = _decode_windows(codec, enc, dst, toks, Hs, src0, dst0, nh, L, rng, use_plan=case % 2 == 0)
    assert status == [0] * n
    torch.cuda.synchronize()
    assert torch.equal(_i16(dst.dense()), want)
    assert dst.untouched()
    # the numpy statement of the format, sliced, says the same (the first container; small ones only, it is slow)
    if ntok[0] * Hs * D <= (1 << 16):
        buf, offs, tot = enc[0], enc[1], enc[2]
        hd, planes = R.decode(buf[offs[0]:offs[0] + tot[0]].cpu().numpy().tobytes())
        assert (hd["H"], hd["D"], hd["ntokens"]) == (Hs, D, ntok[0])
        ref = planes.reshape(2, L, ntok[0], Hs, D).transpose(1, 0, 2, 3, 4)[:, :, :, src0[0]:src0[0] + nh[0]]
        got = _i16(dst.dense()[:, :, :ntok[0], dst0[0]:dst0[0] + nh[0]]).cpu().numpy().view(np.uint16)
        assert np.array_equal(got, ref)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("W_over", [2, 4])
def test_several_shards_into_one_rank_in_one_call(W_over, dtype):
    """W / W' containers at one dst_tok, each whole into its own head range, equal the KV they were encoded from."""
    L, hs, D, T, chunk = 3, 2, 128, 700, 256
    codec = _codec()
    kv = _kv((L, 2, T, hs * W_over, D), dtype, W_over)
    encs = [_encode(codec, kv[:, :, :, r * hs:(r + 1) * hs].contiguous(), chunk) for r in range(W_over)]
    pieces, offs, tot, ntok, toks, src0, dst0, nh = [], [], [], [], [], [], [], []
    o = 0
    for r, (buf, eo, et, en, md, cd) in enumerate(encs):
        for j in range(len(eo)):
            c = buf[eo[j]:eo[j] + et[j]]
            pieces.append(torch.nn.functional.pad(c, (0, (-c.numel()) % 16)))
            offs.append(o)
            o += pieces[-1].numel()
            tot.append(et[j])
            ntok.append(en[j])
            toks.append(j * chunk)
            src0.append(0)
            dst0.append(r * hs)
            nh.append(hs)
    allbuf = torch.cat(pieces + [torch.zeros(640, dtype=torch.uint8, device="cuda")])
    for use_plan in (False, True):
        dst = _Dst("vllm", L, T, hs * W_over, D, dtype, random.Random(0))
        enc = (allbuf, offs, tot, ntok, md, cd)
        status = _decode_windows(codec, enc, dst, toks, hs, src0, dst0, nh, L, random.Random(W_over), use_plan)
        assert status == [0] * len(offs)
        torch.cuda.synchronize()
        assert torch.equal(_i16(dst.blob), _i16(kv))


def test_refused_windows_write_nothing():
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView
    L, Hs, D, T = 2, 4, 64, 100
    codec = _codec()
    kv = _kv((L, 2, T, Hs, D), torch.bfloat16, 1)
    buf, offs, tot, ntok, md, cd = _encode(codec, kv, 64)
    n = len(offs)
    dst = _Dst("vllm", L, T, 2, D, torch.bfloat16, random.Random(0))
    st = torch.full((n,), 77, dtype=torch.int32, device="cuda")
    ok = dict(src_H=Hs, src_head0=[0] * n, dst_head0=[0] * n, n_heads=[2] * n, toks=[0, 64])
    bad = [dict(n_heads=[0, 2]), dict(src_head0=[3, 0]), dict(src_head0=[-1, 0]), dict(dst_head0=[1, 0]),
           dict(dst_head0=[-1, 0]), dict(src_H=0), dict(n_heads=[5, 2], src_head0=[0, 0]),
           dict(toks=[0, 0], n_heads=[1, 2], dst_head0=[1, 0]), dict(toks=[0, 0], dst_head0=[0, 1], n_heads=[2, 1])]

    def plan(a, view=dst.view, md=md):
        return codec.decode_plan_heads(buf.data_ptr(), buf.numel(), offs, tot, ntok, view, a["toks"], md, cd,
                                       a["src_H"], a["src_head0"], a["dst_head0"], a["n_heads"],
                                       torch.cuda.current_stream(), st.data_ptr())
    for b in bad:
        with pytest.raises(N.NativeError, match="lossless_decode_plan_heads"):
            plan(dict(ok, **b))
    # the dtype rule stays: no casting (bf16 containers, an fp16 destination)
    f16 = torch.full((L, 2, T, 2, D), SENT, dtype=torch.int16, device="cuda").view(torch.float16)
    with pytest.raises(N.NativeError, match="lossless_decode_plan_heads"):
        plan(ok, KvView.from_blob(f16, "vllm"))
    # a latent destination has no heads: refused by the library (the codec's own coder check is bypassed on purpose)
    lat = torch.full((L, T, D), SENT, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    lview = KvView.from_blob(lat, "vllm")
    assert lview.latent
    p = N.LosslessDecodePlan()
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    rc = N.lib().b200kv_lossless_decode_plan_heads(
        buf.data_ptr(), buf.numel(), N.i64_array(offs), N.i64_array(tot), N.i32_array(ntok), N.i64_array([0, 64]), n,
        md, ctypes.byref(lview.desc), st.data_ptr(), ws.data_ptr(), ws.numel(), ctypes.byref(p),
        torch.cuda.current_stream().cuda_stream, Hs, N.i32_array([0] * n), N.i32_array([0] * n), N.i32_array([1] * n))
    assert rc < 0 and "latent" in N.last_error()
    # NULL window arrays
    rc = N.lib().b200kv_lossless_decode_plan_heads(
        buf.data_ptr(), buf.numel(), N.i64_array(offs), N.i64_array(tot), N.i32_array(ntok), N.i64_array([0, 64]), n,
        md, ctypes.byref(dst.view.desc), st.data_ptr(), ws.data_ptr(), ws.numel(), ctypes.byref(p),
        torch.cuda.current_stream().cuda_stream, Hs, None, None, None)
    assert rc < 0 and "NULL" in N.last_error()
    assert N.lib().b200kv_lossless_decode_layers(ctypes.byref(p), 0, L, torch.cuda.current_stream().cuda_stream) < 0
    torch.cuda.synchronize()
    assert bool((dst.blob.view(torch.int16) == SENT).all()) and st.tolist() == [77] * n
    assert bool((f16.view(torch.int16) == SENT).all()) and bool((lat.view(torch.int16) == SENT).all())
    # disjoint ranges at one token are fine
    codec.decode_raw_heads(buf.data_ptr(), buf.numel(), offs[:1] * 2, tot[:1] * 2, ntok[:1] * 2, dst.view, [0, 0], md,
                           cd, Hs, [3, 0], [0, 1], [1, 1])
    assert codec.decode_status() == [0, 0]
    torch.cuda.synchronize()
    assert torch.equal(_i16(dst.blob[:, :, :64]), _i16(kv[:, :, :64, [3, 0]]))
    assert bool((dst.blob[:, :, 64:].view(torch.int16) == SENT).all())


def _stream_of(c: bytearray, p: int, ch: int):
    """(byte offset inside the container, length) of the stream of plane p, channel ch"""
    from lmcache_b200.codec import lossless_plane_offsets
    hd = R.parse_header(c)
    C = hd["H"] * hd["D"]
    lo = R.layout(2 * hd["L"], C, hd["ntokens"])
    lens = np.frombuffer(bytes(c[lo["off_lens"] + 2 * p * C:lo["off_lens"] + 2 * (p + 1) * C]), "<u2").astype(np.int64)
    po = lossless_plane_offsets(c)
    return int(po[p] + lens[:ch].sum()), int(lens[ch])


@pytest.mark.parametrize("where", ["inside", "outside"])
def test_damage_inside_the_window_sets_bit_0_and_outside_it_nothing(where):
    from lmcache_b200.codec import KvView
    L, Hs, D, t = 2, 4, 128, 300
    codec = _codec()
    kv = _kv((L, 2, t, Hs, D), torch.bfloat16, 4)
    c = bytearray(codec.encode_to_host(KvView.from_blob(kv, "vllm"), 0, t, t)[0])
    # the window is head 0 (channels [0, 128): tile 0); plane 1's channel 40 is inside, channel 300 (tile 2) outside
    off, ln = _stream_of(c, 1, 40 if where == "inside" else 300)
    assert ln >= 4
    for i in range(4):
        c[off + i] ^= 0x5A                                           # the stream's initial coder state
    dev = torch.zeros(((len(c) + 15) & ~15) + 1024, dtype=torch.uint8, device="cuda")
    dev[:len(c)] = torch.frombuffer(c, dtype=torch.uint8).cuda()
    enc = (dev, [0], [len(c)], [t], 0, codec.coder_for(t))
    for use_plan in (False, True):
        dst = _Dst("vllm", L, t, 1, D, torch.bfloat16, random.Random(0))
        status = _decode_windows(codec, enc, dst, [0], Hs, [0], [0], [1], L, random.Random(1), use_plan)
        torch.cuda.synchronize()
        if where == "inside":
            assert status[0] & 1
            keep = torch.ones(D, dtype=torch.bool, device="cuda")
            keep[40] = False                                         # every other stream of the window is exact
            assert torch.equal(_i16(dst.blob[:, :, :, 0, keep]), _i16(kv[:, :, :, 0, keep]))
        else:
            assert status == [0]
            assert torch.equal(_i16(dst.blob), _i16(kv[:, :, :, 0:1]))


# ---------------------------------------------------------------------------------------------- engine
@pytest.fixture
def server():
    from lmcache_b200 import _native as N
    h = ctypes.c_void_p()
    N.check(N.lib().b200kv_lm_server_start(b"127.0.0.1", 0, ctypes.byref(h)))
    yield h, f"lm://127.0.0.1:{N.lib().b200kv_lm_server_port(h)}"
    N.lib().b200kv_lm_server_stop(h)


def _eng(url, W, r, fmt, local=None, reshard=None, serde="lossless", local_serde=None):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    cfg = LMCacheEngineConfig(256, local, url, serde, False, False, local_serde, reshard_world_sizes=reshard,
                              reshard_lossless=reshard is not None and serde == "lossless")
    return LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, W, r, fmt, "bfloat16"))


def _engine_kv(T, Hg, fmt, seed, L=4, D=128, dtype=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dt = dtype or (torch.bfloat16 if fmt == "vllm" else torch.float16)
    shape = (T, Hg, D) if fmt == "vllm" else (Hg, T, D)
    return [(torch.randn(shape, generator=g, device="cuda").to(dt), torch.randn(shape, generator=g, device="cuda").to(dt))
            for _ in range(L)]


def _heads(kv, a, b, fmt):
    return tuple((k[:, a:b] if fmt == "vllm" else k[a:b], v[:, a:b] if fmt == "vllm" else v[a:b]) for k, v in kv)


def _toks(kv, a, b, fmt):
    return tuple((k[a:b], v[a:b]) if fmt == "vllm" else (k[:, a:b], v[:, a:b]) for k, v in kv)


def _store_layout(url, W, kv, tokens, fmt, Hg, autorelease, upto=None, serde="lossless"):
    """engines of layout W store their head shards; upto[r]: tokens rank r stores"""
    for r in range(W):
        e = autorelease(_eng(url, W, r, fmt, serde=serde))
        n = len(tokens) if upto is None else upto[r]
        e.store(tokens[:n], _toks(_heads(kv, r * Hg // W, (r + 1) * Hg // W, fmt), 0, n, fmt))


def _same(a, b):
    assert len(a) == len(b)
    for (ak, av), (bk, bv) in zip(a, b):
        assert ak.dtype == bk.dtype
        assert torch.equal(_i16(ak), _i16(bk)) and torch.equal(_i16(av), _i16(bv))


def _masked(kv, m, fmt):
    """the tokens of kv where the retrieve mask m is set (a prefix-free suffix: one slice)"""
    idx = torch.nonzero(m).flatten()
    a, b = int(idx[0]), int(idx[-1]) + 1
    return _toks(kv, a, b, fmt)


@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
@pytest.mark.parametrize("W,Wd", [(2, 1), (1, 2), (4, 2), (2, 4)])
def test_retrieve_across_layouts(W, Wd, fmt, server, autorelease):
    from lmcache_b200.cache_engine import sha256_prefix_chain
    from lmcache_b200.utils import CacheEngineKey
    Hg, T = 8, 700                                                   # a ragged tail: 256 + 256 + 188
    tokens = torch.randint(0, 30000, (T,), device="cuda")
    kv = _engine_kv(T, Hg, fmt, W * 10 + Wd)
    _store_layout(server[1], W, kv, tokens, fmt, Hg, autorelease)
    rd = Wd - 1
    mine = _heads(kv, rd * Hg // Wd, (rd + 1) * Hg // Wd, fmt)       # the original KV's heads of rank Wd - 1
    # what layout Wd's own lossless retrieve of the same KV gives (stored under other tokens: other keys)
    tokens2 = tokens + 1
    own_w = autorelease(_eng(server[1], Wd, rd, fmt))
    own_w.store(tokens2, mine)
    mask = torch.ones(T, dtype=torch.bool)
    mask[:300] = False                                               # straddles chunk 1
    for msk in (mask, None):                                         # the store at the end of None comes last
        own_kv, own_m = own_w.retrieve(tokens2, msk)
        e = autorelease(_eng(server[1], Wd, rd, fmt, reshard=[W]))     # retrieve-only: geometry and dtype from a header
        got, m = e.retrieve(tokens, msk)
        want = mine if msk is None else _masked(mine, m, fmt)
        assert torch.equal(m, own_m) and int(m.sum()) == (T if msk is None else T - 300)
        _same(got, want)
        _same(got, own_kv)
        assert e.reshard_stats()[W]["chunks"] == (3 if msk is None else 2)
        lw = e.retrieve_layerwise(tokens, msk)
        lw.synchronize()
        assert torch.equal(lw.ret_mask, m)
        _same(lw.kv, want)
        if fmt == "vllm":                                            # paged, scrambled slots
            L, D = len(kv), 128
            nslots = T + 50
            slots = torch.randperm(nslots, device="cuda")[:T]
            caches = [(torch.zeros((nslots, Hg // Wd, D), dtype=torch.bfloat16, device="cuda"),
                       torch.zeros((nslots, Hg // Wd, D), dtype=torch.bfloat16, device="cuda")) for _ in range(L)]
            pm = e.retrieve_paged(tokens, caches, slots, msk)
            assert torch.equal(pm, m)
            sel = slots[m.cuda()]
            for (kc, vc), (k, v) in zip(caches, want):
                assert torch.equal(_i16(kc[sel]), _i16(k)) and torch.equal(_i16(vc[sel]), _i16(v))
        # never stored: nothing was written under this engine's keys; its ordinary store() then lands the same bits
        if msk is None:
            hashes = sha256_prefix_chain(tokens, 256)
            assert not any(e.engine_.contains(CacheEngineKey(fmt, MODEL, Wd, rd, h)) for h in hashes)
            e.store(tokens, got)
            again, m2 = autorelease(_eng(server[1], Wd, rd, fmt)).retrieve(tokens)
            assert int(m2.sum()) == T
            _same(again, mine)


def test_partial_shards_stop_at_the_first_incomplete_chunk(server, autorelease):
    Hg, T = 8, 1024
    tokens = torch.randint(0, 30000, (T,), device="cuda")
    kv = _engine_kv(T, Hg, "vllm", 5)
    _store_layout(server[1], 2, kv, tokens, "vllm", Hg, autorelease, upto=[1024, 512])
    e = autorelease(_eng(server[1], 1, 0, "vllm", reshard=[2]))
    got, m = e.retrieve(tokens)
    assert int(m.sum()) == 512
    _same(got, _toks(kv, 0, 512, "vllm"))
    assert e.reshard_stats()[2]["chunks"] == 2


def test_own_prefix_then_continuation_with_a_lossless_hybrid(server, autorelease):
    from lmcache_b200.cache_engine import sha256_prefix_chain
    from lmcache_b200.utils import CacheEngineKey
    Hg, T = 8, 1024
    tokens = torch.randint(0, 30000, (T,), device="cuda")
    kv = _engine_kv(T, Hg, "vllm", 9)
    _store_layout(server[1], 2, kv, tokens, "vllm", Hg, autorelease)                # all four chunks at W = 2
    own = autorelease(_eng(server[1], 1, 0, "vllm", local="cpu", local_serde="lossless", reshard=[2]))
    own.store(tokens[:512], _toks(kv, 0, 512, "vllm"))                               # two chunks at W = 1
    got, m = own.retrieve(tokens)
    assert int(m.sum()) == T
    _same(got, kv)
    assert own.reshard_stats()[2]["chunks"] == 2
    hashes = sha256_prefix_chain(tokens, 256)
    lt = own.engine_.local_store
    assert all(lt.contains(CacheEngineKey("vllm", MODEL, 1, 0, h)) for h in hashes[:2])
    assert not any(lt.contains(CacheEngineKey("vllm", MODEL, w, r, h)) for h in hashes for w, r in
                   ((1, 0), (2, 0), (2, 1)) if not (w == 1 and h in hashes[:2]))


def test_retrieve_only_replica_learns_an_fp16_geometry_from_the_source_header(server, autorelease):
    Hg, T = 4, 600
    tokens = torch.randint(0, 30000, (T,), device="cuda")
    kv = _engine_kv(T, Hg, "vllm", 13, L=3, D=64, dtype=torch.float16)
    _store_layout(server[1], 1, kv, tokens, "vllm", Hg, autorelease)
    e = autorelease(_eng(server[1], 4, 2, "vllm", reshard=[1]))
    got, m = e.retrieve(tokens)
    assert int(m.sum()) == T and len(got) == 3 and got[0][0].shape == (T, 1, 64)
    _same(got, _heads(kv, 2, 3, "vllm"))


@pytest.mark.parametrize("stored,wanted", [("cachegen", "lossless"), ("lossless", "cachegen")])
def test_a_source_of_the_other_family_is_a_total_miss(stored, wanted, server, autorelease):
    Hg, T = 8, 512
    tokens = torch.randint(0, 30000, (T,), device="cuda")
    kv = _engine_kv(T, Hg, "vllm", 3)
    _store_layout(server[1], 2, kv, tokens, "vllm", Hg, autorelease, serde=stored)
    e = autorelease(_eng(server[1], 1, 0, "vllm", reshard=[2], serde=wanted))
    got, m = e.retrieve(tokens)
    assert len(got) == 0 and int(m.sum()) == 0
    assert e.reshard_stats() == {}


def test_a_dtype_mismatch_is_a_miss(server, autorelease):
    Hg, T, L, D = 8, 512, 4, 128
    tokens = torch.randint(0, 30000, (T,), device="cuda")
    kv = _engine_kv(T, Hg, "vllm", 21)                                             # bf16
    _store_layout(server[1], 2, kv, tokens, "vllm", Hg, autorelease)
    e = autorelease(_eng(server[1], 1, 0, "vllm", reshard=[2]))
    slots = torch.randperm(T + 16, device="cuda")[:T]
    caches = [(torch.full((T + 16, Hg, D), SENT, dtype=torch.int16, device="cuda").view(torch.float16),
               torch.full((T + 16, Hg, D), SENT, dtype=torch.int16, device="cuda").view(torch.float16)) for _ in range(L)]
    pm = e.retrieve_paged(tokens, caches, slots)
    assert int(pm.sum()) == 0
    assert all(bool((c.view(torch.int16) == SENT).all()) for kv_ in caches for c in kv_)
    # the same engine with bf16 caches gets every chunk
    caches = [(torch.zeros((T + 16, Hg, D), dtype=torch.bfloat16, device="cuda"),
               torch.zeros((T + 16, Hg, D), dtype=torch.bfloat16, device="cuda")) for _ in range(L)]
    assert int(e.retrieve_paged(tokens, caches, slots).sum()) == T
    for (kc, vc), (k, v) in zip(caches, kv):
        assert torch.equal(_i16(kc[slots]), _i16(k)) and torch.equal(_i16(vc[slots]), _i16(v))
