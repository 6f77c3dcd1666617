"""GPU: decoding another tensor-parallel layout's CacheGen containers into this rank's KV heads.

Kernel: b200kv_decode_plan_heads (through CacheGenCodec.decode_raw_heads / decode_plan_heads) against whole decodes of
the same containers (b200kv_decode_chunks) and the oracle, over seeded random shapes, container versions, destinations
and layer splits; bytes outside the windows stay untouched; refused arguments write nothing.
Engine: stores of one layout retrieved by engines of another through an in-process lm:// server."""
import ctypes
import random

import numpy as np
import pytest
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu
MODEL = "mistralai/Mistral-7B-Instruct-v0.2"
SENT = -21555                      # sentinel int16 pattern of destination bytes nobody may write
CODERS = ["rans_compact", "rans", "ac"]


def _codec(coder):
    from lmcache_b200.codec import CacheGenCodec
    return CacheGenCodec(MODEL, coder=coder)


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
                     [j * ntok[0] for j in range(len(offs))], md, cd)
    assert codec.decode_status() == [0] * len(offs)
    return out


class _Dst:
    """A destination of H heads and T tokens in one of three layouts, filled with the sentinel; dense() reads it back as
    [L,2,T,H,D], untouched() says whether everything outside the token rows is still the sentinel."""

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


def _i16(t):
    return t.contiguous().view(torch.int16)


def _layer_splits(L, rng):
    cuts = sorted(rng.sample(range(1, L), rng.randint(0, L - 1))) if L > 1 else []
    return list(zip([0] + cuts, cuts + [L]))


# ---------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("case", range(40))
def test_windowed_decode_is_the_head_slice_of_a_whole_decode(case):
    rng = random.Random(1000 + case)
    torch.manual_seed(case)
    coder = CODERS[case % 3]
    Hs = [1, 2, 4, 8, 32][case % 5]
    D = rng.choice([64, 128])
    dtype = rng.choice([torch.bfloat16, torch.float16])
    kind = ["vllm", "huggingface", "paged"][(case // 3) % 3]
    L = rng.choice([1, 2, 3, 4])
    multi = coder != "rans_compact" and case % 2 == 0           # version 1 / 2 containers of two or three groups
    chunk = rng.choice([300, 600]) if multi else rng.choice([16, 100, 256])
    nch = rng.randint(1, 3)
    T = chunk * (nch - 1) + rng.randint(1, chunk)
    codec = _codec(coder)
    kv = (torch.randn((L, 2, T, Hs, D), device="cuda") * (1 + 3 * torch.rand((1, 1, 1, Hs, D), device="cuda"))).to(dtype)
    enc = _encode(codec, kv, chunk)
    full = _full_decode(codec, enc, kv.shape, dtype)
    n = len(enc[1])
    ntok = enc[3]
    # per chunk a random window, landing at a random head of a destination with more heads
    src0 = [rng.randrange(Hs) for _ in range(n)]
    nh = [rng.randint(1, Hs - s) for s in src0]
    Hd = max(nh) + rng.randint(0, 3)
    dst0 = [rng.randint(0, Hd - k) for k in nh]
    dst = _Dst(kind, L, T, Hd, D, dtype, rng)
    want = torch.full((L, 2, T, Hd, D), SENT, dtype=torch.int16, device="cuda")
    for j in range(n):
        a = j * chunk
        want[:, :, a:a + ntok[j], dst0[j]:dst0[j] + nh[j]] = _i16(full[:, :, a:a + ntok[j], src0[j]:src0[j] + nh[j]])
    buf, offs, tot, _, md, cd = enc
    toks = [j * chunk for j in range(n)]
    if case % 2:
        codec.decode_raw_heads(buf.data_ptr(), buf.numel(), offs, tot, ntok, dst.view, toks, md, cd, Hs, src0, dst0, nh)
        assert codec.decode_status() == [0] * n
    else:
        stream = torch.cuda.current_stream()
        st = torch.zeros(n, dtype=torch.int32, device="cuda")
        plan, ws = codec.decode_plan_heads(buf.data_ptr(), buf.numel(), offs, tot, ntok, dst.view, toks, md, cd, Hs,
                                           src0, dst0, nh, stream, st.data_ptr())
        for a, b in _layer_splits(L, rng):
            codec.decode_layers(plan, a, b, stream)
        torch.cuda.synchronize()
        assert st.tolist() == [0] * n
        del ws
    torch.cuda.synchronize()
    assert torch.equal(_i16(dst.dense()), want)
    assert dst.untouched()


@pytest.mark.parametrize("case", range(4))
def test_windowed_decode_matches_the_oracle(case):
    rng = random.Random(7 + case)
    coder = CODERS[case % 3]
    L, Hs, D, t = 2, [2, 4, 8, 1][case], [128, 64][case % 2], [64, 256, 200, 33][case]
    bits = O.synth_kv_bits(L, t, Hs * D, seed=case)
    kv = torch.from_numpy(bits.view(np.int16)).view(torch.bfloat16).reshape(L, 2, t, Hs, D).cuda()
    codec = _codec(coder)
    enc = _encode(codec, kv, 256)
    kb, vb = O.make_bins(MODEL)
    ref = O.decode_chunk(O.encode_chunk(bits, O.DT_BF16, kb[:L], vb[:L], O.CODER_RANS), O.DT_BF16, kb[:L], vb[:L],
                         O.DT_BF16).reshape(L, 2, t, Hs, D)
    s0 = rng.randrange(Hs)
    k = rng.randint(1, Hs - s0)
    dst = _Dst("vllm", L, t, k, D, torch.bfloat16, rng)
    buf, offs, tot, ntok, md, cd = enc
    codec.decode_raw_heads(buf.data_ptr(), buf.numel(), offs, tot, ntok, dst.view, [0], md, cd, Hs, [s0], [0], [k])
    torch.cuda.synchronize()
    got = dst.blob.view(torch.int16).cpu().numpy().view(np.uint16)
    assert np.array_equal(got, ref[:, :, :, s0:s0 + k])


@pytest.mark.parametrize("W_over", [2, 4])
@pytest.mark.parametrize("coder", CODERS)
def test_several_shards_into_one_rank_in_one_call(W_over, coder):
    """W / W' containers at one dst_tok, each whole into its own head range, equal the concatenation of their decodes."""
    torch.manual_seed(W_over)
    L, hs, D, T, chunk = 3, 2, 128, 300, 256 if coder == "rans_compact" else 300
    codec = _codec(coder)
    kv = (torch.randn((L, 2, T, hs * W_over, D), device="cuda") * 2).to(torch.bfloat16)
    encs = [_encode(codec, kv[:, :, :, r * hs:(r + 1) * hs].contiguous(), chunk) for r in range(W_over)]
    want = torch.cat([_full_decode(codec, e, (L, 2, T, hs, D), torch.bfloat16) for e in encs], dim=3)
    # all shards' containers in one buffer
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
    dst = _Dst("vllm", L, T, hs * W_over, D, torch.bfloat16, random.Random(0))
    codec.decode_raw_heads(allbuf.data_ptr(), allbuf.numel(), offs, tot, ntok, dst.view, toks, md, cd, hs, src0, dst0, nh)
    assert codec.decode_status() == [0] * len(offs)
    assert torch.equal(_i16(dst.blob), _i16(want))


def test_refused_windows_write_nothing():
    from lmcache_b200 import _native as N
    L, Hs, D, T = 2, 4, 64, 100
    codec = _codec("rans_compact")
    kv = torch.randn((L, 2, T, Hs, D), device="cuda").to(torch.bfloat16)
    buf, offs, tot, ntok, md, cd = _encode(codec, kv, 64)
    n = len(offs)
    dst = _Dst("vllm", L, T, 2, D, torch.bfloat16, random.Random(0))
    st = torch.full((n,), 77, dtype=torch.int32, device="cuda")
    ok = dict(src_H=Hs, src_head0=[0] * n, dst_head0=[0] * n, n_heads=[2] * n, toks=[0, 64])
    bad = [dict(n_heads=[0, 2]), dict(src_head0=[3, 0]), dict(src_head0=[-1, 0]), dict(dst_head0=[1, 0]),
           dict(dst_head0=[-1, 0]), dict(src_H=0), dict(n_heads=[5, 2], src_head0=[0, 0]),
           dict(toks=[0, 0], n_heads=[1, 2], dst_head0=[1, 0]), dict(toks=[0, 0], dst_head0=[0, 1], n_heads=[2, 1])]
    for b in bad:
        a = dict(ok, **b)
        with pytest.raises(N.NativeError, match="decode_plan_heads"):
            codec.decode_plan_heads(buf.data_ptr(), buf.numel(), offs, tot, ntok, dst.view, a["toks"], md, cd,
                                    a["src_H"], a["src_head0"], a["dst_head0"], a["n_heads"],
                                    torch.cuda.current_stream(), st.data_ptr())
    torch.cuda.synchronize()
    assert bool((dst.blob.view(torch.int16) == SENT).all()) and st.tolist() == [77] * n
    # disjoint ranges at one token are fine
    a = dict(ok, toks=[0, 0], dst_head0=[0, 1], n_heads=[1, 1], src_head0=[3, 0])
    codec.decode_raw_heads(buf.data_ptr(), buf.numel(), offs[:1] * 2, tot[:1] * 2, ntok[:1] * 2, dst.view, a["toks"], md,
                           cd, Hs, a["src_head0"], a["dst_head0"], a["n_heads"])
    full = _full_decode(codec, (buf, offs, tot, ntok, md, cd), kv.shape, torch.bfloat16)
    torch.cuda.synchronize()
    assert torch.equal(_i16(dst.blob[:, :, :64]), _i16(full[:, :, :64, [3, 0]]))


# ---------------------------------------------------------------------------------------------- engine
@pytest.fixture
def server():
    from lmcache_b200 import _native as N
    h = ctypes.c_void_p()
    N.check(N.lib().b200kv_lm_server_start(b"127.0.0.1", 0, ctypes.byref(h)))
    yield h, f"lm://127.0.0.1:{N.lib().b200kv_lm_server_port(h)}"
    N.lib().b200kv_lm_server_stop(h)


def _eng(url, W, r, fmt, local=None, reshard=None):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    cfg = LMCacheEngineConfig(256, local, url, "cachegen", False, False, "cachegen" if local == "cpu" else None,
                              reshard_world_sizes=reshard)
    return LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, W, r, fmt, "bfloat16"))


def _kv(T, Hg, fmt, seed, L=4, D=128):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dt = torch.bfloat16 if fmt == "vllm" else torch.float16
    shape = (T, Hg, D) if fmt == "vllm" else (Hg, T, D)
    return [(torch.randn(shape, generator=g, device="cuda").to(dt), torch.randn(shape, generator=g, device="cuda").to(dt))
            for _ in range(L)]


def _heads(kv, a, b, fmt):
    return tuple((k[:, a:b] if fmt == "vllm" else k[a:b], v[:, a:b] if fmt == "vllm" else v[a:b]) for k, v in kv)


def _store_layout(url, W, kv, tokens, fmt, Hg, upto=None, autorelease=None):
    """engines of layout W store their head shards; upto[r]: tokens rank r stores"""
    for r in range(W):
        e = autorelease(_eng(url, W, r, fmt))
        n = len(tokens) if upto is None else upto[r]
        part = _heads(kv, r * Hg // W, (r + 1) * Hg // W, fmt)
        e.store(tokens[:n], tuple((k[:n], v[:n]) if fmt == "vllm" else (k[:, :n], v[:, :n]) for k, v in part))


def _own(url, W, r, tokens, fmt, mask=None, autorelease=None):
    """what each source rank retrieves of its own layout"""
    e = autorelease(_eng(url, W, r, fmt))
    kv, m = e.retrieve(tokens, mask)
    return kv, m


def _cat_heads(parts, fmt):
    d = 1 if fmt == "vllm" else 0
    return tuple((torch.cat([p[l][0] for p in parts], d), torch.cat([p[l][1] for p in parts], d))
                 for l in range(len(parts[0])))


def _expected(url, W, Wd, rd, tokens, fmt, Hg, mask, autorelease):
    """rank rd of layout Wd out of layout W's own retrieves: concatenation (W > Wd) or slice (W < Wd)"""
    from lmcache_b200.reshard import source_shards
    parts, m0 = [], None
    for s in source_shards(Hg, W, Wd, rd):
        kv, m = _own(url, W, s.rank, tokens, fmt, mask, autorelease)
        m0 = m if m0 is None else m0
        assert torch.equal(m, m0)
        parts.append(_heads(kv, s.src_head0, s.src_head0 + s.n_heads, fmt))
    return _cat_heads(parts, fmt), m0


def _same(a, b):
    assert len(a) == len(b)
    for (ak, av), (bk, bv) in zip(a, b):
        assert torch.equal(_i16(ak), _i16(bk)) and torch.equal(_i16(av), _i16(bv))


@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
@pytest.mark.parametrize("W,Wd", [(2, 1), (1, 2), (4, 2), (2, 4)])
def test_retrieve_across_layouts(W, Wd, fmt, server, autorelease):
    Hg, T = 8, 700                                                   # a ragged tail: 256 + 256 + 188
    tokens = torch.randint(0, 30000, (T,), device="cuda")
    kv = _kv(T, Hg, fmt, W * 10 + Wd)
    _store_layout(server[1], W, kv, tokens, fmt, Hg, autorelease=autorelease)
    mask = torch.ones(T, dtype=torch.bool)
    mask[:300] = False                                               # straddles chunk 1
    for msk in (None, mask):
        want, wm = _expected(server[1], W, Wd, Wd - 1, tokens, fmt, Hg, msk, autorelease)
        e = autorelease(_eng(server[1], Wd, Wd - 1, fmt, reshard=[W]))
        got, m = e.retrieve(tokens, msk)
        assert torch.equal(m, wm) and int(m.sum()) == (T if msk is None else T - 300)
        _same(got, want)
        assert e.reshard_stats()[W]["chunks"] == (3 if msk is None else 2)
        lw = e.retrieve_layerwise(tokens, msk)
        lw.synchronize()
        assert torch.equal(lw.ret_mask, wm)
        _same(lw.kv, want)
        if fmt == "vllm":                                            # paged, scrambled slots
            L, D = len(kv), 128
            nslots = T + 50
            slots = torch.randperm(nslots, device="cuda")[:T]
            caches = [(torch.zeros((nslots, Hg // Wd, D), dtype=torch.bfloat16, device="cuda"),
                       torch.zeros((nslots, Hg // Wd, D), dtype=torch.bfloat16, device="cuda")) for _ in range(L)]
            pm = e.retrieve_paged(tokens, caches, slots, msk)
            assert torch.equal(pm, wm)
            sel = slots[wm.cuda()]
            for (kc, vc), (k, v) in zip(caches, want):
                assert torch.equal(_i16(kc[sel]), _i16(k)) and torch.equal(_i16(vc[sel]), _i16(v))


def test_partial_shards_stop_at_the_first_incomplete_chunk(server, autorelease):
    Hg, T = 8, 1024
    tokens = torch.randint(0, 30000, (T,), device="cuda")
    kv = _kv(T, Hg, "vllm", 5)
    _store_layout(server[1], 2, kv, tokens, "vllm", Hg, upto=[1024, 512], autorelease=autorelease)
    e = autorelease(_eng(server[1], 1, 0, "vllm", reshard=[2]))
    got, m = e.retrieve(tokens)
    assert int(m.sum()) == 512
    want, _ = _expected(server[1], 2, 1, 0, tokens[:512], "vllm", Hg, None, autorelease)
    _same(got, want)


@pytest.mark.parametrize("local", [None, "cpu"])
def test_own_prefix_then_continuation(local, server, autorelease):
    Hg, T = 8, 1024
    tokens = torch.randint(0, 30000, (T,), device="cuda")
    kv = _kv(T, Hg, "vllm", 9)
    _store_layout(server[1], 2, kv, tokens, "vllm", Hg, autorelease=autorelease)        # all four chunks at W = 2
    own = autorelease(_eng(server[1], 1, 0, "vllm", local=local, reshard=[2]))
    own.store(tokens[:512], tuple((k[:512], v[:512]) for k, v in kv))                  # two chunks at W = 1
    own_kv, _ = own.retrieve(tokens[:512])
    got, m = own.retrieve(tokens)
    assert int(m.sum()) == T
    _same(tuple((k[:512], v[:512]) for k, v in got), own_kv)
    want, _ = _expected(server[1], 2, 1, 0, tokens, "vllm", Hg, None, autorelease)
    _same(tuple((k[512:], v[512:]) for k, v in got), tuple((k[512:], v[512:]) for k, v in want))
    assert own.reshard_stats()[2]["chunks"] == 2
    if local == "cpu":
        from lmcache_b200.cache_engine import sha256_prefix_chain
        from lmcache_b200.utils import CacheEngineKey
        hashes = sha256_prefix_chain(tokens, 256)
        lt = own.engine_.local_store
        assert not any(lt.contains(CacheEngineKey("vllm", MODEL, w, r, h)) for h in hashes for w, r in
                       ((1, 0), (2, 0), (2, 1)) if not (w == 1 and h in hashes[:2]))


def test_off_by_default_is_a_total_miss_without_extra_requests(server, autorelease, monkeypatch):
    from lmcache_b200.storage_backend.remote_backend import LMCRemoteBackend
    Hg, T = 8, 512
    tokens = torch.randint(0, 30000, (T,), device="cuda")
    kv = _kv(T, Hg, "vllm", 3)
    _store_layout(server[1], 2, kv, tokens, "vllm", Hg, autorelease=autorelease)
    e = autorelease(_eng(server[1], 1, 0, "vllm"))
    seen = []
    orig_contains, orig_fetch = LMCRemoteBackend.contains, LMCRemoteBackend._fetch
    monkeypatch.setattr(LMCRemoteBackend, "contains", lambda self, k: seen.append(k) or orig_contains(self, k))
    monkeypatch.setattr(LMCRemoteBackend, "_fetch", lambda self, k, *a: seen.append(k) or orig_fetch(self, k, *a))
    got, m = e.retrieve(tokens)
    assert len(got) == 0 and int(m.sum()) == 0
    assert all(k.world_size == 1 for k in seen) and e.reshard_stats() == {}
