"""GPU: LMCacheEngine with a latent KV (metadata.use_mla, DeepSeek-V2/V3: one [T, D] tensor per layer) on every tier.

Round trips are bit-exact to the input on the raw tiers (cpu, cuda, lm:// with the torch serde) and bit-exact to
CacheGenCodec's own version-4 encode + decode on the CacheGen tiers (cpu + cachegen, a directory, lm:// with the cachegen
serde, hybrid), which the oracle checks in turn.  Then: prefix and suffix-mask semantics, the paged forms with a shuffled
slot mapping, the layer-wise store and retrieve, the device-cache level and a bounded tier, a disk restart, the keys
shared by tensor-parallel ranks (rank 0 alone puts to the server) and the clean miss of a (K, V) engine on those keys."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle as O

import mla_ref

pytestmark = pytest.mark.gpu
MODEL = "deepseek-ai/DeepSeek-V3"
CHUNK = 256
SENT = -21555


def _cfg(L):
    return dict(key_first_layers=min(3, L), key_second_layers=min(20, L), key_third_layers=L, key_first_bins=32,
                key_second_bins=16, key_third_bins=12, value_first_layers=2, value_first_bins=32, value_second_bins=16)


def _latent(L, T, D, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    sigma = torch.exp(0.5 * torch.randn((L, 1, D), device="cuda", generator=g)).clamp_(0.1, 8.0)
    return (torch.randn((L, T, D), device="cuda", generator=g) * sigma).to(dtype)


def _tokens(T, seed=0):
    return torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(seed))


def _bits(x):
    return x.contiguous().view(torch.int16)


@pytest.fixture
def server():
    from lmcache_b200 import _native as N
    h = ctypes.c_void_p()
    N.check(N.lib().b200kv_lm_server_start(b"127.0.0.1", 0, ctypes.byref(h)))
    yield f"lm://127.0.0.1:{N.lib().b200kv_lm_server_port(h)}", h
    N.lib().b200kv_lm_server_stop(h)


def _num_keys(server):
    from lmcache_b200 import _native as N
    return N.lib().b200kv_lm_server_num_keys(server[1])


TIERS = ["cpu", "cuda", "lm_torch", "cpu_cachegen", "disk", "lm_cachegen", "hybrid"]
RAW = {"cpu", "cuda", "lm_torch"}


def _config(tier, L, tmp_path=None, server=None, **kw):
    from lmcache_b200.config import LMCacheEngineConfig
    cg = _cfg(L)
    url = server[0] if server is not None else None
    if tier in ("cpu", "cuda"):
        return LMCacheEngineConfig(CHUNK, tier, None, None, False, False, cachegen_config=cg, **kw)
    if tier == "cpu_cachegen":
        return LMCacheEngineConfig(CHUNK, "cpu", None, None, False, False, "cachegen", cachegen_config=cg, **kw)
    if tier == "disk":
        return LMCacheEngineConfig(CHUNK, f"{tmp_path}/", None, None, False, False, cachegen_config=cg, **kw)
    if tier == "lm_torch":
        return LMCacheEngineConfig(CHUNK, None, url, "torch", False, False, cachegen_config=cg, **kw)
    if tier == "lm_cachegen":
        return LMCacheEngineConfig(CHUNK, None, url, "cachegen", False, False, cachegen_config=cg, **kw)
    assert tier == "hybrid"
    return LMCacheEngineConfig(CHUNK, "cpu", url, "cachegen", False, False, "cachegen", cachegen_config=cg, **kw)


def _engine(autorelease, tier, L, tmp_path=None, server=None, ws=1, rank=0, mla=True, **kw):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineMetadata
    meta = LMCacheEngineMetadata(MODEL, ws, rank, "vllm", "bfloat16", mla)
    return autorelease(LMCacheEngine(_config(tier, L, tmp_path, server, **kw), meta))


def _want(tier, x):
    """what a retrieve of the whole of x [L, T, D] returns on `tier`: x itself on a raw tier; CacheGenCodec's version-4
    encode in 256-token chunks, decoded into bf16 (the vllm format's output dtype), on a CacheGen tier"""
    from lmcache_b200.codec import CacheGenCodec, KvView
    if tier in RAW:
        return x
    L, T, D = x.shape
    codec = CacheGenCodec(MODEL, cachegen_config=_cfg(L))
    batch = codec.encode(KvView.from_blob(x, "vllm"), 0, T, CHUNK)
    out = torch.full((L, T, D), SENT, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    n = len(batch.sizes)
    codec.decode_device_batch(batch, [min(CHUNK, T - j * CHUNK) for j in range(n)], KvView.from_blob(out, "vllm"),
                              [j * CHUNK for j in range(n)])
    assert codec.decode_status() == [0] * n
    torch.cuda.synchronize()
    return out


def _stack(kv):
    return torch.stack(list(kv))


def _needs(tier):
    return tier.startswith("lm") or tier == "hybrid"


# ---------------------------------------------------------------------------------------------- round trips
CASES = [(torch.bfloat16, 1, 512), (torch.float16, 27, 576), (torch.bfloat16, 61, 576), (torch.float16, 128, 512)]


@pytest.mark.parametrize("case", range(len(CASES)), ids=lambda c: "{}-L{}-D{}".format(
    str(CASES[c][0]).split(".")[-1], CASES[c][1], CASES[c][2]))
@pytest.mark.parametrize("tier", TIERS)
def test_store_retrieve_round_trip(tier, case, tmp_path, autorelease, request):
    dtype, L, D = CASES[case]
    srv = request.getfixturevalue("server") if _needs(tier) else None
    T = 600                                                   # two whole chunks and a ragged tail
    x = _latent(L, T, D, dtype, seed=case)
    tokens = _tokens(T, case)
    eng = _engine(autorelease, tier, L, tmp_path, srv)
    eng.store(tokens, tuple(x[l] for l in range(L)))
    # a shared tier is read by a second engine that knows no geometry (it peeks a header / blob)
    reader = _engine(autorelease, tier, L, tmp_path, srv) if tier in ("lm_torch", "lm_cachegen") else eng
    kv, mask = reader.retrieve(tokens)
    assert len(kv) == L and all(t.shape == (T, D) for t in kv)
    assert int(mask.sum()) == T
    want = _want(tier, x)
    assert kv[0].dtype == want.dtype
    assert torch.equal(_bits(_stack(kv)), _bits(want))
    if tier in RAW:
        return
    # the codec's bits are the oracle's: dequantised symbols of the oracle's own quantiser, chunk by chunk
    if case in (0, 1):
        from lmcache_b200.storage_backend.serde.cachegen_basics import CacheGenConfig
        kb = np.asarray(CacheGenConfig.for_engine(MODEL, _cfg(L)).key_bins_list(), np.float32)
        xb = x.view(torch.int16).cpu().numpy().view(np.uint16)
        dt = O.DT_BF16 if dtype == torch.bfloat16 else O.DT_FP16
        got = _bits(want).cpu().numpy().view(np.uint16)
        for c0 in range(0, T, CHUNK):
            part = np.ascontiguousarray(xb[:, c0:c0 + CHUNK])
            enc = mla_ref.encode_chunk_latent(part, dt, kb)
            assert np.array_equal(mla_ref.decode_latent(enc, dt, kb, O.DT_BF16), got[:, c0:c0 + CHUNK])


# ---------------------------------------------------------------------------------------------- prefix and masks
@pytest.mark.parametrize("tier", ["cpu", "cpu_cachegen", "lm_cachegen", "lm_torch"])
def test_prefix_and_suffix_mask(tier, tmp_path, autorelease, request):
    srv = request.getfixturevalue("server") if _needs(tier) else None
    L, D, T = 5, 576, 1000
    x = _latent(L, T, D, torch.bfloat16, seed=11)
    tokens = _tokens(T, 11)
    eng = _engine(autorelease, tier, L, tmp_path, srv)
    eng.store(tokens[:612], tuple(x[l, :612] for l in range(L)))        # chunks 0, 1 and a 100-token tail
    want = _want(tier, x[:, :612].contiguous())
    # a longer prompt: chunks 0 and 1 match, the stored tail is another chunk's prefix
    kv, mask = eng.retrieve(tokens)
    assert int(mask.sum()) == 512 and bool(mask[:512].all())
    assert torch.equal(_bits(_stack(kv)), _bits(want[:, :512]))
    # the same prompt: the ragged tail too
    kv, mask = eng.retrieve(tokens[:612])
    assert int(mask.sum()) == 612 and torch.equal(_bits(_stack(kv)), _bits(want))
    # a suffix mask whose first chunk straddles it: tokens 300.. of 612
    m = torch.ones(612, dtype=torch.bool)
    m[:300] = False
    kv, mask = eng.retrieve(tokens[:612], m)
    assert not bool(mask[:300].any()) and bool(mask[300:].all())
    assert torch.equal(_bits(_stack(kv)), _bits(want[:, 300:]))
    # a total miss
    kv, mask = eng.retrieve(_tokens(300, 99))
    assert kv == () and not bool(mask.any())


# ---------------------------------------------------------------------------------------------- paged
def _paged(L, nslots, D, dtype, block=16):
    return [torch.full((nslots // block, block, D), SENT, dtype=torch.int16, device="cuda").view(dtype)
            for _ in range(L)]


@pytest.mark.parametrize("tier", ["cuda", "cpu", "cpu_cachegen", "lm_cachegen", "lm_torch"])
def test_paged_store_and_retrieve(tier, tmp_path, autorelease, request):
    srv = request.getfixturevalue("server") if _needs(tier) else None
    L, D, T, nslots = 4, 576, 700, 1024
    x = _latent(L, T, D, torch.bfloat16, seed=21)
    tokens = _tokens(T, 21)
    slots = torch.randperm(nslots, generator=torch.Generator().manual_seed(3))[:T].cuda()
    src = _paged(L, nslots, D, torch.bfloat16)
    for l in range(L):
        src[l].view(-1, D)[slots] = x[l]
    eng = _engine(autorelease, tier, L, tmp_path, srv)
    eng.store_paged(tokens, src, slots)
    want = _want(tier, x)
    for mask_from in (0, 300):
        dst = _paged(L, nslots, D, torch.bfloat16)
        m = None
        if mask_from:
            m = torch.ones(T, dtype=torch.bool)
            m[:mask_from] = False
        ret = eng.retrieve_paged(tokens, dst, slots, m)
        assert int(ret.sum()) == T - mask_from and bool(ret[mask_from:].all())
        rows = slots[mask_from:]
        rest = torch.ones(nslots, dtype=torch.bool, device="cuda")
        rest[rows] = False
        for l in range(L):
            flat = dst[l].view(-1, D)
            assert torch.equal(_bits(flat[rows]), _bits(want[l, mask_from:]))
            assert bool((flat.view(torch.int16)[rest] == SENT).all())          # rows not retrieved stay untouched
    # the paged store is the blob store: a blob retrieve gets the same bits
    kv, _ = eng.retrieve(tokens)
    assert torch.equal(_bits(_stack(kv)), _bits(want))


# ---------------------------------------------------------------------------------------------- layer-wise
def _containers(eng, tokens):
    from lmcache_b200.cache_engine import sha256_prefix_chain
    out = []
    for h in sha256_prefix_chain(tokens, CHUNK):
        e = eng.engine_._lookup(eng._make_key(h, "vllm"))
        e.ready.wait()
        out.append(bytes(e.rec.blk.view()[:e.rec.nbytes]))
    return out


def test_layerwise_store_writes_the_containers_of_store(autorelease):
    L, D, T = 61, 576, 700
    x = _latent(L, T, D, torch.bfloat16, seed=31)
    tokens = _tokens(T, 31)
    a = _engine(autorelease, "cpu_cachegen", L)
    a.store(tokens, tuple(x[l] for l in range(L)))
    b = _engine(autorelease, "cpu_cachegen", L)
    st = b.store_layerwise(tokens, tuple(x[l] for l in range(L)))
    assert st.num_layers == L and st._enc is not None              # encoded layer by layer, not at finish()
    for l in range(L):
        st.save_layer(l)
    st.finish()
    ca, cb = _containers(a, tokens), _containers(b, tokens)
    assert len(ca) == 3 and ca == cb
    assert all(c[4] == 4 for c in ca)                              # version 4
    # the paged layer-wise store as well
    nslots = 1024
    slots = torch.randperm(nslots, generator=torch.Generator().manual_seed(4))[:T].cuda()
    src = _paged(L, nslots, D, torch.bfloat16)
    for l in range(L):
        src[l].view(-1, D)[slots] = x[l]
    c = _engine(autorelease, "cpu_cachegen", L)
    st = c.store_paged_layerwise(tokens, src, slots)
    for l in range(L):
        st.save_layer(l)
    st.finish()
    assert _containers(c, tokens) == ca


@pytest.mark.parametrize("tier", ["cpu_cachegen", "disk"])
def test_layerwise_retrieve_equals_retrieve(tier, tmp_path, autorelease):
    L, D, T = 61, 576, 700
    x = _latent(L, T, D, torch.bfloat16, seed=41)
    tokens = _tokens(T, 41)
    eng = _engine(autorelease, tier, L, tmp_path)
    eng.store(tokens, tuple(x[l] for l in range(L)))
    m = torch.ones(T, dtype=torch.bool)
    m[:300] = False
    for mask in (None, m):
        kv, ret = eng.retrieve(tokens, mask)
        want = _bits(_stack(kv))
        r = eng.retrieve_layerwise(tokens, mask)
        assert r.num_layers == L and torch.equal(r.ret_mask, ret) and len(r.kv) == L
        assert r._upload.num_layers == L and r._upload.n > 0      # the layer-major path ran
        side = torch.cuda.Stream()
        for l in (0, L // 2, L - 1):                              # layer l may be read once wait_layer(l) was called
            r.wait_layer(l, side)
            with torch.cuda.stream(side):
                got = r.kv[l].clone()
            side.synchronize()
            assert torch.equal(_bits(got), want[l])
        r.synchronize()
        assert torch.equal(_bits(_stack(r.kv)), want)
        # the paged form
        nslots = 1024
        slots = torch.randperm(nslots, generator=torch.Generator().manual_seed(5))[:T].cuda()
        d1, d2 = _paged(L, nslots, D, torch.bfloat16), _paged(L, nslots, D, torch.bfloat16)
        ret1 = eng.retrieve_paged(tokens, d1, slots, mask)
        rp = eng.retrieve_paged_layerwise(tokens, d2, slots, mask)
        assert rp.kv is None and rp.num_layers == L and torch.equal(rp.ret_mask, ret1)
        rp.synchronize()
        assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(d1, d2))


# ---------------------------------------------------------------------------------------------- device cache, eviction
def test_device_cache_hits_decode_the_same_bits(autorelease):
    L, D, T = 27, 576, 700
    x = _latent(L, T, D, torch.bfloat16, seed=51)
    tokens = _tokens(T, 51)
    eng = _engine(autorelease, "cpu_cachegen", L, device_cache_bytes=256 << 20)
    eng.store(tokens, tuple(x[l] for l in range(L)))
    want = _bits(_want("cpu_cachegen", x))
    for _ in range(2):
        kv, mask = eng.retrieve(tokens)
        assert int(mask.sum()) == T and torch.equal(_bits(_stack(kv)), want)
        r = eng.retrieve_layerwise(tokens)
        r.synchronize()
        assert torch.equal(_bits(_stack(r.kv)), want)
    stats = eng.engine_.device_cache_stats()
    assert stats["hits"] >= 3 and stats["bytes_in_use"] > 0


def test_bounded_tier_keeps_a_retrievable_prefix(autorelease):
    from lmcache_b200.codec import CacheGenCodec, KvView
    L, D, T = 27, 576, 1024
    xa, xb = _latent(L, T, D, torch.bfloat16, seed=61), _latent(L, T, D, torch.bfloat16, seed=62)
    ta, tb = _tokens(T, 61), _tokens(T, 62)
    size = max(CacheGenCodec(MODEL, cachegen_config=_cfg(L)).encode(KvView.from_blob(xa, "vllm"), 0, T, CHUNK).sizes)
    eng = _engine(autorelease, "cpu_cachegen", L, local_capacity_bytes=int(2.5 * size) + 4096)
    eng.store(ta, tuple(xa[l] for l in range(L)))
    eng.store(tb, tuple(xb[l] for l in range(L)))
    for x, tok in ((xa, ta), (xb, tb)):
        kv, mask = eng.retrieve(tok)
        n = int(mask.sum())
        assert n % CHUNK == 0 and n < T and bool(mask[:n].all())
        if n:
            assert torch.equal(_bits(_stack(kv)), _bits(_want("cpu_cachegen", x)[:, :n]))
    kv, mask = eng.retrieve(tb)
    assert int(mask.sum()) >= CHUNK                                 # the latest store keeps its head
    assert eng.engine_.host_bytes() <= int(2.5 * size) + 4096


# ---------------------------------------------------------------------------------------------- disk restart
def test_disk_restart(tmp_path, autorelease):
    L, D, T = 61, 576, 600
    x = _latent(L, T, D, torch.float16, seed=71)
    tokens = _tokens(T, 71)
    eng = _engine(autorelease, "disk", L, tmp_path)
    eng.store(tokens, tuple(x[l] for l in range(L)))
    eng.retrieve(tokens)                         # the files are complete once a retrieve has waited for the store
    eng.close()
    assert len(list(tmp_path.glob("*.b2kv"))) == 3
    again = _engine(autorelease, "disk", L, tmp_path)
    kv, mask = again.retrieve(tokens)
    assert int(mask.sum()) == T and torch.equal(_bits(_stack(kv)), _bits(_want("disk", x)))
    # a (K, V) engine of the same model on the same directory indexes none of them
    kveng = _engine(autorelease, "disk", L, tmp_path, mla=False)
    assert len(kveng.engine_.dict) == 0
    kv, mask = kveng.retrieve(tokens)
    assert kv == () and not bool(mask.any())


# ---------------------------------------------------------------------------------------------- TP ranks, cross-kind
@pytest.mark.parametrize("tier", ["lm_cachegen", "lm_torch"])
def test_tensor_parallel_ranks_share_rank_0s_chunks(tier, server, autorelease):
    L, D, T = 27, 576, 600
    x = _latent(L, T, D, torch.bfloat16, seed=81)
    tokens = _tokens(T, 81)
    kv_in = tuple(x[l] for l in range(L))
    r0 = _engine(autorelease, tier, L, server=server, ws=2, rank=0)
    r1 = _engine(autorelease, tier, L, server=server, ws=2, rank=1)
    w1 = _engine(autorelease, tier, L, server=server, ws=1, rank=0)
    r1.store(tokens, kv_in)
    assert _num_keys(server) == 0                                   # rank 1 puts nothing to the shared tier
    kv, mask = r1.retrieve(tokens)
    assert kv == () and not bool(mask.any())
    r0.store(tokens, kv_in)
    want = _bits(_want(tier, x))
    for eng in (r0, r1, w1):                    # r0's lookups go over the connection its puts took: they are in
        kv, mask = eng.retrieve(tokens)
        assert int(mask.sum()) == T and torch.equal(_bits(_stack(kv)), want)
    assert _num_keys(server) == 3
    w1.store(tokens, kv_in)                                          # the same keys: nothing new
    w1.retrieve(tokens)
    assert _num_keys(server) == 3
    # a (K, V) engine of the same model name finds the keys but not its kind of chunk: a clean miss
    kveng = _engine(autorelease, tier, L, server=server, mla=False)
    kv, mask = kveng.retrieve(tokens)
    assert kv == () and not bool(mask.any())


def test_hybrid_rank_1_fills_its_local_tier_only(server, autorelease):
    L, D, T = 27, 576, 600
    x = _latent(L, T, D, torch.bfloat16, seed=91)
    tokens = _tokens(T, 91)
    r1 = _engine(autorelease, "hybrid", L, server=server, ws=2, rank=1)
    r1.store(tokens, tuple(x[l] for l in range(L)))
    assert _num_keys(server) == 0
    want = _bits(_want("hybrid", x))
    kv, mask = r1.retrieve(tokens)
    assert int(mask.sum()) == T and torch.equal(_bits(_stack(kv)), want)
    r0 = _engine(autorelease, "hybrid", L, server=server, ws=2, rank=0)
    r0.store(tokens, tuple(x[l] for l in range(L)))                # blocking: ends with a round trip per connection
    assert _num_keys(server) == 3
    w1 = _engine(autorelease, "lm_cachegen", L, server=server)
    kv, mask = w1.retrieve(tokens)
    assert int(mask.sum()) == T and torch.equal(_bits(_stack(kv)), want)
