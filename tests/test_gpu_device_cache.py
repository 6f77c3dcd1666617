"""GPU: the device level of the CacheGen host and disk tiers (config.device_cache_bytes).  Every case compares with the
same engine configuration without the level: what a retrieve returns must be the same bits whether its containers were
decoded in the level's pool or uploaded from the tier."""
import pytest
import torch

from test_gpu_host_tier import _blob_of, _kv, _meta

pytestmark = pytest.mark.gpu
CS = 256
L = 6


def _cfg(backend="cpu", device_cache=None, capacity=None):
    from lmcache_b200.config import LMCacheEngineConfig
    return LMCacheEngineConfig.from_legacy(chunk_size=CS, backend=backend, local_serde="cachegen",
                                           local_capacity_bytes=capacity, device_cache_bytes=device_cache)


def _engines(autorelease, fmt="vllm", device_cache=1 << 30, backend="cpu", backend_ref="cpu", capacity=None):
    from lmcache_b200.cache_engine import LMCacheEngine
    ref = autorelease(LMCacheEngine(_cfg(backend_ref, None, capacity), _meta(fmt)))
    eng = autorelease(LMCacheEngine(_cfg(backend, device_cache, capacity), _meta(fmt)))
    return ref, eng


def _bits(x):
    return x.contiguous().view(torch.int16)


def _seq(T, fmt="vllm", seed=0):
    g = torch.Generator(device="cuda").manual_seed(500 + seed)
    return torch.randint(0, 32000, (T,), device="cuda", generator=g), _kv(T, fmt, L=L, seed=seed)


def _same_retrieve(ref, eng, tokens):
    a, ma = ref.retrieve(tokens)
    b, mb = eng.retrieve(tokens)
    torch.cuda.synchronize()
    assert torch.equal(ma, mb) and int(ma.sum()) > 0
    assert torch.equal(_bits(_blob_of(a)), _bits(_blob_of(b)))
    return int(mb.sum())


def _keys(eng, tokens):
    be = eng.engine_
    return [be._dict_key(eng._make_key(h, eng.metadata.fmt)) for h in eng._prefix_hash(tokens)]


def _entries(eng):
    return [e for e in eng.engine_.dict.values() if e.rec is not None and e.error is None]


def _resident_bytes(be):
    torch.cuda.synchronize()
    be._dcache.release.sweep()
    return sum(e.rec.dev.cap for e in be.dict.values() if e.rec is not None and e.rec.dev is not None)


@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
def test_resident_retrieve_is_bit_identical_and_uploads_nothing(fmt, autorelease):
    ref, eng = _engines(autorelease, fmt)
    tokens, kv = _seq(2300, fmt, seed=1)
    ref.store(tokens, kv)
    eng.store(tokens, kv)
    be = eng.engine_
    n = len(_entries(eng))
    assert n == 9 and all(e.rec.dev is not None for e in _entries(eng))
    assert _same_retrieve(ref, eng, tokens) == 2300
    st = be.device_cache_stats()
    assert st["hits"] == n and st["promotions"] == 0
    assert all(e.rec.last_read is None for e in _entries(eng))          # no host block was read
    assert st["bytes_in_use"] == _resident_bytes(be) <= st["budget_bytes"]


def test_resident_paged_retrieve_is_bit_identical(autorelease):
    ref, eng = _engines(autorelease)
    T, bs, H, D = 1500, 16, 2, 128
    tokens, kv = _seq(T, seed=2)
    ref.store(tokens, kv)
    eng.store(tokens, kv)
    nblk = (T + bs - 1) // bs + 4
    slots = torch.randperm(nblk * bs, device="cuda")[:T]
    caches = [[(torch.zeros((nblk, bs, H, D), device="cuda", dtype=torch.bfloat16),
                torch.zeros((nblk, bs, H, D), device="cuda", dtype=torch.bfloat16)) for _ in range(L)] for _ in range(2)]
    ma = ref.retrieve_paged(tokens, caches[0], slots)
    mb = eng.retrieve_paged(tokens, caches[1], slots)
    torch.cuda.synchronize()
    assert torch.equal(ma, mb) and int(mb.sum()) == T
    for (k0, v0), (k1, v1) in zip(*caches):
        assert torch.equal(_bits(k0), _bits(k1)) and torch.equal(_bits(v0), _bits(v1))
    assert eng.engine_.device_cache_stats()["hits"] == len(_entries(eng))


def test_partial_residency_mixes_waves_and_stays_bit_identical(autorelease):
    from lmcache_b200.pipeline import wave_chunks_default
    from lmcache_b200.slab import block_bytes
    tokens, kv = _seq(4096, seed=3)
    probe, _ = _engines(autorelease, device_cache=None)
    probe.store(tokens, kv)
    seq = sum(block_bytes(e.rec.nbytes) for e in _entries(probe))
    budget = int(0.4 * seq)                       # about 6.4 of 16 chunks: the boundary falls inside the second wave
    ref, eng = _engines(autorelease, device_cache=budget)
    ref.store(tokens, kv)
    eng.store(tokens, kv)
    be = eng.engine_
    ents = [be.dict[k] for k in _keys(eng, tokens)]
    resident = [e.rec.dev is not None for e in ents]
    k = sum(resident)
    assert 0 < k < len(ents) and resident == [True] * k + [False] * (len(ents) - k)   # the store kept its head
    W = wave_chunks_default()
    assert any(0 < sum(resident[w:w + W]) < len(resident[w:w + W]) for w in range(0, len(ents), W))   # a mixed wave
    for rnd in (1, 2):
        assert _same_retrieve(ref, eng, tokens) == 4096
        st = be.device_cache_stats()
        assert st["hits"] == rnd * k                                # every resident chunk is served from the level
        assert [e.rec.dev is not None for e in ents] == resident    # promotions never evict the retrieve's own copies
    assert all((e.rec.last_read is None) == res for e, res in zip(ents, resident))   # only the tail was uploaded
    assert st["bytes_in_use"] <= st["budget_bytes"] and _resident_bytes(be) <= budget


def test_disk_tier_promotes_on_first_retrieve_then_hits(tmp_path, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    tokens, kv = _seq(2048, seed=4)
    backend = "file://" + str(tmp_path / "kv") + "/"
    ref = autorelease(LMCacheEngine(_cfg("cpu"), _meta()))
    ref.store(tokens, kv)
    first = LMCacheEngine(_cfg(backend, 1 << 30), _meta())
    first.store(tokens, kv)
    assert first.engine_.device_cache_stats()["bytes_in_use"] > 0
    first.close()
    eng = autorelease(LMCacheEngine(_cfg(backend, 1 << 30), _meta()))   # a restart: the level starts empty
    assert eng.engine_.device_cache_stats()["bytes_in_use"] == 0
    n = len(_entries(eng))
    assert _same_retrieve(ref, eng, tokens) == 2048
    st = eng.engine_.device_cache_stats()
    assert (st["hits"], st["promotions"]) == (0, n)
    assert _same_retrieve(ref, eng, tokens) == 2048
    st = eng.engine_.device_cache_stats()
    assert (st["hits"], st["promotions"]) == (n, n)


def test_tier_eviction_frees_the_device_copy(autorelease):
    from lmcache_b200.slab import block_bytes
    probe, _ = _engines(autorelease, device_cache=None)
    seqs = [_seq(2048, seed=10 + i) for i in range(3)]
    probe.store(*seqs[0])
    seq = sum(block_bytes(e.rec.nbytes) for e in _entries(probe))
    ref, eng = _engines(autorelease, capacity=int(1.5 * seq))
    for tok, kv in seqs:
        ref.store(tok, kv)
        eng.store(tok, kv)
    be = eng.engine_
    assert be.evicted > 0
    assert be.device_cache_stats()["bytes_in_use"] == _resident_bytes(be)  # no copy outlives its entry
    assert _same_retrieve(ref, eng, seqs[2][0]) == 2048


@pytest.mark.parametrize("tier", ["host", "disk"])
def test_overwrite_serves_the_new_kv(tier, tmp_path, autorelease):
    backend = "cpu" if tier == "host" else "file://" + str(tmp_path / "kv") + "/"
    ref, eng = _engines(autorelease, backend=backend)
    tokens, kv = _seq(1024, seed=5)
    _, kv2 = _seq(1024, seed=6)
    eng.store(tokens, kv)
    eng.retrieve(tokens)
    eng.store(tokens, kv2, skip_existing=False, blocking=False)    # overwrite while nothing waits for the old one
    ref.store(tokens, kv2)
    assert _same_retrieve(ref, eng, tokens) == 1024
    assert eng.engine_.device_cache_stats()["bytes_in_use"] == _resident_bytes(eng.engine_)


def test_a_container_larger_than_the_budget_is_not_cached(autorelease):
    ref, eng = _engines(autorelease, device_cache=4096)
    tokens, kv = _seq(1024, seed=7)
    ref.store(tokens, kv)
    eng.store(tokens, kv)
    st = eng.engine_.device_cache_stats()
    assert st["bytes_in_use"] == 0 and st["not_cached"] >= len(_entries(eng))
    assert _same_retrieve(ref, eng, tokens) == 1024
    assert eng.engine_.device_cache_stats()["bytes_in_use"] == 0


@pytest.mark.parametrize("tier", ["host", "disk"])
@pytest.mark.parametrize("budget", ["all", "half"])
def test_layerwise_retrieve_from_the_level(tier, budget, tmp_path, autorelease):
    from lmcache_b200.slab import block_bytes
    tokens, kv = _seq(3000, seed=8)
    backend = "cpu" if tier == "host" else "file://" + str(tmp_path / "kv") + "/"
    probe, _ = _engines(autorelease, device_cache=None)
    probe.store(tokens, kv)
    seq = sum(block_bytes(e.rec.nbytes) for e in _entries(probe))
    _, eng = _engines(autorelease, device_cache=seq if budget == "all" else seq // 2, backend=backend)
    eng.store(tokens, kv)
    ref, ref_mask = eng.retrieve(tokens)
    torch.cuda.synchronize()
    hits0 = eng.engine_.device_cache_stats()["hits"]
    resident = sum(eng.engine_.dict[k].rec.dev is not None for k in _keys(eng, tokens))
    r = eng.retrieve_layerwise(tokens)
    assert r.num_layers == L and torch.equal(r.ret_mask, ref_mask)
    for layer in range(L):
        ev = r._upload.ready(layer)
        assert isinstance(ev, torch.cuda.Event)
        ev.synchronize()
        for j in range(2):
            assert torch.equal(_bits(r.kv[layer][j]), _bits(ref[layer][j]))
    hits = eng.engine_.device_cache_stats()["hits"] - hits0
    assert hits == resident > 0 and (budget == "half" or resident == 12)
    # paged form over the same level
    T, bs, H, D = 3000, 16, 2, 128
    nblk = (T + bs - 1) // bs + 4
    slots = torch.randperm(nblk * bs, device="cuda")[:T]
    caches = [[(torch.zeros((nblk, bs, H, D), device="cuda", dtype=torch.bfloat16),
                torch.zeros((nblk, bs, H, D), device="cuda", dtype=torch.bfloat16)) for _ in range(L)] for _ in range(2)]
    want = eng.retrieve_paged(tokens, caches[0], slots)
    r = eng.retrieve_paged_layerwise(tokens, caches[1], slots)
    r.synchronize()
    torch.cuda.synchronize()
    assert torch.equal(r.ret_mask, want)
    for (k0, v0), (k1, v1) in zip(*caches):
        assert torch.equal(_bits(k0), _bits(k1)) and torch.equal(_bits(v0), _bits(v1))


@pytest.mark.parametrize("tier", ["host", "disk"])
def test_layerwise_store_fills_the_level_with_the_landed_bytes(tier, tmp_path, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    backend = "cpu" if tier == "host" else "file://" + str(tmp_path / "kv") + "/"
    eng = autorelease(LMCacheEngine(_cfg(backend, 1 << 30), _meta()))
    tokens, kv = _seq(2300, seed=9)
    h = eng.store_layerwise(tokens, kv)
    for layer in range(L):
        h.save_layer(layer)
    h.finish()
    be = eng.engine_
    for e in be.dict.values():
        e.ready.wait()
    ents = _entries(eng)
    assert len(ents) == 9 and all(e.rec.dev is not None for e in ents)
    pool = be._dcache.pool.buf
    torch.cuda.synchronize()
    for e in ents:
        if e.rec.blk is not None:
            want = bytes(e.rec.blk.view())[:e.rec.nbytes]
        else:
            with open(e.path, "rb") as f:
                want = f.read()
        got = pool[e.rec.dev.offset:e.rec.dev.offset + e.rec.nbytes].cpu().numpy().tobytes()
        assert got == want
    ref = autorelease(LMCacheEngine(_cfg("cpu"), _meta()))
    ref.store(tokens, kv)
    assert _same_retrieve(ref, eng, tokens) == 2300
