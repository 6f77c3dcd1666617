"""CPU: the device level of the CacheGen tiers (config.device_cache_bytes) -- its configuration key, where the backend
factory rejects it, and the bookkeeping of lmcache_b200.device_cache.DeviceCache driven with plain memory and stand-in
events."""
import random

import pytest

from lmcache_b200.device_cache import DeviceCache
from lmcache_b200.slab import block_bytes
from test_slab_cpu import _FakeSeg

MODEL = "lmsys/longchat-7b-16k"


# ---------------------------------------------------------------------------------------------- configuration
def test_device_cache_config_key_yaml_and_constructors(tmp_path):
    from lmcache_b200.config import LMCacheEngineConfig
    p = tmp_path / "cfg.yaml"
    p.write_text("chunk_size: 256\nlocal_device: cpu\nremote_url: null\nlocal_serde: cachegen\n"
                 "device_cache_bytes: 2147483648\n")
    assert LMCacheEngineConfig.from_file(str(p)).device_cache_bytes == 2 << 30
    p.write_text("chunk_size: 256\nlocal_device: cpu\nremote_url: null\n")
    assert LMCacheEngineConfig.from_file(str(p)).device_cache_bytes is None
    assert LMCacheEngineConfig.from_defaults(device_cache_bytes=5).device_cache_bytes == 5
    assert LMCacheEngineConfig.from_legacy(backend="cpu", local_serde="cachegen",
                                           device_cache_bytes=7).device_cache_bytes == 7
    assert LMCacheEngineConfig.from_legacy(backend="cpu").device_cache_bytes is None
    for bad in (0, -1, 1.5, True, "1024"):
        with pytest.raises(ValueError, match="device cache"):
            LMCacheEngineConfig.from_legacy(backend="cpu", local_serde="cachegen", device_cache_bytes=bad)
        with pytest.raises(ValueError, match="device cache"):
            LMCacheEngineConfig.from_defaults(device_cache_bytes=bad)
    p.write_text("chunk_size: 256\nlocal_device: cpu\ndevice_cache_bytes: -3\n")
    with pytest.raises(ValueError):
        LMCacheEngineConfig.from_file(str(p))


@pytest.mark.parametrize("local,remote,serde", [("cpu", None, None), ("cuda", None, None), ("cuda", None, "cachegen"),
                                                (None, "lm://127.0.0.1:1", None),
                                                ("cpu", "lm://127.0.0.1:1", None),
                                                ("cuda", "lm://127.0.0.1:1", "cachegen")])
def test_device_cache_is_rejected_where_no_cachegen_tier_exists(local, remote, serde):
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    from lmcache_b200.storage_backend import CreateStorageBackend
    cfg = LMCacheEngineConfig(256, local, remote, "cachegen", False, False, serde, device_cache_bytes=1 << 30)
    with pytest.raises(ValueError, match="device_cache_bytes"):
        CreateStorageBackend(cfg, LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16"))


@pytest.mark.parametrize("local", ["cpu", "/tmp/kv/"])
def test_hybrid_hands_the_key_to_its_local_tier(local, monkeypatch):
    import lmcache_b200.storage_backend as sb
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    from lmcache_b200.storage_backend.hybrid_backend import LMCHybridBackend
    made = []
    monkeypatch.setattr(sb, "CreateStorageBackend", lambda cfg, meta: made.append(cfg) or object())
    cfg = LMCacheEngineConfig(256, local, "lm://127.0.0.1:1", "cachegen", False, False, "cachegen",
                              local_capacity_bytes=3 << 30, device_cache_bytes=1 << 30)
    LMCHybridBackend(cfg, LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16"))
    local_cfg, remote_cfg = made
    assert (local_cfg.local_device, local_cfg.remote_url) == (local, None)
    assert local_cfg.device_cache_bytes == 1 << 30 and local_cfg.local_capacity_bytes == 3 << 30
    assert remote_cfg.local_device is None and remote_cfg.device_cache_bytes is None


# ---------------------------------------------------------------------------------------------- bookkeeping
class _Ev:
    def __init__(self, done=False):
        self.done = done

    def query(self):
        return self.done

    def synchronize(self):
        self.done = True


class _Rec:
    def __init__(self, nbytes):
        self.nbytes = nbytes
        self.dev = self.dev_ready = self.dev_read = None


class _Entry:
    """the tier's entry as the level sees it"""

    def __init__(self, nbytes):
        self.rec = _Rec(nbytes)
        self.pins = 0


def _fill(cache, entries, ready=None):
    blocks = [cache.alloc(e.rec.nbytes) for e in entries]
    cache.attach(entries, blocks, ready)
    return blocks


def _in_use(cache, entries):
    return sum(e.rec.dev.cap for e in entries if e.rec.dev is not None)


def test_fills_evict_the_coldest_copy_tail_first_and_stay_within_the_budget():
    cache = DeviceCache(10 * 256, alloc_fn=_FakeSeg)
    a = [_Entry(256) for _ in range(4)]
    b = [_Entry(256) for _ in range(4)]
    _fill(cache, a)
    _fill(cache, b)
    cache.touch(a)                                   # a retrieve of chain a: b is now the colder chain
    c = [_Entry(256) for _ in range(4)]
    got = _fill(cache, c)
    assert all(blk is not None for blk in got)
    assert [e.rec.dev is not None for e in b] == [True, True, False, False]   # b's tail went first
    assert all(e.rec.dev is not None for e in a)
    assert cache.evictions == 2 and cache.skipped == 0
    assert cache.slab.bytes_in_use == _in_use(cache, a + b + c) <= cache.budget
    offs = sorted((e.rec.dev.offset, e.rec.dev.cap) for e in a + b + c if e.rec.dev is not None)
    assert all(o + n <= p for (o, n), (p, _) in zip(offs, offs[1:]))         # no two copies overlap
    assert offs[-1][0] + offs[-1][1] <= cache.budget                         # the read slack stays outside every block


def test_pinned_copies_and_unfinished_fills_or_decodes_are_never_victims():
    cache = DeviceCache(4 * 256, alloc_fn=_FakeSeg)
    ents = [_Entry(256) for _ in range(4)]
    _fill(cache, ents[:1])
    _fill(cache, ents[1:2], ready=_Ev(False))        # a promotion whose copy has not run
    _fill(cache, ents[2:4])
    ents[2].pins = 1                                 # a retrieve between lookup and enqueue
    ents[3].rec.dev_read = _Ev(False)                # a decode still reading it
    cache.touch(ents)
    new = _Entry(256)
    got = _fill(cache, [new])[0]
    assert got is not None and ents[0].rec.dev is None and cache.evictions == 1
    assert all(e.rec.dev is not None for e in ents[1:])
    new.pins = 1
    assert _fill(cache, [_Entry(256)])[0] is None    # everything else is busy: not cached, no wait
    assert cache.skipped == 1
    ents[1].rec.dev_ready.done = True                # the fill completed: now a victim
    assert _fill(cache, [_Entry(256)])[0] is not None and ents[1].rec.dev is None


def test_a_full_pool_or_an_oversized_container_is_skipped_not_waited_for():
    cache = DeviceCache(4 * 256, alloc_fn=_FakeSeg)
    assert cache.alloc(4 * 256 + 1) is None and cache.skipped == 1          # larger than the budget
    assert cache.pool is None                                                # ... and nothing was allocated
    ents = [_Entry(2 * 256) for _ in range(2)]
    _fill(cache, ents)
    for e in ents:
        e.pins = 1
    assert _fill(cache, [_Entry(256)])[0] is None and cache.skipped == 2     # every copy is pinned
    assert cache.slab.bytes_in_use == 4 * 256 and cache.evictions == 0
    ents[1].pins = 0
    assert _fill(cache, [_Entry(256)])[0] is not None and ents[1].rec.dev is None


def test_tier_drop_frees_after_the_last_reader():
    cache = DeviceCache(4 * 256, alloc_fn=_FakeSeg)
    ents = [_Entry(2 * 256) for _ in range(2)]
    _fill(cache, ents)
    reader = _Ev(False)
    ents[0].rec.dev_read = reader
    cache.drop(ents[0])                              # the tier evicted or overwrote the entry
    assert ents[0].rec.dev is None and ents[0] not in cache.order
    ents[1].pins = 1
    assert _fill(cache, [_Entry(2 * 256)])[0] is None                       # its block is still being read
    assert cache.slab.bytes_in_use == 4 * 256
    reader.done = True
    late = _Entry(2 * 256)
    assert _fill(cache, [late])[0] is not None       # freed once the decode completed
    assert ents[1].rec.dev is not None and cache.evictions == 0


@pytest.mark.parametrize("seed", range(4))
def test_random_fills_touches_and_drops_keep_the_invariants(seed):
    rng = random.Random(seed)
    budget = 64 * 256
    cache = DeviceCache(budget, alloc_fn=_FakeSeg)
    live = []
    for step in range(1500):
        r = rng.random()
        if r < 0.45:
            ents = [_Entry(rng.randint(1, 6 * 256)) for _ in range(rng.randint(1, 4))]
            ready = _Ev(rng.random() < 0.5) if rng.random() < 0.5 else None
            _fill(cache, ents, ready)
            live += ents
        elif r < 0.6 and live:
            cache.touch(rng.sample(live, min(len(live), 5)))
        elif r < 0.7 and live:
            e = rng.choice(live)
            if not e.pins:
                live.remove(e)
                cache.drop(e)
        elif r < 0.85 and live:
            e = rng.choice(live)
            e.pins = 1 - e.pins
        elif live:
            e = rng.choice(live)
            if e.rec.dev_ready is not None:
                e.rec.dev_ready.done = True
            e.rec.dev_read = _Ev(rng.random() < 0.7)
        res = [e for e in live if e.rec.dev is not None]
        assert cache.slab.bytes_in_use <= budget
        held = sum(b.cap for _, blocks in cache.release._held for b in blocks)
        assert cache.slab.bytes_in_use == sum(e.rec.dev.cap for e in res) + held
        for e in res:
            assert e in cache.order
            assert e.rec.dev.offset + block_bytes(e.rec.nbytes) <= budget
    assert cache.evictions > 0 and cache.skipped > 0
    st = cache.stats()
    assert st["budget_bytes"] == budget and st["bytes_in_use"] == cache.slab.bytes_in_use


def test_a_store_keeps_its_own_copies_and_its_chain_order():
    """keep= protects the filling call's copies; copies stamped as parts of one call keep chain order"""
    cache = DeviceCache(6 * 256, alloc_fn=_FakeSeg)
    old = [_Entry(256) for _ in range(2)]
    _fill(cache, old)
    mine = [_Entry(256) for _ in range(8)]
    tick = cache.order.new_tick()
    got = []
    for c0 in range(0, 8, 2):                        # waves of two chunks, one tick for the whole store
        wave = mine[c0:c0 + 2]
        blocks = [cache.alloc(e.rec.nbytes, keep=lambda h: h in mine) for e in wave]
        cache.attach(wave, blocks, at=(tick, c0))
        got += blocks
    assert [b is not None for b in got] == [True] * 6 + [False] * 2          # the older copies went, never its own
    assert all(e.rec.dev is None for e in old) and cache.evictions == 2
    assert cache.order.victim(lambda h: True) is mine[5]                     # tail first within the store
    newer = [_Entry(256) for _ in range(2)]
    _fill(cache, newer)                              # a later call evicts the store's tail, its head stays
    assert [e.rec.dev is not None for e in mine[:6]] == [True] * 4 + [False] * 2


def test_touch_at_stamps_parts_of_one_call():
    from lmcache_b200.eviction import PrefixLRU
    o = PrefixLRU()
    t = o.new_tick()
    o.touch_at(["a0", "a1"], t)
    o.touch(["b0"])
    o.touch_at(["a2", "a3"], t, 2)
    assert o.stamp("a3") == (t, -3) and o.tick == t + 1
    out = []
    while (k := o.victim(lambda k: True)) is not None:
        o.discard(k)
        out.append(k)
    assert out == ["a3", "a2", "a1", "a0", "b0"]
