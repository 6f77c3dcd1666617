"""CPU: the eviction order of the bounded CacheGen tiers (lmcache_b200/eviction.py), the slab's byte budget, and the
local_capacity_bytes configuration key."""
import random

import pytest

from lmcache_b200.eviction import PrefixLRU
from lmcache_b200.slab import PinnedSlab, SlabFull
from test_slab_cpu import _FakeSeg


def _drain(order, eligible=lambda k: True):
    out = []
    while True:
        k = order.victim(eligible)
        if k is None:
            return out
        order.discard(k)
        out.append(k)


# ---------------------------------------------------------------------------------------------- policy
def test_victims_come_out_in_tick_then_tail_first_order():
    o = PrefixLRU()
    o.touch(["a0", "a1", "a2"])
    o.touch(["b0", "b1"])
    o.touch(["a0", "a1"])                        # a retrieve of A's first two chunks
    assert o.stamp("a2") == (1, -2) and o.stamp("a1") == (3, -1) and o.stamp("b0") == (2, 0)
    assert _drain(o) == ["a2", "b1", "b0", "a1", "a0"]
    assert len(o) == 0 and o.victim(lambda k: True) is None


def test_ineligible_entries_are_never_chosen_and_keep_their_place():
    o = PrefixLRU()
    o.touch(["p0", "p1"])                        # pinned by a retrieve
    o.touch(["n0"])                              # not landed yet
    o.touch(["s0", "s1"])                        # belongs to the store that is landing
    o.touch(["x0", "x1"])
    blocked = {"p0", "p1", "n0", "s0", "s1"}
    assert _drain(o, lambda k: k not in blocked) == ["x1", "x0"]
    assert o.victim(lambda k: k not in blocked) is None
    assert _drain(o) == ["p1", "p0", "n0", "s1", "s0"]   # once unblocked, in their original order


def test_heap_stays_bounded_under_repeated_touches():
    o = PrefixLRU()
    keys = [f"k{i}" for i in range(8)]
    for _ in range(10000):
        o.touch(keys)
    assert len(o._heap) <= 2 * len(keys) + 64 + len(keys)
    assert _drain(o) == keys[::-1]


class _ModelTier:
    """The bounded tier's bookkeeping without the GPU: the same policy, the same eligibility rule (never a chunk of the
    store that is landing, nor one touched since the touch that preceded the store), drops behind the first chunk that
    does not fit; chunk sizes in abstract units."""

    def __init__(self, capacity):
        self.capacity = capacity
        self.order = PrefixLRU()
        self.held = {}                           # key -> (size, store id)
        self.used = 0

    def contains(self, k):
        return k in self.held

    def touch(self, keys):
        self.order.touch([k for k in keys if k in self.held])

    def put(self, keys, sizes, store):
        """put_kv_chunks + its sink: insert, stamp as one call, then land chunk by chunk"""
        since = self.order.tick
        for k in keys:
            if k in self.held:                   # overwrite: the old container leaves
                self.used -= self.held.pop(k)[0]
        dropped = False
        landed = []
        for k in keys:
            size = sizes[k]
            while not dropped and self.used + size > self.capacity:
                v = self.order.victim(lambda v: v not in self.held or (self.held[v][1] != store and
                                                                       self.order.stamp(v)[0] < since))
                if v is None:
                    dropped = True
                    break
                self.order.discard(v)
                if v in self.held:
                    self.used -= self.held.pop(v)[0]
            if dropped:
                break
            self.held[k] = (size, store)
            self.used += size
            landed.append(k)
        self.touch(landed)
        assert self.used <= self.capacity


def _engine_store(tier, chain, sizes, store, skip_existing):
    start = 0
    if skip_existing:
        start = len(chain)
        for i, k in enumerate(chain):
            if not tier.contains(k):
                start = i
                break
    tier.touch(chain[:start])
    if start < len(chain):
        tier.put(chain[start:], sizes, store)
        tier.touch(chain)


def _engine_retrieve(tier, chain, skip):
    n = 0
    for k in chain[skip:]:
        if not tier.contains(k):
            break
        n += 1
    tier.touch(chain[:skip + n])
    return n


@pytest.mark.parametrize("seed", range(6))
def test_random_operations_keep_every_chain_a_prefix(seed):
    rng = random.Random(seed)
    tier = _ModelTier(capacity=40)
    sizes = {}
    chains = []

    def new_chain():
        if chains and rng.random() < 0.5:             # shares a prefix with an earlier chain
            base = rng.choice(chains)
            chain = base[:rng.randint(1, len(base))]
        else:
            chain = []
        chain = chain + [f"c{len(chains)}_{i}" for i in range(rng.randint(1, 10))]
        for k in chain:
            sizes.setdefault(k, rng.randint(1, 4))
        chains.append(chain)
        return chain

    for step in range(400):
        r = rng.random()
        if r < 0.4 or not chains:
            _engine_store(tier, new_chain(), sizes, step, skip_existing=rng.random() < 0.8)
        elif r < 0.6:
            _engine_store(tier, rng.choice(chains), sizes, step, skip_existing=rng.random() < 0.8)
        else:
            chain = rng.choice(chains)
            _engine_retrieve(tier, chain, rng.randint(0, len(chain) - 1))
        for chain in chains:
            have = [tier.contains(k) for k in chain]
            assert have == sorted(have, reverse=True), (step, chain, have)


def test_a_chain_larger_than_the_capacity_keeps_its_longest_fitting_prefix():
    tier = _ModelTier(capacity=10)
    _engine_store(tier, ["o0", "o1"], {"o0": 3, "o1": 3}, 0, True)
    chain = [f"k{i}" for i in range(8)]
    _engine_store(tier, chain, {k: 3 for k in chain}, 1, True)
    assert [tier.contains(k) for k in chain] == [True] * 3 + [False] * 5
    assert not tier.contains("o0") and not tier.contains("o1")


# ---------------------------------------------------------------------------------------------- slab budget
def test_budgeted_slab_never_exceeds_its_segments():
    rng = random.Random(1)
    slab = PinnedSlab(segment_bytes=1 << 16, alloc_fn=_FakeSeg, max_segments=3)
    live, refused = [], 0
    for _ in range(3000):
        if live and rng.random() < 0.4:
            live.pop(rng.randrange(len(live))).free()
        else:
            try:
                live.append(slab.alloc(rng.randint(1, 20000)))
            except SlabFull:
                refused += 1
        assert slab.stats()[0] <= 3 and slab.stats()[1] <= 3 << 16
    assert refused > 0
    assert slab.stats()[2] == sum(b.cap for b in live)


def test_alloc_beyond_the_budget_fails_without_growing():
    slab = PinnedSlab(segment_bytes=1 << 16, alloc_fn=_FakeSeg, max_segments=2)
    a = slab.alloc(60000)
    b = slab.alloc(60000)
    assert slab.stats()[0] == 2
    with pytest.raises(SlabFull):
        slab.alloc(10000)                        # no extent left and no third segment
    with pytest.raises(SlabFull):
        slab.alloc(1 << 17)                      # larger than a segment: never gets its own under a budget
    assert slab.stats()[0] == 2
    a.free()
    assert slab.alloc(10000).seg == a.seg        # the freed extent serves it
    b.free()
    slab.reserve(1 << 20)                        # reserve is capped by the budget as well
    assert slab.stats()[0] == 2
    unbounded = PinnedSlab(segment_bytes=1 << 16, alloc_fn=_FakeSeg)
    unbounded.alloc(1 << 17)
    assert unbounded.stats()[0] == 1


# ---------------------------------------------------------------------------------------------- configuration
def test_capacity_config_key_yaml_and_constructors(tmp_path):
    from lmcache_b200.config import LMCacheEngineConfig
    p = tmp_path / "cfg.yaml"
    p.write_text("chunk_size: 256\nlocal_device: cpu\nremote_url: null\nlocal_serde: cachegen\n"
                 "local_capacity_bytes: 1073741824\n")
    assert LMCacheEngineConfig.from_file(str(p)).local_capacity_bytes == 1 << 30
    p.write_text("chunk_size: 256\nlocal_device: cpu\nremote_url: null\n")
    assert LMCacheEngineConfig.from_file(str(p)).local_capacity_bytes is None
    assert LMCacheEngineConfig.from_defaults(local_capacity_bytes=5).local_capacity_bytes == 5
    assert LMCacheEngineConfig.from_legacy(backend="cpu", local_serde="cachegen",
                                           local_capacity_bytes=7).local_capacity_bytes == 7
    assert LMCacheEngineConfig.from_legacy(backend="cpu").local_capacity_bytes is None
    for bad in (0, -1, 1.5, True, "1024"):
        with pytest.raises(ValueError):
            LMCacheEngineConfig.from_legacy(backend="cpu", local_serde="cachegen", local_capacity_bytes=bad)
    p.write_text("chunk_size: 256\nlocal_device: cpu\nlocal_capacity_bytes: -3\n")
    with pytest.raises(ValueError):
        LMCacheEngineConfig.from_file(str(p))


@pytest.mark.parametrize("local,remote,serde", [("cpu", None, None), ("cuda", None, None), ("cuda", None, "cachegen"),
                                                (None, "lm://127.0.0.1:1", None),
                                                ("cpu", "lm://127.0.0.1:1", None),
                                                ("cuda", "lm://127.0.0.1:1", "cachegen")])
def test_capacity_is_rejected_where_no_cachegen_tier_honours_it(local, remote, serde):
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    from lmcache_b200.storage_backend import CreateStorageBackend
    cfg = LMCacheEngineConfig(256, local, remote, "cachegen", False, False, serde, local_capacity_bytes=1 << 30)
    with pytest.raises(ValueError, match="local_capacity_bytes"):
        CreateStorageBackend(cfg, LMCacheEngineMetadata("lmsys/longchat-7b-16k", 1, 0, "vllm", "bfloat16"))
