"""GPU: capacity-bounded CacheGen tiers (local_capacity_bytes) behind LMCacheEngine.store()/retrieve().  Whatever a
bounded tier still returns must be the reference's own decode of the stored chunks bit for bit (tests/ref_torch.py, as in
test_gpu_host_tier.py), and what it keeps must be a prefix of every chain."""
import math
import os
import socket
import subprocess
import sys
import threading
import time

import pytest
import torch

from test_gpu_host_tier import MODEL, _blob_of, _kv, _meta, _want

pytestmark = pytest.mark.gpu
CS, T = 256, 2048                                      # 8 chunks per sequence (two store waves of 4)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(capacity, backend="cpu"):
    from lmcache_b200.config import LMCacheEngineConfig
    return LMCacheEngineConfig.from_legacy(chunk_size=CS, backend=backend, local_serde="cachegen",
                                           local_capacity_bytes=capacity)


def _seq(seed, n=T):
    g = torch.Generator(device="cuda").manual_seed(1000 + seed)
    return torch.randint(0, 32000, (n,), device="cuda", generator=g), _kv(n, "vllm", seed=seed)


_SEQ_BYTES = {}


def _seq_bytes():
    """(slab bytes, container bytes) one sequence takes in an unbounded tier"""
    if not _SEQ_BYTES:
        from lmcache_b200.cache_engine import LMCacheEngine
        eng = LMCacheEngine(_cfg(None), _meta())
        eng.store(*_seq(0))
        ents = list(eng.engine_.dict.values())
        _SEQ_BYTES["v"] = (sum(e.blk.cap for e in ents), sum(e.nbytes for e in ents))
        eng.close()
    return _SEQ_BYTES["v"]


def _keys(engine, tokens):
    return [engine._make_key(h, "vllm") for h in engine._prefix_hash(tokens)]


def _held(engine, tokens):
    have = [engine.engine_.contains(k) for k in _keys(engine, tokens)]
    assert have == sorted(have, reverse=True), f"not a prefix: {have}"     # contains is a prefix of the chain
    return sum(have)


def _check_retrieve(engine, tokens, kv, full=False):
    """retrieve; the ret_mask is a prefix of whole chunks and the KV it marks is the reference decode, bit for bit"""
    ret, mask = engine.retrieve(tokens)
    got = int(mask.sum())
    assert bool(mask[:got].all()) and not bool(mask[got:].any())
    assert got % CS == 0 or got == len(tokens)
    if full:
        assert got == len(tokens)
    if got:
        want = _want(kv, "vllm", CS, got)
        assert torch.equal(_blob_of(ret).view(torch.int16), want.view(torch.int16))
    return got // CS if got < len(tokens) else -(-got // CS)


def _check_bound(be, capacity):
    seg = be.slab.segment_bytes
    assert be.host_bytes() <= capacity
    assert be.slab.stats()[1] <= math.ceil(capacity / seg) * seg


def test_bounded_host_tier_keeps_newest_and_prefixes(autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    cap = int(2.5 * _seq_bytes()[0])
    engine = autorelease(LMCacheEngine(_cfg(cap), _meta()))
    be = engine.engine_
    seqs = [_seq(i) for i in range(3)]
    for tok, kv in seqs:
        engine.store(tok, kv)
        _check_bound(be, cap)
    assert be.evicted > 0
    assert _check_retrieve(engine, *seqs[2], full=True) == T // CS
    held_a = _held(engine, seqs[0][0])
    assert held_a < T // CS
    assert _check_retrieve(engine, *seqs[0]) == held_a
    for tok, _ in seqs[1:]:
        _held(engine, tok)


def test_retrieve_makes_a_sequence_recent(autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    cap = int(2.5 * _seq_bytes()[0])
    engine = autorelease(LMCacheEngine(_cfg(cap), _meta()))
    (ta, ka), (tb, kb), (tc, kc) = (_seq(i) for i in (10, 11, 12))
    engine.store(ta, ka)
    engine.store(tb, kb)
    _check_retrieve(engine, ta, ka, full=True)
    engine.store(tc, kc)
    assert engine.engine_.evicted > 0
    assert _held(engine, tb) < T // CS                     # B went first ...
    assert _held(engine, ta) == T // CS                    # ... and none of A
    _check_retrieve(engine, ta, ka, full=True)


def test_stored_prefix_outlives_the_extension_tail(autorelease):
    """A, then A + an extension (skip_existing matches A): the engine touches A's chunks with the whole chain, so under
    pressure the extension's tail goes before any of A"""
    from lmcache_b200.cache_engine import LMCacheEngine
    cap = int(2.2 * _seq_bytes()[0])
    engine = autorelease(LMCacheEngine(_cfg(cap), _meta()))
    tok, kv = _seq(20)
    half = T // 2
    engine.store(tok[:half], tuple((k[:half], v[:half]) for k, v in kv))
    engine.store(tok, kv)
    assert _held(engine, tok) == T // CS
    be = engine.engine_
    stamps = [be._order.stamp(k) for k in _keys(engine, tok)]
    assert stamps == sorted(stamps, reverse=True) and len(set(s[0] for s in stamps)) == 1   # one call, tail first
    for i in range(6):                                     # half-length sequences: ~0.5 of A + extension each
        engine.store(*_seq(21 + i, half))
        n = _held(engine, tok)                             # asserts that what is left of the chain is a prefix
        if n < T // CS:
            break
    else:
        pytest.fail("no pressure reached the extension")
    assert _check_retrieve(engine, tok, kv) == n


def test_store_larger_than_the_capacity_keeps_longest_prefix(autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    cap = int(0.5 * _seq_bytes()[0])
    engine = autorelease(LMCacheEngine(_cfg(cap), _meta()))
    tok, kv = _seq(30)
    engine.store(tok, kv)                                  # returns normally: the tail is dropped, not an error
    _check_bound(engine.engine_, cap)
    n = _held(engine, tok)
    assert 1 <= n < T // CS
    assert _check_retrieve(engine, tok, kv) == n


def test_concurrent_store_under_pressure_and_retrieve(autorelease):
    """one thread stores fresh sequences (every store evicts) while another retrieves one sequence: pins keep each
    container's block alive until its upload is enqueued, so every reported prefix decodes bit-exact"""
    from lmcache_b200.cache_engine import LMCacheEngine
    cap = int(2.5 * _seq_bytes()[0])
    engine = autorelease(LMCacheEngine(_cfg(cap), _meta()))
    tok0, kv0 = _seq(40)
    engine.store(tok0, kv0)
    fresh = [_seq(41 + i) for i in range(6)]
    torch.cuda.synchronize()
    errs = []

    def writer():
        try:
            torch.cuda.set_device(0)
            for i, (tok, kv) in enumerate(fresh):
                engine.store(tok, kv, blocking=(i % 2 == 0))
        except Exception as e:      # noqa: BLE001
            errs.append(e)

    th = threading.Thread(target=writer)
    th.start()
    for _ in range(8):
        _check_retrieve(engine, tok0, kv0)
    th.join()
    assert not errs and engine.engine_.evicted > 0
    _check_retrieve(engine, *fresh[-1], full=True)


def test_bounded_disk_tier_and_restart_with_smaller_capacity(tmp_path, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    d = str(tmp_path / "kvdisk") + "/"
    per_seq = _seq_bytes()[1]

    def disk_bytes():
        return sum(os.path.getsize(d + f) for f in os.listdir(d) if f.endswith(".b2kv"))

    cap = int(2.5 * per_seq)
    engine = LMCacheEngine(_cfg(cap, "file://" + d), _meta())
    seqs = [_seq(50 + i) for i in range(3)]
    for tok, kv in seqs:
        engine.store(tok, kv)
        assert disk_bytes() <= cap
        time.sleep(0.05)                                  # the next sequence's files are strictly newer (mtime)
    assert engine.engine_.evicted > 0
    _check_retrieve(engine, *seqs[2], full=True)
    engine.close()
    small = int(1.3 * per_seq)
    engine2 = autorelease(LMCacheEngine(_cfg(small, "file://" + d), _meta()))
    assert disk_bytes() <= small
    assert _held(engine2, seqs[0][0]) == 0
    _check_retrieve(engine2, *seqs[2], full=True)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.fixture(scope="module")
def lmserver():
    port = _free_port()
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    proc = subprocess.Popen([sys.executable, "-m", "lmcache_b200.server", "127.0.0.1", str(port)], env=env)
    for _ in range(100):
        try:
            socket.create_connection(("127.0.0.1", port), timeout=0.2).close()
            break
        except OSError:
            time.sleep(0.1)
    yield f"lm://127.0.0.1:{port}"
    proc.terminate()
    proc.wait()


def test_hybrid_serves_locally_evicted_chunks_from_remote(lmserver, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig
    cap = int(2.5 * _seq_bytes()[0])
    cfg = LMCacheEngineConfig(CS, "cpu", lmserver, "cachegen", False, False, "cachegen", local_capacity_bytes=cap)
    engine = autorelease(LMCacheEngine(cfg, _meta()))
    local = engine.engine_.local_store
    assert local.capacity == cap
    seqs = [_seq(60 + i) for i in range(3)]
    for tok, kv in seqs:
        engine.store(tok, kv)
    keys = _keys(engine, seqs[0][0])
    have = [local.contains(k) for k in keys]
    assert have == sorted(have, reverse=True) and not all(have)
    _check_retrieve(engine, *seqs[0], full=True)          # local prefix + remote rest, one blob
