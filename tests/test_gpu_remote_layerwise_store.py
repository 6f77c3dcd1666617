"""GPU: layer-by-layer store (store_paged_layerwise / store_layerwise) on the lm:// remote and hybrid tiers.  Whatever
the server and the local tier hold after save_layer for every layer and finish() is compared byte for byte with what
store_paged() / store() put there for the same KV under other tokens, and every retrieve bit for bit.  In the hybrids
whose parts keep the same containers, the encode is counted: one per store."""
import os
import socket
import subprocess
import sys
import time

import pytest
import torch

from test_gpu_host_tier import MODEL
from test_gpu_paged_layouts import _layout
from test_gpu_remote_layerwise import _Native

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L, H, D, CS, BS = 4, 2, 128, 256, 16


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


_TOK = [0]


def _tokens(T):
    """tokens no other store of the module used: distinct keys on the shared server"""
    _TOK[0] += 1
    return torch.arange(T, device="cuda") + 100000 * _TOK[0]


def _engine(autorelease, url, serde="cachegen", local=None, local_serde=None, pipelined=False, cs=CS, mla=False,
            rank=0, capacity=None, cg=None):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    cfg = LMCacheEngineConfig(cs, local, url, serde, pipelined, False, local_serde, capacity, cachegen_config=cg)
    return autorelease(LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, 2 if mla else 1, rank, "vllm", "bfloat16", mla)))


def _kv(T, dtype, seed, mla=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    shape = (L, T, D) if mla else (L, 2, T, H, D)
    return torch.randn(shape, device="cuda", generator=g).to(dtype)


def _paged(kv, slots, kind="flash", mla=False):
    """caches of every layer holding kv's token i at slots[i]"""
    T = kv.shape[1] if mla else kv.shape[2]
    nb = (int(slots.max()) + 1 + BS - 1) // BS + 2
    if mla:
        out = []
        for l in range(L):
            c = torch.zeros(nb, BS, D, dtype=kv.dtype, device="cuda")
            c.view(-1, D)[slots] = kv[l]
            out.append(c)
        return out
    out = []
    for l in range(L):
        rows = [torch.zeros(nb * BS, H, D, dtype=kv.dtype, device="cuda") for _ in range(2)]
        for i in range(2):
            rows[i].view(torch.uint8 if kv.element_size() == 1 else torch.int16)[slots] = \
                kv[l, i].view(torch.uint8 if kv.element_size() == 1 else torch.int16)
        out.append(_layout(kind, rows, nb, BS, H, D))
    assert T == len(slots)
    return out


def _slots(T, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randperm(((T + BS - 1) // BS + 4) * BS, device="cuda", generator=g)[:T]


def _remote_of(eng):
    return getattr(eng.engine_, "remote_store", eng.engine_)


def _server_bytes(url, eng, tokens):
    """the raw bytes of a GET of every chunk key of `tokens` (None for a miss)"""
    from lmcache_b200.storage_backend.connector import CreateConnector
    c = CreateConnector(url)
    try:
        keys = [eng._make_key(h, "vllm") for h in eng._prefix_hash(tokens)]
        out = []
        for k in keys:
            b = c.get(k.to_string())
            out.append(None if not b else bytes(b))
        return out
    finally:
        c.close()


def _layerwise(eng, tokens, caches, slots, order=None):
    h = eng.store_paged_layerwise(tokens, caches, slots)
    layered = h._enc is not None
    for l in (order or range(len(caches))):
        h.save_layer(l)
    h.finish()
    return layered


def _bits(caches):
    out = []
    for c in caches:
        for t in (c if isinstance(c, tuple) else (c,)):
            out.append(t.contiguous().view(torch.uint8))
    return out


def _same_caches(a, b):
    for x, y in zip(_bits(a), _bits(b)):
        assert torch.equal(x, y)


def _retrieve_paged(eng, tokens, like, slots):
    out = [tuple(torch.zeros_like(t) for t in c) if isinstance(c, tuple) else torch.zeros_like(c) for c in like]
    mask = eng.retrieve_paged(tokens, out, slots)
    torch.cuda.synchronize()
    return mask, out


# ---------------------------------------------------------------------------------------------- remote tier
@pytest.mark.parametrize("pipelined", [False, True])
@pytest.mark.parametrize("serde,dtype", [("cachegen", torch.bfloat16), ("cachegen", torch.float16),
                                         ("lossless", torch.bfloat16), ("lossless", torch.float16),
                                         ("lossless", torch.float8_e4m3fn)])
def test_remote_containers_equal_store_paged(serde, dtype, pipelined, lmserver, autorelease):
    T = 1100                                                       # a ragged tail
    kv, slots = _kv(T, dtype, seed=1), _slots(T)
    caches = _paged(kv, slots)
    ta, tb = _tokens(T), _tokens(T)
    eng = _engine(autorelease, lmserver, serde, pipelined=pipelined)
    eng.store_paged(ta, caches, slots)
    assert _layerwise(eng, tb, caches, slots)
    reader = _engine(autorelease, lmserver, serde, pipelined=pipelined)   # right after finish(): no sleep
    a, b = _server_bytes(lmserver, eng, ta), _server_bytes(lmserver, eng, tb)
    assert len(a) == 5 and None not in a and a == b
    ma, oa = _retrieve_paged(reader, ta, caches, slots)
    mb, ob = _retrieve_paged(reader, tb, caches, slots)
    assert int(ma.sum()) == T and torch.equal(ma, mb)
    _same_caches(oa, ob)


@pytest.mark.parametrize("form", ["flashinfer", "tuple"])
@pytest.mark.parametrize("serde", ["cachegen", "lossless"])
def test_remote_flashinfer_and_tuple_forms(form, serde, lmserver, autorelease):
    T = 700
    kv, slots = _kv(T, torch.bfloat16, seed=2), _slots(T, 2)
    ta, tb = _tokens(T), _tokens(T)
    eng = _engine(autorelease, lmserver, serde)
    if form == "flashinfer":
        caches = _paged(kv, slots, "strided")
        eng.store_paged(ta, caches, slots)
        assert _layerwise(eng, tb, caches, slots)
    else:
        tup = tuple((kv[l, 0].clone(), kv[l, 1].clone()) for l in range(L))
        eng.store(ta, tup)
        dst = tuple((torch.full_like(k, float("nan")), torch.full_like(v, float("nan"))) for k, v in tup)
        h = eng.store_layerwise(tb, dst)
        assert h._enc is not None
        for l in range(L):
            dst[l][0].copy_(tup[l][0])
            dst[l][1].copy_(tup[l][1])
            h.save_layer(l)
        h.finish()
    a, b = _server_bytes(lmserver, eng, ta), _server_bytes(lmserver, eng, tb)
    assert None not in a and a == b


@pytest.mark.parametrize("serde", ["cachegen", "lossless"])
def test_remote_mla_rank0_stores_rank1_sends_nothing(serde, lmserver, autorelease, monkeypatch):
    from lmcache_b200.codec import CacheGenCodec, LosslessCodec
    from test_gpu_mla_engine import _cfg as mla_cfg
    cg = mla_cfg(L) if serde == "cachegen" else None
    T = 600
    kv, slots = _kv(T, torch.bfloat16, seed=3, mla=True), _slots(T, 3)
    caches = _paged(kv, slots, mla=True)
    ta, tb, tc = _tokens(T), _tokens(T), _tokens(T)
    r0 = _engine(autorelease, lmserver, serde, mla=True, rank=0, cg=cg)
    r1 = _engine(autorelease, lmserver, serde, mla=True, rank=1, cg=cg)
    r0.store_paged(ta, caches, slots)
    assert _layerwise(r0, tb, caches, slots)
    a, b = _server_bytes(lmserver, r0, ta), _server_bytes(lmserver, r0, tb)
    assert None not in a and a == b and len(a) == 3
    plans = []
    for cls in (CacheGenCodec, LosslessCodec):
        orig = cls.encode_layers_plan
        monkeypatch.setattr(cls, "encode_layers_plan", lambda self, *a, _o=orig, **k: plans.append(1) or _o(self, *a, **k))
    _layerwise(r1, tc, caches, slots)
    assert plans == [] and _server_bytes(lmserver, r1, tc) == [None] * 3
    m0, o0 = _retrieve_paged(r0, ta, caches, slots)
    m1, o1 = _retrieve_paged(r1, tb, caches, slots)                 # rank 1 reads what rank 0 stored
    assert int(m1.sum()) == T and torch.equal(m0, m1)
    _same_caches(o0, o1)


# ---------------------------------------------------------------------------------------------- hybrid tier
LOCALS = {"raw_cpu": ("cpu", None), "raw_cuda": ("cuda", None), "cachegen_host": ("cpu", "cachegen"),
          "lossless_host": ("cpu", "lossless"), "disk": ("file", "cachegen")}
SHARED = {("cachegen_host", "cachegen"), ("lossless_host", "lossless"), ("disk", "cachegen")}


def _local_bytes(eng, tokens):
    """what the hybrid's local tier holds for every chunk key of `tokens`: container bytes, or a raw blob's bytes"""
    local = eng.engine_.local_store
    out = []
    for h in eng._prefix_hash(tokens):
        k = eng._make_key(h, "vllm")
        if hasattr(local, "_lookup"):
            e = local._lookup(k)
            if e is None:
                out.append(None)
                continue
            e.ready.wait()
            if e.error is not None or e.rec is None:
                out.append(None)
            elif e.rec.blk is not None:
                out.append(bytes(e.rec.blk.view())[:e.rec.nbytes])
            else:
                with open(e.path, "rb") as f:
                    out.append(f.read())
        else:
            v = local.dict.get(k)
            if v is None:
                out.append(None)
            else:
                if hasattr(v, "wait"):
                    v.wait()
                t = v.host if hasattr(v, "host") else v
                out.append(bytes(t.contiguous().view(torch.uint8).cpu().numpy()))
    return out


class _Counts:
    def __init__(self, monkeypatch):
        from lmcache_b200.codec import CacheGenCodec, LosslessCodec, _ContainerIO
        self.plans, self.encodes = 0, 0
        for cls in (CacheGenCodec, LosslessCodec):
            orig = cls.encode_layers_plan

            def plan(codec, *a, _o=orig, **k):
                self.plans += 1
                return _o(codec, *a, **k)
            monkeypatch.setattr(cls, "encode_layers_plan", plan)
        orig_enc = _ContainerIO.encode_async

        def enc(codec, *a, **k):
            self.encodes += 1
            return orig_enc(codec, *a, **k)
        monkeypatch.setattr(_ContainerIO, "encode_async", enc)


@pytest.mark.parametrize("remote", ["cachegen", "lossless"])
@pytest.mark.parametrize("local", list(LOCALS))
def test_hybrid_both_tiers_hold_store_paged_bytes(local, remote, lmserver, tmp_path, autorelease, monkeypatch):
    dev, lserde = LOCALS[local]
    if dev == "file":
        dev = f"file://{tmp_path}/"
    T = 9 * CS + 50                                                 # three waves of 4 chunks
    kv, slots = _kv(T, torch.bfloat16, seed=4), _slots(T, 4)
    caches = _paged(kv, slots)
    ta, tb = _tokens(T), _tokens(T)
    eng = _engine(autorelease, lmserver, remote, local=dev, local_serde=lserde)
    counts = _Counts(monkeypatch)
    eng.store_paged(ta, caches, slots)
    shared = (local, remote) in SHARED
    containers = lserde is not None
    assert counts.encodes == (1 if shared else 1 + containers) * 3
    assert _layerwise(eng, tb, caches, slots)
    assert counts.plans == (1 if shared else 1 + containers)
    n = 10
    a, b = _server_bytes(lmserver, eng, ta), _server_bytes(lmserver, eng, tb)
    assert len(a) == n and None not in a and a == b
    la, lb = _local_bytes(eng, ta), _local_bytes(eng, tb)
    assert None not in la and la == lb
    if shared:
        assert la == a                                              # the same containers in both tiers
    for reader in (eng, _engine(autorelease, lmserver, remote)):      # local tier first, then the remote tier alone
        ma, oa = _retrieve_paged(reader, ta, caches, slots)
        mb, ob = _retrieve_paged(reader, tb, caches, slots)
        assert int(ma.sum()) == T and torch.equal(ma, mb)
        _same_caches(oa, ob)


@pytest.mark.parametrize("serde", ["cachegen", "lossless"])
def test_hybrid_evicting_local_tier_is_backed_by_the_server(serde, lmserver, autorelease):
    T = 2 * CS
    kv, slots = _kv(T, torch.bfloat16, seed=5), _slots(T, 5)
    caches = _paged(kv, slots)
    t0, ta, tb = _tokens(T), _tokens(T), _tokens(T)
    probe = _engine(autorelease, lmserver, serde, local="cpu", local_serde=serde)
    probe.store_paged(t0, caches, slots)
    size = max(len(b) for b in _local_bytes(probe, t0))
    eng = _engine(autorelease, lmserver, serde, local="cpu", local_serde=serde, capacity=int(2.5 * size) + 4096)
    assert _layerwise(eng, ta, caches, slots, order=range(L)) and _layerwise(eng, tb, caches, slots)
    assert None in _local_bytes(eng, ta) and None not in _local_bytes(eng, tb)     # b's store evicted a's head
    assert None not in _server_bytes(lmserver, eng, ta)
    ma, oa = _retrieve_paged(eng, ta, caches, slots)               # the server serves a's evicted chunks
    mb, ob = _retrieve_paged(eng, tb, caches, slots)
    assert int(ma.sum()) == T and torch.equal(ma, mb)
    _same_caches(oa, ob)


# ---------------------------------------------------------------------------------------------- edge cases
@pytest.mark.parametrize("tier", ["remote", "hybrid"])
def test_skip_existing_prefix_on_the_server(tier, lmserver, autorelease):
    T = 6 * CS
    kv, slots = _kv(T, torch.bfloat16, seed=6), _slots(T, 6)
    caches = _paged(kv, slots)
    ta, tb = _tokens(T), _tokens(T)
    local = ("cpu", "cachegen") if tier == "hybrid" else (None, None)
    eng = _engine(autorelease, lmserver, "cachegen", local=local[0], local_serde=local[1])
    for t, lw in ((ta, False), (tb, True)):
        eng.store_paged(t[:3 * CS], caches, slots[:3 * CS])
        if lw:
            assert _layerwise(eng, t, caches, slots)
        else:
            eng.store_paged(t, caches, slots)
    assert _server_bytes(lmserver, eng, ta) == _server_bytes(lmserver, eng, tb)
    reader = _engine(autorelease, lmserver, "cachegen")
    ma, oa = _retrieve_paged(reader, ta, caches, slots)
    mb, ob = _retrieve_paged(reader, tb, caches, slots)
    assert int(mb.sum()) == T and torch.equal(ma, mb)
    _same_caches(oa, ob)


def test_arena_limit_keeps_the_same_prefix_in_both_tiers(lmserver, autorelease, monkeypatch):
    T = 16 * CS
    g = torch.Generator(device="cuda").manual_seed(7)
    kv = (torch.rand((L, 2, T, H, D), device="cuda", generator=g) * 2 - 1).to(torch.bfloat16)   # ~4 bits per symbol
    slots = _slots(T, 7)
    caches = _paged(kv, slots)
    ta, tb = _tokens(T), _tokens(T)
    eng = _engine(autorelease, lmserver, "cachegen", local="cpu", local_serde="cachegen")
    eng.store_paged(ta, caches, slots)
    total = sum(len(b) for b in _server_bytes(lmserver, eng, ta))
    monkeypatch.setenv("LMCACHE_B200_LAYERWISE_STORE_MB", str(max(1, total // 2 >> 20)))
    assert (max(1, total // 2 >> 20) << 20) < total
    assert _layerwise(eng, tb, caches, slots)
    remote, local = _server_bytes(lmserver, eng, tb), _local_bytes(eng, tb)
    k = remote.index(None)
    assert 0 < k < 16 and all(x is None for x in remote[k:])
    assert local[:k] == remote[:k] == _server_bytes(lmserver, eng, ta)[:k] and all(x is None for x in local[k:])


@pytest.mark.parametrize("tier", ["remote", "hybrid"])
def test_save_errors_are_those_of_the_host_tier(tier, lmserver, autorelease):
    T = 600
    kv, slots = _kv(T, torch.bfloat16, seed=8), _slots(T, 8)
    caches = _paged(kv, slots)
    tokens = _tokens(T)
    local = ("cuda", None) if tier == "hybrid" else (None, None)
    eng = _engine(autorelease, lmserver, "lossless", local=local[0], local_serde=local[1])
    h = eng.store_paged_layerwise(tokens, caches, slots)
    h.save_layer(2)
    with pytest.raises(ValueError):
        h.save_layer(2)
    with pytest.raises(ValueError):
        h.save_layer(L)
    with pytest.raises(ValueError):
        h.finish()                                                  # layers 0, 1, 3 missing
    assert _server_bytes(lmserver, eng, tokens) == [None] * 3
    assert _layerwise(eng, tokens, caches, slots, order=[3, 1, 0, 2])
    m, out = _retrieve_paged(_engine(autorelease, lmserver, "lossless"), tokens, caches, slots)
    assert int(m.sum()) == T
    _same_caches(out, caches)


def _stored_anyway(fn):
    """run a store whose remote sends may fail against a stopped server: it may raise, as store_paged() would"""
    try:
        fn()
    except Exception:               # noqa: BLE001
        pass


def test_server_closed_before_finish(autorelease):
    """A server stopped before finish(): the remote part's chunks are misses, the shared slots go back to their pools,
    and the engine keeps storing into and serving from its local tier, layer-wise and not."""
    srv = _Native()
    try:
        url = f"lmn://127.0.0.1:{srv.port}"
        T = 700
        kv, slots = _kv(T, torch.bfloat16, seed=9), _slots(T, 9)
        caches = _paged(kv, slots)
        ta, tb, tc = _tokens(T), _tokens(T), _tokens(T)
        eng = _engine(autorelease, url, "lossless", local="cpu", local_serde="lossless")
        local, remote = eng.engine_.local_store, _remote_of(eng)
        h = eng.store_paged_layerwise(ta, caches, slots)
        for l in range(L):
            h.save_layer(l)
        srv.stop()                  # before any send: every send of this engine opens its connection then, and fails
        _stored_anyway(h.finish)
        assert not any(remote.contains(k) for k in eng._keys_of(eng._prefix_hash(ta), "vllm"))
        pool = local._segments
        assert len(pool._free) == 1 and pool._free[0].refs == 0        # both sinks released the shared slot
        _stored_anyway(lambda: eng.store_paged(tb, caches, slots))
        ring = local._pipe.ring
        assert ring._free.qsize() == len(ring._all)                    # every shared wave slot is free again
        _stored_anyway(lambda: _layerwise(eng, tc, caches, slots))
        for t in (ta, tb, tc):
            m, out = _retrieve_paged(eng, t, caches, slots)            # the local tier serves every chunk
            assert int(m.sum()) == T
            _same_caches(out, caches)
    finally:
        srv.stop()


@pytest.mark.parametrize("why", ["torch", "chunk512"])
def test_fallbacks_equal_store_paged(why, lmserver, autorelease):
    T = 1100
    kv, slots = _kv(T, torch.bfloat16, seed=10), _slots(T, 10)
    caches = _paged(kv, slots)
    ta, tb = _tokens(T), _tokens(T)
    serde, cs = ("torch", CS) if why == "torch" else ("cachegen", 512)
    eng = _engine(autorelease, lmserver, serde, cs=cs)
    eng.store_paged(ta, caches, slots)
    assert not _layerwise(eng, tb, caches, slots)
    ma, oa = _retrieve_paged(eng, ta, caches, slots)
    mb, ob = _retrieve_paged(eng, tb, caches, slots)
    assert int(ma.sum()) == T and torch.equal(ma, mb)
    _same_caches(oa, ob)
