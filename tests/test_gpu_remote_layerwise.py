"""GPU: layer-by-layer retrieve from the lm:// remote and hybrid tiers over ranged reads (OPEN / READ / CLOSE).  Every
result is compared bit for bit with retrieve() / retrieve_paged() of the same tier, which the other GPU tests hold to
the reference decode; each case also shows that the path really was layer-major (one event per layer, ranged bytes
counted by the backend)."""
import ctypes
import threading
import time

import pytest
import torch

from test_gpu_host_tier import MODEL
from test_remote_ranges_cpu import _ReferenceStub

pytestmark = pytest.mark.gpu


class _Native:
    def __init__(self):
        from lmcache_b200 import _native as N
        self.lib = N.lib()
        self.h = ctypes.c_void_p()
        N.check(self.lib.b200kv_lm_server_start(b"127.0.0.1", 0, ctypes.byref(self.h)))
        self.port = self.lib.b200kv_lm_server_port(self.h)
        self.live = True

    def num_handles(self):
        return self.lib.b200kv_lm_server_num_handles(self.h)

    def stop(self):
        if self.live:
            self.live = False
            self.lib.b200kv_lm_server_stop(self.h)


class _Python:
    def __init__(self):
        from lmcache_b200.server.__main__ import LMCacheServer
        self.srv = LMCacheServer("127.0.0.1", 0)
        self.port = self.srv.sock.getsockname()[1]
        threading.Thread(target=self.srv.run, daemon=True).start()

    def num_handles(self):
        return self.srv.num_handles()

    def stop(self):
        self.srv.sock.close()


@pytest.fixture(autouse=True)
def remote_layerwise(monkeypatch):
    """the layer-major remote get is opt-in; every engine of these tests opts in unless a test says otherwise"""
    monkeypatch.setenv("LMCACHE_B200_REMOTE_LAYERWISE", "1")
    return monkeypatch


@pytest.fixture
def server():
    s = _Native()
    yield s
    s.stop()


def _engine(autorelease, port, serde="cachegen", cs=256, fmt="vllm", mla=False, scheme="lmn", local=None,
            local_serde=None, reshard=None, ws=1, rank=0, cg=None):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    cfg = LMCacheEngineConfig(cs, local, f"{scheme}://127.0.0.1:{port}", serde, False, False, local_serde,
                              cachegen_config=cg, reshard_world_sizes=reshard,
                              reshard_lossless=reshard is not None and serde == "lossless")
    return autorelease(LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, ws, rank, fmt, "bfloat16", mla)))


def _kv(T, fmt, dtype, L=4, H=2, D=128, seed=0, mla=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if mla:
        return tuple(torch.randn((T, D), device="cuda", generator=g).to(dtype) for _ in range(L))
    shape = (T, H, D) if fmt == "vllm" else (H, T, D)
    return tuple((torch.randn(shape, device="cuda", generator=g).to(dtype),
                  torch.randn(shape, device="cuda", generator=g).to(dtype)) for _ in range(L))


def _cut(kv, n, fmt, mla=False):
    if mla:
        return tuple(x[:n] for x in kv)
    return tuple((k[:n], v[:n]) if fmt == "vllm" else (k[:, :n], v[:, :n]) for k, v in kv)


def _flat(ret):
    out = []
    for x in ret:
        out += list(x) if isinstance(x, tuple) else [x]
    return [t.contiguous().view(torch.int16) for t in out]


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(_flat(a), _flat(b)):
        assert torch.equal(x, y)


def _remote(engine):
    be = engine.engine_
    return getattr(be, "remote_store", be)


def _layer_major(r, backend, reads_before):
    evs = [r._upload.ready(layer) for layer in range(r.num_layers)]
    assert len({id(e) for e in evs}) == r.num_layers            # one event per layer
    assert backend.ranged_stats["reads"] > reads_before and backend.ranged_stats["bytes"] > 0


def _no_leaks(server, engine):
    for _ in range(500):
        if server.num_handles() == 0:
            break
        time.sleep(0.01)
    assert server.num_handles() == 0
    be = _remote(engine)
    engine.close()
    assert be._release.pending() == 0


# ---------------------------------------------------------------------------------------------- equality
CASES = [("cachegen", 256, "vllm", torch.bfloat16, False), ("cachegen", 256, "huggingface", torch.float16, False),
         ("lossless", 256, "vllm", torch.bfloat16, False), ("lossless", 1024, "vllm", torch.float16, False),
         ("lossless", 256, "huggingface", torch.bfloat16, False), ("cachegen", 256, "vllm", torch.bfloat16, True),
         ("lossless", 256, "vllm", torch.bfloat16, True)]


@pytest.mark.parametrize("serde,cs,fmt,dtype,mla", CASES)
@pytest.mark.parametrize("case", ["plain", "masked", "miss"])
@pytest.mark.parametrize("scheme", ["lmn", "lm"])
def test_layerwise_equals_retrieve(serde, cs, fmt, dtype, mla, case, scheme, server, autorelease):
    cg = None
    if mla and serde == "cachegen":
        from test_gpu_mla_engine import _cfg as mla_cfg
        cg = mla_cfg(4)
    T = 3 * cs + 37                                                # a ragged tail
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    kv = _kv(T, fmt, dtype, mla=mla, seed=3)
    writer = _engine(autorelease, server.port, serde, cs, fmt, mla, cg=cg)
    writer.store(tokens[:2 * cs] if case == "miss" else tokens, _cut(kv, 2 * cs if case == "miss" else T, fmt, mla))
    mask = None
    if case == "masked":
        mask = torch.ones(T, dtype=torch.bool)
        mask[:cs + 37] = False                                     # the first retrieved chunk straddles the mask
    ref, ref_mask = _engine(autorelease, server.port, serde, cs, fmt, mla, scheme, cg=cg).retrieve(tokens, mask)
    for eng in (writer, _engine(autorelease, server.port, serde, cs, fmt, mla, scheme, cg=cg)):   # + a replica (peek)
        be = _remote(eng)
        before = be.ranged_stats["reads"]
        r = eng.retrieve_layerwise(tokens, mask)
        r.synchronize()
        torch.cuda.synchronize()
        assert torch.equal(r.ret_mask, ref_mask) and int(ref_mask.sum()) > 0
        _same(r.kv, ref)
        _layer_major(r, be, before)
    _no_leaks(server, writer)


@pytest.mark.parametrize("serde", ["cachegen", "lossless"])
@pytest.mark.parametrize("skip", [0, 300])
def test_paged_layerwise_equals_retrieve_paged(serde, skip, server, autorelease):
    cs, T, L, H, D, bs = 256, 1000, 4, 2, 128, 16
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    kv = _kv(T, "vllm", torch.bfloat16, L=L, H=H, D=D, seed=6)
    eng = _engine(autorelease, server.port, serde, cs)
    eng.store(tokens[:900], _cut(kv, 900, "vllm"))
    nblk = (T + bs - 1) // bs + 8
    slots = torch.randperm(nblk * bs, device="cuda")[:T]
    mask = None
    if skip:
        mask = torch.ones(T, dtype=torch.bool)
        mask[:skip] = False
    caches = []
    for _ in range(2):
        g = torch.Generator(device="cuda").manual_seed(9)
        caches.append([(torch.randn((nblk, bs, H, D), device="cuda", generator=g).to(torch.bfloat16),
                        torch.randn((nblk, bs, H, D), device="cuda", generator=g).to(torch.bfloat16)) for _ in range(L)])
    want = eng.retrieve_paged(tokens, caches[0], slots, mask)
    before = _remote(eng).ranged_stats["reads"]
    r = eng.retrieve_paged_layerwise(tokens, caches[1], slots, mask)
    r.synchronize()
    torch.cuda.synchronize()
    assert torch.equal(r.ret_mask, want) and int(want.sum()) == 768 - skip
    _same(caches[0], caches[1])
    _layer_major(r, _remote(eng), before)
    _no_leaks(server, eng)


def test_lossless_dtype_switch_mid_chain(server, autorelease):
    cs, T = 256, 1024
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    _engine(autorelease, server.port, "lossless").store(tokens[:512], _cut(_kv(T, "vllm", torch.bfloat16, seed=1), 512,
                                                                           "vllm"))
    _engine(autorelease, server.port, "lossless").store(tokens, _kv(T, "vllm", torch.float16, seed=2))   # chunks 2, 3: fp16
    ref, ref_mask = _engine(autorelease, server.port, "lossless").retrieve(tokens)
    eng = _engine(autorelease, server.port, "lossless")
    r = eng.retrieve_layerwise(tokens)
    r.synchronize()
    assert int(ref_mask.sum()) == 512 and torch.equal(r.ret_mask, ref_mask)
    _same(r.kv, ref)
    _layer_major(r, _remote(eng), 0)
    _no_leaks(server, eng)


@pytest.mark.parametrize("kind", ["native", "python"])
@pytest.mark.parametrize("serde", ["cachegen", "lossless"])
def test_retrieve_only_replica_on_both_servers(kind, serde, autorelease):
    srv = _Native() if kind == "native" else _Python()
    try:
        T = 700
        tokens = torch.randint(0, 32000, (T,), device="cuda")
        _engine(autorelease, srv.port, serde).store(tokens, _kv(T, "vllm", torch.bfloat16, seed=5))
        ref, ref_mask = _engine(autorelease, srv.port, serde).retrieve(tokens)
        eng = _engine(autorelease, srv.port, serde)
        r = eng.retrieve_layerwise(tokens)
        r.synchronize()
        assert torch.equal(r.ret_mask, ref_mask) and int(ref_mask.sum()) == T
        _same(r.kv, ref)
        _layer_major(r, _remote(eng), 0)
        _no_leaks(srv, eng)
    finally:
        srv.stop()


def test_wait_layer_orders_a_side_stream(server, autorelease):
    import random
    L, T = 8, 2048
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    eng = _engine(autorelease, server.port, "lossless")
    kv = _kv(T, "vllm", torch.bfloat16, L=L, seed=8)
    eng.store(tokens, kv)
    ref, _ = eng.retrieve(tokens)
    torch.cuda.synchronize()
    r = eng.retrieve_layerwise(tokens)
    copies = []
    for layer in random.Random(0).sample(range(L), L):
        s = torch.cuda.Stream()
        r.wait_layer(layer, s)
        with torch.cuda.stream(s):
            copies.append((layer, s, r.kv[layer][0].clone(), r.kv[layer][1].clone()))
    for layer, s, k, v in copies:
        s.synchronize()
        _same([(k, v)], [ref[layer]])


def test_overwrite_after_the_call_returns_the_first_version(server, autorelease):
    T = 2048
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    first = _engine(autorelease, server.port, "lossless")
    first.store(tokens, _kv(T, "vllm", torch.bfloat16, L=8, seed=1))
    ref, ref_mask = first.retrieve(tokens)
    torch.cuda.synchronize()
    eng = _engine(autorelease, server.port, "lossless")
    other = _engine(autorelease, server.port, "cachegen")      # keys do not name the serde
    r = eng.retrieve_layerwise(tokens)
    other.store(tokens, _kv(T, "vllm", torch.bfloat16, L=8, seed=2), skip_existing=False)
    r.synchronize()
    assert torch.equal(r.ret_mask, ref_mask)
    _same(r.kv, ref)
    again, _ = _engine(autorelease, server.port, "cachegen").retrieve(tokens)
    assert not all(torch.equal(a, b) for a, b in zip(_flat(again), _flat(ref)))     # the overwrite did land


# ---------------------------------------------------------------------------------------------- fallbacks
@pytest.mark.parametrize("why", ["reference", "chunk512", "torch", "not_opted_in"])
def test_fallbacks_equal_retrieve(why, server, autorelease, remote_layerwise):
    if why == "not_opted_in":
        remote_layerwise.delenv("LMCACHE_B200_REMOTE_LAYERWISE")
    stub = _ReferenceStub() if why == "reference" else None
    try:
        port = stub.port if stub else server.port
        scheme = "lm" if stub else "lmn"
        serde = "torch" if why == "torch" else "cachegen"
        cs = 512 if why == "chunk512" else 256
        T = 1100
        tokens = torch.randint(0, 32000, (T,), device="cuda")
        _engine(autorelease, port, serde, cs, scheme=scheme).store(tokens, _kv(T, "vllm", torch.bfloat16, seed=4))
        time.sleep(0.2)
        ref, ref_mask = _engine(autorelease, port, serde, cs, scheme=scheme).retrieve(tokens)
        eng = _engine(autorelease, port, serde, cs, scheme=scheme)
        r = eng.retrieve_layerwise(tokens)
        r.synchronize()
        assert torch.equal(r.ret_mask, ref_mask) and int(ref_mask.sum()) > 0
        _same(r.kv, ref)
        assert len({id(r._upload.ready(layer)) for layer in range(r.num_layers)}) == 1     # one event for every layer
        assert _remote(eng).ranged_stats["retrieves"] == 0
        if why == "not_opted_in":
            assert _remote(eng)._ranges is None                 # the probe was never sent
        if stub:
            assert max(stub.commands) <= 4
    finally:
        if stub:
            stub.close()


# ---------------------------------------------------------------------------------------------- hybrid, reshard
def test_hybrid_both_parts_layer_major(server, autorelease):
    T = 1024
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    kv = _kv(T, "vllm", torch.bfloat16, seed=7)
    hyb = _engine(autorelease, server.port, local="cpu", local_serde="cachegen")
    hyb.store(tokens[:512], _cut(kv, 512, "vllm"))                                    # the local tier: chunks 0, 1
    _engine(autorelease, server.port).store(tokens, kv)                               # the remote tier: every chunk
    ref, ref_mask = _engine(autorelease, server.port).retrieve(tokens)
    r = hyb.retrieve_layerwise(tokens)
    r.synchronize()
    assert torch.equal(r.ret_mask, ref_mask) and int(ref_mask.sum()) == T
    _same(r.kv, ref)
    parts = r._upload.parts
    assert len(parts) == 2 and parts[0].n == 2 and parts[1].n == 2
    for p in parts:
        assert len({id(p.ready(layer)) for layer in range(r.num_layers)}) == r.num_layers
    assert _remote(hyb).ranged_stats["reads"] > 0


def test_reshard_continuation_is_ready_with_layer_0(server, autorelease):
    T, Hg, fmt = 1024, 4, "vllm"
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    kv = _kv(T, fmt, torch.bfloat16, H=Hg, seed=11)
    for r_ in range(2):
        _engine(autorelease, server.port, ws=2, rank=r_).store(
            tokens, tuple((k[:, 2 * r_:2 * r_ + 2], v[:, 2 * r_:2 * r_ + 2]) for k, v in kv))
    own = _engine(autorelease, server.port, reshard=[2])
    own.store(tokens[:512], _cut(kv, 512, fmt))
    ref, ref_mask = own.retrieve(tokens)
    torch.cuda.synchronize()
    r = own.retrieve_layerwise(tokens)
    assert torch.equal(r.ret_mask, ref_mask) and int(ref_mask.sum()) == T
    from lmcache_b200.pipeline import JoinedUpload
    assert isinstance(r._upload, JoinedUpload) and len(r._upload.parts) == 2
    prefix, rest = r._upload.parts
    assert prefix.n == 2 and len({id(prefix.ready(l)) for l in range(r.num_layers)}) == r.num_layers   # layer-major
    assert rest.n == 2 and len({id(rest.ready(l)) for l in range(r.num_layers)}) == 1                 # chunk-major
    s = torch.cuda.Stream()
    r.wait_layer(0, s)
    with torch.cuda.stream(s):
        tail = [(k[512:].clone(), v[512:].clone()) for k, v in r.kv]                  # every layer, after ready(0) only
    s.synchronize()
    _same(tail, [(k[512:], v[512:]) for k, v in ref])
    r.synchronize()
    _same(r.kv, ref)


# ---------------------------------------------------------------------------------------------- errors
def test_lost_server_after_the_match(server, autorelease, monkeypatch):
    from lmcache_b200.storage_backend import remote_backend
    T = 2048
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    eng = _engine(autorelease, server.port, "lossless")
    eng.store(tokens, _kv(T, "vllm", torch.bfloat16, L=8, seed=3))
    torch.cuda.synchronize()
    go = threading.Event()
    run = remote_backend.RangedFetch._run

    def held(self, c):
        go.wait(30)
        return run(self, c)
    monkeypatch.setattr(remote_backend.RangedFetch, "_run", held)
    r = eng.retrieve_layerwise(tokens)
    assert int(r.ret_mask.sum()) == T                          # promised at the call
    server.stop()
    go.set()
    with pytest.raises(Exception):
        r.synchronize()
    with pytest.raises(Exception):
        r.wait_layer(r.num_layers - 1)
    be = _remote(eng)
    t = threading.Thread(target=eng.close)
    t.start()
    t.join(60)
    assert not t.is_alive()
    assert be._release.pending() == 0
