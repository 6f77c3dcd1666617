"""GPU: layer-by-layer store (LMCacheEngine.store_layerwise / store_paged_layerwise) and the encode it rests on
(b200kv_encode_layers_plan + b200kv_encode_layers + b200kv_encode_layers_finish).  What lands is compared byte for byte
with what store() / store_paged() land for the same inputs, and every retrieve bit for bit with the reference decode."""
import os
import socket
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from test_gpu_host_tier import MODEL, _blob_of, _meta, _want

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L, H, D, CS = 4, 2, 128, 256


def _cfg(tier, tmp_path, name, cs=CS, capacity=None):
    from lmcache_b200.config import LMCacheEngineConfig
    backend = "cpu" if tier == "host" else "file://" + str(tmp_path / name) + "/"
    return LMCacheEngineConfig.from_legacy(chunk_size=cs, backend=backend, local_serde="cachegen",
                                           local_capacity_bytes=capacity)


def _source(T, entropy, dtype, seed=0):
    """[L,2,T,H,D] KV: 'low' ~0.6 coder bits per symbol, 'high' ~4 bits"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if entropy == "low":
        kv = torch.randn((L, 2, T, H, D), device="cuda", generator=g) * 0.05
        kv[..., 0] = 4.0
    else:
        kv = torch.rand((L, 2, T, H, D), device="cuda", generator=g) * 2 - 1
    return kv.to(dtype)


def _landed(engine):
    """key -> (container bytes, plane offsets) of every chunk the engine's tier holds, once landed"""
    out = {}
    for k, e in engine.engine_.dict.items():
        e.ready.wait()
        if e.error is not None or e.rec is None:
            continue
        if e.rec.blk is not None:
            data = bytes(e.rec.blk.view())[:e.rec.nbytes]
        else:
            with open(e.path, "rb") as f:
                data = f.read()
        # the disk tier keys its entries by file path: compare tiers in different directories by file name
        out[os.path.basename(k) if isinstance(k, str) else k] = (data, None if e.rec.planes is None else e.rec.planes.tolist())
    return out


def _paged(T, dtype, fill=float("nan"), bs=16):
    nblk = (T + bs - 1) // bs + 4
    slots = torch.randperm(nblk * bs, device="cuda")[:T]
    caches = [(torch.full((nblk, bs, H, D), fill, device="cuda", dtype=dtype),
               torch.full((nblk, bs, H, D), fill, device="cuda", dtype=dtype)) for _ in range(L)]
    return caches, slots


def _write_layer(caches, slots, kv, l):
    caches[l][0].view(-1, H, D)[slots] = kv[l, 0]
    caches[l][1].view(-1, H, D)[slots] = kv[l, 1]


def _save_all(handle, write, order):
    """write layer l on the current stream, then save it; finish, then overwrite every layer on the same stream"""
    for l in order:
        write(l)
        handle.save_layer(l)
    handle.finish()


@pytest.mark.parametrize("tier", ["host", "disk"])
@pytest.mark.parametrize("dtype,T,entropy,reverse", [
    (torch.bfloat16, 200, "low", False),        # one chunk
    (torch.float16, 2300, "high", True),        # ragged last chunk
    (torch.bfloat16, 2300, "high", False),
    (torch.bfloat16, 8192, "low", False),       # 32 chunks
])
def test_paged_layerwise_lands_store_paged_bytes(tier, dtype, T, entropy, reverse, tmp_path, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    kv = _source(T, entropy, dtype, seed=T)
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    ref = autorelease(LMCacheEngine(_cfg(tier, tmp_path, "a"), _meta()))
    caches_a, slots = _paged(T, dtype)
    for l in range(L):
        _write_layer(caches_a, slots, kv, l)
    ref.store_paged(tokens, caches_a, slots)
    eng = autorelease(LMCacheEngine(_cfg(tier, tmp_path, "b"), _meta()))
    caches_b = [(torch.full_like(k, float("nan")), torch.full_like(v, float("nan"))) for k, v in caches_a]
    h = eng.store_paged_layerwise(tokens, caches_b, slots)
    assert h.num_layers == L
    _save_all(h, lambda l: _write_layer(caches_b, slots, kv, l), range(L - 1, -1, -1) if reverse else range(L))
    for k, v in caches_b:                           # the cache is reused right after finish(), in stream order
        k.fill_(-7.0)
        v.fill_(float("nan"))
    ret_b, mask_b = eng.retrieve(tokens)            # waits for the landing (read your writes)
    ret_a, mask_a = ref.retrieve(tokens)
    torch.cuda.synchronize()
    assert int(mask_b.sum()) == T and torch.equal(mask_a, mask_b)
    assert torch.equal(_blob_of(ret_b).view(torch.int16), _blob_of(ret_a).view(torch.int16))
    if dtype == torch.bfloat16:
        want = _want(tuple((kv[l, 0], kv[l, 1]) for l in range(L)), "vllm", CS, T)
        assert torch.equal(_blob_of(ret_b).view(torch.int16), want.view(torch.int16))
    a, b = _landed(ref), _landed(eng)
    assert len(a) == -(-T // CS) and a.keys() == b.keys()
    for k in a:
        assert a[k][0] == b[k][0], "container bytes differ"
        assert a[k][1] == b[k][1] and b[k][1] is not None, "plane offsets differ"


@pytest.mark.parametrize("tier", ["host", "disk"])
@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
def test_dense_layerwise_lands_store_bytes(tier, fmt, tmp_path, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    T = 2300
    dtype = torch.bfloat16 if fmt == "vllm" else torch.float16
    src = _source(T, "high" if fmt == "vllm" else "low", dtype, seed=5)
    kv = tuple((src[l, 0], src[l, 1]) if fmt == "vllm" else (src[l, 0].transpose(0, 1).contiguous(),
                                                              src[l, 1].transpose(0, 1).contiguous()) for l in range(L))
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    ref = autorelease(LMCacheEngine(_cfg(tier, tmp_path, "a"), _meta(fmt)))
    ref.store(tokens, kv)
    eng = autorelease(LMCacheEngine(_cfg(tier, tmp_path, "b"), _meta(fmt)))
    dst = tuple((torch.full_like(k, float("nan")), torch.full_like(v, float("nan"))) for k, v in kv)
    h = eng.store_layerwise(tokens, dst)

    def write(l):
        dst[l][0].copy_(kv[l][0])
        dst[l][1].copy_(kv[l][1])
    _save_all(h, write, range(L))
    for k, v in dst:
        k.fill_(3.0)
        v.fill_(float("nan"))
    ret_b, mask_b = eng.retrieve(tokens)
    torch.cuda.synchronize()
    assert int(mask_b.sum()) == T
    assert torch.equal(_blob_of(ret_b).view(torch.int16), _want(kv, fmt, CS, T).view(torch.int16))
    a, b = _landed(ref), _landed(eng)
    assert len(a) == 9 and a.keys() == b.keys()
    for k in a:
        assert a[k] == b[k]


def test_skip_existing_writes_only_the_missing_chunks_and_touches_like_store_paged(tmp_path, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    T = 8 * CS
    kv = _source(T, "low", torch.bfloat16, seed=21)
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    stamps, landed = [], []
    for mode in ("paged", "layerwise"):
        eng = autorelease(LMCacheEngine(_cfg("host", tmp_path, mode, capacity=1 << 30), _meta()))
        caches, slots = _paged(T, torch.bfloat16)
        for l in range(L):
            _write_layer(caches, slots, kv, l)
        eng.store_paged(tokens[:4 * CS], caches, slots[:4 * CS])
        first = {k: id(e) for k, e in eng.engine_.dict.items()}
        if mode == "paged":
            eng.store_paged(tokens, caches, slots)
        else:
            h = eng.store_paged_layerwise(tokens, caches, slots)
            _save_all(h, lambda l: None, range(L))
        keys = [eng._make_key(x, "vllm") for x in eng._prefix_hash(tokens)]
        ret, mask = eng.retrieve(tokens)
        torch.cuda.synchronize()
        assert int(mask.sum()) == T
        assert all(id(eng.engine_.dict[k]) == first[k] for k in keys[:4])          # chunks 0-3 were not rewritten
        assert len(eng.engine_.dict) == 8
        stamps.append([eng.engine_._order.stamp(k) for k in keys])
        landed.append(_landed(eng))
    assert stamps[0] == stamps[1]
    assert landed[0] == landed[1]


@pytest.mark.parametrize("tier", ["host", "disk"])
def test_arena_overflow_keeps_the_longest_fitting_prefix(tier, tmp_path, autorelease, monkeypatch):
    from lmcache_b200.cache_engine import LMCacheEngine
    T = 16 * CS
    kv = _source(T, "high", torch.bfloat16, seed=31)
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    ref = autorelease(LMCacheEngine(_cfg(tier, tmp_path, "a"), _meta()))
    caches, slots = _paged(T, torch.bfloat16)
    for l in range(L):
        _write_layer(caches, slots, kv, l)
    ref.store_paged(tokens, caches, slots)
    total = sum(len(c) for c, _ in _landed(ref).values())
    monkeypatch.setenv("LMCACHE_B200_LAYERWISE_STORE_MB", str(max(1, total // 2 >> 20)))
    eng = autorelease(LMCacheEngine(_cfg(tier, tmp_path, "b"), _meta()))
    budget = max(1, total // 2 >> 20) << 20
    assert budget < total
    h = eng.store_paged_layerwise(tokens, caches, slots)
    _save_all(h, lambda l: None, range(L))
    ret, mask = eng.retrieve(tokens)
    torch.cuda.synchronize()
    got = int(mask.sum())
    assert 0 < got < T and got % CS == 0
    assert bool(mask[:got].all()) and not bool(mask[got:].any())
    want = _want(tuple((kv[l, 0], kv[l, 1]) for l in range(L)), "vllm", CS, got)
    assert torch.equal(_blob_of(ret).view(torch.int16), want.view(torch.int16))
    a, b = _landed(ref), _landed(eng)
    assert len(b) == got // CS and all(a[k] == b[k] for k in b)


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


@pytest.mark.parametrize("kind", ["remote", "hybrid", "raw", "chunk512"])
def test_fallback_tiers_store_what_store_paged_stores(kind, lmserver, tmp_path, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig
    T = 1100
    kv = _source(T, "low", torch.bfloat16, seed=41)
    caches, slots = _paged(T, torch.bfloat16)
    for l in range(L):
        _write_layer(caches, slots, kv, l)
    results = []
    for mode in ("paged", "layerwise"):
        tokens = torch.arange(T, device="cuda") + (0 if mode == "paged" else 50000)   # distinct keys on a shared server
        if kind == "remote":
            cfg = LMCacheEngineConfig(CS, None, lmserver, "cachegen", False, False, "cachegen")
        elif kind == "hybrid":
            cfg = LMCacheEngineConfig(CS, "cpu", lmserver, "cachegen", False, False, "cachegen")
        elif kind == "raw":
            cfg = LMCacheEngineConfig.from_legacy(chunk_size=CS, backend="cpu")
        else:
            cfg = _cfg("host", tmp_path, mode, cs=512)
        eng = autorelease(LMCacheEngine(cfg, _meta()))
        if mode == "paged":
            eng.store_paged(tokens, caches, slots)
        else:
            h = eng.store_paged_layerwise(tokens, caches, slots)
            _save_all(h, lambda l: None, range(L))
        out = [(torch.zeros_like(k), torch.zeros_like(v)) for k, v in caches]
        mask = eng.retrieve_paged(tokens, out, slots)
        torch.cuda.synchronize()
        results.append((mask, out))
    (ma, oa), (mb, ob) = results
    assert torch.equal(ma, mb) and int(ma.sum()) == T
    for (ka, va), (kb, vb) in zip(oa, ob):
        assert torch.equal(ka.view(torch.int16), kb.view(torch.int16)) and torch.equal(va.view(torch.int16), vb.view(torch.int16))


def test_errors_store_nothing(tmp_path, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    T = 600
    eng = autorelease(LMCacheEngine(_cfg("host", tmp_path, "a"), _meta()))
    caches, slots = _paged(T, torch.bfloat16, fill=1.0)
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    h = eng.store_paged_layerwise(tokens, caches, slots)
    h.save_layer(0)
    with pytest.raises(ValueError):
        h.save_layer(0)
    with pytest.raises(ValueError):
        h.save_layer(L)
    with pytest.raises(ValueError):
        h.save_layer(-1)
    h.save_layer(2)
    with pytest.raises(ValueError):
        h.finish()                                   # layers 1 and 3 missing
    assert len(eng.engine_.dict) == 0
    h2 = eng.store_paged_layerwise(tokens, caches, slots)
    h2.save_layer(1)
    del h2                                           # dropped: its pool slot goes back
    pool = eng.engine_._segments
    assert pool is not None and len(pool._free) >= 1
    h3 = eng.store_paged_layerwise(tokens, caches, slots)
    _save_all(h3, lambda l: None, range(L))
    _, mask = eng.retrieve(tokens)
    assert int(mask.sum()) == T and len(eng.engine_.dict) == 3


# ---------------------------------------------------------------------------------------------- ABI level
@pytest.mark.parametrize("calls", [[1, 1, 1, 1, 1, 1], [2, 3, 1], [6]])
def test_encode_layers_partition_equals_encode_chunks(calls):
    """any partition of the layers into calls lands b200kv_encode_chunks' containers"""
    import ctypes

    from lmcache_b200 import _native as N
    from lmcache_b200.codec import CacheGenCodec, KvView
    codec = CacheGenCodec(MODEL)
    Ln, T, cs = 6, 700, 256
    g = torch.Generator(device="cuda").manual_seed(3)
    blob = (torch.rand((Ln, 2, T, H, D), device="cuda", generator=g) * 2 - 1).to(torch.bfloat16)
    view = KvView.from_blob(blob, "vllm")
    want = codec.encode_to_host(view, 0, T, cs)
    n, last = 3, T - 2 * cs
    lib = N.lib()
    lo = N.container_layout(Ln, H, D, cs, N.CODER_RANS_COMPACT)
    stride = (lo.off_payload + 15) & ~15
    arena = torch.empty(n * lo.max_total_bytes, dtype=torch.uint8, device="cuda")
    fixed = torch.full((n * stride,), 0xAB, dtype=torch.uint8, device="cuda")
    ws = torch.empty(lib.b200kv_encode_layers_workspace_bytes(Ln, H, D, cs, n, max(calls)), dtype=torch.uint8, device="cuda")
    from lmcache_b200.codec import PinnedBuffer
    seg, sizes = PinnedBuffer(16 * 2 * Ln * n), PinnedBuffer(8 * n)
    plan = N.EncodePlan()
    s = torch.cuda.current_stream().cuda_stream
    N.check(lib.b200kv_encode_layers_plan(ctypes.byref(view.desc), 0, n, cs, last, codec._kb, codec._vb,
                                          N.CODER_RANS_COMPACT, arena.data_ptr(), arena.numel(), fixed.data_ptr(), stride,
                                          seg.dev_ptr, sizes.dev_ptr, max(calls), ws.data_ptr(), ws.numel(),
                                          ctypes.byref(plan), s))
    a = 0
    for c in calls:
        N.check(lib.b200kv_encode_layers(ctypes.byref(plan), a, a + c, s))
        assert lib.b200kv_encode_layers(ctypes.byref(plan), a, a + 1, s) < 0        # a layer is encoded once
        a += c
    N.check(lib.b200kv_encode_layers_finish(ctypes.byref(plan), s))
    torch.cuda.synchronize()
    sz = list((ctypes.c_uint64 * n).from_address(sizes.host_ptr))
    rows = np.frombuffer(seg.view(), dtype=np.int64, count=n * 2 * Ln * 2).reshape(n, 2 * Ln, 2)
    fx, ar = fixed.cpu().numpy(), arena.cpu().numpy()
    for j in range(n):
        lj = N.container_layout(Ln, H, D, cs if j < n - 1 else last, N.CODER_RANS_COMPACT)
        got = bytes(fx[j * stride: j * stride + lj.off_payload]) + b"".join(
            bytes(ar[o: o + m]) for o, m in rows[j])
        assert sz[j] == len(want[j]) and got == want[j], j
