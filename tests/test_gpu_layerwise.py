"""GPU: layer-by-layer retrieve (LMCacheEngine.retrieve_layerwise / retrieve_paged_layerwise) and the decode it rests on
(b200kv_decode_plan + b200kv_decode_layers).  Everything is compared bit for bit with retrieve() / retrieve_paged() /
b200kv_decode_chunks, which the other GPU tests hold to the reference decode."""
import random
import time

import numpy as np
import pytest
import torch

from test_gpu_host_tier import MODEL, _blob_of, _kv, _meta, _want

pytestmark = pytest.mark.gpu


def _cfg(cs, backend="cpu", capacity=None):
    from lmcache_b200.config import LMCacheEngineConfig
    return LMCacheEngineConfig.from_legacy(chunk_size=cs, backend=backend, local_serde="cachegen",
                                           local_capacity_bytes=capacity)


def _bits(x):
    return x.contiguous().view(torch.int16)


@pytest.mark.parametrize("tier", ["host", "disk"])
@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
@pytest.mark.parametrize("cs", [256, 100])
@pytest.mark.parametrize("masked", [False, True])
def test_layerwise_equals_retrieve(tier, fmt, cs, masked, tmp_path, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    backend = "cpu" if tier == "host" else "file://" + str(tmp_path / "kv") + "/"
    engine = autorelease(LMCacheEngine(_cfg(cs, backend), _meta(fmt)))
    T = 1100
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    kv = _kv(T, fmt, seed=4)
    engine.store(tokens[:900], tuple((k[:900], v[:900]) if fmt == "vllm" else (k[:, :900], v[:, :900]) for k, v in kv))
    mask = None
    if masked:
        mask = torch.ones(T, dtype=torch.bool)
        mask[:cs + 37] = False                     # the first retrieved chunk straddles the mask
    ref, ref_mask = engine.retrieve(tokens, mask)
    r = engine.retrieve_layerwise(tokens, mask)
    assert r.num_layers == len(kv)
    r.synchronize()
    torch.cuda.synchronize()
    assert torch.equal(r.ret_mask, ref_mask) and int(ref_mask.sum()) > 0
    assert len(r.kv) == len(ref)
    assert torch.equal(_bits(_blob_of(r.kv)), _bits(_blob_of(ref)))


def test_layerwise_total_miss(autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    engine = autorelease(LMCacheEngine(_cfg(256), _meta()))
    tokens = torch.randint(0, 32000, (600,), device="cuda")
    r = engine.retrieve_layerwise(tokens)
    r.synchronize()
    assert not bool(r.ret_mask.any()) and len(r.kv) == 0


@pytest.mark.parametrize("skip", [0, 300])
def test_paged_layerwise_equals_retrieve_paged(skip, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    cs, T, L, H, D, bs = 256, 1000, 6, 2, 128, 16
    engine = autorelease(LMCacheEngine(_cfg(cs), _meta()))
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    kv = _kv(T, "vllm", L=L, H=H, D=D, seed=6)
    engine.store(tokens[:800], tuple((k[:800], v[:800]) for k, v in kv))
    nblk = (T + bs - 1) // bs + 8
    slots = torch.randperm(nblk * bs, device="cuda")[:T]
    mask = None
    if skip:
        mask = torch.ones(T, dtype=torch.bool)
        mask[:skip] = False                        # 300 = chunk 1 + 44 tokens: chunk 1 straddles the mask
    caches = []
    for _ in range(2):
        g = torch.Generator(device="cuda").manual_seed(9)
        caches.append([(torch.randn((nblk, bs, H, D), device="cuda", generator=g).to(torch.bfloat16),
                        torch.randn((nblk, bs, H, D), device="cuda", generator=g).to(torch.bfloat16)) for _ in range(L)])
    before = [(k.clone(), v.clone()) for k, v in caches[1]]
    want_mask = engine.retrieve_paged(tokens, caches[0], slots, mask)
    r = engine.retrieve_paged_layerwise(tokens, caches[1], slots, mask)
    assert r.kv is None and r.num_layers == L
    r.synchronize()
    torch.cuda.synchronize()
    assert torch.equal(r.ret_mask, want_mask)
    for (k0, v0), (k1, v1) in zip(caches[0], caches[1]):
        assert torch.equal(_bits(k0), _bits(k1)) and torch.equal(_bits(v0), _bits(v1))
    got = int(want_mask.sum())
    assert got == 768 - skip                       # chunk 3 was stored as a 32-token tail: a different key
    untouched = torch.ones(nblk * bs, dtype=torch.bool, device="cuda")
    untouched[slots[want_mask.cuda()]] = False
    for (k1, v1), (kb, vb) in zip(caches[1], before):
        assert torch.equal(_bits(k1.view(-1, H, D)[untouched]), _bits(kb.view(-1, H, D)[untouched]))
        assert torch.equal(_bits(v1.view(-1, H, D)[untouched]), _bits(vb.view(-1, H, D)[untouched]))


def test_wait_layer_orders_a_side_stream(autorelease):
    """wait_layer(l) on a fresh stream, then a copy of layer l on that stream -- no device-wide synchronisation"""
    from lmcache_b200.cache_engine import LMCacheEngine
    L, T = 8, 2048
    engine = autorelease(LMCacheEngine(_cfg(256), _meta()))
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    kv = _kv(T, "vllm", L=L, seed=8)
    engine.store(tokens, kv)
    torch.cuda.synchronize()
    want = _want(kv, "vllm", 256, T)
    r = engine.retrieve_layerwise(tokens)
    copies = []
    for layer in random.Random(0).sample(range(L), L):
        s = torch.cuda.Stream()
        r.wait_layer(layer, s)
        with torch.cuda.stream(s):
            copies.append((layer, s, r.kv[layer][0].clone(), r.kv[layer][1].clone()))
    for layer, s, k, v in copies:
        s.synchronize()
        assert torch.equal(_bits(k), _bits(want[layer, 0])) and torch.equal(_bits(v), _bits(want[layer, 1])), layer


# ---------------------------------------------------------------------------------------------- ABI level
def _containers(kind, L=8, H=4, D=128, T=700, cs=256):
    """(codec, container bytes, their 16-byte aligned offsets in a staging buffer, its size, kv, chunk size) at a low
    (peaked) or high (uniform) entropy"""
    from lmcache_b200.codec import CacheGenCodec, KvView
    g = torch.Generator(device="cuda").manual_seed(5)
    if kind == "peaked":
        kv = torch.randn((L, 2, T, H, D), device="cuda", generator=g) * 0.05
        kv[:, :, :, :, 0] = 4.0
    else:
        kv = torch.rand((L, 2, T, H, D), device="cuda", generator=g) * 2 - 1
    kv = kv.to(torch.bfloat16)
    codec = CacheGenCodec(MODEL)
    blobs = [bytes(b) for b in codec.encode_to_host(KvView.from_blob(kv, "vllm"), 0, T, cs)]
    fixed = codec.layout(L, H, D, cs).fixed_bytes
    bps = 8.0 * sum(len(b) - fixed for b in blobs) / kv.numel()
    assert (bps < 1.0) if kind == "peaked" else (bps > 4.0), bps       # the two table layouts (rows / transposed)
    offs, o = [], 0
    for b in blobs:
        offs.append(o)
        o += (len(b) + 15) & ~15
    return codec, blobs, offs, o, kv, cs


def _stage(blobs, offs, total):
    host = np.zeros(total + 640, np.uint8)
    for b, o in zip(blobs, offs):
        host[o:o + len(b)] = np.frombuffer(b, np.uint8)
    return torch.from_numpy(host).cuda()


def _plan(codec, dev, blobs, offs, out, cs, status, stream):
    from lmcache_b200.codec import KvView, parse_header
    hd = parse_header(blobs[0])
    return codec.decode_plan(dev.data_ptr(), dev.numel(), offs, [len(b) for b in blobs],
                             [int(parse_header(b).ntokens) for b in blobs], KvView.from_blob(out, "vllm"),
                             [j * cs for j in range(len(blobs))], int(hd.max_dtype), int(hd.version) - 1, stream,
                             status.data_ptr())


@pytest.mark.parametrize("kind", ["peaked", "uniform"])
def test_plan_and_layers_equal_decode_chunks(kind):
    from lmcache_b200.codec import KvView
    codec, blobs, offs, total, kv, cs = _containers(kind)
    L = kv.shape[0]
    dev = _stage(blobs, offs, total)
    want = torch.zeros_like(kv)
    codec.decode(blobs, KvView.from_blob(want, "vllm"), [j * cs for j in range(len(blobs))])
    torch.cuda.synchronize()
    assert codec.decode_status() == [0] * len(blobs)
    order = list(range(L))
    random.Random(1).shuffle(order)
    splits = {"all": [(0, L)], "one_by_one_shuffled": [(l, l + 1) for l in order], "uneven": [(0, 3), (3, 4), (4, L)]}
    s = torch.cuda.current_stream()
    for name, ranges in splits.items():
        out = torch.zeros_like(kv)
        status = torch.full((len(blobs),), 7, dtype=torch.int32, device="cuda")
        plan, ws = _plan(codec, dev, blobs, offs, out, cs, status, s)
        for a, b in ranges:
            codec.decode_layers(plan, a, b, s)
        torch.cuda.synchronize()
        assert torch.equal(_bits(out), _bits(want)), name
        assert status.tolist() == [0] * len(blobs), name


@pytest.mark.parametrize("kind", ["peaked", "uniform"])
def test_layer_major_upload_ignores_bytes_past_each_range(kind):
    """only the fixed sections, then layer by layer only that layer's two planes, are in place when the layer is decoded;
    every other byte of the staging buffer -- later planes, the gaps and the read slack -- is 0xFF"""
    from lmcache_b200.codec import KvView, parse_header, plane_offsets
    from lmcache_b200.pipeline import layer_copy_ranges
    codec, blobs, offs, total, kv, cs = _containers(kind)
    L = kv.shape[0]
    want = torch.zeros_like(kv)
    codec.decode(blobs, KvView.from_blob(want, "vllm"), [j * cs for j in range(len(blobs))])
    po = [plane_offsets(b) for b in blobs]
    assert all(p is not None for p in po)
    fixed, start, size = layer_copy_ranges(po, [len(b) for b in blobs], L)
    n = len(blobs)
    host = np.zeros(total, np.uint8)
    for b, o in zip(blobs, offs):
        host[o:o + len(b)] = np.frombuffer(b, np.uint8)
    host_t = torch.from_numpy(host).pin_memory()
    dev = torch.full((total + 640,), 0xFF, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream()
    for j in range(n):
        dev[offs[j]:offs[j] + fixed[j]].copy_(host_t[offs[j]:offs[j] + fixed[j]])
    out = torch.zeros_like(kv)
    status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    plan, ws = _plan(codec, dev, blobs, offs, out, cs, status, s)
    for layer in range(L):
        for k in range(2 * n):
            j = k % n
            a, z = offs[j] + int(start[layer, k]), offs[j] + int(start[layer, k] + size[layer, k])
            dev[a:z].copy_(host_t[a:z])
        codec.decode_layers(plan, layer, layer + 1, s)
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(want))
    assert status.tolist() == [0] * n


def test_multi_group_chunks_take_the_fallback(autorelease):
    """chunk_size 512: version-2 containers of two groups; retrieve_layerwise is retrieve() plus one event"""
    from lmcache_b200.cache_engine import LMCacheEngine
    engine = autorelease(LMCacheEngine(_cfg(512), _meta()))
    T = 1300
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    kv = _kv(T, "vllm", seed=12)
    engine.store(tokens, kv)
    ref, ref_mask = engine.retrieve(tokens)
    r = engine.retrieve_layerwise(tokens)
    r.synchronize()
    assert torch.equal(r.ret_mask, ref_mask) and int(ref_mask.sum()) == T
    assert torch.equal(_bits(_blob_of(r.kv)), _bits(_blob_of(ref)))
    assert r._upload.ready(0) is r._upload.ready(len(kv) - 1)


def test_bounded_tier_evicting_during_layerwise_retrieve(autorelease):
    """stores that must evict the retrieved sequence's own chunks are issued while its layer-wise upload is in flight
    (before synchronize): pins until the last copy is enqueued, then DeferredFree until that copy has run, keep every
    block alive under its upload, so the retrieve decodes bit-exact"""
    from lmcache_b200.cache_engine import LMCacheEngine
    from test_gpu_eviction import CS, T, _cfg as _evict_cfg, _held, _keys, _seq, _seq_bytes
    cap = int(2.5 * _seq_bytes()[0])
    engine = autorelease(LMCacheEngine(_evict_cfg(cap), _meta()))
    (ta, ka), (tb, kb), (tc, kc), (td, kd) = (_seq(70 + i) for i in range(4))
    want = _want(ka, "vllm", CS, T)
    engine.store(ta, ka)
    engine.store(tb, kb)
    torch.cuda.synchronize()
    # A's copies are queued behind a ~0.1 s sleep kernel on the uploader's copy stream: the worker enqueues them and
    # unpins A at once, but they cannot run before the stores below have evicted A's tail and landed their own
    # containers -- unless the tier waits for them (DeferredFree), which is what is tested
    be = engine.engine_
    with torch.cuda.stream(be._layerwise_uploader(torch.device("cuda", 0)).copy_stream):
        torch.cuda._sleep(200_000_000)
    r = engine.retrieve_layerwise(ta)               # touches A: B is now the coldest chain, then A
    entries = [be.dict[k] for k in _keys(engine, ta)]
    for _ in range(10_000):                         # the worker unpins A once its last copy is enqueued
        if not any(e.pins for e in entries):
            break
        time.sleep(0.001)
    assert not any(e.pins for e in entries)
    engine.store(tc, kc)
    engine.store(td, kd)                            # evicts the rest of B, then A's tail
    assert _held(engine, ta) < T // CS and engine.engine_.evicted > 0
    r.synchronize()
    assert int(r.ret_mask.sum()) == T
    assert torch.equal(_bits(_blob_of(r.kv)), _bits(want))


def test_total_miss_on_a_fresh_engine_waits_for_nothing(autorelease):
    """a retrieve-only replica that has never seen a chunk does not know L: num_layers is 0 and wait_layer is a no-op"""
    from lmcache_b200.cache_engine import LMCacheEngine
    engine = autorelease(LMCacheEngine(_cfg(256), _meta()))
    r = engine.retrieve_layerwise(torch.randint(0, 32000, (600,), device="cuda"))
    assert r.num_layers == 0 and not bool(r.ret_mask.any())
    for layer in range(4):
        r.wait_layer(layer)
    r.synchronize()


def test_device_plane_offsets_equal_the_host_ones(autorelease):
    """the offsets land() reads on the device match the host-side computation, and a damaged container gets none"""
    import ctypes

    from lmcache_b200 import _native as N
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.codec import plane_offsets
    engine = autorelease(LMCacheEngine(_cfg(256), _meta()))
    T = 1100
    engine.store(torch.randint(0, 32000, (T,), device="cuda"), _kv(T, "vllm", seed=13))
    recs = [e.rec for e in engine.engine_.dict.values()]
    assert len(recs) == 5
    for rec in recs:
        want = plane_offsets(rec.blk.view()[:rec.nbytes])
        assert want is not None and np.array_equal(rec.planes, want)
    # two containers on the device, the second with one damaged half-length byte
    raw = bytes(recs[0].blk.view()[:recs[0].nbytes])
    stride = (len(raw) + 15) & ~15
    lo = N.container_layout(recs[0].L, recs[0].H, recs[0].D, recs[0].ntokens, N.CODER_RANS_COMPACT)
    bad = bytearray(raw)
    bad[lo.off_lengths] ^= 1
    host = np.zeros(2 * stride, np.uint8)
    host[:len(raw)] = np.frombuffer(raw, np.uint8)
    host[stride:stride + len(raw)] = np.frombuffer(bytes(bad), np.uint8)
    dev = torch.from_numpy(host).cuda()
    out = torch.full((2, N.MAX_PLANES + 1), 7, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream()
    N.check(N.lib().b200kv_plane_offsets_device(ctypes.c_void_p(dev.data_ptr()), stride, 2, ctypes.c_void_p(out.data_ptr()),
                                                s.cuda_stream))
    got = out.cpu().numpy()
    assert np.array_equal(got[0, :2 * recs[0].L + 1], plane_offsets(raw)) and got[1, 0] == -1
