"""GPU: layer-by-layer store and retrieve on the raw cpu and cuda tiers, and the mover calls they rest on
(b200kv_pack_chunks_layers / b200kv_unpack_chunks_layers).  The kernels are compared byte for byte with
b200kv_pack_chunks / b200kv_unpack_chunks, the tiers with store / store_paged / retrieve / retrieve_paged."""
import ctypes
import random

import numpy as np
import pytest
import torch

from test_gpu_host_tier import MODEL

pytestmark = pytest.mark.gpu
L, H, D = 4, 2, 64
DTYPES = [torch.bfloat16, torch.float16, torch.uint8, torch.float8_e4m3fn, torch.float8_e5m2]
KINDS = ["blob", "tuple", "hf", "paged", "latent"]


def _rand(shape, dtype, gen):
    es = torch.empty((), dtype=dtype).element_size()
    n = int(np.prod(shape))
    return torch.randint(0, 256, (n * es,), dtype=torch.uint8, device="cuda", generator=gen).view(dtype).view(shape)


def _kv(kind, T, dtype, seed=0, fill=None):
    """(view, planes): a KvView of `kind` over fresh KV, and its planes as [rows, bytes] uint8 views (plane kv*L + l;
    a paged plane's rows are cache slots).  fill: every byte of the KV (a sentinel) instead of random bytes"""
    from lmcache_b200.codec import KvView
    g = torch.Generator(device="cuda").manual_seed(seed)

    def make(shape):
        if fill is None:
            return _rand(shape, dtype, g)
        es = torch.empty((), dtype=dtype).element_size()
        return torch.full((int(np.prod(shape)) * es,), fill, dtype=torch.uint8, device="cuda").view(dtype).view(shape)
    b = lambda x: x.contiguous().view(torch.uint8).reshape(x.shape[0], -1) if x.is_contiguous() else None  # noqa: E731
    if kind == "blob":
        blob = make((L, 2, T, H, D))
        return KvView.from_blob(blob, "vllm"), [blob[l, kv].view(torch.uint8).reshape(T, -1)
                                                for kv in range(2) for l in range(L)]
    if kind == "hf":
        blob = make((L, 2, H, T, D))
        return KvView.from_blob(blob, "huggingface"), [blob[l, kv].view(torch.uint8).transpose(0, 1).reshape(T, -1)
                                                       for kv in range(2) for l in range(L)]
    if kind == "tuple":
        kv = [(make((T, H, D)), make((T, H, D))) for _ in range(L)]
        return KvView.from_tuple(kv, "vllm"), [b(kv[l][k]) for k in range(2) for l in range(L)]
    if kind == "latent":
        blob = make((L, T, 2 * D))
        return KvView.from_blob(blob, "vllm"), [blob[l].view(torch.uint8) for l in range(L)]
    nslots = (T // 16 + 3) * 16
    slots = torch.randperm(nslots, device="cuda", generator=g)[:T]
    caches = [(make((nslots // 16, 16, H, D)), make((nslots // 16, 16, H, D))) for _ in range(L)]
    return KvView.from_paged(caches, slots), [caches[l][k].view(torch.uint8).reshape(nslots, -1)
                                               for k in range(2) for l in range(L)]


def _table(ptrs):
    return torch.tensor(np.asarray(ptrs, dtype=np.uint64).view(np.int64), device="cuda")


def _slices(view, tok_begin, cs):
    n_tok = view.ntokens - tok_begin
    n = (n_tok + cs - 1) // cs
    sizes = [min(cs, n_tok - j * cs) for j in range(n)]
    row = view.planes // view.L * view.H * view.D * view.dtype.itemsize
    return sizes, row


def _pack_layers(view, tok_begin, cs, ranges, buf, stride):
    """pack_chunks_layers over `ranges` into a buffer laid out as pack_chunks lays it out (chunk j at j * stride)"""
    from lmcache_b200 import _native as N
    sizes, row = _slices(view, tok_begin, cs)
    for lb, le in ranges:
        t = _table([buf.data_ptr() + j * stride + lb * t * row for j, t in enumerate(sizes)])
        N.check(N.lib().b200kv_pack_chunks_layers(ctypes.byref(view.desc), tok_begin, len(sizes), cs, sizes[-1],
                                                  int(view.fmt == "huggingface"), lb, le, ctypes.c_void_p(t.data_ptr()),
                                                  torch.cuda.current_stream().cuda_stream))


def _partition(rng):
    cuts = sorted(rng.sample(range(1, L), rng.randint(0, L - 1)))
    b = [0] + cuts + [L]
    return list(zip(b, b[1:]))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", KINDS)
def test_pack_layers_gives_pack_chunks_bytes(kind, dtype):
    T, cs, tok_begin = 700, 256, 37                                   # ragged last chunk
    view, _ = _kv(kind, T, dtype, seed=1)
    want, _ = view.pack_chunks(tok_begin, cs)
    want = want.view(torch.uint8)
    sizes, row = _slices(view, tok_begin, cs)
    stride = L * row * cs
    blob = torch.zeros(want.numel(), dtype=torch.bool, device="cuda")      # the bytes of the chunk blobs
    for j, t in enumerate(sizes):
        blob[j * stride: j * stride + L * row * t] = True

    def check(got, what):
        assert torch.equal(got[blob], want[blob]), what
        assert bool((got[~blob] == 0x5A).all()), what                     # nothing past a blob is written
    rng = random.Random(hash((kind, str(dtype))))
    for ranges in ([(0, L)], [(l, l + 1) for l in range(L)], _partition(rng)):
        got = torch.full_like(want, 0x5A)
        _pack_layers(view, tok_begin, cs, ranges, got, stride)
        torch.cuda.synchronize()
        check(got, ranges)
    # a chunk pointer that is not 16-byte aligned takes the element path; the bytes are the same
    es = view.dtype.itemsize
    raw = torch.full((want.numel() + 16,), 0x5A, dtype=torch.uint8, device="cuda")
    mis = raw[es:es + want.numel()]
    _pack_layers(view, tok_begin, cs, [(0, 1), (1, L)], mis, stride)
    torch.cuda.synchronize()
    check(mis, "misaligned")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", KINDS)
def test_unpack_layers_writes_only_its_rows_and_planes(kind, dtype):
    from lmcache_b200 import _native as N
    T, cs, tok_begin = 700, 256, 37
    src, _ = _kv(kind, T, dtype, seed=2)
    packed, _ = src.pack_chunks(tok_begin, cs)
    sizes, row = _slices(src, tok_begin, cs)
    stride = L * row * cs
    ref, ref_planes = _kv(kind, T, dtype, seed=3, fill=0xC3)          # unpack_chunks of everything
    N.check(N.lib().b200kv_unpack_chunks(ctypes.c_void_p(packed.data_ptr()), stride, len(sizes), cs, sizes[-1],
                                         int(src.fmt == "huggingface"), ctypes.byref(ref.desc), tok_begin,
                                         torch.cuda.current_stream().cuda_stream))
    P = src.planes
    ppl = P // L
    es = src.dtype.itemsize
    for lb, le, shift in ((1, 3, 0), (0, L, 0), (L - 1, L, es)):       # shift: a table entry off 16-byte alignment
        dst, planes = _kv(kind, T, dtype, seed=3, fill=0xC3)
        sentinel = [p.clone() for p in planes]
        blob = torch.empty(packed.numel() * es + 16, dtype=torch.uint8, device="cuda")[shift:shift + packed.numel() * es]
        blob.copy_(packed.view(torch.uint8))
        t = _table([blob.data_ptr() + j * stride + lb * t * row for j, t in enumerate(sizes)])
        N.check(N.lib().b200kv_unpack_chunks_layers(ctypes.c_void_p(t.data_ptr()), len(sizes), cs, sizes[-1],
                                                    int(src.fmt == "huggingface"), lb, le, ctypes.byref(dst.desc),
                                                    tok_begin, torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        for p in range(P):
            inside = lb <= p % L < le
            assert torch.equal(planes[p], ref_planes[p] if inside else sentinel[p]), (lb, le, p)
        assert ppl in (1, 2)


def test_layers_calls_refuse_bad_arguments():
    from lmcache_b200 import _native as N
    view, _ = _kv("blob", 300, torch.bfloat16)
    buf = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    t = _table([buf.data_ptr(), buf.data_ptr() + (1 << 19)])
    s = torch.cuda.current_stream().cuda_stream
    lib = N.lib()
    tp = ctypes.c_void_p(t.data_ptr())
    for args in [(None, 0, L), (tp, -1, L), (tp, 2, 2), (tp, 3, 1), (tp, 0, L + 1)]:
        assert lib.b200kv_pack_chunks_layers(ctypes.byref(view.desc), 0, 2, 256, 44, 0, args[1], args[2], args[0], s) < 0
        assert lib.b200kv_unpack_chunks_layers(args[0], 2, 256, 44, 0, args[1], args[2], ctypes.byref(view.desc), 0, s) < 0
    for n, ct, lt in [(0, 256, 44), (2, 0, 1), (2, 256, 300), (2, 256, 0)]:       # the chunkings pack_chunks refuses
        assert lib.b200kv_pack_chunks_layers(ctypes.byref(view.desc), 0, n, ct, lt, 0, 0, L, tp, s) < 0
        assert lib.b200kv_unpack_chunks_layers(tp, n, ct, lt, 0, 0, L, ctypes.byref(view.desc), 0, s) < 0
    assert lib.b200kv_pack_chunks_layers(None, 0, 2, 256, 44, 0, 0, L, tp, s) < 0
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- the tiers
def _engine(autorelease, device, cs, fmt="vllm", mla=False):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    return autorelease(LMCacheEngine(LMCacheEngineConfig(cs, device, None, None, False, False, None),
                                     LMCacheEngineMetadata(MODEL, 1, 0, fmt, "bfloat16", mla)))


def _tuple_kv(T, fmt, dtype, seed, mla=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if mla:
        return tuple(_rand((T, 2 * D), dtype, g) for _ in range(L))
    shape = (T, H, D) if fmt == "vllm" else (H, T, D)
    return tuple((_rand(shape, dtype, g), _rand(shape, dtype, g)) for _ in range(L))


def _bytes(ret):
    out = []
    for x in ret:
        out += list(x) if isinstance(x, tuple) else [x]
    return [t.contiguous().view(torch.uint8) for t in out]


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(_bytes(a), _bytes(b)):
        assert torch.equal(x, y)


def _per_layer(r):
    evs = [r._upload.ready(l) for l in range(r.num_layers)]
    assert len({id(e) for e in evs}) == r.num_layers                 # one event per layer, not one for all


@pytest.mark.parametrize("device", ["cpu", "cuda"])
@pytest.mark.parametrize("cs", [256, 1024])
@pytest.mark.parametrize("fmt,dtype,mla", [("vllm", torch.bfloat16, False), ("huggingface", torch.float16, False),
                                           ("vllm", torch.float8_e4m3fn, False), ("vllm", torch.bfloat16, True)])
@pytest.mark.parametrize("case", ["full", "suffix", "partial"])
def test_retrieve_layerwise_equals_retrieve(device, cs, fmt, dtype, mla, case, autorelease):
    T = 2 * cs + 300
    eng = _engine(autorelease, device, cs, fmt, mla)
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    kv = _tuple_kv(T, fmt, dtype, seed=cs, mla=mla)
    if case == "partial":                                            # the first chunk and a half only
        n = cs + cs // 2
        cut = tuple(x[:n] for x in kv) if mla else \
            tuple((k[:n], v[:n]) if fmt == "vllm" else (k[:, :n], v[:, :n]) for k, v in kv)
        eng.store(tokens[:n], cut)
    else:
        eng.store(tokens, kv)
    mask = None
    if case == "suffix":                                             # the mask straddles the first chunk
        mask = torch.ones(T, dtype=torch.bool)
        mask[:cs // 2 + 3] = False
    want, want_mask = eng.retrieve(tokens, mask)
    r = eng.retrieve_layerwise(tokens, mask)
    assert torch.equal(r.ret_mask, want_mask)
    _per_layer(r)
    side = torch.cuda.Stream()
    got = []
    for l in range(L):                                               # layer l is final once waited for
        r.wait_layer(l, side)
        with torch.cuda.stream(side):
            x = r.kv[l]
            got.append(x.clone() if mla else (x[0].clone(), x[1].clone()))
    side.synchronize()
    _same(got, want)
    r.synchronize()
    _same(r.kv, want)


@pytest.mark.parametrize("device", ["cpu", "cuda"])
@pytest.mark.parametrize("cs,dtype,mla,skip", [(256, torch.bfloat16, False, 0), (1024, torch.float8_e4m3fn, False, 300),
                                               (256, torch.bfloat16, True, 0)])
def test_retrieve_paged_layerwise_equals_retrieve_paged(device, cs, dtype, mla, skip, autorelease):
    T, bs = 2 * cs + 300, 16
    eng = _engine(autorelease, device, cs, mla=mla)
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    kv = _tuple_kv(T, "vllm", dtype, seed=7, mla=mla)
    eng.store(tokens, kv)
    nblk = T // bs + 8
    slots = torch.randperm(nblk * bs, device="cuda")[:T]
    mask = None
    if skip:
        mask = torch.ones(T, dtype=torch.bool)
        mask[:skip] = False

    def caches():
        def one():
            es = torch.empty((), dtype=dtype).element_size()
            shape = (nblk, bs, 2 * D) if mla else (nblk, bs, H, D)
            return torch.full((int(np.prod(shape)) * es,), 0x77, dtype=torch.uint8, device="cuda").view(dtype).view(shape)
        return [one() for _ in range(L)] if mla else [(one(), one()) for _ in range(L)]
    a, b = caches(), caches()
    want_mask = eng.retrieve_paged(tokens, a, slots, mask)
    r = eng.retrieve_paged_layerwise(tokens, b, slots, mask)
    assert torch.equal(r.ret_mask, want_mask)
    _per_layer(r)
    r.synchronize()
    _same(b, a)


def _stored(eng):
    """key -> bytes of every stored blob"""
    from lmcache_b200.storage_backend.local_backend import _HostEntry
    out = {}
    for k, v in eng.engine_.dict.items():
        if isinstance(v, _HostEntry):
            v.wait()
            v = v.host
        out[k] = v.contiguous().view(torch.uint8).cpu()
    return out


@pytest.mark.parametrize("device", ["cpu", "cuda"])
@pytest.mark.parametrize("cs,fmt,dtype,mla", [(256, "vllm", torch.bfloat16, False), (1024, "vllm", torch.float8_e4m3fn, False),
                                              (256, "huggingface", torch.float16, False), (256, "vllm", torch.bfloat16, True)])
def test_store_layerwise_stores_store_bytes(device, cs, fmt, dtype, mla, autorelease):
    T = 3 * cs + 77
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    kv = _tuple_kv(T, fmt, dtype, seed=11, mla=mla)
    ref = _engine(autorelease, device, cs, fmt, mla)
    ref.store(tokens, kv)
    want = _stored(ref)
    for seed in range(2):
        eng = _engine(autorelease, device, cs, fmt, mla)
        h = eng.store_layerwise(tokens, kv)
        order = list(range(L))
        random.Random(seed).shuffle(order)
        for l in order:
            h.save_layer(l)
        h.finish()
        torch.cuda.current_stream().synchronize()
        got = _stored(eng)
        assert got.keys() == want.keys()
        for k in want:
            assert torch.equal(got[k], want[k])
        r = eng.retrieve_layerwise(tokens)                            # and the stored blobs serve a retrieve
        r.synchronize()
        assert int(r.ret_mask.sum()) == T


@pytest.mark.parametrize("device", ["cpu", "cuda"])
@pytest.mark.parametrize("dtype,mla", [(torch.bfloat16, False), (torch.float8_e5m2, False), (torch.bfloat16, True)])
def test_store_paged_layerwise_stores_store_paged_bytes(device, dtype, mla, autorelease):
    cs, T, bs = 256, 900, 16
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    kv = _tuple_kv(T, "vllm", dtype, seed=5, mla=mla)
    nblk = T // bs + 8
    slots = torch.randperm(nblk * bs, device="cuda")[:T]
    es = torch.empty((), dtype=dtype).element_size()
    shape = (nblk, bs, 2 * D) if mla else (nblk, bs, H, D)
    new = lambda: torch.zeros((int(np.prod(shape)) * es,), dtype=torch.uint8, device="cuda").view(dtype).view(shape)  # noqa: E731
    caches = [new() for _ in range(L)] if mla else [(new(), new()) for _ in range(L)]

    def write(l):
        if mla:
            caches[l].view(-1, 2 * D)[slots] = kv[l]
        else:
            caches[l][0].view(-1, H, D)[slots] = kv[l][0]
            caches[l][1].view(-1, H, D)[slots] = kv[l][1]
    ref = _engine(autorelease, device, cs, mla=mla)
    pre = _engine(autorelease, device, cs, mla=mla)
    pre.store(tokens[:cs], tuple(x[:cs] for x in kv) if mla else tuple((k[:cs], v[:cs]) for k, v in kv))
    kept = {k: v for k, v in pre.engine_.dict.items()}
    h = pre.store_paged_layerwise(tokens, caches, slots)             # skip_existing: chunk 0 is there already
    for l in (3, 0, 2, 1):
        write(l)
        h.save_layer(l)
    h.finish()
    for l in range(L):                                               # overwritten after finish(), in stream order
        (caches[l] if mla else caches[l][0]).zero_()
    torch.cuda.current_stream().synchronize()
    for l in range(L):
        write(l)
    ref.store_paged(tokens, caches, slots)
    want, got = _stored(ref), _stored(pre)
    assert got.keys() == want.keys()
    for k in want:
        assert torch.equal(got[k], want[k])
        if k in kept:
            assert pre.engine_.dict[k] is kept[k]                    # not stored again
    with pytest.raises(ValueError):
        h2 = ref.store_paged_layerwise(tokens, caches, slots, skip_existing=False)
        h2.save_layer(0)
        h2.save_layer(0)


def test_hybrid_with_raw_local_tier_retrieves_layerwise():
    from test_gpu_remote_layerwise import _Native

    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    srv = _Native()
    eng = None
    try:
        cfg = LMCacheEngineConfig(256, "cpu", f"lm://127.0.0.1:{srv.port}", "lossless", False, False, None)
        eng = LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16"))
        T = 1100
        tokens = torch.randint(0, 32000, (T,), device="cuda")
        eng.store(tokens, _tuple_kv(T, "vllm", torch.bfloat16, seed=9))
        want, want_mask = eng.retrieve(tokens)
        r = eng.retrieve_layerwise(tokens)
        assert torch.equal(r.ret_mask, want_mask) and int(want_mask.sum()) == T
        _per_layer(r)
        r.synchronize()
        _same(r.kv, want)
    finally:
        if eng is not None:
            eng.close()
        srv.stop()
