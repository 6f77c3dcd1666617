"""GPU: engine-level behaviour, mirroring the reference's tests/test_cache_engine.py / test_backends.py
(lossless round trips, prefix / mixed / suffix-mask semantics, device placement), plus the hash kernel and the
pack / mover primitives."""
import hashlib
import json
import os
import socket
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def dumb_metadata(fmt="vllm", model="test_model"):
    from lmcache_b200.config import LMCacheEngineMetadata
    return LMCacheEngineMetadata(model, 3, 123, fmt, "half")


def generate_kv_cache(num_tokens, fmt, device, num_layers=32, num_heads=8, head_size=128):
    shape = [num_tokens, num_heads, head_size] if fmt == "vllm" else [num_heads, num_tokens, head_size]
    dtype = torch.bfloat16 if fmt == "vllm" else torch.float16
    return tuple((torch.rand(shape, dtype=dtype, device=device), torch.rand(shape, dtype=dtype, device=device))
                 for _ in range(num_layers))


def generate_tokens(num_tokens, device):
    return torch.randint(0, 10000, size=[num_tokens]).to(device)


def concatenate_kv_caches(kv_chunks, fmt):
    dim = 1 if fmt == "huggingface" else 0
    return tuple((torch.cat([c[l][0] for c in kv_chunks], dim=dim), torch.cat([c[l][1] for c in kv_chunks], dim=dim))
                 for l in range(len(kv_chunks[0])))


def check_kv_cache_equal(left, right, num_tokens, fmt):
    for (lk, lv), (rk, rv) in zip(left, right):
        rk, rv = rk.to(lk.device), rv.to(lv.device)
        assert lk.dim() == 3 and rk.dim() == 3
        if fmt == "huggingface":
            assert (lk[:, :num_tokens, :] == rk[:, :num_tokens, :]).all()
            assert (lv[:, :num_tokens, :] == rv[:, :num_tokens, :]).all()
        else:
            assert (lk[:num_tokens] == rk[:num_tokens]).all()
            assert (lv[:num_tokens] == rv[:num_tokens]).all()


# ---------------------------------------------------------------- hash kernel (a1)
def test_gpu_hash_matches_reference_goldens():
    from lmcache_b200.cache_engine import sha256_prefix_chain
    h = json.load(open(os.path.join(HERE, "golden", "golden_hash.json")))
    rng = np.random.default_rng(1234)
    for c in h["cases"]:
        toks = np.arange(c["n"], dtype=c["dtype"]) if c["label"].startswith("arange") else \
            rng.integers(0, 32000, c["n"], dtype=np.int64)
        got = sha256_prefix_chain(torch.from_numpy(toks).cuda(), c["chunk_size"])
        assert got == c["hashes"], c["label"]
        assert sha256_prefix_chain(torch.from_numpy(toks), c["chunk_size"]) == c["hashes"]   # host tokens: uploaded


def test_gpu_hash_many_sequences_and_sizes():
    from lmcache_b200.cache_engine import sha256_prefix_chain
    rng = np.random.default_rng(7)
    lens = [4096] * 16 + [1, 255, 256, 257, 0, 1000]
    offs = np.concatenate([[0], np.cumsum(lens)])
    toks = rng.integers(0, 32000, offs[-1], dtype=np.int64)
    got = sha256_prefix_chain(torch.from_numpy(toks).cuda(), 256, [int(o) for o in offs])
    want = []
    for i in range(len(lens)):
        want += O.sha256_chain(toks[offs[i]:offs[i + 1]], 256)
    assert got == want
    # plain sha256 of arbitrary byte strings (chunk_size larger than the message -> single block chain)
    for n in [1, 55, 56, 63, 64, 65, 119, 120, 1000, 4097]:
        b = rng.integers(0, 256, n, dtype=np.uint8)
        assert sha256_prefix_chain(torch.from_numpy(b).cuda(), 1 << 20) == [hashlib.sha256(b.tobytes()).hexdigest()]


def test_full_size_chain_property():
    """65536 tokens / 256: checksum-of-checksums vs the oracle (size-independent property at BASELINE config 3)."""
    from lmcache_b200.cache_engine import sha256_prefix_chain
    toks = np.random.default_rng(3).integers(0, 32000, 65536, dtype=np.int64)
    got = sha256_prefix_chain(torch.from_numpy(toks).cuda(), 256)
    assert hashlib.sha256("".join(got).encode()).hexdigest() == \
        hashlib.sha256("".join(O.sha256_chain(toks, 256)).encode()).hexdigest()


# ---------------------------------------------------------------- pack / unpack / mover (a4, a14)
@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
def test_pack_unpack_match_reference_blob_ops(fmt):
    import ctypes

    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView
    L, H, D, T, cs = 5, 3, 64, 300, 128
    kv = generate_kv_cache(T, fmt, "cuda", L, H, D)
    # reference: stack/stack/stack/permute then split + contiguous (cache_engine.py:98-161)
    blob = torch.stack((torch.stack([k for k, _ in kv]), torch.stack([v for _, v in kv]))).permute(1, 0, 2, 3, 4)
    tdim = 2 if fmt == "vllm" else 3
    want = [x.contiguous() for x in torch.split(blob, cs, dim=tdim)]
    view = KvView.from_tuple(kv, fmt)
    per_tok = 2 * L * H * D
    buf = torch.zeros(3 * cs * per_tok, dtype=kv[0][0].dtype, device="cuda")
    N.check(N.lib().b200kv_pack_chunks(ctypes.byref(view.desc), 0, 3, cs, T - 2 * cs, int(fmt == "huggingface"),
                                       ctypes.c_void_p(buf.data_ptr()), cs * per_tok * 2,
                                       torch.cuda.current_stream().cuda_stream))
    for j, w in enumerate(want):
        got = buf[j * cs * per_tok: j * cs * per_tok + w.numel()].view(w.shape)
        assert torch.equal(got, w), j
    # scatter back into fresh tensors
    kv2 = tuple((torch.zeros_like(k), torch.zeros_like(v)) for k, v in kv)
    view2 = KvView.from_tuple(kv2, fmt)
    N.check(N.lib().b200kv_unpack_chunks(ctypes.c_void_p(buf.data_ptr()), cs * per_tok * 2, 3, cs, T - 2 * cs,
                                         int(fmt == "huggingface"), ctypes.byref(view2.desc), 0,
                                         torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    check_kv_cache_equal(kv2, kv, T, fmt)


def test_mover_primitives_roundtrip():
    import ctypes

    from lmcache_b200 import _native as N
    from lmcache_b200.codec import PinnedBuffer
    lib = N.lib()
    n = 1 << 20
    src = torch.randint(0, 255, (n,), dtype=torch.uint8, device="cuda")
    pin = PinnedBuffer(n)
    s, e0, e1 = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
    N.check(lib.b200kv_stream_create(ctypes.byref(s)))
    N.check(lib.b200kv_event_create(ctypes.byref(e0)))
    N.check(lib.b200kv_event_create(ctypes.byref(e1)))
    torch.cuda.synchronize()
    N.check(lib.b200kv_event_record(e0, s))
    N.check(lib.b200kv_copy_async(pin.host_ptr, src.data_ptr(), n, s))
    N.check(lib.b200kv_event_record(e1, s))
    N.check(lib.b200kv_event_sync(e1))
    assert lib.b200kv_event_query(e1) == 0
    ms = ctypes.c_float()
    N.check(lib.b200kv_event_elapsed_ms(e0, e1, ctypes.byref(ms)))
    assert ms.value >= 0
    assert bytes(pin.view()) == src.cpu().numpy().tobytes()
    dst = torch.zeros_like(src)
    N.check(lib.b200kv_copy_async(dst.data_ptr(), pin.host_ptr, n, s))
    # 2-D: rows of 1000 bytes at pitch 1024 -> packed
    packed = torch.zeros(1000 * 1000, dtype=torch.uint8, device="cuda")
    N.check(lib.b200kv_copy2d_async(packed.data_ptr(), 1000, src.data_ptr(), 1024, 1000, 1000, s))
    N.check(lib.b200kv_stream_sync(s))
    assert torch.equal(dst, src)
    assert torch.equal(packed.view(1000, 1000), src[:1024 * 1000].view(1000, 1024)[:, :1000])
    for ev in (e0, e1):
        N.check(lib.b200kv_event_destroy(ev))
    N.check(lib.b200kv_stream_destroy(s))
    pin.close()


# ---------------------------------------------------------------- engine (reference tests/test_cache_engine.py)
@pytest.mark.parametrize("src_device", ["cuda:0", "cuda", "cpu"])
@pytest.mark.parametrize("backend", ["cuda", "cpu"])
def test_retrieve_device(backend, src_device, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig
    tokens = generate_tokens(500, src_device)
    kv_cache = generate_kv_cache(500, "vllm", src_device)
    engine = autorelease(LMCacheEngine(LMCacheEngineConfig.from_legacy(chunk_size=256, backend=backend), dumb_metadata()))
    engine.store(tokens, kv_cache)
    retrieved, _ = engine.retrieve(tokens)
    for k, v in retrieved:
        assert k.device == torch.device("cuda:0") and v.device == torch.device("cuda:0")


@pytest.fixture(params=["fast", "generic"])
def engine_path(request, monkeypatch):
    """Run engine tests through both code paths: the native fast path (backend consumes the caller's KV tensors /
    fills one blob) and the generic per-chunk plugin path every third-party backend would take."""
    if request.param == "generic":
        from lmcache_b200.storage_backend.local_backend import LMCLocalBackend
        from lmcache_b200.storage_backend.remote_backend import LMCRemoteBackend
        monkeypatch.setattr(LMCLocalBackend, "supports_kv_view", lambda self: False)
        monkeypatch.setattr(LMCRemoteBackend, "supports_kv_view", lambda self: False)
    return request.param


@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
@pytest.mark.parametrize("backend", ["cuda", "cpu"])
@pytest.mark.parametrize("blocking", [True, False])
def test_same_retrieve_store(fmt, backend, blocking, autorelease, engine_path):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig
    device = "cpu" if backend == "cpu" else "cuda"
    num_tokens = 2000
    tokens = generate_tokens(num_tokens, device)
    kv_cache = generate_kv_cache(num_tokens, fmt, device)
    engine = autorelease(LMCacheEngine(LMCacheEngineConfig.from_legacy(chunk_size=256, backend=backend), dumb_metadata(fmt)))
    retrieved, ret_mask = engine.retrieve(tokens)
    assert len(retrieved) == 0 and torch.sum(ret_mask) == 0
    engine.store(tokens, kv_cache, blocking=blocking)
    retrieved, ret_mask = engine.retrieve(tokens)
    assert torch.sum(ret_mask) == num_tokens
    check_kv_cache_equal(retrieved, kv_cache, num_tokens, fmt)


@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
@pytest.mark.parametrize("chunk_size", [128, 256])
@pytest.mark.parametrize("backend", ["cuda", "cpu"])
def test_retrieve_prefix(fmt, chunk_size, backend, autorelease, engine_path):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig
    num_tokens, new_num_tokens = 2000, 1000
    tokens = generate_tokens(num_tokens, "cuda")
    kv_cache = generate_kv_cache(num_tokens, fmt, "cuda")
    new_tokens = generate_tokens(new_num_tokens, "cuda")
    engine = autorelease(LMCacheEngine(LMCacheEngineConfig.from_legacy(chunk_size=chunk_size, backend=backend),
                                       dumb_metadata(fmt)))
    engine.store(tokens, kv_cache)
    retrieved, ret_mask = engine.retrieve(torch.cat([tokens, new_tokens]))
    expected = (num_tokens // chunk_size) * chunk_size
    assert torch.sum(ret_mask) == expected
    check_kv_cache_equal(retrieved, kv_cache, expected, fmt)


@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
@pytest.mark.parametrize("chunk_size", [128, 256])
def test_mixed_retrieve(fmt, chunk_size, autorelease, engine_path):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig
    num_tokens, new_num_tokens = 2000, 1000
    tokens = generate_tokens(num_tokens, "cuda")
    kv_cache = generate_kv_cache(num_tokens, fmt, "cuda")
    new_tokens = generate_tokens(new_num_tokens, "cuda")
    new_kv_cache = generate_kv_cache(new_num_tokens, fmt, "cuda")
    engine = autorelease(LMCacheEngine(LMCacheEngineConfig.from_legacy(chunk_size=chunk_size, backend="cuda"),
                                       dumb_metadata(fmt)))
    engine.store(tokens, kv_cache)
    engine.store(new_tokens, new_kv_cache)
    retrieved, ret_mask = engine.retrieve(torch.cat([tokens, new_tokens]))
    expected = (num_tokens // chunk_size) * chunk_size
    assert torch.sum(ret_mask) == expected
    check_kv_cache_equal(retrieved, kv_cache, expected, fmt)
    retrieved, ret_mask = engine.retrieve(new_tokens)
    assert torch.sum(ret_mask) == new_num_tokens
    check_kv_cache_equal(retrieved, new_kv_cache, new_num_tokens, fmt)
    final_tokens = torch.cat([tokens, new_tokens])
    final_kv = concatenate_kv_caches([kv_cache, generate_kv_cache(new_num_tokens, fmt, "cuda")], fmt)
    engine.store(final_tokens, final_kv)
    retrieved, ret_mask = engine.retrieve(final_tokens)
    assert torch.sum(ret_mask) == num_tokens + new_num_tokens
    check_kv_cache_equal(retrieved, final_kv, num_tokens + new_num_tokens, fmt)


def test_golden_engine_semantics(autorelease, engine_path):
    """The scalars recorded from the reference engine in this container (tests/golden/golden_engine.json)."""
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig
    gold = json.load(open(os.path.join(HERE, "golden", "golden_engine.json")))
    engine = autorelease(LMCacheEngine(LMCacheEngineConfig.from_legacy(chunk_size=256, backend="cpu"), dumb_metadata()))
    T = 600
    tokens = torch.arange(T, dtype=torch.int64)
    kv = generate_kv_cache(T, "vllm", "cuda", 3, 2, 8)
    r0, m0 = engine.retrieve(tokens)
    assert (len(r0), int(m0.sum())) == (gold["empty_retrieve"]["n_layers"], gold["empty_retrieve"]["mask_sum"])
    engine.store(tokens, kv)
    r1, m1 = engine.retrieve(tokens)
    assert (int(m1.sum()), r1[0][0].shape[0]) == (gold["full_retrieve"]["mask_sum"], gold["full_retrieve"]["ntok"])
    check_kv_cache_equal(r1, kv, T, "vllm")
    longer = torch.cat([tokens, torch.arange(1000, 1400, dtype=torch.int64)])
    r2, m2 = engine.retrieve(longer)
    assert (int(m2.sum()), r2[0][0].shape[0]) == (gold["prefix_of_longer"]["mask_sum"], gold["prefix_of_longer"]["ntok"])
    nz = m2.nonzero()
    assert [int(nz[0]), int(nz[-1])] == gold["prefix_of_longer"]["mask_true_idx"]
    mask = torch.ones(T, dtype=torch.bool)
    mask[:300] = False
    r3, m3 = engine.retrieve(tokens, mask)
    assert (int(m3.sum()), r3[0][0].shape[0], int(m3.nonzero()[0])) == \
        (gold["suffix_mask_300"]["mask_sum"], gold["suffix_mask_300"]["ntok"], gold["suffix_mask_300"]["first_true"])
    assert torch.equal(r3[0][0], kv[0][0][300:])
    r4, m4 = engine.retrieve(torch.arange(5000, 5300, dtype=torch.int64))
    assert (len(r4), int(m4.sum())) == (gold["miss"]["n_layers"], gold["miss"]["mask_sum"])


def test_store_asserts_and_builder(autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine, LMCacheEngineBuilder
    from lmcache_b200.config import LMCacheEngineConfig
    cfg = LMCacheEngineConfig.from_legacy(chunk_size=256, backend="cuda")
    engine = autorelease(LMCacheEngine(cfg, dumb_metadata()))
    kv = generate_kv_cache(10, "vllm", "cuda", 2, 2, 8)
    with pytest.raises(AssertionError):
        engine.store(torch.zeros(2, 5, dtype=torch.int64), kv)
    with pytest.raises(AssertionError):
        engine.store(torch.arange(11), kv)
    with pytest.raises(AssertionError):
        engine.store(torch.arange(10), ())
    assert LMCacheEngineBuilder.get("test_b200") is None
    e1 = autorelease(LMCacheEngineBuilder.get_or_create("test_b200", cfg, dumb_metadata()))
    assert LMCacheEngineBuilder.get("test_b200") is e1
    with pytest.raises(ValueError):
        LMCacheEngineBuilder.get_or_create("test_b200", LMCacheEngineConfig.from_legacy(chunk_size=512, backend="cuda"),
                                           dumb_metadata())
    LMCacheEngineBuilder.destroy("test_b200")


# ---------------------------------------------------------------- engine over lm:// (serde plugin boundary)
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


@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
def test_remote_torch_serde_lossless(fmt, lmserver, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig
    tokens = generate_tokens(600, "cuda")
    kv = generate_kv_cache(600, fmt, "cuda", 4, 2, 64)
    cfg = LMCacheEngineConfig.from_legacy(chunk_size=256, backend=lmserver, remote_serde="torch")
    engine = autorelease(LMCacheEngine(cfg, dumb_metadata(fmt, "m_torch_" + fmt)))
    engine.store(tokens, kv)
    r, m = engine.retrieve(tokens)
    assert torch.sum(m) == 600
    check_kv_cache_equal(r, kv, 600, fmt)
    # a second engine (another "instance") sees the same chunks through the shared server
    engine2 = autorelease(LMCacheEngine(cfg, dumb_metadata(fmt, "m_torch_" + fmt)))
    r2, m2 = engine2.retrieve(torch.cat([tokens, generate_tokens(100, "cuda")]))
    assert torch.sum(m2) == 512
    check_kv_cache_equal(r2, kv, 512, fmt)


@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
@pytest.mark.parametrize("pipelined", [False, True])
def test_remote_cachegen_matches_reference_chain(fmt, pipelined, lmserver, autorelease, engine_path):
    import ref_torch
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig
    model = "mistralai/Mistral-7B-Instruct-v0.2"
    T = 700
    tokens = generate_tokens(T, "cuda")
    kv = generate_kv_cache(T, fmt, "cuda", 32, 8, 128)
    cfg = LMCacheEngineConfig(256, None, lmserver, "cachegen", pipelined, False)
    engine = autorelease(LMCacheEngine(cfg, dumb_metadata(fmt, model)))
    assert engine._fast_path() == (engine_path == "fast")
    engine.store(tokens, kv, blocking=not pipelined)
    if pipelined:
        engine.engine_.drain()              # non-blocking store: wait until the server holds every chunk
    r, m = engine.retrieve(tokens)
    assert torch.sum(m) == T
    kb, vb = (torch.tensor(b) for b in O.make_bins(model))
    blob = torch.stack((torch.stack([k for k, _ in kv]), torch.stack([v for _, v in kv]))).permute(1, 0, 2, 3, 4)
    blob_v = blob if fmt == "vllm" else blob.permute(0, 1, 3, 2, 4)
    tdim = 2
    want = torch.cat([ref_torch.roundtrip(c, kb, vb, fmt) for c in torch.split(blob_v, 256, dim=tdim)],
                     dim=2 if fmt == "vllm" else 3)
    got = torch.stack([torch.stack(p) for p in r])
    assert got.shape == want.shape and got.dtype == want.dtype
    assert torch.equal(got.view(torch.int16), want.contiguous().view(torch.int16))
    # a second, fresh engine ("another vLLM instance") sharing the server: full hit, and a suffix-mask retrieve
    engine2 = autorelease(LMCacheEngine(cfg, dumb_metadata(fmt, model)))
    r2, m2 = engine2.retrieve(tokens)
    assert torch.sum(m2) == T
    assert torch.equal(torch.stack([torch.stack(p) for p in r2]).view(torch.int16), want.contiguous().view(torch.int16))
    mask = torch.ones(T, dtype=torch.bool)
    mask[:300] = False
    r3, m3 = engine2.retrieve(tokens, mask)
    assert torch.sum(m3) == T - 300 and int(m3.nonzero()[0]) == 300
    tdim = 2 if fmt == "vllm" else 3
    assert torch.equal(torch.stack([torch.stack(p) for p in r3]).view(torch.int16),
                       want.narrow(tdim, 300, T - 300).contiguous().view(torch.int16))


# ---------------------------------------------------------------- paged KV caches in place (SURVEY 8f rank 3)
def _paged_caches(kv, slots, nrows, fill):
    """scatter the dense per-layer (K, V) [T,H,D] into fresh paged caches [nrows/16, 16, H, D]"""
    out = []
    for k, v in kv:
        kc = torch.full((nrows // 16, 16) + tuple(k.shape[1:]), fill, dtype=k.dtype, device="cuda")
        vc = torch.full((nrows // 16, 16) + tuple(k.shape[1:]), fill, dtype=k.dtype, device="cuda")
        kc.view(-1, *k.shape[1:])[slots] = k
        vc.view(-1, *k.shape[1:])[slots] = v
        out.append((kc, vc))
    return out


@pytest.mark.parametrize("backend", ["cuda", "cpu", "lm-cachegen", "lm-torch"])
def test_engine_paged_store_and_retrieve(backend, lmserver, autorelease):
    """store_paged / retrieve_paged against a scattered cache give exactly what store / retrieve give on the
    gathered tensors: same chunks in the store, same values in the mapped rows, unmapped / unretrieved rows untouched;
    prefix hit, miss and a suffix mask that is not chunk aligned."""
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig
    model = "mistralai/Mistral-7B-Instruct-v0.2"
    T, cs, nrows = 700, 256, 1024
    L, H, D = (32, 8, 128) if backend == "lm-cachegen" else (4, 2, 64)
    tokens = generate_tokens(T, "cuda")
    kv = generate_kv_cache(T, "vllm", "cuda", L, H, D)
    g = torch.Generator().manual_seed(3)
    slots = torch.randperm(nrows, generator=g)[:T].cuda()
    caches = _paged_caches(kv, slots, nrows, 9.0)
    if backend.startswith("lm-"):
        cfg = LMCacheEngineConfig(cs, None, lmserver, backend[3:], False, False)
    else:
        cfg = LMCacheEngineConfig.from_legacy(chunk_size=cs, backend=backend)
    name = model if backend == "lm-cachegen" else "paged_" + backend
    eng = autorelease(LMCacheEngine(cfg, dumb_metadata("vllm", name)))
    # in two steps, so that the second call skips the two chunks already present and starts at token 512
    # (tok_begin > 0 through the slot mapping)
    eng.store_paged(tokens[:512], [(k, v) for k, v in caches], slots[:512])
    eng.store_paged(tokens, caches, slots)
    dense, m = eng.retrieve(tokens)                       # what the store now holds, as the dense API sees it
    assert torch.sum(m) == T
    ref = autorelease(LMCacheEngine(LMCacheEngineConfig.from_legacy(chunk_size=cs, backend="cuda"), dumb_metadata("vllm", name)))
    if backend == "lm-cachegen":                          # lossy codec: compare with a dense store through the same codec
        cfg2 = LMCacheEngineConfig(cs, None, lmserver, "cachegen", False, False)
        ref = autorelease(LMCacheEngine(cfg2, dumb_metadata("vllm", model)))
    ref.store(tokens, kv, skip_existing=False)            # same keys: overwrites with the dense-encoded chunks
    want, _ = ref.retrieve(tokens)
    for (a, b), (c, d) in zip(dense, want):
        assert torch.equal(a.view(torch.int16), c.view(torch.int16)) and torch.equal(b.view(torch.int16), d.view(torch.int16))
    # retrieve into a fresh cache with another mapping: longer query -> prefix hit of the 2 full chunks + tail chunk miss
    slots2 = torch.randperm(nrows, generator=g)[:T + 100].cuda()
    caches2 = [(torch.full_like(k, 5.0), torch.full_like(v, 5.0)) for k, v in caches]
    q = torch.cat([tokens, generate_tokens(100, "cuda")])
    m2 = eng.retrieve_paged(q, caches2, slots2)
    assert int(torch.sum(m2)) == 512 and bool(m2[:512].all())
    untouched = torch.ones(nrows, dtype=torch.bool, device="cuda")
    untouched[slots2[:512]] = False
    for l, (kc, vc) in enumerate(caches2):
        for kvi, c in enumerate((kc, vc)):
            flat = c.view(-1, H, D)
            assert torch.equal(flat[slots2[:512]].view(torch.int16), want[l][kvi][:512].view(torch.int16)), (l, kvi)
            assert bool((flat[untouched] == 5.0).all())
    # suffix mask (300 tokens skipped, not chunk aligned) on the exact sequence: rows of tokens < 300 stay as they are
    caches3 = [(torch.full_like(k, 5.0), torch.full_like(v, 5.0)) for k, v in caches]
    mask = torch.ones(T, dtype=torch.bool)
    mask[:300] = False
    m3 = eng.retrieve_paged(tokens, caches3, slots, mask)
    assert int(torch.sum(m3)) == T - 300 and int(m3.nonzero()[0]) == 300
    untouched = torch.ones(nrows, dtype=torch.bool, device="cuda")
    untouched[slots[300:]] = False
    for l, (kc, vc) in enumerate(caches3):
        for kvi, c in enumerate((kc, vc)):
            flat = c.view(-1, H, D)
            assert torch.equal(flat[slots[300:]].view(torch.int16), want[l][kvi][300:].view(torch.int16)), (l, kvi)
            assert bool((flat[untouched] == 5.0).all())
    # total miss
    m4 = eng.retrieve_paged(generate_tokens(T, "cuda") + 20000, caches3, slots)
    assert int(torch.sum(m4)) == 0


# ---------------------------------------------------------------- hybrid backend, wide dtypes
@pytest.mark.parametrize("serde", ["torch", "cachegen"])
def test_hybrid_backend_write_through_and_fall_through(serde, lmserver, autorelease):
    """local + remote (lmcache/storage_backend/hybrid_backend.py): a store lands in both tiers; a second engine whose
    local tier is empty is served by the remote tier; the first engine is served locally (its remote connection can go)"""
    import ref_torch
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig
    from lmcache_b200.storage_backend.hybrid_backend import LMCHybridBackend
    model = "mistralai/Mistral-7B-Instruct-v0.2"
    T = 700
    tokens = generate_tokens(T, "cuda")
    kv = generate_kv_cache(T, "vllm", "cuda", 8, 2, 128)
    cfg = LMCacheEngineConfig(256, "cuda", lmserver, serde, False, False)
    e1 = autorelease(LMCacheEngine(cfg, dumb_metadata("vllm", model)))
    assert isinstance(e1.engine_, LMCHybridBackend)
    e1.store(tokens, kv)
    r1, m1 = e1.retrieve(tokens)                                   # local tier: raw, lossless
    assert int(m1.sum()) == T
    check_kv_cache_equal(r1, kv, T, "vllm")
    e2 = autorelease(LMCacheEngine(cfg, dumb_metadata("vllm", model)))
    r2, m2 = e2.retrieve(tokens)                                   # empty local tier: the remote tier answers
    assert int(m2.sum()) == T
    if serde == "torch":
        check_kv_cache_equal(r2, kv, T, "vllm")
    else:
        kb, vb = (torch.tensor(b) for b in O.make_bins(model))
        blob = torch.stack((torch.stack([k for k, _ in kv]), torch.stack([v for _, v in kv]))).permute(1, 0, 2, 3, 4)
        want = torch.cat([ref_torch.roundtrip(c.contiguous(), kb, vb, "vllm") for c in torch.split(blob, 256, dim=2)], dim=2)
        got = torch.stack([torch.stack(p) for p in r2])
        assert torch.equal(got.view(torch.int16), want.view(torch.int16))


@pytest.mark.parametrize("backend", ["cpu-cachegen", "disk", "lm-cachegen"])
def test_kv_dtype_change_ends_the_match(backend, lmserver, tmp_path, autorelease):
    """Chunks 0-3 stored from fp16 KV, chunks 4-7 from bf16 KV: every CacheGen tier returns exactly chunks 0-3, decoded
    as the reference decodes them.  A retrieve ends at the first container whose KV dtype differs from chunk 0's, also
    when the change falls on a wave boundary (waves of 4 chunks by default)."""
    import ref_torch
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig
    model = "mistralai/Mistral-7B-Instruct-v0.2"
    cs, T = 256, 8 * 256
    if backend == "cpu-cachegen":
        cfg = LMCacheEngineConfig.from_legacy(chunk_size=cs, backend="cpu", local_serde="cachegen")
    elif backend == "disk":
        cfg = LMCacheEngineConfig.from_legacy(chunk_size=cs, backend="file://" + str(tmp_path / "kvdisk") + "/")
    else:
        cfg = LMCacheEngineConfig(cs, None, lmserver, "cachegen", False, False)
    tokens = generate_tokens(T, "cuda")
    kv = generate_kv_cache(T, "vllm", "cuda", 8, 2, 128)                # bf16
    kv16 = tuple((k[:4 * cs].half(), v[:4 * cs].half()) for k, v in kv)
    engine = autorelease(LMCacheEngine(cfg, dumb_metadata("vllm", model)))
    engine.store(tokens[:4 * cs], kv16)
    engine.store(tokens, kv, skip_existing=True)                         # chunks 4-7 are bf16 containers
    r, m = engine.retrieve(tokens)
    assert int(m.sum()) == 4 * cs and r[0][0].shape[0] == 4 * cs
    kb, vb = (torch.tensor(b) for b in O.make_bins(model))
    blob = torch.stack((torch.stack([k for k, _ in kv16]), torch.stack([v for _, v in kv16]))).permute(1, 0, 2, 3, 4)
    want = torch.cat([ref_torch.roundtrip(c.contiguous(), kb, vb, "vllm") for c in torch.split(blob, cs, dim=2)], dim=2)
    got = torch.stack([torch.stack(p) for p in r])
    assert got.dtype == want.dtype and torch.equal(got.view(torch.int16), want.view(torch.int16))


@pytest.mark.parametrize("backend", ["cuda", "cpu"])
def test_fp32_kv_takes_the_generic_path(backend, autorelease):
    """the reference's local tiers accept any dtype (local_backend.py:95-100); the 16-bit kernels do not, so such KV goes
    through torch's blob ops on the GPU and the per-chunk plugin interface -- still lossless"""
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig
    T = 600
    tokens = generate_tokens(T, "cuda")
    kv = tuple((torch.rand(T, 2, 16, device="cuda"), torch.rand(T, 2, 16, device="cuda")) for _ in range(3))
    engine = autorelease(LMCacheEngine(LMCacheEngineConfig.from_legacy(chunk_size=256, backend=backend), dumb_metadata()))
    engine.store(tokens, kv)
    r, m = engine.retrieve(torch.cat([tokens, generate_tokens(50, "cuda")]))
    assert int(m.sum()) == 512 and r[0][0].dtype == torch.float32
    check_kv_cache_equal(r, kv, 512, "vllm")


@pytest.mark.gpu
def test_lazy_hash_chain_matches_oracle_in_any_order():
    """sha256_prefix_chain_lazy: digests become readable while the chain is still running; whatever order they are asked
    for in, they are the oracle's (and the reference's: the oracle is pinned to its goldens)."""
    from lmcache_b200.cache_engine import LazySeq, sha256_prefix_chain, sha256_prefix_chain_lazy
    toks = torch.randint(0, 32000, (8192 + 77,), dtype=torch.int64, device="cuda")
    want = O.sha256_chain(toks.cpu().numpy(), 256)
    lz = sha256_prefix_chain_lazy(toks, 256)
    assert isinstance(lz, LazySeq) and len(lz) == 33
    assert lz[32] == want[32] and lz[0] == want[0] and lz[-2] == want[31]        # the last one first: waits for the whole chain
    assert list(lz[5:9]) == want[5:9] and list(lz) == want
    # several runs in flight at once (each owns its landing buffer and epoch), consumed in reverse order of launch
    runs = [(t, sha256_prefix_chain_lazy(t, 256)) for t in (torch.randint(0, 32000, (n,), dtype=torch.int64, device="cuda")
                                                             for n in (300, 4096, 1, 2048))]
    for t, r in reversed(runs):
        assert list(r) == O.sha256_chain(t.cpu().numpy(), 256)
    # several chains in one launch
    offs = [0, 300, 300, 1000]
    assert sha256_prefix_chain(toks[:1000], 256, offs) == O.sha256_chain(toks[:300].cpu().numpy(), 256) + \
        O.sha256_chain(toks[300:1000].cpu().numpy(), 256)
    assert list(sha256_prefix_chain_lazy(toks[:0], 256)) == []
