"""GPU: models of 65 to 128 layers (B200KV_MAX_PLANES = 256) and CacheGen bin layouts from cachegen_config.

* b200kv_encode_chunks / b200kv_decode_chunks at L = 65, 80 and 128 with every coder and blob, tuple and paged sources:
  container bytes section by section and decoded KV bit for bit the oracle's, with random per-layer bins.
* The layer-wise encode split across the old 64-layer word boundary, finish refusing a missing layer >= 64, the split
  decode across layer 64, b200kv_plane_offsets_device at 128 layers and its rejections, and L = 129 refused everywhere.
* The engine with an 80-layer bf16 tuple on every tier: raw cuda / cpu (bit-exact), the compressed host tier with a
  cachegen_config (the oracle's values), the layer-wise paths, the disk tier across a restart, lm:// with the CacheGen
  serde, and the containers a cachegen_config engine must treat as misses."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle as O
from test_gpu_layer_split import (_Dest, _a16, _check_sections, _containers, _decode, _encode_chunks, _encode_layers, _kv,
                                  _rand_bins, _s, _source)

pytestmark = pytest.mark.gpu

DEEP = "meta-llama/Llama-3.1-70B-Instruct"        # not in the bin table
LLAMA70B = dict(key_first_layers=10, key_second_layers=20, key_third_layers=80, key_first_bins=32, key_second_bins=16,
                key_third_bins=16, value_first_layers=2, value_first_bins=32, value_second_bins=16)
LONGCHAT = dict(LLAMA70B, key_third_layers=32)


def _N():
    from lmcache_b200 import _native as N
    return N


def _bins(cfg):
    from lmcache_b200.storage_backend.serde.cachegen_basics import CacheGenConfig
    c = CacheGenConfig(**cfg)
    return np.array(c.key_bins_list(), np.float32), np.array(c.value_bins_list(), np.float32)


# ------------------------------------------------------------------------------------------------ 1. codec vs oracle
@pytest.mark.parametrize("src", ["blob", "tuple", "paged"])
@pytest.mark.parametrize("coder", [0, 1, 2])
@pytest.mark.parametrize("D", [20, 128])
@pytest.mark.parametrize("L", [65, 80, 128])
def test_encode_decode_deep_vs_oracle(L, D, coder, src):
    """two chunks (128 + 72 tokens) of an L-layer KV: every section of both containers is the oracle's, and decoding
    them gives the oracle's values, with nothing outside the destination rows written"""
    rng = np.random.default_rng(L * 1000 + D * 10 + coder)
    H = 1 if D == 128 else 3
    T, cs = 200, 128
    n, last = 2, T - cs
    dt = int(rng.integers(0, 2))
    kb, vb = _rand_bins(rng, L)
    x, bits = _kv(L, T, H, D, dt, seed=L + D + coder)
    view = _source(src, x, rng)
    raws = _encode_chunks(view, 0, n, cs, last, kb, vb, coder)
    encs = [_check_sections(raws[j], bits[:, :, j * cs: j * cs + (cs if j == 0 else last)], dt, kb, vb, coder)
            for j in range(n)]
    out_dt = int(rng.integers(0, 2))
    dest = _Dest("vllm", L, H, D, T, out_dt, 4, None)
    assert _decode(raws, coder, dest, [4, 4 + cs], kb, vb, dt) == [0, 0]
    want = np.concatenate([O.decode_chunk(e, dt, kb, vb, out_dt) for e in encs], axis=2)
    assert np.array_equal(dest.bits(), want)
    assert dest.rest_untouched()


# ------------------------------------------------------------------------------------------------ 2. layer split
@pytest.mark.parametrize("D", [20, 128])
def test_layer_split_at_128_layers(D):
    """the layer-wise encode as [(0,1),(1,127),(127,128)] and as 128 single layers in reverse order is byte for byte
    encode_chunks' containers; the split decode across layer 64 gives the oracle's values"""
    N = _N()
    rng = np.random.default_rng(D + 1)
    L, H, T, cs = 128, 1, 300, 256
    n, last = 2, T - cs
    kb, vb = _rand_bins(rng, L)
    x, bits = _kv(L, T, H, D, 0, seed=D + 5)
    view = _source("blob", x, rng)
    want = _encode_chunks(view, 0, n, cs, last, kb, vb, N.CODER_RANS_COMPACT)
    for calls in ([(0, 1), (1, 127), (127, 128)], [(l, l + 1) for l in range(L - 1, -1, -1)], [(0, 128)]):
        assert _containers(_encode_layers(view, 0, n, cs, last, kb, vb, calls)) == want, len(calls)
    encs = [_check_sections(want[j], bits[:, :, j * cs: j * cs + (cs if j == 0 else last)], 0, kb, vb,
                            O.CODER_RANS_COMPACT) for j in range(n)]
    wantd = np.concatenate([O.decode_chunk(e, 0, kb, vb, 0) for e in encs], axis=2)
    for parts in ([(0, 40), (40, 90), (90, 128)], [(64, 128), (0, 64)], [(63, 65), (0, 63), (65, 128)]):
        dest = _Dest("vllm", L, H, D, T, 0, 2, None)
        assert _decode(want, N.CODER_RANS_COMPACT, dest, [2, 2 + cs], kb, vb, 0, parts=parts) == [0, 0]
        assert np.array_equal(dest.bits(), wantd) and dest.rest_untouched()


@pytest.mark.parametrize("missing", [3, 64, 100, 127])
def test_finish_refuses_a_missing_layer(missing):
    """finish() fails with a message unless every one of the 128 layers was encoded, including those past 63; a layer
    range that overlaps an earlier one is refused across the word boundary too"""
    N = _N()
    lib = N.lib()
    L, H, D, T = 128, 1, 16, 40
    rng = np.random.default_rng(missing)
    kb, vb = _rand_bins(rng, L)
    x, _ = _kv(L, T, H, D, 0, seed=missing)
    view = _source("blob", x, rng)
    lo = N.container_layout(L, H, D, T, N.CODER_RANS_COMPACT)
    stride = _a16(lo.off_payload)
    arena_bytes = lo.max_total_bytes
    arena = torch.empty(arena_bytes, dtype=torch.uint8, device="cuda")
    fixed = torch.empty(stride, dtype=torch.uint8, device="cuda")
    seg = torch.empty(2 * L * 2, dtype=torch.int64, device="cuda")
    sizes = torch.empty(1, dtype=torch.int64, device="cuda")
    wsb = N.check(lib.b200kv_encode_layers_workspace_bytes(L, H, D, T, 1, L), "encode_layers_workspace_bytes")
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    plan = N.EncodePlan()
    N.check(lib.b200kv_encode_layers_plan(ctypes.byref(view.desc), 0, 1, T, T, N.float_array(kb), N.float_array(vb),
                                          N.CODER_RANS_COMPACT, arena.data_ptr(), arena_bytes, fixed.data_ptr(), stride,
                                          seg.data_ptr(), sizes.data_ptr(), L, ws.data_ptr(), wsb, ctypes.byref(plan),
                                          _s()), "encode_layers_plan")
    if missing > 0:
        N.check(lib.b200kv_encode_layers(ctypes.byref(plan), 0, missing, _s()), "encode_layers")
    if missing + 1 < L:
        N.check(lib.b200kv_encode_layers(ctypes.byref(plan), missing + 1, L, _s()), "encode_layers")
    assert lib.b200kv_encode_layers(ctypes.byref(plan), max(missing - 1, 0), missing + 1, _s()) < 0
    assert "encoded before" in N.last_error()
    assert lib.b200kv_encode_layers_finish(ctypes.byref(plan), _s()) < 0
    assert "never encoded" in N.last_error()
    N.check(lib.b200kv_encode_layers(ctypes.byref(plan), missing, missing + 1, _s()), "encode_layers")
    N.check(lib.b200kv_encode_layers_finish(ctypes.byref(plan), _s()), "encode_layers_finish")
    torch.cuda.synchronize()
    assert int(sizes.cpu()[0]) > lo.off_payload


# ------------------------------------------------------------------------------------------------ 3. plane offsets
def test_plane_offsets_device_at_128_layers():
    """device rows == host offsets at 128 layers (zeros past 2L + 1); a header claiming 129 layers, or more layers than
    its bytes hold, or one whose fixed sections overrun the row stride, gives -1"""
    N = _N()
    lib = N.lib()
    rng = np.random.default_rng(12)
    raws = []
    for L, H, D, T, cs in [(128, 1, 128, 300, 256), (128, 2, 20, 5, 5), (97, 3, 16, 64, 64), (4, 1, 8, 40, 40)]:
        kb, vb = _rand_bins(rng, L)
        x, _ = _kv(L, T, H, D, 0, seed=L + T)
        n = (T + cs - 1) // cs
        raws += _encode_chunks(_source("blob", x, rng), 0, n, cs, T - (n - 1) * cs, kb, vb, N.CODER_RANS_COMPACT)
    n_valid = len(raws)

    def mutate(src, pos, val):
        b = bytearray(src)
        b[pos:pos + 4] = int(val).to_bytes(4, "little")
        return bytes(b)
    bad = [mutate(raws[0], 8, 129),           # L = 129
           mutate(raws[2], 8, 129),
           mutate(raws[-1], 8, 128),          # 4 layers of bytes claiming 128: fixed sections longer than total_bytes
           mutate(raws[-1], 8, 100),
           mutate(raws[3], 12, 1 << 20),      # H so large the lengths section overruns the row
           mutate(raws[2], 8, 127)]           # one layer short: the half-lengths do not add up
    allc = raws + bad
    stride = _a16(max(len(c) for c in allc))
    host = np.zeros(len(allc) * stride, np.uint8)
    for j, c in enumerate(allc):
        host[j * stride: j * stride + len(c)] = np.frombuffer(c, np.uint8)
    buf = torch.from_numpy(host).cuda()
    out = torch.full((len(allc), N.MAX_PLANES + 1), -5, dtype=torch.int64, device="cuda")
    N.check(lib.b200kv_plane_offsets_device(buf.data_ptr(), stride, len(allc), out.data_ptr(), _s()),
            "plane_offsets_device")
    torch.cuda.synchronize()
    dev = out.cpu().numpy()
    for j, c in enumerate(allc):
        a = np.frombuffer(c, np.uint8)
        o = np.zeros(N.MAX_PLANES + 1, np.int64)
        rc = lib.b200kv_plane_offsets(a.ctypes.data, a.size, o.ctypes.data, o.size)
        if j < n_valid:
            L = int(a[8:12].view(np.uint32)[0])
            assert rc == 0 and o[2 * L] == len(c)
            assert np.array_equal(dev[j], o), j
        else:
            assert rc != 0, j
            assert dev[j, 0] == -1, j


# ------------------------------------------------------------------------------------------------ 4. bad calls
def test_129_layers_are_refused_with_a_message():
    """L = 129 (258 planes) is refused by encode, the layer-wise plan, decode, the decode plan, pack and unpack: rc < 0,
    a message, and nothing written"""
    N = _N()
    lib = N.lib()
    L, H, D, t = 129, 1, 8, 4
    src = torch.zeros((L, 2, t, H, D), dtype=torch.bfloat16, device="cuda")
    d = N.KvDesc()
    d.base = src.data_ptr()
    d.planes = None
    d.sL, d.sKV, d.sT, d.sH = 2 * t * H * D, t * H * D, H * D, D
    d.L, d.H, d.D, d.dtype = L, H, D, N.DT_BF16
    bins = N.float_array([16.0] * L)
    out = torch.full((1 << 16,), 0x5A, dtype=torch.uint8, device="cuda")
    sizes = torch.full((4,), 7, dtype=torch.int64, device="cuda")
    ws = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def refused(rc, what):
        assert rc < 0, what
        assert N.last_error(), what
    for coder in (0, 1, 2):
        refused(lib.b200kv_encode_chunks(ctypes.byref(d), 0, 1, t, t, bins, bins, coder, out.data_ptr(), 1 << 15,
                                         sizes.data_ptr(), ws.data_ptr(), ws.numel(), _s()), f"encode {coder}")
    plan = N.EncodePlan()
    refused(lib.b200kv_encode_layers_plan(ctypes.byref(d), 0, 1, t, t, bins, bins, N.CODER_RANS_COMPACT, out.data_ptr(),
                                          1 << 15, out.data_ptr() + (1 << 15), 1 << 14, sizes.data_ptr(),
                                          sizes.data_ptr(), 1, ws.data_ptr(), ws.numel(), ctypes.byref(plan), _s()),
            "encode_layers_plan")
    args = (out.data_ptr(), out.numel(), N.i64_array([0]), N.i64_array([1024]), N.i32_array([t]), N.i64_array([0]), 1,
            N.DT_BF16, N.CODER_RANS_COMPACT, ctypes.byref(d), bins, bins, None, ws.data_ptr(), ws.numel())
    refused(lib.b200kv_decode_chunks(*args, _s()), "decode_chunks")
    dplan = N.DecodePlan()
    refused(lib.b200kv_decode_plan(*args, ctypes.byref(dplan), _s()), "decode_plan")
    refused(lib.b200kv_pack_chunks(ctypes.byref(d), 0, 1, t, t, 0, out.data_ptr(), 1 << 15, _s()), "pack")
    refused(lib.b200kv_unpack_chunks(out.data_ptr(), 1 << 15, 1, t, t, 0, ctypes.byref(d), 0, _s()), "unpack")
    torch.cuda.synchronize()
    assert bool((out == 0x5A).all()) and bool((sizes == 7).all()) and bool((src == 0).all())
    # 128 layers pass the same checks
    d.L = 128
    N.check(lib.b200kv_pack_chunks(ctypes.byref(d), 0, 1, t, t, 0, out.data_ptr(), 1 << 15, _s()), "pack")
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ 5. engine
T_ENG, H_ENG, D_ENG = 600, 2, 64


def _deep_kv(L=80, T=T_ENG, seed=0):
    """an L-layer bf16 KV: the tuple store() takes, and its bits [L,2,T,C]"""
    bits = O.synth_kv_bits(L, T, H_ENG * D_ENG, seed=seed)
    x = torch.from_numpy(bits.view(np.int16)).view(torch.bfloat16).reshape(L, 2, T, H_ENG, D_ENG).cuda()
    return tuple((x[l, 0], x[l, 1]) for l in range(L)), bits


def _bits_of(kv):
    L = len(kv)
    x = torch.stack([torch.stack([k, v]) for k, v in kv])
    return x.contiguous().cpu().view(torch.int16).numpy().view(np.uint16).reshape(L, 2, x.shape[2], -1)


def _oracle(bits, cfg, cs=256):
    kb, vb = _bins(cfg)
    return np.concatenate([O.decode_chunk(O.encode_chunk(bits[:, :, a:a + cs], O.DT_BF16, kb, vb, O.CODER_RANS),
                                          O.DT_BF16, kb, vb, O.DT_BF16) for a in range(0, bits.shape[2], cs)], axis=2)


def _engine(model=DEEP, **kw):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    return LMCacheEngine(LMCacheEngineConfig.from_legacy(chunk_size=256, **kw),
                         LMCacheEngineMetadata(model, 1, 0, "vllm", "bfloat16"))


def _tokens(T=T_ENG, seed=1):
    return torch.randint(0, 32000, (T,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed))


def _containers_of(engine):
    return {k: bytes(e.rec.blk.view()[:e.rec.nbytes]) for k, e in engine.engine_.dict.items()}


@pytest.mark.parametrize("backend", ["cuda", "cpu"])
def test_raw_tiers_store_and_retrieve_80_layers(backend, autorelease):
    eng = autorelease(_engine(backend=backend))
    kv, bits = _deep_kv(seed=3)
    tokens = _tokens()
    eng.store(tokens, kv)
    ret, mask = eng.retrieve(tokens)
    torch.cuda.synchronize()
    assert int(mask.sum()) == T_ENG and len(ret) == 80
    assert np.array_equal(_bits_of(ret), bits)


@pytest.fixture(scope="module")
def deep_case():
    kv, bits = _deep_kv(seed=5)
    return kv, bits, _oracle(bits, LLAMA70B)


def test_compressed_host_tier_with_cachegen_config(deep_case, autorelease):
    kv, _, want = deep_case
    eng = autorelease(_engine(backend="cpu", local_serde="cachegen", cachegen_config=LLAMA70B))
    tokens = _tokens()
    eng.store(tokens, kv)
    ret, mask = eng.retrieve(tokens)
    torch.cuda.synchronize()
    assert int(mask.sum()) == T_ENG
    assert np.array_equal(_bits_of(ret), want)
    assert all(c[4] == 3 for c in _containers_of(eng).values())
    # a prefix and a suffix mask are served as by the table models
    ret2, mask2 = eng.retrieve(tokens[:300])
    torch.cuda.synchronize()
    assert int(mask2.sum()) == 256 and np.array_equal(_bits_of(ret2), want[:, :, :256])


def test_layerwise_paths_equal_the_ordinary_ones(deep_case, autorelease):
    kv, _, want = deep_case
    tokens = _tokens()
    plain = autorelease(_engine(backend="cpu", local_serde="cachegen", cachegen_config=LLAMA70B))
    plain.store(tokens, kv)
    plain.retrieve(tokens)
    lw = autorelease(_engine(backend="cpu", local_serde="cachegen", cachegen_config=LLAMA70B))
    st = lw.store_layerwise(tokens, kv)
    for l in range(80):
        st.save_layer(l)
    st.finish()
    r = lw.retrieve_layerwise(tokens)
    r.synchronize()
    assert int(r.ret_mask.sum()) == T_ENG
    assert np.array_equal(_bits_of(r.kv), want)
    assert _containers_of(lw) == _containers_of(plain)
    # layer by layer: each layer is complete after its own wait
    r = plain.retrieve_layerwise(tokens)
    for l in (0, 63, 64, 79):
        r.wait_layer(l)
        torch.cuda.current_stream().synchronize()
        assert np.array_equal(_bits_of(r.kv[l:l + 1]), want[l:l + 1]), l
    r.synchronize()
    assert np.array_equal(_bits_of(r.kv), want)


def test_disk_tier_rebuilds_its_index_after_a_restart(deep_case, tmp_path, autorelease):
    kv, _, want = deep_case
    tokens = _tokens()
    eng = _engine(backend=f"file://{tmp_path}/", cachegen_config=LLAMA70B)
    eng.store(tokens, kv)
    eng.retrieve(tokens)                 # the files are complete once a retrieve has waited for the store
    eng.close()
    assert len(list(tmp_path.glob("*.b2kv"))) == 3
    again = autorelease(_engine(backend=f"file://{tmp_path}/", cachegen_config=LLAMA70B))
    ret, mask = again.retrieve(tokens)
    torch.cuda.synchronize()
    assert int(mask.sum()) == T_ENG and np.array_equal(_bits_of(ret), want)


@pytest.fixture
def server():
    N = _N()
    h = ctypes.c_void_p()
    N.check(N.lib().b200kv_lm_server_start(b"127.0.0.1", 0, ctypes.byref(h)))
    yield f"lm://127.0.0.1:{N.lib().b200kv_lm_server_port(h)}"
    N.lib().b200kv_lm_server_stop(h)


def test_lm_remote_tier_with_cachegen_serde(deep_case, server, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    kv, _, want = deep_case
    tokens = _tokens()

    def make():
        cfg = LMCacheEngineConfig(256, None, server, "cachegen", False, False, cachegen_config=LLAMA70B)
        return autorelease(LMCacheEngine(cfg, LMCacheEngineMetadata(DEEP, 1, 0, "vllm", "bfloat16")))
    make().store(tokens, kv)
    ret, mask = make().retrieve(tokens)
    torch.cuda.synchronize()
    assert int(mask.sum()) == T_ENG and np.array_equal(_bits_of(ret), want)


def test_cachegen_config_settings_that_cannot_record_bins_are_refused(monkeypatch, tmp_path):
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    from lmcache_b200.storage_backend.serde import CreateSerde
    meta = LMCacheEngineMetadata(DEEP, 1, 0, "vllm", "bfloat16")
    with pytest.raises(ValueError):
        _engine(backend="cpu", local_serde="cachegen")                    # not in the table, no cachegen_config
    for name in ("rans", "ac"):
        monkeypatch.setenv("LMCACHE_B200_CODER", name)
        with pytest.raises(ValueError):
            _engine(backend="cpu", local_serde="cachegen", cachegen_config=LLAMA70B)
        with pytest.raises(ValueError):
            CreateSerde("cachegen", LMCacheEngineConfig.from_defaults(cachegen_config=LLAMA70B), meta)
    monkeypatch.delenv("LMCACHE_B200_CODER")
    for kw in (dict(backend="cpu", local_serde="cachegen"), dict(backend=f"file://{tmp_path}/")):
        with pytest.raises(ValueError):
            from lmcache_b200.cache_engine import LMCacheEngine
            LMCacheEngine(LMCacheEngineConfig.from_legacy(chunk_size=512, cachegen_config=LLAMA70B, **kw), meta)
    with pytest.raises(ValueError):
        CreateSerde("cachegen", LMCacheEngineConfig.from_defaults(chunk_size=512, cachegen_config=LLAMA70B), meta)


@pytest.mark.parametrize("writer", ["v2", "v3_other_bins", "v3_same_bins"])
def test_containers_a_cachegen_config_engine_cannot_read_are_misses(writer, tmp_path, monkeypatch, autorelease):
    """a table engine (longchat) stores on disk; a cachegen_config engine of the same model name reads the directory:
    its version-2 containers, and version-3 ones written with other bins, are misses; with the table's own bins it hits"""
    model = "lmsys/longchat-7b-16k"
    kv, bits = _deep_kv(L=32, seed=8)
    tokens = _tokens(seed=4)
    if writer == "v2":
        monkeypatch.setenv("LMCACHE_B200_CODER", "rans")
    w = _engine(model, backend=f"file://{tmp_path}/")
    w.store(tokens, kv)
    w.retrieve(tokens)
    w.close()
    monkeypatch.delenv("LMCACHE_B200_CODER", raising=False)
    cfg = dict(LONGCHAT, key_first_bins=24) if writer == "v3_other_bins" else LONGCHAT
    r = autorelease(_engine(model, backend=f"file://{tmp_path}/", cachegen_config=cfg))
    ret, mask = r.retrieve(tokens)
    torch.cuda.synchronize()
    if writer == "v3_same_bins":
        assert int(mask.sum()) == T_ENG and np.array_equal(_bits_of(ret), _oracle(bits, LONGCHAT))
    else:
        assert int(mask.sum()) == 0
