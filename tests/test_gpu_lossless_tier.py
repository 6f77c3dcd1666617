"""GPU: LMCacheEngine on the lossless local tiers (local_serde="lossless"): the compressed host tier and the disk tier
give back the stored bits for every store and retrieve entry point, bounded tiers evict and keep a prefix, a disk tier
restarts on its directory and leaves the other container family's files alone, the device level serves hits in place,
layer-major retrieves are exact layer by layer for chunks of up to 4096 tokens, a layer-wise store lands what store()
lands, and a hybrid puts a lossless local tier in front of an lm:// server."""
import ctypes
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
MODEL = "lmsys/longchat-7b-16k"
SENT = -21555


def _kv(shape, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, device="cuda", generator=g) * torch.exp(2 * torch.randn(shape[-1], device="cuda", generator=g))
    return x.to(dtype)


def _toks(T, seed):
    return torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(seed))


def _engine(local, cs=256, fmt="vllm", dtype="bfloat16", mla=False, serde="lossless", remote=None, rserde=None, **kw):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    cfg = LMCacheEngineConfig(cs, local, remote, rserde, False, False, serde, **kw)
    return LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, 1, 0, fmt, dtype, use_mla=mla))


def _local(tier, tmp_path):
    return "cpu" if tier == "host" else str(tmp_path) + "/"


def _pairs(blob):
    return tuple((blob[l, 0], blob[l, 1]) for l in range(blob.shape[0]))


def _stack(kv):
    return torch.stack([torch.stack([k, v]) for k, v in kv])


def _bits(x):
    return x.contiguous().view(torch.int16)


@pytest.fixture
def server():
    from lmcache_b200 import _native as N
    h = ctypes.c_void_p()
    N.check(N.lib().b200kv_lm_server_start(b"127.0.0.1", 0, ctypes.byref(h)))
    yield f"lm://127.0.0.1:{N.lib().b200kv_lm_server_port(h)}"
    N.lib().b200kv_lm_server_stop(h)


@pytest.mark.parametrize("tier", ["host", "disk"])
@pytest.mark.parametrize("fmt,dtype", [("vllm", torch.bfloat16), ("vllm", torch.float16),
                                       ("huggingface", torch.bfloat16), ("huggingface", torch.float16)])
def test_store_retrieve_is_bit_exact(tier, fmt, dtype, tmp_path):
    L, T, H, D = 4, 700, 8, 128                       # a ragged last chunk of 188 tokens
    shape = (L, 2, T, H, D) if fmt == "vllm" else (L, 2, H, T, D)
    blob = _kv(shape, dtype, 3)
    toks = _toks(T, 1)
    e = _engine(_local(tier, tmp_path), fmt=fmt, dtype=str(dtype).split(".")[1])
    e.store(toks, _pairs(blob))
    kv, mask = e.retrieve(toks)
    assert int(mask.sum()) == T and kv[0][0].dtype == dtype
    assert torch.equal(_bits(_stack(kv)), _bits(blob))
    m = torch.ones(T, dtype=torch.bool)
    m[:300] = False
    kv, mask = e.retrieve(toks, m)
    td = 2 if fmt == "vllm" else 3
    assert int(mask.sum()) == T - 300 and torch.equal(_bits(_stack(kv)), _bits(blob.narrow(td, 300, T - 300)))
    # a fresh engine on the same tier object learns the geometry (and the stored dtype) from a header
    e._geom = None
    kv, mask = e.retrieve(toks)
    assert int(mask.sum()) == T and torch.equal(_bits(_stack(kv)), _bits(blob))
    e.close()


@pytest.mark.parametrize("tier", ["host", "disk"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_paged_store_retrieve_is_bit_exact(tier, dtype, tmp_path):
    L, T, H, D = 3, 600, 4, 64
    blob = _kv((L, 2, T, H, D), dtype, 5)
    toks = _toks(T, 2)
    slots = torch.randperm(1024, generator=torch.Generator().manual_seed(5))[:T].cuda()
    caches = [(torch.zeros(64, 16, H, D, dtype=dtype, device="cuda"), torch.zeros(64, 16, H, D, dtype=dtype, device="cuda"))
              for _ in range(L)]
    for l, (k, v) in enumerate(caches):
        k.view(-1, H, D)[slots] = blob[l, 0]
        v.view(-1, H, D)[slots] = blob[l, 1]
    e = _engine(_local(tier, tmp_path), dtype=str(dtype).split(".")[1])
    e.store_paged(toks, caches, slots)
    dst = [(torch.full_like(_bits(k), SENT).view(dtype), torch.full_like(_bits(v), SENT).view(dtype)) for k, v in caches]
    m = torch.ones(T, dtype=torch.bool)
    m[:256] = False
    mask = e.retrieve_paged(toks, dst, slots, m)
    torch.cuda.synchronize()
    assert int(mask.sum()) == T - 256
    for l, (k, v) in enumerate(dst):
        assert torch.equal(_bits(k.view(-1, H, D)[slots[256:]]), _bits(blob[l, 0, 256:]))
        assert torch.equal(_bits(v.view(-1, H, D)[slots[256:]]), _bits(blob[l, 1, 256:]))
        assert (_bits(k.view(-1, H, D)[slots[:256]]) == SENT).all()
    e.close()


@pytest.mark.parametrize("tier", ["host", "disk"])
def test_mla_engine(tier, tmp_path):
    L, T, D, cs = 4, 1300, 576, 1024                  # version-6 containers of more than 256 tokens
    lat = _kv((L, T, D), torch.bfloat16, 7)
    toks = _toks(T, 3)
    e = _engine(_local(tier, tmp_path), cs=cs, mla=True)
    e.store(toks, tuple(lat[l] for l in range(L)))
    kv, mask = e.retrieve(toks)
    assert int(mask.sum()) == T and torch.equal(_bits(torch.stack(list(kv))), _bits(lat))
    r = e.retrieve_layerwise(toks)
    assert r._upload.n == 2                           # went layer-major
    r.synchronize()
    assert torch.equal(_bits(torch.stack(list(r.kv))), _bits(lat))
    e.close()


@pytest.mark.parametrize("tier", ["host", "disk"])
def test_bounded_tier_evicts_and_keeps_a_prefix(tier, tmp_path):
    L, T, H, D = 2, 1024, 4, 128
    a, b = _kv((L, 2, T, H, D), torch.bfloat16, 11), _kv((L, 2, T, H, D), torch.bfloat16, 12)
    ta, tb = _toks(T, 11), _toks(T, 12)
    probe = _engine(_local(tier, tmp_path / "probe"))
    probe.store(ta, _pairs(a))
    one = max(en.nbytes for en in probe.engine_.dict.values())
    probe.close()
    cap = 3 * one + one // 2                          # three chunks of the four
    e = _engine(_local(tier, tmp_path / "t"), local_capacity_bytes=cap)
    e.store(ta, _pairs(a))
    kv, mask = e.retrieve(ta)
    n = int(mask.sum())
    assert 0 < n < T and n % 256 == 0 and torch.equal(_bits(_stack(kv)), _bits(a[:, :, :n]))
    e.store(tb, _pairs(b))
    assert e.engine_.evicted > 0
    kv, mask = e.retrieve(tb)
    n = int(mask.sum())
    assert n > 0 and torch.equal(_bits(_stack(kv)), _bits(b[:, :, :n]))
    if tier == "host":
        assert e.engine_.host_bytes() <= cap
    else:
        assert sum(os.path.getsize(tmp_path / "t" / f) for f in os.listdir(tmp_path / "t")) <= cap
    e.close()


def test_disk_restart_and_the_other_family(tmp_path):
    L, T, H, D = 2, 600, 4, 128
    a, c = _kv((L, 2, T, H, D), torch.bfloat16, 21), _kv((L, 2, T, H, D), torch.bfloat16, 22)
    ta, tc = _toks(T, 21), _toks(T, 22)
    d = str(tmp_path) + "/"
    e = _engine(d)
    e.store(ta, _pairs(a))
    e.close()
    cg = _engine(d, serde=None)                       # a CacheGen disk tier on the same directory
    assert len(cg.engine_.dict) == 0                  # the lossless files are not its chunks ...
    cg.store(tc, _pairs(c))
    kv, mask = cg.retrieve(ta)
    assert int(mask.sum()) == 0
    cg.close()
    files = sorted(os.listdir(d))
    assert len(files) == 6                            # ... and stay on disk
    e2 = _engine(d)                                   # the lossless tier restarts on its three files only
    assert len(e2.engine_.dict) == 3
    kv, mask = e2.retrieve(ta)
    assert int(mask.sum()) == T and torch.equal(_bits(_stack(kv)), _bits(a))
    kv, mask = e2.retrieve(tc)
    assert int(mask.sum()) == 0
    e2.close()
    cg2 = _engine(d, serde="cachegen")
    assert len(cg2.engine_.dict) == 3
    kv, mask = cg2.retrieve(tc)
    assert int(mask.sum()) == T
    cg2.close()
    assert sorted(os.listdir(d)) == files


@pytest.mark.parametrize("tier", ["host", "disk"])
def test_device_cache_hits_are_bit_exact(tier, tmp_path):
    L, T, H, D = 4, 900, 8, 128
    blob = _kv((L, 2, T, H, D), torch.float16, 31)
    toks = _toks(T, 31)
    e = _engine(_local(tier, tmp_path), dtype="float16", device_cache_bytes=64 << 20)
    e.store(toks, _pairs(blob))
    for _ in range(2):
        kv, mask = e.retrieve(toks)
        assert int(mask.sum()) == T and torch.equal(_bits(_stack(kv)), _bits(blob))
    r = e.retrieve_layerwise(toks)
    r.synchronize()
    assert torch.equal(_bits(_stack(r.kv)), _bits(blob))
    st = e.engine_.device_cache_stats()
    assert st["hits"] >= 3 * 4 and st["bytes_in_use"] > 0
    e.close()


@pytest.mark.parametrize("tier", ["host", "disk"])
@pytest.mark.parametrize("cs", [256, 1024, 4096])
def test_layerwise_retrieve(tier, cs, tmp_path):
    L, H, D = 4, 8, 128
    T = cs + cs // 2 + 5
    blob = _kv((L, 2, T, H, D), torch.bfloat16, cs)
    toks = _toks(T, cs)
    e = _engine(_local(tier, tmp_path), cs=cs)
    e.store(toks, _pairs(blob))
    r = e.retrieve_layerwise(toks)
    assert r._upload.n == 2 and int(r.ret_mask.sum()) == T
    for l in range(L):
        r.wait_layer(l)
        k, v = r.kv[l]
        assert torch.equal(_bits(k), _bits(blob[l, 0])) and torch.equal(_bits(v), _bits(blob[l, 1])), l
    kv, _ = e.retrieve(toks)
    assert torch.equal(_bits(_stack(r.kv)), _bits(_stack(kv)))
    # paged form
    slots = torch.randperm(T + 64, generator=torch.Generator().manual_seed(cs))[:T].cuda()
    nb = (T + 64 + 15) // 16
    dst = [(torch.zeros(nb, 16, H, D, dtype=torch.bfloat16, device="cuda"),
            torch.zeros(nb, 16, H, D, dtype=torch.bfloat16, device="cuda")) for _ in range(L)]
    r = e.retrieve_paged_layerwise(toks, dst, slots)
    for l in range(L):
        r.wait_layer(l)
        k, v = dst[l]
        assert torch.equal(_bits(k.view(-1, H, D)[slots]), _bits(blob[l, 0]))
        assert torch.equal(_bits(v.view(-1, H, D)[slots]), _bits(blob[l, 1]))
    e.close()


@pytest.mark.parametrize("tier", ["host", "disk"])
def test_store_layerwise_lands_what_store_lands(tier, tmp_path):
    L, T, H, D = 3, 700, 4, 128
    blob = _kv((L, 2, T, H, D), torch.bfloat16, 41)
    toks = _toks(T, 41)
    a = _engine(_local(tier, tmp_path / "a"))
    a.store(toks, _pairs(blob))
    b = _engine(_local(tier, tmp_path / "b"))
    s = b.store_layerwise(toks, _pairs(blob))
    for l in range(L):
        s.save_layer(l)
    s.finish()

    def containers(eng, path):
        if tier == "host":
            out = {}
            for k, en in eng.engine_.dict.items():
                en.ready.wait()
                out[k] = bytes(en.rec.blk.view())
            return out
        return {f: open(os.path.join(path, f), "rb").read() for f in os.listdir(path)}
    ca, cb = containers(a, tmp_path / "a"), containers(b, tmp_path / "b")
    assert len(ca) == 3 and ca == cb
    kv, mask = b.retrieve(toks)
    assert int(mask.sum()) == T and torch.equal(_bits(_stack(kv)), _bits(blob))
    a.close(), b.close()


@pytest.mark.parametrize("rserde", ["lossless", "cachegen"])
def test_hybrid_with_a_lossless_local_tier(server, rserde):
    L, T, H, D = 4, 600, 8, 128
    blob = _kv((L, 2, T, H, D), torch.bfloat16, 51)
    toks = _toks(T, 51)
    h = _engine("cpu", remote=server, rserde=rserde)
    h.store(toks, _pairs(blob))
    kv, mask = h.retrieve(toks)                       # served by the lossless local tier: exact
    assert int(mask.sum()) == T and torch.equal(_bits(_stack(kv)), _bits(blob))
    h2 = _engine("cpu", remote=server, rserde=rserde)  # an empty local tier: the remote tier serves
    kv, mask = h2.retrieve(toks)
    assert int(mask.sum()) == T
    if rserde == "lossless":
        assert torch.equal(_bits(_stack(kv)), _bits(blob))
    # fp16 chunks in the local tier of a CacheGen hybrid (which decodes a vllm KV into bf16) are a miss, not a cast
    if rserde == "cachegen":
        h3 = _engine("cpu", remote=None, dtype="float16")
        f16 = blob.to(torch.float16)
        h3.store(toks, _pairs(f16))
        from lmcache_b200.codec import KvView
        out = torch.empty_like(blob)
        n = h3.engine_.get_kv_into([h3._make_key(x, "vllm") for x in h3._prefix_hash(toks)], KvView.from_blob(out, "vllm"),
                                   0, 256)
        assert n == 0
        h3.close()
    h.close(), h2.close()
