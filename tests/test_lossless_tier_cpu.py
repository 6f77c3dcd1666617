"""CPU: the lossless local tiers (local_serde="lossless") -- configuration and factory rules, the MLA chunk-size rule, the
host-side stream offsets of a lossless container (b200kv_lossless_plane_offsets) against the numpy statement in
tests/lossless_ref.py, and the byte ranges of a layer-major upload of lossless containers."""
import numpy as np
import pytest

import lossless_ref as R
from lmcache_b200 import _native as N
from lmcache_b200.codec import lossless_plane_offsets
from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
from lmcache_b200.pipeline import layer_copy_ranges
from lmcache_b200.storage_backend import CreateStorageBackend

MODEL = "lmsys/longchat-7b-16k"


def _meta(mla=False):
    return LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16", use_mla=mla)


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:       # noqa: BLE001
        return False


# ---------------------------------------------------------------------------------------------- configuration
def test_local_serde_lossless_is_accepted_everywhere(tmp_path, monkeypatch):
    assert LMCacheEngineConfig(256, "cpu", None, None, False, False, "lossless").local_serde == "lossless"
    assert LMCacheEngineConfig.from_defaults(local_device="cpu", local_serde="lossless").local_serde == "lossless"
    assert LMCacheEngineConfig.from_legacy(backend="cpu", local_serde="lossless").local_serde == "lossless"
    cfg = LMCacheEngineConfig.from_legacy(backend=f"file://{tmp_path}/", local_serde="lossless", local_capacity_bytes=9)
    assert (cfg.local_device, cfg.local_serde, cfg.local_capacity_bytes) == (f"{tmp_path}/", "lossless", 9)
    p = tmp_path / "cfg.yaml"
    p.write_text(f"chunk_size: 4096\nlocal_device: file://{tmp_path}/\nlocal_serde: lossless\n"
                 f"device_cache_bytes: 1024\n")
    cfg = LMCacheEngineConfig.from_file(str(p))
    assert (cfg.chunk_size, cfg.local_serde, cfg.device_cache_bytes) == (4096, "lossless", 1024)
    monkeypatch.setenv("LMCACHE_B200_LOCAL_SERDE", "lossless")
    assert LMCacheEngineConfig.from_defaults(local_device="cpu").local_serde == "lossless"
    assert LMCacheEngineConfig.from_defaults(local_device="cpu", local_serde="cachegen").local_serde == "cachegen"
    for bad in ("Lossless", "fast", "torch"):
        with pytest.raises(ValueError, match="Invalid local serde"):
            LMCacheEngineConfig.from_defaults(local_device="cpu", local_serde=bad)
    p.write_text("chunk_size: 256\nlocal_device: cpu\nlocal_serde: zstd\n")
    with pytest.raises(ValueError, match="Invalid local serde"):
        LMCacheEngineConfig.from_file(str(p))


# ---------------------------------------------------------------------------------------------- factory
def _factory(monkeypatch):
    """CreateStorageBackend with every tier class replaced by a recorder: the factory's choice, without a device"""
    from lmcache_b200.storage_backend import hybrid_backend, local_backend
    made = []

    def fake(name):
        class T:
            def __init__(self, config, metadata):
                made.append((name, config.local_serde))
        return T
    for name in ("LMCLocalBackend", "LMCLocalCompressedBackend", "LMCLocalDiskBackend"):
        monkeypatch.setattr(local_backend, name, fake(name))
    monkeypatch.setattr(hybrid_backend, "LMCHybridBackend", fake("LMCHybridBackend"))
    return made


def test_factory_choices(tmp_path, monkeypatch):
    made = _factory(monkeypatch)
    d = str(tmp_path)

    def make(local, serde, remote=None, rserde="cachegen", **kw):
        made.clear()
        CreateStorageBackend(LMCacheEngineConfig(256, local, remote, rserde, False, False, serde, **kw), _meta())
        return made[0]
    assert make("cpu", "lossless") == ("LMCLocalCompressedBackend", "lossless")
    assert make(d, "lossless") == ("LMCLocalDiskBackend", "lossless")
    assert make(d, None) == ("LMCLocalDiskBackend", None)                  # a directory stays CacheGen
    assert make(d, "cachegen") == ("LMCLocalDiskBackend", "cachegen")
    assert make("cuda", "lossless") == ("LMCLocalBackend", "lossless")     # as "cuda" with "cachegen": raw blobs
    assert make("cuda", "cachegen") == ("LMCLocalBackend", "cachegen")
    for local in ("cpu", d):                                               # both lossless tiers are bounded and cached
        assert make(local, "lossless", local_capacity_bytes=1 << 20, device_cache_bytes=1 << 20)[1] == "lossless"
    for rserde in ("cachegen", "lossless", "torch"):
        assert make("cpu", "lossless", "lm://127.0.0.1:1", rserde)[0] == "LMCHybridBackend"


def test_factory_errors(tmp_path, monkeypatch):
    _factory(monkeypatch)
    for local in ("cpu", str(tmp_path)):
        cfg = LMCacheEngineConfig(8192, local, None, None, False, False, "lossless")
        with pytest.raises(ValueError, match="4096"):
            CreateStorageBackend(cfg, _meta())
    CreateStorageBackend(LMCacheEngineConfig(4096, "cpu", None, None, False, False, "lossless"), _meta())
    with pytest.raises(ValueError, match="4096"):      # the hybrid's local tier as well
        CreateStorageBackend(LMCacheEngineConfig(8192, "cpu", "lm://127.0.0.1:1", "lossless", False, False, "lossless"),
                             _meta())
    # the raw tiers still refuse a capacity and a device level, whatever the serde
    for kw, name in (({"local_capacity_bytes": 1 << 20}, "local_capacity_bytes"),
                     ({"device_cache_bytes": 1 << 20}, "device_cache_bytes")):
        with pytest.raises(ValueError, match=name):
            CreateStorageBackend(LMCacheEngineConfig(256, "cuda", None, None, False, False, "lossless", **kw), _meta())
    # resharding stays a CacheGen feature of the remote tier
    with pytest.raises(ValueError, match="reshard_world_sizes"):
        CreateStorageBackend(LMCacheEngineConfig(256, "cpu", "lm://127.0.0.1:1", "lossless", False, False, "lossless",
                                                 reshard_world_sizes=[2]), _meta())


def test_mla_chunk_size_rule(tmp_path):
    from lmcache_b200.cache_engine import LMCacheEngine
    d = str(tmp_path)
    # a lossless disk or host tier is not a CacheGen tier: version-6 containers hold up to 4096 tokens
    for local in (d, "cpu"):
        LMCacheEngine._check_mla_config(LMCacheEngineConfig(4096, local, None, None, False, False, "lossless"),
                                        _meta(True))
    # a CacheGen disk tier (no serde named, or "cachegen") keeps the 256-token limit
    for serde in (None, "cachegen"):
        with pytest.raises(ValueError, match="256"):
            LMCacheEngine._check_mla_config(LMCacheEngineConfig(512, d, None, None, False, False, serde), _meta(True))
    # and so does a CacheGen remote tier behind a lossless local one
    with pytest.raises(ValueError, match="256"):
        LMCacheEngine._check_mla_config(LMCacheEngineConfig(512, "cpu", "lm://127.0.0.1:1", "cachegen", False, False,
                                                            "lossless"), _meta(True))


@pytest.mark.skipif(_has_gpu(), reason="checks the no-device failure")
def test_lossless_tier_needs_a_device():
    with pytest.raises(RuntimeError, match="CUDA|no CPU fallback"):
        CreateStorageBackend(LMCacheEngineConfig(256, "cpu", None, None, False, False, "lossless"), _meta())


# ---------------------------------------------------------------------------------------------- stream offsets
def _container(P, C, t, seed, latent=False, H=None):
    rng = np.random.default_rng(seed)
    e = rng.integers(0x78, 0x84, size=(P, t, C))                       # bf16 exponents near 1.0
    kv = ((e << 7) | rng.integers(0, 128, size=(P, t, C)) | (rng.integers(0, 2, size=(P, t, C)) << 15)).astype(np.uint16)
    H = H or 1
    L = P if latent else P // 2
    return R.encode(kv, L, H, C // H, R.DT_BF16, latent)


def _numpy_offsets(blob):
    hd = R.parse_header(blob)
    P = hd["L"] if hd["version"] == 6 else 2 * hd["L"]
    C = hd["H"] * hd["D"]
    lo = R.layout(P, C, hd["ntokens"])
    lens = np.frombuffer(blob[lo["off_lens"]:lo["off_lens"] + 2 * P * C], dtype="<u2").reshape(P, C).astype(np.int64)
    return np.concatenate([[lo["off_payload"]], lo["off_payload"] + np.cumsum(lens.sum(axis=1))]), lo


@pytest.mark.parametrize("P,C,t,latent", [(2, 8, 1, False), (4, 128, 7, False), (6, 200, 33, False), (3, 64, 5, True),
                                          (1, 576, 2, True), (2, 16, 300, False)])
def test_plane_offsets_match_the_lengths_section(P, C, t, latent):
    blob = _container(P, C, t, seed=P * 1000 + t, latent=latent)
    want, lo = _numpy_offsets(blob)
    got = lossless_plane_offsets(bytearray(blob))
    assert got is not None and np.array_equal(got, want) and got[-1] == len(blob)
    # only the header and the lengths are read: a buffer that ends at off_raw gives the same offsets
    got2 = np.empty(P + 1, np.int64)
    fixed = np.frombuffer(bytearray(blob[:lo["off_raw"]]), np.uint8)
    assert N.lib().b200kv_lossless_plane_offsets(fixed.ctypes.data, fixed.size, got2.ctypes.data, P + 1) == 0
    assert np.array_equal(got2, want)
    # too short a buffer or too small an output is refused
    assert N.lib().b200kv_lossless_plane_offsets(fixed.ctypes.data, lo["off_raw"] - 1, got2.ctypes.data, P + 1) < 0
    assert N.lib().b200kv_lossless_plane_offsets(fixed.ctypes.data, fixed.size, got2.ctypes.data, P) < 0


def test_plane_offsets_of_a_damaged_or_foreign_container():
    P, C, t = 4, 64, 9
    blob = bytearray(_container(P, C, t, seed=3))
    lo = R.layout(P, C, t)
    bad = bytearray(blob)
    bad[lo["off_lens"] + 2 * C + 3] ^= 0x10                             # one length of plane 1: no longer adds up
    assert lossless_plane_offsets(bad) is None
    o = np.empty(P + 1, np.int64)
    src = np.frombuffer(bad, np.uint8)
    assert N.lib().b200kv_lossless_plane_offsets(src.ctypes.data, src.size, o.ctypes.data, P + 1) == 1
    want, _ = _numpy_offsets(bytes(bad))
    assert np.array_equal(o, want)                                      # still the sums of what the section says
    for off, val in ((4, 3), (4, 7), (0, 0)):                            # CacheGen versions, an unknown one, no magic
        other = bytearray(blob)
        other[off:off + 4] = int(val).to_bytes(4, "little")
        if off == 4:
            assert lossless_plane_offsets(other) is None
        src = np.frombuffer(other, np.uint8)
        assert N.lib().b200kv_lossless_plane_offsets(src.ctypes.data, src.size, o.ctypes.data, P + 1) < 0
    short = bytearray(blob)
    short[40:48] = int(lo["off_payload"] - 16).to_bytes(8, "little")    # total_bytes inside the fixed sections
    src = np.frombuffer(short, np.uint8)
    assert N.lib().b200kv_lossless_plane_offsets(src.ctypes.data, src.size, o.ctypes.data, P + 1) < 0


# ---------------------------------------------------------------------------------------------- layer-major ranges
@pytest.mark.parametrize("L,ppl,C,ts", [(3, 2, 64, [7, 7, 2]), (4, 1, 96, [5, 1]), (1, 2, 16, [300]),
                                        (2, 2, 128, [4096 // 64])])
def test_layer_copy_ranges_of_lossless_containers(L, ppl, C, ts):
    latent = ppl == 1
    blobs = [_container(ppl * L, C, t, seed=10 + j, latent=latent) for j, t in enumerate(ts)]
    offs = [lossless_plane_offsets(bytearray(b)) for b in blobs]
    raw = [(R.layout(ppl * L, C, t)["off_raw"], t * C) for t in ts]
    fixed, start, size = layer_copy_ranges(offs, [len(b) for b in blobs], L, ppl, raw)
    n = len(blobs)
    assert start.shape == size.shape == (L, 2 * ppl * n)
    for j, b in enumerate(blobs):
        lo = R.layout(ppl * L, C, ts[j])
        assert fixed[j] == lo["off_raw"]
        raw_end = lo["off_raw"] + ppl * L * ts[j] * C
        cover = np.zeros(len(b), np.int32)
        cover[:fixed[j]] += 1
        for l in range(L):
            cols = [k * n + j for k in range(2 * ppl)]
            got = sorted((int(start[l, c]), int(size[l, c])) for c in cols)
            want = []
            for k in range(ppl):
                p = k * L + l
                want.append((lo["off_raw"] + p * ts[j] * C, ts[j] * C))                   # the plane's raw rows
                s0 = raw_end if p == 0 else int(offs[j][p])       # plane 0's streams take the alignment gap before them
                want.append((s0, int(offs[j][p + 1]) - s0))                               # the plane's streams
            assert got == sorted(want)
            for s, z in got:
                cover[s:s + z] += 1
        assert (cover == 1).all()                                       # the union is exactly the container
    # a container without offsets (damaged lengths) is copied whole, in its fixed part
    fixed2, _, size2 = layer_copy_ranges([None] + offs[1:], [len(b) for b in blobs], L, ppl, raw)
    assert fixed2[0] == len(blobs[0]) and (size2[:, [k * n for k in range(2 * ppl)]] == 0).all()
