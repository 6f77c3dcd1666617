"""CPU: LMCacheEngine with a latent KV (metadata.use_mla, DeepSeek-V2/V3) -- the metadata field, the settings it rules
out, the (K, V) / latent argument checks, the keys every tensor-parallel rank shares, the rank-0-only rule of the remote
tier (remote-only and hybrid), the layer-major copy ranges and segment rows of one plane per layer, and the disk index
that admits version-4 containers for a latent engine only.  Stand-in backends and connectors; no GPU."""
import os

import numpy as np
import pytest
import torch

from lmcache_b200 import _native as N
from oracle import oracle as O

import mla_ref

MODEL = "deepseek-ai/DeepSeek-V3"


def _meta(ws=1, rank=0, fmt="vllm", mla=True):
    from lmcache_b200.config import LMCacheEngineMetadata
    return LMCacheEngineMetadata(MODEL, ws, rank, fmt, "bfloat16", mla)


class _Backend:
    def contains(self, key):
        return False

    def close(self):
        pass


def _engine(monkeypatch, meta, **cfg):
    import lmcache_b200.cache_engine as ce
    from lmcache_b200.config import LMCacheEngineConfig
    monkeypatch.setattr(ce, "CreateStorageBackend", lambda c, m: _Backend())
    return ce.LMCacheEngine(LMCacheEngineConfig.from_defaults(**cfg), meta)


# ---------------------------------------------------------------------------------------------- metadata
def test_use_mla_is_the_last_field_and_defaults_to_false():
    import dataclasses

    from lmcache_b200.config import LMCacheEngineMetadata
    fields = [f.name for f in dataclasses.fields(LMCacheEngineMetadata)]
    assert fields == ["model_name", "world_size", "worker_id", "fmt", "dtype", "use_mla"]
    m = LMCacheEngineMetadata(MODEL, 2, 1, "vllm", "bfloat16")
    assert m.use_mla is False
    assert LMCacheEngineMetadata(MODEL, 2, 1, "vllm", "bfloat16", True).use_mla is True
    assert m != LMCacheEngineMetadata(MODEL, 2, 1, "vllm", "bfloat16", use_mla=True)


def test_builder_tells_an_mla_engine_from_a_kv_engine(monkeypatch):
    from lmcache_b200.cache_engine import LMCacheEngineBuilder
    import lmcache_b200.cache_engine as ce
    from lmcache_b200.config import LMCacheEngineConfig
    monkeypatch.setattr(ce, "CreateStorageBackend", lambda c, m: _Backend())
    cfg = LMCacheEngineConfig.from_defaults(local_device="cpu", remote_url=None)
    try:
        e = LMCacheEngineBuilder.get_or_create("mla-test", cfg, _meta())
        assert LMCacheEngineBuilder.get_or_create("mla-test", cfg, _meta()) is e
        with pytest.raises(ValueError, match="different"):
            LMCacheEngineBuilder.get_or_create("mla-test", cfg, _meta(mla=False))
    finally:
        LMCacheEngineBuilder.destroy("mla-test")


# ---------------------------------------------------------------------------------------------- refusals
def test_mla_refuses_the_huggingface_layout(monkeypatch):
    with pytest.raises(ValueError, match="vllm"):
        _engine(monkeypatch, _meta(fmt="huggingface"), local_device="cpu", remote_url=None)
    _engine(monkeypatch, _meta(fmt="huggingface", mla=False), local_device="cpu", remote_url=None)


def test_mla_refuses_reshard_world_sizes(monkeypatch):
    with pytest.raises(ValueError, match="reshard_world_sizes"):
        _engine(monkeypatch, _meta(), local_device=None, remote_url="lm://127.0.0.1:1", remote_serde="cachegen",
                reshard_world_sizes=[2])


@pytest.mark.parametrize("local,serde,remote,rserde", [("cpu", "cachegen", None, "torch"), ("/tmp/mla-kv/", None, None, "torch"),
                                                       (None, None, "lm://127.0.0.1:1", "cachegen"),
                                                       ("cpu", None, "lm://127.0.0.1:1", "cachegen")])
def test_mla_refuses_cachegen_chunks_over_256_tokens(monkeypatch, local, serde, remote, rserde):
    kw = dict(chunk_size=512, local_device=local, local_serde=serde, remote_url=remote, remote_serde=rserde)
    with pytest.raises(ValueError, match="256"):
        _engine(monkeypatch, _meta(), **kw)
    _engine(monkeypatch, _meta(), **dict(kw, chunk_size=256))
    _engine(monkeypatch, _meta(mla=False), **kw)


@pytest.mark.parametrize("local,remote,rserde", [("cpu", None, "torch"), ("cuda", None, "torch"),
                                                 (None, "lm://127.0.0.1:1", "torch")])
def test_mla_raw_tiers_take_any_chunk_size(monkeypatch, local, remote, rserde):
    _engine(monkeypatch, _meta(), chunk_size=512, local_device=local, remote_url=remote, remote_serde=rserde)


def test_pairs_to_an_mla_engine_and_latents_to_a_kv_engine_are_assertion_errors(monkeypatch):
    L, T, D = 3, 5, 8
    tokens = torch.arange(T)
    lat = tuple(torch.zeros(T, D, dtype=torch.bfloat16) for _ in range(L))
    pairs = tuple((torch.zeros(T, 1, D, dtype=torch.bfloat16),) * 2 for _ in range(L))
    paged_lat = [torch.zeros(2, 4, D, dtype=torch.bfloat16) for _ in range(L)]
    paged_pairs = [(torch.zeros(2, 4, 1, D, dtype=torch.bfloat16),) * 2 for _ in range(L)]
    slots = torch.arange(T)
    mla = _engine(monkeypatch, _meta(), local_device="cpu", remote_url=None)
    kv = _engine(monkeypatch, _meta(mla=False), local_device="cpu", remote_url=None)
    for eng, wrong, wrong_paged in ((mla, pairs, paged_pairs), (kv, lat, paged_lat)):
        with pytest.raises(AssertionError, match="pair"):
            eng.store(tokens, wrong)
        with pytest.raises(AssertionError, match="pair"):
            eng.store_layerwise(tokens, wrong)
        with pytest.raises(AssertionError, match="pair"):
            eng.store_paged(tokens, wrong_paged, slots)
        with pytest.raises(AssertionError, match="pair"):
            eng.store_paged_layerwise(tokens, wrong_paged, slots)
        with pytest.raises(AssertionError, match="pair"):
            eng.retrieve_paged(tokens, wrong_paged, slots)
        with pytest.raises(AssertionError, match="pair"):
            eng.retrieve_paged_layerwise(tokens, wrong_paged, slots)
    # the right kind gets past the argument checks: the token count is read from the latent's first dimension
    assert mla._num_tokens_in_kv(lat, "vllm") == T
    with pytest.raises(AssertionError, match="Number of tokens"):
        mla.store(torch.arange(T + 1), lat)


# ---------------------------------------------------------------------------------------------- keys
def test_every_rank_of_an_mla_engine_makes_the_keys_of_a_one_rank_layout(monkeypatch):
    from lmcache_b200.utils import CacheEngineKey
    one = _engine(monkeypatch, _meta(1, 0), local_device="cpu", remote_url=None)
    want = [one._make_key(h, "vllm") for h in ("a", "b")]
    assert want == [CacheEngineKey("vllm", MODEL, 1, 0, h) for h in ("a", "b")]
    for ws in (2, 4, 8):
        for rank in range(ws):
            eng = _engine(monkeypatch, _meta(ws, rank), local_device="cpu", remote_url=None)
            assert [eng._make_key(h, "vllm") for h in ("a", "b")] == want
            assert list(eng._keys_of(["a", "b"], "vllm")) == want
    kv = _engine(monkeypatch, _meta(8, 3, mla=False), local_device="cpu", remote_url=None)
    assert kv._make_key("a", "vllm") == CacheEngineKey("vllm", MODEL, 8, 3, "a")


# ---------------------------------------------------------------------------------------------- remote puts
class _Conn:
    def __init__(self):
        self.sets = []

    def set(self, key, value):
        self.sets.append(key)

    def exists(self, key):
        return key in self.sets

    def close(self):
        pass


class _Ser:
    def to_bytes(self, t):
        return b"x"

    def view_to_bytes_batch(self, view, chunk_size, tok_begin, n_tokens):
        return [b"x"] * ((n_tokens + chunk_size - 1) // chunk_size)


class _Deser:
    def from_bytes(self, bs):
        return None

    def decode_into(self, blobs, dst, toks):
        pass


class _View:
    ntokens = 600
    desc = None


def _remote(monkeypatch, meta):
    from lmcache_b200.config import LMCacheEngineConfig
    from lmcache_b200.storage_backend import remote_backend as rb
    monkeypatch.setattr(rb, "CreateConnector", lambda url: _Conn())
    monkeypatch.setattr(rb, "CreateSerde", lambda s, c, m: (_Ser(), _Deser()))
    cfg = LMCacheEngineConfig.from_defaults(local_device=None, remote_url="lm://127.0.0.1:1", remote_serde="torch")
    return rb.LMCRemoteBackend(cfg, meta)


def _keys(n):
    from lmcache_b200.utils import CacheEngineKey
    return [CacheEngineKey("vllm", MODEL, 1, 0, f"h{i}") for i in range(n)]


@pytest.mark.parametrize("ws,rank,mla", [(2, 0, True), (2, 1, True), (8, 7, True), (2, 1, False)])
def test_remote_tier_takes_latent_stores_from_rank_0_only(monkeypatch, ws, rank, mla):
    be = _remote(monkeypatch, _meta(ws, rank, mla=mla))
    try:
        stores = rank == 0 or not mla
        chunk = torch.zeros(1)
        be.put(_keys(1)[0], chunk)
        be.put(_keys(2)[1], chunk, blocking=False)
        be.batched_put(zip(_keys(4)[2:], [chunk] * 2))
        n = be.put_kv_chunks(_keys(3), _View(), 0, 256, blocking=True)
        be.put_kv_chunks(_keys(3), _View(), 0, 256, blocking=False)
        be.drain()
        assert n == (3 if stores else 0)
        assert len(be.connection.sets) == (10 if stores else 0)
        assert be.put_queue.empty()
    finally:
        be.close()


class _Local:
    def __init__(self):
        self.puts = []

    def put(self, key, chunk, blocking=True):
        self.puts.append(key)

    def put_kv_chunks(self, keys, view, tok_begin, chunk_size, blocking=True):
        self.puts.extend(keys)
        return len(keys)

    def close(self):
        pass


@pytest.mark.parametrize("rank", [0, 1])
def test_hybrid_fills_its_local_tier_on_every_rank_and_the_remote_one_from_rank_0(monkeypatch, rank):
    import lmcache_b200.storage_backend as sb
    from lmcache_b200.config import LMCacheEngineConfig
    from lmcache_b200.storage_backend import remote_backend as rb
    from lmcache_b200.storage_backend.hybrid_backend import LMCHybridBackend
    monkeypatch.setattr(rb, "CreateConnector", lambda url: _Conn())
    monkeypatch.setattr(rb, "CreateSerde", lambda s, c, m: (_Ser(), _Deser()))
    local = _Local()
    monkeypatch.setattr(sb, "CreateStorageBackend",
                        lambda c, m: rb.LMCRemoteBackend(c, m) if c.remote_url else local)
    cfg = LMCacheEngineConfig.from_defaults(local_device="cpu", remote_url="lm://127.0.0.1:1", remote_serde="torch",
                                            cachegen_config=mla_cfg(4))
    hy = LMCHybridBackend(cfg, _meta(2, rank))
    try:
        assert hy.remote_store.puts == (rank == 0)
        assert hy.put_kv_chunks(_keys(3), _View(), 0, 256) == 3
        hy.put(_keys(4)[3], torch.zeros(1))
        assert local.puts == _keys(4)
        assert len(hy.remote_store.connection.sets) == (4 if rank == 0 else 0)
    finally:
        hy.close()


def mla_cfg(L):
    return dict(key_first_layers=1, key_second_layers=2, key_third_layers=L, key_first_bins=32, key_second_bins=16,
                key_third_bins=8, value_first_layers=2, value_first_bins=32, value_second_bins=16)


# ---------------------------------------------------------------------------------------------- layer-major uploads
def test_layer_copy_ranges_of_one_plane_per_layer():
    from lmcache_b200.pipeline import layer_copy_ranges
    L = 5
    rng = np.random.default_rng(3)
    offs, sizes = [], []
    for j in range(4):
        o = np.concatenate([[100 + j], 100 + j + np.cumsum(rng.integers(0, 50, L))]).astype(np.int64)
        offs.append(o)
        sizes.append(int(o[-1]))
    offs[2] = None                               # no plane offsets: uploaded whole with the fixed sections
    sizes[2] = 777
    fixed, start, size = layer_copy_ranges(offs, sizes, L, 1)
    assert start.shape == size.shape == (L, 4)
    assert list(fixed) == [100, 101, 777, 103]
    for j, o in enumerate(offs):
        if o is None:
            assert (size[:, j] == 0).all()
            continue
        assert list(start[:, j]) == list(o[:L]) and list(size[:, j]) == list(np.diff(o))
        # fixed sections then the L planes cover the container exactly once
        cover = np.zeros(sizes[j], np.int32)
        cover[:fixed[j]] += 1
        for l in range(L):
            cover[start[l, j]:start[l, j] + size[l, j]] += 1
        assert (cover == 1).all()
    # two planes per layer: what the (K, V) upload has always taken
    po = [np.arange(2 * L + 1, dtype=np.int64) * 10 + 64]
    f2, s2, z2 = layer_copy_ranges(po, [int(po[0][-1])], L)
    assert s2.shape == (L, 2) and list(s2[:, 0]) == list(po[0][:L]) and list(s2[:, 1]) == list(po[0][L:2 * L])
    assert (z2 == 10).all() and list(f2) == [64]


def test_segment_rows_are_sized_for_the_planes_of_a_chunk():
    from lmcache_b200.pipeline import SegmentSlot

    class _T:
        def __init__(self, n):
            self.n = n

        def numel(self):
            return self.n

    class _B:
        def __init__(self, n):
            self.nbytes = n

    L, n = 61, 3
    s = SegmentSlot.__new__(SegmentSlot)
    s.arena, s.fixed, s.ws = _T(1000), _T(1000), _T(1000)
    s.sizes, s.seg = _B(8 * n), _B(16 * L * n)               # (offset, bytes) rows of L planes per chunk
    assert s.holds(1000, 1000, 1000, n, L)                   # a latent KV: P = L
    assert not s.holds(1000, 1000, 1000, n, 2 * L)           # the (K, V) pairs of the same model: P = 2L
    s.seg = _B(16 * 2 * L * n)
    assert s.holds(1000, 1000, 1000, n, 2 * L)


# ---------------------------------------------------------------------------------------------- disk index
def _disk_index(path, latent):
    from lmcache_b200.storage_backend.local_backend import LMCLocalDiskBackend
    b = LMCLocalDiskBackend.__new__(LMCLocalDiskBackend)
    b.path, b.dict, b.capacity, b.latent = str(path) + "/", {}, None, latent
    b._rebuild_index()
    return {os.path.basename(p): e.rec for p, e in b.dict.items()}


def test_disk_index_admits_version_4_for_a_latent_engine_only(tmp_path):
    t, D = 7, 64
    kb = np.full(4, 16, np.float32)
    v4, ends, _ = mla_ref.v4_container(O.synth_kv_bits(2, t, D, seed=5)[:, 0], O.DT_BF16, kb, 1, D)
    # version 3 of one layer is, byte for byte, version 4 of its two planes with another header
    raw3 = bytearray(v4)
    raw3[4:12] = (3).to_bytes(4, "little") + (1).to_bytes(4, "little")
    v4b, _, _ = mla_ref.v4_container(O.synth_kv_bits(1, t, D, seed=6)[:, 0], O.DT_BF16, kb, 1, D)
    (tmp_path / "a.b2kv").write_bytes(v4)
    (tmp_path / "b.b2kv").write_bytes(bytes(raw3))
    (tmp_path / "c.b2kv").write_bytes(v4b)
    (tmp_path / "d.b2kv").write_bytes(v4b[:-3])              # truncated: never part of the cache
    (tmp_path / "e.b2kv.tmp").write_bytes(v4b)               # an unfinished write
    lat = _disk_index(tmp_path, True)
    assert sorted(lat) == ["a.b2kv", "c.b2kv"]
    assert all(r.coder == N.CODER_LATENT for r in lat.values())
    assert (lat["a.b2kv"].L, lat["a.b2kv"].H, lat["a.b2kv"].D, lat["a.b2kv"].ntokens) == (2, 1, D, t)
    assert lat["a.b2kv"].nbytes == len(v4) == ends[-1]
    kv = _disk_index(tmp_path, False)
    assert sorted(kv) == ["b.b2kv"] and kv["b.b2kv"].coder == N.CODER_RANS_COMPACT and kv["b.b2kv"].L == 1
