"""CPU: serving another tensor-parallel layout's chunks -- the head arithmetic of lmcache_b200.reshard, the
reshard_world_sizes configuration key and its rejections, and the engine's choice of layout and source groups against a
stand-in backend."""
import pytest

from lmcache_b200.reshard import Shard, first_source_rank, source_shards

MODEL = "lmsys/longchat-7b-16k"


# ---------------------------------------------------------------------------------------------- head arithmetic
@pytest.mark.parametrize("Hg", range(1, 33))
def test_source_shards_cover_every_destination_head_once(Hg):
    for W in range(1, 9):
        for Wd in range(1, 9):
            for r in range(Wd):
                shards = source_shards(Hg, W, Wd, r)
                if Hg % W or Hg % Wd:
                    assert shards == []
                    continue
                hs, hd = Hg // W, Hg // Wd
                got = {}
                for s in shards:
                    assert isinstance(s, Shard) and s.n_heads >= 1
                    assert 0 <= s.src_head0 and s.src_head0 + s.n_heads <= hs
                    for k in range(s.n_heads):
                        d = s.dst_head0 + k
                        assert d not in got, "a destination head is covered twice"
                        got[d] = s.rank * hs + s.src_head0 + k           # the model head the source stores there
                assert got == {d: r * hd + d for d in range(hd)}      # every head, from the right model head
                assert [s.rank for s in shards] == sorted(s.rank for s in shards)
                assert shards[0].rank == first_source_rank(W, Wd, r)
                if W % Wd == 0 or Wd % W == 0:                     # one container partly, or W / W' whole
                    assert len(shards) == max(1, W // Wd)
                    assert all(s.n_heads == hs for s in shards) if W >= Wd else shards[0].n_heads == hd


def test_source_shards_examples():
    assert source_shards(8, 1, 2, 1) == [Shard(0, 4, 4, 0)]
    assert source_shards(8, 4, 2, 1) == [Shard(2, 0, 2, 0), Shard(3, 0, 2, 2)]
    assert source_shards(6, 2, 3, 1) == [Shard(0, 2, 1, 0), Shard(1, 0, 1, 1)]
    assert source_shards(4, 8, 1, 0) == []            # KV heads replicated above Hg: out of scope
    assert source_shards(8, 2, 1, 1) == []            # no rank 1 in a one-rank layout
    assert first_source_rank(2, 1, 1) is None


# ---------------------------------------------------------------------------------------------- configuration
def test_reshard_config_key_yaml_and_constructors(tmp_path):
    from lmcache_b200.config import LMCacheEngineConfig
    p = tmp_path / "cfg.yaml"
    p.write_text("chunk_size: 256\nremote_url: lm://127.0.0.1:65000\nremote_serde: cachegen\n"
                 "reshard_world_sizes: [2, 4]\n")
    assert LMCacheEngineConfig.from_file(str(p)).reshard_world_sizes == [2, 4]
    p.write_text("chunk_size: 256\nremote_url: lm://127.0.0.1:65000\n")
    assert LMCacheEngineConfig.from_file(str(p)).reshard_world_sizes is None
    assert LMCacheEngineConfig.from_defaults(reshard_world_sizes=[1]).reshard_world_sizes == [1]
    assert LMCacheEngineConfig.from_legacy(backend="lm://127.0.0.1:1", remote_serde="cachegen",
                                           reshard_world_sizes=(8, 2)).reshard_world_sizes == [8, 2]
    assert LMCacheEngineConfig.from_legacy(backend="cpu").reshard_world_sizes is None
    for bad in ([], [0], [-2], [2, 2], [1.0], [True], "2", 2, [None]):
        with pytest.raises(ValueError, match="reshard"):
            LMCacheEngineConfig.from_defaults(reshard_world_sizes=bad)
        with pytest.raises(ValueError, match="reshard"):
            LMCacheEngineConfig.from_legacy(backend="lm://127.0.0.1:1", reshard_world_sizes=bad)
    p.write_text("chunk_size: 256\nremote_url: lm://127.0.0.1:65000\nreshard_world_sizes: [2, 2]\n")
    with pytest.raises(ValueError, match="reshard"):
        LMCacheEngineConfig.from_file(str(p))


@pytest.mark.parametrize("local,remote,serde", [("cpu", None, "cachegen"), ("/tmp/kv/", None, "cachegen"),
                                                (None, "lm://127.0.0.1:1", "torch"),
                                                ("cpu", "lm://127.0.0.1:1", "torch")])
def test_reshard_is_rejected_without_a_cachegen_remote_tier(local, remote, serde):
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    from lmcache_b200.storage_backend import CreateStorageBackend
    cfg = LMCacheEngineConfig(256, local, remote, serde, False, False, reshard_world_sizes=[2])
    with pytest.raises(ValueError, match="reshard_world_sizes"):
        CreateStorageBackend(cfg, LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16"))


def test_engine_rejects_its_own_world_size(monkeypatch):
    import lmcache_b200.cache_engine as ce
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    monkeypatch.setattr(ce, "CreateStorageBackend", lambda cfg, meta: _FakeBackend(set()))
    cfg = LMCacheEngineConfig.from_defaults(remote_url="lm://127.0.0.1:1", remote_serde="cachegen",
                                            reshard_world_sizes=[1, 2])
    with pytest.raises(ValueError, match="own world size"):
        ce.LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, 2, 0, "vllm", "bfloat16"))
    ce.LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, 4, 3, "vllm", "bfloat16"))


# ---------------------------------------------------------------------------------------------- engine
class _FakeBackend:
    """Holds a set of keys; get_kv_shards_into serves a group when every key of it is held, up to the first that is not."""

    def __init__(self, held):
        self.held = held
        self.contains_calls = []
        self.calls = []

    def contains(self, key):
        self.contains_calls.append(key)
        return key in self.held

    def get_kv_shards_into(self, groups, dst, dst_tok0, chunk_size, stats=None):
        self.calls.append((groups, dst_tok0))
        n = 0
        for g in groups:
            if not all(k in self.held for k, _ in g):
                break
            n += 1
        if stats is not None:
            stats["bytes"] = stats.get("bytes", 0) + 100 * n
        return n

    def close(self):
        pass


class _View:
    def __init__(self, H):
        self.H = H


def _engine(monkeypatch, held, ws, rank, sizes):
    import lmcache_b200.cache_engine as ce
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    be = _FakeBackend(held)
    monkeypatch.setattr(ce, "CreateStorageBackend", lambda cfg, meta: be)
    cfg = LMCacheEngineConfig.from_defaults(remote_url="lm://127.0.0.1:1", remote_serde="cachegen",
                                            reshard_world_sizes=sizes)
    return ce.LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, ws, rank, "vllm", "bfloat16")), be


def _key(h, W, r):
    from lmcache_b200.utils import CacheEngineKey
    return CacheEngineKey("vllm", MODEL, W, r, h)


def test_engine_takes_the_first_complete_layout_and_stops_at_an_incomplete_chunk(monkeypatch):
    hashes = [f"h{i}" for i in range(6)]
    held = set()
    for i in range(6):
        held.add(_key(hashes[i], 4, 2))                       # layout 4 lacks rank 3 of every chunk: never complete
    for i in range(4):
        held.add(_key(hashes[i], 1, 0))                       # layout 1 holds chunks 0..3
    held |= {_key(hashes[i], 8, r) for i in range(6) for r in range(4, 8)}     # layout 8 would hold all, but comes last
    eng, be = _engine(monkeypatch, held, 2, 1, [4, 1, 8])     # Hg = 8 at W' = 2: rank 1 owns heads 4..7
    layout, n = eng._reshard_get(hashes[1:], "vllm", _View(4), 256)
    assert (layout, n) == (1, 3)                              # chunks 1..3; chunk 4 is missing
    groups, tok0 = be.calls[-1]
    assert tok0 == 256 and len(groups) == 5
    (k, w), = groups[0]
    assert k == _key("h1", 1, 0) and tuple(w) == (8, 4, 4, 0)
    assert eng.reshard_stats() == {1: {"chunks": 3, "bytes": 300}}
    # a continuation keeps its layout: no new choice
    nc = len(be.contains_calls)
    assert eng._reshard_get(hashes[4:], "vllm", _View(4), 0, 8) == (8, 2)
    assert len(be.contains_calls) == nc
    assert [k for k, _ in be.calls[-1][0][0]] == [_key("h4", 8, r) for r in range(4, 8)]
    assert eng.reshard_stats() == {1: {"chunks": 3, "bytes": 300}, 8: {"chunks": 2, "bytes": 200}}


def test_engine_groups_for_a_larger_source_layout(monkeypatch):
    eng, _ = _engine(monkeypatch, set(), 2, 1, [4])
    groups = eng._reshard_groups(["a", "b"], "huggingface", 4, 8)
    assert len(groups) == 2
    assert [(k.world_size, k.worker_id, k.fmt, k.chunk_hash) for k, _ in groups[1]] == \
        [(4, 2, "huggingface", "b"), (4, 3, "huggingface", "b")]
    assert [tuple(w) for _, w in groups[1]] == [(2, 0, 2, 0), (2, 0, 2, 2)]


def test_engine_without_a_complete_layout_serves_nothing(monkeypatch):
    eng, be = _engine(monkeypatch, {_key("h0", 2, 0)}, 1, 0, [2])     # rank 1 of layout 2 is missing
    assert eng._reshard_get(["h0", "h1"], "vllm", _View(8), 0) == (None, 0)
    assert be.calls == [] and eng.reshard_stats() == {}


def test_engine_is_off_without_the_key(monkeypatch):
    import lmcache_b200.cache_engine as ce
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    be = _FakeBackend({_key("h0", 2, 0), _key("h0", 2, 1)})
    monkeypatch.setattr(ce, "CreateStorageBackend", lambda cfg, meta: be)
    eng = ce.LMCacheEngine(LMCacheEngineConfig.from_defaults(remote_url="lm://127.0.0.1:1", remote_serde="cachegen"),
                           LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16"))
    assert eng._reshard_get(["h0"], "vllm", _View(8), 0) == (None, 0)
    assert be.contains_calls == [] and be.calls == []
