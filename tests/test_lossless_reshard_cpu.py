"""CPU: retrieving another tensor-parallel layout's lossless containers -- the reshard_lossless configuration key, the
factory accepting reshard_world_sizes with remote_serde="lossless" once reshard_lossless is set (every tier class
replaced by a recorder: no server, no device) and refusing it otherwise, an MLA engine still refusing it, and the new
entry point b200kv_lossless_decode_plan_heads declared in include/b200kv.h and bound in lmcache_b200/_native.py."""
import ctypes
import os
import re

import pytest

from lmcache_b200 import _native as N
from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
from lmcache_b200.storage_backend import CreateStorageBackend

MODEL = "lmsys/longchat-7b-16k"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _meta(mla=False, W=1, r=0):
    return LMCacheEngineMetadata(MODEL, W, r, "vllm", "bfloat16", use_mla=mla)


def _factory(monkeypatch):
    """CreateStorageBackend with every tier class replaced by a recorder: the factory's choice, without a device or a
    server"""
    from lmcache_b200.storage_backend import hybrid_backend, local_backend, remote_backend
    made = []

    def fake(name):
        class T:
            def __init__(self, config, metadata):
                made.append((name, config.remote_serde, config.reshard_world_sizes))
        return T
    for name in ("LMCLocalBackend", "LMCLocalCompressedBackend", "LMCLocalDiskBackend"):
        monkeypatch.setattr(local_backend, name, fake(name))
    for name in ("LMCRemoteBackend", "LMCPipelinedRemoteBackend"):
        monkeypatch.setattr(remote_backend, name, fake(name))
    monkeypatch.setattr(hybrid_backend, "LMCHybridBackend", fake("LMCHybridBackend"))
    return made


# ---------------------------------------------------------------------------------------------- the configuration key
def test_reshard_lossless_key_yaml_and_constructors(tmp_path):
    url = "lm://127.0.0.1:1"
    assert LMCacheEngineConfig(256, None, url, "lossless", False, False).reshard_lossless is False
    assert LMCacheEngineConfig.from_defaults(remote_url=url, remote_serde="lossless").reshard_lossless is False
    cfg = LMCacheEngineConfig.from_defaults(local_device=None, remote_url=url, remote_serde="lossless",
                                            reshard_world_sizes=[2], reshard_lossless=True)
    assert (cfg.reshard_world_sizes, cfg.reshard_lossless) == ([2], True)
    cfg = LMCacheEngineConfig.from_legacy(backend=url, remote_serde="lossless", reshard_world_sizes=[4, 2],
                                          reshard_lossless=True)
    assert (cfg.remote_url, cfg.reshard_world_sizes, cfg.reshard_lossless) == (url, [4, 2], True)
    p = tmp_path / "cfg.yaml"
    p.write_text(f"chunk_size: 256\nremote_url: {url}\nremote_serde: lossless\nreshard_world_sizes: [2]\n"
                 f"reshard_lossless: true\n")
    assert LMCacheEngineConfig.from_file(str(p)).reshard_lossless is True
    p.write_text(f"chunk_size: 256\nremote_url: {url}\nremote_serde: lossless\nreshard_world_sizes: [2]\n")
    assert LMCacheEngineConfig.from_file(str(p)).reshard_lossless is False


@pytest.mark.parametrize("kw", [dict(reshard_world_sizes=None), dict(remote_serde="cachegen"),
                                dict(remote_serde="torch"), dict(reshard_lossless=1), dict(reshard_lossless="yes")])
def test_reshard_lossless_key_is_validated(kw):
    a = dict(local_device=None, remote_url="lm://127.0.0.1:1", remote_serde="lossless", reshard_world_sizes=[2],
             reshard_lossless=True)
    a.update(kw)
    with pytest.raises(ValueError, match="reshard_lossless"):
        LMCacheEngineConfig.from_defaults(**a)


# ---------------------------------------------------------------------------------------------- the factory's gate
@pytest.mark.parametrize("local,lserde,pipelined,want", [
    (None, None, False, "LMCRemoteBackend"), (None, None, True, "LMCPipelinedRemoteBackend"),
    ("cpu", "lossless", False, "LMCHybridBackend"), ("cpu", "cachegen", False, "LMCHybridBackend")])
def test_reshard_is_accepted_with_a_lossless_remote_tier_that_opts_in(local, lserde, pipelined, want, monkeypatch):
    made = _factory(monkeypatch)
    cfg = LMCacheEngineConfig(256, local, "lm://127.0.0.1:1", "lossless", pipelined, False, lserde,
                              reshard_world_sizes=[2, 4], reshard_lossless=True)
    CreateStorageBackend(cfg, _meta())
    assert made == [(want, "lossless", [2, 4])]


@pytest.mark.parametrize("local,lserde", [(None, None), ("cpu", "lossless"), ("cpu", "cachegen")])
def test_reshard_with_a_lossless_remote_tier_is_refused_without_the_opt_in(local, lserde, monkeypatch):
    made = _factory(monkeypatch)
    cfg = LMCacheEngineConfig(256, local, "lm://127.0.0.1:1", "lossless", False, False, lserde, reshard_world_sizes=[2])
    with pytest.raises(ValueError, match="reshard_world_sizes.*reshard_lossless"):
        CreateStorageBackend(cfg, _meta())
    assert made == []


def test_reshard_is_still_accepted_with_a_cachegen_remote_tier(monkeypatch):
    made = _factory(monkeypatch)
    CreateStorageBackend(LMCacheEngineConfig(256, None, "lm://127.0.0.1:1", "cachegen", False, False,
                                             reshard_world_sizes=[2]), _meta())
    assert made == [("LMCRemoteBackend", "cachegen", [2])]


@pytest.mark.parametrize("local,remote,serde,lserde", [
    (None, "lm://127.0.0.1:1", "torch", None), ("cpu", "lm://127.0.0.1:1", "torch", "lossless"),
    ("cpu", None, "lossless", "lossless"), ("cpu", None, "cachegen", "cachegen"), ("/tmp/kv/", None, "lossless", "lossless"),
    ("cuda", None, "lossless", None)])
def test_reshard_is_refused_without_a_container_remote_tier(local, remote, serde, lserde, monkeypatch):
    made = _factory(monkeypatch)
    cfg = LMCacheEngineConfig(256, local, remote, serde, False, False, lserde, reshard_world_sizes=[2])
    with pytest.raises(ValueError, match="reshard_world_sizes"):
        CreateStorageBackend(cfg, _meta())
    assert made == []


def test_mla_still_refuses_reshard_with_the_lossless_serde(monkeypatch):
    import lmcache_b200.cache_engine as ce
    monkeypatch.setattr(ce, "CreateStorageBackend", lambda c, m: pytest.fail("the backend must not be made"))
    cfg = LMCacheEngineConfig.from_defaults(chunk_size=256, local_device=None, remote_url="lm://127.0.0.1:1",
                                            remote_serde="lossless", reshard_world_sizes=[2], reshard_lossless=True)
    with pytest.raises(ValueError, match="reshard_world_sizes"):
        ce.LMCacheEngine(cfg, _meta(mla=True))


def test_engine_with_a_lossless_reshard_config_is_made(monkeypatch):
    """past the factory, the engine adds no rule of its own for the lossless serde (its own world size stays refused)"""
    import lmcache_b200.cache_engine as ce
    made = _factory(monkeypatch)
    cfg = LMCacheEngineConfig.from_defaults(chunk_size=256, local_device=None, remote_url="lm://127.0.0.1:1",
                                            remote_serde="lossless", reshard_world_sizes=[2], reshard_lossless=True)
    e = ce.LMCacheEngine(cfg, _meta(W=1))
    assert made == [("LMCRemoteBackend", "lossless", [2])] and e.reshard_stats() == {}
    with pytest.raises(ValueError, match="own world size"):
        ce.LMCacheEngine(cfg, _meta(W=2, r=1))


# ---------------------------------------------------------------------------------------------- the C ABI
def test_plan_heads_symbol_is_declared_and_bound():
    name = "b200kv_lossless_decode_plan_heads"
    with open(os.path.join(ROOT, "include", "b200kv.h")) as f:
        hdr = f.read()
    m = re.search(r"int\s+" + name + r"\(([^;]*)\);", hdr)
    assert m is not None, "not declared in include/b200kv.h"
    nargs = len([a for a in m.group(1).split(",") if a.strip()])
    res, args = N.SIGNATURES[name]
    assert res is ctypes.c_int32 and len(args) == nargs == 18
    # the whole plan's arguments, then (src_H, src_head0, dst_head0, n_heads)
    assert args[:14] == N.SIGNATURES["b200kv_lossless_decode_plan"][1]
    assert args[14:] == [ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    # listed among the symbols added without changing B200KV_VERSION
    vblock = hdr[hdr.index("#define B200KV_VERSION"):]
    vblock = vblock[:vblock.index("*/")]
    assert name in vblock


def test_lossless_codec_offers_the_window_calls_of_the_cachegen_codec():
    import inspect

    from lmcache_b200.codec import CacheGenCodec, LosslessCodec
    for fn in ("decode_raw_heads", "decode_plan_heads"):
        a = list(inspect.signature(getattr(CacheGenCodec, fn)).parameters)
        b = list(inspect.signature(getattr(LosslessCodec, fn)).parameters)
        assert a == b, fn
