"""CPU: models of up to 128 layers and CacheGen bin layouts outside the five-model table.

* LMCacheEngineConfig.cachegen_config: the YAML key, both constructors, every rejection, and the bin lists it gives
  (a layout that mirrors longchat's is the reference's golden lists).
* parse_header / check_header at L = 128 and 129.
* b200kv_plane_offsets (host) on a 128-layer version-3 container assembled from the oracle's encode.
* The plan structs' sizes: b200kv_encode_plan_t grew to 512 words with the plane table; b200kv_decode_plan_t keeps its
  256, and the decode workspace holds the table of a model deeper than 64 layers."""
import ctypes

import numpy as np
import pytest

from lmcache_b200 import _native as N
from lmcache_b200.codec import check_header, parse_header, plane_offsets
from lmcache_b200.config import LMCacheEngineConfig
from oracle import oracle as O

LONGCHAT = dict(key_first_layers=10, key_second_layers=20, key_third_layers=32, key_first_bins=32, key_second_bins=16,
                key_third_bins=16, value_first_layers=2, value_first_bins=32, value_second_bins=16)
LLAMA70B = dict(LONGCHAT, key_third_layers=80)


def _bins(cfg):
    from lmcache_b200.storage_backend.serde.cachegen_basics import CacheGenConfig
    c = CacheGenConfig(**cfg)
    return np.array(c.key_bins_list(), np.float32), np.array(c.value_bins_list(), np.float32)


def _v3_container(L, t, H, D, kb, vb, seed):
    """one chunk's version-3 container (include/b200kv.h), assembled on the host from the oracle's encode"""
    bits = O.synth_kv_bits(L, t, H * D, seed=seed)
    enc = O.encode_chunk(bits, O.DT_BF16, kb, vb, O.CODER_RANS_COMPACT)
    (bs, ln, _), = enc["groups"]
    nb = O.nb_map(kb, vb, L)
    payload, half = O.v3_pack(enc["counts"], nb, ln, bs)
    NL, C = 2 * L, H * D
    lo = N.container_layout(L, H, D, t, N.CODER_RANS_COMPACT)
    total = lo.off_payload + payload.size
    buf = bytearray(total)
    hd = N.Header()
    hd.magic, hd.version, hd.L, hd.H, hd.D, hd.ntokens, hd.ngroups = N.MAGIC, 3, L, H, D, t, 1
    hd.max_dtype, hd.payload_bytes, hd.total_bytes = N.DT_BF16, payload.size, total
    buf[:N.HEADER_BYTES] = bytes(hd)
    buf[lo.off_cdf:lo.off_cdf + NL] = bytes(nb)
    buf[lo.off_maxes:lo.off_maxes + enc["maxes"].nbytes] = enc["maxes"].tobytes()
    buf[lo.off_lengths:lo.off_lengths + NL * C] = half.tobytes()
    buf[lo.off_payload:] = payload.tobytes()
    ends = lo.off_payload + np.concatenate([[0], np.cumsum(2 * half.reshape(NL, C).astype(np.int64).sum(axis=1))])
    return bytes(buf), ends


# ------------------------------------------------------------------------------------------------ cachegen_config
def test_cachegen_config_default_is_none_and_table_unchanged():
    from lmcache_b200.storage_backend.serde.cachegen_basics import CacheGenConfig
    assert LMCacheEngineConfig.from_defaults().cachegen_config is None
    assert LMCacheEngineConfig.from_legacy().cachegen_config is None
    with pytest.raises(ValueError):
        CacheGenConfig.from_model_name("meta-llama/Llama-3.1-70B-Instruct")
    with pytest.raises(ValueError):
        CacheGenConfig.for_engine("meta-llama/Llama-3.1-70B-Instruct")
    assert CacheGenConfig.for_engine("lmsys/longchat-7b-16k") == CacheGenConfig.from_model_name("lmsys/longchat-7b-16k")


def test_cachegen_config_constructors_and_yaml(tmp_path):
    a = LMCacheEngineConfig.from_defaults(cachegen_config=LLAMA70B)
    b = LMCacheEngineConfig.from_legacy(chunk_size=256, backend="cpu", cachegen_config=LLAMA70B)
    assert a.cachegen_config == LLAMA70B and b.cachegen_config == LLAMA70B
    assert a.cachegen_config is not LLAMA70B            # a copy: the caller's mapping may change later
    p = tmp_path / "deep.yaml"
    p.write_text("chunk_size: 256\nlocal_device: cpu\nlocal_serde: cachegen\ncachegen_config:\n" +
                 "".join(f"  {k}: {v}\n" for k, v in LLAMA70B.items()))
    c = LMCacheEngineConfig.from_file(str(p))
    assert c.cachegen_config == LLAMA70B and c.local_device == "cpu"
    p.write_text("chunk_size: 256\nlocal_device: cpu\n")
    assert LMCacheEngineConfig.from_file(str(p)).cachegen_config is None
    p.write_text("chunk_size: 256\ncachegen_config:\n  key_third_layers: 80\n")
    with pytest.raises(ValueError):
        LMCacheEngineConfig.from_file(str(p))
    # the reference's own type is accepted too, as its nine fields
    from lmcache_b200.storage_backend.serde.cachegen_basics import CacheGenConfig
    assert LMCacheEngineConfig.from_defaults(cachegen_config=CacheGenConfig(**LLAMA70B)).cachegen_config == LLAMA70B


@pytest.mark.parametrize("bad", [
    "not a mapping", [1, 2], {},
    {k: v for k, v in LLAMA70B.items() if k != "value_second_bins"},          # a field missing
    dict(LLAMA70B, extra=1),                                                  # a field too many
    dict(LLAMA70B, key_third_layers=0), dict(LLAMA70B, key_third_layers=129), dict(LLAMA70B, key_third_layers=-3),
    dict(LLAMA70B, key_third_layers=80.0), dict(LLAMA70B, key_third_layers="80"), dict(LLAMA70B, key_first_bins=True),
    dict(LLAMA70B, key_first_layers=-1), dict(LLAMA70B, key_second_layers=-1), dict(LLAMA70B, value_first_layers=-1),
    dict(LLAMA70B, key_first_bins=3), dict(LLAMA70B, key_first_bins=33), dict(LLAMA70B, key_second_bins=2),
    dict(LLAMA70B, key_third_bins=64), dict(LLAMA70B, value_first_bins=0), dict(LLAMA70B, value_second_bins=40),
])
def test_cachegen_config_rejections(bad):
    for make in (lambda: LMCacheEngineConfig.from_defaults(cachegen_config=bad),
                 lambda: LMCacheEngineConfig.from_legacy(cachegen_config=bad),
                 lambda: LMCacheEngineConfig(256, "cpu", None, "torch", False, False, cachegen_config=bad)):
        with pytest.raises(ValueError):
            make()


def test_cachegen_config_bins_that_no_layer_gets_are_not_checked():
    """a bin count that no layer gets says nothing about the quantiser: such a layout is accepted"""
    ok = [dict(LLAMA70B, key_first_layers=0, key_first_bins=0),                     # no first key band
          dict(LLAMA70B, key_second_layers=10, key_second_bins=99),                 # second band inside the first
          dict(LLAMA70B, key_second_layers=80, key_third_bins=1),                   # second band reaches the last layer
          dict(LLAMA70B, value_first_layers=0, value_first_bins=-5),
          dict(LLAMA70B, value_first_layers=200, value_second_bins=1),
          dict(LLAMA70B, key_third_layers=1), dict(LLAMA70B, key_third_layers=128)]
    for cfg in ok:
        c = LMCacheEngineConfig.from_defaults(cachegen_config=cfg).cachegen_config
        kb, vb = _bins(c)
        assert len(kb) == len(vb) == cfg["key_third_layers"]
        assert ((kb >= 4) & (kb <= 32)).all() and ((vb >= 4) & (vb <= 32)).all()


def test_cachegen_config_mirroring_longchat_gives_reference_golden_bins(golden):
    from lmcache_b200.storage_backend.serde.cachegen_basics import CacheGenConfig
    cfg = LMCacheEngineConfig.from_defaults(cachegen_config=LONGCHAT).cachegen_config
    c = CacheGenConfig.for_engine("any/model-name", cfg)
    assert c.key_bins_list() == golden["key_bins"].tolist()
    assert c.value_bins_list() == golden["value_bins"].tolist()
    assert c == CacheGenConfig.from_model_name("lmsys/longchat-7b-16k")
    kb, vb = _bins(LLAMA70B)
    assert kb.tolist() == [32.0] * 10 + [16.0] * 70 and vb.tolist() == [32.0] * 2 + [16.0] * 78


# ------------------------------------------------------------------------------------------------ headers
def test_max_planes_admits_128_layers():
    assert N.MAX_PLANES == 256
    assert ctypes.sizeof(N.EncodePlan) == 4096            # the encode plan holds the 256-plane parameter block
    assert ctypes.sizeof(N.DecodePlan) == 2048            # the decode plan keeps its size: deep tables go to the workspace
    lib = N.lib()
    small = lib.b200kv_decode_workspace_bytes(64, 8, 128, 256, 4)
    deep = lib.b200kv_decode_workspace_bytes(65, 8, 128, 256, 4)
    assert deep >= small + 3072                            # ... which counts the table beyond 64 layers


@pytest.mark.parametrize("version", [1, 2, 3])
def test_check_header_at_128_and_129_layers(version):
    L, H, D, t = 128, 1, 8, 4
    lo = N.container_layout(L, H, D, t, version - 1)
    hd = N.Header()
    hd.magic, hd.version, hd.L, hd.H, hd.D, hd.ntokens, hd.ngroups = N.MAGIC, version, L, H, D, t, 1
    hd.max_dtype = N.DT_BF16
    hd.payload_bytes = 4 * 2 * L * H * D
    hd.total_bytes = lo.off_payload + hd.payload_bytes
    nb = [16] * (2 * L)
    check_header(hd, nb if version == 3 else None)
    hd.L = 129
    with pytest.raises(ValueError):
        check_header(hd, [16] * 258 if version == 3 else None)


def test_parse_header_at_128_and_129_layers():
    kb, vb = _bins(dict(LLAMA70B, key_third_layers=128))
    raw, _ = _v3_container(128, 3, 1, 16, kb, vb, seed=5)
    hd = parse_header(raw)
    assert (hd.version, hd.L, hd.ntokens) == (3, 128, 3)
    assert hd.nb == O.nb_map(kb, vb, 128)
    bad = bytearray(raw)
    bad[8:12] = (129).to_bytes(4, "little")
    with pytest.raises(ValueError):
        parse_header(bytes(bad))


def test_host_plane_offsets_on_128_layer_oracle_container():
    rng = np.random.default_rng(3)
    L, t, H, D = 128, 17, 2, 20
    kb = rng.integers(4, 33, size=L).astype(np.float32)
    vb = rng.integers(4, 33, size=L).astype(np.float32)
    raw, ends = _v3_container(L, t, H, D, kb, vb, seed=9)
    a = np.frombuffer(raw, np.uint8)
    o = np.full(N.MAX_PLANES + 1, -5, np.int64)
    assert N.lib().b200kv_plane_offsets(a.ctypes.data, a.size, o.ctypes.data, o.size) == 0
    assert np.array_equal(o[:2 * L + 1], ends) and o[2 * L] == len(raw)
    assert (o[2 * L + 1:] == -5).all()
    assert np.array_equal(plane_offsets(raw), ends)
    # too small an output, and a header that claims 129 layers, are refused
    assert N.lib().b200kv_plane_offsets(a.ctypes.data, a.size, o.ctypes.data, 2 * L) < 0
    bad = bytearray(raw)
    bad[8:12] = (129).to_bytes(4, "little")
    b = np.frombuffer(bytes(bad), np.uint8)
    assert N.lib().b200kv_plane_offsets(b.ctypes.data, b.size, o.ctypes.data, o.size) < 0
