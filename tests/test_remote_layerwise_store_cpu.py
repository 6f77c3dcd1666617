"""CPU: the host-side rules of the layer-wise store on the remote and hybrid tiers -- when two codecs write the same
containers (pipeline.same_containers), which handle a hybrid tier returns (one shared encode, a fan-out of both parts'
handles, or None), and the reference count that returns a slot two sinks land to its pool only after both."""
import queue
import threading
from types import SimpleNamespace

import pytest

from lmcache_b200 import _native as N
from lmcache_b200.codec import CacheGenCodec, LosslessCodec
from lmcache_b200.pipeline import EncodeRing, FanOutEncode, SegmentPool, layerwise_encodes, same_containers
from lmcache_b200.storage_backend.hybrid_backend import LMCHybridBackend
from lmcache_b200.storage_backend.serde.cachegen_basics import CacheGenConfig

MODEL = "lmsys/longchat-7b-16k"


def _cg_config(L=4, vbins=16):
    return dict(key_first_layers=min(3, L), key_second_layers=min(20, L), key_third_layers=L, key_first_bins=32,
                key_second_bins=16, key_third_bins=12, value_first_layers=2, value_first_bins=32, value_second_bins=vbins)


def _cachegen(model=MODEL, coder="rans_compact", cachegen_config=None):
    """a CacheGenCodec's rule-bearing fields, without the device buffers its constructor makes"""
    c = object.__new__(CacheGenCodec)
    c.coder = N.CODERS[coder]
    c.v3_only = cachegen_config is not None
    c.config = CacheGenConfig.for_engine(model, cachegen_config)
    return c


def _lossless():
    return object.__new__(LosslessCodec)


# ---------------------------------------------------------------------------------------------- same_containers
@pytest.mark.parametrize("latent", [False, True])
def test_same_codec_settings_share(latent):
    assert same_containers(_cachegen(), _cachegen(), 256, latent)
    assert same_containers(_cachegen(cachegen_config=_cg_config()), _cachegen("other/model", cachegen_config=_cg_config()),
                           256, latent)
    assert same_containers(_lossless(), _lossless(), 256, latent)
    assert same_containers(_lossless(), _lossless(), 4096, latent)


def test_different_bins_coders_or_families_do_not_share():
    assert not same_containers(_cachegen(cachegen_config=_cg_config(vbins=16)),
                               _cachegen(cachegen_config=_cg_config(vbins=10)), 256, False)
    assert not same_containers(_cachegen(cachegen_config=_cg_config(L=4)), _cachegen(cachegen_config=_cg_config(L=8)),
                               256, False)
    assert not same_containers(_cachegen(), _cachegen(cachegen_config=_cg_config()), 256, False)
    assert not same_containers(_cachegen(), _cachegen(coder="rans"), 256, False)
    assert not same_containers(_cachegen(), _cachegen(coder="ac"), 256, False)
    assert not same_containers(_cachegen(), _lossless(), 256, False)
    assert not same_containers(_lossless(), _cachegen(), 256, False)
    assert not same_containers(None, _lossless(), 256, False)           # a raw local tier
    assert not same_containers(_cachegen(), None, 256, False)


def test_chunk_sizes_a_codec_refuses_do_not_share():
    assert not same_containers(_lossless(), _lossless(), 8192, False)
    assert not same_containers(_cachegen(coder="rans"), _cachegen(coder="rans"), 256, True)    # no latent container
    assert not same_containers(_cachegen(cachegen_config=_cg_config()), _cachegen(cachegen_config=_cg_config()), 512,
                               False)
    # two table codecs at 512 tokens both write version 2: the same containers, which the layer-wise encode does not write
    assert same_containers(_cachegen(), _cachegen(), 512, False)
    assert not layerwise_encodes(_cachegen(), 512, False)


def test_layerwise_encodes():
    assert layerwise_encodes(_cachegen(), 256, False) and layerwise_encodes(_cachegen(), 256, True)
    assert not layerwise_encodes(_cachegen(coder="rans"), 256, False)
    assert not layerwise_encodes(_cachegen(coder="ac"), 256, False)
    assert layerwise_encodes(_lossless(), 4096, False) and not layerwise_encodes(_lossless(), 4097, False)


# ---------------------------------------------------------------------------------------------- hybrid's choice
class _Part:
    def __init__(self, name):
        self.name, self.calls, self.abandoned = name, [], False

    def encode_layer(self, layer, stream, ready=None):
        self.calls.append((layer, stream, ready))

    def abandon(self):
        self.abandoned = True


class _Tier:
    def __init__(self, codec=None, handle=True, striped=True, puts=True, begins=True):
        self.codec = codec
        self.serializer = SimpleNamespace(codec=codec)
        self.puts = puts
        self._is_striped = striped
        self.begun = []
        self.handle = handle
        if begins:
            self.begin_layerwise_store = self._begin

    def _striped(self):
        return self._is_striped

    def _begin(self, view, tok_begin, chunk_size):
        h = _Part(len(self.begun)) if self.handle else None
        self.begun.append(h)
        return h


def _hybrid(local, remote):
    h = object.__new__(LMCHybridBackend)
    h.local_store, h.remote_store = local, remote
    h._join = SimpleNamespace(device="dev")
    return h


VIEW = SimpleNamespace(latent=False, device="dev")


def test_identical_containers_share_one_encode():
    local, remote = _Tier(_cachegen()), _Tier(_cachegen())
    enc = _hybrid(local, remote).begin_layerwise_store(VIEW, 0, 256)
    assert enc is local.begun[0] and remote.begun == []


@pytest.mark.parametrize("pair", ["raw_local", "cachegen_lossless", "bins", "not_striped_match"])
def test_different_containers_fan_out(pair):
    local, remote = {"raw_local": (_Tier(None), _Tier(_lossless())),
                     "cachegen_lossless": (_Tier(_cachegen()), _Tier(_lossless())),
                     "bins": (_Tier(_cachegen(cachegen_config=_cg_config(vbins=16))),
                              _Tier(_cachegen(cachegen_config=_cg_config(vbins=10)))),
                     "not_striped_match": (_Tier(_lossless()), _Tier(_lossless(), striped=False))}[pair]
    enc = _hybrid(local, remote).begin_layerwise_store(VIEW, 0, 256)
    assert isinstance(enc, FanOutEncode) and enc.parts == [local.begun[0], remote.begun[0]]
    ready = object()
    enc.encode_layer(2, "caller", ready=ready)
    assert enc.parts[0].calls == enc.parts[1].calls == [(2, "caller", ready)]    # one event for both parts
    enc.abandon()
    assert all(p.abandoned for p in enc.parts)


@pytest.mark.parametrize("which", ["local", "remote", "remote_has_none"])
def test_either_part_refusing_gives_none(which):
    local = _Tier(None, handle=which != "local")
    remote = _Tier(_lossless(), handle=which != "remote", begins=which != "remote_has_none")
    assert _hybrid(local, remote).begin_layerwise_store(VIEW, 0, 256) is None
    assert all(h.abandoned for h in local.begun if h is not None)       # a local part already begun is dropped


# ---------------------------------------------------------------------------------------------- shared slots
def _pool():
    p = object.__new__(SegmentPool)
    p.keep, p._free, p._lock = 2, [], threading.Lock()
    return p


def test_segment_slot_returns_after_the_last_sink():
    pool = _pool()
    slot = SimpleNamespace(refs=1, ticket="t", close=lambda: None)
    pool.hold(slot)
    pool.release(slot)
    assert pool._free == [] and slot.ticket == "t"           # the other sink still lands it
    pool.release(slot)
    assert pool._free == [slot] and slot.ticket is None


def test_wave_slot_returns_after_the_last_sink():
    ring = object.__new__(EncodeRing)
    ring._free, ring._lock = queue.Queue(), threading.Lock()
    slot = SimpleNamespace(refs=1, ticket="t")
    ring.hold(slot)
    ring.release(slot)
    assert ring._free.empty()
    ring.release(slot)
    assert ring._free.get_nowait() is slot and slot.ticket is None


class _Sinking:
    """a tier whose put_kv_chunks(encoded=) does what its worker does: the sink, then release of the slot"""

    def __init__(self, log, name, puts=True, fail=False):
        self.log, self.name, self.puts, self.fail = log, name, puts, fail

    def put_kv_chunks(self, keys, view, tok_begin, chunk_size, blocking=True, encoded=None):
        if self.fail:
            raise RuntimeError("landing failed before the submit")
        self.log.append((self.name, encoded.slot.refs))
        encoded.pool.release(encoded.slot)
        return len(keys)


@pytest.mark.parametrize("case", ["both", "remote_skips", "local_fails"])
def test_hybrid_shared_put_releases_after_both(case):
    log = []
    pool = _pool()
    slot = SimpleNamespace(refs=1, ticket="t", close=lambda: None)
    enc = SimpleNamespace(pool=pool, slot=slot)
    local = _Sinking(log, "local", fail=case == "local_fails")
    remote = _Sinking(log, "remote", puts=case != "remote_skips")
    hyb = _hybrid(local, remote)
    if case == "local_fails":
        with pytest.raises(RuntimeError):
            hyb.put_kv_chunks(["k0", "k1"], None, 0, 256, encoded=enc)
        assert slot.refs == 1 and pool._free == []    # the local reference is the failed landing's own
        return
    assert hyb.put_kv_chunks(["k0", "k1"], None, 0, 256, encoded=enc) == 2
    if case == "both":
        assert log == [("local", 2), ("remote", 1)]
    else:
        assert log == [("local", 1)]
    assert pool._free == [slot] and slot.refs == 0
