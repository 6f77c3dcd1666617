"""LMCHybridBackend -- local tier in front of a remote one (lmcache/storage_backend/hybrid_backend.py): writes go to
both, reads are served locally when possible and fall through to the remote tier (whose chunks are then kept locally).
The reference prefetches the whole remote store into the local tier at start-up (hybrid_backend.py:26-62: list() + one
get/put per key -- a full deserialise of everything the server holds); here the local tier fills on demand.

Both tiers keep their engine fast paths: a store hands the caller's KV view to each tier once -- or, when both keep the
same containers (pipeline.same_containers), encodes it once and lands every container in both -- and a retrieve asks
the local tier for the longest prefix it holds and the remote tier for the rest, all decoded / copied straight into the
one destination blob."""
from typing import Iterable, List, Optional, Tuple

import torch

from lmcache_b200 import _native as N
from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
from lmcache_b200.storage_backend.abstract_backend import LMCBackendInterface
from lmcache_b200.utils import CacheEngineKey


class LMCHybridBackend(LMCBackendInterface):

    def __init__(self, config: LMCacheEngineConfig, metadata: LMCacheEngineMetadata):
        super().__init__()
        from lmcache_b200.storage_backend import CreateStorageBackend
        # a capacity bounds the local tier (one of the CacheGen tiers); chunks it evicts are still served by the remote one.
        # A device level belongs to the local tier as well.  Both tiers code with the engine's bin layout.
        local_cfg = LMCacheEngineConfig(config.chunk_size, config.local_device, None, None, False, config.save_decode_cache,
                                        config.local_serde, config.local_capacity_bytes, config.device_cache_bytes,
                                        cachegen_config=config.cachegen_config)
        remote_cfg = LMCacheEngineConfig(config.chunk_size, None, config.remote_url, config.remote_serde,
                                         config.pipelined_backend, config.save_decode_cache, None,
                                         cachegen_config=config.cachegen_config)
        # an MLA engine's remote tier takes stores from rank 0 only (LMCRemoteBackend); the local tier, which is this
        # process's own, takes every rank's
        self.local_store = CreateStorageBackend(local_cfg, metadata)
        self.remote_store = CreateStorageBackend(remote_cfg, metadata)
        self._join: Optional[torch.cuda.Stream] = None     # where a FanOutEncode joins its parts' finish events

    def contains(self, key: CacheEngineKey) -> bool:
        return self.local_store.contains(key) or self.remote_store.contains(key)

    def put(self, key: CacheEngineKey, kv_chunk: torch.Tensor, blocking: bool = True) -> None:
        self.local_store.put(key, kv_chunk, blocking=True)
        self.remote_store.put(key, kv_chunk, blocking)

    def get(self, key: CacheEngineKey) -> Optional[torch.Tensor]:
        val = self.local_store.get(key)
        if val is None:
            val = self.remote_store.get(key)
            if val is not None:
                self.local_store.put(key, val, blocking=True)
        return val

    def batched_put(self, keys_and_chunks: Iterable[Tuple[CacheEngineKey, torch.Tensor]], blocking=True) -> int:
        n = 0
        for key, chunk in keys_and_chunks:
            self.put(key, chunk, blocking=blocking)
            n += 1
        return n

    # ------------------------------------------------------------------ engine fast paths
    def supports_kv_view(self) -> bool:
        f, g = getattr(self.local_store, "supports_kv_view", None), getattr(self.remote_store, "supports_kv_view", None)
        return bool(f and f() and g and g())

    def supports_split_view(self) -> bool:
        """both parts take a split paged view as it is; otherwise the engine stages it once for both"""
        f, g = getattr(self.local_store, "supports_split_view", None), getattr(self.remote_store, "supports_split_view", None)
        return bool(f and f() and g and g())

    def _shares_containers(self, chunk_size: int, view) -> bool:
        """Do both parts keep the same containers for chunks of `chunk_size` of `view`'s kind (pipeline.same_containers
        of the local tier's codec and the remote serializer's), so that one encode serves both?  The remote part must be on its
        striped path: that path lands containers from a device slot."""
        from lmcache_b200.pipeline import same_containers
        remote = self.remote_store
        striped = getattr(remote, "_striped", None)
        if striped is None or not striped():
            return False
        return same_containers(getattr(self.local_store, "codec", None), getattr(remote.serializer, "codec", None),
                               chunk_size, view.latent)

    def put_kv_chunks(self, keys: List[CacheEngineKey], view, tok_begin: int, chunk_size: int, blocking: bool = True,
                      encoded=None) -> int:
        """The local tier's put (blocking), then the remote tier's.  When both keep the same containers, the chunks are
        encoded once: on the caller's stream, wave by wave, each wave landed by both tiers' workers from the same device
        slot (pipeline.SharedWaves); or, with `encoded`, one layer-wise encode whose slot both land.  `encoded` of two
        tiers that do not (a pipeline.FanOutEncode) gives each tier its own part."""
        from lmcache_b200.pipeline import FanOutEncode, SharedWaves
        local, remote = self.local_store, self.remote_store
        if isinstance(encoded, FanOutEncode):
            try:
                n = local.put_kv_chunks(keys, None, tok_begin, chunk_size, blocking=True, encoded=encoded.parts[0])
            except BaseException:
                encoded.parts[1].abandon()
                raise
            remote.put_kv_chunks(keys, None, tok_begin, chunk_size, blocking=blocking, encoded=encoded.parts[1])
            return n
        if encoded is not None:
            # one slot, two sinks: the remote part's reference is taken before the local worker can release the slot
            if not remote.puts:
                return local.put_kv_chunks(keys, None, tok_begin, chunk_size, blocking=True, encoded=encoded)
            encoded.pool.hold(encoded.slot)
            try:
                n = local.put_kv_chunks(keys, None, tok_begin, chunk_size, blocking=True, encoded=encoded)
            except BaseException:
                encoded.pool.release(encoded.slot)
                raise
            remote.put_kv_chunks(keys, None, tok_begin, chunk_size, blocking=blocking, encoded=encoded)
            return n
        if not (getattr(remote, "puts", False) and self._shares_containers(chunk_size, view)):
            n = local.put_kv_chunks(keys, view, tok_begin, chunk_size, blocking=True)
            remote.put_kv_chunks(keys, view, tok_begin, chunk_size, blocking=blocking)
            return n
        shared = SharedWaves(remote._pipeline(), keys)
        n = local.put_kv_chunks(keys, view, tok_begin, chunk_size, blocking=True, shared=shared)
        if blocking:
            shared.job.wait()
            remote.flush()
        return n

    @property
    def layerwise_store_blocking(self) -> bool:
        """Yes: finish() returns once the server holds the containers (the remote part's guarantee), after the local
        part has landed them."""
        return True

    def begin_layerwise_store(self, view, tok_begin: int, chunk_size: int, budget: Optional[int] = None):
        """A layer-wise store into both parts, or None when either part cannot take one (a torch-serde remote tier, a
        chunk size over a part's limit): the engine then stores both at finish().  When both parts keep the same
        containers it is one pipeline.LayerwiseEncode on the local tier's pool, whose slot put_kv_chunks lands into
        both; otherwise a pipeline.FanOutEncode of the two parts' own handles.  `budget` goes to both parts."""
        from lmcache_b200.pipeline import FanOutEncode
        begins = [getattr(s, "begin_layerwise_store", None) for s in (self.local_store, self.remote_store)]
        if None in begins:
            return None
        kw = {} if budget is None else {"budget": budget}
        if self._shares_containers(chunk_size, view):
            return begins[0](view, tok_begin, chunk_size, **kw)
        local = begins[0](view, tok_begin, chunk_size, **kw)
        if local is None:
            return None
        try:
            remote = begins[1](view, tok_begin, chunk_size, **kw)
        except BaseException:
            local.abandon()
            raise
        if remote is None:
            local.abandon()
            return None
        if self._join is None or self._join.device != view.device:
            self._join = torch.cuda.Stream(device=view.device)
        return FanOutEncode([local, remote], self._join)

    def get_kv_into(self, keys: List[CacheEngineKey], dst, dst_tok0: int, chunk_size: int) -> int:
        n = self.local_store.get_kv_into(keys, dst, dst_tok0, chunk_size)
        if n < len(keys):
            n += self.remote_store.get_kv_into(keys[n:], dst, dst_tok0 + n * chunk_size, chunk_size)
        return n

    def get_kv_shards_into(self, groups, dst, dst_tok0: int, chunk_size: int, stats=None) -> int:
        """Chunks of another tensor-parallel layout come from the remote tier alone: the local tier holds this process's
        keys only, and the chunks served are not kept in it (they are another layout's quantisation, not this one's)."""
        f = getattr(self.remote_store, "get_kv_shards_into", None)
        return f(groups, dst, dst_tok0, chunk_size, stats) if f is not None else 0

    @property
    def layerwise_max_tokens(self) -> int:
        """the smaller of the two tiers' (a tier without a layer-major path counts with one group of 256 tokens)"""
        return min(getattr(s, "layerwise_max_tokens", N.GROUP_TOKENS) for s in (self.local_store, self.remote_store))

    def supports_layerwise_get(self) -> bool:
        return any(s.supports_layerwise_get() for s in (self.local_store, self.remote_store))

    def get_kv_layerwise(self, keys, dst, dst_tok0: int, chunk_size: int):
        """get_kv_into with each part layer-major where its tier can: the local tier's prefix, then the remote tier's
        rest.  A part whose tier cannot is decoded chunk-major and counts as ready for every layer.  Returns one handle
        whose ready(l) comes after both parts' layer l (pipeline.join_uploads)."""
        from lmcache_b200.pipeline import join_uploads
        parts: list = []
        n = self._get_part(self.local_store, keys, dst, dst_tok0, chunk_size, parts)
        if n < len(keys):
            self._get_part(self.remote_store, keys[n:], dst, dst_tok0 + n * chunk_size, chunk_size, parts)
        return join_uploads(parts, dst.L)

    def get_kv_layerwise_runs(self, runs, dst, chunk_size: int, rotation=None):
        """get_kv_layerwise_runs as get_kv_into would serve each run: its keys from the local tier, then from the remote
        tier where the local one missed; then (when the keys missed) its fallback keys the same way.  Each part is one
        multi-run get of one tier (a tier that cannot go layer-major decodes its part chunk-major), each chunk is in
        exactly one part, and each part turns only the rows it wrote (`rotation`).  Returns ([(key hits, fallback
        hits)] per run, one handle whose ready(l) comes after every part's layer l)."""
        from lmcache_b200.pipeline import join_uploads
        parts: list = []
        own = self._runs_parts([(keys, tok0) for keys, _, tok0 in runs], dst, chunk_size, rotation, parts)
        fb = [(f[h:] if f is not None and h < len(f) else [], tok0 + h * chunk_size)
              for (_, f, tok0), h in zip(runs, own)]
        more = self._runs_parts(fb, dst, chunk_size, rotation, parts)
        return list(zip(own, more)), join_uploads(parts, dst.L)

    def _runs_parts(self, runs, dst, chunk_size: int, rotation, parts: list) -> list:
        """runs of (keys, destination token) from the local tier, then their rest (rest_runs) from the remote tier;
        returns the hits per run"""
        from lmcache_b200.pipeline import rest_runs
        hits = [0] * len(runs)
        for store in (self.local_store, self.remote_store):
            if any(len(keys) for keys, _ in runs):
                n = self._runs_part(store, runs, dst, chunk_size, rotation, parts)
                hits = [h + m for h, m in zip(hits, n)]
                runs = rest_runs(runs, n, chunk_size)
        return hits

    @staticmethod
    def _runs_part(store, runs, dst, chunk_size: int, rotation, parts: list) -> list:
        from lmcache_b200.pipeline import LayerwiseUpload
        f = getattr(store, "get_kv_layerwise_runs", None)
        if f is not None and store.supports_layerwise_get() and \
                chunk_size <= getattr(store, "layerwise_max_tokens", N.GROUP_TOKENS):
            hits, up = f([(keys, None, tok0) for keys, tok0 in runs], dst, chunk_size, rotation)
            parts.append(up)
            return [h for h, _ in hits]
        # chunk-major: every run through get_kv_into, then the rows written turned for every layer at once
        n = [store.get_kv_into(keys, dst, tok0, chunk_size) if len(keys) else 0 for keys, tok0 in runs]
        stream = torch.cuda.current_stream()
        rot = None if rotation is None else rotation.prepare(
            [(r, tok0 + j * chunk_size, min(chunk_size, dst.ntokens - tok0 - j * chunk_size))
             for r, ((_, tok0), m) in enumerate(zip(runs, n)) for j in range(m)], dst.device)
        if rot is not None:
            rot.shift_layers(dst, 0, dst.L, stream)
        ev = torch.cuda.Event()
        ev.record(stream)
        parts.append(LayerwiseUpload.completed(sum(n), dst.L, ev))
        return n

    @staticmethod
    def _get_part(store, keys, dst, dst_tok0: int, chunk_size: int, parts: list) -> int:
        from lmcache_b200.pipeline import LayerwiseUpload
        if store.supports_layerwise_get() and chunk_size <= getattr(store, "layerwise_max_tokens", N.GROUP_TOKENS):
            parts.append(store.get_kv_layerwise(keys, dst, dst_tok0, chunk_size))
        else:
            n = store.get_kv_into(keys, dst, dst_tok0, chunk_size)
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream())
            parts.append(LayerwiseUpload.completed(n, dst.L, ev))
        return parts[-1].n

    def touch(self, keys) -> None:
        f = getattr(self.local_store, "touch", None)
        if f is not None:
            f(keys)

    def peek_geometry(self, key: CacheEngineKey, fmt: str = "vllm"):
        for store in (self.local_store, self.remote_store):
            f = getattr(store, "peek_geometry", None)
            g = f(key, fmt) if f is not None else None
            if g is not None:
                return g
        return None

    def out_dtype(self):
        f = getattr(self.remote_store, "out_dtype", None) or \
            getattr(getattr(self.remote_store, "deserializer", None), "out_dtype", None)
        return f() if f is not None else None

    def close(self):
        self.local_store.close()
        self.remote_store.close()
