"""LMCRemoteBackend -- serde + connector (lmcache/storage_backend/remote_backend.py:24-180) and the pipelined
variant (:183-275).  This is the caller of the serde plugins: put = to_bytes -> connection.set,
get = connection.get -> from_bytes.  The generic per-chunk path keeps the reference's single put worker thread.

Engine fast paths (CacheGen serde + a connector with get_into), both pipelined and striped over several connections:
  put   waves of chunks are encoded on the caller's stream (enqueue only -- this is also the snapshot a non-blocking
        store needs, the caller may reuse its KV buffers in stream order); a worker moves each finished wave's containers
        to a page-locked slab and sends them over k connections in parallel;
  get   the containers of all requested chunks are fetched by k connections into the slab while the main thread uploads
        and decodes the waves that are already complete (network || H2D || decode: what remote_backend.py:183-275 does
        with a network thread and a deserialize thread, here also on the engine's one-blob path).
LMCACHE_B200_REMOTE_CONNS sets k (default 4; one TCP stream is slower than the GPU side)."""
import os
import queue
import threading
from concurrent.futures import ThreadPoolExecutor
from typing import Iterable, Iterator, List, Optional, Set, Tuple, Union

import torch

from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
from lmcache_b200.logging import init_logger
from lmcache_b200.pipeline import DeferredFree
from lmcache_b200.storage_backend.abstract_backend import LMCBackendInterface
from lmcache_b200.storage_backend.connector import CreateConnector
from lmcache_b200.storage_backend.serde import CreateSerde
from lmcache_b200.utils import CacheEngineKey, _lmcache_nvtx_annotate

logger = init_logger(__name__)


class RemoteBackendEndSignal:
    pass


class LazyFlat:
    """The keys of groups of (key, window), k per group, in order; a group is read when one of its keys is reached."""

    def __init__(self, groups, k: int):
        self.groups, self.k = groups, k

    def __len__(self) -> int:
        return len(self.groups) * self.k

    def __getitem__(self, i: int):
        return self.groups[i // self.k][i % self.k][0]

    def __iter__(self):
        for g in self.groups:
            for key, _ in g:
                yield key


def _grouped(recs, k: int, sizes: List[int]):
    """recs (fetched container records) k at a time; the container bytes of each group yielded go to `sizes`.  Records
    of a group the consumer never received are freed when it stops."""
    buf: list = []
    try:
        for r in recs:
            buf.append(r)
            if len(buf) == k:
                out, buf = buf, []
                sizes.append(sum(x.nbytes for x in out if x is not None))
                yield out
    finally:
        for r in buf:
            if r is not None and r.blk is not None:
                r.blk.free()


class LMCRemoteBackend(LMCBackendInterface):

    def __init__(self, config: LMCacheEngineConfig, metadata: LMCacheEngineMetadata):
        super().__init__()
        self.existing_keys: Set[CacheEngineKey] = set()
        self.put_thread = None
        self.connection = None
        assert config.remote_url is not None, "Need to provide remote_url when using LMCRemoteBackend"
        assert config.remote_serde is not None, "Need to provide remote_serde when using LMCRemoteBackend"
        self.connection = CreateConnector(config.remote_url)
        self.serializer, self.deserializer = CreateSerde(config.remote_serde, config, metadata)
        # a latent KV (metadata.use_mla) is the same on every tensor-parallel rank and its keys are shared: rank 0
        # alone puts it to the shared tier, the other ranks only read
        self.latent = bool(getattr(metadata, "use_mla", False))
        self.puts = not (self.latent and metadata.worker_id != 0)
        self.dst_device = "cuda"
        self._device = torch.cuda.current_device() if torch.cuda.is_available() else None
        self.put_queue: "queue.Queue[Union[Tuple[CacheEngineKey, torch.Tensor], RemoteBackendEndSignal]]" = \
            queue.Queue()
        self.put_thread = threading.Thread(target=self.put_worker, args=(), daemon=True)
        self.put_thread.start()
        # fast-path machinery, built on first use
        self._url = config.remote_url
        self._nconn = max(1, int(os.environ.get("LMCACHE_B200_REMOTE_CONNS", "4")))
        self._pool: Optional[ThreadPoolExecutor] = None
        self._tls = threading.local()
        self._conns: List = []
        self._conns_lock = threading.Lock()
        self._slab = None
        self._pipe = None
        self._upload = None
        self._release = DeferredFree()   # fetched blocks that uploads may still read
        self._peek = None            # (key, HostContainer): the container peek_geometry fetched, reused by get_kv_into

    @_lmcache_nvtx_annotate
    def put_worker(self):
        if self._device is not None:
            torch.cuda.set_device(self._device)
        while True:
            item = self.put_queue.get()
            if isinstance(item, RemoteBackendEndSignal):
                self.put_queue.task_done()
                break
            try:
                if item[0] == "view":
                    _, keys, view, tok_begin, chunk_size = item
                    self._put_view_blocking(keys, view, tok_begin, chunk_size)
                else:
                    key, value = item
                    self.put_blocking(key, value)
            except Exception as e:   # a failed background put is a cache miss later, not a crash
                logger.error(f"background put failed: {e}")
            finally:
                self.put_queue.task_done()

    def _combine_key(self, key: CacheEngineKey) -> str:
        return key.to_string()

    def _split_key(self, key: str) -> CacheEngineKey:
        return CacheEngineKey.from_string(key)

    def list(self) -> List[CacheEngineKey]:
        keys = [self._split_key(k) for k in self.connection.list()]
        self.existing_keys.update(keys)
        return keys

    def contains(self, key: CacheEngineKey) -> bool:
        if key in self.existing_keys:
            return True
        flag = self.connection.exists(self._combine_key(key))
        if flag:
            self.existing_keys.add(key)
        return flag

    def put_blocking(self, key: CacheEngineKey, kv_chunk: torch.Tensor) -> None:
        bs = self.serializer.to_bytes(kv_chunk)
        self.connection.set(self._combine_key(key), bs)
        self.existing_keys.add(key)

    def put(self, key: CacheEngineKey, kv_chunk: torch.Tensor, blocking: bool = True) -> None:
        if not self.puts:
            return
        if blocking:
            self.put_blocking(key, kv_chunk)
        else:
            self.put_queue.put((key, kv_chunk))

    @_lmcache_nvtx_annotate
    def get(self, key: CacheEngineKey) -> Optional[torch.Tensor]:
        if not self.contains(key):
            return None
        bs = self.connection.get(self._combine_key(key))
        if bs is None or len(bs) == 0:
            return None
        return self.deserializer.from_bytes(bs).to(self.dst_device)

    # ------------------------------------------------------------------ engine fast paths (no per-chunk blobs)
    def supports_kv_view(self) -> bool:
        """True when the serde plugin can encode / decode straight from / into the engine's KV tensors."""
        return hasattr(self.serializer, "view_to_bytes_batch") and hasattr(self.deserializer, "decode_into")

    def _striped(self) -> bool:
        return hasattr(self.connection, "get_into") and hasattr(self.serializer, "codec") and \
            hasattr(self.deserializer, "container_bound")

    # k connections, one per pool thread (a connection serialises whole request / response exchanges)
    def _conn(self):
        c = getattr(self._tls, "conn", None)
        if c is None:
            c = CreateConnector(self._url)
            self._tls.conn = c
            with self._conns_lock:
                self._conns.append(c)
        return c

    def _executor(self) -> ThreadPoolExecutor:
        if self._pool is None:
            self._pool = ThreadPoolExecutor(max_workers=self._nconn, thread_name_prefix="b200kv-net")
        return self._pool

    def _host_slab(self):
        if self._slab is None:
            from lmcache_b200.slab import PinnedSlab
            self._slab = PinnedSlab()
        return self._slab

    # ---- put
    def _sink(self, slot, batch, c0, keys) -> None:
        """store worker: one wave's containers -> page-locked slab (land() raises on a nonzero encoder status: nothing
        corrupt leaves the host), then k-way send"""
        from lmcache_b200.pipeline import land
        blocks = [rec.blk for rec in land(self._host_slab(), slot, batch, codec=self.serializer.codec)]
        try:
            def send(key, blk):
                self._conn().set(self._combine_key(key), blk.view())
                return key
            for key in self._executor().map(send, keys, blocks):
                self.existing_keys.add(key)
        finally:
            for blk in blocks:
                blk.free()

    def _put_view_blocking(self, keys, view, tok_begin: int, chunk_size: int) -> None:
        n_tokens = view.ntokens - tok_begin
        if hasattr(self.serializer, "view_to_pinned_batch"):
            # containers are sent from the page-locked slab the device->host copies landed in
            with self.serializer.view_to_pinned_batch(view, chunk_size, tok_begin, n_tokens) as blobs:
                assert len(blobs) == len(keys)
                for key, mv in zip(keys, blobs):
                    self.connection.set(self._combine_key(key), mv)
                    self.existing_keys.add(key)
            return
        blobs = self.serializer.view_to_bytes_batch(view, chunk_size, tok_begin, n_tokens)
        assert len(blobs) == len(keys)
        for key, bs in zip(keys, blobs):
            self.connection.set(self._combine_key(key), bs)
            self.existing_keys.add(key)

    def put_kv_chunks(self, keys: List[CacheEngineKey], view, tok_begin: int, chunk_size: int,
                      blocking: bool = True) -> int:
        """Store tokens [tok_begin, T) of `view` as len(keys) chunks.  Striped path: every wave is encoded on the caller's
        stream before this returns (so a non-blocking store has consumed the caller's KV in stream order -- paged caches
        included -- like the reference's materialised chunk list, cache_engine.py:274-275); D2H and the sends happen on
        the pipeline's worker.  Other serdes: one batched encode, then one set() per chunk.  A latent KV's rank other
        than 0 stores nothing (returns 0)."""
        if not self.puts:
            return 0
        if self._striped():
            if self._pipe is None:
                from lmcache_b200.pipeline import EncodePipeline
                self._pipe = EncodePipeline(self.serializer.codec, self._sink, name="b200kv-remote-store")
            job = self._pipe.submit(view, tok_begin, chunk_size, keys)      # keys may be lazy: a wave's are read when it is queued
            if blocking:
                job.wait()
                self.flush()
            return len(keys)
        if blocking or getattr(view.desc, "slot_map", None):
            # a paged view aliases vLLM's live cache: never queue it for a later encode
            self._put_view_blocking(keys, view, tok_begin, chunk_size)
        else:
            self.put_queue.put(("view", list(keys), view, tok_begin, chunk_size))
        return len(keys)

    def flush(self) -> None:
        """PUT carries no acknowledgement (lmcache/server/__main__.py:46-48), but a connection is served in order: one
        EXIST round trip per connection means the server has processed every PUT sent before it.  A blocking store ends
        with this, so another engine's retrieve that starts afterwards finds the chunks."""
        with self._conns_lock:
            conns = list(self._conns)
        for c in conns:
            try:
                c.exists("b200kv-flush")
            except Exception:       # noqa: BLE001
                pass

    def drain(self) -> None:
        """Wait until every queued / in-flight put of this backend has reached the server."""
        self.put_queue.join()
        if self._pipe is not None and self._pipe.ring is not None:
            self._pipe.ring.drain()
        self.flush()

    # ---- get
    def _fetch(self, key: CacheEngineKey, bound: int, conn=None):
        """one GET into a fresh slab block (on a pool thread: over that thread's connection) -> its HostContainer, or
        None on a miss or a damaged / foreign container"""
        from lmcache_b200.pipeline import read_container
        blk = self._host_slab().alloc(bound)
        try:
            n = (conn or self._conn()).get_into(self._combine_key(key), blk.host_ptr, bound)
        except Exception:      # noqa: BLE001 -- a broken connection is a miss
            n = None
        if not n:
            blk.free()
            return None
        blk.shrink(int(n))                      # the bound covers the largest container version; a v3 one is a tenth of it
        return read_container(self.deserializer.codec, blk, int(n), self.latent)

    def peek_geometry(self, key: CacheEngineKey, fmt: str = "vllm"):
        """(L, H, D, output dtype) from the header of the first chunk's container -- the stored dtype when the serde
        decodes into it (out_dtype() None: the lossless serde).  The fetched container is kept for the get_kv_into call
        that follows, so a retrieve-only replica neither decodes nor fetches chunk 0 twice."""
        if not (self._striped() and hasattr(self.deserializer, "out_dtype")):
            return None
        rec = self._fetch(key, 256 << 20, self.connection)       # the geometry is what we are asking for: be generous
        if rec is None:
            return None
        if self._peek is not None:
            self._peek[1].blk.free()
        self._peek = (key, rec)
        od = self.deserializer.out_dtype()
        if od is None:
            from lmcache_b200.codec import dtype_of_code
            od = dtype_of_code(rec.max_dtype)
        return (rec.L, rec.H, rec.D, od)

    def get_kv_into(self, keys: List[CacheEngineKey], dst, dst_tok0: int, chunk_size: int) -> int:
        """Fetch consecutive chunks until the first miss and decode them straight into `dst` (chunk i lands at token
        dst_tok0 + i * chunk_size).  Returns the number of chunks."""
        if self._striped() and hasattr(self.deserializer, "codec"):
            return self._get_striped(keys, dst, dst_tok0, chunk_size)        # keys may be lazy: read as the fetch window moves
        blobs = []
        for key in keys:
            if not self.contains(key):
                break
            bs = self.connection.get(self._combine_key(key))
            if bs is None or len(bs) == 0:
                break
            blobs.append(bs)
        if blobs:
            self.deserializer.decode_into(blobs, dst, [dst_tok0 + i * chunk_size for i in range(len(blobs))])
        return len(blobs)

    def _get_striped(self, keys, dst, dst_tok0: int, chunk_size: int) -> int:
        return self._get_striped_groups(keys, None, dst, dst_tok0, chunk_size)

    def get_kv_shards_into(self, groups, dst, dst_tok0: int, chunk_size: int, stats: Optional[dict] = None) -> int:
        """Serve chunks that another tensor-parallel layout stored: groups[i] lists (key, HeadWindow) for chunk i -- the
        source containers and the window of each that makes up this rank's heads (the same windows for every chunk).
        They are fetched over the striped connections and decoded into `dst` (chunk i at token dst_tok0 + i *
        chunk_size) up to the first chunk that is incomplete.  Returns the number of whole chunks served; with `stats`,
        stats["bytes"] grows by the container bytes of those chunks.  CacheGen and lossless serdes; nothing is kept."""
        if not (len(groups) and self._striped()):
            return 0
        return self._get_striped_groups(groups, [w for _, w in groups[0]], dst, dst_tok0, chunk_size, stats)

    def _get_striped_groups(self, items, windows, dst, dst_tok0: int, chunk_size: int, stats=None) -> int:
        """items: keys (windows None), or groups of (key, window) (see get_kv_shards_into)"""
        import contextlib
        from concurrent.futures import Future

        from lmcache_b200.pipeline import UploadRing, fetched_in_order, upload_decode, wave_chunks_default
        self._release.sweep()
        H = dst.H if windows is None else windows[0].src_H
        bound = (self.deserializer.container_bound(dst.L, H, dst.D, chunk_size, dst.latent) + 255) & ~255
        ex = self._executor()
        keys = items if windows is None else LazyFlat(items, len(windows))
        peek, self._peek = self._peek, None
        if peek is not None and not (len(keys) and peek[0] == keys[0]):
            peek[1].blk.free()
            peek = None

        def gets():
            for i, key in enumerate(keys):
                if i == 0 and peek is not None:
                    f = Future()
                    f.set_result(peek[1])                               # already in host memory (peek_geometry)
                    yield f
                else:
                    yield ex.submit(self._fetch, key, bound)
        if self._upload is None or self._upload.device != dst.device:
            self._upload = UploadRing(dst.device)
        window = max(2 * self._nconn, 2 * wave_chunks_default())       # fetches in flight ahead of the consumer
        with contextlib.closing(fetched_in_order(gets(), window)) as recs:
            if windows is None:
                return upload_decode(self.deserializer.codec, self._upload, recs, dst, dst_tok0, chunk_size,
                                     self._release)
            sizes: List[int] = []
            with contextlib.closing(_grouped(recs, len(windows), sizes)) as grecs:
                n = upload_decode(self.deserializer.codec, self._upload, grecs, dst, dst_tok0, chunk_size,
                                  self._release, windows=windows)
            if stats is not None:
                stats["bytes"] = stats.get("bytes", 0) + sum(sizes[:n])
            return n

    def close(self):
        if self.put_thread is not None and self.put_thread.is_alive():
            self.put_queue.put(RemoteBackendEndSignal())
            self.put_thread.join()
        if getattr(self, "_pipe", None) is not None:
            self._pipe.close()
            self._pipe = None
        if getattr(self, "_pool", None) is not None:
            self._pool.shutdown(wait=True)
            self._pool = None
        if getattr(self, "_release", None) is not None:
            self._release.drain()
        if getattr(self, "_peek", None) is not None:
            self._peek[1].blk.free()
            self._peek = None
        for c in getattr(self, "_conns", []):
            try:
                c.close()
            except Exception:       # noqa: BLE001
                pass
        self._conns = []
        if getattr(self, "_slab", None) is not None:
            self._slab.close()
            self._slab = None
        if self.connection is not None:
            self.connection.close()
            self.connection = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class LMCPipelinedRemoteBackend(LMCRemoteBackend):
    """batched_get with the network fetch of chunk i+1 overlapped with the decode of chunk i
    (remote_backend.py:183-275: network thread + deserialize thread)."""

    def __init__(self, config: LMCacheEngineConfig, metadata: LMCacheEngineMetadata):
        super().__init__(config, metadata)

    @_lmcache_nvtx_annotate
    def batched_get(self, keys: Iterator[CacheEngineKey]) -> Iterable[Optional[torch.Tensor]]:
        keys = list(keys)
        fetched: "queue.Queue" = queue.Queue()

        def network_worker():
            for key in keys:
                data = None
                if self.contains(key):
                    data = self.connection.get(self._combine_key(key))
                fetched.put(data)
                if data is None:
                    break

        th = threading.Thread(target=network_worker, daemon=True)
        th.start()
        results: List[Optional[torch.Tensor]] = []
        for _ in keys:
            data = fetched.get()
            if data is None or len(data) == 0:
                results.append(None)
                break
            results.append(self.deserializer.from_bytes(data).to(self.dst_device))
        th.join()
        return results
