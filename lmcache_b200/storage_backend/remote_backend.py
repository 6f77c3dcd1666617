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
  get, layer-major (get_kv_layerwise, on a server with ranged reads): every matched container is OPENed -- its fixed
        sections arrive with the OPEN -- and then k network threads READ every chunk's layer l before any chunk's layer
        l + 1, while the uploader copies and decodes each layer as soon as its bytes are in host memory.
LMCACHE_B200_REMOTE_CONNS sets k (default 4; one TCP stream is slower than the GPU side).  The layer-major get is opt-in,
LMCACHE_B200_REMOTE_LAYERWISE=1: over loopback it brings layer 0 sooner but the last layer later than the chunk-major get
(DESIGN.md section 4), so by default retrieve_layerwise on this tier stays retrieve() plus one event for every layer."""
import collections
import os
import queue
import threading
import time
from concurrent.futures import Future, ThreadPoolExecutor
from typing import Callable, Iterable, Iterator, List, Optional, Set, Tuple, Union

import numpy as np
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


READ_BATCH_BYTES = 4 << 20      # a network thread merges the READs of consecutive layers (after layer 0) up to this


class RangedFetch:
    """The network side of a layer-major remote retrieve: for each of the k connections a pool thread sends, layer after
    layer, that connection's READs of pipeline.ranged_read_plan (small layers merged, see _batch), straight into the
    containers' blocks, and publishes how many layers it has completed.  wait(l) -- the uploader's host_ready -- returns once every connection has completed
    layer l, and raises once a READ has failed (a lost connection, or a READ the server refused) and every thread has
    stopped: no block is released while a thread may still write it.  finish() waits for the threads and CLOSEs the
    handles."""

    def __init__(self, conns, reads, handles: List[Optional[int]], ptrs: List[int], num_layers: int,
                 count: Callable[..., None]):
        self.conns, self.reads, self.handles, self.ptrs = conns, reads, handles, ptrs
        self.L = num_layers
        self.count = count                 # count(reads=, bytes=, read_s=, thread_s=): the backend's ranged_stats
        self._done = [0] * len(conns)
        self._left = len(conns)            # threads still running
        self._error: Optional[BaseException] = None
        self._cv = threading.Condition()
        self._futs: List[Future] = []

    def start(self, pool: ThreadPoolExecutor) -> None:
        self._futs = [pool.submit(self._run, c) for c in range(len(self.conns))]

    def _run(self, c: int) -> None:
        conn, handles = self.conns[c], self.handles
        ptrs = np.asarray(self.ptrs, dtype=np.int64)
        t_start = time.perf_counter()
        try:
            layer = 0
            while layer < self.L:
                batch, end = self._batch(c, layer)
                for e in batch:
                    if self._error is not None:
                        return
                    j, off, nb = e[:, 0], e[:, 1], e[:, 2]
                    t0 = time.perf_counter()
                    if not conn.read_ranges([handles[i] for i in j.tolist()], off, nb, ptrs[j] + off):
                        raise RuntimeError(f"lm:// READ of layers {layer}..{end - 1} refused by the server")
                    self.count(reads=1, bytes=int(nb.sum()), read_s=time.perf_counter() - t0)
                with self._cv:
                    self._done[c] = end
                    self._cv.notify_all()
                layer = end
        except BaseException as e:          # noqa: BLE001 -- the upload fails in wait()
            with self._cv:
                if self._error is None:
                    self._error = e
        finally:
            self.count(thread_s=time.perf_counter() - t_start)
            with self._cv:
                self._left -= 1
                self._cv.notify_all()

    def _batch(self, c: int, layer: int):
        """(READs, end): connection c's READs for layers [layer, end).  Layer 0 goes alone, so that it is ready as soon
        as possible; after it, layers whose READ is a single one are merged into one READ until it carries
        READ_BATCH_BYTES -- each exchange costs a round trip, which dominates when a layer's share is small."""
        from lmcache_b200.pipeline import READ_MAX_BYTES, READ_MAX_RANGES
        reads = self.reads[c]
        batch, end = list(reads[layer]), layer + 1
        if layer == 0 or len(batch) > 1:
            return batch, end
        nbytes = int(batch[0][:, 2].sum()) if batch else 0
        nrng = len(batch[0]) if batch else 0
        while end < self.L and len(reads[end]) <= 1 and nbytes < READ_BATCH_BYTES:
            b = int(reads[end][0][:, 2].sum()) if reads[end] else 0
            r = len(reads[end][0]) if reads[end] else 0
            if nbytes + b > READ_MAX_BYTES or nrng + r > READ_MAX_RANGES:
                break
            batch += reads[end]
            nbytes, nrng, end = nbytes + b, nrng + r, end + 1
        return ([np.concatenate(batch)] if len(batch) > 1 else batch), end

    def wait(self, layer: int) -> None:
        with self._cv:
            while min(self._done) <= layer:
                if self._error is not None and self._left == 0:
                    raise self._error
                self._cv.wait()

    def finish(self) -> None:
        for f in self._futs:
            f.result()
        by_conn = collections.defaultdict(list)
        for j, h in enumerate(self.handles):
            if h is not None:
                by_conn[j % len(self.conns)].append(h)
        for c, hs in by_conn.items():
            try:
                self.conns[c].close_handles(hs)
            except Exception:      # noqa: BLE001 -- a lost connection has dropped its handles
                pass


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
        self._segments = None            # pipeline.SegmentPool, made by the first layer-wise store
        self._upload = None
        self._release = DeferredFree()   # fetched blocks that uploads may still read
        self._peek = None            # (key, HostContainer): the container peek_geometry fetched, reused by get_kv_into
        # layer-major retrieve (get_kv_layerwise, opt-in): does the server have ranged reads (None: not asked yet), its
        # own k connections (chunk j's handle lives on connection j mod k), a pool for the OPENs of the match and one for
        # the READ threads (a retrieve's match does not wait behind an earlier retrieve's whole fetch), the uploader, and
        # what it fetched: ranged_stats counts OPENs, READs, bytes, and host seconds spent in them (open_s: in OPEN
        # exchanges on the pool threads; match_s: the calling thread's match; read_s: inside READ exchanges; thread_s:
        # the READ threads' whole lives)
        self._lw_enabled = os.environ.get("LMCACHE_B200_REMOTE_LAYERWISE", "0") == "1"
        self._ranges: Optional[bool] = None
        self._lw_conns: List = []
        self._lw_open_pool: Optional[ThreadPoolExecutor] = None
        self._lw_pool: Optional[ThreadPoolExecutor] = None
        self._layerwise = None
        self._stats_lock = threading.Lock()
        self.ranged_stats = {"retrieves": 0, "opens": 0, "reads": 0, "bytes": 0, "open_s": 0.0, "match_s": 0.0,
                             "read_s": 0.0, "thread_s": 0.0}

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

    def _pipeline(self):
        if self._pipe is None:
            from lmcache_b200.pipeline import EncodePipeline
            self._pipe = EncodePipeline(self.serializer.codec, self._sink, name="b200kv-remote-store")
        return self._pipe

    def put_kv_chunks(self, keys: List[CacheEngineKey], view, tok_begin: int, chunk_size: int,
                      blocking: bool = True, encoded=None) -> int:
        """Store tokens [tok_begin, T) of `view` as len(keys) chunks.  Striped path: every wave is encoded on the caller's
        stream before this returns (so a non-blocking store has consumed the caller's KV in stream order -- paged caches
        included -- like the reference's materialised chunk list, cache_engine.py:274-275); D2H and the sends happen on
        the pipeline's worker.  encoded: a finished pipeline.LayerwiseEncode of these chunks (begin_layerwise_store),
        whose containers are landed and sent instead of encoding `view`.  Other serdes: one batched encode, then one
        set() per chunk.  A latent KV's rank other than 0 stores nothing (returns 0)."""
        if not self.puts:
            return 0
        if self._striped():
            pipe = self._pipeline()
            if encoded is None:
                job = pipe.submit(view, tok_begin, chunk_size, keys)   # keys may be lazy: a wave's are read when it is queued
            else:
                job = pipe.submit_encoded(encoded, keys)
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

    # ---- layer-major get (ranged reads)
    @property
    def layerwise_max_tokens(self) -> int:
        """the largest chunk a layer-major retrieve takes: one group per container (256 tokens for CacheGen, 4096 for
        lossless); 0 for a serde without containers"""
        codec = getattr(self.deserializer, "codec", None)
        return getattr(codec, "layerwise_max_tokens", 0) if self._striped() else 0

    # ---- layer-wise store
    @property
    def layerwise_store_blocking(self) -> bool:
        """Yes: a layer-wise store's finish() returns only once the server holds every container (the pipeline's job,
        then flush()), as the blocking store() it replaced did, so that another engine's retrieve that starts after
        finish() finds the chunks."""
        return True

    def begin_layerwise_store(self, view, tok_begin: int, chunk_size: int, budget: Optional[int] = None):
        """A pipeline.LayerwiseEncode of tokens [tok_begin, T) of `view` (whose KV may not be written yet) on this tier's
        own SegmentPool; put_kv_chunks(..., encoded=it) lands and sends its containers.  None off the striped path (a
        serde without containers) and when the containers for `chunk_size` are not ones a layer-wise encode writes
        (pipeline.layerwise_encodes).  A latent KV's rank other than 0 gets a pipeline.NoEncode: it stores nothing, so
        nothing is encoded.  `budget`: the cap of its arena (default LMCACHE_B200_LAYERWISE_STORE_MB)."""
        from lmcache_b200.pipeline import LayerwiseEncode, NoEncode, layerwise_encodes, segment_pool_for
        if not (self._striped() and layerwise_encodes(self.serializer.codec, chunk_size, view.latent)):
            return None
        if not self.puts:
            return NoEncode()
        self._segments = segment_pool_for(self._segments, view.device)
        return LayerwiseEncode(self.serializer.codec, self._segments, view, tok_begin, chunk_size, budget)

    def _count(self, **kw) -> None:
        with self._stats_lock:
            for key, v in kw.items():
                self.ranged_stats[key] += v

    def supports_layerwise_get(self) -> bool:
        """Opted in (LMCACHE_B200_REMOTE_LAYERWISE=1), a container serde on the striped path, and a server that answers
        the ranged-read probe (asked once, on the first layer-wise retrieve: the reference server does not have ranged
        reads).  Without the opt-in nothing is sent."""
        if not (self._lw_enabled and self._striped() and hasattr(self.deserializer, "codec") and hasattr(self.connection, "supports_ranges")):
            return False
        if self._ranges is None:
            try:
                self._ranges = bool(self.connection.supports_ranges())
            except Exception:       # noqa: BLE001 -- a broken connection: chunk-major, as every get would be
                self._ranges = False
        return self._ranges

    def _lw_connections(self):
        if not self._lw_conns:
            self._lw_conns = [CreateConnector(self._url) for _ in range(self._nconn)]
            self._lw_open_pool = ThreadPoolExecutor(max_workers=self._nconn, thread_name_prefix="b200kv-open")
            self._lw_pool = ThreadPoolExecutor(max_workers=self._nconn, thread_name_prefix="b200kv-ranges")
        return self._lw_conns

    def _layerwise_uploader(self, device):
        from lmcache_b200.pipeline import LayerwiseUploader
        if self._layerwise is None or self._layerwise.device != device:
            if self._layerwise is not None:
                self._layerwise.close()
            self._layerwise = LayerwiseUploader(device)
        return self._layerwise

    def _open(self, conn, key: CacheEngineKey, prefix: int, bound: int):
        """OPEN one container into a fresh slab block of its size (on a pool thread): (HostContainer or None, handle or
        None, prefix bytes received).  A miss, a broken connection, a container larger than `bound` and a damaged or
        foreign one all give no record; a handle that was opened is still returned, for CLOSE."""
        from lmcache_b200.pipeline import read_container

        def alloc(size: int):
            if size > bound or size == 0:
                raise ValueError("not a container this retrieve can take")
            blk = self._host_slab().alloc(size)
            return blk.host_ptr, blk
        t0 = time.perf_counter()
        try:
            r = conn.open_into(self._combine_key(key), prefix, alloc)
        except Exception:           # noqa: BLE001 -- a miss, as in _fetch
            return None, None, 0
        finally:
            self._count(open_s=time.perf_counter() - t0)
        if r is None:
            return None, None, 0
        handle, size, got, blk = r
        return read_container(self.deserializer.codec, blk, size, self.latent, prefix=got), handle, got

    def get_kv_layerwise(self, keys, dst, dst_tok0: int, chunk_size: int):
        """get_kv_into in layer-major order, over ranged reads (supports_layerwise_get must be True).  On the calling
        thread: the keys are OPENed in chain order, pipelined over the k connections, each container's fixed sections
        landing in a slab block of its size, and matched as get_kv_into matches them (first miss, damaged or foreign
        container, change of dtype or coder); the handles past the match are closed.  Then the network threads READ
        layer 0 of every matched chunk, then layer 1, ... into those blocks, and the uploader copies and decodes layer l
        once its bytes are there (pipeline.upload_decode_layerwise with host_ready).  Returns the
        pipeline.LayerwiseUpload: n is known, ready(l) is the event after layer l's decode.  Every matched container
        sits in page-locked memory until its last copy.  A failed READ fails the upload: ready(l) raises for the layers
        not yet published (n was promised already), the blocks and handles are released."""
        return self.get_kv_layerwise_runs([(keys, None, dst_tok0)], dst, chunk_size)[1]

    def get_kv_layerwise_runs(self, runs, dst, chunk_size: int, rotation=None):
        """get_kv_layerwise of several runs in one ranged fetch and one upload: each run is (keys, fallback keys or None,
        destination token of its chunk 0).  A run's keys are OPENed and matched as get_kv_layerwise matches them, then
        (when it missed) its fallback keys from that index on; every container matches against the call's first one.
        `rotation` (rope.Rotation) turns the keys of the chunks written, layer by layer, after each layer's decode
        (pipeline.upload_decode_layerwise_runs).  Returns ([(key hits, fallback hits)] per run, LayerwiseUpload)."""
        from lmcache_b200.pipeline import (LayerwiseUpload, _continues_match, layer_copy_ranges, ranged_read_plan,
                                           upload_decode_layerwise_runs, wave_chunks_default)
        self._release.sweep()
        codec = self.deserializer.codec
        conns = self._lw_connections()
        k, pool = len(conns), self._lw_open_pool
        t_match = time.perf_counter()
        prefix = codec.plan_prefix(dst.L, dst.H, dst.D, chunk_size, dst.latent)     # the fixed sections of a full chunk
        bound = (self.deserializer.container_bound(dst.L, dst.H, dst.D, chunk_size, dst.latent) + 255) & ~255
        peek, self._peek = self._peek, None
        keys0 = runs[0][0] if runs else []
        if peek is not None and not (len(keys0) and peek[0] == keys0[0]):
            peek[1].blk.free()
            peek = None
        window = max(2 * k, 2 * wave_chunks_default())
        recs, handles, got, conn_of = [], [], [], []
        stale = collections.defaultdict(list)          # handles past the match, per connection

        def drop(c, rec, h):
            if rec is not None:
                rec.blk.free()
            if h is not None:
                stale[c].append(h)

        def match(keys, tok0: int, use_peek: bool) -> int:
            """OPEN `keys` in chain order over the k connections and append their records up to the first miss"""
            pending: "collections.deque" = collections.deque()
            keys_it = enumerate(keys)
            n0 = len(recs)

            def fill():
                while len(pending) < window:
                    try:
                        j, key = next(keys_it)
                    except StopIteration:
                        return
                    if j == 0 and use_peek and peek is not None:
                        f = Future()
                        f.set_result((peek[1], None, peek[1].nbytes))    # fetched whole by peek_geometry: used as it is
                    else:
                        f = pool.submit(self._open, conns[j % k], key, prefix, bound)
                    pending.append((j, f))
            try:
                fill()
                while pending:
                    j, f = pending.popleft()
                    rec, h, g = f.result()
                    if rec is None or not _continues_match(rec, recs[0] if recs else None, dst,
                                                           tok0 + (len(recs) - n0) * chunk_size):
                        drop(j % k, rec, h)
                        break
                    recs.append(rec)
                    handles.append(h)
                    got.append(g)
                    conn_of.append(j % k)
                    fill()
            finally:
                for j, f in pending:
                    drop(j % k, *f.result()[:2])
            return len(recs) - n0

        bounds = []                                    # per run: its records are recs[a:b] (keys), recs[b:c] (fallback)
        try:
            for i, (keys, fb, tok0) in enumerate(runs):
                a = len(recs)
                own = match(keys, tok0, i == 0)
                if fb is not None and own < len(fb):
                    match(fb[own:], tok0 + own * chunk_size, False)
                bounds.append((a, a + own, len(recs)))
        except BaseException:
            for c, rec, h in zip(conn_of, recs, handles):
                drop(c, rec, h)
            recs = []
            raise
        finally:
            for c, hs in stale.items():
                try:
                    conns[c].close_handles(hs)
                except Exception:      # noqa: BLE001 -- a lost connection has dropped its handles
                    pass
        n = len(recs)
        hits = [(b - a, c - b) for a, b, c in bounds]
        self._count(retrieves=1, opens=sum(h is not None for h in handles), match_s=time.perf_counter() - t_match,
                    bytes=sum(g for g, h in zip(got, handles) if h is not None))
        if n == 0:
            with torch.cuda.device(dst.device):
                ev = torch.cuda.Event()
                ev.record(torch.cuda.current_stream())
            return hits, LayerwiseUpload.completed(0, dst.L, ev)
        L = dst.L
        try:
            fixed, start, size = layer_copy_ranges([r.planes for r in recs], [r.nbytes for r in recs], L,
                                                   dst.planes // L, codec.raw_rows(recs, dst.latent))
            reads = ranged_read_plan(fixed, start, size, got, conn_of, k)
            fetch = RangedFetch(conns, reads, handles, [r.blk.host_ptr for r in recs], L, self._count)
            fetch.start(self._lw_pool)
        except BaseException:                 # nothing reads the blocks yet: free them, close the handles
            left = collections.defaultdict(list)
            for c, rec, h in zip(conn_of, recs, handles):
                rec.blk.free()
                if h is not None:
                    left[c].append(h)
            for c, hs in left.items():
                try:
                    conns[c].close_handles(hs)
                except Exception:      # noqa: BLE001
                    pass
            raise

        def done():
            try:
                fetch.finish()
            finally:
                self._release.add(recs[0].last_read, [r.blk for r in recs])
        matched = [(iter(recs[a:b]), (lambda i, rest=recs[b:c]: iter(rest)) if c > b else None, run[2])
                   for (a, b, c), run in zip(bounds, runs)]
        return upload_decode_layerwise_runs(codec, self._layerwise_uploader(dst.device), matched, dst, chunk_size,
                                            on_done=done, host_ready=fetch.wait, rotation=rotation)

    def close(self):
        if getattr(self, "_layerwise", None) is not None:
            self._layerwise.close()            # every layer-major job has ended (its fetch stopped, its blocks released)
            self._layerwise = None
        for attr in ("_lw_open_pool", "_lw_pool"):
            if getattr(self, attr, None) is not None:
                getattr(self, attr).shutdown(wait=True)
                setattr(self, attr, None)
        for c in getattr(self, "_lw_conns", []):
            try:
                c.close()
            except Exception:       # noqa: BLE001
                pass
        self._lw_conns = []
        if self.put_thread is not None and self.put_thread.is_alive():
            self.put_queue.put(RemoteBackendEndSignal())
            self.put_thread.join()
        if getattr(self, "_pipe", None) is not None:
            self._pipe.close()
            self._pipe = None
        if getattr(self, "_segments", None) is not None:
            self._segments.close()
            self._segments = None
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
