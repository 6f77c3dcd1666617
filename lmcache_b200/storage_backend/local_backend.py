"""LMCLocalBackend -- KV chunks in local GPU memory or page-locked host memory.

Reference: lmcache/storage_backend/local_backend.py:28-153.  There the "cpu" tier is a pageable
`tensor.to("cpu")` (pinned branch disabled, `torch.cuda.synchronize()` per put :82-100), a queue plus a
worker thread for non-blocking puts, and `.to("cuda")` on get (:141-144).

Here the host tier is the mover of include/b200kv.h: every put is one `b200kv_copy_async` into page-locked
memory on a dedicated side stream, completion is a CUDA event (no device-wide synchronize, no worker thread:
a "non-blocking put" is simply a put whose event has not been waited on yet), and a get is an async upload
ordered on the caller's stream.
"""
import ctypes
import threading
from typing import Dict, Optional

import torch

from lmcache_b200 import _native as N
from lmcache_b200.config import LMCacheEngineConfig
from lmcache_b200.logging import init_logger
from lmcache_b200.storage_backend.abstract_backend import LMCBackendInterface
from lmcache_b200.utils import CacheEngineKey, _lmcache_nvtx_annotate

logger = init_logger(__name__)


class _HostEntry:
    __slots__ = ("host", "event", "src")

    def __init__(self, host: torch.Tensor, event: Optional[torch.cuda.Event], src):
        self.host = host      # page-locked copy
        self.event = event    # completion of the device->host copy (None: already complete)
        self.src = src        # keeps the source alive until the copy has run

    def wait(self):
        if self.event is not None:
            self.event.synchronize()
            self.event = None
            self.src = None


def _copy_async(dst: torch.Tensor, src: torch.Tensor, stream: torch.cuda.Stream) -> None:
    N.check(N.lib().b200kv_copy_async(ctypes.c_void_p(dst.data_ptr()), ctypes.c_void_p(src.data_ptr()),
                                      src.numel() * src.element_size(), stream.cuda_stream), "copy_async")


class LMCLocalBackend(LMCBackendInterface):

    def __init__(self, config: LMCacheEngineConfig):
        super().__init__()
        N.require_cuda()
        self.chunk_size = config.chunk_size
        self.config = config
        self.device = config.local_device       # "cpu" | "cuda"
        self.dst_device = "cuda"                # like the reference (:53): gets land on the GPU
        self.dict: Dict[CacheEngineKey, object] = {}
        self.update_lock = threading.Lock()
        self._side: Optional[torch.cuda.Stream] = None
        self._inflight = []   # (event, pinned tensor) of uploads still reading host memory

    def _side_stream(self, device) -> torch.cuda.Stream:
        if self._side is None or self._side.device != device:
            self._side = torch.cuda.Stream(device=device)
        return self._side

    def contains(self, key: CacheEngineKey) -> bool:
        return key in self.dict

    @_lmcache_nvtx_annotate
    def put(self, key: CacheEngineKey, kv_chunk: torch.Tensor, blocking: bool = True) -> None:
        if self.device == "cuda":
            # reference: kv_chunk.to("cuda") -- a no-op for GPU chunks, an upload for host chunks
            val = kv_chunk if kv_chunk.is_cuda else kv_chunk.to("cuda", non_blocking=False)
            with self.update_lock:
                self.dict[key] = val
            return
        # host tier
        if not kv_chunk.is_cuda:
            entry = _HostEntry(kv_chunk.detach().clone().pin_memory(), None, None)
        else:
            src = kv_chunk if kv_chunk.is_contiguous() else kv_chunk.contiguous()
            host = torch.empty(src.shape, dtype=src.dtype, pin_memory=True)
            side = self._side_stream(src.device)
            side.wait_stream(torch.cuda.current_stream(src.device))   # producer kernels finished first
            _copy_async(host, src, side)
            ev = torch.cuda.Event()
            ev.record(side)
            entry = _HostEntry(host, ev, src)
            if blocking:
                entry.wait()
        with self.update_lock:
            self.dict[key] = entry

    @_lmcache_nvtx_annotate
    def get(self, key: CacheEngineKey) -> Optional[torch.Tensor]:
        val = self.dict.get(key, None)
        if val is None:
            return None
        if isinstance(val, _HostEntry):
            val.wait()
            out = torch.empty(val.host.shape, dtype=val.host.dtype, device=self.dst_device)
            stream = torch.cuda.current_stream(out.device)
            _copy_async(out, val.host, stream)   # ordered on the consumer's stream
            # the pinned block must outlive the DMA even if the key is overwritten meanwhile
            ev = torch.cuda.Event()
            ev.record(stream)
            self._inflight = [(e, h) for e, h in self._inflight if not e.query()]
            self._inflight.append((ev, val.host))
            return out
        return val.to(self.dst_device)

    # ------------------------------------------------------------------ engine fast paths
    def supports_kv_view(self) -> bool:
        return True

    def peek_geometry(self, key, fmt: str = "vllm"):
        """(L, H, D, dtype) of a stored chunk blob, from its shape (no copy): [L,2,t,H,D] (vllm) / [L,2,H,t,D] (hf)."""
        val = self.dict.get(key, None)
        if val is None:
            return None
        t = val.host if isinstance(val, _HostEntry) else val
        if t.dim() != 5:
            return None
        return (t.shape[0], t.shape[2], t.shape[4], t.dtype) if fmt == "huggingface" else \
            (t.shape[0], t.shape[3], t.shape[4], t.dtype)

    def put_kv_chunks(self, keys, view, tok_begin: int, chunk_size: int, blocking: bool = True) -> int:
        """Store tokens [tok_begin, T) of `view` as len(keys) chunk blobs: ONE gather kernel (b200kv_pack_chunks)
        builds every chunk blob; for the host tier ONE device->host DMA moves them all into a page-locked slab."""
        fmt_hf = getattr(view, "fmt", "vllm") == "huggingface"
        n_tok = view.ntokens - tok_begin
        n_chunks = len(keys)
        assert n_chunks == (n_tok + chunk_size - 1) // chunk_size
        last = n_tok - (n_chunks - 1) * chunk_size
        per_tok = 2 * view.L * view.H * view.D
        stride = per_tok * chunk_size
        dev = torch.empty(n_chunks * stride, dtype=view.dtype, device=view.device)
        with torch.cuda.device(view.device):
            cur = torch.cuda.current_stream()
            N.check(N.lib().b200kv_pack_chunks(ctypes.byref(view.desc), tok_begin, n_chunks, chunk_size, last,
                                               1 if fmt_hf else 0, ctypes.c_void_p(dev.data_ptr()),
                                               stride * dev.element_size(), cur.cuda_stream), "pack_chunks")

            def shape(t):
                return (view.L, 2, view.H, t, view.D) if fmt_hf else (view.L, 2, t, view.H, view.D)

            if self.device == "cuda":
                vals = [dev[j * stride: j * stride + per_tok * (chunk_size if j < n_chunks - 1 else last)]
                        .view(shape(chunk_size if j < n_chunks - 1 else last)) for j in range(n_chunks)]
            else:
                host = torch.empty(n_chunks * stride, dtype=view.dtype, pin_memory=True)
                side = self._side_stream(view.device)
                side.wait_stream(cur)
                _copy_async(host, dev, side)
                ev = torch.cuda.Event()
                ev.record(side)
                vals = []
                for j in range(n_chunks):
                    t = chunk_size if j < n_chunks - 1 else last
                    vals.append(_HostEntry(host[j * stride: j * stride + per_tok * t].view(shape(t)), ev, dev))
                if blocking:
                    ev.synchronize()
                    for v in vals:
                        v.event, v.src = None, None
        with self.update_lock:
            for key, v in zip(keys, vals):
                self.dict[key] = v
        return n_chunks

    def get_kv_into(self, keys, dst, dst_tok0: int, chunk_size: int) -> int:
        """Copy consecutive chunks (until the first miss) straight into the destination blob view `dst` at token
        offsets dst_tok0 + i * chunk_size: strided 2-D copies (host tier: async uploads), no intermediate chunk tensors,
        no torch.cat."""
        fmt_hf = getattr(dst, "fmt", "vllm") == "huggingface"
        blob = dst.blob
        if blob is None:
            return self._get_kv_scatter(keys, dst, dst_tok0, chunk_size)
        n = 0
        with torch.cuda.device(blob.device):
            stream = torch.cuda.current_stream()
            for i, key in enumerate(keys):
                val = self.dict.get(key, None)
                if val is None:
                    break
                src = val.host if isinstance(val, _HostEntry) else val
                if isinstance(val, _HostEntry):
                    val.wait()
                elif not src.is_cuda:
                    src = src.cuda()
                t = src.shape[3] if fmt_hf else src.shape[2]
                tok = dst_tok0 + i * chunk_size
                if tok + t > dst.ntokens or src.dtype != blob.dtype:
                    break
                es = blob.element_size()
                if fmt_hf:      # rows = (l, kv, h): t*D contiguous elements each
                    rows, row_bytes = blob.shape[0] * 2 * blob.shape[2], t * blob.shape[4] * es
                    dst_pitch = blob.shape[3] * blob.shape[4] * es
                    dptr = blob.data_ptr() + tok * blob.shape[4] * es
                else:           # rows = (l, kv): t*H*D contiguous elements each
                    rows, row_bytes = blob.shape[0] * 2, t * blob.shape[3] * blob.shape[4] * es
                    dst_pitch = blob.shape[2] * blob.shape[3] * blob.shape[4] * es
                    dptr = blob.data_ptr() + tok * blob.shape[3] * blob.shape[4] * es
                N.check(N.lib().b200kv_copy2d_async(ctypes.c_void_p(dptr), dst_pitch, ctypes.c_void_p(src.data_ptr()),
                                                    row_bytes, row_bytes, rows, stream.cuda_stream), "copy2d")
                if isinstance(val, _HostEntry):
                    ev = torch.cuda.Event()
                    ev.record(stream)
                    self._inflight = [(e, h) for e, h in self._inflight if not e.query()]
                    self._inflight.append((ev, val.host))
                n += 1
        return n

    def _get_kv_scatter(self, keys, dst, dst_tok0: int, chunk_size: int) -> int:
        """get_kv_into for destinations that are not one blob (the engine's 2L tensors, or a paged KV cache with its
        slot mapping): each hit chunk is scattered by ONE b200kv_unpack_chunks launch (host tier: after one upload)."""
        n = 0
        hf = getattr(dst, "fmt", "vllm") == "huggingface"      # chunk blobs carry the engine's layout
        with torch.cuda.device(dst.device):
            stream = torch.cuda.current_stream()
            for i, key in enumerate(keys):
                val = self.dict.get(key, None)
                if val is None:
                    break
                if isinstance(val, _HostEntry):
                    val.wait()
                    src = val.host.to(dst.device, non_blocking=True)
                else:
                    src = val if val.is_cuda else val.cuda()
                t = src.shape[3] if hf else src.shape[2]
                tok = dst_tok0 + i * chunk_size
                if tok + t > dst.ntokens or src.dtype != dst.dtype:
                    break
                src = src.contiguous()
                N.check(N.lib().b200kv_unpack_chunks(ctypes.c_void_p(src.data_ptr()), src.numel() * src.element_size(), 1,
                                                     t, t, 1 if hf else 0, ctypes.byref(dst.desc), tok,
                                                     stream.cuda_stream), "unpack_chunks")
                src.record_stream(stream)
                n += 1
        return n

    def close(self):
        for val in list(self.dict.values()):
            if isinstance(val, _HostEntry):
                val.wait()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---------------------------------------------------------------------------------------------- compressed host tier
class _CEntry:
    """One CacheGen container in the page-locked slab."""
    __slots__ = ("blk", "path", "nbytes", "ntokens", "L", "H", "D", "max_dtype", "coder", "ready", "error", "last_read")

    def __init__(self):
        self.blk = None
        self.path = None                     # disk tier: the container's file (then blk is None)
        self.nbytes = 0
        self.ntokens = 0
        self.L = self.H = self.D = 0
        self.max_dtype = 0
        self.coder = 0
        self.ready = threading.Event()       # set by the store worker once the container is in host memory
        self.error: Optional[BaseException] = None
        self.last_read: Optional[torch.cuda.Event] = None   # most recent upload out of the block


class LMCLocalCompressedBackend(LMCBackendInterface):
    """local_device="cpu" + local_serde="cachegen": the host tier keeps CacheGen containers instead of raw blobs.

    Replaces LMCLocalBackend("cpu") (lmcache/storage_backend/local_backend.py:28-153) for BASELINE configs[2]: the
    bytes crossing PCIe and sitting in host memory shrink by the codec's ratio (5.9x on the SURVEY 8d data), and both
    directions are pipelined (lmcache_b200/pipeline.py):
      store     waves of chunks are encoded on the caller's stream (enqueue only) while a worker thread moves the
                previous wave's containers -- exactly their bytes -- into the page-locked slab on a copy stream;
      retrieve  the containers of wave i+1 are uploaded on a copy stream while wave i is decoded straight into the
                destination; slot reuse is ordered by events, the host never waits.
    Every container lives in one PinnedSlab (one cudaHostAlloc per GiB, not one per put)."""

    def __init__(self, config: LMCacheEngineConfig, metadata):
        super().__init__()
        from lmcache_b200.codec import CacheGenCodec
        from lmcache_b200.pipeline import EncodePipeline, UploadRing
        from lmcache_b200.slab import PinnedSlab
        N.require_cuda()
        self.chunk_size = config.chunk_size
        self.fmt = metadata.fmt
        if self.fmt not in ("vllm", "huggingface"):
            raise ValueError(f"Invalid format: {self.fmt}")
        self.codec = CacheGenCodec(metadata.model_name)      # ValueError for models outside the bin table
        self.slab = PinnedSlab()
        self.dict: Dict[CacheEngineKey, _CEntry] = {}
        self.update_lock = threading.Lock()
        self._copy_stream: Optional[torch.cuda.Stream] = None
        self._pipe = EncodePipeline(self.codec, self._sink)
        self._upload: Optional[UploadRing] = None
        self._retired = []                                    # (event, block): overwritten entries still being read
        self._closed = False

    # ------------------------------------------------------------------ store
    def _land(self, slot, batch, entries) -> None:
        """worker thread: the wave's containers -> slab blocks (one async copy each, exactly `size` bytes); fills the
        entries from the container headers.  Raises (after marking the entries) when anything is wrong."""
        dev = slot.dev.device
        with torch.cuda.device(dev):
            if self._copy_stream is None or self._copy_stream.device != dev:
                self._copy_stream = torch.cuda.Stream(device=dev)
            cs = self._copy_stream
            try:
                blocks = []
                for j, size in enumerate(batch.sizes):
                    blk = self.slab.alloc(size)
                    blocks.append(blk)
                    N.check(N.lib().b200kv_copy_async(ctypes.c_void_p(blk.host_ptr),
                                                      ctypes.c_void_p(slot.dev.data_ptr() + j * batch.stride), size,
                                                      cs.cuda_stream), "copy_async")
                cs.synchronize()
                from lmcache_b200.codec import parse_header
                for e, blk in zip(entries, blocks):
                    hd = parse_header(blk.view())              # raises on a nonzero encoder status
                    e.blk, e.nbytes, e.ntokens = blk, blk.nbytes, int(hd.ntokens)
                    e.L, e.H, e.D, e.max_dtype, e.coder = int(hd.L), int(hd.H), int(hd.D), int(hd.max_dtype), int(hd.version) - 1
            except BaseException as err:     # noqa: BLE001
                for e in entries:
                    e.error = err
                raise

    def _sink(self, slot, batch, c0, entries) -> None:
        """store pipeline sink: land the wave in host memory, then publish the entries (readers wait on `ready`)"""
        try:
            self._land(slot, batch, entries)
        finally:
            for e in entries:
                e.ready.set()

    def _retire(self, e: _CEntry) -> None:
        if e.blk is None:
            return
        if e.last_read is not None and not e.last_read.query():
            self._retired.append((e.last_read, e.blk))
        else:
            e.blk.free()
        e.blk = None

    def _sweep(self) -> None:
        keep = []
        for ev, blk in self._retired:
            if ev.query():
                blk.free()
            else:
                keep.append((ev, blk))
        self._retired = keep

    def put_kv_chunks(self, keys, view, tok_begin: int, chunk_size: int, blocking: bool = True) -> int:
        # `keys` may be lazy (the engine's hash chain produces key i after keys 0..i-1): the encode waves
        # need no keys, so they are enqueued first; the entries are published as their keys arrive.  Readers wait on `ready`.
        entries = [_CEntry() for _ in range(len(keys))]
        job = self._pipe.submit(view, tok_begin, chunk_size, entries)
        old = []
        for k, e in zip(keys, entries):
            with self.update_lock:
                prev = self.dict.get(k)
                if prev is not None:
                    old.append(prev)
                self.dict[k] = e
        for prev in old:                            # an overwritten container leaves once nobody reads it any more
            prev.ready.wait()
            self._retire(prev)
        self._sweep()
        if blocking:
            job.wait()
        return len(keys)

    @_lmcache_nvtx_annotate
    def put(self, key: CacheEngineKey, kv_chunk: torch.Tensor, blocking: bool = True) -> None:
        from lmcache_b200.codec import KvView
        if not kv_chunk.is_cuda:
            kv_chunk = kv_chunk.cuda()              # reference: tensor.cuda() in the serializer (cachegen_encoder.py:383)
        view = KvView.from_blob(kv_chunk, self.fmt)
        self.put_kv_chunks([key], view, 0, view.ntokens, blocking=blocking)

    # ------------------------------------------------------------------ lookup
    def contains(self, key: CacheEngineKey) -> bool:
        e = self.dict.get(key)
        if e is None:
            return False
        if e.ready.is_set() and e.error is not None:
            return False
        return True

    def _ready_entry(self, key) -> Optional[_CEntry]:
        e = self.dict.get(key)
        if e is None:
            return None
        e.ready.wait()
        return None if e.error is not None or e.blk is None else e

    def peek_geometry(self, key, fmt: str = "vllm"):
        """(L, H, D, output dtype) of the stored chunks, read from a container header (no decode)."""
        e = self._ready_entry(key)
        return None if e is None else (e.L, e.H, e.D, self.out_dtype())

    def out_dtype(self) -> torch.dtype:
        # the reference's decoder casts by format, ignoring metadata.dtype (cachegen_decoder.py:189-200)
        return torch.bfloat16 if self.fmt == "vllm" else torch.float16

    # ------------------------------------------------------------------ retrieve
    def supports_kv_view(self) -> bool:
        return True

    def get_kv_into(self, keys, dst, dst_tok0: int, chunk_size: int) -> int:
        """Upload + decode consecutive chunks (until the first miss) straight into `dst`; chunk i lands at token
        dst_tok0 + i * chunk_size.  Everything is enqueued: copies on the copy stream, decodes on the current stream."""
        from lmcache_b200.pipeline import UploadRing, wave_chunks_default
        W = wave_chunks_default()
        lib = N.lib()
        n_hits = 0
        first = None
        with torch.cuda.device(dst.device):
            if self._upload is None or self._upload.device != dst.device:
                self._upload = UploadRing(dst.device)
            up = self._upload
            cur = torch.cuda.current_stream()

            def flush(wave, w0):
                offs, o = [], 0
                for e in wave:
                    offs.append(o)
                    o += (e.nbytes + 15) & ~15
                slot, buf = up.next_slot(o)
                for e, off in zip(wave, offs):
                    N.check(lib.b200kv_copy_async(ctypes.c_void_p(buf.data_ptr() + off), ctypes.c_void_p(e.blk.host_ptr),
                                                  e.nbytes, up.copy_stream.cuda_stream), "copy_async")
                ev = torch.cuda.Event()
                ev.record(up.copy_stream)
                for e in wave:
                    e.last_read = ev
                cur.wait_event(ev)
                self.codec.decode_raw(buf.data_ptr(), buf.numel(), offs, [e.nbytes for e in wave],
                                      [e.ntokens for e in wave], dst,
                                      [dst_tok0 + (w0 + j) * chunk_size for j in range(len(wave))],
                                      wave[0].max_dtype, wave[0].coder, cur)
                up.mark_read(slot, cur)

            # keys may be lazy (the hash chain is still running): every full wave is uploaded and decoded as soon as its
            # keys exist, while the chain works on the later chunks
            wave = []
            for i, key in enumerate(keys):
                e = self._ready_entry(key)
                if e is None or (e.L, e.H, e.D) != (dst.L, dst.H, dst.D):
                    break
                if dst_tok0 + i * chunk_size + e.ntokens > dst.ntokens:
                    break
                if first is not None and (e.max_dtype, e.coder) != (first.max_dtype, first.coder):
                    break
                first = first or e
                wave.append(e)
                n_hits += 1
                if len(wave) == W:
                    flush(wave, n_hits - W)
                    wave = []
            if wave:
                flush(wave, n_hits - len(wave))
        return n_hits

    @_lmcache_nvtx_annotate
    def get(self, key: CacheEngineKey) -> Optional[torch.Tensor]:
        from lmcache_b200.codec import KvView
        e = self._ready_entry(key)
        if e is None:
            return None
        shape = (e.L, 2, e.ntokens, e.H, e.D) if self.fmt == "vllm" else (e.L, 2, e.H, e.ntokens, e.D)
        out = torch.empty(shape, dtype=self.out_dtype(), device=torch.device("cuda", torch.cuda.current_device()))
        if self.get_kv_into([key], KvView.from_blob(out, self.fmt), 0, e.ntokens) != 1:
            return None
        return out

    def reserve_host(self, nbytes: int) -> None:
        """Page-lock at least nbytes of slab up front (a cudaHostAlloc of 1 GiB takes ~0.3 s: better at start-up than
        inside a store)."""
        self.slab.reserve(int(nbytes))

    def host_bytes(self) -> int:
        """bytes of containers currently held (for reports)"""
        return self.slab.stats()[2]

    def close(self):
        if self._closed:
            return
        self._closed = True
        self._pipe.close()
        try:
            torch.cuda.synchronize()
        except Exception:       # noqa: BLE001 -- interpreter shutdown
            pass
        self.slab.close()

    def __del__(self):
        try:
            self.close()
        except Exception:       # noqa: BLE001
            pass


# ---------------------------------------------------------------------------------------------- disk tier
class LMCLocalDiskBackend(LMCLocalCompressedBackend):
    """local_device = "file://<dir>/": CacheGen containers as files, one per chunk (SURVEY.md 8f rank 4).

    Replaces LMCLocalDiskBackend of the reference (lmcache/storage_backend/local_backend.py:163-310: one raw safetensors
    file per key, a synchronous save per chunk, an in-memory key set that is empty after a restart).  Here
      * a chunk on disk is its B2KV container (5.9x smaller on the SURVEY 8d data), written by the store pipeline's
        worker from the page-locked block the device->host copy landed in, to `<key>.b2kv.tmp` and renamed -- a file
        that exists is complete;
      * the index (key -> file, size, geometry) is rebuilt from the directory when the backend starts: headers are read
        and checked, damaged or foreign files are ignored -- a restart keeps the cache;
      * retrieve reads the files of the requested chunks with a small thread pool straight into page-locked blocks while
        earlier waves upload and decode (disk || H2D || decode, lmcache_b200/pipeline.py fetch_decode)."""

    SUFFIX = ".b2kv"

    def __init__(self, config: LMCacheEngineConfig, metadata):
        import os
        from concurrent.futures import ThreadPoolExecutor
        path = config.local_device
        assert path is not None, "Need to specify local path if when using LMCLocalDiskBackend"
        self.path = path if path.endswith("/") else path + "/"
        os.makedirs(self.path, exist_ok=True)
        super().__init__(config, metadata)
        self._io = ThreadPoolExecutor(max_workers=max(1, int(os.environ.get("LMCACHE_B200_DISK_THREADS", "4"))),
                                      thread_name_prefix="b200kv-disk")
        self._inflight_reads = []               # (event, [blocks]) of uploads out of transient read blocks
        self._rebuild_index()

    # ---- index
    def _key_to_path(self, key: CacheEngineKey) -> str:
        return self.path + key.to_string().replace("/", "-") + self.SUFFIX      # reference naming rule (:228)

    def _rebuild_index(self) -> int:
        import os

        from lmcache_b200.codec import check_header
        n = 0
        for name in os.listdir(self.path):
            if not name.endswith(self.SUFFIX):
                continue
            full = self.path + name
            try:
                size = os.path.getsize(full)
                if size < N.HEADER_BYTES:
                    continue
                with open(full, "rb") as f:
                    head = f.read(N.HEADER_BYTES + N.MAX_PLANES)
                hd = N.Header.from_buffer_copy(head[:N.HEADER_BYTES])
                if hd.magic != N.MAGIC or hd.version not in (1, 2, 3) or hd.status != 0 or int(hd.total_bytes) != size:
                    continue
                check_header(hd, list(head[N.HEADER_BYTES:N.HEADER_BYTES + 2 * hd.L]) if hd.version == 3 else None)
            except (OSError, ValueError):
                continue                         # damaged / foreign file: not part of the cache
            # "/" in a model name was written as "-": the key of a lookup goes through the same rule, so index by path
            e = _CEntry()
            e.path, e.nbytes, e.ntokens = full, size, int(hd.ntokens)
            e.L, e.H, e.D, e.max_dtype, e.coder = int(hd.L), int(hd.H), int(hd.D), int(hd.max_dtype), int(hd.version) - 1
            e.ready.set()
            self._by_path[full] = e
            n += 1
        return n

    # the dict is keyed by file path: CacheEngineKey -> path is many-to-one ("/" and "-"), exactly as in the reference
    @property
    def _by_path(self):
        return self.dict

    def _lookup(self, key: CacheEngineKey):
        return self.dict.get(self._key_to_path(key))

    def contains(self, key: CacheEngineKey) -> bool:
        e = self._lookup(key)
        return e is not None and not (e.ready.is_set() and e.error is not None)

    def _ready_entry(self, key):
        e = self._lookup(key)
        if e is None:
            return None
        e.ready.wait()
        return None if e.error is not None or e.path is None else e

    # ---- store: the pipeline's sink writes files instead of keeping blocks
    def _sink(self, slot, batch, c0, entries) -> None:
        import os
        try:
            self._land(slot, batch, entries)             # containers -> page-locked blocks, headers parsed
            for e in entries:
                tmp = e.path + ".tmp"
                try:
                    with open(tmp, "wb") as f:
                        f.write(e.blk.view())
                    os.replace(tmp, e.path)               # a file that exists is complete
                except OSError as err:
                    e.error = err
        finally:
            for e in entries:
                if e.blk is not None:
                    e.blk.free()
                    e.blk = None
                e.ready.set()                             # readers see the entry only once its file is in place

    def put_kv_chunks(self, keys, view, tok_begin: int, chunk_size: int, blocking: bool = True) -> int:
        entries = [_CEntry() for _ in keys]
        for k, e in zip(keys, entries):
            e.path = self._key_to_path(k)
            e.ready.clear()
        with self.update_lock:
            for e in entries:
                self.dict[e.path] = e                     # an overwritten chunk's file is replaced atomically by the rename
        # the parent's sink sets `ready` before the file exists: keep readers out until the file is written
        job = self._pipe.submit(view, tok_begin, chunk_size, entries)
        if blocking:
            job.wait()
        return len(keys)

    # ---- retrieve
    def _read_file(self, e: _CEntry):
        blk = self.slab.alloc(e.nbytes)
        try:
            with open(e.path, "rb", buffering=0) as f:
                got = f.readinto(blk.view())
                while got is not None and 0 < got < e.nbytes:
                    more = f.readinto(blk.view()[got:])
                    if not more:
                        break
                    got += more
            if got != e.nbytes:
                raise OSError("short read")
            return blk, e.nbytes
        except OSError:
            blk.free()
            return None

    def get_kv_into(self, keys, dst, dst_tok0: int, chunk_size: int) -> int:
        from lmcache_b200.pipeline import UploadRing, fetch_decode
        keep = []
        for ev, blocks in self._inflight_reads:          # transient read blocks of earlier calls
            if ev.query():
                for b in blocks:
                    b.free()
            else:
                keep.append((ev, blocks))
        self._inflight_reads = keep
        futs = []
        for key in keys:
            e = self._ready_entry(key)
            if e is None:
                break
            futs.append(self._io.submit(self._read_file, e))
        if not futs:
            return 0
        with torch.cuda.device(dst.device):
            if self._upload is None or self._upload.device != dst.device:
                self._upload = UploadRing(dst.device)
        return fetch_decode(self.codec, self._upload, futs, dst, dst_tok0, chunk_size, self._inflight_reads)

    def host_bytes(self) -> int:
        return sum(e.nbytes for e in self.dict.values() if e.path is not None)

    def close(self):
        if self._closed:
            return
        self._pipe.close()
        self._io.shutdown(wait=True)
        try:
            torch.cuda.synchronize()
        except Exception:       # noqa: BLE001
            pass
        for _, blocks in self._inflight_reads:
            for b in blocks:
                b.free()
        self._inflight_reads = []
        self._closed = True
        self.slab.close()
