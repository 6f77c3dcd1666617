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
import sys
import threading
import time
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from lmcache_b200 import _native as N
from lmcache_b200.codec import KvView
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


# ---------------------------------------------------------------------------------------------- layer slices of raw blobs
# A raw chunk blob of t tokens holds its layers back to back: layer l is one contiguous slice of t * row bytes at
# l * t * row, where row = ppl * H * D * element bytes (ppl = 2 for [L,2,t,H,D] / [L,2,H,t,D], 1 for a latent [L,t,D]).
LAYER_SLOTS = 3          # staging ring of the raw cpu tier's layer-wise paths: a layer's copy overlaps the previous unpack


def layer_row_bytes(H: int, D: int, elem_bytes: int, latent: bool) -> int:
    """bytes per token of one layer slice of a raw chunk blob (H = 1 for a latent KV)"""
    return (1 if latent else 2) * H * D * elem_bytes


def layer_table(bases: Sequence[int], tokens: Sequence[int], row_bytes: int, layer: int) -> np.ndarray:
    """uint64 [n]: where layer `layer` of chunk j starts, for chunk blobs at bases[j] of tokens[j] tokens each -- the
    chunk_ptrs of b200kv_pack_chunks_layers / b200kv_unpack_chunks_layers for the range [layer, layer + 1).  A staging
    area that holds one layer of every chunk back to back is layer_table(area + packed_offsets(tokens, row), ..., 0)."""
    return np.asarray(bases, dtype=np.uint64) + np.uint64(layer * row_bytes) * np.asarray(tokens, dtype=np.uint64)


def packed_offsets(tokens: Sequence[int], row_bytes: int) -> np.ndarray:
    """uint64 [n]: offset of chunk j's slice in an area that holds one layer slice of each chunk back to back"""
    sl = np.asarray(tokens, dtype=np.uint64) * np.uint64(row_bytes)
    return np.concatenate([np.zeros(1, np.uint64), np.cumsum(sl, dtype=np.uint64)[:-1]]) if len(sl) else sl


def chunk_runs(tokens: Sequence[int], chunk_size: int) -> List[tuple]:
    """The chunk ranges [a, b) one mover launch takes: every chunk but the range's last has chunk_size tokens, and its
    last at most that many; a chunk of any other size moves alone.  Returns (a, b, chunk_tokens, last_chunk_tokens)."""
    runs, a = [], 0
    for j, t in enumerate(tokens):
        if t > chunk_size and a < j:                 # a longer chunk is never the tail of a run
            runs.append((a, j, chunk_size, tokens[j - 1]))
            a = j
        if t != chunk_size or j == len(tokens) - 1:
            runs.append((a, j + 1, chunk_size if j > a else t, t))
            a = j + 1
    return runs


def _device_table(rows: np.ndarray, device, stream: torch.cuda.Stream) -> torch.Tensor:
    """a pointer table in device memory, uploaded on `stream` (which is also the stream the allocator ties it to)"""
    with torch.cuda.stream(stream):
        return torch.from_numpy(np.ascontiguousarray(rows).view(np.int64)).pin_memory().to(device, non_blocking=True)


def _mover_layers(pack: bool, view, table_ptr: int, tok_begin: int, run: tuple, layer: int, stream) -> None:
    a, b, ct, lt = run
    hf = int(getattr(view, "fmt", "vllm") == "huggingface")
    if pack:
        rc = N.lib().b200kv_pack_chunks_layers(ctypes.byref(view.desc), tok_begin, b - a, ct, lt, hf, layer, layer + 1,
                                               ctypes.c_void_p(table_ptr + 8 * a), stream.cuda_stream)
    else:
        rc = N.lib().b200kv_unpack_chunks_layers(ctypes.c_void_p(table_ptr + 8 * a), b - a, ct, lt, hf, layer, layer + 1,
                                                 ctypes.byref(view.desc), tok_begin, stream.cuda_stream)
    N.check(rc, "pack_chunks_layers" if pack else "unpack_chunks_layers")


class RawLayerwiseStore:
    """One layer-wise store into a raw tier (LMCLocalBackend.begin_layerwise_store): what LayerwiseStore uses of a
    pipeline.LayerwiseEncode.  encode_layer(l, stream) packs layer l of every chunk (b200kv_pack_chunks_layers) on the
    tier's pack stream behind an event on `stream`.  The cuda tier packs straight into the final blobs; the cpu tier
    packs into a device ring of LAYER_SLOTS layer slots and moves each layer into the store's page-locked buffer with one
    strided copy on the copy stream, so that the store holds a few layers of HBM, not the whole store.  The blobs are
    byte for byte those of KvView.pack_chunks (store / store_paged)."""

    def __init__(self, tier: "LMCLocalBackend", view, tok_begin: int, chunk_size: int):
        n_tok = view.ntokens - tok_begin
        n = (n_tok + chunk_size - 1) // chunk_size
        self.tier, self.view, self.tok_begin, self.cs = tier, view, tok_begin, chunk_size
        self.L, self.H, self.D, self.latent, self.fmt = view.L, view.H, view.D, view.latent, view.fmt
        self.sizes = [min(chunk_size, n_tok - j * chunk_size) for j in range(n)]
        self.run = (0, n, chunk_size, self.sizes[-1])
        es = view.dtype.itemsize
        self.row = layer_row_bytes(view.H, view.D, es, view.latent)
        self.stride = view.L * self.row * chunk_size             # bytes between chunk blobs, as in pack_chunks
        self.ps, self.cs_stream = tier._layer_streams(view.device)
        self.saves = 0
        self.copied: List[torch.cuda.Event] = []                 # cpu tier: the copy event of each save, in save order
        self.done: Optional[torch.cuda.Event] = None
        self.host = None
        with torch.cuda.device(view.device):
            view.record_stream(self.ps)                          # the caller's KV outlives the last pack that reads it
            if tier.device == "cuda":
                # allocated on the caller's stream like pack_chunks' buffer: the entries are read there afterwards
                self.buf = torch.empty(n * self.stride // es, dtype=view.dtype, device=view.device)
                self.buf.record_stream(self.ps)
                rows = np.stack([layer_table(self.buf.data_ptr() + self.stride * np.arange(n, dtype=np.uint64),
                                             self.sizes, self.row, l) for l in range(view.L)])
            else:
                self.host = torch.empty(n * self.stride // es, dtype=view.dtype, pin_memory=True)
                self.slot_bytes = n_tok * self.row
                with torch.cuda.stream(self.ps):
                    self.buf = torch.empty(LAYER_SLOTS * self.slot_bytes, dtype=torch.uint8, device=view.device)
                self.buf.record_stream(self.cs_stream)
                offs = packed_offsets(self.sizes, self.row)
                rows = np.stack([np.uint64(self.buf.data_ptr() + r * self.slot_bytes) + offs for r in range(LAYER_SLOTS)])
            self.table = _device_table(rows, view.device, self.ps)

    def encode_layer(self, layer: int, stream: torch.cuda.Stream, ready: Optional[torch.cuda.Event] = None) -> None:
        """`ready`: an event already recorded on `stream` after layer `layer` was written (pipeline.FanOutEncode's)"""
        with torch.cuda.device(self.view.device):
            ev = ready
            if ev is None:
                ev = torch.cuda.Event()
                ev.record(stream)
            self.ps.wait_event(ev)
            k, self.saves = self.saves, self.saves + 1
            if self.host is None:
                _mover_layers(True, self.view, self.table[layer].data_ptr(), self.tok_begin, self.run, layer, self.ps)
                return
            slot = k % LAYER_SLOTS
            if k >= LAYER_SLOTS:
                self.ps.wait_event(self.copied[k - LAYER_SLOTS])      # the slot's previous layer has left it
            _mover_layers(True, self.view, self.table[slot].data_ptr(), self.tok_begin, self.run, layer, self.ps)
            packed = torch.cuda.Event()
            packed.record(self.ps)
            self.cs_stream.wait_event(packed)
            src = self.buf.data_ptr() + slot * self.slot_bytes
            dst = self.host.data_ptr() + layer * self.cs * self.row
            full = len(self.sizes) if self.sizes[-1] == self.cs else len(self.sizes) - 1
            sl = self.cs * self.row
            N.check(N.lib().b200kv_copy2d_async(ctypes.c_void_p(dst), self.stride, ctypes.c_void_p(src), sl, sl, full,
                                                self.cs_stream.cuda_stream), "copy2d")
            if full < len(self.sizes):                              # the ragged last chunk's slice
                t = self.sizes[-1]
                N.check(N.lib().b200kv_copy_async(ctypes.c_void_p(self.host.data_ptr() + full * self.stride +
                                                                  layer * t * self.row),
                                                  ctypes.c_void_p(src + full * sl), t * self.row,
                                                  self.cs_stream.cuda_stream), "copy_async")
            copied = torch.cuda.Event()
            copied.record(self.cs_stream)
            self.copied.append(copied)

    def finish(self) -> torch.cuda.Event:
        """the event after the last pack: the caller's KV is no longer read.  self.done: the blobs are complete"""
        with torch.cuda.device(self.view.device):
            last = torch.cuda.Event()
            last.record(self.ps)
            if self.host is None:
                self.done = last
            else:
                self.done = torch.cuda.Event()
                self.done.record(self.cs_stream)
        self.view = None
        return last

    def blobs(self) -> list:
        """the chunk blobs (device tensors, or page-locked views for the cpu tier), after finish()"""
        out = []
        base = self.buf if self.host is None else self.host
        es = base.element_size()
        for j, t in enumerate(self.sizes):
            shape = (self.L, t, self.D) if self.latent else KvView.blob_shape(self.fmt, self.L, self.H, self.D, t)
            off = j * self.stride // es
            out.append(base[off: off + t * self.L * self.row // es].view(shape))
        return out

    def abandon(self) -> None:
        """drop the store; copies still queued keep the page-locked buffer alive until they have run"""
        if self.host is not None and self.copied:
            self.tier._keep_until(self.copied[-1], self.host)
        self.view, self.host, self.buf = None, None, None


class LMCLocalBackend(LMCBackendInterface):

    def __init__(self, config: LMCacheEngineConfig, metadata=None):
        super().__init__()
        N.require_cuda()
        self.chunk_size = config.chunk_size
        self.config = config
        # the engine's KV is latent (metadata.use_mla): chunk blobs are [L,t,D], and only those are its chunks
        self.latent = bool(getattr(metadata, "use_mla", False))
        self.device = config.local_device       # "cpu" | "cuda"
        self.dst_device = "cuda"                # like the reference (:53): gets land on the GPU
        self.dict: Dict[CacheEngineKey, object] = {}
        self.update_lock = threading.Lock()
        self._side: Optional[torch.cuda.Stream] = None
        self._layer: Optional[tuple] = None   # (mover stream, copy stream) of the layer-wise paths
        self._inflight = []   # (event, pinned tensor) of uploads still reading host memory

    def _side_stream(self, device) -> torch.cuda.Stream:
        if self._side is None or self._side.device != device:
            self._side = torch.cuda.Stream(device=device)
        return self._side

    def _layer_streams(self, device) -> tuple:
        """the streams of the layer-wise store and retrieve: one for the pack / unpack kernels, one for the copies"""
        device = torch.device(device)
        if self._layer is None or self._layer[0].device != device:
            self._layer = (torch.cuda.Stream(device=device), torch.cuda.Stream(device=device))
        return self._layer

    def _keep_until(self, event: torch.cuda.Event, host) -> None:
        """the page-locked block(s) `host` outlive the copies before `event` even if nothing else holds them"""
        self._inflight = [(e, h) for e, h in self._inflight if not e.query()]
        self._inflight.append((event, host))

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

    def supports_split_view(self) -> bool:
        """a split paged view (PagedAttention's layout) is read and written by the mover alone: taken as it is"""
        return True

    def peek_geometry(self, key, fmt: str = "vllm"):
        """(L, H, D, dtype) of a stored chunk blob, from its shape (no copy): [L,2,t,H,D] (vllm) / [L,2,H,t,D] (hf); for
        a latent engine [L,t,D] (H = 1).  None for a blob of the other kind."""
        val = self.dict.get(key, None)
        if val is None:
            return None
        t = val.host if isinstance(val, _HostEntry) else val
        return KvView.blob_geometry(t, fmt) if t.dim() == (3 if self.latent else 5) else None

    @property
    def layerwise_max_tokens(self) -> int:
        """the largest chunk a layer-major retrieve or a layer-wise store takes: raw blobs have no group limit"""
        return sys.maxsize

    def begin_layerwise_store(self, view, tok_begin: int, chunk_size: int,
                              budget: Optional[int] = None) -> RawLayerwiseStore:
        """A layer-wise store of tokens [tok_begin, T) of `view`, whose KV may not be written yet (RawLayerwiseStore);
        put_kv_chunks(..., encoded=it) publishes its blobs after finish().  `budget` is ignored: raw blobs need no
        encode arena."""
        return RawLayerwiseStore(self, view, tok_begin, chunk_size)

    def put_kv_chunks(self, keys, view, tok_begin: int, chunk_size: int, blocking: bool = True,
                      encoded: Optional[RawLayerwiseStore] = None) -> int:
        """Store tokens [tok_begin, T) of `view` as len(keys) chunk blobs: ONE gather kernel (b200kv_pack_chunks)
        builds every chunk blob; for the host tier ONE device->host DMA moves them all into a page-locked slab.
        encoded: a finished layer-wise store of these chunks (store_layerwise), whose blobs are published instead: the
        host tier's entries complete with its last copy, which nothing waits for here unless `blocking`."""
        if encoded is not None:
            vals = encoded.blobs()
            assert len(vals) == len(keys)
            if encoded.host is not None:
                vals = [_HostEntry(v, encoded.done, None) for v in vals]
                if blocking:
                    encoded.done.synchronize()
                    for v in vals:
                        v.event = None
            with self.update_lock:
                for key, v in zip(keys, vals):
                    self.dict[key] = v
            return len(vals)
        with torch.cuda.device(view.device):
            dev, vals = view.pack_chunks(tok_begin, chunk_size)
            assert len(vals) == len(keys)
            if self.device != "cuda":
                host = torch.empty(dev.numel(), dtype=dev.dtype, pin_memory=True)
                side = self._side_stream(view.device)
                side.wait_stream(torch.cuda.current_stream())
                _copy_async(host, dev, side)
                ev = torch.cuda.Event()
                ev.record(side)
                # each host chunk sits at its device chunk's offset
                vals = [_HostEntry(host.as_strided(c.shape, c.stride(), c.storage_offset()), ev, dev) for c in vals]
                if blocking:
                    ev.synchronize()
                    for v in vals:
                        v.event, v.src = None, None
        with self.update_lock:
            for key, v in zip(keys, vals):
                self.dict[key] = v
        return len(vals)

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
                if src.dim() != blob.dim():
                    break                                   # a chunk of the other kind (latent / (K, V)): a miss
                t = src.shape[KvView.token_dim(dst.fmt, dst.latent)]
                tok = dst_tok0 + i * chunk_size
                if tok + t > dst.ntokens or src.dtype != blob.dtype:
                    break
                es = blob.element_size()
                if dst.latent:  # rows = l: t*D contiguous elements each
                    rows, row_bytes = blob.shape[0], t * blob.shape[2] * es
                    dst_pitch = blob.shape[1] * blob.shape[2] * es
                    dptr = blob.data_ptr() + tok * blob.shape[2] * es
                elif fmt_hf:    # rows = (l, kv, h): t*D contiguous elements each
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
                if src.dim() != (3 if dst.latent else 5):
                    break                                   # a chunk of the other kind (latent / (K, V)): a miss
                t = src.shape[KvView.token_dim(dst.fmt, dst.latent)]
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

    def get_kv_layerwise(self, keys, dst, dst_tok0: int, chunk_size: int):
        """get_kv_into in layer-major order: the hits (the rules of _get_kv_scatter) are known when this returns, with a
        pipeline.LayerwiseUpload whose ready(l) is the event after layer l of every hit chunk is in `dst`.  Per layer,
        one b200kv_unpack_chunks_layers over every hit chunk on the tier's mover stream: from the stored device blobs
        (cuda tier), or (cpu tier) from a device slot of a LAYER_SLOTS ring that one batched copy on the copy stream
        has filled with the layer's slice of every chunk, so that layer l + 1's copy runs while layer l is unpacked.
        Everything is enqueued before this returns; the host never waits."""
        return self.get_kv_layerwise_runs([(keys, None, dst_tok0)], dst, chunk_size)[1]

    def get_kv_layerwise_runs(self, runs, dst, chunk_size: int, rotation=None):
        """get_kv_layerwise of several runs in one upload: each run is (keys, fallback keys or None, destination token
        of its chunk 0), and takes its keys up to the first miss, then its fallback keys from that index on
        (pipeline.match_runs).  Each layer is unpacked for every hit chunk of every run before the next layer.
        `rotation` (rope.Rotation): each layer of every chunk is unpacked with its keys turned by its run's table row in
        one b200kv_unpack_chunks_layers_rope launch, on the mover stream, before layer l's ready event.  Returns ([(key hits, fallback hits)] per
        run, LayerwiseUpload)."""
        from lmcache_b200.pipeline import LayerwiseUpload, _batch_copy, match_runs
        t0 = time.perf_counter()
        L = dst.L

        def fits(val, tok: int) -> bool:
            src = val.host if isinstance(val, _HostEntry) else val
            if src.dim() != (3 if dst.latent else 5):
                return False                                # a chunk of the other kind (latent / (K, V)): a miss
            t = src.shape[KvView.token_dim(dst.fmt, dst.latent)]
            if tok + t > dst.ntokens or src.dtype != dst.dtype:
                return False
            # another geometry: its slices are not this KV's layers
            return src.numel() == dst.planes * dst.H * dst.D * t
        per_run = match_runs([(map(self.dict.get, keys), None if fb is None else (lambda i, fb=fb: map(self.dict.get, fb[i:])),
                               tok0) for keys, fb, tok0 in runs], chunk_size, fits)
        hit_counts = [(own, len(got) - own) for got, own in per_run]
        hits = []                                            # (stored value, source blob, tokens)
        placed = []                                          # (run, destination token, tokens)
        mover_runs = []                                      # (chunk_runs entry over the call's chunks, token of its first)
        for k, (got, _) in enumerate(per_run):
            base = len(hits)
            for val, tok in got:
                src = val.host if isinstance(val, _HostEntry) else val
                t = src.shape[KvView.token_dim(dst.fmt, dst.latent)]
                hits.append((val, src, t))
                placed.append((k, tok, t))
            if got:
                for a, b, ct, lt in chunk_runs([h[2] for h in hits[base:]], chunk_size):
                    mover_runs.append(((base + a, base + b, ct, lt), got[a][1]))
        n = len(hits)
        with torch.cuda.device(dst.device):
            srcs = []
            for val, src, _ in hits:
                if isinstance(val, _HostEntry):
                    if not src.is_contiguous():
                        src = src.contiguous().pin_memory()
                elif not src.is_cuda or not src.is_contiguous():
                    src = src.contiguous().to(dst.device)        # on the current stream, before `start`
                srcs.append(src)
            fused = None            # with a rotation: one fused unpack-and-turn launch per layer over every chunk
            if rotation is not None and n:
                from lmcache_b200.rope import chunk_arrays
                fused = tuple(torch.from_numpy(a).to(dst.device, non_blocking=True)
                              for a in chunk_arrays(placed, rotation.run_rows))
            start = torch.cuda.Event()
            start.record(torch.cuda.current_stream())
            if n == 0:
                return hit_counts, LayerwiseUpload.completed(0, L, start)
            ms, cs = self._layer_streams(dst.device)
            if fused is not None:
                for a in fused:
                    a.record_stream(ms)
                rotation.table.record_stream(ms)
            ms.wait_event(start)
            cs.wait_event(start)
            for val, _, _ in hits:
                if isinstance(val, _HostEntry) and val.event is not None:
                    cs.wait_event(val.event)                # a store's copy into the block is still queued
            dst.record_stream(ms)
            tokens = [t for _, _, t in hits]
            row = layer_row_bytes(dst.H, dst.D, dst.dtype.itemsize, dst.latent)
            bases = np.array([s.data_ptr() for s in srcs], dtype=np.uint64)
            host = self.device != "cuda"
            if host:
                slot_bytes = sum(tokens) * row
                with torch.cuda.stream(ms):
                    staging = torch.empty(LAYER_SLOTS * slot_bytes, dtype=torch.uint8, device=dst.device)
                staging.record_stream(cs)
                offs = packed_offsets(tokens, row)
                rows = np.stack([np.uint64(staging.data_ptr() + r * slot_bytes) + offs for r in range(LAYER_SLOTS)])
                sizes = np.ascontiguousarray(np.asarray(tokens, dtype=np.int64) * row)
            else:
                for s in srcs:
                    s.record_stream(ms)
                rows = np.stack([layer_table(bases, tokens, row, l) for l in range(L)])
            table = _device_table(rows, dst.device, ms)
            upload = LayerwiseUpload(n, L)
            copied = None
            t1 = time.perf_counter()
            upload.enqueue_s.append(t1 - t0)
            upload.wait_s.append(0.0)
            for layer in range(L):
                if host:
                    slot = layer % LAYER_SLOTS
                    if layer >= LAYER_SLOTS:
                        cs.wait_event(upload._ready[layer - LAYER_SLOTS])   # the slot's previous layer is unpacked
                    dsts = np.ascontiguousarray(rows[slot])
                    hsrc = layer_table(bases, tokens, row, layer)
                    _batch_copy(dsts, hsrc, sizes, cs)
                    copied = torch.cuda.Event()
                    copied.record(cs)
                    ms.wait_event(copied)
                    tp = table[slot].data_ptr()
                else:
                    tp = table[layer].data_ptr()
                if fused is not None:
                    from lmcache_b200.rope import unpack_rope_layers
                    unpack_rope_layers(dst, tp, fused, max(tokens), layer, layer + 1, rotation, ms)
                else:
                    for run, tok in mover_runs:
                        _mover_layers(False, dst, tp, tok, run, layer, ms)
                ev = torch.cuda.Event(enable_timing=True)     # a caller may time the layers against each other
                ev.record(ms)
                upload._publish(ev)
                t0, t1 = t1, time.perf_counter()
                upload.enqueue_s.append(t1 - t0)
                upload.wait_s.append(0.0)
            if host:
                self._keep_until(copied, srcs)
        return hit_counts, upload

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
def _copy_ptr(dst: int, src: int, nbytes: int, stream: torch.cuda.Stream) -> None:
    N.check(N.lib().b200kv_copy_async(ctypes.c_void_p(dst), ctypes.c_void_p(src), nbytes, stream.cuda_stream), "copy_async")


class _Store:
    """One put_kv_chunks call.  A bounded tier never evicts a call's entries to make room for its later chunks, nor an
    entry touched since `since` -- the latest touch on the calling thread, which for LMCacheEngine is the prefix its
    skip_existing scan matched: evicting that prefix would make the chunks being stored unreachable.  Once one of its
    containers does not fit, the rest are dropped as well: behind a gap they could never be hit.  The device level
    likewise never evicts the call's own copies, stamps them all with one tick (`dtick`) in chain order, and once one
    of its chunks is not cached it caches none of the later ones (`dgap`): what the level holds of the call is a prefix."""
    __slots__ = ("dropped", "since", "dtick", "dgap")

    def __init__(self, since: Optional[int] = None):
        self.dropped = False
        self.since = since
        self.dtick: Optional[int] = None
        self.dgap = False


def _miss_beyond(entries, batch) -> None:
    """A layer-wise store's batch holds the prefix of its chunks that fit the device arena: the rest are misses."""
    for e in entries[len(batch.sizes):]:
        if e.error is None:
            e.error = MemoryError("chunk did not fit the layer-wise store's device arena (LMCACHE_B200_LAYERWISE_STORE_MB)")


class _CEntry:
    """One stored chunk: its container's record (pipeline.HostContainer) plus the tier's bookkeeping."""
    __slots__ = ("rec", "path", "ready", "error", "store", "pins", "retired")

    def __init__(self, store: Optional[_Store] = None):
        self.rec = None                      # None until the container has landed (and again once it is retired)
        self.path = None                     # disk tier: the container's file (then rec.blk is None)
        self.ready = threading.Event()       # set by the store worker once the container is in host memory
        self.error: Optional[BaseException] = None
        self.store = store                   # the put_kv_chunks call that made it (None: found on disk at start-up)
        self.pins = 0                        # retrieves between lookup and upload: the block is neither evicted nor freed
        self.retired = False                 # retired while pinned: the last unpin hands the block to DeferredFree

    # read by reports (bench.py's e2e counts the container bytes a retrieve uploads)
    @property
    def blk(self):
        return None if self.rec is None else self.rec.blk

    @property
    def nbytes(self) -> int:
        return 0 if self.rec is None else self.rec.nbytes


class _Level:
    """pipeline.DeviceLevel of one retrieve: chunk i of the call is entries[i], pinned by the retrieve"""

    def __init__(self, tier: "LMCLocalCompressedBackend", entries: list, device):
        self.tier, self.entries, self.cache = tier, entries, tier._dcache
        self.device = torch.device(device)

    def resident(self, r) -> bool:
        return r.dev is not None and self.cache.serves(self.device)

    def promote(self, i: int, r, src_ptr: int, stream: torch.cuda.Stream) -> bool:
        return self.tier._promote(self.entries[i], r, src_ptr, stream)

    def hit(self, n: int) -> None:
        with self.tier.update_lock:
            self.cache.hits += n

    def mark_read(self, recs, stream: torch.cuda.Stream) -> None:
        from lmcache_b200.pipeline import mark_dev_read
        with self.tier.update_lock:
            mark_dev_read(recs, stream)


class LMCLocalCompressedBackend(LMCBackendInterface):
    """local_device="cpu" + local_serde="cachegen": the host tier keeps CacheGen containers instead of raw blobs.

    Replaces LMCLocalBackend("cpu") (lmcache/storage_backend/local_backend.py:28-153) for BASELINE configs[2]: the
    bytes crossing PCIe and sitting in host memory shrink by the codec's ratio (5.9x on the SURVEY 8d data), and both
    directions are pipelined (lmcache_b200/pipeline.py):
      store     waves of chunks are encoded on the caller's stream (enqueue only) while a worker thread moves the
                previous wave's containers -- exactly their bytes -- into the page-locked slab on a copy stream;
      retrieve  the containers of wave i+1 are uploaded on a copy stream while wave i is decoded straight into the
                destination; slot reuse is ordered by events, the host never waits.
    Every container lives in one PinnedSlab (one cudaHostAlloc per GiB, not one per put).

    With config.local_capacity_bytes the slab never holds more than that many bytes: the store worker evicts chunks in
    the order of lmcache_b200.eviction.PrefixLRU before it lands a wave, and drops what does not fit even then.

    With config.device_cache_bytes the tier has a device level (lmcache_b200/device_cache.py): containers are copied
    into one device pool as they land and as retrieves upload them, and a retrieve decodes the resident ones in place
    (pipeline.DeviceLevel).  The level is inclusive -- a device copy leaves with its entry -- and filling it never
    waits: what does not find room at once is not cached.

    With config.local_serde="lossless" the containers are lossless ones (versions 5 and 6, codec.LosslessCodec), with
    every feature above: a retrieve gives back the stored bits in the stored dtype, and a chunk whose dtype or kind
    differs from the destination's is a miss."""

    lossless = False                          # the tier keeps lossless containers (set from config.local_serde)

    def __init__(self, config: LMCacheEngineConfig, metadata):
        super().__init__()
        from lmcache_b200.codec import LosslessCodec, engine_codec
        from lmcache_b200.eviction import PrefixLRU
        from lmcache_b200.pipeline import DeferredFree, EncodePipeline, UploadRing
        N.require_cuda()
        self.chunk_size = config.chunk_size
        self.fmt = metadata.fmt
        if self.fmt not in ("vllm", "huggingface"):
            raise ValueError(f"Invalid format: {self.fmt}")
        # the engine's KV is latent (metadata.use_mla): its containers are version 4, and only those are its chunks
        self.latent = bool(getattr(metadata, "use_mla", False))
        # ValueError for models outside the bin table (without config.cachegen_config), and for settings that
        # config.cachegen_config rules out.  local_serde="lossless": lossless containers, in the stored dtype
        self.lossless = config.local_serde == "lossless"
        self.codec = LosslessCodec() if self.lossless else engine_codec(config, metadata.model_name)
        self.capacity: Optional[int] = config.local_capacity_bytes
        self.slab = self._new_slab()
        self._order = PrefixLRU()             # eviction order of a bounded tier, keyed like self.dict
        self._touched = threading.local()     # .tick: the order's tick after this thread's latest touch
        self.evicted = 0                      # chunks evicted so far (reports)
        self.dict: Dict[CacheEngineKey, _CEntry] = {}
        self.update_lock = threading.Lock()
        self._pipe = EncodePipeline(self.codec, self._sink)
        self._upload: Optional[UploadRing] = None
        self._layerwise = None                # pipeline.LayerwiseUploader, made by the first layer-wise retrieve
        self._segments = None                 # pipeline.SegmentPool, made by the first layer-wise store
        self._release = DeferredFree()        # blocks uploads may still read: retired entries, the disk tier's file reads
        self._dcache = None                   # device_cache.DeviceCache: the device level (config.device_cache_bytes)
        if config.device_cache_bytes is not None:
            from lmcache_b200.device_cache import DeviceCache
            self._dcache = DeviceCache(config.device_cache_bytes)
        self._closed = False

    def _new_slab(self):
        """bounded: segments of min(LMCACHE_B200_SLAB_SEGMENT_MB, capacity), at most ceil(capacity / segment) of them"""
        from lmcache_b200.slab import PinnedSlab, _default_segment_bytes
        if self.capacity is None:
            return PinnedSlab()
        seg = min(_default_segment_bytes(), self.capacity)
        return PinnedSlab(seg, max_segments=-(-self.capacity // seg))

    # ------------------------------------------------------------------ store
    def _sink(self, slot, batch, c0, entries) -> None:
        """store pipeline sink: land the wave in host memory, then publish the entries (readers wait on `ready`)"""
        from lmcache_b200.pipeline import land
        dblocks = None
        try:
            blocks = None if self.capacity is None else self._make_room(batch.sizes, entries)
            if self._dcache is None:
                recs = land(self.slab, slot, batch, blocks, codec=self.codec) if blocks is None or blocks else []
            else:
                dblocks = self._fill_blocks(batch.sizes[:len(batch.sizes) if blocks is None else len(blocks)], slot,
                                            entries[0].store)
                recs = land(self.slab, slot, batch, blocks, self._fill_ptrs(dblocks), self.codec) if dblocks else []
            for e, rec in zip(entries, recs):
                e.rec = rec
            if dblocks:
                with self.update_lock:
                    self._dcache.attach(entries, dblocks, at=self._fill_stamp(entries[0].store, c0))  # landed with the wave
                dblocks = None
            _miss_beyond(entries, batch)
        except BaseException as err:     # noqa: BLE001 -- the entries become misses; the job reports the error
            for e in entries:
                e.error = err
            raise
        finally:
            for blk in dblocks or ():
                if blk is not None:
                    blk.free()
            for e in entries:
                e.ready.set()

    def _make_room(self, sizes, entries) -> list:
        """Bounded tier, on the store worker: a slab block for each container of the wave, in chunk order, while the
        slab's bytes in use stay within the capacity; chunks are evicted until each one fits.  The first container that
        does not fit even then is dropped with every later chunk of its store: their entries become misses."""
        from lmcache_b200.slab import SlabFull, block_bytes
        store = entries[0].store
        blocks = []
        for size in sizes:
            blk = None
            while not store.dropped:
                if self.slab.bytes_in_use + block_bytes(size) <= self.capacity:
                    try:
                        blk = self.slab.alloc(size)
                        break
                    except SlabFull:             # first-fit fragmentation: free more, never open another segment
                        pass
                if self._release.pending():
                    self._release.sweep(wait=True)    # victims an upload may still read: wait here, off the caller's thread
                elif not self._evict_one(store):
                    store.dropped = True
            if blk is None:
                break
            blocks.append(blk)
        for e in entries[len(blocks):]:
            e.error = MemoryError(f"chunk does not fit within local_capacity_bytes={self.capacity}")
        return blocks

    def _evictable(self, k, store: Optional[_Store]) -> bool:
        e = self.dict.get(k)
        if e is None:
            return True
        if not e.ready.is_set() or e.pins:
            return False
        return store is None or (e.store is not store and (store.since is None or self._order.stamp(k)[0] < store.since))

    def _evict_one(self, store: Optional[_Store]) -> bool:
        """Evict the eligible entry with the smallest stamp (never one of `store`'s, a pinned one or one that has not
        landed).  False: there is none."""
        with self.update_lock:
            k = self._order.victim(lambda k: self._evictable(k, store))
            if k is None:
                return False
            self._order.discard(k)
            e = self.dict.pop(k, None)
            if e is not None:
                self.evicted += 1
        if e is not None:
            self._drop(e)
        return True

    def _drop(self, e: _CEntry) -> None:
        """an evicted entry's bytes leave the tier"""
        self._retire(e)

    def _retire(self, e: _CEntry) -> None:
        with self.update_lock:
            if e.pins:
                e.retired = True                 # a retrieve still holds it: the last unpin frees the block
                return
            if self._dcache is not None:
                e.retired = True                 # a promotion must not fill it any more
            rec = self._detach(e)
        self._free_rec(rec)

    def _detach(self, e: _CEntry):
        """under the lock: the record whose bytes retiring `e` frees (and its device copy leaves the level)"""
        rec, e.rec = e.rec, None
        if rec is not None and self._dcache is not None:
            self._dcache.order.discard(e)
            self._dcache.detach(rec)
        return rec

    def _free_rec(self, rec) -> None:
        if rec is not None and rec.blk is not None:
            self._release.add(rec.last_read, [rec.blk])

    def touch(self, keys) -> None:
        """Recency update of one call: `keys` in chain order, chunk 0 first (LMCacheEngine passes every key of a stored
        sequence and every key of a retrieved prefix, lmcache_b200/eviction.py).  Keys the tier does not hold are
        skipped.  The device level's order gets the same call, over the entries it holds.  No-op on an unbounded tier
        without a device level."""
        if self.capacity is None and self._dcache is None:
            return
        dks = [self._dict_key(k) for k in keys]
        with self.update_lock:
            if self.capacity is not None:
                self._order.touch([k for k in dks if k in self.dict])
                self._touched.tick = self._order.tick
            if self._dcache is not None:
                self._dcache.touch([self.dict.get(k) for k in dks])

    def _new_store(self) -> _Store:
        return _Store(getattr(self._touched, "tick", None) if self.capacity is not None else None)

    def _submit(self, view, tok_begin: int, chunk_size: int, entries, encoded, shared=None):
        return self._pipe.submit(view, tok_begin, chunk_size, entries, shared=shared) if encoded is None else \
            self._pipe.submit_encoded(encoded, entries)

    def put_kv_chunks(self, keys, view, tok_begin: int, chunk_size: int, blocking: bool = True, encoded=None,
                      shared=None) -> int:
        # `keys` may be lazy (the engine's hash chain produces key i after keys 0..i-1): the encode waves
        # need no keys, so they are enqueued first; the entries are published as their keys arrive.  Readers wait on `ready`.
        # encoded: a finished pipeline.LayerwiseEncode of these chunks (store_layerwise), landed instead of encoding `view`
        # shared: a pipeline.SharedWaves whose pipeline lands every encoded wave as well (LMCHybridBackend)
        store = self._new_store()
        entries = [_CEntry(store) for _ in range(len(keys))]
        job = self._submit(view, tok_begin, chunk_size, entries, encoded, shared)
        old = []
        for k, e in zip(keys, entries):
            with self.update_lock:
                prev = self.dict.get(k)
                if prev is not None:
                    old.append(prev)
                self.dict[k] = e
        self.touch(keys)                            # one call, positions relative to tok_begin; the engine's touch follows
        for prev in old:                            # an overwritten container leaves once nobody reads it any more
            prev.ready.wait()
            self._retire(prev)
        self._release.sweep()
        if blocking:
            job.wait()
        return len(keys)

    @_lmcache_nvtx_annotate
    def put(self, key: CacheEngineKey, kv_chunk: torch.Tensor, blocking: bool = True) -> None:
        if not kv_chunk.is_cuda:
            kv_chunk = kv_chunk.cuda()              # reference: tensor.cuda() in the serializer (cachegen_encoder.py:383)
        view = KvView.from_blob(kv_chunk, self.fmt)
        self.put_kv_chunks([key], view, 0, view.ntokens, blocking=blocking)

    # ------------------------------------------------------------------ lookup
    def _dict_key(self, key: CacheEngineKey):
        return key

    def _lookup(self, key: CacheEngineKey) -> Optional[_CEntry]:
        return self.dict.get(self._dict_key(key))

    def contains(self, key: CacheEngineKey) -> bool:
        e = self._lookup(key)
        return e is not None and not (e.ready.is_set() and e.error is not None)

    def _ready_entry(self, key) -> Optional[_CEntry]:
        e = self._lookup(key)
        if e is None:
            return None
        e.ready.wait()
        return None if e.error is not None or e.rec is None else e

    def peek_geometry(self, key, fmt: str = "vllm"):
        """(L, H, D, output dtype) of the stored chunks, read from a container header (no decode).  None for a container
        of the other kind (version 4 for a (K, V) engine, or the reverse)."""
        e = self._ready_entry(key)
        if e is None or bool(e.rec.coder & N.KV_LATENT) != self.latent:
            return None
        return e.rec.L, e.rec.H, e.rec.D, self._dtype_of(e.rec)

    def out_dtype(self) -> Optional[torch.dtype]:
        """The dtype a retrieve decodes into: by format for CacheGen containers (the reference's decoder casts by format,
        ignoring metadata.dtype, cachegen_decoder.py:189-200); None for lossless ones, which decode into the dtype they
        were stored in (peek_geometry says which)."""
        if self.lossless:
            return None
        return torch.bfloat16 if self.fmt == "vllm" else torch.float16

    def _dtype_of(self, rec) -> torch.dtype:
        from lmcache_b200.codec import dtype_of_code
        return self.out_dtype() or dtype_of_code(rec.max_dtype)

    @property
    def layerwise_store_blocking(self) -> bool:
        """Does a layer-wise store's finish() return only once its containers have landed?  Not on a host tier: nothing
        outside the tier sees an entry before it lands, and a retrieve of its keys waits for it."""
        return False

    @property
    def layerwise_max_tokens(self) -> int:
        """the largest chunk a layer-major retrieve or a layer-wise store takes: one group per container"""
        return self.codec.layerwise_max_tokens

    # ------------------------------------------------------------------ retrieve
    def supports_kv_view(self) -> bool:
        return True

    def get_kv_into(self, keys, dst, dst_tok0: int, chunk_size: int) -> int:
        """Upload + decode consecutive chunks (until the first miss) straight into `dst`; chunk i lands at token
        dst_tok0 + i * chunk_size.  Everything is enqueued: copies on the copy stream, decodes on the current stream."""
        from lmcache_b200.pipeline import upload_decode
        # keys may be lazy (the hash chain is still running): every full wave is uploaded and decoded as soon as its
        # keys exist, while the chain works on the later chunks.  The records were checked when they landed.
        pinned = []
        try:
            return upload_decode(self.codec, self._upload_ring(dst.device), self._pinned_records(keys, pinned), dst,
                                 dst_tok0, chunk_size, level=self._level(dst.device, pinned))
        finally:
            self._unpin(pinned)             # every wave's upload event is recorded in its records' last_read by now

    def get_kv_layerwise(self, keys, dst, dst_tok0: int, chunk_size: int):
        """get_kv_into in layer-major order (pipeline.upload_decode_layerwise): returns once the hit count is known, with
        a pipeline.LayerwiseUpload whose ready(l) is the event after layer l's decode.  The entries stay pinned until
        the last copy is enqueued."""
        from lmcache_b200.pipeline import upload_decode_layerwise
        pinned = []
        return upload_decode_layerwise(self.codec, self._layerwise_uploader(dst.device), self._pinned_records(keys, pinned),
                                       dst, dst_tok0, chunk_size, on_done=lambda: self._unpin(pinned),
                                       level=self._level(dst.device, pinned))

    def get_kv_layerwise_runs(self, runs, dst, chunk_size: int, rotation=None):
        """get_kv_layerwise of several runs in one upload (pipeline.upload_decode_layerwise_runs): each run is (keys,
        fallback keys or None, destination token of its chunk 0); a run takes its keys up to the first miss, then its
        fallback keys from that index on.  `rotation` (rope.Rotation) turns the keys of the chunks written, layer by
        layer.  Returns ([(key hits, fallback hits)] per run, LayerwiseUpload).  The device level is neither read nor
        filled here (its chunks are decoded from their host copies, which an inclusive level keeps)."""
        from lmcache_b200.pipeline import upload_decode_layerwise_runs
        pinned = []
        recs = [(self._pinned_records(keys, pinned),
                 None if fb is None else (lambda i, fb=fb: self._pinned_records(fb[i:], pinned)), tok0)
                for keys, fb, tok0 in runs]
        return upload_decode_layerwise_runs(self.codec, self._layerwise_uploader(dst.device), recs, dst, chunk_size,
                                            on_done=lambda: self._unpin(pinned), rotation=rotation)

    def begin_layerwise_store(self, view, tok_begin: int, chunk_size: int, budget: Optional[int] = None):
        """A pipeline.LayerwiseEncode of tokens [tok_begin, T) of `view` (whose KV may not be written yet), or None
        when this tier's containers for `chunk_size` are not ones a layer-wise encode writes: versions 3 and 4 (CacheGen,
        chunks of at most 256 tokens), versions 5 and 6 (lossless, at most 4096).  `budget`: the cap of its arena
        (default LMCACHE_B200_LAYERWISE_STORE_MB)."""
        from lmcache_b200.pipeline import LayerwiseEncode, layerwise_encodes, segment_pool_for
        if not layerwise_encodes(self.codec, chunk_size, view.latent):
            return None
        self._segments = segment_pool_for(self._segments, view.device)
        return LayerwiseEncode(self.codec, self._segments, view, tok_begin, chunk_size, budget)

    def _layerwise_uploader(self, device):
        from lmcache_b200.pipeline import LayerwiseUploader
        if self._layerwise is None or self._layerwise.device != device:
            if self._layerwise is not None:
                self._layerwise.close()
            self._layerwise = LayerwiseUploader(device)
        return self._layerwise

    def _pinned_records(self, keys, pinned: list):
        """the records of `keys` in order (None: a miss), each entry pinned from its lookup on: neither eviction nor an
        overwrite frees its block before the upload that reads it is enqueued and recorded"""
        for key in keys:
            dk = self._dict_key(key)
            with self.update_lock:
                e = self.dict.get(dk)
                if e is not None:
                    e.pins += 1
                    pinned.append(e)
            if e is None:
                yield None
                return
            e.ready.wait()
            yield None if e.error is not None else e.rec

    def _unpin(self, pinned: list) -> None:
        free = []
        with self.update_lock:
            for e in pinned:
                e.pins -= 1
                if e.pins == 0 and e.retired and e.rec is not None:
                    free.append(self._detach(e))
        for rec in free:
            self._free_rec(rec)

    # ------------------------------------------------------------------ device level
    def _level(self, device, entries: list):
        """the pipeline's view of the device level for one retrieve into `device`, whose chunk i is entries[i] (an
        entry pinned from its lookup on), or None without a level"""
        return None if self._dcache is None else _Level(self, entries, device)

    def _fill_stamp(self, store: _Store, c0: int):
        """under the lock: (tick, chain position) of the store's copies from chunk c0 on -- one tick per store"""
        if store.dtick is None:
            store.dtick = self._dcache.order.new_tick()
        return store.dtick, c0

    def _fill_blocks(self, sizes, slot, store: _Store) -> list:
        """store worker: a device block for each landing container, or None where it is not cached.  The store's own
        copies are never evicted for its later chunks: a sequence larger than the level keeps its head resident."""
        from lmcache_b200.pipeline import SegmentSlot
        device = (slot.arena if isinstance(slot, SegmentSlot) else slot.dev).device
        c = self._dcache
        with self.update_lock, torch.cuda.device(device):
            if c.pool is not None and not c.serves(device):
                return [None] * len(sizes)
            out = []
            for size in sizes:
                blk = None if store.dgap else c.alloc(size, keep=lambda h: h.store is store)
                if blk is None:
                    c.skipped += store.dgap          # alloc counted the first one
                    store.dgap = True
                out.append(blk)
            return out

    def _fill_ptrs(self, dblocks) -> list:
        base = self._dcache.pool.dev_ptr if any(b is not None for b in dblocks) else 0
        return [None if b is None else base + b.offset for b in dblocks]

    def _promote(self, e: _CEntry, r, src_ptr: int, stream: torch.cuda.Stream) -> bool:
        """a retrieve uploaded `r` (entry e's container) to src_ptr: copy it into the level on `stream` when a block is
        free without waiting.  True: the copy is enqueued."""
        c = self._dcache
        with self.update_lock:
            if e.retired or e.rec is None or e.rec.dev is not None or e.rec.nbytes != r.nbytes:
                return False
            if c.pool is not None and not c.serves(stream.device):
                return False
            with torch.cuda.device(stream.device):
                blk = c.alloc(r.nbytes)
                if blk is None:
                    return False
                try:
                    _copy_ptr(c.pool.dev_ptr + blk.offset, src_ptr, r.nbytes, stream)
                except BaseException:
                    blk.free()
                    raise
                ev = torch.cuda.Event()
                ev.record(stream)
            c.attach([e], [blk], ev)
            c.promotions += 1
        return True

    def reserve_device(self) -> None:
        """Make the device level's pool now, on the current device (the first store makes it otherwise).  No-op without
        a level."""
        if self._dcache is not None:
            with self.update_lock:
                self._dcache.reserve()

    def device_cache_stats(self) -> Optional[dict]:
        """bytes_in_use, budget_bytes, hits, promotions, evictions, not_cached (chunks that found no room without
        waiting) of the device level; None without one"""
        if self._dcache is None:
            return None
        with self.update_lock:
            return self._dcache.stats()

    def _upload_ring(self, device):
        from lmcache_b200.pipeline import UploadRing
        if self._upload is None or self._upload.device != device:
            self._upload = UploadRing(device)
        return self._upload

    @_lmcache_nvtx_annotate
    def get(self, key: CacheEngineKey) -> Optional[torch.Tensor]:
        e = self._ready_entry(key)
        if e is None:
            return None
        r = e.rec
        out = torch.empty(KvView.blob_shape(self.fmt, r.L, r.H, r.D, r.ntokens, bool(r.coder & N.KV_LATENT)),
                          dtype=self._dtype_of(r),
                          device=torch.device("cuda", torch.cuda.current_device()))
        if self.get_kv_into([key], KvView.from_blob(out, self.fmt), 0, r.ntokens) != 1:
            return None
        self.touch([key])
        return out

    def reserve_host(self, nbytes: int) -> None:
        """Page-lock at least nbytes of slab up front (a cudaHostAlloc of 1 GiB takes ~0.3 s: better at start-up than
        inside a store).  A bounded tier reserves at most its capacity."""
        self.slab.reserve(int(nbytes) if self.capacity is None else min(int(nbytes), self.capacity))

    def host_bytes(self) -> int:
        """bytes of containers currently held (for reports)"""
        return self.slab.stats()[2]

    def close(self):
        if self._closed:
            return
        self._closed = True
        self._pipe.close()
        if self._segments is not None:
            self._segments.close()
        if self._layerwise is not None:
            self._layerwise.close()
        try:
            torch.cuda.synchronize()
        except Exception:       # noqa: BLE001 -- interpreter shutdown
            pass
        self.slab.close()
        if self._dcache is not None:
            self._dcache.close()

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
        earlier waves upload and decode (disk || H2D || decode, lmcache_b200/pipeline.py upload_decode);
      * with config.local_capacity_bytes the .b2kv files total at most that many bytes: the store worker removes files in
        the order of lmcache_b200.eviction.PrefixLRU before it writes one.  A reader that loses the race to a removal gets
        an OSError or a short read, which is a miss.  At start-up the order is seeded oldest file (mtime) first, and a
        directory over the capacity is evicted down to it; the prefix guarantee holds within one process only."""

    SUFFIX = ".b2kv"

    def __init__(self, config: LMCacheEngineConfig, metadata):
        import os
        from concurrent.futures import ThreadPoolExecutor
        path = config.local_device
        assert path is not None, "Need to specify local path if when using LMCLocalDiskBackend"
        self.path = path if path.endswith("/") else path + "/"
        os.makedirs(self.path, exist_ok=True)
        self._file_bytes: Dict[str, int] = {}        # bounded tier: size of every indexed file
        self._disk_bytes = 0                         # ... and their total
        super().__init__(config, metadata)
        self._io = ThreadPoolExecutor(max_workers=max(1, int(os.environ.get("LMCACHE_B200_DISK_THREADS", "4"))),
                                      thread_name_prefix="b200kv-disk")
        self._rebuild_index()

    def _new_slab(self):
        from lmcache_b200.slab import PinnedSlab
        return PinnedSlab()                  # transient blocks only: the capacity bounds the files

    # ---- index
    def _key_to_path(self, key: CacheEngineKey) -> str:
        return self.path + key.to_string().replace("/", "-") + self.SUFFIX      # reference naming rule (:228)

    def _rebuild_index(self) -> int:
        import os

        from lmcache_b200.codec import parse_header, parse_lossless_header
        from lmcache_b200.pipeline import HostContainer
        # the tier's own family only: a CacheGen tier indexes versions 1 to 4, a lossless one 5 and 6
        parse = parse_lossless_header if self.lossless else parse_header
        found = []
        for name in os.listdir(self.path):
            if not name.endswith(self.SUFFIX):
                continue
            full = self.path + name
            try:
                st = os.stat(full)
                size = st.st_size
                with open(full, "rb") as f:
                    hd = parse(f.read(N.HEADER_BYTES + N.MAX_PLANES), size)
                if int(hd.total_bytes) != size or bool(N.coder_of_version(hd.version) & N.KV_LATENT) != self.latent:
                    continue                     # versions 4 and 6 hold a latent KV: containers of a latent engine only
            except (OSError, ValueError):
                continue                         # damaged / foreign file (the other family's too): left as it is
            # "/" in a model name was written as "-": the key of a lookup goes through the same rule, so index by path
            e = _CEntry()
            e.path, e.rec = full, HostContainer(None, size, hd)
            e.ready.set()
            found.append((st.st_mtime_ns, full, e))
        found.sort(key=lambda f: f[:2])                  # oldest first: the eviction order of a bounded tier
        for _, full, e in found:
            self._by_path[full] = e
            if self.capacity is not None:
                self._order.touch([full])
                self._file_bytes[full] = e.rec.nbytes
                self._disk_bytes += e.rec.nbytes
        while self.capacity is not None and self._disk_bytes > self.capacity and self._evict_one(None):
            pass
        return len(self.dict)

    @property
    def layerwise_store_blocking(self) -> bool:
        """On a lossless disk tier, yes: its layer-wise store replaced a blocking store() at finish(), and the directory
        is read by other engines and by a restarted tier, so finish() keeps returning with the files in place (the
        encode still runs layer by layer on the side stream).  A CacheGen disk tier's layer-wise store lands in the
        background, as it always has."""
        return self.lossless

    # the dict is keyed by file path: CacheEngineKey -> path is many-to-one ("/" and "-"), exactly as in the reference
    @property
    def _by_path(self):
        return self.dict

    def _dict_key(self, key: CacheEngineKey) -> str:
        return self._key_to_path(key)

    def _drop(self, e: _CEntry) -> None:
        """evicted: the file goes (on the store worker, or at start-up), and its device copy with it"""
        import os
        try:
            os.remove(e.path)
        except OSError:
            pass
        self._disk_bytes -= self._file_bytes.pop(e.path, 0)
        if self._dcache is not None:
            self._retire(e)

    def _detach(self, e: _CEntry):
        """the index record stays (readers of the entry may still open its path); only the device copy leaves"""
        if e.rec is not None and self._dcache is not None:
            self._dcache.order.discard(e)
            self._dcache.detach(e.rec)
        return None

    def _make_file_room(self, e: _CEntry, nbytes: int) -> bool:
        """bounded tier: evict until the file of `e` (replacing any file at its path) fits within the capacity"""
        while not e.store.dropped:
            if self._disk_bytes - self._file_bytes.get(e.path, 0) + nbytes <= self.capacity:
                return True
            if not self._evict_one(e.store):
                e.store.dropped = True
        return False

    # ---- store: the pipeline's sink writes files instead of keeping blocks
    def _sink(self, slot, batch, c0, entries) -> None:
        import os

        from lmcache_b200.pipeline import land
        recs = []
        dblocks = None
        try:
            if self._dcache is None:
                recs = land(self.slab, slot, batch, codec=self.codec)   # containers -> page-locked blocks, headers parsed
            else:
                dblocks = self._fill_blocks(batch.sizes, slot, entries[0].store)
                recs = land(self.slab, slot, batch, None, self._fill_ptrs(dblocks), self.codec)
        except BaseException as err:     # noqa: BLE001
            for e in entries:
                e.error = err
            raise
        else:
            _miss_beyond(entries, batch)
            for j, (e, rec) in enumerate(zip(entries, recs)):
                e.rec = rec
                if self.capacity is not None and not self._make_file_room(e, rec.nbytes):
                    e.error = OSError(f"chunk does not fit within local_capacity_bytes={self.capacity}")
                    continue
                tmp = e.path + ".tmp"
                try:
                    with open(tmp, "wb") as f:
                        f.write(rec.blk.view())
                    os.replace(tmp, e.path)               # a file that exists is complete
                except OSError as err:
                    e.error = err
                    continue
                if self.capacity is not None:
                    self._disk_bytes += rec.nbytes - self._file_bytes.get(e.path, 0)
                    self._file_bytes[e.path] = rec.nbytes
                if dblocks is not None and dblocks[j] is not None:
                    with self.update_lock:                # inclusive: only beside a file that is in place
                        if not e.retired:                 # an overwrite retired it: its copy would never be served
                            self._dcache.attach([e], [dblocks[j]], at=self._fill_stamp(e.store, c0 + j))
                            dblocks[j] = None
        finally:
            for blk in dblocks or ():
                if blk is not None:
                    blk.free()
            for rec in recs:
                rec.blk.free()
                rec.blk = None
            for e in entries:
                e.ready.set()                             # readers see the entry only once its file is in place

    def put_kv_chunks(self, keys, view, tok_begin: int, chunk_size: int, blocking: bool = True, encoded=None,
                      shared=None) -> int:
        store = self._new_store()
        entries = [_CEntry(store) for _ in keys]
        for k, e in zip(keys, entries):
            e.path = self._key_to_path(k)
            e.ready.clear()
        old = []
        with self.update_lock:
            for e in entries:
                if self._dcache is not None and e.path in self.dict:
                    old.append(self.dict[e.path])
                self.dict[e.path] = e                     # an overwritten chunk's file is replaced atomically by the rename
        # the parent's sink sets `ready` before the file exists: keep readers out until the file is written
        job = self._submit(view, tok_begin, chunk_size, entries, encoded, shared)
        self.touch(keys)
        for prev in old:      # an overwritten chunk's device copy is never served again (its sink checks `retired`)
            self._retire(prev)
        if blocking:
            job.wait()
        return len(keys)

    # ---- retrieve
    def _read_file(self, e: _CEntry):
        """reader pool: the container file -> a fresh slab block -> its record, or None (a miss)"""
        from lmcache_b200.pipeline import read_container
        nbytes = e.rec.nbytes
        blk = self.slab.alloc(nbytes)
        try:
            with open(e.path, "rb", buffering=0) as f:
                got = f.readinto(blk.view())
                while got is not None and 0 < got < nbytes:
                    more = f.readinto(blk.view()[got:])
                    if not more:
                        break
                    got += more
            if got != nbytes:
                raise OSError("short read")
        except OSError:
            blk.free()
            return None
        return read_container(self.codec, blk, nbytes, self.latent)

    def _reads(self, keys, level: Optional[_Level]) -> list:
        """futures of the records of `keys` up to the first miss: file reads, or with a device level the index
        record of a resident entry (no read).  With a level every entry is pinned into level.entries."""
        from concurrent.futures import Future
        reads = []
        for key in keys:
            if level is None:
                e = self._ready_entry(key)
            else:
                rec = next(self._pinned_records([key], level.entries))
                e = level.entries[-1] if rec is not None else None
            if e is None:
                break
            if level is not None and level.resident(e.rec):
                f = Future()
                f.set_result(e.rec)
                reads.append(f)
            else:
                reads.append(self._io.submit(self._read_file, e))
        return reads

    def get_kv_into(self, keys, dst, dst_tok0: int, chunk_size: int) -> int:
        import contextlib

        from lmcache_b200.pipeline import fetched_in_order, upload_decode
        self._release.sweep()                            # transient read blocks of earlier calls
        level = self._level(dst.device, [])
        try:
            reads = self._reads(keys, level)
            with contextlib.closing(fetched_in_order(reads)) as recs:
                return upload_decode(self.codec, self._upload_ring(dst.device), recs, dst, dst_tok0, chunk_size,
                                     self._release, level)
        finally:
            if level is not None:
                self._unpin(level.entries)

    def get_kv_layerwise(self, keys, dst, dst_tok0: int, chunk_size: int):
        import contextlib

        from lmcache_b200.pipeline import fetched_in_order, upload_decode_layerwise
        self._release.sweep()
        level = self._level(dst.device, [])
        try:
            reads = self._reads(keys, level)
        except BaseException:
            if level is not None:
                self._unpin(level.entries)
            raise
        with contextlib.closing(fetched_in_order(reads)) as recs:
            return upload_decode_layerwise(self.codec, self._layerwise_uploader(dst.device), recs, dst, dst_tok0,
                                           chunk_size, self._release,
                                           on_done=None if level is None else (lambda: self._unpin(level.entries)),
                                           level=level)

    def get_kv_layerwise_runs(self, runs, dst, chunk_size: int, rotation=None):
        """LMCLocalCompressedBackend.get_kv_layerwise_runs over container files: every run's files are read on the
        reader pool (a fallback's once its run has missed), and the device level is not used."""
        import contextlib

        from lmcache_b200.pipeline import fetched_in_order, upload_decode_layerwise_runs
        self._release.sweep()
        with contextlib.ExitStack() as opened:
            def recs(keys):
                return opened.enter_context(contextlib.closing(fetched_in_order(self._reads(keys, None))))
            srcs = [(recs(keys), None if fb is None else (lambda i, fb=fb: recs(fb[i:])), tok0) for keys, fb, tok0 in runs]
            return upload_decode_layerwise_runs(self.codec, self._layerwise_uploader(dst.device), srcs, dst, chunk_size,
                                                self._release, rotation=rotation)

    def host_bytes(self) -> int:
        return sum(e.rec.nbytes for e in self.dict.values() if e.rec is not None)

    def close(self):
        self._io.shutdown(wait=True)
        super().close()              # the slab, transient read blocks included, goes after a device synchronise
