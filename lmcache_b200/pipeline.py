"""Wave pipelines between the codec and a host-side tier: encode || device->host on the way out, host->device ||
decode on the way in (SURVEY.md section 7 step 7, BASELINE configs[2]).

A store is cut into waves of a few chunks.  Each wave owns a *slot*: a device staging area for its containers and a
page-locked array for their sizes.  The caller's thread only enqueues kernels (CacheGenCodec.encode_async on the
caller's stream: the KV is consumed in stream order, nothing is synchronised) and hands the slot to a worker thread;
the worker waits for the wave's event, learns the container sizes, and hands the wave to the tier's sink, which `land`s
exactly those bytes in a page-locked slab (and keeps them, writes them to files or sends them over sockets).  While it
does, the next wave is already encoding.  Scratch is bounded by slots x wave size instead of the whole block (round 1
staged every chunk of a store at once: ~4 GB of device scratch for a 4 GiB block).

On the way in, every tier hands `upload_decode` its containers in chunk order as `HostContainer` records -- the ones it
keeps, or disk reads / GETs still in flight (`fetched_in_order`) -- and `DeferredFree` releases transient blocks once
their uploads are done.

The reference does none of this: LMCLocalBackend.put_nonblocking hands whole chunk tensors to a queue and its worker
calls tensor.to("cpu") + torch.cuda.synchronize() per chunk (lmcache/storage_backend/local_backend.py:82-117).
"""
from __future__ import annotations

import collections
import ctypes
import functools
import os
import queue
import threading
import time
from concurrent.futures import Future
from typing import Callable, Iterable, Iterator, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch

from lmcache_b200 import _native as N
from lmcache_b200.codec import CacheGenCodec, EncodedBatch, EncodeTicket, KvView, PinnedBuffer, SegmentLayout


def wave_chunks_default() -> int:
    return max(1, int(os.environ.get("LMCACHE_B200_WAVE_CHUNKS", "4")))


def wave_slots_default() -> int:
    return max(2, int(os.environ.get("LMCACHE_B200_WAVE_SLOTS", "3")))


class WaveSlot:
    """Device staging + sizes for one wave of at most `wave` chunks of one geometry."""

    def __init__(self, nbytes: int, wave: int, device):
        self.dev = torch.empty(nbytes + N.READ_SLACK, dtype=torch.uint8, device=device)
        self.sizes = PinnedBuffer(max(64, 8 * wave))
        self.planes = PinnedBuffer(8 * (N.MAX_PLANES + 1) * wave)      # b200kv_plane_offsets_device rows, one per chunk
        self.ticket: Optional[EncodeTicket] = None
        self.refs = 1                       # sinks that still land this wave (EncodeRing.hold / release)

    def close(self):
        self.sizes.close()
        self.planes.close()
        self.dev = None


class EncodeRing:
    """A fixed set of WaveSlots for one (L, H, D, chunk_size, device); acquire() blocks the calling host thread while
    every slot is still in flight -- the only back-pressure of the store pipeline."""

    def __init__(self, codec: CacheGenCodec, L: int, H: int, D: int, chunk_size: int, device, wave: Optional[int] = None,
                 slots: Optional[int] = None, latent: bool = False):
        self.codec = codec
        self.geom = (L, H, D, chunk_size, torch.device(device), latent)
        self.wave = wave or wave_chunks_default()
        self.stride = codec.out_stride(L, H, D, chunk_size, latent)
        n = slots or wave_slots_default()
        self._free: "queue.Queue[WaveSlot]" = queue.Queue()
        self._lock = threading.Lock()
        self._all: List[WaveSlot] = []
        for _ in range(n):
            s = WaveSlot(self.stride * self.wave, self.wave, device)
            self._all.append(s)
            self._free.put(s)

    def matches(self, L, H, D, chunk_size, device, latent: bool = False) -> bool:
        return self.geom == (L, H, D, chunk_size, torch.device(device), latent)

    def scratch_bytes(self) -> int:
        return sum(s.dev.numel() for s in self._all)

    def acquire(self) -> WaveSlot:
        slot = self._free.get()
        slot.refs = 1
        return slot

    def hold(self, slot: WaveSlot) -> None:
        """one more release() is needed before `slot` is free again (a wave that two sinks land)"""
        with self._lock:
            slot.refs += 1

    def release(self, slot: WaveSlot) -> None:
        with self._lock:
            slot.refs -= 1
            if slot.refs > 0:
                return
        slot.ticket = None
        self._free.put(slot)

    def drain(self) -> None:
        """Wait until every slot is back (no wave in flight)."""
        got = [self._free.get() for _ in self._all]
        for s in got:
            self._free.put(s)

    def close(self) -> None:
        self.drain()
        for s in self._all:
            s.close()
        self._all = []


class StoreJob:
    """Completion of one put_kv_chunks call: counts its waves; `wait()` blocks until the sink took all of them."""

    def __init__(self, n_waves: int):
        self._left = n_waves
        self._cv = threading.Condition()
        self.error: Optional[BaseException] = None

    def wave_done(self, err: Optional[BaseException] = None) -> None:
        with self._cv:
            if err is not None and self.error is None:
                self.error = err
            self._left -= 1
            if self._left <= 0:
                self._cv.notify_all()

    def wait(self) -> None:
        with self._cv:
            while self._left > 0:
                self._cv.wait()
        if self.error is not None:
            raise self.error


class SharedWaves:
    """The second sink of an encode that two tiers land (EncodePipeline.submit's `shared`): `pipe`, the other tier's
    EncodePipeline, whose worker hands every wave to its own sink; `items`, that sink's per-chunk payload; `job`, set by
    submit, which completes when that sink has taken every wave.  The first pipeline's worker passes each wave on to
    `pipe` once its own sink is done with it, so the first tier holds a wave's chunks before the second one does, and
    the two sinks never use the slot at the same time."""

    def __init__(self, pipe: "EncodePipeline", items: Sequence):
        self.pipe, self.items = pipe, items
        self.job: Optional[StoreJob] = None


class EncodePipeline:
    """encode waves on the caller's stream; a worker thread hands every finished wave to `sink`.

    sink(slot, batch, first_chunk, items) is called on the worker thread with the wave's EncodedBatch (sizes known,
    containers still in slot.dev) and items = the caller's per-chunk payload (keys); it must be done with slot.dev
    when it returns -- the slot is recycled right after."""

    def __init__(self, codec: CacheGenCodec, sink: Callable, name: str = "b200kv-store"):
        self.codec = codec
        self.sink = sink
        self.ring: Optional[EncodeRing] = None
        self._q: "queue.Queue" = queue.Queue()
        self._device = torch.cuda.current_device()
        self._thread = threading.Thread(target=self._worker, name=name, daemon=True)
        self._thread.start()
        self._closed = False

    # ------------------------------------------------------------------ caller side
    def _ring_for(self, view: KvView, chunk_size: int) -> EncodeRing:
        if self.ring is None or not self.ring.matches(view.L, view.H, view.D, chunk_size, view.device, view.latent):
            if self.ring is not None:
                self.ring.close()
            self.ring = EncodeRing(self.codec, view.L, view.H, view.D, chunk_size, view.device, latent=view.latent)
        return self.ring

    def submit_encoded(self, enc: "LayerwiseEncode", items: Sequence) -> StoreJob:
        """Hand a finished layer-wise encode (LayerwiseEncode.finish has been called) to the worker: it lands the
        containers that fit the arena, as one wave, in submission order with the other stores."""
        job = StoreJob(1)
        self._q.put((enc.pool, enc.slot, 0, list(items), job, None))
        return job

    def submit(self, view: KvView, tok_begin: int, chunk_size: int, items: Sequence,
               stream: Optional[torch.cuda.Stream] = None, shared: Optional["SharedWaves"] = None) -> StoreJob:
        """Enqueue the encode of tokens [tok_begin, T) of `view`, len(items) chunks, in waves.  Returns once every wave
        is enqueued on `stream` (default: the current stream); the job completes when the sink has taken them all.
        shared: another pipeline whose sink lands every wave too, from the same slot, with its own items, after this
        pipeline's sink (a hybrid tier whose parts keep the same containers); shared.job completes when that sink has
        taken them all, and a slot is free again only after both sinks."""
        n_tok = view.ntokens - tok_begin
        n_chunks = len(items)
        assert n_chunks == (n_tok + chunk_size - 1) // chunk_size and n_chunks > 0
        ring = self._ring_for(view, chunk_size)
        W = ring.wave
        job = StoreJob((n_chunks + W - 1) // W)
        if shared is not None:
            shared.job = StoreJob((n_chunks + W - 1) // W)
        with torch.cuda.device(view.device):
            for c0 in range(0, n_chunks, W):
                k = min(W, n_chunks - c0)
                t0 = tok_begin + c0 * chunk_size
                nt = min(k * chunk_size, view.ntokens - t0)
                slot = ring.acquire()
                try:
                    slot.ticket = self.codec.encode_async(view, t0, nt, chunk_size, stream, out=slot.dev, sizes=slot.sizes)
                except BaseException as e:       # noqa: BLE001 -- give the slot back, fail the job, re-raise
                    ring.release(slot)
                    job.wave_done(e)
                    if shared is not None:
                        shared.job.wave_done(e)
                    raise
                then = None
                if shared is not None:
                    ring.hold(slot)             # the second sink's reference, taken before this worker can release it
                    then = (shared.pipe, list(shared.items[c0:c0 + k]), shared.job)
                self._q.put((ring, slot, c0, list(items[c0:c0 + k]), job, then))
        return job

    # ------------------------------------------------------------------ worker side
    def _worker(self) -> None:
        torch.cuda.set_device(self._device)
        while True:
            item = self._q.get()
            if item is None:
                return
            ring, slot, c0, items, job, then = item
            err = None
            try:
                batch = slot.ticket.wait()          # host wait on this wave's kernels -- on the worker thread only
                self.sink(slot, batch, c0, items)
            except BaseException as e:              # noqa: BLE001 -- a failed background store is a miss later
                err = e
            finally:
                if then is not None:                # SharedWaves: the second sink lands the wave after this one
                    pipe, items2, job2 = then
                    pipe._q.put((ring, slot, c0, items2, job2, None))
                ring.release(slot)
                job.wave_done(err)

    def close(self) -> None:
        if self._closed:
            return
        self._closed = True
        self._q.put(None)
        self._thread.join()
        if self.ring is not None:
            self.ring.close()
            self.ring = None


class UploadRing:
    """Device staging for containers on their way in: two slots filled by host->device copies on a copy stream while the
    decoder works on the other one.  Slot reuse is ordered by events on the streams -- the host never waits."""

    def __init__(self, device):
        self.device = torch.device(device)
        self.copy_stream = torch.cuda.Stream(device=device)
        self._bufs: List[Optional[torch.Tensor]] = [None, None]
        self._busy: List[Optional[torch.cuda.Event]] = [None, None]     # decode that last read the slot
        self._i = 0

    def next_slot(self, nbytes: int):
        """(slot index, device buffer of >= nbytes + read slack); the copy stream already waits for the slot's last reader"""
        i = self._i
        self._i ^= 1
        need = nbytes + N.READ_SLACK
        if self._busy[i] is not None:
            if self._bufs[i] is None or self._bufs[i].numel() < need:
                self._busy[i].synchronize()          # growing: the old buffer must not be freed under a kernel
            else:
                self.copy_stream.wait_event(self._busy[i])
        if self._bufs[i] is None or self._bufs[i].numel() < need:
            self._bufs[i] = torch.empty(max(need, need * 5 // 4), dtype=torch.uint8, device=self.device)
        return i, self._bufs[i]

    def mark_read(self, i: int, stream: torch.cuda.Stream) -> None:
        ev = torch.cuda.Event()
        ev.record(stream)
        self._busy[i] = ev


class HostContainer:
    """One container (CacheGen, or lossless: versions 5 and 6) in a page-locked slab block, with the header fields its
    upload and decode need."""
    __slots__ = ("blk", "nbytes", "ntokens", "L", "H", "D", "max_dtype", "coder", "last_read", "planes", "dev",
                 "dev_ready", "dev_read")

    def __init__(self, blk, nbytes: int, hd: "N.Header", planes: Optional[np.ndarray] = None):
        self.blk = blk                       # None once the tier no longer keeps the bytes (the disk tier's index)
        self.nbytes = int(nbytes)
        self.ntokens = int(hd.ntokens)
        self.L, self.H, self.D = int(hd.L), int(hd.H), int(hd.D)
        self.max_dtype = int(hd.max_dtype)
        self.coder = N.coder_of_version(hd.version)          # N.CODER_LATENT for version 4 (one plane per layer)
        self.last_read: Optional[torch.cuda.Event] = None   # most recent upload out of the block
        # codec.plane_offsets: where each plane's streams lie, for a layer-major upload; None: upload it whole.  Made by
        # whoever makes the record (land, read_container), never on the thread of a retrieve.
        self.planes = planes
        # the tier's device level (lmcache_b200/device_cache.py): the container's block in the level's pool, the event
        # after which that block holds the container (None: it does), and the latest decode that read it
        self.dev = None
        self.dev_ready: Optional[torch.cuda.Event] = None
        self.dev_read: Optional[torch.cuda.Event] = None


@functools.lru_cache(maxsize=None)
def _d2h_stream(device: torch.device) -> torch.cuda.Stream:
    return torch.cuda.Stream(device=device)


def land(slab, slot: WaveSlot, batch, blocks: Optional[list] = None,
         dev_dst: Optional[Sequence[Optional[int]]] = None, codec=CacheGenCodec) -> List[HostContainer]:
    """Store-pipeline sink side: copy a finished wave's containers out of slot.dev into fresh blocks of `slab` (exactly
    their bytes, on the device's copy stream), wait for the copies, and parse every header.  Raises -- with every block
    freed -- when a copy fails or a container carries an encoder error.  `blocks`: blocks the caller allocated for the
    first len(blocks) containers (a bounded tier); only those are landed.  `dev_dst`: per container, a device address
    that gets a copy of it as well (None: none), on the same stream and before the same wait.  `codec`: the codec (or
    codec class) that wrote the wave: its header check and its plane-offset kernel (a lossless codec's for its
    containers).  A layer-wise store's slot (SegmentSlot) lands through land_segments."""
    if isinstance(slot, SegmentSlot):
        return land_segments(slab, slot, batch, blocks, dev_dst, codec)
    parse = codec.parse_header
    dev = slot.dev.device
    cs = _d2h_stream(dev)
    if blocks is None:
        blocks = [slab.alloc(size) for size in batch.sizes]
    try:
        with torch.cuda.device(dev):
            try:
                # plane offsets of the wave, read on the device before the bytes leave it: no host pass over the
                # lengths sections (on the store worker such a pass made every e2e store ~2 ms slower, measured)
                codec.plane_offsets_device(slot.dev.data_ptr(), batch.stride, len(blocks), slot.planes.dev_ptr,
                                           cs.cuda_stream)
                for j, (blk, size) in enumerate(zip(blocks, batch.sizes)):
                    N.check(N.lib().b200kv_copy_async(ctypes.c_void_p(blk.host_ptr),
                                                      ctypes.c_void_p(slot.dev.data_ptr() + j * batch.stride), size,
                                                      cs.cuda_stream), "copy_async")
                for j, (ptr, size) in enumerate(zip(dev_dst or (), batch.sizes)):
                    if ptr is not None:
                        N.check(N.lib().b200kv_copy_async(ctypes.c_void_p(ptr),
                                                          ctypes.c_void_p(slot.dev.data_ptr() + j * batch.stride), size,
                                                          cs.cuda_stream), "copy_async")
            finally:
                cs.synchronize()             # no block leaves this function while a copy may still write it
        po = np.frombuffer(slot.planes.view(), dtype=np.int64, count=len(blocks) * (N.MAX_PLANES + 1))
        po = po.reshape(len(blocks), N.MAX_PLANES + 1)
        recs = []
        for j, blk in enumerate(blocks):
            hd = parse(blk.view())
            P = N.planes_of(hd.version, hd.L)
            recs.append(HostContainer(blk, blk.nbytes, hd, po[j, :P + 1].copy() if po[j, 0] >= 0 else None))
        return recs
    except BaseException:
        for blk in blocks:
            blk.free()
        raise


def layerwise_store_budget_default() -> int:
    """LMCACHE_B200_LAYERWISE_STORE_MB: the most device arena one layer-wise store takes (default 1024 MB, about what
    the ordinary store's EncodeRing holds)."""
    return max(1, int(os.environ.get("LMCACHE_B200_LAYERWISE_STORE_MB", "1024"))) << 20


def arena_placement(seg_bytes: np.ndarray, arena_bytes: int, layers: Optional[Sequence[int]] = None):
    """Host statement of the layer-wise store's arena rule (arena_place in common.cuh, which both encoders' placement
    kernels run), for tests and sizing.  seg_bytes[c, j]: bytes of chunk j's segment in layer call c (CacheGen: the
    payload of its K planes, then its V planes; lossless: its raw part, then those streams); layers[c]: the layers
    of call c (default 1 each).  Calls are placed in order; within a call, chunk j's bytes go 16-byte aligned at the
    cursor.  Chunk j fits if, after chunks 0..j of the call, the arena still holds the layers still to come at this
    call's size per layer (a reserve, so that a later call finds room for the chunks an earlier one accepted).  A chunk
    that does not fit fails, and so does every later chunk, in this call and every later one.  Returns (base
    int64[calls, n], -1 in every call for the chunks that failed; the number of chunks that fit).
    The device's seg_sizes_out rows differ for the failed chunks: the calls before the one in which they failed had
    placed them, and their rows keep those arena offsets (the bytes stay in the arena, unused); only the rows of the
    failing call and the later ones are -1.  sizes_out is 0 for every failed chunk, so no reader looks at those rows.
    Zeroing seg_bytes of the calls after c gives the placement as it stood after call c."""
    seg_bytes = np.asarray(seg_bytes, dtype=np.int64)
    calls, n = seg_bytes.shape
    layers = list(layers) if layers is not None else [1] * calls
    base = np.full((calls, n), -1, dtype=np.int64)
    cursor, fail = 0, n
    for c in range(calls):
        left = sum(layers[c + 1:])
        start = cursor
        for j in range(min(n, fail)):
            size = (int(seg_bytes[c, j]) + 15) & ~15
            if cursor + size + (cursor + size - start) * left // layers[c] > arena_bytes:
                fail = j
                break
            base[c, j] = cursor
            cursor += size
    base[:, fail:] = -1                      # a failed chunk's earlier segments stay in the arena, unused
    return base, fail


class SegmentSlot:
    """Device scratch of one layer-wise store: the arena, the chunks' fixed-section images, the encode workspace, and in
    mapped page-locked memory the container sizes and the segment row of every (chunk, plane): `row` int64 each (the
    codec's seg_row: 2 for CacheGen, 3 for lossless).  P: planes per chunk, 2L for (K, V) pairs, L for a latent KV."""

    def __init__(self, arena_bytes: int, fixed_bytes: int, ws_bytes: int, n_chunks: int, P: int, device, row: int = 2):
        self.arena = torch.empty(max(16, arena_bytes), dtype=torch.uint8, device=device)
        self.fixed = torch.empty(max(16, fixed_bytes), dtype=torch.uint8, device=device)
        self.ws = torch.empty(max(16, ws_bytes), dtype=torch.uint8, device=device)
        self.sizes = PinnedBuffer(max(64, 8 * n_chunks))
        self.seg = PinnedBuffer(max(64, 8 * row * P * n_chunks))
        self.arena_bytes = arena_bytes
        self.ticket = None
        self.refs = 1                       # sinks that still land this slot (SegmentPool.hold / release)
        self.layouts: tuple = ()            # (SegmentLayout of a full chunk, of the last chunk)
        self.fixed_stride = 0
        self.coder = N.CODER_RANS_COMPACT   # the coder that names the containers' version (N.CODER_LATENT: 4)
        self.n_chunks, self.P, self.seg_row = 0, P, row

    def holds(self, arena_bytes: int, fixed_bytes: int, ws_bytes: int, n_chunks: int, P: int, row: int = 2) -> bool:
        return (self.arena.numel() >= arena_bytes and self.fixed.numel() >= fixed_bytes and self.ws.numel() >= ws_bytes
                and self.sizes.nbytes >= 8 * n_chunks and self.seg.nbytes >= 8 * row * P * n_chunks)

    def close(self) -> None:
        self.sizes.close()
        self.seg.close()
        self.arena = self.fixed = self.ws = None


class SegmentPool:
    """Reusable SegmentSlots for the layer-wise stores of one tier and device, and the stream they encode on.  A slot
    is reused by the next store that fits it; at most `keep` idle slots are kept.  Every kernel that touches a slot runs
    on `stream` and its tensors are allocated there, so reuse and release are ordered by the stream; the worker hands a
    slot back only after its device->host copies have completed.  A slot that several sinks land (a hybrid tier whose two
    parts keep the same containers) takes one hold() per extra sink and goes back with the last release()."""

    def __init__(self, device, keep: int = 2):
        self.device = torch.device(device)
        self.stream = torch.cuda.Stream(device=self.device)
        self.keep = keep
        self._free: List[SegmentSlot] = []
        self._lock = threading.Lock()

    def acquire(self, arena_bytes: int, fixed_bytes: int, ws_bytes: int, n_chunks: int, P: int,
                row: int = 2) -> SegmentSlot:
        with self._lock:
            for s in self._free:
                if s.holds(arena_bytes, fixed_bytes, ws_bytes, n_chunks, P, row):
                    self._free.remove(s)
                    s.refs = 1
                    return s
        with torch.cuda.device(self.device), torch.cuda.stream(self.stream):
            return SegmentSlot(arena_bytes, fixed_bytes, ws_bytes, n_chunks, P, self.device, row)

    def hold(self, slot: SegmentSlot) -> None:
        """one more release() is needed before `slot` goes back to the pool"""
        with self._lock:
            slot.refs += 1

    def release(self, slot: SegmentSlot) -> None:
        with self._lock:
            slot.refs -= 1
            if slot.refs > 0:
                return
            slot.ticket = None
            self._free.append(slot)
            drop = self._free[:-self.keep] if len(self._free) > self.keep else []
            self._free = self._free[len(drop):]
        for s in drop:
            s.close()

    def close(self) -> None:
        with self._lock:
            free, self._free = self._free, []
        self.stream.synchronize()
        for s in free:
            s.close()


class _SegmentTicket:
    """The EncodeTicket of a layer-wise store: wait() blocks the worker until the finish step has run and returns the
    batch of the containers that fit the arena (a prefix of the chunks)."""

    def __init__(self, slot: SegmentSlot, event: torch.cuda.Event, keep):
        self.slot, self.event, self.keep = slot, event, keep

    def wait(self) -> EncodedBatch:
        self.event.synchronize()
        self.keep = None
        sizes = list((ctypes.c_uint64 * self.slot.n_chunks).from_address(self.slot.sizes.host_ptr))
        k = next((j for j, s in enumerate(sizes) if s == 0), len(sizes))
        return EncodedBatch(self.slot.fixed, self.slot.fixed_stride, [int(s) for s in sizes[:k]], 0, self.slot.coder)


class LayerwiseEncode:
    """One layer-wise store's encode on the pool's stream, through the codec's three calls (CacheGen:
    b200kv_encode_layers_plan / _layers / _finish; lossless: b200kv_lossless_encode_layers_*).  The plan is made at
    once; encode_layer(l, stream) makes the encode stream wait for `stream` and enqueues layer l; finish() enqueues the
    headers and returns the event after which the KV is no longer read and the containers are complete.  The host never
    waits.  The arena is the airtight bound of the chunks (the codec's layerwise_chunk_bound each), capped at `budget`:
    past the cap the later chunks fail and become misses."""

    def __init__(self, codec: CacheGenCodec, pool: SegmentPool, view: KvView, tok_begin: int, chunk_size: int,
                 budget: Optional[int] = None):
        n_tok = view.ntokens - tok_begin
        n = (n_tok + chunk_size - 1) // chunk_size
        last = n_tok - (n - 1) * chunk_size
        L, H, D, latent = view.L, view.H, view.D, view.latent
        coder = codec.coder_for(chunk_size, latent)
        dt = view.dtype_code
        layouts = (codec.segment_layout(L, H, D, chunk_size, latent, dt), codec.segment_layout(L, H, D, last, latent, dt))
        stride = (layouts[0].head + 15) & ~15
        arena = min(n * codec.layerwise_chunk_bound(L, H, D, chunk_size, latent),
                    budget or layerwise_store_budget_default())
        ws_bytes = codec.layerwise_workspace_bytes(L, H, D, chunk_size, n, latent)
        self.codec, self.pool, self.view, self.L, self.n_chunks = codec, pool, view, L, n
        self.arena_bytes = arena            # the arena this store takes of its budget (begin_runs)
        self.slot = pool.acquire(arena, n * stride, ws_bytes, n, view.planes, codec.seg_row)
        s = self.slot
        s.n_chunks, s.P, s.seg_row, s.fixed_stride, s.coder = n, view.planes, codec.seg_row, stride, coder
        s.arena_bytes, s.layouts = arena, layouts
        self.done: Optional[torch.cuda.Event] = None
        try:
            with torch.cuda.device(pool.device):
                view.record_stream(pool.stream)          # the caller's KV outlives the encode's last read of it
                self.plan = codec.encode_layers_plan(view, tok_begin, n, chunk_size, last, s, pool.stream)
        except BaseException:
            self.abandon()
            raise

    def encode_layer(self, layer: int, stream: torch.cuda.Stream, ready: Optional[torch.cuda.Event] = None) -> None:
        """`ready`: an event already recorded on `stream` after layer `layer` was written (FanOutEncode's)"""
        with torch.cuda.device(self.pool.device):
            self.pool.stream.wait_event(ready or _recorded(stream))
            self.codec.encode_layers(self.plan, layer, layer + 1, self.pool.stream)

    def finish(self) -> torch.cuda.Event:
        with torch.cuda.device(self.pool.device):
            self.codec.encode_layers_finish(self.plan, self.pool.stream)
            self.done = torch.cuda.Event()
            self.done.record(self.pool.stream)
        self.slot.ticket = _SegmentTicket(self.slot, self.done, self.view)
        self.view = None
        return self.done

    def abandon(self) -> None:
        """give the slot back without landing anything (the kernels already enqueued run on; the pool's stream orders
        the slot's next user after them)"""
        if self.slot is not None:
            slot, self.slot, self.view = self.slot, None, None
            self.pool.release(slot)


def _recorded(stream: torch.cuda.Stream) -> torch.cuda.Event:
    ev = torch.cuda.Event()
    ev.record(stream)
    return ev


# the containers a layer-wise encode writes: versions 3 and 4 (CacheGen), 5 and 6 (lossless)
LAYERWISE_CODERS = (N.CODER_RANS_COMPACT, N.CODER_LATENT, N.CODER_LOSSLESS, N.CODER_LOSSLESS_LATENT)


def layerwise_encodes(codec, chunk_size: int, latent: bool) -> bool:
    """Does a layer-wise encode write `codec`'s containers for chunks of `chunk_size`?  Not for CacheGen chunks of more
    than 256 tokens, the 'rans' and 'ac' coders, or lossless chunks of more than 4096 tokens."""
    try:
        return codec.coder_for(chunk_size, latent) in LAYERWISE_CODERS
    except ValueError:
        return False


def same_containers(a, b, chunk_size: int, latent: bool) -> bool:
    """Do codecs `a` and `b` write byte-identical containers for chunks of `chunk_size` (a latent KV if `latent`)?  Yes
    when both are of one family and write the same coder for this chunk size, and CacheGen codecs code with the same key
    and value bins (the same cachegen_config, or the same model row).  None (a tier without containers) is never the
    same."""
    if a is None or b is None or type(a) is not type(b):
        return False
    try:
        if a.coder_for(chunk_size, latent) != b.coder_for(chunk_size, latent):
            return False
    except ValueError:
        return False
    ca, cb = getattr(a, "config", None), getattr(b, "config", None)
    if ca is None or cb is None:
        return ca is cb
    return ca.key_bins_list() == cb.key_bins_list() and ca.value_bins_list() == cb.value_bins_list()


def segment_pool_for(pool: Optional[SegmentPool], device) -> SegmentPool:
    """`pool` when it serves `device`; otherwise `pool` is closed and a new one made"""
    if pool is None or pool.device != torch.device(device):
        if pool is not None:
            pool.close()
        pool = SegmentPool(device)
    return pool


class NoEncode:
    """A layer-wise store that encodes and stores nothing: the handle of a tier that takes no stores from this engine
    (an MLA engine's remote tier on ranks other than 0).  No GPU work is enqueued."""

    def encode_layer(self, layer: int, stream: torch.cuda.Stream, ready: Optional[torch.cuda.Event] = None) -> None:
        pass

    def finish(self) -> torch.cuda.Event:
        """an event that was never recorded: waiting on it waits for nothing"""
        return torch.cuda.Event()

    def abandon(self) -> None:
        pass


class FanOutEncode:
    """One layer-wise store into two tiers that do not keep the same containers (a hybrid tier): `parts` are the
    tiers' own handles (LayerwiseEncode, local_backend.RawLayerwiseStore, NoEncode), in the hybrid's order (local,
    remote).  encode_layer records one event on the caller's stream and every part enqueues its own launches behind
    it; finish() returns an event after every part's; abandon() drops every part."""

    def __init__(self, parts: Sequence, stream: torch.cuda.Stream):
        self.parts = list(parts)
        self._stream = stream           # where the join of the parts' finish events is recorded

    def encode_layer(self, layer: int, stream: torch.cuda.Stream, ready: Optional[torch.cuda.Event] = None) -> None:
        ready = ready or _recorded(stream)
        for p in self.parts:
            p.encode_layer(layer, stream, ready=ready)

    def finish(self) -> torch.cuda.Event:
        evs = [p.finish() for p in self.parts]
        with torch.cuda.device(self._stream.device):
            for ev in evs:
                self._stream.wait_event(ev)
            return _recorded(self._stream)

    def abandon(self) -> None:
        for p in self.parts:
            p.abandon()

    @property
    def arena_bytes(self) -> int:
        """each part got the same budget: the larger of the parts' arenas is what the store took of it"""
        return max(arena_of(p) for p in self.parts)


def arena_of(handle) -> int:
    """the device arena a tier's layer-wise store handle took of its budget (0: a raw tier's, or NoEncode)"""
    return int(getattr(handle, "arena_bytes", 0))


def begin_runs(begin: Callable, views: Sequence, chunk_size: int, budget: int) -> Optional[list]:
    """One layer-wise store handle per run of a layer-wise segment store: begin(view, 0, chunk_size, budget=...) (a
    tier's begin_layerwise_store) of each run's staged blob, in plan order.  `budget` (LMCACHE_B200_LAYERWISE_STORE_MB)
    bounds the store as a whole: each run gets what the runs before it left, so the arenas do not grow with the number
    of segments, and a run that finds too little keeps the prefix of its chunks that fits (the others become misses, as
    past the budget of one layer-wise store).  None, with every handle made so far abandoned, when the tier takes no
    layer-wise store for these views."""
    handles = []
    left = budget
    try:
        for v in views:
            h = begin(v, 0, chunk_size, budget=max(1, left))
            if h is None:
                for x in handles:
                    x.abandon()
                return None
            handles.append(h)
            left -= arena_of(h)
    except BaseException:
        for x in handles:
            x.abandon()
        raise
    return handles


class SegmentsEncode:
    """The encode a layer-wise segment store's LayerwiseStore drives: `head`, the LayerwiseStore of a segment at token
    0 (store_paged_layerwise / store_layerwise of tokens[:end]) or None; `handles`, one tier handle per run (begin_runs),
    fed from `gather` (rope.StagedGather; None without runs).  encode_layer(l, stream) forwards save_layer to the head,
    then gathers layer l of every run on the gather's side stream and enqueues each run's encode of it behind that
    gather; finish() finishes every run's handle and returns an event after them and every gather (the head is
    finished by the engine's publish step, which also puts it); abandon() drops every part."""

    def __init__(self, head, handles: Sequence, gather):
        self.head, self.handles, self.gather = head, list(handles), gather

    def encode_layer(self, layer: int, stream, ready=None) -> None:
        if self.head is not None:
            self.head.save_layer(layer, stream)
        if self.handles:
            done = self.gather.layer(layer, stream)
            for h in self.handles:
                h.encode_layer(layer, self.gather.side, ready=done)

    def finish(self):
        if not self.handles:
            return torch.cuda.Event()           # never recorded: waiting on it waits for nothing
        return self.gather.join([h.finish() for h in self.handles])

    def abandon(self) -> None:
        head, self.head = self.head, None
        handles, self.handles = self.handles, []
        if head is not None:
            head.close()
        for h in handles:
            h.abandon()


def segment_copy_ranges(seg: np.ndarray, layouts: Sequence[SegmentLayout]):
    """Where the bytes of layer-wise stored containers come from (pure host arithmetic).  seg: int64 [n, P, w], the
    segment rows of n containers of P planes -- w = 2: (arena offset, bytes) of each plane's streams (CacheGen); w = 3:
    (arena offset of its raw rows, arena offset of its streams, stream bytes) (lossless).  layouts[j]: container j's
    SegmentLayout.  Returns (dst, src, nbytes, planes): per container its copy ranges in order -- int64 [n, R] offset in
    the container, source (-1: offset 0 of the chunk's fixed image; otherwise an arena offset) and length; R = 1 + P
    (the fixed image, then each plane's streams) or 1 + 2P (the fixed image, each plane's raw rows -- the last plane's
    running up to the payload --, each plane's streams) -- and int64 [n, P + 1] the plane offsets: payload + the running
    sum of the stream bytes, what codec.plane_offsets / lossless_plane_offsets return for the same container."""
    seg = np.asarray(seg, dtype=np.int64)
    n, P, w = seg.shape
    head = np.array([lo.head for lo in layouts], dtype=np.int64)[:, None]
    pay = np.array([lo.payload for lo in layouts], dtype=np.int64)[:, None]
    sbytes = seg[:, :, w - 1]
    planes = np.concatenate([pay, pay + np.cumsum(sbytes, axis=1)], axis=1)
    dst = [np.zeros((n, 1), dtype=np.int64)]
    src = [np.full((n, 1), -1, dtype=np.int64)]
    lens = [head]
    if w == 3:
        rp = np.array([lo.raw_plane for lo in layouts], dtype=np.int64)[:, None]
        rlen = np.repeat(rp, P, axis=1)
        rlen[:, -1:] = pay - head - (P - 1) * rp
        dst.append(head + np.arange(P, dtype=np.int64)[None, :] * rp)
        src.append(seg[:, :, 0])
        lens.append(rlen)
    dst.append(planes[:, :-1])
    src.append(seg[:, :, w - 2])
    lens.append(sbytes)
    return np.concatenate(dst, axis=1), np.concatenate(src, axis=1), np.concatenate(lens, axis=1), planes


def land_segments(slab, slot: SegmentSlot, batch, blocks: Optional[list] = None,
                  dev_dst: Optional[Sequence[Optional[int]]] = None, codec=CacheGenCodec) -> List[HostContainer]:
    """land() for a layer-wise store: container j is assembled in a fresh block of `slab` from its fixed-section image
    and its segments in the arena (one batched device->host copy of the ranges segment_copy_ranges gives, all
    containers in one call), its plane offsets come from the segment rows, and its header is checked by `codec`'s
    parse_header.  `dev_dst` as in land(): those containers are assembled at their device address too, by the same
    batched copy.  Raises -- with every block freed -- when a copy fails, the segments do not add up to the container's
    size, or a header carries an encoder error."""
    if blocks is None:
        blocks = [slab.alloc(size) for size in batch.sizes]
    n, P, w = len(blocks), slot.P, slot.seg_row     # P planes per container: 2L, or L for a latent KV
    try:
        if n == 0:
            return []
        seg = np.frombuffer(slot.seg.view(), dtype=np.int64, count=slot.n_chunks * P * w)
        seg = seg.reshape(slot.n_chunks, P, w)[:n]
        full, last = slot.layouts
        dst, src, lens, planes = segment_copy_ranges(seg, [last if j == slot.n_chunks - 1 else full for j in range(n)])
        sizes = np.asarray([b.nbytes for b in blocks], dtype=np.int64)
        if (src[:, 1:] < 0).any() or not np.array_equal(planes[:, -1], np.asarray(batch.sizes[:n], dtype=np.int64)):
            raise N.NativeError("layer-wise store: plane segments do not add up to the container sizes")
        assert (lens.sum(axis=1) == sizes).all()
        host = np.array([b.host_ptr for b in blocks], dtype=np.int64)
        dsts = host[:, None] + dst
        fbase = slot.fixed.data_ptr() + np.arange(n, dtype=np.int64) * slot.fixed_stride
        srcs = np.where(src < 0, fbase[:, None], slot.arena.data_ptr() + src)
        resident = [j for j, ptr in enumerate(list(dev_dst or ())[:n]) if ptr is not None]
        if resident:
            dptr = np.array([dev_dst[j] for j in resident], dtype=np.int64)
            dsts = np.concatenate([dsts, dptr[:, None] + dst[resident]])
            srcs = np.concatenate([srcs, srcs[resident]])
            lens = np.concatenate([lens, lens[resident]])
        dev = slot.arena.device
        cs = _d2h_stream(dev)
        with torch.cuda.device(dev):
            try:
                _batch_copy(np.ascontiguousarray(dsts.ravel().astype(np.uint64)),
                            np.ascontiguousarray(srcs.ravel().astype(np.uint64)), np.ascontiguousarray(lens.ravel()), cs)
            finally:
                cs.synchronize()             # no block leaves this function while a copy may still write it
        return [HostContainer(blk, blk.nbytes, codec.parse_header(blk.view()), planes[j].copy())
                for j, blk in enumerate(blocks)]
    except BaseException:
        for blk in blocks:
            blk.free()
        raise


def read_container(codec: CacheGenCodec, blk, nbytes: int, latent: bool = False,
                   prefix: Optional[int] = None) -> Optional[HostContainer]:
    """The record of a container a disk read or a GET put into the first `nbytes` of `blk`, or None -- with the block
    freed -- when it is damaged, was written with another model's bins, or holds the other kind of KV than `latent`
    says (version 4 for a latent engine, versions 1 to 3 otherwise; versions 6 and 5 for a lossless codec): a miss, not an
    error.  The header is checked by the codec's own parse_header, so a container of the other codec family is a miss.
    `prefix`: only the container's first `prefix` bytes are in `blk` yet (a ranged read; the container is `nbytes`
    long): the header is checked against nbytes, and the plane offsets are read when the prefix holds the fixed sections
    (None otherwise: the container is then uploaded whole)."""
    got = nbytes if prefix is None else min(int(prefix), nbytes)
    try:
        hd = codec.parse_header(blk.view()[:got], nbytes)
        if codec.accepts(hd, latent):
            try:
                planes = codec.plane_offsets(blk.view()[:got])      # on the reader's thread
            except N.NativeError:
                if prefix is None:
                    raise
                planes = None                                      # the prefix stops inside the fixed sections
            return HostContainer(blk, nbytes, hd, planes)
    except ValueError:
        pass
    blk.free()
    return None


class DeferredFree:
    """Slab blocks that host->device copies may still be reading: each group is freed once the event recorded after
    those copies has completed (an event of None: nothing reads them)."""

    def __init__(self):
        self._held: list = []              # (event, [blocks])
        self._lock = threading.Lock()

    def add(self, event: Optional[torch.cuda.Event], blocks: list) -> None:
        with self._lock:
            self._held.append((event, blocks))

    def sweep(self, wait: bool = False) -> None:
        """Free every group whose event has completed (wait=True: wait for all of them first)."""
        with self._lock:
            keep = []
            for ev, blocks in self._held:
                if wait and ev is not None:
                    ev.synchronize()
                if ev is None or ev.query():
                    for b in blocks:
                        b.free()
                else:
                    keep.append((ev, blocks))
            self._held = keep

    def pending(self) -> int:
        """groups still held"""
        with self._lock:
            return len(self._held)

    def drain(self) -> None:
        """Blocking: free everything once its copies are done (a tier's close())."""
        self.sweep(wait=True)


def fetched_in_order(futures: Iterable[Future], window: Optional[int] = None) -> Iterator[Optional[HostContainer]]:
    """Results of container fetches (futures of a HostContainer, None for a miss) in the order given, with at most
    `window` of them taken from `futures` ahead of the consumer (None: all of them) -- `futures` may submit each fetch
    as it is taken.  When the consumer stops early, the fetches already issued run to completion and their blocks are
    freed."""
    pending: "collections.deque[Future]" = collections.deque()
    try:
        for f in futures:
            pending.append(f)
            if window is not None and len(pending) >= window:
                yield pending.popleft().result()
        while pending:
            yield pending.popleft().result()
    finally:
        for f in pending:
            rec = f.result()
            if rec is not None and rec.blk is not None:     # a record without a block: a device copy, not a read
                rec.blk.free()


class HeadWindow(NamedTuple):
    """What upload_decode takes of a container of src_H heads: heads [src_head0, src_head0 + n_heads), written at the
    destination's head dst_head0 (lmcache_b200/reshard.py says which)."""
    src_H: int
    src_head0: int
    n_heads: int
    dst_head0: int


def _continues_match(r: HostContainer, first: Optional[HostContainer], dst: KvView, tok: int,
                     src_H: Optional[int] = None) -> bool:
    """May container `r`, landing at token `tok` of `dst`, extend a match that began with `first` (None: r is first)?
    src_H: the heads r must hold when it is decoded through a head window (None: dst's).  A version-4 or version-6
    container fits a latent destination only, and every other version a (K, V) one; a lossless container (versions 5
    and 6) fits a destination of its own dtype only."""
    return (r.L, r.H, r.D) == (dst.L, dst.H if src_H is None else src_H, dst.D) and tok + r.ntokens <= dst.ntokens and \
        bool(r.coder & N.KV_LATENT) == dst.latent and \
        ((r.coder & 0xff) != N.CODER_LOSSLESS or r.max_dtype == dst.dtype_code) and \
        (first is None or (r.max_dtype, r.coder) == (first.max_dtype, first.coder))


class DeviceLevel:
    """What upload_decode and upload_decode_layerwise need from a tier's device level (lmcache_b200/device_cache.py):
    `cache`, the DeviceCache; resident(r): may record r be decoded from the level (it has a device copy in a pool on the
    destination's device); promote(i, r, src_ptr, stream): r, chunk i of the call, has just been uploaded to src_ptr --
    the tier may enqueue a copy of it into the level on `stream` (never waiting) and returns whether it did;
    mark_read(recs, stream): the decodes just enqueued on `stream` read recs' device copies (mark_dev_read, under the
    tier's lock); hit(n): n chunks were served from it.
    The tier keeps every resident record's device copy alive until the call has recorded its decode in `dev_read`."""
    cache = None

    def resident(self, r: HostContainer) -> bool:
        raise NotImplementedError

    def promote(self, i: int, r: HostContainer, src_ptr: int, stream: torch.cuda.Stream) -> bool:
        raise NotImplementedError

    def hit(self, n: int) -> None:
        raise NotImplementedError

    def mark_read(self, recs: Sequence[HostContainer], stream: torch.cuda.Stream) -> None:
        raise NotImplementedError


def mark_dev_read(recs: Sequence[HostContainer], stream: torch.cuda.Stream) -> None:
    """Record on `stream` the event after which no decode reads recs' device copies any more.  A copy that another
    stream may still be decoding keeps that reader too: `stream` waits for the previous `dev_read` before the event, so
    the one event stands for both.  Call under the tier's lock (concurrent retrieves may read the same copies)."""
    seen = set()
    for r in recs:
        if r.dev_read is not None and id(r.dev_read) not in seen:
            seen.add(id(r.dev_read))
            stream.wait_event(r.dev_read)
    ev = _recorded(stream)
    for r in recs:
        r.dev_read = ev


def _wait_filled(recs: Sequence[HostContainer], stream: torch.cuda.Stream) -> None:
    seen = set()
    for r in recs:
        if r.dev_ready is not None and id(r.dev_ready) not in seen:
            seen.add(id(r.dev_ready))
            stream.wait_event(r.dev_ready)


def upload_decode(codec: CacheGenCodec, upload: UploadRing, records: Iterable[Optional[HostContainer]], dst: KvView,
                  dst_tok0: int, chunk_size: int, release: Optional[DeferredFree] = None,
                  level: Optional[DeviceLevel] = None, windows: Optional[Sequence[HeadWindow]] = None) -> int:
    """Upload + decode consecutive chunks straight into `dst`: records[i] (None: a miss) is chunk i and lands at token
    dst_tok0 + i * chunk_size.  Wave by wave the containers are copied into an UploadRing slot on its copy stream and
    decoded on the current stream; nothing is synchronised, and the records are consumed as the caller produces them
    (later fetches / hash-chain keys overlap earlier waves).  Every uploaded record's `last_read` is set to its wave's
    upload event.  Returns the number of chunks decoded: the match stops at the first miss, at the first container whose
    geometry differs from `dst` or that does not fit it, and at the first whose (max_dtype, coder) differs from the
    first container's.  With `release`, the records' blocks are transient: each wave's go to `release` with its upload
    event, and the block of the record the match stopped at is freed.

    With a device `level`, a wave's resident records are not uploaded: they are decoded where they are, in one call at
    their pool offsets after their fill events, and the rest of the wave in a second call from the slot.  Their
    `last_read` is left alone and their `dev_read` becomes that decode's event.  Each uploaded record is offered to the
    level (level.promote) right after its wave's upload.

    With `windows`, chunk i is a group of containers: records[i] is a sequence aligned with `windows` (None: a miss),
    and container k of the group is decoded through head window windows[k] (CacheGenCodec.decode_raw_heads): the chunk
    is what another tensor-parallel layout stored for this rank's heads.  A chunk matches only when every container of
    its group is there, holds windows[k].src_H heads and continues the match; the stopped group's blocks are freed as
    above.  A wave then counts containers, not chunks."""
    W = wave_chunks_default()
    lib = N.lib()
    wave: List[HostContainer] = []
    wtok: List[int] = []                  # destination token of each wave entry
    wwin: List[Optional[HeadWindow]] = []
    widx: List[int] = []                  # chunk index of each wave entry
    n = 0
    first = None
    with torch.cuda.device(dst.device):
        cur = torch.cuda.current_stream()

        def decode(base_ptr: int, buf_bytes: int, offs: List[int], sel: List[int]) -> None:
            recs = [wave[j] for j in sel]
            args = (base_ptr, buf_bytes, offs, [r.nbytes for r in recs], [r.ntokens for r in recs], dst,
                    [wtok[j] for j in sel], wave[0].max_dtype, wave[0].coder)
            if windows is None:
                codec.decode_raw(*args, cur)
            else:
                ws = [wwin[j] for j in sel]
                codec.decode_raw_heads(*args, ws[0].src_H, [w.src_head0 for w in ws], [w.dst_head0 for w in ws],
                                       [w.n_heads for w in ws], cur)

        def flush():
            if not wave:
                return
            res = [j for j, r in enumerate(wave) if level is not None and level.resident(r)]
            up = [j for j in range(len(wave)) if j not in res] if res else list(range(len(wave)))
            if res:
                pool = level.cache.pool
                recs = [wave[j] for j in res]
                _wait_filled(recs, cur)
                decode(pool.dev_ptr, pool.buf.numel(), [r.dev.offset for r in recs], res)
                level.mark_read(recs, cur)
                level.hit(len(recs))
            if up:
                recs = [wave[j] for j in up]
                offs, o = [], 0
                for r in recs:
                    offs.append(o)
                    o += (r.nbytes + 15) & ~15
                slot, buf = upload.next_slot(o)
                for r, off in zip(recs, offs):
                    N.check(lib.b200kv_copy_async(ctypes.c_void_p(buf.data_ptr() + off), ctypes.c_void_p(r.blk.host_ptr),
                                                  r.nbytes, upload.copy_stream.cuda_stream), "copy_async")
                ev = torch.cuda.Event()
                ev.record(upload.copy_stream)
                for r in recs:
                    r.last_read = ev
                if release is not None:
                    release.add(ev, [r.blk for r in recs])
                promoted = None
                if level is not None:       # after the wave's event: the decode does not wait for these copies
                    if sum(level.promote(widx[j], r, buf.data_ptr() + off, upload.copy_stream)
                           for j, r, off in zip(up, recs, offs)):
                        promoted = torch.cuda.Event()
                        promoted.record(upload.copy_stream)
                cur.wait_event(ev)
                decode(buf.data_ptr(), buf.numel(), offs, up)
                if promoted is not None:    # the slot's next writer (or its replacement) waits for the promotion's reads
                    cur.wait_event(promoted)
                upload.mark_read(slot, cur)
            for lst in (wave, wtok, wwin, widx):
                lst.clear()

        for item in records:
            if item is None:
                break
            group = [item] if windows is None else list(item)
            wins = [None] if windows is None else list(windows)
            tok = dst_tok0 + n * chunk_size
            ok = len(group) == len(wins) and all(r is not None for r in group)
            ok = ok and all(_continues_match(r, first or group[0], dst, tok, w.src_H if w is not None else None) and
                            r.ntokens == group[0].ntokens for r, w in zip(group, wins))
            if not ok:
                if release is not None:
                    for r in group:
                        if r is not None and r.blk is not None:
                            r.blk.free()
                break
            first = first or group[0]
            for r, w in zip(group, wins):
                wave.append(r)
                wtok.append(tok)
                wwin.append(w)
                widx.append(n)
            n += 1
            if len(wave) >= W:
                flush()
        flush()
    return n


class LayerwiseUpload:
    """One layer-major upload + decode in flight (upload_decode_layerwise): `n` chunks matched, and per layer the event
    recorded after that layer's decode.  A worker thread records the events one layer after another; `ready(l)` blocks
    the calling host thread until event l has been recorded -- not until it has completed."""

    def __init__(self, n: int, num_layers: int):
        self.n = n
        self.num_layers = num_layers
        self.enqueue_s: List[float] = []    # host seconds the worker spent enqueueing: fixed sections + plan, then per layer
        self.wait_s: List[float] = []       # of which host_ready waits (bytes still on their way), in the same order
        self._ready: List[torch.cuda.Event] = []
        self._error: Optional[BaseException] = None
        self._cv = threading.Condition()

    @classmethod
    def completed(cls, n: int, num_layers: int, event: torch.cuda.Event) -> "LayerwiseUpload":
        """a handle whose every layer is ready with `event` (a retrieve that was not layer-major)"""
        u = cls(n, num_layers)
        u._ready = [event] * num_layers
        return u

    def _publish(self, event: torch.cuda.Event) -> None:
        with self._cv:
            self._ready.append(event)
            self._cv.notify_all()

    def _fail(self, err: BaseException) -> None:
        with self._cv:
            self._error = err
            self._cv.notify_all()

    def ready(self, layer: int) -> torch.cuda.Event:
        if not 0 <= layer < self.num_layers:
            raise IndexError(f"layer {layer} out of range [0, {self.num_layers})")
        with self._cv:
            while len(self._ready) <= layer and self._error is None:
                self._cv.wait()
            if len(self._ready) <= layer:
                raise self._error
            return self._ready[layer]


class JoinedUpload:
    """Several LayerwiseUploads of one retrieve as one handle (a hybrid tier's local and remote parts, or a layer-major
    prefix followed by chunk-major chunks): ready(l) is an event after every part's layer l, recorded on a stream of the
    handle's own that waits for them.  A part's error is raised by ready() as the part raises it."""

    def __init__(self, parts: Sequence[LayerwiseUpload], num_layers: int):
        self.parts = list(parts)
        self.n = sum(p.n for p in self.parts)
        self.num_layers = num_layers
        self.enqueue_s: List[float] = []
        self.wait_s: List[float] = []
        self._ready: dict = {}
        self._stream: Optional[torch.cuda.Stream] = None
        self._lock = threading.Lock()

    def ready(self, layer: int) -> torch.cuda.Event:
        evs = [p.ready(layer) for p in self.parts]
        if len(evs) == 1:
            return evs[0]
        with self._lock:
            ev = self._ready.get(layer)
            if ev is None:
                if self._stream is None:
                    self._stream = torch.cuda.Stream()
                for e in evs:
                    self._stream.wait_event(e)
                ev = torch.cuda.Event(enable_timing=True)
                ev.record(self._stream)
                self._ready[layer] = ev
            return ev


def join_uploads(parts: Sequence, num_layers: int):
    """one handle for the uploads of one retrieve (the part itself when there is one)"""
    return parts[0] if len(parts) == 1 else JoinedUpload(parts, num_layers)


class LayerwiseUploader:
    """A copy stream, a decode stream and the worker thread that enqueues layer-major uploads on them (one per tier and
    device).  Jobs run one after another in submission order."""

    def __init__(self, device):
        self.device = torch.device(device)
        self.copy_stream = torch.cuda.Stream(device=self.device)
        self.decode_stream = torch.cuda.Stream(device=self.device)
        self._q: "queue.Queue" = queue.Queue()
        self._thread = threading.Thread(target=self._worker, name="b200kv-layerwise", daemon=True)
        self._thread.start()

    def _worker(self) -> None:
        torch.cuda.set_device(self.device)
        while True:
            job = self._q.get()
            if job is None:
                return
            job()
            job = None               # a finished job's destination must not live on until the next job arrives

    def submit(self, job: Callable[[], None]) -> None:
        self._q.put(job)

    def close(self) -> None:
        """wait for every submitted job to be enqueued, then stop the worker"""
        if self._thread is not None:
            self._q.put(None)
            self._thread.join()
            self._thread = None


def _batch_copy(dsts: np.ndarray, srcs: np.ndarray, sizes: np.ndarray, stream: torch.cuda.Stream) -> None:
    """one b200kv_copy_batch_async for contiguous uint64 / uint64 / int64 arrays of equal length"""
    N.check(N.lib().b200kv_copy_batch_async(dsts.ctypes.data, srcs.ctypes.data, sizes.ctypes.data, len(sizes),
                                            stream.cuda_stream), "copy_batch_async")


def layer_copy_ranges(plane_offs: Sequence[Optional[np.ndarray]], nbytes: Sequence[int], L: int, ppl: int = 2,
                      raw: Optional[Sequence[Tuple[int, int]]] = None):
    """The copies of a layer-major upload of n containers, as offsets into each container: (fixed int64[n],
    start int64[L, ppl * n], size int64[L, ppl * n]).  Container j's first fixed[j] bytes go first (its fixed sections;
    all of it when it has no plane offsets); row l holds the key ranges (plane l) of containers 0..n-1, then their value
    ranges (plane L + l).  A latent KV (ppl = 1, version 4: plane l is layer l) has one range per container in row l.
    Lossless containers (versions 5 and 6) pass `raw`, their (off_raw, bytes per plane) (codec.raw_rows): then
    fixed[j] is off_raw, the part the decode plan reads, and a plane is two ranges, its raw rows and its streams, so the
    rows are [L, 2 * ppl * n]: the raw ranges of every plane of the row, then the stream ranges.  Together they cover
    every container exactly once."""
    n = len(nbytes)
    P = ppl * L
    po = np.stack([o if o is not None else np.zeros(P + 1, np.int64) for o in plane_offs]).astype(np.int64)
    split = np.array([o is not None for o in plane_offs])
    start = np.ascontiguousarray(np.concatenate([po[:, k * L:(k + 1) * L] for k in range(ppl)]).T)     # [L, ppl * n]
    size = np.ascontiguousarray(np.concatenate([po[:, k * L + 1:(k + 1) * L + 1] - po[:, k * L:(k + 1) * L]
                                                for k in range(ppl)]).T)
    assert start.shape == (L, ppl * n)
    if raw is None:
        fixed = np.where(split, po[:, 0], np.asarray(nbytes, dtype=np.int64)).astype(np.int64)
        return fixed, start, size
    off_raw = np.asarray([r[0] for r in raw], dtype=np.int64)
    row = np.asarray([r[1] for r in raw], dtype=np.int64)
    fixed = np.where(split, off_raw, np.asarray(nbytes, dtype=np.int64)).astype(np.int64)
    pad = np.where(split, po[:, 0] - (off_raw + P * row), 0)     # alignment between the raw rows and the streams:
    start[0, :n] -= pad                                          # copied with plane 0's streams, so that the ranges
    size[0, :n] += pad                                           # cover the container exactly
    planes = np.concatenate([np.arange(L)[:, None] + k * L for k in range(ppl)], axis=0)         # [ppl * L, 1]
    rstart = (off_raw[None, :] + planes * row[None, :]).reshape(ppl, L, n).transpose(1, 0, 2).reshape(L, ppl * n)
    rsize = np.tile(row, (L, ppl))
    rsize = np.where(np.tile(split, ppl)[None, :], rsize, 0)
    start = np.ascontiguousarray(np.concatenate([rstart, start], axis=1))
    size = np.ascontiguousarray(np.concatenate([rsize, size], axis=1))
    return fixed, start, size


READ_MAX_BYTES = (1 << 31) - 1      # an lm:// reply's length is an int32 (protocol.MAX_REPLY)
READ_MAX_RANGES = 1 << 20          # ranges per READ: a request body of 24 MiB at most


def ranged_read_plan(fixed: np.ndarray, start: np.ndarray, size: np.ndarray, got: Sequence[int],
                     conn_of: Sequence[int], k: int, max_bytes: int = READ_MAX_BYTES,
                     max_ranges: int = READ_MAX_RANGES) -> List[List[List[np.ndarray]]]:
    """The READs of a layer-major remote fetch (pure host arithmetic).  fixed, start, size: layer_copy_ranges of n
    containers (column i of start / size belongs to container i % n); got[j]: the first bytes of container j that OPEN
    already delivered; conn_of[j]: the connection (0 .. k-1) that holds its handle.  Returns reads[c][l], the READs
    connection c sends for layer l, each an int64 [m, 3] array of (container, offset, nbytes).  Layer 0 also carries
    bytes [got, fixed) of a container whose prefix stops short of its fixed sections (one uploaded whole).  Ranges are
    clipped to what the prefix lacks, so the prefix and the READs cover every container exactly once; empty ranges are
    dropped.  A READ asks for at most max_bytes in at most max_ranges ranges; a longer range is split."""
    n = len(got)
    L = start.shape[0]
    reads: List[List[List[np.ndarray]]] = [[[] for _ in range(L)] for _ in range(k)]
    if n == 0:
        return reads
    got = np.asarray(got, dtype=np.int64)
    conn_of = np.asarray(conn_of, dtype=np.int64)
    col = np.arange(start.shape[1]) % n
    g = got[col][None, :]
    lo = np.maximum(start, g)
    ln = np.maximum(start + size, g) - lo
    rest = np.asarray(fixed, dtype=np.int64) - got
    for layer in range(L):
        ent = np.stack([col, lo[layer], ln[layer]], axis=1)
        if layer == 0 and (rest > 0).any():
            j = np.nonzero(rest > 0)[0]
            ent = np.concatenate([np.stack([j, got[j], rest[j]], axis=1), ent])
        ent = ent[ent[:, 2] > 0]
        for c in range(k):
            e = ent[conn_of[ent[:, 0]] == c]
            if len(e) == 0:
                continue
            if len(e) <= max_ranges and int(e[:, 2].sum()) <= max_bytes:
                reads[c][layer].append(np.ascontiguousarray(e))
                continue
            cur, tot = [], 0
            for j, off, nb in e.tolist():
                while nb > 0:
                    if len(cur) == max_ranges or tot == max_bytes:
                        reads[c][layer].append(np.array(cur, dtype=np.int64))
                        cur, tot = [], 0
                    take = min(nb, max_bytes - tot)
                    cur.append((j, off, take))
                    tot += take
                    off += take
                    nb -= take
            if cur:
                reads[c][layer].append(np.array(cur, dtype=np.int64))
    return reads


def match_runs(runs: Sequence[Tuple[Iterable, Optional[Callable[[int], Iterable]], int]], chunk_size: int,
               fits: Callable[[object, int], bool]) -> List[Tuple[List[Tuple[object, int]], int]]:
    """The match of a multi-run fetch (get_kv_layerwise_runs), on the calling thread.  Each run is (primary items,
    fallback(i) -> the items that continue it from its chunk i (None: no continuation), destination token of its chunk
    0).  A run takes its primary items up to the first miss -- None, or an item that fits(item, destination token)
    refuses -- then fallback(k) from that index k on, up to their first miss.  A miss ends only its own run.  Returns
    per run ([(item, destination token)], number of primary items among them)."""
    out = []
    for primary, fallback, tok0 in runs:
        got: List[Tuple[object, int]] = []
        own = None
        for src in (primary, None):
            if src is None:
                own = len(got)
                if fallback is None:
                    break
                src = fallback(own)
            for it in src:
                tok = tok0 + len(got) * chunk_size
                if it is None or not fits(it, tok):
                    break
                got.append((it, tok))
        out.append((got, len(got) if own is None else own))
    return out


def rest_runs(runs: Sequence[Tuple[Sequence, int]], hits: Sequence[int], chunk_size: int) -> List[Tuple[Sequence, int]]:
    """What another tier is asked for after one served `hits[i]` chunks of each run (keys, destination token of its
    chunk 0): the keys after them, at the token after them.  Each chunk of a run is served by one tier only."""
    return [(keys[h:], tok0 + h * chunk_size) for (keys, tok0), h in zip(runs, hits)]


def upload_decode_layerwise(codec: CacheGenCodec, uploader: LayerwiseUploader, records: Iterable[Optional[HostContainer]],
                            dst: KvView, dst_tok0: int, chunk_size: int, release: Optional[DeferredFree] = None,
                            on_done: Optional[Callable[[], None]] = None,
                            level: Optional[DeviceLevel] = None,
                            host_ready: Optional[Callable[[int], None]] = None) -> LayerwiseUpload:
    """upload_decode in layer-major order, so that layer 0 of every chunk is decoded after ~1/L of the bytes.

    The match follows upload_decode's rules and is made on the calling thread, which consumes `records` to its end
    (n is known when this returns).  A worker then enqueues, on the uploader's streams:
      1. the fixed sections of every matched container (whole containers without plane offsets) into one device staging
         buffer, and the decode plan (stream offsets) after them;
      2. for each layer l: the byte ranges of planes l (keys) and L + l (values) of every container, one batched copy,
         then the decode of layer l, then the layer's ready event.
    The decode stream first waits for the calling thread's current stream (the destination may have just been
    allocated there).  Every record's `last_read` is the last copy's event; `release` (transient blocks) gets the blocks
    with that event; `on_done` runs once that event is recorded (or when the call fails) -- e.g. to unpin the entries.

    With a device `level`, resident records take no copies: they get a plan of their own over the level's pool (after
    their fill events), and each layer is decoded by both plans before its ready event.  Their `last_read` is left
    alone and their `dev_read` becomes the last decode's event.  The uploaded records are offered to the level
    (level.promote) after the last copy.

    `host_ready(l)`: the records' blocks are still being filled (a ranged remote read, RangedFetch.wait): the worker
    calls it before it enqueues the fixed sections (l = 0) and before each layer l's copy, and it returns once the bytes
    those copies read are in host memory, or raises -- which fails the upload."""
    return upload_decode_layerwise_runs(codec, uploader, [(records, None, dst_tok0)], dst, chunk_size, release, on_done,
                                        level, host_ready)[1]


def upload_decode_layerwise_runs(codec: CacheGenCodec, uploader: LayerwiseUploader,
                                 runs: Sequence[Tuple[Iterable[Optional[HostContainer]],
                                                      Optional[Callable[[int], Iterable[Optional[HostContainer]]]], int]],
                                 dst: KvView, chunk_size: int, release: Optional[DeferredFree] = None,
                                 on_done: Optional[Callable[[], None]] = None, level: Optional[DeviceLevel] = None,
                                 host_ready: Optional[Callable[[int], None]] = None, rotation=None):
    """upload_decode_layerwise of several runs of chunks, each at its own destination (match_runs: a run is its
    records, a callable that continues it from chunk i with other records or None, and its destination token), in one
    upload: each layer is copied and decoded for every chunk of every run before the next layer.  Every record matches
    against the first one of the call.  `rotation` (rope.Rotation, whose rows are per run): the keys of layer l of the
    chunks written are turned on the decode stream after layer l's decode, before its ready event.  Returns ([(primary
    hits, fallback hits)] per run, LayerwiseUpload)."""
    matched: List[HostContainer] = []
    L = dst.L
    submitted = False
    try:
        first = None

        def fits(r: HostContainer, tok: int) -> bool:
            nonlocal first
            if not _continues_match(r, first, dst, tok):
                if release is not None and r.blk is not None:
                    r.blk.free()
                return False
            first = first or r
            matched.append(r)                  # runs match one after another: matched is in run order
            return True
        per_run = match_runs(runs, chunk_size, fits)
        hits = [(own, len(got) - own) for got, own in per_run]
        placed = [(k, tok, r.ntokens) for k, (got, _) in enumerate(per_run) for r, tok in got]
        dst_tok = [tok for got, _ in per_run for _, tok in got]
        n = len(matched)
        res_j = [j for j, r in enumerate(matched) if level is not None and level.resident(r)]
        up_j = [j for j in range(n) if j not in res_j] if res_j else list(range(n))
        res = [matched[j] for j in res_j]
        up = [matched[j] for j in up_j]
        if res:
            level.hit(len(res))
        with torch.cuda.device(dst.device):
            start = torch.cuda.Event()
            start.record(torch.cuda.current_stream())
            if n == 0:
                submitted = True
                if on_done is not None:
                    on_done()
                return hits, LayerwiseUpload.completed(0, L, start)
            offs, o = [], 0
            for r in up:
                offs.append(o)
                o += (r.nbytes + 15) & ~15
            staging = None
            if up:
                staging = torch.empty(o + N.READ_SLACK, dtype=torch.uint8, device=dst.device)
                staging.record_stream(uploader.copy_stream)
                staging.record_stream(uploader.decode_stream)
            dst.record_stream(uploader.decode_stream)
            rot = None if rotation is None else rotation.prepare(placed, dst.device)
            if rot is not None:
                rot.record_stream(uploader.decode_stream)
                start.record(torch.cuda.current_stream())       # after the upload of its seg_of_tok

        if up:
            base = staging.data_ptr()
            host = np.array([r.blk.host_ptr for r in up], dtype=np.uint64)
            dev = base + np.array(offs, dtype=np.uint64)
            ppl = dst.planes // L
            fixed, lo, sz = layer_copy_ranges([r.planes for r in up], [r.nbytes for r in up], L, ppl,
                                              codec.raw_rows(up, dst.latent))
            k = lo.shape[1] // len(up)
            lay_src = np.ascontiguousarray(np.tile(np.concatenate([host] * k), (L, 1)) + lo.astype(np.uint64))
            lay_dst = np.ascontiguousarray(np.tile(np.concatenate([dev] * k), (L, 1)) + lo.astype(np.uint64))
        upload = LayerwiseUpload(n, L)

        def job():
            cs, ds = uploader.copy_stream, uploader.decode_stream
            last = None
            plans = []
            try:
                with torch.cuda.device(uploader.device):
                    t0 = time.perf_counter()
                    waited = 0.0
                    cs.wait_event(start)
                    ds.wait_event(start)
                    if res:
                        pool = level.cache.pool
                        _wait_filled(res, ds)
                        plans.append(codec.decode_plan(pool.dev_ptr, pool.buf.numel(), [r.dev.offset for r in res],
                                                       [r.nbytes for r in res], [r.ntokens for r in res], dst,
                                                       [dst_tok[j] for j in res_j], first.max_dtype, first.coder, ds))
                    if up:
                        if host_ready is not None:
                            w0 = time.perf_counter()
                            host_ready(0)
                            waited = time.perf_counter() - w0
                        _batch_copy(dev, host, fixed, cs)
                        last = torch.cuda.Event()
                        last.record(cs)
                        ds.wait_event(last)
                        plans.append(codec.decode_plan(base, staging.numel(), offs, [r.nbytes for r in up],
                                                       [r.ntokens for r in up], dst, [dst_tok[j] for j in up_j],
                                                       first.max_dtype, first.coder, ds))
                    t1 = time.perf_counter()
                    upload.enqueue_s.append(t1 - t0 - waited)
                    upload.wait_s.append(waited)
                    for layer in range(L):
                        waited = 0.0
                        if up:
                            if host_ready is not None:
                                w0 = time.perf_counter()
                                host_ready(layer)
                                waited = time.perf_counter() - w0
                            _batch_copy(lay_dst[layer], lay_src[layer], sz[layer], cs)
                            last = torch.cuda.Event()
                            last.record(cs)
                            ds.wait_event(last)
                        for plan, _ in plans:
                            codec.decode_layers(plan, layer, layer + 1, ds)
                        if rot is not None:
                            rot.shift_layer(dst, layer, ds)
                        ev = torch.cuda.Event(enable_timing=True)     # a caller may time the layers against each other
                        ev.record(ds)
                        upload._publish(ev)
                        t0, t1 = t1, time.perf_counter()
                        upload.enqueue_s.append(t1 - t0 - waited)
                        upload.wait_s.append(waited)
                    if level is not None:             # staging is recorded on the copy stream: freed after these
                        for j, r, off in zip(up_j, up, offs):
                            level.promote(j, r, base + off, cs)
                    plans.clear()                     # workspaces are recorded on the decode stream
            except BaseException as e:               # noqa: BLE001 -- the caller sees it in ready()
                upload._fail(e)
                cs.synchronize()                      # no block is released while a copy that reads it may be queued
                last = None
            finally:
                for r in up:
                    r.last_read = last
                if res:
                    level.mark_read(res, uploader.decode_stream)
                if release is not None:
                    release.add(last, [r.blk for r in up])
                if on_done is not None:
                    on_done()

        uploader.submit(job)
        submitted = True
        return hits, upload
    finally:
        if not submitted:                             # failed before the worker took over: nothing was enqueued
            if release is not None:
                for r in matched:
                    if r.blk is not None:
                        r.blk.free()
            if on_done is not None:
                on_done()


def _recorded(stream: torch.cuda.Stream) -> torch.cuda.Event:
    ev = torch.cuda.Event()
    ev.record(stream)
    return ev
