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
from typing import Callable, Iterable, Iterator, List, Optional, Sequence

import numpy as np
import torch

from lmcache_b200 import _native as N
from lmcache_b200.codec import CacheGenCodec, EncodeTicket, KvView, PinnedBuffer, parse_header, plane_offsets


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

    def close(self):
        self.sizes.close()
        self.planes.close()
        self.dev = None


class EncodeRing:
    """A fixed set of WaveSlots for one (L, H, D, chunk_size, device); acquire() blocks the calling host thread while
    every slot is still in flight -- the only back-pressure of the store pipeline."""

    def __init__(self, codec: CacheGenCodec, L: int, H: int, D: int, chunk_size: int, device, wave: Optional[int] = None,
                 slots: Optional[int] = None):
        self.codec = codec
        self.geom = (L, H, D, chunk_size, torch.device(device))
        self.wave = wave or wave_chunks_default()
        self.stride = codec.out_stride(L, H, D, chunk_size)
        n = slots or wave_slots_default()
        self._free: "queue.Queue[WaveSlot]" = queue.Queue()
        self._all: List[WaveSlot] = []
        for _ in range(n):
            s = WaveSlot(self.stride * self.wave, self.wave, device)
            self._all.append(s)
            self._free.put(s)

    def matches(self, L, H, D, chunk_size, device) -> bool:
        return self.geom == (L, H, D, chunk_size, torch.device(device))

    def scratch_bytes(self) -> int:
        return sum(s.dev.numel() for s in self._all)

    def acquire(self) -> WaveSlot:
        return self._free.get()

    def release(self, slot: WaveSlot) -> None:
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
        if self.ring is None or not self.ring.matches(view.L, view.H, view.D, chunk_size, view.device):
            if self.ring is not None:
                self.ring.close()
            self.ring = EncodeRing(self.codec, view.L, view.H, view.D, chunk_size, view.device)
        return self.ring

    def submit(self, view: KvView, tok_begin: int, chunk_size: int, items: Sequence,
               stream: Optional[torch.cuda.Stream] = None) -> StoreJob:
        """Enqueue the encode of tokens [tok_begin, T) of `view`, len(items) chunks, in waves.  Returns once every wave
        is enqueued on `stream` (default: the current stream); the job completes when the sink has taken them all."""
        n_tok = view.ntokens - tok_begin
        n_chunks = len(items)
        assert n_chunks == (n_tok + chunk_size - 1) // chunk_size and n_chunks > 0
        ring = self._ring_for(view, chunk_size)
        W = ring.wave
        job = StoreJob((n_chunks + W - 1) // W)
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
                    raise
                self._q.put((ring, slot, c0, list(items[c0:c0 + k]), job))
        return job

    # ------------------------------------------------------------------ worker side
    def _worker(self) -> None:
        torch.cuda.set_device(self._device)
        while True:
            item = self._q.get()
            if item is None:
                return
            ring, slot, c0, items, job = item
            err = None
            try:
                batch = slot.ticket.wait()          # host wait on this wave's kernels -- on the worker thread only
                self.sink(slot, batch, c0, items)
            except BaseException as e:              # noqa: BLE001 -- a failed background store is a miss later
                err = e
            finally:
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
    """One CacheGen container in a page-locked slab block, with the header fields its upload and decode need."""
    __slots__ = ("blk", "nbytes", "ntokens", "L", "H", "D", "max_dtype", "coder", "last_read", "planes")

    def __init__(self, blk, nbytes: int, hd: "N.Header", planes: Optional[np.ndarray] = None):
        self.blk = blk                       # None once the tier no longer keeps the bytes (the disk tier's index)
        self.nbytes = int(nbytes)
        self.ntokens = int(hd.ntokens)
        self.L, self.H, self.D = int(hd.L), int(hd.H), int(hd.D)
        self.max_dtype = int(hd.max_dtype)
        self.coder = int(hd.version) - 1
        self.last_read: Optional[torch.cuda.Event] = None   # most recent upload out of the block
        # codec.plane_offsets: where each plane's streams lie, for a layer-major upload; None: upload it whole.  Made by
        # whoever makes the record (land, read_container), never on the thread of a retrieve.
        self.planes = planes


@functools.lru_cache(maxsize=None)
def _d2h_stream(device: torch.device) -> torch.cuda.Stream:
    return torch.cuda.Stream(device=device)


def land(slab, slot: WaveSlot, batch, blocks: Optional[list] = None) -> List[HostContainer]:
    """Store-pipeline sink side: copy a finished wave's containers out of slot.dev into fresh blocks of `slab` (exactly
    their bytes, on the device's copy stream), wait for the copies, and parse every header.  Raises -- with every block
    freed -- when a copy fails or a container carries an encoder error.  `blocks`: blocks the caller allocated for the
    first len(blocks) containers (a bounded tier); only those are landed."""
    dev = slot.dev.device
    cs = _d2h_stream(dev)
    if blocks is None:
        blocks = [slab.alloc(size) for size in batch.sizes]
    try:
        with torch.cuda.device(dev):
            try:
                # plane offsets of the wave, read on the device before the bytes leave it: no host pass over the
                # lengths sections (on the store worker such a pass made every e2e store ~2 ms slower, measured)
                N.check(N.pylib().b200kv_plane_offsets_device(ctypes.c_void_p(slot.dev.data_ptr()), batch.stride,
                                                            len(blocks), ctypes.c_void_p(slot.planes.dev_ptr),
                                                            cs.cuda_stream), "plane_offsets_device")
                for j, (blk, size) in enumerate(zip(blocks, batch.sizes)):
                    N.check(N.lib().b200kv_copy_async(ctypes.c_void_p(blk.host_ptr),
                                                      ctypes.c_void_p(slot.dev.data_ptr() + j * batch.stride), size,
                                                      cs.cuda_stream), "copy_async")
            finally:
                cs.synchronize()             # no block leaves this function while a copy may still write it
        po = np.frombuffer(slot.planes.view(), dtype=np.int64, count=len(blocks) * (N.MAX_PLANES + 1))
        po = po.reshape(len(blocks), N.MAX_PLANES + 1)
        recs = []
        for j, blk in enumerate(blocks):
            hd = parse_header(blk.view())
            recs.append(HostContainer(blk, blk.nbytes, hd, po[j, :2 * hd.L + 1].copy() if po[j, 0] >= 0 else None))
        return recs
    except BaseException:
        for blk in blocks:
            blk.free()
        raise


def read_container(codec: CacheGenCodec, blk, nbytes: int) -> Optional[HostContainer]:
    """The record of a container a disk read or a GET put into the first `nbytes` of `blk`, or None -- with the block
    freed -- when it is damaged or was written with another model's bins (a miss, not an error)."""
    try:
        hd = parse_header(blk.view()[:nbytes])
        if codec.accepts(hd):
            return HostContainer(blk, nbytes, hd, plane_offsets(blk.view()[:nbytes]))   # on the reader's thread
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
            if rec is not None:
                rec.blk.free()


def _continues_match(r: HostContainer, first: Optional[HostContainer], dst: KvView, tok: int) -> bool:
    """May container `r`, landing at token `tok` of `dst`, extend a match that began with `first` (None: r is first)?"""
    return (r.L, r.H, r.D) == (dst.L, dst.H, dst.D) and tok + r.ntokens <= dst.ntokens and \
        (first is None or (r.max_dtype, r.coder) == (first.max_dtype, first.coder))


def upload_decode(codec: CacheGenCodec, upload: UploadRing, records: Iterable[Optional[HostContainer]], dst: KvView,
                  dst_tok0: int, chunk_size: int, release: Optional[DeferredFree] = None) -> int:
    """Upload + decode consecutive chunks straight into `dst`: records[i] (None: a miss) is chunk i and lands at token
    dst_tok0 + i * chunk_size.  Wave by wave the containers are copied into an UploadRing slot on its copy stream and
    decoded on the current stream; nothing is synchronised, and the records are consumed as the caller produces them
    (later fetches / hash-chain keys overlap earlier waves).  Every uploaded record's `last_read` is set to its wave's
    upload event.  Returns the number of chunks decoded: the match stops at the first miss, at the first container whose
    geometry differs from `dst` or that does not fit it, and at the first whose (max_dtype, coder) differs from the
    first container's.  With `release`, the records' blocks are transient: each wave's go to `release` with its upload
    event, and the block of the record the match stopped at is freed."""
    W = wave_chunks_default()
    lib = N.lib()
    wave: List[HostContainer] = []
    n = 0
    first = None
    with torch.cuda.device(dst.device):
        cur = torch.cuda.current_stream()

        def flush():
            if not wave:
                return
            offs, o = [], 0
            for r in wave:
                offs.append(o)
                o += (r.nbytes + 15) & ~15
            slot, buf = upload.next_slot(o)
            for r, off in zip(wave, offs):
                N.check(lib.b200kv_copy_async(ctypes.c_void_p(buf.data_ptr() + off), ctypes.c_void_p(r.blk.host_ptr),
                                              r.nbytes, upload.copy_stream.cuda_stream), "copy_async")
            ev = torch.cuda.Event()
            ev.record(upload.copy_stream)
            for r in wave:
                r.last_read = ev
            if release is not None:
                release.add(ev, [r.blk for r in wave])
            cur.wait_event(ev)
            w0 = n - len(wave)
            codec.decode_raw(buf.data_ptr(), buf.numel(), offs, [r.nbytes for r in wave], [r.ntokens for r in wave], dst,
                             [dst_tok0 + (w0 + j) * chunk_size for j in range(len(wave))], wave[0].max_dtype,
                             wave[0].coder, cur)
            upload.mark_read(slot, cur)
            wave.clear()

        for r in records:
            if r is None:
                break
            if not _continues_match(r, first, dst, dst_tok0 + n * chunk_size):
                if release is not None:
                    r.blk.free()
                break
            first = first or r
            wave.append(r)
            n += 1
            if len(wave) == W:
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


def layer_copy_ranges(plane_offs: Sequence[Optional[np.ndarray]], nbytes: Sequence[int], L: int):
    """The copies of a layer-major upload of n containers, as offsets into each container: (fixed int64[n],
    start int64[L, 2n], size int64[L, 2n]).  Container j's first fixed[j] bytes go first (its fixed sections; all of it
    when it has no plane offsets); row l holds the key ranges (plane l) of containers 0..n-1, then their value ranges
    (plane L + l).  Together they cover every container exactly once."""
    n = len(nbytes)
    po = np.stack([o if o is not None else np.zeros(2 * L + 1, np.int64) for o in plane_offs]).astype(np.int64)
    split = np.array([o is not None for o in plane_offs])
    fixed = np.where(split, po[:, 0], np.asarray(nbytes, dtype=np.int64)).astype(np.int64)
    start = np.ascontiguousarray(np.concatenate([po[:, :L], po[:, L:2 * L]]).T)                   # [L, 2n]
    size = np.ascontiguousarray(np.concatenate([po[:, 1:L + 1] - po[:, :L], po[:, L + 1:] - po[:, L:2 * L]]).T)
    assert start.shape == (L, 2 * n)
    return fixed, start, size


def upload_decode_layerwise(codec: CacheGenCodec, uploader: LayerwiseUploader, records: Iterable[Optional[HostContainer]],
                            dst: KvView, dst_tok0: int, chunk_size: int, release: Optional[DeferredFree] = None,
                            on_done: Optional[Callable[[], None]] = None) -> LayerwiseUpload:
    """upload_decode in layer-major order, so that layer 0 of every chunk is decoded after ~1/L of the bytes.

    The match follows upload_decode's rules and is made on the calling thread, which consumes `records` to its end
    (n is known when this returns).  A worker then enqueues, on the uploader's streams:
      1. the fixed sections of every matched container (whole containers without plane offsets) into one device staging
         buffer, and the decode plan (stream offsets) after them;
      2. for each layer l: the byte ranges of planes l (keys) and L + l (values) of every container, one batched copy,
         then the decode of layer l, then the layer's ready event.
    The decode stream first waits for the calling thread's current stream (the destination may have just been
    allocated there).  Every record's `last_read` is the last copy's event; `release` (transient blocks) gets the blocks
    with that event; `on_done` runs once that event is recorded (or when the call fails) -- e.g. to unpin the entries."""
    matched: List[HostContainer] = []
    L = dst.L
    submitted = False
    try:
        first = None
        for r in records:
            if r is None:
                break
            if not _continues_match(r, first, dst, dst_tok0 + len(matched) * chunk_size):
                if release is not None:
                    r.blk.free()
                break
            first = first or r
            matched.append(r)
        n = len(matched)
        with torch.cuda.device(dst.device):
            start = torch.cuda.Event()
            start.record(torch.cuda.current_stream())
            if n == 0:
                submitted = True
                if on_done is not None:
                    on_done()
                return LayerwiseUpload.completed(0, L, start)
            offs, o = [], 0
            for r in matched:
                offs.append(o)
                o += (r.nbytes + 15) & ~15
            staging = torch.empty(o + N.READ_SLACK, dtype=torch.uint8, device=dst.device)
            staging.record_stream(uploader.copy_stream)
            staging.record_stream(uploader.decode_stream)
            dst.record_stream(uploader.decode_stream)

        base = staging.data_ptr()
        host = np.array([r.blk.host_ptr for r in matched], dtype=np.uint64)
        dev = base + np.array(offs, dtype=np.uint64)
        fixed, lo, sz = layer_copy_ranges([r.planes for r in matched], [r.nbytes for r in matched], L)
        lay_src = np.ascontiguousarray(np.tile(np.concatenate([host, host]), (L, 1)) + lo.astype(np.uint64))
        lay_dst = np.ascontiguousarray(np.tile(np.concatenate([dev, dev]), (L, 1)) + lo.astype(np.uint64))
        upload = LayerwiseUpload(n, L)
        totals = [r.nbytes for r in matched]
        ntoks = [r.ntokens for r in matched]
        dst_tok = [dst_tok0 + j * chunk_size for j in range(n)]

        def job():
            cs, ds = uploader.copy_stream, uploader.decode_stream
            last = None
            try:
                with torch.cuda.device(uploader.device):
                    t0 = time.perf_counter()
                    cs.wait_event(start)
                    ds.wait_event(start)
                    _batch_copy(dev, host, fixed, cs)
                    last = torch.cuda.Event()
                    last.record(cs)
                    ds.wait_event(last)
                    plan, ws = codec.decode_plan(base, staging.numel(), offs, totals, ntoks, dst, dst_tok,
                                                 first.max_dtype, first.coder, ds)
                    t1 = time.perf_counter()
                    upload.enqueue_s.append(t1 - t0)
                    for layer in range(L):
                        _batch_copy(lay_dst[layer], lay_src[layer], sz[layer], cs)
                        last = torch.cuda.Event()
                        last.record(cs)
                        ds.wait_event(last)
                        codec.decode_layers(plan, layer, layer + 1, ds)
                        ev = torch.cuda.Event(enable_timing=True)     # a caller may time the layers against each other
                        ev.record(ds)
                        upload._publish(ev)
                        t0, t1 = t1, time.perf_counter()
                        upload.enqueue_s.append(t1 - t0)
                    del ws                            # recorded on the decode stream: reused only after the decodes
            except BaseException as e:               # noqa: BLE001 -- the caller sees it in ready()
                upload._fail(e)
                cs.synchronize()                      # no block is released while a copy that reads it may be queued
                last = None
            finally:
                for r in matched:
                    r.last_read = last
                if release is not None:
                    release.add(last, [r.blk for r in matched])
                if on_done is not None:
                    on_done()

        uploader.submit(job)
        submitted = True
        return upload
    finally:
        if not submitted:                             # failed before the worker took over: nothing was enqueued
            if release is not None:
                for r in matched:
                    r.blk.free()
            if on_done is not None:
                on_done()
