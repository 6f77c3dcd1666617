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
from concurrent.futures import Future
from typing import Callable, Iterable, Iterator, List, Optional, Sequence

import torch

from lmcache_b200 import _native as N
from lmcache_b200.codec import CacheGenCodec, EncodeTicket, KvView, PinnedBuffer, parse_header


def wave_chunks_default() -> int:
    return max(1, int(os.environ.get("LMCACHE_B200_WAVE_CHUNKS", "4")))


def wave_slots_default() -> int:
    return max(2, int(os.environ.get("LMCACHE_B200_WAVE_SLOTS", "3")))


class WaveSlot:
    """Device staging + sizes for one wave of at most `wave` chunks of one geometry."""

    def __init__(self, nbytes: int, wave: int, device):
        self.dev = torch.empty(nbytes + N.READ_SLACK, dtype=torch.uint8, device=device)
        self.sizes = PinnedBuffer(max(64, 8 * wave))
        self.ticket: Optional[EncodeTicket] = None

    def close(self):
        self.sizes.close()
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
    __slots__ = ("blk", "nbytes", "ntokens", "L", "H", "D", "max_dtype", "coder", "last_read")

    def __init__(self, blk, nbytes: int, hd: "N.Header"):
        self.blk = blk                       # None once the tier no longer keeps the bytes (the disk tier's index)
        self.nbytes = int(nbytes)
        self.ntokens = int(hd.ntokens)
        self.L, self.H, self.D = int(hd.L), int(hd.H), int(hd.D)
        self.max_dtype = int(hd.max_dtype)
        self.coder = int(hd.version) - 1
        self.last_read: Optional[torch.cuda.Event] = None   # most recent upload out of the block


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
                for j, (blk, size) in enumerate(zip(blocks, batch.sizes)):
                    N.check(N.lib().b200kv_copy_async(ctypes.c_void_p(blk.host_ptr),
                                                      ctypes.c_void_p(slot.dev.data_ptr() + j * batch.stride), size,
                                                      cs.cuda_stream), "copy_async")
            finally:
                cs.synchronize()             # no block leaves this function while a copy may still write it
        return [HostContainer(blk, blk.nbytes, parse_header(blk.view())) for blk in blocks]
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
            return HostContainer(blk, nbytes, hd)
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
            if (r.L, r.H, r.D) != (dst.L, dst.H, dst.D) or dst_tok0 + n * chunk_size + r.ntokens > dst.ntokens or \
                    (first is not None and (r.max_dtype, r.coder) != (first.max_dtype, first.coder)):
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
