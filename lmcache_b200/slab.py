"""PinnedSlab -- page-locked host memory for the KV tiers, allocated in large segments and carved up by a first-fit
free list.

Replaces the per-put host allocations of the reference's local tier (lmcache/storage_backend/local_backend.py:82-100:
a pageable `tensor.to("cpu")` per chunk) and this package's round-1 per-put `pin_memory=True` tensors: a
cudaHostAlloc costs about as much as encoding a whole chunk, so the slab pays it once per segment (1 GiB by default)
and every chunk after that is an offset.  Segments are mapped into the device address space (b200kv_pinned_alloc), so
kernels can write into them as well as copy engines.

The allocator is host-side bookkeeping only (a sorted free list per segment, coalescing on free); nothing here touches
the GPU path.  Thread-safe.
"""
from __future__ import annotations

import bisect
import os
import threading
from typing import List, Optional, Tuple

ALIGN = 256          # allocation granularity: keeps every block aligned for 16-byte vector copies and DMA bursts


def _default_segment_bytes() -> int:
    return int(os.environ.get("LMCACHE_B200_SLAB_SEGMENT_MB", "1024")) << 20


def block_bytes(nbytes: int) -> int:
    """slab bytes a block of nbytes takes (its `cap`)"""
    return max(ALIGN, (int(nbytes) + ALIGN - 1) // ALIGN * ALIGN)


class SlabBlock:
    """One allocation: `nbytes` at `offset` of segment `seg`; host_ptr / dev_ptr are absolute addresses."""
    __slots__ = ("slab", "seg", "offset", "nbytes", "cap")

    def __init__(self, slab: "PinnedSlab", seg: int, offset: int, nbytes: int, cap: int):
        self.slab, self.seg, self.offset, self.nbytes, self.cap = slab, seg, offset, nbytes, cap

    @property
    def host_ptr(self) -> int:
        return self.slab._segs[self.seg].host_ptr + self.offset

    @property
    def dev_ptr(self) -> int:
        return self.slab._segs[self.seg].dev_ptr + self.offset

    def view(self) -> memoryview:
        return self.slab._segs[self.seg].view(self.offset, self.nbytes)

    def free(self) -> None:
        self.slab.free(self)

    def shrink(self, nbytes: int) -> None:
        """Give the tail back: a receive buffer is reserved for the largest possible payload and usually holds far less."""
        self.slab.shrink(self, nbytes)


class _FreeList:
    """Sorted, coalescing list of free extents of one segment."""

    def __init__(self, size: int):
        self.offs: List[int] = [0]
        self.lens: List[int] = [size]

    def take(self, n: int) -> Optional[int]:
        for i, ln in enumerate(self.lens):          # first fit
            if ln >= n:
                off = self.offs[i]
                if ln == n:
                    del self.offs[i], self.lens[i]
                else:
                    self.offs[i] += n
                    self.lens[i] -= n
                return off
        return None

    def give(self, off: int, n: int) -> None:
        i = bisect.bisect_left(self.offs, off)
        if i > 0 and self.offs[i - 1] + self.lens[i - 1] == off:      # merge with the extent before
            i -= 1
            self.lens[i] += n
        else:
            self.offs.insert(i, off)
            self.lens.insert(i, n)
        if i + 1 < len(self.offs) and self.offs[i] + self.lens[i] == self.offs[i + 1]:   # and with the one after
            self.lens[i] += self.lens[i + 1]
            del self.offs[i + 1], self.lens[i + 1]

    def free_bytes(self) -> int:
        return sum(self.lens)


class SlabFull(MemoryError):
    """No free extent fits the request and the slab may not reserve another segment."""


class PinnedSlab:

    def __init__(self, segment_bytes: Optional[int] = None, alloc_fn=None, max_segments: Optional[int] = None):
        """alloc_fn(nbytes) -> object with host_ptr / dev_ptr / view(offset, nbytes) / close(); defaults to the
        library's page-locked allocator (lmcache_b200.codec.PinnedBuffer).  Tests pass a plain-memory stand-in.
        max_segments: the slab's byte budget in segments (None: unbounded); beyond it `alloc` raises SlabFull instead of
        page-locking more memory, and requests larger than a segment always do."""
        self.segment_bytes = int(segment_bytes or _default_segment_bytes())
        self.max_segments = max_segments
        self._alloc_fn = alloc_fn
        self._segs: list = []
        self._free: List[_FreeList] = []
        self._lock = threading.Lock()
        self.bytes_in_use = 0

    def _new_segment(self, nbytes: int) -> int:
        if self._alloc_fn is None:
            from lmcache_b200.codec import PinnedBuffer
            self._alloc_fn = PinnedBuffer
        self._segs.append(self._alloc_fn(nbytes))
        self._free.append(_FreeList(nbytes))
        return len(self._segs) - 1

    def reserve(self, nbytes: int) -> None:
        """Make sure at least nbytes are available without a further cudaHostAlloc (start-up warm-up)."""
        with self._lock:
            have = sum(f.free_bytes() for f in self._free)
            while have < nbytes and (self.max_segments is None or len(self._segs) < self.max_segments):
                self._new_segment(self.segment_bytes)
                have += self.segment_bytes

    def alloc(self, nbytes: int) -> SlabBlock:
        cap = block_bytes(nbytes)
        with self._lock:
            for s, fl in enumerate(self._free):
                off = fl.take(cap)
                if off is not None:
                    self.bytes_in_use += cap
                    return SlabBlock(self, s, off, int(nbytes), cap)
            if self.max_segments is not None and (len(self._segs) >= self.max_segments or cap > self.segment_bytes):
                raise SlabFull(f"no free extent of {cap} bytes within {self.max_segments} segments")
            s = self._new_segment(max(self.segment_bytes, cap))       # oversized requests get their own segment
            off = self._free[s].take(cap)
            self.bytes_in_use += cap
            return SlabBlock(self, s, off, int(nbytes), cap)

    def shrink(self, blk: SlabBlock, nbytes: int) -> None:
        keep = max(ALIGN, (int(nbytes) + ALIGN - 1) // ALIGN * ALIGN)
        with self._lock:
            if blk.cap and keep < blk.cap:
                self._free[blk.seg].give(blk.offset + keep, blk.cap - keep)
                self.bytes_in_use -= blk.cap - keep
                blk.cap = keep
                blk.nbytes = min(blk.nbytes, keep)

    def free(self, blk: SlabBlock) -> None:
        with self._lock:
            if blk.cap:
                self._free[blk.seg].give(blk.offset, blk.cap)
                self.bytes_in_use -= blk.cap
                blk.cap = 0

    def stats(self) -> Tuple[int, int, int]:
        """(segments, bytes reserved from the OS, bytes in use)"""
        with self._lock:
            return len(self._segs), sum(getattr(s, "nbytes", 0) for s in self._segs), self.bytes_in_use

    def close(self) -> None:
        with self._lock:
            for s in self._segs:
                s.close()
            self._segs, self._free, self.bytes_in_use = [], [], 0
