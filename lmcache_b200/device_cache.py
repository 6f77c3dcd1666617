"""DeviceCache -- the device-memory level of the CacheGen host and disk tiers (config.device_cache_bytes).

The level is inclusive: a container is copied into device memory only beside the tier's own copy (a slab block or a
.b2kv file), so losing a device copy never loses data.  A retrieve decodes a resident container where it is, with the
same decode entry points as an uploaded one; nothing crosses PCIe for it.

One device allocation of `budget + N.READ_SLACK` bytes holds every copy.  It is carved by the slab allocator
(lmcache_b200.slab.PinnedSlab) as a single segment of `budget` bytes, so every block ends at least READ_SLACK bytes
before the end of the allocation: the decoder's look-ahead past a container stays inside it, and a container at
`base + block.offset` is decoded with `base` and the allocation's size like any container in a staging buffer.

Filling never waits.  A container is copied in when its store lands or when a retrieve has uploaded it (a promotion);
room is made by evicting device copies in the order of a PrefixLRU of their own, and only copies nobody can still read
are victims: not pinned by a retrieve between its lookup and its enqueue, fill copy and latest decode completed.  A
store never evicts its own copies (its caller's `keep`): a sequence larger than the level keeps the head of its chain,
and the tail is not cached.  When that is not enough (or first-fit fragmentation leaves no extent) the container is
simply not cached.

Bookkeeping only: the holders are the tier's entries (anything with `.rec` and `.pins`), the device copy is
`holder.rec.dev` with the events `rec.dev_ready` (fill done) and `rec.dev_read` (latest decode).  Not thread-safe: the
tier calls every method under its own lock.  No method needs CUDA when `alloc_fn` and the events are stand-ins.
"""
from __future__ import annotations

from typing import Dict, Iterable, Optional

from lmcache_b200.eviction import PrefixLRU
from lmcache_b200.slab import PinnedSlab, SlabBlock, SlabFull, block_bytes


def _done(ev) -> bool:
    return ev is None or ev.query()


class DevicePool:
    """The level's one device allocation: `nbytes + N.READ_SLACK` bytes on the current device (a PinnedSlab segment of
    `nbytes`; the slack stays outside every block)."""

    def __init__(self, nbytes: int):
        import torch

        from lmcache_b200 import _native as N
        self.nbytes = int(nbytes)
        self.buf = torch.empty(self.nbytes + N.READ_SLACK, dtype=torch.uint8,
                               device=torch.device("cuda", torch.cuda.current_device()))
        self.device = self.buf.device
        self.dev_ptr = self.buf.data_ptr()
        self.host_ptr = None

    def view(self, offset: int, nbytes: int):
        raise TypeError("device pool blocks have no host view")

    def close(self) -> None:
        self.buf = None


class DeviceCache:

    def __init__(self, budget: int, alloc_fn=None):
        from lmcache_b200.pipeline import DeferredFree
        self.budget = int(budget)
        self.slab = PinnedSlab(self.budget, alloc_fn=alloc_fn or DevicePool, max_segments=1)
        self.order = PrefixLRU()             # over the holders whose record has a device copy
        self.release = DeferredFree()        # evicted / retired blocks a decode or a fill may still touch
        self.hits = 0                        # chunks decoded from the level
        self.promotions = 0                  # chunks copied in by a retrieve
        self.evictions = 0                   # device copies evicted to make room
        self.skipped = 0                     # chunks not cached: no room without waiting

    # ------------------------------------------------------------------ the allocation
    def reserve(self) -> None:
        """make the allocation now (on the current device) instead of at the first fill"""
        self.slab.reserve(self.budget)

    @property
    def pool(self):
        """the DevicePool, or None before the first fill"""
        segs = self.slab._segs
        return segs[0] if segs else None

    def serves(self, device) -> bool:
        """may containers in the level be decoded into tensors on `device`?"""
        p = self.pool
        return p is not None and getattr(p, "device", None) == device

    # ------------------------------------------------------------------ filling
    def alloc(self, nbytes: int, keep=None) -> Optional[SlabBlock]:
        """A block of `nbytes` for a new device copy, or None (counted as skipped).  Evicts idle copies while the
        container does not fit, except the holders for which keep(holder) holds; never waits for one."""
        self.release.sweep()
        if block_bytes(nbytes) > self.budget:
            self.skipped += 1
            return None
        while True:
            try:
                return self.slab.alloc(nbytes)
            except SlabFull:
                pass
            h = self.order.victim(self._idle if keep is None else (lambda h: self._idle(h) and not keep(h)))
            if h is None:
                self.skipped += 1
                return None
            self.order.discard(h)
            if h.rec is not None and h.rec.dev is not None:
                self.evictions += 1
                self.detach(h.rec)
                self.release.sweep()

    def _idle(self, h) -> bool:
        r = h.rec
        if r is None or r.dev is None:
            return True                      # stale: its copy is gone already
        return not h.pins and _done(r.dev_ready) and _done(r.dev_read)

    def attach(self, holders: Iterable, blocks: Iterable[Optional[SlabBlock]], ready=None, at=None) -> None:
        """Give each holder's record its block (None: not cached), valid once `ready` has completed (None: now).  The
        holders are stamped in chain order, first to last: as one call, or with at=(tick, first) as the part of the call
        of `tick` whose first holder is at chain position `first` (a store's waves share its tick, so the head of its
        chain outlives the tail)."""
        tick, first = at if at is not None else (self.order.new_tick(), 0)
        for i, (h, blk) in enumerate(zip(holders, blocks)):
            if blk is None:
                continue
            h.rec.dev, h.rec.dev_ready, h.rec.dev_read = blk, ready, None
            self.order.touch_at([h], tick, first + i)

    def detach(self, rec) -> None:
        """The record's device copy leaves the level; its block is freed once the last fill or decode that touches it
        has completed."""
        blk, rec.dev = rec.dev, None
        if blk is None:
            return
        last = rec.dev_read or rec.dev_ready
        rec.dev_ready = rec.dev_read = None
        self.release.add(last, [blk])

    def drop(self, holder) -> None:
        """the tier dropped (or replaced) `holder`: its device copy goes with it"""
        self.order.discard(holder)
        if holder.rec is not None:
            self.detach(holder.rec)

    # ------------------------------------------------------------------ order and reports
    def touch(self, holders: Iterable) -> None:
        """The tier's touch of one call (chain order): resident holders are stamped together."""
        self.order.touch([h for h in holders if h is not None and h.rec is not None and h.rec.dev is not None])

    def stats(self) -> Dict[str, int]:
        return {"bytes_in_use": self.slab.bytes_in_use, "budget_bytes": self.budget, "hits": self.hits,
                "promotions": self.promotions, "evictions": self.evictions, "not_cached": self.skipped}

    def close(self) -> None:
        """after a device synchronise: every pending free is done"""
        self.release.sweep(wait=True)
        self.slab.close()
