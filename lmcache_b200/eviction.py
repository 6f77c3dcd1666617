"""Eviction order of the capacity-bounded CacheGen tiers (LMCLocalCompressedBackend, LMCLocalDiskBackend).

A retrieve matches chunks front to back and stops at the first miss, so a chunk whose predecessor is gone can never be
hit again: it only holds memory.  Plain LRU evicts exactly that predecessor -- a retrieve reads chunk 0 first, which makes
chunk 0 the least recent.  Here every `touch(keys)` (keys in chain order, chunk 0 first) is one call with a fresh tick T,
and key i of the call gets the stamp (T, -i).  The victim is the eligible key with the smallest stamp: the oldest call,
and within it the chunk furthest along the chain.  As long as every call that touches chunk i also touches chunks
0..i-1, a chunk's predecessor always carries a larger stamp than the chunk itself and is evicted after it.

Not thread-safe: the tiers call it under their own lock.
"""
from __future__ import annotations

import heapq
import itertools
from typing import Callable, Dict, Hashable, Iterable, List, Optional, Tuple

Stamp = Tuple[int, int]


class PrefixLRU:

    def __init__(self):
        self._tick = 0
        self._stamp: Dict[Hashable, Stamp] = {}
        self._heap: List[tuple] = []            # (stamp, seq, key); entries whose stamp is no longer current are stale
        self._seq = itertools.count()           # tie-break: keys need not be orderable

    def __len__(self) -> int:
        return len(self._stamp)

    def __contains__(self, key) -> bool:
        return key in self._stamp

    def touch(self, keys: Iterable[Hashable]) -> None:
        """One call: keys[i] (chain position i, counted from chunk 0) gets the stamp (T, -i)."""
        self.touch_at(keys, self.new_tick())

    def new_tick(self) -> int:
        """a fresh tick for a call whose keys are stamped in several parts (touch_at)"""
        self._tick += 1
        return self._tick

    def touch_at(self, keys: Iterable[Hashable], tick: int, first: int = 0) -> None:
        """Part of the call of `tick`: keys[i] is at chain position first + i and gets the stamp (tick, -(first + i))."""
        for i, k in enumerate(keys):
            s = (tick, -(first + i))
            self._stamp[k] = s
            heapq.heappush(self._heap, (s, next(self._seq), k))
        if len(self._heap) > 2 * len(self._stamp) + 64:     # drop stale entries: the heap stays O(live keys)
            self._heap = [(s, next(self._seq), k) for k, s in self._stamp.items()]
            heapq.heapify(self._heap)

    @property
    def tick(self) -> int:
        """tick of the latest touch"""
        return self._tick

    def stamp(self, key) -> Optional[Stamp]:
        return self._stamp.get(key)

    def discard(self, key) -> None:
        self._stamp.pop(key, None)

    def victim(self, eligible: Callable[[Hashable], bool]) -> Optional[Hashable]:
        """The key with the smallest stamp for which eligible(key) holds (None: there is none).  The key stays in the
        order until the caller discards it."""
        skipped = []
        try:
            while self._heap:
                s, _, k = self._heap[0]
                if self._stamp.get(k) != s:
                    heapq.heappop(self._heap)
                    continue
                if eligible(k):
                    return k
                skipped.append(heapq.heappop(self._heap))
            return None
        finally:
            for item in skipped:
                heapq.heappush(self._heap, item)
