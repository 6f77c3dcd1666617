"""Backend plugin interface (lmcache/storage_backend/abstract_backend.py:12-121): same methods, same
None-on-miss / never-raise contract, same default batched loops."""
import abc
from typing import Iterable, Optional, Tuple

import torch

from lmcache_b200.utils import CacheEngineKey


class LMCBackendInterface(metaclass=abc.ABCMeta):

    @abc.abstractmethod
    def put(self, key: CacheEngineKey, kv_chunk: torch.Tensor, blocking=True) -> None:
        """Store one KV chunk blob under `key`; with blocking=False return once it is enqueued."""
        raise NotImplementedError

    @abc.abstractmethod
    def contains(self, key: CacheEngineKey) -> bool:
        raise NotImplementedError

    @abc.abstractmethod
    def get(self, key: CacheEngineKey) -> Optional[torch.Tensor]:
        """The chunk blob on the GPU, or None when the key is absent (a miss is not an error)."""
        raise NotImplementedError

    def batched_put(self, keys_and_chunks: Iterable[Tuple[CacheEngineKey, torch.Tensor]], blocking=True) -> int:
        n = 0
        for key, kv_chunk in keys_and_chunks:
            self.put(key, kv_chunk, blocking=blocking)
            n += 1
        return n

    def batched_get(self, keys: Iterable[CacheEngineKey]) -> Iterable[Optional[torch.Tensor]]:
        """Lazy: the engine stops consuming at the first None (prefix semantics, cache_engine.py:339-343)."""
        for key in keys:
            if self.contains(key):
                yield self.get(key)
            else:
                yield None

    def supports_layerwise_get(self) -> bool:
        """Can get_kv_layerwise serve this tier's chunks layer-major?  A tier that has the method can; the remote tier
        also needs a server with ranged reads, and asks it once."""
        return getattr(self, "get_kv_layerwise", None) is not None

    @abc.abstractmethod
    def close(self):
        pass
