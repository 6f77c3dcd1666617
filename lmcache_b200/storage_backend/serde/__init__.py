"""Serde plugin factory (lmcache/storage_backend/serde/__init__.py:19-41)."""
from typing import Optional, Tuple

from lmcache_b200.config import GlobalConfig, LMCacheEngineConfig, LMCacheEngineMetadata
from lmcache_b200.storage_backend.serde.serde import (Deserializer, DeserializerDebugWrapper, Serializer,
                                                      SerializerDebugWrapper)
from lmcache_b200.storage_backend.serde.torch_serde import TorchDeserializer, TorchSerializer


def CreateSerde(serde_type: str, config: LMCacheEngineConfig,
                metadata: LMCacheEngineMetadata) -> Tuple[Serializer, Deserializer]:
    s: Optional[Serializer] = None
    d: Optional[Deserializer] = None
    if serde_type == "torch":
        s, d = TorchSerializer(), TorchDeserializer()
    elif serde_type == "cachegen":
        from lmcache_b200.storage_backend.serde.cachegen_decoder import CacheGenDeserializer
        from lmcache_b200.storage_backend.serde.cachegen_encoder import CacheGenSerializer
        s, d = CacheGenSerializer(config, metadata), CacheGenDeserializer(config, metadata)
    elif serde_type == "lossless":
        # not in the reference: bit-exact containers (B2KV versions 5 and 6), exponent bytes rANS-coded on the GPU
        from lmcache_b200.storage_backend.serde.lossless import LosslessDeserializer, LosslessSerializer
        s, d = LosslessSerializer(config, metadata), LosslessDeserializer(config, metadata)
    elif serde_type in ("safetensor", "fast"):
        # alternative lossless serdes of the reference (safe_serde.py / fast_serde.py) are outside the
        # rebuilt hot path (SURVEY.md section 2 row 8)
        raise ValueError(f"serde type {serde_type} is not provided by lmcache_b200 (use 'torch', 'cachegen' or "
                         f"'lossless')")
    else:
        raise ValueError(f"Invalid serde type: {serde_type}")
    if GlobalConfig.is_debug():
        return SerializerDebugWrapper(s), DeserializerDebugWrapper(d)
    return s, d


def __getattr__(name):   # lazy: importing the package must not require CUDA
    if name == "CacheGenSerializer":
        from lmcache_b200.storage_backend.serde.cachegen_encoder import CacheGenSerializer
        return CacheGenSerializer
    if name == "CacheGenDeserializer":
        from lmcache_b200.storage_backend.serde.cachegen_decoder import CacheGenDeserializer
        return CacheGenDeserializer
    if name in ("LosslessSerializer", "LosslessDeserializer"):
        from lmcache_b200.storage_backend.serde import lossless
        return getattr(lossless, name)
    raise AttributeError(name)


__all__ = ["Serializer", "Deserializer", "TorchSerializer", "TorchDeserializer", "CacheGenDeserializer",
           "CacheGenSerializer", "LosslessSerializer", "LosslessDeserializer", "CreateSerde"]
