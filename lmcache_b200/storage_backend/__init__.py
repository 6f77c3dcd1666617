"""Backend factory (lmcache/storage_backend/__init__.py:13-44): same (local_device, remote_url) dispatch."""
from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
from lmcache_b200.storage_backend.abstract_backend import LMCBackendInterface


def CreateStorageBackend(config: LMCacheEngineConfig, metadata: LMCacheEngineMetadata) -> LMCBackendInterface:
    local, remote = config.local_device, config.remote_url
    # the compressed host tier: page-locked containers, CacheGen or lossless; "cuda" keeps raw blobs whatever the serde
    compressed_host = local == "cpu" and config.local_serde in ("cachegen", "lossless")
    if config.local_capacity_bytes is not None:
        # only the container tiers evict: the raw tiers keep views of one shared buffer per store, so evicting one view
        # would free nothing; a remote-only configuration has no local tier
        if local is None:
            raise ValueError("local_capacity_bytes needs a local tier; a remote-only configuration has none")
        if local in ("cpu", "cuda") and not compressed_host:
            raise ValueError(f"local_capacity_bytes is honoured by the CacheGen tiers only (local_device='cpu' with "
                             f"local_serde='cachegen', or a directory), and by their lossless forms "
                             f"(local_serde='lossless'), not by local_device={local!r}")
    if config.device_cache_bytes is not None:
        # the device level keeps copies of containers: only the container local tiers have any
        if local is None:
            raise ValueError("device_cache_bytes needs a local CacheGen tier; a remote-only configuration has none")
        if local in ("cpu", "cuda") and not compressed_host:
            raise ValueError(f"device_cache_bytes is honoured by the CacheGen tiers only (local_device='cpu' with "
                             f"local_serde='cachegen', or a directory), and by their lossless forms "
                             f"(local_serde='lossless'), not by local_device={local!r}")
    if config.local_serde == "lossless" and local not in (None, "cuda"):
        # the compressed host tier or the disk tier holds lossless containers: one container per chunk
        from lmcache_b200.storage_backend.serde.lossless import _check_chunk_size
        _check_chunk_size(config)
    if config.reshard_world_sizes is not None:
        # another layout's chunks exist only on a shared remote tier, and only containers can be decoded a window of
        # heads at a time: CacheGen ones, or lossless ones when the configuration opts in (reshard_lossless)
        lossless = config.remote_serde == "lossless" and config.reshard_lossless
        if remote is None or not (config.remote_serde == "cachegen" or lossless):
            raise ValueError("reshard_world_sizes needs a remote tier with remote_serde='cachegen', or with "
                             "remote_serde='lossless' and reshard_lossless=True, not "
                             f"remote_url={remote!r} with remote_serde={config.remote_serde!r}")
    if local is None and isinstance(remote, str):
        from lmcache_b200.storage_backend.remote_backend import LMCPipelinedRemoteBackend, LMCRemoteBackend
        return (LMCPipelinedRemoteBackend if config.pipelined_backend else LMCRemoteBackend)(config, metadata)
    if isinstance(local, str) and remote is None:
        if compressed_host:
            from lmcache_b200.storage_backend.local_backend import LMCLocalCompressedBackend
            return LMCLocalCompressedBackend(config, metadata)
        if local in ("cpu", "cuda"):
            from lmcache_b200.storage_backend.local_backend import LMCLocalBackend
            return LMCLocalBackend(config, metadata)
        # a directory: the disk tier (LMCLocalDiskBackend, local_backend.py:163-310), here with CacheGen containers, or
        # lossless ones with local_serde="lossless"
        from lmcache_b200.storage_backend.local_backend import LMCLocalDiskBackend
        return LMCLocalDiskBackend(config, metadata)
    if isinstance(local, str) and isinstance(remote, str):
        from lmcache_b200.storage_backend.hybrid_backend import LMCHybridBackend
        return LMCHybridBackend(config, metadata)
    raise ValueError(f"Invalid configuration: {config}")


__all__ = ["CreateStorageBackend", "LMCBackendInterface"]
