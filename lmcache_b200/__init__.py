"""lmcache_b200 -- H100-native KV-cache store/load hot path behind LMCache v0.1.2's
LMCacheEngine.store()/retrieve() + storage_backend + serde plugin surface.

Only the hot path is rebuilt (CacheGen encode/decode, chunk hash / prefix match, GPU<->pinned-host
mover); it runs as hand-written sm_90a CUDA in libb200kv.so (include/b200kv.h).  No CPU fallback.
"""
__version__ = "0.1.0"
