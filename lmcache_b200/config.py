"""Engine configuration / metadata types -- same names, fields, constructors and validation
as lmcache/config.py:8-139 so existing callers (lmcache-vllm adapter, YAML files) keep working."""
from __future__ import annotations

import re
from dataclasses import dataclass
from typing import Dict, List, Optional

import yaml

_DISK_RE = re.compile(r"file://(.*)/")
_URL_RE = re.compile(r"(.*)://(.*):(\d+)")


@dataclass
class LMCacheEngineMetadata:
    model_name: str   # LLM name; selects the CacheGen bin table
    world_size: int   # tensor-parallel world size (part of the key)
    worker_id: int    # tensor-parallel rank (part of the key)
    fmt: str          # "vllm" | "huggingface"
    dtype: str        # dtype of the kv tensors
    # not in the reference: the model caches one latent vector per token and layer (multi-head latent attention,
    # DeepSeek-V2/V3) instead of a (K, V) pair.  The engine then takes and returns one [T, D] tensor per layer, its
    # CacheGen tiers keep version-4 containers, and every tensor-parallel rank uses the keys of rank 0 of a one-rank
    # layout: the latent is the same on every rank, so one copy serves all of them (LMCacheEngine).
    use_mla: bool = False


@dataclass
class LMCacheEngineConfig:
    chunk_size: int
    local_device: Optional[str]
    remote_url: Optional[str]
    remote_serde: Optional[str]   # "torch" | "cachegen" | ...
    pipelined_backend: bool
    save_decode_cache: bool
    # not in the reference: how the LOCAL host tier keeps chunks.  None = raw blobs, as the reference does
    # (local_backend.py:95-100); "cachegen" = CacheGen containers in page-locked memory (LMCLocalCompressedBackend);
    # "lossless" = lossless containers (versions 5 and 6), in page-locked memory or, for a directory, in the files of the
    # disk tier, which are CacheGen containers otherwise.  The environment variable LMCACHE_B200_LOCAL_SERDE sets the
    # default for configurations that do not name it.
    local_serde: Optional[str] = None
    # not in the reference: the most bytes the local CacheGen tier keeps (slab blocks of the host tier, .b2kv files of the
    # disk tier); beyond it chunks are evicted from the tail of the coldest chain (lmcache_b200/eviction.py).  None = no
    # bound.  Only the two CacheGen tiers and their lossless forms honour it (CreateStorageBackend rejects it elsewhere).
    local_capacity_bytes: Optional[int] = None
    # not in the reference: bytes of device memory that keep copies of the local CacheGen tier's containers, so that a
    # retrieve of a resident chunk decodes it in place instead of uploading it (lmcache_b200/device_cache.py).  None =
    # off.  The level is inclusive: every device copy has its tier copy beside it.  Only the two CacheGen tiers and their
    # lossless forms take it.
    device_cache_bytes: Optional[int] = None
    # not in the reference: other tensor-parallel world sizes whose stored chunks a retrieve may decode into this rank's
    # KV heads once its own layout's prefix ends (lmcache_b200/reshard.py), tried in this order.  None = off.  Needs a
    # remote tier with the CacheGen serde, or with the lossless serde and reshard_lossless (CreateStorageBackend).  Must
    # not hold the engine's own world size (LMCacheEngine).
    reshard_world_sizes: Optional[List[int]] = None
    # not in the reference as a key (it is the reference's nine-field CacheGenConfig): the CacheGen bin layout of a model
    # outside the five-name table of CacheGenConfig.from_model_name, e.g. a 70B model's 80 layers.  A mapping of exactly
    # the nine fields; None = the table.  When set, the engine's CacheGen tiers and serdes use it for any model name, and
    # write and read version-3 containers only -- the one version that records the bins (chunk_size <= 256).
    cachegen_config: Optional[Dict[str, int]] = None
    # not in the reference: with remote_serde "lossless", let reshard_world_sizes decode other layouts' lossless
    # containers (b200kv_lossless_decode_plan_heads): this rank's heads come back bit for bit as it would have stored them.
    # False = a lossless remote tier refuses reshard_world_sizes, as it did before the key existed; True needs
    # reshard_world_sizes and remote_serde "lossless", and every layout named there must store lossless containers too.
    reshard_lossless: bool = False

    def __post_init__(self):
        if self.local_serde is None:
            import os
            self.local_serde = os.environ.get("LMCACHE_B200_LOCAL_SERDE") or None
        if self.local_serde not in (None, "cachegen", "lossless"):
            raise ValueError(f"Invalid local serde: {self.local_serde}")
        c = self.local_capacity_bytes
        if c is not None and (isinstance(c, bool) or not isinstance(c, int) or c <= 0):
            raise ValueError(f"Invalid local capacity: {c!r} (a positive number of bytes, or None)")
        d = self.device_cache_bytes
        if d is not None and (isinstance(d, bool) or not isinstance(d, int) or d <= 0):
            raise ValueError(f"Invalid device cache size: {d!r} (a positive number of bytes, or None)")
        r = self.reshard_world_sizes
        if r is not None and (not isinstance(r, (list, tuple)) or not r or len(set(r)) != len(r) or
                              any(isinstance(w, bool) or not isinstance(w, int) or w <= 0 for w in r)):
            raise ValueError(f"Invalid reshard world sizes: {r!r} (a non-empty list of distinct positive ints, or None)")
        if r is not None:
            self.reshard_world_sizes = list(r)
        if self.cachegen_config is not None:
            self.cachegen_config = check_cachegen_config(self.cachegen_config)
        if not isinstance(self.reshard_lossless, bool):
            raise ValueError(f"Invalid reshard_lossless: {self.reshard_lossless!r} (True or False)")
        if self.reshard_lossless and (self.reshard_world_sizes is None or self.remote_serde != "lossless"):
            raise ValueError("reshard_lossless needs reshard_world_sizes and remote_serde='lossless', not "
                             f"reshard_world_sizes={self.reshard_world_sizes!r} with remote_serde={self.remote_serde!r}")

    @staticmethod
    def from_defaults(chunk_size: int = 256, local_device: str = "cuda",
                      remote_url: str = "redis://localhost:6379", remote_serde: str = "torch",
                      pipelined_backend: bool = False, save_decode_cache: bool = False,
                      local_serde: Optional[str] = None,
                      local_capacity_bytes: Optional[int] = None,
                      device_cache_bytes: Optional[int] = None,
                      reshard_world_sizes: Optional[List[int]] = None,
                      cachegen_config: Optional[Dict[str, int]] = None,
                      reshard_lossless: bool = False) -> "LMCacheEngineConfig":
        return LMCacheEngineConfig(chunk_size, local_device, remote_url, remote_serde, pipelined_backend,
                                   save_decode_cache, local_serde, local_capacity_bytes, device_cache_bytes,
                                   reshard_world_sizes, cachegen_config, reshard_lossless)

    @staticmethod
    def from_legacy(chunk_size: int = 256, backend: str = "cuda", persist_path: Optional[str] = None,
                    remote_serde: Optional[str] = "torch", pipelined_backend: bool = False,
                    save_decode_cache: bool = False, local_serde: Optional[str] = None,
                    local_capacity_bytes: Optional[int] = None,
                    device_cache_bytes: Optional[int] = None,
                    reshard_world_sizes: Optional[List[int]] = None,
                    cachegen_config: Optional[Dict[str, int]] = None,
                    reshard_lossless: bool = False) -> "LMCacheEngineConfig":
        """backend: "cpu" | "cuda" | "file://<dir>/" | "<scheme>://<host>:<port>" (config.py:51-82)."""
        local_device: Optional[str] = None
        remote_url: Optional[str] = None
        if backend in ("cpu", "cuda"):
            local_device = backend
        elif _DISK_RE.match(backend):
            local_device = backend[7:]
        elif _URL_RE.match(backend):
            remote_url = backend
        return LMCacheEngineConfig(chunk_size, local_device, remote_url, remote_serde, pipelined_backend,
                                   save_decode_cache, local_serde, local_capacity_bytes, device_cache_bytes,
                                   reshard_world_sizes, cachegen_config, reshard_lossless)

    @staticmethod
    def from_file(file_path: str) -> "LMCacheEngineConfig":
        """YAML loader with the reference's validation rules (config.py:84-124)."""
        with open(file_path, "r") as fin:
            cfg = yaml.safe_load(fin)
        chunk_size = cfg.get("chunk_size", 256)
        local_device = cfg.get("local_device", None)
        remote_url = cfg.get("remote_url", None)
        remote_serde = cfg.get("remote_serde", "torch")
        pipelined_backend = cfg.get("pipelined_backend", False)
        save_decode_cache = cfg.get("save_decode_cache", False)
        local_serde = cfg.get("local_serde", None)
        local_capacity_bytes = cfg.get("local_capacity_bytes", None)
        device_cache_bytes = cfg.get("device_cache_bytes", None)
        reshard_world_sizes = cfg.get("reshard_world_sizes", None)
        cachegen_config = cfg.get("cachegen_config", None)
        reshard_lossless = cfg.get("reshard_lossless", False)

        if local_device in ("cpu", "cuda", None):
            pass
        elif isinstance(local_device, str) and _DISK_RE.match(local_device):
            local_device = local_device[7:]
        else:
            raise ValueError(f"Invalid local storage device: {local_device}")

        if remote_url is not None and not (isinstance(remote_url, str) and _URL_RE.match(remote_url)):
            raise ValueError(f"Invalid remote storage url: {remote_url}")

        return LMCacheEngineConfig(chunk_size, local_device, remote_url, remote_serde, pipelined_backend,
                                   save_decode_cache, local_serde, local_capacity_bytes, device_cache_bytes,
                                   reshard_world_sizes, cachegen_config, reshard_lossless)


CACHEGEN_CONFIG_FIELDS = ("key_first_layers", "key_second_layers", "key_third_layers", "key_first_bins",
                          "key_second_bins", "key_third_bins", "value_first_layers", "value_first_bins",
                          "value_second_bins")
MAX_LAYERS = 128        # B200KV_MAX_PLANES / 2
MIN_BINS, MAX_BINS = 4, 32      # the quantiser range of the kernels: bins // 2 - 1 in [1, 15]


def check_cachegen_config(c) -> Dict[str, int]:
    """The nine CacheGenConfig fields of `c` (a mapping, or a CacheGenConfig) as a plain dict, or ValueError.
    key_third_layers is the model's layer count (1..128); every bin count that some layer gets lies in [4, 32].
    Layer i's key bins are key_first_bins for i < key_first_layers, else key_second_bins for i < key_second_layers,
    else key_third_bins; its value bins value_first_bins for i < value_first_layers, else value_second_bins
    (make_key_bins / make_value_bins of the reference)."""
    import dataclasses
    from collections.abc import Mapping
    if dataclasses.is_dataclass(c) and not isinstance(c, type):
        c = dataclasses.asdict(c)
    if not isinstance(c, Mapping) or set(c) != set(CACHEGEN_CONFIG_FIELDS):
        raise ValueError(f"Invalid cachegen_config: {c!r} (a mapping of exactly the fields {', '.join(CACHEGEN_CONFIG_FIELDS)})")
    for k in CACHEGEN_CONFIG_FIELDS:
        if isinstance(c[k], bool) or not isinstance(c[k], int):
            raise ValueError(f"Invalid cachegen_config: {k} = {c[k]!r} is not an int")
    c = {k: int(c[k]) for k in CACHEGEN_CONFIG_FIELDS}
    L = c["key_third_layers"]
    if not 1 <= L <= MAX_LAYERS:
        raise ValueError(f"Invalid cachegen_config: key_third_layers = {L} (the layer count, 1..{MAX_LAYERS})")
    for k in ("key_first_layers", "key_second_layers", "value_first_layers"):
        if c[k] < 0:
            raise ValueError(f"Invalid cachegen_config: {k} = {c[k]} is negative")
    k1, k2 = min(c["key_first_layers"], L), min(c["key_second_layers"], L)
    v1 = min(c["value_first_layers"], L)
    applies = {"key_first_bins": k1 > 0, "key_second_bins": k2 > k1, "key_third_bins": L > max(k1, k2),
               "value_first_bins": v1 > 0, "value_second_bins": L > v1}
    for k, used in applies.items():
        if used and not MIN_BINS <= c[k] <= MAX_BINS:
            raise ValueError(f"Invalid cachegen_config: {k} = {c[k]} (bins must lie in [{MIN_BINS}, {MAX_BINS}])")
    return c


class GlobalConfig:
    """Process-wide switches (config.py:130-139)."""
    enable_debug: bool = True

    @classmethod
    def set_debug(cls, enable: bool):
        cls.enable_debug = enable

    @classmethod
    def is_debug(cls) -> bool:
        return cls.enable_debug
