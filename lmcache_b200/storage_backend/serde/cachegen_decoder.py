"""CacheGenDeserializer -- the decode-side serde plugin (lmcache/storage_backend/serde/cachegen_decoder.py:109-202).

from_bytes = one host->device copy of the container + one decode (b200kv_decode_plan + _layers) that writes the final
bf16 (vllm) / fp16 (huggingface) blob directly (no uint8 / fp32 intermediates, no stack/permute/cast passes).
"""
from typing import List, Optional, Sequence

import torch

from lmcache_b200.codec import KvView, engine_codec, parse_header
from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
from lmcache_b200.storage_backend.serde.cachegen_basics import CacheGenConfig
from lmcache_b200.storage_backend.serde.serde import Deserializer
from lmcache_b200.utils import _lmcache_nvtx_annotate


class CacheGenDeserializer(Deserializer):

    def __init__(self, config: LMCacheEngineConfig, metadata: LMCacheEngineMetadata):
        self.cachegen_config = CacheGenConfig.for_engine(metadata.model_name, config.cachegen_config)
        self.chunk_size = config.chunk_size
        self.fmt = metadata.fmt
        if self.fmt not in ("vllm", "huggingface"):
            raise RuntimeError("Unknown format %s" % self.fmt)
        self.codec = engine_codec(config, metadata.model_name)

    def _out_dtype(self) -> torch.dtype:
        # reference casts by format, ignoring metadata.dtype (cachegen_decoder.py:189-200)
        return torch.bfloat16 if self.fmt == "vllm" else torch.float16

    def _alloc(self, L: int, H: int, D: int, t: int, device, latent: bool = False) -> torch.Tensor:
        return torch.empty(KvView.blob_shape(self.fmt, L, H, D, t, latent), dtype=self._out_dtype(), device=device)

    @_lmcache_nvtx_annotate
    def from_bytes(self, bs) -> torch.Tensor:
        """one container -> its chunk blob: [L,2,t,H,D] / [L,2,H,t,D], or [L,t,D] for a version-4 (latent) one"""
        hd = parse_header(bs)
        out = self._alloc(hd.L, hd.H, hd.D, hd.ntokens, torch.device("cuda", torch.cuda.current_device()),
                          hd.version == 4)
        self.codec.decode([bs], KvView.from_blob(out, self.fmt), [0])
        return out

    @_lmcache_nvtx_annotate
    def decode_into(self, containers: Sequence, dst: KvView, dst_tok: Sequence[int]) -> None:
        """Engine fast path: decode containers straight into a destination view at the given token offsets."""
        self.codec.decode(list(containers), dst, list(dst_tok))

    def out_dtype(self) -> torch.dtype:
        return self._out_dtype()

    def container_bound(self, L: int, H: int, D: int, chunk_tokens: int, latent: bool = False) -> int:
        """Upper bound of one container's size (what a receive slab must reserve per chunk); `latent`: a version-4
        container of one plane per layer."""
        return self.codec.max_container_bytes(L, H, D, chunk_tokens, latent)

    def pinned_staging(self, nbytes: int):
        return self.codec.pinned_staging(nbytes)

    @_lmcache_nvtx_annotate
    def from_bytes_batch(self, containers: Sequence, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Decode consecutive chunks into ONE blob (the retrieve-side torch.cat disappears):
        container j lands at token offset sum(ntokens[:j])."""
        heads = [parse_header(c) for c in containers]
        total = sum(h.ntokens for h in heads)
        h0 = heads[0]
        if out is None:
            out = self._alloc(h0.L, h0.H, h0.D, total, torch.device("cuda", torch.cuda.current_device()))
        offs, o = [], 0
        for h in heads:
            offs.append(o)
            o += h.ntokens
        self.codec.decode(list(containers), KvView.from_blob(out, self.fmt), offs)
        return out
