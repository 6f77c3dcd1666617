"""CacheGenSerializer -- the encode-side serde plugin (lmcache/storage_backend/serde/cachegen_encoder.py:328-389).

The reference's to_bytes runs ~25 torch launches + 3 torchac_cuda kernels + a pickle of CUDA tensors per
256 tokens.  Here to_bytes is: one b200kv_encode_chunks call (absmax -> fused quantise/CDF/arithmetic-code/
compact -> header) + one device->host copy of the finished container.
"""
from typing import List, Optional, Sequence

import torch

from lmcache_b200.codec import KvView, engine_codec
from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
from lmcache_b200.storage_backend.serde.cachegen_basics import CacheGenConfig
from lmcache_b200.storage_backend.serde.serde import Serializer
from lmcache_b200.utils import _lmcache_nvtx_annotate


class CacheGenSerializer(Serializer):

    def __init__(self, config: LMCacheEngineConfig, metadata: LMCacheEngineMetadata):
        # ValueError for models outside the bin table, like the reference (cachegen_basics.py:77-78), unless
        # config.cachegen_config gives the layout
        self.cachegen_config = CacheGenConfig.for_engine(metadata.model_name, config.cachegen_config)
        self.chunk_size = config.chunk_size
        self.fmt = metadata.fmt
        self.codec = engine_codec(config, metadata.model_name)
        self.key_bins = torch.tensor(self.cachegen_config.key_bins_list())
        self.value_bins = torch.tensor(self.cachegen_config.value_bins_list())

    def _view(self, tensor: torch.Tensor) -> KvView:
        if not tensor.is_cuda:
            tensor = tensor.cuda()   # reference: tensor.cuda() at cachegen_encoder.py:383
        return KvView.from_blob(tensor, self.fmt)   # hf layout handled by strides, no permute copy (:377-378)

    @_lmcache_nvtx_annotate
    def to_bytes(self, tensor: torch.Tensor) -> bytes:
        """tensor: [L,2,t,H,D] (vllm) / [L,2,H,t,D] (huggingface) chunk -> one B2KV container."""
        view = self._view(tensor)
        return self.codec.encode_to_host(view, 0, view.ntokens, view.ntokens)[0]

    @_lmcache_nvtx_annotate
    def to_bytes_batch(self, tensor: torch.Tensor, chunk_size: Optional[int] = None) -> List[bytes]:
        """Encode a multi-chunk blob in one launch: tokens are split into `chunk_size` chunks, each an
        independent container (what LMCacheEngine.store feeds the backend chunk by chunk)."""
        view = self._view(tensor)
        return self.codec.encode_to_host(view, 0, view.ntokens, chunk_size or self.chunk_size)

    @_lmcache_nvtx_annotate
    def kv_to_bytes_batch(self, kv: Sequence, chunk_size: Optional[int] = None, tok_begin: int = 0,
                          n_tokens: Optional[int] = None) -> List[bytes]:
        """Same, straight from the engine's tuple of per-layer (K, V) tensors (no blob is ever built)."""
        return self.view_to_bytes_batch(KvView.from_tuple(kv, self.fmt), chunk_size, tok_begin, n_tokens)

    @_lmcache_nvtx_annotate
    def view_to_bytes_batch(self, view: KvView, chunk_size: Optional[int] = None, tok_begin: int = 0,
                            n_tokens: Optional[int] = None) -> List[bytes]:
        """Engine fast path: encode tokens [tok_begin, tok_begin + n_tokens) of a KvView, one container per chunk,
        with one launch sequence and one device->host copy pass."""
        n = view.ntokens - tok_begin if n_tokens is None else n_tokens
        return self.codec.encode_to_host(view, tok_begin, n, chunk_size or self.chunk_size)

    def view_to_pinned_batch(self, view: KvView, chunk_size: Optional[int] = None, tok_begin: int = 0,
                             n_tokens: Optional[int] = None):
        """Same, as a context manager yielding memoryviews over the codec's page-locked slab: a connector can send the
        containers from where the device->host copy put them (no bytes objects, no extra host copy)."""
        n = view.ntokens - tok_begin if n_tokens is None else n_tokens
        return self.codec.encode_to_pinned(view, tok_begin, n, chunk_size or self.chunk_size)
