"""LosslessSerializer / LosslessDeserializer -- the `lossless` serde: KV chunks in lossless B2KV containers (versions 5
and 6, include/b200kv.h), coded and decoded on the GPU by LosslessCodec.  A decode gives back the stored bits exactly, in
the stored dtype (bf16, fp16, or one-byte: uint8, float8_e4m3fn, float8_e5m2); a KV of another dtype is refused.

The plugins carry the same engine fast-path methods as the CacheGen serde (view_to_bytes_batch, view_to_pinned_batch,
decode_into, container_bound, .codec), so the remote tier runs its striped pipelines with them: k connections,
pipelined fetch / upload / decode, and non-blocking stores that read the caller's KV in stream order."""
from typing import List, Optional, Sequence

import torch

from lmcache_b200 import _native as N
from lmcache_b200.codec import NATIVE_DTYPES, KvView, LosslessCodec, dtype_of_code, parse_lossless_header
from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
from lmcache_b200.storage_backend.serde.serde import Deserializer, Serializer


def _check_chunk_size(config: LMCacheEngineConfig) -> None:
    if not 0 < config.chunk_size <= N.LOSSLESS_MAX_TOKENS:
        raise ValueError(f"chunk_size {config.chunk_size}: a lossless container holds at most {N.LOSSLESS_MAX_TOKENS} "
                         f"tokens")


class LosslessSerializer(Serializer):

    def __init__(self, config: LMCacheEngineConfig, metadata: LMCacheEngineMetadata):
        _check_chunk_size(config)
        self.chunk_size = config.chunk_size
        self.fmt = metadata.fmt
        if self.fmt not in ("vllm", "huggingface"):
            raise RuntimeError("Unknown format %s" % self.fmt)
        self.codec = LosslessCodec()

    def _view(self, tensor: torch.Tensor) -> KvView:
        if tensor.dtype not in NATIVE_DTYPES:
            raise TypeError(f"the lossless serde codes bfloat16 and float16 KV and one-byte KV (uint8, float8_e4m3fn, "
                            f"float8_e5m2) only, not {tensor.dtype}")
        if not tensor.is_cuda:
            tensor = tensor.cuda()
        return KvView.from_blob(tensor, self.fmt)

    def to_bytes(self, tensor: torch.Tensor) -> bytes:
        """tensor: [L,2,t,H,D] (vllm) / [L,2,H,t,D] (huggingface) chunk, or a latent [L,t,D] -> one container"""
        view = self._view(tensor)
        return self.codec.encode_to_host(view, 0, view.ntokens, view.ntokens)[0]

    def view_to_bytes_batch(self, view: KvView, chunk_size: Optional[int] = None, tok_begin: int = 0,
                            n_tokens: Optional[int] = None) -> List[bytes]:
        """Engine fast path: tokens [tok_begin, tok_begin + n_tokens) of a KvView, one container per chunk."""
        n = view.ntokens - tok_begin if n_tokens is None else n_tokens
        return self.codec.encode_to_host(view, tok_begin, n, chunk_size or self.chunk_size)

    def view_to_pinned_batch(self, view: KvView, chunk_size: Optional[int] = None, tok_begin: int = 0,
                             n_tokens: Optional[int] = None):
        """Same, as a context manager yielding memoryviews over the codec's page-locked slab."""
        n = view.ntokens - tok_begin if n_tokens is None else n_tokens
        return self.codec.encode_to_pinned(view, tok_begin, n, chunk_size or self.chunk_size)


class LosslessDeserializer(Deserializer):

    def __init__(self, config: LMCacheEngineConfig, metadata: LMCacheEngineMetadata):
        _check_chunk_size(config)
        self.chunk_size = config.chunk_size
        self.fmt = metadata.fmt
        if self.fmt not in ("vllm", "huggingface"):
            raise RuntimeError("Unknown format %s" % self.fmt)
        self.codec = LosslessCodec()

    def from_bytes(self, bs) -> torch.Tensor:
        """one container -> its chunk blob in the stored dtype: [L,2,t,H,D] / [L,2,H,t,D], or [L,t,D] for version 6"""
        hd = parse_lossless_header(bs)
        latent = hd.version == 6
        out = torch.empty(KvView.blob_shape(self.fmt, hd.L, hd.H, hd.D, hd.ntokens, latent),
                          dtype=dtype_of_code(hd.max_dtype), device=torch.device("cuda", torch.cuda.current_device()))
        self.codec.decode([bs], KvView.from_blob(out, self.fmt), [0])
        return out

    def decode_into(self, containers: Sequence, dst: KvView, dst_tok: Sequence[int]) -> None:
        """Engine fast path: decode containers straight into a destination view at the given token offsets."""
        self.codec.decode(list(containers), dst, list(dst_tok))

    def out_dtype(self) -> None:
        """None: a lossless container is decoded into the dtype it was stored in."""
        return None

    def container_bound(self, L: int, H: int, D: int, chunk_tokens: int, latent: bool = False) -> int:
        """Upper bound of one container's size (what a receive slab must reserve per chunk)."""
        return self.codec.max_container_bytes(L, H, D, chunk_tokens, latent)

    def pinned_staging(self, nbytes: int):
        return self.codec.pinned_staging(nbytes)
