"""LMCacheEngine -- store()/retrieve() with the reference's signatures and semantics
(lmcache/cache_engine.py:16-436), rebuilt around the CUDA hot path:

  * chunk hashes: one b200kv_sha256_chain launch on the token ids (no per-chunk tokens.cpu() sync,
    cache_engine.py:58-96); digests are bit-identical to hashlib's.
  * blob pack + chunking: one b200kv_pack_chunks gather from the caller's 2L tensors straight into per-chunk
    blobs (replaces 3x torch.stack + permute + split + .contiguous() per chunk, :98-161).
  * retrieve assembles chunks into one preallocated blob (replaces torch.cat, :362-368).
Prefix-match / mask semantics are unchanged: chunks are matched front to back through `contains`, the first
miss ends the match, everything after the first missing chunk is (re)stored (:183-208).
"""
from __future__ import annotations

import ctypes
import threading
import time
from typing import Any, Callable, Dict, Iterable, List, Optional, Sequence, Tuple, Union

import torch

from lmcache_b200 import _native as N
from lmcache_b200.blend import (BatchBlendPlan, BlendPlan, BlendSpec, check_blend_args, check_blend_batch_args,
                                 check_blend_dtype)
from lmcache_b200.codec import NATIVE_DTYPES, KvView, PinnedBuffer, paged_layout
from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
from lmcache_b200.logging import init_logger
from lmcache_b200.storage_backend import CreateStorageBackend
from lmcache_b200.pipeline import (HeadWindow, LayerwiseUpload, SegmentsEncode, arena_of, begin_runs, join_uploads,
                                   layerwise_store_budget_default)
from lmcache_b200.reshard import first_source_rank, source_shards
from lmcache_b200.rope import (RopeSpec, Rotation, StagedGather, derived_digest, hash_input, pack_rope,
                                plan_segment_store, plan_segments, rope_shift, rope_table, seg_of_tok, skip_chunks)
from lmcache_b200.utils import CacheEngineKey, KVCache, _lmcache_nvtx_annotate

logger = init_logger(__name__)



def _bytes_of(t: torch.Tensor) -> torch.Tensor:
    """A one-byte (FP8) tensor as its bytes, any other as it is: the paged gathers and scatters index the bytes, as
    indexed reads and writes do not take every float8 dtype."""
    return t.view(torch.uint8) if t.element_size() == 1 else t

class LazySeq:
    """A read-only sequence whose items are computed on access: fn(base[i]).  Slices stay lazy.  The engine passes its
    chunk keys around in this form: item i only exists once the hash chain has reached chunk i (one chunk after another), and a
    consumer that walks the sequence front to back -- look up / fetch / encode wave by wave -- overlaps with the chain
    instead of waiting for its end."""

    def __init__(self, fn, base, start: int = 0, stop: Optional[int] = None):
        self._fn, self._base = fn, base
        self._start = start
        self._stop = len(base) if stop is None else stop

    def __len__(self) -> int:
        return self._stop - self._start

    def __getitem__(self, i):
        if isinstance(i, slice):
            a, b, step = i.indices(len(self))
            if step != 1:
                return [self[k] for k in range(a, b, step)]
            return LazySeq(self._fn, self._base, self._start + a, self._start + max(a, b))
        if i < 0:
            i += len(self)
        if not 0 <= i < len(self):
            raise IndexError(i)
        v = self._base[self._start + i]
        return v if self._fn is None else self._fn(v)

    def __iter__(self):
        for i in range(len(self)):
            yield self[i]


class _HashRun:
    """One hash-chain launch: digests and their ready words land in mapped page-locked memory; item i blocks (a short
    spin on the ready word) until the kernel has produced digest i."""
    _pool: List[PinnedBuffer] = []
    _pool_lock = threading.Lock()
    _epoch = 0
    _streams: dict = {}

    def __init__(self, dev_tokens: torch.Tensor, chunk_size: int, offs: List[int], nchunks: int):
        self.n = nchunks
        need = 36 * nchunks                                  # 32-byte digests, then one ready word each
        with _HashRun._pool_lock:
            _HashRun._epoch = (_HashRun._epoch % 0x7fffffff) + 1
            self.epoch = _HashRun._epoch
            # a pooled buffer whose own finaliser ran after it was pooled (both were garbage of one reference cycle,
            # such as an error's traceback that reaches this run) is closed: drop it, never hand it out
            _HashRun._pool = [b for b in _HashRun._pool if b.host_ptr]
            fit = [b for b in _HashRun._pool if b.nbytes >= need]
            if fit:
                self.buf = min(fit, key=lambda b: b.nbytes)
                _HashRun._pool.remove(self.buf)
            else:
                self.buf = PinnedBuffer(max(1 << 14, 2 * need))     # cudaHostAlloc zero-fills: no stale epoch inside
        self.cap = self.buf.nbytes // 36
        self._tokens = dev_tokens                            # alive until the kernel has run
        self._hex: List[Optional[str]] = [None] * nchunks
        self._flags = (ctypes.c_uint32 * self.cap).from_address(self.buf.host_ptr + 32 * self.cap)
        dev = dev_tokens.device
        with torch.cuda.device(dev):
            # its own stream: the chain is one warp on one SM; the caller's encode / decode kernels must not queue behind it
            side = _HashRun._streams.get(dev.index)
            if side is None:
                side = _HashRun._streams[dev.index] = torch.cuda.Stream(device=dev)
            ready = torch.cuda.Event()
            ready.record(torch.cuda.current_stream())
            side.wait_event(ready)
            N.check(N.lib().b200kv_sha256_chain_ready(ctypes.c_void_p(dev_tokens.data_ptr()), dev_tokens.element_size(),
                                                      N.i64_array(offs), len(offs) - 1, chunk_size,
                                                      ctypes.c_void_p(self.buf.dev_ptr),
                                                      ctypes.c_void_p(self.buf.dev_ptr + 32 * self.cap), self.epoch,
                                                      side.cuda_stream), "sha256_chain")
            self.done = torch.cuda.Event()
            self.done.record(side)
            dev_tokens.record_stream(side)

    def __len__(self) -> int:
        return self.n

    def __getitem__(self, i: int) -> str:
        h = self._hex[i]
        if h is None:
            spins = 0
            while self._flags[i] != self.epoch:
                spins += 1
                if spins % 4096 == 0 and self.done.query():
                    # the kernel is over: either the word is there now, or the launch failed
                    if self._flags[i] != self.epoch:
                        self.done.synchronize()
                        raise N.NativeError("hash chain kernel finished without producing every digest")
            h = self._hex[i] = bytes(self.buf.view(32 * i, 32)).hex()
        return h

    def __del__(self):
        try:
            if not self.done.query():
                self.done.synchronize()                      # the kernel still writes into the buffer
            with _HashRun._pool_lock:
                # a buffer the cyclic collector finalised first is closed already: it must not be handed out again
                if len(_HashRun._pool) < 8 and self.buf.host_ptr:
                    _HashRun._pool.append(self.buf)
                    self.buf = None
            if self.buf is not None:
                self.buf.close()
        except Exception:       # noqa: BLE001 -- interpreter shutdown
            pass


def sha256_prefix_chain_lazy(tokens: torch.Tensor, chunk_size: int, seq_offsets: Optional[List[int]] = None) -> LazySeq:
    """sha256_prefix_chain without waiting for the end of the chain: returns at once with a lazy sequence of hex digests;
    digest i becomes available once the chain has hashed chunks 0..i."""
    N.require_cuda()
    if tokens.dim() != 1:
        raise ValueError(f"Invalid shape of tokens: {tokens.shape}")
    n = tokens.shape[0]
    offs = [0, n] if seq_offsets is None else list(seq_offsets)
    n_seq = len(offs) - 1
    nchunks = sum((offs[i + 1] - offs[i] + chunk_size - 1) // chunk_size for i in range(n_seq))
    if nchunks == 0:
        return LazySeq(None, [])
    dev_tokens = tokens if tokens.is_cuda else tokens.to("cuda", non_blocking=False)
    return LazySeq(None, _HashRun(dev_tokens.contiguous(), chunk_size, offs, nchunks))


def sha256_prefix_chain(tokens: torch.Tensor, chunk_size: int, seq_offsets: Optional[List[int]] = None) -> List[str]:
    """Hex digests h_i = sha256(hex(h_{i-1}) || bytes(chunk_i)) for every chunk of every sequence
    (cache_engine.py:58-96), computed on the GPU.  tokens: 1-D integer tensor on any device; the bytes hashed
    are the tensor's native little-endian dtype, as in the reference.  seq_offsets: token boundaries of
    independent sequences (default: one sequence)."""
    return list(sha256_prefix_chain_lazy(tokens, chunk_size, seq_offsets))


class LayerwiseRetrieval:
    """What retrieve_layerwise / retrieve_paged_layerwise return: the hit is known (`ret_mask`, and for the blob form the
    per-layer (K, V) views `kv`, or an MLA engine's latent views), the KV arrives layer by layer.  Layer l may be read on a stream once wait_layer(l,
    stream) has been called -- what vLLM's KV connector does in wait_for_layer_load before attention layer l."""

    def __init__(self, ret_mask: torch.Tensor, kv: Optional[KVCache], num_layers: int, upload):
        self.ret_mask = ret_mask
        self.kv = kv                        # None for the paged form
        self.num_layers = num_layers
        self._upload = upload               # pipeline.LayerwiseUpload

    def wait_layer(self, layer: int, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Make `stream` (default: the current one) wait for layer `layer`.  Blocks the host only until the layer's
        decode has been enqueued, never until it has run.  A no-op when num_layers is 0: a total miss before the engine
        knew the model's geometry retrieved nothing, so there is no layer to wait for."""
        if self.num_layers == 0:
            return
        (stream or torch.cuda.current_stream()).wait_event(self._upload.ready(layer))

    def synchronize(self) -> None:
        """Block the host until every layer is in place."""
        if self.num_layers > 0:
            self._upload.ready(self.num_layers - 1).synchronize()     # the layers are decoded in order on one stream


class LayerwiseStore:
    """What store_layerwise / store_paged_layerwise return: a store whose KV is handed over one layer at a time, as
    vLLM's KV connector does with save_kv_layer after each attention layer and wait_for_save at the end of the forward
    pass.  save_layer(l, stream) says that layer l is written in `stream` order; finish(stream) completes the store.
    Neither waits on the host, except finish() on a lossless disk tier, which returns once the files are written, and on
    the remote and hybrid tiers, which returns once the server holds the containers, as the store() it replaced did (the
    tier's layerwise_store_blocking).  On the compressed host and disk tiers and the remote tier each layer is encoded
    on a side stream as soon as it is saved (pipeline.LayerwiseEncode), and on the raw cpu and cuda tiers packed into
    its chunk blobs (local_backend.RawLayerwiseStore); a hybrid tier does both parts so (once, when they keep the same
    containers); elsewhere save_layer only records the layer and finish() runs the ordinary store.  A handle dropped without finish() stores nothing and gives its device scratch back."""

    def __init__(self, num_layers: int, enc, on_finish: Callable):
        self.num_layers = num_layers
        self._enc = enc                     # pipeline.LayerwiseEncode, or None: nothing is encoded layer by layer
        self._on_finish = on_finish         # on_finish(stream, enc): publish / store, on the calling thread
        self._saved = [False] * num_layers
        self._finished = False

    def save_layer(self, layer: int, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Layer `layer` is complete in `stream` order (default: the current stream): its encode is enqueued behind an
        event on that stream.  ValueError for a layer out of range or saved before, or after finish()."""
        if self._finished:
            raise ValueError("save_layer after finish()")
        if not 0 <= layer < self.num_layers:
            raise ValueError(f"layer {layer} out of range [0, {self.num_layers})")
        if self._saved[layer]:
            raise ValueError(f"layer {layer} was saved before")
        self._saved[layer] = True
        if self._enc is not None:
            self._enc.encode_layer(layer, stream or torch.cuda.current_stream())

    def finish(self, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Complete the store: `stream` (default: the current stream) waits for the encode's last read of the KV, so
        the caller may overwrite the cache in that stream's order; the containers land on the tier's worker thread, and
        a later retrieve of these keys waits for them (a lossless disk tier waits here for its files to be written).
        ValueError, and nothing is stored, when a layer was never saved."""
        if self._finished:
            raise ValueError("finish() was called before")
        self._finished = True
        missing = [l for l, s in enumerate(self._saved) if not s]
        if missing:
            self.close()
            raise ValueError(f"finish() before layers {missing} were saved; nothing is stored")
        stream = stream or torch.cuda.current_stream()
        enc, self._enc = self._enc, None
        if enc is not None:
            stream.wait_event(enc.finish())
        self._on_finish(stream, enc)

    def close(self) -> None:
        """drop an unfinished store: its device scratch goes back to the tier's pool"""
        enc, self._enc = self._enc, None
        if enc is not None:
            enc.abandon()

    def __del__(self):
        try:
            self.close()
        except Exception:       # noqa: BLE001 -- interpreter shutdown
            pass


class LMCacheEngine:

    def __init__(self, config: LMCacheEngineConfig, metadata: LMCacheEngineMetadata):
        self.config = config
        self.metadata = metadata
        self.chunk_size = config.chunk_size
        self.save_decode_cache = config.save_decode_cache
        if config.reshard_world_sizes is not None and metadata.world_size in config.reshard_world_sizes:
            raise ValueError(f"reshard_world_sizes {config.reshard_world_sizes} holds this engine's own world size "
                             f"{metadata.world_size}: its chunks are served by the ordinary retrieve")
        self._mla = bool(getattr(metadata, "use_mla", False))
        if self._mla:
            self._check_mla_config(config, metadata)
        self.engine_ = CreateStorageBackend(config, metadata)
        self._reshard_counts: Dict[int, Dict[str, int]] = {}
        self._seg_stream: Optional[torch.cuda.Stream] = None    # the layer-wise segment store's gathers
        logger.debug(f"Current storage backend type {type(self.engine_)}")

    @staticmethod
    def _check_mla_config(config: LMCacheEngineConfig, metadata: LMCacheEngineMetadata) -> None:
        """the settings a latent KV (use_mla) rules out"""
        if metadata.fmt != "vllm":
            raise ValueError(f"use_mla: a latent KV has the vllm layout only, not fmt={metadata.fmt!r}")
        if config.reshard_world_sizes is not None:
            raise ValueError("use_mla: the keys of a latent KV are shared by every tensor-parallel size already, "
                             "reshard_world_sizes must be None")
        local = config.local_device
        # a directory keeps CacheGen containers unless local_serde is "lossless" (version 6 then, up to 4096 tokens)
        cachegen_tier = ((local == "cpu" and config.local_serde == "cachegen") or
                         (local not in (None, "cpu", "cuda") and config.local_serde != "lossless") or
                         (config.remote_url is not None and config.remote_serde == "cachegen"))
        if cachegen_tier and config.chunk_size > N.GROUP_TOKENS:
            raise ValueError(f"use_mla: a CacheGen tier keeps a latent KV in version-4 containers, which hold at most "
                             f"{N.GROUP_TOKENS} tokens; chunk_size is {config.chunk_size}")

    # ------------------------------------------------------------------ keys / hashes
    def _make_key(self, chunk_hash: str, fmt: str) -> CacheEngineKey:
        if self._mla:
            # every rank holds the same latent: one key for all of them, that of a one-rank layout
            return CacheEngineKey(fmt, self.metadata.model_name, 1, 0, chunk_hash)
        return CacheEngineKey(fmt, self.metadata.model_name, self.metadata.world_size, self.metadata.worker_id,
                              chunk_hash)

    def _first(self, kv) -> torch.Tensor:
        """the first tensor of a store's KV: layer 0's latent, or layer 0's K"""
        return kv[0] if self._mla else kv[0][0]

    def _tensors(self, kv) -> List[torch.Tensor]:
        return list(kv) if self._mla else [t for pair in kv for t in pair]

    def _num_tokens_in_kv(self, kv_tensors: Union[KVCache, torch.Tensor], fmt: str) -> int:
        if fmt not in ("vllm", "huggingface"):
            raise ValueError(f"Invalid format: {fmt}")
        if self._mla:
            return kv_tensors[0].shape[0]                                  # a layer's latent is [T, D]
        return kv_tensors[0][0].shape[KvView.token_dim(fmt) - 2]         # a layer's K is a blob without its [L, 2] dims

    def _check_kind(self, kv, what: str) -> None:
        """AssertionError unless `kv` holds one tensor per layer (a latent KV) on an MLA engine, a (K, V) pair per
        layer otherwise"""
        if self._mla:
            assert all(isinstance(t, torch.Tensor) for t in kv), \
                f"an MLA engine (use_mla) takes one latent tensor per layer in {what}, not (K, V) pairs"
        else:
            assert not any(isinstance(t, torch.Tensor) for t in kv), \
                f"a (K, V) engine takes a (K, V) pair per layer in {what}; latent tensors need use_mla"

    def _prefix_hash(self, tokens: torch.Tensor, num_skip_chunk: Optional[int] = 0):
        """All chunk digests of `tokens` (the whole chain is hashed, then the first num_skip_chunk digests are
        dropped, like cache_engine.py:86-96).  A lazy sequence: digest i is there once the chain has reached chunk i."""
        return sha256_prefix_chain_lazy(tokens, self.chunk_size)[num_skip_chunk or 0:]

    def _keys_of(self, chunk_hashes, fmt: str) -> LazySeq:
        return LazySeq(lambda h: self._make_key(h, fmt), chunk_hashes)

    # ------------------------------------------------------------------ blob helpers
    def _pack_chunks_torch(self, kv: KVCache, tok_begin: int, fmt: str) -> List[torch.Tensor]:
        """_tuple_kv_to_blob + _slice_kv_at with torch ops (cache_engine.py:98-161), for dtypes the kernels do not move"""
        if self._mla:
            blob = torch.stack(list(kv))                                   # [L, T, D]
        else:
            k = torch.stack([x[0] for x in kv])
            v = torch.stack([x[1] for x in kv])
            blob = torch.stack((k, v)).permute(1, 0, 2, 3, 4)
        tdim = KvView.token_dim(fmt, self._mla)
        blob = blob.narrow(tdim, tok_begin, blob.shape[tdim] - tok_begin)
        return [c.contiguous() for c in torch.split(blob, self.chunk_size, dim=tdim)]

    def _as_cuda_kv(self, kv_tensors_raw: KVCache) -> KVCache:
        if self._first(kv_tensors_raw).is_cuda:
            return kv_tensors_raw
        if self._mla:
            return tuple(x.cuda() for x in kv_tensors_raw)
        return tuple((k.cuda(), v.cuda()) for k, v in kv_tensors_raw)

    def _blob_to_tuple_kv(self, blob: torch.Tensor) -> KVCache:
        if self._mla:
            return tuple(torch.unbind(blob, dim=0))                        # L views [T, D] of the [L, T, D] blob
        return tuple((layer[0], layer[1]) for layer in torch.unbind(blob, dim=0))

    def _mover_paged(self, kv_caches) -> Optional[str]:
        """The layout of a paged (K, V) cache whose rows torch indexing cannot reach in place ("strided", "split"): its
        gathers and scatters go through the mover with a KvView.  None for the FlashAttention layout and latent caches."""
        if self._mla:
            return None
        kind = paged_layout(*kv_caches[0]).kind
        return None if kind == "flash" else kind

    def _stages_split(self, kv_caches) -> bool:
        """A split cache on a tier that reads KV views through the codec kernels (every container tier): its stores and
        retrieves go through one device blob of the raw bytes of the tokens moved (KvView.staged / unpack_blob).  The raw
        cpu and cuda tiers move a split view themselves (supports_split_view)."""
        if self._mover_paged(kv_caches) != "split":
            return False
        f = getattr(self.engine_, "supports_split_view", None)
        return not (f and f())

    def _flat_paged(self, kv_caches) -> list:
        """the paged caches as [num_slots, ...] views: per layer a latent cache, or a (key, value) pair"""
        if self._mla:
            return [c.reshape(-1, c.shape[-1]) for c in kv_caches]
        return [(k.reshape(-1, k.shape[-2], k.shape[-1]), v.reshape(-1, v.shape[-2], v.shape[-1])) for k, v in kv_caches]

    # ------------------------------------------------------------------ arguments and masks
    def _check_store_args(self, tokens: torch.Tensor, kv_tensors_raw: KVCache, fmt: str) -> None:
        assert len(tokens.shape) == 1, f"Invalid shape of tokens: {tokens.shape}"
        assert len(kv_tensors_raw) > 0, "Empty kv_tensors"
        self._check_kind(kv_tensors_raw, "kv_tensors_raw")
        assert len(tokens) == self._num_tokens_in_kv(kv_tensors_raw, fmt), \
            "Number of tokens in the kv cache does not match the input tokens"

    def _check_paged_args(self, tokens: torch.Tensor, slot_mapping: torch.Tensor, kv_caches=None) -> None:
        """The paged methods' argument checks; the stores pass their kv_caches, which are checked too."""
        if self.metadata.fmt != "vllm":
            raise ValueError(f"paged KV caches use the vllm layout, engine fmt is {self.metadata.fmt}")
        if kv_caches is not None:
            assert len(tokens.shape) == 1, f"Invalid shape of tokens: {tokens.shape}"
            assert len(kv_caches) > 0, "Empty kv_caches"
            self._check_kind(kv_caches, "kv_caches")
        assert len(tokens) == slot_mapping.numel(), "Number of slots does not match the input tokens"

    def _split_mask(self, tokens: torch.Tensor, mask: Optional[torch.Tensor]) -> Tuple[torch.Tensor, int, int, int]:
        """A retrieve's suffix mask (None: every token): (ret_mask with the masked-off tokens cleared, num_skip_tok
        masked-off tokens, num_skip_chunk whole chunks among them, extra masked-off tokens in the first chunk fetched)"""
        num_skip_tok = 0 if mask is None else int(len(mask) - torch.sum(mask))
        num_skip_chunk = num_skip_tok // self.chunk_size
        ret_mask = torch.ones_like(tokens, dtype=torch.bool)
        ret_mask[:num_skip_tok] = False
        return ret_mask, num_skip_tok, num_skip_chunk, num_skip_tok - num_skip_chunk * self.chunk_size

    @staticmethod
    def _trim_mask(ret_mask: torch.Tensor, num_skip_tok: int, n_tok: int) -> torch.Tensor:
        """ret_mask of a retrieve that got the n_tok tokens after the masked-off ones (none if n_tok <= 0)"""
        if n_tok <= 0:
            ret_mask[:] = False
        else:
            ret_mask[num_skip_tok + n_tok:] = False
        return ret_mask

    # ------------------------------------------------------------------ store
    def _skip_scan(self, chunk_hashes, fmt: str) -> int:
        """store()'s skip_existing scan: the first chunk whose key the tier does not hold"""
        for i, h in enumerate(chunk_hashes):
            if not self.engine_.contains(self._make_key(h, fmt)):
                return i
        return len(chunk_hashes)

    def _store_put(self, chunk_hashes, start: int, fmt: str, put: Optional[Callable]) -> int:
        """Every store after its scan: touch the matched chunks [0, start), put(keys, tok_begin) the rest if there is
        any (and put is not None), then touch the whole chain.  Returns the number of chunks put."""
        self._touch(chunk_hashes[:start], fmt)
        if put is None or start == len(chunk_hashes):
            return 0
        n = put(self._keys_of(chunk_hashes[start:], fmt), start * self.chunk_size)
        self._touch(chunk_hashes, fmt)
        return n

    @_lmcache_nvtx_annotate
    @torch.no_grad()
    def store(self, tokens: torch.Tensor, kv_tensors_raw: KVCache, skip_existing=True, blocking=True) -> None:
        """Store the KV cache of `tokens`.  kv_tensors_raw: nested tuple of per-layer (K, V), each
        [num_tokens, num_heads, head_size] (vllm) or [num_heads, num_tokens, head_size] (huggingface),
        without a batch dimension.  An MLA engine (metadata.use_mla) takes one latent [num_tokens, D] per layer."""
        start_time = time.perf_counter()
        fmt = self.metadata.fmt
        self._check_store_args(tokens, kv_tensors_raw, fmt)
        chunk_hashes = self._prefix_hash(tokens)
        start = self._skip_scan(chunk_hashes, fmt) if skip_existing else 0

        def put(keys, tok_begin):
            kv_cuda = self._as_cuda_kv(kv_tensors_raw)
            if self._first(kv_cuda).dtype not in NATIVE_DTYPES:
                # the native pack / codec kernels move 16-bit and one-byte (FP8) KV; any other dtype (the reference's
                # local and torch-serde paths accept every dtype) takes the reference's own blob ops on the GPU
                # (cache_engine.py:98-161)
                chunks = self._pack_chunks_torch(kv_cuda, tok_begin, fmt)
                return self.engine_.batched_put(zip(keys, chunks), blocking=blocking)
            view = KvView.from_tuple(kv_cuda, fmt)
            self._geom = (view.L, view.H, view.D, view.dtype)
            if self._fast_path():
                # native path: the backend consumes the caller's 2L tensors directly (batched encode / one gather)
                return self.engine_.put_kv_chunks(keys, view, tok_begin, self.chunk_size, blocking=blocking)
            _, chunks = view.pack_chunks(tok_begin, self.chunk_size)
            return self.engine_.batched_put(zip(keys, chunks), blocking=blocking)
        n_chunks = self._store_put(chunk_hashes, start, fmt, put)
        logger.info(f"Stored/updated {n_chunks} chunks, total time {time.perf_counter() - start_time:.2f}s")

    # ------------------------------------------------------------------ retrieve
    @_lmcache_nvtx_annotate
    @torch.no_grad()
    def retrieve(self, tokens: torch.Tensor, mask: Optional[torch.Tensor] = None) -> Tuple[KVCache, torch.Tensor]:
        """Retrieve the longest cached prefix of `tokens` (optionally only the suffix selected by a boolean
        suffix `mask`).  Returns (kv tuple -- empty tuple on a total miss, ret_mask marking retrieved tokens).  An MLA
        engine returns one latent [T, D] per layer: views of one [L, T, D] blob."""
        return self._retrieve(tokens, mask)

    def _retrieve(self, tokens, mask, get_kv=None) -> Tuple[KVCache, torch.Tensor]:
        """retrieve(); get_kv(keys, view, tok0, chunk_size) -> chunks decoded fetches this layout's chunks on the native
        path (default: the backend's get_kv_into).  A get_kv comes from _layerwise_get, which has checked that path."""
        ret_mask, num_skip_tok, num_skip_chunk, extra = self._split_mask(tokens, mask)
        st = time.perf_counter()
        fmt = self.metadata.fmt
        if fmt not in ("vllm", "huggingface"):
            raise ValueError(f"Invalid format: {fmt}")
        full_chain = self._prefix_hash(tokens)
        chunk_hashes = full_chain[num_skip_chunk:]
        native = get_kv is not None or self._fast_path()
        if native and len(chunk_hashes) > 0 and not getattr(self, "_wide_dtype", False):
            try:
                return self._retrieve_into_blob(tokens, full_chain, ret_mask, num_skip_tok, num_skip_chunk, extra, fmt,
                                                st, get_kv)
            except TypeError:
                self._wide_dtype = True      # chunks of a dtype the kernels do not move: per-chunk path from now on
        retrieved: List[torch.Tensor] = []
        for chunk in self.engine_.batched_get(self._make_key(h, fmt) for h in chunk_hashes):
            # a blob of the other kind (a latent [L,t,D] for a (K, V) engine, or the reverse) is a miss
            if chunk is None or chunk.dim() != (3 if self._mla else 5):
                break
            retrieved.append(chunk)
        self._touch(full_chain[:num_skip_chunk + len(retrieved)], fmt)
        if len(retrieved) == 0:
            logger.info("Retrieved 0 chunks")
            return (), self._trim_mask(ret_mask, num_skip_tok, 0)

        # assemble into one blob; drop the extra leading tokens of the first chunk (suffix mask)
        tdim = KvView.token_dim(fmt, self._mla)
        sizes = [c.shape[tdim] for c in retrieved]
        total = sum(sizes) - extra
        first = retrieved[0]
        shape = list(first.shape)
        shape[tdim] = total
        blob = torch.empty(shape, dtype=first.dtype, device=first.device)
        pos = 0
        for i, c in enumerate(retrieved):
            src = c.narrow(tdim, extra, sizes[i] - extra) if i == 0 else c
            n = src.shape[tdim]
            blob.narrow(tdim, pos, n).copy_(src)
            pos += n
        logger.info(f"Retrieved {len(retrieved)} chunks ({total} tokens in total) -- "
                    f"elapsed time {time.perf_counter() - st}")
        return self._blob_to_tuple_kv(blob), self._trim_mask(ret_mask, num_skip_tok, total)

    # ------------------------------------------------------------------ paged KV caches, in place
    @_lmcache_nvtx_annotate
    @torch.no_grad()
    def store_paged(self, tokens: torch.Tensor, kv_caches, slot_mapping: torch.Tensor, skip_existing=True,
                    blocking=True) -> None:
        """store() for a vLLM paged KV cache: token i's K/V live in row slot_mapping[i] of every layer's
        (key_cache, value_cache) [num_blocks, block_size, H, D].  What lmcache-vllm's lmcache_store_kv does with a
        torch gather per layer + store() (LLM_Engine.rst:91-99); here the backend's kernels read the cache rows
        directly (cachegen: quantise + code from the rows; local tiers: one gather straight into the chunk blobs).
        An MLA engine takes one latent cache [num_blocks, block_size, D] (or [num_slots, D]) per layer."""
        self._check_paged_args(tokens, slot_mapping, kv_caches)
        if not self._fast_path():
            if self._mover_paged(kv_caches):
                # the mover gathers the rows a torch index cannot reach in place
                blob = KvView.from_paged(kv_caches, slot_mapping.cuda()).staged(0).blob
                return self.store(tokens, tuple((blob[l, 0], blob[l, 1]) for l in range(blob.shape[0])), skip_existing,
                                  blocking)
            flat = self._flat_paged(kv_caches)
            idx = slot_mapping.to(self._first(flat).device)
            g = lambda c: _bytes_of(c)[idx].view(c.dtype)  # noqa: E731
            kv = tuple(g(c) for c in flat) if self._mla else tuple((g(k), g(v)) for k, v in flat)
            return self.store(tokens, kv, skip_existing, blocking)
        chunk_hashes = self._prefix_hash(tokens)
        start = self._skip_scan(chunk_hashes, "vllm") if skip_existing else 0

        def put(keys, tok_begin):
            view = KvView.from_paged(kv_caches, slot_mapping.cuda())
            self._geom = (view.L, view.H, view.D, view.dtype)
            if self._stages_split(kv_caches):
                # one blob of the stored range for every part of the tier; the view keeps it alive for the tier's kernels
                view, tok_begin = view.staged(tok_begin), 0
            return self.engine_.put_kv_chunks(keys, view, tok_begin, self.chunk_size, blocking=blocking)
        self._store_put(chunk_hashes, start, "vllm", put)

    @_lmcache_nvtx_annotate
    @torch.no_grad()
    def retrieve_paged(self, tokens: torch.Tensor, kv_caches, slot_mapping: torch.Tensor,
                       mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """retrieve() straight into a paged KV cache: the longest cached prefix of `tokens` (optionally only the
        suffix selected by `mask`) is written to rows slot_mapping[i]; returns ret_mask as retrieve() does.  Rows of
        tokens that are not retrieved -- misses and the masked-off prefix -- are left untouched."""
        return self._retrieve_paged(tokens, kv_caches, slot_mapping, mask)

    def _retrieve_paged(self, tokens, kv_caches, slot_mapping, mask, get_kv=None) -> torch.Tensor:
        """retrieve_paged; get_kv as in _retrieve, for every chunk but a first one that straddles the mask"""
        self._check_paged_args(tokens, slot_mapping)
        self._check_kind(kv_caches, "kv_caches")
        mover = self._mover_paged(kv_caches)
        flat = None if mover else self._flat_paged(kv_caches)      # a strided cache's reshape would be a copy
        dev = self._first(kv_caches).device
        slots = slot_mapping.to(dev)
        if not self._fast_path():
            kv, ret_mask = self.retrieve(tokens, mask)
            if len(kv) > 0 and self._mover_paged(kv_caches):
                # the retrieved tokens are one run after the masked-off prefix: the mover scatters them
                a = 0 if mask is None else int(len(mask) - torch.sum(mask))
                blob = torch.stack([torch.stack(p) for p in kv]).to(self._first(kv_caches).dtype)
                KvView.from_paged(kv_caches, slots[a:]).unpack_blob(blob, 0)
            elif len(kv) > 0:
                idx = slots[ret_mask.to(dev)]
                if self._mla:
                    for c, x in zip(flat, kv):
                        _bytes_of(c)[idx] = _bytes_of(x.to(c.dtype))
                else:
                    for (kc, vc), (k, v) in zip(flat, kv):
                        _bytes_of(kc)[idx] = _bytes_of(k.to(kc.dtype))
                        _bytes_of(vc)[idx] = _bytes_of(v.to(vc.dtype))
            return ret_mask
        cs = self.chunk_size
        ret_mask, num_skip_tok, num_skip_chunk, extra = self._split_mask(tokens, mask)
        full_chain = self._prefix_hash(tokens)
        chunk_hashes = full_chain[num_skip_chunk:]
        base = num_skip_chunk * cs
        view = KvView.from_paged(kv_caches, slots[base:])
        first = 1 if extra > 0 and len(chunk_hashes) > 0 else 0
        layout, own, got_chunks = None, 0, 0      # layout: the other one that serves the chunks after this engine's own
        if first:
            # the first chunk straddles the mask: decode it next to the cache and scatter only its unmasked tail
            t0 = min(cs, len(tokens) - base)
            tmp = torch.empty(KvView.blob_shape("vllm", view.L, view.H, view.D, t0, self._mla), dtype=view.dtype,
                              device=dev)
            layout, own, got_chunks = self._fetch(chunk_hashes[:1], "vllm", KvView.from_blob(tmp, "vllm"), 0)
            if got_chunks and mover:
                view.unpack_blob(tmp[:, :, extra:], extra)
            elif got_chunks:
                idx = slots[base + extra: base + t0]
                if self._mla:
                    for l, c in enumerate(flat):
                        _bytes_of(c)[idx] = _bytes_of(tmp[l, extra:])
                else:
                    for l, (kc, vc) in enumerate(flat):
                        _bytes_of(kc)[idx] = _bytes_of(tmp[l, 0, extra:])
                        _bytes_of(vc)[idx] = _bytes_of(tmp[l, 1, extra:])
        if got_chunks == first and len(chunk_hashes) > first:       # not after a straddling chunk that missed
            dst, tok0 = view, first * cs
            if self._stages_split(kv_caches):
                # decoded into a blob of the tokens asked for, then only the retrieved ones unpacked into the cache
                n_stage = view.ntokens - tok0
                dst = KvView.from_blob(torch.empty(KvView.blob_shape("vllm", view.L, view.H, view.D, n_stage),
                                                   dtype=view.dtype, device=dev), "vllm")
                tok0 = 0
            layout, own_rest, n = self._fetch(chunk_hashes[first:], "vllm", dst, tok0, get_kv, layout)
            if dst is not view and n:
                view.unpack_blob(dst.blob.narrow(2, 0, min(n * cs, n_stage)), first * cs)
            own += own_rest
            got_chunks += n
        self._touch(full_chain[:num_skip_chunk + own], "vllm")
        return self._trim_mask(ret_mask, num_skip_tok, min(base + got_chunks * cs, len(tokens)) - num_skip_tok)

    # ------------------------------------------------------------------ other tensor-parallel layouts
    def _foreign_key(self, chunk_hash: str, fmt: str, world_size: int, rank: int) -> CacheEngineKey:
        return CacheEngineKey(fmt, self.metadata.model_name, world_size, rank, chunk_hash)

    def _reshard_layout(self, chunk_hash: str, fmt: str, Hg: int) -> Optional[int]:
        """The first world size of reshard_world_sizes under which every shard of this rank's heads of the chunk exists."""
        ws, rank = self.metadata.world_size, self.metadata.worker_id
        for W in self.config.reshard_world_sizes:
            shards = source_shards(Hg, W, ws, rank)
            if shards and all(self.engine_.contains(self._foreign_key(chunk_hash, fmt, W, s.rank)) for s in shards):
                return W
        return None

    def _reshard_groups(self, chunk_hashes, fmt: str, W: int, Hg: int) -> LazySeq:
        """Per chunk, the (key, HeadWindow) of every container of layout W that this rank's heads are made of."""
        wins = [(s.rank, HeadWindow(Hg // W, s.src_head0, s.n_heads, s.dst_head0))
                for s in source_shards(Hg, W, self.metadata.world_size, self.metadata.worker_id)]
        return LazySeq(lambda h: [(self._foreign_key(h, fmt, W, r), w) for r, w in wins], chunk_hashes)

    def _reshard_get(self, chunk_hashes, fmt: str, view: KvView, tok0: int,
                     layout: Optional[int] = None) -> Tuple[Optional[int], int]:
        """Continue a retrieve whose own-layout prefix has ended: decode the chunks of `chunk_hashes` (the first at token
        tok0 of `view`) from another layout's shards, up to the first incomplete chunk.  The layout is `layout`, or the
        first of reshard_world_sizes that holds every shard of the first chunk.  Returns (layout, chunks served).  Off
        (no request at all) unless reshard_world_sizes is set."""
        get = getattr(self.engine_, "get_kv_shards_into", None)
        if not self.config.reshard_world_sizes or get is None or len(chunk_hashes) == 0:
            return layout, 0
        Hg = view.H * self.metadata.world_size
        if layout is None:
            layout = self._reshard_layout(chunk_hashes[0], fmt, Hg)
            if layout is None:
                return None, 0
        stats: Dict[str, int] = {}
        n = get(self._reshard_groups(chunk_hashes, fmt, layout, Hg), view, tok0, self.chunk_size, stats)
        if n:
            c = self._reshard_counts.setdefault(layout, {"chunks": 0, "bytes": 0})
            c["chunks"] += n
            c["bytes"] += stats.get("bytes", 0)
        return layout, n

    def _reshard_geometry(self, chunk_hash: str, fmt: str):
        """(L, H, D, dtype) of this rank's chunks for a replica that knows no geometry and whose own layout misses: read
        from the header of the first source container of the first layout that has one (Hg = its H * W).  The backend
        keeps that container for the fetch that follows."""
        peek = getattr(self.engine_, "peek_geometry", None)
        if peek is None:
            return None
        ws, rank = self.metadata.world_size, self.metadata.worker_id
        for W in self.config.reshard_world_sizes:
            g = peek(self._foreign_key(chunk_hash, fmt, W, first_source_rank(W, ws, rank)), fmt)
            if g is not None and source_shards(g[1] * W, W, ws, rank):
                return (g[0], g[1] * W // ws) + tuple(g[2:])
        return None

    def reshard_stats(self) -> Dict[int, Dict[str, int]]:
        """Chunks served from other tensor-parallel layouts since the engine started, per source world size: {"chunks":
        whole chunks decoded, "bytes": container bytes fetched for them}."""
        return {W: dict(c) for W, c in self._reshard_counts.items()}

    def _touch(self, chunk_hashes, fmt: str) -> None:
        """Recency update for a bounded local tier (lmcache_b200/eviction.py): one call with the keys of a chain prefix,
        chunk 0 first -- every key of a stored sequence, the skipped and hit keys of a retrieve.  Touching a chunk only
        together with all of its predecessors is what keeps a tier's eviction from cutting a chain in the middle.  A store
        touches the prefix its scan matched (possibly none) right before it stores the rest: the tier protects what was
        touched since then while that store lands."""
        f = getattr(self.engine_, "touch", None)
        if f is not None:
            f(self._keys_of(chunk_hashes, fmt))

    # ------------------------------------------------------------------ native fast paths
    def _fast_path(self) -> bool:
        f = getattr(self.engine_, "supports_kv_view", None)
        return bool(f and f())

    def _kv_geometry(self):
        """(L, H, D, dtype) of this engine's chunks, learnt from the first store / a probe get."""
        return getattr(self, "_geom", None)

    def _fetch(self, chunk_hashes, fmt: str, view: KvView, tok0: int, get_kv=None, layout: Optional[int] = None,
               own_miss: bool = False) -> Tuple[Optional[int], int, int]:
        """Decode the chunks of `chunk_hashes` into `view`, the first at token tok0, up to the first miss: this layout's
        through get_kv (default: the backend's get_kv_into) -- unless another `layout` was chosen before or this one is
        known to miss the first chunk (own_miss) -- then the chunks after them from another layout (_reshard_get).
        Returns (layout, chunks of this layout, chunks in all)."""
        own = 0
        if layout is None and not own_miss:
            own = (get_kv or self.engine_.get_kv_into)(self._keys_of(chunk_hashes, fmt), view, tok0, self.chunk_size)
        layout, n = self._reshard_get(chunk_hashes[own:], fmt, view, tok0 + own * self.chunk_size, layout)
        uploads = getattr(get_kv, "uploads", None)
        if n and uploads:
            # chunk-major chunks after a layer-major prefix: every layer's ready event also comes after their decode
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream())
            uploads.append(LayerwiseUpload.completed(n, view.L, ev))
        return layout, own, own + n

    def _retrieve_into_blob(self, tokens, full_chain, ret_mask, num_skip_tok, num_skip_chunk, extra, fmt, st, get_kv):
        """retrieve() without per-chunk tensors or torch.cat: the backend decodes / uploads every hit chunk straight
        into one preallocated blob; the suffix-mask trim of the first chunk is a view offset, not a copy."""
        chunk_hashes = full_chain[num_skip_chunk:]
        geom = self._kv_geometry()
        own_miss = False         # this layout holds not even the first chunk: only another layout can serve it
        if geom is None:
            # shapes unknown (nothing stored through this engine yet -- the normal case for a retrieve-only replica):
            # read them from the first chunk's container header / stored blob; only backends without that door pay
            # for a full get of chunk 0
            key0 = self._make_key(chunk_hashes[0], fmt)
            peek = getattr(self.engine_, "peek_geometry", None)
            if peek is not None:
                geom = peek(key0, fmt)
            else:
                first = self.engine_.get(key0)
                if first is not None and first.dim() == (3 if self._mla else 5):     # the other kind's blob: a miss
                    geom = KvView.blob_geometry(first, fmt)
            if geom is None and self.config.reshard_world_sizes:
                geom = self._reshard_geometry(chunk_hashes[0], fmt)
                own_miss = geom is not None
            if geom is None:
                self._touch(full_chain[:num_skip_chunk], fmt)
                logger.info("Retrieved 0 chunks")
                return (), self._trim_mask(ret_mask, num_skip_tok, 0)
            self._geom = geom
        L, H, D, dtype = geom
        od = getattr(self.engine_, "out_dtype", None) or getattr(getattr(self.engine_, "deserializer", None), "out_dtype", None)
        if od is not None and od() is not None:
            dtype = od()
        n_tok_max = len(tokens) - num_skip_chunk * self.chunk_size
        blob = torch.empty(KvView.blob_shape(fmt, L, H, D, n_tok_max, self._mla), dtype=dtype,
                           device=torch.device("cuda", torch.cuda.current_device()))
        _, own, n = self._fetch(chunk_hashes, fmt, KvView.from_blob(blob, fmt), 0, get_kv, own_miss=own_miss)
        self._touch(full_chain[:num_skip_chunk + own], fmt)
        if n == 0:
            logger.info("Retrieved 0 chunks")
            return (), self._trim_mask(ret_mask, num_skip_tok, 0)
        got = min(n * self.chunk_size, n_tok_max) - extra      # the last hit chunk may be the ragged tail
        logger.info(f"Retrieved {n} chunks ({got} tokens in total) -- elapsed time {time.perf_counter() - st}")
        kv = self._blob_to_tuple_kv(blob.narrow(KvView.token_dim(fmt, self._mla), extra, got))
        return kv, self._trim_mask(ret_mask, num_skip_tok, got)

    # ------------------------------------------------------------------ layer-wise retrieve
    def _layerwise_get(self):
        """(get_kv for _retrieve / _retrieve_paged, whose `uploads` list receives the LayerwiseUploads), or None: the
        backend cannot serve this engine's chunks layer-major -- it says so (supports_layerwise_get: a remote tier whose
        server has no ranged reads, a serde without containers), or its containers hold several groups
        (CacheGen containers of more than 256 tokens; a lossless container is always one group)"""
        f = getattr(self.engine_, "get_kv_layerwise", None)
        ok = getattr(self.engine_, "supports_layerwise_get", None)
        if f is None or ok is None or not self._fast_path() or \
                self.chunk_size > getattr(self.engine_, "layerwise_max_tokens", N.GROUP_TOKENS) or not ok():
            return None
        uploads: List[LayerwiseUpload] = []

        def get_kv(keys, view, tok0, cs):
            uploads.append(f(keys, view, tok0, cs))
            return uploads[-1].n
        get_kv.uploads = uploads
        return get_kv, uploads

    @staticmethod
    def _layerwise_result(ret_mask, kv, num_layers: int, uploads) -> LayerwiseRetrieval:
        if uploads:
            return LayerwiseRetrieval(ret_mask, kv, num_layers, join_uploads(uploads, num_layers))
        # nothing went layer-major: everything this call enqueued is before one event
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        return LayerwiseRetrieval(ret_mask, kv, num_layers, LayerwiseUpload.completed(0, num_layers, ev))

    @torch.no_grad()
    def retrieve_layerwise(self, tokens: torch.Tensor, mask: Optional[torch.Tensor] = None) -> LayerwiseRetrieval:
        """retrieve(), with the KV made available one layer at a time: returns once the hit is known; ret_mask and the
        KV after synchronize() are those of retrieve().  On the compressed host and disk tiers the containers are
        uploaded and decoded layer-major, so layer 0 is ready after about 1/L of the bytes; on the raw cpu and cuda tiers
        each layer of every chunk blob is copied and unpacked in one launch per layer.  On the remote tier, opted in
        with LMCACHE_B200_REMOTE_LAYERWISE=1 and with a server that has ranged reads (this project's), they are also
        fetched layer-major: every chunk's layer l before
        any chunk's layer l + 1.  A hybrid tier does both parts so and joins them.  Chunks served from another
        tensor-parallel layout after a layer-major prefix are decoded whole, before every layer's event.  On every other
        tier (and for CacheGen chunks of more than 256 tokens) this is retrieve() followed by one event that stands for
        every layer.  A remote fetch that fails after the match (a lost server) raises in wait_layer / synchronize for
        the layers not yet released: ret_mask was already promised."""
        get_kv, uploads = self._layerwise_get() or (None, [])
        kv, ret_mask = self._retrieve(tokens, mask, get_kv)
        geom = self._kv_geometry()
        return self._layerwise_result(ret_mask, kv, len(kv) or (geom[0] if geom else 0), uploads)

    @torch.no_grad()
    def retrieve_paged_layerwise(self, tokens: torch.Tensor, kv_caches, slot_mapping: torch.Tensor,
                                 mask: Optional[torch.Tensor] = None) -> LayerwiseRetrieval:
        """retrieve_paged(), with the KV made available one layer at a time (see retrieve_layerwise: the same tiers go
        layer-major, the remote one included).  A first chunk that straddles the mask is decoded and scattered whole
        before layer 0's wait; `kv` is None."""
        self._check_kind(kv_caches, "kv_caches")
        # a split cache on a container tier is retrieved whole through its staging blob: one event for every layer
        get_kv, uploads = (None if self._stages_split(kv_caches) else self._layerwise_get()) or (None, [])
        ret_mask = self._retrieve_paged(tokens, kv_caches, slot_mapping, mask, get_kv)
        return self._layerwise_result(ret_mask, None, len(kv_caches), uploads)

    # ------------------------------------------------------------------ layer-wise store
    def _layerwise_store_ok(self, dtype: torch.dtype) -> bool:
        """Can this store be encoded layer by layer?  The compressed host and disk tiers and the lm:// remote tier with
        the cachegen or lossless serde can, for the KV their codec encodes (CacheGen: 16-bit; lossless: 16-bit and
        one-byte) and chunks of at most the tier's layerwise_max_tokens (256 for CacheGen's version-3 containers, 4096
        for lossless ones); the raw cpu and cuda tiers can for every chunk size and every KV the mover moves; a hybrid
        tier can when both its parts can.  A remote tier with the torch serde cannot (layerwise_max_tokens 0)."""
        return (getattr(self.engine_, "begin_layerwise_store", None) is not None and self._fast_path() and
                self.chunk_size <= self.engine_.layerwise_max_tokens and dtype in NATIVE_DTYPES)

    def _begin_layerwise(self, tokens, view_fn, fmt: str, num_layers: int, skip_existing: bool,
                         fallback: Callable) -> LayerwiseStore:
        """The hash chain and the skip_existing scan run here, on the calling thread: the scan blocks until the chain
        has produced the digest of the first chunk the tier does not hold (one 256-token SHA-256 step per chunk) plus
        one dict lookup per chunk.  The plan (no KV read) is enqueued on the tier's encode stream.  finish() makes the
        touches and the put that store() / store_paged() make, in the same order."""
        chunk_hashes = self._prefix_hash(tokens)
        start = self._skip_scan(chunk_hashes, fmt) if skip_existing else 0
        enc = None
        if start < len(chunk_hashes):
            view = view_fn()
            self._geom = (view.L, view.H, view.D, view.dtype)
            enc = self.engine_.begin_layerwise_store(view, start * self.chunk_size, self.chunk_size)
            if enc is None:
                return LayerwiseStore(num_layers, None, fallback)

        def publish(stream, enc):
            # enc is None when the scan matched every chunk, or when the handle was closed: nothing to put.  The put
            # waits for the landing on a tier that asks for it (a lossless disk tier: layerwise_store_blocking)
            blocking = bool(getattr(self.engine_, "layerwise_store_blocking", False))
            put = None if enc is None else lambda keys, tok_begin: self.engine_.put_kv_chunks(
                keys, None, tok_begin, self.chunk_size, blocking=blocking, encoded=enc)
            self._store_put(chunk_hashes, start, fmt, put)
        return LayerwiseStore(num_layers, enc, publish)

    @torch.no_grad()
    def store_paged_layerwise(self, tokens: torch.Tensor, kv_caches, slot_mapping: torch.Tensor,
                              skip_existing=True) -> LayerwiseStore:
        """store_paged(), with the KV handed over one layer at a time: the caches may still be unwritten when this is
        called; call save_layer(l) once layer l is written and finish() after the last layer (LayerwiseStore).  The keys
        stored, the containers and the eviction touches are those of store_paged(tokens, kv_caches, slot_mapping,
        skip_existing).  Layer by layer on the compressed host and disk tiers, the raw cpu and cuda tiers, the lm://
        remote tier with the cachegen or lossless serde, and hybrids of these (one encode for both parts when they keep
        the same containers); on the remote and hybrid tiers finish() returns once the server holds every chunk.  Every
        other case, and a split (PagedAttention) cache on a container tier, runs store_paged() at finish()."""
        self._check_paged_args(tokens, slot_mapping, kv_caches)

        def fallback(stream, enc):
            with torch.cuda.stream(stream):
                self.store_paged(tokens, kv_caches, slot_mapping, skip_existing)
        if not self._layerwise_store_ok(self._first(kv_caches).dtype) or self._stages_split(kv_caches):
            # a split cache on a container tier is staged whole: the store runs at finish()
            return LayerwiseStore(len(kv_caches), None, fallback)
        return self._begin_layerwise(tokens, lambda: KvView.from_paged(kv_caches, slot_mapping.cuda()), "vllm",
                                     len(kv_caches), skip_existing, fallback)

    def _in_place(self, kv_tensors_raw: KVCache) -> bool:
        """do all of store()'s tensors share layer 0's strides, with a contiguous last dimension (KvView.from_tuple
        reads them in place)?"""
        k0 = self._first(kv_tensors_raw)
        return all(t.stride() == k0.stride() and t.stride(-1) == 1 for t in self._tensors(kv_tensors_raw))

    @torch.no_grad()
    def store_layerwise(self, tokens: torch.Tensor, kv_tensors_raw: KVCache, skip_existing=True) -> LayerwiseStore:
        """store(), with the KV handed over one layer at a time (see store_paged_layerwise): kv_tensors_raw is store()'s
        per-layer (K, V) tuple (or an MLA engine's latent per layer) on the GPU, possibly not yet written."""
        fmt = self.metadata.fmt
        self._check_store_args(tokens, kv_tensors_raw, fmt)

        def fallback(stream, enc):
            with torch.cuda.stream(stream):
                self.store(tokens, kv_tensors_raw, skip_existing)
        k0 = self._first(kv_tensors_raw)
        # the kernels must read the caller's tensors in place (KvView.from_tuple would copy tensors of other strides
        # now, before they are written): anything else takes the ordinary store at finish()
        if not k0.is_cuda or not self._in_place(kv_tensors_raw) or not self._layerwise_store_ok(k0.dtype):
            return LayerwiseStore(len(kv_tensors_raw), None, fallback)
        return self._begin_layerwise(tokens, lambda: KvView.from_tuple(kv_tensors_raw, fmt), fmt, len(kv_tensors_raw),
                                     skip_existing, fallback)

    # ------------------------------------------------------------------ non-prefix segments
    @staticmethod
    def _check_rope_dtype(dtype: torch.dtype) -> None:
        if dtype not in (torch.bfloat16, torch.float16):
            raise TypeError(f"segment retrieve rotates 16-bit keys only, not {dtype}: rotating an FP8 key would round it "
                            f"a third time")

    def _segment_hashes(self, tokens: torch.Tensor, plans) -> list:
        """every segment's chunk digests, its tokens hashed as their own sequence: one hash-chain launch for all"""
        toks, offs = hash_input(tokens, plans)
        chain = sha256_prefix_chain_lazy(toks, self.chunk_size, offs)
        return [chain[p.chunk_begin:p.chunk_begin + p.n_chunks] for p in plans]

    def _segments_prologue(self, tokens: torch.Tensor, segments, rope: RopeSpec):
        """the plan and the refusals every segment retrieve makes before it fetches anything"""
        assert len(tokens.shape) == 1, f"Invalid shape of tokens: {tokens.shape}"
        if not isinstance(rope, RopeSpec):
            raise TypeError(f"rope must be a RopeSpec, got {type(rope).__name__}")
        plans = plan_segments(len(tokens), segments, self.chunk_size)
        md = str(self.metadata.dtype).lower()
        if any(s in md for s in ("fp8", "float8", "uint8")):
            raise TypeError(f"segment retrieve rotates 16-bit keys only; this engine's KV dtype is {self.metadata.dtype}")
        return plans

    def _derived_key(self, chunk_hash: str, fmt: str) -> CacheEngineKey:
        """the key of a chunk of a segment stored from inside a longer prompt (rope.derived_digest)"""
        return self._make_key(derived_digest(chunk_hash), fmt)

    def _derived_keys(self, chunk_hashes, fmt: str) -> LazySeq:
        return LazySeq(lambda h: self._derived_key(h, fmt), chunk_hashes)

    def _chain_keys(self, chunk_hashes, p: int, n: int, fmt: str) -> list:
        """the keys of a segment's chunks [0, n): prefix keys for [0, p), derived keys after"""
        return [self._make_key(h, fmt) for h in chunk_hashes[:p]] + \
            [self._derived_key(h, fmt) for h in chunk_hashes[p:n]]

    def _touch_chain(self, chunk_hashes, p: int, n: int, fmt: str) -> None:
        """_touch of a segment's chunks [0, n) as one chain, chunk 0 first, under the keys they hit"""
        f = getattr(self.engine_, "touch", None)
        if f is not None:
            f(self._chain_keys(chunk_hashes, p, n, fmt))

    def _get_chunks(self, keys) -> List[torch.Tensor]:
        """batched_get of `keys` up to the first miss (a blob of the other kind is one)"""
        chunks = []
        for c in self.engine_.batched_get(iter(keys)):
            if c is None or c.dim() != (3 if self._mla else 5):
                break
            chunks.append(c)
        return chunks

    def _rotate(self, view: KvView, written, rope: RopeSpec) -> None:
        """one rope shift of the written key rows of every segment that does not start at token 0"""
        sot, lo, hi, shifts = seg_of_tok(view.ntokens, written)
        if hi > lo:
            seg = torch.tensor(sot, dtype=torch.int32).to(view.device)
            sh = torch.tensor(shifts, dtype=torch.int64).to(view.device)
            rope_shift(view, lo, seg, sh, rope)

    def _segments_geometry(self, plans, hashes, fmt: str, rope: Optional[RopeSpec]):
        """(L, H, D, dtype of the result) of a segment retrieve on a native-path tier: the engine's, or read from the
        first chunk any segment has stored; None when neither tells.  The dtype, and D against `rope`, are checked."""
        geom = self._kv_geometry()
        peek = getattr(self.engine_, "peek_geometry", None)
        for p, hs in zip(plans, hashes):
            # a segment inside the prompt may be stored under its derived keys only
            for key0 in [self._make_key(hs[0], fmt)] + ([self._derived_key(hs[0], fmt)] if p.start > 0 else []):
                if geom is not None:
                    break
                if peek is not None:
                    geom = peek(key0, fmt)
                else:
                    first = self.engine_.get(key0)
                    if first is not None and first.dim() == (3 if self._mla else 5):
                        geom = KvView.blob_geometry(first, fmt)
        if geom is None:
            return None
        self._geom = geom
        L, H, D, dtype = geom
        od = getattr(self.engine_, "out_dtype", None) or \
            getattr(getattr(self.engine_, "deserializer", None), "out_dtype", None)
        if od is not None and od() is not None:
            dtype = od()
        self._check_rope_dtype(dtype)
        if rope is not None:
            rope.check(D)
        return L, H, D, dtype

    def _segments_blob(self, tokens, plans, hashes, fmt: str, rope: Optional[RopeSpec] = None):
        """Every segment's longest stored prefix of chunks in one zeroed blob of the request's T tokens, each at its
        start (unrotated).  Returns (blob or None when nothing was found, [(plan, tokens written)]).  With `rope`, the
        geometry's dtype and D are checked against it once known, before any chunk is written."""
        T, cs = len(tokens), self.chunk_size
        tdim = KvView.token_dim(fmt, self._mla)
        dev = torch.device("cuda", torch.cuda.current_device())
        written, blob = [], None
        fast = self._fast_path()
        if fast:
            geom = self._segments_geometry(plans, hashes, fmt, rope)
            if geom is not None:
                L, H, D, dtype = geom
                blob = torch.zeros(KvView.blob_shape(fmt, L, H, D, T, self._mla), dtype=dtype, device=dev)
        dst = None if blob is None else KvView.from_blob(blob, fmt)
        for p, hs in zip(plans, hashes):
            n_tok = 0
            if fast and blob is not None:
                own = self.engine_.get_kv_into(self._keys_of(hs, fmt), dst, p.start, cs)
                more = 0
                if p.start > 0 and own < len(hs):
                    more = self.engine_.get_kv_into(self._derived_keys(hs[own:], fmt), dst, p.start + own * cs, cs)
                self._touch_chain(hs, own, own + more, fmt)
                n_tok = min((own + more) * cs, p.end - p.start)
            elif not fast:
                chunks = self._get_chunks(self._keys_of(hs, fmt))
                own = len(chunks)
                if p.start > 0 and own < len(hs):
                    chunks += self._get_chunks(self._derived_keys(hs[own:], fmt))
                self._touch_chain(hs, own, len(chunks), fmt)
                if chunks and blob is None:
                    L, H, D, dtype = KvView.blob_geometry(chunks[0], fmt)
                    self._check_rope_dtype(dtype)
                    if rope is not None:
                        rope.check(D)
                    blob = torch.zeros(KvView.blob_shape(fmt, L, H, D, T, self._mla), dtype=dtype, device=dev)
                for k, c in enumerate(chunks):
                    t = c.shape[tdim]
                    blob.narrow(tdim, p.start + k * cs, t).copy_(c)
                    n_tok += t
            written.append((p, n_tok))
        return blob, written

    @_lmcache_nvtx_annotate
    @torch.no_grad()
    def retrieve_segments(self, tokens: torch.Tensor, segments, rope: RopeSpec) -> Tuple[KVCache, torch.Tensor]:
        """Non-prefix retrieve (a RAG prompt's documents, seen before as prompts of their own, at new positions).
        segments: (start, end) token ranges of `tokens`, non-overlapping, in any order.  Each segment gets its longest
        stored prefix of chunks, keyed by the hash chain of its own tokens (what a store of tokens[start:end] alone
        stored), at tokens start... of the result, its keys turned by `start` positions (rope).  Returns (kv, ret_mask):
        kv is retrieve()'s per-layer views of one [L, 2, T, H, D] blob (an MLA engine: [L, T, D]) in which every token
        not retrieved is zero, or () when no segment hits; ret_mask marks exactly the tokens written.  One segment
        (0, T) gives retrieve(tokens)'s rows and ret_mask.  TypeError for FP8 KV, ValueError for empty, overlapping or
        out-of-range segments and for a rotary range that does not fit a key head, all before anything is fetched.
        reshard_world_sizes is not consulted."""
        fmt = self.metadata.fmt
        if fmt not in ("vllm", "huggingface"):
            raise ValueError(f"Invalid format: {fmt}")
        plans = self._segments_prologue(tokens, segments, rope)
        geom = self._kv_geometry()
        if geom is not None:
            self._check_rope_dtype(geom[3])
            rope.check(geom[2])
        blob, written = self._segments_blob(tokens, plans, self._segment_hashes(tokens, plans), fmt, rope)
        ret_mask = torch.zeros(len(tokens), dtype=torch.bool)
        if blob is None:
            return (), ret_mask
        for p, n in written:
            ret_mask[p.start:p.start + n] = True
        self._rotate(KvView.from_blob(blob, fmt), written, rope)
        return self._blob_to_tuple_kv(blob), ret_mask

    @_lmcache_nvtx_annotate
    @torch.no_grad()
    def retrieve_paged_segments(self, tokens: torch.Tensor, kv_caches, slot_mapping: torch.Tensor, segments,
                                rope: RopeSpec) -> torch.Tensor:
        """retrieve_segments straight into a paged KV cache (any layout retrieve_paged takes): each segment's stored
        chunks are written to rows slot_mapping[start...], through the fetch step of retrieve_paged on every tier, then
        one rope shift turns the written key rows of every segment by its start (a segment at 0 is not rotated).
        Returns ret_mask, marking exactly the tokens written; every other row is untouched.  One segment (0, T) gives
        retrieve_paged(tokens, kv_caches, slot_mapping)'s ret_mask and rows bit for bit.  An MLA engine takes
        RopeSpec(64, inv_freq, "gptj", offset=512): only the decoupled RoPE channels of its latent turn."""
        self._check_paged_args(tokens, slot_mapping)
        self._check_kind(kv_caches, "kv_caches")
        plans = self._segments_prologue(tokens, segments, rope)
        first = self._first(kv_caches)
        self._check_rope_dtype(first.dtype)
        rope.check(first.shape[-1] if self._mla else paged_layout(*kv_caches[0]).D)
        dev, cs = first.device, self.chunk_size
        slots = slot_mapping.to(dev)
        hashes = self._segment_hashes(tokens, plans)
        if not self._fast_path():
            # the tier hands out chunk blobs: assemble them, then scatter each segment's run as retrieve_paged does
            blob, written = self._segments_blob(tokens, plans, hashes, "vllm")
            for p, n in written:
                if n == 0:
                    continue
                if self._mla:
                    idx = slots[p.start:p.start + n]
                    for l, c in enumerate(self._flat_paged(kv_caches)):
                        c[idx] = blob[l, p.start:p.start + n].to(c.dtype)
                else:
                    KvView.from_paged(kv_caches, slots[p.start:p.start + n]).unpack_blob(
                        blob[:, :, p.start:p.start + n].to(first.dtype), 0)
        else:
            stage = self._stages_split(kv_caches)
            view = KvView.from_paged(kv_caches, slots)
            written = []
            for p, hs in zip(plans, hashes):
                dst, tok0 = view, p.start
                if stage:
                    # decoded into a blob of the segment, then only the retrieved tokens unpacked into the cache
                    dst = KvView.from_blob(torch.empty(KvView.blob_shape("vllm", view.L, view.H, view.D, p.end - p.start),
                                                       dtype=view.dtype, device=dev), "vllm")
                    tok0 = 0
                own = self.engine_.get_kv_into(self._keys_of(hs, "vllm"), dst, tok0, cs)
                more = 0
                if p.start > 0 and own < len(hs):
                    # continued in the namespace of segments stored from inside a longer prompt
                    more = self.engine_.get_kv_into(self._derived_keys(hs[own:], "vllm"), dst, tok0 + own * cs, cs)
                self._touch_chain(hs, own, own + more, "vllm")
                n = min((own + more) * cs, p.end - p.start)
                if dst is not view and n:
                    view.unpack_blob(dst.blob.narrow(2, 0, n), p.start)
                written.append((p, n))
        ret_mask = torch.zeros(len(tokens), dtype=torch.bool)
        for p, n in written:
            ret_mask[p.start:p.start + n] = True
        self._rotate(KvView.from_paged(kv_caches, slots), written, rope)
        return ret_mask

    # ------------------------------------------------------------------ layer-wise segment retrieve
    def _segments_runs_get(self, kv_caches=None):
        """The tier's multi-run layer-major get (get_kv_layerwise_runs) when it can serve this engine's chunks so
        (retrieve_layerwise's conditions, and no split cache staged through a blob), else None"""
        f = getattr(self.engine_, "get_kv_layerwise_runs", None)
        if f is None or self._layerwise_get() is None or (kv_caches is not None and self._stages_split(kv_caches)):
            return None
        return f

    def _segments_layerwise(self, get, plans, hashes, fmt: str, view: KvView, rope: RopeSpec, n_tokens: int):
        """Every segment's stored chunks fetched into `view` by ONE layer-major get, each at its start: its prefix keys,
        then (start > 0) its derived keys from their first miss on; the keys of every segment at start > 0 turned by its
        start, layer by layer, inside the upload.  Touches each segment's chain.  Returns (ret_mask, LayerwiseUpload)."""
        shifted = [p for p in plans if p.shift != 0]
        rotation = None
        if shifted:
            with torch.cuda.device(view.device):
                table = rope_table(torch.tensor([p.shift for p in shifted], dtype=torch.int64).to(view.device), rope)
            rows = {p.index: k for k, p in enumerate(shifted)}
            rotation = Rotation(rope, table, [rows.get(p.index, -1) for p in plans], [p.end for p in plans])
        runs = [(self._keys_of(hs, fmt), self._derived_keys(hs, fmt) if p.start > 0 else None, p.start)
                for p, hs in zip(plans, hashes)]
        with torch.cuda.device(view.device):
            hits, upload = get(runs, view, self.chunk_size, rotation)
        ret_mask = torch.zeros(n_tokens, dtype=torch.bool)
        for p, hs, (own, more) in zip(plans, hashes, hits):
            self._touch_chain(hs, own, own + more, fmt)
            ret_mask[p.start:p.start + min((own + more) * self.chunk_size, p.end - p.start)] = True
        return ret_mask, upload

    @torch.no_grad()
    def retrieve_paged_segments_layerwise(self, tokens: torch.Tensor, kv_caches, slot_mapping: torch.Tensor, segments,
                                          rope: RopeSpec) -> LayerwiseRetrieval:
        """retrieve_paged_segments, with the KV made available one layer at a time (`kv` is None): returns once every
        segment's hit is known; after wait_layer(l, stream) layer l's rows are written and turned by each segment's
        start; after synchronize() ret_mask and every row are retrieve_paged_segments'.  On every tier with a
        layer-major get (raw, CacheGen and lossless host and disk, lm:// with ranged reads, hybrid), every segment's
        chunks go through one layer-major upload (the tier's get_kv_layerwise_runs), each layer's keys turned as that
        layer lands.  Every other case -- the remote tier without the opt-in or ranged reads, the torch serde, CacheGen
        chunks of more than 256 tokens, a split (PagedAttention) cache on a container tier -- runs
        retrieve_paged_segments with one event for every layer.  The refusals are
        retrieve_paged_segments', raised before anything is hashed or fetched."""
        self._check_paged_args(tokens, slot_mapping)
        self._check_kind(kv_caches, "kv_caches")
        plans = self._segments_prologue(tokens, segments, rope)
        first = self._first(kv_caches)
        self._check_rope_dtype(first.dtype)
        rope.check(first.shape[-1] if self._mla else paged_layout(*kv_caches[0]).D)
        get = self._segments_runs_get(kv_caches)
        if get is None:
            ret_mask = self.retrieve_paged_segments(tokens, kv_caches, slot_mapping, segments, rope)
            return self._layerwise_result(ret_mask, None, len(kv_caches), [])
        view = KvView.from_paged(kv_caches, slot_mapping.to(first.device))
        ret_mask, upload = self._segments_layerwise(get, plans, self._segment_hashes(tokens, plans), "vllm", view, rope,
                                                    len(tokens))
        return LayerwiseRetrieval(ret_mask, None, len(kv_caches), upload)

    @torch.no_grad()
    def retrieve_segments_layerwise(self, tokens: torch.Tensor, segments, rope: RopeSpec) -> LayerwiseRetrieval:
        """retrieve_segments, with the KV made available one layer at a time: `kv` holds retrieve_segments' per-layer
        views of one blob (rows not retrieved are zero), whose layer l may be read once wait_layer(l, stream) was called.
        The same tiers go layer-major as for retrieve_paged_segments_layerwise.  On a total miss before the geometry is
        known, kv is () and num_layers 0."""
        fmt = self.metadata.fmt
        if fmt not in ("vllm", "huggingface"):
            raise ValueError(f"Invalid format: {fmt}")
        plans = self._segments_prologue(tokens, segments, rope)
        geom = self._kv_geometry()
        if geom is not None:
            self._check_rope_dtype(geom[3])
            rope.check(geom[2])
        get = self._segments_runs_get()
        if get is None:
            kv, ret_mask = self.retrieve_segments(tokens, segments, rope)
            geom = self._kv_geometry()
            return self._layerwise_result(ret_mask, kv, len(kv) or (geom[0] if geom else 0), [])
        hashes = self._segment_hashes(tokens, plans)
        geom = self._segments_geometry(plans, hashes, fmt, rope)
        if geom is None:
            return self._layerwise_result(torch.zeros(len(tokens), dtype=torch.bool), (), 0, [])
        L, H, D, dtype = geom
        blob = torch.zeros(KvView.blob_shape(fmt, L, H, D, len(tokens), self._mla), dtype=dtype,
                           device=torch.device("cuda", torch.cuda.current_device()))
        ret_mask, upload = self._segments_layerwise(get, plans, hashes, fmt, KvView.from_blob(blob, fmt), rope,
                                                    len(tokens))
        return LayerwiseRetrieval(ret_mask, self._blob_to_tuple_kv(blob), L, upload)

    # ------------------------------------------------------------------ segment store
    def _segment_store_check(self, tokens: torch.Tensor, segments, rope: RopeSpec, first: torch.Tensor, D: int):
        """the plan and the refusals every segment store makes before it hashes or stores anything"""
        plans = self._segments_prologue(tokens, segments, rope)
        self._check_rope_dtype(first.dtype)
        rope.check(D)
        return plans

    def _segment_store_plan(self, tokens: torch.Tensor, plans, fmt: str, prefix_store: Callable[[int], Any],
                            skip_existing: bool):
        """Every segment store after its refusals: a segment at 0 through prefix_store(end), then every other segment's
        hash chain, skip scan (with the touches of the chains it hit) and staging plan (plan_segment_store).  Returns
        (prefix_store's result, or None without a segment at 0; the digests of the segments inside the prompt; runs,
        rows, seg_of_tok and shifts of plan_segment_store)."""
        cs = self.chunk_size
        # the segments inside the prompt, planned again: their hash input and chain offsets leave out a segment at 0
        inner = plan_segments(len(tokens), [(p.start, p.end) for p in plans if p.start > 0], cs)
        head = None
        for p in plans:
            if p.start == 0:
                # exactly a prefill of tokens[:end]: its ordinary prefix keys, unrotated
                head = prefix_store(p.end)
        if not inner:
            return head, [], [], [], [], []
        hashes = self._segment_hashes(tokens, inner)
        hits = []
        for p, hs in zip(inner, hashes):
            if not skip_existing:
                hits.append((0, 0))
                continue
            has = lambda k: lambda i: self.engine_.contains(k(hs[i], fmt))   # noqa: E731
            ph, dh = skip_chunks(p.n_chunks, has(self._make_key), has(self._derived_key))
            self._touch_chain(hs, ph, ph + dh, fmt)
            hits.append((ph, dh))
        return (head, hashes) + tuple(plan_segment_store(inner, hits, cs))

    def _store_segments(self, tokens: torch.Tensor, segments, rope: RopeSpec, fmt: str, first: torch.Tensor, D: int,
                        view_fn: Callable[[], KvView], prefix_store: Callable[[int], None], skip_existing: bool,
                        blocking: bool) -> None:
        """Every segment store: the refusals, then a segment at 0 through prefix_store(end), then every other segment's
        skip scan, one table and one b200kv_pack_chunks_rope launch into one staging blob, and one put per segment
        under its derived keys."""
        plans = self._segment_store_check(tokens, segments, rope, first, D)
        _, hashes, runs, rows, sot, shifts = self._segment_store_plan(tokens, plans, fmt, prefix_store, skip_existing)
        if not runs:
            return
        cs = self.chunk_size
        view = view_fn()
        self._geom = (view.L, view.H, view.D, view.dtype)
        dev = view.device
        with torch.cuda.device(dev):
            src = view.rows(torch.tensor(rows, dtype=torch.int64).to(dev))
            blob = torch.empty(KvView.blob_shape(fmt, view.L, view.H, view.D, len(rows), self._mla), dtype=view.dtype,
                               device=dev)
            pack_rope(src, blob, torch.tensor(sot, dtype=torch.int32).to(dev),
                      rope_table(torch.tensor(shifts, dtype=torch.int64).to(dev), rope), rope)
        tdim = KvView.token_dim(fmt, self._mla)
        fast = self._fast_path()
        for r in runs:
            hs = hashes[r.plan.index]
            part = KvView.from_blob(blob.narrow(tdim, r.stage_begin, r.n_tok), fmt)
            keys = self._derived_keys(hs[r.first:], fmt)
            if fast:
                self.engine_.put_kv_chunks(keys, part, 0, cs, blocking=blocking)
            else:
                _, chunks = part.pack_chunks(0, cs)
                self.engine_.batched_put(zip(keys, chunks), blocking=blocking)
            self._touch_chain(hs, r.prefix_hits, len(hs), fmt)
        logger.info(f"Stored {len(rows)} tokens of {len(runs)} segments under derived keys")

    @_lmcache_nvtx_annotate
    @torch.no_grad()
    def store_paged_segments(self, tokens: torch.Tensor, kv_caches, slot_mapping: torch.Tensor, segments,
                             rope: RopeSpec, skip_existing=True, blocking=True) -> None:
        """Store documents from inside a longer prompt, for retrieve_paged_segments / retrieve_segments at any later
        position.  segments: (start, end) token ranges of `tokens`, non-overlapping, in any order (plan_segments).  A
        segment at start > 0 is stored as a prefill of tokens[start:end] alone would have laid it out: chunks aligned to
        its start, its keys turned by -start (rope) on the way into one staging blob (one b200kv_pack_chunks_rope launch
        for all segments), keyed by the derived digests of its own hash chain (rope.derived_digest) -- a namespace that
        retrieve() / retrieve_paged() never look up, since that KV attended to the tokens before it.  A segment at 0 is
        store_paged(tokens[:end], kv_caches, slot_mapping[:end]).  skip_existing: chunks held under the segment's prefix
        keys (stored alone), then under its derived keys, are skipped.  Any layout store_paged takes, every tier; the
        staging costs the raw bytes of the tokens stored.  TypeError for FP8 KV, ValueError for bad segments or a
        rotary range that does not fit, all before anything is hashed or written.  reshard_world_sizes is not
        consulted."""
        self._check_paged_args(tokens, slot_mapping, kv_caches)
        first = self._first(kv_caches)
        D = first.shape[-1] if self._mla else paged_layout(*kv_caches[0]).D
        slots = slot_mapping.to(first.device)
        self._store_segments(
            tokens, segments, rope, "vllm", first, D, lambda: KvView.from_paged(kv_caches, slots),
            lambda end: self.store_paged(tokens[:end], kv_caches, slot_mapping[:end], skip_existing, blocking),
            skip_existing, blocking)

    @_lmcache_nvtx_annotate
    @torch.no_grad()
    def store_segments(self, tokens: torch.Tensor, kv_tensors_raw: KVCache, segments, rope: RopeSpec,
                       skip_existing=True, blocking=True) -> None:
        """store_paged_segments for store()'s KV (per-layer (K, V) in the engine's vllm or huggingface format, or an MLA
        engine's latent per layer): a segment at 0 is store(tokens[:end], the KV's first end tokens)."""
        fmt = self.metadata.fmt
        self._check_store_args(tokens, kv_tensors_raw, fmt)
        first = self._first(kv_tensors_raw)
        self._store_segments(
            tokens, segments, rope, fmt, first, first.shape[-1],
            lambda: KvView.from_tuple(self._as_cuda_kv(kv_tensors_raw), fmt),
            lambda end: self.store(tokens[:end], self._kv_head(kv_tensors_raw, end, fmt), skip_existing, blocking),
            skip_existing, blocking)

    def _kv_head(self, kv_tensors_raw: KVCache, end: int, fmt: str) -> KVCache:
        """the first `end` tokens of store()'s KV, as views"""
        if self._mla:
            return tuple(t[:end] for t in kv_tensors_raw)
        tdim = KvView.token_dim(fmt) - 2         # a layer's token dimension
        return tuple((k.narrow(tdim, 0, end), v.narrow(tdim, 0, end)) for k, v in kv_tensors_raw)

    # ------------------------------------------------------------------ layer-wise segment store
    def _seg_side_stream(self, device) -> torch.cuda.Stream:
        """the engine's side stream of the layer-wise segment store's gathers on `device`"""
        s = self._seg_stream
        if s is None or s.device != torch.device(device):
            s = self._seg_stream = torch.cuda.Stream(device=device)
        return s

    def _store_segments_layerwise(self, tokens: torch.Tensor, segments, rope: RopeSpec, fmt: str, first: torch.Tensor,
                                  D: int, num_layers: int, ok: bool, view_fn: Callable[[], KvView],
                                  prefix_store: Callable[[int], LayerwiseStore], fallback: Callable,
                                  skip_existing: bool) -> LayerwiseStore:
        """Every layer-wise segment store.  At the call: the whole form's refusals; where the store cannot go layer by
        layer (not `ok`), a handle that runs the whole form at finish(); otherwise the whole form's plan, with the
        segment at 0 through prefix_store(end) (a layer-wise store handle), the staging (rope.StagedGather) and one
        tier handle per run (pipeline.begin_runs).  finish() then finishes the segment at 0 (its touches and put) and
        makes one put and one chain touch per run, in the whole form's order."""
        plans = self._segment_store_check(tokens, segments, rope, first, D)
        if not ok:
            return LayerwiseStore(num_layers, None, fallback)
        head, hashes, runs, _, _, shifts = self._segment_store_plan(tokens, plans, fmt, prefix_store, skip_existing)
        cs = self.chunk_size
        handles, gather = [], None
        if runs:
            try:
                view = view_fn()
                self._geom = (view.L, view.H, view.D, view.dtype)
                gather = StagedGather(view, runs, shifts, fmt, self._mla, rope, self._seg_side_stream(view.device),
                                      KvView.blob_shape)
                # one budget for the whole store: the segment at 0's encode takes its arena first
                budget = layerwise_store_budget_default() - (0 if head is None else arena_of(head._enc))
                handles = begin_runs(self.engine_.begin_layerwise_store,
                                     [KvView.from_blob(b, fmt) for b in gather.blobs], cs, budget)
            except BaseException:
                if head is not None:
                    head.close()
                raise
            if handles is None:
                # the tier writes no layer-wise containers for these chunks: the whole form runs at finish()
                if head is not None:
                    head.close()
                return LayerwiseStore(num_layers, None, fallback)

        def publish(stream, enc):
            if enc is None:                     # closed before finish(): nothing is stored
                return
            if enc.head is not None:
                enc.head.finish(stream)
            blocking = bool(getattr(self.engine_, "layerwise_store_blocking", False))
            for r, h in zip(runs, enc.handles):
                hs = hashes[r.plan.index]
                self.engine_.put_kv_chunks(self._derived_keys(hs[r.first:], fmt), None, 0, cs, blocking=blocking,
                                           encoded=h)
                self._touch_chain(hs, r.prefix_hits, len(hs), fmt)
        return LayerwiseStore(num_layers, SegmentsEncode(head, handles, gather), publish)

    @torch.no_grad()
    def store_paged_segments_layerwise(self, tokens: torch.Tensor, kv_caches, slot_mapping: torch.Tensor, segments,
                                       rope: RopeSpec, skip_existing=True) -> LayerwiseStore:
        """store_paged_segments(), with the KV handed over one layer at a time (LayerwiseStore: save_layer(l, stream)
        once layer l is written, finish(stream) after the last): the caches may still be unwritten when this is called.
        The refusals, the hash chain, the skip scan with its touches and the staging plan are made here; a segment at 0
        is store_paged_layerwise(tokens[:end], kv_caches, slot_mapping[:end], skip_existing).  Each save_layer(l)
        gathers layer l of every other segment, its keys turned by -start, into its own staged chunk blob with one
        b200kv_pack_chunks_layers_rope launch on the engine's side stream, and each segment's tier handle encodes (or,
        on the raw tiers, packs) it behind that launch.  LMCACHE_B200_LAYERWISE_STORE_MB bounds the encode arenas of the
        whole store (pipeline.begin_runs).  After finish() the tier holds the keys and bytes store_paged_segments
        stores.  Where store_paged_layerwise cannot go layer by layer (a torch-serde remote tier, a chunk size over the
        tier's layerwise_max_tokens) finish() runs store_paged_segments; a split (PagedAttention) cache needs no such
        fallback, since the encoders read the staged blobs."""
        self._check_paged_args(tokens, slot_mapping, kv_caches)
        first = self._first(kv_caches)
        D = first.shape[-1] if self._mla else paged_layout(*kv_caches[0]).D

        def fallback(stream, enc):
            with torch.cuda.stream(stream):
                self.store_paged_segments(tokens, kv_caches, slot_mapping, segments, rope, skip_existing)
        slots = slot_mapping.to(first.device)
        return self._store_segments_layerwise(
            tokens, segments, rope, "vllm", first, D, len(kv_caches), self._layerwise_store_ok(first.dtype),
            lambda: KvView.from_paged(kv_caches, slots),
            lambda end: self.store_paged_layerwise(tokens[:end], kv_caches, slot_mapping[:end], skip_existing),
            fallback, skip_existing)

    @torch.no_grad()
    def store_segments_layerwise(self, tokens: torch.Tensor, kv_tensors_raw: KVCache, segments, rope: RopeSpec,
                                 skip_existing=True) -> LayerwiseStore:
        """store_segments(), with the KV handed over one layer at a time (see store_paged_segments_layerwise):
        kv_tensors_raw is store()'s per-layer (K, V) tuple (or an MLA engine's latent per layer) on the GPU, possibly not
        yet written.  A segment at 0 is store_layerwise(tokens[:end], the KV's first end tokens).  KV that is not on the
        GPU or not laid out for the kernels to read in place (store_layerwise's rule) is stored by store_segments at
        finish()."""
        fmt = self.metadata.fmt
        self._check_store_args(tokens, kv_tensors_raw, fmt)
        first = self._first(kv_tensors_raw)

        def fallback(stream, enc):
            with torch.cuda.stream(stream):
                self.store_segments(tokens, kv_tensors_raw, segments, rope, skip_existing)
        ok = first.is_cuda and self._in_place(kv_tensors_raw) and self._layerwise_store_ok(first.dtype)
        return self._store_segments_layerwise(
            tokens, segments, rope, fmt, first, first.shape[-1], len(kv_tensors_raw), ok,
            lambda: KvView.from_tuple(kv_tensors_raw, fmt),
            lambda end: self.store_layerwise(tokens[:end], self._kv_head(kv_tensors_raw, end, fmt), skip_existing),
            fallback, skip_existing)

    # ------------------------------------------------------------------ CacheBlend's selective recomputation
    def blend_paged(self, kv_caches, slot_mapping: torch.Tensor, ret_mask: torch.Tensor, spec: BlendSpec) -> BlendPlan:
        """The plan of a blended prefill over the paged caches a (layer-wise) retrieve_paged_segments filled, in any
        layout it takes (an MLA engine: its latent caches): which tokens the model recomputes at each layer and, at each
        check layer of `spec`, the deviation of its fresh keys from the cached ones and the choice that follows
        (BlendPlan.check).  ret_mask: the retrieve's.  TypeError for an FP8 cache; ValueError for a spec that is not a
        BlendSpec or names a layer the caches do not have, and for a ret_mask of another length than slot_mapping.
        Nothing is enqueued but the mask's upload."""
        if self.metadata.fmt != "vllm":
            raise ValueError(f"paged KV caches use the vllm layout, engine fmt is {self.metadata.fmt}")
        self._check_kind(kv_caches, "kv_caches")
        first = self._first(kv_caches)
        check_blend_dtype(first.dtype)
        check_blend_args(spec, len(kv_caches), slot_mapping.numel(), ret_mask)
        slots = slot_mapping.to(first.device)
        return BlendPlan(KvView.from_paged(kv_caches, slots), ret_mask, spec, slots)

    def blend_paged_batch(self, kv_caches, slot_mapping: torch.Tensor, ret_masks: Sequence[torch.Tensor],
                          spec: BlendSpec) -> BatchBlendPlan:
        """blend_paged for a whole prefill batch: slot_mapping is the flattened batch's (as vLLM hands it to attention)
        and ret_masks holds one mask per request, in batch order -- the ret_mask of its (layer-wise)
        retrieve_paged_segments; a request that retrieved nothing (a decode step, a prompt whose documents all
        missed) is all False and all its rows are computed.  Each request keeps its own budgets; every check is one
        launch sequence for the whole batch (BatchBlendPlan.check).  The layouts and the refusals are blend_paged's,
        and ret_masks that is not a non-empty list of 1-D bool CPU tensors whose lengths add up to slot_mapping's is
        a ValueError.  Nothing is enqueued but the masks' upload."""
        if self.metadata.fmt != "vllm":
            raise ValueError(f"paged KV caches use the vllm layout, engine fmt is {self.metadata.fmt}")
        self._check_kind(kv_caches, "kv_caches")
        first = self._first(kv_caches)
        check_blend_dtype(first.dtype)
        check_blend_batch_args(spec, len(kv_caches), slot_mapping.numel(), ret_masks)
        slots = slot_mapping.to(first.device)
        return BatchBlendPlan(KvView.from_paged(kv_caches, slots), ret_masks, spec, slots)

    def blend(self, kv: KVCache, ret_mask: torch.Tensor, spec: BlendSpec) -> BlendPlan:
        """blend_paged for the dense per-layer views retrieve_segments / retrieve_segments_layerwise return (an MLA
        engine: its [T, D] latents).  A dense caller writes the fresh K / V of rows_at(layer) into the views itself
        (index_copy_ along the token dimension); BlendStep.slots is None.  The refusals are blend_paged's, and a kv of
        no layers (a total miss) is a ValueError: there is nothing to blend."""
        fmt = self.metadata.fmt
        if not len(kv):
            raise ValueError("blend needs the KV of a retrieve that hit: kv holds no layers")
        self._check_kind(kv, "kv")
        first = self._first(kv)
        check_blend_dtype(first.dtype)
        view = KvView.from_tuple(kv, fmt)
        check_blend_args(spec, view.L, view.ntokens, ret_mask)
        return BlendPlan(view, ret_mask, spec)

    def close(self):
        self.engine_.close()


class LMCacheEngineBuilder:
    """Process-wide engine registry (cache_engine.py:387-436)."""
    _instances: Dict[str, LMCacheEngine] = {}
    _cfgs: Dict[str, LMCacheEngineConfig] = {}
    _metadatas: Dict[str, LMCacheEngineMetadata] = {}

    @classmethod
    def get_or_create(cls, instance_id: str, config: LMCacheEngineConfig,
                      metadata: LMCacheEngineMetadata) -> LMCacheEngine:
        if instance_id not in cls._instances:
            engine = LMCacheEngine(config, metadata)
            cls._instances[instance_id] = engine
            cls._cfgs[instance_id] = config
            cls._metadatas[instance_id] = metadata
            return engine
        if cls._cfgs[instance_id] != config or cls._metadatas[instance_id] != metadata:
            raise ValueError(f"Instance {instance_id} already exists with a different configuration or metadata.")
        return cls._instances[instance_id]

    @classmethod
    def get(cls, instance_id: str) -> Optional[LMCacheEngine]:
        return cls._instances.get(instance_id)

    @classmethod
    def destroy(cls, instance_id: str) -> None:
        if instance_id in cls._instances:
            cls._instances[instance_id].close()
            cls._instances.pop(instance_id, None)
            cls._cfgs.pop(instance_id, None)
            cls._metadatas.pop(instance_id, None)
