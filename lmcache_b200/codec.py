"""Host-side driver of the CUDA codec: descriptors, buffers, and batched encode / decode calls.

This is plumbing above the C ABI (include/b200kv.h): PyTorch supplies device memory and streams,
libb200kv does all the work.  The serde plugins (storage_backend/serde/*.py) and the engine fast
paths are thin layers over `CacheGenCodec` and `LosslessCodec`, which share one host-side flow (`_ContainerIO`) and
differ only in their native calls and container checks.
"""
from __future__ import annotations

import contextlib
import ctypes
import threading
from dataclasses import dataclass
from typing import List, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from lmcache_b200 import _native as N

_DTYPE_CODE = {torch.bfloat16: N.DT_BF16, torch.float16: N.DT_FP16, torch.uint8: N.DT_U8,
               torch.float8_e4m3fn: N.DT_FP8_E4M3, torch.float8_e5m2: N.DT_FP8_E5M2}
_CODE_DTYPE = {v: k for k, v in _DTYPE_CODE.items()}
NATIVE_DTYPES = tuple(_DTYPE_CODE)      # the element dtypes the kernels move and the lossless codec stores
# CacheGen quantises 16-bit KV only; what a CacheGen serde or tier says to a one-byte (FP8) KV
_CACHEGEN_FP8 = ("CacheGen codes bfloat16 and float16 KV only, not {}: FP8 KV is stored bit-exact by the lossless codec "
                 "(local_serde: lossless / remote_serde: lossless), or raw on the cpu / cuda tiers")


def _stream_ptr(stream: Optional[torch.cuda.Stream]) -> int:
    return (stream if stream is not None else torch.cuda.current_stream()).cuda_stream


class PinnedBuffer:
    """Page-locked, device-mapped host memory from b200kv_pinned_alloc (replaces the reference's
    pageable .to("cpu") staging, local_backend.py:82-100)."""

    def __init__(self, nbytes: int):
        N.require_cuda()
        self.nbytes = int(nbytes)
        p = ctypes.c_void_p()
        N.check(N.lib().b200kv_pinned_alloc(ctypes.byref(p), self.nbytes), "pinned_alloc")
        self.host_ptr = p.value
        d = ctypes.c_void_p()
        N.check(N.lib().b200kv_host_device_ptr(p, ctypes.byref(d)), "host_device_ptr")
        self.dev_ptr = d.value
        self._arr = (ctypes.c_uint8 * self.nbytes).from_address(self.host_ptr)

    def view(self, offset: int = 0, nbytes: Optional[int] = None) -> memoryview:
        n = self.nbytes - offset if nbytes is None else nbytes
        return memoryview(self._arr)[offset:offset + n]

    def close(self):
        if self.host_ptr:
            self._arr = None
            N.lib().b200kv_pinned_free(ctypes.c_void_p(self.host_ptr))
            self.host_ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PagedLayout(NamedTuple):
    """A paged (key, value) cache pair as paged_layout recognises it.  kind: "flash" (FlashAttention: contiguous
    [nb, bs, H, D] or [num_slots, H, D] rows), "strided" (FlashInfer's kv[:, 0] / kv[:, 1] of a [nb, 2, bs, H, D] cache:
    [nb, bs, H, D] rows whose blocks start rows_per_block rows apart) or "split" (PagedAttention / xFormers: key
    [nb, H, D/x, bs, x], value [nb, H, D, bs], x elements per 16-byte key vector)."""
    kind: str
    nb: int
    bs: int
    H: int
    D: int
    rows_per_block: int      # "strided": block stride in rows; "flash": bs ([num_slots, H, D]: 1); "split": bs
    x: int                   # "split": elements per 16-byte key vector; 0 otherwise


def paged_layout(key: torch.Tensor, value: torch.Tensor) -> PagedLayout:
    """The layout of one layer's (key_cache, value_cache) pair, from shapes, strides and dtype alone (no data is read,
    any device).  ValueError for a pair no rule matches: key and value that disagree on nb, bs, H or D, D % x != 0, a
    split or strided pair in a dtype the mover does not move, or strides of no known layout."""
    if key.dtype != value.dtype:
        raise ValueError(f"key and value caches differ in dtype ({key.dtype}, {value.dtype})")
    native = key.dtype in _DTYPE_CODE
    if key.dim() == 5:
        if not native:
            raise ValueError(f"a split paged cache must hold a dtype the mover moves ({NATIVE_DTYPES}), not {key.dtype}")
        x = 16 // key.element_size()
        nb, H, dx, bs, kx = key.shape
        if value.dim() != 4:
            raise ValueError(f"a split key cache [nb, H, D/x, bs, x] needs a value cache [nb, H, D, bs], got "
                             f"{tuple(value.shape)}")
        vnb, vH, D, vbs = value.shape
        if (vnb, vH, vbs) != (nb, H, bs) or dx * kx != D:
            raise ValueError(f"split key {tuple(key.shape)} and value {tuple(value.shape)} caches disagree on nb, bs, H "
                             f"or D")
        if kx != x or D % x != 0:
            raise ValueError(f"a split paged cache of {key.dtype} needs x = {x} (16 bytes) and D % x == 0, got x = {kx}, "
                             f"D = {D}")
        if not (key.is_contiguous() and value.is_contiguous()):
            raise ValueError("split paged caches must be contiguous (they are written in place)")
        return PagedLayout("split", nb, bs, H, D, bs, x)
    if key.dim() not in (3, 4) or key.shape != value.shape:
        raise ValueError(f"paged key {tuple(key.shape)} and value {tuple(value.shape)} caches disagree on nb, bs, H or D "
                         f"(or are of no known layout)")
    if key.stride() != value.stride():
        raise ValueError("paged key and value caches must share strides")
    if key.dim() == 3:
        nb, bs, (H, D) = key.shape[0], 1, key.shape[1:]
    else:
        nb, bs, H, D = key.shape
    if key.is_contiguous():
        return PagedLayout("flash", nb, bs, H, D, bs, 0)
    HD = H * D
    if key.dim() == 4 and key.stride()[1:] == (HD, D, 1) and key.stride(0) % HD == 0 and key.stride(0) >= bs * HD:
        if not native:
            raise ValueError(f"a block-strided paged cache must hold a dtype the mover moves ({NATIVE_DTYPES}), not "
                             f"{key.dtype}")
        return PagedLayout("strided", nb, bs, H, D, key.stride(0) // HD, 0)
    raise ValueError("paged K/V caches must be contiguous [nb, bs, H, D] rows, block-strided rows (FlashInfer's kv[:, 0] "
                     "and kv[:, 1]) or PagedAttention's split pair (they are written in place)")


def strided_slots(slot_mapping: torch.Tensor, bs: int, rows_per_block: int) -> torch.Tensor:
    """The row of each slot in a block-strided cache, on the slot map's device: (s // bs) * rows_per_block + s % bs."""
    return torch.div(slot_mapping, bs, rounding_mode="floor") * rows_per_block + torch.remainder(slot_mapping, bs)


class KvView:
    """A KV source / destination for the native library: either one strided blob tensor or the engine's
    tuple of 2L per-layer tensors (no stack / permute / contiguous copies).  Keeps the tensors alive.

    A latent KV (multi-head latent attention, e.g. DeepSeek-V2/V3: one [T, 576] vector per token and layer, no V) is
    one tensor per layer where a (K, V) pair would be: a [L, T, D] blob, a tuple of L [T, D] tensors, or L paged
    [num_blocks, block_size, D] caches.  Its descriptor carries N.KV_LATENT; its L planes are coded with the key bins
    into version-4 containers."""

    def __init__(self, desc: N.KvDesc, keep, ntokens: int, device: torch.device, dtype: torch.dtype,
                 fmt: str = "vllm", blob: Optional[torch.Tensor] = None):
        self.desc = desc
        self._keep = keep
        self.ntokens = ntokens
        self.device = device
        self.dtype = dtype
        self.fmt = fmt
        self.blob = blob      # the single blob tensor behind this view, when there is one
        self.layout: Optional[str] = None    # a paged (K, V) view: "flash", "strided" or "split" (see paged_layout)
        self.slots: Optional[torch.Tensor] = None   # a paged view: the slot map its descriptor reads (rows if strided)

    @property
    def L(self): return self.desc.L
    @property
    def H(self): return self.desc.H
    @property
    def D(self): return self.desc.D
    @property
    def latent(self) -> bool: return bool(self.desc.dtype & N.KV_LATENT)
    @property
    def planes(self) -> int:
        """P: planes of the KV, L for a latent KV, 2L otherwise."""
        return self.L if self.latent else 2 * self.L
    @property
    def dtype_code(self) -> int:
        """N.DT_* of the elements (the descriptor's dtype without the latent and split flags)."""
        return int(self.desc.dtype) & ~(N.KV_LATENT | N.KV_PAGED_SPLIT)
    @property
    def split(self) -> bool:
        """a paged cache in PagedAttention's split layout: only the mover (pack / unpack) reads and writes it"""
        return bool(self.desc.dtype & N.KV_PAGED_SPLIT)

    def record_stream(self, stream: torch.cuda.Stream) -> None:
        """Mark every tensor behind the view as used by work on `stream`: the caching allocator reuses none of them
        before that work has run, even if the caller lets go of them first."""
        todo = [self._keep]
        while todo:
            x = todo.pop()
            if isinstance(x, torch.Tensor):
                x.record_stream(stream)
            elif isinstance(x, (list, tuple)):
                todo.extend(x)

    @staticmethod
    def _code(dtype: torch.dtype) -> int:
        if dtype not in _DTYPE_CODE:
            raise TypeError(f"KV dtype must be bfloat16, float16 or a one-byte type (uint8, float8_e4m3fn, "
                            f"float8_e5m2), got {dtype}")
        return _DTYPE_CODE[dtype]

    # A chunk blob holds t tokens of every layer: [L,2,t,H,D] (vllm) or [L,2,H,t,D] (huggingface); a latent one [L,t,D]
    # (vllm only).  Its token dimension, its shape, and the (L, H, D, dtype) read back from one (H = 1 for a latent blob,
    # as in its descriptor):
    @staticmethod
    def token_dim(fmt: str, latent: bool = False) -> int: return 1 if latent else 2 if fmt == "vllm" else 3
    @staticmethod
    def blob_shape(fmt: str, L: int, H: int, D: int, t: int, latent: bool = False) -> Tuple[int, ...]:
        if latent:
            return (L, t, D)
        return (L, 2, t, H, D) if fmt == "vllm" else (L, 2, H, t, D)
    @staticmethod
    def blob_geometry(blob: torch.Tensor, fmt: str) -> Tuple[int, int, int, torch.dtype]:
        if blob.dim() == 3:
            return blob.shape[0], 1, blob.shape[2], blob.dtype
        return blob.shape[0], blob.shape[3 if fmt == "vllm" else 2], blob.shape[4], blob.dtype

    @staticmethod
    def _latent_desc(L: int, D: int, dtype: torch.dtype) -> N.KvDesc:
        d = N.KvDesc()
        d.sKV = 0
        d.L, d.H, d.D = L, 1, D
        d.dtype = KvView._code(dtype) | N.KV_LATENT
        return d

    @staticmethod
    def from_blob(blob: torch.Tensor, fmt: str) -> "KvView":
        """blob: [L,2,T,H,D] (vllm) or [L,2,H,T,D] (huggingface); any strides with a contiguous last dim.
        A latent KV: [L,T,D] (vllm format only)."""
        if blob.dim() == 3:
            if fmt != "vllm":
                raise ValueError("a latent KV blob [L,T,D] has the vllm format only")
            if not blob.is_cuda:
                raise RuntimeError("KV blob must live on a CUDA device (no CPU fallback)")
            if blob.stride(2) != 1:
                blob = blob.contiguous()
            L, T, D = blob.shape
            d = KvView._latent_desc(L, D, blob.dtype)
            d.base = blob.data_ptr()
            d.planes = None
            d.sL, d.sT, d.sH = blob.stride(0), blob.stride(1), D
            return KvView(d, blob, T, blob.device, blob.dtype, fmt, blob)
        if blob.dim() != 5 or blob.shape[1] != 2:
            raise ValueError(f"expected a [L,2,..] KV blob, got {tuple(blob.shape)}")
        if not blob.is_cuda:
            raise RuntimeError("KV blob must live on a CUDA device (no CPU fallback)")
        if blob.stride(4) != 1:
            blob = blob.contiguous()
        if fmt == "vllm":
            L, _, T, H, D = blob.shape
            sL, sKV, sT, sH, _ = blob.stride()
        elif fmt == "huggingface":
            L, _, H, T, D = blob.shape
            sL, sKV, sH, sT, _ = blob.stride()
        else:
            raise ValueError(f"Invalid format: {fmt}")
        d = N.KvDesc()
        d.base = blob.data_ptr()
        d.planes = None
        d.sL, d.sKV, d.sT, d.sH = sL, sKV, sT, sH
        d.L, d.H, d.D = L, H, D
        d.dtype = KvView._code(blob.dtype)
        return KvView(d, blob, T, blob.device, blob.dtype, fmt, blob)

    @staticmethod
    def from_tuple(kv: Sequence[Tuple[torch.Tensor, torch.Tensor]], fmt: str) -> "KvView":
        """kv: L pairs of [T,H,D] (vllm) / [H,T,D] (huggingface) tensors, as passed to LMCacheEngine.store; or, for a
        latent KV, L [T,D] tensors (vllm format only)."""
        L = len(kv)
        if L == 0:
            raise ValueError("Empty kv_tensors")
        if isinstance(kv[0], torch.Tensor):
            return KvView._from_latent_tuple(kv, fmt)
        ref = kv[0][0]
        if not ref.is_cuda:
            raise RuntimeError("KV tensors must live on a CUDA device (no CPU fallback)")
        keep = []
        ptrs = (ctypes.c_void_p * (2 * L))()
        for l, (k, v) in enumerate(kv):
            for kvi, t in ((0, k), (1, v)):
                if t.shape != ref.shape or t.dtype != ref.dtype or t.device != ref.device:
                    raise ValueError("all K/V tensors must share shape, dtype and device")
                if t.stride() != ref.stride() or t.stride(2) != 1:
                    t = t.contiguous()
                    if t.stride() != ref.stride():
                        return KvView.from_tuple(tuple((a.contiguous(), b.contiguous()) for a, b in kv), fmt)
                keep.append(t)
                ptrs[kvi * L + l] = t.data_ptr()
        if fmt == "vllm":
            T, H, D = ref.shape
            sT, sH, _ = ref.stride()
        elif fmt == "huggingface":
            H, T, D = ref.shape
            sH, sT, _ = ref.stride()
        else:
            raise ValueError(f"Invalid format: {fmt}")
        d = N.KvDesc()
        d.base = None
        d.planes = ctypes.cast(ptrs, ctypes.POINTER(ctypes.c_void_p))
        d.sL = d.sKV = 0
        d.sT, d.sH = sT, sH
        d.L, d.H, d.D = L, H, D
        d.dtype = KvView._code(ref.dtype)
        return KvView(d, (keep, ptrs), T, ref.device, ref.dtype, fmt)

    @staticmethod
    def _from_latent_tuple(kv: Sequence[torch.Tensor], fmt: str) -> "KvView":
        if fmt != "vllm":
            raise ValueError("a latent KV has the vllm format only")
        ref = kv[0]
        if not ref.is_cuda:
            raise RuntimeError("KV tensors must live on a CUDA device (no CPU fallback)")
        if ref.dim() != 2:
            raise ValueError(f"a latent KV takes one [T,D] tensor per layer, got {tuple(ref.shape)}")
        if any(t.shape != ref.shape or t.dtype != ref.dtype or t.device != ref.device for t in kv):
            raise ValueError("all latent tensors must share shape, dtype and device")
        kv = [t if t.stride(1) == 1 else t.contiguous() for t in kv]
        if any(t.stride() != kv[0].stride() for t in kv):
            kv = [t.contiguous() for t in kv]
        L, (T, D) = len(kv), ref.shape
        ptrs = (ctypes.c_void_p * L)(*[t.data_ptr() for t in kv])
        d = KvView._latent_desc(L, D, ref.dtype)
        d.base = None
        d.planes = ctypes.cast(ptrs, ctypes.POINTER(ctypes.c_void_p))
        d.sL = 0
        d.sT, d.sH = kv[0].stride(0), D
        return KvView(d, (list(kv), ptrs), T, ref.device, ref.dtype, fmt)

    @staticmethod
    def _from_latent_paged(kv_caches: Sequence[torch.Tensor], slot_mapping: torch.Tensor) -> "KvView":
        ref = kv_caches[0]
        if not ref.is_cuda:
            raise RuntimeError("KV caches must live on a CUDA device (no CPU fallback)")
        if ref.dim() not in (2, 3):
            raise ValueError(f"a latent paged cache is [num_blocks, block_size, D] or [num_slots, D], got "
                             f"{tuple(ref.shape)}")
        for t in kv_caches:
            if t.shape != ref.shape or t.dtype != ref.dtype or t.device != ref.device:
                raise ValueError("all latent caches must share shape, dtype and device")
            if not t.is_contiguous():
                raise ValueError("paged latent caches must be contiguous (they are written in place)")
        L, D = len(kv_caches), ref.shape[-1]
        ptrs = (ctypes.c_void_p * L)(*[t.data_ptr() for t in kv_caches])
        d = KvView._latent_desc(L, D, ref.dtype)
        d.base = None
        d.planes = ctypes.cast(ptrs, ctypes.POINTER(ctypes.c_void_p))
        d.sL = 0
        d.sT, d.sH = D, D
        d.slot_map = slot_mapping.data_ptr()
        view = KvView(d, ([slot_mapping] + list(kv_caches), ptrs), slot_mapping.numel(), ref.device, ref.dtype, "vllm")
        view.slots = slot_mapping
        return view

    @staticmethod
    def from_paged(kv_caches: Sequence[Tuple[torch.Tensor, torch.Tensor]], slot_mapping: torch.Tensor) -> "KvView":
        """vLLM's paged KV cache used in place: `kv_caches` holds, per layer, the (key_cache, value_cache) pair shaped
        [num_blocks, block_size, H, D] (or already flattened [num_slots, H, D]); `slot_mapping` (int64, CUDA) gives the
        cache row of every token of the sequence (block * block_size + offset) -- what lmcache-vllm's
        lmcache_store_kv / lmcache_retrieve_kv gather and scatter with torch indexing (LLM_Engine.rst:91-109).
        The codec kernels read (encode) and write (decode) the rows directly; token i of the view is row
        slot_mapping[i].  A latent KV (vLLM's MLA cache): one [num_blocks, block_size, D] (or [num_slots, D]) tensor per
        layer instead of a pair."""
        L = len(kv_caches)
        if L == 0:
            raise ValueError("Empty kv_caches")
        if slot_mapping.dtype != torch.int64 or not slot_mapping.is_cuda or slot_mapping.dim() != 1:
            raise ValueError("slot_mapping must be a 1-D int64 CUDA tensor")
        slot_mapping = slot_mapping.contiguous()
        if isinstance(kv_caches[0], torch.Tensor):
            return KvView._from_latent_paged(kv_caches, slot_mapping)
        ref = kv_caches[0][0]
        if not ref.is_cuda:
            raise RuntimeError("KV caches must live on a CUDA device (no CPU fallback)")
        lay = paged_layout(*kv_caches[0])
        keep = [slot_mapping]
        ptrs = (ctypes.c_void_p * (2 * L))()
        for l, (k, v) in enumerate(kv_caches):
            if paged_layout(k, v) != lay or k.dtype != ref.dtype or k.device != ref.device or v.device != ref.device:
                raise ValueError("all K/V caches must share layout, shape, strides, dtype and device")
            for kvi, t in ((0, k), (1, v)):
                keep.append(t)
                ptrs[kvi * L + l] = t.data_ptr()
        H, D = lay.H, lay.D
        d = N.KvDesc()
        d.base = None
        d.planes = ctypes.cast(ptrs, ctypes.POINTER(ctypes.c_void_p))
        d.sL = d.sKV = 0
        d.sT, d.sH = H * D, D
        d.L, d.H, d.D = L, H, D
        d.dtype = KvView._code(ref.dtype)
        if lay.kind == "strided":
            # block b's rows start rows_per_block rows apart: every kernel reads the cache as rows through this slot map
            slot_mapping = strided_slots(slot_mapping, lay.bs, lay.rows_per_block)
            keep[0] = slot_mapping
        elif lay.kind == "split":
            d.sT, d.sH = lay.bs, 0                  # B200KV_KV_PAGED_SPLIT: sT carries the block size
            d.dtype |= N.KV_PAGED_SPLIT
        d.slot_map = slot_mapping.data_ptr()
        view = KvView(d, (keep, ptrs), slot_mapping.numel(), ref.device, ref.dtype, "vllm")
        view.layout = lay.kind
        view.slots = slot_mapping
        return view

    def rows(self, tokens: torch.Tensor) -> "KvView":
        """The same planes with token i of the new view at token tokens[i] of this one (int64 CUDA): a paged view reads
        through its slot map composed with `tokens`, a tuple view (no slot map) through `tokens` as rows.  Not for blob
        views, whose descriptor has no slot map to compose."""
        if self.blob is not None:
            raise ValueError("a blob view has no rows to compose")
        d = N.KvDesc.from_buffer_copy(self.desc)
        slots = tokens if self.slots is None else self.slots[tokens]
        slots = slots.contiguous()
        d.slot_map = slots.data_ptr()
        view = KvView(d, (self._keep, slots), slots.numel(), self.device, self.dtype, self.fmt)
        view.layout = self.layout
        view.slots = slots
        return view

    def staged(self, tok_begin: int) -> "KvView":
        """Tokens [tok_begin, T) of this view packed into one device blob [L, 2, T - tok_begin, H, D] by one mover launch
        on the current stream, as a blob view (the view keeps the blob alive).  What the container tiers encode from when
        the cache is split: its HBM cost is the raw bytes of those tokens."""
        n = self.ntokens - tok_begin
        buf, (blob,) = self.pack_chunks(tok_begin, n)
        return KvView.from_blob(blob, "vllm")

    def unpack_blob(self, blob: torch.Tensor, tok_begin: int) -> None:
        """Write the t tokens of a vllm blob [L, 2, t, H, D] to tokens [tok_begin, tok_begin + t) of this view with one
        b200kv_unpack_chunks launch on the current stream (the mover: any layout the view has)."""
        t = blob.shape[2]
        if t == 0:
            return
        blob = blob.contiguous()
        with torch.cuda.device(self.device):
            N.check(N.lib().b200kv_unpack_chunks(ctypes.c_void_p(blob.data_ptr()), blob.numel() * blob.element_size(),
                                                 1, t, t, 0, ctypes.byref(self.desc), tok_begin, _stream_ptr(None)),
                    "unpack_chunks")

    def pack_chunks(self, tok_begin: int, chunk_size: int) -> Tuple[torch.Tensor, List[torch.Tensor]]:
        """Gather tokens [tok_begin, T), at least one, into blobs of chunk_size tokens (the last may be shorter) with one
        b200kv_pack_chunks launch on the current stream.  Returns the buffer and the blobs, back to back views of it."""
        n_tok = self.ntokens - tok_begin
        n_chunks = (n_tok + chunk_size - 1) // chunk_size
        per_tok = self.planes * self.H * self.D
        stride = per_tok * chunk_size
        buf = torch.empty(n_chunks * stride, dtype=self.dtype, device=self.device)
        with torch.cuda.device(self.device):
            N.check(N.lib().b200kv_pack_chunks(ctypes.byref(self.desc), tok_begin, n_chunks, chunk_size,
                                               n_tok - (n_chunks - 1) * chunk_size, int(self.fmt == "huggingface"),
                                               ctypes.c_void_p(buf.data_ptr()), stride * buf.element_size(),
                                               _stream_ptr(None)), "pack_chunks")
        sizes = [min(chunk_size, n_tok - j * chunk_size) for j in range(n_chunks)]
        shape = (lambda t: (self.L, t, self.D)) if self.latent else \
            (lambda t: self.blob_shape(self.fmt, self.L, self.H, self.D, t))
        return buf, [buf[j * stride: j * stride + per_tok * t].view(shape(t)) for j, t in enumerate(sizes)]


def _parse_preamble(buf, total: Optional[int], versions: Tuple[int, ...],
                    bad_version: str) -> Tuple[memoryview, N.Header]:
    """The checks every B2KV header parse starts with: the buffer holds a header, the magic, a version of `versions`
    (else ValueError(bad_version with the version)), total_bytes within the container (`total`: its size, when `buf` is
    a prefix of it) and no encoder error status.  Returns the buffer's memoryview and the header."""
    mv = memoryview(buf)
    if mv.nbytes < N.HEADER_BYTES:
        raise ValueError("buffer too small for a B2KV container")
    hd = N.Header.from_buffer_copy(bytes(mv[:N.HEADER_BYTES]))
    if hd.magic != N.MAGIC:
        raise ValueError("not a B2KV container (bad magic)")
    if hd.version not in versions:
        raise ValueError(bad_version.format(hd.version))
    if hd.total_bytes > (mv.nbytes if total is None else total):
        raise ValueError("truncated B2KV container")
    if hd.status != 0:
        raise ValueError(f"B2KV container carries encoder error status {hd.status}")
    return mv, hd


def _plane_offsets(buf, versions: Tuple[int, ...], native, what: str) -> Optional[np.ndarray]:
    """plane_offsets / lossless_plane_offsets: `native` (b200kv_plane_offsets or b200kv_lossless_plane_offsets) on a
    container of one of `versions`, None for any other version and for lengths that do not add up."""
    src = np.frombuffer(buf, dtype=np.uint8)
    version, L = (int(v) for v in src[4:12].view(np.uint32))
    if version not in versions:
        return None
    o = np.empty(N.planes_of(version, L) + 1, dtype=np.int64)
    rc = N.check(native(src.ctypes.data, src.size, o.ctypes.data, o.size), what)
    return o if rc == 0 else None


def parse_header(buf, total: Optional[int] = None) -> N.Header:
    """Validate and return the 64-byte header of a B2KV container (bytes / bytearray / memoryview).  `buf` is the whole
    container, or -- when `total`, the size of the whole container, is given -- a prefix of it that holds the header
    and, for versions 3 and 4, the nb map after it."""
    mv, hd = _parse_preamble(buf, total, (1, 2, 3, 4), "unsupported B2KV version {}")
    nb = None
    if hd.version >= 3:
        P = N.planes_of(hd.version, hd.L)
        if not 0 < hd.L <= N.MAX_PLANES // 2 or mv.nbytes < N.HEADER_BYTES + P:
            raise ValueError("B2KV header carries an impossible shape")
        nb = list(bytes(mv[N.HEADER_BYTES:N.HEADER_BYTES + P]))
    check_header(hd, nb)
    return hd


def plane_offsets(buf) -> Optional[np.ndarray]:
    """Boundaries of the planes' streams in a version-3 or version-4 container (`buf`: at least its fixed sections), from
    its half-lengths section: int64[P + 1] (P = 2L planes, keys of layer p then values of layer p - L; P = L latent
    planes in version 4), plane p is bytes [o[p], o[p + 1]) of the container; o[0] is the start of the payload and
    o[P] == total_bytes.  None for versions 1 and 2, and when the lengths do not add up to the header's payload (a
    damaged container: it is only ever uploaded whole)."""
    return _plane_offsets(buf, (3, 4), N.lib().b200kv_plane_offsets, "plane_offsets")


def container_layout_of(hd: "N.Header") -> "N.Layout":
    """Section offsets of a parsed container."""
    return N.container_layout(hd.L, hd.H, hd.D, hd.ntokens, N.coder_of_version(hd.version))


def check_header(hd: "N.Header", nb: Optional[Sequence[int]] = None) -> None:
    """Structural checks that make a damaged blob a miss (ValueError) instead of bad device addresses: the section
    offsets follow from (L, H, D, ntokens, version), so total_bytes must be exactly fixed sections + payload.  A compact
    container (version 3, or 4 for a latent KV) also carries its nb map -- the P bytes after the header (P = 2L, or L),
    passed as `nb` and attached to the header as `hd.nb`: the symbols per plane its writer's bin table allowed."""
    if not (0 < hd.L <= N.MAX_PLANES // 2 and hd.H > 0 and hd.D > 0 and hd.ntokens > 0):
        raise ValueError("B2KV header carries an impossible shape")
    if hd.max_dtype not in (N.DT_BF16, N.DT_FP16):
        raise ValueError("B2KV header carries an unknown max_dtype")
    hd.nb = None
    P = N.planes_of(hd.version, hd.L)
    if hd.version >= 3:
        if nb is None or len(nb) != P or any(v < 4 or v > 32 or v % 2 for v in nb):
            raise ValueError(f"B2KV v{hd.version} header: bad nb map")
        if hd.ntokens > N.GROUP_TOKENS:
            raise ValueError(f"B2KV v{hd.version} header: more than 256 tokens")
        hd.nb = [int(v) for v in nb]
    lo = container_layout_of(hd)
    if hd.ngroups != (hd.ntokens + N.GROUP_TOKENS - 1) // N.GROUP_TOKENS:
        raise ValueError("B2KV header: ngroups does not match ntokens")
    if hd.total_bytes != lo.off_payload + hd.payload_bytes:
        raise ValueError("B2KV header: total_bytes != fixed sections + payload_bytes (truncated or corrupt)")
    nstreams = P * hd.H * hd.D * hd.ngroups
    per_stream = 1 if hd.version == 1 else 4          # rANS streams are >= 4 bytes, arithmetic-coder streams >= 1
    if hd.payload_bytes < per_stream * nstreams or hd.payload_bytes > lo.max_total_bytes:
        raise ValueError("B2KV header: payload_bytes impossible for this shape")


class SegmentLayout(NamedTuple):
    """How a layer-wise store assembles a container of some number of tokens (pipeline.segment_copy_ranges): bytes
    [0, head) come from the chunk's fixed image, the streams start at `payload`, and -- lossless containers only -- plane
    p's raw rows lie at head + p * raw_plane, raw_plane bytes each (the last plane's range runs up to `payload`)."""
    head: int
    payload: int
    raw_plane: int = 0


@dataclass
class EncodedBatch:
    """Device-resident result of one encode call: n containers at `stride` in `buf`."""
    buf: torch.Tensor            # uint8 device staging
    stride: int
    sizes: List[int]             # total bytes per container (host, valid after the call returns)
    max_dtype: int = 0           # dtype code of the stored row maxima (== input dtype)
    coder: int = N.CODER_RANS    # which entropy coder filled the payloads (container version - 1)

    def container(self, j: int) -> torch.Tensor:
        return self.buf[j * self.stride: j * self.stride + self.sizes[j]]


@dataclass
class EncodeTicket:
    """An encode in flight (encode_async).  `wait()` blocks the calling host thread -- not the stream --
    until the kernels are done and returns the batch with its sizes."""
    buf: torch.Tensor
    stride: int
    n_chunks: int
    sizes_buf: "PinnedBuffer"
    event: torch.cuda.Event
    max_dtype: int
    coder: int
    keep: object = None          # keeps the source view (and through it the KV tensors) alive until the kernels ran
    codec: object = None         # told the measured bits per symbol (picks the next call's kernel variant)
    stats: tuple = (0, 0.0)      # (fixed bytes per container, symbols in this call)

    def wait(self) -> EncodedBatch:
        self.event.synchronize()
        self.keep = None
        sizes = list((ctypes.c_uint64 * self.n_chunks).from_address(self.sizes_buf.host_ptr))
        for j, s in enumerate(sizes):
            if s < N.HEADER_BYTES or s > self.stride:
                raise N.NativeError(f"encoder produced an invalid container size {s} for chunk {j}")
        if self.codec is not None and self.stats[1] > 0:
            self.codec._last_bits_per_symbol = 8.0 * (sum(sizes) - self.n_chunks * self.stats[0]) / self.stats[1]
            self.codec = None
        return EncodedBatch(self.buf, self.stride, [int(s) for s in sizes], self.max_dtype, self.coder)


class _ContainerIO:
    """The host-side flow both codecs share around their own native calls: encode_async and its blocking and host-copy
    forms, decode (header checks, then the upload of host containers through the codec's staging), decode_raw /
    decode_raw_heads and the decode plan calls, and the ordering of calls that share buffers.  A codec provides its
    container check (parse_header, accepts), coder_for, layout, out_stride, decode_layers, and these hooks:

    _check_source(view)                     ValueError for a KV the codec cannot encode (default: none)
    _encode_ws_bytes(view, chunk_size, n_chunks, coder)
    _encode_launch(view, tok_begin, n_tokens, chunk_size, n_chunks, last, coder, out, stride, sizes, stream)
                                            enqueue the encode; returns the EncodeTicket fields it sets
    _decode_ws_bytes(dst, src_H, tmax, n)   a decode plan's workspace bytes (never negative)
    _plan_native(args, coder, dst, status, ws, stream, window)
                                            the plan call, whole (window ()) or over head windows; returns the plan
    _check_container(hd, dst)               decode()'s check of a header beyond its kind and shape"""

    def _init_io(self) -> None:
        self._enc_lock = threading.RLock()
        self._dec_lock = threading.Lock()
        self._enc_event: Optional[torch.cuda.Event] = None
        self._enc_ws: Optional[torch.Tensor] = None
        self._dec_ws: Optional[torch.Tensor] = None
        self._enc_out: Optional[torch.Tensor] = None
        self._sizes: Optional[PinnedBuffer] = None
        self._dec_in: Optional[torch.Tensor] = None
        self._dec_event: Optional[torch.cuda.Event] = None
        self._dec_status: Optional[PinnedBuffer] = None   # uint32 per chunk of the last decode call (mapped host memory)
        self._dec_status_n = 0
        self._pin_lock = threading.Lock()
        self._pin_in_lock = threading.Lock()
        self._pin_out: Optional[PinnedBuffer] = None      # containers on their way out (encode_to_pinned)
        self._pin_in: Optional[PinnedBuffer] = None       # containers on their way in (pinned_staging)

    @staticmethod
    def _grow(t: Optional[torch.Tensor], nbytes: int, device) -> torch.Tensor:
        if t is None or t.numel() < nbytes or t.device != device:
            t = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
        return t

    def _check_source(self, view: KvView) -> None:
        """ValueError for a KV this codec cannot encode"""

    # ------------------------------------------------------------------ encode
    def encode_async(self, view: KvView, tok_begin: int, n_tokens: int, chunk_size: int,
                     stream: Optional[torch.cuda.Stream] = None, out: Optional[torch.Tensor] = None,
                     sizes: Optional[PinnedBuffer] = None) -> EncodeTicket:
        """Enqueue the encode of tokens [tok_begin, tok_begin + n_tokens) of `view` as ceil(n_tokens / chunk_size)
        containers on `stream` and return at once: no host synchronisation.  The containers land in `out` (device,
        `out_stride` apart; the codec's own staging when None) and their sizes in `sizes` (mapped page-locked memory,
        8 bytes per chunk; the codec's own when None) -- both are valid once the ticket's event has completed.
        The KV is read in stream order, so the caller may reuse it for later work on the same stream (this is the
        snapshot a non-blocking store needs; reference cache_engine.py:274-275 materialises chunk copies instead)."""
        if n_tokens <= 0:
            raise ValueError("n_tokens must be positive")
        self._check_source(view)
        coder = self.coder_for(chunk_size, view.latent)
        n_chunks = (n_tokens + chunk_size - 1) // chunk_size
        last = n_tokens - (n_chunks - 1) * chunk_size
        stride = self.out_stride(view.L, view.H, view.D, chunk_size, view.latent)
        with self._enc_lock, torch.cuda.device(view.device):
            tstream = stream if stream is not None else torch.cuda.current_stream()
            ws_bytes = self._encode_ws_bytes(view, chunk_size, n_chunks, coder)
            own_out, own_sizes = out is None, sizes is None
            need_out = stride * n_chunks + N.READ_SLACK if own_out else 0
            # the workspace (and the codec's own staging) are shared by consecutive calls: order after the previous
            # encode on whatever stream it ran; never free a buffer a kernel may still be using
            if self._enc_event is not None:
                grow = (self._enc_ws is None or self._enc_ws.numel() < ws_bytes or self._enc_ws.device != view.device or
                        (own_out and (self._enc_out is None or self._enc_out.numel() < need_out)))
                if grow:
                    self._enc_event.synchronize()
                else:
                    tstream.wait_event(self._enc_event)
            self._enc_ws = self._grow(self._enc_ws, ws_bytes, view.device)
            if own_out:
                self._enc_out = self._grow(self._enc_out, need_out, view.device)
                out = self._enc_out
            elif out.numel() < stride * n_chunks:
                raise ValueError("encode output buffer too small")
            if own_sizes:
                if self._sizes is None or self._sizes.nbytes < 8 * n_chunks:
                    self._sizes = PinnedBuffer(max(4096, 8 * n_chunks))
                sizes = self._sizes
            elif sizes.nbytes < 8 * n_chunks:
                raise ValueError("sizes buffer too small")
            extra = self._encode_launch(view, tok_begin, n_tokens, chunk_size, n_chunks, last, coder, out, stride, sizes,
                                        tstream)
            ev = torch.cuda.Event()
            ev.record(tstream)
            self._enc_event = ev
            return EncodeTicket(out, stride, n_chunks, sizes, ev, view.dtype_code, coder, view, **extra)

    def encode(self, view: KvView, tok_begin: int, n_tokens: int, chunk_size: int,
               stream: Optional[torch.cuda.Stream] = None, out: Optional[torch.Tensor] = None) -> EncodedBatch:
        """encode_async + one event wait: blocks until the containers' sizes are known; payloads stay on the device.
        With out=None the batch aliases the codec's staging, which the next encode call overwrites."""
        return self.encode_async(view, tok_begin, n_tokens, chunk_size, stream, out).wait()

    def encode_to_host(self, view: KvView, tok_begin: int, n_tokens: int, chunk_size: int,
                       stream: Optional[torch.cuda.Stream] = None) -> List[bytes]:
        """encode + one device->host copy per container through the codec's page-locked slab, returned as immutable
        bytes (the Serializer.to_bytes contract, serde.py:12-27).  The encoder lock is held until the copies are done:
        the staging the batch aliases cannot be overwritten by a concurrent encode."""
        with self._enc_lock, self.encode_to_pinned(view, tok_begin, n_tokens, chunk_size, stream) as views:
            return [bytes(v) for v in views]

    @contextlib.contextmanager
    def encode_to_pinned(self, view: KvView, tok_begin: int, n_tokens: int, chunk_size: int,
                         stream: Optional[torch.cuda.Stream] = None):
        """encode + one device->host copy per container into the codec's page-locked slab (kept across calls, grown on
        demand); yields one writable memoryview per container.  The views -- e.g. handed to a socket send -- are valid
        inside the `with` block only: the slab is reused by the next call (serialised by a lock)."""
        with self._enc_lock, self._pin_lock:
            batch = self.encode(view, tok_begin, n_tokens, chunk_size, stream)
            total = sum((s + 15) & ~15 for s in batch.sizes)
            if self._pin_out is None or self._pin_out.nbytes < total:
                if self._pin_out is not None:
                    self._pin_out.close()
                self._pin_out = PinnedBuffer(max(total, 1) * 5 // 4)
            pin = self._pin_out
            lib = N.lib()
            sp = _stream_ptr(stream)
            offs, o = [], 0
            with torch.cuda.device(view.device):
                for j, s in enumerate(batch.sizes):
                    N.check(lib.b200kv_copy_async(pin.host_ptr + o, batch.buf.data_ptr() + j * batch.stride, s, sp), "copy")
                    offs.append(o)
                    o += (s + 15) & ~15
                N.check(lib.b200kv_stream_sync(sp), "stream_sync")
            views = [pin.view(offs[j], batch.sizes[j]) for j in range(len(offs))]
            for v in views:
                self.parse_header(v)        # raises on encoder error status
            try:
                yield views
            finally:
                del views

    # ------------------------------------------------------------------ decode
    @contextlib.contextmanager
    def pinned_staging(self, nbytes: int):
        """A page-locked receive slab of at least nbytes (kept across calls): a remote tier reads containers straight
        into it and decode() uploads from it with true asynchronous copies."""
        with self._pin_in_lock:
            if self._pin_in is None or self._pin_in.nbytes < nbytes:
                if self._pin_in is not None:
                    self._dec_sync()
                    self._pin_in.close()
                self._pin_in = PinnedBuffer(max(nbytes, 1) * 5 // 4)
            try:
                yield self._pin_in
            finally:
                self._dec_sync()       # the uploads out of the slab must finish before the next user overwrites it

    def _dec_sync(self) -> None:
        if self._dec_event is not None:
            self._dec_event.synchronize()

    def _order_decode(self, tstream, need_in: int, need_ws: int) -> None:
        """staging / workspace are reused across calls: order after the previous decode and never free a
        buffer a kernel may still be reading."""
        if self._dec_event is None:
            return
        if ((self._dec_in is not None and self._dec_in.numel() < need_in) or
                (self._dec_ws is not None and self._dec_ws.numel() < need_ws)):
            self._dec_event.synchronize()
        else:
            tstream.wait_event(self._dec_event)

    def _status_buffer(self, n: int) -> PinnedBuffer:
        """the mapped page-locked status words of a decode call of n containers (grown on demand)"""
        if self._dec_status is None or self._dec_status.nbytes < 4 * n:
            if self._dec_status is not None:
                self._dec_sync()
            self._dec_status = PinnedBuffer(max(4096, 8 * n))
        self._dec_status_n = n
        return self._dec_status

    def decode_status(self) -> List[int]:
        """Wait for the most recent decode call and return its per-chunk status words (0 = clean; bit 0: a rANS stream
        did not return to its initial state, bit 1: stream offsets beyond the payload, bit 2: the header's version is not
        the one the call's coder named).  A nonzero word means the container's bytes were damaged after its header was
        written, or it was handed to the wrong decode: treat the chunk as a miss."""
        with self._dec_lock:
            if self._dec_status is None or self._dec_event is None:
                return []
            self._dec_event.synchronize()
            return list((ctypes.c_uint32 * self._dec_status_n).from_address(self._dec_status.host_ptr))

    def decode_raw(self, base_ptr: int, buf_bytes: int, offsets: Sequence[int], totals: Sequence[int],
                   ntokens: Sequence[int], dst: KvView, dst_tok: Sequence[int], max_dtype: int, coder: int,
                   stream: Optional[torch.cuda.Stream] = None, _locked: bool = False) -> None:
        """Decode containers that already sit in device memory at base_ptr + offsets[j] (asynchronous): decode_plan on
        the codec's own workspace and status words, then decode_layers over every layer.  `buf_bytes` is the size of the
        buffer behind base_ptr: it must extend N.READ_SLACK bytes past every container (checked by the library);
        totals[j] = header.total_bytes.  max_dtype and coder are the headers' (N.coder_of_version); a lossless
        container's max_dtype is its element dtype, which must be dst's."""
        self._decode_raw(base_ptr, buf_bytes, offsets, totals, ntokens, dst, dst_tok, max_dtype, coder, stream, _locked)

    def decode_raw_heads(self, base_ptr: int, buf_bytes: int, offsets: Sequence[int], totals: Sequence[int],
                         ntokens: Sequence[int], dst: KvView, dst_tok: Sequence[int], max_dtype: int, coder: int,
                         src_H: int, src_head0: Sequence[int], dst_head0: Sequence[int], n_heads: Sequence[int],
                         stream: Optional[torch.cuda.Stream] = None) -> None:
        """decode_raw for a window of each container's heads (decode_plan_heads): every container holds src_H heads, and
        its heads [src_head0[j], src_head0[j] + n_heads[j]) land in dst's heads from dst_head0[j] on, at token
        dst_tok[j] (a lossless container's bit for bit as the source layout stored them).  The rest of dst is left as it
        was."""
        self._decode_raw(base_ptr, buf_bytes, offsets, totals, ntokens, dst, dst_tok, max_dtype, coder, stream, False,
                         (src_H, src_head0, dst_head0, n_heads))

    def _decode_raw(self, base_ptr, buf_bytes, offsets, totals, ntokens, dst: KvView, dst_tok, max_dtype, coder, stream,
                    _locked: bool, heads=None) -> None:
        n = len(offsets)
        if n == 0:
            return

        def run():
            tstream = stream if stream is not None else torch.cuda.current_stream()
            ws_bytes = self._decode_ws_bytes(dst, heads[0] if heads else dst.H, max(ntokens), n)
            if not _locked:
                self._order_decode(tstream, 0, ws_bytes)
            self._dec_ws = self._grow(self._dec_ws, ws_bytes, dst.device)
            plan, _ = self._plan(base_ptr, buf_bytes, offsets, totals, ntokens, dst, dst_tok, max_dtype, coder, heads,
                                 self._dec_ws, self._status_buffer(n).dev_ptr, tstream)
            self.decode_layers(plan, 0, dst.L, tstream)
            if self._dec_event is None:
                self._dec_event = torch.cuda.Event()
            self._dec_event.record(tstream)

        if _locked:
            run()
        else:
            with self._dec_lock, torch.cuda.device(dst.device):
                run()

    def decode_plan(self, base_ptr: int, buf_bytes: int, offsets: Sequence[int], totals: Sequence[int],
                    ntokens: Sequence[int], dst: KvView, dst_tok: Sequence[int], max_dtype: int, coder: int,
                    stream: torch.cuda.Stream, status_ptr: int = 0) -> Tuple[ctypes.Structure, torch.Tensor]:
        """First half of decode_raw (b200kv_decode_plan; b200kv_lossless_decode_plan): enqueue on `stream` the kernels
        that read what the plan needs of every container -- its fixed sections; [0, off_raw) of a lossless one -- and
        return (plan, workspace).  The payloads may still be uploading; decode_layers decodes a range of layers once its
        bytes are there.  The workspace is the caller's (not the codec's shared one), so plans of concurrent retrieves do
        not order after each other; it must be released only after the plan's last decode_layers (it is recorded on
        `stream`: run those on the same stream)."""
        return self._plan(base_ptr, buf_bytes, offsets, totals, ntokens, dst, dst_tok, max_dtype, coder, None, None,
                          status_ptr, stream)

    def decode_plan_heads(self, base_ptr: int, buf_bytes: int, offsets: Sequence[int], totals: Sequence[int],
                          ntokens: Sequence[int], dst: KvView, dst_tok: Sequence[int], max_dtype: int, coder: int,
                          src_H: int, src_head0: Sequence[int], dst_head0: Sequence[int], n_heads: Sequence[int],
                          stream: torch.cuda.Stream, status_ptr: int = 0) -> Tuple[ctypes.Structure, torch.Tensor]:
        """decode_plan for head windows (see decode_raw_heads); decode_layers runs the plan."""
        return self._plan(base_ptr, buf_bytes, offsets, totals, ntokens, dst, dst_tok, max_dtype, coder,
                          (src_H, src_head0, dst_head0, n_heads), None, status_ptr, stream)

    def _plan(self, base_ptr, buf_bytes, offsets, totals, ntokens, dst: KvView, dst_tok, max_dtype, coder, heads, ws,
              status_ptr, stream) -> Tuple[ctypes.Structure, torch.Tensor]:
        """the plan call of decode_plan (heads None) or decode_plan_heads (heads: (src_H, src_head0, dst_head0,
        n_heads)); ws None: a workspace of the caller's own, recorded on `stream`"""
        n = len(offsets)
        if ws is None:
            ws = torch.empty(self._decode_ws_bytes(dst, heads[0] if heads else dst.H, max(ntokens), n),
                             dtype=torch.uint8, device=dst.device)
            ws.record_stream(stream)
        args = (base_ptr, int(buf_bytes), N.i64_array(list(offsets)), N.i64_array(list(totals)),
                N.i32_array(list(ntokens)), N.i64_array(list(dst_tok)), n, int(max_dtype))
        window = () if heads is None else (int(heads[0]), *(N.i32_array(list(h)) for h in heads[1:]))
        return self._plan_native(args, coder, dst, status_ptr or None, ws, stream, window), ws

    def decode(self, containers: Sequence[Union[bytes, bytearray, memoryview, torch.Tensor]], dst: KvView,
               dst_tok: Sequence[int], stream: Optional[torch.cuda.Stream] = None) -> None:
        """Decode containers into `dst` at token offsets `dst_tok` (asynchronous on `stream`).  Host containers are
        uploaded first; a single 16-byte-aligned device tensor is used in place.  ValueError for a container that is not
        of this codec's family, whose kind (one plane per layer or a (K, V) pair) or shape is not dst's, that the codec
        refuses (CacheGen: written with other bins; lossless: of another dtype than dst's), or that does not fit dst's
        tokens; and for containers of one call that differ in max_dtype or version."""
        n = len(containers)
        if n == 0:
            return
        heads = []
        for c in containers:
            if isinstance(c, torch.Tensor):
                hd = self.parse_header(c[:N.HEADER_BYTES + N.MAX_PLANES].cpu().numpy().tobytes(), c.numel())
            else:
                hd = self.parse_header(c)
            if (hd.version in (4, 6)) != dst.latent:          # versions 4 and 6 hold one plane per layer
                raise ValueError(f"a version-{hd.version} container does not fit a destination of "
                                 f"{'one plane' if dst.latent else 'a (K, V) pair'} per layer")
            self._check_container(hd, dst)
            if (hd.L, hd.H, hd.D) != (dst.L, dst.H, dst.D):
                raise ValueError(f"container shape L/H/D={hd.L}/{hd.H}/{hd.D} does not match destination "
                                 f"{dst.L}/{dst.H}/{dst.D}")
            heads.append(hd)
        max_dtype = heads[0].max_dtype
        if any(h.max_dtype != max_dtype or h.version != heads[0].version for h in heads):
            raise ValueError("containers of one decode call must share max_dtype and container version")
        coder = N.coder_of_version(heads[0].version)
        totals = [int(h.total_bytes) for h in heads]
        ntoks = [int(h.ntokens) for h in heads]
        for tok, nt in zip(dst_tok, ntoks):
            if tok < 0 or tok + nt > dst.ntokens:
                raise ValueError(f"container of {nt} tokens at offset {tok} does not fit a {dst.ntokens}-token destination")
        lib = N.lib()
        with self._dec_lock, torch.cuda.device(dst.device):
            tstream = stream if stream is not None else torch.cuda.current_stream()
            sp = tstream.cuda_stream
            need_in = sum((t + 15) & ~15 for t in totals) + N.READ_SLACK
            self._order_decode(tstream, need_in, self._decode_ws_bytes(dst, dst.H, max(ntoks), n))
            if n == 1 and isinstance(containers[0], torch.Tensor) and containers[0].is_cuda \
                    and containers[0].data_ptr() % 16 == 0 and containers[0].numel() >= totals[0] + N.READ_SLACK:
                keep_dev = containers[0]
                self.decode_raw(keep_dev.data_ptr(), keep_dev.numel(), [0], totals, ntoks, dst, dst_tok, max_dtype, coder,
                                tstream, _locked=True)
                return
            self._dec_in = self._grow(self._dec_in, need_in, dst.device)
            base_ptr = self._dec_in.data_ptr()
            offsets, o = [], 0
            for c, nb in zip(containers, totals):
                if isinstance(c, torch.Tensor):
                    keep = c
                    src_ptr = c.data_ptr()
                else:
                    keep = np.frombuffer(c, dtype=np.uint8, count=nb)   # zero-copy view of bytes/bytearray/memoryview
                    src_ptr = keep.ctypes.data
                # pageable sources are staged by the driver before the call returns
                N.check(lib.b200kv_copy_async(base_ptr + o, src_ptr, nb, sp), "copy")
                del keep
                offsets.append(o)
                o += (nb + 15) & ~15
            self.decode_raw(base_ptr, self._dec_in.numel(), offsets, totals, ntoks, dst, dst_tok, max_dtype, coder, tstream,
                            _locked=True)


class CacheGenCodec(_ContainerIO):
    """Batched CacheGen encode / decode on the current CUDA device.

    Thread model: one encoder and one decoder may run concurrently from different threads (the
    reference's put_worker / deserialize_worker, remote_backend.py:61-69,234-246); each direction owns
    its buffers and is guarded by its own lock.
    """

    def __init__(self, model_name: str, coder: Optional[str] = None, cachegen_config=None):
        """coder: "rans_compact" (container version 3, the default: rANS payload + symbol counts instead of CDF rows;
        chunks of more than 256 tokens fall back to version 2), "rans" (version 2) or "ac" (version 1, the
        torchac-lineage arithmetic coder); the environment variable LMCACHE_B200_CODER overrides the default.
        Decoding accepts all three.

        cachegen_config: the nine CacheGenConfig fields (LMCacheEngineConfig.cachegen_config), used instead of the bin
        table for any model name.  Only version 3 records the bins a container was written with, so such a codec writes
        and reads version 3 only: another coder is a ValueError here, chunks of more than 256 tokens one in coder_for,
        and accepts() refuses versions 1 and 2 (their values would be dequantised with a step they were not written
        with)."""
        import os
        from lmcache_b200.storage_backend.serde.cachegen_basics import CacheGenConfig
        N.require_cuda()
        name = (coder or os.environ.get("LMCACHE_B200_CODER", "rans_compact")).lower()
        if name not in N.CODERS:
            raise ValueError(f"unknown coder {name!r} (expected one of {sorted(N.CODERS)})")
        self.coder = N.CODERS[name]
        self.v3_only = cachegen_config is not None
        if self.v3_only and self.coder != N.CODER_RANS_COMPACT:
            raise ValueError(f"coder {name!r} writes containers that do not record their bins: with cachegen_config "
                             f"only 'rans_compact' (container version 3) is possible")
        self.config = CacheGenConfig.for_engine(model_name, cachegen_config)
        kb, vb = self.config.key_bins_list(), self.config.value_bins_list()
        self.nlayers = len(kb)
        self._kb = N.float_array(kb)
        self._vb = N.float_array(vb)
        self._nb = (N.nb_map(kb, vb, len(kb)))          # keys then values, all layers of the model
        self._init_io()
        self._last_bits_per_symbol = 0.0        # payload bits per symbol of the most recent encode whose sizes were read

    # ------------------------------------------------------------------ helpers
    parse_header = staticmethod(parse_header)    # the CacheGen container check (versions 1 to 4)
    plane_offsets = staticmethod(plane_offsets)  # where a version-3 / version-4 container's planes lie
    layerwise_max_tokens = N.GROUP_TOKENS         # a layer-major retrieve needs one group per container

    @staticmethod
    def plane_offsets_device(containers: int, stride: int, n: int, out: int, stream) -> None:
        """plane_offsets for n containers `stride` apart in device memory (b200kv_plane_offsets_device, pipeline.land):
        int64[N.MAX_PLANES + 1] rows into `out`.  Through N.pylib(): the call keeps the GIL."""
        N.check(N.pylib().b200kv_plane_offsets_device(ctypes.c_void_p(containers), stride, n, ctypes.c_void_p(out),
                                                      stream), "b200kv_plane_offsets_device")

    @staticmethod
    def raw_rows(records, latent: bool = False) -> None:
        """layer_copy_ranges' `raw` for these containers: None, a plane of a CacheGen container is its streams"""
        return None

    def plan_prefix(self, L: int, H: int, D: int, chunk_tokens: int, latent: bool = False) -> int:
        """bytes [0, n) of a full chunk's container that decode_plan reads: its fixed sections"""
        return int(self.layout(L, H, D, chunk_tokens, latent).off_payload)

    def coder_for(self, chunk_tokens: int, latent: bool = False) -> int:
        """The container this codec writes for chunks of `chunk_tokens`: the compact one holds <= 256 tokens.  A latent
        KV is written as version 4 (N.CODER_LATENT), which exists for the compact coder and <= 256 tokens only."""
        if latent:
            if self.coder != N.CODER_RANS_COMPACT or chunk_tokens > N.GROUP_TOKENS:
                raise ValueError(f"a latent KV is coded into version-4 containers: coder 'rans_compact' and chunks of "
                                 f"at most {N.GROUP_TOKENS} tokens only")
            return N.CODER_LATENT
        if self.coder == N.CODER_RANS_COMPACT and chunk_tokens > N.GROUP_TOKENS:
            if self.v3_only:
                raise ValueError(f"chunks of {chunk_tokens} tokens: with cachegen_config the containers are version 3, "
                                 f"which holds at most {N.GROUP_TOKENS} tokens")
            return N.CODER_RANS
        return self.coder

    def layout(self, L: int, H: int, D: int, chunk_tokens: int, latent: bool = False) -> "N.Layout":
        return N.container_layout(L, H, D, chunk_tokens, self.coder_for(chunk_tokens, latent))

    def accepts(self, hd: "N.Header", latent: bool = False) -> bool:
        """Can this codec decode the container into a destination of one plane per layer (`latent`) or of (K, V) pairs?
        The container's plane layout must be the destination's: version 4 for a latent destination, versions 1 to 3
        otherwise.  A compact container must have been written with this model's bins (a latent plane with the key
        bins); a codec made from a cachegen_config reads compact containers only (the others do not say which bins they
        used)."""
        if (hd.version == 4) != latent:
            return False
        n = self.nlayers
        if hd.version == 4:
            return hd.L <= n and hd.nb == self._nb[:hd.L]
        if hd.version != 3:
            return not self.v3_only
        return hd.L <= n and hd.nb == self._nb[:hd.L] + self._nb[n:n + hd.L]

    def max_container_bytes(self, L: int, H: int, D: int, chunk_tokens: int, latent: bool = False) -> int:
        """Upper bound of a container of ANY version this codec can decode (what a receive slab must reserve when the
        writer may have been configured differently): version 2's sections are the largest.  A latent KV (one plane per
        layer) is read from version 4 only: that container's own bound."""
        if latent:
            return self.out_stride(L, H, D, chunk_tokens, latent=True)
        lo = N.container_layout(L, H, D, chunk_tokens)
        if chunk_tokens <= N.GROUP_TOKENS:
            return (lo.fixed_bytes + 2 * L * H * D * (chunk_tokens + 4) + 16 + 15) & ~15
        return lo.max_total_bytes

    def out_stride(self, L: int, H: int, D: int, chunk_tokens: int, latent: bool = False) -> int:
        """Bytes reserved per container.  Chunks of <= 256 tokens are coded with their own empirical CDF,
        so a stream costs <= 8 bits/symbol (+ flush); larger chunks may reach 16 bits/symbol."""
        lo = self.layout(L, H, D, chunk_tokens, latent)
        if chunk_tokens <= N.GROUP_TOKENS:
            hdr = N.HDR_MAX if self.coder_for(chunk_tokens, latent) & 0xff == N.CODER_RANS_COMPACT else 0
            return (lo.fixed_bytes + (1 if latent else 2) * L * H * D * (chunk_tokens + 4 + hdr) + 16 + 15) & ~15
        return lo.max_total_bytes

    def _check_source(self, view: KvView) -> None:
        if view.dtype_code in N.ONE_BYTE_DTYPES:
            raise TypeError(_CACHEGEN_FP8.format(view.dtype))
        if view.L > self.nlayers:
            raise ValueError(f"KV has {view.L} layers but the bin table of this model has {self.nlayers}")

    # ------------------------------------------------------------------ layer-wise encode (pipeline.LayerwiseEncode)
    # b200kv_encode_layers_plan / _layers / _finish, version-3 (version-4) containers; a segment row per (chunk, plane)
    # is (arena offset, bytes) of the plane's streams
    seg_row = 2

    def segment_layout(self, L: int, H: int, D: int, ntokens: int, latent: bool = False,
                       dtype: int = N.DT_BF16) -> SegmentLayout:
        """dtype: the KV's N.DT_* (16-bit: the only kind this codec encodes)"""
        lo = N.container_layout(L, H, D, ntokens, N.CODER_LATENT if latent else N.CODER_RANS_COMPACT)
        return SegmentLayout(int(lo.off_payload), int(lo.off_payload))

    def layerwise_chunk_bound(self, L: int, H: int, D: int, chunk_tokens: int, latent: bool = False) -> int:
        """arena bytes a chunk can take: its worst-case payload and the alignment of one segment per layer"""
        lo = N.container_layout(L, H, D, chunk_tokens, N.CODER_LATENT if latent else N.CODER_RANS_COMPACT)
        return int(lo.max_total_bytes - lo.off_payload) + 16 * L

    def layerwise_workspace_bytes(self, L: int, H: int, D: int, chunk_tokens: int, n_chunks: int,
                                  latent: bool = False) -> int:
        return N.check(N.lib().b200kv_encode_layers_workspace_bytes(L, H, D, chunk_tokens, n_chunks, 1),
                       "encode_layers_workspace")

    def encode_layers_plan(self, view: KvView, tok_begin: int, n: int, chunk_tokens: int, last: int, slot,
                           stream: torch.cuda.Stream) -> "N.EncodePlan":
        """b200kv_encode_layers_plan into a pipeline.SegmentSlot, one layer per call; returns the plan"""
        self._check_source(view)
        plan = N.EncodePlan()
        N.check(N.lib().b200kv_encode_layers_plan(ctypes.byref(view.desc), tok_begin, n, chunk_tokens, last, self._kb,
                                                  self._vb, N.CODER_RANS_COMPACT, slot.arena.data_ptr(), slot.arena_bytes,
                                                  slot.fixed.data_ptr(), slot.fixed_stride, slot.seg.dev_ptr,
                                                  slot.sizes.dev_ptr, 1, slot.ws.data_ptr(), slot.ws.numel(),
                                                  ctypes.byref(plan), stream.cuda_stream), "encode_layers_plan")
        return plan

    @staticmethod
    def encode_layers(plan: "N.EncodePlan", layer_begin: int, layer_end: int, stream: torch.cuda.Stream) -> None:
        """b200kv_encode_layers: enqueue the encode of layers [layer_begin, layer_end)"""
        N.check(N.lib().b200kv_encode_layers(ctypes.byref(plan), int(layer_begin), int(layer_end), stream.cuda_stream),
                "encode_layers")

    @staticmethod
    def encode_layers_finish(plan: "N.EncodePlan", stream: torch.cuda.Stream) -> None:
        """b200kv_encode_layers_finish: enqueue the headers and container sizes"""
        N.check(N.lib().b200kv_encode_layers_finish(ctypes.byref(plan), stream.cuda_stream), "encode_layers_finish")

    # ------------------------------------------------------------------ encode / decode hooks of _ContainerIO
    def _encode_ws_bytes(self, view: KvView, chunk_size: int, n_chunks: int, coder: int) -> int:
        return N.lib().b200kv_encode_workspace_bytes(view.L, view.H, view.D, chunk_size, n_chunks, coder)

    def _encode_launch(self, view: KvView, tok_begin: int, n_tokens: int, chunk_size: int, n_chunks: int, last: int,
                       coder: int, out: torch.Tensor, stride: int, sizes: PinnedBuffer, stream) -> dict:
        # KV statistics of one model are stable from call to call: the previous call's measured entropy picks the
        # compaction kernel's shared-memory stage size for this one (byte-identical output either way)
        # (the threshold is in coder bits per symbol; a version-3 payload also holds ~0.4 bits of stream headers)
        b = self._last_bits_per_symbol - (0.4 if coder & 0xff == N.CODER_RANS_COMPACT else 0.0)
        flags = (coder & 0xff) | (N.ENCODE_HINT_MID_ENTROPY if b > 1.2 else 0)   # the descriptor says latent
        N.check(N.lib().b200kv_encode_chunks(ctypes.byref(view.desc), tok_begin, n_chunks, chunk_size, last, self._kb,
                                             self._vb, flags, out.data_ptr(), stride, sizes.dev_ptr,
                                             self._enc_ws.data_ptr(), self._enc_ws.numel(), stream.cuda_stream),
                "encode_chunks")
        # the ticket measures this call's bits per symbol for the next one
        fixed = self.layout(view.L, view.H, view.D, chunk_size, view.latent).fixed_bytes
        return dict(codec=self, stats=(fixed, float(view.planes) * view.H * view.D * n_tokens))

    def _decode_ws_bytes(self, dst: KvView, src_H: int, tmax: int, n: int) -> int:
        # < 0: a shape the plan call refuses, with its reason
        return max(N.lib().b200kv_decode_workspace_bytes(dst.L, int(src_H), dst.D, tmax, n), 0)

    def _plan_native(self, args: tuple, coder: int, dst: KvView, status, ws: torch.Tensor, stream,
                     window: tuple) -> "N.DecodePlan":
        if dst.dtype_code in N.ONE_BYTE_DTYPES:
            raise TypeError(_CACHEGEN_FP8.format(dst.dtype))
        plan = N.DecodePlan()
        args += (int(coder), ctypes.byref(dst.desc), self._kb, self._vb, status, ws.data_ptr(), ws.numel(),
                 ctypes.byref(plan), stream.cuda_stream)
        if window:
            N.check(N.lib().b200kv_decode_plan_heads(*args, *window), "decode_plan_heads")
        else:
            N.check(N.lib().b200kv_decode_plan(*args), "decode_plan")
        return plan

    @staticmethod
    def decode_layers(plan: "N.DecodePlan", layer_begin: int, layer_end: int, stream: torch.cuda.Stream) -> None:
        """Second half of decode_raw (b200kv_decode_layers): enqueue the decode of layers [layer_begin, layer_end)."""
        N.check(N.lib().b200kv_decode_layers(ctypes.byref(plan), int(layer_begin), int(layer_end), stream.cuda_stream),
                "decode_layers")

    def _check_container(self, hd: "N.Header", dst: KvView) -> None:
        if dst.dtype_code in N.ONE_BYTE_DTYPES:
            raise TypeError(_CACHEGEN_FP8.format(dst.dtype))
        if not self.accepts(hd, dst.latent):
            raise ValueError("compact container written with another model's bins" if hd.version >= 3 else
                             f"a codec made from a cachegen_config reads version 3 only, not version {hd.version}")

    def decode_device_batch(self, batch: EncodedBatch, ntokens: Sequence[int], dst: KvView, dst_tok: Sequence[int],
                            stream: Optional[torch.cuda.Stream] = None) -> None:
        """Decode an EncodedBatch straight from its device staging buffer (no host hop, no header reads)."""
        self.decode_raw(batch.buf.data_ptr(), batch.buf.numel(), [j * batch.stride for j in range(len(batch.sizes))],
                        batch.sizes, ntokens, dst, dst_tok, batch.max_dtype, batch.coder, stream)


def dtype_of_code(code: int) -> torch.dtype:
    """torch dtype of an N.DT_* code"""
    return _CODE_DTYPE[int(code)]


def parse_lossless_header(buf, total: Optional[int] = None) -> N.Header:
    """Validate and return the 64-byte header of a lossless B2KV container (versions 5 and 6; ValueError for anything
    else, CacheGen containers included).  `buf` is the whole container, or a prefix of at least the header when `total`,
    the size of the whole container, is given."""
    hd = _parse_preamble(buf, total, (5, 6), "not a lossless B2KV container (version {})")[1]
    check_lossless_header(hd)
    return hd


def check_lossless_header(hd: "N.Header") -> None:
    """Structural checks of a lossless header: a possible shape (L <= 128 layers, 1..4096 tokens), a known element dtype
    (16-bit or one-byte), one group, and total_bytes = fixed sections + payload_bytes with a payload between 4 bytes per
    stream and the worst case."""
    if not (0 < hd.L <= N.MAX_PLANES // 2 and hd.H > 0 and hd.D > 0 and hd.H * hd.D < (1 << 24) and
            0 < hd.ntokens <= N.LOSSLESS_MAX_TOKENS):
        raise ValueError("B2KV header carries an impossible shape")
    if hd.max_dtype not in _CODE_DTYPE:
        raise ValueError("B2KV header carries an unknown element dtype")
    if hd.ngroups != 1 or any(hd.reserved):
        raise ValueError("B2KV lossless header: ngroups must be 1 and reserved 0")
    lo = N.lossless_layout(hd.L, hd.H, hd.D, hd.ntokens, hd.version == 6, hd.max_dtype)
    if hd.total_bytes != lo.off_payload + hd.payload_bytes:
        raise ValueError("B2KV header: total_bytes != fixed sections + payload_bytes (truncated or corrupt)")
    nstreams = N.planes_of(hd.version, hd.L) * hd.H * hd.D
    if hd.payload_bytes < 4 * nstreams or hd.total_bytes > lo.max_total_bytes:
        raise ValueError("B2KV header: payload_bytes impossible for this shape")


def lossless_plane_offsets(buf) -> Optional[np.ndarray]:
    """Where the streams of each plane lie in a lossless container (`buf`: at least its header, frequency rows and
    lengths), from its lengths section: int64[P + 1] (P = 2L, or L for version 6), the streams of plane p are bytes
    [o[p], o[p + 1]) of the container, o[0] is off_payload and o[P] == total_bytes.  None when the lengths do not add up
    to the header's total (a damaged container: it is only ever uploaded whole).  Plane p's raw rows (none for one-byte
    elements) come from the layout: LosslessCodec.raw_rows."""
    return _plane_offsets(buf, (5, 6), N.lib().b200kv_lossless_plane_offsets, "lossless_plane_offsets")


class LosslessCodec(_ContainerIO):
    """Lossless encode / decode on the current CUDA device (container versions 5 and 6, include/b200kv.h): every
    element's high byte after a one-bit rotation (bf16: the exponent) is rANS-coded per (plane, channel) against one
    frequency row per plane, the low byte is kept verbatim, and the decode gives back the same bits.  A one-byte element
    (FP8, uint8) is coded whole: its container has no raw section.  Sizes this codec reserves (out_stride,
    max_container_bytes, layerwise_chunk_bound) are those of 16-bit elements, which bound the one-byte ones; the exact
    layouts (layout, segment_layout, raw_rows) follow the element dtype.  It presents what the
    remote tier's pipelines take from CacheGenCodec; it needs no model table, and decodes into the stored dtype only.

    Thread model as CacheGenCodec: one encoder and one decoder may run concurrently from different threads."""

    def __init__(self):
        N.require_cuda()
        self._init_io()

    parse_header = staticmethod(parse_lossless_header)
    plane_offsets = staticmethod(lossless_plane_offsets)
    layerwise_max_tokens = N.LOSSLESS_MAX_TOKENS   # a lossless container is always one group

    @staticmethod
    def plane_offsets_device(containers: int, stride: int, n: int, out: int, stream) -> None:
        """CacheGenCodec.plane_offsets_device for lossless containers (b200kv_lossless_plane_offsets_device)"""
        N.check(N.pylib().b200kv_lossless_plane_offsets_device(ctypes.c_void_p(containers), stride, n,
                                                               ctypes.c_void_p(out), stream),
                "b200kv_lossless_plane_offsets_device")

    @staticmethod
    def raw_rows(records, latent: bool = False) -> List[Tuple[int, int]]:
        """layer_copy_ranges' `raw` for these containers (records with L, H, D, ntokens and max_dtype): per container
        (off_raw, bytes per plane), plane p's raw rows are bytes [off_raw + p * t * C, off_raw + (p + 1) * t * C); 0
        bytes per plane for one-byte elements"""
        return [(int(N.lossless_layout(r.L, r.H, r.D, r.ntokens, latent, r.max_dtype).off_raw),
                 0 if r.max_dtype in N.ONE_BYTE_DTYPES else int(r.ntokens) * r.H * r.D) for r in records]

    def plan_prefix(self, L: int, H: int, D: int, chunk_tokens: int, latent: bool = False) -> int:
        """bytes [0, n) of a full chunk's container that decode_plan reads: [0, off_raw)"""
        return int(self.layout(L, H, D, chunk_tokens, latent).off_raw)

    @staticmethod
    def coder_for(chunk_tokens: int, latent: bool = False) -> int:
        """The coder value HostContainer / EncodedBatch carry for this codec's containers (version 6 for a latent KV)."""
        if not 0 < chunk_tokens <= N.LOSSLESS_MAX_TOKENS:
            raise ValueError(f"a lossless container holds 1 to {N.LOSSLESS_MAX_TOKENS} tokens, not {chunk_tokens}")
        return N.CODER_LOSSLESS_LATENT if latent else N.CODER_LOSSLESS

    def accepts(self, hd: "N.Header", latent: bool = False) -> bool:
        """Does a container that passed parse_lossless_header fit a destination of one plane per layer (`latent`: version
        6) or of (K, V) pairs (version 5)?"""
        return hd.version in (5, 6) and (hd.version == 6) == latent

    def layout(self, L: int, H: int, D: int, chunk_tokens: int, latent: bool = False,
               dtype: int = N.DT_BF16) -> "N.LosslessLayout":
        """the container of elements of `dtype` (N.DT_*); the 16-bit one by default, which bounds the one-byte one"""
        self.coder_for(chunk_tokens, latent)
        return N.lossless_layout(L, H, D, chunk_tokens, latent, dtype)

    def out_stride(self, L: int, H: int, D: int, chunk_tokens: int, latent: bool = False) -> int:
        """Bytes reserved per container: the worst case, every stream at 12 bits per symbol."""
        return int(self.layout(L, H, D, chunk_tokens, latent).max_total_bytes)

    def max_container_bytes(self, L: int, H: int, D: int, chunk_tokens: int, latent: bool = False) -> int:
        """Upper bound of a container this codec can decode (there is one lossless layout per shape)."""
        return self.out_stride(L, H, D, chunk_tokens, latent)

    # ------------------------------------------------------------------ layer-wise encode (pipeline.LayerwiseEncode)
    # b200kv_lossless_encode_layers_plan / _layers / _finish; a segment row per (chunk, plane) is (arena offset of the
    # plane's raw rows, arena offset of its streams, stream bytes)
    seg_row = 3

    def segment_layout(self, L: int, H: int, D: int, ntokens: int, latent: bool = False,
                       dtype: int = N.DT_BF16) -> SegmentLayout:
        lo = self.layout(L, H, D, ntokens, latent, dtype)
        return SegmentLayout(int(lo.off_raw), int(lo.off_payload), 0 if dtype in N.ONE_BYTE_DTYPES else int(ntokens) * H * D)

    def layerwise_chunk_bound(self, L: int, H: int, D: int, chunk_tokens: int, latent: bool = False) -> int:
        """arena bytes a chunk can take: everything of its worst case after the fixed image, and per layer the alignment
        of one segment and of the streams inside it"""
        lo = self.layout(L, H, D, chunk_tokens, latent)
        return int(lo.max_total_bytes - lo.off_raw) + 32 * L

    def layerwise_workspace_bytes(self, L: int, H: int, D: int, chunk_tokens: int, n_chunks: int,
                                  latent: bool = False) -> int:
        return N.check(N.lib().b200kv_lossless_encode_layers_workspace_bytes(L, H, D, chunk_tokens, n_chunks,
                                                                             int(latent), 1),
                       "lossless_encode_layers_workspace")

    def encode_layers_plan(self, view: KvView, tok_begin: int, n: int, chunk_tokens: int, last: int, slot,
                           stream: torch.cuda.Stream) -> "N.LosslessEncodePlan":
        """b200kv_lossless_encode_layers_plan into a pipeline.SegmentSlot, one layer per call; returns the plan"""
        plan = N.LosslessEncodePlan()
        N.check(N.lib().b200kv_lossless_encode_layers_plan(ctypes.byref(view.desc), tok_begin, n, chunk_tokens, last,
                                                           slot.arena.data_ptr(), slot.arena_bytes, slot.fixed.data_ptr(),
                                                           slot.fixed_stride, slot.seg.dev_ptr, slot.sizes.dev_ptr, 1,
                                                           slot.ws.data_ptr(), slot.ws.numel(), ctypes.byref(plan),
                                                           stream.cuda_stream), "lossless_encode_layers_plan")
        return plan

    @staticmethod
    def encode_layers(plan: "N.LosslessEncodePlan", layer_begin: int, layer_end: int, stream: torch.cuda.Stream) -> None:
        """b200kv_lossless_encode_layers: enqueue the encode of layers [layer_begin, layer_end)"""
        N.check(N.lib().b200kv_lossless_encode_layers(ctypes.byref(plan), int(layer_begin), int(layer_end),
                                                      stream.cuda_stream), "lossless_encode_layers")

    @staticmethod
    def encode_layers_finish(plan: "N.LosslessEncodePlan", stream: torch.cuda.Stream) -> None:
        """b200kv_lossless_encode_layers_finish: enqueue the headers and container sizes"""
        N.check(N.lib().b200kv_lossless_encode_layers_finish(ctypes.byref(plan), stream.cuda_stream),
                "lossless_encode_layers_finish")

    # ------------------------------------------------------------------ encode / decode hooks of _ContainerIO
    def _encode_ws_bytes(self, view: KvView, chunk_size: int, n_chunks: int, coder: int) -> int:
        return N.check(N.lib().b200kv_lossless_workspace_bytes(view.L, view.H, view.D, chunk_size, n_chunks,
                                                               int(view.latent), 0), "lossless_workspace_bytes")

    def _encode_launch(self, view: KvView, tok_begin: int, n_tokens: int, chunk_size: int, n_chunks: int, last: int,
                       coder: int, out: torch.Tensor, stride: int, sizes: PinnedBuffer, stream) -> dict:
        # the KV is read in stream order twice: histogram, then coding
        N.check(N.lib().b200kv_lossless_encode(ctypes.byref(view.desc), tok_begin, n_chunks, chunk_size, last,
                                               out.data_ptr(), stride, sizes.dev_ptr, self._enc_ws.data_ptr(),
                                               self._enc_ws.numel(), stream.cuda_stream), "lossless_encode")
        return {}

    def _decode_ws_bytes(self, dst: KvView, src_H: int, tmax: int, n: int) -> int:
        # < 0: a shape the plan call refuses, with its reason
        return max(N.lib().b200kv_lossless_workspace_bytes(dst.L, int(src_H), dst.D, tmax, n, int(dst.latent), 1), 16)

    def _plan_native(self, args: tuple, coder: int, dst: KvView, status, ws: torch.Tensor, stream,
                     window: tuple) -> "N.LosslessDecodePlan":
        # the library takes no coder: the destination says which version it decodes (6 for a latent one)
        if coder not in (N.CODER_LOSSLESS, N.CODER_LOSSLESS_LATENT) or bool(coder & N.KV_LATENT) != dst.latent:
            raise ValueError(f"coder {coder} does not name the lossless container of this destination")
        plan = N.LosslessDecodePlan()
        args += (ctypes.byref(dst.desc), status, ws.data_ptr(), ws.numel(), ctypes.byref(plan), stream.cuda_stream)
        if window:
            N.check(N.lib().b200kv_lossless_decode_plan_heads(*args, *window), "lossless_decode_plan_heads")
        else:
            N.check(N.lib().b200kv_lossless_decode_plan(*args), "lossless_decode_plan")
        return plan

    @staticmethod
    def decode_layers(plan: "N.LosslessDecodePlan", layer_begin: int, layer_end: int, stream: torch.cuda.Stream) -> None:
        """Second half of the decode (b200kv_lossless_decode_layers): enqueue the decode of layers [layer_begin,
        layer_end)."""
        N.check(N.lib().b200kv_lossless_decode_layers(ctypes.byref(plan), int(layer_begin), int(layer_end),
                                                      stream.cuda_stream), "lossless_decode_layers")

    def _check_container(self, hd: "N.Header", dst: KvView) -> None:
        if hd.max_dtype != dst.dtype_code:
            raise ValueError(f"container holds {dtype_of_code(hd.max_dtype)}, destination is {dst.dtype}: a lossless "
                             f"container is decoded into its own dtype")


def engine_codec(config, model_name: str) -> CacheGenCodec:
    """The codec of an engine's CacheGen tier or serde: the bins of config.cachegen_config when it is set (then the
    containers are version 3, so chunk_size must be <= 256: a ValueError here, when the tier or serde is made, not at
    the first store), the model's row of the bin table otherwise (ValueError for a name outside it)."""
    cg = config.cachegen_config
    if cg is not None and config.chunk_size > N.GROUP_TOKENS:
        raise ValueError(f"chunk_size {config.chunk_size}: with cachegen_config the containers are version 3, which "
                         f"holds at most {N.GROUP_TOKENS} tokens")
    return CacheGenCodec(model_name, cachegen_config=cg)
