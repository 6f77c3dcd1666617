"""CacheGen configuration and wire-container views.

Mirrors lmcache/storage_backend/serde/cachegen_basics.py:
  * CACHEGEN_GPU_MAX_TOKENS_PER_CHUNK (:13), CacheGenConfig.from_model_name (:16-78): identical bin table;
    CacheGenConfig.for_engine also takes an operator-supplied layout (LMCacheEngineConfig.cachegen_config).
  * CacheGenGPUBytestream / CacheGenGPUEncoderOutput (:109-142): same field names, but `to_bytes` /
    `from_bytes` speak the flat "B2KV" container (include/b200kv.h) that the encode kernel writes on the
    device, instead of pickling CUDA tensors.  `from_bytes` gives the same object a reference consumer
    would unpickle (test_serde.py:60-62 reads .num_heads / .head_size).
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import torch

from lmcache_b200 import _native as N

CACHEGEN_GPU_MAX_TOKENS_PER_CHUNK = N.GROUP_TOKENS

_FAMILY_LAYERS = {
    "mistralai/Mistral-7B-Instruct-v0.2": 32,
    "lmsys/longchat-7b-16k": 32,
    "Qwen/Qwen-7B": 32,
    "meta-llama/Llama-3.1-8B-Instruct": 32,
    "THUDM/glm-4-9b-chat": 40,
}


@dataclass
class CacheGenConfig:
    key_first_layers: int
    key_second_layers: int
    key_third_layers: int
    key_first_bins: int
    key_second_bins: int
    key_third_bins: int
    value_first_layers: int
    value_first_bins: int
    value_second_bins: int

    def __getitem__(self, key: str) -> int:
        return getattr(self, key)

    @staticmethod
    def from_model_name(model_name: str) -> "CacheGenConfig":
        if model_name not in _FAMILY_LAYERS:
            raise ValueError(f"Model {model_name} is not supported")
        return CacheGenConfig(
            key_first_layers=10, key_second_layers=20, key_third_layers=_FAMILY_LAYERS[model_name],
            key_first_bins=32, key_second_bins=16, key_third_bins=16,
            value_first_layers=2, value_first_bins=32, value_second_bins=16)

    @staticmethod
    def for_engine(model_name: str, cachegen_config=None) -> "CacheGenConfig":
        """The layout an engine uses: `cachegen_config` (LMCacheEngineConfig.cachegen_config: the nine fields, checked
        by config.check_cachegen_config) for any model name when it is given, the table of from_model_name otherwise."""
        if cachegen_config is None:
            return CacheGenConfig.from_model_name(model_name)
        from lmcache_b200.config import check_cachegen_config
        return CacheGenConfig(**check_cachegen_config(cachegen_config))

    def key_bins_list(self) -> List[float]:
        """make_key_bins (cachegen_encoder.py:339-344): per-layer fp32 bin counts."""
        bins = [float(self.key_third_bins)] * self.key_third_layers
        for i in range(min(self.key_second_layers, self.key_third_layers)):
            bins[i] = float(self.key_second_bins)
        for i in range(min(self.key_first_layers, self.key_third_layers)):
            bins[i] = float(self.key_first_bins)
        return bins

    def value_bins_list(self) -> List[float]:
        """make_value_bins (cachegen_encoder.py:346-350)."""
        bins = [float(self.value_second_bins)] * self.key_third_layers
        for i in range(min(self.value_first_layers, self.key_third_layers)):
            bins[i] = float(self.value_first_bins)
        return bins


@dataclass
class CacheGenGPUBytestream:
    bytestream: torch.Tensor          # uint8 [N]
    bytestream_lengths: torch.Tensor  # int32 [2L, C]
    ntokens: int

    def __getitem__(self, key: str):
        return getattr(self, key)


_HALF = {N.DT_BF16: torch.bfloat16, N.DT_FP16: torch.float16}


def cdf_from_counts(counts: np.ndarray, ntokens: int) -> np.ndarray:
    """The CDF tensor the reference stores, as a function of the symbol histogram (what a version-3 container keeps):
    counts [..., 33] (entry 32 is 0) -> int16 [..., 33].  Restates the in-tree spec of torchac_cuda.calculate_cdf
    (cachegen_encoder.py:95-126,185-196) the way the kernels evaluate it (csrc/ac_core.cuh, CdfAccum):
    p_i = fl32(n_i / t); cdf_f[i] = fl32(sum_{k<i} p_k accumulated in double); cdf[i] = int16(rint(cdf_f[i] * 65504) + i).
    Host-side helper of the from_bytes shim -- the decoder evaluates this on the device."""
    counts = np.asarray(counts)
    p = (counts.astype(np.float32) / np.float32(ntokens)).astype(np.float32)
    cum = np.zeros(counts.shape[:-1], np.float64)
    out = np.empty(counts.shape, np.int16)
    for i in range(counts.shape[-1]):
        prev = cum.astype(np.float32)
        r = np.rint(prev * np.float32(65504.0)).astype(np.int64) + i
        out[..., i] = (r & 0xFFFF).astype(np.uint16).view(np.int16)
        cum = cum + p[..., i].astype(np.float64)
    return out


def _v3_parse_streams(payload: np.ndarray, half: np.ndarray, nb: List[int], C: int, t: int):
    """Version-3 payload -> (counts int32 [S, 33], rANS lengths int32 [S], rANS bytes u8): every stream starts with its
    histogram header (include/b200kv.h).  Vectorised over the S = 2L * C streams; raises ValueError on a malformed one."""
    S = half.size
    total = half.astype(np.int64) * 2
    start = np.cumsum(total) - total
    if S == 0 or int(start[-1] + total[-1]) != payload.size:
        raise ValueError("B2KV v3: stream lengths do not add up to the payload")
    nbs = np.repeat(np.asarray(nb, np.int64), C)
    mb = (nbs + 7) // 8
    if np.any(total < mb + 4):
        raise ValueError("B2KV v3: stream shorter than its header")
    pad = np.concatenate([payload, np.zeros(8, np.uint8)])
    mask = np.zeros(S, np.int64)
    for k in range(4):
        mask |= np.where(k < mb, pad[start + k].astype(np.int64), 0) << (8 * k)
    mask &= (np.int64(1) << nbs) - 1
    bits = ((mask[:, None] >> np.arange(32)[None, :]) & 1).astype(bool)
    nz = bits.sum(axis=1)
    if np.any(nz == 0):
        raise ValueError("B2KV v3: empty symbol mask")
    hlen = mb + nz - 1
    hlen += hlen & 1
    if np.any(hlen + 4 > total):
        raise ValueError("B2KV v3: stream shorter than its header")
    rank = np.cumsum(bits, axis=1) - 1
    last = bits & (rank == (nz - 1)[:, None])
    stored = bits & ~last
    counts = np.zeros((S, N.LP), np.int32)
    view = counts[:, :32]
    idx = (start + mb)[:, None] + rank
    view[stored] = payload[idx[stored]]
    if np.any(view[stored] == 0):
        raise ValueError("B2KV v3: zero count for a symbol the mask lists")
    rest = t - view.sum(axis=1)
    if np.any(rest <= 0):
        raise ValueError("B2KV v3: counts exceed the token count")
    view[last] = rest
    rlen = (total - hlen).astype(np.int32)
    keep = np.ones(payload.size, bool)
    hpos = np.repeat(start, hlen) + (np.arange(int(hlen.sum())) - np.repeat(np.cumsum(hlen) - hlen, hlen))
    keep[hpos] = False
    return counts, rlen, payload[keep]


def _v3_build_streams(counts: np.ndarray, nb: List[int], C: int, rlen: np.ndarray, rans: np.ndarray):
    """Inverse of _v3_parse_streams: (payload u8, half-lengths u8 [S])."""
    S = counts.shape[0]
    nbs = np.repeat(np.asarray(nb, np.int64), C)
    mb = (nbs + 7) // 8
    view = counts[:, :32]
    bits = view > 0
    nz = bits.sum(axis=1)
    hlen = mb + np.maximum(nz, 1) - 1
    hlen += hlen & 1
    rlen = rlen.astype(np.int64)
    total = hlen + rlen
    if np.any(total % 2) or np.any(total // 2 > 255):
        raise ValueError("stream too long for a version-3 container")
    start = np.cumsum(total) - total
    out = np.zeros(int(total.sum()), np.uint8)
    mask = (bits.astype(np.int64) << np.arange(32)[None, :]).sum(axis=1)
    for k in range(4):
        sel = k < mb
        out[(start + k)[sel]] = ((mask[sel] >> (8 * k)) & 0xFF).astype(np.uint8)
    rank = np.cumsum(bits, axis=1) - 1
    stored = bits & ~(bits & (rank == (nz - 1)[:, None]))
    idx = (start + mb)[:, None] + rank
    out[idx[stored]] = view[stored].astype(np.uint8)
    rstart = np.cumsum(rlen) - rlen
    dst = np.repeat(start + hlen - rstart, rlen) + np.arange(int(rlen.sum()))
    out[dst] = rans
    return out, (total // 2).astype(np.uint8)


@dataclass
class CacheGenGPUEncoderOutput:
    data_chunks: List[CacheGenGPUBytestream]
    cdf: torch.Tensor                 # int16 [2L, C, 33]
    max_tensors_key: torch.Tensor     # half [L, t, 1]
    max_tensors_value: torch.Tensor   # half [L, t, 1]
    num_heads: int
    head_size: int
    coder: int = N.CODER_RANS         # entropy coder of the bytestreams = container version - 1 (not in the reference)
    counts: Optional[torch.Tensor] = None   # version 3 only: int32 [2L, C, 33] symbol histogram the CDF was rebuilt from
    nb: Optional[List[int]] = None          # version 3 only: counts stored per stream of each plane (the container's nb map)

    def __getitem__(self, key: str):
        return getattr(self, key)

    @staticmethod
    def from_bytes(bs) -> "CacheGenGPUEncoderOutput":
        """Parse a B2KV container into host tensors (zero-copy views where possible)."""
        from lmcache_b200.codec import parse_header
        from lmcache_b200.codec import container_layout_of
        hd = parse_header(bs)
        if hd.version == 4:
            raise ValueError("a version-4 container (one latent plane per layer) has no (key, value) object form")
        L, H, D, t, G = hd.L, hd.H, hd.D, hd.ntokens, hd.ngroups
        C = H * D
        lo = container_layout_of(hd)
        raw = np.frombuffer(bs, dtype=np.uint8, count=int(hd.total_bytes))

        def section(off, count, dtype):
            return torch.from_numpy(raw[off:off + count * np.dtype(dtype).itemsize].view(dtype).copy())

        counts_t = None
        payload = raw[lo.off_payload: lo.off_payload + int(hd.payload_bytes)]
        if hd.version == 3:
            # compact container: every stream carries its histogram; rebuild the reference's CDF tensor from it and
            # hand out the bare rANS streams with their lengths, as a version-2 container would
            half = raw[lo.off_lengths: lo.off_lengths + 2 * L * C]
            counts, rlen, payload = _v3_parse_streams(payload, half, hd.nb, C, t)
            counts = counts.reshape(2 * L, C, N.LP)
            cdf = torch.from_numpy(cdf_from_counts(counts, t))
            counts_t = torch.from_numpy(counts)
            lengths = torch.from_numpy(rlen).reshape(G, 2 * L, C)
        else:
            cdf = section(lo.off_cdf, 2 * L * C * N.LP, np.int16).reshape(2 * L, C, N.LP)
            lengths = section(lo.off_lengths, G * 2 * L * C, np.int32).reshape(G, 2 * L, C)
        maxes = section(lo.off_maxes, 2 * L * t, np.int16).view(_HALF[hd.max_dtype]).reshape(2, L, t, 1)
        chunks, pos = [], 0
        for g in range(G):
            nb = int(lengths[g].sum())
            gt = min(N.GROUP_TOKENS, t - g * N.GROUP_TOKENS)
            chunks.append(CacheGenGPUBytestream(torch.from_numpy(payload[pos:pos + nb].copy()), lengths[g], gt))
            pos += nb
        return CacheGenGPUEncoderOutput(chunks, cdf, maxes[0], maxes[1], H, D, int(hd.version) - 1, counts_t, hd.nb)

    def to_bytes(self) -> bytes:
        """Re-assemble the flat container from the logical fields (host side; used by tests / tools).  A version-3
        object (rANS bytestreams + the histogram) is written back as version 3; without the histogram the same
        bytestreams go into a version-2 container with the CDF tensor."""
        L = self.max_tensors_key.shape[0]
        t = self.max_tensors_key.shape[1]
        H, D = self.num_heads, self.head_size
        C = H * D
        compact = int(self.coder) == N.CODER_RANS_COMPACT and self.counts is not None and self.nb is not None
        coder = int(self.coder) if compact or int(self.coder) != N.CODER_RANS_COMPACT else N.CODER_RANS
        lens = torch.stack([c.bytestream_lengths.reshape(2 * L, C) for c in self.data_chunks])
        payload = b"".join(c.bytestream.cpu().numpy().tobytes() for c in self.data_chunks)
        lo = N.container_layout(L, H, D, t, coder)
        if compact:
            pl, half = _v3_build_streams(self.counts.numpy().reshape(2 * L * C, N.LP), self.nb, C,
                                         lens.numpy().reshape(-1), np.frombuffer(payload, np.uint8))
            payload = pl.tobytes()
        total = lo.off_payload + len(payload)
        buf = bytearray(total)
        hd = N.Header.from_buffer(buf)
        hd.magic, hd.version = N.MAGIC, coder + 1
        hd.L, hd.H, hd.D, hd.ntokens, hd.ngroups = L, H, D, t, len(self.data_chunks)
        hd.max_dtype = N.DT_BF16 if self.max_tensors_key.dtype == torch.bfloat16 else N.DT_FP16
        hd.payload_bytes, hd.total_bytes, hd.status = len(payload), total, 0
        del hd

        def put(off, tensor):
            b = tensor.contiguous().cpu().view(torch.uint8).numpy().tobytes()
            buf[off:off + len(b)] = b

        if compact:
            buf[lo.off_cdf:lo.off_cdf + 2 * L] = bytes(self.nb)
            buf[lo.off_lengths:lo.off_lengths + half.size] = half.tobytes()
        else:
            put(lo.off_cdf, self.cdf.reshape(2 * L, C, N.LP))
            put(lo.off_lengths, lens.to(torch.int32))
        put(lo.off_maxes, torch.stack([self.max_tensors_key.reshape(L, t), self.max_tensors_value.reshape(L, t)]))
        buf[lo.off_payload:] = payload
        return bytes(buf)


# the legacy (CPU coder) container name the reference test imports (test_serde.py:5,60)
CacheGenEncoderOutput = CacheGenGPUEncoderOutput
