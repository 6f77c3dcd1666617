"""Latent-KV (one plane per layer) reference built from the CPU oracle: the oracle's quantiser, histogram, rANS and
version-3 stream framing take any plane count, so a latent plane is coded exactly as the K plane of a (K, V) pair.
Used by tests/test_mla_cpu.py and tests/test_gpu_mla.py."""
import numpy as np

from lmcache_b200 import _native as N
from oracle import oracle as O


def encode_chunk_latent(x_bits: np.ndarray, dtype: int, key_bins):
    """x_bits uint16 [L, t, C] -> dict(sym [L,t,C], maxes u16 [L,t], counts, cdf, bytestream, lengths [L,C]): the K half
    of the oracle's quantize on [L, 2, t, C], then its CDF / histogram / rANS streams over those L planes."""
    L, t, C = x_bits.shape
    pair = np.ascontiguousarray(np.stack([x_bits, x_bits], axis=1))
    kb = np.ascontiguousarray(key_bins[:L], np.float32)
    sym, maxes = O.quantize(pair, dtype, kb, kb)
    sym = np.ascontiguousarray(sym[:L])
    c = O.cdf(sym)
    bs, ln = O.encode_group(c, sym, 0, t, O.CODER_RANS)
    return dict(sym=sym, maxes=np.ascontiguousarray(maxes[0]), counts=O.counts(sym), cdf=c, bytestream=bs, lengths=ln)


def nb_latent(key_bins, L: int):
    return [2 * (int(b) // 2) for b in list(key_bins)[:L]]


def v4_container(x_bits: np.ndarray, dtype: int, key_bins, H: int, D: int):
    """One chunk's version-4 container assembled on the host (include/b200kv.h) and the end of every plane's streams."""
    L, t, C = x_bits.shape
    enc = encode_chunk_latent(x_bits, dtype, key_bins)
    nb = nb_latent(key_bins, L)
    payload, half = O.v3_pack(enc["counts"], nb, enc["lengths"], enc["bytestream"])
    lo = N.container_layout(L, H, D, t, N.CODER_LATENT)
    total = lo.off_payload + payload.size
    buf = bytearray(total)
    hd = N.Header()
    hd.magic, hd.version, hd.L, hd.H, hd.D, hd.ntokens, hd.ngroups = N.MAGIC, 4, L, H, D, t, 1
    hd.max_dtype, hd.payload_bytes, hd.total_bytes = dtype, payload.size, total
    buf[:N.HEADER_BYTES] = bytes(hd)
    buf[lo.off_cdf:lo.off_cdf + L] = bytes(nb)
    buf[lo.off_maxes:lo.off_maxes + enc["maxes"].nbytes] = enc["maxes"].tobytes()
    buf[lo.off_lengths:lo.off_lengths + L * C] = half.tobytes()
    buf[lo.off_payload:] = payload.tobytes()
    ends = lo.off_payload + np.concatenate([[0], np.cumsum(2 * half.reshape(L, C).astype(np.int64).sum(axis=1))])
    return bytes(buf), ends, enc


def decode_latent(enc: dict, dtype: int, key_bins, out_dtype: int) -> np.ndarray:
    """The oracle's dequantised values of encode_chunk_latent's symbols: uint16 bits [L, t, C]."""
    sym = enc["sym"].astype(np.uint8)
    L, t, C = sym.shape
    kb = np.ascontiguousarray(key_bins[:L], np.float32)
    both = np.ascontiguousarray(np.concatenate([sym, sym]))
    maxes = np.ascontiguousarray(np.stack([enc["maxes"], enc["maxes"]]))
    return O.dequantize(both, maxes, dtype, kb, kb, out_dtype)[:, 0]
