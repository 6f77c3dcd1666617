"""Plain numpy statement of the lossless container (B2KV versions 5 and 6, include/b200kv.h): encoder and decoder.

It produces byte-identical containers to b200kv_lossless_encode and is the oracle of the tests: the streams of a call are
coded in lockstep over tokens, one numpy operation per token for every (plane, channel) stream at once.

kv: uint16 [P, t, C] -- the bits of plane p (keys of layers 0..L-1, then values; or the L latent planes), token i,
channel c = h * D + d."""
import struct

import numpy as np

MAGIC = 0x564B3242
HEADER_BYTES = 64
HEADER_FMT = "<8I2QI3I"
M = 4096                 # probability precision (12 bits)
RANS_LOW = 1 << 16
MAX_TOKENS = 4096
DT_BF16, DT_FP16 = 0, 1


def align16(x: int) -> int:
    return (x + 15) & ~15


def max_stream_bytes(t: int) -> int:
    """4 state bytes + at most ceil(3t/4) + 1 renormalisation halfwords"""
    return 4 + 2 * ((3 * t + 3) // 4) + 2


def layout(P: int, C: int, t: int) -> dict:
    off_freq = HEADER_BYTES
    off_lens = off_freq + P * 256 * 2
    off_raw = align16(off_lens + 2 * P * C)
    off_payload = align16(off_raw + P * t * C)
    return dict(off_freq=off_freq, off_lens=off_lens, off_raw=off_raw, off_payload=off_payload,
                max_stream=max_stream_bytes(t), max_total=align16(off_payload + P * C * max_stream_bytes(t)))


def split(u: np.ndarray):
    """u (uint16) -> (sym, raw): v = rotl16(u, 1), sym = v >> 8, raw = v & 0xff"""
    u = u.astype(np.uint32)
    v = ((u << 1) | (u >> 15)) & 0xFFFF
    return (v >> 8).astype(np.uint8), (v & 0xFF).astype(np.uint8)


def join(sym: np.ndarray, raw: np.ndarray) -> np.ndarray:
    v = (sym.astype(np.uint32) << 8) | raw.astype(np.uint32)
    return (((v >> 1) | (v << 15)) & 0xFFFF).astype(np.uint16)


def normalise(counts: np.ndarray) -> np.ndarray:
    """the frequency row of a histogram: K = symbols that occur, f = 1 + floor(n * (4096 - K) / N) for each of them, and
    the remainder 4096 - sum(f) to the symbol with the largest count (the smallest symbol among equals)"""
    counts = np.asarray(counts, dtype=np.int64)
    N = int(counts.sum())
    K = int((counts > 0).sum())
    f = np.where(counts > 0, 1 + (counts * (M - K)) // N, 0)
    f[int(np.argmax(counts))] += M - int(f.sum())       # argmax: the first (smallest) of equal maxima
    assert f.sum() == M and (f[counts > 0] >= 1).all()
    return f.astype(np.int64)


def header_bytes(version, L, H, D, t, dtype, payload, total, status=0) -> bytes:
    return struct.pack(HEADER_FMT, MAGIC, version, L, H, D, t, 1, dtype, payload, total, status, 0, 0, 0)


def parse_header(buf) -> dict:
    v = struct.unpack(HEADER_FMT, bytes(buf[:HEADER_BYTES]))
    keys = ("magic", "version", "L", "H", "D", "ntokens", "ngroups", "max_dtype", "payload_bytes", "total_bytes",
            "status", "r0", "r1", "r2")
    return dict(zip(keys, v))


def encode(kv: np.ndarray, L: int, H: int, D: int, dtype: int, latent: bool = False) -> bytes:
    """One container of the P = 2L (or L) planes kv [P, t, C] (uint16)."""
    kv = np.ascontiguousarray(kv, dtype=np.uint16)
    P, t, C = kv.shape
    assert P == (L if latent else 2 * L) and C == H * D and 1 <= t <= MAX_TOKENS
    lo = layout(P, C, t)
    sym, raw = split(kv)                                      # [P, t, C]
    freq = np.stack([normalise(np.bincount(sym[p].ravel(), minlength=256)) for p in range(P)])   # [P, 256]
    start = np.concatenate([np.zeros((P, 1), np.int64), np.cumsum(freq, axis=1)[:, :-1]], axis=1)
    # every (plane, channel) stream at once: columns in (plane, channel) order
    S = P * C
    plane = np.repeat(np.arange(P), C)
    s_all = sym.transpose(1, 0, 2).reshape(t, S).astype(np.int64)     # [t, S]
    x = np.full(S, RANS_LOW, dtype=np.int64)
    push = np.zeros((t, S), dtype=bool)
    word = np.zeros((t, S), dtype=np.uint16)
    for i in range(t - 1, -1, -1):
        f = freq[plane, s_all[i]]
        st = start[plane, s_all[i]]
        p = (x >> 20) >= f                                    # x >> 20, not x >= f << 20: f = 4096 would overflow 32 bits
        push[i] = p
        word[i] = (x & 0xFFFF).astype(np.uint16)
        x = np.where(p, x >> 16, x)
        x = ((x // f) << 12) + (x % f) + st
        assert (x < (1 << 32)).all() and (x >= RANS_LOW).all()
    k = push.sum(axis=0)                                      # halfwords per stream
    lens = 4 + 2 * k
    if (lens > lo["max_stream"]).any():
        raise OverflowError("a stream outgrew the 12-bit-per-symbol bound")
    # stream = LE32 state, then the pushed halfwords in reverse push order = ascending token order
    words = word.T[push.T]                                    # stream-major, ascending i within a stream
    hw = np.empty(int(lens.sum()) // 2, dtype=np.uint16)
    first = np.concatenate([[0], np.cumsum(lens // 2)[:-1]])
    keep = np.ones(hw.size, dtype=bool)
    keep[first] = keep[first + 1] = False
    hw[first] = (x & 0xFFFF).astype(np.uint16)
    hw[first + 1] = (x >> 16).astype(np.uint16)
    hw[keep] = words
    payload = hw.tobytes()
    total = lo["off_payload"] + len(payload)
    out = bytearray(lo["off_payload"])
    out[:HEADER_BYTES] = header_bytes(6 if latent else 5, L, H, D, t, dtype, len(payload), total)
    out[lo["off_freq"]:lo["off_lens"]] = freq.astype("<u2").tobytes()
    out[lo["off_lens"]:lo["off_lens"] + 2 * S] = lens.astype("<u2").tobytes()
    out[lo["off_raw"]:lo["off_raw"] + P * t * C] = raw.tobytes()
    return bytes(out) + payload


class Damaged(ValueError):
    pass


def decode(buf) -> tuple:
    """(header dict, kv uint16 [P, t, C]) of a container; Damaged when a frequency row, a length or a stream is not
    what the encoder writes."""
    buf = np.frombuffer(bytes(buf), dtype=np.uint8)
    hd = parse_header(buf)
    if hd["magic"] != MAGIC or hd["version"] not in (5, 6):
        raise Damaged("not a lossless container")
    L, H, D, t = hd["L"], hd["H"], hd["D"], hd["ntokens"]
    P, C = (L if hd["version"] == 6 else 2 * L), H * D
    lo = layout(P, C, t)
    if hd["total_bytes"] != lo["off_payload"] + hd["payload_bytes"] or hd["total_bytes"] > buf.size:
        raise Damaged("bad sizes")
    freq = buf[lo["off_freq"]:lo["off_lens"]].view("<u2").reshape(P, 256).astype(np.int64)
    if (freq.sum(axis=1) != M).any():
        raise Damaged("a frequency row does not sum to 4096")
    start = np.concatenate([np.zeros((P, 1), np.int64), np.cumsum(freq, axis=1)[:, :-1]], axis=1)
    slot2sym = np.stack([np.repeat(np.arange(256), freq[p]) for p in range(P)])       # [P, 4096]
    lens = buf[lo["off_lens"]:lo["off_lens"] + 2 * P * C].view("<u2").astype(np.int64)
    off = np.concatenate([[0], np.cumsum(lens)[:-1]])
    if off[-1] + lens[-1] > hd["payload_bytes"] or (lens < 4).any() or (lens % 2).any():
        raise Damaged("bad stream lengths")
    raw = buf[lo["off_raw"]:lo["off_raw"] + P * t * C].reshape(P, t, C)
    hw = buf[lo["off_payload"]:lo["off_payload"] + hd["payload_bytes"] // 2 * 2].view("<u2").astype(np.int64)
    S = P * C
    plane = np.repeat(np.arange(P), C)
    h0 = off // 2
    x = hw[h0] | (hw[h0 + 1] << 16)
    nw = (lens - 4) // 2
    k = np.zeros(S, dtype=np.int64)
    sym = np.empty((t, S), dtype=np.uint8)
    for i in range(t):
        slot = x & (M - 1)
        s = slot2sym[plane, slot]
        sym[i] = s
        x = freq[plane, s] * (x >> 12) + slot - start[plane, s]
        r = x < RANS_LOW
        nxt = np.where(k < nw, hw[np.minimum(h0 + 2 + k, hw.size - 1)], 0)
        x = np.where(r, (x << 16) | nxt, x)
        k = k + r
    if (x != RANS_LOW).any() or (k != nw).any():
        raise Damaged("a stream did not return to its initial state")
    sym = sym.reshape(t, P, C).transpose(1, 0, 2)
    return hd, join(sym, raw)


def planes_of_blob(blob: np.ndarray, fmt: str = "vllm", latent: bool = False) -> np.ndarray:
    """[L,2,t,H,D] (vllm) / [L,2,H,t,D] (huggingface) / latent [L,t,D] uint16 -> [P, t, C]"""
    if latent:
        return blob
    if fmt == "huggingface":
        blob = blob.transpose(0, 1, 3, 2, 4)
    L, _, t, H, D = blob.shape
    return np.ascontiguousarray(blob.transpose(1, 0, 2, 3, 4)).reshape(2 * L, t, H * D)
