"""Plain numpy statement of the lossless container for one-byte elements (B2KV versions 5 and 6 with header.max_dtype
B200KV_DT_U8, _FP8_E4M3 or _FP8_E5M2; include/b200kv.h): encoder and decoder.

Everything is the 16-bit container of tests/lossless_ref.py (whose header, normaliser and stream bound it uses) except
that an element is its own symbol, sym = the byte, and there is no raw section: its length is 0, so off_payload ==
off_raw.  The streams are coded in lockstep over tokens, as there.

kv: uint8 [P, t, C] -- the bytes of plane p (keys of layers 0..L-1, then values; or the L latent planes), token i,
channel c = h * D + d."""
import numpy as np

from lossless_ref import (HEADER_BYTES, M, MAGIC, MAX_TOKENS, RANS_LOW, Damaged, align16, header_bytes,
                          max_stream_bytes, normalise, parse_header)

DT_U8, DT_FP8_E4M3, DT_FP8_E5M2 = 2, 3, 4
ONE_BYTE = (DT_U8, DT_FP8_E4M3, DT_FP8_E5M2)


def layout(P: int, C: int, t: int) -> dict:
    off_freq = HEADER_BYTES
    off_lens = off_freq + P * 256 * 2
    off_raw = align16(off_lens + 2 * P * C)
    off_payload = off_raw                                     # no raw section
    return dict(off_freq=off_freq, off_lens=off_lens, off_raw=off_raw, off_payload=off_payload,
                max_stream=max_stream_bytes(t), max_total=align16(off_payload + P * C * max_stream_bytes(t)))


def code_streams(sym: np.ndarray, freq: np.ndarray, max_stream: int):
    """rANS streams of the symbols sym [P, t, C] against the frequency rows freq [P, 256]: (lens int64 [P * C],
    payload bytes), streams in (plane, channel) order"""
    P, t, C = sym.shape
    start = np.concatenate([np.zeros((P, 1), np.int64), np.cumsum(freq, axis=1)[:, :-1]], axis=1)
    S = P * C
    plane = np.repeat(np.arange(P), C)
    s_all = sym.transpose(1, 0, 2).reshape(t, S).astype(np.int64)
    x = np.full(S, RANS_LOW, dtype=np.int64)
    push = np.zeros((t, S), dtype=bool)
    word = np.zeros((t, S), dtype=np.uint16)
    for i in range(t - 1, -1, -1):
        f = freq[plane, s_all[i]]
        st = start[plane, s_all[i]]
        p = (x >> 20) >= f
        push[i] = p
        word[i] = (x & 0xFFFF).astype(np.uint16)
        x = np.where(p, x >> 16, x)
        x = ((x // f) << 12) + (x % f) + st
        assert (x < (1 << 32)).all() and (x >= RANS_LOW).all()
    lens = 4 + 2 * push.sum(axis=0)
    if (lens > max_stream).any():
        raise OverflowError("a stream outgrew the 12-bit-per-symbol bound")
    words = word.T[push.T]
    hw = np.empty(int(lens.sum()) // 2, dtype=np.uint16)
    first = np.concatenate([[0], np.cumsum(lens // 2)[:-1]])
    keep = np.ones(hw.size, dtype=bool)
    keep[first] = keep[first + 1] = False
    hw[first] = (x & 0xFFFF).astype(np.uint16)
    hw[first + 1] = (x >> 16).astype(np.uint16)
    hw[keep] = words
    return lens, hw.tobytes()


def encode(kv: np.ndarray, L: int, H: int, D: int, dtype: int, latent: bool = False) -> bytes:
    """One container of the P = 2L (or L) planes kv [P, t, C] (uint8)."""
    assert dtype in ONE_BYTE
    kv = np.ascontiguousarray(kv, dtype=np.uint8)
    P, t, C = kv.shape
    assert P == (L if latent else 2 * L) and C == H * D and 1 <= t <= MAX_TOKENS
    lo = layout(P, C, t)
    freq = np.stack([normalise(np.bincount(kv[p].ravel(), minlength=256)) for p in range(P)])
    lens, payload = code_streams(kv, freq, lo["max_stream"])
    total = lo["off_payload"] + len(payload)
    out = bytearray(lo["off_payload"])
    out[:HEADER_BYTES] = header_bytes(6 if latent else 5, L, H, D, t, dtype, len(payload), total)
    out[lo["off_freq"]:lo["off_lens"]] = freq.astype("<u2").tobytes()
    out[lo["off_lens"]:lo["off_lens"] + 2 * P * C] = lens.astype("<u2").tobytes()
    return bytes(out) + payload


def decode(buf) -> tuple:
    """(header dict, kv uint8 [P, t, C]) of a one-byte container; Damaged when a frequency row, a length or a stream is
    not what the encoder writes."""
    buf = np.frombuffer(bytes(buf), dtype=np.uint8)
    hd = parse_header(buf)
    if hd["magic"] != MAGIC or hd["version"] not in (5, 6) or hd["max_dtype"] not in ONE_BYTE:
        raise Damaged("not a one-byte lossless container")
    L, H, D, t = hd["L"], hd["H"], hd["D"], hd["ntokens"]
    P, C = (L if hd["version"] == 6 else 2 * L), H * D
    lo = layout(P, C, t)
    if hd["total_bytes"] != lo["off_payload"] + hd["payload_bytes"] or hd["total_bytes"] > buf.size:
        raise Damaged("bad sizes")
    freq = buf[lo["off_freq"]:lo["off_lens"]].view("<u2").reshape(P, 256).astype(np.int64)
    if (freq.sum(axis=1) != M).any():
        raise Damaged("a frequency row does not sum to 4096")
    start = np.concatenate([np.zeros((P, 1), np.int64), np.cumsum(freq, axis=1)[:, :-1]], axis=1)
    slot2sym = np.stack([np.repeat(np.arange(256), freq[p]) for p in range(P)])
    lens = buf[lo["off_lens"]:lo["off_lens"] + 2 * P * C].view("<u2").astype(np.int64)
    off = np.concatenate([[0], np.cumsum(lens)[:-1]])
    if off[-1] + lens[-1] > hd["payload_bytes"] or (lens < 4).any() or (lens % 2).any():
        raise Damaged("bad stream lengths")
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
    return hd, np.ascontiguousarray(sym.reshape(t, P, C).transpose(1, 0, 2))
