"""CPU: the lossless container for one-byte (FP8 / uint8) elements -- its numpy statement (tests/lossless8_ref.py) at the
format's edges, the layout arithmetic of the library for every element size, the header checks, and the dtype codes."""
import ctypes

import numpy as np
import pytest
import torch

import lossless8_ref as R8
import lossless_ref as R
from lmcache_b200 import _native as N
from lmcache_b200.codec import KvView, dtype_of_code, parse_lossless_header


def _roundtrip(kv, L, H, D, dtype=R8.DT_FP8_E4M3, latent=False):
    blob = R8.encode(kv, L, H, D, dtype, latent)
    hd, got = R8.decode(blob)
    assert np.array_equal(got, kv)
    assert hd["version"] == (6 if latent else 5) and hd["ngroups"] == 1 and hd["max_dtype"] == dtype
    assert hd["total_bytes"] == len(blob)
    return blob


def test_dtype_codes():
    assert (N.DT_U8, N.DT_FP8_E4M3, N.DT_FP8_E5M2) == (R8.DT_U8, R8.DT_FP8_E4M3, R8.DT_FP8_E5M2) == (2, 3, 4)
    assert KvView._code(torch.uint8) == N.DT_U8
    assert KvView._code(torch.float8_e4m3fn) == N.DT_FP8_E4M3
    assert KvView._code(torch.float8_e5m2) == N.DT_FP8_E5M2
    assert dtype_of_code(N.DT_FP8_E5M2) == torch.float8_e5m2
    with pytest.raises(TypeError):
        KvView._code(torch.float32)
    assert N.lib().b200kv_version() == 4


def test_every_byte_value_roundtrips():
    kv = np.arange(256, dtype=np.uint8).reshape(1, 16, 16)
    kv = np.concatenate([kv, kv[:, ::-1]])
    for dt in R8.ONE_BYTE:
        blob = _roundtrip(kv, 1, 2, 8, dt)
        lo = R8.layout(2, 16, 16)
        assert lo["off_payload"] == lo["off_raw"]
        freq = np.frombuffer(blob[lo["off_freq"]:lo["off_lens"]], dtype="<u2").reshape(2, 256)
        assert (freq == 16).all()                               # 256 equally frequent symbols: 4096 / 256 each


def test_single_symbol_plane():
    kv = np.full((2, 300, 16), 0x38, dtype=np.uint8)            # E4M3 1.0 everywhere
    blob = _roundtrip(kv, 1, 2, 8)
    lo = R8.layout(2, 16, 300)
    freq = np.frombuffer(blob[lo["off_freq"]:lo["off_lens"]], dtype="<u2").reshape(2, 256)
    assert (freq[:, 0x38] == 4096).all()
    lens = np.frombuffer(blob[lo["off_lens"]:lo["off_lens"] + 64], dtype="<u2")
    assert (lens == 4).all()
    assert len(blob) == lo["off_payload"] + 4 * 32


def test_256_symbol_plane_with_rare_symbols():
    rng = np.random.default_rng(2)
    t, C = 256, 64
    sym = np.full((1, t, C), 0x80, dtype=np.uint8)
    pos = rng.choice(t * C, size=256, replace=False)
    sym.reshape(-1)[pos] = np.arange(256, dtype=np.uint8)
    _roundtrip(np.concatenate([sym, sym[:, ::-1]]), 1, 1, 64, R8.DT_FP8_E5M2)
    f = R.normalise(np.bincount(sym.ravel(), minlength=256))
    assert (f > 0).all() and (f == 1).sum() >= 250 and f.sum() == 4096


@pytest.mark.parametrize("t", [1, 255, 256, 4096])
def test_token_counts(t):
    rng = np.random.default_rng(t)
    C = 8 if t == 4096 else 32
    kv = rng.integers(0, 256, size=(2, t, C), dtype=np.uint8)
    kv[:, :, : C // 2] = (rng.standard_normal((2, t, C // 2)) * 4).astype(np.int64).astype(np.uint8)
    _roundtrip(kv, 1, 1, C, R8.DT_U8)


def test_latent_roundtrip():
    rng = np.random.default_rng(5)
    kv = rng.integers(0x30, 0x48, size=(3, 40, 72), dtype=np.uint8)
    _roundtrip(kv, 3, 1, 72, R8.DT_FP8_E4M3, latent=True)


def test_stream_bound_on_incompressible_input():
    # uniform bytes: 8 bits per symbol, well inside the 12-bit bound the layout reserves
    rng = np.random.default_rng(3)
    for t in (1, 2, 3, 64, 4096):
        C = 4
        kv = rng.integers(0, 256, size=(2, t, C), dtype=np.uint8)
        blob = _roundtrip(kv, 1, 1, C)
        lo = R8.layout(2, C, t)
        lens = np.frombuffer(blob[lo["off_lens"]:lo["off_lens"] + 4 * C], dtype="<u2")
        assert (lens <= lo["max_stream"]).all() and len(blob) <= lo["max_total"]


def _native_layout(L, H, D, t, latent, dt):
    lo = N.LosslessLayout()
    N.check(N.lib().b200kv_lossless_layout_dt(L, H, D, t, int(latent), dt, ctypes.byref(lo)), "layout_dt")
    return lo


@pytest.mark.parametrize("dt", [2, 3, 4])
def test_layout_dt_matches_spec(dt):
    for L, H, D, t, latent in [(1, 1, 8, 1, False), (32, 8, 128, 256, False), (4, 1, 576, 100, True),
                               (128, 2, 64, 4096, False), (3, 3, 5, 17, False)]:
        lo = _native_layout(L, H, D, t, latent, dt)
        P = L if latent else 2 * L
        ref = R8.layout(P, H * D, t)
        assert (lo.off_freq, lo.off_lens, lo.off_raw, lo.off_payload, lo.fixed_bytes, lo.max_stream_bytes,
                lo.max_total_bytes) == (ref["off_freq"], ref["off_lens"], ref["off_raw"], ref["off_payload"],
                                        ref["off_payload"], ref["max_stream"], ref["max_total"])
        # the 16-bit layout of the same shape bounds it field by field
        w = N.lossless_layout(L, H, D, t, latent)
        assert w.off_raw == lo.off_raw and w.off_payload >= lo.off_payload and w.max_total_bytes >= lo.max_total_bytes
        assert N.lossless_layout(L, H, D, t, latent, dt).off_payload == lo.off_payload


def test_16bit_layout_unchanged():
    for L, H, D, t, latent in [(32, 8, 128, 256, False), (4, 1, 576, 100, True)]:
        P = L if latent else 2 * L
        ref = R.layout(P, H * D, t)
        for dt in (N.DT_BF16, N.DT_FP16):
            lo = _native_layout(L, H, D, t, latent, dt)
            assert (lo.off_raw, lo.off_payload, lo.max_total_bytes) == (ref["off_raw"], ref["off_payload"],
                                                                        ref["max_total"])
        lo = N.LosslessLayout()
        N.check(N.lib().b200kv_lossless_layout(L, H, D, t, int(latent), ctypes.byref(lo)), "layout")
        assert (lo.off_raw, lo.off_payload, lo.max_total_bytes) == (ref["off_raw"], ref["off_payload"], ref["max_total"])
    lo = N.LosslessLayout()
    assert N.lib().b200kv_lossless_layout_dt(1, 1, 8, 1, 0, 5, ctypes.byref(lo)) < 0     # unknown dtype


@pytest.mark.parametrize("dt", [2, 3, 4])
def test_host_plane_offsets_match_spec(dt):
    rng = np.random.default_rng(dt)
    L, H, D, t = 3, 2, 16, 37
    kv = rng.integers(0x20, 0x50, size=(2 * L, t, H * D), dtype=np.uint8)
    blob = R8.encode(kv, L, H, D, dt)
    lo = R8.layout(2 * L, H * D, t)
    out = (ctypes.c_int64 * (2 * L + 1))()
    buf = np.frombuffer(blob, dtype=np.uint8)
    assert N.lib().b200kv_lossless_plane_offsets(buf.ctypes.data, len(blob), out, 2 * L + 1) == 0
    lens = np.frombuffer(blob[lo["off_lens"]:lo["off_lens"] + 4 * L * H * D], dtype="<u2").astype(np.int64)
    want = lo["off_payload"] + np.concatenate([[0], np.cumsum(lens.reshape(2 * L, -1).sum(axis=1))])
    assert list(out) == list(want) and out[0] == lo["off_raw"] and out[2 * L] == len(blob)
    # the same bytes under a 16-bit dtype code name a container with a raw section: the lengths no longer add up
    bad = bytearray(blob)
    bad[28:32] = (0).to_bytes(4, "little")
    assert N.lib().b200kv_lossless_plane_offsets((ctypes.c_uint8 * len(bad)).from_buffer(bad), len(bad), out,
                                                 2 * L + 1) != 0


def test_parse_lossless_header_dtypes():
    rng = np.random.default_rng(9)
    kv = rng.integers(0, 256, size=(2, 8, 16), dtype=np.uint8)
    for dt in R8.ONE_BYTE:
        blob = R8.encode(kv, 1, 1, 16, dt)
        hd = parse_lossless_header(blob)
        assert hd.max_dtype == dt and hd.total_bytes == len(blob)
    for dt in (5, 7, 255):
        bad = bytearray(R8.encode(kv, 1, 1, 16, R8.DT_U8))
        bad[28:32] = dt.to_bytes(4, "little")
        with pytest.raises(ValueError, match="dtype"):
            parse_lossless_header(bytes(bad))
    # a one-byte container relabelled as bf16 is refused by its sizes: it has no raw section
    bad = bytearray(R8.encode(kv, 1, 1, 16, R8.DT_FP8_E4M3))
    bad[28:32] = (0).to_bytes(4, "little")
    with pytest.raises(ValueError):
        parse_lossless_header(bytes(bad))


def test_lossless_serde_dtype_rule():
    from lmcache_b200.storage_backend.serde.lossless import LosslessSerializer
    ser = LosslessSerializer.__new__(LosslessSerializer)
    ser.fmt = "vllm"
    with pytest.raises(TypeError, match="bfloat16 and float16"):
        ser._view(torch.zeros(1, 2, 1, 1, 8, dtype=torch.float32))
