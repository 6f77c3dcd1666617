"""CPU: the lossless container (B2KV versions 5 and 6) -- its numpy statement (tests/lossless_ref.py) at the format's
edges, the layout arithmetic of the library, the header checks that keep the CacheGen and lossless families apart, and
the `lossless` serde's construction rules."""
import struct

import numpy as np
import pytest

import lossless_ref as R
from lmcache_b200 import _native as N
from lmcache_b200.codec import parse_header, parse_lossless_header
from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata


def _roundtrip(kv, L, H, D, dtype=R.DT_BF16, latent=False):
    blob = R.encode(kv, L, H, D, dtype, latent)
    hd, got = R.decode(blob)
    assert np.array_equal(got, kv)
    assert hd["version"] == (6 if latent else 5) and hd["ngroups"] == 1 and hd["max_dtype"] == dtype
    assert hd["total_bytes"] == len(blob)
    return blob


def test_every_bit_pattern_roundtrips():
    # one plane of 256 tokens x 256 channels holds each of the 65536 patterns once: NaN payloads, +-inf, -0, subnormals
    kv = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).reshape(1, 256, 256)
    kv = np.concatenate([kv, kv[:, ::-1]])                       # K and V planes of one layer
    for dt in (R.DT_BF16, R.DT_FP16):
        _roundtrip(kv, 1, 2, 128, dt)
    sym, raw = R.split(kv)
    assert np.array_equal(R.join(sym, raw), kv)
    # bf16: the symbol is the exponent; fp16: the 5 exponent bits and the 3 top mantissa bits
    u = np.array([0x3F80, 0xBF80, 0x7F80, 0x0001, 0x8000], dtype=np.uint16)
    assert list(R.split(u)[0]) == [0x7F, 0x7F, 0xFF, 0x00, 0x00]
    assert list(R.split(u)[1]) == [0x00, 0x01, 0x00, 0x02, 0x01]


def test_single_symbol_plane():
    # every element has the same high byte: f = 4096, the case where the renormalisation bound f << 20 overflows
    rng = np.random.default_rng(1)
    kv = (0x3F00 | rng.integers(0, 128, size=(2, 300, 16))).astype(np.uint16)    # sign 0, exponent 0x7E
    blob = _roundtrip(kv, 1, 2, 8)
    lo = R.layout(2, 16, 300)
    freq = np.frombuffer(blob[lo["off_freq"]:lo["off_lens"]], dtype="<u2").reshape(2, 256)
    assert (freq.max(axis=1) == 4096).all()
    lens = np.frombuffer(blob[lo["off_lens"]:lo["off_lens"] + 64], dtype="<u2")
    assert (lens == 4).all()                                    # the state alone, still 2^16
    assert blob[lo["off_payload"]:lo["off_payload"] + 4] == (1 << 16).to_bytes(4, "little")


def test_256_symbol_plane_with_rare_symbols():
    # one dominant symbol and 255 that occur once each: every rare frequency is the floor 1
    rng = np.random.default_rng(2)
    t, C = 256, 64
    sym = np.full((1, t, C), 0x80, dtype=np.uint8)
    pos = rng.choice(t * C, size=256, replace=False)
    sym.reshape(-1)[pos] = np.arange(256, dtype=np.uint8)
    raw = rng.integers(0, 256, size=(1, t, C), dtype=np.uint8)
    kv = R.join(np.concatenate([sym, sym[:, ::-1]]), np.concatenate([raw, raw]))
    _roundtrip(kv, 1, 1, 64)
    f = R.normalise(np.bincount(sym.ravel(), minlength=256))
    assert (f > 0).all() and (f == 1).sum() >= 250 and f.sum() == 4096


def test_normalise_rule():
    assert list(R.normalise(np.eye(256, dtype=np.int64)[7] * 5)[[6, 7, 8]]) == [0, 4096, 0]
    f = R.normalise(np.array([3, 3] + [0] * 254))
    assert f[0] == 2048 and f[1] == 2048                       # ties: the smaller symbol gets the remainder (0 here)
    f = R.normalise(np.array([1, 2, 2, 0, 1] + [0] * 251))
    assert f.sum() == 4096 and f[1] >= f[2] and f[3] == 0 and f[0] >= 1


@pytest.mark.parametrize("t", [1, 2, 255, 256, 257, 4096])
def test_token_counts(t):
    rng = np.random.default_rng(t)
    C = 9 if t == 4096 else 24
    x = rng.standard_normal((2, t, C)).astype(np.float32)
    kv = (x.view(np.uint32) >> 16).astype(np.uint16)           # bf16 bits of normal data
    _roundtrip(kv, 1, 3, C // 3, R.DT_BF16)
    _roundtrip(kv[:1], 1, 3, C // 3, R.DT_FP16, latent=True)


@pytest.mark.parametrize("t", [1, 3, 256, 4096])
def test_stream_bound_on_incompressible_input(t):
    # uniform 16-bit patterns (every symbol near 1/256) and the adversarial case: one channel made of the rarest symbol
    # of a wide plane (f = 1, 12 bits per symbol)
    rng = np.random.default_rng(10 + t)
    C = 64 if t < 4096 else 16
    kv = rng.integers(0, 1 << 16, size=(2, t, C), dtype=np.uint64).astype(np.uint16)
    blob = _roundtrip(kv, 1, 1, C)
    lo = R.layout(2, C, t)
    lens = np.frombuffer(blob[lo["off_lens"]:lo["off_lens"] + 4 * C], dtype="<u2")
    assert lens.max() <= lo["max_stream"] <= 0xFFFF
    wide = 4096
    sym = np.zeros((1, t, wide), dtype=np.uint8)
    sym[0, :, 0] = 0xAB                                         # t of t * 4096 symbols: f = 1
    for trial in range(2):
        kv1 = R.join(sym, rng.integers(0, 256, size=sym.shape, dtype=np.uint8))
        if trial:
            kv1[0, :, 0] = R.join(np.full(t, 0xAB, np.uint8), np.zeros(t, np.uint8))
        b = R.encode(kv1, 1, 1, wide, R.DT_BF16, latent=True)
        lo1 = R.layout(1, wide, t)
        l1 = np.frombuffer(b[lo1["off_lens"]:lo1["off_lens"] + 2 * wide], dtype="<u2")
        assert l1[0] <= lo1["max_stream"] and l1[0] >= 4 + 2 * ((3 * t) // 4) - 2
        assert np.array_equal(R.decode(b)[1], kv1)
    assert R.max_stream_bytes(4096) == 4 + 2 * 3072 + 2 <= 0xFFFF


def test_layout_matches_library():
    for (L, H, D, t, latent) in [(32, 8, 128, 256, False), (1, 1, 1, 1, False), (61, 1, 576, 64, True),
                                 (128, 32, 128, 4096, False), (3, 5, 7, 257, True)]:
        lo = N.lossless_layout(L, H, D, t, latent)
        ref = R.layout(L if latent else 2 * L, H * D, t)
        assert (lo.off_freq, lo.off_lens, lo.off_raw, lo.off_payload) == \
            (ref["off_freq"], ref["off_lens"], ref["off_raw"], ref["off_payload"])
        assert lo.fixed_bytes == lo.off_payload and lo.max_stream_bytes == ref["max_stream"]
        assert lo.max_total_bytes == ref["max_total"]
        assert all(o % 16 == 0 for o in (lo.off_freq, lo.off_lens, lo.off_raw, lo.off_payload, lo.max_total_bytes))
    for bad in [(0, 1, 1, 1), (129, 1, 1, 1), (1, 1, 1, 0), (1, 1, 1, 4097), (1, 0, 8, 8)]:
        with pytest.raises(N.NativeError):
            N.lossless_layout(*bad)
    lib = N.lib()
    assert lib.b200kv_lossless_workspace_bytes(32, 8, 128, 4097, 1, 0, 0) < 0
    assert lib.b200kv_lossless_workspace_bytes(32, 8, 128, 256, 4, 0, 0) > lib.b200kv_lossless_workspace_bytes(
        32, 8, 128, 256, 4, 0, 1) > 0
    # the CacheGen layout and version number are unchanged
    assert lib.b200kv_version() == 4
    with pytest.raises(N.NativeError):
        N.container_layout(2, 1, 8, 16, 3)
    assert N.coder_of_version(5) == N.CODER_LOSSLESS and N.coder_of_version(6) == N.CODER_LOSSLESS_LATENT
    assert N.planes_of(6, 61) == 61 and N.planes_of(5, 61) == 122


def _sample(latent=False, t=40):
    rng = np.random.default_rng(5)
    P = 2 if latent else 4
    x = rng.standard_normal((P, t, 16)).astype(np.float32)
    kv = (x.view(np.uint32) >> 16).astype(np.uint16)
    return R.encode(kv, 2 if not latent else P, 2, 8, R.DT_BF16, latent)


def test_lossless_header_check():
    blob = _sample()
    hd = parse_lossless_header(blob)
    assert hd.version == 5 and hd.total_bytes == len(blob)
    assert parse_lossless_header(_sample(latent=True)).version == 6
    assert parse_lossless_header(blob[:64], len(blob)).ntokens == 40

    def patched(off, fmt, val, base=blob):
        b = bytearray(base)
        struct.pack_into("<" + fmt, b, off, val)
        return bytes(b)
    damaged = [blob[:63], blob[:-2],                              # too short, truncated
               patched(0, "I", 0x12345678),                       # magic
               patched(8, "I", 0), patched(8, "I", 129),          # L
               patched(20, "I", 0), patched(20, "I", 4097),       # ntokens
               patched(24, "I", 2),                               # ngroups
               patched(28, "I", 2),                               # dtype
               patched(32, "Q", 1), patched(40, "Q", len(blob) - 2),   # payload / total mismatch
               patched(48, "I", 1),                               # encoder status
               patched(52, "I", 7)]                               # reserved
    for b in damaged:
        with pytest.raises(ValueError):
            parse_lossless_header(b)
    # the families stay apart: CacheGen's check refuses versions 5 and 6, the lossless check versions 1 to 4
    with pytest.raises(ValueError, match="unsupported B2KV version 5"):
        parse_header(blob)
    with pytest.raises(ValueError, match="unsupported B2KV version 6"):
        parse_header(_sample(latent=True))
    for v in (1, 2, 3, 4, 7):
        with pytest.raises(ValueError, match="not a lossless"):
            parse_lossless_header(patched(4, "I", v))


def test_reference_decoder_refuses_damage():
    blob = bytearray(_sample())
    lo = R.layout(4, 16, 40)
    for off, val in [(lo["off_freq"] + 2, 0xFFFF), (lo["off_lens"], 3), (lo["off_payload"] + 1, 0x55)]:
        b = bytearray(blob)
        b[off] ^= val & 0xFF
        with pytest.raises(R.Damaged):
            R.decode(bytes(b))


def test_create_serde_and_config():
    from lmcache_b200.storage_backend.serde import CreateSerde
    meta = LMCacheEngineMetadata("lmsys/longchat-7b-16k", 1, 0, "vllm", "bfloat16")
    cfg = LMCacheEngineConfig.from_defaults(chunk_size=8192, remote_url="lm://localhost:1", remote_serde="lossless")
    with pytest.raises(ValueError, match="4096"):
        CreateSerde("lossless", cfg, meta)
    with pytest.raises(ValueError, match="lossless"):
        CreateSerde("fast", cfg, meta)
    cfg = LMCacheEngineConfig.from_defaults(chunk_size=4096, remote_url="lm://localhost:1", remote_serde="lossless")
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:       # noqa: BLE001
        has_gpu = False
    if not has_gpu:        # the codec needs a device: the serde fails loudly, with no CPU fallback
        with pytest.raises(RuntimeError, match="CUDA|no CPU fallback"):
            CreateSerde("lossless", cfg, meta)
    # resharding stays a CacheGen feature
    from lmcache_b200.storage_backend import CreateStorageBackend
    with pytest.raises(ValueError, match="cachegen"):
        CreateStorageBackend(LMCacheEngineConfig.from_defaults(chunk_size=256, local_device=None,
                                                               remote_url="lm://localhost:1", remote_serde="lossless",
                                                               reshard_world_sizes=[2]), meta)
