"""CPU: container version 4 -- one latent plane per layer (multi-head latent attention, e.g. DeepSeek-V2/V3).

* Layout arithmetic of version 4 next to version 3, and the coders that have no latent layout.
* parse_header / check_header / plane_offsets / b200kv_plane_offsets on version-4 containers assembled on the host from
  the oracle, at L = 1, 27, 61 and 128.
* A version-4 container is refused where version 3 is expected, and the reverse."""
import numpy as np
import pytest

from lmcache_b200 import _native as N
from lmcache_b200.codec import check_header, parse_header, plane_offsets
from oracle import oracle as O

import mla_ref


def _bins(L, seed):
    return np.random.default_rng(seed).integers(4, 33, size=L).astype(np.float32)


def test_latent_flag_values():
    assert N.KV_LATENT == 0x100 and N.CODER_LATENT == N.CODER_RANS_COMPACT | N.KV_LATENT
    assert N.lib().b200kv_version() == 4
    assert N.coder_of_version(4) == N.CODER_LATENT and [N.coder_of_version(v) for v in (1, 2, 3)] == [0, 1, 2]
    assert N.planes_of(4, 61) == 61 and N.planes_of(3, 61) == 122


@pytest.mark.parametrize("L,H,D,t", [(1, 1, 576, 256), (61, 1, 576, 256), (27, 1, 20, 7), (128, 2, 64, 1)])
def test_v4_layout_is_v3_with_L_planes(L, H, D, t):
    C = H * D
    a16 = lambda x: (x + 15) & ~15
    lo = N.container_layout(L, H, D, t, N.CODER_LATENT)
    assert lo.off_cdf == 64
    assert lo.off_maxes == a16(64 + L)
    assert lo.off_lengths == a16(lo.off_maxes + L * t * 2)
    assert lo.off_payload == a16(lo.off_lengths + L * C) == lo.fixed_bytes
    assert lo.max_total_bytes == a16(lo.off_payload + L * C * (2 * t + 4 + N.HDR_MAX) + 16)
    # version 3 of 2L planes; version 4 at 2L layers is that, plane for plane
    v3 = N.container_layout(L, H, D, t, N.CODER_RANS_COMPACT)
    assert v3.off_payload == a16(a16(a16(64 + 2 * L) + 2 * L * t * 2) + 2 * L * C)
    if 2 * L <= 128:
        assert N.container_layout(2 * L, H, D, t, N.CODER_LATENT).fixed_bytes == v3.fixed_bytes


def test_v4_layout_refusals():
    for coder in (N.CODER_AC | N.KV_LATENT, N.CODER_RANS | N.KV_LATENT, 3):
        with pytest.raises(N.NativeError):
            N.container_layout(4, 1, 576, 16, coder)
    with pytest.raises(N.NativeError):                        # a compact container holds <= 256 tokens
        N.container_layout(4, 1, 576, 257, N.CODER_LATENT)
    lib = N.lib()
    assert lib.b200kv_encode_workspace_bytes(4, 1, 576, 256, 2, N.CODER_RANS | N.KV_LATENT) < 0
    lat = lib.b200kv_encode_workspace_bytes(61, 1, 576, 256, 4, N.CODER_LATENT)
    pair = lib.b200kv_encode_workspace_bytes(61, 1, 576, 256, 4, N.CODER_RANS_COMPACT)
    assert 0 < lat < pair


@pytest.mark.parametrize("L", [1, 27, 61, 128])
def test_parse_header_and_plane_offsets_on_oracle_v4(L):
    H, D = (1, 20) if L > 27 else (1, 576)
    t = {1: 256, 27: 33, 61: 5, 128: 3}[L]
    kb = _bins(L, L)
    bits = O.synth_kv_bits(L, t, H * D, seed=L)[:, 0]
    raw, ends, enc = mla_ref.v4_container(bits, O.DT_BF16, kb, H, D)
    hd = parse_header(raw)
    assert (hd.version, hd.L, hd.H, hd.D, hd.ntokens, hd.ngroups) == (4, L, H, D, t, 1)
    assert hd.nb == mla_ref.nb_latent(kb, L)
    assert np.array_equal(plane_offsets(raw), ends) and ends[-1] == len(raw)
    a = np.frombuffer(raw, np.uint8)
    o = np.full(N.MAX_PLANES + 1, -5, np.int64)
    assert N.lib().b200kv_plane_offsets(a.ctypes.data, a.size, o.ctypes.data, o.size) == 0
    assert np.array_equal(o[:L + 1], ends) and (o[L + 1:] == -5).all()
    assert N.lib().b200kv_plane_offsets(a.ctypes.data, a.size, o.ctypes.data, L) < 0      # needs L + 1 entries
    # the oracle decodes its own streams back to the symbols
    out = np.zeros((L, t, H * D), np.uint8)
    O.decode_group(enc["cdf"], enc["bytestream"], enc["lengths"], out, 0, t, O.CODER_RANS)
    assert np.array_equal(out, enc["sym"].astype(np.uint8))
    # a damaged nb map, a length that does not add up, more layers than the table holds
    bad = bytearray(raw)
    bad[64] = 3
    with pytest.raises(ValueError):
        parse_header(bytes(bad))
    bad = bytearray(raw)
    bad[8:12] = (129).to_bytes(4, "little")
    with pytest.raises(ValueError):
        parse_header(bytes(bad))
    with pytest.raises(ValueError):
        parse_header(raw[:-2])


def test_v4_refused_where_v3_expected_and_the_reverse():
    from lmcache_b200.codec import CacheGenCodec
    from lmcache_b200.storage_backend.serde.cachegen_basics import CacheGenGPUEncoderOutput
    L, t, H, D = 4, 9, 1, 576
    kb, vb = O.make_bins("lmsys/longchat-7b-16k")
    raw4, _, _ = mla_ref.v4_container(O.synth_kv_bits(L, t, H * D, seed=1)[:, 0], O.DT_BF16, kb, H, D)
    hd4 = parse_header(raw4)
    # the header of a version-3 container with the same bytes after it (2L-entry nb map) is not a valid version 4
    hd3 = parse_header(raw4)
    hd3.version = 3
    with pytest.raises(ValueError):
        check_header(hd3, hd4.nb)
    hd4b = parse_header(raw4)
    with pytest.raises(ValueError):
        check_header(hd4b, hd4.nb + hd4.nb)
    with pytest.raises(ValueError):                       # the reference-shaped object form has (K, V) planes only
        CacheGenGPUEncoderOutput.from_bytes(raw4)
    # the match rule of a codec: plane layout first, then bins
    codec = CacheGenCodec.__new__(CacheGenCodec)
    codec.nlayers, codec.v3_only, codec._nb = len(kb), False, N.nb_map(kb, vb, len(kb))
    assert not codec.accepts(hd4) and codec.accepts(hd4, latent=True)
    hd4.nb = [32] * L if hd4.nb != [32] * L else [16] * L
    assert not codec.accepts(hd4, latent=True)
    hdv3 = N.Header()
    hdv3.version, hdv3.L, hdv3.nb = 3, L, N.nb_map(kb, vb, L)
    assert codec.accepts(hdv3) and not codec.accepts(hdv3, latent=True)
    # device-side plane offsets read version 4 too (checked on the GPU); the host one refuses versions 1 and 2
    a = np.frombuffer(bytes(bytearray(raw4[:4]) + (2).to_bytes(4, "little") + raw4[8:]), np.uint8)
    o = np.zeros(N.MAX_PLANES + 1, np.int64)
    assert N.lib().b200kv_plane_offsets(a.ctypes.data, a.size, o.ctypes.data, o.size) < 0
