"""CPU: where each plane's streams lie in a version-3 container (codec.plane_offsets), and the copies a layer-major upload
makes of it (pipeline.layer_copy_ranges), on containers assembled from the oracle's own encode."""
import ctypes

import numpy as np
import pytest

from lmcache_b200 import _native as N
from lmcache_b200.codec import parse_header, plane_offsets
from lmcache_b200.pipeline import layer_copy_ranges
from oracle import oracle as O

MODEL = "lmsys/longchat-7b-16k"


def _v3_container(L, t, H, D, seed):
    """(container bytes, per-plane stream bytes) of one chunk, laid out as include/b200kv.h describes version 3"""
    kb, vb = O.make_bins(MODEL)
    bits = O.synth_kv_bits(L, t, H * D, seed=seed)
    enc = O.encode_chunk(bits, O.DT_BF16, kb, vb, O.CODER_RANS_COMPACT)
    (bs, ln, _), = enc["groups"]
    nb = O.nb_map(kb, vb, L)
    payload, half = O.v3_pack(enc["counts"], nb, ln, bs)
    NL, C = 2 * L, H * D
    # each plane packed on its own: what plane p's byte range must hold
    ends = np.concatenate([[0], np.cumsum(ln.reshape(NL, C).sum(axis=1))])
    planes = [O.v3_pack(enc["counts"][p:p + 1], nb[p:p + 1], ln[p:p + 1], bs[ends[p]:ends[p + 1]])[0] for p in range(NL)]
    lo = N.container_layout(L, H, D, t, N.CODER_RANS_COMPACT)
    total = lo.off_payload + payload.size
    buf = bytearray(total)
    hd = N.Header()
    hd.magic, hd.version, hd.L, hd.H, hd.D, hd.ntokens, hd.ngroups = N.MAGIC, 3, L, H, D, t, 1
    hd.max_dtype, hd.payload_bytes, hd.total_bytes = N.DT_BF16, payload.size, total
    buf[:N.HEADER_BYTES] = bytes(hd)
    buf[lo.off_cdf:lo.off_cdf + NL] = bytes(nb)
    buf[lo.off_maxes:lo.off_maxes + enc["maxes"].nbytes] = enc["maxes"].tobytes()
    buf[lo.off_lengths:lo.off_lengths + NL * C] = half.tobytes()
    buf[lo.off_payload:] = payload.tobytes()
    return bytes(buf), planes


@pytest.mark.parametrize("L,t,H,D,seed", [(4, 256, 2, 64, 0), (3, 100, 1, 128, 1), (2, 17, 4, 32, 2), (32, 64, 1, 64, 3)])
def test_plane_offsets_partition_the_payload(L, t, H, D, seed):
    buf, planes = _v3_container(L, t, H, D, seed)
    hd = parse_header(buf)
    o = plane_offsets(buf)
    lo = N.container_layout(L, H, D, t, N.CODER_RANS_COMPACT)
    assert o.dtype == np.int64 and o.shape == (2 * L + 1,)
    assert o[0] == lo.off_payload and o[-1] == hd.total_bytes == len(buf)
    assert np.all(np.diff(o) > 0)
    for p in range(2 * L):
        assert buf[o[p]:o[p + 1]] == planes[p].tobytes(), f"plane {p}"


def test_layer_copies_cover_every_container_once():
    bufs = [_v3_container(4, t, 2, 64, s)[0] for s, t in enumerate((256, 256, 100))]
    L = 4
    offs = [plane_offsets(b) for b in bufs]
    offs.append(None)                     # a container without plane offsets is copied whole with the fixed sections
    sizes = [len(b) for b in bufs] + [4096]
    fixed, start, size = layer_copy_ranges(offs, sizes, L)
    n = len(sizes)
    assert start.shape == size.shape == (L, 2 * n)
    for j in range(n):
        spans = [(0, int(fixed[j]))]
        for layer in range(L):
            for k in (j, n + j):
                if size[layer, k]:
                    spans.append((int(start[layer, k]), int(start[layer, k] + size[layer, k])))
        spans.sort()
        pos = 0
        for a, b in spans:
            assert a == pos, f"container {j}: gap or overlap at {pos}"
            pos = b
        assert pos == sizes[j]
    assert fixed[-1] == 4096 and not size[:, n - 1].any() and not size[:, 2 * n - 1].any()


def test_damaged_lengths_give_no_plane_offsets():
    buf, _ = _v3_container(2, 64, 1, 64, 4)
    lo = N.container_layout(2, 1, 64, 64, N.CODER_RANS_COMPACT)
    bad = bytearray(buf)
    bad[lo.off_lengths] ^= 1                    # one stream one halfword longer / shorter: sums no longer match
    assert plane_offsets(bytes(bad)) is None
    v2 = bytearray(buf)
    v2[4] = 2
    assert plane_offsets(bytes(v2)) is None
    assert ctypes.sizeof(N.DecodePlan) == 2048
