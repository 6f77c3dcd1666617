"""CPU: the host-side parts of the layer-wise store on the lossless tiers -- the copy ranges that assemble a container
from its fixed image and its arena segments (pipeline.segment_copy_ranges), the arena rule with lossless segment sizes
(pipeline.arena_placement), and the engine's gate, which asks the tier for its largest chunk."""
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import lossless_ref as ref
from lmcache_b200.codec import SegmentLayout, lossless_plane_offsets
from lmcache_b200.pipeline import arena_placement, segment_copy_ranges

# (L, H, D, chunk tokens, last chunk tokens, latent): gaps after the lengths and after the raw rows are non-empty in the
# first two (2 * P * C and P * t * C not multiples of 16), the third is version 6
GEOMS = [(3, 1, 5, 3, 2, False), (2, 3, 3, 5, 5, False), (3, 1, 7, 5, 3, True), (2, 2, 8, 16, 9, False)]


def _containers(L, H, D, cs, last, latent, n=3, seed=0):
    rng = np.random.default_rng(seed)
    P = L if latent else 2 * L
    out = []
    for j in range(n):
        t = last if j == n - 1 else cs
        kv = rng.normal(0, 1, (P, t, H * D)).astype(np.float32)
        bits = torch.from_numpy(kv).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
        if j == 1:
            bits[0] = bits[0, 0, 0]                          # one single-symbol plane (frequency 4096)
        out.append(ref.encode(bits, L, H, D, ref.DT_BF16, latent))
    return out


def _local_planes(L, latent, a, b):
    """the planes of a call over layers [a, b), in the order the device codes them: keys, then values"""
    return list(range(a, b)) if latent else list(range(a, b)) + list(range(L + a, L + b))


def _segment(cont, L, C, latent, a, b):
    """the segment the device writes for one container in a call over layers [a, b): [raw rows of the call's planes
    (and the zero gap up to off_payload in the call that holds the last plane), zeros to 16 bytes][the call's streams];
    and per plane its (raw offset, stream offset, stream bytes) inside the segment"""
    t, P = ref.parse_header(cont)["ntokens"], (L if latent else 2 * L)
    lo = ref.layout(P, C, t)
    lens = np.frombuffer(cont[lo["off_lens"]:lo["off_lens"] + 2 * P * C], dtype="<u2").reshape(P, C).astype(np.int64)
    soff = lo["off_payload"] + np.concatenate([[0], np.cumsum(lens.sum(axis=1))])
    planes = _local_planes(L, latent, a, b)
    raw = b"".join(cont[lo["off_raw"] + p * t * C: lo["off_raw"] + (p + 1) * t * C] for p in planes)
    if b == L:
        raw += cont[lo["off_raw"] + P * t * C: lo["off_payload"]]
    raw += bytes(ref.align16(len(raw)) - len(raw))
    rows, streams = {}, b""
    for i, p in enumerate(planes):
        rows[p] = (i * t * C, len(raw) + len(streams), int(soff[p + 1] - soff[p]))
        streams += cont[soff[p]:soff[p + 1]]
    return raw + streams, rows


def _partitions(L):
    rng = random.Random(L)
    parts = [[1] * L, [L]]
    for _ in range(3):
        cuts = sorted(rng.sample(range(1, L), rng.randint(1, L - 1))) if L > 1 else []
        parts.append([b - a for a, b in zip([0] + cuts, cuts + [L])])
    return parts


@pytest.mark.parametrize("geom", GEOMS)
def test_segments_reassemble_the_whole_container(geom):
    L, H, D, cs, last, latent = geom
    C, P = H * D, (L if latent else 2 * L)
    conts = _containers(L, H, D, cs, last, latent, seed=L * 7 + D)
    n = len(conts)
    for calls in _partitions(L):
        bounds = np.cumsum([0] + calls)
        fwd = [(int(bounds[i]), int(bounds[i + 1])) for i in range(len(calls))]
        for ranges in (fwd, fwd[::-1]):                   # the calls in layer order, and the last layers first
            segs = [[_segment(c, L, C, latent, a, b) for c in conts] for a, b in ranges]
            seg_bytes = np.array([[len(s) for s, _ in row] for row in segs], dtype=np.int64)
            base, fit = arena_placement(seg_bytes, 1 << 30, [b - a for a, b in ranges])
            assert fit == n
            arena = bytearray(int(base.max() + seg_bytes.max()) + 16)
            rows = np.zeros((n, P, 3), dtype=np.int64)
            for ci, row in enumerate(segs):
                for j, (data, prow) in enumerate(row):
                    o = int(base[ci, j])
                    arena[o:o + len(data)] = data
                    for p, (r, s, m) in prow.items():
                        rows[j, p] = (o + r, o + s, m)
            layouts = []
            for c in conts:
                t = ref.parse_header(c)["ntokens"]
                lo = ref.layout(P, C, t)
                layouts.append(SegmentLayout(lo["off_raw"], lo["off_payload"], t * C))
            dst, src, lens, planes = segment_copy_ranges(rows, layouts)
            assert dst.shape == (n, 1 + 2 * P)
            for j, c in enumerate(conts):
                fixed = c[:layouts[j].head]               # the fixed image: header, frequency rows, lengths, zero gap
                got = bytearray(int(lens[j].sum()))
                for d, s, m in zip(dst[j], src[j], lens[j]):
                    got[d:d + m] = fixed[:m] if s < 0 else arena[s:s + m]
                assert bytes(got) == c, (geom, ranges, j)
                assert planes[j].tolist() == lossless_plane_offsets(c).tolist()


def test_segment_rows_of_a_single_call_are_contiguous_and_cover_the_gap():
    L, H, D, cs, last, latent = GEOMS[0]
    C, P = H * D, 2 * L
    (c,) = _containers(L, H, D, cs, cs, latent, n=1)
    lo = ref.layout(P, C, cs)
    assert lo["off_raw"] > lo["off_lens"] + 2 * P * C and lo["off_payload"] > lo["off_raw"] + P * cs * C  # both gaps
    assert c[lo["off_lens"] + 2 * P * C:lo["off_raw"]] == bytes(lo["off_raw"] - lo["off_lens"] - 2 * P * C)
    seg, rows = _segment(c, L, C, latent, 0, L)
    rows = np.array([rows[p] for p in range(P)], dtype=np.int64)[None]
    dst, src, lens, planes = segment_copy_ranges(rows, [SegmentLayout(lo["off_raw"], lo["off_payload"], cs * C)])
    assert lens[0, P] == lo["off_payload"] - lo["off_raw"] - (P - 1) * cs * C    # the last raw range runs to the payload
    assert int(lens[0].sum()) == len(c) and planes[0, -1] == len(c)


def test_cachegen_rows_keep_their_ranges():
    seg = np.array([[[100, 6], [106, 10]], [[200, 4], [204, 8]]], dtype=np.int64)
    dst, src, lens, planes = segment_copy_ranges(seg, [SegmentLayout(48, 48), SegmentLayout(32, 32)])
    assert dst.tolist() == [[0, 48, 54], [0, 32, 36]]
    assert src.tolist() == [[-1, 100, 106], [-1, 200, 204]]
    assert lens.tolist() == [[48, 6, 10], [32, 4, 8]]
    assert planes.tolist() == [[48, 54, 64], [32, 36, 44]]


def test_arena_placement_with_lossless_segments_keeps_a_prefix():
    L, H, D, cs, last, latent = GEOMS[3]
    C, P = H * D, 2 * L
    conts = _containers(L, H, D, cs, last, latent, n=6, seed=3)
    seg = np.array([[len(_segment(c, L, C, latent, l, l + 1)[0]) for c in conts] for l in range(L)], dtype=np.int64)
    total = int(((seg + 15) // 16 * 16).sum())
    for budget in (total // 3, total // 2, total - 1):
        base, fit = arena_placement(seg, budget)
        assert 0 < fit < len(conts)
        assert (base[:, :fit] >= 0).all() and (base[:, fit:] == -1).all()
        assert int(((seg[:, :fit] + 15) // 16 * 16).sum()) <= budget
    base, fit = arena_placement(seg, total)
    assert fit == len(conts)


@pytest.mark.parametrize("serde_max,cs,ok", [(4096, 256, True), (4096, 1024, True), (4096, 4096, True),
                                             (4096, 8192, False), (256, 256, True), (256, 512, False)])
def test_store_gate_follows_the_tiers_limit(serde_max, cs, ok):
    from lmcache_b200.cache_engine import LMCacheEngine
    tier = SimpleNamespace(begin_layerwise_store=lambda *a: None, layerwise_max_tokens=serde_max)
    eng = SimpleNamespace(engine_=tier, _fast_path=lambda: True, chunk_size=cs)
    assert LMCacheEngine._layerwise_store_ok(eng, torch.bfloat16) is ok
    assert LMCacheEngine._layerwise_store_ok(eng, torch.float32) is False
    assert LMCacheEngine._layerwise_store_ok(SimpleNamespace(engine_=SimpleNamespace(layerwise_max_tokens=4096),
                                                             _fast_path=lambda: True, chunk_size=cs),
                                             torch.bfloat16) is False          # no layer-wise store (raw, remote tiers)
