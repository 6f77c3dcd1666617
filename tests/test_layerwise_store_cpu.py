"""CPU: the host-testable parts of the layer-by-layer store -- the arena placement rule (pipeline.arena_placement, the
statement of codec.cu's place_kernel), the plane-range tile remap of encode_kernel / absmax_kernel (codec.cu
launch_plane), and the LayerwiseStore handle's state machine against a fake encode."""
import itertools
import random

import numpy as np
import pytest

from lmcache_b200.cache_engine import LayerwiseStore
from lmcache_b200.pipeline import arena_placement


def test_arena_placement_fits_everything_in_order():
    seg = np.array([[100, 17, 32], [5, 5, 5]])
    base, fit = arena_placement(seg, 1 << 20)
    assert fit == 3
    assert base.tolist() == [[0, 112, 144], [176, 192, 208]]          # 16-byte aligned, (call, chunk) order


def test_arena_placement_keeps_a_prefix_across_calls():
    seg = np.array([[64, 64, 64, 64], [64, 64, 64, 64]])
    base, fit = arena_placement(seg, 64 * 6)
    assert fit == 3                                  # call 1 keeps room for call 2: chunks 0-2 (192 B + 192 B reserve)
    assert (base[:, 3:] == -1).all() and (base[:, :3] >= 0).all()
    seg = np.array([[64] * 4, [64] * 4, [100] * 4])  # the last call is larger than the reserve: its tail chunk fails
    base, fit = arena_placement(seg, 64 * 3 * 3 + 16)
    assert 0 < fit < 3 and (base[:, fit:] == -1).all()
    rng = random.Random(1)
    for _ in range(200):
        calls, n = rng.randint(1, 6), rng.randint(1, 9)
        seg = np.array([[rng.randint(0, 300) for _ in range(n)] for _ in range(calls)])
        cap = rng.randint(0, 4000)
        base, fit = arena_placement(seg, cap)
        assert (base[:, :fit] >= 0).all() and (base[:, fit:] == -1).all()
        used = sum((int(s) + 15) & ~15 for s in seg[:, :fit].ravel())
        assert used <= cap
        ends = [(int(base[c, j]), int(base[c, j]) + int(seg[c, j])) for c in range(calls) for j in range(fit)]
        ends.sort()
        assert all(a[1] <= b[0] for a, b in zip(ends, ends[1:])), "segments overlap"


def _launch_tiles(L, tpp, lb, nlay):
    """(plane, channel tile) of every tile of a launch over layers [lb, lb + nlay): codec.cu's decode_tile + launch_plane
    for one group -- K planes lb.., then V planes L + lb.."""
    out = []
    for tile in range(2 * nlay * tpp):
        local, ct = divmod(tile, tpp)
        nl = local + (lb if local < nlay else L - nlay + lb)
        out.append((nl, ct))
    return out


@pytest.mark.parametrize("L,tpp", [(1, 1), (4, 2), (6, 3), (32, 32)])
def test_plane_range_remap_covers_every_tile_once(L, tpp):
    rng = random.Random(L * 100 + tpp)
    parts = [[1] * L, [L]]
    for _ in range(20):
        cuts = sorted(rng.sample(range(1, L), rng.randint(0, L - 1))) if L > 1 else []
        parts.append([b - a for a, b in zip([0] + cuts, cuts + [L])])
    for part in parts:
        seen = []
        lb = 0
        for nlay in part:
            tiles = _launch_tiles(L, tpp, lb, nlay)
            planes = {nl for nl, _ in tiles}
            assert planes == set(range(lb, lb + nlay)) | set(range(L + lb, L + lb + nlay))
            seen += tiles
            lb += nlay
        assert sorted(seen) == sorted(itertools.product(range(2 * L), range(tpp)))
    assert _launch_tiles(L, tpp, 0, L) == list(itertools.product(range(2 * L), range(tpp)))   # identity for all layers


class _Stream:
    def __init__(self):
        self.waited = []

    def wait_event(self, ev):
        self.waited.append(ev)


class _FakeEncode:
    def __init__(self):
        self.layers, self.finished, self.abandoned = [], False, False

    def encode_layer(self, layer, stream):
        self.layers.append((layer, stream))

    def finish(self):
        self.finished = True
        return "done-event"

    def abandon(self):
        self.abandoned = True


def _handle(L=4):
    enc, calls = _FakeEncode(), []
    return LayerwiseStore(L, enc, lambda stream, e: calls.append((stream, e))), enc, calls


def test_handle_encodes_each_saved_layer_and_publishes_on_finish():
    h, enc, calls = _handle()
    s = _Stream()
    for layer in (3, 1, 0, 2):
        h.save_layer(layer, s)
    assert [l for l, _ in enc.layers] == [3, 1, 0, 2] and all(st is s for _, st in enc.layers)
    assert not calls
    h.finish(s)
    assert enc.finished and s.waited == ["done-event"] and calls == [(s, enc)] and not enc.abandoned
    with pytest.raises(ValueError):
        h.finish(s)
    with pytest.raises(ValueError):
        h.save_layer(0, s)


def test_handle_rejects_bad_layers_and_incomplete_finish():
    h, enc, calls = _handle()
    s = _Stream()
    h.save_layer(0, s)
    for bad in (0, 4, -1):
        with pytest.raises(ValueError):
            h.save_layer(bad, s)
    assert [l for l, _ in enc.layers] == [0]
    with pytest.raises(ValueError):
        h.finish(s)
    assert enc.abandoned and not enc.finished and not calls            # nothing stored, scratch given back


def test_dropped_handle_gives_its_scratch_back():
    h, enc, _ = _handle()
    h.save_layer(0, _Stream())
    del h
    assert enc.abandoned


def test_fallback_handle_runs_the_ordinary_store_at_finish():
    calls = []
    h = LayerwiseStore(2, None, lambda stream, e: calls.append((stream, e)))
    s = _Stream()
    h.save_layer(1, s)
    h.save_layer(0, s)
    assert not calls
    h.finish(s)
    assert calls == [(s, None)] and s.waited == []
