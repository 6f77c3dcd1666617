"""CPU: the pure parts of the layer-wise segment retrieve -- the match of a multi-run fetch with its fallback keys
(pipeline.match_runs) and the seg_of_tok a tier builds for the chunks it wrote (rope.written_seg_of_tok)."""
import pytest

import numpy as np

from lmcache_b200.pipeline import match_runs, rest_runs
from lmcache_b200.rope import chunk_arrays, plan_segments, written_seg_of_tok

CS = 4


def _run(stored, names, fb_names=None, tok0=0, log=None):
    """a run over `names`, its items the stored values (None: a miss); fallback names continue it"""
    def items(ns):
        for n in ns:
            if log is not None:
                log.append(n)
            yield stored.get(n)
    fb = None if fb_names is None else (lambda i: items(fb_names[i:]))
    return items(names), fb, tok0


def test_miss_ends_only_its_run():
    stored = {"a0": 1, "a1": 2, "b0": 3, "b2": 4}
    out = match_runs([_run(stored, ["a0", "a1", "a2"]), _run(stored, ["b0", "b1", "b2"], tok0=100)], CS,
                     lambda it, tok: True)
    assert out == [([(1, 0), (2, 4)], 2), ([(3, 100)], 1)]


def test_continuation_starts_at_the_first_primary_miss():
    stored = {"p0": 1, "p1": 2, "d2": 5, "d3": 6, "d0": 9, "d1": 9}
    log = []
    out = match_runs([_run(stored, ["p0", "p1", "p2", "p3", "p4"], ["d0", "d1", "d2", "d3", "d4"], tok0=10, log=log)],
                     CS, lambda it, tok: True)
    # primary hits 0 and 1, then derived keys from index 2 on: d0 and d1 are never looked up
    assert out == [([(1, 10), (2, 14), (5, 18), (6, 22)], 2)]
    assert log == ["p0", "p1", "p2", "d2", "d3", "d4"]


def test_no_fallback_and_full_primary_hit():
    stored = {"p0": 1, "p1": 2, "d0": 7}
    out = match_runs([_run(stored, ["p0", "p1"], ["d0", "d1"]), _run(stored, ["x"], None), _run(stored, [], ["d0"])],
                     CS, lambda it, tok: True)
    assert out == [([(1, 0), (2, 4)], 2), ([], 0), ([(7, 0)], 0)]


def test_refused_item_is_a_miss_of_its_run_only():
    stored = {"a0": 1, "a1": -1, "a2": 3, "b0": 4, "b1": 5}
    seen = []

    def fits(it, tok):
        seen.append((it, tok))
        return it > 0
    out = match_runs([_run(stored, ["a0", "a1", "a2"], ["c0", "c1", "c2"]), _run(stored, ["b0", "b1"], tok0=50)], CS,
                     fits)
    assert out == [([(1, 0)], 1), ([(4, 50), (5, 54)], 2)]
    assert seen == [(1, 0), (-1, 4), (4, 50), (5, 54)]          # c1 is a miss: fits is never asked


def test_written_seg_of_tok_tails_and_start_zero():
    # run 0 starts at token 0 (row -1), run 1 at 20 (row 0) with a short tail chunk, run 2 at 40 (row 1)
    chunks = [(0, 0, 4), (0, 4, 4), (1, 20, 4), (1, 24, 4), (1, 28, 2), (2, 40, 3)]
    lo, sot = written_seg_of_tok(chunks, [-1, 0, 1], [8, 30, 43])
    assert lo == 20 and len(sot) == 23 and sot.dtype == np.int32
    assert list(sot[:10]) == [0] * 10 and list(sot[10:20]) == [-1] * 10 and list(sot[20:]) == [1] * 3
    covered = [lo + i for i, x in enumerate(sot) if x >= 0]
    assert covered == list(range(20, 30)) + list(range(40, 43))     # every written token of a turned run, once


def test_written_seg_of_tok_clips_to_the_segment_end():
    lo, sot = written_seg_of_tok([(0, 10, 4), (0, 14, 4)], [0], [16])
    assert lo == 10 and list(sot) == [0] * 6


def test_written_seg_of_tok_nothing_turns():
    assert len(written_seg_of_tok([(0, 0, 4), (0, 4, 1)], [-1], [5])[1]) == 0
    assert len(written_seg_of_tok([], [0, 1], [4, 8])[1]) == 0


def test_chunk_arrays_per_chunk():
    """chunk_ntok / dst_tok / chunk_seg from the matched chunks: tail chunks keep their size, a segment at 0 gets -1, and
    together the chunks cover every written token exactly once"""
    plans = plan_segments(200, [(100, 170), (0, 9), (30, 64)], CS * 4)        # chunks of 16 tokens
    hits = {0: 1, 1: 3, 2: 5}                                               # chunks matched per plan
    placed = [(r, p.start + k * 16, min(16, p.end - p.start - k * 16)) for r, p in enumerate(plans)
              for k in range(min(hits[r], p.n_chunks))]
    ntok, dst, seg = chunk_arrays(placed, [-1, 0, 1])
    assert ntok.dtype == np.int32 and dst.dtype == np.int64 and seg.dtype == np.int32
    assert list(ntok) == [9, 16, 16, 2, 16, 16, 16, 16, 6]
    assert list(dst) == [0, 30, 46, 62, 100, 116, 132, 148, 164]
    assert list(seg) == [-1, 0, 0, 0, 1, 1, 1, 1, 1]
    toks = np.concatenate([np.arange(t, t + n) for t, n in zip(dst, ntok)])
    assert len(np.unique(toks)) == len(toks)
    assert set(toks) == set(range(0, 9)) | set(range(30, 64)) | set(range(100, 170))


class _FakeTier:
    """a tier holding some keys, serving get_kv_layerwise_runs up to each run's first miss, and recording what it served"""

    def __init__(self, held):
        self.held, self.served = set(held), []

    def supports_layerwise_get(self):
        return True

    def get_kv_layerwise_runs(self, runs, dst, chunk_size, rotation=None):
        hits = []
        for keys, fb, tok0 in runs:
            assert fb is None
            n = 0
            while n < len(keys) and keys[n] in self.held:
                self.served.append((keys[n], tok0 + n * chunk_size))
                n += 1
            hits.append((n, 0))
        return hits, _FakeUpload(sum(h for h, _ in hits))


class _FakeUpload:
    def __init__(self, n):
        self.n = n


class _Dst:
    L = 2


def test_hybrid_splits_runs_into_local_and_remote_parts():
    from lmcache_b200.storage_backend.hybrid_backend import LMCHybridBackend
    hy = object.__new__(LMCHybridBackend)
    hy.local_store = _FakeTier({"a0", "a1", "b0", "da3"})
    hy.remote_store = _FakeTier({"a2", "a3", "b1", "b2", "da4", "c0"})
    runs = [(["a0", "a1", "a2", "a3", "a4", "a5"], ["da0", "da1", "da2", "da3", "da4", "da5"], 10),
            (["b0", "b1", "b2"], None, 100),
            (["c0", "c1"], ["dc0", "dc1"], 200)]
    hits, _ = hy.get_kv_layerwise_runs(runs, _Dst(), 4)
    # prefix keys: local, then remote from the local miss; derived keys from the first prefix miss, local then remote
    assert hits == [(4, 1), (3, 0), (1, 0)]
    assert hy.local_store.served == [("a0", 10), ("a1", 14), ("b0", 100)]
    assert hy.remote_store.served == [("a2", 18), ("a3", 22), ("b1", 104), ("b2", 108), ("c0", 200), ("da4", 26)]
    toks = [t for _, t in hy.local_store.served + hy.remote_store.served]
    assert len(toks) == len(set(toks))                                       # each chunk in exactly one part


def test_rest_runs():
    assert rest_runs([(["a", "b", "c"], 0), (["d"], 50)], [1, 1], 8) == [(["b", "c"], 8), ([], 58)]
