"""CPU: the plan of a segment store (store_paged_segments / store_segments) -- the skip scan over prefix-keyed and
derived-keyed hits, the staged token ranges, seg_of_tok and the shifts -- the derived digests that key a segment stored
from inside a longer prompt, and the bound of a key turned twice (by -s at store, by s' at retrieve)."""
import hashlib
import itertools

import numpy as np
import pytest
import torch

from rope_ref import partner, rotate
from rope_twice_ref import tolerance_twice

from lmcache_b200.rope import (DERIVED_TAG, derived_digest, plan_segment_store, plan_segments, skip_chunks)
from lmcache_b200.utils import CacheEngineKey


# ---------------------------------------------------------------------------------------------- skip scan
@pytest.mark.parametrize("n", [1, 2, 4])
def test_skip_scan_every_hit_pattern(n):
    """prefix hits end the first walk at their first miss; derived hits continue from there to their own first miss"""
    for pre in itertools.product([False, True], repeat=n):
        for der in itertools.product([False, True], repeat=n):
            asked = []

            def has(kind, hits):
                def f(i):
                    asked.append((kind, i))
                    return hits[i]
                return f
            p, d = skip_chunks(n, has("p", pre), has("d", der))
            want_p = next((i for i in range(n) if not pre[i]), n)
            want_d = next((i for i in range(want_p, n) if not der[i]), n) - want_p
            assert (p, d) == (want_p, want_d), (pre, der)
            # only what the walk needs is looked up: prefix keys up to their first miss, then derived keys
            assert asked == [("p", i) for i in range(min(want_p + 1, n))] + \
                [("d", i) for i in range(want_p, min(want_p + want_d + 1, n))]


# ---------------------------------------------------------------------------------------------- the plan
def test_plan_stages_the_chunks_after_the_hits():
    cs = 64
    plans = plan_segments(1000, [(300, 500), (30, 222), (600, 601), (700, 900)], cs)
    assert [p.start for p in plans] == [30, 300, 600, 700]
    hits = [(1, 0), (0, 2), (0, 0), (1, 3)]        # the last: every chunk hit (prefix 1, derived 3 > its 4 - 1)
    runs, rows, sot, shifts = plan_segment_store(plans, hits, cs)
    # segment 30..222: chunk 0 hit under its prefix key -> tokens 94..222; 300..500: chunks 0-1 derived -> 428..500;
    # 600..601: everything; 700..900 (4 chunks): nothing
    assert [(r.plan.start, r.first, r.prefix_hits, r.begin, r.stage_begin, r.n_tok, r.row) for r in runs] == [
        (30, 1, 1, 94, 0, 128, 0), (300, 2, 0, 428, 128, 72, 1), (600, 0, 0, 600, 200, 1, 2)]
    assert rows == list(range(94, 222)) + list(range(428, 500)) + [600]
    assert sot == [0] * 128 + [1] * 72 + [2]
    assert -1 not in sot                            # every staged token is stored
    assert shifts == [-30, -300, -600]


def test_plan_of_nothing_to_store_and_the_start_0_refusal():
    plans = plan_segments(300, [(10, 100), (100, 300)], 64)
    assert plan_segment_store(plans, [(2, 0), (1, 3)], 64) == ([], [], [], [])
    with pytest.raises(ValueError, match="token 0"):
        plan_segment_store(plan_segments(300, [(0, 100)], 64), [(0, 0)], 64)


def test_plan_runs_are_chunk_aligned_to_their_segment():
    """the staged part of a segment starts on one of its own chunk boundaries, so its chunks are those of a store of
    the segment alone"""
    cs = 16
    rng = np.random.default_rng(1)
    for _ in range(200):
        cuts = sorted(rng.choice(np.arange(1, 400), size=6, replace=False).tolist())
        segs = [(cuts[i], cuts[i + 1]) for i in range(0, 6, 2)]
        plans = plan_segments(400, segs, cs)
        hits = [(int(rng.integers(0, 3)), int(rng.integers(0, 3))) for _ in plans]
        runs, rows, sot, shifts = plan_segment_store(plans, hits, cs)
        assert len(rows) == len(sot) == sum(r.n_tok for r in runs)
        for r in runs:
            assert (r.begin - r.plan.start) % cs == 0 and r.begin + r.n_tok == r.plan.end
            assert rows[r.stage_begin:r.stage_begin + r.n_tok] == list(range(r.begin, r.plan.end))
            assert shifts[r.row] == -r.plan.start
            assert set(sot[r.stage_begin:r.stage_begin + r.n_tok]) == {r.row}


# ---------------------------------------------------------------------------------------------- derived digests
def test_derived_digests():
    chain, h = [], ""
    for i in range(64):
        h = hashlib.sha256(h.encode() + bytes([i]) * 8).hexdigest()
        chain.append(h)
    derived = [derived_digest(c) for c in chain]
    assert derived == [derived_digest(c) for c in chain]                       # deterministic
    assert all(len(d) == 64 and int(d, 16) >= 0 and d == d.lower() for d in derived)
    assert len(set(derived)) == len(derived) and not set(derived) & set(chain)
    assert derived[5] == hashlib.sha256(DERIVED_TAG + bytes.fromhex(chain[5])).hexdigest()
    # derived of derived is yet another digest: the namespace does not fold back onto the prefix one
    assert derived_digest(derived[0]) not in set(chain) | set(derived)
    # a derived key string has the shape and length of the prefix key it stands beside
    model = "meta-llama/Meta-Llama-3.1-70B-Instruct"
    for c, d in zip(chain, derived):
        key = CacheEngineKey("huggingface", model, 1024, 1023, d).to_string()
        assert len(key) == len(CacheEngineKey("huggingface", model, 1024, 1023, c).to_string()) <= 150, len(key)
        assert CacheEngineKey.from_string(key).chunk_hash == d


# ---------------------------------------------------------------------------------------------- two turns
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("style", ["neox", "gptj"])
def test_turn_back_and_forth_within_the_two_rounding_bound(dtype, style):
    """turned by -s and rounded, then by s' and rounded: within tolerance_twice of one turn by s' - s"""
    name = {torch.bfloat16: "bfloat16", torch.float16: "float16"}[dtype]
    D, rd, off = 128, 96, 16
    inv = (1.0 / (10000.0 ** (torch.arange(0, rd, 2, dtype=torch.float) / rd))).numpy()
    rng = np.random.default_rng(3)
    x = torch.from_numpy(rng.standard_normal((512, 4, D)) * 4).to(dtype).double().numpy()
    p = partner(rd, style, off, D)
    r = lambda a: torch.from_numpy(a).to(dtype).double().numpy()      # noqa: E731 -- round to the dtype
    for s, s2 in ((1, 1), (255, 4096), (4096, 17), (65535, 65535), (70, 65535)):
        once = r(rotate(x, -s, inv, rd, style, off))
        twice = r(rotate(once, s2, inv, rd, style, off))
        want = r(rotate(x, s2 - s, inv, rd, style, off))
        tol = tolerance_twice(want, twice, x, x[..., p], name)
        err = np.abs(twice - want)
        assert (err <= tol).all(), (s, s2, float((err - tol).max()))
        assert np.array_equal(twice[..., :off], x[..., :off]) and np.array_equal(twice[..., off + rd:], x[..., off + rd:])
