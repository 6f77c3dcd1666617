"""CPU: the host side of a batched blend (lmcache_b200/blend.py) -- the per-request arithmetic of every check (segment
starts, budgets, output starts, lens_at / cu_rows_at) against check_sizes and against tests/blend_ref.py's walk of each
request alone, and the refusals of LMCacheEngine.blend_paged_batch that run before anything is enqueued."""
import types

import numpy as np
import pytest
import torch

import blend_ref as R
from lmcache_b200.blend import (BatchBlendPlan, BlendSpec, batch_checks, check_blend_batch_args, check_sizes)


def _view(L=6):
    """what the plan reads of a view before any check: its device and layer count"""
    return types.SimpleNamespace(device=torch.device("cpu"), L=L, H=2, D=64, dtype=torch.bfloat16)


def _masks(rng, shapes):
    """one ret_mask per request: 'none' retrieved nothing, 'all' everything, 'one' is a 1-token request, an int a
    random request of that many tokens"""
    out = []
    for s in shapes:
        if s == "none":
            out.append(torch.zeros(int(rng.integers(1, 50)), dtype=torch.bool))
        elif s == "all":
            out.append(torch.ones(int(rng.integers(1, 50)), dtype=torch.bool))
        elif s == "one":
            out.append(torch.tensor([bool(rng.integers(0, 2))]))
        else:
            out.append(torch.from_numpy(rng.random(s) < rng.random()))
    return out


def test_batch_checks_arithmetic():
    spec = BlendSpec([1, 3], [0.5, 0.1])
    n, r = [10, 1, 40, 7], [0, 1, 30, 7]
    got = batch_checks(spec, n, r)
    # request sizes by hand: (n_in, k, n_out) per check
    #   10 tokens, none retrieved: (10, 0, 10), (10, 0, 10); 1 token retrieved: (1, 1, 1), (1, 1, 1)
    #   40 tokens, 30 retrieved: (40, 15, 25), (25, 3, 13); 7 of 7 retrieved: (7, 4, 4), (4, 1, 1)
    assert got[0].seg == [0, 10, 11, 51, 58] and got[0].k == [0, 1, 15, 4] and got[0].out == [0, 10, 11, 36, 40]
    assert got[1].seg == got[0].out and got[1].k == [0, 1, 3, 1] and got[1].out == [0, 10, 11, 24, 25]
    for j, c in enumerate(got):
        for b in range(len(n)):
            n_in, k, n_out = check_sizes(spec, n[b], r[b])[j]
            assert c.seg[b + 1] - c.seg[b] == n_in and c.k[b] == k and c.out[b + 1] - c.out[b] == n_out


@pytest.mark.parametrize("seed", range(5))
def test_plan_lens_and_cu_rows(seed):
    rng = np.random.default_rng(seed)
    masks = _masks(rng, ["none", "one", 300, "all", 17, "one", "none"])
    spec = BlendSpec([1, 2, 4], [0.6, 0.3, 0.05])
    plan = BatchBlendPlan(_view(), masks, spec)
    assert plan.B == len(masks) and plan.n_tokens == sum(m.numel() for m in masks)
    assert plan.lens_at(0) == plan.lens_at(1) == [m.numel() for m in masks]
    assert torch.equal(plan.cu_rows_at(1), torch.tensor(plan.checks[0].seg, dtype=torch.int32))
    assert plan.cu_rows_at(0).dtype == torch.int32 and plan.cu_rows_at(0).numel() == len(masks) + 1
    for j, c in enumerate(plan.checks):
        assert torch.equal(plan._seg[j], torch.tensor(c.seg)) and torch.equal(plan._k[j], torch.tensor(c.k))
        assert torch.equal(plan._cu[j + 1], torch.tensor(c.out, dtype=torch.int32))
        for b, m in enumerate(masks):
            n_in, k, n_out = check_sizes(spec, m.numel(), int(m.sum()))[j]
            assert (c.seg[b + 1] - c.seg[b], c.k[b], c.out[b + 1] - c.out[b]) == (n_in, k, n_out)
    assert torch.equal(plan._mask, torch.cat(masks).to(torch.uint8))
    with pytest.raises(ValueError):
        plan.lens_at(2)                                   # past a check not yet run
    with pytest.raises(ValueError):
        plan.cu_rows_at(6)


@pytest.mark.parametrize("seed", range(6))
def test_segmented_walk_matches_each_request_alone(seed):
    """a batch walked with the per-segment statement of the select, on the plan's segment starts and budgets, is the
    concatenation of blend_ref.walk of each request alone, offset by the request's first token"""
    rng = np.random.default_rng(100 + seed)
    masks = _masks(rng, ["one", int(rng.integers(1, 200)), "none", "all", int(rng.integers(1, 200)), "one"])
    ratios = sorted(rng.random(int(rng.integers(1, 4))).tolist(), reverse=True)
    spec = BlendSpec(list(range(1, len(ratios) + 1)), ratios)
    checks = batch_checks(spec, [m.numel() for m in masks], [int(m.sum()) for m in masks])
    starts = np.cumsum([0] + [m.numel() for m in masks])
    flat = torch.cat(masks).numpy()
    rows = np.arange(len(flat))
    devs = [[] for _ in masks]
    for c in checks:
        dev = rng.random(len(rows)).astype(np.float32)
        dev[rng.random(len(rows)) < 0.1] = np.nan
        dev[rng.random(len(rows)) < 0.1] = 0.5                # ties
        sel = []
        for b in range(len(masks)):
            a, e = c.seg[b], c.seg[b + 1]
            devs[b].append(dev[a:e])
            sel.append(a + R.select(dev[a:e], flat[rows[a:e]], c.k[b]))
            assert len(sel[-1]) == c.out[b + 1] - c.out[b]
        rows = rows[np.concatenate(sel)]
        assert len(rows) == c.out[-1]
    want = np.concatenate([starts[b] + R.walk(m.numpy(), ratios, devs[b])[-1] for b, m in enumerate(masks)])
    assert np.array_equal(rows, want)


def test_batch_args_refusals():
    spec = BlendSpec([1], [0.15])
    m = [torch.zeros(4, dtype=torch.bool), torch.ones(6, dtype=torch.bool)]
    check_blend_batch_args(spec, 4, 10, m)
    check_blend_batch_args(spec, 4, 10, tuple(m))
    for args in ((spec, 4, 11, m), (spec, 4, 10, []), (spec, 4, 10, m[0]), (spec, 4, 10, [m[0], m[1].to(torch.uint8)]),
                 (spec, 4, 10, [m[0], m[1].view(2, 3)]), (BlendSpec([4], [0.1]), 4, 10, m), ("spec", 4, 10, m),
                 (spec, 4, 10, [m[0], "mask"]), (spec, 4, 10, None)):
        with pytest.raises(ValueError):
            check_blend_batch_args(*args)


def test_engine_refusals_before_anything():
    """LMCacheEngine.blend_paged_batch's refusals need no GPU: they run on the arguments alone"""
    from lmcache_b200.cache_engine import LMCacheEngine
    eng = types.SimpleNamespace(metadata=types.SimpleNamespace(fmt="vllm"), _mla=False)
    eng._check_kind = lambda kv, what: LMCacheEngine._check_kind(eng, kv, what)
    eng._first = lambda kv: LMCacheEngine._first(eng, kv)
    caches = [(torch.zeros(2, 16, 2, 64, dtype=torch.bfloat16),) * 2 for _ in range(4)]
    slots = torch.arange(10)
    m = [torch.zeros(4, dtype=torch.bool), torch.ones(6, dtype=torch.bool)]
    spec = BlendSpec([1], [0.1])
    for bad_spec, masks in ((spec, m[:1]), (spec, []), (spec, m[0]), (BlendSpec([4], [0.1]), m), ("x", m),
                            (spec, [m[0], m[1].to(torch.uint8)])):
        with pytest.raises(ValueError):
            LMCacheEngine.blend_paged_batch(eng, caches, slots, masks, bad_spec)
    fp8 = [tuple(t.view(torch.uint8)[..., :64].view(torch.float8_e4m3fn) for t in p) for p in caches]
    with pytest.raises(TypeError):
        LMCacheEngine.blend_paged_batch(eng, fp8, slots, m, spec)
    eng.metadata.fmt = "huggingface"
    with pytest.raises(ValueError):
        LMCacheEngine.blend_paged_batch(eng, caches, slots, m, spec)
