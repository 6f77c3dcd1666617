"""CPU: the host side of CacheBlend's selective recomputation (lmcache_b200/blend.py) -- BlendSpec's rules, the k_j
arithmetic, the rows, candidates and forced rows of a blended prefill across several check layers (driven by the
statement of the select in tests/blend_ref.py), and the refusals that run before anything is enqueued."""
import math

import numpy as np
import pytest
import torch

import blend_ref as R
from lmcache_b200.blend import (BlendSpec, check_blend_args, check_blend_dtype, check_sizes, fresh_row_stride)


@pytest.mark.parametrize("layers,ratios", [([], []), ([1], []), ([1, 2], [0.5]), ([2, 1], [0.5, 0.1]),
                                           ([1, 1], [0.5, 0.1]), ([-1], [0.1]), ([1.0], [0.1]), ([True], [0.1]),
                                           ([1], [1.5]), ([1], [-0.1]), ([1], [float("nan")]), ([1, 2], [0.1, 0.2]),
                                           ([1], ["0.1"])])
def test_spec_refusals(layers, ratios):
    with pytest.raises(ValueError):
        BlendSpec(layers, ratios)


def test_spec_accepts():
    s = BlendSpec([1], [0.15])
    assert s.check_layers == [1] and s.ratios == [0.15]
    s = BlendSpec((1, 5, 9), (1, 0.5, 0.5))
    assert s.check_layers == [1, 5, 9] and s.ratios == [1.0, 0.5, 0.5]
    BlendSpec([0], [0])


def test_budgets():
    assert BlendSpec([1], [0.15]).budgets(100) == [15]                # the decimal ratio: no spurious 16 or 5
    assert BlendSpec([1], [0.1]).budgets(40) == [4]
    assert BlendSpec([1], [0.15]).budgets(1) == [1]                   # ceil at small R
    assert BlendSpec([1], [0.15]).budgets(7) == [2]
    assert BlendSpec([1], [0.0]).budgets(50) == [0]
    assert BlendSpec([1], [1.0]).budgets(50) == [50]
    assert BlendSpec([1], [0.15]).budgets(0) == [0]
    assert BlendSpec([1, 2, 3], [1.0, 0.3, 0.0]).budgets(10) == [10, 3, 0]
    assert BlendSpec([1, 2], [0.5, 0.5]).budgets(3) == [2, 2]
    for R_ in range(0, 300, 7):
        for rs in ([0.15], [0.5, 0.15], [0.33, 0.33, 0.05], [1.0, 0.01]):
            assert BlendSpec(list(range(1, len(rs) + 1)), rs).budgets(R_) == R.budgets(rs, R_), (R_, rs)
            for k in BlendSpec(list(range(1, len(rs) + 1)), rs).budgets(R_):
                assert 0 <= k <= R_


def test_check_sizes():
    assert check_sizes(BlendSpec([1, 3], [0.3, 0.1]), 50, 40) == [(50, 12, 22), (22, 4, 14)]
    assert check_sizes(BlendSpec([1], [0.0]), 10, 10) == [(10, 0, 0)]
    assert check_sizes(BlendSpec([1], [1.0]), 10, 0) == [(10, 0, 10)]


@pytest.mark.parametrize("seed", range(6))
def test_walk_bookkeeping(seed):
    """several checks driven by the statement: each check sees the rows the previous one kept; forced (not retrieved)
    tokens are always kept, first, in request order; the sizes are check_sizes' and known before any deviation"""
    rng = np.random.default_rng(seed)
    T = int(rng.integers(1, 400))
    mask = rng.random(T) < rng.random()
    ratios = sorted(rng.random(int(rng.integers(1, 4))).tolist(), reverse=True)
    if seed == 0:
        ratios = [1.0, 0.0]
    spec = BlendSpec(list(range(1, len(ratios) + 1)), ratios)
    sizes = check_sizes(spec, T, int(mask.sum()))
    forced = np.nonzero(~mask)[0]
    rows = np.arange(T)
    devs = []
    for j, (n_in, k, n_out) in enumerate(sizes):
        assert len(rows) == n_in
        dev = rng.random(n_in).astype(np.float32)
        dev[rng.random(n_in) < 0.1] = np.nan
        devs.append(dev)
        cand = mask[rows]
        assert int((~cand).sum()) == len(forced)
        sel = R.select(dev, cand, k)
        assert len(sel) == n_out
        assert np.array_equal(rows[sel[:len(forced)]], forced)
        picked = rows[sel[len(forced):]]
        assert mask[picked].all() and np.all(np.diff(sel[len(forced):]) > 0)
        # the k largest of the candidates: every candidate left out ranks below every one taken
        key = np.where(np.isnan(dev), np.inf, dev)
        out = np.setdiff1d(np.nonzero(cand)[0], sel)
        if len(out) and k:
            taken = sel[len(forced):]
            worst = min(taken, key=lambda i: (key[i], -i))
            assert all((key[o], -o) < (key[worst], -worst) for o in out)
        rows = rows[sel]
    walked = R.walk(mask, ratios, devs)
    assert np.array_equal(walked[-1], rows)


def test_select_statement_edges():
    assert R.select([1.0], [1], 1).tolist() == [0]
    assert R.select([1.0], [0], 1).tolist() == [0]
    assert R.select([1.0, 1.0, 1.0], [1, 1, 1], 2).tolist() == [0, 1]                  # ties: the lower rows
    assert R.select([0.0, np.nan, np.inf, 5.0], [1, 1, 1, 1], 2).tolist() == [1, 2]     # NaN as +inf, then row order
    assert R.select([3.0, 2.0, 1.0], [1, 0, 1], 1).tolist() == [1, 0]                  # forced first
    assert R.select([3.0, 2.0, 1.0], [1, 0, 1], 0).tolist() == [1]
    assert R.select([3.0, 2.0, 1.0], [1, 1, 1], 9).tolist() == [0, 1, 2]


def test_refusals():
    with pytest.raises(TypeError):
        check_blend_dtype(torch.float8_e4m3fn)
    with pytest.raises(TypeError):
        check_blend_dtype(torch.uint8)
    check_blend_dtype(torch.bfloat16)
    check_blend_dtype(torch.float16)
    spec = BlendSpec([1], [0.15])
    mask = torch.zeros(10, dtype=torch.bool)
    check_blend_args(spec, 4, 10, mask)
    for args in ((spec, 4, 11, mask), (BlendSpec([4], [0.1]), 4, 10, mask), ("spec", 4, 10, mask),
                 (spec, 4, 10, mask.to(torch.uint8)), (spec, 4, 10, mask.view(2, 5))):
        with pytest.raises(ValueError):
            check_blend_args(*args)
    dev = torch.device("cpu")
    f = torch.zeros(5, 2, 64, dtype=torch.bfloat16)
    assert fresh_row_stride(f, 5, 128, torch.bfloat16, dev) == 128
    assert fresh_row_stride(f.view(5, 128), 5, 128, torch.bfloat16, dev) == 128
    wide = torch.zeros(5, 131, dtype=torch.bfloat16)
    assert fresh_row_stride(wide[:, :128], 5, 128, torch.bfloat16, dev) == 131
    assert fresh_row_stride(wide[:1, :128], 1, 128, torch.bfloat16, dev) == 128
    for bad in (f[:4], f.to(torch.float16), torch.zeros(5, 2, 63, dtype=torch.bfloat16), f.transpose(1, 2),
                torch.zeros(5, dtype=torch.bfloat16), "f"):
        with pytest.raises(ValueError):
            fresh_row_stride(bad, 5, 128, torch.bfloat16, dev)
    with pytest.raises(ValueError):
        fresh_row_stride(f, 5, 128, torch.bfloat16, torch.device("cuda", 0))


def test_budget_ceiling_is_exact():
    for R_ in range(1, 200):
        for r in (0.05, 0.1, 0.15, 0.3, 0.7):
            k = BlendSpec([1], [r]).budgets(R_)[0]
            assert k == math.ceil(round(r * R_, 9))
