"""The numpy statement of the blend kernels (lmcache_b200/csrc/blend.cu) and of a blended prefill's bookkeeping.

deviation: dev[i] = sum over the H * D channels of (fresh - cached)^2, in float64 (the kernel's fp32 sum is within
summation error of it).  select: the rows with cand == 0 in row order, then the k candidate rows of largest dev in row
order, ranked by sorted(range(n), key=(-key, i)) with NaN as +inf."""
import math

import numpy as np


def deviation(fresh, cached):
    """fresh, cached: [n, H * D] (any float dtype) -> float64 [n]"""
    d = np.asarray(fresh, dtype=np.float64) - np.asarray(cached, dtype=np.float64)
    return (d * d).sum(axis=1)


def _key(v):
    v = float(v)
    return math.inf if math.isnan(v) else v


def select(dev, cand, k):
    dev, cand = np.asarray(dev), np.asarray(cand)
    n = len(dev)
    forced = [i for i in range(n) if not cand[i]]
    cands = [i for i in range(n) if cand[i]]
    if len(cands) > 4096:                                  # the same order, faster: lexsort by (-key, i)
        keys = dev[cands].astype(np.float64)
        keys = np.where(np.isnan(keys), np.inf, keys)
        idx = np.asarray(cands, dtype=np.int64)
        order = np.lexsort((idx, -keys))
        chosen = sorted(idx[order[:k]].tolist())
    else:
        chosen = sorted(sorted(cands, key=lambda i: (-_key(dev[i]), i))[:k])
    return np.asarray(forced + chosen, dtype=np.int64)


def budgets(ratios, R):
    """k_j = min(ceil(r_j * R), k_{j-1}), k_{-1} = R, with r_j the decimal the float prints as"""
    from fractions import Fraction
    out, prev = [], R
    for r in ratios:
        prev = min(math.ceil(Fraction(repr(float(r))) * R), prev)
        out.append(prev)
    return out


def walk(ret_mask, ratios, devs):
    """The tokens computed after each check of a blended prefill whose check j sees deviations devs[j] (indexed by the
    rows computed at that check): a list of int64 token arrays, one per check"""
    ret_mask = np.asarray(ret_mask, dtype=bool)
    rows = np.arange(len(ret_mask))
    out = []
    for k, dev in zip(budgets(ratios, int(ret_mask.sum())), devs):
        sel = select(dev, ret_mask[rows], k)
        rows = rows[sel]
        out.append(rows)
    return out
