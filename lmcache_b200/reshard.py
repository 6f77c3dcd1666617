"""Head arithmetic of tensor-parallel layouts: which stored shards of another layout make up this rank's KV heads.

Layout W (a TP world size) stores rank r's chunk as the model's KV heads [r * Hg / W, (r + 1) * Hg / W) under the key
(fmt, model, W, r, chunk hash); Hg is the model's KV head count.  The hash chain depends on the tokens alone, so one
chunk has the same hash under every rank and every layout.  This module is the one place that knows that rule: the
engine and the storage tiers ask it and do not restate it."""
from __future__ import annotations

from typing import List, NamedTuple, Optional


class Shard(NamedTuple):
    """The part of source rank `rank`'s container that a destination rank needs: its heads
    [src_head0, src_head0 + n_heads), written at the destination's head dst_head0."""
    rank: int
    src_head0: int
    n_heads: int
    dst_head0: int


def _divides(Hg: int, W: int) -> bool:
    return Hg > 0 and W > 0 and Hg % W == 0


def source_shards(Hg: int, W_src: int, W_dst: int, r_dst: int) -> List[Shard]:
    """The shards of layout W_src that rank r_dst of layout W_dst is made of, in head order: plain interval intersection
    of the two ranks' head ranges.  W_src < W_dst gives one container, partly decoded; W_src > W_dst gives W_src / W_dst
    containers, each whole.  [] when either size does not divide Hg (vLLM replicates KV heads when TP exceeds them:
    not a layout this module describes) or r_dst is not a rank of W_dst."""
    if not (_divides(Hg, W_src) and _divides(Hg, W_dst)) or not 0 <= r_dst < W_dst:
        return []
    hs, hd = Hg // W_src, Hg // W_dst
    lo, hi = r_dst * hd, (r_dst + 1) * hd
    out = []
    for r in range(lo // hs, (hi - 1) // hs + 1):
        a, b = max(lo, r * hs), min(hi, (r + 1) * hs)
        out.append(Shard(r, a - r * hs, b - a, a - lo))
    return out


def first_source_rank(W_src: int, W_dst: int, r_dst: int) -> Optional[int]:
    """The source rank holding rank r_dst's first head, whatever Hg is (as long as both sizes divide it): the rank whose
    container tells a replica that knows no geometry yet what Hg is.  None when r_dst is not a rank of W_dst."""
    if W_src <= 0 or not 0 <= r_dst < W_dst:
        return None
    return r_dst * W_src // W_dst
