"""Non-prefix KV reuse: the rotation a retrieved segment's keys need, and the plan of a segment retrieve.

vLLM caches K after the rotary embedding.  A document prefilled alone at positions 0..n-1 holds R(i)·k_i; served at
positions s..s+n-1 its keys must be R(s + i)·k_i = R(s)·(R(i)·k_i), so each retrieved key row is rotated by s·θ_j
(b200kv_rope_shift).  V carries no position.  A document stored as its own prompt is keyed by the hash chain of its own
tokens, which is exactly what a segment lookup recomputes from those tokens inside a longer request: existing caches
serve as segments without being stored again."""
from __future__ import annotations

import ctypes
from typing import List, NamedTuple, Sequence, Tuple

import torch

from lmcache_b200 import _native as N

STYLES = {"neox": 0, "gptj": 1}


class RopeSpec:
    """The rotary embedding of the model whose keys are shifted: `rotary_dim` channels from channel `offset` of every
    key head (offset 512, rotary_dim 64, style "gptj" for the decoupled RoPE part of DeepSeek's 576-channel latent),
    paired as in vLLM's RotaryEmbedding -- "neox": (d, d + rotary_dim/2), "gptj": (2d, 2d + 1) -- and turned by
    position · inv_freq[j].  inv_freq: float32 [rotary_dim/2], as vLLM's rotary_emb computes it (any scaling that only
    rescales frequencies: plain theta, Llama-3's, YaRN's).  Dynamic NTK, whose frequencies depend on the sequence
    length, cannot be expressed."""

    def __init__(self, rotary_dim: int, inv_freq: torch.Tensor, style: str = "neox", offset: int = 0):
        if isinstance(rotary_dim, bool) or not isinstance(rotary_dim, int) or rotary_dim <= 0 or rotary_dim % 2:
            raise ValueError(f"rotary_dim must be a positive even int, got {rotary_dim!r}")
        if style not in STYLES:
            raise ValueError(f"style must be one of {sorted(STYLES)}, got {style!r}")
        if isinstance(offset, bool) or not isinstance(offset, int) or offset < 0:
            raise ValueError(f"offset must be a non-negative int, got {offset!r}")
        if not isinstance(inv_freq, torch.Tensor) or inv_freq.dtype != torch.float32 or \
                tuple(inv_freq.shape) != (rotary_dim // 2,):
            raise ValueError(f"inv_freq must be a float32 tensor of rotary_dim/2 = {rotary_dim // 2} frequencies")
        self.rotary_dim = rotary_dim
        self.inv_freq = inv_freq
        self.style = style
        self.offset = offset

    @staticmethod
    def from_base(rotary_dim: int, base: float, style: str = "neox", offset: int = 0) -> "RopeSpec":
        """inv_freq = base ** (-arange(0, rotary_dim, 2) / rotary_dim) in float32: vLLM's RotaryEmbedding._compute_inv_freq"""
        inv = 1.0 / (base ** (torch.arange(0, rotary_dim, 2, dtype=torch.float) / rotary_dim))
        return RopeSpec(rotary_dim, inv, style, offset)

    def check(self, D: int) -> None:
        """ValueError unless channels [offset, offset + rotary_dim) lie in a key head of D channels"""
        if self.offset + self.rotary_dim > D:
            raise ValueError(f"rotary channels [{self.offset}, {self.offset + self.rotary_dim}) do not fit a key head of "
                             f"{D} channels")

    def __repr__(self) -> str:
        return f"RopeSpec(rotary_dim={self.rotary_dim}, style={self.style!r}, offset={self.offset})"


class SegmentPlan(NamedTuple):
    """One segment [start, end) of a request: its tokens are hashed as their own sequence, tokens [hash_begin,
    hash_begin + end - start) of the concatenated hash input; its digests are [chunk_begin, chunk_begin + n_chunks) of
    the one hash launch; its KV lands at destination token `start` and its keys turn by `shift` positions."""
    index: int               # position in the caller's list
    start: int
    end: int
    shift: int
    hash_begin: int
    chunk_begin: int
    n_chunks: int

    def chunk_bounds(self, chunk_size: int) -> List[Tuple[int, int]]:
        """request tokens of each chunk: aligned to the segment's own start, the last one possibly short, as a store
        of the segment alone made them"""
        return [(a, min(a + chunk_size, self.end)) for a in range(self.start, self.end, chunk_size)]


def plan_segments(n_tokens: int, segments: Sequence[Tuple[int, int]], chunk_size: int) -> List[SegmentPlan]:
    """The plan of a segment retrieve, in request order (by start).  ValueError, before anything is enqueued, for an
    empty segment, one outside [0, n_tokens), and overlapping segments."""
    if chunk_size <= 0:
        raise ValueError(f"chunk_size must be positive, got {chunk_size}")
    segs = []
    for i, seg in enumerate(segments):
        try:
            a, b = (int(x) for x in seg)
        except (TypeError, ValueError):
            raise ValueError(f"segment {i} must be a (start, end) pair, got {seg!r}") from None
        if a >= b:
            raise ValueError(f"segment {i} ({a}, {b}) is empty")
        if a < 0 or b > n_tokens:
            raise ValueError(f"segment {i} ({a}, {b}) lies outside the request's tokens [0, {n_tokens})")
        segs.append((a, b, i))
    segs.sort()
    for (a0, b0, i0), (a1, b1, i1) in zip(segs, segs[1:]):
        if a1 < b0:
            raise ValueError(f"segments {i0} ({a0}, {b0}) and {i1} ({a1}, {b1}) overlap")
    out, h, c = [], 0, 0
    for a, b, i in segs:
        n = (b - a + chunk_size - 1) // chunk_size
        out.append(SegmentPlan(i, a, b, a, h, c, n))
        h += b - a
        c += n
    return out


def hash_input(tokens: torch.Tensor, plans: Sequence[SegmentPlan]) -> Tuple[torch.Tensor, List[int]]:
    """The tokens of every segment back to back and the sequence offsets of one b200kv_sha256_chain launch"""
    toks = torch.cat([tokens[p.start:p.end] for p in plans])
    return toks, [p.hash_begin for p in plans] + [len(toks)]


def seg_of_tok(n_tokens: int, written: Sequence[Tuple[SegmentPlan, int]]) -> Tuple[List[int], int, int, List[int]]:
    """The shift's arguments for the tokens written, (plan, tokens written from its start) per segment: (seg_of_tok of
    tokens [lo, hi), lo, hi, shift per table row).  A segment at start 0, or with nothing written, has no table row
    and its tokens stay -1.  hi == lo: nothing to rotate."""
    shifts, rows = [], []
    for p, n in written:
        if n > 0 and p.shift != 0:
            rows.append((p.start, p.start + n, len(shifts)))
            shifts.append(p.shift)
    if not rows:
        return [], 0, 0, []
    lo, hi = min(r[0] for r in rows), max(r[1] for r in rows)
    sot = [-1] * (hi - lo)
    for a, b, k in rows:
        sot[a - lo:b - lo] = [k] * (b - a)
    return sot, lo, hi, shifts


def rope_shift(view, tok_begin: int, seg: torch.Tensor, shifts: torch.Tensor, rope: RopeSpec) -> None:
    """Rotate the keys of tokens [tok_begin, tok_begin + len(seg)) of a KvView on the current stream: one table launch
    (b200kv_rope_table) and one shift launch (b200kv_rope_shift).  seg: int32 CUDA, a row of the table per token or -1;
    shifts: int64 CUDA, one per table row."""
    dev = view.device
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        inv = rope.inv_freq.to(dev, non_blocking=True)
        table = torch.empty(shifts.numel(), rope.rotary_dim // 2, 2, dtype=torch.float32, device=dev)
        N.check(N.lib().b200kv_rope_table(ctypes.c_void_p(shifts.data_ptr()), shifts.numel(),
                                          ctypes.c_void_p(inv.data_ptr()), rope.rotary_dim,
                                          ctypes.c_void_p(table.data_ptr()), st), "rope_table")
        N.check(N.lib().b200kv_rope_shift(ctypes.byref(view.desc), tok_begin, seg.numel(),
                                          ctypes.c_void_p(seg.data_ptr()), ctypes.c_void_p(table.data_ptr()),
                                          rope.rotary_dim, rope.offset, STYLES[rope.style], st), "rope_shift")
