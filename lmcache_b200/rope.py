"""Non-prefix KV reuse: the rotation a retrieved segment's keys need, and the plans of a segment retrieve and store.

vLLM caches K after the rotary embedding.  A document prefilled alone at positions 0..n-1 holds R(i)·k_i; served at
positions s..s+n-1 its keys must be R(s + i)·k_i = R(s)·(R(i)·k_i), so each retrieved key row is rotated by s·θ_j
(b200kv_rope_shift).  V carries no position.  A document stored as its own prompt is keyed by the hash chain of its own
tokens, which is exactly what a segment lookup recomputes from those tokens inside a longer request: existing caches
serve as segments without being stored again.

A document stored from position s > 0 of a longer prompt is turned back by -s (b200kv_pack_chunks_rope), so its keys
are those of position 0 on.  Its KV still attended to the tokens before s, which a prefill of the document alone did
not: it is keyed in a namespace of its own (derived_digest), which retrieve() never looks up.  A segment lookup
continues there from the first chunk the prefix keys miss."""
from __future__ import annotations

import ctypes
import hashlib
from typing import Callable, List, NamedTuple, Sequence, Tuple

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


def rope_table(shifts: torch.Tensor, rope: RopeSpec) -> torch.Tensor:
    """(cos, sin) of every shift (int64 CUDA) times every frequency, float32 [n, rotary_dim/2, 2]: one
    b200kv_rope_table launch on the current stream of the shifts' device"""
    dev = shifts.device
    with torch.cuda.device(dev):
        inv = rope.inv_freq.to(dev, non_blocking=True)
        table = torch.empty(shifts.numel(), rope.rotary_dim // 2, 2, dtype=torch.float32, device=dev)
        N.check(N.lib().b200kv_rope_table(ctypes.c_void_p(shifts.data_ptr()), shifts.numel(),
                                          ctypes.c_void_p(inv.data_ptr()), rope.rotary_dim,
                                          ctypes.c_void_p(table.data_ptr()), torch.cuda.current_stream().cuda_stream),
                "rope_table")
    return table


def rope_shift(view, tok_begin: int, seg: torch.Tensor, shifts: torch.Tensor, rope: RopeSpec) -> None:
    """Rotate the keys of tokens [tok_begin, tok_begin + len(seg)) of a KvView on the current stream: one table launch
    (b200kv_rope_table) and one shift launch (b200kv_rope_shift).  seg: int32 CUDA, a row of the table per token or -1;
    shifts: int64 CUDA, one per table row."""
    dev = view.device
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        table = rope_table(shifts, rope)
        N.check(N.lib().b200kv_rope_shift(ctypes.byref(view.desc), tok_begin, seg.numel(),
                                          ctypes.c_void_p(seg.data_ptr()), ctypes.c_void_p(table.data_ptr()),
                                          rope.rotary_dim, rope.offset, STYLES[rope.style], st), "rope_shift")


def pack_rope(view, blob: torch.Tensor, seg: torch.Tensor, table: torch.Tensor, rope: RopeSpec) -> None:
    """Tokens [0, T) of a KvView packed into `blob`, one chunk of T tokens in the view's chunk layout, with the keys of
    token i turned by table row seg[i] (-1: copied) on the way: one b200kv_pack_chunks_rope launch on the current
    stream.  seg: int32 CUDA [T]; table: rope_table's."""
    t = view.ntokens
    with torch.cuda.device(view.device):
        N.check(N.lib().b200kv_pack_chunks_rope(ctypes.byref(view.desc), 0, 1, t, t, int(view.fmt == "huggingface"),
                                                ctypes.c_void_p(blob.data_ptr()), blob.numel() * blob.element_size(),
                                                ctypes.c_void_p(seg.data_ptr()), ctypes.c_void_p(table.data_ptr()),
                                                rope.rotary_dim, rope.offset, STYLES[rope.style],
                                                torch.cuda.current_stream().cuda_stream), "pack_chunks_rope")


# ---------------------------------------------------------------------------------------------- segment store
DERIVED_TAG = b"lmcache-b200 contextual kv v1\0"


def derived_digest(chunk_hash: str) -> str:
    """The key digest of a chunk of a segment stored from inside a longer prompt: sha256(DERIVED_TAG || raw chain
    digest) as 64 hex characters.  A key string keeps its shape and length, and no prefix digest equals one unless
    SHA-256 collides."""
    return hashlib.sha256(DERIVED_TAG + bytes.fromhex(chunk_hash)).hexdigest()


def skip_chunks(n_chunks: int, prefix_has: Callable[[int], bool], derived_has: Callable[[int], bool]) -> Tuple[int, int]:
    """A segment store's skip scan: (p, d) -- chunks [0, p) hit under their prefix keys (the document was stored alone),
    chunks [p, p + d) under their derived keys; the chunks from p + d on are stored.  Each lookup runs only while the
    walk is still hitting."""
    p = 0
    while p < n_chunks and prefix_has(p):
        p += 1
    d = 0
    while p + d < n_chunks and derived_has(p + d):
        d += 1
    return p, d


class StoreRun(NamedTuple):
    """The part of one segment (start > 0) that a segment store stores: chunks [first, n_chunks) of its plan, request
    tokens [begin, plan.end), staged at tokens [stage_begin, stage_begin + n_tok) of the staging blob, turned by table row
    `row` (shift -start)."""
    plan: SegmentPlan
    prefix_hits: int
    first: int
    begin: int
    stage_begin: int
    n_tok: int
    row: int


def plan_segment_store(plans: Sequence[SegmentPlan], hits: Sequence[Tuple[int, int]],
                       chunk_size: int) -> Tuple[List[StoreRun], List[int], List[int], List[int]]:
    """The staging of a segment store, from the plans of segments at start > 0 and their skip scans (p, d):
    (runs of the segments with chunks to store, the request token of every staged token, seg_of_tok of every staged
    token, the shift of every table row).  A run's tokens are staged back to back in plan order and each segment with
    something to store has one table row, shift -start; every staged token is stored, so seg_of_tok holds no -1."""
    runs: List[StoreRun] = []
    rows: List[int] = []
    sot: List[int] = []
    shifts: List[int] = []
    for p, (ph, dh) in zip(plans, hits):
        if p.start <= 0:
            raise ValueError(f"segment ({p.start}, {p.end}) starts at token 0: it is stored under its prefix keys")
        first = min(ph + dh, p.n_chunks)
        begin = p.start + first * chunk_size
        if begin >= p.end:
            continue
        n = p.end - begin
        runs.append(StoreRun(p, min(ph, first), first, begin, len(rows), n, len(shifts)))
        rows.extend(range(begin, p.end))
        sot.extend([len(shifts)] * n)
        shifts.append(-p.start)
    return runs, rows, sot, shifts
