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
from typing import Callable, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np
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


def rope_shift_layers(view, layer_begin: int, layer_end: int, tok_begin: int, seg: torch.Tensor, table: torch.Tensor,
                      rope: RopeSpec, stream: torch.cuda.Stream) -> None:
    """rope_shift of the key planes of layers [layer_begin, layer_end) only, by a prepared table (rope_table's), on
    `stream`: one b200kv_rope_shift_layers launch"""
    N.check(N.lib().b200kv_rope_shift_layers(ctypes.byref(view.desc), layer_begin, layer_end, tok_begin, seg.numel(),
                                             ctypes.c_void_p(seg.data_ptr()), ctypes.c_void_p(table.data_ptr()),
                                             rope.rotary_dim, rope.offset, STYLES[rope.style], stream.cuda_stream),
            "rope_shift_layers")


def written_seg_of_tok(chunks: Sequence[Tuple[int, int, int]], run_rows: Sequence[int],
                       run_ends: Sequence[int]) -> Tuple[int, np.ndarray]:
    """The shift's arguments for the chunks a multi-run fetch wrote, (run, destination token, tokens) each:
    (lo, int32 seg_of_tok of tokens [lo, lo + len)).  A chunk of run r turns by table row run_rows[r], its tokens
    clipped to the run's end run_ends[r]; -1 (a segment at token 0) leaves it alone, like every token no chunk wrote.
    Empty when nothing turns.  The runs are segments of one plan, which never overlap (plan_segments)."""
    turned = [(tok, min(tok + n, run_ends[r]), run_rows[r]) for r, tok, n in chunks if run_rows[r] >= 0]
    turned = [t for t in turned if t[1] > t[0]]
    if not turned:
        return 0, np.zeros(0, np.int32)
    lo, hi = min(a for a, _, _ in turned), max(b for _, b, _ in turned)
    sot = np.full(hi - lo, -1, dtype=np.int32)
    for a, b, k in turned:
        sot[a - lo:b - lo] = k
    return lo, sot


def chunk_arrays(chunks: Sequence[Tuple[int, int, int]], run_rows: Sequence[int]):
    """The per-chunk arguments of b200kv_unpack_chunks_layers_rope for the chunks a multi-run fetch wrote, (run,
    destination token, tokens) each: (chunk_ntok int32, dst_tok int64, chunk_seg int32), chunk_seg the run's table row
    (-1: a segment at token 0, copied)."""
    return (np.array([n for _, _, n in chunks], dtype=np.int32), np.array([t for _, t, _ in chunks], dtype=np.int64),
            np.array([run_rows[r] for r, _, _ in chunks], dtype=np.int32))


def unpack_rope_layers(view, table_ptr: int, arrays, chunk_tokens: int, layer_begin: int, layer_end: int,
                       rot: "Rotation", stream: torch.cuda.Stream) -> None:
    """one b200kv_unpack_chunks_layers_rope launch on `stream`: chunk j's layer range starts at the device pointer
    table_ptr[j]; arrays: device (chunk_ntok, dst_tok, chunk_seg) of chunk_arrays"""
    ntok, dst_tok, seg = arrays
    N.check(N.lib().b200kv_unpack_chunks_layers_rope(
        ctypes.c_void_p(table_ptr), ntok.numel(), chunk_tokens, ctypes.c_void_p(ntok.data_ptr()),
        ctypes.c_void_p(dst_tok.data_ptr()), ctypes.c_void_p(seg.data_ptr()), int(view.fmt == "huggingface"),
        layer_begin, layer_end, ctypes.byref(view.desc), ctypes.c_void_p(rot.table.data_ptr()), rot.rope.rotary_dim,
        rot.rope.offset, STYLES[rot.rope.style], stream.cuda_stream), "unpack_chunks_layers_rope")


class Rotation:
    """The turn a layer-major multi-run fetch (a tier's get_kv_layerwise_runs) gives the keys it writes: the chunks of
    run r turn by row run_rows[r] of `table` (rope_table's: one row per segment that does not start at token 0; -1 for
    one that does), up to the run's segment end run_ends[r].  The tier turns each layer on the stream that wrote it,
    before that layer's ready event."""

    def __init__(self, rope: RopeSpec, table: torch.Tensor, run_rows: Sequence[int], run_ends: Sequence[int]):
        self.rope, self.table, self.run_rows, self.run_ends = rope, table, list(run_rows), list(run_ends)

    def prepare(self, chunks: Sequence[Tuple[int, int, int]], device) -> Optional["PreparedRotation"]:
        """The rotation of the chunks a fetch matched, (run, destination token, tokens) each, or None when none of them
        turns.  Its seg_of_tok is uploaded on the current stream: call it before the fetch's start event."""
        lo, sot = written_seg_of_tok(chunks, self.run_rows, self.run_ends)
        if not len(sot):
            return None
        return PreparedRotation(self, lo, torch.from_numpy(sot).to(device, non_blocking=True))


class PreparedRotation:
    def __init__(self, rot: Rotation, lo: int, seg: torch.Tensor):
        self.rot, self.lo, self.seg = rot, lo, seg

    def shift_layers(self, view, layer_begin: int, layer_end: int, stream: torch.cuda.Stream) -> None:
        """turn the written keys of layers [layer_begin, layer_end) on `stream` (the stream that wrote them)"""
        rope_shift_layers(view, layer_begin, layer_end, self.lo, self.seg, self.rot.table, self.rot.rope, stream)

    def shift_layer(self, view, layer: int, stream: torch.cuda.Stream) -> None:
        self.shift_layers(view, layer, layer + 1, stream)

    def record_stream(self, stream: torch.cuda.Stream) -> None:
        self.seg.record_stream(stream)
        self.rot.table.record_stream(stream)


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


# ---------------------------------------------------------------------------------------------- layer-wise segment store
def store_run_arrays(runs: Sequence[StoreRun]) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The per-chunk arguments of b200kv_pack_chunks_layers_rope for a layer-wise segment store, in which each run of
    plan_segment_store is one chunk of its n_tok tokens from request token `begin`, turned by its table row:
    (chunk_ntok int32, src_tok int64, chunk_seg int32)."""
    return (np.array([r.n_tok for r in runs], dtype=np.int32), np.array([r.begin for r in runs], dtype=np.int64),
            np.array([r.row for r in runs], dtype=np.int32))


def staging_layout(runs: Sequence[StoreRun], shape_of: Callable[[int], Tuple[int, ...]],
                   layer_elems: Callable[[int], int], L: int) -> Tuple[List[Tuple[int, ...]], List[int], np.ndarray]:
    """Where a layer-wise segment store stages its runs: each run's own chunk blob (shape_of(n_tok)) back to back in
    one allocation.  Returns (the blob shapes, each blob's element offset, int64 [L, runs] the element offset of layer l
    of each run's blob -- the chunk_ptrs of layer l, in elements).  layer_elems(t): elements of one layer of a blob of
    t tokens."""
    shapes = [tuple(shape_of(r.n_tok)) for r in runs]
    sizes = [int(np.prod(s)) for s in shapes]
    offs = [int(x) for x in np.concatenate([[0], np.cumsum(sizes, dtype=np.int64)[:-1]])] if runs else []
    per = np.array([layer_elems(r.n_tok) for r in runs], dtype=np.int64)
    layer_offs = np.array(offs, dtype=np.int64)[None, :] + np.arange(L, dtype=np.int64)[:, None] * per[None, :]
    return shapes, offs, layer_offs


def pack_rope_layers(view, ptrs_ptr: int, arrays, chunk_tokens: int, layer_begin: int, layer_end: int,
                     table: torch.Tensor, rope: RopeSpec, stream: torch.cuda.Stream) -> None:
    """one b200kv_pack_chunks_layers_rope launch on `stream`: chunk j's layer range goes to the device pointer
    ptrs_ptr[j]; arrays: device (chunk_ntok, src_tok, chunk_seg) of store_run_arrays; table: rope_table's"""
    ntok, src_tok, seg = arrays
    N.check(N.lib().b200kv_pack_chunks_layers_rope(
        ctypes.byref(view.desc), ntok.numel(), chunk_tokens, ctypes.c_void_p(ntok.data_ptr()),
        ctypes.c_void_p(src_tok.data_ptr()), ctypes.c_void_p(seg.data_ptr()), int(view.fmt == "huggingface"),
        layer_begin, layer_end, ctypes.c_void_p(ptrs_ptr), ctypes.c_void_p(table.data_ptr()), rope.rotary_dim,
        rope.offset, STYLES[rope.style], stream.cuda_stream), "pack_chunks_layers_rope")


class StagedGather:
    """The staging of a layer-wise segment store.  One device allocation holds each run's own chunk blob
    (KvView.blob_shape of its n_tok tokens) back to back -- the raw bytes of the tokens stored, as the whole form's one
    staging blob.  layer(l, stream) makes the side stream wait for `stream` and fills layer l of every run's blob with
    one b200kv_pack_chunks_layers_rope launch there, keys turned by -start; it returns the event after it.  Everything
    the launches read is made on the current stream at construction, which the side stream waits for."""

    def __init__(self, view, runs: Sequence[StoreRun], shifts: Sequence[int], fmt: str, latent: bool, rope: RopeSpec,
                 side: torch.cuda.Stream, blob_shape: Callable):
        dev = view.device
        self.view, self.rope, self.side, self.R = view, rope, side, len(runs)
        self.chunk_tokens = max(r.n_tok for r in runs)
        L, H, D = view.L, view.H, view.D
        per_tok = (1 if latent else 2) * H * D                # elements of one token of one layer
        shapes, offs, layer_offs = staging_layout(runs, lambda t: blob_shape(fmt, L, H, D, t, latent),
                                                  lambda t: per_tok * t, L)
        es = view.dtype.itemsize
        with torch.cuda.device(dev):
            self.staging = torch.empty(offs[-1] + int(np.prod(shapes[-1])), dtype=view.dtype, device=dev)
            self.blobs = [self.staging.narrow(0, o, int(np.prod(s))).view(s) for o, s in zip(offs, shapes)]
            self.ptrs = torch.from_numpy(self.staging.data_ptr() + es * layer_offs).to(dev)
            self.arrays = tuple(torch.from_numpy(a).to(dev) for a in store_run_arrays(runs))
            self.table = rope_table(torch.tensor(list(shifts), dtype=torch.int64).to(dev), rope)
            ready = torch.cuda.Event()
            ready.record(torch.cuda.current_stream())
        side.wait_event(ready)
        view.record_stream(side)                             # the caller's KV outlives the last gather that reads it
        for t in (self.staging, self.ptrs, self.table) + self.arrays:
            t.record_stream(side)

    def layer(self, layer: int, stream: torch.cuda.Stream) -> torch.cuda.Event:
        with torch.cuda.device(self.view.device):
            written = torch.cuda.Event()
            written.record(stream)
            self.side.wait_event(written)
            pack_rope_layers(self.view, self.ptrs.data_ptr() + 8 * self.R * layer, self.arrays, self.chunk_tokens,
                             layer, layer + 1, self.table, self.rope, self.side)
            done = torch.cuda.Event()
            done.record(self.side)
        return done

    def join(self, events: Sequence[torch.cuda.Event]) -> torch.cuda.Event:
        """an event after `events` and every gather"""
        with torch.cuda.device(self.view.device):
            for ev in events:
                self.side.wait_event(ev)
            done = torch.cuda.Event()
            done.record(self.side)
        return done
