"""The paged movers at their edges: a plain torch statement of what the split (PagedAttention / xFormers) and
block-strided (FlashInfer) pack and unpack move, a Python model of the launch rule the split kernel runs under, and the
table of cases that drives the kernel to every branch of that rule.

The statement works on one layer's caches held as bits (int16 for two-byte elements, uint8 for one-byte ones) on the
CPU, with torch views, permutes and indexing only.  It shares nothing with the native library: not the kernels, not the
address formulas of include/b200kv.h, not the layout detection of codec.py.

The model restates launch_split (lmcache_b200/csrc/mover.cu) on the host side -- vector width, heads per unit, shared
memory, the 48 KB and 200 KB decisions, the alignment fallbacks -- and, per group of bs call tokens, the kernel's tile
test.  It tells a failing test which path the failing group took, and `coverage` checks that CASES reaches every branch.
"""
from typing import Dict, List, NamedTuple, Optional, Sequence, Set, Tuple

import numpy as np
import torch

H100_SMS = 132                 # H100 SXM; the GPU tests read the device's own count
SMEM_OPT_IN = 48 * 1024        # above this the kernel's dynamic shared memory needs cudaFuncSetAttribute
SMEM_TILE_MAX = 200 * 1024     # above this launch_split gives up the tile path
TILE_TARGET = 16384            # heads per unit: the most whose tile hb * bs * D * es fits in 16 KB


def bits_dtype(es: int) -> torch.dtype:
    return torch.int16 if es == 2 else torch.uint8


# ---------------------------------------------------------------------------------------------- the statement
class PagedLayoutLike(NamedTuple):
    """the fields of codec.PagedLayout the statement reads, for caches built without codec.paged_layout"""
    kind: str
    nb: int
    bs: int
    H: int
    D: int
    rows_per_block: int
    x: int


def _strided_view(layout, t: torch.Tensor) -> torch.Tensor:
    """the [nb, bs, H, D] rows of a block-strided cache: block b starts rows_per_block rows after block b - 1"""
    nb, bs, H, D, rpb = layout.nb, layout.bs, layout.H, layout.D, layout.rows_per_block
    return torch.as_strided(t, (nb, bs, H, D), (rpb * H * D, H * D, D, 1), t.storage_offset())


def _row_views(layout, key: torch.Tensor, value: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """views of one layer's caches as [nb, bs, H, D] rows (the key of a split cache as [nb, bs, H, D/x, x])"""
    nb, bs, H, D = layout.nb, layout.bs, layout.H, layout.D
    if layout.kind == "split":
        x = layout.x
        return (key.view(nb, H, D // x, bs, x).permute(0, 3, 1, 2, 4),
                value.view(nb, H, D, bs).permute(0, 3, 1, 2))
    if layout.kind == "strided":
        return _strided_view(layout, key), _strided_view(layout, value)
    return key.view(nb, bs, H, D), value.view(nb, bs, H, D)


def ref_rows(layout, key: torch.Tensor, value: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """One layer's (key, value) caches in `layout` (a codec.PagedLayout or anything with its fields) as two
    [nb * bs, H, D] FlashAttention row tensors (copies).  A strided cache is passed as the view the engine gets
    (FlashInfer's kv[:, 0] / kv[:, 1]); only its storage and offset are used, its rows are placed by rows_per_block."""
    n = layout.nb * layout.bs
    return tuple(v.reshape(n, layout.H, layout.D).clone() for v in _row_views(layout, key, value))


def ref_write_rows(layout, key: torch.Tensor, value: torch.Tensor, rows_k: torch.Tensor, rows_v: torch.Tensor) -> None:
    """The inverse of ref_rows: write [nb * bs, H, D] rows into the caches in place (rows only: a strided cache's other
    rows and a padded allocation's spare rows are left alone)."""
    for view, rows in zip(_row_views(layout, key, value), (rows_k, rows_v)):
        view.copy_(rows.view(view.shape))


def _chunking(T: int, tok_begin: int, chunk_tokens: int) -> List[Tuple[int, int]]:
    """(first call token, tokens) of every chunk of a move of tokens [tok_begin, T)"""
    return [(a, min(chunk_tokens, T - a)) for a in range(tok_begin, T, chunk_tokens)]


def ref_pack(layout, caches: Sequence[Tuple[torch.Tensor, torch.Tensor]], slots: torch.Tensor, tok_begin: int,
             chunk_tokens: int, layers: Optional[Tuple[int, int]] = None) -> List[torch.Tensor]:
    """The vllm chunk blobs [nl, 2, t, H, D] that a pack of call tokens [tok_begin, len(slots)) in chunks of
    chunk_tokens (the last may be shorter) gathers from `caches` (one (key, value) pair per layer); token i of the call
    is cache row slots[i].  layers = (a, b): layers a .. b - 1 only, layer a first."""
    a, b = layers if layers is not None else (0, len(caches))
    rows = [ref_rows(layout, *caches[l]) for l in range(a, b)]
    out = []
    for c0, t in _chunking(len(slots), tok_begin, chunk_tokens):
        s = slots[c0:c0 + t].long()
        out.append(torch.stack([torch.stack([rk[s], rv[s]]) for rk, rv in rows]))
    return out


def ref_unpack(layout, caches: Sequence[Tuple[torch.Tensor, torch.Tensor]], slots: torch.Tensor, tok_begin: int,
               chunk_tokens: int, blobs: Sequence[torch.Tensor], layers: Optional[Tuple[int, int]] = None) -> None:
    """Scatter vllm chunk blobs (as ref_pack makes them) into `caches` in place: the inverse of ref_pack on the rows it
    addresses; every other element of the caches keeps its value."""
    a, b = layers if layers is not None else (0, len(caches))
    chunks = _chunking(len(slots), tok_begin, chunk_tokens)
    assert len(chunks) == len(blobs)
    for li, l in enumerate(range(a, b)):
        rk, rv = ref_rows(layout, *caches[l])
        for (c0, t), blob in zip(chunks, blobs):
            s = slots[c0:c0 + t].long()
            rk[s] = blob[li, 0]
            rv[s] = blob[li, 1]
        ref_write_rows(layout, caches[l][0], caches[l][1], rk, rv)


# ---------------------------------------------------------------------------------------------- slot maps
def make_slots(kind: str, T: int, nb: int, bs: int, seed: int) -> torch.Tensor:
    """T distinct slots in [0, nb * bs) (CPU int64).
    vllm:    a block table's slots from the first token of a block (every whole group is a tile);
    mid:     the same, from the middle of the first block (no group is);
    shift:   consecutive slots from bs // 2: runs of bs slots that cross a block boundary;
    inblock: whole blocks, each with its slots in a scrambled order;
    alt:     vllm, with every second block scrambled (tile and element-wise groups interleave);
    perm:    any slots."""
    g = torch.Generator().manual_seed(seed)
    if kind == "perm":
        return torch.randperm(nb * bs, generator=g)[:T]
    if kind == "shift":
        s = torch.arange(T) + max(1, bs // 2)
        assert bs > 1 and int(s[-1]) < nb * bs
        return s
    blocks = torch.randperm(nb, generator=g)
    inner = torch.arange(bs).repeat(nb, 1)
    for i in range(nb):
        if kind == "inblock" or (kind == "alt" and i % 2 == 1):
            p = torch.randperm(bs, generator=g)
            if bs > 1 and bool((p == torch.arange(bs)).all()):
                p[[0, 1]] = p[[1, 0]]
            inner[i] = p
    start = max(1, bs // 2) if kind == "mid" else 0
    s = (blocks.view(-1, 1) * bs + inner).flatten()[start:start + T]
    assert s.numel() == T, "too few blocks for T tokens"
    return s


# ---------------------------------------------------------------------------------------------- the launch model
class Launch(NamedTuple):
    es: int
    bs: int
    H: int
    D: int
    vw_bs: int            # value vector bytes the block size allows (16, 8 or 0)
    vw: int               # what the launch runs with (0: element-wise only)
    hb: int               # heads per unit
    nhb: int              # head blocks per group
    pitch: int            # shared-memory bytes per row
    tile_smem: int        # hb * bs * pitch: the tile's shared memory
    smem: int             # dynamic shared memory of the launch (0 without a tile path)
    opt_in: bool          # smem > 48 KB: cudaFuncSetAttribute before the launch
    refused: bool         # the tile would exceed 200 KB
    misaligned: Tuple[str, ...]   # whole-launch alignment fallbacks that apply: chunk_buffer, stride, plane
    table: bool


def launch_model(es: int, bs: int, H: int, D: int, *, table: bool, chunk_off: int = 0, stride: int = 0,
                 plane_off: int = 0) -> Launch:
    """launch_split's host rule.  chunk_off: the chunk buffer's address mod 16 (contiguous form); stride: its chunk
    stride in bytes; plane_off: the planes' addresses mod 16; table: the device-table form (b200kv_*_chunks_layers),
    whose entries the kernel checks per chunk."""
    head_bytes = bs * D * es
    hb = next(h for h in range(H, 0, -1) if H % h == 0 and (h * head_bytes <= TILE_TARGET or h == 1))
    pitch = D * es + 16
    vw_bs = 16 if (bs * es) % 16 == 0 else 8 if (bs * es) % 8 == 0 else 0
    mis = []
    if not table and chunk_off % 16 != 0:
        mis.append("chunk_buffer")
    if not table and stride % 16 != 0:
        mis.append("stride")
    if plane_off % 16 != 0:
        mis.append("plane")
    tile_smem = hb * bs * pitch
    refused = tile_smem > SMEM_TILE_MAX
    vw = 0 if mis or refused else vw_bs
    smem = tile_smem if vw else 0
    return Launch(es, bs, H, D, vw_bs, vw, hb, H // hb, pitch, tile_smem, smem, smem > SMEM_OPT_IN, refused,
                  tuple(mis), table)


def group_paths(launch: Launch, slots: Sequence[int], tok_begin: int, chunk_tokens: int,
                table_offs: Optional[Sequence[int]] = None) -> List[Tuple[int, str]]:
    """(g0, path) of every group the launch visits, in order: "tile" where the kernel's tile test passes, else why not:
    "vw0" (no tile path in this launch), "edge" (the group reaches outside the call), "chunk_boundary" (a chunk ends
    inside it), "table_entry" (its chunk's table entry is not 16-byte aligned), "run_off_block" (consecutive slots
    from a slot that is not a block's first), "permuted_block" (one block's slots, out of order), "scattered"."""
    bs = launch.bs
    T = len(slots)
    s = np.asarray(slots, dtype=np.int64)
    out = []
    for k in range(tok_begin // bs, (T - 1) // bs + 1):
        g0 = k * bs
        if launch.vw == 0:
            why = "vw0"
        elif g0 < tok_begin or g0 + bs > T:
            why = "edge"
        else:
            j, tok0 = divmod(g0 - tok_begin, chunk_tokens)
            run = s[g0:g0 + bs]
            if tok0 + bs > min(chunk_tokens, T - tok_begin - j * chunk_tokens):
                why = "chunk_boundary"
            elif table_offs is not None and table_offs[j % len(table_offs)] % 16 != 0:
                why = "table_entry"
            elif np.array_equal(run, run[0] + np.arange(bs)):
                why = "tile" if run[0] % bs == 0 else "run_off_block"
            elif np.array_equal(np.sort(run), (run[0] // bs) * bs + np.arange(bs)):
                why = "permuted_block"
            else:
                why = "scattered"
        out.append((g0, why))
    return out


def cta_mixes(launch: Launch, paths: Sequence[Tuple[int, str]], nl: int, sms: int) -> bool:
    """Whether one CTA of the grid-stride loop runs both a tile unit and an element-wise one (it then reuses its
    shared-memory rows after element-wise work): units (group, plane, head block), grid min(units, sms * 32)."""
    n_groups = len(paths)
    units = n_groups * 2 * nl * launch.nhb
    blocks = max(1, min(units, sms * 8 * 4))
    u = np.arange(units)
    tile = np.array([p == "tile" for _, p in paths])[(u // launch.nhb) % n_groups]
    cta = u % blocks
    n_tile = np.bincount(cta, weights=tile, minlength=blocks)
    n_all = np.bincount(cta, minlength=blocks)
    return bool(((n_tile > 0) & (n_tile < n_all)).any())


# ---------------------------------------------------------------------------------------------- the cases
DTYPES = {"bf16": (torch.bfloat16, 2), "fp16": (torch.float16, 2), "u8": (torch.uint8, 1),
          "e4m3": (torch.float8_e4m3fn, 1), "e5m2": (torch.float8_e5m2, 1)}


class Case(NamedTuple):
    name: str
    dtype: str                  # a DTYPES key
    bs: int
    H: int
    D: int
    L: int
    nb: int
    slots: str                  # a make_slots kind
    T: int
    tok_begin: int
    chunk_tokens: int
    layers: Tuple[int, int]     # the layer range of the device-table form (the contiguous form moves every layer)
    buf: str = "device"         # chunks in "device" memory or in mapped page-locked ("pinned") host memory
    chunk_off: int = 0          # contiguous form: the chunk buffer starts this many bytes past a 16-byte boundary
    stride_pad: int = 0         # contiguous form: chunk stride = chunk bytes + stride_pad
    table_offs: Tuple[int, ...] = (0,)   # table form: chunk j starts table_offs[j % len] bytes past a 16-byte boundary
    plane_off: int = 0          # every key and value cache starts this many bytes past a 16-byte boundary

    @property
    def es(self) -> int:
        return DTYPES[self.dtype][1]

    @property
    def torch_dtype(self) -> torch.dtype:
        return DTYPES[self.dtype][0]

    @property
    def seed(self) -> int:
        return sum(ord(c) * (i + 1) for i, c in enumerate(self.name))

    def chunk_bytes(self, nl: int) -> int:
        return nl * 2 * self.chunk_tokens * self.H * self.D * self.es

    def forms(self) -> List[Tuple[str, int, int]]:
        """(form, first layer, end layer): the contiguous buffer over every layer and the device table over `layers`"""
        return [("contig", 0, self.L), ("table", *self.layers)]

    def launch(self, form: str) -> Launch:
        if form == "table":
            return launch_model(self.es, self.bs, self.H, self.D, table=True, plane_off=self.plane_off)
        return launch_model(self.es, self.bs, self.H, self.D, table=False, chunk_off=self.chunk_off,
                            stride=self.chunk_bytes(self.L) + self.stride_pad, plane_off=self.plane_off)

    def paths(self, form: str, slots: Optional[torch.Tensor] = None) -> List[Tuple[int, str]]:
        if slots is None:
            slots = make_slots(self.slots, self.T, self.nb, self.bs, self.seed)
        return group_paths(self.launch(form), slots.tolist(), self.tok_begin, self.chunk_tokens,
                           self.table_offs if form == "table" else None)


def _c(*a, **k) -> Case:
    return Case(*a, **k)


CASES: List[Case] = [
    # name                      dtype  bs   H  D   L  nb  slots     T     tb  cs   layers
    # baselines: every whole group a tile (16-byte value vectors), and scrambled slots
    _c("bf16_bs16_vllm",        "bf16", 16, 8, 64, 3, 20, "vllm",   16 * 9 + 5, 16, 48, (1, 3)),
    _c("e4m3_bs32_perm",        "e4m3", 32, 2, 128, 2, 12, "perm",  300, 7, 64, (0, 1)),
    _c("fp16_bs16_mid",         "fp16", 16, 4, 64, 2, 16, "mid",    200, 0, 64, (1, 2)),
    # 8-byte value vectors: VO = 4 for 16-bit elements (bs * es = 8, 24), VO = 8 for one-byte ones (8, 24)
    _c("bf16_bs4_vw8",          "bf16", 4, 2, 64, 2, 40, "vllm",    101, 4, 32, (0, 2)),
    _c("fp16_bs12_vw8",         "fp16", 12, 3, 128, 3, 14, "vllm",  12 * 9 + 5, 12, 36, (1, 3)),
    _c("e4m3_bs8_vw8",          "e4m3", 8, 4, 64, 2, 16, "vllm",    90, 3, 32, (1, 2)),
    _c("u8_bs24_vw8",           "u8", 24, 2, 32, 2, 8, "vllm",      24 * 6 + 1, 24, 48, (0, 2)),
    # no tile path from the block size: bs * es not a multiple of 8
    _c("bf16_bs1_vw0",          "bf16", 1, 2, 64, 2, 80, "vllm",    70, 3, 16, (1, 2)),
    _c("bf16_bs2_vw0",          "bf16", 2, 2, 64, 2, 40, "vllm",    70, 2, 16, (0, 2)),
    _c("bf16_bs3_vw0",          "bf16", 3, 1, 128, 2, 30, "vllm",   70, 3, 18, (0, 1)),
    _c("e5m2_bs4_vw0",          "e5m2", 4, 2, 64, 2, 30, "vllm",    90, 4, 32, (1, 2)),
    _c("u8_bs12_vw0",           "u8", 12, 2, 32, 2, 10, "vllm",     100, 12, 36, (0, 2)),
    # heads per unit: a proper divisor of H that is not a power of two
    _c("bf16_H6_hb3",           "bf16", 16, 6, 128, 2, 12, "vllm",  16 * 10 + 7, 16, 64, (1, 2)),
    _c("fp16_H12_hb6",          "fp16", 16, 12, 64, 2, 10, "vllm",  16 * 8 + 3, 0, 32, (0, 2)),
    _c("bf16_H40_hb5",          "bf16", 16, 40, 80, 2, 8, "vllm",   16 * 6 + 9, 16, 48, (0, 1)),
    _c("e4m3_H6_hb3",           "e4m3", 32, 6, 128, 2, 8, "vllm",   32 * 5 + 7, 32, 64, (1, 2)),
    _c("u8_H12_hb6",            "u8", 32, 12, 64, 2, 6, "vllm",     32 * 4 + 1, 0, 64, (0, 2)),
    # shared memory above 48 KB (68 and 132 KB), and a tile refused above 200 KB
    _c("bf16_bs256_D128_68k",   "bf16", 256, 2, 128, 2, 6, "vllm",  256 * 4 + 100, 256, 512, (1, 2)),
    _c("bf16_bs256_D256_132k",  "bf16", 256, 1, 256, 2, 5, "vllm",  256 * 3 + 50, 0, 256, (0, 2)),
    _c("e4m3_bs256_D256_68k",   "e4m3", 256, 2, 256, 2, 5, "vllm",  256 * 3 + 9, 256, 512, (0, 1)),
    _c("bf16_bs512_D256_refused", "bf16", 512, 1, 256, 2, 4, "vllm", 512 * 3 + 20, 512, 512, (1, 2)),
    _c("u8_bs1024_D256_refused", "u8", 1024, 1, 256, 2, 3, "vllm",  1024 * 2 + 30, 0, 1024, (0, 2)),
    # a device table that mixes 16-byte aligned and misaligned chunk pointers
    _c("bf16_table_mixed",      "bf16", 16, 2, 64, 3, 16, "vllm",   16 * 11 + 4, 16, 32, (0, 3),
       table_offs=(0, 2, 0, 8)),
    _c("e4m3_table_mixed",      "e4m3", 16, 2, 64, 2, 16, "vllm",   16 * 11 + 4, 0, 32, (1, 2),
       table_offs=(0, 1, 8, 0)),
    # whole-launch fallbacks: a misaligned chunk buffer, a chunk stride % 16 != 0, misaligned planes
    _c("bf16_chunk_buf_off2",   "bf16", 16, 2, 64, 2, 12, "vllm",   150, 16, 64, (0, 2), chunk_off=2),
    _c("e5m2_chunk_buf_off1",   "e5m2", 16, 2, 64, 2, 12, "vllm",   150, 0, 64, (1, 2), chunk_off=1),
    _c("fp16_stride_pad8",      "fp16", 16, 2, 64, 2, 12, "vllm",   150, 16, 64, (0, 2), stride_pad=8),
    _c("u8_stride_pad4",        "u8", 16, 2, 64, 2, 12, "vllm",     150, 16, 64, (0, 1), stride_pad=4),
    _c("bf16_plane_off2",       "bf16", 16, 2, 64, 2, 12, "vllm",   150, 16, 64, (1, 2), plane_off=2),
    _c("fp16_plane_off8",       "fp16", 8, 4, 128, 2, 20, "vllm",   150, 8, 64, (0, 2), plane_off=8),
    _c("e4m3_plane_off8",       "e4m3", 16, 2, 64, 2, 12, "vllm",   150, 16, 64, (0, 2), plane_off=8),
    _c("u8_plane_off2",         "u8", 32, 2, 64, 2, 8, "vllm",      150, 0, 64, (1, 2), plane_off=2),
    # a chunk boundary inside a block: chunk_tokens not a multiple of bs, and chunk_tokens < bs
    _c("bf16_cs24_bs16",        "bf16", 16, 2, 64, 2, 14, "vllm",   16 * 12 + 5, 16, 24, (0, 2)),
    _c("fp16_cs12_bs32",        "fp16", 32, 2, 64, 2, 8, "vllm",    32 * 5 + 3, 32, 12, (1, 2)),
    _c("e4m3_cs40_bs32",        "e4m3", 32, 2, 64, 2, 8, "vllm",    32 * 6 + 1, 0, 40, (0, 2)),
    _c("u8_cs8_bs16",           "u8", 16, 2, 64, 2, 12, "vllm",     16 * 9 + 2, 16, 8, (0, 1)),
    # consecutive slots from the middle of a block, and blocks with scrambled slots
    _c("bf16_run_off_block",    "bf16", 16, 2, 64, 2, 12, "shift",  16 * 9 + 3, 16, 64, (0, 2)),
    _c("u8_run_off_block",      "u8", 16, 2, 64, 2, 12, "shift",    16 * 9 + 3, 0, 64, (1, 2)),
    _c("fp16_permuted_blocks",  "fp16", 8, 2, 64, 2, 20, "inblock", 8 * 15 + 2, 8, 32, (0, 2)),
    _c("e5m2_permuted_blocks",  "e5m2", 16, 2, 64, 2, 12, "inblock", 16 * 9 + 3, 16, 64, (0, 1)),
    # more units than SMs x 32, tile and element-wise groups interleaved: CTAs alternate between the two paths
    _c("bf16_cta_mix",          "bf16", 4, 2, 64, 4, 680, "alt",    2700, 0, 256, (1, 3)),
    _c("u8_cta_mix",            "u8", 8, 2, 64, 4, 610, "alt",      4800, 8, 256, (0, 2)),
    # chunks in mapped page-locked host memory: the pack writes over PCIe, the unpack reads over it
    _c("bf16_pinned",           "bf16", 16, 4, 128, 2, 12, "vllm",  16 * 9 + 7, 16, 48, (0, 2), buf="pinned",
       table_offs=(0, 2)),
    _c("e4m3_pinned",           "e4m3", 8, 2, 64, 2, 20, "alt",     8 * 16 + 3, 8, 32, (1, 2), buf="pinned",
       table_offs=(0, 8)),
]


# the branches of launch_split / split_kernel the suite must reach, for both directions and both element sizes
BRANCHES = {
    "vw8": "8-byte value vectors on the tile path (VO = 4 for 16-bit elements, 8 for one-byte ones)",
    "vw0_block_size": "no tile path because bs * es is not a multiple of 8",
    "hb_not_pow2": "heads per unit a proper divisor of H that is not a power of two, on the tile path",
    "smem_opt_in": "dynamic shared memory above 48 KB (cudaFuncSetAttribute), on the tile path",
    "smem_refused": "tile refused because it would exceed 200 KB",
    "table_entry_misaligned": "per-chunk fallback for a misaligned table entry, next to tiles in the same launch",
    "chunk_buffer_misaligned": "whole-launch fallback: chunk buffer not 16-byte aligned",
    "stride_misaligned": "whole-launch fallback: chunk stride % 16 != 0",
    "plane_misaligned": "whole-launch fallback: a cache plane not 16-byte aligned",
    "chunk_boundary_in_block": "a chunk boundary inside a group (tok0 + bs > t)",
    "chunk_smaller_than_block": "chunk_tokens < bs",
    "run_off_block": "a run of consecutive slots that does not start at a block boundary",
    "permuted_block": "a block whose slots are permuted",
    "cta_mixes_paths": "one CTA runs tile and element-wise units under the grid stride",
    "mapped_pinned": "pack into and unpack from mapped page-locked memory",
}
DIRECTIONS = ("pack", "unpack")


def branches_of(case: Case, sms: Optional[int] = None) -> Set[str]:
    """The BRANCHES keys the case reaches (in either form; each form runs in both directions).  sms: the SM count
    (default: the device's, or an H100 SXM's without a GPU)."""
    sms = sm_count(H100_SMS) if sms is None else sms
    hit = set()
    slots = make_slots(case.slots, case.T, case.nb, case.bs, case.seed)
    for form, a, b in case.forms():
        lc = case.launch(form)
        paths = case.paths(form, slots)
        kinds = {p for _, p in paths}
        tiles = "tile" in kinds
        if lc.vw == 8 and tiles:
            hit.add("vw8")
        if lc.vw_bs == 0:
            hit.add("vw0_block_size")
        if tiles and lc.hb < case.H and lc.hb & (lc.hb - 1) != 0:
            hit.add("hb_not_pow2")
        if tiles and lc.opt_in:
            hit.add("smem_opt_in")
        if lc.refused and lc.vw_bs:
            hit.add("smem_refused")
        if tiles and "table_entry" in kinds:
            hit.add("table_entry_misaligned")
        if lc.vw_bs and not lc.refused:
            for m in lc.misaligned:
                hit.add({"chunk_buffer": "chunk_buffer_misaligned", "stride": "stride_misaligned",
                         "plane": "plane_misaligned"}[m])
        if "chunk_boundary" in kinds:
            hit.add("chunk_boundary_in_block")
            if case.chunk_tokens < case.bs:
                hit.add("chunk_smaller_than_block")
        if "run_off_block" in kinds:
            hit.add("run_off_block")
        if "permuted_block" in kinds:
            hit.add("permuted_block")
        if tiles and cta_mixes(lc, paths, b - a, sms):
            hit.add("cta_mixes_paths")
        if case.buf == "pinned" and tiles:
            hit.add("mapped_pinned")
    return hit


def coverage(cases: Sequence[Case] = CASES, sms: Optional[int] = None) -> Dict[Tuple[str, str, int], List[str]]:
    """(branch, direction, element size) -> the cases that reach it; every key of BRANCHES x DIRECTIONS x (1, 2)"""
    out: Dict[Tuple[str, str, int], List[str]] = {(br, d, es): [] for br in BRANCHES for d in DIRECTIONS
                                                  for es in (1, 2)}
    for c in cases:
        for br in branches_of(c, sms):
            for d in DIRECTIONS:
                out[(br, d, c.es)].append(c.name)
    return out


def sm_count(default: Optional[int] = None) -> int:
    """The device's SM count when a GPU is present, else `default`."""
    if torch.cuda.is_available():
        return torch.cuda.get_device_properties(0).multi_processor_count
    if default is None:
        raise RuntimeError("no GPU: pass the SM count")
    return default
