"""CacheBlend's selective recomputation, the cache's side: which reused tokens a RAG prefill recomputes.

A document served at a new position (retrieve_paged_segments) carries KV that, at layers >= 1, was computed without
attending to the tokens now in front of it.  CacheBlend (Yao et al., 2024) recomputes a small share of the reused tokens:
those whose cached KV deviates most from a fresh computation, chosen at a check layer from the deviation of the keys.
The model computes; this module measures and chooses on the GPU, over the engine's own layouts:

  * b200kv_blend_deviation compares the model's fresh keys of a check layer with the cached key rows of that layer, in
    every layout the segment calls write (FlashAttention, FlashInfer block-strided and PagedAttention split caches, dense
    views, MLA latents).  Its summation order depends on (H, D) only, so tensor-parallel ranks that all-reduce their
    per-head partial sums hold the same totals.
  * b200kv_blend_select keeps the tokens that were not retrieved (always recomputed) and the k retrieved tokens of
    largest deviation, ties to the lower row: the same choice on every rank, with no host sync.
  * b200kv_blend_select_batch makes that choice per request of a prefill batch whose rows are concatenated, in one
    launch sequence whatever the number of requests.

BatchBlendPlan walks a prefill batch through the check layers of a BlendSpec (CacheBlend's gradual filtering), each
request with its own budgets; BlendPlan is its one-request case."""
from __future__ import annotations

import ctypes
from fractions import Fraction
from typing import Callable, List, NamedTuple, Optional, Sequence, Tuple

import torch

from lmcache_b200 import _native as N


class BlendSpec:
    """Check layers, strictly increasing, and the fraction of the retrieved tokens kept after each, in [0, 1] and not
    increasing: after check layer j the model recomputes the tokens that were not retrieved and k_j retrieved ones,
    k_j = min(ceil(ratios[j] * R), k_{j-1}) for R retrieved tokens, k_{-1} = R.  The ceiling is exact, of the ratio as
    written (its shortest decimal form) times R: 0.1 of 40 is 4 and 0.15 of 100 is 15.  BlendSpec([1], [0.15]) is
    CacheBlend's usual setting."""

    def __init__(self, check_layers: Sequence[int], ratios: Sequence[float]):
        layers, rs = list(check_layers), list(ratios)
        if not layers or len(layers) != len(rs):
            raise ValueError(f"a BlendSpec needs one ratio per check layer and at least one, got {layers!r} / {rs!r}")
        for c in layers:
            if isinstance(c, bool) or not isinstance(c, int) or c < 0:
                raise ValueError(f"check layers must be non-negative ints, got {c!r}")
        if any(b <= a for a, b in zip(layers, layers[1:])):
            raise ValueError(f"check layers must be strictly increasing, got {layers}")
        for r in rs:
            if isinstance(r, bool) or not isinstance(r, (int, float)) or not 0.0 <= r <= 1.0:
                raise ValueError(f"ratios must lie in [0, 1], got {r!r}")
        if any(b > a for a, b in zip(rs, rs[1:])):
            raise ValueError(f"ratios must not increase, got {rs}")
        self.check_layers = layers
        self.ratios = [float(r) for r in rs]

    def budgets(self, n_retrieved: int) -> List[int]:
        """k_j of every check layer for n_retrieved retrieved tokens"""
        out, prev = [], int(n_retrieved)
        for r in self.ratios:
            k = -((-Fraction(repr(r)) * n_retrieved) // 1)     # exact ceiling of the decimal ratio
            prev = min(int(k), prev)
            out.append(prev)
        return out

    def __repr__(self) -> str:
        return f"BlendSpec({self.check_layers}, {self.ratios})"


def check_sizes(spec: BlendSpec, n_tokens: int, n_retrieved: int) -> List[Tuple[int, int, int]]:
    """Per check layer j: (rows the model computes there, k_j, rows it computes after it).  All n_tokens at the first
    check; after check j the n_tokens - n_retrieved tokens that were not retrieved and k_j retrieved ones."""
    forced = n_tokens - n_retrieved
    out, n_in = [], n_tokens
    for k in spec.budgets(n_retrieved):
        out.append((n_in, k, forced + k))
        n_in = forced + k
    return out


def check_blend_dtype(dtype: torch.dtype) -> None:
    """TypeError unless the cache holds 16-bit keys: the segment calls that fill it refuse FP8"""
    if dtype not in (torch.bfloat16, torch.float16):
        raise TypeError(f"blend compares 16-bit keys only, not {dtype}: the segment retrieve it follows refuses FP8 KV")


def _check_spec(spec: BlendSpec, num_layers: int) -> None:
    if not isinstance(spec, BlendSpec):
        raise ValueError(f"spec must be a BlendSpec, got {type(spec).__name__}")
    if spec.check_layers[-1] >= num_layers:
        raise ValueError(f"check layer {spec.check_layers[-1]} outside the model's {num_layers} layers")


def _check_mask(ret_mask) -> None:
    if not isinstance(ret_mask, torch.Tensor) or ret_mask.dtype != torch.bool or ret_mask.dim() != 1 or \
            ret_mask.is_cuda:
        raise ValueError("ret_mask must be the 1-D bool CPU tensor a segment retrieve returns")


def check_blend_args(spec: BlendSpec, num_layers: int, n_tokens: int, ret_mask: torch.Tensor) -> None:
    """ValueError for a spec that is not a BlendSpec or names a layer outside [0, num_layers), and for a ret_mask that
    is not a 1-D bool CPU tensor of n_tokens entries"""
    _check_spec(spec, num_layers)
    _check_mask(ret_mask)
    if ret_mask.numel() != n_tokens:
        raise ValueError(f"ret_mask holds {ret_mask.numel()} tokens, the KV {n_tokens}")


def check_blend_batch_args(spec: BlendSpec, num_layers: int, n_tokens: int, ret_masks) -> None:
    """check_blend_args for a batch: ValueError unless ret_masks is a non-empty sequence (list or tuple) of 1-D bool
    CPU tensors, one per request in batch order, whose lengths add up to n_tokens"""
    _check_spec(spec, num_layers)
    if not isinstance(ret_masks, (list, tuple)) or not ret_masks:
        raise ValueError("ret_masks must be a non-empty list of the requests' ret_mask, in batch order")
    for m in ret_masks:
        _check_mask(m)
    total = sum(m.numel() for m in ret_masks)
    if total != n_tokens:
        raise ValueError(f"ret_masks hold {total} tokens, the batch's slot_mapping {n_tokens}")


def fresh_row_stride(fresh_k: torch.Tensor, n: int, C: int, dtype: torch.dtype, device: torch.device) -> int:
    """The row stride, in elements, of the model's fresh keys: n rows of C = H * D channels ([n, H, D] or [n, H * D],
    any row stride, each row contiguous) of the cache's dtype on its device.  ValueError otherwise."""
    if not isinstance(fresh_k, torch.Tensor):
        raise ValueError(f"fresh_k must be a tensor, got {type(fresh_k).__name__}")
    if fresh_k.dtype != dtype:
        raise ValueError(f"fresh_k is {fresh_k.dtype}, the cache {dtype}")
    if fresh_k.device != device:
        raise ValueError(f"fresh_k is on {fresh_k.device}, the cache on {device}")
    shape = tuple(fresh_k.shape)
    inner = 1
    for s in shape[1:]:
        inner *= s
    if len(shape) < 2 or shape[0] != n or inner != C:
        raise ValueError(f"fresh_k must hold {n} rows of H * D = {C} keys, got shape {shape}")
    step = 1
    for s, st in zip(reversed(shape[1:]), reversed(fresh_k.stride()[1:])):
        if s != 1 and st != step:
            raise ValueError("each row of fresh_k must be contiguous")
        step *= s
    return fresh_k.stride(0) if n > 1 else C


def deviation(view, layer: int, tok: torch.Tensor, fresh: torch.Tensor, stride: int, out: torch.Tensor,
              stream) -> None:
    """one b200kv_blend_deviation launch on `stream`: out[i] = the squared distance of fresh row i from the key row of
    view token tok[i] at `layer`"""
    N.check(N.lib().b200kv_blend_deviation(ctypes.byref(view.desc), layer, tok.numel(), ctypes.c_void_p(tok.data_ptr()),
                                           ctypes.c_void_p(fresh.data_ptr()), stride,
                                           ctypes.c_void_p(out.data_ptr()), stream.cuda_stream), "blend_deviation")


def select(dev: torch.Tensor, cand: torch.Tensor, k: int, n_out: int, stream) -> torch.Tensor:
    """b200kv_blend_select on `stream`: the rows with cand == 0, then the k candidates of largest dev, each part in
    row order; n_out = the forced rows + min(k, candidates), which the caller knows"""
    n = dev.numel()
    ws = torch.empty(max(1, N.lib().b200kv_blend_select_workspace_bytes(n)), dtype=torch.uint8, device=dev.device)
    rows = torch.empty(max(n_out, 1), dtype=torch.int64, device=dev.device)     # never a NULL pointer
    N.check(N.lib().b200kv_blend_select(ctypes.c_void_p(dev.data_ptr()), ctypes.c_void_p(cand.data_ptr()), n, int(k),
                                        ctypes.c_void_p(rows.data_ptr()), ctypes.c_void_p(ws.data_ptr()), ws.numel(),
                                        stream.cuda_stream), "blend_select")
    return rows[:n_out]


def select_batch(dev: torch.Tensor, cand: torch.Tensor, seg: torch.Tensor, k: torch.Tensor, n_out: int,
                 stream) -> torch.Tensor:
    """b200kv_blend_select_batch on `stream`: per segment s of rows [seg[s], seg[s+1]) (DEVICE int64 [B+1]), its rows
    with cand == 0, then its k[s] (DEVICE int64 [B]) candidates of largest dev, each part in row order, as global rows;
    n_out = the total of those blocks, which the caller knows"""
    n, B = dev.numel(), k.numel()
    ws = torch.empty(max(1, N.lib().b200kv_blend_select_batch_workspace_bytes(n, B)), dtype=torch.uint8,
                     device=dev.device)
    rows = torch.empty(max(n_out, 1), dtype=torch.int64, device=dev.device)     # never a NULL pointer
    N.check(N.lib().b200kv_blend_select_batch(ctypes.c_void_p(dev.data_ptr()), ctypes.c_void_p(cand.data_ptr()), n, B,
                                              ctypes.c_void_p(seg.data_ptr()), ctypes.c_void_p(k.data_ptr()),
                                              ctypes.c_void_p(rows.data_ptr()), ctypes.c_void_p(ws.data_ptr()),
                                              ws.numel(), stream.cuda_stream), "blend_select_batch")
    return rows[:n_out]


class BatchCheck(NamedTuple):
    """The per-request arithmetic of one check of a batch, known on the host from the masks and the spec: seg[r] is
    where request r's rows start among the check's input rows (B + 1 entries, the last = the rows in), k[r] its budget,
    out[r] where its block starts among the rows computed after the check (B + 1 entries, the last = the rows out)."""
    seg: List[int]
    k: List[int]
    out: List[int]


def _starts(lens: Sequence[int]) -> List[int]:
    out = [0]
    for n in lens:
        out.append(out[-1] + n)
    return out


def batch_checks(spec: BlendSpec, n_tokens: Sequence[int], n_retrieved: Sequence[int]) -> List[BatchCheck]:
    """BatchCheck of every check layer of spec for requests of n_tokens[r] tokens, n_retrieved[r] of them retrieved:
    check_sizes of each request, laid side by side"""
    per = [check_sizes(spec, n, r) for n, r in zip(n_tokens, n_retrieved)]
    return [BatchCheck(_starts([p[j][0] for p in per]), [p[j][1] for p in per], _starts([p[j][2] for p in per]))
            for j in range(len(spec.check_layers))]


class BatchBlendStep(NamedTuple):
    """What a check of a batch chose.  rows index the rows of the fresh keys passed, tokens are those rows' indices in
    the flattened batch, slots their cache slots (None for a dense view): one block per request in batch order, inside
    it the forced tokens (not retrieved), then the chosen retrieved ones, each part in token order.  cu_rows (DEVICE
    int32 [B + 1]) are the blocks' starts, the cu_seqlens_q of the rows computed after the check."""
    rows: torch.Tensor
    tokens: torch.Tensor
    slots: Optional[torch.Tensor]
    cu_rows: torch.Tensor


class BlendStep(NamedTuple):
    """What a check chose: `rows` index the rows of the fresh keys passed (the model subsets its hidden states with
    them), `tokens` are those rows' request tokens, `slots` their cache slots (None for a dense view).  Forced tokens
    (not retrieved) come first, then the chosen retrieved ones, each part in request order."""
    rows: torch.Tensor
    tokens: torch.Tensor
    slots: Optional[torch.Tensor]


class BatchBlendPlan:
    """A prefill batch's walk through the check layers of a BlendSpec, made by LMCacheEngine.blend_paged_batch: B
    requests flattened into one token dimension (vLLM's), sharing one view, one slot_mapping and one spec, each with its
    own ret_mask and budgets k_{j,r} = spec.budgets(R_r)[j].  The choice is per request; the GPU work of a check is one
    launch sequence for the whole batch.  rows_at(layer) are the batch tokens the model computes at `layer`: all of them
    up to and including the first check layer, the latest selection after it, one block per request in batch order.
    Every per-request array the checks need is computed on the host when the plan is made and uploaded in one copy,
    with the masks."""

    def __init__(self, view, ret_masks: Sequence[torch.Tensor], spec: BlendSpec,
                 slot_mapping: Optional[torch.Tensor] = None):
        self.view, self.spec = view, spec
        self.B = len(ret_masks)
        self.n_tokens_each = [m.numel() for m in ret_masks]
        self.n_retrieved_each = [int(m.sum()) for m in ret_masks]
        self.n_tokens, self.n_retrieved = sum(self.n_tokens_each), sum(self.n_retrieved_each)
        self.checks = batch_checks(spec, self.n_tokens_each, self.n_retrieved_each)
        self._cu_host = [_starts(self.n_tokens_each)] + [c.out for c in self.checks]
        n, C, B = self.n_tokens, len(self.checks), self.B
        # one upload: the masks (uint8), then seg and k of every check (int64), then the cu_rows of every stage (int32)
        mask = torch.cat([m.reshape(-1) for m in ret_masks]).to(torch.uint8)
        i64 = torch.tensor([v for c in self.checks for v in c.seg + c.k], dtype=torch.int64)
        i32 = torch.tensor([v for cu in self._cu_host for v in cu], dtype=torch.int32)
        o64 = -(-n // 8) * 8
        o32 = o64 + 8 * i64.numel()
        host = torch.zeros(o32 + 4 * i32.numel(), dtype=torch.uint8)
        host[:n] = mask
        host[o64:o32] = i64.view(torch.uint8)
        host[o32:] = i32.view(torch.uint8)
        dev = view.device
        buf = host.to(dev)
        self._mask = buf[:n]
        d64 = buf[o64:o32].view(torch.int64)
        self._seg = [d64[j * (2 * B + 1):j * (2 * B + 1) + B + 1] for j in range(C)]
        self._k = [d64[j * (2 * B + 1) + B + 1:(j + 1) * (2 * B + 1)] for j in range(C)]
        d32 = buf[o32:].view(torch.int32)
        self._cu = [d32[i * (B + 1):(i + 1) * (B + 1)] for i in range(C + 1)]
        self._all = torch.arange(n, dtype=torch.int64, device=dev)
        self._slot_mapping = None if slot_mapping is None else slot_mapping.to(dev)
        self._steps: list = []

    @property
    def num_checks(self) -> int:
        """checks run so far"""
        return len(self._steps)

    def _after(self, layer: int) -> int:
        """check layers before `layer`; ValueError for a layer outside the model or past a check not yet run"""
        if not 0 <= layer < self.view.L:
            raise ValueError(f"layer {layer} outside [0, {self.view.L})")
        j = sum(1 for c in self.spec.check_layers if c < layer)
        if j > len(self._steps):
            raise ValueError(f"layer {layer} follows check layer {self.spec.check_layers[j - 1]}, which has not been "
                             f"checked yet")
        return j

    def rows_at(self, layer: int) -> torch.Tensor:
        """DEVICE int64: the batch tokens the model computes at `layer`"""
        j = self._after(layer)
        return self._all if j == 0 else self._steps[j - 1].tokens

    def slots_at(self, layer: int) -> Optional[torch.Tensor]:
        """slot_mapping at rows_at(layer) (what vLLM's reshape_and_cache takes); None for a dense view"""
        j = self._after(layer)
        return self._slot_mapping if j == 0 else self._steps[j - 1].slots

    def cu_rows_at(self, layer: int) -> torch.Tensor:
        """DEVICE int32 [B + 1]: where each request's block starts in rows_at(layer), the cu_seqlens_q of FlashAttention's
        varlen call for that layer.  No sync: it was uploaded with the plan."""
        return self._cu[self._after(layer)]

    def lens_at(self, layer: int) -> List[int]:
        """the rows of each request in rows_at(layer), on the host: the differences of cu_rows_at(layer)"""
        cu = self._cu_host[self._after(layer)]
        return [b - a for a, b in zip(cu, cu[1:])]

    def _step(self, rows, tokens, slots, j):
        return BatchBlendStep(rows, tokens, slots, self._cu[j + 1])

    def check(self, layer: int, fresh_k: torch.Tensor, stream: Optional[torch.cuda.Stream] = None,
              reduce: Optional[Callable[[torch.Tensor], None]] = None):
        """The choice at check layer `layer` for every request of the batch: fresh_k ([n, H, D] or [n, H * D], the keys
        after the rotary embedding of rows_at(layer), in that order and the cache's dtype) against the cached key rows
        -- one deviation launch over all n rows, then reduce(dev) once if given (e.g. lambda d: dist.all_reduce(d,
        group=tp): the engine calls no collective), then one segmented select (a batch of one request takes
        b200kv_blend_select, the same choice), then the gathers of tokens and slots, all on `stream` (default: the
        current stream), with no host sync and the same operations whatever B.  Order it after wait_layer(layer,
        stream) of a layer-wise retrieve.  ValueError, before anything is enqueued, for a layer that is not the next
        check layer of the spec and for a fresh_k of another shape, dtype or device."""
        j = len(self._steps)
        if j >= len(self.spec.check_layers) or layer != self.spec.check_layers[j]:
            nxt = self.spec.check_layers[j] if j < len(self.spec.check_layers) else None
            raise ValueError(f"check at layer {layer}: the next check layer of {self.spec} is {nxt}")
        c = self.checks[j]
        n, n_out = c.seg[-1], c.out[-1]
        v = self.view
        stride = fresh_row_stride(fresh_k, n, v.H * v.D, v.dtype, v.device)
        toks = self._all if j == 0 else self._steps[j - 1].tokens
        stream = stream or torch.cuda.current_stream(v.device)
        with torch.cuda.device(v.device), torch.cuda.stream(stream):
            cand = self._mask if j == 0 else self._mask[toks]
            dev = torch.empty(n, dtype=torch.float32, device=v.device)
            deviation(v, layer, toks, fresh_k, stride, dev, stream)
            if reduce is not None:
                reduce(dev)
            if self.B == 1:
                rows = select(dev, cand, c.k[0], n_out, stream)
            else:
                rows = select_batch(dev, cand, self._seg[j], self._k[j], n_out, stream)
            tokens = toks[rows]
            slots = None if self._slot_mapping is None else self._slot_mapping[tokens]
        step = self._step(rows, tokens, slots, j)
        self._steps.append(step)
        return step


class BlendPlan(BatchBlendPlan):
    """One request's walk through the check layers of a BlendSpec, made by LMCacheEngine.blend_paged / blend: the
    batch plan of one request, whose checks return BlendSteps.  rows_at(layer) are the request tokens the model computes
    at `layer`: all of them up to and including the first check layer, the latest selection after it.  At each check
    layer, in order, the model computes its keys for rows_at(layer) and calls check() before it writes them to the cache
    (the check compares them with the cached rows); then it writes the KV it computed, as at every layer -- the engine
    adds no scatter."""

    def __init__(self, view, ret_mask: torch.Tensor, spec: BlendSpec, slot_mapping: Optional[torch.Tensor] = None):
        super().__init__(view, [ret_mask], spec, slot_mapping)
        self.sizes = check_sizes(spec, self.n_tokens, self.n_retrieved)

    def _step(self, rows, tokens, slots, j):
        return BlendStep(rows, tokens, slots)
