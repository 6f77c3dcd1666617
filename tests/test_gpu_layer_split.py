"""GPU: the layer-split entry points, driven through the raw C ABI and held to the CPU oracle.

* b200kv_encode_layers_plan / b200kv_encode_layers / b200kv_encode_layers_finish: random shapes (scalar and vector
  absmax, partial channel tiles), both dtypes, every kind of source, tok_begin, 1..256-token chunks, per-plane bins from
  4 to 32 (1-, 2-, 3- and 4-byte stream-header masks), random layer partitions issued in random order.  Every container
  is assembled from its fixed image and its plane rows and must be byte for byte b200kv_encode_chunks' container and,
  section by section, the oracle's.
* b200kv_decode_plan / b200kv_decode_layers on containers of every version, multi-group containers mixed with short
  ones, both rANS table layouts, vllm / huggingface / paged destinations in either dtype.
* The ABI maximum of 64 layers, the arena placement of the device (place_kernel) against its host statement
  (pipeline.arena_placement), the engine's layer-wise store when late layers overflow the arena,
  b200kv_plane_offsets_device against b200kv_plane_offsets, and the argument checks of the split entry points."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle as O
from test_gpu_codec import _bits_to_tensor, _eq_nan, _tensor_bits

pytestmark = pytest.mark.gpu
TDT = (torch.bfloat16, torch.float16)
FILL = 3.0                  # destination sentinel: rows a decode must not write keep it
ARENA_FILL = 0xAB           # arena / fixed-image sentinel: bytes no kernel may write keep it
BIN_SETS = {
    "any": list(range(4, 33)),          # odd values too: nb = 2 * (bins // 2)
    "small": list(range(4, 10)),        # nb <= 8: 1-byte stream-header masks, 4-step rANS search
    "wide": list(range(17, 26)),        # nb 16..24: 3-byte masks
}


def _N():
    from lmcache_b200 import _native as N
    return N


def _s():
    return torch.cuda.current_stream().cuda_stream


def _a16(x):
    return (int(x) + 15) & ~15


def _rand_bins(rng, L, mode="any"):
    vals = BIN_SETS[mode]
    return rng.choice(vals, size=L).astype(np.float32), rng.choice(vals, size=L).astype(np.float32)


def _rand_partition(rng, L):
    """a random partition of layers [0, L) into ranges, in a random order"""
    cuts = sorted(int(c) for c in rng.choice(np.arange(1, L), size=int(rng.integers(0, L)), replace=False)) if L > 1 else []
    b = [0] + cuts + [L]
    calls = [(b[i], b[i + 1]) for i in range(len(b) - 1)]
    return [calls[i] for i in rng.permutation(len(calls))]


def _kv(L, T, H, D, dt, seed):
    """[L,2,T,H,D] device KV of the given dtype and its bit pattern [L,2,T,C]"""
    bits = O.synth_kv_bits(L, T, H * D, seed=seed)
    x = _bits_to_tensor(bits, 0).float().to(TDT[dt]).reshape(L, 2, T, H, D).cuda()
    return x, _tensor_bits(x).reshape(L, 2, T, H * D)


def _source(kind, x, rng):
    """a KvView of x [L,2,T,H,D]: vllm blob, huggingface blob, tuple of 2L planes, or a paged cache (rows scattered by a
    random slot mapping, the rows no token maps to hold NaN)"""
    from lmcache_b200.codec import KvView
    L, _, T, H, D = x.shape
    if kind == "blob":
        return KvView.from_blob(x, "vllm")
    if kind == "hf":
        return KvView.from_blob(x.permute(0, 1, 3, 2, 4).contiguous(), "huggingface")
    if kind == "tuple":
        return KvView.from_tuple(tuple((x[l, 0].clone(), x[l, 1].clone()) for l in range(L)), "vllm")
    nslots = T + int(rng.integers(0, 64))
    slots = torch.from_numpy(rng.permutation(nslots)[:T].astype(np.int64)).cuda()
    caches = []
    for l in range(L):
        k = torch.full((nslots, H, D), float("nan"), dtype=x.dtype, device="cuda")
        v = torch.full_like(k, float("nan"))
        k[slots] = x[l, 0]
        v[slots] = x[l, 1]
        caches.append((k, v))
    return KvView.from_paged(caches, slots)


def _encode_chunks(view, tok_begin, n, cs, last, kb, vb, coder):
    """b200kv_encode_chunks: the n containers, as bytes"""
    N = _N()
    lib = N.lib()
    L, H, D = view.L, view.H, view.D
    stride = _a16(N.container_layout(L, H, D, cs, coder).max_total_bytes)
    out = torch.empty(n * stride, dtype=torch.uint8, device="cuda")
    sizes = torch.zeros(n, dtype=torch.int64, device="cuda")
    wsb = N.check(lib.b200kv_encode_workspace_bytes(L, H, D, cs, n, coder), "encode_workspace_bytes")
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    N.check(lib.b200kv_encode_chunks(ctypes.byref(view.desc), tok_begin, n, cs, last, N.float_array(kb), N.float_array(vb),
                                     coder, out.data_ptr(), stride, sizes.data_ptr(), ws.data_ptr(), wsb, _s()),
            "encode_chunks")
    torch.cuda.synchronize()
    sz = sizes.cpu().tolist()
    buf = out.cpu().numpy()
    assert all(0 < s <= stride for s in sz), sz
    return [bytes(buf[j * stride: j * stride + sz[j]]) for j in range(n)]


def _encode_layers(view, tok_begin, n, cs, last, kb, vb, calls, max_layers=None, arena_bytes=None, extra_stride=0,
                   guard=4096):
    """plan + one b200kv_encode_layers call per range of `calls` (in that order) + finish, into an arena and fixed
    images filled with ARENA_FILL (and `guard` bytes behind each).  Returns the outputs, copied back."""
    N = _N()
    lib = N.lib()
    L, H, D = view.L, view.H, view.D
    lo = N.container_layout(L, H, D, cs, N.CODER_RANS_COMPACT)
    stride = _a16(lo.off_payload) + extra_stride
    if arena_bytes is None:               # airtight: every chunk fits
        arena_bytes = n * (lo.max_total_bytes - lo.off_payload + 16 * L)
    arena = torch.full((arena_bytes + guard,), ARENA_FILL, dtype=torch.uint8, device="cuda")
    fixed = torch.full((n * stride + guard,), ARENA_FILL, dtype=torch.uint8, device="cuda")
    seg = torch.full((n * 2 * L * 2,), -7, dtype=torch.int64, device="cuda")
    sizes = torch.full((n,), -7, dtype=torch.int64, device="cuda")
    ml = max_layers or max(b - a for a, b in calls)
    wsb = N.check(lib.b200kv_encode_layers_workspace_bytes(L, H, D, cs, n, ml), "encode_layers_workspace_bytes")
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    plan = N.EncodePlan()
    N.check(lib.b200kv_encode_layers_plan(ctypes.byref(view.desc), tok_begin, n, cs, last, N.float_array(kb),
                                          N.float_array(vb), N.CODER_RANS_COMPACT, arena.data_ptr(), arena_bytes,
                                          fixed.data_ptr(), stride, seg.data_ptr(), sizes.data_ptr(), ml, ws.data_ptr(),
                                          wsb, ctypes.byref(plan), _s()), "encode_layers_plan")
    for a, b in calls:
        N.check(lib.b200kv_encode_layers(ctypes.byref(plan), a, b, _s()), "encode_layers")
    N.check(lib.b200kv_encode_layers_finish(ctypes.byref(plan), _s()), "encode_layers_finish")
    torch.cuda.synchronize()
    offp = [N.container_layout(L, H, D, cs if j < n - 1 else last, N.CODER_RANS_COMPACT).off_payload for j in range(n)]
    return dict(arena=arena.cpu().numpy(), fixed=fixed.cpu().numpy(), seg=seg.cpu().numpy().reshape(n, 2 * L, 2),
                sizes=sizes.cpu().numpy(), stride=stride, arena_bytes=arena_bytes, offp=offp, n=n, L=L, guard=guard)


def _status(r, j):
    """header.status of chunk j's fixed image"""
    s = r["stride"] * j
    return int(r["fixed"][s + 48: s + 52].view(np.uint32)[0])


def _containers(r):
    """the containers of the chunks that fit (sizes_out != 0), assembled from fixed image || 2L plane rows, after
    checking everything around them: fixed images zero past off_payload, the fixed buffer untouched past the n images,
    arena bytes outside every placed row -- behind the cursor, past arena_bytes -- untouched, rows inside the arena and
    adding up to sizes_out"""
    n, stride, arena, fixed = r["n"], r["stride"], r["arena"], r["fixed"]
    covered = np.zeros(arena.size, dtype=bool)
    out = []
    for j in range(n):
        img = fixed[j * stride: (j + 1) * stride]
        assert not img[r["offp"][j]:].any(), f"fixed image {j} is not zero past off_payload"
        rows = r["seg"][j]
        assert (rows[:, 1] >= 0).all()
        for o, m in rows:
            if o >= 0:
                assert o + m <= r["arena_bytes"], (j, o, m)
                covered[o: o + m] = True
        size = int(r["sizes"][j])
        if size == 0:
            out.append(None)
            continue
        assert (rows[:, 0] >= 0).all(), f"chunk {j} fits but has a row marked failed"
        assert _status(r, j) == 0
        assert size == r["offp"][j] + int(rows[:, 1].sum()), f"plane rows of chunk {j} do not add up to sizes_out"
        out.append(bytes(img[:r["offp"][j]]) + b"".join(bytes(arena[o: o + m]) for o, m in rows))
        assert len(out[-1]) == size
    assert (fixed[n * stride:] == ARENA_FILL).all(), "fixed images written past the n-th"
    assert (arena[~covered] == ARENA_FILL).all(), "arena bytes outside every plane row were written"
    return out


def _check_sections(raw, bits, dt, kb, vb, coder, nan_maxes=False):
    """every section of the container == the oracle's encode of the chunk bits [L,2,t,C]; returns that encode"""
    from lmcache_b200.codec import container_layout_of, parse_header
    L, _, t, C = bits.shape
    enc = O.encode_chunk(bits, dt, kb, vb, coder)
    hd = parse_header(raw)
    assert (hd.version, hd.L, hd.ntokens, hd.H * hd.D, hd.max_dtype) == (coder + 1, L, t, C, dt)
    lo = container_layout_of(hd)
    a = np.frombuffer(raw, np.uint8)
    maxes = a[lo.off_maxes: lo.off_maxes + 4 * L * t].view(np.uint16).reshape(2, L, t)
    if nan_maxes:
        assert _eq_nan(maxes, enc["maxes"], dt)
    else:
        assert np.array_equal(maxes, enc["maxes"])
    if coder == O.CODER_RANS_COMPACT:
        nb = O.nb_map(kb, vb, L)
        assert hd.nb == nb
        (b0, ln0, _), = enc["groups"]
        pl, half = O.v3_pack(enc["counts"], nb, ln0, b0)
        assert np.array_equal(a[lo.off_lengths: lo.off_lengths + half.size], half.ravel())
        assert bytes(a[lo.off_payload:]) == pl.tobytes()
    else:
        G = hd.ngroups
        cdf = a[lo.off_cdf: lo.off_cdf + 2 * L * C * 33 * 2].view(np.int16).reshape(2 * L, C, 33)
        assert np.array_equal(cdf, enc["cdf"])
        lengths = a[lo.off_lengths: lo.off_lengths + G * 2 * L * C * 4].view(np.int32).reshape(G, 2 * L, C)
        assert np.array_equal(lengths, np.stack([ln for _, ln, _ in enc["groups"]]))
        assert bytes(a[lo.off_payload:]) == np.concatenate([b for b, _, _ in enc["groups"]]).tobytes()
    return enc


class _Dest:
    """A decode destination for n_tok tokens, with rows the decode must not touch: a vllm or huggingface blob with `pad`
    tokens in front and 5 behind, or a paged cache whose slot mapping leaves rows out.  Filled with FILL."""

    def __init__(self, kind, L, H, D, n_tok, dt, pad, rng):
        from lmcache_b200.codec import KvView
        tdt = TDT[dt]
        self.kind, self.L, self.n, self.pad = kind, L, n_tok, pad
        if kind == "paged":
            nslots = n_tok + pad + 5
            self.slots = torch.from_numpy(rng.permutation(nslots)[:n_tok].astype(np.int64)).cuda()
            self.caches = [tuple(torch.full((nslots, H, D), FILL, dtype=tdt, device="cuda") for _ in range(2))
                           for _ in range(L)]
            self.view = KvView.from_paged(self.caches, self.slots)
            self.tok0 = 0
            self.unmapped = torch.ones(nslots, dtype=torch.bool, device="cuda")
            self.unmapped[self.slots] = False
        else:
            shape = (L, 2, pad + n_tok + 5, H, D) if kind == "vllm" else (L, 2, H, pad + n_tok + 5, D)
            self.out = torch.full(shape, FILL, dtype=tdt, device="cuda")
            self.view = KvView.from_blob(self.out, "vllm" if kind == "vllm" else "huggingface")
            self.tok0 = pad

    def tokens(self):
        """[L,2,n_tok,H,D]: the rows the decode writes"""
        if self.kind == "paged":
            return torch.stack([torch.stack([c[self.slots] for c in pair]) for pair in self.caches])
        o = self.out if self.kind == "vllm" else self.out.transpose(2, 3)
        return o[:, :, self.pad: self.pad + self.n]

    def bits(self):
        return _tensor_bits(self.tokens()).reshape(self.L, 2, self.n, -1)

    def rest_untouched(self) -> bool:
        if self.kind == "paged":
            return all(bool((c[self.unmapped] == FILL).all()) for pair in self.caches for c in pair)
        o = self.out if self.kind == "vllm" else self.out.transpose(2, 3)
        return bool((o[:, :, :self.pad] == FILL).all()) and bool((o[:, :, self.pad + self.n:] == FILL).all())


def _decode(raws, coder, dest, dst_tok, kb, vb, max_dtype, parts=None, after_first=None):
    """containers -> dest through b200kv_decode_chunks (parts None) or b200kv_decode_plan + one b200kv_decode_layers call
    per range of `parts`; after_first() runs after the first of those calls has completed.  Returns the status words."""
    from lmcache_b200.codec import parse_header
    N = _N()
    lib = N.lib()
    n = len(raws)
    offs, o = [], 0
    for r in raws:
        offs.append(o)
        o = _a16(o + len(r))
    total = o + N.READ_SLACK
    host = np.zeros(total, np.uint8)
    for r, off in zip(raws, offs):
        host[off: off + len(r)] = np.frombuffer(r, np.uint8)
    buf = torch.from_numpy(host).cuda()
    ntok = [int(parse_header(r).ntokens) for r in raws]
    v = dest.view
    wsb = N.check(lib.b200kv_decode_workspace_bytes(v.L, v.H, v.D, max(ntok), n), "decode_workspace_bytes")
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    status = torch.full((n,), 0x5555, dtype=torch.int32, device="cuda")
    args = (buf.data_ptr(), total, N.i64_array(offs), N.i64_array([len(r) for r in raws]), N.i32_array(ntok),
            N.i64_array(dst_tok), n, max_dtype, coder, ctypes.byref(v.desc), N.float_array(kb), N.float_array(vb),
            status.data_ptr(), ws.data_ptr(), wsb)
    if parts is None:
        N.check(lib.b200kv_decode_chunks(*args, _s()), "decode_chunks")
    else:
        plan = N.DecodePlan()
        N.check(lib.b200kv_decode_plan(*args, ctypes.byref(plan), _s()), "decode_plan")
        for i, (a, b) in enumerate(parts):
            N.check(lib.b200kv_decode_layers(ctypes.byref(plan), a, b, _s()), "decode_layers")
            if i == 0 and after_first is not None:
                torch.cuda.synchronize()
                after_first()
    torch.cuda.synchronize()
    return status.cpu().tolist()


# ------------------------------------------------------------------------------------------------ 1. encode sweep
SOURCES = ("blob", "hf", "tuple", "paged")


@pytest.mark.parametrize("seed", range(28))
def test_encode_layers_sweep_vs_encode_chunks_and_oracle(seed):
    """Random shapes, dtypes, sources, tok_begin, chunk sizes from 1 to 256, per-plane bins and layer partitions issued
    in random order: every container is b200kv_encode_chunks' bytes and the oracle's sections, nothing outside the plane
    rows is written; the containers decode through a random layer partition to the oracle's values, and nothing
    outside the mapped destination is written."""
    N = _N()
    rng = np.random.default_rng(4200 + seed)
    L = int(rng.integers(1, 7))
    H = int(rng.integers(1, 5))
    D = int(rng.choice([8, 20, 33, 64, 72, 80, 128]))
    T = int(rng.integers(1, 701))
    cs = 1 if seed % 7 == 3 else int(rng.choice([1, 16, 64, 200, 256]))
    dt = (seed // 4) % 2
    src = SOURCES[seed % 4]
    tok_begin = int(rng.integers(0, T)) if T > 1 and rng.random() < 0.5 else 0
    kb, vb = _rand_bins(rng, L, ("any", "small", "wide")[seed % 3])
    calls = _rand_partition(rng, L)
    max_layers = int(rng.integers(max(b - a for a, b in calls), L + 1))
    x, bits = _kv(L, T, H, D, dt, seed=700 + seed)
    view = _source(src, x, rng)
    n_tok = T - tok_begin
    n = (n_tok + cs - 1) // cs
    last = n_tok - (n - 1) * cs
    want = _encode_chunks(view, tok_begin, n, cs, last, kb, vb, N.CODER_RANS_COMPACT)
    r = _encode_layers(view, tok_begin, n, cs, last, kb, vb, calls, max_layers=max_layers,
                       extra_stride=int(rng.choice([0, 16, 48])))
    got = _containers(r)
    encs = []
    for j in range(n):
        assert got[j] == want[j], (seed, j)
        t0 = tok_begin + j * cs
        encs.append(_check_sections(got[j], bits[:, :, t0: t0 + (cs if j < n - 1 else last)], dt, kb, vb,
                                    O.CODER_RANS_COMPACT))
    out_dt = int(rng.integers(0, 2))
    dest = _Dest(str(rng.choice(["vllm", "hf", "paged"])), L, H, D, n_tok, out_dt, int(rng.integers(0, 40)), rng)
    status = _decode(got, N.CODER_RANS_COMPACT, dest, [dest.tok0 + j * cs for j in range(n)], kb, vb, dt,
                     parts=_rand_partition(rng, L))
    assert status == [0] * n
    wantd = np.concatenate([O.decode_chunk(e, dt, kb, vb, out_dt) for e in encs], axis=2)
    assert np.array_equal(dest.bits(), wantd), seed
    assert dest.rest_untouched(), "decode wrote outside its destination rows"


@pytest.mark.parametrize("dt", [0, 1])
@pytest.mark.parametrize("H,D", [(1, 128), (2, 33)])
def test_encode_decode_layers_extreme_rows(dt, H, D):
    """zero layers, +/-inf and NaN entries, a near-max column: layer-split encode == encode_chunks == oracle sections
    (maxima with NaN matching NaN), split decode == oracle"""
    N = _N()
    L, T, cs = 4, 100, 64
    C = H * D
    big = 1e30 if dt == 0 else 6e4
    x = torch.randn((L, 2, T, H, D), generator=torch.Generator().manual_seed(dt * 100 + D)).to(TDT[dt])
    x[0] = 0
    x[1, 0, 3, 0, 5] = float("inf")
    x[1, 1, 70, 0, 6] = float("-inf")
    x[2, 1, 4, 0, 6] = float("nan")
    x[2, 0, 80:, 0, 1] = float("nan")
    x[3, 0, :, 0, 7] = big
    bits = x.view(torch.int16).numpy().view(np.uint16).reshape(L, 2, T, C)
    x = x.cuda()
    view = _source("blob", x, None)
    kb, vb = np.array([4, 9, 32, 24], np.float32), np.array([17, 5, 16, 31], np.float32)
    n, last = 2, T - cs
    want = _encode_chunks(view, 0, n, cs, last, kb, vb, N.CODER_RANS_COMPACT)
    got = _containers(_encode_layers(view, 0, n, cs, last, kb, vb, [(2, 4), (0, 1), (1, 2)]))
    assert got == want
    encs = [_check_sections(got[j], bits[:, :, j * cs: j * cs + (cs if j == 0 else last)], dt, kb, vb,
                            O.CODER_RANS_COMPACT, nan_maxes=True) for j in range(n)]
    dest = _Dest("vllm", L, H, D, T, dt, 3, None)
    assert _decode(got, N.CODER_RANS_COMPACT, dest, [3, 3 + cs], kb, vb, dt, parts=[(1, 3), (3, 4), (0, 1)]) == [0, 0]
    wantd = np.concatenate([O.decode_chunk(e, dt, kb, vb, dt) for e in encs], axis=2)
    assert _eq_nan(dest.bits(), wantd, dt)
    assert dest.rest_untouched()


# ------------------------------------------------------------------------------------------------ 2. every version
@pytest.mark.parametrize("coder,table", [(0, None), (1, "rows"), (1, "transposed"), (2, "rows"), (2, "transposed")])
def test_decode_layers_every_container_version(coder, table, monkeypatch):
    """containers of every version from b200kv_encode_chunks (multi-group ones of 512 and 700 tokens in one call with a
    37-token one for versions 1 / 2), C = 240 (a partial channel tile), random bins: their sections == the oracle's, and
    any layer partition of the decode writes what b200kv_decode_chunks writes == the oracle's values, into every kind of
    destination; after the first layer range, the other layers are untouched"""
    N = _N()
    if table is not None:
        monkeypatch.setenv("B200KV_DECODE_TABLE", table)
    rng = np.random.default_rng(31 + 7 * coder + (table == "transposed"))
    L, H, D = 5, 3, 80
    kb, vb = _rand_bins(rng, L)
    if coder == N.CODER_RANS_COMPACT:
        pieces = [(0, 3, 256, 256), (768, 2, 200, 13)]           # (tok_begin, n, chunk, last): 256, 256, 256, 200, 13
    else:
        pieces = [(0, 2, 512, 512), (1024, 2, 700, 37)]          # 512, 512, 700, 37 tokens: 2, 2, 3, 1 groups
    T = pieces[-1][0] + (pieces[-1][1] - 1) * pieces[-1][2] + pieces[-1][3]
    x, bits = _kv(L, T, H, D, 0, seed=90 + coder)
    view = _source("blob", x, rng)
    raws, ntoks, starts = [], [], []
    for tb, n, cs, last in pieces:
        raws += _encode_chunks(view, tb, n, cs, last, kb, vb, coder)
        for j in range(n):
            starts.append(tb + j * cs)
            ntoks.append(cs if j < n - 1 else last)
    encs = [_check_sections(raw, bits[:, :, s: s + t], 0, kb, vb, coder) for raw, s, t in zip(raws, starts, ntoks)]
    for trial, kind in enumerate(("vllm", "hf", "paged")):
        out_dt = trial % 2
        wantd = np.concatenate([O.decode_chunk(e, 0, kb, vb, out_dt) for e in encs], axis=2)
        whole = _Dest(kind, L, H, D, T, out_dt, 7, np.random.default_rng(trial))
        assert _decode(raws, coder, whole, [whole.tok0 + s for s in starts], kb, vb, 0) == [0] * len(raws)
        split = _Dest(kind, L, H, D, T, out_dt, 7, np.random.default_rng(trial))
        parts = _rand_partition(rng, L)
        if len(parts) == 1:
            parts = [(2, 4), (0, 2), (4, 5)]

        def untouched_after_first():
            a, b = parts[0]
            tok = split.tokens()
            others = [l for l in range(L) if not a <= l < b]
            assert bool((tok[others] == FILL).all()), "decode_layers wrote layers outside its range"
            assert np.array_equal(split.bits()[a:b], wantd[a:b])
        assert _decode(raws, coder, split, [split.tok0 + s for s in starts], kb, vb, 0, parts=parts,
                       after_first=untouched_after_first) == [0] * len(raws)
        assert torch.equal(split.tokens().view(torch.int16), whole.tokens().view(torch.int16))
        assert np.array_equal(split.bits(), wantd), kind
        assert split.rest_untouched() and whole.rest_untouched()


# ------------------------------------------------------------------------------------------------ 3. L = 64
@pytest.mark.parametrize("D", [20, 128])
def test_sixty_four_layers(D):
    """the ABI maximum (128 planes): encode as one call of 64 layers, as 64 single-layer calls in reverse order and as
    [1, 62, 1]; decode split the same ways; host and device plane offsets -- all against encode_chunks and the oracle"""
    N = _N()
    lib = N.lib()
    rng = np.random.default_rng(D)
    L, H, T, cs = 64, 1, 300, 256
    n, last = 2, T - cs
    kb, vb = _rand_bins(rng, L)
    x, bits = _kv(L, T, H, D, 0, seed=D)
    view = _source("blob", x, rng)
    want = _encode_chunks(view, 0, n, cs, last, kb, vb, N.CODER_RANS_COMPACT)
    encs = [_check_sections(want[j], bits[:, :, j * cs: j * cs + (cs if j == 0 else last)], 0, kb, vb,
                            O.CODER_RANS_COMPACT) for j in range(n)]
    splits = ([(0, 64)], [(l, l + 1) for l in range(63, -1, -1)], [(0, 1), (1, 63), (63, 64)])
    for calls in splits:
        assert _containers(_encode_layers(view, 0, n, cs, last, kb, vb, calls)) == want, len(calls)
    wantd = np.concatenate([O.decode_chunk(e, 0, kb, vb, 0) for e in encs], axis=2)
    for parts in splits:
        dest = _Dest("vllm", L, H, D, T, 0, 2, None)
        assert _decode(want, N.CODER_RANS_COMPACT, dest, [2, 2 + cs], kb, vb, 0, parts=parts) == [0, 0]
        assert np.array_equal(dest.bits(), wantd) and dest.rest_untouched()
    stride = _a16(max(len(w) for w in want))
    host = np.zeros(n * stride, np.uint8)
    for j, w in enumerate(want):
        host[j * stride: j * stride + len(w)] = np.frombuffer(w, np.uint8)
    out = torch.full((n, N.MAX_PLANES + 1), -5, dtype=torch.int64, device="cuda")
    buf = torch.from_numpy(host).cuda()
    N.check(lib.b200kv_plane_offsets_device(buf.data_ptr(), stride, n, out.data_ptr(), _s()), "plane_offsets_device")
    torch.cuda.synchronize()
    dev = out.cpu().numpy()
    for j, w in enumerate(want):
        a = np.frombuffer(w, np.uint8)
        o = np.zeros(N.MAX_PLANES + 1, np.int64)
        assert lib.b200kv_plane_offsets(a.ctypes.data, a.size, o.ctypes.data, o.size) == 0
        assert o[2 * L] == len(w) and np.array_equal(dev[j], o)


# ------------------------------------------------------------------------------------------------ 4. arena placement
def _plane_sizes(view, tok_begin, n, cs, last, kb, vb):
    """bytes of every (chunk, plane), and the full containers, from a run with an airtight arena"""
    L = view.L
    r = _encode_layers(view, tok_begin, n, cs, last, kb, vb, [(l, l + 1) for l in range(L)])
    full = _containers(r)
    assert all(c is not None for c in full)
    return r["seg"][:, :, 1].copy(), full


def _call_bytes(sz, calls, L):
    """seg_bytes[c, j] of arena_placement: chunk j's bytes in call c (its K planes, then its V planes)"""
    return np.array([[int(sz[j, a:b].sum() + sz[j, L + a:L + b].sum()) for j in range(sz.shape[0])] for a, b in calls],
                    dtype=np.int64)


def _check_placement(view, tok_begin, n, cs, last, kb, vb, calls, arena, sz, full):
    """one run at `arena` bytes against pipeline.arena_placement; returns (chunks that fit, the latest call in which a
    chunk failed, or the number of calls when none did)"""
    from lmcache_b200.pipeline import arena_placement
    L = view.L
    layers = [b - a for a, b in calls]
    seg_bytes = _call_bytes(sz, calls, L)
    base, fit = arena_placement(seg_bytes, arena, layers)
    # Row c of the device is the placement as it stood after call c: the host model with the later calls emptied (which
    # changes no decision up to c).  A chunk placed in call c and failed in a later one keeps its row of call c.
    want_base = np.empty_like(base)
    for c in range(len(calls)):
        head = seg_bytes.copy()
        head[c + 1:] = 0
        want_base[c] = arena_placement(head, arena, layers)[0][c]
    assert np.array_equal(want_base[-1], base[-1])
    fail_call = [int(np.argmax(want_base[:, j] < 0)) if j >= fit else len(calls) for j in range(n)]
    r = _encode_layers(view, tok_begin, n, cs, last, kb, vb, calls, arena_bytes=arena)
    got = _containers(r)
    assert [c is not None for c in got] == [j < fit for j in range(n)], (arena, fit)
    for j in range(n):
        if j < fit:
            assert got[j] == full[j]
        else:
            assert int(r["sizes"][j]) == 0 and _status(r, j) & 16, j
        assert np.array_equal(r["seg"][j, :, 1], sz[j])
    for c, (a, b) in enumerate(calls):
        planes = list(range(a, b)) + list(range(L + a, L + b))
        for j in range(n):
            rows = r["seg"][j, planes]
            if want_base[c, j] >= 0:              # placed at the host model's base, its planes back to back
                assert rows[0, 0] == want_base[c, j], (arena, c, j)
                assert np.array_equal(rows[:, 0], rows[0, 0] + np.concatenate([[0], np.cumsum(rows[:-1, 1])])), (c, j)
            else:                                 # failed in this call or an earlier one
                assert c >= fail_call[j] and (rows[:, 0] == -1).all(), (arena, c, j)
    return fit, max(fail_call[fit:], default=len(calls))


@pytest.mark.parametrize("order", ["cheap_first", "random"])
def test_arena_placement_matches_host_model(order):
    """Device arena placement == pipeline.arena_placement at the exact total, one byte less and random sizes in between,
    for single-layer calls and a random partition.  With cheap layers (bins 4) encoded first the reserve underestimates
    the later layers, so chunks are accepted early and fail late: sizes_out 0, header status bit 16, rows -1 from the
    failing call on."""
    rng = np.random.default_rng(5 if order == "cheap_first" else 6)
    L, H, D, cs, n = 8, 2, 64, 128, 12
    T = n * cs - 50
    last = T - (n - 1) * cs
    if order == "cheap_first":
        kb = vb = np.array([4] * 4 + [32] * 4, np.float32)
    else:
        kb, vb = _rand_bins(rng, L)
    g = torch.Generator(device="cuda").manual_seed(9)
    x = (torch.rand((L, 2, T, H, D), device="cuda", generator=g) * 2 - 1).to(torch.bfloat16)
    view = _source("blob", x, rng)
    sz, full = _plane_sizes(view, 0, n, cs, last, kb, vb)
    late = 0
    partitions = [[(l, l + 1) for l in range(L)], [(0, 3), (3, 4), (4, 8)]]
    if order == "random":
        partitions.append(_rand_partition(rng, L))
    for calls in partitions:
        total = int(sum(_a16(v) for v in _call_bytes(sz, calls, L).ravel()))
        arenas = [total, total - 1] + [int(a) for a in rng.integers(total // 4, total, size=4)]
        for arena in arenas:
            fit, fail_call = _check_placement(view, 0, n, cs, last, kb, vb, calls, arena, sz, full)
            if arena == total - 1:
                assert fit < n                    # the bytes of every chunk need the whole total
            late += 0 < fail_call < len(calls)
    if order == "cheap_first":
        assert late >= 2, "no run failed a chunk in a later call than the first"


@pytest.mark.parametrize("L", [1, 2])
def test_place_kernel_second_batch(L):
    """1100 one-token chunks: place_kernel's loop takes a second batch of 1024; the cut at chunk 1050 (arena exactly
    enough for 1050, and one byte less) matches the host model"""
    from lmcache_b200.pipeline import arena_placement
    rng = np.random.default_rng(L)
    H, D, n = 1, 8, 1100
    kb, vb = _rand_bins(rng, L)
    x, _ = _kv(L, n, H, D, 0, seed=L)
    view = _source("blob", x, rng)
    sz, full = _plane_sizes(view, 0, n, 1, 1, kb, vb)
    calls = [(l, l + 1) for l in range(L)]
    seg_bytes = _call_bytes(sz, calls, L)
    total = int(sum(_a16(v) for v in seg_bytes.ravel()))
    if L == 1:                                     # one call: what fits grows with the arena
        lo, hi = 0, total
        while lo < hi:                             # the smallest arena in which 1050 chunks fit
            mid = (lo + hi) // 2
            if arena_placement(seg_bytes, mid, [1])[1] >= 1050:
                hi = mid
            else:
                lo = mid + 1
        arenas = (lo, lo - 1)
    else:                                          # the reserve makes it non-monotone: take a size that cuts in batch 2
        cands = [int(total * f) for f in np.linspace(0.5, 1.5, 401)]
        arenas = (next(a for a in cands if 1024 < arena_placement(seg_bytes, a, [1] * L)[1] < n),)
    fits = [_check_placement(view, 0, n, 1, 1, kb, vb, calls, a, sz, full)[0] for a in arenas + (4 * total,)]
    assert all(1024 < f < n for f in fits[:-1]) and fits[-1] == n
    if L == 1:
        assert fits[0] == 1050 > fits[1]


# ------------------------------------------------------------------------------------------------ 5. engine
@pytest.mark.parametrize("tier", ["host", "disk"])
def test_engine_layerwise_store_late_overflow(tier, tmp_path, autorelease, monkeypatch):
    """store_paged_layerwise, 12 layers with the model's bins, saved in reverse order (the 16-bin layers first) under a
    tight arena: the retrieve returns a bit-exact prefix of whole chunks, and no chunk past it lands"""
    from lmcache_b200.cache_engine import LMCacheEngine
    from test_gpu_host_tier import _blob_of, _meta, _want
    from test_gpu_layerwise_store import _cfg, _landed
    L, H, D, cs, T = 12, 2, 128, 256, 16 * 256
    g = torch.Generator(device="cuda").manual_seed(12)
    kv = (torch.rand((L, 2, T, H, D), device="cuda", generator=g) * 2 - 1).to(torch.bfloat16)
    tokens = torch.randint(0, 32000, (T,), device="cuda", generator=None)
    nblk = T // 16 + 4
    slots = torch.randperm(nblk * 16, device="cuda")[:T]
    caches = [(torch.full((nblk, 16, H, D), float("nan"), device="cuda", dtype=torch.bfloat16),
               torch.full((nblk, 16, H, D), float("nan"), device="cuda", dtype=torch.bfloat16)) for _ in range(L)]
    for l in range(L):
        caches[l][0].view(-1, H, D)[slots] = kv[l, 0]
        caches[l][1].view(-1, H, D)[slots] = kv[l, 1]
    ref = autorelease(LMCacheEngine(_cfg(tier, tmp_path, "a"), _meta()))
    ref.store_paged(tokens, caches, slots)
    a = _landed(ref)
    total = sum(len(c) for c, _ in a.values())
    mb = max(1, (total // 2) >> 20)
    assert (mb << 20) < total
    monkeypatch.setenv("LMCACHE_B200_LAYERWISE_STORE_MB", str(mb))
    eng = autorelease(LMCacheEngine(_cfg(tier, tmp_path, "b"), _meta()))
    h = eng.store_paged_layerwise(tokens, caches, slots)
    for l in range(L - 1, -1, -1):
        h.save_layer(l)
    h.finish()
    ret, mask = eng.retrieve(tokens)
    torch.cuda.synchronize()
    got = int(mask.sum())
    assert 0 < got < T and got % cs == 0
    assert bool(mask[:got].all()) and not bool(mask[got:].any())
    want = _want(tuple((kv[l, 0], kv[l, 1]) for l in range(L)), "vllm", cs, got)
    assert torch.equal(_blob_of(ret).view(torch.int16), want.view(torch.int16))
    b = _landed(eng)
    assert len(b) == got // cs and all(a[k] == b[k] for k in b)


# ------------------------------------------------------------------------------------------------ 6. plane offsets
def test_plane_offsets_device_across_shapes():
    """a few hundred containers in one launch -- C % 16 != 0 (scalar sums), t = 1, L = 64, partial tiles -- equal the host
    b200kv_plane_offsets; -1 in entry 0 for each kind of input it rejects"""
    N = _N()
    lib = N.lib()
    rng = np.random.default_rng(77)
    raws = []
    for L, H, D, T, cs in [(1, 1, 8, 240, 1), (3, 2, 20, 300, 64), (2, 3, 33, 256, 256), (4, 2, 64, 200, 200),
                           (5, 3, 80, 129, 128), (64, 1, 20, 44, 44), (64, 1, 128, 3, 1), (6, 1, 72, 70, 16)]:
        kb, vb = _rand_bins(rng, L)
        x, _ = _kv(L, T, H, D, int(rng.integers(0, 2)), seed=L * 1000 + D)
        n = (T + cs - 1) // cs
        raws += _encode_chunks(_source("blob", x, rng), 0, n, cs, T - (n - 1) * cs, kb, vb, N.CODER_RANS_COMPACT)
    n_valid = len(raws)
    assert n_valid > 250
    bad = []

    def mutate(src, pos, fmt, val):
        b = bytearray(src)
        np.frombuffer(b, np.uint8)[pos: pos + np.dtype(fmt).itemsize].view(fmt)[0] = val
        return bytes(b)
    from lmcache_b200.codec import container_layout_of, parse_header
    for k, base in enumerate((raws[3], raws[241], raws[-1])):          # C = 8 at t = 1, C = 40, C = 72
        bad.append(mutate(base, 4, np.uint32, 2))                   # version 2
        bad.append(mutate(base, 8, np.uint32, 0))                   # L = 0
        bad.append(mutate(base, 8, np.uint32, 65))                  # L = 65
        bad.append(mutate(base, 20, np.uint32, 257))                # t = 257
        lo = container_layout_of(parse_header(base))
        hd = parse_header(base)
        half = np.frombuffer(base, np.uint8)[lo.off_lengths: lo.off_lengths + 2 * hd.L * hd.H * hd.D]
        i = int(np.flatnonzero(half < 255)[k])
        bad.append(mutate(base, lo.off_lengths + i, np.uint8, half[i] + 1))       # one half-length one too long
        i = int(np.flatnonzero(half > 0)[-1 - k])
        bad.append(mutate(base, lo.off_lengths + i, np.uint8, half[i] - 1))       # one too short
    allc = raws + bad
    stride = _a16(max(len(c) for c in allc))
    host = np.zeros(len(allc) * stride, np.uint8)
    for j, c in enumerate(allc):
        host[j * stride: j * stride + len(c)] = np.frombuffer(c, np.uint8)
    buf = torch.from_numpy(host).cuda()
    out = torch.full((len(allc), N.MAX_PLANES + 1), -5, dtype=torch.int64, device="cuda")
    N.check(lib.b200kv_plane_offsets_device(buf.data_ptr(), stride, len(allc), out.data_ptr(), _s()),
            "plane_offsets_device")
    torch.cuda.synchronize()
    dev = out.cpu().numpy()
    for j, c in enumerate(allc):
        a = np.frombuffer(c, np.uint8)
        o = np.zeros(N.MAX_PLANES + 1, np.int64)
        rc = lib.b200kv_plane_offsets(a.ctypes.data, a.size, o.ctypes.data, o.size)
        if j < n_valid:
            L = int(a[8:12].view(np.uint32)[0])
            assert rc == 0 and o[2 * L] == len(c)
            assert np.array_equal(dev[j, :2 * L + 1], o[:2 * L + 1]), j
        else:
            assert rc != 0, j
            assert dev[j, 0] == -1, j


# ------------------------------------------------------------------------------------------------ 7. ABI checks
def test_split_entry_points_reject_bad_arguments():
    """every bad argument of the split entry points returns < 0 with a message and enqueues nothing: the buffers keep
    their sentinels, and the same plan / buffers then produce encode_chunks' containers and the oracle's decode"""
    N = _N()
    lib = N.lib()
    L, H, D, T, cs = 4, 1, 64, 300, 256
    n, last = 2, T - cs
    kb, vb = np.array([16, 5, 32, 9], np.float32), np.array([8, 24, 17, 32], np.float32)
    kba, vba = N.float_array(kb), N.float_array(vb)
    x, bits = _kv(L, T, H, D, 0, seed=3)
    view = _source("blob", x, None)
    want = _encode_chunks(view, 0, n, cs, last, kb, vb, N.CODER_RANS_COMPACT)
    lo = N.container_layout(L, H, D, cs, N.CODER_RANS_COMPACT)
    stride = _a16(lo.off_payload)
    arena_bytes = n * (lo.max_total_bytes - lo.off_payload + 16 * L)
    arena = torch.full((arena_bytes,), ARENA_FILL, dtype=torch.uint8, device="cuda")
    fixed = torch.full((n * stride + 64,), ARENA_FILL, dtype=torch.uint8, device="cuda")
    seg = torch.full((n * 2 * L * 2,), -7, dtype=torch.int64, device="cuda")
    sizes = torch.full((n,), -7, dtype=torch.int64, device="cuda")
    wsb = lib.b200kv_encode_layers_workspace_bytes(L, H, D, cs, n, 2)
    ws = torch.full((wsb,), 0xCD, dtype=torch.uint8, device="cuda")
    good = dict(kv=ctypes.byref(view.desc), tok_begin=0, n=n, cs=cs, last=last, kb=kba, vb=vba, coder=N.CODER_RANS_COMPACT,
                arena=arena.data_ptr(), arena_bytes=arena_bytes, fixed=fixed.data_ptr(), stride=stride,
                seg=seg.data_ptr(), sizes=sizes.data_ptr(), max_layers=2, ws=ws.data_ptr(), wsb=wsb)

    def plan_rc(plan, **over):
        a = dict(good, **over)
        return lib.b200kv_encode_layers_plan(a["kv"], a["tok_begin"], a["n"], a["cs"], a["last"], a["kb"], a["vb"],
                                             a["coder"], a["arena"], a["arena_bytes"], a["fixed"], a["stride"], a["seg"],
                                             a["sizes"], a["max_layers"], a["ws"], a["wsb"], plan, _s())

    def untouched():
        torch.cuda.synchronize()
        return (bool((fixed == ARENA_FILL).all()) and bool((ws == 0xCD).all()) and bool((arena == ARENA_FILL).all())
                and bool((seg == -7).all()) and bool((sizes == -7).all()))

    def refused(rc):
        return rc < 0 and len(N.last_error()) > 0

    plan = N.EncodePlan()
    for over in (dict(coder=0), dict(coder=1), dict(cs=257, last=257), dict(max_layers=0), dict(max_layers=L + 1),
                 dict(fixed=fixed.data_ptr() + 8), dict(stride=stride + 8), dict(stride=_a16(lo.off_payload) - 16),
                 dict(wsb=wsb - 1), dict(arena=None), dict(fixed=None), dict(seg=None), dict(sizes=None)):
        assert refused(plan_rc(ctypes.byref(plan), **over)), over
        assert refused(lib.b200kv_encode_layers(ctypes.byref(plan), 0, 1, _s())), over      # the plan was not made
        assert untouched(), over
    assert refused(plan_rc(None))
    assert refused(lib.b200kv_encode_layers(ctypes.byref(N.EncodePlan()), 0, 1, _s()))     # never planned
    assert refused(lib.b200kv_encode_layers_finish(ctypes.byref(N.EncodePlan()), _s()))
    assert untouched()
    N.check(plan_rc(ctypes.byref(plan)), "encode_layers_plan")
    for a, b in ((1, 1), (2, 1), (-1, 1), (3, L + 1), (L, L + 1), (0, 3)):    # empty, reversed, outside, > max_layers
        assert refused(lib.b200kv_encode_layers(ctypes.byref(plan), a, b, _s())), (a, b)
    N.check(lib.b200kv_encode_layers(ctypes.byref(plan), 2, 4, _s()), "encode_layers")
    assert refused(lib.b200kv_encode_layers(ctypes.byref(plan), 3, 4, _s()))                # encoded before
    N.check(lib.b200kv_encode_layers(ctypes.byref(plan), 0, 1, _s()), "encode_layers")
    assert refused(lib.b200kv_encode_layers_finish(ctypes.byref(plan), _s()))              # layer 1 missing
    torch.cuda.synchronize()
    assert bool((sizes == -7).all()), "a refused finish wrote sizes_out"
    N.check(lib.b200kv_encode_layers(ctypes.byref(plan), 1, 2, _s()), "encode_layers")
    N.check(lib.b200kv_encode_layers_finish(ctypes.byref(plan), _s()), "encode_layers_finish")
    torch.cuda.synchronize()
    r = dict(arena=arena.cpu().numpy(), fixed=fixed.cpu().numpy(), seg=seg.cpu().numpy().reshape(n, 2 * L, 2),
             sizes=sizes.cpu().numpy(), stride=stride, arena_bytes=arena_bytes, n=n, L=L,
             offp=[lo.off_payload, N.container_layout(L, H, D, last, N.CODER_RANS_COMPACT).off_payload])
    got = _containers(r)
    assert got == want

    # decode_layers
    dest = _Dest("vllm", L, H, D, T, 0, 4, None)
    host =np.zeros(_a16(len(got[0])) + len(got[1]) + N.READ_SLACK, np.uint8)
    offs = [0, _a16(len(got[0]))]
    for o, c in zip(offs, got):
        host[o: o + len(c)] = np.frombuffer(c, np.uint8)
    buf = torch.from_numpy(host).cuda()
    dws = torch.empty(lib.b200kv_decode_workspace_bytes(L, H, D, cs, n), dtype=torch.uint8, device="cuda")
    status = torch.full((n,), 0x5555, dtype=torch.int32, device="cuda")
    dplan = N.DecodePlan()
    assert refused(lib.b200kv_decode_layers(ctypes.byref(dplan), 0, L, _s()))               # never planned
    N.check(lib.b200kv_decode_plan(buf.data_ptr(), host.size, N.i64_array(offs), N.i64_array([len(c) for c in got]),
                                   N.i32_array([cs, last]), N.i64_array([4, 4 + cs]), n, 0, N.CODER_RANS_COMPACT,
                                   ctypes.byref(dest.view.desc), kba, vba, status.data_ptr(), dws.data_ptr(), dws.numel(),
                                   ctypes.byref(dplan), _s()), "decode_plan")
    for a, b in ((0, 0), (2, 1), (-1, 2), (0, L + 1), (L, L + 1)):
        assert refused(lib.b200kv_decode_layers(ctypes.byref(dplan), a, b, _s())), (a, b)
    torch.cuda.synchronize()
    assert bool((dest.tokens() == FILL).all()), "a refused decode_layers wrote its destination"
    N.check(lib.b200kv_decode_layers(ctypes.byref(dplan), 1, L, _s()), "decode_layers")
    N.check(lib.b200kv_decode_layers(ctypes.byref(dplan), 0, 1, _s()), "decode_layers")
    torch.cuda.synchronize()
    assert status.cpu().tolist() == [0, 0]
    wantd = np.concatenate([O.decode_chunk(O.encode_chunk(bits[:, :, j * cs: j * cs + t], 0, kb, vb, O.CODER_RANS_COMPACT),
                                           0, kb, vb, 0) for j, t in enumerate((cs, last))], axis=2)
    assert np.array_equal(dest.bits(), wantd) and dest.rest_untouched()
