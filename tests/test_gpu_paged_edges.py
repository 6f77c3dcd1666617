"""GPU: the split (PagedAttention / xFormers) and block-strided (FlashInfer) paged movers against the torch statement
of paged_edges, at every branch of the split kernel's launch rule (paged_edges.CASES): pack_chunks and
pack_chunks_layers give ref_pack's bytes and leave the rest of the chunk buffer as it was; unpack_chunks and
unpack_chunks_layers into sentinel-filled caches give ref_unpack's caches byte for byte.  Then the strided layout
through the mover and both codecs, and an engine round trip through the lossless host tier from a split cache whose
tile needs more than 48 KB of shared memory."""
import ctypes

import numpy as np
import pytest
import torch

import paged_edges as P

pytestmark = pytest.mark.gpu
FILL = 0xA5          # chunk buffers
SENTINEL = 0x5A      # destination caches


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _u8(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.uint8).reshape(-1)


# ---------------------------------------------------------------------------------------------- caches
class _Split:
    """L split (key, value) pairs on the device, each plane its own allocation starting plane_off bytes past a 16-byte
    boundary, with their CPU bits"""

    def __init__(self, case: P.Case, seed: int, fill=None):
        c = case
        self.case = c
        x = 16 // c.es
        self.layout = P.PagedLayoutLike("split", c.nb, c.bs, c.H, c.D, c.bs, x)
        shapes = ((c.nb, c.H, c.D // x, c.bs, x), (c.nb, c.H, c.D, c.bs))
        nbytes = c.nb * c.bs * c.H * c.D * c.es
        g = torch.Generator().manual_seed(seed)
        self.dev, self.bits = [], []
        for _ in range(c.L):
            pair, bits = [], []
            for shape in shapes:
                if fill is None:
                    b = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, generator=g)
                else:
                    b = torch.full((nbytes,), fill, dtype=torch.uint8)
                raw = torch.empty(nbytes + 32, dtype=torch.uint8, device="cuda")
                lo = (-raw.data_ptr()) % 16 + c.plane_off
                plane = raw[lo:lo + nbytes]
                plane.copy_(b)
                assert plane.data_ptr() % 16 == c.plane_off % 16
                pair.append(plane.view(c.torch_dtype).view(shape))
                bits.append(b.view(P.bits_dtype(c.es)).view(shape))
            self.dev.append(tuple(pair))
            self.bits.append(tuple(bits))

    def cpu_bits(self):
        return [tuple(t.view(torch.uint8).cpu().view(P.bits_dtype(self.case.es)) for t in p) for p in self.dev]


# ---------------------------------------------------------------------------------------------- chunk buffers
class _Buffer:
    """FILL-initialised chunk memory on the device or in mapped page-locked host memory"""

    def __init__(self, kind: str, nbytes: int):
        self.kind = kind
        self.nbytes = nbytes + 16
        if kind == "pinned":
            from lmcache_b200.codec import PinnedBuffer
            self.pin = PinnedBuffer(self.nbytes)
            self.host = np.frombuffer(self.pin.view(), dtype=np.uint8)
            self.host[:] = FILL
            ptr = self.pin.dev_ptr
        else:
            self.t = torch.full((self.nbytes,), FILL, dtype=torch.uint8, device="cuda")
            ptr = self.t.data_ptr()
        self.lo = (-ptr) % 16
        self.ptr = ptr + self.lo                # 16-byte aligned

    def read(self) -> torch.Tensor:
        torch.cuda.synchronize()
        if self.kind == "pinned":
            return torch.from_numpy(self.host[self.lo:].copy())
        return self.t[self.lo:].cpu()

    def write(self, off: int, data: torch.Tensor) -> None:
        if self.kind == "pinned":
            self.host[self.lo + off:self.lo + off + data.numel()] = data.numpy()
        else:
            self.t[self.lo + off:self.lo + off + data.numel()].copy_(data)

    def close(self):
        if self.kind == "pinned":
            self.host = None
            self.pin.close()


def _placement(case: P.Case, form: str, a: int, b: int, n: int):
    """the start of every chunk in the buffer, and the buffer's size"""
    if form == "contig":
        stride = case.chunk_bytes(case.L) + case.stride_pad
        return [case.chunk_off + j * stride for j in range(n)], case.chunk_off + n * stride + 16
    ts = (case.chunk_bytes(b - a) + 32 + 15) & ~15
    return [j * ts + case.table_offs[j % len(case.table_offs)] for j in range(n)], n * ts


def _move(pack: bool, case: P.Case, form: str, a: int, b: int, view, buf: _Buffer, starts, n: int, last: int):
    from lmcache_b200 import _native as N
    lib, cs, tb = N.lib(), case.chunk_tokens, case.tok_begin
    if form == "contig":
        stride = case.chunk_bytes(case.L) + case.stride_pad
        ptr = ctypes.c_void_p(buf.ptr + starts[0])
        if pack:
            rc = lib.b200kv_pack_chunks(ctypes.byref(view.desc), tb, n, cs, last, 0, ptr, stride, _stream())
        else:
            rc = lib.b200kv_unpack_chunks(ptr, stride, n, cs, last, 0, ctypes.byref(view.desc), tb, _stream())
    else:
        table = torch.tensor(np.asarray([buf.ptr + s for s in starts], dtype=np.uint64).view(np.int64), device="cuda")
        tp = ctypes.c_void_p(table.data_ptr())
        if pack:
            rc = lib.b200kv_pack_chunks_layers(ctypes.byref(view.desc), tb, n, cs, last, 0, a, b, tp, _stream())
        else:
            rc = lib.b200kv_unpack_chunks_layers(tp, n, cs, last, 0, a, b, ctypes.byref(view.desc), tb, _stream())
    N.check(rc, f"{'pack' if pack else 'unpack'} ({form})")
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- diagnostics
def _path_of(paths, bs, g):
    return dict(paths).get((g // bs) * bs, "not visited")


def _explain_pack(case, form, a, paths, slots, j, rel, blob):
    """where byte `rel` of chunk j's blob (shape [nl, 2, t, H, D]) comes from"""
    if rel < 0 or rel >= blob.numel() * case.es:
        return f"{case.name} {form} pack: chunk {j} written outside its blob at byte {rel}"
    li, kv, tok, h, d = np.unravel_index(rel // case.es, tuple(blob.shape))
    g = case.tok_begin + j * case.chunk_tokens + int(tok)
    return (f"{case.name} {form} pack: chunk {j} layer {a + int(li)} kv {int(kv)} head {int(h)} channel {int(d)} "
            f"token {g} slot {int(slots[g])}: group {(g // case.bs) * case.bs} took path {_path_of(paths, case.bs, g)}")


def _explain_unpack(case, form, layout, paths, slots, l, got, want):
    rg, rw = P.ref_rows(layout, *got), P.ref_rows(layout, *want)
    for kv in range(2):
        diff = (rg[kv] != rw[kv]).nonzero()
        if diff.numel():
            row, h, d = (int(v) for v in diff[0])
            hit = (slots == row).nonzero()
            if hit.numel() == 0:
                return (f"{case.name} {form} unpack: layer {l} kv {kv} head {h} channel {d}: slot {row}, which no "
                        f"call token addresses, was written")
            g = int(hit[0])
            return (f"{case.name} {form} unpack: layer {l} kv {kv} head {h} channel {d} token {g} slot {row}: group "
                    f"{(g // case.bs) * case.bs} took path {_path_of(paths, case.bs, g)}")
    return f"{case.name} {form} unpack: layer {l}: the caches differ"


# ---------------------------------------------------------------------------------------------- the split mover
@pytest.mark.parametrize("case", P.CASES, ids=lambda c: c.name)
def test_split_mover_equals_torch(case):
    from lmcache_b200.codec import KvView
    slots = P.make_slots(case.slots, case.T, case.nb, case.bs, case.seed)
    slots_dev = slots.cuda()
    src = _Split(case, case.seed)
    view = KvView.from_paged(src.dev, slots_dev)
    assert view.split
    cs, tb = case.chunk_tokens, case.tok_begin
    n = (case.T - tb + cs - 1) // cs
    last = case.T - tb - (n - 1) * cs
    for form, a, b in case.forms():
        paths = case.paths(form, slots)
        blobs = P.ref_pack(src.layout, src.bits, slots, tb, cs, (a, b))
        starts, size = _placement(case, form, a, b, n)
        # pack: ref_pack's bytes at each chunk's start, FILL everywhere else
        buf = _Buffer(case.buf, size)
        try:
            _move(True, case, form, a, b, view, buf, starts, n, last)
            got = buf.read()
        finally:
            buf.close()
        want = torch.full_like(got, FILL)
        for s, blob in zip(starts, blobs):
            want[s:s + blob.numel() * case.es] = _u8(blob)
        if not torch.equal(got, want):
            i = int((got != want).nonzero()[0])
            j = max(k for k, s in enumerate(starts) if s <= i) if i >= starts[0] else 0
            pytest.fail(_explain_pack(case, form, a, paths, slots, j, i - starts[j], blobs[j]))
        # unpack: ref_pack's blobs into sentinel-filled caches give ref_unpack's caches
        dst = _Split(case, 0, fill=SENTINEL)
        dview = KvView.from_paged(dst.dev, slots_dev)
        buf = _Buffer(case.buf, size)
        try:
            for s, blob in zip(starts, blobs):
                buf.write(s, _u8(blob))
            _move(False, case, form, a, b, dview, buf, starts, n, last)
        finally:
            buf.close()
        want_caches = [tuple(t.clone() for t in p) for p in dst.bits]
        P.ref_unpack(dst.layout, want_caches, slots, tb, cs, blobs, (a, b))
        got_caches = dst.cpu_bits()
        for l in range(case.L):
            if not all(torch.equal(x, y) for x, y in zip(got_caches[l], want_caches[l])):
                pytest.fail(_explain_unpack(case, form, dst.layout, paths, slots, l, got_caches[l], want_caches[l]))


# ---------------------------------------------------------------------------------------------- block-strided
def _strided(nb, planes, bs, H, D, L, gen, fill=None):
    """L FlashInfer pairs kv[:, 0], kv[:, 1] of [nb, planes, bs, H, D] bf16 allocations (planes 3: a spare plane)"""
    allocs = []
    for _ in range(L):
        if fill is None:
            b = torch.randint(0, 256, (nb * planes * bs * H * D * 2,), dtype=torch.uint8, generator=gen)
        else:
            b = torch.full((nb * planes * bs * H * D * 2,), fill, dtype=torch.uint8)
        allocs.append(b.cuda().view(torch.bfloat16).view(nb, planes, bs, H, D))
    return allocs, [(x[:, 0], x[:, 1]) for x in allocs]


def _cpu_pairs(allocs):
    """the allocations' bits on the CPU, and the pairs as the same views of them"""
    cpu = [x.view(torch.int16).cpu() for x in allocs]
    return cpu, [(x[:, 0], x[:, 1]) for x in cpu]


@pytest.mark.parametrize("bs", [1, 256])
@pytest.mark.parametrize("planes", [2, 3])
def test_strided_mover_and_codecs(bs, planes):
    """rows_per_block = 2 bs (FlashInfer's kv[:, 0]) and 3 bs (a padded allocation): the mover gives ref_pack's blobs
    and ref_unpack's caches; CacheGen and lossless encode straight from the cache give the containers of the same KV in
    FlashAttention layout, and decode straight into it writes what they write there, and nothing else"""
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import CacheGenCodec, KvView, LosslessCodec
    from test_gpu_host_tier import MODEL
    L, H, D = 2, 2, 64
    nb, T, cs = (700, 600, 128) if bs == 1 else (4, 600, 256)
    gen = torch.Generator().manual_seed(bs * 10 + planes)
    lay = P.PagedLayoutLike("strided", nb, bs, H, D, planes * bs, 0)
    slots = P.make_slots("vllm", T, nb, bs, seed=planes)
    slots_dev = slots.cuda()
    allocs, pairs = _strided(nb, planes, bs, H, D, L, gen)
    view = KvView.from_paged(pairs, slots_dev)
    assert view.layout == "strided"
    _, cpu_pairs = _cpu_pairs(allocs)
    # the mover, from token 5 in chunks of cs
    tb = 5
    blobs = P.ref_pack(lay, cpu_pairs, slots, tb, cs)
    _, got = view.pack_chunks(tb, cs)
    for j, (g, w) in enumerate(zip(got, blobs)):
        assert torch.equal(g.view(torch.int16).cpu(), w), (bs, planes, "pack", j)
    dallocs, dpairs = _strided(nb, planes, bs, H, D, L, gen, fill=SENTINEL)
    dview = KvView.from_paged(dpairs, slots_dev)
    buf = torch.cat([_u8(b) for b in blobs]).cuda()
    n = len(blobs)
    N.check(N.lib().b200kv_unpack_chunks(ctypes.c_void_p(buf.data_ptr()), cs * L * 2 * H * D * 2, n, cs,
                                         T - tb - (n - 1) * cs, 0, ctypes.byref(dview.desc), tb, _stream()), "unpack")
    torch.cuda.synchronize()
    want_allocs, want_pairs = _cpu_pairs(dallocs)
    want_allocs = [x.clone() for x in want_allocs]
    want_pairs = [(x[:, 0], x[:, 1]) for x in want_allocs]
    P.ref_unpack(lay, want_pairs, slots, tb, cs, blobs)
    got_allocs, _ = _cpu_pairs(dallocs)
    for l in range(L):
        assert torch.equal(got_allocs[l], want_allocs[l]), (bs, planes, "unpack", l)
    # the codecs: the same KV as contiguous FlashAttention rows, through the same slot map
    flash_rows = [P.ref_rows(lay, *p) for p in cpu_pairs]
    flash = [tuple(r.view(nb, bs, H, D).cuda().view(torch.bfloat16) for r in p) for p in flash_rows]
    fview = KvView.from_paged(flash, slots_dev)
    assert fview.layout == "flash"
    moved = torch.zeros(nb * bs, dtype=torch.bool)
    moved[slots] = True
    for codec in (CacheGenCodec(MODEL), LosslessCodec()):
        raws = codec.encode_to_host(view, 0, T, cs)
        assert raws == codec.encode_to_host(fview, 0, T, cs), (bs, planes, type(codec).__name__)
        dallocs, dpairs = _strided(nb, planes, bs, H, D, L, gen, fill=SENTINEL)
        fdst = [tuple(torch.full((nb, bs, H, D), SENTINEL, dtype=torch.uint8, device="cuda").repeat(1, 1, 1, 2)
                      .view(torch.bfloat16) for _ in range(2)) for _ in range(L)]
        starts = list(range(0, T, cs))
        codec.decode(raws, KvView.from_paged(dpairs, slots_dev), starts)
        codec.decode(raws, KvView.from_paged(fdst, slots_dev), starts)
        torch.cuda.synchronize()
        got_allocs, got_pairs = _cpu_pairs(dallocs)
        for l in range(L):
            rows = P.ref_rows(lay, *got_pairs[l])
            for kv in range(2):
                frows = fdst[l][kv].view(torch.int16).cpu().view(nb * bs, H, D)
                assert torch.equal(rows[kv], frows), (bs, planes, type(codec).__name__, l, kv)
                assert bool((rows[kv][~moved].view(torch.uint8) == SENTINEL).all())
                if isinstance(codec, LosslessCodec):
                    assert torch.equal(rows[kv][moved], flash_rows[l][kv][moved])
            if planes == 3:
                assert bool((got_allocs[l][:, 2].view(torch.uint8) == SENTINEL).all())


# ---------------------------------------------------------------------------------------------- the engine
def test_engine_lossless_host_tier_round_trip_at_bs256(tmp_path, autorelease):
    """store_paged from and retrieve_paged into a split cache at bs = 256 (a tile of 68 KB of shared memory) through
    the lossless host tier: the container tiers stage a split cache through the mover (KvView.staged, unpack_blob)"""
    from test_gpu_host_tier import MODEL
    from test_gpu_paged_layouts import _engine
    case = P.Case("engine_bs256", "bf16", 256, 2, 128, 2, 4, "vllm", 256 * 2 + 77, 0, 256, (0, 2))
    assert P.launch_model(2, 256, 2, 128, table=False, stride=case.chunk_bytes(2)).opt_in
    slots = P.make_slots("vllm", case.T, case.nb, case.bs, seed=21)
    slots_dev = slots.cuda()
    tokens = torch.randint(0, 32000, (case.T,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(22))
    src = _Split(case, 23)
    dst = _Split(case, 0, fill=SENTINEL)
    eng = _engine(autorelease, "host-lossless", case.chunk_tokens, None, tmp_path, MODEL)
    eng.store_paged(tokens, src.dev, slots_dev)
    ret = eng.retrieve_paged(tokens, dst.dev, slots_dev)
    torch.cuda.synchronize()
    assert int(ret.sum()) == case.T
    moved = torch.zeros(case.nb * case.bs, dtype=torch.bool)
    moved[slots] = True
    got = dst.cpu_bits()
    for l in range(case.L):
        want = P.ref_rows(src.layout, *src.bits[l])
        rows = P.ref_rows(dst.layout, *got[l])
        for kv in range(2):
            assert torch.equal(rows[kv][moved], want[kv][moved]), (l, kv)
            assert bool((rows[kv][~moved].view(torch.uint8) == SENTINEL).all()), (l, kv)
