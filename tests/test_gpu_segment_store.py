"""GPU: storing a prompt's documents from inside it.  b200kv_pack_chunks_rope against the composition it fuses
(b200kv_pack_chunks, then b200kv_rope_shift of the packed rows) byte for byte in every layout, chunk layout and
destination, against the float64 statement, and its refusals; LMCacheEngine.store_paged_segments / store_segments on
every tier and paged layout, read back at other positions by retrieve_paged_segments / retrieve_segments."""
import ctypes

import numpy as np
import pytest
import torch

import paged_edges as P
from rope_ref import partner, rotate, tolerance
from rope_twice_ref import tolerance_twice
from test_gpu_host_tier import MODEL
from test_gpu_paged_layouts import (BS, D_E, H_E, L_E, LAYOUTS, NB, TIERS, _all_rows, _cache_rows, _caches, _engine,
                                    _slots, lmserver)  # noqa: F401 -- lmserver is a fixture
from test_gpu_segments import KERNEL_LAYOUTS, NAMES, RAW_EXACT, ROT, _randn_rows, _target

pytestmark = pytest.mark.gpu
SHIFTS = [-1, -255, -4096, -65535]
FILL = 0xA5


def _seg_pattern(n):
    """n tokens: four table rows with -1 gaps, repeating"""
    unit = [-1] * 3 + [0] * 20 + [1] * 15 + [-1] * 5 + [2] * 20 + [3] * 10
    return (unit * (n // len(unit) + 1))[:n]


class _Out:
    """FILL-initialised chunk memory in device memory or mapped page-locked host memory, 16-byte aligned + off"""

    def __init__(self, kind, nbytes, off=0):
        self.kind = kind
        if kind == "pinned":
            from lmcache_b200.codec import PinnedBuffer
            self.pin = PinnedBuffer(nbytes + 32)
            self.host = np.frombuffer(self.pin.view(), dtype=np.uint8)
            self.host[:] = FILL
            base = self.pin.dev_ptr
        else:
            self.t = torch.full((nbytes + 32,), FILL, dtype=torch.uint8, device="cuda")
            base = self.t.data_ptr()
        self.lo = (-base) % 16 + off
        self.ptr = base + self.lo
        self.nbytes = nbytes

    def read(self):
        torch.cuda.synchronize()
        if self.kind == "pinned":
            out = torch.from_numpy(self.host[self.lo:self.lo + self.nbytes].copy())
            self.host = None
            self.pin.close()
            return out
        return self.t[self.lo:self.lo + self.nbytes].cpu()


def _chunking(T, tb, cs):
    n = (T - tb + cs - 1) // cs
    return n, T - tb - (n - 1) * cs


def _fused(view, tb, cs, hf, seg, shifts, spec, out="device", off=0, pad=0):
    """b200kv_pack_chunks_rope of tokens [tb, T) into chunks of cs tokens: the chunk memory's bytes"""
    from lmcache_b200 import _native as N
    from lmcache_b200.rope import STYLES, rope_table
    n, last = _chunking(view.ntokens, tb, cs)
    es = torch.empty((), dtype=view.dtype).element_size()
    stride = view.planes * view.H * view.D * cs * es + pad
    buf = _Out(out, n * stride, off)
    sg = torch.tensor(seg, dtype=torch.int32, device="cuda")
    table = rope_table(torch.tensor(shifts, dtype=torch.int64, device="cuda"), spec)
    N.check(N.lib().b200kv_pack_chunks_rope(ctypes.byref(view.desc), tb, n, cs, last, hf, ctypes.c_void_p(buf.ptr),
                                            stride, ctypes.c_void_p(sg.data_ptr()), ctypes.c_void_p(table.data_ptr()),
                                            spec.rotary_dim, spec.offset, STYLES[spec.style], None), "pack_chunks_rope")
    return buf.read(), stride


def _composed(view, tb, cs, hf, seg, shifts, spec, stride, rope=True):
    """b200kv_pack_chunks into the same chunk placement, then b200kv_rope_shift of each packed chunk's rows"""
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView
    from lmcache_b200.rope import rope_shift
    n, last = _chunking(view.ntokens, tb, cs)
    es = torch.empty((), dtype=view.dtype).element_size()
    buf = torch.full((n * stride + 16,), FILL, dtype=torch.uint8, device="cuda")
    lo = (-buf.data_ptr()) % 16
    N.check(N.lib().b200kv_pack_chunks(ctypes.byref(view.desc), tb, n, cs, last, hf,
                                       ctypes.c_void_p(buf.data_ptr() + lo), stride, None), "pack_chunks")
    if rope:
        fmt = "huggingface" if hf else "vllm"
        for j in range(n):
            t = last if j == n - 1 else cs
            shape = KvView.blob_shape(fmt, view.L, view.H, view.D, t, view.latent)
            nbytes = int(np.prod(shape)) * es
            blob = buf[lo + j * stride: lo + j * stride + nbytes].view(view.dtype).view(shape)
            rope_shift(KvView.from_blob(blob, fmt), 0, torch.tensor(seg[j * cs:j * cs + t], dtype=torch.int32,
                                                                     device="cuda"),
                       torch.tensor(shifts, dtype=torch.int64, device="cuda"), spec)
    torch.cuda.synchronize()
    return buf[lo:lo + n * stride].cpu()


def _same(got, want, what):
    if not torch.equal(got, want):
        i = int((got != want).nonzero()[0])
        pytest.fail(f"{what}: first differing byte {i} of {got.numel()}: {int(got[i])} != {int(want[i])}")


# ---------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("style", ["neox", "gptj"])
@pytest.mark.parametrize("kind", KERNEL_LAYOUTS + ["latent", "latent-paged"])
def test_fused_equals_pack_then_shift(dtype, style, kind):
    """byte for byte, for every rotary range (ROT: full, half, the element-wise 36 / 4, 32 / 16), both chunk layouts
    (the split layout packs vllm chunks only), device and mapped page-locked chunks"""
    from lmcache_b200.rope import RopeSpec
    latent = kind.startswith("latent")
    T, H, D = 96, 4, (576 if latent else 128)
    rots = [(64, 512)] if latent else ROT
    hfs = [0] if kind.startswith("split") or latent else [0, 1]
    for i, (rd, off) in enumerate(rots):
        spec = RopeSpec.from_base(rd, 10000.0, style, off)
        view, _, _ = _target(kind, dtype, T, H, D, seed=i + 10 * len(kind))
        for hf in hfs:
            for out, tb, cs in (("device", 5, 32), ("pinned", 0, 40)):
                seg = _seg_pattern(T - tb)
                got, stride = _fused(view, tb, cs, hf, seg, SHIFTS, spec, out)
                _same(got, _composed(view, tb, cs, hf, seg, SHIFTS, spec, stride),
                      f"{kind} rot {rd}/{off} hf {hf} {out}")


@pytest.mark.parametrize("case", [c for c in P.CASES if c.es == 2], ids=lambda c: c.name)
def test_fused_split_every_branch(case):
    """every 16-bit case of the split kernel's case table (tile and element-wise groups, misaligned chunks and strides,
    mapped chunks, >48 KB tiles): fused equals pack then shift, for an aligned and an element-wise rotary range"""
    from lmcache_b200.codec import KvView
    from lmcache_b200.rope import RopeSpec
    from test_gpu_paged_edges import _Split
    slots = P.make_slots(case.slots, case.T, case.nb, case.bs, case.seed).cuda()
    view = KvView.from_paged(_Split(case, case.seed).dev, slots)
    D = case.D
    for rd, off, style in ((D, 0, "neox"), (D // 2, 8, "gptj"), (D - 12, 6, "neox")):
        spec = RopeSpec.from_base(rd, 10000.0, style, off)
        seg = _seg_pattern(case.T - case.tok_begin)
        got, stride = _fused(view, case.tok_begin, case.chunk_tokens, 0, seg, SHIFTS, spec, case.buf, case.chunk_off,
                             case.stride_pad)
        _same(got, _composed(view, case.tok_begin, case.chunk_tokens, 0, seg, SHIFTS, spec, stride),
              f"{case.name} rot {rd}/{off}/{style}")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("kind", ["tuple", "huggingface", "split-16", "strided-16", "latent-paged"])
def test_fused_against_the_statement(dtype, kind):
    """the rotary channels of turned tokens within tolerance of the float64 statement; every other byte that of
    b200kv_pack_chunks; all rows -1: b200kv_pack_chunks itself"""
    from lmcache_b200.rope import RopeSpec
    latent = kind.startswith("latent")
    T, H, D = 96, 4, (576 if latent else 128)
    spec = RopeSpec.from_base(64, 10000.0, "gptj", 512) if latent else RopeSpec.from_base(96, 10000.0, "neox", 16)
    view, _, _ = _target(kind, dtype, T, H, D, seed=4)
    seg = _seg_pattern(T)
    got, stride = _fused(view, 0, T, 0, seg, SHIFTS, spec)
    plain = _composed(view, 0, T, 0, seg, SHIFTS, spec, stride, rope=False)
    none, _ = _fused(view, 0, T, 0, [-1] * T, SHIFTS, spec)
    _same(none, plain, f"{kind} all -1")
    shape = (view.L, T, D) if latent else (view.L, 2, T, H, D)
    g = got.view(dtype).view(shape)
    w = plain.view(dtype).view(shape)
    k_got, k_src = (g, w) if latent else (g[:, 0], w[:, 0])
    rot = torch.zeros(shape, dtype=torch.bool)
    toks = torch.tensor([i for i, s in enumerate(seg) if s >= 0])
    sel = (slice(None), toks) if latent else (slice(None), 0, toks)
    m = rot[sel]
    m[..., spec.offset:spec.offset + spec.rotary_dim] = True
    rot[sel] = m
    assert torch.equal(got.view(torch.int16).view(shape)[~rot], plain.view(torch.int16).view(shape)[~rot]), kind
    x = k_src[:, toks].double().numpy()
    sh = np.asarray(SHIFTS, dtype=np.int64)[np.asarray(seg)[toks.numpy()]]
    xs = np.moveaxis(x, 1, 0)                                   # [n, L, (H,) D]: per-token shifts on axis 0
    want = np.moveaxis(rotate(xs, sh, spec.inv_freq.numpy(), spec.rotary_dim, spec.style, spec.offset), 0, 1)
    want_r = torch.from_numpy(want).to(dtype).double().numpy()
    gg = k_got[:, toks].double().numpy()
    p = partner(spec.rotary_dim, spec.style, spec.offset, D)
    assert (np.abs(gg - want_r) <= tolerance(want_r, gg, x, x[..., p], NAMES[dtype])).all(), kind


def test_fused_refusals_write_nothing():
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView
    L, T, H, D = 2, 32, 2, 64
    seg = torch.zeros(T, dtype=torch.int32, device="cuda")
    table = torch.zeros(1, D // 2, 2, dtype=torch.float32, device="cuda")
    out = torch.full((L * 2 * T * H * D * 2,), FILL, dtype=torch.uint8, device="cuda")
    lib = N.lib()

    def call(blob, rd, off, style=0, tab=table.data_ptr(), sg=seg.data_ptr(), n=1, last=T):
        view = KvView.from_blob(blob, "vllm")
        return lib.b200kv_pack_chunks_rope(ctypes.byref(view.desc), 0, n, T, last, 0, ctypes.c_void_p(out.data_ptr()),
                                           out.numel(), ctypes.c_void_p(sg), ctypes.c_void_p(tab), rd, off, style, None)
    for dt in (torch.uint8, torch.float8_e4m3fn, torch.float8_e5m2):
        blob = torch.full((L, 2, T, H, D), 0x3C, dtype=torch.uint8, device="cuda").view(dt)
        assert call(blob, D, 0) < 0 and "16-bit" in N.last_error()
    blob = torch.randn(L, 2, T, H, D, device="cuda").to(torch.bfloat16)
    for kw, msg in (({"rd": 63, "off": 0}, "even"), ({"rd": 0, "off": 0}, "even"), ({"rd": 32, "off": 33}, "exceeds"),
                    ({"rd": 64, "off": -2}, "exceeds"), ({"rd": 64, "off": 0, "style": 2}, "style"),
                    ({"rd": 64, "off": 0, "tab": 0}, "NULL"), ({"rd": 64, "off": 0, "sg": 0}, "NULL"),
                    ({"rd": 64, "off": 0, "n": 0}, "chunking"), ({"rd": 64, "off": 0, "last": T + 1}, "chunking")):
        assert call(blob, **kw) < 0, kw
        assert msg in N.last_error(), (msg, N.last_error())
    torch.cuda.synchronize()
    assert bool((out == FILL).all())


# ---------------------------------------------------------------------------------------------- the engine
CS = 64
DOCS = {"A": 2 * CS + 10, "B": 3 * CS, "C": 3 * CS + 20}


def _request(doc_tokens, order, lens, gen):
    """the documents in `order` between filler runs of `lens`: tokens and each document's (start, end)"""
    parts, segs, pos = [], {}, 0
    for i, name in enumerate(order):
        filler = torch.randint(0, 32000, (lens[i],), generator=gen)
        parts += [filler, doc_tokens[name]]
        segs[name] = (pos + lens[i], pos + lens[i] + len(doc_tokens[name]))
        pos += lens[i] + len(doc_tokens[name])
    parts.append(torch.randint(0, 32000, (lens[-1],), generator=gen))
    return torch.cat(parts), segs


def _docs(tag):
    gen = torch.Generator().manual_seed(5)
    return {n: torch.randint(0, 32000, (ln,), generator=gen) + 40000 + 1000 * tag for n, ln in DOCS.items()}


def _drain(eng):
    if hasattr(eng.engine_, "drain"):
        eng.engine_.drain()


def _turned_alone(src_rows, slots, a, b, spec):
    """pack + rope_shift(-a) of the request's rows [a, b): the KV of the document as if prefilled alone"""
    from lmcache_b200.codec import KvView
    from lmcache_b200.rope import rope_shift
    idx = slots[a:b]
    blob = torch.stack([torch.stack((k.view(torch.bfloat16)[idx], v.view(torch.bfloat16)[idx])) for k, v in src_rows])
    rope_shift(KvView.from_blob(blob, "vllm"), 0, torch.zeros(b - a, dtype=torch.int32, device="cuda"),
               torch.tensor([-a], dtype=torch.int64, device="cuda"), spec)
    return blob


@pytest.mark.parametrize("tier", TIERS)
def test_engine_store_then_retrieve_elsewhere(tier, lmserver, tmp_path, autorelease):
    """request 1 [prefix][B][A][gap][C][question] stored with store_paged_segments from each paged layout; request 2
    holds the documents in another order at other offsets.  Its rows equal, bit for bit, those of an engine in which
    each document was stored alone as pack + rope_shift(-start) of the same rows; on the raw and lossless tiers V is the
    source's and K within the two-rounding bound of the source turned by new start - old start."""
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(D_E, 10000.0)
    docs = _docs(TIERS.index(tier))

    def requests(off):
        """requests 1 and 2 with every token id moved by `off`: the engines of one test share a disk directory or a
        server, so each stores under keys of its own"""
        d = {n: t + off for n, t in docs.items()}
        return (_request(d, ["B", "A", "C"], [30, 0, 17, 25], torch.Generator().manual_seed(6)),
                _request(d, ["A", "C", "B"], [45, 3, 64, 9], torch.Generator().manual_seed(16)))
    (tok1, seg1), (tok2, seg2) = requests(0)
    slots1 = _slots("vllm", len(tok1), NB, BS, torch.Generator().manual_seed(7))
    slots2 = _slots("vllm", len(tok2), NB, BS, torch.Generator().manual_seed(8))
    src_rows = _randn_rows(L_E, NB * BS, H_E, D_E, torch.bfloat16, seed=21)
    # the reference: each document stored alone, its KV the source rows turned back by their request-1 start
    ref = _engine(autorelease, tier, CS, lmserver, tmp_path, MODEL)
    flat_src = _cache_rows("flash", _caches("flash", src_rows, NB, BS, H_E, D_E))
    for n, (a, b) in seg1.items():
        blob = _turned_alone(flat_src, slots1, a, b, spec)
        ref.store(docs[n], tuple((blob[l, 0], blob[l, 1]) for l in range(L_E)))
    _drain(ref)
    want_mask = torch.zeros(len(tok2), dtype=torch.bool)
    for a, b in seg2.values():
        want_mask[a:b] = True

    def read(eng, tok2):
        dst = _caches("flash", _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x3C), NB, BS, H_E, D_E)
        ret = eng.retrieve_paged_segments(tok2, dst, slots2, list(seg2.values()), spec)
        torch.cuda.synchronize()
        assert torch.equal(ret, want_mask), tier
        return _cache_rows("flash", dst)
    want = read(ref, tok2)
    for li, layout in enumerate(LAYOUTS):
        eng = _engine(autorelease, tier, CS, lmserver, tmp_path, MODEL)
        (t1, _), (t2, _) = requests(100000 * (li + 1))
        src = _caches(layout, src_rows, NB, BS, H_E, D_E)
        eng.store_paged_segments(t1, src, slots1, [seg1["C"], seg1["B"], seg1["A"]], spec)
        _drain(eng)
        got = read(eng, t2)
        for l in range(L_E):
            for i in range(2):
                assert torch.equal(got[l][i][slots2], want[l][i][slots2]), (tier, layout, l, i)
        if tier in RAW_EXACT and li == 0:
            inv = spec.inv_freq.numpy()
            p = partner(D_E, "neox", 0, D_E)
            for n, (a2, b2) in seg2.items():
                a1 = seg1[n][0]
                for l in range(L_E):
                    assert torch.equal(got[l][1][slots2[a2:b2]], flat_src[l][1][slots1[a1:a1 + b2 - a2]]), (n, l)
                    x = flat_src[l][0][slots1[a1:a1 + b2 - a2]].view(torch.bfloat16).double().cpu().numpy()
                    w = torch.from_numpy(rotate(x, a2 - a1, inv, D_E)).to(torch.bfloat16).double().numpy()
                    g = got[l][0][slots2[a2:b2]].view(torch.bfloat16).double().cpu().numpy()
                    assert (np.abs(g - w) <= tolerance_twice(w, g, x, x[..., p], "bfloat16")).all(), (tier, n, l)


@pytest.mark.parametrize("tier", ["cpu", "host-cachegen", "host-lossless"])
def test_namespace_isolation_and_start_0(tier, lmserver, tmp_path, autorelease):
    """a document stored from inside a prompt never comes back from retrieve_paged / retrieve; a segment at 0 stores
    what store_paged(tokens[:end]) stores"""
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(D_E, 10000.0)
    docs = _docs(50 + TIERS.index(tier))
    tok, seg = _request(docs, ["A", "B"], [0, 40, 7], torch.Generator().manual_seed(9))
    slots = _slots("vllm", len(tok), NB, BS, torch.Generator().manual_seed(10))
    src = _caches("flash", _randn_rows(L_E, NB * BS, H_E, D_E, torch.bfloat16, seed=22), NB, BS, H_E, D_E)
    eng = _engine(autorelease, tier, CS, lmserver, tmp_path, MODEL)
    eng.store_paged_segments(tok, src, slots, [seg["B"], seg["A"]], spec)
    _drain(eng)
    alone = _engine(autorelease, tier, CS, lmserver, tmp_path, MODEL)      # in-process tiers: a store of its own
    a_end = seg["A"][1]
    alone.store_paged(tok[:a_end], src, slots[:a_end])
    _drain(alone)
    # B, stored from position 40 + |A|: its own tokens, or a request that begins with it, miss
    dst = _caches("flash", _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x3C), NB, BS, H_E, D_E)
    q = torch.cat([docs["B"], torch.randint(0, 32000, (20,), generator=torch.Generator().manual_seed(1))])
    assert int(eng.retrieve_paged(q, dst, torch.arange(len(q), device="cuda")).sum()) == 0
    kv, ret = eng.retrieve(docs["B"])
    assert len(kv) == 0 and int(ret.sum()) == 0
    # A, the segment at 0: what store_paged(tokens[:end]) stored, under the same keys
    for e in (eng, alone):
        assert all(e.engine_.contains(e._make_key(h, "vllm")) for h in e._prefix_hash(docs["A"]))
    r = []
    for e in (eng, alone):
        d = _caches("flash", _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x3C), NB, BS, H_E, D_E)
        r.append((e.retrieve_paged(docs["A"], d, slots[:a_end]), _cache_rows("flash", d)))
    assert torch.equal(r[0][0], r[1][0]) and bool(r[0][0].all())
    for l in range(L_E):
        for i in range(2):
            assert torch.equal(r[0][1][l][i], r[1][1][l][i]), (l, i)


def test_skip_and_continuation(lmserver, tmp_path, autorelease):
    """C's first two chunks stored alone: the segment store puts only its later chunks under derived keys, and the
    retrieve serves chunks 0-1 from the prefix keys, the rest from the derived keys"""
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(D_E, 10000.0)
    eng = _engine(autorelease, "cpu", CS, lmserver, tmp_path, f"{MODEL}-skip")
    docs = _docs(70)
    tok, seg = _request(docs, ["C"], [100, 30], torch.Generator().manual_seed(11))
    a, b = seg["C"]
    slots = _slots("vllm", len(tok), NB, BS, torch.Generator().manual_seed(12))
    src_rows = _randn_rows(L_E, NB * BS, H_E, D_E, torch.bfloat16, seed=23)
    flat = _cache_rows("flash", _caches("flash", src_rows, NB, BS, H_E, D_E))
    blob = _turned_alone(flat, slots, a, b, spec)
    eng.store(docs["C"][:2 * CS], tuple((blob[l, 0, :2 * CS], blob[l, 1, :2 * CS]) for l in range(L_E)))
    hs = list(eng._prefix_hash(docs["C"]))
    puts = []
    orig = eng.engine_.put_kv_chunks

    def spy(keys, view, tok0, cs, **kw):
        puts.append([k.chunk_hash for k in keys])
        return orig(keys, view, tok0, cs, **kw)
    eng.engine_.put_kv_chunks = spy
    eng.store_paged_segments(tok, _caches("split", src_rows, NB, BS, H_E, D_E), slots, [seg["C"]], spec)
    from lmcache_b200.rope import derived_digest
    assert puts == [[derived_digest(h) for h in hs[2:]]]
    assert not any(eng.engine_.contains(eng._derived_key(h, "vllm")) for h in hs[:2])
    # a second store finds every chunk and puts nothing
    eng.store_paged_segments(tok, _caches("flash", src_rows, NB, BS, H_E, D_E), slots, [seg["C"]], spec)
    assert len(puts) == 1
    # request 2: C at 7; all of it comes back, the same bytes as a store of C alone in full
    tok2, seg2 = _request(docs, ["C"], [7, 3], torch.Generator().manual_seed(13))
    ref = _engine(autorelease, "cpu", CS, lmserver, tmp_path, f"{MODEL}-skip-ref")
    ref.store(docs["C"], tuple((blob[l, 0], blob[l, 1]) for l in range(L_E)))
    rows = []
    for e in (eng, ref):
        d = _caches("strided", _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x3C), NB, BS, H_E, D_E)
        ret = e.retrieve_paged_segments(tok2, d, torch.arange(len(tok2), device="cuda"), [seg2["C"]], spec)
        assert int(ret.sum()) == DOCS["C"] and bool(ret[seg2["C"][0]:seg2["C"][1]].all())
        rows.append(_cache_rows("strided", d))
    for l in range(L_E):
        for i in range(2):
            assert torch.equal(rows[0][l][i], rows[1][l][i]), (l, i)
    kv, ret = eng.retrieve_segments(tok2, [seg2["C"]], spec)
    assert int(ret.sum()) == DOCS["C"]


@pytest.mark.parametrize("tier", ["cpu", "host-cachegen", "host-lossless"])
def test_mla_turns_only_the_rope_channels(tier, lmserver, tmp_path, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineMetadata
    from lmcache_b200.rope import RopeSpec
    from test_gpu_paged_layouts import _tier_config
    spec = RopeSpec.from_base(64, 10000.0, "gptj", 512)
    eng = autorelease(LMCacheEngine(_tier_config(tier, CS, lmserver, tmp_path),
                                    LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16", True)))
    L, D, nb, bs = 3, 576, 60, 16
    g = torch.Generator(device="cuda").manual_seed(9)
    src = [torch.randn(nb, bs, D, device="cuda", generator=g).to(torch.bfloat16) for _ in range(L)]
    gen = torch.Generator().manual_seed(10)
    doc = torch.randint(0, 32000, (2 * CS + 10,), generator=gen) + 700000 + 1000 * len(tier)
    tokens = torch.cat([torch.randint(0, 32000, (77,), generator=gen), doc])
    slots = _slots("perm", len(tokens), nb, bs, torch.Generator().manual_seed(11))
    eng.store_paged_segments(tokens, src, slots, [(77, len(tokens))], spec)
    _drain(eng)
    # served at position 5: the latent channels as stored, the rope channels turned by 5 - 77
    tok2 = torch.cat([tokens[:5], doc])
    dst = [torch.full((nb, bs, D), 7, dtype=torch.bfloat16, device="cuda") for _ in range(L)]
    slots2 = torch.arange(len(tok2), device="cuda")
    ret = eng.retrieve_paged_segments(tok2, dst, slots2, [(5, len(tok2))], spec)
    torch.cuda.synchronize()
    assert int(ret.sum()) == len(doc)
    if tier == "host-cachegen":
        return                                            # lossy: the bit-exact checks below are for raw / lossless
    p = partner(64, "gptj", 512, D)
    for l in range(L):
        got = dst[l].view(-1, D)[slots2[5:]]
        x_t = src[l].view(-1, D)[slots[77:]]
        assert torch.equal(got[:, :512].view(torch.int16), x_t[:, :512].view(torch.int16)), l
        x = x_t.double().cpu().numpy()
        w = torch.from_numpy(rotate(x, 5 - 77, spec.inv_freq.numpy(), 64, "gptj", 512)).to(torch.bfloat16).double().numpy()
        gg = got.double().cpu().numpy()
        assert (np.abs(gg - w) <= tolerance_twice(w, gg, x, x[..., p], "bfloat16")).all(), l


@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
def test_dense_store_segments(fmt, lmserver, tmp_path, autorelease):
    """store_segments from store()'s per-layer tensors (vllm [T, H, D], huggingface [H, T, D]), non-blocking then
    drained; retrieve_segments at the same positions gives V as stored and K within the two-rounding bound"""
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineMetadata
    from lmcache_b200.rope import RopeSpec
    from test_gpu_paged_layouts import _tier_config
    spec = RopeSpec.from_base(D_E, 10000.0, "gptj")
    eng = autorelease(LMCacheEngine(_tier_config("cpu", CS, lmserver, tmp_path),
                                    LMCacheEngineMetadata(MODEL, 1, 0, fmt, "bfloat16")))
    docs = _docs(80)
    tok, seg = _request(docs, ["A", "B"], [0, 13, 20], torch.Generator().manual_seed(14))
    T = len(tok)
    g = torch.Generator(device="cuda").manual_seed(15)
    rows = [tuple(torch.randn(T, H_E, D_E, device="cuda", generator=g).to(torch.bfloat16) for _ in range(2))
            for _ in range(L_E)]
    kv = tuple((k, v) if fmt == "vllm" else (k.transpose(0, 1).contiguous(), v.transpose(0, 1).contiguous())
               for k, v in rows)
    eng.store_segments(tok, kv, [seg["A"], seg["B"]], spec, blocking=False)
    _drain(eng)
    got, ret = eng.retrieve_segments(tok, [seg["B"], seg["A"]], spec)
    assert int(ret.sum()) == DOCS["A"] + DOCS["B"]
    p = partner(D_E, "gptj", 0, D_E)
    tdim = 0 if fmt == "vllm" else 1
    for l in range(L_E):
        for n, (a, b) in seg.items():
            k = got[l][0].narrow(tdim, a, b - a)
            v = got[l][1].narrow(tdim, a, b - a)
            if fmt == "huggingface":
                k, v = k.transpose(0, 1), v.transpose(0, 1)
            assert torch.equal(v.view(torch.int16), rows[l][1][a:b].view(torch.int16)), (n, l)
            x = rows[l][0][a:b].double().cpu().numpy()
            w = torch.from_numpy(rotate(x, 0, spec.inv_freq.numpy(), D_E, "gptj")).to(torch.bfloat16).double().numpy()
            gg = k.double().cpu().numpy()
            assert (np.abs(gg - w) <= tolerance_twice(w, gg, x, x[..., p], "bfloat16")).all(), (n, l)


def test_refusals_store_nothing(lmserver, tmp_path, autorelease):
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(D_E, 10000.0)
    eng = _engine(autorelease, "cpu", CS, lmserver, tmp_path, f"{MODEL}-refuse")
    docs = _docs(90)
    tok, seg = _request(docs, ["A", "B"], [10, 5, 5], torch.Generator().manual_seed(17))
    slots = _slots("vllm", len(tok), NB, BS, torch.Generator().manual_seed(18))
    src = _caches("flash", _randn_rows(L_E, NB * BS, H_E, D_E, torch.bfloat16, seed=24), NB, BS, H_E, D_E)
    fp8 = _caches("flash", _all_rows(L_E, NB, BS, H_E, D_E, torch.float8_e4m3fn, seed=25), NB, BS, H_E, D_E)
    with pytest.raises(TypeError):
        eng.store_paged_segments(tok, fp8, slots, [seg["A"]], spec)
    with pytest.raises(ValueError, match="overlap"):
        eng.store_paged_segments(tok, src, slots, [seg["A"], (seg["A"][1] - 1, seg["A"][1] + 3)], spec)
    with pytest.raises(ValueError, match="do not fit"):
        eng.store_paged_segments(tok, src, slots, [seg["A"]], RopeSpec.from_base(D_E, 1e4, "neox", 8))
    kv = tuple((k.view(-1, H_E, D_E)[slots], v.view(-1, H_E, D_E)[slots]) for k, v in src)
    with pytest.raises(ValueError, match="overlap"):
        eng.store_segments(tok, kv, [seg["B"], seg["B"]], spec)
    dst = _caches("flash", _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x3C), NB, BS, H_E, D_E)
    assert int(eng.retrieve_paged_segments(tok, dst, slots, [seg["A"], seg["B"]], spec).sum()) == 0
