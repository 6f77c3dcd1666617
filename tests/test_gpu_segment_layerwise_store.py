"""GPU: the layer-by-layer segment store.  b200kv_pack_chunks_layers_rope byte for byte against b200kv_pack_chunks_rope
restricted to the layer range and against b200kv_pack_chunks_layers + b200kv_rope_shift_layers, in every source layout,
at chunks of mixed sizes, misaligned and mapped chunk pointers, and its refusals; store_paged_segments_layerwise /
store_segments_layerwise on every tier and paged layout against the whole forms, with each layer written only just
before it is saved."""
import ctypes
import hashlib

import numpy as np
import pytest
import torch

import paged_edges as P
from test_gpu_host_tier import MODEL
from test_gpu_paged_layouts import (BS, D_E, H_E, L_E, LAYOUTS, NB, TIERS, _all_rows, _cache_rows, _caches, _engine,
                                    _layout, _slots, lmserver)  # noqa: F401 -- lmserver is a fixture
from test_gpu_segment_store import DOCS, FILL, SHIFTS, _docs, _drain, _Out, _request, _same
from test_gpu_segments import KERNEL_LAYOUTS, ROT, _randn_rows, _target

pytestmark = pytest.mark.gpu
CS_E = 64
CHUNKS = [(3, 16, 0), (40, 7, -1), (20, 16, 1), (60, 1, 2), (70, 13, 3)]     # (src_tok, tokens, table row)


def _es(view):
    return torch.empty((), dtype=view.dtype).element_size()


def _slice_bytes(view, t):
    """bytes of one layer of a chunk of t tokens"""
    return (1 if view.latent else 2) * view.H * view.D * t * _es(view)


def _table(spec):
    from lmcache_b200.rope import rope_table
    return rope_table(torch.tensor(SHIFTS, dtype=torch.int64, device="cuda"), spec)


def _fused(view, chunks, ct, hf, l0, l1, spec, out="device", offs=(0,)):
    """b200kv_pack_chunks_layers_rope of `chunks` into FILL-initialised full-L chunk buffers (chunk j's pointer at its
    layer l0): each chunk's bytes, the other layers' FILL included"""
    from lmcache_b200 import _native as N
    from lmcache_b200.rope import STYLES
    bufs = [_Out(out, view.L * _slice_bytes(view, t), offs[j % len(offs)]) for j, (_, t, _) in enumerate(chunks)]
    ptrs = torch.tensor([b.ptr + l0 * _slice_bytes(view, t) for b, (_, t, _) in zip(bufs, chunks)], dtype=torch.int64,
                        device="cuda")
    ntok = torch.tensor([t for _, t, _ in chunks], dtype=torch.int32, device="cuda")
    stok = torch.tensor([a for a, _, _ in chunks], dtype=torch.int64, device="cuda")
    seg = torch.tensor([s for _, _, s in chunks], dtype=torch.int32, device="cuda")
    table = _table(spec)
    N.check(N.lib().b200kv_pack_chunks_layers_rope(
        ctypes.byref(view.desc), len(chunks), ct, ctypes.c_void_p(ntok.data_ptr()), ctypes.c_void_p(stok.data_ptr()),
        ctypes.c_void_p(seg.data_ptr()), hf, l0, l1, ctypes.c_void_p(ptrs.data_ptr()), ctypes.c_void_p(table.data_ptr()),
        spec.rotary_dim, spec.offset, STYLES[spec.style], None), "pack_chunks_layers_rope")
    return [b.read() for b in bufs]


def _composed(view, chunks, hf, l0, l1, spec):
    """b200kv_pack_chunks_layers of each chunk, then b200kv_rope_shift_layers of the packed range"""
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView
    from lmcache_b200.rope import rope_shift_layers
    table = _table(spec)
    fmt = "huggingface" if hf else "vllm"
    out = []
    for a, t, s in chunks:
        sl = _slice_bytes(view, t)
        buf = torch.full((view.L * sl + 16,), FILL, dtype=torch.uint8, device="cuda")
        lo = (-buf.data_ptr()) % 16
        ptr = torch.tensor([buf.data_ptr() + lo + l0 * sl], dtype=torch.int64, device="cuda")
        N.check(N.lib().b200kv_pack_chunks_layers(ctypes.byref(view.desc), a, 1, t, t, hf, l0, l1,
                                                  ctypes.c_void_p(ptr.data_ptr()), None), "pack_chunks_layers")
        if s >= 0:
            shape = KvView.blob_shape(fmt, l1 - l0, view.H, view.D, t, view.latent)
            blob = buf[lo + l0 * sl:lo + l1 * sl].view(view.dtype).view(shape)
            rope_shift_layers(KvView.from_blob(blob, fmt), 0, l1 - l0, 0, torch.full((t,), s, dtype=torch.int32,
                                                                                     device="cuda"),
                              table, spec, torch.cuda.current_stream())
        torch.cuda.synchronize()
        out.append(buf[lo:lo + view.L * sl].cpu())
    return out


def _fused_whole(view, chunks, hf, l0, l1, spec):
    """b200kv_pack_chunks_rope of each chunk (every layer), with the layers outside [l0, l1) set to FILL"""
    from lmcache_b200 import _native as N
    from lmcache_b200.rope import STYLES
    table = _table(spec)
    out = []
    for a, t, s in chunks:
        sl = _slice_bytes(view, t)
        buf = torch.full((view.L * sl + 16,), FILL, dtype=torch.uint8, device="cuda")
        lo = (-buf.data_ptr()) % 16
        seg = torch.full((t,), s, dtype=torch.int32, device="cuda")
        N.check(N.lib().b200kv_pack_chunks_rope(ctypes.byref(view.desc), a, 1, t, t, hf,
                                                ctypes.c_void_p(buf.data_ptr() + lo), view.L * sl,
                                                ctypes.c_void_p(seg.data_ptr()), ctypes.c_void_p(table.data_ptr()),
                                                spec.rotary_dim, spec.offset, STYLES[spec.style], None),
                "pack_chunks_rope")
        torch.cuda.synchronize()
        b = buf[lo:lo + view.L * sl].cpu()
        b[:l0 * sl] = FILL
        b[l1 * sl:] = FILL
        out.append(b)
    return out


def _check_all(view, get, chunks, ct, hf, spec, what, out="device", offs=(0,)):
    before = [tuple(None if x is None else x.clone() for x in p) for p in get()]
    L = view.L
    full = _fused(view, chunks, ct, hf, 0, L, spec, out, offs)
    for l0, l1 in [(0, L)] + [(l, l + 1) for l in range(L)]:
        got = _fused(view, chunks, ct, hf, l0, l1, spec, out, offs)
        for j, (g, c, w) in enumerate(zip(got, _composed(view, chunks, hf, l0, l1, spec),
                                          _fused_whole(view, chunks, hf, l0, l1, spec))):
            _same(g, c, f"{what} [{l0}, {l1}) chunk {j} against pack_layers + shift")
            _same(g, w, f"{what} [{l0}, {l1}) chunk {j} against pack_chunks_rope")
    # ranges covering each layer once give the full range's bytes
    parts = [_fused(view, chunks, ct, hf, l, l + 1, spec, out, offs) for l in range(L)]
    for j, (_, t, _) in enumerate(chunks):
        sl = _slice_bytes(view, t)
        _same(torch.cat([parts[l][j][l * sl:(l + 1) * sl] for l in range(L)]), full[j], f"{what} chunk {j} by layers")
    torch.cuda.synchronize()
    for p, q in zip(before, get()):            # the source is only read
        for x, y in zip(p, q):
            if x is not None:
                assert torch.equal(x.view(torch.int16), y.view(torch.int16)), what


# ---------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("style", ["neox", "gptj"])
@pytest.mark.parametrize("kind", KERNEL_LAYOUTS + ["latent", "latent-paged"])
def test_kernel_equals_pack_rope_and_pack_layers_then_shift(dtype, style, kind):
    """every rotary range of ROT (vector and element-wise paths; 512/64 for a latent KV), both chunk layouts, chunks of
    mixed sizes at non-contiguous source tokens, a -1 row, device chunks (one misaligned) and mapped page-locked ones"""
    from lmcache_b200.rope import RopeSpec
    latent = kind.startswith("latent")
    T, H, D = 96, 4, (576 if latent else 128)
    rots = [(64, 512)] if latent else ROT
    hfs = [0] if kind.startswith("split") or latent else [0, 1]
    for i, (rd, off) in enumerate(rots):
        spec = RopeSpec.from_base(rd, 10000.0, style, off)
        view, get, _ = _target(kind, dtype, T, H, D, seed=i + 10 * len(kind))
        for hf in hfs:
            _check_all(view, get, CHUNKS, 16, hf, spec, f"{kind} rot {rd}/{off} hf {hf}", "device", (0, 2))
            if i == 0:
                _check_all(view, get, CHUNKS[:3], 16, hf, spec, f"{kind} rot {rd}/{off} hf {hf} pinned", "pinned")


@pytest.mark.parametrize("case", [c for c in P.CASES if c.es == 2], ids=lambda c: c.name)
def test_kernel_split_every_case(case):
    """every 16-bit case of the split mover's case table as a source: the case's chunking from its tok_begin, its chunk
    memory and offsets, an aligned and an element-wise rotary range"""
    from lmcache_b200.codec import KvView
    from lmcache_b200.rope import RopeSpec
    from test_gpu_paged_edges import _Split
    slots = P.make_slots(case.slots, case.T, case.nb, case.bs, case.seed).cuda()
    sp = _Split(case, case.seed)
    view = KvView.from_paged(sp.dev, slots)
    chunks = []
    for j, a in enumerate(range(case.tok_begin, case.T, case.chunk_tokens)):
        chunks.append((a, min(case.chunk_tokens, case.T - a), j % 5 - 1))
    D = case.D
    for rd, off, style in ((D, 0, "neox"), (D - 12, 6, "gptj")):
        spec = RopeSpec.from_base(rd, 10000.0, style, off)
        _check_all(view, lambda: [tuple(p) for p in sp.dev], chunks, case.chunk_tokens, 0, spec,
                   f"{case.name} rot {rd}/{off}", case.buf, tuple(o + case.chunk_off for o in case.table_offs))


def test_kernel_refusals_write_nothing():
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView
    L, T, H, D = 2, 32, 2, 64
    out = torch.full((L * 2 * T * H * D * 2,), FILL, dtype=torch.uint8, device="cuda")
    ptrs = torch.tensor([out.data_ptr()], dtype=torch.int64, device="cuda")
    ntok = torch.tensor([T], dtype=torch.int32, device="cuda")
    stok = torch.zeros(1, dtype=torch.int64, device="cuda")
    seg = torch.zeros(1, dtype=torch.int32, device="cuda")
    table = torch.zeros(1, D // 2, 2, dtype=torch.float32, device="cuda")
    lib = N.lib()

    def call(view, rd=D, off=0, style=0, l0=0, l1=L, n=1, ct=T, hf=0, tab=table.data_ptr(), p=ptrs.data_ptr(),
             nt=ntok.data_ptr(), st=stok.data_ptr(), sg=seg.data_ptr()):
        return lib.b200kv_pack_chunks_layers_rope(ctypes.byref(view.desc), n, ct, ctypes.c_void_p(nt),
                                                  ctypes.c_void_p(st), ctypes.c_void_p(sg), hf, l0, l1,
                                                  ctypes.c_void_p(p), ctypes.c_void_p(tab), rd, off, style, None)
    for dt in (torch.uint8, torch.float8_e4m3fn, torch.float8_e5m2):
        blob = torch.full((L, 2, T, H, D), 0x3C, dtype=torch.uint8, device="cuda").view(dt)
        assert call(KvView.from_blob(blob, "vllm")) < 0 and "16-bit" in N.last_error()
    view = KvView.from_blob(torch.randn(L, 2, T, H, D, device="cuda").to(torch.bfloat16), "vllm")
    for kw, msg in (({"rd": 63}, "even"), ({"rd": 0}, "even"), ({"rd": 32, "off": 33}, "exceeds"),
                    ({"off": -2}, "exceeds"), ({"style": 2}, "style"), ({"tab": 0}, "NULL"), ({"p": 0}, "NULL"),
                    ({"nt": 0}, "NULL"), ({"st": 0}, "NULL"), ({"sg": 0}, "NULL"), ({"l0": 1, "l1": 1}, "layer range"),
                    ({"l0": -1}, "layer range"), ({"l1": L + 1}, "layer range"), ({"n": 0}, "chunking"),
                    ({"ct": 0}, "chunking"), ({"hf": 2}, "hf_layout")):
        assert call(view, **kw) < 0, kw
        assert msg in N.last_error(), (msg, N.last_error())
    split = KvView.from_paged(_caches("split", _all_rows(L, 8, 16, H, D, torch.bfloat16, seed=1), 8, 16, H, D),
                              torch.arange(T, device="cuda"))
    assert call(split, hf=1) < 0 and "vllm chunks only" in N.last_error()
    torch.cuda.synchronize()
    assert bool((out == FILL).all())


# ---------------------------------------------------------------------------------------------- the engine
def _held(eng, items):
    """per (kind, chunk hash): sha256 of what the tier holds under the prefix ("p") or derived ("d") key, None where it
    holds nothing -- a container's bytes on the compressed host and disk tiers, a raw blob's on the raw tiers, the
    decoded blob elsewhere"""
    tier = eng.engine_
    torch.cuda.synchronize()
    out = []
    for kind, h in items:
        key = eng._make_key(h, "vllm") if kind == "p" else eng._derived_key(h, "vllm")
        if not tier.contains(key):
            out.append(None)
            continue
        d = getattr(tier, "dict", None)
        e = None if d is None else d.get(tier._key_to_path(key) if hasattr(tier, "_key_to_path") else key)
        if e is not None and hasattr(e, "ready"):
            e.ready.wait()
            if e.rec.blk is not None:
                data = bytes(e.rec.blk.view())[:e.rec.nbytes]
            else:
                with open(e.path, "rb") as f:
                    data = f.read()
        elif e is not None:
            t = e.host if hasattr(e, "host") else e
            data = t.contiguous().cpu().view(torch.uint8).numpy().tobytes()
        else:
            blob = next(iter(tier.batched_get(iter([key]))))
            data = blob.contiguous().cpu().view(torch.uint8).numpy().tobytes()
        out.append(hashlib.sha256(data).hexdigest())
    return out


def _n_held(digests):
    return sum(d is not None for d in digests)


def _items(eng, tok, segs):
    """every prefix and derived key a store of `segs` of `tok` could hold"""
    out = []
    for a, b in segs:
        for h in eng._prefix_hash(tok[a:b]):
            out += [("p", h), ("d", h)]
    return out


def _nan_caches(layout):
    return _caches(layout, _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0xFF), NB, BS, H_E, D_E)


def _write_layer(dst, layout, src_rows, l):
    for a, b in zip(dst[l], _layout(layout, src_rows[l], NB, BS, H_E, D_E)):
        a.copy_(b)


def _save_all(handle, write, order):
    for l in order:
        write(l)
        handle.save_layer(l)
    handle.finish()


def _read(eng, tok2, slots2, segs2, spec):
    dst = _caches("flash", _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x3C), NB, BS, H_E, D_E)
    ret = eng.retrieve_paged_segments(tok2, dst, slots2, segs2, spec)
    torch.cuda.synchronize()
    return ret, _cache_rows("flash", dst)


@pytest.mark.parametrize("tier", TIERS)
def test_engine_layerwise_stores_what_the_whole_form_stores(tier, lmserver, tmp_path, autorelease):
    """[A][gap][B][C][question]: A at token 0, B and C inside.  For every paged layout, an engine fed layer by layer
    (each layer written from NaN only just before its save, forward or reverse) holds the keys and bytes of an engine
    given store_paged_segments, and serves the same rows at other positions"""
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(D_E, 10000.0)
    docs = _docs(200 + TIERS.index(tier))
    tok, seg = _request(docs, ["A", "B", "C"], [0, 30, 17, 25], torch.Generator().manual_seed(26))
    segs = [seg["C"], seg["A"], seg["B"]]
    slots = _slots("vllm", len(tok), NB, BS, torch.Generator().manual_seed(27))
    tok2, seg2 = _request(docs, ["C", "A", "B"], [9, 3, 64, 5], torch.Generator().manual_seed(28))
    slots2 = _slots("vllm", len(tok2), NB, BS, torch.Generator().manual_seed(29))
    src_rows = _randn_rows(L_E, NB * BS, H_E, D_E, torch.bfloat16, seed=30)
    for li, layout in enumerate(LAYOUTS):
        # every token id moved by an offset of the engine's own: the engines of one test share a server or a disk
        # directory, so each stores under keys of its own
        ow, ol = 100000 * (2 * li + 1), 100000 * (2 * li + 2)
        whole = _engine(autorelease, tier, CS_E, lmserver, tmp_path, MODEL)
        whole.store_paged_segments(tok + ow, _caches(layout, src_rows, NB, BS, H_E, D_E), slots, segs, spec)
        _drain(whole)
        eng = _engine(autorelease, tier, CS_E, lmserver, tmp_path, MODEL)
        dst = _nan_caches(layout)
        h = eng.store_paged_segments_layerwise(tok + ol, dst, slots, segs, spec)
        _save_all(h, lambda l: _write_layer(dst, layout, src_rows, l), range(L_E)[::(-1 if li % 2 else 1)])
        _drain(eng)
        want = _held(whole, _items(whole, tok + ow, segs))
        assert _n_held(want) == sum((b - a + CS_E - 1) // CS_E for a, b in segs), (tier, layout)
        assert _held(eng, _items(eng, tok + ol, segs)) == want, (tier, layout)
        r0, rows0 = _read(whole, tok2 + ow, slots2, list(seg2.values()), spec)
        r1, rows1 = _read(eng, tok2 + ol, slots2, list(seg2.values()), spec)
        assert torch.equal(r0, r1) and int(r0.sum()) == sum(DOCS.values()), (tier, layout)
        for l in range(L_E):
            for i in range(2):
                assert torch.equal(rows0[l][i][slots2], rows1[l][i][slots2]), (tier, layout, l, i)


@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
@pytest.mark.parametrize("tier", ["cpu", "host-lossless"])
def test_dense_layerwise(fmt, tier, lmserver, tmp_path, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineMetadata
    from lmcache_b200.rope import RopeSpec
    from test_gpu_paged_layouts import _tier_config
    spec = RopeSpec.from_base(D_E, 10000.0, "gptj")
    docs = _docs(300)
    tok, seg = _request(docs, ["A", "B"], [0, 13, 20], torch.Generator().manual_seed(31))
    T = len(tok)
    g = torch.Generator(device="cuda").manual_seed(32)
    rows = [tuple(torch.randn(T, H_E, D_E, device="cuda", generator=g).to(torch.bfloat16) for _ in range(2))
            for _ in range(L_E)]
    kv = tuple((k, v) if fmt == "vllm" else (k.transpose(0, 1).contiguous(), v.transpose(0, 1).contiguous())
               for k, v in rows)
    engs = [autorelease(LMCacheEngine(_tier_config(tier, CS_E, lmserver, tmp_path),
                                      LMCacheEngineMetadata(MODEL, 1, 0, fmt, "bfloat16")))
            for i in range(2)]
    engs[0].store_segments(tok, kv, [seg["A"], seg["B"]], spec)
    dst = tuple((torch.full_like(k, float("nan")), torch.full_like(v, float("nan"))) for k, v in kv)

    def write(l):
        dst[l][0].copy_(kv[l][0])
        dst[l][1].copy_(kv[l][1])
    _save_all(engs[1].store_segments_layerwise(tok, dst, [seg["A"], seg["B"]], spec), write, range(L_E))
    _drain(engs[1])
    got = []
    for e in engs:
        keys = [e._make_key(h, fmt) for h in e._prefix_hash(tok[:seg["A"][1]])] + \
            [e._derived_key(h, fmt) for h in e._prefix_hash(tok[seg["B"][0]:seg["B"][1]])]
        assert all(e.engine_.contains(k) for k in keys)
        kv2, ret = e.retrieve_segments(tok, [seg["B"], seg["A"]], spec)
        assert int(ret.sum()) == DOCS["A"] + DOCS["B"]
        got.append(kv2)
    for l in range(L_E):
        for i in range(2):
            assert torch.equal(got[0][l][i].view(torch.int16), got[1][l][i].view(torch.int16)), (fmt, l, i)


@pytest.mark.parametrize("tier", ["cpu", "host-cachegen", "host-lossless"])
def test_mla_layerwise(tier, lmserver, tmp_path, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineMetadata
    from lmcache_b200.rope import RopeSpec
    from test_gpu_paged_layouts import _tier_config
    spec = RopeSpec.from_base(64, 10000.0, "gptj", 512)
    L, D, nb, bs = 3, 576, 60, 16
    g = torch.Generator(device="cuda").manual_seed(33)
    src = [torch.randn(nb, bs, D, device="cuda", generator=g).to(torch.bfloat16) for _ in range(L)]
    gen = torch.Generator().manual_seed(34)
    doc = torch.randint(0, 32000, (2 * CS_E + 10,), generator=gen) + 800000
    tokens = torch.cat([torch.randint(0, 32000, (77,), generator=gen), doc])
    slots = _slots("perm", len(tokens), nb, bs, torch.Generator().manual_seed(35))
    engs = [autorelease(LMCacheEngine(_tier_config(tier, CS_E, lmserver, tmp_path),
                                      LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16", True)))
            for i in range(2)]
    engs[0].store_paged_segments(tokens, src, slots, [(77, len(tokens))], spec)
    dst = [torch.full_like(c, float("nan")) for c in src]

    def write(l):
        dst[l].copy_(src[l])
    _save_all(engs[1].store_paged_segments_layerwise(tokens, dst, slots, [(77, len(tokens))], spec), write,
              reversed(range(L)))
    rows = []
    for e in engs:
        _drain(e)
        tok2 = torch.cat([tokens[:5], doc])
        out = [torch.full((nb, bs, D), 7, dtype=torch.bfloat16, device="cuda") for _ in range(L)]
        ret = e.retrieve_paged_segments(tok2, out, torch.arange(len(tok2), device="cuda"), [(5, len(tok2))], spec)
        torch.cuda.synchronize()
        assert int(ret.sum()) == len(doc)
        rows.append(out)
    for l in range(L):
        assert torch.equal(rows[0][l].view(torch.int16), rows[1][l].view(torch.int16)), (tier, l)


def test_skip_existing_and_partial_derived_hits(lmserver, tmp_path, autorelease):
    """B stored alone (prefix keys), C's first two chunks stored from inside a prompt (derived keys): the layer-wise
    form puts only C's later chunks, touches as the whole form does, and a second store puts nothing"""
    from lmcache_b200.rope import RopeSpec, derived_digest
    spec = RopeSpec.from_base(D_E, 10000.0)
    docs = _docs(400)
    tok, seg = _request(docs, ["B", "C"], [20, 11, 30], torch.Generator().manual_seed(36))
    slots = _slots("vllm", len(tok), NB, BS, torch.Generator().manual_seed(37))
    src_rows = _randn_rows(L_E, NB * BS, H_E, D_E, torch.bfloat16, seed=38)
    log = {}
    for form in ("whole", "layerwise"):
        eng = _engine(autorelease, "host-lossless", CS_E, lmserver, tmp_path, MODEL)
        src = _caches("flash", src_rows, NB, BS, H_E, D_E)
        a, b = seg["C"]
        pre = _caches("flash", src_rows, NB, BS, H_E, D_E)
        eng.store_paged_segments(tok[:b], pre, slots[:b], [(a, a + 2 * CS_E)], spec)   # C's chunks 0-1 (derived)
        ba, bb = seg["B"]
        eng.store_paged(tok[ba:bb], pre, slots[ba:bb])                                    # B stored alone
        puts, touches = [], []
        orig_put = eng.engine_.put_kv_chunks
        orig_touch = getattr(eng.engine_, "touch", None)

        def spy(keys, view, tok0, cs, **kw):
            puts.append([k.chunk_hash for k in keys])
            return orig_put(keys, view, tok0, cs, **kw)
        eng.engine_.put_kv_chunks = spy
        if orig_touch is not None:
            eng.engine_.touch = lambda keys: (touches.append([k.chunk_hash for k in keys]), orig_touch(keys))[1]
        if form == "whole":
            eng.store_paged_segments(tok, src, slots, [seg["B"], seg["C"]], spec)
        else:
            dst = _nan_caches("flash")
            h = eng.store_paged_segments_layerwise(tok, dst, slots, [seg["B"], seg["C"]], spec)
            _save_all(h, lambda l: _write_layer(dst, "flash", src_rows, l), range(L_E))
        hs = list(eng._prefix_hash(tok[a:b]))
        assert puts == [[derived_digest(x) for x in hs[2:]]], form
        log[form] = touches
        n = len(puts)
        if form == "whole":
            eng.store_paged_segments(tok, src, slots, [seg["B"], seg["C"]], spec)
        else:
            h = eng.store_paged_segments_layerwise(tok, src, slots, [seg["B"], seg["C"]], spec)
            _save_all(h, lambda l: None, range(L_E))
        assert len(puts) == n, form
    assert log["whole"] == log["layerwise"] and len(log["whole"]) > 0


@pytest.mark.parametrize("tier", ["host-cachegen", "host-lossless"])
def test_arena_overflow_keeps_a_prefix_and_does_not_grow_with_segments(tier, lmserver, tmp_path, autorelease,
                                                                        monkeypatch):
    """with LMCACHE_B200_LAYERWISE_STORE_MB below the first run's airtight bound, the first segment keeps a prefix of
    its chunks, byte-identical to the whole form's, and the later segments, which find the budget spent, keep none"""
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(128, 10000.0)
    L, H, D, cs, bs = 4, 8, 128, 256, 16
    n_doc, T0 = 8 * cs, 64
    T = T0 + 3 * n_doc
    g = torch.Generator(device="cuda").manual_seed(39)
    nb = T // bs + 2
    src = [tuple(torch.rand(nb, bs, H, D, device="cuda", generator=g).mul(2).sub(1).to(torch.bfloat16)
                 for _ in range(2)) for _ in range(L)]
    slots = torch.arange(T, device="cuda")
    tok = torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(40)) + 900000
    segs = [(T0 + i * n_doc, T0 + (i + 1) * n_doc) for i in range(3)]
    whole = _engine(autorelease, tier, cs, lmserver, tmp_path, MODEL)
    whole.store_paged_segments(tok, src, slots, segs, spec)
    items = _items(whole, tok, segs)
    want = _held(whole, items)
    assert _n_held(want) == 24
    monkeypatch.setenv("LMCACHE_B200_LAYERWISE_STORE_MB", "4")
    eng = _engine(autorelease, tier, cs, lmserver, tmp_path, MODEL)
    h = eng.store_paged_segments_layerwise(tok, src, slots, segs, spec)
    arenas = [getattr(x, "arena_bytes", 0) for x in h._enc.handles]
    assert arenas == [4 << 20, 1, 1], arenas        # the later runs find the budget spent: their chunks are misses
    _save_all(h, lambda l: None, range(L))
    _drain(eng)
    got = _held(eng, items)
    first = [i for i, (kind, _) in enumerate(items) if kind == "d"][:8]      # the first segment's derived keys
    kept = [i for i, d in enumerate(got) if d is not None]
    assert 0 < len(kept) < 8 and kept == first[:len(kept)], kept
    assert all(got[i] == want[i] for i in kept)


@pytest.mark.parametrize("tier", ["lm-torch", "host-cachegen"])
def test_fallback_tiers(tier, lmserver, tmp_path, autorelease):
    """the torch-serde remote tier and a CacheGen chunk over 256 tokens take the whole form at finish()"""
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(D_E, 10000.0)
    cs = CS_E if tier == "lm-torch" else 512
    docs = _docs(500)
    tok, seg = _request(docs, ["A", "C"], [0, 40, 9], torch.Generator().manual_seed(41))
    slots = _slots("vllm", len(tok), NB, BS, torch.Generator().manual_seed(42))
    src_rows = _randn_rows(L_E, NB * BS, H_E, D_E, torch.bfloat16, seed=43)
    whole = _engine(autorelease, tier, cs, lmserver, tmp_path, MODEL)
    whole.store_paged_segments(tok + 10 ** 6, _caches("flash", src_rows, NB, BS, H_E, D_E), slots, list(seg.values()),
                               spec)
    eng = _engine(autorelease, tier, cs, lmserver, tmp_path, MODEL)
    dst = _nan_caches("flash")
    h = eng.store_paged_segments_layerwise(tok + 2 * 10 ** 6, dst, slots, list(seg.values()), spec)
    assert h._enc is None
    _save_all(h, lambda l: _write_layer(dst, "flash", src_rows, l), range(L_E))
    for e in (whole, eng):
        _drain(e)
    want = _held(whole, _items(whole, tok + 10 ** 6, list(seg.values())))
    assert _held(eng, _items(eng, tok + 2 * 10 ** 6, list(seg.values()))) == want and _n_held(want) > 0


def test_refusals_and_a_dropped_handle_store_nothing(lmserver, tmp_path, autorelease):
    import gc
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(D_E, 10000.0)
    eng = _engine(autorelease, "host-lossless", CS_E, lmserver, tmp_path, MODEL)
    docs = _docs(600)
    tok, seg = _request(docs, ["A", "B"], [0, 5, 5], torch.Generator().manual_seed(44))
    slots = _slots("vllm", len(tok), NB, BS, torch.Generator().manual_seed(45))
    src = _caches("flash", _randn_rows(L_E, NB * BS, H_E, D_E, torch.bfloat16, seed=46), NB, BS, H_E, D_E)
    fp8 = _caches("flash", _all_rows(L_E, NB, BS, H_E, D_E, torch.float8_e4m3fn, seed=47), NB, BS, H_E, D_E)
    puts = []
    orig = eng.engine_.put_kv_chunks
    eng.engine_.put_kv_chunks = lambda *a, **kw: (puts.append(1), orig(*a, **kw))[1]
    with pytest.raises(TypeError):
        eng.store_paged_segments_layerwise(tok, fp8, slots, [seg["B"]], spec)
    with pytest.raises(ValueError, match="overlap"):
        eng.store_paged_segments_layerwise(tok, src, slots, [seg["B"], (seg["B"][1] - 1, seg["B"][1] + 3)], spec)
    with pytest.raises(ValueError, match="do not fit"):
        eng.store_paged_segments_layerwise(tok, src, slots, [seg["B"]], RopeSpec.from_base(D_E, 1e4, "neox", 8))
    kv = tuple((k.view(-1, H_E, D_E)[slots], v.view(-1, H_E, D_E)[slots]) for k, v in src)
    with pytest.raises(ValueError, match="overlap"):
        eng.store_segments_layerwise(tok, kv, [seg["B"], seg["B"]], spec)
    # a handle dropped without finish(), one closed, one finished with a layer missing
    h = eng.store_paged_segments_layerwise(tok, src, slots, [seg["A"], seg["B"]], spec)
    h.save_layer(0)
    del h
    gc.collect()
    h = eng.store_paged_segments_layerwise(tok, src, slots, [seg["A"], seg["B"]], spec)
    h.close()
    h = eng.store_paged_segments_layerwise(tok, src, slots, [seg["A"], seg["B"]], spec)
    for l in range(L_E - 1):
        h.save_layer(l)
    with pytest.raises(ValueError, match="never|before layers"):
        h.finish()
    torch.cuda.synchronize()
    _drain(eng)
    assert puts == []
    assert _n_held(_held(eng, _items(eng, tok, [seg["A"], seg["B"]]))) == 0
