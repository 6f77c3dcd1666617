"""GPU: the layer-wise segment retrieve.  b200kv_rope_shift_layers against b200kv_rope_shift in every layout a kv_desc
carries, and its refusals; LMCacheEngine.retrieve_paged_segments_layerwise / retrieve_segments_layerwise against the
whole forms on every tier and paged layout, with one event per layer where the tier is layer-major and each layer final
on a side stream right after its wait."""
import ctypes

import pytest
import torch

from test_gpu_host_tier import MODEL
from test_gpu_paged_layouts import (BS, D_E, H_E, L_E, LAYOUTS, NB, TIERS, _all_rows, _cache_rows, _caches, _engine,
                                    _slots, lmserver)  # noqa: F401 -- lmserver is a fixture
from test_gpu_segments import CS, DOCS, KERNEL_LAYOUTS, ROT, SHIFTS, _doc_setup, _request, _seg_pattern, _target

pytestmark = pytest.mark.gpu

# the tiers whose get_kv_layerwise_runs serves segments layer-major; the rest run the whole retrieve
LAYER_MAJOR = ("cpu", "cuda", "host-cachegen", "host-lossless", "disk-cachegen", "disk-lossless", "hybrid")


def _bits(get):
    return [tuple(None if t is None else t.clone().view(torch.int16) for t in p) for p in get()]


def _table(shifts, spec):
    from lmcache_b200.rope import rope_table
    return rope_table(torch.tensor(shifts, dtype=torch.int64, device="cuda"), spec)


def _shift_layers(view, a, b, seg, table, spec):
    from lmcache_b200 import _native as N
    from lmcache_b200.rope import STYLES
    return N.lib().b200kv_rope_shift_layers(ctypes.byref(view.desc), a, b, 5, seg.numel(), ctypes.c_void_p(seg.data_ptr()),
                                            ctypes.c_void_p(table.data_ptr()), spec.rotary_dim, spec.offset,
                                            STYLES[spec.style], None)


def _fresh(kind, dtype, H, D, seed):
    torch.manual_seed(seed)                          # a paged latent cache draws from the default generator
    return _target(kind, dtype, 96, H, D, seed)


def _layer_ranges_equal_whole(kind, dtype, spec, H, D, seed):
    from lmcache_b200 import _native as N
    seg = torch.tensor(_seg_pattern(), dtype=torch.int32, device="cuda")
    table = _table(SHIFTS, spec)
    view, get, _ = _fresh(kind, dtype, H, D, seed)
    N.check(N.lib().b200kv_rope_shift(ctypes.byref(view.desc), 5, seg.numel(), ctypes.c_void_p(seg.data_ptr()),
                                      ctypes.c_void_p(table.data_ptr()), spec.rotary_dim, spec.offset,
                                      0 if spec.style == "neox" else 1, None))
    torch.cuda.synchronize()
    whole = _bits(get)
    view, get, _ = _fresh(kind, dtype, H, D, seed)
    before = _bits(get)
    N.check(_shift_layers(view, 1, 2, seg, table, spec))
    torch.cuda.synchronize()
    mid = _bits(get)
    assert torch.equal(mid[1][0], whole[1][0]), (kind, "layer 1's keys")
    assert torch.equal(mid[0][0], before[0][0]), (kind, "layer 0 touched")
    for l in range(2):
        if mid[l][1] is not None:
            assert torch.equal(mid[l][1], before[l][1]), (kind, l, "V touched")
    N.check(_shift_layers(view, 0, 1, seg, table, spec))           # ranges covering each layer once = one full shift
    torch.cuda.synchronize()
    for got, want in zip(_bits(get), whole):
        for g, w in zip(got, want):
            assert (g is None and w is None) or torch.equal(g, w), kind


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("style", ["neox", "gptj"])
@pytest.mark.parametrize("kind", KERNEL_LAYOUTS)
def test_shift_layers_equals_shift(dtype, style, kind):
    from lmcache_b200.rope import RopeSpec
    for i, (rd, off) in enumerate(ROT):                    # vector and element-wise paths, partial rotary
        _layer_ranges_equal_whole(kind, dtype, RopeSpec.from_base(rd, 10000.0, style, off), 4, 128, seed=30 + i)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("style", ["neox", "gptj"])
@pytest.mark.parametrize("kind", ["latent", "latent-paged"])
def test_shift_layers_latent_offset_512(dtype, style, kind):
    from lmcache_b200.rope import RopeSpec
    _layer_ranges_equal_whole(kind, dtype, RopeSpec.from_base(64, 10000.0, style, 512), 1, 576, seed=40)


def test_shift_layers_refusals_write_nothing():
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(64, 10000.0)
    seg = torch.tensor(_seg_pattern(), dtype=torch.int32, device="cuda")
    table = _table(SHIFTS, spec)
    blob = torch.full((2, 2, 96, 2, 64), 0x3C3C, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    view = KvView.from_blob(blob, "vllm")
    for a, b in ((-1, 1), (1, 1), (1, 0), (0, 3), (2, 3)):
        assert _shift_layers(view, a, b, seg, table, spec) < 0, (a, b)
        assert "layer range" in N.last_error()
    fp8 = torch.full((2, 2, 96, 2, 64), 0x3C, dtype=torch.uint8, device="cuda").view(torch.float8_e4m3fn)
    assert _shift_layers(KvView.from_blob(fp8, "vllm"), 0, 1, seg, table, spec) < 0 and "16-bit" in N.last_error()
    assert _shift_layers(view, 0, 1, seg, table, RopeSpec.from_base(64, 1e4, "neox", 8)) < 0
    assert "exceeds" in N.last_error()
    torch.cuda.synchronize()
    assert bool((blob.view(torch.int16) == 0x3C3C).all()) and bool((fp8.view(torch.uint8) == 0x3C).all())


# ---------------------------------------------------------------------------------------------- the engine
def _per_layer(r):
    evs = [r._upload.ready(l) for l in range(r.num_layers)]
    assert len({id(e) for e in evs}) == r.num_layers                 # one event per layer, not one for all


def _layerwise_paged(eng, tokens, b, slots, segs, spec, layer_major):
    """retrieve_paged_segments_layerwise into a fresh cache of layout b: (ret_mask, final rows, the copy of each layer
    taken on a side stream right after wait_layer)"""
    dst = _caches(b, _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x3C), NB, BS, H_E, D_E)
    r = eng.retrieve_paged_segments_layerwise(tokens, dst, slots, segs, spec)
    assert r.kv is None and r.num_layers == L_E
    if layer_major:
        _per_layer(r)
    early = []
    for l in range(L_E):
        side = torch.cuda.Stream()
        r.wait_layer(l, side)
        with torch.cuda.stream(side):
            early.append(tuple(t.clone() for t in _cache_rows(b, dst)[l]))
        torch.cuda.current_stream().wait_stream(side)
    r.synchronize()
    return r.ret_mask, _cache_rows(b, dst), early


def _whole_paged(eng, tokens, b, slots, segs, spec):
    dst = _caches(b, _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x3C), NB, BS, H_E, D_E)
    ret = eng.retrieve_paged_segments(tokens, dst, slots, segs, spec)
    torch.cuda.synchronize()
    return ret, _cache_rows(b, dst)


def _same_paged(got, want, what):
    ret_g, rows_g, early = got
    ret_w, rows_w = want
    assert torch.equal(ret_g, ret_w), what
    for l in range(L_E):
        for i in range(2):
            assert torch.equal(rows_g[l][i].view(torch.int16), rows_w[l][i].view(torch.int16)), (what, l, i)
            assert torch.equal(early[l][i].view(torch.int16), rows_w[l][i].view(torch.int16)), (what, l, i, "early")


def _same_dense(eng, tokens, segs, spec, layer_major, what):
    kv_w, ret_w = eng.retrieve_segments(tokens, segs, spec)
    r = eng.retrieve_segments_layerwise(tokens, segs, spec)
    if layer_major and r.num_layers:
        _per_layer(r)
    early = []
    for l in range(r.num_layers):
        side = torch.cuda.Stream()
        r.wait_layer(l, side)
        with torch.cuda.stream(side):
            early.append(tuple(t.clone() for t in r.kv[l]))
        torch.cuda.current_stream().wait_stream(side)
    r.synchronize()
    assert torch.equal(r.ret_mask, ret_w), what
    assert len(r.kv) == len(kv_w), what
    for l in range(len(kv_w)):
        for i in range(2):
            assert torch.equal(r.kv[l][i].view(torch.int16), kv_w[l][i].view(torch.int16)), (what, l, i)
            assert torch.equal(early[l][i].view(torch.int16), kv_w[l][i].view(torch.int16)), (what, l, i, "early")


@pytest.mark.parametrize("tier", TIERS)
def test_engine_layerwise_equals_whole(tier, lmserver, tmp_path, autorelease):
    _equals_whole(tier, tier in LAYER_MAJOR, 5, lmserver, tmp_path, autorelease)


@pytest.mark.parametrize("tier", ["lm-cachegen", "lm-lossless", "hybrid"])
def test_engine_layerwise_ranged_remote(tier, lmserver, tmp_path, autorelease, monkeypatch):
    """opted in to ranged reads, the remote tier and both parts of the hybrid tier serve segments layer-major"""
    monkeypatch.setenv("LMCACHE_B200_REMOTE_LAYERWISE", "1")
    _equals_whole(tier, True, 7, lmserver, tmp_path, autorelease)


def _equals_whole(tier, layer_major, ai, lmserver, tmp_path, autorelease):
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(D_E, 10000.0)
    eng = _engine(autorelease, tier, CS, lmserver, tmp_path, MODEL)
    doc_tokens, _ = _doc_setup(eng, tier, ai, 11)
    tokens, segs = _request(doc_tokens, torch.Generator().manual_seed(16))
    order = [segs["C"], segs["A"], segs["B"]]
    slots = _slots("vllm", len(tokens), NB, BS, torch.Generator().manual_seed(17))
    for b in LAYOUTS:
        major = layer_major and not (b == "split" and tier not in ("cpu", "cuda"))
        got = _layerwise_paged(eng, tokens, b, slots, order, spec, major)
        want = _whole_paged(eng, tokens, b, slots, order, spec)
        assert int(want[0].sum()) == sum(DOCS[n][1] for n in DOCS), (tier, b)
        _same_paged(got, want, (tier, b))
    _same_dense(eng, tokens, order, spec, layer_major, tier)
    # a segment at 0: one segment (0, T) is retrieve_paged_layerwise
    toks = doc_tokens["C"]
    T = len(toks)
    sl = _slots("vllm", T, NB, BS, torch.Generator().manual_seed(18))
    for b in LAYOUTS:
        major = layer_major and not (b == "split" and tier not in ("cpu", "cuda"))
        got = _layerwise_paged(eng, toks, b, sl, [(0, T)], spec, major)
        dst = _caches(b, _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x3C), NB, BS, H_E, D_E)
        r = eng.retrieve_paged_layerwise(toks, dst, sl)
        r.synchronize()
        _same_paged(got, (r.ret_mask, _cache_rows(b, dst)), (tier, b, "(0, T)"))


@pytest.mark.parametrize("tier", ["cpu", "cuda", "host-cachegen", "host-lossless", "disk-lossless", "hybrid"])
def test_engine_layerwise_continuation(tier, lmserver, tmp_path, autorelease):
    """a document stored inside one prompt (store_paged_segments, derived keys) and served inside another"""
    from lmcache_b200.rope import RopeSpec
    from test_gpu_segments import _randn_rows
    spec = RopeSpec.from_base(D_E, 10000.0)
    eng = _engine(autorelease, tier, CS, lmserver, tmp_path, MODEL)
    gen = torch.Generator().manual_seed(19)
    doc = torch.randint(0, 32000, (3 * CS + 7,), generator=gen) + 700000 + 1000 * TIERS.index(tier)
    head = doc[:CS]                                     # stored alone: the continuation starts at chunk 1
    pre1, pre2 = torch.randint(0, 32000, (41,), generator=gen), torch.randint(0, 32000, (90,), generator=gen)
    src = _caches("flash", _randn_rows(L_E, NB * BS, H_E, D_E, torch.bfloat16, seed=23), NB, BS, H_E, D_E)
    eng.store_paged(head, src, torch.arange(CS, device="cuda"))
    t1 = torch.cat([pre1, doc])
    eng.store_paged_segments(t1, src, torch.arange(len(t1), device="cuda"), [(len(pre1), len(t1))], spec)
    if hasattr(eng.engine_, "drain"):
        eng.engine_.drain()
    t2 = torch.cat([pre2, doc, pre1[:9]])
    seg = [(len(pre2), len(pre2) + len(doc))]
    slots = _slots("vllm", len(t2), NB, BS, torch.Generator().manual_seed(20))
    for b in LAYOUTS:
        major = tier in LAYER_MAJOR and not (b == "split" and tier not in ("cpu", "cuda"))
        got = _layerwise_paged(eng, t2, b, slots, seg, spec, major)
        want = _whole_paged(eng, t2, b, slots, seg, spec)
        assert int(want[0].sum()) == len(doc), (tier, b)
        _same_paged(got, want, (tier, b))
    _same_dense(eng, t2, seg, spec, tier in LAYER_MAJOR, tier)


@pytest.mark.parametrize("tier", ["cpu", "host-cachegen", "host-lossless"])
def test_engine_layerwise_mla(tier, lmserver, tmp_path, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineMetadata
    from lmcache_b200.rope import RopeSpec
    from test_gpu_paged_layouts import _tier_config
    spec = RopeSpec.from_base(64, 10000.0, "gptj", 512)
    eng = autorelease(LMCacheEngine(_tier_config(tier, CS, lmserver, tmp_path),
                                    LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "bfloat16", True)))
    L, D, nb, bs = 3, 576, 60, 16
    g = torch.Generator(device="cuda").manual_seed(29)
    src = [torch.randn(nb, bs, D, device="cuda", generator=g).to(torch.bfloat16) for _ in range(L)]
    gen = torch.Generator().manual_seed(30)
    doc = torch.randint(0, 32000, (2 * CS + 10,), generator=gen) + 950000 + 1000 * len(tier)
    eng.store_paged(doc, src, torch.arange(len(doc), device="cuda"))
    if hasattr(eng.engine_, "drain"):
        eng.engine_.drain()
    pre = torch.randint(0, 32000, (77,), generator=gen)
    tokens = torch.cat([pre, doc])
    slots = _slots("perm", len(tokens), nb, bs, torch.Generator().manual_seed(31))
    d1 = [torch.full((nb, bs, D), 7, dtype=torch.bfloat16, device="cuda") for _ in range(L)]
    d2 = [torch.full((nb, bs, D), 7, dtype=torch.bfloat16, device="cuda") for _ in range(L)]
    r = eng.retrieve_paged_segments_layerwise(tokens, d1, slots, [(77, len(tokens))], spec)
    _per_layer(r)
    r.synchronize()
    ret = eng.retrieve_paged_segments(tokens, d2, slots, [(77, len(tokens))], spec)
    torch.cuda.synchronize()
    assert torch.equal(r.ret_mask, ret) and int(ret.sum()) == len(doc)
    for a, b in zip(d1, d2):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    kv_w, ret_w = eng.retrieve_segments(tokens, [(77, len(tokens))], spec)
    r = eng.retrieve_segments_layerwise(tokens, [(77, len(tokens))], spec)
    r.synchronize()
    assert torch.equal(r.ret_mask, ret_w)
    for a, b in zip(r.kv, kv_w):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("tier", ["cpu", "host-cachegen", "disk-lossless"])
def test_engine_layerwise_total_miss(tier, lmserver, tmp_path, autorelease):
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(D_E, 10000.0)
    eng = _engine(autorelease, tier, CS, lmserver, tmp_path, MODEL)       # a fresh engine: no geometry known
    tokens = torch.randint(0, 32000, (3 * CS,), generator=torch.Generator().manual_seed(33)) + 990000
    r = eng.retrieve_segments_layerwise(tokens, [(10, 2 * CS)], spec)
    assert r.num_layers == 0 and r.kv == () and not bool(r.ret_mask.any())
    r.wait_layer(0)
    r.synchronize()
    slots = _slots("vllm", len(tokens), NB, BS, torch.Generator().manual_seed(34))
    got = _layerwise_paged(eng, tokens, "flash", slots, [(10, 2 * CS)], spec, False)
    assert not bool(got[0].any())
    for l in range(L_E):
        for i in range(2):
            assert bool((got[1][l][i].view(torch.uint8) == 0x3C).all())


@pytest.mark.parametrize("tier", ["cpu", "host-lossless"])
def test_engine_layerwise_refusals_fetch_nothing(tier, lmserver, tmp_path, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineMetadata
    from lmcache_b200.rope import RopeSpec
    from test_gpu_paged_layouts import _tier_config
    spec = RopeSpec.from_base(D_E, 10000.0)
    eng = _engine(autorelease, tier, CS, lmserver, tmp_path, MODEL)
    doc_tokens, _ = _doc_setup(eng, tier, 6, 13)
    tokens, segs = _request(doc_tokens, torch.Generator().manual_seed(36))
    slots = _slots("vllm", len(tokens), NB, BS, torch.Generator().manual_seed(37))
    calls = []
    tier_obj = eng.engine_
    for name in ("get_kv_layerwise_runs", "get_kv_into", "contains", "touch", "peek_geometry", "get", "batched_get"):
        f = getattr(tier_obj, name, None)
        if f is None:
            continue
        setattr(tier_obj, name, lambda *a, _n=name, _f=f, **k: (calls.append(_n), _f(*a, **k))[1])
    dst = _caches("flash", _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x3C), NB, BS, H_E, D_E)
    bad = [segs["A"], (segs["A"][1] - 1, segs["A"][1] + 5)]
    with pytest.raises(ValueError, match="overlap"):
        eng.retrieve_paged_segments_layerwise(tokens, dst, slots, [segs["B"]] + bad, spec)
    with pytest.raises(ValueError, match="do not fit"):
        eng.retrieve_paged_segments_layerwise(tokens, dst, slots, [segs["B"]], RopeSpec.from_base(D_E, 1e4, "neox", 8))
    with pytest.raises(ValueError, match="overlap"):
        eng.retrieve_segments_layerwise(tokens, [segs["A"], segs["A"]], spec)
    fp8 = _caches("flash", _all_rows(L_E, NB, BS, H_E, D_E, torch.float8_e4m3fn, seed=0, fill=0x3C), NB, BS, H_E, D_E)
    with pytest.raises(TypeError):
        eng.retrieve_paged_segments_layerwise(tokens, fp8, slots, [segs["B"]], spec)
    e8 = autorelease(LMCacheEngine(_tier_config(tier, CS, lmserver, tmp_path),
                                   LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "fp8")))
    with pytest.raises(TypeError):
        e8.retrieve_segments_layerwise(tokens, [segs["B"]], spec)
    assert calls == []
    torch.cuda.synchronize()
    for l in range(L_E):
        for i in range(2):
            assert bool((_cache_rows("flash", dst)[l][i].view(torch.uint8) == 0x3C).all())


# ---------------------------------------------------------------------------------------------- fused unpack + turn
CHUNKS = [(5, 16, 0), (21, 16, 1), (37, 5, -1), (50, 16, 2), (80, 3, 3)]   # (destination token, tokens, table row)


def _chunk_blobs(view, l0, l1, dtype, misalign):
    """one random layer-range blob per chunk (the view's chunk layout), chunk 1 at a misaligned address if asked"""
    ppl = 1 if view.latent else 2
    g = torch.Generator(device="cuda").manual_seed(77)
    blobs, ptrs = [], []
    for i, (_, t, _) in enumerate(CHUNKS):
        n = (l1 - l0) * ppl * t * view.H * view.D
        store = torch.randn(n + 8, generator=g, device="cuda").to(dtype)
        off = 1 if (misalign and i == 1) else 0
        blobs.append(store)
        ptrs.append(store.data_ptr() + 2 * off)
    return blobs, torch.tensor(ptrs, dtype=torch.int64, device="cuda")


def _fused_vs_composed(kind, dtype, spec, H, D, l0, l1, misalign, seed):
    from lmcache_b200 import _native as N
    from lmcache_b200.rope import STYLES
    table = _table(SHIFTS, spec)
    ntok = torch.tensor([t for _, t, _ in CHUNKS], dtype=torch.int32, device="cuda")
    dtok = torch.tensor([a for a, _, _ in CHUNKS], dtype=torch.int64, device="cuda")
    cseg = torch.tensor([s for _, _, s in CHUNKS], dtype=torch.int32, device="cuda")
    sot = [-1] * 96
    for a, t, s in CHUNKS:
        sot[a:a + t] = [s] * t
    seg = torch.tensor(sot, dtype=torch.int32, device="cuda")
    view, get, _ = _fresh(kind, dtype, H, D, seed)
    before = _bits(get)
    blobs, ptrs = _chunk_blobs(view, l0, l1, dtype, misalign)
    hf = int(view.fmt == "huggingface")
    N.check(N.lib().b200kv_unpack_chunks_layers_rope(
        ctypes.c_void_p(ptrs.data_ptr()), len(CHUNKS), 16, ctypes.c_void_p(ntok.data_ptr()),
        ctypes.c_void_p(dtok.data_ptr()), ctypes.c_void_p(cseg.data_ptr()), hf, l0, l1, ctypes.byref(view.desc),
        ctypes.c_void_p(table.data_ptr()), spec.rotary_dim, spec.offset, STYLES[spec.style], None))
    torch.cuda.synchronize()
    fused = _bits(get)
    view, get, _ = _fresh(kind, dtype, H, D, seed)
    for j, (a, t, _) in enumerate(CHUNKS):
        N.check(N.lib().b200kv_unpack_chunks_layers(ctypes.c_void_p(ptrs.data_ptr() + 8 * j), 1, t, t, hf, l0, l1,
                                                    ctypes.byref(view.desc), a, None))
    N.check(N.lib().b200kv_rope_shift_layers(ctypes.byref(view.desc), l0, l1, 0, 96, ctypes.c_void_p(seg.data_ptr()),
                                             ctypes.c_void_p(table.data_ptr()), spec.rotary_dim, spec.offset,
                                             STYLES[spec.style], None))
    torch.cuda.synchronize()
    composed = _bits(get)
    for l, (f, c, b) in enumerate(zip(fused, composed, before)):
        for i in range(2):
            if f[i] is None:
                continue
            assert torch.equal(f[i], c[i]), (kind, l, i, misalign)
            if not l0 <= l < l1:
                assert torch.equal(f[i], b[i]), (kind, l, i, "outside the layer range")
    del blobs


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("style", ["neox", "gptj"])
@pytest.mark.parametrize("kind", KERNEL_LAYOUTS)
def test_fused_unpack_equals_unpack_then_shift(dtype, style, kind):
    from lmcache_b200.rope import RopeSpec
    for i, (rd, off) in enumerate(ROT):                    # vector and element-wise paths, partial rotary
        spec = RopeSpec.from_base(rd, 10000.0, style, off)
        _fused_vs_composed(kind, dtype, spec, 4, 128, 1, 2, misalign=i == 0, seed=50 + i)
        _fused_vs_composed(kind, dtype, spec, 4, 128, 0, 2, misalign=False, seed=60 + i)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("style", ["neox", "gptj"])
@pytest.mark.parametrize("kind", ["latent", "latent-paged"])
def test_fused_unpack_latent_offset_512(dtype, style, kind):
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(64, 10000.0, style, 512)
    _fused_vs_composed(kind, dtype, spec, 1, 576, 0, 1, misalign=True, seed=70)
    _fused_vs_composed(kind, dtype, spec, 1, 576, 0, 2, misalign=False, seed=71)


def test_fused_unpack_refusals_write_nothing():
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView
    spec_rd, L = 64, 2
    blob = torch.full((L, 2, 96, 2, 64), 0x3C3C, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    fp8 = torch.full((L, 2, 96, 2, 64), 0x3C, dtype=torch.uint8, device="cuda").view(torch.float8_e4m3fn)
    src = torch.zeros(2 * 16 * 2 * 64, dtype=torch.bfloat16, device="cuda")
    ptrs = torch.tensor([src.data_ptr()], dtype=torch.int64, device="cuda")
    ntok = torch.tensor([16], dtype=torch.int32, device="cuda")
    dtok = torch.tensor([0], dtype=torch.int64, device="cuda")
    cseg = torch.tensor([0], dtype=torch.int32, device="cuda")
    table = torch.zeros(1, 32, 2, dtype=torch.float32, device="cuda")

    def call(t, l0=0, l1=1, rd=spec_rd, off=0, style=0, tab=table.data_ptr(), p=ptrs.data_ptr(), n=1, ct=16):
        v = KvView.from_blob(t, "vllm")
        return N.lib().b200kv_unpack_chunks_layers_rope(ctypes.c_void_p(p), n, ct, ctypes.c_void_p(ntok.data_ptr()),
                                                        ctypes.c_void_p(dtok.data_ptr()), ctypes.c_void_p(cseg.data_ptr()),
                                                        0, l0, l1, ctypes.byref(v.desc), ctypes.c_void_p(tab), rd, off,
                                                        style, None)
    assert call(fp8) < 0 and "16-bit" in N.last_error()
    for kw, msg in ((dict(l0=1, l1=1), "layer range"), (dict(l1=3), "layer range"), (dict(rd=63), "even"),
                    (dict(off=8), "exceeds"), (dict(style=2), "style"), (dict(tab=0), "NULL"), (dict(p=0), "NULL"),
                    (dict(n=0), "chunking"), (dict(ct=0), "chunking")):
        assert call(blob, **kw) < 0, kw
        assert msg in N.last_error(), (kw, N.last_error())
    torch.cuda.synchronize()
    assert bool((blob.view(torch.int16) == 0x3C3C).all()) and bool((fp8.view(torch.uint8) == 0x3C).all())


def _shift_kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "rope_shift_kernel" in e.name]


def test_shift_layers_alignment_looks_at_the_range_only():
    """a misaligned key plane outside the range keeps the vector path (NP = 8); one inside selects the element path
    (NP = 1); the bits are those of the full shift either way"""
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(64, 10000.0)
    seg = torch.tensor(_seg_pattern(), dtype=torch.int32, device="cuda")
    table = _table(SHIFTS, spec)
    n = 96 * 2 * 64
    g = torch.Generator(device="cuda").manual_seed(90)
    src = [torch.randn(n + 8, generator=g, device="cuda").to(torch.bfloat16) for _ in range(6)]

    def make(skew):
        """layer 0's K plane one element into its storage (misaligned) when skewed"""
        kv = tuple((src[2 * l].clone()[(1 if skew and l == 0 else 0):][:n].view(96, 2, 64),
                    src[2 * l + 1].clone()[:n].view(96, 2, 64)) for l in range(3))
        return kv, KvView.from_tuple(kv, "vllm")
    kv_a, va = make(True)
    assert va.desc is not None and kv_a[0][0].data_ptr() % 16 != 0
    names = _shift_kernel_names(lambda: N.check(_shift_layers(va, 1, 3, seg, table, spec)))
    assert names and all(", 8," in x or "Li8E" in x for x in names), names
    names = _shift_kernel_names(lambda: N.check(_shift_layers(va, 0, 1, seg, table, spec)))
    assert names and all(", 1," in x or "Li1E" in x for x in names), names
    kv_c, vc = make(True)                                  # the same data, turned by one full shift
    N.check(N.lib().b200kv_rope_shift(ctypes.byref(vc.desc), 5, seg.numel(), ctypes.c_void_p(seg.data_ptr()),
                                      ctypes.c_void_p(table.data_ptr()), 64, 0, 0, None))
    torch.cuda.synchronize()
    for l in range(3):
        for i in range(2):
            assert torch.equal(kv_a[l][i].view(torch.int16), kv_c[l][i].view(torch.int16)), (l, i)
