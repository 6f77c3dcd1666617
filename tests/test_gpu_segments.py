"""GPU: non-prefix KV reuse.  b200kv_rope_shift against the float64 statement of tests/rope_ref.py in every layout a
kv_desc carries, its refusals, and LMCacheEngine.retrieve_paged_segments / retrieve_segments on every tier: documents
stored as prompts of their own, served inside a longer request at new positions with their keys turned."""
import ctypes

import numpy as np
import pytest
import torch

from rope_ref import partner, rotate, tolerance
from test_gpu_host_tier import MODEL
from test_gpu_paged_layouts import (BS, D_E, H_E, L_E, LAYOUTS, NB, TIERS, _all_rows, _cache_rows, _caches, _engine,
                                    _layout, _rows, _slots, lmserver)  # noqa: F401 -- lmserver is a fixture

pytestmark = pytest.mark.gpu
NAMES = {torch.bfloat16: "bfloat16", torch.float16: "float16"}
SHIFTS = [1, 255, 4096, 65535]


def _seg_pattern():
    """tokens [5, 85) of 96: four segments with -1 gaps between them"""
    return [-1] * 7 + [0] * 20 + [-1] * 3 + [1] * 15 + [2] * 20 + [-1] * 5 + [3] * 10


def _shift(view, tok_begin, seg, shifts, spec):
    from lmcache_b200.rope import rope_shift
    rope_shift(view, tok_begin, torch.tensor(seg, dtype=torch.int32, device="cuda"),
               torch.tensor(shifts, dtype=torch.int64, device="cuda"), spec)
    torch.cuda.synchronize()


def _randn_rows(L, n, H, D, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [tuple(torch.randn(n, H, D, generator=g, device="cuda").to(dtype) for _ in range(2)) for _ in range(L)]


def _target(kind, dtype, T, H, D, seed):
    """(view, rows(), slot of each token): rows() gives per layer (K, V) as [n_rows, H, D] of the view's storage (V None
    for a latent KV), token t of the view living in row slot[t]"""
    from lmcache_b200.codec import KvView
    L = 2
    if kind.startswith("latent"):
        if kind == "latent":
            blob = torch.randn(L, T, D, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed)).to(dtype)
            return KvView.from_blob(blob, "vllm"), lambda: [(blob[l].unsqueeze(1), None) for l in range(L)], np.arange(T)
        nb, bs = 16, 16
        caches = [torch.randn(nb, bs, D, device="cuda").to(dtype) for _ in range(L)]
        slots = _slots("perm", T, nb, bs, torch.Generator().manual_seed(seed))
        return (KvView.from_paged(caches, slots), lambda: [(c.view(nb * bs, 1, D), None) for c in caches],
                slots.cpu().numpy())
    if kind in ("vllm", "huggingface", "tuple"):
        rows = _randn_rows(L, T, H, D, dtype, seed)
        if kind == "tuple":
            kv = tuple((k.clone(), v.clone()) for k, v in rows)
            return KvView.from_tuple(kv, "vllm"), lambda: list(kv), np.arange(T)
        blob = torch.stack([torch.stack(p) for p in rows])                         # [L, 2, T, H, D]
        if kind == "huggingface":
            blob = blob.transpose(2, 3).contiguous()                               # [L, 2, H, T, D]
            return (KvView.from_blob(blob, kind),
                    lambda: [(blob[l, 0].transpose(0, 1), blob[l, 1].transpose(0, 1)) for l in range(L)], np.arange(T))
        return KvView.from_blob(blob, kind), lambda: [(blob[l, 0], blob[l, 1]) for l in range(L)], np.arange(T)
    layout, bs = kind.rsplit("-", 1)
    bs, nb = int(bs), 40
    rows = _randn_rows(L, nb * bs, H, D, dtype, seed)
    caches = [_layout(layout, r, nb, bs, H, D) for r in rows]
    slots = _slots("perm" if bs == 8 else "vllm", T, nb, bs, torch.Generator().manual_seed(seed))

    def get():
        return [tuple(t.view(dtype) for t in _rows(layout, p, nb, bs, H, D)) for p in caches]
    return KvView.from_paged(caches, slots), get, slots.cpu().numpy()


def _check(before, after, slot, tok_begin, seg, shifts, spec, D, dtype):
    """rotated key rows within tolerance of the statement; every other byte as before"""
    seg = np.asarray(seg)
    toks = np.nonzero(seg >= 0)[0]
    rows = slot[tok_begin + toks]
    sh = np.asarray(shifts, dtype=np.int64)[seg[toks]]
    rd, off = spec.rotary_dim, spec.offset
    inv = spec.inv_freq.numpy()
    p = partner(rd, spec.style, off, D)
    exact = total = 0
    for l, ((k0, v0), (k1, v1)) in enumerate(zip(before, after)):
        if v0 is not None:
            assert torch.equal(v0.view(torch.int16), v1.view(torch.int16)), ("V plane written", l)
        changed = torch.zeros(k0.shape, dtype=torch.bool, device=k0.device)
        changed[torch.as_tensor(rows, device=k0.device), :, off:off + rd] = True
        assert torch.equal(k0.view(torch.int16)[~changed], k1.view(torch.int16)[~changed]), ("untouched bytes", l)
        x = k0.double().cpu().numpy()[rows]
        ref = rotate(x, sh, inv, rd, spec.style, off)
        ref_r = torch.from_numpy(ref).to(dtype).double().numpy()
        got = k1.double().cpu().numpy()[rows]
        tol = tolerance(ref_r, got, x, x[..., p], NAMES[dtype])
        err = np.abs(got - ref_r)[..., off:off + rd]
        bad = err > tol[..., off:off + rd]
        assert not bad.any(), (l, int(bad.sum()), float(err.max()))
        exact += int((err == 0).sum())
        total += err.size
    assert exact >= 0.95 * total, (exact, total)      # nearly every element is the correctly rounded rotation


KERNEL_LAYOUTS = ["vllm", "huggingface", "tuple", "flash-16", "strided-16", "split-8", "split-16", "split-32"]
ROT = [(128, 0), (64, 0), (36, 4), (32, 16)]          # (rotary_dim, offset) of D = 128; 36 / 4: the element-wise path


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("style", ["neox", "gptj"])
@pytest.mark.parametrize("kind", KERNEL_LAYOUTS)
def test_kernel_matches_statement(dtype, style, kind):
    from lmcache_b200.rope import RopeSpec
    T, H, D = 96, 4, 128
    for i, (rd, off) in enumerate(ROT):
        spec = RopeSpec.from_base(rd, 10000.0, style, off)
        view, get, slot = _target(kind, dtype, T, H, D, seed=i + 10 * KERNEL_LAYOUTS.index(kind))
        before = [(k.clone(), None if v is None else v.clone()) for k, v in get()]
        _shift(view, 5, _seg_pattern(), SHIFTS, spec)
        _check(before, get(), slot, 5, _seg_pattern(), SHIFTS, spec, D, dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("style", ["neox", "gptj"])
@pytest.mark.parametrize("kind", ["latent", "latent-paged"])
def test_kernel_latent_offset_512(dtype, style, kind):
    """DeepSeek's latent: only the decoupled RoPE channels [512, 576) of the one plane turn"""
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(64, 10000.0, style, 512)
    view, get, slot = _target(kind, dtype, 96, 1, 576, seed=3)
    before = [(k.clone(), None) for k, _ in get()]
    _shift(view, 5, _seg_pattern(), SHIFTS, spec)
    _check(before, get(), slot, 5, _seg_pattern(), SHIFTS, spec, 576, dtype)


def test_kernel_refusals_write_nothing():
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView
    L, T, H, D = 2, 32, 2, 64
    seg = torch.zeros(T, dtype=torch.int32, device="cuda")
    shifts = torch.tensor([4096], dtype=torch.int64, device="cuda")
    inv = torch.ones(D // 2, dtype=torch.float32, device="cuda")
    table = torch.empty(1, D // 2, 2, dtype=torch.float32, device="cuda")
    lib = N.lib()
    N.check(lib.b200kv_rope_table(ctypes.c_void_p(shifts.data_ptr()), 1, ctypes.c_void_p(inv.data_ptr()), D,
                                  ctypes.c_void_p(table.data_ptr()), None))

    def call(blob, rd, off, style=0, tab=table.data_ptr(), sg=seg.data_ptr()):
        view = KvView.from_blob(blob, "vllm")
        return lib.b200kv_rope_shift(ctypes.byref(view.desc), 0, T, ctypes.c_void_p(sg), ctypes.c_void_p(tab), rd, off,
                                     style, None)
    for dt in (torch.uint8, torch.float8_e4m3fn, torch.float8_e5m2):
        blob = torch.full((L, 2, T, H, D), 0x3C, dtype=torch.uint8, device="cuda").view(dt)
        assert call(blob, D, 0) < 0 and "16-bit" in N.last_error()
        torch.cuda.synchronize()
        assert bool((blob.view(torch.uint8) == 0x3C).all())
    blob = torch.full((L, 2, T, H, D), 0x3C3C, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    for rd, off, style, tab, sg, msg in ((63, 0, 0, table.data_ptr(), seg.data_ptr(), "even"),
                                         (0, 0, 0, table.data_ptr(), seg.data_ptr(), "even"),
                                         (32, 33, 0, table.data_ptr(), seg.data_ptr(), "exceeds"),
                                         (64, -2, 0, table.data_ptr(), seg.data_ptr(), "exceeds"),
                                         (64, 0, 2, table.data_ptr(), seg.data_ptr(), "style"),
                                         (64, 0, 0, 0, seg.data_ptr(), "NULL"),
                                         (64, 0, 0, table.data_ptr(), 0, "NULL")):
        assert call(blob, rd, off, style, tab, sg) < 0, (rd, off, style)
        assert msg in N.last_error(), (msg, N.last_error())
    torch.cuda.synchronize()
    assert bool((blob.view(torch.int16) == 0x3C3C).all())
    assert lib.b200kv_rope_table(ctypes.c_void_p(shifts.data_ptr()), 1, ctypes.c_void_p(inv.data_ptr()), 63,
                                 ctypes.c_void_p(table.data_ptr()), None) < 0


def test_table_angles_in_fp64():
    """the table's (cos, sin) are the fp64 values rounded once to fp32, up to a shift of 2^20 at inv_freq 1"""
    from lmcache_b200 import _native as N
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(128, 10000.0)
    shifts = np.array([0, 1, 255, 4096, 65535, 65536, 1 << 20], dtype=np.int64)
    sh = torch.from_numpy(shifts).cuda()
    inv = spec.inv_freq.cuda()
    table = torch.empty(len(shifts), 64, 2, dtype=torch.float32, device="cuda")
    N.check(N.lib().b200kv_rope_table(ctypes.c_void_p(sh.data_ptr()), len(shifts), ctypes.c_void_p(inv.data_ptr()),
                                      128, ctypes.c_void_p(table.data_ptr()), None))
    torch.cuda.synchronize()
    a = shifts[:, None].astype(np.float64) * spec.inv_freq.numpy().astype(np.float64)[None, :]
    got = table.cpu().numpy().astype(np.float64)
    assert np.abs(got[..., 0] - np.cos(a)).max() <= 2.0 ** -24 * 1.01
    assert np.abs(got[..., 1] - np.sin(a)).max() <= 2.0 ** -24 * 1.01


# ---------------------------------------------------------------------------------------------- the engine
CS = 64
RAW_EXACT = ("cpu", "cuda", "host-lossless", "disk-lossless", "lm-lossless", "lm-torch")
# documents: (length, tokens stored); C has only its first two chunks stored
DOCS = {"A": (2 * CS + 10, 2 * CS + 10), "B": (3 * CS, 3 * CS), "C": (3 * CS + 20, 2 * CS)}
SRC_SLOT0 = {"A": 0, "B": 200, "C": 400}


def _request(doc_tokens, gen):
    """[prefix][B][A][gap][C][question]: tokens and the segments (start, end) of B, A and C"""
    parts, segs, pos = [], {}, 0
    for name in ("prefix", "B", "A", "gap", "C", "question"):
        t = doc_tokens[name] if name in DOCS else torch.randint(0, 32000, ({"prefix": 30, "gap": 17,
                                                                             "question": 25}[name],), generator=gen)
        if name in DOCS:
            segs[name] = (pos, pos + len(t))
        parts.append(t)
        pos += len(t)
    return torch.cat(parts), segs


def _doc_setup(eng, tier, ai, kind_tag):
    """store the documents as prompts of their own from a FlashAttention cache; return their tokens and, per document,
    what retrieve_paged of the document alone gives ([n, H, D] K and V rows) and the source rows"""
    gen = torch.Generator().manual_seed(5)
    base = 300000 * TIERS.index(tier) + 50000 * ai + kind_tag
    doc_tokens = {n: torch.randint(0, 32000, (DOCS[n][0],), generator=gen) + base for n in DOCS}
    src = _caches("flash", _randn_rows(L_E, NB * BS, H_E, D_E, torch.bfloat16, seed=21), NB, BS, H_E, D_E)
    ref = {}
    for n, (ln, stored) in DOCS.items():
        slots = torch.arange(SRC_SLOT0[n], SRC_SLOT0[n] + ln, device="cuda")
        eng.store_paged(doc_tokens[n][:stored], src, slots[:stored])
    if hasattr(eng.engine_, "drain"):
        eng.engine_.drain()
    for n, (ln, stored) in DOCS.items():
        slots = torch.arange(ln, device="cuda")
        dst = _caches("flash", _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x3C), NB, BS, H_E, D_E)
        ret = eng.retrieve_paged(doc_tokens[n], dst, slots)
        torch.cuda.synchronize()
        assert int(ret.sum()) == stored, (tier, n)
        got = _cache_rows("flash", dst)
        ref[n] = [(k[:stored], v[:stored]) for k, v in got]
        if tier in RAW_EXACT:
            want = _cache_rows("flash", src)
            for l in range(L_E):
                for i in range(2):
                    assert torch.equal(ref[n][l][i], want[l][i][SRC_SLOT0[n]:SRC_SLOT0[n] + stored]), (tier, n, l, i)
    return doc_tokens, ref


def _check_segments(rows, slot, segs, ref, spec, dtype=torch.bfloat16):
    """every segment's rows: V bit-identical to the document's, K within tolerance of its rotation to the new start"""
    inv = spec.inv_freq.numpy()
    D = rows[0][0].shape[-1]
    p = partner(spec.rotary_dim, spec.style, spec.offset, D)
    for n, (a, b) in segs.items():
        stored = DOCS[n][1]
        r = slot[a:a + stored]
        for l in range(len(rows)):
            kg, vg = rows[l]
            kr, vr = ref[n][l]
            assert torch.equal(vg[r], vr), (n, l, "V")
            x = kr.view(dtype).double().cpu().numpy()
            want = rotate(x, a, inv, spec.rotary_dim, spec.style, spec.offset)
            want_r = torch.from_numpy(want).to(dtype).double().numpy()
            got = kg[r].view(dtype).double().cpu().numpy()
            tol = tolerance(want_r, got, x, x[..., p], NAMES[dtype])
            assert (np.abs(got - want_r) <= tol).all(), (n, l, float(np.abs(got - want_r).max()))


@pytest.mark.parametrize("tier", TIERS)
def test_engine_segments_every_layout(tier, lmserver, tmp_path, autorelease):
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(D_E, 10000.0)
    eng = _engine(autorelease, tier, CS, lmserver, tmp_path, MODEL)
    doc_tokens, ref = _doc_setup(eng, tier, 0, 0)
    tokens, segs = _request(doc_tokens, torch.Generator().manual_seed(6))
    T = len(tokens)
    order = [segs["C"], segs["A"], segs["B"]]            # any order
    want_mask = torch.zeros(T, dtype=torch.bool)
    for n, (a, b) in segs.items():
        want_mask[a:a + DOCS[n][1]] = True
    slots = _slots("vllm", T, NB, BS, torch.Generator().manual_seed(7))
    slot = slots.cpu().numpy()
    flash_rows = None
    for b in LAYOUTS:
        dst = _caches(b, _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x3C), NB, BS, H_E, D_E)
        ret = eng.retrieve_paged_segments(tokens, dst, slots, order, spec)
        torch.cuda.synchronize()
        assert torch.equal(ret, want_mask), (tier, b)
        rows = _cache_rows(b, dst)
        _check_segments(rows, slot, segs, ref, spec)
        hit = torch.zeros(NB * BS, dtype=torch.bool, device="cuda")
        hit[slots[ret.cuda()]] = True
        for l in range(L_E):
            for i in range(2):
                assert bool((rows[l][i][~hit].view(torch.uint8) == 0x3C).all()), (tier, b, l, i)
        if flash_rows is None:
            flash_rows = rows
        else:                                             # every layout gets the same bytes
            for l in range(L_E):
                for i in range(2):
                    assert torch.equal(rows[l][i][slots], flash_rows[l][i][slots]), (tier, b, l, i)
    # the dense form: the same rows at the request's tokens, zero elsewhere
    kv, ret = eng.retrieve_segments(tokens, order, spec)
    assert torch.equal(ret, want_mask)
    for l in range(L_E):
        for i in range(2):
            t = kv[l][i].reshape(T, H_E, D_E).view(torch.int16)
            assert torch.equal(t[ret.cuda()], flash_rows[l][i][slots[ret.cuda()]]), (tier, l, i)
            assert bool((t[~ret.cuda()] == 0).all())


@pytest.mark.parametrize("tier", TIERS)
def test_engine_one_whole_segment_equals_retrieve(tier, lmserver, tmp_path, autorelease):
    """segment (0, T) gives retrieve_paged's ret_mask and bytes, and retrieve's rows, in every layout"""
    from lmcache_b200.rope import RopeSpec
    spec = RopeSpec.from_base(D_E, 10000.0)
    eng = _engine(autorelease, tier, CS, lmserver, tmp_path, MODEL)
    doc_tokens, _ = _doc_setup(eng, tier, 1, 7)
    for n in ("A", "C"):                                  # C: a partial hit
        toks = doc_tokens[n]
        T = len(toks)
        slots = _slots("vllm", T, NB, BS, torch.Generator().manual_seed(8))
        for b in LAYOUTS:
            d1 = _caches(b, _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x3C), NB, BS, H_E, D_E)
            d2 = _caches(b, _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x3C), NB, BS, H_E, D_E)
            r1 = eng.retrieve_paged_segments(toks, d1, slots, [(0, T)], spec)
            r2 = eng.retrieve_paged(toks, d2, slots)
            torch.cuda.synchronize()
            assert torch.equal(r1, r2), (tier, n, b)
            for (k1, v1), (k2, v2) in zip(_cache_rows(b, d1), _cache_rows(b, d2)):
                assert torch.equal(k1, k2) and torch.equal(v1, v2), (tier, n, b)
        kv1, r1 = eng.retrieve_segments(toks, [(0, T)], spec)
        kv2, r2 = eng.retrieve(toks)
        assert torch.equal(r1, r2)
        got = int(r2.sum())
        for l in range(L_E):
            for i in range(2):
                assert torch.equal(kv1[l][i][:got].view(torch.int16), kv2[l][i][:got].view(torch.int16)), (tier, n, l)


@pytest.mark.parametrize("tier", ["cpu", "host-cachegen", "host-lossless"])
def test_mla_engine_turns_only_the_rope_channels(tier, lmserver, tmp_path, autorelease):
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
    doc = torch.randint(0, 32000, (2 * CS + 10,), generator=gen) + 900000 + 1000 * len(tier)
    eng.store_paged(doc, src, torch.arange(len(doc), device="cuda"))
    if hasattr(eng.engine_, "drain"):
        eng.engine_.drain()
    ref = [torch.full((nb, bs, D), 7, dtype=torch.bfloat16, device="cuda") for _ in range(L)]
    eng.retrieve_paged(doc, ref, torch.arange(len(doc), device="cuda"))
    pre = torch.randint(0, 32000, (77,), generator=gen)
    tokens = torch.cat([pre, doc])
    slots = _slots("perm", len(tokens), nb, bs, torch.Generator().manual_seed(11))
    dst = [torch.full((nb, bs, D), 7, dtype=torch.bfloat16, device="cuda") for _ in range(L)]
    ret = eng.retrieve_paged_segments(tokens, dst, slots, [(77, len(tokens))], spec)
    torch.cuda.synchronize()
    assert int(ret.sum()) == len(doc) and bool(ret[77:].all())
    inv = spec.inv_freq.numpy()
    p = partner(64, "gptj", 512, D)
    rows = slots[77:]
    for l in range(L):
        got = dst[l].view(-1, D)[rows]
        want = ref[l].view(-1, D)[:len(doc)]
        assert torch.equal(got[:, :512].view(torch.int16), want[:, :512].view(torch.int16)), l
        x = want.double().cpu().numpy()
        w = torch.from_numpy(rotate(x, 77, inv, 64, "gptj", 512)).to(torch.bfloat16).double().numpy()
        gg = got.double().cpu().numpy()
        assert (np.abs(gg - w) <= tolerance(w, gg, x, x[..., p], "bfloat16")).all(), l
        others = torch.ones(nb * bs, dtype=torch.bool, device="cuda")
        others[rows] = False
        assert bool((dst[l].view(-1, D)[others] == 7).all())


def test_refusals_before_anything_is_written(lmserver, tmp_path, autorelease):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineMetadata
    from lmcache_b200.rope import RopeSpec
    from test_gpu_paged_layouts import _tier_config
    spec = RopeSpec.from_base(D_E, 10000.0)
    eng = _engine(autorelease, "cpu", CS, lmserver, tmp_path, MODEL)
    doc_tokens, _ = _doc_setup(eng, "cpu", 2, 3)
    tokens, segs = _request(doc_tokens, torch.Generator().manual_seed(6))
    slots = _slots("vllm", len(tokens), NB, BS, torch.Generator().manual_seed(7))
    for b in LAYOUTS:
        dst = _caches(b, _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x3C), NB, BS, H_E, D_E)
        bad = [segs["A"], (segs["A"][1] - 1, segs["A"][1] + 5)]
        with pytest.raises(ValueError, match="overlap"):
            eng.retrieve_paged_segments(tokens, dst, slots, [segs["B"]] + bad, spec)
        with pytest.raises(ValueError, match="do not fit"):
            eng.retrieve_paged_segments(tokens, dst, slots, [segs["B"]], RopeSpec.from_base(D_E, 1e4, "neox", 8))
        torch.cuda.synchronize()
        for l in range(L_E):
            for i in range(2):
                assert bool((_cache_rows(b, dst)[l][i].view(torch.uint8) == 0x3C).all()), (b, l, i)
    with pytest.raises(ValueError, match="overlap"):
        eng.retrieve_segments(tokens, [segs["A"], segs["A"]], spec)
    # FP8 caches and FP8 engines
    fp8 = _caches("flash", _all_rows(L_E, NB, BS, H_E, D_E, torch.float8_e4m3fn, seed=0, fill=0x3C), NB, BS, H_E, D_E)
    with pytest.raises(TypeError):
        eng.retrieve_paged_segments(tokens, fp8, slots, [segs["B"]], spec)
    e8 = autorelease(LMCacheEngine(_tier_config("cpu", CS, lmserver, tmp_path),
                                   LMCacheEngineMetadata(MODEL, 1, 0, "vllm", "fp8")))
    with pytest.raises(TypeError):
        e8.retrieve_segments(tokens, [segs["B"]], spec)
    fp8_store = _caches("flash", _all_rows(L_E, NB, BS, H_E, D_E, torch.float8_e4m3fn, seed=4), NB, BS, H_E, D_E)
    e9 = autorelease(LMCacheEngine(_tier_config("cpu", CS, lmserver, tmp_path),
                                   LMCacheEngineMetadata(MODEL + "-e4m3", 1, 0, "vllm", "bfloat16")))
    e9.store_paged(doc_tokens["A"], fp8_store, torch.arange(len(doc_tokens["A"]), device="cuda"))
    with pytest.raises(TypeError):
        e9.retrieve_segments(tokens, [segs["A"]], spec)
