"""GPU: CacheBlend's selective recomputation.  b200kv_blend_deviation against the float64 statement of tests/blend_ref.py
in every layout a kv_desc carries, bit-identical across layouts and n; b200kv_blend_select index-exact against the
statement; the refusals; BlendPlan.check with no host sync; and a blended prefill of a toy decoder (tests/blend_model.py)
over documents served by retrieve_paged_segments, against its full prefill."""
import ctypes

import numpy as np
import pytest
import torch

import blend_model as M
import blend_ref as R
from test_gpu_host_tier import MODEL
from test_gpu_paged_layouts import _layout, _slots
from test_gpu_segments import KERNEL_LAYOUTS, _target

pytestmark = pytest.mark.gpu


def _dev(view, layer, tok, fresh, stride=None):
    from lmcache_b200 import _native as N
    n = tok.numel()
    out = torch.full((max(n, 1),), -1.0, dtype=torch.float32, device="cuda")
    stride = fresh.stride(0) if stride is None else stride
    N.check(N.lib().b200kv_blend_deviation(ctypes.byref(view.desc), layer, n, ctypes.c_void_p(tok.data_ptr()),
                                           ctypes.c_void_p(fresh.data_ptr()), stride, ctypes.c_void_p(out.data_ptr()),
                                           torch.cuda.current_stream().cuda_stream), "blend_deviation")
    torch.cuda.synchronize()
    return out[:n]


def _fresh(cached, dtype, pad, misalign, seed):
    """[n, C] fresh rows near the cached ones, in a buffer of row stride C + pad, starting `misalign` elements in"""
    n, C = cached.shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.zeros(n * (C + pad) + misalign, dtype=dtype, device="cuda")
    rows = buf[misalign:].view(n, C + pad)[:, :C]
    rows.copy_((cached.float() + 0.05 * torch.randn(n, C, generator=g, device="cuda")).to(dtype))
    rows[0] = cached[0]                                   # one row of deviation 0
    return rows


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("kind", KERNEL_LAYOUTS + ["latent", "latent-paged"])
def test_deviation_matches_statement(dtype, kind):
    T, H, D = 96, (1 if kind.startswith("latent") else 4), (576 if kind.startswith("latent") else 128)
    view, get, slot = _target(kind, dtype, T, H, D, seed=5)
    rows = get()
    gen = torch.Generator().manual_seed(1)
    tok = torch.randperm(T, generator=gen)[:61].cuda()     # scattered tokens, in any order
    for layer in range(view.L):
        cached = rows[layer][0].view(dtype)[torch.as_tensor(slot, device="cuda")[tok]].reshape(61, H * D)
        for pad, mis in ((0, 0), (8, 0), (3, 0), (0, 1)):  # vectors; aligned wider stride; element-wise paths
            fresh = _fresh(cached, dtype, pad, mis, seed=layer * 10 + pad + mis)
            got = _dev(view, layer, tok, fresh).double().cpu().numpy()
            want = R.deviation(fresh.float().cpu().numpy(), cached.float().cpu().numpy())
            assert got[0] == 0.0
            assert np.allclose(got, want, rtol=1e-5, atol=1e-30), (kind, layer, pad, mis, np.abs(got - want).max())


def test_deviation_bit_identical_across_layouts_and_n():
    """the same rows give the same bits in every layout, at every n and row index, on the vector and element paths"""
    from lmcache_b200.codec import KvView
    L, H, D, nb, bs, T = 2, 8, 128, 40, 16, 300
    g = torch.Generator(device="cuda").manual_seed(3)
    K = [torch.randn(T, H, D, generator=g, device="cuda").mul(3).to(torch.bfloat16) for _ in range(L)]
    V = [torch.randn(T, H, D, generator=g, device="cuda").to(torch.bfloat16) for _ in range(L)]
    slots = _slots("perm", T, nb, bs, torch.Generator().manual_seed(4))
    views = {}
    blob = torch.stack([torch.stack((K[l], V[l])) for l in range(L)])            # [L, 2, T, H, D]
    views["vllm"] = KvView.from_blob(blob, "vllm")
    hf = blob.transpose(2, 3).contiguous()
    views["huggingface"] = KvView.from_blob(hf, "huggingface")
    views["tuple"] = KvView.from_tuple([(K[l].clone(), V[l].clone()) for l in range(L)], "vllm")
    for kind in ("flash", "strided", "split"):
        caches = []
        for l in range(L):
            rows = [torch.zeros(nb * bs, H, D, dtype=torch.bfloat16, device="cuda") for _ in range(2)]
            rows[0][slots], rows[1][slots] = K[l], V[l]
            caches.append(_layout(kind, rows, nb, bs, H, D))
        views[kind] = KvView.from_paged(caches, slots)
    fresh = (K[1].float() + torch.randn(T, H, D, generator=g, device="cuda")).to(torch.bfloat16).view(T, H * D)
    tok = torch.arange(T, device="cuda")
    ref = _dev(views["vllm"], 1, tok, fresh)
    wide = torch.zeros(T, H * D + 3, dtype=torch.bfloat16, device="cuda")
    wide[:, :H * D] = fresh
    for name, view in views.items():
        assert torch.equal(_dev(view, 1, tok, fresh), ref), name
        assert torch.equal(_dev(view, 1, tok, wide[:, :H * D]), ref), (name, "element path")
    perm = torch.randperm(T, generator=torch.Generator().manual_seed(9)).cuda()
    for n in (1, 7, 33, 200):
        sub = perm[:n]
        for name in ("vllm", "split"):
            assert torch.equal(_dev(views[name], 1, sub, fresh[sub].contiguous()), ref[sub]), (name, n)
    for _ in range(2):                                    # and on every call
        assert torch.equal(_dev(views["strided"], 1, tok, fresh), ref)


def test_deviation_refusals_enqueue_nothing():
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView
    L, T, H, D = 2, 16, 2, 64
    lib = N.lib()
    tok = torch.arange(T, device="cuda")
    out = torch.full((T,), 7.0, device="cuda")
    for dt in (torch.uint8, torch.float8_e4m3fn):
        blob = torch.zeros(L, 2, T, H, D, dtype=torch.uint8, device="cuda").view(dt)
        fresh = torch.zeros(T, H * D, dtype=torch.uint8, device="cuda").view(dt)
        rc = lib.b200kv_blend_deviation(ctypes.byref(KvView.from_blob(blob, "vllm").desc), 0, T,
                                        ctypes.c_void_p(tok.data_ptr()), ctypes.c_void_p(fresh.data_ptr()), H * D,
                                        ctypes.c_void_p(out.data_ptr()), None)
        assert rc < 0 and "16-bit" in N.last_error()
    blob = torch.zeros(L, 2, T, H, D, dtype=torch.bfloat16, device="cuda")
    view = KvView.from_blob(blob, "vllm")
    fresh = torch.ones(T, H * D, dtype=torch.bfloat16, device="cuda")
    for layer, tp, fp, stride, op, msg in ((L, tok.data_ptr(), fresh.data_ptr(), H * D, out.data_ptr(), "layer"),
                                           (-1, tok.data_ptr(), fresh.data_ptr(), H * D, out.data_ptr(), "layer"),
                                           (0, 0, fresh.data_ptr(), H * D, out.data_ptr(), "NULL"),
                                           (0, tok.data_ptr(), 0, H * D, out.data_ptr(), "NULL"),
                                           (0, tok.data_ptr(), fresh.data_ptr(), H * D, 0, "NULL"),
                                           (0, tok.data_ptr(), fresh.data_ptr(), H * D - 1, out.data_ptr(), "stride")):
        rc = lib.b200kv_blend_deviation(ctypes.byref(view.desc), layer, T, ctypes.c_void_p(tp), ctypes.c_void_p(fp),
                                        stride, ctypes.c_void_p(op), None)
        assert rc < 0 and msg in N.last_error(), (msg, N.last_error())
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())
    # select: negative n or k, NULL pointers, a small workspace
    dev = torch.ones(T, device="cuda")
    cand = torch.ones(T, dtype=torch.uint8, device="cuda")
    rows = torch.full((T,), -5, dtype=torch.int64, device="cuda")
    ws = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    need = lib.b200kv_blend_select_workspace_bytes(T)
    for n, k, dp, wsb, msg in ((-1, 1, dev.data_ptr(), need, "n"), (T, -1, dev.data_ptr(), need, "k"),
                               (T, 1, 0, need, "NULL"), (T, 1, dev.data_ptr(), need - 4, "workspace")):
        rc = lib.b200kv_blend_select(ctypes.c_void_p(dp), ctypes.c_void_p(cand.data_ptr()), n, k,
                                     ctypes.c_void_p(rows.data_ptr()), ctypes.c_void_p(ws.data_ptr()), wsb, None)
        assert rc < 0 and msg in N.last_error(), (msg, N.last_error())
    torch.cuda.synchronize()
    assert bool((rows == -5).all()) and bool((ws == 0).all())


def _select(dev, cand, k):
    from lmcache_b200.blend import select
    dev = torch.as_tensor(dev, dtype=torch.float32).cuda()
    cand = torch.as_tensor(cand, dtype=torch.uint8).cuda()
    n_out = int((cand == 0).sum()) + min(k, int((cand != 0).sum()))
    rows = select(dev, cand, k, n_out, torch.cuda.current_stream())
    return rows.cpu().numpy()


def _cases():
    rng = np.random.default_rng(0)
    yield "random", rng.random(5000).astype(np.float32), rng.random(5000) < 0.8, 700
    yield "all-equal", np.full(3000, 2.5, np.float32), np.ones(3000, bool), 1234
    yield "quantised", rng.integers(0, 4, 4000).astype(np.float32), rng.random(4000) < 0.9, 1500
    d = rng.random(2000).astype(np.float32)
    d[rng.random(2000) < 0.05] = np.nan
    d[rng.random(2000) < 0.05] = np.inf
    d[rng.random(2000) < 0.05] = 0.0
    d[rng.random(2000) < 0.05] = -0.0
    yield "nan-inf", d, rng.random(2000) < 0.7, 300
    yield "k=0", rng.random(1000).astype(np.float32), rng.random(1000) < 0.5, 0
    yield "k>=cand", rng.random(1000).astype(np.float32), rng.random(1000) < 0.5, 10 ** 6
    yield "k=cand", rng.random(1000).astype(np.float32), np.arange(1000) % 3 == 0, 334
    yield "all-forced", rng.random(1000).astype(np.float32), np.zeros(1000, bool), 5
    yield "none-forced", rng.random(1000).astype(np.float32), np.ones(1000, bool), 5
    yield "n=1", np.array([0.5], np.float32), np.array([True]), 1
    yield "n=1-forced", np.array([0.5], np.float32), np.array([False]), 1
    yield "n=1-k0", np.array([0.5], np.float32), np.array([True]), 0
    yield "tiny-values", (rng.random(3000) * 1e-38).astype(np.float32), np.ones(3000, bool), 100
    yield "n=2^20", rng.random(1 << 20).astype(np.float32), rng.random(1 << 20) < 0.85, 150000
    q = rng.integers(0, 3, 1 << 20).astype(np.float32)
    yield "n=2^20-ties", q, rng.random(1 << 20) < 0.85, 400000


@pytest.mark.parametrize("name,dev,cand,k", list(_cases()), ids=[c[0] for c in _cases()])
def test_select_index_exact(name, dev, cand, k):
    got = _select(dev, cand, k)
    want = R.select(dev, cand, k)
    assert np.array_equal(got, want), (name, len(got), len(want))


def _plan(kind="flash", T=80, n_ret=60, spec=None):
    from lmcache_b200.blend import BlendPlan, BlendSpec
    from lmcache_b200.codec import KvView
    cache = M.PagedKV(kind)
    g = torch.Generator(device="cuda").manual_seed(2)
    slots = _slots("perm", T, cache.nb, cache.bs, torch.Generator().manual_seed(3))
    for l in range(M.L):
        cache.write(l, slots, torch.randn(T, M.HKV, M.D, generator=g, device="cuda"),
                    torch.randn(T, M.HKV, M.D, generator=g, device="cuda"))
    mask = torch.zeros(T, dtype=torch.bool)
    mask[10:10 + n_ret] = True
    spec = spec or BlendSpec([1, 2], [0.5, 0.2])
    return BlendPlan(KvView.from_paged(cache.caches, slots), mask, spec, slots), cache, slots, mask


def test_check_no_host_sync_and_reduce_once():
    plan, cache, slots, mask = _plan()
    T = mask.numel()
    g = torch.Generator(device="cuda").manual_seed(8)
    fresh1 = torch.randn(T, M.HKV, M.D, generator=g, device="cuda").to(torch.bfloat16)
    seen = []
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        s1 = plan.check(1, fresh1, reduce=lambda d: seen.append(d))
        n2 = s1.tokens.numel()
        fresh2 = torch.randn(n2, M.HKV * M.D, generator=g, device="cuda").to(torch.bfloat16)
        s2 = plan.check(2, fresh2)
        rows3 = plan.rows_at(3)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(seen) == 1 and seen[0].dtype == torch.float32 and seen[0].numel() == T
    # the choice against the statement
    K1, _ = cache.read(1, slots)
    dev1 = _dev(plan.view, 1, torch.arange(T, device="cuda"), fresh1.view(T, -1)).cpu().numpy()
    want1 = R.deviation(fresh1.float().view(T, -1).cpu().numpy(), K1.view(T, -1).cpu().numpy())
    assert np.allclose(dev1, want1, rtol=1e-5)
    sel1 = R.select(dev1, mask.numpy(), 30)
    assert np.array_equal(s1.rows.cpu().numpy(), sel1)
    assert np.array_equal(s1.tokens.cpu().numpy(), sel1)
    assert torch.equal(s1.slots, slots[s1.tokens])
    toks1 = s1.tokens.cpu().numpy()
    dev2 = _dev(plan.view, 2, s1.tokens, fresh2).cpu().numpy()
    sel2 = R.select(dev2, mask.numpy()[toks1], 12)
    assert np.array_equal(s2.rows.cpu().numpy(), sel2)
    assert np.array_equal(s2.tokens.cpu().numpy(), toks1[sel2])
    assert torch.equal(rows3, s2.tokens) and torch.equal(plan.slots_at(3), slots[s2.tokens])
    assert torch.equal(plan.rows_at(1).cpu(), torch.arange(T)) and torch.equal(plan.rows_at(2), s1.tokens)


def test_check_refusals():
    from lmcache_b200.blend import BlendSpec
    plan, cache, slots, mask = _plan(spec=BlendSpec([1, 3], [0.5, 0.2]))
    T = mask.numel()
    ok = torch.zeros(T, M.HKV, M.D, dtype=torch.bfloat16, device="cuda")
    for layer, f in ((0, ok), (3, ok), (2, ok), (1, ok[:-1]), (1, ok.half()), (1, ok.cpu()),
                     (1, torch.zeros(T, M.HKV, M.D + 1, dtype=torch.bfloat16, device="cuda")),
                     (1, ok.transpose(1, 2))):
        with pytest.raises(ValueError):
            plan.check(layer, f)
    with pytest.raises(ValueError):
        plan.rows_at(2)                                   # past a check not yet run
    with pytest.raises(ValueError):
        plan.rows_at(M.L)
    plan.check(1, ok)
    with pytest.raises(ValueError):
        plan.check(1, ok)                                 # out of order


def test_engine_refusals(autorelease):
    from lmcache_b200.blend import BlendSpec
    from test_gpu_paged_layouts import _engine
    eng = _engine(autorelease, "cuda", 16, None, None, MODEL)
    cache = M.PagedKV("flash")
    slots = torch.arange(40, device="cuda")
    mask = torch.zeros(40, dtype=torch.bool)
    for spec, m in ((BlendSpec([M.L], [0.1]), mask), ("x", mask), (BlendSpec([1], [0.1]), mask[:39]),
                    (BlendSpec([1], [0.1]), mask.cuda())):
        with pytest.raises(ValueError):
            eng.blend_paged(cache.caches, slots, m, spec)
    fp8 = [tuple(t.view(torch.uint8)[..., :M.D].view(torch.float8_e4m3fn) for t in p) for p in cache.caches]
    with pytest.raises(TypeError):
        eng.blend_paged(fp8, slots, mask, BlendSpec([1], [0.1]))
    with pytest.raises(ValueError):
        eng.blend((), mask, BlendSpec([1], [0.1]))


# ---------------------------------------------------------------------------------------------- end to end
SYS, QN, DOC_A, DOC_B = 12, 10, 48, 40


def _e2e(tier, kind, layerwise, autorelease, ratios=(1.0, 0.0, 0.15)):
    from lmcache_b200.blend import BlendSpec
    from lmcache_b200.rope import RopeSpec
    from test_gpu_paged_layouts import _engine
    model = M.ToyDecoder(seed=0)
    g = torch.Generator().manual_seed(1)
    sysp, A, B, q = (torch.randint(0, M.VOCAB, (n,), generator=g) for n in (SYS, DOC_A, DOC_B, QN))
    eng = _engine(autorelease, tier, 16, None, None, MODEL)
    for doc in (A, B):                                    # each document prefilled and stored as its own prompt
        c = M.PagedKV(kind)
        s = torch.arange(len(doc), device="cuda")
        model.prefill(doc.cuda(), c, s)
        eng.store_paged(doc, c.caches, s)
    if hasattr(eng.engine_, "drain"):
        eng.engine_.drain()
    tokens = torch.cat([sysp, A, B, q])
    T = len(tokens)
    segs = [(SYS, SYS + DOC_A), (SYS + DOC_A, SYS + DOC_A + DOC_B)]
    slots = _slots("vllm", T, 16, 16, torch.Generator().manual_seed(2))
    full = model.prefill(tokens.cuda(), M.PagedKV(kind), slots)[-QN:]
    rope = RopeSpec(M.D, model.inv_freq, "neox")
    errs = {}
    for r in ratios:
        cache = M.PagedKV(kind)
        wait = None
        if layerwise:
            lr = eng.retrieve_paged_segments_layerwise(tokens, cache.caches, slots, segs, rope)
            ret = lr.ret_mask
            wait = lr.wait_layer
        else:
            ret = eng.retrieve_paged_segments(tokens, cache.caches, slots, segs, rope)
        assert int(ret.sum()) == DOC_A + DOC_B and not ret[:SYS].any() and not ret[-QN:].any()
        plan = eng.blend_paged(cache.caches, slots, ret, BlendSpec([1], [r]))
        x, toks, steps = model.blended_prefill(tokens.cuda(), cache, slots, plan, wait=wait)
        forced = np.nonzero(~ret.numpy())[0]
        got = steps[0].tokens.cpu().numpy()
        assert np.array_equal(got[:len(forced)], forced)
        if r == 1.0:
            assert np.array_equal(got, np.concatenate([forced, np.nonzero(ret.numpy())[0]]))     # index-exact
        if r == 0.0:
            assert np.array_equal(got, forced)
        assert len(got) == len(forced) + BlendSpec([1], [r]).budgets(int(ret.sum()))[0]
        assert np.array_equal(toks[-QN:].cpu().numpy(), np.arange(T - QN, T))
        errs[r] = M.rel_err(x[-QN:], full)
    assert errs[1.0] <= 1e-5, errs
    assert errs[0.15] < errs[0.0], errs
    return errs


@pytest.mark.parametrize("tier", ["cuda", "host-cachegen"])
def test_blended_prefill_toy_model(tier, autorelease):
    _e2e(tier, "flash", False, autorelease)


def test_blended_prefill_layerwise(autorelease):
    _e2e("host-cachegen", "flash", True, autorelease)


def test_blended_prefill_split_layout(autorelease):
    _e2e("cuda", "split", False, autorelease)


def test_dense_blend_matches_paged(autorelease):
    """engine.blend over dense per-layer views (retrieve_segments') chooses what blend_paged chooses over the same KV"""
    from lmcache_b200.blend import BlendSpec
    from test_gpu_paged_layouts import _engine
    eng = _engine(autorelease, "cuda", 16, None, None, MODEL)
    plan, cache, slots, mask = _plan(spec=BlendSpec([1], [0.3]))
    T = mask.numel()
    blob = torch.zeros(M.L, 2, T, M.HKV, M.D, dtype=torch.bfloat16, device="cuda")
    for l in range(M.L):
        K, V = cache.read(l, slots)
        blob[l, 0], blob[l, 1] = K.to(torch.bfloat16), V.to(torch.bfloat16)
    kv = tuple((blob[l, 0], blob[l, 1]) for l in range(M.L))
    dense = eng.blend(kv, mask, BlendSpec([1], [0.3]))
    fresh = torch.randn(T, M.HKV, M.D, device="cuda").to(torch.bfloat16)
    a, b = plan.check(1, fresh), dense.check(1, fresh)
    assert torch.equal(a.rows, b.rows) and b.slots is None


def test_mla_engine_blend(autorelease):
    """an MLA engine: the deviation runs over all 576 channels of the one latent plane, paged and dense"""
    from lmcache_b200.blend import BlendSpec
    from test_gpu_mla_engine import _engine as mla_engine
    Lm, Dm, nb, bs, T = 3, 576, 12, 16, 150
    eng = mla_engine(autorelease, "cuda", Lm)
    g = torch.Generator(device="cuda").manual_seed(6)
    caches = [torch.randn(nb, bs, Dm, generator=g, device="cuda").to(torch.bfloat16) for _ in range(Lm)]
    slots = _slots("perm", T, nb, bs, torch.Generator().manual_seed(7))
    mask = torch.zeros(T, dtype=torch.bool)
    mask[20:140] = True
    fresh = (caches[1].view(-1, Dm)[slots].float() + torch.randn(T, Dm, generator=g, device="cuda")).to(torch.bfloat16)
    plan = eng.blend_paged(caches, slots, mask, BlendSpec([1], [0.2]))
    step = plan.check(1, fresh)
    dev = _dev(plan.view, 1, torch.arange(T, device="cuda"), fresh).cpu().numpy()
    want = R.deviation(fresh.float().cpu().numpy(), caches[1].view(-1, Dm)[slots].float().cpu().numpy())
    assert np.allclose(dev, want, rtol=1e-5)
    assert np.array_equal(step.rows.cpu().numpy(), R.select(dev, mask.numpy(), 24))
    assert torch.equal(step.slots, slots[step.tokens])
    dense = tuple(c.view(-1, Dm)[slots].clone() for c in caches)           # retrieve_segments' [T, D] views
    dstep = eng.blend(dense, mask, BlendSpec([1], [0.2])).check(1, fresh)
    assert torch.equal(dstep.rows, step.rows) and dstep.slots is None
