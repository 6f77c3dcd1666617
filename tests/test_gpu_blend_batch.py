"""GPU: a batched blend.  b200kv_blend_select_batch index-exact against tests/blend_ref.py's select applied per segment
(cut anywhere: empty and 1-row segments, ties across boundaries, NaN / inf / +-0, B = 1 to 4096, a 2^20-row segment
among tiny ones, boundaries inside and at the edges of the kernel's per-CTA row ranges); its refusals; BatchBlendPlan
against one BlendPlan per request in every paged layout and for an MLA latent cache; check() with no host sync, one
reduce and the same library calls at every B; and a batched blended prefill of the toy decoder over documents served
by retrieve_paged_segments, against each request's own."""
import ctypes

import numpy as np
import pytest
import torch

import blend_model as M
import blend_ref as R
from test_gpu_blend import _cases, _dev
from test_gpu_host_tier import MODEL
from test_gpu_paged_layouts import _layout, _slots

pytestmark = pytest.mark.gpu


def _select_batch(dev, cand, seg, k):
    from lmcache_b200.blend import select_batch
    dev_t = torch.as_tensor(np.asarray(dev, np.float32)).cuda()
    cand_t = torch.as_tensor(np.asarray(cand, bool).astype(np.uint8)).cuda()
    n_out = sum(int((~np.asarray(cand[a:b], bool)).sum()) + min(kk, int(np.asarray(cand[a:b], bool).sum()))
                for a, b, kk in zip(seg, seg[1:], k))
    rows = select_batch(dev_t, cand_t, torch.tensor(seg, device="cuda"), torch.tensor(k, device="cuda"), n_out,
                        torch.cuda.current_stream())
    return rows.cpu().numpy()


def _want(dev, cand, seg, k):
    dev, cand = np.asarray(dev, np.float32), np.asarray(cand, bool)
    out = [a + R.select(dev[a:b], cand[a:b], kk) for a, b, kk in zip(seg, seg[1:], k)]
    return np.concatenate(out) if out else np.zeros(0, np.int64)


def _check(dev, cand, seg, k, name=""):
    got = _select_batch(dev, cand, seg, k)
    want = _want(dev, cand, seg, k)
    assert np.array_equal(got, want), (name, len(got), len(want), np.nonzero(got[:len(want)] != want[:len(got)])[0][:5])


def _cta_ranges(n):
    """the kernel's row split: CTA c owns [c * per, min(n, (c + 1) * per))"""
    ctas = max(1, min(-(-n // 1024), 1024))
    per = -(-n // ctas)
    return per, ctas


def _cut(n, rng, parts):
    cuts = np.sort(rng.integers(0, n + 1, parts - 1))
    return [0] + cuts.tolist() + [n]


def _ks(dev, cand, seg, rng):
    return [int(rng.integers(0, max(1, int(np.asarray(cand[a:b]).sum()) + 2))) for a, b in zip(seg, seg[1:])]


@pytest.mark.parametrize("name,dev,cand,k", list(_cases()), ids=[c[0] for c in _cases()])
def test_select_batch_single_segment_and_cut(name, dev, cand, k):
    n = len(dev)
    _check(dev, cand, [0, n], [k], name)                                     # B = 1
    rng = np.random.default_rng(n)
    for parts in (2, 7, 64):
        seg = _cut(n, rng, parts)
        _check(dev, cand, seg, _ks(dev, cand, seg, rng), (name, parts))


def test_select_batch_edges():
    rng = np.random.default_rng(1)
    n = 3000
    dev = rng.random(n).astype(np.float32)
    cand = rng.random(n) < 0.7
    # empty segments at the start, in the middle, repeated, and at the end
    seg = [0, 0, 0, 10, 10, 1000, 1000, 1000, 2999, 3000, 3000]
    _check(dev, cand, seg, [3, 1, 5, 0, 200, 9, 4, 1, 1, 2], "empty")
    # 1-row segments, forced and not, with k = 0 and 1
    seg = list(range(0, 41)) + [n]
    k = [i % 2 for i in range(41)]
    _check(dev, cand, seg, k, "1-row")
    # k = 0 and k >= candidates everywhere; all-forced and none-forced segments
    seg = [0, 500, 1500, 2200, n]
    c2 = cand.copy()
    c2[500:1500] = False
    c2[1500:2200] = True
    _check(dev, c2, seg, [0, 10 ** 9, 7, 10 ** 6], "k-edges")
    # NaN, inf and +-0, and tie runs that cross segment boundaries
    d = dev.copy()
    d[rng.random(n) < 0.1] = np.nan
    d[rng.random(n) < 0.1] = np.inf
    d[rng.random(n) < 0.1] = 0.0
    d[rng.random(n) < 0.1] = -0.0
    d[1000:1300] = 0.25
    seg = [0, 400, 1100, 1150, 1200, 2000, n]
    _check(d, cand, seg, [50, 100, 10, 30, 5, 300], "nan-inf-ties")
    _check(np.full(n, 1.0, np.float32), np.ones(n, bool), [0, 700, 701, 1800, n], [300, 1, 2, 600], "all-equal")


def test_select_batch_many_segments():
    rng = np.random.default_rng(2)
    B = 4096                                              # a few rows each, so a CTA crosses hundreds of segments
    lens = rng.integers(0, 8, B)
    seg = np.concatenate([[0], np.cumsum(lens)]).tolist()
    n = seg[-1]
    dev = rng.integers(0, 5, n).astype(np.float32)        # quantised: ties everywhere
    cand = rng.random(n) < 0.75
    _check(dev, cand, seg, rng.integers(0, 6, B).tolist(), "B=4096")


def test_select_batch_huge_segment_among_tiny():
    rng = np.random.default_rng(3)
    tiny = 300
    lens = [1] * tiny + [1 << 20] + [int(x) for x in rng.integers(0, 3, tiny)]
    seg = np.concatenate([[0], np.cumsum(lens)]).tolist()
    n = seg[-1]
    dev = rng.random(n).astype(np.float32)
    dev[rng.random(n) < 0.01] = np.nan
    cand = rng.random(n) < 0.85
    k = [int(x) for x in rng.integers(0, 2, len(lens))]
    k[tiny] = 150000
    _check(dev, cand, seg, k, "2^20 among tiny")


def test_select_batch_cta_boundaries():
    """segment boundaries inside a CTA's row range, at its first row and at its last row (per = 1024 here: 8 CTAs)"""
    rng = np.random.default_rng(4)
    n = 8192
    per, ctas = _cta_ranges(n)
    assert (per, ctas) == (1024, 8)
    inside = [per + 300, 3 * per + 1]                    # inside CTA 1 and CTA 3
    at_start = [2 * per, 5 * per]                         # the first rows of CTAs 2 and 5
    at_end = [4 * per - 1, 6 * per - 1, 7 * per - 1]      # the last rows of CTAs 3, 5 and 6
    seg = sorted({0, n, *inside, *at_start, *at_end})
    dev = rng.integers(0, 50, n).astype(np.float32)
    cand = rng.random(n) < 0.8
    for trial in range(3):
        _check(dev, cand, seg, _ks(dev, cand, seg, rng), ("cta", trial))
    # a segment that starts at a CTA's first row and ends at the next CTA's last row, and one of one CTA exactly
    _check(dev, cand, [0, per, 3 * per, 4 * per, n], [100, 1500, 500, 2000], "whole-ctas")
    # a tile boundary (256 rows) of the compaction inside a CTA
    _check(dev, cand, [0, 256, 511, 512, 513, n], [100, 200, 1, 0, 3000], "tiles")


def test_select_batch_refusals_enqueue_nothing():
    from lmcache_b200 import _native as N
    lib = N.lib()
    T, B = 64, 4
    dev = torch.ones(T, device="cuda")
    cand = torch.ones(T, dtype=torch.uint8, device="cuda")
    seg = torch.tensor([0, 10, 20, 30, T], device="cuda")
    k = torch.ones(B, dtype=torch.int64, device="cuda")
    rows = torch.full((T,), -5, dtype=torch.int64, device="cuda")
    need = lib.b200kv_blend_select_batch_workspace_bytes(T, B)
    assert need == 4176 * B + 16 and lib.b200kv_blend_select_batch_workspace_bytes(T, 0) < 0
    assert lib.b200kv_blend_select_batch_workspace_bytes(-1, 1) < 0
    ws = torch.zeros(need + 8, dtype=torch.uint8, device="cuda")
    p = lambda t: t.data_ptr()                                                          # noqa: E731
    for n, b, dp, sp, kp, wp, wsb, msg in (
            (-1, B, p(dev), p(seg), p(k), p(ws), need, "n"), (1 << 31, B, p(dev), p(seg), p(k), p(ws), need, "n"),
            (T, 0, p(dev), p(seg), p(k), p(ws), need, "B"), (T, B, 0, p(seg), p(k), p(ws), need, "NULL"),
            (T, B, p(dev), 0, p(k), p(ws), need, "NULL"), (T, B, p(dev), p(seg), 0, p(ws), need, "NULL"),
            (T, B, p(dev), p(seg), p(k), 0, need, "NULL"), (T, B, p(dev), p(seg), p(k), p(ws), need - 4, "workspace"),
            (T, B, p(dev), p(seg), p(k), p(ws) + 2, need, "aligned")):
        rc = lib.b200kv_blend_select_batch(ctypes.c_void_p(dp), ctypes.c_void_p(cand.data_ptr()), n, b,
                                           ctypes.c_void_p(sp), ctypes.c_void_p(kp), ctypes.c_void_p(rows.data_ptr()),
                                           ctypes.c_void_p(wp), wsb, None)
        assert rc < 0 and msg in N.last_error(), (msg, N.last_error())
    torch.cuda.synchronize()
    assert bool((rows == -5).all()) and bool((ws == 0).all())


# ---------------------------------------------------------------------------------------------- plans
LENS_RET = [(110, (20, 90)), (1, None), (60, None), (200, (0, 150)), (45, (5, 45))]   # (tokens, retrieved range)


def _masks(lens_ret=LENS_RET):
    out = []
    for n, r in lens_ret:
        m = torch.zeros(n, dtype=torch.bool)
        if r is not None:
            m[r[0]:r[1]] = True
        out.append(m)
    return out


def _paged(kind, L, H, D, nb, bs, seed):
    from lmcache_b200.codec import KvView  # noqa: F401
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "latent":
        return [torch.randn(nb, bs, D, generator=g, device="cuda").to(torch.bfloat16) for _ in range(L)]
    return [_layout(kind, [torch.randn(nb * bs, H, D, generator=g, device="cuda").to(torch.bfloat16)
                           for _ in range(2)], nb, bs, H, D) for _ in range(L)]


def _compare_plans(caches, slots, masks, spec, H, D, seed, engine=None):
    """the batch plan against one BlendPlan per request, each fed its own rows of the batch's fresh keys"""
    from lmcache_b200.blend import BatchBlendPlan, BlendPlan
    from lmcache_b200.codec import KvView
    starts = np.cumsum([0] + [m.numel() for m in masks]).tolist()
    if engine is not None:
        batch = engine.blend_paged_batch(caches, slots, masks, spec)
    else:
        batch = BatchBlendPlan(KvView.from_paged(caches, slots), masks, spec, slots)
    singles = [BlendPlan(KvView.from_paged(caches, slots[a:b]), m, spec, slots[a:b])
               for a, b, m in zip(starts, starts[1:], masks)]
    g = torch.Generator(device="cuda").manual_seed(seed)
    for layer in spec.check_layers:
        rows = batch.rows_at(layer)
        # fresh keys near the cached rows of every batch token, then taken at the plan's rows
        allk = torch.randn(starts[-1], H * D, generator=g, device="cuda").to(torch.bfloat16)
        step = batch.check(layer, allk[rows])
        want_rows, want_tok, want_slots, lens = [], [], [], []
        seg0 = 0
        for r, (p, a) in enumerate(zip(singles, starts)):
            pr = p.rows_at(layer)
            s = p.check(layer, allk[a + pr])
            want_rows.append(s.rows + seg0)
            want_tok.append(s.tokens + a)
            want_slots.append(s.slots)
            lens.append(s.tokens.numel())
            seg0 += pr.numel()
        assert torch.equal(step.rows, torch.cat(want_rows)), layer
        assert torch.equal(step.tokens, torch.cat(want_tok)), layer
        assert torch.equal(step.slots, torch.cat(want_slots)) and torch.equal(step.slots, slots[step.tokens])
        cu = torch.tensor(np.cumsum([0] + lens), dtype=torch.int32)
        assert torch.equal(step.cu_rows.cpu(), cu) and step.cu_rows.dtype == torch.int32
        nxt = layer + 1                                   # the spec leaves a layer after its last check
        assert batch.lens_at(nxt) == lens and torch.equal(batch.cu_rows_at(nxt).cpu(), cu)
        assert torch.equal(batch.rows_at(nxt), step.tokens) and torch.equal(batch.slots_at(nxt), step.slots)
    return batch


@pytest.mark.parametrize("kind", ["flash", "strided", "split"])
def test_batch_plan_matches_per_request_plans(kind):
    from lmcache_b200.blend import BlendSpec
    L, H, D, nb, bs = 4, 2, 64, 40, 16
    caches = _paged(kind, L, H, D, nb, bs, seed=1)
    masks = _masks()
    slots = _slots("perm", sum(m.numel() for m in masks), nb, bs, torch.Generator().manual_seed(2))
    _compare_plans(caches, slots, masks, BlendSpec([1, 2], [0.4, 0.1]), H, D, seed=3)


def test_batch_plan_mla_engine(autorelease):
    from lmcache_b200.blend import BlendSpec
    from test_gpu_mla_engine import _engine as mla_engine
    Lm, Dm, nb, bs = 4, 576, 30, 16
    eng = mla_engine(autorelease, "cuda", Lm)
    caches = _paged("latent", Lm, 1, Dm, nb, bs, seed=4)
    masks = _masks(LENS_RET[:4])
    slots = _slots("perm", sum(m.numel() for m in masks), nb, bs, torch.Generator().manual_seed(5))
    _compare_plans(caches, slots, masks, BlendSpec([1, 2], [0.3, 0.05]), 1, Dm, seed=6, engine=eng)


def test_engine_batch_refusals(autorelease):
    from lmcache_b200.blend import BlendSpec
    from test_gpu_paged_layouts import _engine
    eng = _engine(autorelease, "cuda", 16, None, None, MODEL)
    cache = M.PagedKV("flash")
    slots = torch.arange(40, device="cuda")
    m = [torch.zeros(15, dtype=torch.bool), torch.ones(25, dtype=torch.bool)]
    for spec, masks in ((BlendSpec([M.L], [0.1]), m), ("x", m), (BlendSpec([1], [0.1]), m[:1]),
                        (BlendSpec([1], [0.1]), []), (BlendSpec([1], [0.1]), [m[0], m[1].cuda()])):
        with pytest.raises(ValueError):
            eng.blend_paged_batch(cache.caches, slots, masks, spec)
    fp8 = [tuple(t.view(torch.uint8)[..., :M.D].view(torch.float8_e4m3fn) for t in p) for p in cache.caches]
    with pytest.raises(TypeError):
        eng.blend_paged_batch(fp8, slots, m, BlendSpec([1], [0.1]))


def _counting(monkeypatch):
    from lmcache_b200 import _native as N
    real, calls = N.lib(), []

    class Lib:
        def __getattr__(self, name):
            calls.append(name)
            return getattr(real, name)
    monkeypatch.setattr(N, "lib", lambda: Lib())
    return calls


@pytest.mark.parametrize("B", [2, 64])
def test_check_no_sync_one_reduce_constant_calls(B, monkeypatch):
    from lmcache_b200.blend import BatchBlendPlan, BlendSpec
    from lmcache_b200.codec import KvView
    L, H, D, nb, bs = 3, 2, 64, 200, 16
    rng = np.random.default_rng(B)
    masks = [torch.from_numpy(rng.random(int(rng.integers(1, 40))) < 0.7) for _ in range(B)]
    n = sum(m.numel() for m in masks)
    caches = _paged("flash", L, H, D, nb, bs, seed=7)
    slots = _slots("perm", n, nb, bs, torch.Generator().manual_seed(8))
    spec = BlendSpec([1, 2], [0.5, 0.2])
    plan = BatchBlendPlan(KvView.from_paged(caches, slots), masks, spec, slots)
    g = torch.Generator(device="cuda").manual_seed(9)
    fresh1 = torch.randn(n, H, D, generator=g, device="cuda").to(torch.bfloat16)
    n2 = plan.checks[0].out[-1]                           # the rows computed at layer 2, known before check 1
    fresh2 = torch.randn(n2, H * D, generator=g, device="cuda").to(torch.bfloat16)
    seen = []

    def reduce(d):                                        # rewrites dev: the select must follow the reduced values
        seen.append(d.numel())
        d.neg_()
    calls = _counting(monkeypatch)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        s1 = plan.check(1, fresh1, reduce=reduce)
        s2 = plan.check(2, fresh2, reduce=reduce)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    monkeypatch.undo()
    assert seen == [n, n2]
    per_check = ["b200kv_blend_deviation", "b200kv_blend_select_batch_workspace_bytes", "b200kv_blend_select_batch"]
    assert calls == per_check * 2, calls
    flat = torch.cat(masks).numpy()
    c0 = plan.checks[0]
    dev1 = -_dev(plan.view, 1, torch.arange(n, device="cuda"), fresh1.view(n, -1)).cpu().numpy()
    assert np.array_equal(s1.rows.cpu().numpy(), _want(dev1, flat, c0.seg, c0.k))
    toks1 = s1.tokens.cpu().numpy()
    c1 = plan.checks[1]
    dev2 = -_dev(plan.view, 2, s1.tokens, fresh2).cpu().numpy()
    assert np.array_equal(s2.rows.cpu().numpy(), _want(dev2, flat[toks1], c1.seg, c1.k))
    assert np.array_equal(s2.tokens.cpu().numpy(), toks1[s2.rows.cpu().numpy()])


# ---------------------------------------------------------------------------------------------- end to end
SYS, QN, DOC_A, DOC_B = 12, 10, 48, 40


def _batched_prefill(model, tokens, pos, cache, slots, plan, starts):
    """the toy decoder's blended prefill over a flattened batch: every request's rows in one qkv, one plan.check per
    check layer with the fresh keys in the plan's row order, attention per request over its own keys; (the last
    layer's output of the rows computed to the end, those batch tokens, the steps, the fresh keys of each check)"""
    n = tokens.numel()
    x = model.emb[tokens]
    toks = torch.arange(n, device="cuda")
    perm = toks
    steps, fresh = [], {}
    for l in range(M.L):
        q, k, v = model.qkv(l, x, pos[toks])
        step = None
        if l in plan.spec.check_layers:
            fresh[l] = k[perm].to(torch.bfloat16)
            step = plan.check(l, fresh[l])
            steps.append(step)
        cache.write(l, slots[toks], k, v)
        outs = []
        for a, b in zip(starts, starts[1:]):
            sel = torch.nonzero((toks >= a) & (toks < b)).flatten()
            K, V = cache.read(l, slots[a:b])
            outs.append(model.finish(l, x[sel], q[sel], pos[toks[sel]], K, V))
        x = torch.cat(outs)
        if step is not None:
            order = torch.argsort(step.tokens)
            x = x[perm][step.rows][order]
            toks = step.tokens[order]
            perm = torch.argsort(order)
    return x, toks, steps, fresh


class _Fed:
    """a BlendPlan whose checks take the batch's fresh keys of this request instead of the model's own"""

    def __init__(self, plan, keys):
        self.plan, self.keys, self.spec = plan, keys, plan.spec

    def check(self, layer, fresh_k):
        return self.plan.check(layer, self.keys[layer])


def test_batched_blended_prefill_toy_model(autorelease):
    from lmcache_b200.blend import BlendSpec
    from lmcache_b200.rope import RopeSpec
    from test_gpu_paged_layouts import _engine
    model = M.ToyDecoder(seed=0)
    g = torch.Generator().manual_seed(1)
    eng = _engine(autorelease, "cuda", 16, None, None, MODEL)
    docs = [torch.randint(0, M.VOCAB, (n,), generator=g) for n in (DOC_A, DOC_B, DOC_A)]
    for doc in docs:                                      # each document prefilled and stored as its own prompt
        c = M.PagedKV("flash")
        s = torch.arange(len(doc), device="cuda")
        model.prefill(doc.cuda(), c, s)
        eng.store_paged(doc, c.caches, s)
    rope = RopeSpec(M.D, model.inv_freq, "neox")
    sysp, q1, q2 = (torch.randint(0, M.VOCAB, (n,), generator=g) for n in (SYS, QN, QN))
    unseen = torch.randint(0, M.VOCAB, (DOC_B,), generator=g)
    reqs = [(torch.cat([sysp, docs[0], docs[1], q1]), [(SYS, SYS + DOC_A), (SYS + DOC_A, SYS + DOC_A + DOC_B)]),
            (torch.randint(0, M.VOCAB, (1,), generator=g), None),                       # a decode row
            (torch.cat([sysp, unseen, q2]), [(SYS, SYS + DOC_B)]),                       # its document missed
            (torch.cat([sysp, docs[2], q2]), [(SYS, SYS + DOC_A)])]
    lens = [len(t) for t, _ in reqs]
    starts = np.cumsum([0] + lens).tolist()
    nb = 32
    slots = _slots("vllm", starts[-1], nb, 16, torch.Generator().manual_seed(2))
    cache = M.PagedKV("flash", nb=nb)
    masks, alone = [], []
    for (t, segs), a, b in zip(reqs, starts, starts[1:]):
        c1 = M.PagedKV("flash", nb=nb)
        if segs is None:
            m = torch.zeros(len(t), dtype=torch.bool)
        else:
            m = eng.retrieve_paged_segments(t, cache.caches, slots[a:b], segs, rope)
            assert torch.equal(eng.retrieve_paged_segments(t, c1.caches, slots[a:b], segs, rope), m)
        masks.append(m)
        alone.append(c1)
    assert int(masks[0].sum()) == DOC_A + DOC_B and not masks[2].any() and int(masks[3].sum()) == DOC_A
    spec = BlendSpec([1, 2], [0.3, 0.15])
    plan = eng.blend_paged_batch(cache.caches, slots, masks, spec)
    tokens = torch.cat([t for t, _ in reqs]).cuda()
    pos = torch.cat([torch.arange(n) for n in lens]).cuda()
    x, toks, steps, fresh = _batched_prefill(model, tokens, pos, cache, slots, plan, starts)
    for r, ((t, _), a, b) in enumerate(zip(reqs, starts, starts[1:])):
        single = eng.blend_paged(alone[r].caches, slots[a:b], masks[r], spec)
        keys = {}
        for l in spec.check_layers:                       # this request's rows of the batch's fresh keys
            cu = plan.cu_rows_at(l).cpu().tolist()
            keys[l] = fresh[l][cu[r]:cu[r + 1]]
        xr, tr, sr = model.blended_prefill(t.cuda(), alone[r], slots[a:b], _Fed(single, keys))
        for j in range(len(spec.check_layers)):
            cu = steps[j].cu_rows.cpu().tolist()
            assert torch.equal(steps[j].tokens[cu[r]:cu[r + 1]] - a, sr[j].tokens), (r, j)
        sel = (toks >= a) & (toks < b)
        assert torch.equal(toks[sel] - a, tr), r
        assert M.rel_err(x[sel], xr) < 1e-4, (r, M.rel_err(x[sel], xr))
