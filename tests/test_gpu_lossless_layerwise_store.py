"""GPU: the layer-wise store on the lossless host and disk tiers, and the encode it rests on
(b200kv_lossless_encode_layers_plan + b200kv_lossless_encode_layers + b200kv_lossless_encode_layers_finish).  Every
container assembled from a fixed image and arena segments is compared byte for byte with b200kv_lossless_encode's for
the same KV, over layer partitions and call orders; what the engine lands is compared with what store() /
store_paged() land, and every retrieve bit for bit with the stored KV."""
import ctypes
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
MODEL = "lmsys/longchat-7b-16k"
PAT = 0x5A                     # what the output buffers hold before a call


def _kv(shape, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, device="cuda", generator=g) * torch.exp(2 * torch.randn(shape[-1], device="cuda", generator=g))
    return x.to(dtype)


def _whole(view, T, cs):
    """b200kv_lossless_encode's containers, written into a buffer that held PAT"""
    from lmcache_b200.codec import LosslessCodec
    codec = LosslessCodec()
    n = -(-T // cs)
    stride = codec.out_stride(view.L, view.H, view.D, cs, view.latent)
    out = torch.full((n * stride + 1024,), PAT, dtype=torch.uint8, device="cuda")
    batch = codec.encode(view, 0, T, cs, out=out)
    buf = out.cpu().numpy()
    return [bytes(buf[j * stride: j * stride + s]) for j, s in enumerate(batch.sizes)]


class _Layerwise:
    """one b200kv_lossless_encode_layers_plan with every output buffer pre-filled with PAT"""

    def __init__(self, view, T, cs, arena_bytes=None, max_layers=None):
        from lmcache_b200 import _native as N
        from lmcache_b200.codec import LosslessCodec, PinnedBuffer
        self.N, self.view, self.cs = N, view, cs
        L, H, D, lat = view.L, view.H, view.D, view.latent
        self.n, self.last, self.P = -(-T // cs), T - (-(-T // cs) - 1) * cs, view.planes
        codec = LosslessCodec()
        self.layouts = [codec.segment_layout(L, H, D, cs if j < self.n - 1 else self.last, lat) for j in range(self.n)]
        self.stride = self.layouts[0].head
        bound = self.n * codec.layerwise_chunk_bound(L, H, D, cs, lat)
        self.arena = torch.full((bound if arena_bytes is None else max(16, arena_bytes),), PAT, dtype=torch.uint8,
                                device="cuda")
        self.arena_bytes = bound if arena_bytes is None else arena_bytes
        self.fixed = torch.full((self.n * self.stride,), PAT, dtype=torch.uint8, device="cuda")
        self.max_layers = max_layers or L
        wsb = N.lib().b200kv_lossless_encode_layers_workspace_bytes(L, H, D, cs, self.n, int(lat), self.max_layers)
        assert wsb > 0
        self.ws = torch.full((wsb,), PAT, dtype=torch.uint8, device="cuda")
        self.seg, self.sizes = PinnedBuffer(24 * self.P * self.n), PinnedBuffer(8 * self.n)
        ctypes.memset(self.seg.host_ptr, PAT, 24 * self.P * self.n)
        self.plan = N.LosslessEncodePlan()
        self.s = torch.cuda.current_stream().cuda_stream

    def plan_rc(self, **over):
        a = dict(kv=ctypes.byref(self.view.desc), tok=0, n=self.n, cs=self.cs, last=self.last,
                 arena=self.arena.data_ptr(), arena_bytes=self.arena_bytes, fixed=self.fixed.data_ptr(),
                 stride=self.stride, seg=self.seg.dev_ptr, sizes=self.sizes.dev_ptr, max_layers=self.max_layers,
                 ws=self.ws.data_ptr(), ws_bytes=self.ws.numel(), plan=ctypes.byref(self.plan), stream=self.s)
        a.update(over)
        return self.N.lib().b200kv_lossless_encode_layers_plan(*a.values())

    def layers(self, a, b, plan=None):
        return self.N.lib().b200kv_lossless_encode_layers(ctypes.byref(plan or self.plan), a, b, self.s)

    def finish(self, plan=None):
        return self.N.lib().b200kv_lossless_encode_layers_finish(ctypes.byref(plan or self.plan), self.s)

    def run(self, ranges):
        self.N.check(self.plan_rc())
        for a, b in ranges:
            self.N.check(self.layers(a, b))
        self.N.check(self.finish())
        torch.cuda.synchronize()

    def outputs(self):
        sizes = list((ctypes.c_uint64 * self.n).from_address(self.sizes.host_ptr))
        rows = np.frombuffer(self.seg.view(), dtype=np.int64, count=self.n * self.P * 3).reshape(self.n, self.P, 3).copy()
        return sizes, rows

    def containers(self):
        """(containers assembled from the fixed images and the arena by segment_copy_ranges, plane offsets) of the
        chunks whose sizes_out is nonzero"""
        from lmcache_b200.pipeline import segment_copy_ranges
        sizes, rows = self.outputs()
        k = next((j for j, s in enumerate(sizes) if s == 0), self.n)
        if k == 0:
            return [], []
        dst, src, lens, planes = segment_copy_ranges(rows[:k], self.layouts[:k])
        fx, ar = self.fixed.cpu().numpy(), self.arena.cpu().numpy()
        out = []
        for j in range(k):
            got = bytearray(int(lens[j].sum()))
            for d, s, m in zip(dst[j], src[j], lens[j]):
                got[d:d + m] = (fx[j * self.stride: j * self.stride + m] if s < 0 else ar[s:s + m]).tobytes()
            assert len(got) == sizes[j]
            out.append(bytes(got))
        return out, planes


def _ranges(L, part, reverse=False):
    b = np.cumsum([0] + part)
    r = [(int(b[i]), int(b[i + 1])) for i in range(len(part))]
    return r[::-1] if reverse else r


def _view(kind, L, T, H, D, dtype, seed):
    """(KvView, keep-alive) of the source KV"""
    from lmcache_b200.codec import KvView
    if kind == "latent":
        blob = _kv((L, T, D), dtype, seed)
        return KvView.from_tuple([blob[l] for l in range(L)], "vllm"), blob
    if kind == "hf":
        blob = _kv((L, 2, H, T, D), dtype, seed)
        return KvView.from_blob(blob, "huggingface"), blob
    blob = _kv((L, 2, T, H, D), dtype, seed)
    if kind == "tuple":
        return KvView.from_tuple([(blob[l, 0], blob[l, 1]) for l in range(L)], "vllm"), blob
    if kind == "paged":
        bs = 16
        nblk = T // bs + 4
        slots = torch.randperm(nblk * bs, device="cuda")[:T]
        caches = [(torch.zeros((nblk, bs, H, D), dtype=dtype, device="cuda"),
                   torch.zeros((nblk, bs, H, D), dtype=dtype, device="cuda")) for _ in range(L)]
        for l in range(L):
            caches[l][0].view(-1, H, D)[slots] = blob[l, 0]
            caches[l][1].view(-1, H, D)[slots] = blob[l, 1]
        return KvView.from_paged(caches, slots), (caches, slots)
    if kind == "flat":                                # a single-symbol plane (every element equal): frequency 4096
        blob[1, 0] = blob[1, 0, 0, 0, 0]
    return KvView.from_blob(blob, "vllm"), blob


CASES = {   # kind, L, T, H, D, dtype, chunk tokens
    "bf16-vllm": ("blob", 6, 700, 2, 64, torch.bfloat16, 256),
    "fp16-hf": ("hf", 6, 700, 2, 64, torch.float16, 256),
    "tuple": ("tuple", 6, 530, 2, 64, torch.bfloat16, 256),
    "paged": ("paged", 6, 700, 2, 64, torch.float16, 256),
    "latent": ("latent", 6, 700, 1, 72, torch.bfloat16, 256),
    "cs1": ("blob", 6, 5, 2, 64, torch.bfloat16, 1),
    "cs4096": ("blob", 6, 4196, 2, 64, torch.bfloat16, 4096),
    "flat": ("flat", 6, 300, 2, 64, torch.bfloat16, 256),
    "gaps": ("blob", 6, 8, 1, 5, torch.bfloat16, 3),      # 2 P C = 120, P t C = 180: both alignment gaps non-empty
}


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("part,reverse", [("ones", False), ("231", False), ("all", False), ("ones", True)])
def test_layer_partitions_equal_the_whole_encode(case, part, reverse):
    from lmcache_b200.codec import lossless_plane_offsets
    kind, L, T, H, D, dtype, cs = CASES[case]
    if part != "ones" and case not in ("bf16-vllm", "gaps", "latent"):
        pytest.skip("every partition on three cases; the others take [1] * L")
    view, keep = _view(kind, L, T, H, D, dtype, seed=T + D)
    want = _whole(view, T, cs)
    lw = _Layerwise(view, T, cs, max_layers={"ones": 1, "231": 3, "all": L}[part])
    lw.run(_ranges(L, {"ones": [1] * L, "231": [2, 3, 1], "all": [L]}[part], reverse))
    got, planes = lw.containers()
    assert len(got) == len(want) == lw.n
    for j, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"chunk {j} differs"
        assert planes[j].tolist() == lossless_plane_offsets(w).tolist()
    if case == "gaps":                                # the gap bytes are zero in both paths, whatever the buffers held
        from lmcache_b200 import _native as N
        for j, w in enumerate(want):
            t = cs if j < lw.n - 1 else lw.last
            lo = N.lossless_layout(L, H, D, t)
            P, C = 2 * L, H * D
            assert lo.off_raw > lo.off_lens + 2 * P * C and lo.off_payload > lo.off_raw + P * t * C
            assert w[lo.off_lens + 2 * P * C:lo.off_raw] == bytes(lo.off_raw - lo.off_lens - 2 * P * C)
            assert w[lo.off_raw + P * t * C:lo.off_payload] == bytes(lo.off_payload - lo.off_raw - P * t * C)
    del keep


def test_arena_overflow_matches_the_host_model():
    from lmcache_b200.pipeline import arena_placement
    L, T, H, D, cs = 4, 2300, 2, 64, 256
    view, keep = _view("blob", L, T, H, D, torch.bfloat16, 7)
    big = _Layerwise(view, T, cs, max_layers=1)
    big.run(_ranges(L, [1] * L))
    _, rows = big.outputs()
    C = H * D
    # segment bytes per (call, chunk): the raw part (16-byte aligned) and the call's streams
    seg = np.zeros((L, big.n), dtype=np.int64)
    for l in range(L):
        for j in range(big.n):
            ps = [l, L + l]
            seg[l, j] = rows[j, ps[1], 1] - rows[j, ps[0], 0] + rows[j, ps[1], 2]
            assert rows[j, ps[1], 0] - rows[j, ps[0], 0] == big.layouts[j].raw_plane
    total = int(((seg + 15) // 16 * 16).sum())
    for budget in (total // 2, total // 5):
        base, fit = arena_placement(seg, budget)
        assert 0 < fit < big.n
        lw = _Layerwise(view, T, cs, arena_bytes=budget, max_layers=1)
        lw.run(_ranges(L, [1] * L))
        sizes, r = lw.outputs()
        assert all(s > 0 for s in sizes[:fit]) and all(s == 0 for s in sizes[fit:])
        fx = lw.fixed.cpu().numpy()
        for j in range(big.n):
            st = int(np.frombuffer(fx[j * lw.stride + 48: j * lw.stride + 52].tobytes(), dtype=np.uint32)[0])
            assert (st & 16 != 0) == (j >= fit)
        for l in range(L):
            for j in range(fit):
                assert r[j, l, 0] == base[l, j] and r[j, L + l, 0] == base[l, j] + lw.layouts[j].raw_plane
        assert (r[fit:, L - 1, :2] == -1).all() and (r[fit:, 2 * L - 1, :2] == -1).all()   # the last call placed none
        got, _ = lw.containers()
        assert got == _Layerwise.containers(big)[0][:fit]
    del keep


def test_refusals_enqueue_nothing():
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import CacheGenCodec
    L, T, H, D, cs = 4, 600, 2, 64, 256
    view, keep = _view("blob", L, T, H, D, torch.bfloat16, 9)
    lw = _Layerwise(view, T, cs, max_layers=2)

    def snapshot():
        torch.cuda.synchronize()
        return (lw.arena.cpu().clone(), lw.fixed.cpu().clone(), bytes(lw.seg.view()), bytes(lw.sizes.view()))

    def same(a, b):
        return all(torch.equal(x, y) if isinstance(x, torch.Tensor) else x == y for x, y in zip(a, b))

    before = snapshot()
    bad_plans = [dict(arena=lw.arena.data_ptr() + 8), dict(fixed=lw.fixed.data_ptr() + 8), dict(stride=lw.stride - 16),
                 dict(stride=lw.stride + 8), dict(ws_bytes=lw.ws.numel() - 1), dict(cs=4097, last=4097),
                 dict(n=65536), dict(max_layers=0), dict(max_layers=L + 1), dict(last=cs + 1), dict(arena_bytes=-1)]
    for over in bad_plans:
        assert lw.plan_rc(**over) < 0, over
        assert N.last_error()
    desc = N.KvDesc.from_buffer_copy(view.desc)
    desc.L = 129
    assert lw.plan_rc(kv=ctypes.byref(desc)) < 0                       # more than 128 layers
    assert same(before, snapshot())
    assert lw.layers(0, 1) < 0 and lw.finish() < 0                     # a plan that failed is not a plan
    assert lw.layers(0, 1, N.LosslessEncodePlan()) < 0                 # an uninitialised plan
    # a CacheGen plan is of the other family, and the CacheGen calls refuse a lossless plan
    codec = CacheGenCodec(MODEL)
    from lmcache_b200.codec import PinnedBuffer
    cg = N.EncodePlan()
    lo = N.container_layout(L, H, D, cs, N.CODER_RANS_COMPACT)
    fx = torch.empty(3 * ((lo.off_payload + 15) & ~15), dtype=torch.uint8, device="cuda")
    ar = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    wsb = torch.empty(N.lib().b200kv_encode_layers_workspace_bytes(L, H, D, cs, 3, 1), dtype=torch.uint8, device="cuda")
    sg, sz = PinnedBuffer(16 * 2 * L * 3), PinnedBuffer(8 * 3)
    N.check(N.lib().b200kv_encode_layers_plan(ctypes.byref(view.desc), 0, 3, cs, T - 2 * cs, codec._kb, codec._vb,
                                              N.CODER_RANS_COMPACT, ar.data_ptr(), ar.numel(), fx.data_ptr(),
                                              (lo.off_payload + 15) & ~15, sg.dev_ptr, sz.dev_ptr, 1, wsb.data_ptr(),
                                              wsb.numel(), ctypes.byref(cg), lw.s))
    assert N.lib().b200kv_lossless_encode_layers(ctypes.cast(ctypes.byref(cg), ctypes.POINTER(N.LosslessEncodePlan)),
                                                 0, 1, lw.s) < 0
    assert N.lib().b200kv_lossless_encode_layers_finish(
        ctypes.cast(ctypes.byref(cg), ctypes.POINTER(N.LosslessEncodePlan)), lw.s) < 0
    N.check(lw.plan_rc())
    assert N.lib().b200kv_encode_layers(ctypes.cast(ctypes.byref(lw.plan), ctypes.POINTER(N.EncodePlan)), 0, 1,
                                        lw.s) < 0
    N.check(lw.layers(1, 3))
    after_plan = snapshot()
    for a, b in [(-1, 1), (3, 5), (2, 2), (3, 2), (0, 4), (1, 2), (2, 4)]:   # bounds, more than max_layers, encoded before
        assert lw.layers(a, b) < 0, (a, b)
    assert lw.finish() < 0                                              # layers 0 and 3 never encoded
    assert same(after_plan, snapshot())
    N.check(lw.layers(3, 4))
    N.check(lw.layers(0, 1))
    N.check(lw.finish())
    torch.cuda.synchronize()
    assert lw.containers()[0] == _whole(view, T, cs)
    del keep


# ---------------------------------------------------------------------------------------------- engine level
def _engine(local, cs=256, fmt="vllm", dtype="bfloat16", mla=False, **kw):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    cfg = LMCacheEngineConfig(cs, local, None, None, False, False, "lossless", **kw)
    return LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, 1, 0, fmt, dtype, use_mla=mla))


def _local(tier, path):
    return "cpu" if tier == "host" else str(path) + "/"


def _landed(engine):
    """key -> (container bytes, plane offsets) of every chunk the engine's tier holds (disk: by file name)"""
    out = {}
    for k, e in engine.engine_.dict.items():
        e.ready.wait()
        if e.error is not None or e.rec is None:
            continue
        if e.rec.blk is not None:
            data = bytes(e.rec.blk.view())[:e.rec.nbytes]
        else:
            with open(e.path, "rb") as f:
                data = f.read()
        out[os.path.basename(k) if isinstance(k, str) else k] = (data, None if e.rec.planes is None else
                                                                  e.rec.planes.tolist())
    return out


def _bits(x):
    return x.contiguous().view(torch.int16)


def _paged(blob, bs=16):
    L, _, T, H, D = blob.shape
    nblk = T // bs + 4
    slots = torch.randperm(nblk * bs, device="cuda")[:T]
    caches = [(torch.full((nblk, bs, H, D), float("nan"), dtype=blob.dtype, device="cuda"),
               torch.full((nblk, bs, H, D), float("nan"), dtype=blob.dtype, device="cuda")) for _ in range(L)]
    return caches, slots


def _write(caches, slots, blob, l):
    caches[l][0].view(-1, *caches[l][0].shape[2:])[slots] = blob[l, 0]
    caches[l][1].view(-1, *caches[l][1].shape[2:])[slots] = blob[l, 1]


@pytest.mark.parametrize("tier", ["host", "disk"])
@pytest.mark.parametrize("dtype,cs", [(torch.bfloat16, 256), (torch.float16, 1024), (torch.bfloat16, 1024)])
def test_paged_layerwise_lands_store_paged_bytes(tier, dtype, cs, tmp_path):
    L, T, H, D = 4, 2500, 4, 64
    blob = _kv((L, 2, T, H, D), dtype, cs + T)
    toks = torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(cs))
    dn = str(dtype).split(".")[1]
    ref = _engine(_local(tier, tmp_path / "a"), cs, dtype=dn)
    ca, slots = _paged(blob)
    for l in range(L):
        _write(ca, slots, blob, l)
    ref.store_paged(toks, ca, slots)
    eng = _engine(_local(tier, tmp_path / "b"), cs, dtype=dn)
    cb = [(torch.full_like(k, float("nan")), torch.full_like(v, float("nan"))) for k, v in ca]
    h = eng.store_paged_layerwise(toks, cb, slots)
    assert h._enc is not None                        # the layer-wise encode, not the fallback
    for l in reversed(range(L)):
        _write(cb, slots, blob, l)
        h.save_layer(l)
    h.finish()
    for k, v in cb:                                  # the cache is reused right after finish(), in stream order
        k.fill_(-7.0)
        v.fill_(float("nan"))
    a, b = _landed(ref), _landed(eng)
    assert len(a) == -(-T // cs) and a == b and all(p is not None for _, p in b.values())
    out = [(torch.zeros_like(k), torch.zeros_like(v)) for k, v in ca]
    lw = eng.retrieve_paged_layerwise(toks, out, slots)
    assert int(lw.ret_mask.sum()) == T
    for l in range(L):
        lw.wait_layer(l)
        torch.cuda.current_stream().synchronize()
        assert torch.equal(_bits(out[l][0].view(-1, H, D)[slots]), _bits(blob[l, 0]))
        assert torch.equal(_bits(out[l][1].view(-1, H, D)[slots]), _bits(blob[l, 1]))
    kv, mask = eng.retrieve(toks)
    assert int(mask.sum()) == T and torch.equal(_bits(torch.stack([torch.stack(p) for p in kv])), _bits(blob))
    ref.close(), eng.close()


@pytest.mark.parametrize("tier", ["host", "disk"])
@pytest.mark.parametrize("fmt,mla", [("vllm", False), ("huggingface", False), ("vllm", True)])
def test_dense_layerwise_lands_store_bytes(tier, fmt, mla, tmp_path):
    L, T, H, D, cs = 4, 2300, 4, 64, 1024
    dtype = torch.float16 if fmt == "huggingface" else torch.bfloat16
    dn = str(dtype).split(".")[1]
    if mla:
        src = _kv((L, T, 72), dtype, 11)
        kv = tuple(src[l] for l in range(L))
    else:
        src = _kv((L, 2, T, H, D), dtype, 12)
        kv = tuple((src[l, 0], src[l, 1]) if fmt == "vllm" else (src[l, 0].transpose(0, 1).contiguous(),
                                                                  src[l, 1].transpose(0, 1).contiguous())
                   for l in range(L))
    toks = torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(5))
    ref = _engine(_local(tier, tmp_path / "a"), cs, fmt, dn, mla)
    ref.store(toks, kv)
    eng = _engine(_local(tier, tmp_path / "b"), cs, fmt, dn, mla)
    dst = tuple(torch.full_like(x, float("nan")) for x in kv) if mla else \
        tuple((torch.full_like(k, float("nan")), torch.full_like(v, float("nan"))) for k, v in kv)
    h = eng.store_layerwise(toks, dst)
    assert h._enc is not None
    for l in range(L):
        if mla:
            dst[l].copy_(kv[l])
        else:
            dst[l][0].copy_(kv[l][0])
            dst[l][1].copy_(kv[l][1])
        h.save_layer(l)
    h.finish()
    for x in dst:
        for t in (x if isinstance(x, tuple) else (x,)):
            t.fill_(3.0)
    a, b = _landed(ref), _landed(eng)
    assert len(a) == 3 and a == b
    got, mask = eng.retrieve(toks)
    assert int(mask.sum()) == T
    for g, w in zip(got, kv):
        for x, y in zip(g if isinstance(g, tuple) else (g,), w if isinstance(w, tuple) else (w,)):
            assert torch.equal(_bits(x), _bits(y))
    ref.close(), eng.close()


def test_skip_existing_and_touches_like_store_paged(tmp_path):
    L, T, H, D, cs = 4, 8 * 256, 2, 64, 256
    blob = _kv((L, 2, T, H, D), torch.bfloat16, 21)
    toks = torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(21))
    stamps, landed = [], []
    for mode in ("paged", "layerwise"):
        eng = _engine("cpu", cs, local_capacity_bytes=1 << 30)
        caches, slots = _paged(blob)
        for l in range(L):
            _write(caches, slots, blob, l)
        eng.store_paged(toks[:4 * cs], caches, slots[:4 * cs])
        first = {k: id(e) for k, e in eng.engine_.dict.items()}
        if mode == "paged":
            eng.store_paged(toks, caches, slots)
        else:
            h = eng.store_paged_layerwise(toks, caches, slots)
            assert h._enc is not None
            for l in range(L):
                h.save_layer(l)
            h.finish()
        keys = [eng._make_key(x, "vllm") for x in eng._prefix_hash(toks)]
        _, mask = eng.retrieve(toks)
        assert int(mask.sum()) == T
        assert all(id(eng.engine_.dict[k]) == first[k] for k in keys[:4])
        stamps.append([eng.engine_._order.stamp(k) for k in keys])
        landed.append(_landed(eng))
        eng.close()
    assert stamps[0] == stamps[1] and landed[0] == landed[1]


@pytest.mark.parametrize("tier", ["host", "disk"])
def test_small_arena_keeps_the_longest_fitting_prefix(tier, tmp_path, monkeypatch):
    L, T, H, D, cs = 4, 16 * 256, 8, 128, 256
    blob = _kv((L, 2, T, H, D), torch.bfloat16, 31)
    toks = torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(31))
    caches, slots = _paged(blob)
    for l in range(L):
        _write(caches, slots, blob, l)
    ref = _engine(_local(tier, tmp_path / "a"), cs)
    ref.store_paged(toks, caches, slots)
    a = _landed(ref)
    total = sum(len(c) for c, _ in a.values())
    mb = max(1, total // 2 >> 20)
    assert mb << 20 < total
    monkeypatch.setenv("LMCACHE_B200_LAYERWISE_STORE_MB", str(mb))
    eng = _engine(_local(tier, tmp_path / "b"), cs)
    h = eng.store_paged_layerwise(toks, caches, slots)
    for l in range(L):
        h.save_layer(l)
    h.finish()
    kv, mask = eng.retrieve(toks)
    got = int(mask.sum())
    assert 0 < got < T and got % cs == 0 and bool(mask[:got].all())
    assert torch.equal(_bits(torch.stack([torch.stack(p) for p in kv])), _bits(blob[:, :, :got]))
    b = _landed(eng)
    assert len(b) == got // cs and all(a[k] == b[k] for k in b)
    ref.close(), eng.close()


def test_disk_restart_device_level_and_dropped_handle(tmp_path):
    L, T, H, D, cs = 4, 1300, 4, 64, 512
    blob = _kv((L, 2, T, H, D), torch.bfloat16, 51)
    toks = torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(51))
    caches, slots = _paged(blob)
    for l in range(L):
        _write(caches, slots, blob, l)
    eng = _engine(_local("disk", tmp_path / "d"), cs, device_cache_bytes=64 << 20)
    h = eng.store_paged_layerwise(toks, caches, slots)
    assert h._enc is not None
    for l in range(L):
        h.save_layer(l)
    h.finish()
    landed = _landed(eng)
    assert len(landed) == 3
    pool = eng.engine_._dcache.pool.buf
    torch.cuda.synchronize()
    for k, e in eng.engine_.dict.items():          # the device level holds the landed bytes
        assert e.rec.dev is not None
        got = pool[e.rec.dev.offset:e.rec.dev.offset + e.rec.nbytes].cpu().numpy().tobytes()
        assert got == landed[os.path.basename(k) if isinstance(k, str) else k][0]
    out = [(torch.zeros_like(k), torch.zeros_like(v)) for k, v in caches]
    mask = eng.retrieve_paged(toks, out, slots)
    assert int(mask.sum()) == T
    # a dropped handle gives its slot back to the pool
    h2 = eng.store_paged_layerwise(toks + 1, caches, slots)
    h2.save_layer(0)
    del h2
    assert len(eng.engine_._segments._free) >= 1
    eng.close()
    again = _engine(_local("disk", tmp_path / "d"), cs)            # a tier reopened on the directory
    assert {k: d for k, (d, _) in _landed(again).items()} == {k: d for k, (d, _) in landed.items()}   # bytes
    out = [(torch.zeros_like(k), torch.zeros_like(v)) for k, v in caches]
    mask = again.retrieve_paged(toks, out, slots)
    assert int(mask.sum()) == T
    for l in range(L):
        assert torch.equal(_bits(out[l][0].view(-1, H, D)[slots]), _bits(blob[l, 0]))
    again.close()
