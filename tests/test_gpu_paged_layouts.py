"""GPU: paged KV caches in vLLM's block-strided (FlashInfer) and split (PagedAttention / xFormers) layouts.  The mover's
split kernel (B200KV_KV_PAGED_SPLIT) and the strided slot remap must give the FlashAttention layout's blobs byte for
byte and write exactly the addressed elements; the codec refuses split descriptors; and every tier's paged store and
retrieve from and into any of the three layouts equals the FlashAttention layout's."""
import ctypes
import random

import numpy as np
import pytest
import torch

from test_gpu_host_tier import MODEL

pytestmark = pytest.mark.gpu
DTYPES = [torch.bfloat16, torch.float16, torch.uint8, torch.float8_e4m3fn, torch.float8_e5m2]
LAYOUTS = ["flash", "strided", "split"]


def _es(dtype):
    return torch.empty((), dtype=dtype).element_size()


def _rand_rows(n, dtype, gen):
    return torch.randint(0, 256, (n * _es(dtype),), dtype=torch.uint8, device="cuda", generator=gen).view(dtype)


def _layout(kind, rows, nb, bs, H, D):
    """one layer's (key, value) caches in layout `kind` holding rows[kv] ([nb * bs, H, D] FlashAttention rows)"""
    dt = rows[0].dtype
    if kind == "flash":
        return tuple(r.view(nb, bs, H, D).clone() for r in rows)
    if kind == "strided":
        kv = torch.empty(nb, 2, bs, H, D, dtype=dt, device="cuda")
        for i in range(2):
            kv[:, i] = rows[i].view(nb, bs, H, D)
        return kv[:, 0], kv[:, 1]
    x = 16 // _es(dt)
    cache = torch.empty(2, nb, bs * H * D, dtype=dt, device="cuda")      # vLLM: PagedAttention.split_kv_cache
    key, value = cache[0].view(nb, H, D // x, -1, x), cache[1].view(nb, H, D, -1)
    key.copy_(rows[0].view(nb, bs, H, D // x, x).permute(0, 2, 3, 1, 4))
    value.copy_(rows[1].view(nb, bs, H, D).permute(0, 2, 3, 1))
    return key, value


def _rows(kind, pair, nb, bs, H, D):
    """the inverse of _layout: a layer's pair as [nb * bs, H, D] rows, as bytes"""
    k, v = pair
    if kind == "split":
        k = k.permute(0, 3, 1, 2, 4).reshape(nb * bs, H, D)
        v = v.permute(0, 3, 1, 2).reshape(nb * bs, H, D)
    return tuple(t.reshape(nb * bs, H, D).view(torch.uint8) if t.element_size() == 1 else
                 t.reshape(nb * bs, H, D).view(torch.int16) for t in (k, v))


def _caches(kind, all_rows, nb, bs, H, D):
    return [_layout(kind, r, nb, bs, H, D) for r in all_rows]


def _all_rows(L, nb, bs, H, D, dtype, seed, fill=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = nb * bs * H * D
    if fill is not None:
        return [tuple(torch.full((n * _es(dtype),), fill, dtype=torch.uint8, device="cuda").view(dtype).view(nb * bs, H, D)
                      for _ in range(2)) for _ in range(L)]
    return [tuple(_rand_rows(n, dtype, g).view(nb * bs, H, D) for _ in range(2)) for _ in range(L)]


def _slots(kind, T, nb, bs, gen):
    """vllm: a block table's slots from token 0; mid: the same, from a token in the middle of a block; perm: any slots"""
    if kind == "perm":
        return torch.randperm(nb * bs, generator=gen)[:T].cuda()
    blocks = torch.randperm(nb, generator=gen)
    start = 5 if kind == "mid" else 0
    s = (blocks.view(-1, 1) * bs + torch.arange(bs).view(1, -1)).flatten()[start:start + T]
    return s.cuda()


def _pack(view, tok_begin, cs):
    """the chunk blobs' bytes (a ragged last chunk leaves the rest of the buffer unwritten)"""
    _, blobs = view.pack_chunks(tok_begin, cs)
    return torch.cat([b.contiguous().view(torch.uint8).flatten() for b in blobs])


def _shapes():
    out = []
    for dtype in DTYPES:
        x = 16 // _es(dtype)
        for bs in (8, 16, 32):
            for H in (1, 8):
                for D in (64, 80, 128, 256):
                    if D % x == 0:
                        out.append((dtype, bs, H, D))
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_pack_equals_flash_layout(dtype):
    from lmcache_b200.codec import KvView
    L = 3
    gen = torch.Generator().manual_seed(1)
    for dt, bs, H, D in _shapes():
        if dt != dtype:
            continue
        nb = 40
        rows = _all_rows(L, nb, bs, H, D, dtype, seed=bs * H + D)
        caches = {k: _caches(k, rows, nb, bs, H, D) for k in LAYOUTS}
        for skind in ("vllm", "mid", "perm"):
            T = 7 * bs + 3                                             # a ragged last chunk
            slots = _slots(skind, T, nb, bs, gen)
            views = {k: KvView.from_paged(caches[k], slots) for k in LAYOUTS}
            for tok_begin, cs in ((0, 2 * bs), (bs + 1, 3 * bs), (2 * bs, 64)):
                want = _pack(views["flash"], tok_begin, cs)
                for k in ("strided", "split"):
                    assert torch.equal(_pack(views[k], tok_begin, cs), want), (dt, bs, H, D, skind, k, tok_begin, cs)


def _pack_layers(view, tok_begin, cs, layers):
    from lmcache_b200 import _native as N
    n_tok = view.ntokens - tok_begin
    n = (n_tok + cs - 1) // cs
    last = n_tok - (n - 1) * cs
    a, b = layers
    row = 2 * view.H * view.D * view.dtype.itemsize
    stride = (b - a) * row * cs
    buf = torch.full((n * stride,), 0xA5, dtype=torch.uint8, device="cuda")
    table = torch.tensor(np.asarray([buf.data_ptr() + j * stride for j in range(n)], dtype=np.uint64).view(np.int64),
                         device="cuda")
    N.check(N.lib().b200kv_pack_chunks_layers(ctypes.byref(view.desc), tok_begin, n, cs, last, 0, a, b,
                                              ctypes.c_void_p(table.data_ptr()),
                                              torch.cuda.current_stream().cuda_stream), "pack_chunks_layers")
    return buf


@pytest.mark.parametrize("dtype,bs", [(torch.bfloat16, 16), (torch.float8_e4m3fn, 8), (torch.float16, 32)])
def test_pack_layers_equals_flash_layout(dtype, bs):
    from lmcache_b200.codec import KvView
    L, H, D, nb = 4, 8, 128, 30
    rows = _all_rows(L, nb, bs, H, D, dtype, seed=3)
    caches = {k: _caches(k, rows, nb, bs, H, D) for k in LAYOUTS}
    gen = torch.Generator().manual_seed(2)
    for skind in ("vllm", "mid", "perm"):
        slots = _slots(skind, 9 * bs + 5, nb, bs, gen)
        views = {k: KvView.from_paged(caches[k], slots) for k in LAYOUTS}
        for layers in ((0, L), (1, 3), (3, 4)):
            want = _pack_layers(views["flash"], bs, 2 * bs, layers)
            for k in ("strided", "split"):
                assert torch.equal(_pack_layers(views[k], bs, 2 * bs, layers), want), (skind, layers, k)


@pytest.mark.parametrize("dtype,bs,H,D", [(torch.bfloat16, 16, 8, 128), (torch.uint8, 8, 1, 64),
                                          (torch.float8_e5m2, 32, 8, 80), (torch.float16, 8, 1, 256)])
def test_unpack_writes_exactly_the_addressed_elements(dtype, bs, H, D):
    """unpack_chunks and unpack_chunks_layers into a sentinel-filled cache of each layout: the rows a FlashAttention
    cache gets, rearranged, and every other byte keeps the sentinel"""
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView
    L, nb = 3, 30
    gen = torch.Generator().manual_seed(4)
    src_rows = _all_rows(L, nb, bs, H, D, dtype, seed=5)
    for skind in ("vllm", "mid", "perm"):
        T = 6 * bs + 7
        slots = _slots(skind, T, nb, bs, gen)
        src = KvView.from_paged(_caches("flash", src_rows, nb, bs, H, D), slots)
        tok_begin, cs = bs + 3, 2 * bs
        buf, _ = src.pack_chunks(tok_begin, cs)
        n_tok = T - tok_begin
        n = (n_tok + cs - 1) // cs
        stride = L * 2 * H * D * _es(dtype) * cs
        for layers in (None, (1, 3)):
            want = None
            for k in LAYOUTS:
                dst = _caches(k, _all_rows(L, nb, bs, H, D, dtype, seed=0, fill=0x5A), nb, bs, H, D)
                view = KvView.from_paged(dst, slots)
                if layers is None:
                    N.check(N.lib().b200kv_unpack_chunks(ctypes.c_void_p(buf.data_ptr()), stride, n, cs,
                                                         n_tok - (n - 1) * cs, 0, ctypes.byref(view.desc), tok_begin,
                                                         torch.cuda.current_stream().cuda_stream), "unpack")
                else:
                    lay_buf = _pack_layers(src, tok_begin, cs, layers)
                    a, b = layers
                    lstride = (b - a) * 2 * H * D * _es(dtype) * cs
                    table = torch.tensor(np.asarray([lay_buf.data_ptr() + j * lstride for j in range(n)],
                                                    dtype=np.uint64).view(np.int64), device="cuda")
                    N.check(N.lib().b200kv_unpack_chunks_layers(ctypes.c_void_p(table.data_ptr()), n, cs,
                                                                n_tok - (n - 1) * cs, 0, a, b, ctypes.byref(view.desc),
                                                                tok_begin, torch.cuda.current_stream().cuda_stream),
                            "unpack_layers")
                got = [_rows(k, p, nb, bs, H, D) for p in dst]
                if want is None:
                    want = got
                    # the FlashAttention reference itself: addressed rows hold the source, the rest the sentinel
                    moved = slots[tok_begin:].long()
                    for l in range(L):
                        inside = layers is None or layers[0] <= l < layers[1]
                        for i in range(2):
                            w = got[l][i].reshape(nb * bs, -1)
                            s = src_rows[l][i].reshape(nb * bs, H, D)
                            s = (s.view(torch.uint8) if s.element_size() == 1 else s.view(torch.int16)).reshape(nb * bs, -1)
                            mask = torch.zeros(nb * bs, dtype=torch.bool, device="cuda")
                            if inside:
                                mask[moved] = True
                                assert torch.equal(w[mask], s[mask])
                            rest = w[~mask].view(torch.uint8)
                            assert bool((rest == 0x5A).all())
                else:
                    for l in range(L):
                        for i in range(2):
                            assert torch.equal(got[l][i], want[l][i]), (k, skind, layers, l, i)


def test_abi_refusals():
    """every CacheGen and lossless entry point refuses a split descriptor and leaves its outputs untouched; the mover
    refuses hf_layout = 1, a NULL slot map and D % x != 0"""
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import CacheGenCodec, KvView, LosslessCodec
    L, H, D, bs, nb, T = 2, 2, 64, 16, 8, 100
    rows = _all_rows(L, nb, bs, H, D, torch.bfloat16, seed=6)
    slots = torch.arange(T, device="cuda")
    split = KvView.from_paged(_caches("split", rows, nb, bs, H, D), slots)
    flash = KvView.from_paged(_caches("flash", rows, nb, bs, H, D), slots)
    for codec in (CacheGenCodec(MODEL), LosslessCodec()):
        out = torch.full((codec.out_stride(L, H, D, 64) * 2 + N.READ_SLACK,), 0x33, dtype=torch.uint8, device="cuda")
        with pytest.raises(N.NativeError, match="B200KV_KV_PAGED_SPLIT"):
            codec.encode_async(split, 0, 100, 64, out=out)
        torch.cuda.synchronize()
        assert bool((out == 0x33).all())
        raws = codec.encode_to_host(flash, 0, 100, 64)
        dst = _caches("split", _all_rows(L, nb, bs, H, D, torch.bfloat16, seed=0, fill=0x11), nb, bs, H, D)
        with pytest.raises(N.NativeError, match="B200KV_KV_PAGED_SPLIT"):
            codec.decode(raws, KvView.from_paged(dst, slots), [0, 64])
        torch.cuda.synchronize()
        for k, v in dst:
            assert bool((k.view(torch.uint8) == 0x11).all()) and bool((v.view(torch.uint8) == 0x11).all())
    buf = torch.empty(L * 2 * H * D * 64, dtype=torch.bfloat16, device="cuda")
    d = N.KvDesc.from_buffer_copy(split.desc)
    for what, mutate, hf in (("hf_layout", None, 1), ("slot_map", "slot", 0)):
        d = N.KvDesc.from_buffer_copy(split.desc)
        if mutate == "slot":
            d.slot_map = None
        rc = N.lib().b200kv_pack_chunks(ctypes.byref(d), 0, 1, 64, 64, hf, ctypes.c_void_p(buf.data_ptr()),
                                        buf.numel() * 2, torch.cuda.current_stream().cuda_stream)
        assert rc < 0, what
    d = N.KvDesc.from_buffer_copy(split.desc)
    d.D = 72                                                           # x = 8: 72 is fine; fp8 x = 16 is not
    d.dtype = N.DT_U8 | N.KV_PAGED_SPLIT
    rc = N.lib().b200kv_pack_chunks(ctypes.byref(d), 0, 1, 64, 64, 0, ctypes.c_void_p(buf.data_ptr()), buf.numel() * 2,
                                    torch.cuda.current_stream().cuda_stream)
    assert rc < 0 and b"D % x" in N.lib().b200kv_last_error()


def test_codec_refuses_split_in_every_plan():
    """the layer-wise encode plans and the decode plans (whole and head windows) refuse a split view too"""
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import CacheGenCodec, KvView, LosslessCodec
    L, H, D, bs, nb, T = 2, 2, 64, 16, 8, 64
    rows = _all_rows(L, nb, bs, H, D, torch.bfloat16, seed=8)
    slots = torch.arange(T, device="cuda")
    split = KvView.from_paged(_caches("split", rows, nb, bs, H, D), slots)
    flash = KvView.from_paged(_caches("flash", rows, nb, bs, H, D), slots)
    stream = torch.cuda.current_stream()
    scratch = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    p = ctypes.c_void_p(scratch.data_ptr())
    bins = N.float_array([32.0] * L)
    plan = N.EncodePlan()
    assert N.lib().b200kv_encode_layers_plan(ctypes.byref(split.desc), 0, 1, T, T, bins, bins, N.CODER_RANS_COMPACT,
                                             p, 1 << 14, p, 1 << 12, p, p, L, p, 1 << 14, ctypes.byref(plan),
                                             stream.cuda_stream) < 0
    assert b"B200KV_KV_PAGED_SPLIT" in N.lib().b200kv_last_error()
    lplan = N.LosslessEncodePlan()
    assert N.lib().b200kv_lossless_encode_layers_plan(ctypes.byref(split.desc), 0, 1, T, T, p, 1 << 14, p, 1 << 12, p,
                                                      p, L, p, 1 << 14, ctypes.byref(lplan), stream.cuda_stream) < 0
    assert b"B200KV_KV_PAGED_SPLIT" in N.lib().b200kv_last_error()
    torch.cuda.synchronize()
    assert int(scratch.count_nonzero()) == 0                           # nothing was enqueued
    for codec in (CacheGenCodec(MODEL), LosslessCodec()):
        raw = codec.encode_to_host(flash, 0, T, T)[0]
        buf = torch.zeros(len(raw) + N.READ_SLACK, dtype=torch.uint8, device="cuda")
        buf[:len(raw)] = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()
        with pytest.raises(N.NativeError, match="B200KV_KV_PAGED_SPLIT"):
            codec.decode_plan(buf.data_ptr(), buf.numel(), [0], [len(raw)], [T], split, [0], N.DT_BF16,
                              codec.coder_for(T), stream)
        with pytest.raises(N.NativeError, match="B200KV_KV_PAGED_SPLIT"):
            codec.decode_plan_heads(buf.data_ptr(), buf.numel(), [0], [len(raw)], [T], split, [0], N.DT_BF16,
                                    codec.coder_for(T), H, [0], [0], [1], stream)


@pytest.fixture(scope="module")
def lmserver():
    import os
    import socket
    import subprocess
    import sys
    import time
    from test_gpu_engine import ROOT, _free_port
    port = _free_port()
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    proc = subprocess.Popen([sys.executable, "-m", "lmcache_b200.server", "127.0.0.1", str(port)], env=env)
    for _ in range(100):
        try:
            socket.create_connection(("127.0.0.1", port), timeout=0.2).close()
            break
        except OSError:
            time.sleep(0.1)
    yield f"lm://127.0.0.1:{port}"
    proc.terminate()
    proc.wait()


# ---------------------------------------------------------------------------------------------- the tiers
L_E, H_E, D_E, BS, NB = 4, 2, 64, 16, 80


def _tier_config(tier, cs, lmserver, tmp_path):
    from lmcache_b200.config import LMCacheEngineConfig
    if tier in ("cpu", "cuda"):
        return LMCacheEngineConfig(cs, tier, None, None, False, False, None)
    if tier in ("host-cachegen", "host-lossless"):
        return LMCacheEngineConfig(cs, "cpu", None, None, False, False, tier.split("-")[1])
    if tier in ("disk-cachegen", "disk-lossless"):
        return LMCacheEngineConfig(cs, str(tmp_path / f"{tier}-{random.random()}"), None, None, False, False,
                                   tier.split("-")[1])
    if tier.startswith("lm-"):
        return LMCacheEngineConfig(cs, None, lmserver, tier[3:], False, False, None)
    if tier == "hybrid":
        return LMCacheEngineConfig(cs, "cuda", lmserver, "cachegen", False, False, None)
    raise ValueError(tier)


def _engine(autorelease, tier, cs, lmserver, tmp_path, name, ws=1, rank=0, reshard=None):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineMetadata
    cfg = _tier_config(tier, cs, lmserver, tmp_path)
    if reshard is not None:
        cfg.reshard_world_sizes = reshard
    return autorelease(LMCacheEngine(cfg, LMCacheEngineMetadata(name, ws, rank, "vllm", "bfloat16")))


TIERS = ["cpu", "cuda", "host-cachegen", "host-lossless", "disk-cachegen", "disk-lossless", "lm-cachegen",
         "lm-lossless", "lm-torch", "hybrid"]


def _cache_rows(kind, caches):
    return [_rows(kind, p, NB, BS, H_E, D_E) for p in caches]


@pytest.mark.parametrize("tier", TIERS)
def test_engine_round_trips_every_layout_pair(tier, lmserver, tmp_path, autorelease):
    """store_paged from layout A and retrieve_paged into layout B, for all 9 pairs: the same ret_mask and the same
    rows as the FlashAttention store and retrieve, rows outside the hit untouched; a suffix mask with a straddling first
    chunk and a skip_existing second store; FP8 where the tier takes it"""
    cs = 64
    dtypes = [torch.bfloat16] + ([] if "cachegen" in tier or tier == "hybrid" else [torch.float8_e4m3fn])
    for dtype in dtypes:
        T = 4 * cs + 21
        gen = torch.Generator().manual_seed(11)
        slots = _slots("vllm", T, NB, BS, gen)
        tokens = torch.randint(0, 32000, (T,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
        rows = _all_rows(L_E, NB, BS, H_E, D_E, dtype, seed=12)
        mask = torch.ones(T, dtype=torch.bool)
        mask[:cs + 9] = False
        results = {}
        for ai, a in enumerate(LAYOUTS):
            # own tokens per layout and tier: a server shared across engines (lm://) must not serve one's chunks to another
            toks = tokens + 40000 * ai + 1000 * (dtype != torch.bfloat16) + 200000 * TIERS.index(tier)
            eng = _engine(autorelease, tier, cs, lmserver, tmp_path, MODEL)
            src = _caches(a, rows, NB, BS, H_E, D_E)
            eng.store_paged(toks[:2 * cs], [p for p in src], slots[:2 * cs])
            eng.store_paged(toks, src, slots)                            # skip_existing: from chunk 2 on
            if hasattr(eng.engine_, "drain"):
                eng.engine_.drain()
            for b in LAYOUTS:
                for m in (None, mask):
                    dst = _caches(b, _all_rows(L_E, NB, BS, H_E, D_E, dtype, seed=0, fill=0x3C), NB, BS, H_E, D_E)
                    ret = eng.retrieve_paged(toks, dst, slots, m)
                    torch.cuda.synchronize()
                    results[(a, b, m is None)] = (ret.clone(), _cache_rows(b, dst))
        for key, (ret, got) in results.items():
            want_ret, want = results[("flash", "flash", key[2])]
            assert torch.equal(ret, want_ret), (tier, dtype, key)
            for l in range(L_E):
                for i in range(2):
                    assert torch.equal(got[l][i], want[l][i]), (tier, dtype, key, l, i)
        ret, want = results[("flash", "flash", False)]
        hit = slots[ret.cuda()].long()
        untouched = torch.ones(NB * BS, dtype=torch.bool, device="cuda")
        untouched[hit] = False
        assert int(ret.sum()) == T - cs - 9
        assert bool((want[0][0].reshape(NB * BS, -1)[untouched].view(torch.uint8) == 0x3C).all())


@pytest.mark.parametrize("tier", ["cpu", "cuda"])
def test_engine_stores_the_flash_layouts_bytes(tier, lmserver, tmp_path, autorelease):
    """the stored blobs of a split or strided store are those of the FlashAttention store"""
    from test_gpu_raw_layerwise import _stored
    cs, T = 64, 200
    gen = torch.Generator().manual_seed(13)
    slots = _slots("perm", T, NB, BS, gen)
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    rows = _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=14)
    stored = {}
    for a in LAYOUTS:
        eng = _engine(autorelease, tier, cs, lmserver, tmp_path, MODEL)
        eng.store_paged(tokens, _caches(a, rows, NB, BS, H_E, D_E), slots)
        torch.cuda.synchronize()
        stored[a] = _stored(eng)
    for a in ("strided", "split"):
        assert stored[a].keys() == stored["flash"].keys()
        for k in stored["flash"]:
            assert torch.equal(stored[a][k], stored["flash"][k]), (tier, a)


@pytest.mark.parametrize("tier", ["cpu", "cuda", "host-lossless", "host-cachegen"])
def test_layerwise_forms(tier, lmserver, tmp_path, autorelease):
    """store_paged_layerwise and retrieve_paged_layerwise from and into a split cache equal the FlashAttention ones"""
    cs, T = 64, 3 * 64 + 10
    gen = torch.Generator().manual_seed(15)
    slots = _slots("vllm", T, NB, BS, gen)
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    rows = _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=16)
    out = {}
    for a in ("flash", "split"):
        eng = _engine(autorelease, tier, cs, lmserver, tmp_path, MODEL)
        src = _caches(a, rows, NB, BS, H_E, D_E)
        h = eng.store_paged_layerwise(tokens, src, slots)
        for l in (2, 0, 3, 1):
            h.save_layer(l)
        h.finish()
        dst = _caches(a, _all_rows(L_E, NB, BS, H_E, D_E, torch.bfloat16, seed=0, fill=0x21), NB, BS, H_E, D_E)
        r = eng.retrieve_paged_layerwise(tokens, dst, slots)
        r.synchronize()
        out[a] = (r.ret_mask, _cache_rows(a, dst))
    assert torch.equal(out["split"][0], out["flash"][0]) and int(out["flash"][0].sum()) == T
    for l in range(L_E):
        for i in range(2):
            assert torch.equal(out["split"][1][l][i], out["flash"][1][l][i])


def test_reshard_tp2_to_tp1_into_split_cache(lmserver, tmp_path, autorelease):
    """chunks two TP ranks stored (CacheGen, lm://) decode into one rank's split cache as into its FlashAttention one"""
    cs, T, Hg = 64, 150, 4
    gen = torch.Generator().manual_seed(17)
    tokens = torch.randint(0, 32000, (T,), device="cuda")
    full = _all_rows(L_E, NB, BS, Hg, D_E, torch.bfloat16, seed=18)
    slots = _slots("vllm", T, NB, BS, gen)
    name = MODEL
    for r in range(2):
        part = [tuple(x[:, r * 2:(r + 1) * 2].contiguous() for x in p) for p in full]
        e = _engine(autorelease, "lm-cachegen", cs, lmserver, tmp_path, name, ws=2, rank=r)
        e.store_paged(tokens, _caches("flash", part, NB, BS, 2, D_E), slots)
        e.engine_.drain()
    got = {}
    for b in LAYOUTS:
        e = _engine(autorelease, "lm-cachegen", cs, lmserver, tmp_path, name, reshard=[2])
        dst = _caches(b, _all_rows(L_E, NB, BS, Hg, D_E, torch.bfloat16, seed=0, fill=0x44), NB, BS, Hg, D_E)
        ret = e.retrieve_paged(tokens, dst, slots)
        torch.cuda.synchronize()
        got[b] = (ret, [_rows(b, p, NB, BS, Hg, D_E) for p in dst])
    assert int(got["flash"][0].sum()) == T
    for b in ("strided", "split"):
        assert torch.equal(got[b][0], got["flash"][0])
        for l in range(L_E):
            for i in range(2):
                assert torch.equal(got[b][1][l][i], got["flash"][1][l][i])
