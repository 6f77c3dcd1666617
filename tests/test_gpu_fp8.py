"""GPU: one-byte (FP8 / uint8) KV caches through the mover, the lossless codec and every raw and lossless tier.

The mover's pack / unpack equal torch's slicing for blob, huggingface, tuple, paged and latent sources, on the vector and
the scalar path, into device and mapped pinned chunks, and write nothing outside the call; device containers equal
tests/lossless8_ref.py byte for byte; decodes -- whole, by layer ranges, by head windows -- are bit-exact; damage is
refused or flagged; a destination of another dtype and every CacheGen entry point refuse one-byte KV; and LMCacheEngine
round trips are bit-exact on the raw cpu / cuda tiers, the lossless host and disk tiers (bounded, device cache, persistent
index), lm:// with the lossless (also layer-major) and torch serdes, hybrid tiers, MLA latent KV and resharding."""
import ctypes
import os

import numpy as np
import pytest
import torch

import lossless8_ref as R8

pytestmark = pytest.mark.gpu
MODEL = "lmsys/longchat-7b-16k"
SENT = 0xA5
ONE_BYTE = [torch.uint8, torch.float8_e4m3fn, torch.float8_e5m2]
CODE = {torch.uint8: 2, torch.float8_e4m3fn: 3, torch.float8_e5m2: 4}


def _kv(shape, dtype, seed, kind="normal"):
    """FP8 values of a KV-like distribution (uint8: the E4M3 bytes, as vLLM 0.6.x allocates its fp8 cache), or every
    byte value ("bits")"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "bits":
        return torch.randint(0, 256, shape, device="cuda", generator=g, dtype=torch.uint8).view(dtype)
    x = torch.randn(shape, device="cuda", generator=g)
    if kind == "scaled":
        x = x * torch.exp(torch.randn(shape[-1], device="cuda", generator=g))
    f8 = torch.float8_e5m2 if dtype == torch.float8_e5m2 else torch.float8_e4m3fn
    return x.to(f8).view(dtype)


def _u8(x):
    return x.contiguous().view(torch.uint8)


def _np(x):
    return _u8(x).cpu().numpy()


def _sent_like(x):
    return torch.full(x.shape, SENT, dtype=torch.uint8, device=x.device).view(x.dtype)


def _codec():
    from lmcache_b200.codec import LosslessCodec
    return LosslessCodec()


def _toks(T, seed):
    return torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(seed))


def _pairs(blob):
    return tuple((blob[l, 0], blob[l, 1]) for l in range(blob.shape[0]))


def _stack(kv):
    """the bytes of a tuple of per-layer (K, V) as one [L, 2, ...] uint8 tensor"""
    return torch.stack([torch.stack([_u8(k), _u8(v)]) for k, v in kv])


def _paged(blob, nslots, seed, dtype=None):
    """[num_blocks, 16, H, D] caches holding blob's tokens at shuffled slots"""
    L, _, T, H, D = blob.shape
    slots = torch.randperm(nslots, generator=torch.Generator().manual_seed(seed))[:T].cuda()
    caches = [(torch.zeros(nslots // 16, 16, H, D, dtype=torch.uint8, device="cuda").view(dtype or blob.dtype),
               torch.zeros(nslots // 16, 16, H, D, dtype=torch.uint8, device="cuda").view(dtype or blob.dtype))
              for _ in range(L)]
    for l, (k, v) in enumerate(caches):
        _u8(k).view(-1, H, D)[slots] = _u8(blob[l, 0])
        _u8(v).view(-1, H, D)[slots] = _u8(blob[l, 1])
    return caches, slots


# ------------------------------------------------------------------------------------------ mover
def _move(pack, view, tok_begin, n_tok, cs, hf, ptr, stride):
    from lmcache_b200 import _native as N
    n = (n_tok + cs - 1) // cs
    last = n_tok - (n - 1) * cs
    sp = torch.cuda.current_stream().cuda_stream
    if pack:
        rc = N.lib().b200kv_pack_chunks(ctypes.byref(view.desc), tok_begin, n, cs, last, int(hf), ctypes.c_void_p(ptr),
                                        stride, sp)
    else:
        rc = N.lib().b200kv_unpack_chunks(ctypes.c_void_p(ptr), stride, n, cs, last, int(hf), ctypes.byref(view.desc),
                                          tok_begin, sp)
    N.check(rc, "pack" if pack else "unpack")
    torch.cuda.synchronize()
    return n


@pytest.mark.parametrize("D", [64, 128, 576, 20])
@pytest.mark.parametrize("where", ["device", "pinned"])
def test_mover_equals_torch(D, where):
    from lmcache_b200.codec import KvView, PinnedBuffer
    L, T, t0, cs = 2, 200, 37, 64
    H = 1 if D == 576 else 2
    dtype = torch.float8_e4m3fn
    blob = _kv((L, 2, T, H, D), dtype, D, "bits")
    lat = _kv((L, T, D), dtype, D + 1, "bits")
    caches, slots = _paged(blob, 256, D)
    hfb = blob.permute(0, 1, 3, 2, 4).contiguous()
    kinds = {
        "blob": (KvView.from_blob(blob, "vllm"), lambda a, b: _np(blob[:, :, a:b]), False),
        "huggingface": (KvView.from_blob(hfb, "huggingface"), lambda a, b: _np(hfb[:, :, :, a:b]), True),
        "tuple": (KvView.from_tuple(_pairs(blob), "vllm"), lambda a, b: _np(blob[:, :, a:b]), False),
        "paged": (KvView.from_paged(caches, slots), lambda a, b: _np(blob[:, :, a:b]), False),
        "latent": (KvView.from_blob(lat, "vllm"), lambda a, b: _np(lat[:, a:b]), False),
    }
    for name, (view, ref, hf) in kinds.items():
        per_tok = view.planes * view.H * view.D
        stride = (per_tok * cs + 16 + 15) & ~15                   # a sentinel gap after every chunk
        n = (T - t0 + cs - 1) // cs
        if where == "device":
            buf = torch.full((n * stride,), SENT, dtype=torch.uint8, device="cuda")
            ptr, host = buf.data_ptr(), (lambda: buf.cpu().numpy())
        else:
            pin = PinnedBuffer(n * stride)
            np.frombuffer(pin.view(), dtype=np.uint8)[:] = SENT
            ptr, host = pin.dev_ptr, (lambda: np.frombuffer(pin.view(), dtype=np.uint8).copy())
        _move(True, view, t0, T - t0, cs, hf, ptr, stride)
        got = host()
        for j in range(n):
            a, b = t0 + j * cs, min(T, t0 + (j + 1) * cs)
            want = ref(a, b).reshape(-1)
            c = got[j * stride:(j + 1) * stride]
            assert np.array_equal(c[:want.size], want), (name, j)
            assert (c[want.size:] == SENT).all(), (name, j, "write outside the chunk")
        # unpack into a destination of the same kind full of sentinels: the call's rows only
        if name == "paged":
            dst_c = [(_sent_like(k), _sent_like(v)) for k, v in caches]
            dview = KvView.from_paged(dst_c, slots)
        elif name == "tuple":
            dst_c = tuple((_sent_like(blob[l, 0]), _sent_like(blob[l, 1])) for l in range(L))
            dview = KvView.from_tuple(dst_c, "vllm")
        else:
            src = {"blob": blob, "huggingface": hfb, "latent": lat}[name]
            dst_c = _sent_like(src)
            dview = KvView.from_blob(dst_c, "huggingface" if hf else "vllm")
        _move(False, dview, t0, T - t0, cs, hf, ptr, stride)
        if name == "paged":
            out = torch.stack([torch.stack([_u8(k).view(-1, H, D)[slots], _u8(v).view(-1, H, D)[slots]])
                               for k, v in dst_c])
            rest = torch.ones(256, dtype=torch.bool, device="cuda")
            rest[slots[t0:]] = False
            assert all((_u8(k).view(-1, H, D)[rest] == SENT).all() and (_u8(v).view(-1, H, D)[rest] == SENT).all()
                       for k, v in dst_c)
            assert torch.equal(out[:, :, t0:], _u8(blob[:, :, t0:]))
            continue
        out = _u8(_stack(dst_c)) if name == "tuple" else _u8(dst_c)
        src = _u8(blob if name == "tuple" else {"blob": blob, "huggingface": hfb, "latent": lat}[name])
        tdim = 3 if name == "huggingface" else 1 if name == "latent" else 2
        assert torch.equal(out.narrow(tdim, t0, T - t0), src.narrow(tdim, t0, T - t0)), name
        assert (out.narrow(tdim, 0, t0) == SENT).all(), name


# ------------------------------------------------------------------------------------------ lossless containers
@pytest.mark.parametrize("dtype", ONE_BYTE)
def test_containers_match_spec_and_decode_everywhere(dtype):
    from lmcache_b200.codec import KvView
    L, T, H, D, cs, t0 = 3, 700, 4, 128, 256, 37
    dt = CODE[dtype]
    blob = _kv((L, 2, T, H, D), dtype, dt, "scaled")
    bits = _np(blob)
    codec = _codec()
    ref = [R8.encode(np.ascontiguousarray(bits[:, :, a:a + cs].transpose(1, 0, 2, 3, 4)).reshape(2 * L, -1, H * D),
                     L, H, D, dt) for a in range(t0, T, cs)]
    hfb = blob.permute(0, 1, 3, 2, 4).contiguous()
    caches, slots = _paged(blob, 1024, 3)
    for name, view in (("blob", KvView.from_blob(blob, "vllm")), ("huggingface", KvView.from_blob(hfb, "huggingface")),
                       ("tuple", KvView.from_tuple(_pairs(blob), "vllm")), ("paged", KvView.from_paged(caches, slots))):
        assert codec.encode_to_host(view, t0, T - t0, cs) == ref, name
    dst_tok = [j * cs for j in range(len(ref))]
    n_tok = T - t0
    # whole decode into every destination kind, sentinels around the call's tokens
    out = _sent_like(torch.empty((L, 2, n_tok + 8, H, D), dtype=torch.uint8, device="cuda")).view(dtype)
    codec.decode(ref, KvView.from_blob(out, "vllm"), [4 + d for d in dst_tok])
    torch.cuda.synchronize()
    assert codec.decode_status() == [0] * len(ref)
    assert torch.equal(_u8(out)[:, :, 4:4 + n_tok], _u8(blob[:, :, t0:]))
    assert (_u8(out)[:, :, :4] == SENT).all() and (_u8(out)[:, :, 4 + n_tok:] == SENT).all()
    out_hf = _sent_like(hfb[:, :, :, t0:].contiguous())
    codec.decode(ref, KvView.from_blob(out_hf, "huggingface"), dst_tok)
    out_t = tuple((_sent_like(blob[l, 0, t0:]), _sent_like(blob[l, 1, t0:])) for l in range(L))
    codec.decode(ref, KvView.from_tuple(out_t, "vllm"), dst_tok)
    pc = [(_sent_like(k), _sent_like(v)) for k, v in caches]
    codec.decode(ref, KvView.from_paged(pc, slots[t0:]), dst_tok)
    torch.cuda.synchronize()
    assert torch.equal(_u8(out_hf), _u8(hfb[:, :, :, t0:]))
    assert torch.equal(_u8(_stack(out_t)), _u8(blob[:, :, t0:]))
    for l, (k, v) in enumerate(pc):
        assert torch.equal(_u8(k).view(-1, H, D)[slots[t0:]], _u8(blob[l, 0, t0:]))
        assert torch.equal(_u8(v).view(-1, H, D)[slots[t0:]], _u8(blob[l, 1, t0:]))
        assert (_u8(k).view(-1, H, D)[slots[:t0]] == SENT).all()
    # layer ranges in any order equal the whole decode
    batch = codec.encode(KvView.from_blob(blob, "vllm"), t0, n_tok, cs)
    offs = [j * batch.stride for j in range(len(batch.sizes))]
    nt = [min(cs, n_tok - j * cs) for j in range(len(batch.sizes))]
    part = _sent_like(blob[:, :, t0:].contiguous())
    s = torch.cuda.current_stream()
    plan, ws = codec.decode_plan(batch.buf.data_ptr(), batch.buf.numel(), offs, batch.sizes, nt,
                                 KvView.from_blob(part, "vllm"), dst_tok, batch.max_dtype, batch.coder, s)
    for a, b in ((2, 3), (0, 1), (1, 2)):
        codec.decode_layers(plan, a, b, s)
    torch.cuda.synchronize()
    assert batch.max_dtype == dt and torch.equal(_u8(part), _u8(blob[:, :, t0:]))
    # a head window: source heads [1, 3) into a 2-head destination
    win = _sent_like(torch.empty((L, 2, n_tok, 2, D), dtype=torch.uint8, device="cuda")).view(dtype)
    codec.decode_raw_heads(batch.buf.data_ptr(), batch.buf.numel(), offs, batch.sizes, nt, KvView.from_blob(win, "vllm"),
                           dst_tok, batch.max_dtype, batch.coder, H, [1] * len(nt), [0] * len(nt), [2] * len(nt))
    torch.cuda.synchronize()
    assert torch.equal(_u8(win), _u8(blob[:, :, t0:, 1:3]))
    # a lossless container decodes into its own dtype only: another one-byte dtype, uint8 vs fp8, bf16
    for other in [d for d in ONE_BYTE if d != dtype] + [torch.bfloat16]:
        o = torch.empty((L, 2, n_tok, H, D), dtype=other, device="cuda")
        with pytest.raises(ValueError, match="own dtype"):
            codec.decode(ref, KvView.from_blob(o, "vllm"), dst_tok)


def test_latent_fp8_version6_and_single_symbol_planes():
    from lmcache_b200.codec import KvView
    L, T, D, cs = 4, 520, 576, 256
    lat = _kv((L, T, D), torch.float8_e4m3fn, 11, "scaled")
    lat[1] = torch.tensor(1.0).to(torch.float8_e4m3fn)           # one symbol in a plane: f = 4096
    codec = _codec()
    conts = codec.encode_to_host(KvView.from_blob(lat, "vllm"), 0, T, cs)
    bits = _np(lat)
    for j, c in enumerate(conts):
        assert c[4] == 6 and c == R8.encode(bits[:, j * cs:(j + 1) * cs], L, 1, D, 3, latent=True)
    out = _sent_like(lat)
    codec.decode(conts, KvView.from_blob(out, "vllm"), [0, cs, 2 * cs])
    torch.cuda.synchronize()
    assert torch.equal(_u8(out), _u8(lat))
    y = _kv((1, 2, 4096, 1, 16), torch.uint8, 4, "bits")         # t = 4096, incompressible
    c = codec.encode_to_host(KvView.from_blob(y, "vllm"), 0, 4096, 4096)[0]
    assert c == R8.encode(_np(y).reshape(2, 4096, 16), 1, 1, 16, 2)
    out = torch.empty_like(y)
    codec.decode([c], KvView.from_blob(out, "vllm"), [0])
    torch.cuda.synchronize()
    assert torch.equal(out, y)


def test_damaged_containers_are_refused_or_flagged():
    from lmcache_b200.codec import KvView
    L, T, H, D = 2, 96, 2, 64
    x = _kv((L, 2, T, H, D), torch.float8_e4m3fn, 21, "scaled")
    codec = _codec()
    good = codec.encode_to_host(KvView.from_blob(x, "vllm"), 0, T, T)[0]
    lo = R8.layout(2 * L, H * D, T)
    rng = np.random.default_rng(1234)
    outcomes = {"refused": 0, "flagged": 0}
    for trial in range(40):
        b = bytearray(good)
        lo_b, hi_b = [(0, 64), (lo["off_freq"], lo["off_lens"]), (lo["off_lens"], lo["off_raw"]),
                      (lo["off_payload"], len(good))][trial % 4]
        for _ in range(1 + trial % 3):
            b[int(rng.integers(lo_b, hi_b))] ^= int(rng.integers(1, 256))
        out = _sent_like(torch.empty((L, 2, T + 32, H, D), dtype=torch.uint8, device="cuda")).view(x.dtype)
        try:
            codec.decode([bytes(b)], KvView.from_blob(out, "vllm"), [16])
            st = codec.decode_status()
        except (ValueError, TypeError):
            outcomes["refused"] += 1
            st = None
        got = _u8(out)
        assert (got[:, :, :16] == SENT).all() and (got[:, :, 16 + T:] == SENT).all(), "write outside the call's rows"
        if st is None:
            continue
        if st[0] != 0:
            outcomes["flagged"] += 1
        else:
            assert torch.equal(got[:, :, 16:16 + T], _u8(x)), f"trial {trial}: damage neither refused nor flagged"
    assert outcomes["refused"] > 0 and outcomes["flagged"] > 0


def test_native_decode_refuses_another_dtype():
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView
    L, T, H, D = 2, 64, 2, 32
    x = _kv((L, 2, T, H, D), torch.float8_e4m3fn, 5)
    codec = _codec()
    batch = codec.encode(KvView.from_blob(x, "vllm"), 0, T, T)
    for other in (torch.float8_e5m2, torch.uint8):
        dst = _sent_like(x.view(torch.uint8)).view(other)
        plan = N.LosslessDecodePlan()
        ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
        rc = N.lib().b200kv_lossless_decode_plan(
            ctypes.c_void_p(batch.buf.data_ptr()), batch.buf.numel(), N.i64_array([0]), N.i64_array(batch.sizes),
            N.i32_array([T]), N.i64_array([0]), 1, 3, ctypes.byref(KvView.from_blob(dst, "vllm").desc), None,
            ctypes.c_void_p(ws.data_ptr()), ws.numel(), ctypes.byref(plan), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert rc < 0 and (_u8(dst) == SENT).all()


def test_every_cachegen_entry_point_refuses_one_byte_kv():
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import CacheGenCodec, KvView, PinnedBuffer
    L, T, H, D = 2, 64, 2, 32
    cg = CacheGenCodec(MODEL)
    kb, vb = cg._kb, cg._vb
    src16 = torch.randn(L, 2, T, H, D, device="cuda").to(torch.bfloat16)
    good = cg.encode(KvView.from_blob(src16, "vllm"), 0, T, T)
    sp = torch.cuda.current_stream().cuda_stream
    lib = N.lib()
    for dtype in ONE_BYTE:
        x = _kv((L, 2, T, H, D), dtype, 1)
        view = KvView.from_blob(x, "vllm")
        out = torch.full((1 << 20,), SENT, dtype=torch.uint8, device="cuda")
        ws = torch.zeros(8 << 20, dtype=torch.uint8, device="cuda")
        pin = PinnedBuffer(4096)                                 # mapped: sizes and segment rows
        words = np.frombuffer(pin.view(), dtype=np.uint64)
        words[:] = 7
        rc = lib.b200kv_encode_chunks(ctypes.byref(view.desc), 0, 1, T, T, kb, vb, N.CODER_RANS_COMPACT,
                                      ctypes.c_void_p(out.data_ptr()), 1 << 19, ctypes.c_void_p(pin.dev_ptr),
                                      ctypes.c_void_p(ws.data_ptr()), ws.numel(), sp)
        assert rc < 0
        plan = N.EncodePlan()
        rc = lib.b200kv_encode_layers_plan(ctypes.byref(view.desc), 0, 1, T, T, kb, vb, N.CODER_RANS_COMPACT,
                                           ctypes.c_void_p(out.data_ptr()), 1 << 18,
                                           ctypes.c_void_p(out.data_ptr() + (1 << 19)), 1 << 16,
                                           ctypes.c_void_p(pin.dev_ptr + 1024), ctypes.c_void_p(pin.dev_ptr), 1,
                                           ctypes.c_void_p(ws.data_ptr()), ws.numel(), ctypes.byref(plan), sp)
        assert rc < 0
        dst = _sent_like(x.view(torch.uint8)).view(dtype)
        dview = KvView.from_blob(dst, "vllm")
        args = (ctypes.c_void_p(good.buf.data_ptr()), good.buf.numel(), N.i64_array([0]), N.i64_array(good.sizes),
                N.i32_array([T]), N.i64_array([0]), 1, good.max_dtype, good.coder, ctypes.byref(dview.desc), kb, vb,
                None, ctypes.c_void_p(ws.data_ptr()), ws.numel())
        assert lib.b200kv_decode_chunks(*args, sp) < 0
        assert lib.b200kv_decode_plan(*args, ctypes.byref(N.DecodePlan()), sp) < 0
        assert lib.b200kv_decode_plan_heads(*args, ctypes.byref(N.DecodePlan()), sp, H, N.i32_array([0]),
                                            N.i32_array([0]), N.i32_array([H])) < 0
        torch.cuda.synchronize()
        assert (out == SENT).all() and (_u8(dst) == SENT).all() and (words == 7).all()
        pin.close()
        # and the Python codec says what to use instead
        with pytest.raises(TypeError, match="lossless"):
            cg.encode(view, 0, T, T)
        with pytest.raises(TypeError, match="lossless"):
            cg.decode_raw(good.buf.data_ptr(), good.buf.numel(), [0], good.sizes, [T], dview, [0], good.max_dtype,
                          good.coder)


# ------------------------------------------------------------------------------------------ engines
@pytest.fixture
def server():
    from lmcache_b200 import _native as N
    h = ctypes.c_void_p()
    N.check(N.lib().b200kv_lm_server_start(b"127.0.0.1", 0, ctypes.byref(h)))
    yield f"lm://127.0.0.1:{N.lib().b200kv_lm_server_port(h)}"
    N.lib().b200kv_lm_server_stop(h)


def _engine(local=None, remote=None, rserde=None, lserde=None, cs=256, mla=False, W=1, r=0, **kw):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    cfg = LMCacheEngineConfig(cs, local, remote, rserde, False, False, lserde, **kw)
    return LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, W, r, "vllm", "fp8", use_mla=mla))


TIERS = ["cpu", "cuda", "host_lossless", "disk_lossless", "lm_lossless", "lm_lossless_layerwise", "lm_torch", "hybrid"]


def _tier_engine(tier, url, tmp_path):
    if tier in ("cpu", "cuda"):
        return _engine(tier)
    if tier == "host_lossless":
        return _engine("cpu", lserde="lossless", local_capacity_bytes=1 << 30, device_cache_bytes=64 << 20)
    if tier == "disk_lossless":
        return _engine(str(tmp_path) + "/", lserde="lossless", device_cache_bytes=64 << 20)
    if tier in ("lm_lossless", "lm_lossless_layerwise"):
        return _engine(remote=url, rserde="lossless")
    if tier == "lm_torch":
        return _engine(remote=url, rserde="torch")
    return _engine("cpu", remote=url, rserde="lossless")


@pytest.mark.parametrize("dtype", [torch.uint8, torch.float8_e4m3fn])
@pytest.mark.parametrize("tier", TIERS)
def test_engine_round_trips_are_bit_exact(tier, dtype, server, tmp_path, monkeypatch):
    if tier == "lm_lossless_layerwise":
        monkeypatch.setenv("LMCACHE_B200_REMOTE_LAYERWISE", "1")
    L, T, H, D = 3, 600, 4, 64
    blob = _kv((L, 2, T, H, D), dtype, 31, "scaled")
    toks = _toks(T, 1)
    e = _tier_engine(tier, server, tmp_path)
    e.store(toks, _pairs(blob))
    kv, mask = e.retrieve(toks)
    assert int(mask.sum()) == T and kv[0][0].dtype == dtype and torch.equal(_u8(_stack(kv)), _u8(blob))
    m = torch.ones(T, dtype=torch.bool)
    m[:300] = False                                              # straddles chunk 1
    kv, mask = e.retrieve(toks, m)
    assert int(mask.sum()) == T - 300 and torch.equal(_u8(_stack(kv)), _u8(blob[:, :, 300:]))
    # vLLM-shaped paged caches: store_paged / retrieve_paged, with and without a suffix mask
    toks2 = _toks(T, 2)
    caches, slots = _paged(blob, 1024, 7)
    e.store_paged(toks2, caches, slots)
    for msk, lo in ((None, 0), (m, 300)):
        dst = [(_sent_like(k), _sent_like(v)) for k, v in caches]
        pm = e.retrieve_paged(toks2, dst, slots, msk)
        torch.cuda.synchronize()
        assert int(pm.sum()) == T - lo
        for l, (k, v) in enumerate(dst):
            assert torch.equal(_u8(k).view(-1, H, D)[slots[lo:]], _u8(blob[l, 0, lo:]))
            assert torch.equal(_u8(v).view(-1, H, D)[slots[lo:]], _u8(blob[l, 1, lo:]))
            assert (_u8(k).view(-1, H, D)[slots[:lo]] == SENT).all()
    # both layer-wise forms
    toks3 = _toks(T, 3)
    s = e.store_paged_layerwise(toks3, caches, slots)
    for l in range(L):
        s.save_layer(l)
    s.finish()
    r = e.retrieve_layerwise(toks3)
    for l in range(L):
        r.wait_layer(l)
    assert int(r.ret_mask.sum()) == T and torch.equal(_u8(_stack(r.kv)), _u8(blob))
    dst = [(_sent_like(k), _sent_like(v)) for k, v in caches]
    r = e.retrieve_paged_layerwise(toks3, dst, slots)
    for l in range(L):
        r.wait_layer(l)
        k, v = dst[l]
        assert torch.equal(_u8(k).view(-1, H, D)[slots], _u8(blob[l, 0]))
        assert torch.equal(_u8(v).view(-1, H, D)[slots], _u8(blob[l, 1]))
    e.close()


@pytest.mark.parametrize("tier", ["host", "disk"])
def test_layerwise_store_lands_the_whole_encode_and_the_disk_index_persists(tier, tmp_path):
    L, T, H, D = 3, 700, 4, 128
    blob = _kv((L, 2, T, H, D), torch.float8_e4m3fn, 41, "scaled")
    toks = _toks(T, 41)
    path = lambda n: "cpu" if tier == "host" else str(tmp_path / n) + "/"  # noqa: E731
    a = _engine(path("a"), lserde="lossless")
    a.store(toks, _pairs(blob))
    b = _engine(path("b"), lserde="lossless")
    s = b.store_layerwise(toks, _pairs(blob))
    for l in range(L):
        s.save_layer(l)
    s.finish()

    def containers(eng, n):
        if tier == "host":
            out = {}
            for k, en in eng.engine_.dict.items():
                en.ready.wait()
                out[k] = bytes(en.rec.blk.view())
            return out
        return {f: open(os.path.join(tmp_path / n, f), "rb").read() for f in os.listdir(tmp_path / n)}
    ca, cb = containers(a, "a"), containers(b, "b")
    assert len(ca) == 3 and ca == cb
    bits = _np(blob)
    want = {R8.encode(np.ascontiguousarray(bits[:, :, x:x + 256].transpose(1, 0, 2, 3, 4)).reshape(2 * L, -1, H * D),
                      L, H, D, 3) for x in range(0, T, 256)}
    assert set(cb.values()) == want
    a.close(), b.close()
    if tier == "disk":                                           # a new engine on the same directory finds every chunk
        c = _engine(path("b"), lserde="lossless")
        kv, mask = c.retrieve(toks)
        assert int(mask.sum()) == T and torch.equal(_u8(_stack(kv)), _u8(blob))
        c.close()


@pytest.mark.parametrize("where", ["host", "lm"])
def test_mla_latent_fp8(where, server):
    L, T, D = 3, 520, 576
    lat = _kv((L, T, D), torch.float8_e4m3fn, 53, "scaled")
    toks = _toks(T, 6)
    mk = (lambda: _engine("cpu", lserde="lossless", mla=True, cs=512)) if where == "host" else \
        (lambda: _engine(remote=server, rserde="lossless", mla=True, cs=512))
    m = mk()
    m.store(toks, tuple(lat[l] for l in range(L)))
    kv, mask = (m if where == "host" else mk()).retrieve(toks)
    assert int(mask.sum()) == T and torch.equal(torch.stack([_u8(x) for x in kv]), _u8(lat))
    m.close()


@pytest.mark.parametrize("W,Wd", [(2, 1), (1, 2)])
def test_reshard_lossless_fp8(W, Wd, server):
    Hg, T, L, D = 8, 600, 3, 64
    blob = _kv((L, 2, T, Hg, D), torch.float8_e4m3fn, 10 * W + Wd, "scaled")
    toks = _toks(T, 9)
    engines = []
    for r in range(W):
        e = _engine(remote=server, rserde="lossless", W=W, r=r)
        a, b = r * Hg // W, (r + 1) * Hg // W
        e.store(toks, _pairs(blob[:, :, :, a:b]))
        engines.append(e)
    for rd in range(Wd):
        e = _engine(remote=server, rserde="lossless", W=Wd, r=rd, reshard_world_sizes=[W], reshard_lossless=True)
        a, b = rd * Hg // Wd, (rd + 1) * Hg // Wd
        kv, mask = e.retrieve(toks)
        assert int(mask.sum()) == T and kv[0][0].dtype == torch.float8_e4m3fn
        assert torch.equal(_u8(_stack(kv)), _u8(blob[:, :, :, a:b]))
        engines.append(e)
    for e in engines:
        e.close()


def test_cachegen_tiers_refuse_fp8(tmp_path):
    e = _engine("cpu", lserde="cachegen")
    kv = _pairs(_kv((2, 2, 64, 2, 32), torch.float8_e4m3fn, 1))
    with pytest.raises(TypeError, match="local_serde: lossless"):
        e.store(torch.arange(64), kv)
    e.close()
