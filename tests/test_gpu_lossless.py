"""GPU: the lossless codec (B2KV versions 5 and 6) and the `lossless` remote serde.

Device containers equal the numpy statement (tests/lossless_ref.py) byte for byte for every source kind (blob, tuple,
huggingface strides, paged), both dtypes, (K, V) and latent KV, tok_begin > 0, ragged last chunks and many chunks per
call; decodes are bit-exact into every destination kind and write nothing outside the call's rows; a seeded set of
damaged containers is refused or flagged.  Then LMCacheEngine round trips through a local lm:// server: blob and paged
store / retrieve, suffix masks, a retrieve-only replica, a hybrid engine, huggingface fp16, MLA, and CacheGen and lossless
engines that share one server (a clean miss both ways)."""
import ctypes

import numpy as np
import pytest
import torch

import lossless_ref as R

pytestmark = pytest.mark.gpu
MODEL = "lmsys/longchat-7b-16k"
SENT = -21555


def _kv(shape, dtype, seed, kind="normal"):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, device="cuda", generator=g)
    if kind == "scaled":       # per-channel scales: more exponents per plane
        x = x * torch.exp(2 * torch.randn(shape[-1], device="cuda", generator=g))
    if kind == "bits":         # every bit pattern: NaNs, infinities, subnormals
        return torch.randint(-32768, 32768, shape, device="cuda", generator=g, dtype=torch.int32).to(torch.int16).view(dtype)
    return x.to(dtype)


def _np(x):
    return x.contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def _codec():
    from lmcache_b200.codec import LosslessCodec
    return LosslessCodec()


def _encode(codec, view, tok_begin, n_tokens, cs):
    return codec.encode_to_host(view, tok_begin, n_tokens, cs)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("H", [1, 8, 32])
def test_blob_matches_spec_and_roundtrips(dtype, H):
    from lmcache_b200.codec import KvView
    L, T, D, cs, t0 = 3, 700, 128 if H < 32 else 32, 256, 37
    blob = _kv((L, 2, T, H, D), dtype, H, "scaled")
    codec = _codec()
    conts = _encode(codec, KvView.from_blob(blob, "vllm"), t0, T - t0, cs)
    assert len(conts) == 3 and [c[4] for c in conts] == [5, 5, 5]
    bits = _np(blob)
    for j, c in enumerate(conts):
        a, b = t0 + j * cs, min(T, t0 + (j + 1) * cs)
        want = R.encode(R.planes_of_blob(bits[:, :, a:b]), L, H, D, 0 if dtype == torch.bfloat16 else 1)
        assert c == want, f"container {j} differs from the spec"
    # decode into a destination with sentinel rows around the call's tokens
    out = torch.full((L, 2, T + 8, H, D), SENT, dtype=torch.int16, device="cuda").view(dtype)
    codec.decode(conts, KvView.from_blob(out, "vllm"), [4 + j * cs for j in range(len(conts))])
    torch.cuda.synchronize()
    assert codec.decode_status() == [0, 0, 0]
    got = _np(out)
    assert np.array_equal(got[:, :, 4:4 + T - t0], bits[:, :, t0:])
    assert (got[:, :, :4].view(np.int16) == SENT).all() and (got[:, :, 4 + T - t0:].view(np.int16) == SENT).all()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_every_source_and_destination_kind(dtype):
    from lmcache_b200.codec import KvView
    L, T, H, D, cs = 2, 300, 4, 64, 128
    dt = 0 if dtype == torch.bfloat16 else 1
    blob = _kv((L, 2, T, H, D), dtype, 7, "bits")
    bits = _np(blob)
    codec = _codec()
    ref = [R.encode(R.planes_of_blob(bits[:, :, a:a + cs]), L, H, D, dt) for a in range(0, T, cs)]
    # tuple of per-layer tensors
    kv = tuple((blob[l, 0].clone(), blob[l, 1].clone()) for l in range(L))
    assert _encode(codec, KvView.from_tuple(kv, "vllm"), 0, T, cs) == ref
    # huggingface strides [L, 2, H, T, D]
    hf = blob.permute(0, 1, 3, 2, 4).contiguous()
    assert _encode(codec, KvView.from_blob(hf, "huggingface"), 0, T, cs) == ref
    # paged: a shuffled slot mapping into [num_blocks, 16, H, D] caches
    slots = torch.randperm(400, generator=torch.Generator().manual_seed(3))[:T].cuda()
    caches = [(torch.zeros(25, 16, H, D, dtype=dtype, device="cuda"), torch.zeros(25, 16, H, D, dtype=dtype, device="cuda"))
              for _ in range(L)]
    for l, (k, v) in enumerate(caches):
        k.view(-1, H, D)[slots] = blob[l, 0]
        v.view(-1, H, D)[slots] = blob[l, 1]
    assert _encode(codec, KvView.from_paged(caches, slots), 0, T, cs) == ref
    # decode into each kind
    out_hf = torch.full_like(hf.view(torch.int16), SENT).view(dtype)
    codec.decode(ref, KvView.from_blob(out_hf, "huggingface"), [0, cs, 2 * cs])
    pc = [(torch.full_like(k.view(torch.int16), SENT).view(dtype), torch.full_like(v.view(torch.int16), SENT).view(dtype))
          for k, v in caches]
    codec.decode(ref, KvView.from_paged(pc, slots), [0, cs, 2 * cs])
    out_t = tuple((torch.empty_like(a), torch.empty_like(b)) for a, b in kv)
    codec.decode(ref, KvView.from_tuple(out_t, "vllm"), [0, cs, 2 * cs])
    torch.cuda.synchronize()
    assert np.array_equal(_np(out_hf), _np(hf))
    for (k, v), (k0, v0), (tk, tv) in zip(pc, caches, out_t):
        kk, vv = k.view(-1, H, D), v.view(-1, H, D)
        assert torch.equal(kk[slots].view(torch.int16), k0.view(-1, H, D)[slots].view(torch.int16))
        assert torch.equal(vv[slots].view(torch.int16), v0.view(-1, H, D)[slots].view(torch.int16))
        rest = torch.ones(400, dtype=torch.bool, device="cuda")
        rest[slots] = False
        assert (kk[rest].view(torch.int16) == SENT).all() and (vv[rest].view(torch.int16) == SENT).all()
    for l in range(L):
        assert torch.equal(out_t[l][0].view(torch.int16), blob[l, 0].view(torch.int16))
        assert torch.equal(out_t[l][1].view(torch.int16), blob[l, 1].view(torch.int16))
    # a lossless codec does not cast: the other 16-bit dtype is refused
    other = torch.empty_like(blob, dtype=torch.float16 if dtype == torch.bfloat16 else torch.bfloat16)
    with pytest.raises(ValueError, match="own dtype"):
        codec.decode(ref, KvView.from_blob(other, "vllm"), [0, cs, 2 * cs])


def test_latent_kv_version6():
    from lmcache_b200.codec import KvView
    L, T, D, cs = 5, 520, 576, 256
    lat = _kv((L, T, D), torch.bfloat16, 11, "scaled")
    codec = _codec()
    conts = _encode(codec, KvView.from_blob(lat, "vllm"), 0, T, cs)
    bits = _np(lat)
    for j, c in enumerate(conts):
        assert c[4] == 6
        assert c == R.encode(bits[:, j * cs:(j + 1) * cs], L, 1, D, 0, latent=True)
    out = torch.empty_like(lat)
    codec.decode(conts, KvView.from_blob(out, "vllm"), [0, cs, 2 * cs])
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), lat.view(torch.int16))
    kvdst = torch.empty((L, 2, T, 1, D), dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError):
        codec.decode(conts, KvView.from_blob(kvdst, "vllm"), [0, cs, 2 * cs])


def test_single_symbol_and_many_chunks():
    from lmcache_b200.codec import KvView
    L, T, H, D, cs = 2, 4096 + 100, 2, 64, 1024
    x = torch.full((L, 2, T, H, D), 1.5, dtype=torch.bfloat16, device="cuda")        # one symbol per plane: f = 4096
    codec = _codec()
    conts = _encode(codec, KvView.from_blob(x, "vllm"), 0, T, cs)
    assert len(conts) == 5
    for j, c in enumerate(conts):
        assert c == R.encode(R.planes_of_blob(_np(x)[:, :, j * cs:(j + 1) * cs]), L, H, D, 0)
    y = _kv((1, 2, 4096, 1, 16), torch.float16, 4, "bits")                     # t = 4096, incompressible
    c = _encode(codec, KvView.from_blob(y, "vllm"), 0, 4096, 4096)[0]
    assert c == R.encode(R.planes_of_blob(_np(y)), 1, 1, 16, 1)
    out = torch.empty_like(y)
    codec.decode([c], KvView.from_blob(out, "vllm"), [0])
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), y.view(torch.int16))


def test_damaged_containers_are_refused_or_flagged():
    from lmcache_b200.codec import KvView
    L, T, H, D = 2, 96, 2, 64
    x = _kv((L, 2, T, H, D), torch.bfloat16, 21, "scaled")
    codec = _codec()
    good = _encode(codec, KvView.from_blob(x, "vllm"), 0, T, T)[0]
    lo = R.layout(2 * L, H * D, T)
    rng = np.random.default_rng(1234)
    outcomes = {"refused": 0, "flagged": 0}
    for trial in range(40):
        b = bytearray(good)
        region = trial % 4
        lo_b, hi_b = [(0, 64), (lo["off_freq"], lo["off_lens"]), (lo["off_lens"], lo["off_raw"]),
                      (lo["off_payload"], len(good))][region]
        for _ in range(1 + trial % 3):
            b[int(rng.integers(lo_b, hi_b))] ^= int(rng.integers(1, 256))
        out = torch.full((L, 2, T + 32, H, D), SENT, dtype=torch.int16, device="cuda").view(torch.bfloat16)
        try:
            codec.decode([bytes(b)], KvView.from_blob(out, "vllm"), [16])
            st = codec.decode_status()
        except ValueError:
            outcomes["refused"] += 1
            st = None
        got = out.view(torch.int16)
        assert (got[:, :, :16] == SENT).all() and (got[:, :, 16 + T:] == SENT).all(), "write outside the call's rows"
        if st is None:
            continue
        same = torch.equal(got[:, :, 16:16 + T], x.view(torch.int16))
        if st[0] != 0:
            outcomes["flagged"] += 1
        else:
            assert same, f"trial {trial}: damage neither refused nor flagged, and the KV differs"
    assert outcomes["refused"] > 0 and outcomes["flagged"] > 0


# ------------------------------------------------------------------------------------------ engines over lm://
@pytest.fixture
def server():
    from lmcache_b200 import _native as N
    h = ctypes.c_void_p()
    N.check(N.lib().b200kv_lm_server_start(b"127.0.0.1", 0, ctypes.byref(h)))
    yield f"lm://127.0.0.1:{N.lib().b200kv_lm_server_port(h)}", h
    N.lib().b200kv_lm_server_stop(h)


def _engine(url, serde="lossless", fmt="vllm", local=None, cs=256, mla=False, dtype="bfloat16"):
    from lmcache_b200.cache_engine import LMCacheEngine
    from lmcache_b200.config import LMCacheEngineConfig, LMCacheEngineMetadata
    cfg = LMCacheEngineConfig(cs, local, url, serde, False, False)
    return LMCacheEngine(cfg, LMCacheEngineMetadata(MODEL, 1, 0, fmt, dtype, use_mla=mla))


def _pairs(blob, fmt="vllm"):
    return tuple((blob[l, 0], blob[l, 1]) for l in range(blob.shape[0]))


def _stack(kv):
    return torch.stack([torch.stack([k, v]) for k, v in kv])


def test_engine_store_retrieve_replica_and_mask(server):
    L, T, H, D = 4, 700, 8, 128
    blob = _kv((L, 2, T, H, D), torch.bfloat16, 31, "scaled")
    toks = torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(1))
    w = _engine(server[0])
    w.store(toks, _pairs(blob))
    kv, mask = w.retrieve(toks)
    assert int(mask.sum()) == T and torch.equal(_stack(kv).view(torch.int16), blob.view(torch.int16))
    r = _engine(server[0])                      # a retrieve-only replica learns the geometry from the first header
    kv, mask = r.retrieve(toks)
    assert int(mask.sum()) == T and kv[0][0].dtype == torch.bfloat16
    assert torch.equal(_stack(kv).view(torch.int16), blob.view(torch.int16))
    m = torch.ones(T, dtype=torch.bool)
    m[:300] = False
    kv, mask = r.retrieve(toks, m)
    assert int(mask.sum()) == T - 300 and torch.equal(_stack(kv).view(torch.int16), blob[:, :, 300:].view(torch.int16))
    # a longer prompt: its whole chunks that were stored are served; the stored ragged tail chunk hashes differently
    toks2 = torch.cat([toks, torch.arange(100)])
    kv, mask = r.retrieve(toks2)
    assert int(mask.sum()) == 512 and torch.equal(_stack(kv).view(torch.int16), blob[:, :, :512].view(torch.int16))
    w.close(), r.close()


def test_engine_paged_and_nonblocking(server):
    L, T, H, D = 3, 600, 4, 64
    blob = _kv((L, 2, T, H, D), torch.float16, 41, "bits")
    toks = torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(2))
    slots = torch.randperm(1024, generator=torch.Generator().manual_seed(5))[:T].cuda()
    caches = [(torch.zeros(64, 16, H, D, dtype=torch.float16, device="cuda"),
               torch.zeros(64, 16, H, D, dtype=torch.float16, device="cuda")) for _ in range(L)]
    for l, (k, v) in enumerate(caches):
        k.view(-1, H, D)[slots] = blob[l, 0]
        v.view(-1, H, D)[slots] = blob[l, 1]
    e = _engine(server[0], dtype="float16")
    e.store_paged(toks, caches, slots, blocking=False)
    for k, v in caches:                          # the store has read the caches in stream order
        k.fill_(0)
        v.fill_(0)
    e.engine_.drain()
    dst = [(torch.full_like(k.view(torch.int16), SENT).view(torch.float16),
            torch.full_like(v.view(torch.int16), SENT).view(torch.float16)) for k, v in caches]
    mask = e.retrieve_paged(toks, dst, slots)
    torch.cuda.synchronize()
    assert int(mask.sum()) == T
    for l, (k, v) in enumerate(dst):
        assert torch.equal(k.view(-1, H, D)[slots].view(torch.int16), blob[l, 0].view(torch.int16))
        assert torch.equal(v.view(-1, H, D)[slots].view(torch.int16), blob[l, 1].view(torch.int16))
    e.close()


def test_engine_huggingface_fp16_hybrid_and_mla(server):
    L, T, H, D = 2, 300, 4, 64
    hf = _kv((L, 2, H, T, D), torch.float16, 51, "scaled")
    toks = torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(3))
    e = _engine(server[0], fmt="huggingface", dtype="float16")
    e.store(toks, _pairs(hf))
    r = _engine(server[0], fmt="huggingface", dtype="float16")
    kv, mask = r.retrieve(toks)
    assert int(mask.sum()) == T and kv[0][0].dtype == torch.float16
    assert torch.equal(_stack(kv).view(torch.int16), hf.view(torch.int16))
    e.close(), r.close()
    # hybrid: a raw host tier in front of the lossless remote tier; a second engine reads the remote half
    blob = _kv((L, 2, T, H, D), torch.bfloat16, 52, "scaled")
    toks = torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(4))
    h = _engine(server[0], local="cpu")
    h.store(toks, _pairs(blob))
    h2 = _engine(server[0], local="cpu")
    kv, mask = h2.retrieve(toks)
    assert int(mask.sum()) == T and torch.equal(_stack(kv).view(torch.int16), blob.view(torch.int16))
    h.close(), h2.close()
    # MLA: version-6 containers, one key for every rank
    lat = _kv((3, 520, 576), torch.bfloat16, 53, "scaled")
    toks = torch.randint(0, 32000, (520,), generator=torch.Generator().manual_seed(6))
    m = _engine(server[0], mla=True, cs=512)
    m.store(toks, tuple(lat[l] for l in range(3)))
    m2 = _engine(server[0], mla=True, cs=512)
    kv, mask = m2.retrieve(toks)
    assert int(mask.sum()) == 520 and torch.equal(torch.stack(kv).view(torch.int16), lat.view(torch.int16))
    m.close(), m2.close()


def test_engine_refuses_wide_dtype(server):
    L, T, H, D = 2, 64, 2, 32
    e = _engine(server[0])
    kv = tuple((torch.zeros(T, H, D, device="cuda"), torch.zeros(T, H, D, device="cuda")) for _ in range(L))
    with pytest.raises(TypeError, match="bfloat16 and float16"):
        e.store(torch.arange(T), kv)
    e.close()


def test_cachegen_and_lossless_engines_share_a_server(server):
    L, T, H, D = 2, 512, 4, 64
    blob = _kv((L, 2, T, H, D), torch.bfloat16, 61, "scaled")
    toks = torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(7))
    toks_b = torch.randint(0, 32000, (T,), generator=torch.Generator().manual_seed(8))
    cg = _engine(server[0], serde="cachegen")
    ll = _engine(server[0], serde="lossless")
    cg.store(toks, _pairs(blob))
    ll.store(toks_b, _pairs(blob))
    # each engine meets the other's container under a key it asks for: a clean miss, nothing written
    out_ll = _engine(server[0], serde="lossless")
    kv, mask = out_ll.retrieve(toks)
    assert int(mask.sum()) == 0 and len(kv) == 0
    out_cg = _engine(server[0], serde="cachegen")
    kv, mask = out_cg.retrieve(toks_b)
    assert int(mask.sum()) == 0 and len(kv) == 0
    # with a known geometry the miss writes nothing into the destination
    slots = torch.arange(T, device="cuda")
    dst = [(torch.full((T, H, D), SENT, dtype=torch.int16, device="cuda").view(torch.bfloat16),
            torch.full((T, H, D), SENT, dtype=torch.int16, device="cuda").view(torch.bfloat16)) for _ in range(L)]
    ll.retrieve(toks_b)                          # its own chunks: a hit (sets nothing up beyond the geometry)
    assert int(ll.retrieve_paged(toks, dst, slots).sum()) == 0
    assert int(cg.retrieve_paged(toks_b, dst, slots).sum()) == 0
    assert all((k.view(torch.int16) == SENT).all() and (v.view(torch.int16) == SENT).all() for k, v in dst)
    # and each still reads its own
    kv, mask = out_ll.retrieve(toks_b)
    assert int(mask.sum()) == T and torch.equal(_stack(kv).view(torch.int16), blob.view(torch.int16))
    for e in (cg, ll, out_ll, out_cg):
        e.close()
