"""GPU parity tests of the CUDA codec, through the C ABI (ctypes) and the serde plugins.

Bar: every container section (CDF, maxima, stream lengths, payload bytes) bit-identical to the oracle; decoded KV
bit-identical to the reference goldens (the north-star tolerance is 1e-3 max-abs; we hold 0)."""
import numpy as np
import pytest
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu
MODEL = "lmsys/longchat-7b-16k"


def _bits_to_tensor(bits: np.ndarray, dt: int) -> torch.Tensor:
    return torch.from_numpy(bits.view(np.int16).copy()).view(torch.bfloat16 if dt == 0 else torch.float16)


def _tensor_bits(t: torch.Tensor) -> np.ndarray:
    return t.contiguous().cpu().view(torch.int16).numpy().view(np.uint16)


def _eq_nan(a: np.ndarray, b: np.ndarray, dt: int) -> bool:
    """bit equality, except that any NaN matches any NaN (payloads differ between x86 and the GPU)."""
    if np.array_equal(a, b):
        return True
    f = (lambda u: (u.astype(np.uint32) << 16).view(np.float32)) if dt == 0 else (lambda u: u.view(np.float16))
    fa, fb = f(a), f(b)
    both_nan = np.isnan(fa) & np.isnan(fb)
    return bool(np.all((a == b) | both_nan))


@pytest.fixture(scope="module", params=["rans_compact", "rans", "ac"])
def codec(request):
    """all container formats: version 3 (rANS + symbol counts, the default), 2 (rANS + CDF rows), 1 (arithmetic coder)"""
    from lmcache_b200.codec import CacheGenCodec
    return CacheGenCodec(MODEL, coder=request.param)


def _oenc(codec, *args):
    """the oracle's encode with the coder under test (the compact container holds chunks of <= 256 tokens only)"""
    return O.encode_chunk(*args, coder=codec.coder_for(args[0].shape[2]))


def _sections(raw: bytes, L, H, D, t):
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import parse_header
    from lmcache_b200.codec import container_layout_of
    hd = parse_header(raw)
    assert (hd.L, hd.H, hd.D, hd.ntokens) == (L, H, D, t)
    lo = container_layout_of(hd)
    C = H * D
    G = (t + 255) // 256
    a = np.frombuffer(raw, np.uint8)
    payload = a[lo.off_payload: lo.off_payload + hd.payload_bytes]
    if hd.version == 3:
        # compact container: every stream carries its histogram in place of a CDF row.  Unpacked with the ORACLE's
        # parser; the CDF is rebuilt with the oracle's arithmetic (callers compare it with the reference-made goldens)
        kb, vb = O.make_bins(MODEL)
        nb = O.nb_map(kb, vb, L)
        assert list(a[lo.off_cdf: lo.off_cdf + 2 * L]) == nb == hd.nb
        half = a[lo.off_lengths: lo.off_lengths + 2 * L * C].reshape(2 * L, C)
        cnt, ln, payload = O.v3_unpack(payload, half, nb, t)
        assert np.all(cnt.sum(axis=2) == t)
        cdf = O.cdf_from_counts(cnt, t)
        lengths = ln.reshape(1, 2 * L, C)
    else:
        cdf = a[lo.off_cdf: lo.off_cdf + 2 * L * C * 33 * 2].view(np.int16).reshape(2 * L, C, 33)
        lengths = a[lo.off_lengths: lo.off_lengths + G * 2 * L * C * 4].view(np.int32).reshape(G, 2 * L, C)
    maxes = a[lo.off_maxes: lo.off_maxes + 2 * L * t * 2].view(np.uint16).reshape(2, L, t)
    assert hd.total_bytes == lo.off_payload + hd.payload_bytes == len(raw)
    return cdf, maxes, lengths, payload


GOLDEN_CASES = ["bf16_t1", "bf16_t7_L32", "bf16_t40", "bf16_t236", "bf16_t256", "bf16_t300", "bf16_uniform_t16",
                "fp16_t40", "fp16_uniform_t128"]


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_encode_container_bit_exact_vs_oracle_and_goldens(codec, golden, name):
    from lmcache_b200.codec import KvView
    x = golden[f"{name}/x"]
    dt = int(golden[f"{name}/dtype"][0])
    L, _, t, H, D = x.shape
    kv = _bits_to_tensor(x, dt).cuda()
    raw = codec.encode_to_host(KvView.from_blob(kv, "vllm"), 0, t, t)[0]
    cdf, maxes, lengths, payload = _sections(raw, L, H, D, t)
    # against vectors made by the reference's own functions
    assert np.array_equal(cdf, golden[f"{name}/cdf"])
    assert np.array_equal(maxes[0], golden[f"{name}/max_k"].reshape(L, t))
    assert np.array_equal(maxes[1], golden[f"{name}/max_v"].reshape(L, t))
    # against the oracle's bitstream
    kb, vb = golden["key_bins"], golden["value_bins"]
    enc = _oenc(codec, x.reshape(L, 2, t, H * D), dt, kb, vb)
    assert np.array_equal(np.stack([ln for _, ln, _ in enc["groups"]]), lengths)
    assert np.array_equal(np.concatenate([b for b, _, _ in enc["groups"]]), payload)
    if raw[4] == 3:     # the packed streams (histogram headers included) and their lengths, byte for byte
        from lmcache_b200.codec import container_layout_of, parse_header
        lo = container_layout_of(parse_header(raw))
        (b0, ln0, _), = enc["groups"]
        pl, half = O.v3_pack(enc["counts"], O.nb_map(kb, vb, L), ln0, b0)
        assert bytes(raw[lo.off_payload:]) == pl.tobytes()
        assert bytes(raw[lo.off_lengths:lo.off_lengths + half.size]) == half.tobytes()


@pytest.mark.parametrize("name", GOLDEN_CASES)
@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
def test_decode_bit_exact_vs_reference_goldens(codec, golden, name, fmt):
    from lmcache_b200.codec import KvView
    x = golden[f"{name}/x"]
    dt = int(golden[f"{name}/dtype"][0])
    L, _, t, H, D = x.shape
    kv = _bits_to_tensor(x, dt).cuda()
    raw = codec.encode_to_host(KvView.from_blob(kv, "vllm"), 0, t, t)[0]
    if fmt == "vllm":
        out = torch.zeros((L, 2, t, H, D), dtype=torch.bfloat16, device="cuda")
        want = golden[f"{name}/deq_vllm_bf16"]
    else:
        out = torch.zeros((L, 2, H, t, D), dtype=torch.float16, device="cuda")
        want = golden[f"{name}/deq_hf_fp16"]
    codec.decode([raw], KvView.from_blob(out, fmt), [0])
    torch.cuda.synchronize()
    assert _eq_nan(_tensor_bits(out), want, 0 if fmt == "vllm" else 1)


@pytest.mark.parametrize("name", ["bf16_t300", "bf16_t236", "bf16_t256"])
def test_oracle_made_container_decodes_on_gpu(codec, golden, name):
    """Decoder accepts a container assembled entirely on the CPU by the oracle (wire compatibility both ways)."""
    from lmcache_b200.codec import KvView
    from lmcache_b200.storage_backend.serde.cachegen_basics import CacheGenGPUBytestream, CacheGenGPUEncoderOutput
    x = golden[f"{name}/x"]
    L, _, t, H, D = x.shape
    enc = _oenc(codec, x.reshape(L, 2, t, H * D), 0, golden["key_bins"], golden["value_bins"])
    mk = torch.from_numpy(enc["maxes"][0].view(np.int16)).view(torch.bfloat16).reshape(L, t, 1)
    mv = torch.from_numpy(enc["maxes"][1].view(np.int16)).view(torch.bfloat16).reshape(L, t, 1)
    raw = CacheGenGPUEncoderOutput(
        [CacheGenGPUBytestream(torch.from_numpy(b), torch.from_numpy(ln), g) for b, ln, g in enc["groups"]],
        torch.from_numpy(enc["cdf"]), mk, mv, H, D, codec.coder_for(t), torch.from_numpy(O.counts(enc["sym"]).astype(np.int32)),
        O.nb_map(golden["key_bins"], golden["value_bins"], L)).to_bytes()
    assert raw[4] == codec.coder_for(t) + 1
    out = torch.zeros((L, 2, t, H, D), dtype=torch.bfloat16, device="cuda")
    codec.decode([raw], KvView.from_blob(out, "vllm"), [0])
    torch.cuda.synchronize()
    assert np.array_equal(_tensor_bits(out), golden[f"{name}/deq_vllm_bf16"])


@pytest.mark.parametrize("T,cs", [(600, 256), (256, 64), (700, 300), (100, 256), (1030, 512)])
@pytest.mark.parametrize("source", ["blob", "tuple", "hf_blob"])
def test_multichunk_ragged_vs_oracle(codec, T, cs, source):
    """Several chunks per launch incl. a ragged tail, chunks > 256 tokens (split kernels), tuple and hf sources."""
    from lmcache_b200.codec import KvView
    L, H, D = 6, 2, 72                      # C = 144: one full tile + a partial one
    C = H * D
    bits = O.synth_kv_bits(L, T, C, seed=T + cs)
    kv = _bits_to_tensor(bits, 0).reshape(L, 2, T, H, D).cuda()
    if source == "blob":
        view = KvView.from_blob(kv, "vllm")
    elif source == "hf_blob":
        view = KvView.from_blob(kv.permute(0, 1, 3, 2, 4).contiguous(), "huggingface")
    else:
        view = KvView.from_tuple(tuple((kv[l, 0].clone(), kv[l, 1].clone()) for l in range(L)), "vllm")
    raws = codec.encode_to_host(view, 0, T, cs)
    kb, vb = O.make_bins(MODEL)
    n_chunks = (T + cs - 1) // cs
    assert len(raws) == n_chunks
    out = torch.zeros((L, 2, T, H, D), dtype=torch.bfloat16, device="cuda")
    offs = []
    for j, raw in enumerate(raws):
        t0, t1 = j * cs, min(T, (j + 1) * cs)
        enc = _oenc(codec, bits[:, :, t0:t1], 0, kb, vb)
        cdf, maxes, lengths, payload = _sections(raw, L, H, D, t1 - t0)
        assert np.array_equal(cdf, enc["cdf"]), j
        assert np.array_equal(maxes, enc["maxes"]), j
        assert np.array_equal(lengths, np.stack([ln for _, ln, _ in enc["groups"]])), j
        assert np.array_equal(payload, np.concatenate([b for b, _, _ in enc["groups"]])), j
        offs.append(t0)
    codec.decode(raws, KvView.from_blob(out, "vllm"), offs)
    torch.cuda.synchronize()
    want = np.concatenate([O.decode_chunk(_oenc(codec, bits[:, :, j * cs:min(T, (j + 1) * cs)], 0, kb, vb), 0, kb, vb, 0)
                           for j in range(n_chunks)], axis=2)
    assert np.array_equal(_tensor_bits(out).reshape(L, 2, T, C), want)


@pytest.mark.parametrize("T,cs,dt", [(600, 256, 0), (300, 64, 1), (700, 512, 0)])
def test_paged_kv_cache_in_place(codec, T, cs, dt):
    """vLLM-style paged KV cache + slot_mapping (KvView.from_paged): encoding the scattered rows gives the very
    container the contiguous gather gives, and decoding scatters straight into the cache rows -- no pack / unpack
    copies (SURVEY 8f rank 3).  Fused (chunk <= 256) and split (chunk 512) kernels, bf16 and fp16, ragged tails."""
    from lmcache_b200.codec import KvView
    L, H, D, bs, nblocks = 4, 3, 80, 16, 64               # C = 240: a full tile + a partial one
    C = H * D
    g = torch.Generator().manual_seed(T + cs)
    slots = torch.randperm(nblocks * bs, generator=g)[:T].to(torch.int64)          # token i -> cache row slots[i]
    bits = O.synth_kv_bits(L, T, C, seed=5 * T + cs)
    tdt = torch.bfloat16 if dt == 0 else torch.float16
    dense = _bits_to_tensor(bits, 0).float().to(tdt).reshape(L, 2, T, H, D).cuda()
    bits = _tensor_bits(dense).reshape(L, 2, T, C)
    caches = []
    for l in range(L):
        k = torch.full((nblocks, bs, H, D), 7.0, dtype=tdt, device="cuda")
        v = torch.full((nblocks, bs, H, D), -7.0, dtype=tdt, device="cuda")
        k.view(-1, H, D)[slots.cuda()] = dense[l, 0]
        v.view(-1, H, D)[slots.cuda()] = dense[l, 1]
        caches.append((k, v))
    paged = KvView.from_paged(caches, slots.cuda())
    assert paged.ntokens == T
    raws_paged = codec.encode_to_host(paged, 0, T, cs)
    raws_dense = codec.encode_to_host(KvView.from_blob(dense, "vllm"), 0, T, cs)
    for j, (a, b) in enumerate(zip(raws_paged, raws_dense)):
        tj = min(cs, T - j * cs)
        for u, v in zip(_sections(a, L, H, D, tj), _sections(b, L, H, D, tj)):
            assert np.array_equal(u, v), j
    # and against the oracle
    kb, vb = O.make_bins(MODEL)
    n_chunks = (T + cs - 1) // cs
    for j, raw in enumerate(raws_paged):
        t0, t1 = j * cs, min(T, (j + 1) * cs)
        enc = _oenc(codec, bits[:, :, t0:t1], dt, kb, vb)
        cdf, maxes, lengths, payload = _sections(raw, L, H, D, t1 - t0)
        assert np.array_equal(cdf, enc["cdf"]) and np.array_equal(maxes, enc["maxes"]), j
        assert np.array_equal(lengths, np.stack([ln for _, ln, _ in enc["groups"]])), j
        assert np.array_equal(payload, np.concatenate([b_ for b_, _, _ in enc["groups"]])), j
    # decode into a fresh paged cache through a different mapping; untouched rows must stay untouched
    slots2 = torch.randperm(nblocks * bs, generator=g)[:T].to(torch.int64)
    caches2 = [(torch.full((nblocks, bs, H, D), 3.0, dtype=tdt, device="cuda"),
                torch.full((nblocks, bs, H, D), 3.0, dtype=tdt, device="cuda")) for _ in range(L)]
    codec.decode(raws_paged, KvView.from_paged(caches2, slots2.cuda()), [j * cs for j in range(n_chunks)])
    torch.cuda.synchronize()
    want = np.concatenate([O.decode_chunk(_oenc(codec, bits[:, :, j * cs:min(T, (j + 1) * cs)], dt, kb, vb), dt, kb, vb, dt)
                           for j in range(n_chunks)], axis=2)                     # [L,2,T,C]
    mask = torch.ones(nblocks * bs, dtype=torch.bool)
    mask[slots2] = False
    for l in range(L):
        for kvi in range(2):
            flat = caches2[l][kvi].view(-1, H, D)
            got = _tensor_bits(flat[slots2.cuda()]).reshape(T, C)
            assert np.array_equal(got, want[l, kvi]), (l, kvi)
            assert bool((flat[mask.cuda()] == 3.0).all()), "decode wrote outside the mapped rows"


def test_split_mode_oversized_tiles_take_the_direct_path(codec):
    """One 2048-token chunk (CDF over the whole chunk): seven groups of near-constant values and one group of values
    spread over all bins.  That group's symbols are rare chunk-wide (~10 bits each), so its tiles exceed the
    compaction kernel's shared-memory stage and are written by the per-thread direct path; the rest is staged.
    Container and decoded values must equal the oracle's either way."""
    from lmcache_b200.codec import KvView
    L, H, D, T = 2, 1, 128, 2048
    C = H * D
    rng = np.random.default_rng(77)
    x = np.zeros((L, 2, T, C), np.float32)
    x[:, :, :, 0] = 8.0                                            # row max in every row: the scale is fixed
    x[:, :, 768:1024, 1:] = rng.uniform(-8.0, 8.0, size=(L, 2, 256, C - 1)).astype(np.float32)
    x[:, :, :768, 1:] += rng.choice([0.0, 0.6], size=(L, 2, 768, C - 1), p=[0.95, 0.05]).astype(np.float32)
    bits = O.f32_to_bf16_bits(x)
    kv = _bits_to_tensor(bits, 0).reshape(L, 2, T, H, D).cuda()
    raw = codec.encode_to_host(KvView.from_blob(kv, "vllm"), 0, T, T)[0]
    kb, vb = O.make_bins(MODEL)
    enc = _oenc(codec, bits, 0, kb, vb)
    cdf, maxes, lengths, payload = _sections(raw, L, H, D, T)
    assert np.array_equal(cdf, enc["cdf"]) and np.array_equal(maxes, enc["maxes"])
    want_len = np.stack([ln for _, ln, _ in enc["groups"]])
    assert np.array_equal(lengths, want_len)
    assert int(want_len[3].reshape(-1, 128).sum(axis=1).max()) > 128 * 196 + 32      # group 3's tiles really are oversized
    assert np.array_equal(payload, np.concatenate([b for b, _, _ in enc["groups"]]))
    out = torch.empty_like(kv)
    codec.decode([raw], KvView.from_blob(out, "vllm"), [0])
    torch.cuda.synchronize()
    assert np.array_equal(_tensor_bits(out).reshape(L, 2, T, C), O.decode_chunk(enc, 0, kb, vb, 0))


def test_tok_begin_and_device_container_decode(codec):
    """Encoding a token sub-range, and decoding straight from the device staging buffer (no host hop)."""
    from lmcache_b200.codec import KvView
    L, H, D, T = 4, 1, 128, 512
    bits = O.synth_kv_bits(L, T, H * D, seed=11)
    kv = _bits_to_tensor(bits, 0).reshape(L, 2, T, H, D).cuda()
    batch = codec.encode(KvView.from_blob(kv, "vllm"), 128, 256, 256)
    dev_container = batch.container(0).clone()
    out = torch.zeros((L, 2, 256, H, D), dtype=torch.bfloat16, device="cuda")
    codec.decode([dev_container], KvView.from_blob(out, "vllm"), [0])
    torch.cuda.synchronize()
    kb, vb = O.make_bins(MODEL)
    want = O.decode_chunk(_oenc(codec, bits[:, :, 128:384], 0, kb, vb), 0, kb, vb, 0)
    assert np.array_equal(_tensor_bits(out).reshape(L, 2, 256, H * D), want)


def test_full_width_chunk_vs_torch_reference_chain(codec):
    """C = 4096 (Llama-7B width), t = 256: decoded KV vs the reference's torch op chain run on the same GPU
    (size-independent check; the C oracle is used at small sizes)."""
    import ref_torch
    from lmcache_b200.codec import KvView
    L, H, D, t = 32, 32, 128, 256
    g = torch.Generator(device="cuda").manual_seed(1)
    sigma = torch.exp(0.5 * torch.randn((L, 2, 1, H * D), device="cuda", generator=g)).clamp(0.1, 8.0)
    sigma = torch.where(torch.rand((L, 2, 1, H * D), device="cuda", generator=g) < 0.01, sigma * 10, sigma)
    kv = (torch.randn((L, 2, t, H * D), device="cuda", generator=g) * sigma).to(torch.bfloat16).reshape(L, 2, t, H, D)
    kb, vb = (torch.tensor(b) for b in O.make_bins(MODEL))
    want = ref_torch.roundtrip(kv, kb, vb, "vllm")
    raw = codec.encode_to_host(KvView.from_blob(kv, "vllm"), 0, t, t)[0]
    out = torch.empty_like(kv)
    codec.decode([raw], KvView.from_blob(out, "vllm"), [0])
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), want.view(torch.int16))
    sym = ref_torch.quantize(kv, kb, vb)[0]
    bits_per_sym = 8.0 * (len(raw)) / sym.numel()
    assert bits_per_sym < 8.0
    # idempotence: re-encoding the decoded KV reproduces the same symbols -> the same decode
    raw2 = codec.encode_to_host(KvView.from_blob(out, "vllm"), 0, t, t)[0]
    out2 = torch.empty_like(kv)
    codec.decode([raw2], KvView.from_blob(out2, "vllm"), [0])
    torch.cuda.synchronize()
    assert torch.equal(out2.view(torch.int16), out.view(torch.int16))


def test_baseline_block_full_size_properties(codec):
    """BASELINE configs[1] at full size (32L/32H/128D, 8192 tokens = 4 GiB, 32 chunks in ONE batched call):
    decoded block == the reference's torch op chain applied chunk by chunk (bit-exact); containers of the batched
    call == containers of per-chunk calls (checksum of checksums); decode(encode(decoded)) == decoded (idempotence);
    total size below 8 bits/symbol."""
    import zlib
    import ref_torch
    from lmcache_b200.codec import KvView
    if codec.coder != 2:
        pytest.skip("the 4 GiB block runs once, on the default container")
    L, H, D, T, cs = 32, 32, 128, 8192, 256
    g = torch.Generator(device="cuda").manual_seed(2)
    sigma = torch.exp(0.5 * torch.randn((L, 2, 1, H * D), device="cuda", generator=g)).clamp(0.1, 8.0)
    kv = torch.empty((L, 2, T, H * D), dtype=torch.bfloat16, device="cuda")
    for t0 in range(0, T, 1024):                                  # generate in slabs: no 16 GiB fp32 temporary
        kv[:, :, t0:t0 + 1024] = (torch.randn((L, 2, 1024, H * D), device="cuda", generator=g) * sigma).to(torch.bfloat16)
    kv = kv.reshape(L, 2, T, H, D)
    view = KvView.from_blob(kv, "vllm")
    raws = codec.encode_to_host(view, 0, T, cs)
    assert len(raws) == T // cs
    crc_batched = zlib.crc32(b"".join(zlib.crc32(bytes(r)[64:]).to_bytes(4, "little") for r in raws))
    crc_single = zlib.crc32(b"".join(
        zlib.crc32(bytes(codec.encode_to_host(view, j * cs, cs, cs)[0])[64:]).to_bytes(4, "little") for j in range(T // cs)))
    assert crc_batched == crc_single
    assert sum(len(r) for r in raws) * 8 < 8.0 * kv.numel()
    out = torch.empty_like(kv)
    codec.decode(raws, KvView.from_blob(out, "vllm"), [j * cs for j in range(T // cs)])
    torch.cuda.synchronize()
    kb, vb = (torch.tensor(b) for b in O.make_bins(MODEL))
    for j in range(T // cs):
        want = ref_torch.roundtrip(kv[:, :, j * cs:(j + 1) * cs], kb, vb, "vllm")
        assert torch.equal(out[:, :, j * cs:(j + 1) * cs].view(torch.int16), want.view(torch.int16)), j
    del want
    raws2 = codec.encode_to_host(KvView.from_blob(out, "vllm"), 0, T, cs)
    out2 = torch.empty_like(kv)
    codec.decode(raws2, KvView.from_blob(out2, "vllm"), [j * cs for j in range(T // cs)])
    torch.cuda.synchronize()
    assert torch.equal(out2.view(torch.int16), out.view(torch.int16))


@pytest.mark.parametrize("seed", range(24))
def test_random_shapes_layouts_and_offsets_vs_oracle(codec, seed):
    """Seeded sweep over shapes the fixed cases do not pin: odd head sizes (scalar kernels), partial channel tiles,
    1..700 tokens, chunk sizes on both sides of 256, both dtypes, blob / tuple / huggingface sources, tok_begin > 0,
    decode at a destination offset into a larger blob.  Container sections and decoded values == oracle."""
    from lmcache_b200.codec import KvView
    rng = np.random.default_rng(9000 + seed)
    L = int(rng.integers(1, 5))
    H = int(rng.integers(1, 5))
    D = int(rng.choice([8, 20, 33, 64, 72, 80, 128]))
    T = int(rng.integers(1, 701))
    cs = int(rng.choice([16, 64, 200, 256, 300, 512]))
    dt = int(rng.integers(0, 2))
    src = str(rng.choice(["blob", "tuple", "hf_blob"]))
    tok_begin = int(rng.integers(0, T)) if T > 1 and rng.random() < 0.5 else 0
    C = H * D
    bits = O.synth_kv_bits(L, T, C, seed=seed)
    tdt = torch.bfloat16 if dt == 0 else torch.float16
    kv = _bits_to_tensor(bits, 0).float().to(tdt).reshape(L, 2, T, H, D).cuda()
    bits = _tensor_bits(kv).reshape(L, 2, T, C)
    if src == "blob":
        view = KvView.from_blob(kv, "vllm")
    elif src == "hf_blob":
        view = KvView.from_blob(kv.permute(0, 1, 3, 2, 4).contiguous(), "huggingface")
    else:
        view = KvView.from_tuple(tuple((kv[l, 0].clone(), kv[l, 1].clone()) for l in range(L)), "vllm")
    n = T - tok_begin
    raws = codec.encode_to_host(view, tok_begin, n, cs)
    kb, vb = O.make_bins(MODEL)
    n_chunks = (n + cs - 1) // cs
    assert len(raws) == n_chunks
    pad = int(rng.integers(0, 40))
    out = torch.full((L, 2, pad + n, H, D), 2.0, dtype=tdt, device="cuda")
    wants = []
    for j, raw in enumerate(raws):
        t0, t1 = tok_begin + j * cs, min(T, tok_begin + (j + 1) * cs)
        enc = _oenc(codec, bits[:, :, t0:t1], dt, kb, vb)
        cdf, maxes, lengths, payload = _sections(raw, L, H, D, t1 - t0)
        assert np.array_equal(cdf, enc["cdf"]) and np.array_equal(maxes, enc["maxes"]), (seed, j)
        assert np.array_equal(lengths, np.stack([ln for _, ln, _ in enc["groups"]])), (seed, j)
        assert np.array_equal(payload, np.concatenate([b for b, _, _ in enc["groups"]])), (seed, j)
        wants.append(O.decode_chunk(enc, dt, kb, vb, dt))
    codec.decode(raws, KvView.from_blob(out, "vllm"), [pad + j * cs for j in range(n_chunks)])
    torch.cuda.synchronize()
    got = _tensor_bits(out).reshape(L, 2, pad + n, C)
    assert np.array_equal(got[:, :, pad:], np.concatenate(wants, axis=2)), seed
    if pad:
        assert bool((out[:, :, :pad] == 2.0).all()), "decode wrote in front of its destination offset"


def test_extreme_inputs(codec):
    """all-zero block, single outlier rows, +/-inf and NaN rows: no crash, parity with the oracle."""
    from lmcache_b200.codec import KvView
    L, H, D, t = 3, 1, 128, 64
    x = torch.randn(L, 2, t, H, D).to(torch.bfloat16)
    x[0] = 0
    x[1, 0, 3, 0, 5] = float("inf")
    x[1, 1, 4, 0, 6] = float("nan")
    x[2, 0, :, 0, 7] = 1e30
    bits = x.view(torch.int16).numpy().view(np.uint16).reshape(L, 2, t, H * D)
    raw = codec.encode_to_host(KvView.from_blob(x.cuda(), "vllm"), 0, t, t)[0]
    kb, vb = O.make_bins(MODEL)
    enc = _oenc(codec, bits, 0, kb, vb)
    cdf, maxes, lengths, payload = _sections(raw, L, H, D, t)
    assert np.array_equal(cdf, enc["cdf"])
    assert np.array_equal(lengths[0], enc["groups"][0][1])
    assert np.array_equal(payload, enc["groups"][0][0])
    out = torch.zeros((L, 2, t, H, D), dtype=torch.bfloat16, device="cuda")
    codec.decode([raw], KvView.from_blob(out, "vllm"), [0])
    torch.cuda.synchronize()
    assert _eq_nan(_tensor_bits(out).reshape(L, 2, t, H * D), O.decode_chunk(enc, 0, kb, vb, 0), 0)


# ---------------------------------------------------------------- serde plugins (mirrors reference tests/test_serde.py)
def _generate_kv_cache(num_tokens, fmt, device):
    shape = [num_tokens, 8, 128] if fmt == "vllm" else [8, num_tokens, 128]
    dtype = torch.bfloat16 if fmt == "vllm" else torch.float16
    return tuple((torch.rand(shape, dtype=dtype, device=device), torch.rand(shape, dtype=dtype, device=device))
                 for _ in range(32))


def _to_blob(kv):
    return torch.stack([torch.stack(p, dim=0) for p in kv], dim=0)


def _meta(fmt):
    from lmcache_b200.config import LMCacheEngineMetadata
    return LMCacheEngineMetadata("mistralai/Mistral-7B-Instruct-v0.2", 1, 0, fmt, "bfloat16")


@pytest.mark.parametrize("chunk_size", [16, 128, 256])
def test_cachegen_encoder(chunk_size):
    from lmcache_b200.config import LMCacheEngineConfig
    from lmcache_b200.storage_backend.serde.cachegen_basics import CacheGenEncoderOutput
    from lmcache_b200.storage_backend.serde.cachegen_encoder import CacheGenSerializer
    cfg = LMCacheEngineConfig.from_defaults(chunk_size=chunk_size)
    s1, s2 = CacheGenSerializer(cfg, _meta("vllm")), CacheGenSerializer(cfg, _meta("huggingface"))
    kv = _to_blob(_generate_kv_cache(chunk_size, "vllm", "cuda"))
    out1 = s1.to_bytes(kv)
    out2 = s2.to_bytes(kv.permute([0, 1, 3, 2, 4]))
    assert abs(len(out1) - len(out2)) < 10
    assert out1 == out2          # same tokens, same bits: the layouts differ only by strides
    od = CacheGenEncoderOutput.from_bytes(out1)
    assert od.num_heads == 8 and od.head_size == 128


@pytest.mark.parametrize("fmt", ["vllm", "huggingface"])
@pytest.mark.parametrize("chunk_size", [16, 128, 256])
def test_cachegen_decoder(fmt, chunk_size):
    import ref_torch
    from lmcache_b200.config import LMCacheEngineConfig
    from lmcache_b200.storage_backend.serde import CreateSerde
    cfg = LMCacheEngineConfig.from_defaults(chunk_size=chunk_size)
    ser, des = CreateSerde("cachegen", cfg, _meta(fmt))
    kv = _to_blob(_generate_kv_cache(chunk_size, fmt, "cuda"))
    dec = des.from_bytes(ser.to_bytes(kv))
    assert dec.shape == kv.shape and dec.mean() != 0
    assert dec.dtype == (torch.bfloat16 if fmt == "vllm" else torch.float16)
    kb, vb = (torch.tensor(b) for b in O.make_bins(MODEL))
    kv_v = kv if fmt == "vllm" else kv.permute(0, 1, 3, 2, 4)
    want = ref_torch.roundtrip(kv_v, kb, vb, fmt)
    assert torch.equal(dec.view(torch.int16), want.contiguous().view(torch.int16))
    assert torch.equal(des.from_bytes(bytearray(ser.to_bytes(kv))), dec)      # bytearray from the socket path


def test_cachegen_unmatched_size():
    from lmcache_b200.config import LMCacheEngineConfig
    from lmcache_b200.storage_backend.serde import CreateSerde
    ser, des = CreateSerde("cachegen", LMCacheEngineConfig.from_defaults(chunk_size=256), _meta("vllm"))
    kv = _to_blob(_generate_kv_cache(236, "vllm", "cuda"))
    dec = des.from_bytes(ser.to_bytes(kv))
    assert dec.shape == kv.shape and dec.mean() != 0


def test_batched_plugin_paths_match_per_chunk_calls():
    from lmcache_b200.config import LMCacheEngineConfig
    from lmcache_b200.storage_backend.serde.cachegen_decoder import CacheGenDeserializer
    from lmcache_b200.storage_backend.serde.cachegen_encoder import CacheGenSerializer
    cfg = LMCacheEngineConfig.from_defaults(chunk_size=128)
    ser, des = CacheGenSerializer(cfg, _meta("vllm")), CacheGenDeserializer(cfg, _meta("vllm"))
    kvt = _generate_kv_cache(300, "vllm", "cuda")
    blob = _to_blob(kvt)
    per_chunk = [ser.to_bytes(blob[:, :, a:min(300, a + 128)].contiguous()) for a in range(0, 300, 128)]
    assert ser.to_bytes_batch(blob) == per_chunk
    assert ser.kv_to_bytes_batch(kvt) == per_chunk
    whole = des.from_bytes_batch(per_chunk)
    parts = torch.cat([des.from_bytes(b) for b in per_chunk], dim=2)
    assert torch.equal(whole, parts)


def test_torch_serde_gpu_lossless():
    from lmcache_b200.storage_backend.serde.torch_serde import TorchDeserializer, TorchSerializer
    t = torch.randn(4, 2, 256, 4, 64, device="cuda").to(torch.bfloat16)     # BASELINE config 1 shape
    back = TorchDeserializer().from_bytes(TorchSerializer().to_bytes(t))
    assert back.device.type == "cpu" and torch.equal(back, t.cpu())


@pytest.mark.parametrize("coder", ["rans_compact", "rans"])
@pytest.mark.parametrize("kind", ["peaked", "uniform"])
def test_decoder_table_layouts_agree(kind, coder, monkeypatch):
    """the row-major and the transposed decoder table produce identical KV (the product picks by the containers' bits
    per symbol; B200KV_DECODE_TABLE forces one)"""
    from lmcache_b200.codec import CacheGenCodec, KvView
    L, H, D, T, cs = 8, 4, 128, 700, 256
    g = torch.Generator(device="cuda").manual_seed(5)
    if kind == "peaked":
        kv = (torch.randn((L, 2, T, H, D), device="cuda", generator=g) * 0.05)
        kv[:, :, :, :, 0] = 4.0                                        # one loud channel pins every row's maximum
    else:
        kv = torch.rand((L, 2, T, H, D), device="cuda", generator=g) * 2 - 1
    kv = kv.to(torch.bfloat16)
    codec = CacheGenCodec(MODEL, coder=coder)
    blobs = [bytes(b) for b in codec.encode_to_host(KvView.from_blob(kv, "vllm"), 0, T, cs)]
    decs = {}
    for table in ("rows", "transposed"):
        monkeypatch.setenv("B200KV_DECODE_TABLE", table)
        out = torch.zeros_like(kv)
        codec.decode(blobs, KvView.from_blob(out, "vllm"), [j * cs for j in range(len(blobs))])
        torch.cuda.synchronize()
        assert codec.decode_status() == [0] * len(blobs)
        decs[table] = out
    assert torch.equal(decs["rows"].view(torch.int16), decs["transposed"].view(torch.int16))
    kb, vb = O.make_bins(MODEL)
    bits = _tensor_bits(kv).reshape(L, 2, T, H * D)
    want = np.concatenate([O.decode_chunk(O.encode_chunk(bits[:, :, j * cs:min(T, (j + 1) * cs)], 0, kb, vb, O.CODER_RANS), 0, kb, vb, 0)
                           for j in range(len(blobs))], axis=2)
    assert np.array_equal(_tensor_bits(decs["rows"]).reshape(L, 2, T, H * D), want)


@pytest.mark.parametrize("kind", ["peaked", "uniform"])
def test_damaged_containers_never_fault(codec, kind):
    """A container whose bytes were damaged after its header was written (a remote tier, a disk) must decode to SOMETHING
    without touching memory outside the caller's buffer: random byte flips in the lengths section, the stream headers /
    CDF rows, the payload and the maxima of every container version.  The header itself stays intact (a damaged header is
    rejected on the host, tests/test_abi_and_host.py).  rANS containers flag the damage in their status words; a clean
    decode afterwards proves the context is alive."""
    from lmcache_b200 import _native as N
    from lmcache_b200.codec import KvView, container_layout_of, parse_header
    L, H, D, T = 4, 2, 128, 256
    g = torch.Generator(device="cuda").manual_seed(11)
    if kind == "peaked":
        kv = torch.randn((L, 2, T, H, D), device="cuda", generator=g) * 0.05
        kv[:, :, :, :, 0] = 4.0
    else:
        kv = torch.rand((L, 2, T, H, D), device="cuda", generator=g) * 2 - 1
    kv = kv.to(torch.bfloat16)
    raw = bytes(codec.encode_to_host(KvView.from_blob(kv, "vllm"), 0, T, T)[0])
    lo = container_layout_of(parse_header(raw))
    rng = np.random.default_rng(3)
    sections = {"lengths": (lo.off_lengths, lo.off_payload), "payload": (lo.off_payload, len(raw)),
                "front": (lo.off_cdf, lo.off_maxes), "maxes": (lo.off_maxes, lo.off_lengths),
                "payload_head": (lo.off_payload, min(len(raw), lo.off_payload + 4096))}
    flagged = 0
    for name, (a, b) in sections.items():
        for n_flips in (1, 64, 4096):
            bad = bytearray(raw)
            for pos in rng.integers(a, b, size=n_flips):
                bad[pos] = int(rng.integers(0, 256))
            out = torch.zeros_like(kv)
            try:
                codec.decode([bytes(bad)], KvView.from_blob(out, "vllm"), [0])
            except ValueError:
                continue                                   # the host-side checks caught it (e.g. the nb map): a miss
            torch.cuda.synchronize()                       # would raise on an illegal address
            flagged += any(codec.decode_status())
    if codec.coder != N.CODER_AC:
        assert flagged > 0                                 # the rANS final-state check notices damaged streams
    out = torch.zeros_like(kv)
    codec.decode([raw], KvView.from_blob(out, "vllm"), [0])
    torch.cuda.synchronize()
    assert codec.decode_status() == [0]
    bits = _tensor_bits(kv).reshape(L, 2, T, H * D)
    kb, vb = O.make_bins(MODEL)
    want = O.decode_chunk(O.encode_chunk(bits, 0, kb, vb, O.CODER_RANS), 0, kb, vb, 0)
    assert np.array_equal(_tensor_bits(out).reshape(L, 2, T, H * D), want)
