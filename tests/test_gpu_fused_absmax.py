"""GPU: the per-token maxima computed inside the persistent encode_kernel (chunks of <= 256 tokens), held to the CPU
oracle byte for byte.

encode_kernel<FUSED = true> claims tickets that interleave absmax items (8 token rows of one (chunk, plane) over all
channels) with the tiles of the unit eight steps behind; a tile waits for its unit's items.  These tests check that what
comes out is exactly what the separate absmax pass produced: every container version (1, 2, 3 and the latent version
4), bf16 and fp16, vector and scalar row loads, a paged slot map, a ragged last chunk, H = 8 and H = 32, rows whose
maximum is zero, subnormal, infinite or NaN, calls with more units than the device holds CTAs at once, and the
layer-split encode (b200kv_encode_layers) in random layer partitions."""
import numpy as np
import pytest
import torch

import mla_ref
from oracle import oracle as O
from test_gpu_layer_split import _check_sections, _containers, _encode_chunks, _encode_layers, _rand_partition, _source

pytestmark = pytest.mark.gpu
TDT = (torch.bfloat16, torch.float16)


def _N():
    from lmcache_b200 import _native as N
    return N


def _extreme_kv(L, T, H, D, dt, seed):
    """[L,2,T,H,D] normal KV with rows whose maximum is 0, subnormal, +inf (a -inf entry), NaN, and a row whose maximum
    sits in the last channel; returns the CPU tensor and its bits [L,2,T,C]"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((L, 2, T, H, D), generator=g).to(TDT[dt])
    sub = torch.tensor(1e-40 if dt == 0 else 3e-6, dtype=torch.float32).to(TDT[dt])   # a subnormal of the dtype
    x[0, 0, 5] = 0
    x[0, 1, 6] = sub * torch.sign(torch.randn((H, D), generator=g)).to(TDT[dt])
    x[L - 1, 0, 7, H - 1, D - 1] = float("-inf")
    x[L - 1, 1, T - 1, 0, 0] = float("nan")
    x[0, 0, 9] *= 0.01
    x[0, 0, 9, H - 1, D - 1] = 50.0
    x[L - 1, 0, 260 % T] = 0                         # in the ragged last chunk when T > 260
    return x, x.view(torch.int16).numpy().view(np.uint16).reshape(L, 2, T, H * D)


@pytest.mark.parametrize("src", ["blob", "paged", "hf"])
@pytest.mark.parametrize("H,D", [(8, 128), (32, 128), (3, 33)])
@pytest.mark.parametrize("dt", [0, 1], ids=["bf16", "fp16"])
@pytest.mark.parametrize("coder", [0, 1, 2])
def test_encode_chunks_vs_oracle(coder, dt, H, D, src):
    """b200kv_encode_chunks, 256-token chunks plus a ragged one: every section == the oracle's (maxima NaN for NaN).
    D = 128 takes the 128-bit row loads, 3 x 33 the scalar ones and a partial channel tile."""
    L, cs = 2, 256
    T = 2 * cs + 45
    x, bits = _extreme_kv(L, T, H, D, dt, seed=31 * coder + 7 * dt + H)
    view = _source(src, x.cuda(), np.random.default_rng(H + dt))
    kb, vb = np.array([32, 9], np.float32), np.array([16, 5], np.float32)
    n, last = 3, T - 2 * cs
    raws = _encode_chunks(view, 0, n, cs, last, kb, vb, coder)
    for j in range(n):
        t = cs if j < n - 1 else last
        _check_sections(raws[j], bits[:, :, j * cs: j * cs + t], dt, kb, vb, coder, nan_maxes=True)


@pytest.mark.parametrize("src", ["blob", "paged"])
def test_many_units_and_tok_begin(src):
    """32 layers x 5 chunks = 320 (chunk, plane) units, far more work items than resident CTAs, chunks of 200 tokens
    starting at token 37 of the source: the containers == the oracle's"""
    N = _N()
    L, H, D, cs = 32, 8, 128, 200
    T = 37 + 4 * cs + 130
    x, bits = _extreme_kv(L, T, H, D, 0, seed=5)
    view = _source(src, x.cuda(), np.random.default_rng(3))
    rng = np.random.default_rng(11)
    kb, vb = rng.integers(4, 33, L).astype(np.float32), rng.integers(4, 33, L).astype(np.float32)
    n, last = 5, 130
    raws = _encode_chunks(view, 37, n, cs, last, kb, vb, N.CODER_RANS_COMPACT)
    for j in range(n):
        a = 37 + j * cs
        _check_sections(raws[j], bits[:, :, a: a + (cs if j < n - 1 else last)], 0, kb, vb, O.CODER_RANS_COMPACT,
                        nan_maxes=True)


@pytest.mark.parametrize("src", ["blob", "paged"])
@pytest.mark.parametrize("dt", [0, 1], ids=["bf16", "fp16"])
@pytest.mark.parametrize("H", [8, 32])
def test_encode_layers_vs_encode_chunks_and_oracle(H, dt, src):
    """b200kv_encode_layers in a random layer partition (the maxima of each call's layers only): every container ==
    b200kv_encode_chunks' and the oracle's"""
    N = _N()
    L, D, cs = 6, 128, 128
    T = 2 * cs + 19
    x, bits = _extreme_kv(L, T, H, D, dt, seed=H + dt)
    rng = np.random.default_rng(100 * H + dt)
    view = _source(src, x.cuda(), rng)
    kb, vb = rng.integers(4, 33, L).astype(np.float32), rng.integers(4, 33, L).astype(np.float32)
    n, last = 3, T - 2 * cs
    want = _encode_chunks(view, 0, n, cs, last, kb, vb, N.CODER_RANS_COMPACT)
    got = _containers(_encode_layers(view, 0, n, cs, last, kb, vb, _rand_partition(rng, L)))
    assert got == want
    for j in range(n):
        _check_sections(got[j], bits[:, :, j * cs: j * cs + (cs if j < n - 1 else last)], dt, kb, vb,
                        O.CODER_RANS_COMPACT, nan_maxes=True)


@pytest.mark.parametrize("paged", [False, True], ids=["blob", "paged"])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("L,D", [(61, 576), (9, 20)])
def test_latent_v4_vs_oracle(L, D, dt, paged):
    """a latent KV (one plane per layer, container version 4), 256-token chunks and a ragged one: == the oracle's"""
    from lmcache_b200.codec import CacheGenCodec, KvView
    N = _N()
    cs, rag = 256, 29
    T = cs + rag
    bits = O.synth_kv_bits(L, T, D, seed=L + D)[:, 0]
    if dt == torch.float16:
        bits = O.bf16_bits_to_f32(bits).astype(np.float16).view(np.uint16)
    bits = np.ascontiguousarray(bits)
    bits[0, 3] = 0                                              # a zero row
    x = torch.from_numpy(bits.view(np.int16)).view(dt).cuda()
    cfg = dict(key_first_layers=min(3, L), key_second_layers=min(20, L), key_third_layers=L, key_first_bins=32,
               key_second_bins=16, key_third_bins=8, value_first_layers=2, value_first_bins=32, value_second_bins=16)
    codec = CacheGenCodec("lmsys/longchat-7b-16k", cachegen_config=cfg)
    kb = np.array(codec.config.key_bins_list(), np.float32)
    if paged:
        nblk = (T + 63) // 64 + 2
        store = torch.zeros((L, nblk, 64, D), dtype=dt, device="cuda")
        slots = torch.randperm(nblk * 64, generator=torch.Generator().manual_seed(L))[:T].cuda()
        store.view(L, -1, D)[:, slots] = x
        view = KvView.from_paged([store[l] for l in range(L)], slots)
    else:
        view = KvView.from_blob(x, "vllm")
    batch = codec.encode(view, 0, T, cs)
    assert batch.coder == N.CODER_LATENT
    dtc = N.DT_BF16 if dt == torch.bfloat16 else N.DT_FP16
    for j, (a, t) in enumerate([(0, cs), (cs, rag)]):
        want, _, _ = mla_ref.v4_container(bits[:, a:a + t], dtc, kb, 1, D)
        assert batch.container(j).cpu().numpy().tobytes() == want, f"chunk {j}"
