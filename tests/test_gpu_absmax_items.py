"""GPU: the absmax items of the persistent encode_kernel across row sizes and source layouts, held to the CPU oracle
byte for byte.

An item reduces kAbsRows token rows of one (chunk, plane) over all channels, with 128-bit loads when every row is
16-byte aligned and 2-byte loads otherwise.  Covered: rows of 2, 8 and 16 KB (H = 8, 32, 64 heads of 128), heads at a
pitch other than D (a padded vllm blob and a huggingface blob), a paged cache with a scattered
slot map, a ragged last chunk after tok_begin != 0, fp16, rows of zeros, -0, +-inf and NaN, a view 2 bytes past a
16-byte boundary (2-byte loads at D = 128), and back-to-back calls that share one workspace and output buffer."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle as O
from test_gpu_layer_split import _a16, _check_sections, _encode_chunks, _s, _source

pytestmark = pytest.mark.gpu
TDT = (torch.bfloat16, torch.float16)
CS = 256


def _N():
    from lmcache_b200 import _native as N
    return N


def _special_kv(L, T, H, D, dt, seed):
    """[L,2,T,H,D] normal KV with rows of zeros, of -0, with +inf / -inf entries, with NaN, and one whose maximum sits
    in its last channel; returns the CPU tensor and its bits [L,2,T,C]"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((L, 2, T, H, D), generator=g).to(TDT[dt])
    x[0, 0, 1] = 0
    x[0, 1, 2] = -0.0
    x[L - 1, 0, 3, H // 2, D - 1] = float("inf")
    x[L - 1, 1, 4, H - 1, 0] = float("-inf")
    x[0, 0, T - 1, 0, D // 2] = float("nan")
    x[0, 1, 8] *= 0.01
    x[0, 1, 8, H - 1, D - 1] = 40.0
    return x, x.view(torch.int16).numpy().view(np.uint16).reshape(L, 2, T, H * D)


def _bins(L, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(4, 33, L).astype(np.float32), rng.integers(4, 33, L).astype(np.float32)


def _check_all(raws, bits, tok_begin, n, last, dt, kb, vb):
    for j in range(n):
        a = tok_begin + j * CS
        _check_sections(raws[j], bits[:, :, a: a + (CS if j < n - 1 else last)], dt, kb, vb, O.CODER_RANS_COMPACT,
                        nan_maxes=True)


@pytest.mark.parametrize("H,src", [(64, "blob"), (64, "hf"), (8, "padded"), (32, "padded"), (64, "padded")])
def test_row_sizes_and_head_pitch(H, src):
    """rows of 2, 8 and 16 KB, contiguous heads and heads at a pitch (D + 8 or T * D channels): == the oracle.
    8- and 32-head blobs are in test_gpu_fused_absmax.py"""
    N = _N()
    L, D = 2, 128
    tok_begin, n, last = 21, 2, 77
    T = tok_begin + CS + last
    x, bits = _special_kv(L, T, H, D, 0, seed=H)
    if src == "padded":                 # vllm blob, heads 136 channels apart
        pad = torch.zeros((L, 2, T, H, D + 8), dtype=x.dtype, device="cuda")
        pad[..., :D] = x.cuda()
        from lmcache_b200.codec import KvView
        view = KvView.from_blob(pad[..., :D], "vllm")
        assert view.desc.sH == D + 8
    else:
        view = _source(src, x.cuda(), np.random.default_rng(H))
    kb, vb = _bins(L, H)
    raws = _encode_chunks(view, tok_begin, n, CS, last, kb, vb, N.CODER_RANS_COMPACT)
    _check_all(raws, bits, tok_begin, n, last, 0, kb, vb)


@pytest.mark.parametrize("dt", [0, 1], ids=["bf16", "fp16"])
def test_paged_scattered_slot_map(dt):
    """16 KB rows of a paged cache, scattered by a random slot map (one source address per token row), fp16 and bf16"""
    N = _N()
    L, H, D = 2, 64, 128
    tok_begin, n, last = 5, 2, 130
    T = tok_begin + CS + last
    x, bits = _special_kv(L, T, H, D, dt, seed=10 + H + dt)
    view = _source("paged", x.cuda(), np.random.default_rng(H + dt))
    kb, vb = _bins(L, 7 + dt)
    raws = _encode_chunks(view, tok_begin, n, CS, last, kb, vb, N.CODER_RANS_COMPACT)
    _check_all(raws, bits, tok_begin, n, last, dt, kb, vb)


@pytest.mark.parametrize("dt", [0, 1], ids=["bf16", "fp16"])
def test_misaligned_view(dt):
    """a blob 2 bytes past a 16-byte boundary: the items take 2-byte loads; == the oracle"""
    N = _N()
    from lmcache_b200.codec import KvView
    L, H, D = 2, 32, 128
    T = CS + 40
    x, bits = _special_kv(L, T, H, D, dt, seed=3 + dt)
    flat = torch.empty(x.numel() + 8, dtype=x.dtype, device="cuda")
    mis = flat[1: 1 + x.numel()].view(x.shape)
    mis.copy_(x.cuda())
    assert mis.data_ptr() % 16 == 2
    view = KvView.from_blob(mis, "vllm")
    kb, vb = _bins(L, 5)
    raws = _encode_chunks(view, 0, 2, CS, T - CS, kb, vb, N.CODER_RANS_COMPACT)
    _check_all(raws, bits, 0, 2, T - CS, dt, kb, vb)


def test_back_to_back_calls_share_a_workspace():
    """several encode calls on one workspace and one output buffer, each with other data, shapes of rows and chunk
    counts: every container == the oracle's (the ticket and ready counters start from zero in every call)"""
    N = _N()
    lib = N.lib()
    L, D = 2, 128
    cases = [(32, 3, 0, 200), (8, 1, 7, 256), (64, 2, 3, 31), (32, 4, 100, 1), (8, 2, 0, 256)]
    Hmax, nmax = 64, 4
    stride = _a16(N.container_layout(L, Hmax, D, CS, N.CODER_RANS_COMPACT).max_total_bytes)
    out = torch.empty(nmax * stride, dtype=torch.uint8, device="cuda")
    sizes = torch.zeros(nmax, dtype=torch.int64, device="cuda")
    wsb = max(N.check(lib.b200kv_encode_workspace_bytes(L, H, D, CS, nmax, N.CODER_RANS_COMPACT), "workspace")
              for H, _, _, _ in cases)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    for i, (H, n, tok_begin, last) in enumerate(cases):
        T = tok_begin + (n - 1) * CS + last
        x, bits = _special_kv(L, T, H, D, 0, seed=50 + i)
        view = _source("blob", x.cuda(), None)
        kb, vb = _bins(L, 60 + i)
        N.check(lib.b200kv_encode_chunks(ctypes.byref(view.desc), tok_begin, n, CS, last, N.float_array(kb),
                                         N.float_array(vb), N.CODER_RANS_COMPACT, out.data_ptr(), stride,
                                         sizes.data_ptr(), ws.data_ptr(), wsb, _s()), "encode_chunks")
        torch.cuda.synchronize()
        sz = sizes.cpu().tolist()
        buf = out.cpu().numpy()
        raws = [bytes(buf[j * stride: j * stride + sz[j]]) for j in range(n)]
        _check_all(raws, bits, tok_begin, n, last, 0, kb, vb)
