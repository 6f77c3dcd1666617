"""CPU: the C ABI of the layer-range mover calls and the slice arithmetic the raw tiers' layer-wise paths use."""
import ctypes
import os
import re

import numpy as np
import pytest

from lmcache_b200 import _native as N
from lmcache_b200.storage_backend.local_backend import chunk_runs, layer_row_bytes, layer_table, packed_offsets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ctypes.POINTER(N.KvDesc)


@pytest.mark.parametrize("name,want", [
    ("b200kv_pack_chunks_layers", [P, ctypes.c_int64] + [ctypes.c_int32] * 6 + [ctypes.c_void_p, ctypes.c_void_p]),
    ("b200kv_unpack_chunks_layers", [ctypes.c_void_p] + [ctypes.c_int32] * 6 + [P, ctypes.c_int64, ctypes.c_void_p]),
])
def test_layers_symbols_are_declared_bound_and_listed(name, want):
    with open(os.path.join(ROOT, "include", "b200kv.h")) as f:
        hdr = f.read()
    m = re.search(r"int\s+" + name + r"\(([^;]*)\);", hdr)
    assert m is not None
    assert len(m.group(1).split(",")) == len(want) == 10
    res, args = N.SIGNATURES[name]
    assert res is ctypes.c_int32 and args == want
    vblock = hdr[hdr.index("#define B200KV_VERSION"):]
    assert name in vblock[:vblock.index("*/")]


# hand-computed: L = 3, H = 2, D = 4, 2-byte elements, chunks of 5 tokens, a ragged last chunk of 2
@pytest.mark.parametrize("kind,H,D,row", [("vllm", 2, 4, 2 * 2 * 4 * 2), ("huggingface", 2, 4, 2 * 2 * 4 * 2),
                                          ("latent", 1, 8, 8 * 2)])
def test_layer_slices_of_raw_blobs(kind, H, D, row):
    L, es, tokens = 3, 2, [5, 5, 2]
    assert layer_row_bytes(H, D, es, kind == "latent") == row
    stride = L * row * 5                                       # pack_chunks' chunk stride
    bases = [1000 + j * stride for j in range(3)]
    for layer in range(L):
        # a layer slice of t tokens is [2,t,H,D] / [2,H,t,D] / [t,D]: t * row bytes at layer * t * row
        assert layer_table(bases, tokens, row, layer).tolist() == [bases[0] + layer * 5 * row,
                                                                   bases[1] + layer * 5 * row,
                                                                   bases[2] + layer * 2 * row]
    assert layer_table(bases, tokens, row, 0).dtype == np.uint64
    assert packed_offsets(tokens, row).tolist() == [0, 5 * row, 10 * row]
    assert packed_offsets([], row).tolist() == []


def test_layer_slices_of_a_vllm_blob_match_numpy_offsets():
    L, H, D, t = 4, 3, 8, 7
    blob = np.arange(L * 2 * t * H * D, dtype=np.int16).reshape(L, 2, t, H, D)
    row = layer_row_bytes(H, D, 2, False)
    for layer in range(L):
        off = int(layer_table([0], [t], row, layer)[0])
        assert off == blob[layer].ctypes.data - blob.ctypes.data
        assert np.array_equal(blob.view(np.uint8).reshape(-1)[off:off + t * row], blob[layer].view(np.uint8).reshape(-1))


@pytest.mark.parametrize("tokens,want", [
    ([256, 256, 100], [(0, 3, 256, 100)]),
    ([256], [(0, 1, 256, 256)]),
    ([100], [(0, 1, 100, 100)]),
    ([256, 100, 256, 256], [(0, 2, 256, 100), (2, 4, 256, 256)]),
    ([256, 300, 256], [(0, 1, 256, 256), (1, 2, 300, 300), (2, 3, 256, 256)]),
])
def test_chunk_runs(tokens, want):
    assert chunk_runs(tokens, 256) == want
