"""Plain references for the prefix-hash chain: hashlib over the tokens' native bytes, exactly as the reference engine
hashes a chunk (lmcache/cache_engine.py:58-96: sha256(prefix_hex.encode("ascii") + chunk.tobytes()).hexdigest(), with an
empty prefix for the first chunk).  Shared by the CPU test that pins it to the goldens and the oracle, and by the GPU
test of the kernels."""
import hashlib
from typing import Dict, List, Sequence

import numpy as np

NP_DTYPE = {1: np.uint8, 2: np.int16, 4: np.int32, 8: np.int64}

# Per element size, chunk sizes whose token bytes cs * es fall in every reachable class mod 64 among 0, 1, 54, 55, 56,
# 57 and 63: the classes where SHA-256 padding (0x80, zeros, 8 length bytes) just fits, just spills into one more block,
# or leaves a whole block of padding.  A chained chunk hashes a 64-byte hex prefix block in front, so the class of the
# token bytes is also the class of the whole message.
PAD_CHUNK_SIZES: Dict[int, List[int]] = {
    1: [1, 54, 55, 56, 57, 63, 64, 65, 119, 120],
    2: [1, 27, 28, 32, 59, 60],
    4: [1, 14, 16, 30, 32],
    8: [1, 7, 8, 15, 16],
}


def pad_class(chunk_size: int, elem_size: int) -> int:
    return chunk_size * elem_size % 64


def ref_chain(tokens: np.ndarray, chunk_size: int) -> List[str]:
    """Hex digests of the chain over one sequence."""
    data = np.ascontiguousarray(tokens)
    out, prefix = [], b""
    for i in range(0, data.shape[0], chunk_size):
        h = hashlib.sha256(prefix + data[i:i + chunk_size].tobytes()).hexdigest()
        out.append(h)
        prefix = h.encode("ascii")
    return out


def ref_chain_seqs(tokens: np.ndarray, offsets: Sequence[int], chunk_size: int) -> List[str]:
    """ref_chain of every sequence [offsets[s], offsets[s + 1]), concatenated in sequence order."""
    out = []
    for a, b in zip(offsets[:-1], offsets[1:]):
        out += ref_chain(tokens[a:b], chunk_size)
    return out


def n_chunks(offsets: Sequence[int], chunk_size: int) -> int:
    return sum((b - a + chunk_size - 1) // chunk_size for a, b in zip(offsets[:-1], offsets[1:]))


def random_tokens(rng: np.random.Generator, n: int, elem_size: int) -> np.ndarray:
    """n tokens of the element size's dtype over its whole bit range."""
    return rng.integers(0, 256, n * elem_size, dtype=np.uint8).view(NP_DTYPE[elem_size])
