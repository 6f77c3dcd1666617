"""CPU: the hashlib chain the GPU hash tests compare against (hash_mover_ref.ref_chain) is pinned to the digests the
reference engine made (golden_hash.json) and to the CPU oracle, at every element size and SHA-256 padding class."""
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import oracle as O

from hash_mover_ref import PAD_CHUNK_SIZES, pad_class, random_tokens, ref_chain, ref_chain_seqs

HERE = os.path.dirname(os.path.abspath(__file__))


def _golden_cases():
    h = json.load(open(os.path.join(HERE, "golden", "golden_hash.json")))
    rng = np.random.default_rng(1234)        # the rng cases are drawn one after another, in file order
    out = []
    for c in h["cases"]:
        if c["label"].startswith("arange"):
            toks = np.arange(c["n"], dtype=c["dtype"])
        else:
            toks = rng.integers(0, 32000, c["n"], dtype=np.int64)
        assert hashlib.sha256(toks.tobytes()).hexdigest() == c["tokens_sha256"], c["label"]
        out.append((c, toks))
    return h, out


def test_ref_chain_matches_reference_goldens():
    h, cases = _golden_cases()
    for c, toks in cases:
        assert ref_chain(toks, c["chunk_size"]) == c["hashes"], c["label"]
    # the lm:// key string the reference's server and clients use embeds the first digest as it is
    first = ref_chain(cases[0][1], cases[0][0]["chunk_size"])[0]
    assert h["key_string_example"] == f"vllm@m@1@0@{first}"


def test_padding_classes_cover_every_reachable_class():
    for es, sizes in PAD_CHUNK_SIZES.items():
        reachable = {c for c in (0, 1, 54, 55, 56, 57, 63) if any((cs * es) % 64 == c for cs in range(1, 64))}
        assert reachable <= {pad_class(cs, es) for cs in sizes}, es


@pytest.mark.parametrize("es", [1, 2, 4, 8])
def test_ref_chain_matches_oracle(es):
    rng = np.random.default_rng(100 + es)
    for cs in PAD_CHUNK_SIZES[es]:
        # at least three chunks, so every class occurs on chained chunks; a ragged and a full last chunk
        for n in (3 * cs, 3 * cs + max(1, cs // 2), 4 * cs - 1):
            toks = random_tokens(rng, n, es)
            assert ref_chain(toks, cs) == O.sha256_chain(toks, cs), (es, cs, n)


def test_ref_chain_seqs_concatenates_in_order():
    rng = np.random.default_rng(5)
    toks = random_tokens(rng, 100, 2)
    offs = [0, 0, 17, 17, 64, 100]
    want = []
    for a, b in zip(offs[:-1], offs[1:]):
        want += O.sha256_chain(toks[a:b], 16)
    assert ref_chain_seqs(toks, offs, 16) == want
    assert ref_chain(toks[:0], 16) == []
