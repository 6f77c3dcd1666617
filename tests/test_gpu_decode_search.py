"""GPU: the rANS decode loop's symbol search (rans_decode_stream) at both search depths and in both table layouts.

One container per token count t in 1..5 and 253..256 (one coder group of t symbols per stream), two layers whose four
planes hold 4, 16, 18 and 32 symbols: key bins 4 and 18, value bins 16 and 32.  The 4- and 16-symbol planes search 4
levels (the transposed table with its LUT replica, whatever the host picks); the 18- and 32-symbol ones search 5, in the
table layout B200KV_DECODE_TABLE names.  Channel 0 of every plane is symbol 0 on every token, so each row's maximum is
MAX, the factor is 1 and x = s - MAX quantises to s exactly; the other channels hold prescribed symbol columns:

* every symbol the plane can hold, ascending and descending; a single symbol (the top one, the centre one); the two
  ends alternating -- so the search lands on every entry the plane uses and must step over the empty entries past nb
  (one slot each) and the entries of symbols a stream does not use (no slots);
* the columns of tests/golden/rans_edges.npz that fit the plane, and 256-token random columns found by a seeded search,
  which together make every symbol of every plane decode at least once from its first slot (slot == cdf[s]) and once
  from its last (slot == cdf[s + 1] - 1) -- asserted from the spec decoder's trace (rans_edges.decode_as_kernel);
* random columns with random sparse histograms fill the rest.

Both container versions that carry rANS streams (2: CDF rows in the container, 3: per-stream histograms) go through
b200kv_decode_chunks into a vllm blob or a paged cache, in both output dtypes, and must give the oracle's values bit for
bit with status 0."""
import numpy as np
import pytest
import torch

from oracle import oracle as O

import rans_edges as R
from test_gpu_layer_split import _Dest, _check_sections, _decode, _encode_chunks, _source

pytestmark = pytest.mark.gpu
KB = np.array([4, 18], np.float32)
VB = np.array([16, 32], np.float32)
PLANE_MAX = [1, 8, 7, 15]                     # planes K0, K1, V0, V1: 4, 18, 16 and 32 symbols
TOKENS = [1, 2, 3, 4, 5, 253, 254, 255, 256]
H, D = 2, 80                                  # C = 160: a full channel tile and a partial one
C = H * D


def _trace(col, M):
    """(slot, symbol) of every decode step of the own-CDF stream of `col` on a plane of MAX M, and the table"""
    cdf = R.own_cdf(col)
    start, freq = R.table(cdf)
    tr = []
    out, _ = R.decode_as_kernel(cdf, R.encode(cdf, col), col.size, nsteps=4 if M <= 7 else 5, trace=tr)
    assert np.array_equal(out, col)
    return [(slot, s) for slot, s, _, _ in tr], start, freq


def _edges(col, M):
    """{(symbol, 'first' | 'last')} the stream of `col` decodes from the first / last slot of that symbol"""
    tr, start, freq = _trace(col, M)
    hit = set()
    for slot, s in tr:
        if slot == start[s]:
            hit.add((s, "first"))
        if slot == start[s] + freq[s] - 1:
            hit.add((s, "last"))
    return hit


def _random_col(rng, t, M):
    syms = rng.choice(2 * M + 1, size=int(rng.integers(1, min(2 * M + 1, 6) + 1)), replace=False)
    w = rng.dirichlet(np.full(syms.size, 0.3))
    return rng.choice(syms, size=t, p=w).astype(np.uint8)


@pytest.fixture(scope="module")
def columns():
    """{(plane, t): [columns]} and the slot-edge coverage they reach per plane"""
    rng = np.random.default_rng(20261018)
    fixture = [col for col, _ in R.own_rows(R.load())]
    cols = {(p, t): [] for p in range(len(PLANE_MAX)) for t in TOKENS}
    cover = {}
    for p, M in enumerate(PLANE_MAX):
        top = 2 * M
        want = {(s, e) for s in range(top + 1) for e in ("first", "last")}
        got = set()
        for t in TOKENS:
            i = np.arange(t)
            cols[p, t] += [i % (top + 1), (top - i) % (top + 1), np.full(t, top), np.full(t, M),
                           np.where(i % 2 == 1, top, 0)]
            cols[p, t] += [c for c in fixture if c.size == t and c.max() <= top]
        for (q, t), cs in cols.items():
            if q == p:
                for c in cs:
                    got |= _edges(np.asarray(c, np.uint8), M)
        # the rest: 256-token columns in which a missing symbol is rare (few slots, so a decode of it starts at either
        # end of its range with a fair chance)
        for k in range(6000):
            miss = sorted(want - got)
            if not miss:
                break
            s = miss[k % len(miss)][0]
            c = _random_col(rng, 256, M)
            c[rng.choice(256, size=int(rng.integers(1, 4)), replace=False)] = s
            new = _edges(c, M) - got
            if new:
                got |= new
                cols[p, 256].append(c)
        cover[p] = (want, got)
    for (p, t), cs in cols.items():
        assert len(cs) < C, (p, t, len(cs))
        while len(cs) < C - 1:
            cs.append(_random_col(rng, t, PLANE_MAX[p]))
    return cols, cover


def test_search_columns_reach_every_slot_edge(columns):
    """the columns make every symbol of every plane decode from its first and from its last slot (host-side spec)"""
    _, cover = columns
    for p, (want, got) in cover.items():
        assert got >= want, (PLANE_MAX[p], sorted(want - got))


def _chunk_bits(cols, t):
    """KV bits [2, 2, t, C] (bf16) whose plane p holds symbol column c in channel 1 + c; channel 0 is symbol 0"""
    sym = np.zeros((len(PLANE_MAX), t, C), np.int64)
    for p in range(len(PLANE_MAX)):
        for c, col in enumerate(cols[p, t]):
            sym[p, :, 1 + c] = col
    x = (sym - np.array(PLANE_MAX)[:, None, None]).astype(np.float32)
    planes = torch.from_numpy(x).to(torch.bfloat16)                      # integers |x| <= 15: exact
    kv = planes.reshape(2, 2, t, C).transpose(0, 1).contiguous()         # planes (K0, K1, V0, V1) -> [L, 2, t, C]
    return kv, kv.view(torch.int16).numpy().view(np.uint16)


@pytest.mark.parametrize("table", ["rows", "transposed"])
@pytest.mark.parametrize("coder", [1, 2], ids=["v2", "v3"])      # B200KV_CODER_RANS, B200KV_CODER_RANS_COMPACT
def test_decode_search_matches_oracle(columns, coder, table, monkeypatch):
    monkeypatch.setenv("B200KV_DECODE_TABLE", table)
    cols, _ = columns
    for k, t in enumerate(TOKENS):
        kv, bits = _chunk_bits(cols, t)
        view = _source("blob", kv.reshape(2, 2, t, H, D).cuda(), None)
        raws = _encode_chunks(view, 0, 1, t, t, KB, VB, coder)
        enc = _check_sections(raws[0], bits, 0, KB, VB, coder)
        out_dt = k % 2
        dest = _Dest("paged" if k % 3 == 2 else "vllm", 2, H, D, t, out_dt, 3, np.random.default_rng(k))
        assert _decode(raws, coder, dest, [dest.tok0], KB, VB, 0) == [0], (coder, table, t)
        want = O.decode_chunk(enc, 0, KB, VB, out_dt)
        assert np.array_equal(dest.bits(), want), (coder, table, t)
        assert dest.rest_untouched()
