"""CPU: the statement the paged-edge GPU tests compare against (paged_edges.ref_rows / ref_pack / ref_unpack) is pinned
to hand-built caches and to the layouts codec.paged_layout and codec.strided_slots recognise; the launch model gives the
vector widths and head blocks worked out by hand; and CASES reaches every branch of the split kernel's launch rule."""
import pytest
import torch

from lmcache_b200.codec import paged_layout, strided_slots

import paged_edges as P


def _bits(n, es, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n * es,), dtype=torch.uint8, generator=g).view(P.bits_dtype(es))


def _hand_split(K, V, nb, bs, H, D, x):
    """a split pair filled element by element from [nb * bs, H, D] rows (vLLM's PagedAttention layout)"""
    key = torch.empty(nb, H, D // x, bs, x, dtype=K.dtype)
    value = torch.empty(nb, H, D, bs, dtype=V.dtype)
    for s in range(nb * bs):
        b, o = divmod(s, bs)
        for h in range(H):
            for d in range(D):
                key[b, h, d // x, o, d % x] = K[s, h, d]
                value[b, h, d, o] = V[s, h, d]
    return key, value


@pytest.mark.parametrize("dtype,es", [(torch.bfloat16, 2), (torch.float8_e4m3fn, 1)])
@pytest.mark.parametrize("bs", [1, 3, 4])
def test_ref_rows_split_matches_hand_built_cache(dtype, es, bs):
    nb, H, D = 3, 2, 32
    x = 16 // es
    K, V = (_bits(nb * bs * H * D, es, s).view(nb * bs, H, D) for s in (1, 2))
    key, value = _hand_split(K, V, nb, bs, H, D, x)
    lay = paged_layout(key.view(dtype), value.view(dtype))
    assert (lay.kind, lay.nb, lay.bs, lay.H, lay.D, lay.x) == ("split", nb, bs, H, D, x)
    rk, rv = P.ref_rows(lay, key, value)
    assert torch.equal(rk, K) and torch.equal(rv, V)
    # the inverse writes the same elements back
    k2, v2 = torch.zeros_like(key), torch.zeros_like(value)
    P.ref_write_rows(lay, k2, v2, K, V)
    assert torch.equal(k2, key) and torch.equal(v2, value)


@pytest.mark.parametrize("planes", [2, 3])
@pytest.mark.parametrize("bs", [1, 4])
def test_ref_rows_strided_matches_hand_built_cache_and_strided_slots(planes, bs):
    """FlashInfer's kv[:, 0] / kv[:, 1] of a [nb, 2, bs, H, D] cache, and of a padded [nb, 3, bs, H, D] allocation"""
    nb, H, D = 4, 2, 16
    K, V = (_bits(nb * bs * H * D, 2, s).view(nb * bs, H, D) for s in (3, 4))
    alloc = _bits(nb * planes * bs * H * D, 2, 5).view(nb, planes, bs, H, D)
    spare = alloc[:, 2:].clone()
    for s in range(nb * bs):
        b, o = divmod(s, bs)
        alloc[b, 0, o] = K[s]
        alloc[b, 1, o] = V[s]
    key, value = alloc[:, 0], alloc[:, 1]
    lay = paged_layout(key.view(torch.bfloat16), value.view(torch.bfloat16))
    assert (lay.kind, lay.bs, lay.rows_per_block) == ("strided", bs, planes * bs)
    rk, rv = P.ref_rows(lay, key, value)
    assert torch.equal(rk, K) and torch.equal(rv, V)
    # codec.strided_slots names the row of the cache's storage, counted from the key's first row, that holds each slot
    slots = torch.arange(nb * bs)
    flat = alloc.view(-1, H, D)
    assert torch.equal(flat[strided_slots(slots, bs, lay.rows_per_block)], K)
    assert torch.equal(flat[bs + strided_slots(slots, bs, lay.rows_per_block)], V)
    P.ref_write_rows(lay, key, value, torch.zeros_like(K), torch.zeros_like(V))
    assert int(alloc[:, :2].count_nonzero()) == 0 and torch.equal(alloc[:, 2:], spare)


def test_ref_rows_flash_is_the_rows():
    nb, bs, H, D = 3, 4, 2, 8
    K, V = (_bits(nb * bs * H * D, 2, s).view(nb, bs, H, D) for s in (6, 7))
    lay = paged_layout(K.view(torch.float16), V.view(torch.float16))
    assert lay.kind == "flash"
    rk, rv = P.ref_rows(lay, K, V)
    assert torch.equal(rk, K.view(-1, H, D)) and torch.equal(rv, V.view(-1, H, D))


def _caches(lay, L, es, seed, fill=None):
    """L (key, value) pairs in `lay` and the allocations behind them (a strided pair shares one [nb, R, bs, H, D])"""
    n = lay.nb * lay.bs * lay.H * lay.D
    caches, allocs = [], []
    for l in range(L):
        if lay.kind == "split":
            key = _bits(n, es, seed + 2 * l).view(lay.nb, lay.H, lay.D // lay.x, lay.bs, lay.x).clone()
            value = _bits(n, es, seed + 2 * l + 1).view(lay.nb, lay.H, lay.D, lay.bs).clone()
            allocs += [key, value]
        else:
            alloc = _bits(n * lay.rows_per_block // lay.bs, es, seed + l).view(lay.nb, -1, lay.bs, lay.H, lay.D).clone()
            key, value = alloc[:, 0], alloc[:, 1]
            allocs.append(alloc)
        caches.append((key, value))
    if fill is not None:
        for a in allocs:
            a.fill_(fill)
    return caches, allocs


def _layout(kind, nb, bs, H, D, es, rpb=None):
    x = 16 // es
    return P.PagedLayoutLike(kind, nb, bs, H, D, rpb or bs, x if kind == "split" else 0)


@pytest.mark.parametrize("kind,rpb_mult", [("split", 1), ("strided", 2), ("strided", 3)])
@pytest.mark.parametrize("es", [1, 2])
@pytest.mark.parametrize("slots_kind,T,tok_begin,cs,layers", [
    ("vllm", 53, 0, 16, None), ("perm", 61, 5, 24, (1, 3)), ("shift", 40, 3, 7, (2, 3)), ("alt", 64, 16, 64, None)])
def test_ref_pack_then_unpack_is_the_identity_on_the_addressed_elements(kind, rpb_mult, es, slots_kind, T, tok_begin,
                                                                          cs, layers):
    L, nb, bs, H, D = 3, 12, 8, 2, 32
    lay = _layout(kind, nb, bs, H, D, es, rpb_mult * bs)
    src, _ = _caches(lay, L, es, seed=10)
    slots = P.make_slots(slots_kind, T, nb, bs, seed=T)
    blobs = P.ref_pack(lay, src, slots, tok_begin, cs, layers)
    # chunk shapes: chunk_tokens each, a ragged last one
    a, b = layers or (0, L)
    n_tok = T - tok_begin
    assert [bl.shape for bl in blobs] == [(b - a, 2, min(cs, n_tok - j * cs), H, D) for j in range(len(blobs))]
    # blob element (l, kv, tok, h, d) is the source rows' element at the token's slot
    srows = [P.ref_rows(lay, *p) for p in src]
    for j, bl in enumerate(blobs):
        for tok in (0, bl.shape[2] - 1):
            s = int(slots[tok_begin + j * cs + tok])
            assert torch.equal(bl[-1, 1, tok], srows[b - 1][1][s])
    sentinel = 0x5A if es == 1 else 0x5A5A
    dst, allocs = _caches(lay, L, es, seed=0, fill=sentinel)
    P.ref_unpack(lay, dst, slots, tok_begin, cs, blobs, layers)
    moved = torch.zeros(nb * bs, dtype=torch.bool)
    moved[slots[tok_begin:].long()] = True
    for l in range(L):
        got = P.ref_rows(lay, *dst[l])
        for i in range(2):
            if a <= l < b:
                assert torch.equal(got[i][moved], srows[l][i][moved])
                assert bool((got[i][~moved] == sentinel).all())
            else:
                assert bool((got[i] == sentinel).all())
    if kind == "strided":                      # the spare rows of a padded allocation are not rows of either cache
        assert all(bool((al[:, 2:] == sentinel).all()) for al in allocs)
    assert all(torch.equal(x, y) for x, y in zip(P.ref_pack(lay, dst, slots, tok_begin, cs, layers), blobs))


def test_launch_model_by_hand():
    m = P.launch_model
    # value vector bytes: 16 when bs * es % 16 == 0, else 8 when bs * es % 8 == 0 (8, 24, 40 bytes), else 0
    for es, bs, vw in ((2, 8, 16), (2, 4, 8), (2, 12, 8), (2, 20, 8), (1, 8, 8), (1, 24, 8), (1, 16, 16),
                       (2, 1, 0), (2, 2, 0), (2, 3, 0), (1, 4, 0), (1, 12, 0)):
        assert m(es, bs, 2, 64, table=True).vw == vw, (es, bs)
    # heads per unit: the largest divisor of H whose hb * bs * D * es fits 16 KB
    for es, bs, H, D, hb in ((2, 16, 6, 128, 3), (2, 16, 12, 64, 6), (2, 16, 40, 80, 5), (2, 16, 8, 128, 4),
                             (1, 32, 6, 128, 3), (2, 16, 7, 128, 1), (2, 256, 8, 128, 1), (1, 8, 32, 64, 32)):
        lc = m(es, bs, H, D, table=True)
        assert (lc.hb, lc.nhb) == (hb, H // hb), (es, bs, H, D)
    lc = m(2, 256, 2, 128, table=True)
    assert (lc.pitch, lc.smem, lc.opt_in, lc.refused) == (272, 256 * 272, True, False)
    lc = m(2, 256, 1, 256, table=True)
    assert (lc.smem, lc.opt_in) == (256 * 528, True)
    lc = m(2, 512, 1, 256, table=True)
    assert (lc.vw_bs, lc.vw, lc.smem, lc.refused) == (16, 0, 0, True)
    assert m(2, 16, 2, 64, table=True).smem == 2 * 16 * 144 and not m(2, 16, 2, 64, table=True).opt_in
    # whole-launch alignment fallbacks: the contiguous form's buffer and stride, either form's planes
    assert m(2, 16, 2, 64, table=False, chunk_off=2, stride=4096).vw == 0
    assert m(2, 16, 2, 64, table=False, chunk_off=0, stride=4104).vw == 0
    assert m(2, 16, 2, 64, table=True, plane_off=8).vw == 0
    assert m(2, 16, 2, 64, table=True, chunk_off=2, stride=4104).vw == 16     # a table's entries are checked per chunk


def test_group_paths_by_hand():
    lc = P.launch_model(2, 4, 1, 64, table=True)
    slots = [8, 9, 10, 11,  13, 14, 15, 16,  3, 2, 1, 0,  23, 22, 21, 20,  40, 41, 42, 43,  4, 5]
    paths = P.group_paths(lc, slots, tok_begin=4, chunk_tokens=6, table_offs=None)
    # chunks hold call tokens 4 .. 9, 10 .. 15, 16 .. 21.  The launch starts at group 1 (tok_begin // bs), a run from
    # slot 13; group 2 (8 .. 11) crosses a chunk boundary; group 3 is block 5 scrambled; group 4 a tile; group 5 ragged
    assert paths == [(4, "run_off_block"), (8, "chunk_boundary"), (12, "permuted_block"), (16, "tile"), (20, "edge")]
    assert P.group_paths(lc, slots, tok_begin=3, chunk_tokens=6)[0] == (0, "edge")
    paths = P.group_paths(lc, slots, tok_begin=0, chunk_tokens=4, table_offs=(0, 0, 0, 0, 2))
    assert paths[4] == (16, "table_entry") and paths[0] == (0, "tile")


def test_cases_stay_inside_the_kernel_contract():
    names = set()
    for c in P.CASES:
        assert c.name not in names
        names.add(c.name)
        s = P.make_slots(c.slots, c.T, c.nb, c.bs, c.seed)
        assert s.numel() == c.T and int(s.min()) >= 0 and int(s.max()) < c.nb * c.bs
        assert torch.unique(s).numel() == c.T                         # an unpack writes each row once
        assert c.D % (16 // c.es) == 0 and 0 <= c.tok_begin < c.T
        assert 0 <= c.layers[0] < c.layers[1] <= c.L
        # misalignments are element-aligned: the element-wise path's accesses stay aligned
        assert all(o % c.es == 0 for o in (c.chunk_off, c.stride_pad, c.plane_off) + c.table_offs)


def test_coverage_is_complete():
    cov = P.coverage(sms=P.H100_SMS)
    missing = sorted(k for k, v in cov.items() if not v)
    assert not missing, "branches no case reaches: " + ", ".join(f"{b} ({d}, {es}-byte)" for b, d, es in missing)
    assert {k[0] for k in cov} == set(P.BRANCHES)
