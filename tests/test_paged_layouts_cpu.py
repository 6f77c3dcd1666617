"""CPU: the paged cache layouts KvView.from_paged recognises (codec.paged_layout), the slot remap of the block-strided
(FlashInfer) layout, and the address formulas of the split (PagedAttention / xFormers) layout that the mover's
B200KV_KV_PAGED_SPLIT descriptor implements.  Shapes and strides only: no device needed."""
import pytest
import torch

from lmcache_b200.codec import paged_layout, strided_slots

ONE_BYTE = [torch.uint8, torch.float8_e4m3fn, torch.float8_e5m2]


def _x(dtype):
    return 16 // torch.empty((), dtype=dtype).element_size()


def split_kv_cache(kv_cache, H, D, x):
    """vLLM's PagedAttention.split_kv_cache on a [2, nb, bs * H * D] layer cache"""
    nb = kv_cache.shape[1]
    key = kv_cache[0].view(nb, H, D // x, -1, x)
    value = kv_cache[1].view(nb, H, D, -1)
    return key, value


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16] + ONE_BYTE)
def test_recognises_the_three_layouts(dtype):
    nb, bs, H, D = 5, 16, 2, 64
    flash = torch.empty(nb, bs, H, D, dtype=dtype)
    assert paged_layout(flash, flash.clone()) == ("flash", nb, bs, H, D, bs, 0, )
    flat = torch.empty(nb * bs, H, D, dtype=dtype)
    assert paged_layout(flat, flat.clone()).kind == "flash"
    kv = torch.empty(nb, 2, bs, H, D, dtype=dtype)
    lay = paged_layout(kv[:, 0], kv[:, 1])
    assert lay == ("strided", nb, bs, H, D, 2 * bs, 0)
    x = _x(dtype)
    k, v = split_kv_cache(torch.empty(2, nb, bs * H * D, dtype=dtype), H, D, x)
    assert paged_layout(k, v) == ("split", nb, bs, H, D, bs, x)


def test_refusals():
    nb, bs, H, D = 4, 16, 2, 64
    bf = torch.bfloat16
    k, v = split_kv_cache(torch.empty(2, nb, bs * H * D, dtype=bf), H, D, 8)
    with pytest.raises(ValueError, match="disagree"):                  # nb
        paged_layout(k, v[:nb - 1])
    with pytest.raises(ValueError, match="disagree"):                  # bs
        paged_layout(k, torch.empty(nb, H, D, bs // 2, dtype=bf))
    with pytest.raises(ValueError, match="disagree"):                  # H
        paged_layout(k, torch.empty(nb, H + 1, D, bs, dtype=bf))
    with pytest.raises(ValueError, match="disagree"):                  # D
        paged_layout(k, torch.empty(nb, H, D + 8, bs, dtype=bf))
    with pytest.raises(ValueError, match="disagree"):                  # flash pair of different shapes
        paged_layout(torch.empty(nb, bs, H, D, dtype=bf), torch.empty(nb, bs, H, D + 8, dtype=bf))
    with pytest.raises(ValueError, match="x = 8"):                     # x of another element size
        paged_layout(torch.empty(nb, H, D // 16, bs, 16, dtype=bf), torch.empty(nb, H, D, bs, dtype=bf))
    with pytest.raises(ValueError, match="D % x"):                     # fp8: D = 72 is not a multiple of x = 16
        paged_layout(torch.empty(nb, H, 4, bs, 18, dtype=torch.uint8), torch.empty(nb, H, 72, bs, dtype=torch.uint8))
    with pytest.raises(ValueError, match="dtype the mover moves"):     # split float32
        paged_layout(torch.empty(nb, H, D // 4, bs, 4), torch.empty(nb, H, D, bs))
    kv = torch.empty(nb, 2, bs, H, D)
    with pytest.raises(ValueError, match="dtype the mover moves"):     # strided float32
        paged_layout(kv[:, 0], kv[:, 1])
    assert paged_layout(torch.empty(nb, bs, H, D), torch.empty(nb, bs, H, D)).kind == "flash"   # today's, any dtype
    with pytest.raises(ValueError, match="dtype"):
        paged_layout(k, v.view(torch.float16))
    with pytest.raises(ValueError, match="contiguous"):                # a split pair that is not in place
        paged_layout(k.transpose(0, 1).contiguous().transpose(0, 1), v)
    with pytest.raises(ValueError, match="block-strided"):             # rows that are not block-strided
        t = torch.empty(nb, bs, H, 2 * D, dtype=bf)[..., :D]
        paged_layout(t, t)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.uint8])
@pytest.mark.parametrize("bs", [8, 16, 32])
def test_strided_slot_remap_matches_byte_offsets(dtype, bs):
    nb, H, D = 7, 3, 32
    kv = torch.empty(nb, 2, bs, H, D, dtype=dtype)
    es = kv.element_size()
    for kvi in range(2):
        t = kv[:, kvi]
        lay = paged_layout(t, t)
        slots = torch.randperm(nb * bs, generator=torch.Generator().manual_seed(bs))
        got = strided_slots(slots, lay.bs, lay.rows_per_block)
        for s, r in zip(slots.tolist(), got.tolist()):
            off = t[s // bs, s % bs].data_ptr() - t.data_ptr()         # brute force: where the row's bytes are
            assert off == r * H * D * es


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16] + ONE_BYTE)
@pytest.mark.parametrize("bs", [8, 16])
@pytest.mark.parametrize("D", [64, 128])
def test_split_address_formulas(dtype, bs, D):
    """include/b200kv.h's two formulas for B200KV_KV_PAGED_SPLIT, as torch, against split_kv_cache's views"""
    nb, H = 3, 2
    x = _x(dtype)
    n = nb * bs * H * D
    kv_cache = torch.arange(2 * n, dtype=torch.int64).view(2, nb, bs * H * D)
    key, value = split_kv_cache(kv_cache, H, D, x)
    s = torch.arange(nb * bs).view(-1, 1, 1)
    h = torch.arange(H).view(1, -1, 1)
    d = torch.arange(D).view(1, 1, -1)
    b, o = s // bs, s % bs
    koff = ((b * H + h) * (D // x) + d // x) * bs * x + o * x + d % x
    voff = ((b * H + h) * D + d) * bs + o
    assert torch.equal(kv_cache[0].flatten()[koff], key[b, h, d // x, o, d % x])
    assert torch.equal(kv_cache[1].flatten()[voff], value[b, h, d, o])
    # every element is addressed exactly once
    assert torch.equal(koff.flatten().sort().values, torch.arange(n))
    assert torch.equal(voff.flatten().sort().values, torch.arange(n))
