"""CPU: the rope shift's numpy statement, the segment plan and RopeSpec (no GPU needed)."""
import numpy as np
import pytest
import torch

from rope_ref import angles, partner, rotate, rotate_complex, tolerance, ulp


def _inv(rotary_dim, base=10000.0):
    return (1.0 / (base ** (np.arange(0, rotary_dim, 2, dtype=np.float32) / np.float32(rotary_dim)))).astype(np.float32)


CASES = [(128, 128, "neox", 0), (128, 128, "gptj", 0), (128, 64, "neox", 0), (128, 32, "gptj", 16),
         (576, 64, "gptj", 512), (576, 64, "neox", 512), (80, 36, "neox", 4)]


@pytest.mark.parametrize("D,rd,style,offset", CASES)
def test_statement_equals_complex_multiplication(D, rd, style, offset):
    rng = np.random.default_rng(D + rd + offset)
    k = rng.standard_normal((5, 3, D))
    inv = _inv(rd)
    for shift in (1, 255, 4096, 65535, np.array([0, 1, 7, 65535, 1 << 20])):
        np.testing.assert_allclose(rotate(k, shift, inv, rd, style, offset),
                                   rotate_complex(k, shift, inv, rd, style, offset), rtol=0, atol=1e-12)


@pytest.mark.parametrize("D,rd,style,offset", CASES)
def test_statement_touches_only_the_rotary_channels_and_keeps_norms(D, rd, style, offset):
    rng = np.random.default_rng(1)
    k = rng.standard_normal((4, 2, D))
    out = rotate(k, 4096, _inv(rd), rd, style, offset)
    outside = np.ones(D, dtype=bool)
    outside[offset:offset + rd] = False
    assert np.array_equal(out[..., outside], k[..., outside])
    p = partner(rd, style, offset, D)
    pair_norm = lambda t: t ** 2 + t[..., p] ** 2          # noqa: E731
    np.testing.assert_allclose(pair_norm(out), pair_norm(k), rtol=1e-12)


@pytest.mark.parametrize("D,rd,style,offset", CASES)
def test_shift_composes_with_the_stored_position(D, rd, style, offset):
    """R(s)·R(i)·k = R(s + i)·k in float64: a key stored at position i and shifted by s is the key at s + i"""
    rng = np.random.default_rng(2)
    k = rng.standard_normal((6, 2, D))
    inv = _inv(rd)
    i = np.array([0, 1, 5, 300, 2047, 9000])
    for s in (1, 255, 4096, 65535):
        stored = rotate(k, i, inv, rd, style, offset)
        np.testing.assert_allclose(rotate(stored, s, inv, rd, style, offset), rotate(k, i + s, inv, rd, style, offset),
                                   rtol=0, atol=1e-9)


def test_angles_are_float64_products_of_float32_frequencies():
    inv = np.array([1.0, 0.1, 1e-4], dtype=np.float32)
    a = angles(65536, inv)
    assert a.dtype == np.float64
    assert a[0] == 65536.0 and a[1] == 65536.0 * float(np.float32(0.1))
    # an fp32 product at a shift of 65535 would be off by more than 1e-4 rad for some frequency: beyond a bf16 ulp
    # of the small keys' rotations
    inv = _inv(128)
    a = angles(65535, inv)
    assert np.max(np.abs((np.float32(65535) * inv).astype(np.float64) - a)) > 1e-4


def test_ulp_and_tolerance():
    assert ulp(1.0, "bfloat16") == 2.0 ** -7 and ulp(1.0, "float16") == 2.0 ** -10
    assert ulp(0.0, "float16") == 2.0 ** -24 and ulp(3.0, "bfloat16") == 2.0 ** -6
    t = tolerance(np.array([1.0]), np.array([1.0]), np.array([1.0]), np.array([1.0]), "bfloat16")
    assert t[0] == 2.0 ** -7 + 2.0 ** -20


# ---------------------------------------------------------------------------------------------- the plan
def test_plan_unaligned_segments_and_short_last_chunk():
    from lmcache_b200.rope import plan_segments
    plans = plan_segments(1000, [(700, 1000), (10, 300), (300, 301)], 256)
    assert [(p.index, p.start, p.end, p.shift) for p in plans] == [(1, 10, 300, 10), (2, 300, 301, 300),
                                                                   (0, 700, 1000, 700)]
    assert [(p.hash_begin, p.chunk_begin, p.n_chunks) for p in plans] == [(0, 0, 2), (290, 2, 1), (291, 3, 2)]
    assert plans[0].chunk_bounds(256) == [(10, 266), (266, 300)]
    assert plans[1].chunk_bounds(256) == [(300, 301)]
    assert plans[2].chunk_bounds(256) == [(700, 956), (956, 1000)]
    one = plan_segments(512, [(0, 512)], 256)
    assert one[0].shift == 0 and one[0].chunk_bounds(256) == [(0, 256), (256, 512)]


@pytest.mark.parametrize("segs,what", [([(0, 10), (9, 20)], "overlap"), ([(5, 5)], "empty"), ([(6, 5)], "empty"),
                                       ([(-1, 5)], "outside"), ([(90, 101)], "outside"),
                                       ([(0, 50), (60, 70), (40, 55)], "overlap"), ([(1, 2, 3)], "pair"),
                                       ([None], "pair")])
def test_plan_refusals(segs, what):
    from lmcache_b200.rope import plan_segments
    with pytest.raises(ValueError, match=what):
        plan_segments(100, segs, 16)


def test_hash_input_and_seg_of_tok():
    from lmcache_b200.rope import hash_input, plan_segments, seg_of_tok
    tokens = torch.arange(100)
    plans = plan_segments(100, [(50, 60), (0, 20), (70, 75)], 8)
    toks, offs = hash_input(tokens, plans)
    assert offs == [0, 20, 30, 35]
    assert toks.tolist() == list(range(0, 20)) + list(range(50, 60)) + list(range(70, 75))
    # segment at 0 and a segment with nothing written get no table row
    sot, lo, hi, shifts = seg_of_tok(100, [(plans[0], 16), (plans[1], 8), (plans[2], 0)])
    assert (lo, hi, shifts) == (50, 58, [50])
    assert sot == [0] * 8
    sot, lo, hi, shifts = seg_of_tok(100, [(plans[0], 20), (plans[1], 4), (plans[2], 5)])
    assert (lo, hi, shifts) == (50, 75, [50, 70])
    assert sot == [0] * 4 + [-1] * 16 + [1] * 5
    assert seg_of_tok(100, [(plans[0], 20)]) == ([], 0, 0, [])


# ---------------------------------------------------------------------------------------------- RopeSpec
def test_from_base_matches_vllm_formula():
    from lmcache_b200.rope import RopeSpec
    for rd, base in ((128, 10000.0), (64, 500000.0), (96, 1e6), (2, 10000.0)):
        spec = RopeSpec.from_base(rd, base)
        want = 1.0 / (base ** (np.arange(0, rd, 2, dtype=np.float32) / np.float32(rd)))
        assert spec.inv_freq.dtype == torch.float32 and spec.inv_freq.shape == (rd // 2,)
        np.testing.assert_allclose(spec.inv_freq.numpy(), want.astype(np.float32), rtol=3e-7)
        assert spec.style == "neox" and spec.offset == 0


def test_rope_spec_validation():
    from lmcache_b200.rope import RopeSpec
    inv = torch.ones(32, dtype=torch.float32)
    RopeSpec(64, inv, "gptj", 512).check(576)
    with pytest.raises(ValueError, match="do not fit"):
        RopeSpec(64, inv, "gptj", 513).check(576)
    with pytest.raises(ValueError, match="do not fit"):
        RopeSpec(64, inv).check(48)
    with pytest.raises(ValueError, match="even"):
        RopeSpec(63, torch.ones(31))
    with pytest.raises(ValueError, match="even"):
        RopeSpec(0, torch.ones(0))
    with pytest.raises(ValueError, match="style"):
        RopeSpec(64, inv, "glm")
    with pytest.raises(ValueError, match="offset"):
        RopeSpec(64, inv, "neox", -1)
    with pytest.raises(ValueError, match="float32"):
        RopeSpec(64, inv.double())
    with pytest.raises(ValueError, match="float32"):
        RopeSpec(64, torch.ones(31, dtype=torch.float32))
    with pytest.raises(ValueError, match="float32"):
        RopeSpec(64, [1.0] * 32)
