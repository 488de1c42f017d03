"""CPU: the numpy restatement of the int4 weight format (tests/int4_ref.py) against hand-worked groups: the packed byte
order, ties to even, the clamp after the scale is rounded, and a zero group. tests/test_int4_gpu.py trusts it."""
import numpy as np

import int4_ref as R


def test_pack_places_each_code_where_the_header_says():
    q = np.zeros((2, 128), np.int8)
    q[0, 8] = 3             # row 0, k = 8: block 0, h = 1, t = 0, b = 0 -> byte 1, low nibble
    q[1, 1] = -5            # row 1, k = 1: h = 0, t = 0, b = 1 -> byte 2, high nibble
    q[0, 16 + 7] = -7       # row 0, k = 23: block 1, k' = 7 = 8*0 + 2*3 + 1 -> byte 16 + 4*3 + 2 = 30, low nibble
    q[1, 127] = 7           # row 1, k = 127: block 7, k' = 15 = 8 + 2*3 + 1 -> byte 112 + 12 + 2 + 1 = 127, high nibble
    p = R.pack(q)
    want = np.full((1, 128), 0x88, np.uint8)
    want[0, 1] = 0x80 | (3 + 8)
    want[0, 2] = ((-5 + 8) << 4) | 0x8
    want[0, 30] = 0x80 | (-7 + 8)
    want[0, 127] = ((7 + 8) << 4) | 0x8
    assert np.array_equal(p, want)
    # the first word: bytes 0..3 hold k = 0, 8, 1, 9 of rows 0 (low) and 1 (high)
    q2 = np.zeros((2, 128), np.int8)
    q2[0, [0, 8, 1, 9]] = [1, 2, 3, 4]
    q2[1, [0, 8, 1, 9]] = [-1, -2, -3, -4]
    assert R.pack(q2)[0, :4].tolist() == [(7 << 4) | 9, (6 << 4) | 10, (5 << 4) | 11, (4 << 4) | 12]


def test_pack_round_trips():
    q = np.random.default_rng(0).integers(-7, 8, size=(24, 384)).astype(np.int8)
    assert np.array_equal(R.unpack(R.pack(q)), q)


def test_ties_round_to_even():
    w = np.zeros((8, 128), np.float32)
    vals = [7.0, 0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 6.5, -6.5, 3.5, -3.5]   # absmax 7: s = 1 exactly
    w[0, :len(vals)] = vals
    q, s = R.quantize(w)
    assert s[0, 0] == 1.0
    assert q[0, :len(vals)].tolist() == [7, 0, 2, 2, 0, -2, -2, 6, -6, 4, -4]


def test_clamp_after_scale_rounding():
    # a = 7.0625 (a bf16): a / 7 = 1.00893 rounds down to the bf16 1.0078125, so a / s = 7.0078 > 7; q stays at +-7
    w = np.zeros((8, 128), np.float32)
    w[0, 0], w[0, 5], w[0, 6] = 7.0625, -7.0625, 3.5
    q, s = R.quantize(w)
    assert s[0, 0] == np.float32(1.0078125) and 7.0625 / s[0, 0] > 7
    assert q[0, [0, 5, 6]].tolist() == [7, -7, 3]      # 3.5 / 1.0078125 = 3.473 -> 3
    assert R.dequantize(q, s)[0, 0] == R.bf16_rne(np.float32(7 * 1.0078125))


def test_zero_group_gives_zero_scale_and_codes():
    w = np.zeros((8, 256), np.float32)
    w[0, 128:] = np.linspace(-1, 1, 128, dtype=np.float32)
    q, s = R.quantize(w)
    assert s[0, 0] == 0 and not q[0, :128].any()
    assert s[0, 1] == R.bf16_rne(np.float32(1.0) / np.float32(7.0)) and np.abs(q[0, 128:]).max() == 7
    assert np.array_equal(R.pack(q)[0, :128], np.full(128, 0x88, np.uint8))


def test_bf16_rne_ties_to_even():
    one = np.float32(1.0)
    ulp = np.float32(2.0 ** -7)
    assert R.bf16_rne(np.float32(one + ulp / 2)) == one                 # tie, 1.0 is even
    assert R.bf16_rne(np.float32(one + ulp * 1.5)) == one + 2 * ulp     # tie, 1 + 2 ulp is even
    assert R.bf16_rne(np.float32(one + ulp / 2 + 2.0 ** -20)) == one + ulp
