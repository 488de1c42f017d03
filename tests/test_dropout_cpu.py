"""CPU: the numpy Philox4x32-10 the dropout tests rebuild masks with (Random123 known-answer vectors), the counter layouts of
include/fsb200.h, and the effective drop rate of the 8-bit threshold."""
import numpy as np
import pytest

import philox_ref as R


@pytest.mark.parametrize("key,ctr,want", [
    ((0, 0), (0, 0, 0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff, 0xffffffff), (0xffffffff,) * 4, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0xa4093822, 0x299f31d0), (0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(key, ctr, want):
    got = R.philox4x32_10(ctr, key)
    assert tuple(int(x) for x in got) == want


@pytest.mark.parametrize("p", [0.0, 0.1, 0.2, 0.5, 0.9, 0.999])
def test_effective_rate_within_2_pow_minus_9(p):
    assert abs(R.p_eff(p) - p) <= 2.0 ** -9


def test_hidden_layout_uses_one_call_per_16_columns():
    seed, stream = 0x0123456789abcdef, (5 << 32) | 7
    keep = R.hidden_keep(seed, stream, 3, 40, 0.5)
    w = R.philox4x32_10((2, 1, 7, 5), (0x89abcdef, 0x01234567))   # row 1, columns 32..47
    byte = lambda col: (int(w[(col % 16) // 4]) >> (8 * (col % 4))) & 0xFF
    for col in range(32, 40):
        assert keep[1, col] == (byte(col) >= 128)


def test_attention_layout_matches_the_documented_counter():
    seed, stream, H = 99, 3, 3
    keep = R.attn_keep(seed, stream, 2, H, 40, 40, 0.5)
    for (b, h, q, k) in [(0, 0, 0, 0), (1, 2, 9, 17), (0, 1, 33, 8), (1, 0, 31, 39)]:
        qa, qh, qs, qp = q >> 4, (q >> 3) & 1, (q >> 1) & 3, q & 1
        ka, kh, ks, kp = k >> 4, (k >> 3) & 1, (k >> 1) & 3, k & 1
        w = R.philox4x32_10(((ka * 4 + ks) | ((qa * 4 + qs) << 16), b * H + h, 3, 0), (99, 0))
        r = (int(w[2 * qp + kp]) >> (8 * (2 * qh + kh))) & 0xFF
        assert keep[b, h, q, k] == (r >= 128)


def test_masks_have_the_expected_rate_and_differ_between_streams():
    p = 0.1
    a = R.hidden_keep(1, 0, 512, 1024, p)
    b = R.hidden_keep(1, 1, 512, 1024, p)
    n, pe = a.size, R.p_eff(p)
    assert abs((~a).mean() - pe) < 5 * np.sqrt(pe * (1 - pe) / n)
    agree = (a == b).mean()
    want = pe * pe + (1 - pe) ** 2
    assert abs(agree - want) < 5 * np.sqrt(want * (1 - want) / n)
