"""CPU checks of the FP8 recipe (include/fsb200.h, fsb_fp8_quantize / fsb_gemm_fp8): the numpy restatement of the casts
against torch's float8 dtypes, the per-tensor scale rule on hand-worked cases, and proofs that the GEMM tests' integer
constructions are exact (every 128-deep block sum below 2^11, every fp32 running sum below 2^24)."""
import numpy as np
import pytest
import torch

from fp8_ref import FORMATS, NAN_CODE, block_sums, decode, encode, exact_operands, quantize, scale_exp

TORCH = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}


def _all_bf16():
    """every finite bf16 value, as fp32"""
    v = (np.arange(1 << 16, dtype=np.uint32) << 16).view(np.float32)
    return v[np.isfinite(v)]


@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
def test_encode_matches_torch_on_every_in_range_bf16(fmt):
    fmax = FORMATS[fmt][3]
    v = _all_bf16()
    v = v[np.abs(v) <= fmax]   # beyond it torch's cast does not saturate (see below)
    want = torch.from_numpy(v).to(TORCH[fmt]).view(torch.uint8).numpy()
    got = encode(v, fmt)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, [(float(v[i]), int(got[i]), int(want[i])) for i in bad[:5]]
    # subnormals, signed zero and round-half-even are among the values above; pin a few by hand
    tiny = np.ldexp(1.0, 1 - FORMATS[fmt][2] - FORMATS[fmt][1])   # the smallest subnormal
    assert encode(np.float32([0.0, -0.0]), fmt).tolist() == [0x00, 0x80]
    assert encode(np.float32([tiny, tiny / 2, tiny * 1.5, -tiny / 4]), fmt).tolist() == [0x01, 0x00, 0x02, 0x80]


@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
def test_decode_inverts_encode(fmt):
    codes = np.arange(256, dtype=np.uint8)
    vals = decode(codes, fmt)
    fin = np.isfinite(vals)
    assert np.array_equal(encode(vals[fin].astype(np.float32), fmt), codes[fin])


@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
def test_saturation_and_nan(fmt):
    _, _, _, fmax, maxcode, _ = FORMATS[fmt]
    big = np.float32([fmax * 1.1, -fmax * 4, np.inf, -np.inf, 3e38])
    assert encode(big, fmt).tolist() == [maxcode, maxcode | 0x80, maxcode, maxcode | 0x80, maxcode]
    assert encode(np.float32([np.nan, -np.nan]), fmt).tolist() == [NAN_CODE, NAN_CODE]
    # torch's cast does not saturate: beyond the range it gives NaN (e4m3fn) or inf (e5m2), which the kernel never does
    t = torch.tensor([fmax * 4], dtype=torch.float32).to(TORCH[fmt]).float().item()
    assert not np.isfinite(t)
    # values that round onto the largest finite value from below
    below = np.float32(fmax - np.ldexp(1.0, FORMATS[fmt][5] - FORMATS[fmt][1] - 1) * 0.99)
    assert encode(np.float32([below]), fmt).tolist() == [maxcode]


def test_scale_rule_hand_cases():
    # amax = 0 -> scale 1; non-finite amax -> scale_inv NaN
    assert scale_exp(0.0, "e4m3") == (0, 1.0)
    for bad in (np.inf, np.nan):
        e, sinv = scale_exp(bad, "e4m3")
        assert e == 0 and np.isnan(sinv)
    # amax a power of two: 448 / 2 = 224 -> 2^7; 57344 / 1 -> 2^15
    assert scale_exp(2.0, "e4m3")[0] == 7 and scale_exp(1.0, "e5m2")[0] == 15
    # amax just above / below one: 448 / (1 + 2^-7) = 444.5 -> 2^8; 448 / (1 - 2^-8) = 449.8 -> 2^8
    assert scale_exp(1.0 + 2.0 ** -7, "e4m3")[0] == 8 and scale_exp(1.0 - 2.0 ** -8, "e4m3")[0] == 8
    # the boundary m = 1.75: amax = 448 -> 2^0, amax just above -> 2^-1
    assert scale_exp(448.0, "e4m3")[0] == 0 and scale_exp(np.nextafter(np.float32(448), np.float32(1e9)), "e4m3")[0] == -1
    assert scale_exp(57344.0, "e5m2")[0] == 0 and scale_exp(57345.0, "e5m2")[0] == -1
    # tiny amax: the scale clamps at 2^126 (scale and 1 / scale stay normal fp32)
    e, sinv = scale_exp(np.float32(2.0 ** -130), "e4m3")
    assert e == 126 and sinv == np.float32(2.0 ** -126)
    # huge amax: 448 / 3e38 ~ 2^-119.4 -> 2^-120
    assert scale_exp(np.float32(3e38), "e4m3")[0] == -120
    # after scaling, amax never exceeds the largest finite value and is at least half of it (unless clamped)
    rng = np.random.default_rng(0)
    for a in np.exp(rng.uniform(-80, 80, 2000)).astype(np.float32):
        for fmt in ("e4m3", "e5m2"):
            e, _ = scale_exp(a, fmt)
            s = np.ldexp(np.float64(a), e)
            assert s <= FORMATS[fmt][3] and (abs(e) == 126 or s > FORMATS[fmt][3] / 2), (a, fmt, e)


def test_quantize_layouts_and_zero():
    x = np.arange(32 * 16, dtype=np.float32).reshape(32, 16) - 200
    y, yt, sinv = quantize(x, "e4m3")
    assert np.array_equal(yt, y.T) and sinv == np.float32(1.0)   # amax 311: 448 / 311 = 1.44 -> scale 2^0
    y0, _, s0 = quantize(np.zeros((16, 16), np.float32), "e5m2")
    assert not y0.any() and s0 == 1.0


@pytest.mark.parametrize("m,n,k,positive", [(64, 48, 1024, False), (16, 16, 8192, True)])
def test_exact_gemm_constructions_are_exact(m, n, k, positive):
    """The GPU tests' exact inputs: every k-block partial sum below 2^11 in magnitude (exact in the tensor cores' reduced
    accumulator) and every fp32 running sum below 2^24; the all-positive k = 8192 case sums past 2^14, so a GEMM that did not
    promote its partial sums into fp32 would lose bits."""
    a, b = exact_operands(m, n, k, seed=k + m, positive=positive)
    for fmt in ("e4m3", "e5m2"):   # every value is exact in both formats
        assert np.array_equal(decode(encode(a.astype(np.float32), fmt), fmt), a)
    bs = block_sums(a, b)
    assert np.abs(bs).max() < 2 ** 11
    run = np.cumsum(bs, axis=0)
    assert np.abs(run).max() < 2 ** 24
    if positive:
        assert run[-1].min() > 2 ** 14
