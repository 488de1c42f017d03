"""numpy restatement of the FP8 quantiser of include/fsb200.h (fsb_fp8_quantize) and the exact-GEMM constructions the FP8 tests
share. Pure numpy: the CPU tests check it against torch's casts and the GPU tests check the kernels against it."""
import numpy as np

# name -> (exponent bits, mantissa bits, exponent bias, largest finite value, its code, exponent of that value)
FORMATS = {"e4m3": (4, 3, 7, 448.0, 0x7E, 8), "e5m2": (5, 2, 15, 57344.0, 0x7B, 15)}
NAN_CODE = 0x7F   # the NaN both casts produce (sign dropped)


def encode(x, fmt):
    """fp32 values -> uint8 codes as cvt.rn.satfinite.{e4m3,e5m2}x2.f32 produces them: round to nearest even on the format's
    grid (subnormals included), magnitudes beyond the largest finite value (and inf) saturate to it, the sign of a zero is
    kept, NaN gives NAN_CODE."""
    _, mb, bias, fmax, maxcode, _ = FORMATS[fmt]
    x = np.asarray(x, dtype=np.float32)
    a = np.abs(x).astype(np.float64)
    sign = (np.signbit(x).astype(np.uint8) << 7)
    emin = 1 - bias                                     # exponent of the smallest normal
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        _, e = np.frexp(np.where(np.isfinite(a) & (a > 0), a, 1.0))
        e = np.maximum(e - 1, emin)                     # a = m 2^e, m in [1, 2) (subnormal range: the fixed step 2^(emin - mb))
        ulp = np.ldexp(1.0, e - mb)
        q = np.rint(a / ulp) * ulp                      # exact in float64; rint is round-half-even
        sat = ~(q <= fmax)                              # beyond the largest finite value, or inf
        q = np.where(sat, fmax, q)
        _, e2 = np.frexp(np.where(q > 0, q, 1.0))
        e2 = e2 - 1
        normal = q >= np.ldexp(1.0, emin)
        mant = np.where(normal, q / np.ldexp(1.0, e2 - mb) - 2 ** mb, q / np.ldexp(1.0, emin - mb))
        expf = np.where(normal, e2 + bias, 0)
        code = (expf.astype(np.int64) << mb) | np.rint(mant).astype(np.int64)
    code = np.where(sat, maxcode, code).astype(np.uint8) | sign
    return np.where(np.isnan(x), NAN_CODE, code).astype(np.uint8)


def decode(codes, fmt):
    """uint8 codes -> float64 values (NaN for the NaN codes)."""
    eb, mb, bias, _, _, _ = FORMATS[fmt]
    c = np.asarray(codes, dtype=np.int64)
    s = np.where(c & 0x80, -1.0, 1.0)
    ex = (c >> mb) & ((1 << eb) - 1)
    m = c & ((1 << mb) - 1)
    v = np.where(ex == 0, np.ldexp(m.astype(np.float64), 1 - bias - mb),
                 np.ldexp((m + (1 << mb)).astype(np.float64), ex - bias - mb))
    nan = ((c & 0x7F) == 0x7F) if fmt == "e4m3" else (ex == (1 << eb) - 1) & (m != 0)
    inf = (fmt == "e5m2") & (ex == (1 << eb) - 1) & (m == 0)
    v = np.where(inf, np.inf, v)
    return np.where(nan, np.nan, s * v)


def scale_exp(amax, fmt):
    """-> (e, scale_inv) of the scale 2^e: e = floor(log2(fmax / amax)) clamped to [-126, 126]; amax == 0 gives e = 0;
    a non-finite amax gives e = 0 and scale_inv = NaN."""
    a = np.float32(amax)
    if not np.isfinite(a):
        return 0, np.float32(np.nan)
    if a == 0:
        return 0, np.float32(1.0)
    m, ea = np.frexp(np.float64(a))                     # a = m 2^ea, m in [0.5, 1)
    e = FORMATS[fmt][5] - (ea - 1) - (1 if 2 * m > 1.75 else 0)
    e = int(min(max(e, -126), 126))
    return e, np.float32(np.ldexp(1.0, -e))


def quantize(x, fmt):
    """bf16 values (as fp32) [rows, cols] -> (codes [rows, cols], transposed codes, scale_inv) as fsb_fp8_quantize writes them."""
    x = np.asarray(x, dtype=np.float32)
    with np.errstate(invalid="ignore"):
        amax = np.max(np.abs(x)) if not np.isnan(x).any() else np.float32(np.nan)
    e, sinv = scale_exp(amax, fmt)
    y = encode(x * np.float32(np.ldexp(1.0, e)), fmt)
    return y, np.ascontiguousarray(y.T), sinv


def exact_operands(m, n, k, seed, positive=False):
    """Small-integer GEMM operands whose every product and sum is exact: A [m, k], B [n, k] int64 in [-3, 3] (in [1, 3] when
    `positive`), each value exact in e4m3 and e5m2. A 128-deep block sum stays within 128 * 9 = 1152 < 2^11."""
    rng = np.random.default_rng(seed)
    lo = 1 if positive else -3
    return rng.integers(lo, 4, size=(m, k)), rng.integers(lo, 4, size=(n, k))


def block_sums(a, b, block=128):
    """[k / block, m, n] int64 partial sums of a @ b.T over consecutive k-blocks (the GEMM's promotion interval)."""
    k = a.shape[1]
    return np.stack([a[:, j:j + block] @ b[:, j:j + block].T for j in range(0, k, block)])
