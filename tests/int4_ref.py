"""The int4 weight format of include/fsb200.h (fsb_quantize_w4) restated in numpy float32, without the library: group-wise
scales, the 4-bit codes, their packed byte layout and the dequantised weight W^ = bf16(q * s). tests/test_int4_cpu.py pins
it to hand-worked groups; tests/test_int4_gpu.py checks the CUDA quantiser and GEMM against it."""
import numpy as np

GROUP = 128


def bf16_rne(x):
    """float32 -> the nearest bf16 (ties to even), returned as float32. Finite inputs only."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    r = (b + np.uint32(0x7FFF) + ((b >> np.uint32(16)) & np.uint32(1))) & np.uint32(0xFFFF0000)
    return r.view(np.float32)


def quantize(w):
    """w float32 [n, k] (bf16 values) -> (q int8 [n, k] in [-7, 7], s float32 [n, k / 128] holding bf16 values):
    s = bf16(absmax(group) / 7), q = clamp(rint(w / s), -7, 7), q = 0 where s == 0."""
    w = np.asarray(w, dtype=np.float32)
    n, k = w.shape
    g = w.reshape(n, k // GROUP, GROUP)
    s = bf16_rne(np.abs(g).max(axis=2) / np.float32(7.0))
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.rint(g / s[:, :, None])
    q = np.clip(r, -7, 7)
    q[np.broadcast_to(s[:, :, None] == 0, q.shape)] = 0
    return q.reshape(n, k).astype(np.int8), s


def pack(q):
    """q int8 [n, k] -> uint8 [n / 2, k]: line p holds rows 2p (low nibble) and 2p + 1 (high nibble) as q + 8; inside each
    16-k block, byte 4t + 2b + h holds k = 8h + 2t + b."""
    n, k = q.shape
    u = (q.astype(np.int16) + 8).astype(np.uint8).reshape(n // 2, 2, k // 16, 2, 4, 2)   # [p, row, block, h, t, b]
    u = u.transpose(0, 2, 4, 5, 3, 1)                                                  # [p, block, t, b, h, row]
    return (u[..., 0] | (u[..., 1] << 4)).reshape(n // 2, k)


def unpack(packed):
    """The inverse of pack."""
    p2, k = packed.shape
    b = packed.reshape(p2, k // 16, 4, 2, 2)                                           # [p, block, t, b, h]
    u = np.stack([b & 0xF, b >> 4], axis=-1).astype(np.int16) - 8                      # [p, block, t, b, h, row]
    return u.transpose(0, 5, 1, 4, 2, 3).reshape(2 * p2, k).astype(np.int8)


def dequantize(q, s):
    """W^ = bf16(q * s) as float32: the exact product (at most 11 significant bits, exact in float32) rounded once."""
    n, k = q.shape
    prod = q.astype(np.float32).reshape(n, k // GROUP, GROUP) * s[:, :, None]
    return bf16_rne(prod).reshape(n, k)
