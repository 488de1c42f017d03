"""The int8 weight format of include/fsb200.h (fsb_quantize_w8) restated in numpy float32, without the library. The GPU
tests check the CUDA quantiser against it."""
import numpy as np


def quantize(w):
    """The quantiser's contract in numpy float32: s = absmax / 127, q = clamp(rint(w / s), -127, 127), zero rows 0."""
    w = np.asarray(w, dtype=np.float32)
    s = (np.abs(w).max(axis=1) / np.float32(127.0)).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.rint(w / s[:, None])
    q = np.clip(r, -127, 127)
    q[s == 0] = 0
    return q.astype(np.int8), s
