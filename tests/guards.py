"""Sentinel-filled output buffers for the kernel parity tests.

A kernel under test writes into a view of a larger allocation. Everything outside the view is a guard: the test checks
that the kernel wrote every element of the view (no NaN sentinel left) and that no guard element changed (bit equality).
Also the bf16-ulp comparison for kernels that round their fp32 result to bf16 once.
"""
import torch

_BITS = {torch.bfloat16: torch.int16, torch.float16: torch.int16, torch.float32: torch.int32}


def bits(t):
    return t.view(_BITS[t.dtype])


class Guarded:
    """buf: the whole allocation, already filled; sel(t) returns the view the kernel writes (the same slicing works on
    a bool mask of buf's shape)."""

    def __init__(self, buf, sel):
        self.buf, self.sel = buf, sel
        self.before = buf.clone()
        mask = torch.zeros(buf.shape, dtype=torch.bool, device=buf.device)
        sel(mask).fill_(True)
        self.guard = ~mask
        self.view = sel(buf)

    def check(self, what="", written=True):
        """Guards bit-identical; with written=True also no NaN left inside the view."""
        if written:
            nan = torch.isnan(self.view.float())
            assert not nan.any(), f"{what}: {int(nan.sum())}/{nan.numel()} elements of the output were never written"
        same = torch.equal(bits(self.buf)[self.guard], bits(self.before)[self.guard])
        assert same, f"{what}: guard elements outside the output view were modified"

    def reset(self):
        self.buf.copy_(self.before)


def guarded_2d(rows, cols, dtype, fill=float("nan"), init=None, pad_rows=3, pad_cols=8, device="cuda"):
    """[rows, cols] view inside a [rows + 2 pad_rows, ld] buffer, ld > cols a multiple of 8, 16-byte aligned view.
    init: optional finite content for the view (accumulating kernels)."""
    ld = (cols + 2 * pad_cols + 7) // 8 * 8
    buf = torch.full((rows + 2 * pad_rows, ld), fill, dtype=dtype, device=device)
    sel = lambda t: t[pad_rows:pad_rows + rows, pad_cols:pad_cols + cols]   # noqa: E731
    if init is not None:
        sel(buf).copy_(init)
    return Guarded(buf, sel)


def guarded_1d(n, dtype, fill=float("nan"), init=None, pad=8, device="cuda"):
    buf = torch.full((n + 2 * pad,), fill, dtype=dtype, device=device)
    sel = lambda t: t[pad:pad + n]   # noqa: E731
    if init is not None:
        sel(buf).copy_(init)
    return Guarded(buf, sel)


def bf16_ulp(ref):
    """Spacing of bf16 numbers at |ref| (8 significant bits); the smallest normal spacing below 2^-126."""
    _, e = torch.frexp(ref.double().abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(ref, dtype=torch.float64), e - 8)


def assert_ulp_close(got, ref, what="", ulps=1.0, floor=0.0):
    """|got - ref| <= ulps * bf16_ulp(ref) + floor elementwise, ref in fp64. floor: a number or a tensor that broadcasts
    against ref (an absolute allowance for fp32 cancellation, stated by the caller). NaN in got fails."""
    ref = ref.double()
    err = (got.double() - ref).abs()
    tol = ulps * bf16_ulp(ref) + floor
    bad = ~(err <= tol)
    if bad.any():
        i = int(bad.reshape(-1).nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} elements beyond {ulps} bf16 ulp + floor; first at "
                             f"flat index {i}: got {got.reshape(-1)[i].item():.6g}, want {ref.reshape(-1)[i].item():.6g}; "
                             f"max err {err.max().item():.4g}")
