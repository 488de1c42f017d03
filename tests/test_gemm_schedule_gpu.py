"""Every schedule and tile shape the bf16 GEMM's plan can pick, on inputs whose product is known to the bit.

The plan (csrc/gemm.cu, gemm_plan) picks per call between the cooperative kernel on 128 x 128, 128 x 192 or 128 x 256 tiles
and the ping-pong kernel on 64 x 256 tiles (K <= 1024), from the shape and the SMs the GEMM may use. `plan` below restates that rule so
that each case can be built to land on the plan and the wave count it names; the test checks that the shapes chosen really
do. Operands are small integers (tests/exact_inputs.py), so fp32 accumulation is exact in any order and the only rounding
is the final store: every output must equal the fp64 product rounded once, bit for bit, whatever the schedule. The one
exception is GELU, whose fast device formula is held to one bf16 ulp of the fp64 value plus the formula's own error.
"""
import pytest
import torch

import exact_inputs as X
from guards import assert_ulp_close, bits, guarded_2d

pytestmark = pytest.mark.gpu

from fsb200 import lib as L, ops  # noqa: E402

DEV = "cuda"
BF16, F32 = torch.bfloat16, torch.float32
_NAME = {L.GEMM_NT: "NT", L.GEMM_NN: "NN", L.GEMM_TN: "TN"}
PP_MAX_K = 1024


def plan(layout, M, N, K, sms, plain=True):
    """(schedule, tile rows, tile width, K-splits, tiles) as gemm_plan chooses them for an unbatched call."""
    tm = -(-M // 128)
    tiles256 = tm * -(-N // 256)
    bn = 256 if (N > 128 and tiles256 * 10 >= sms * 7) else 128
    if layout == L.GEMM_TN and plain and N % 4 == 0 and (M * N) % 8 == 0 and K >= 4096:
        wide = N >= 256
        tiles = tm * (-(-N // 256) if wide else -(-N // 128))
        splits = min(sms // tiles, 16)
        while splits > 1 and (K % (splits * 64) != 0 or K // splits < 1024):
            splits -= 1
        if splits >= 2 and tiles * 2 <= sms:
            return ("coop", 128, 256 if wide else bn, splits, tiles * splits)
    if bn == 256 and K <= PP_MAX_K:
        return ("pingpong", 64, 256, 1, -(-M // 64) * -(-N // 256))
    if bn == 128 and layout == L.GEMM_TN and N > 128:
        t128, t192 = tm * -(-N // 128), tm * -(-N // 192)
        last = t128 % sms
        if last and last * 2 < sms and -(-t192 // sms) < -(-t128 // sms):
            return ("coop", 128, 192, 1, t192)
    return ("coop", 128, bn, 1, tm * -(-N // bn))


def _sms(reserved):
    return torch.cuda.get_device_properties(0).multi_processor_count - reserved


def _dev(t):
    """bf16 copy on the device as a strided view (ld a multiple of 8 beyond the width)."""
    rows, cols = t.shape
    ld = (cols + 8 + 7) // 8 * 8
    buf = torch.full((rows, ld), 7.0, dtype=BF16, device=DEV)
    buf[:, :cols] = t.to(BF16)
    return buf[:, :cols]


def _assert_bits(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape)
    g, w = bits(got.contiguous()), bits(want.contiguous())
    if not torch.equal(g, w):
        bad = (g != w).nonzero()
        i = tuple(int(v) for v in bad[0])
        raise AssertionError(f"{what}: {len(bad)}/{got.numel()} elements differ; first at {i}: got {got[i].item()!r}, "
                             f"want {want[i].item()!r}")


def _want(exact, dt):
    return exact.float() if dt == F32 else X.bf16_of(exact)


def _shapes(sms):
    """(name, layout, M, N, K, expected plan, expected waves): each plan at the wave counts that stress its tile walk."""
    K_pp, K_long = 768, 4160
    # 192-wide: a TN call whose 128 x 128 tiles leave a last wave less than half full (GPT-2's mlp_proj wgrad on 132 SMs)
    tm192 = next(t for t in range(1, 4 * sms) if plan(L.GEMM_TN, 128 * t, 768, 2048, sms)[2] == 192)
    out = []
    for layout in (L.GEMM_NT, L.GEMM_NN, L.GEMM_TN):
        n = _NAME[layout]
        out += [
            # ping-pong: the CTA's last tile on warpgroup 0 (odd count per CTA), on warpgroup 1, and many tiles per CTA
            (f"{n} pingpong 2 waves + 1", layout, 64 * (2 * sms + 1), 256, K_pp, ("pingpong", 256), 3),
            (f"{n} pingpong 2 waves - 1", layout, 64 * (2 * sms - 1), 256, K_pp, ("pingpong", 256), 2),
            (f"{n} pingpong many, ragged", layout, 64 * 61 + 24, 1024 + 8, 1024, ("pingpong", 256), None),
            # cooperative 128 x 256 at long K: a few tiles over one wave
            (f"{n} coop 256 wave + few", layout, 128 * (sms // 8 + 1), 256 * 8, K_long, ("coop", 256), 2),
            # cooperative 128 x 128: exactly one wave, one tile over
            (f"{n} coop 128 one wave", layout, 128 * sms, 128, 1024, ("coop", 128), 1),
            (f"{n} coop 128 wave + 1", layout, 128 * (sms + 1), 128, 1024, ("coop", 128), 2),
        ]
    out += [("TN coop 192 one wave", L.GEMM_TN, 128 * tm192, 768, 2048, ("coop", 192), 1),
            ("TN coop 192 ragged", L.GEMM_TN, 128 * tm192 - 40, 768 - 8, 2048, ("coop", 192), 1)]
    return out


@pytest.mark.parametrize("reserved", [0, 16])
def test_every_plan_exact(reserved):
    sms = _sms(reserved)
    try:
        ops.set_reserved_sms(reserved)
        for i, (what, layout, M, N, K, want_plan, waves) in enumerate(_shapes(sms)):
            sched, _, bn, splits, tiles = plan(layout, M, N, K, sms)
            assert (sched, bn) == want_plan and splits == 1, (what, sched, bn, splits)
            if waves is not None:
                assert -(-tiles // sms) == waves, (what, tiles, sms)
            A, B = X.int_operands(M, N, K, seed=100 + i)
            a, b = (_dev(t) for t in X.to_layout(layout, A, B))
            exact = A.to(DEV) @ B.to(DEV)
            for dt in (BF16, F32):
                d = guarded_2d(M, N, dt)
                ops.gemm(layout, a, b, out=d.view)
                d.check(f"{what} reserved {reserved} {dt}")
                _assert_bits(d.view, _want(exact, dt), f"{what} reserved {reserved} {dt}")
    finally:
        ops.set_reserved_sms(0)


EPILOGUES = [  # (bias dtype or None, activation, aux, accumulate, D dtype)
    (BF16, L.EPI_NONE, False, False, BF16),
    (F32, L.EPI_NONE, True, False, BF16),
    (BF16, L.EPI_GELU_TANH, True, False, BF16),
    (BF16, L.EPI_GELU_ERF, True, False, BF16),
    (None, L.EPI_GELU_TANH, False, False, BF16),
    (None, L.EPI_NONE, False, True, BF16),
    (F32, L.EPI_NONE, False, True, F32),
    (BF16, L.EPI_GELU_ERF, True, True, F32),
]


def _gelu(x, epi):
    return X.gelu_tanh(x) if epi == L.EPI_GELU_TANH else X.gelu_erf(x)


@pytest.mark.parametrize("reserved", [0, 16])
@pytest.mark.parametrize("layout", [L.GEMM_NT, L.GEMM_NN, L.GEMM_TN])
def test_pingpong_epilogues(layout, reserved):
    """Bias, GELU, the pre-activation copy and accumulation under the ping-pong schedule, over a ragged tile grid that leaves
    warpgroup 0 the last tile of some CTAs."""
    sms = _sms(reserved)
    M, N, K = 64 * (2 * sms + 1) - 24, 512 + 8, 768
    assert plan(layout, M, N, K, sms, plain=False)[0] == "pingpong"
    A, B = X.int_operands(M, N, K, seed=7)
    a, b = (_dev(t) for t in X.to_layout(layout, A, B))
    exact = A.to(DEV) @ B.to(DEV)
    try:
        ops.set_reserved_sms(reserved)
        for j, (bias_dt, epi, want_aux, accumulate, dt) in enumerate(EPILOGUES):
            what = f"{_NAME[layout]} reserved {reserved} bias {bias_dt} epi {epi} aux {want_aux} acc {accumulate} {dt}"
            pre = exact.clone()
            bias = None
            if bias_dt is not None:
                bv = X.int_vector(N, seed=20 + j).to(DEV)
                bias = bv.to(bias_dt)
                pre = pre + bv
            old = X.int_vector(M * N, seed=40 + j).view(M, N).to(DEV) if accumulate else None
            d = guarded_2d(M, N, dt, init=old.to(dt) if accumulate else None)
            aux = guarded_2d(M, N, BF16) if want_aux else None
            ops.gemm(layout, a, b, out=d.view, bias=bias, epilogue=epi, accumulate=accumulate,
                     aux=aux.view if want_aux else None)
            d.check(what)
            if want_aux:
                aux.check(what + " aux")
                _assert_bits(aux.view, X.bf16_of(pre), what + " aux")
            if epi == L.EPI_NONE:
                total = pre + old if accumulate else pre
                _assert_bits(d.view, _want(total, dt), what)
            else:
                act = _gelu(pre, epi)
                total = act + old if accumulate else act
                # the device erfc (Abramowitz & Stegun 7.1.26) is good to 1.5e-7 absolute, which the far negative tail
                # (values ~1e-12) shows as a relative error: allow 1e-7 |x| on top of the ulp
                assert_ulp_close(d.view, total, what, ulps=1.0, floor=1e-7 * pre.abs())
    finally:
        ops.set_reserved_sms(0)


def test_two_runs_identical_bits():
    """Random bf16 operands, where the summation order does show in the result: two calls of each plan give the same bits."""
    sms = _sms(0)
    g = torch.Generator(device="cpu").manual_seed(5)
    cases = [(L.GEMM_NN, 64 * (2 * sms + 1), 768, 768), (L.GEMM_NT, 8192, 3072, 768), (L.GEMM_TN, 768, 3072, 8192),
             (L.GEMM_NT, 128 * (sms + 1), 256, 4608)]
    for layout, M, N, K in cases:
        A = torch.randn(M, K, generator=g).double()
        B = torch.randn(K, N, generator=g).double()
        a, b = (_dev(t) for t in X.to_layout(layout, A, B))
        bias = torch.randn(N, generator=g).to(BF16).to(DEV)
        for kw in ({}, {"bias": bias, "epilogue": L.EPI_GELU_TANH}):
            r1 = ops.gemm(layout, a, b, **kw)
            r2 = ops.gemm(layout, a, b, **kw)
            _assert_bits(r2, r1, f"{_NAME[layout]} {M}x{N}x{K} {plan(layout, M, N, K, sms, plain=not kw)[:3]} run 2")
