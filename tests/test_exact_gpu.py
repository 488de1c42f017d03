"""Exact-answer tests of the GEMM (fsb_gemm_bf16) and the weight-only GEMMs (fsb_gemm_w8a16 / fsb_gemm_w4a16).

The inputs come from tests/exact_inputs.py: integers whose every partial sum stays below 2^20, so fp32 accumulation is exact
in any order, any K split and any tile walk. What is compared:
- fp32 D: bit-equal to the exact integer. bf16 D and aux: bit-equal to its round-to-nearest-even. No tolerance.
- the copy GEMM (A a row selector): D reproduces arbitrary normal bf16 bit patterns of B, bit for bit.
- the GELU epilogues, over every normal bf16 pre-activation in [-128, 128] and zero (aux must equal the pre-activation bit
  for bit), against the fp64 formula:
    tanh form  x / (1 + 2^a), a = c x (1 + 0.044715 x^2): `a` is the product of three fp32 roundings, so |da| <= 3 * 2^-24 |a|,
      and 2^a is off by at most ln2 |da| + 2^-22 (ex2.approx.ftz) relative; that error reaches the result damped by
      t / (1 + t) <= 1, and __fdividef and the 1 + t add cost 2^-22 + 2^-24 more. Bound: |err| <= (2^-21 + 2^-22 |a|) |ref|
      + 2^-119 (below 2^-119 the true value is under fp32's flush-to-zero of a 128 / 2^126 quotient).
    erf form   Abramowitz & Stegun 7.1.26 bounds erfc absolutely by 1.5e-7, and the result is 0.5 x erfc (or x minus it), so
      |err| <= 0.75e-7 |x| + 2^-21 |ref| (the second term: ex2.approx, __fdividef and five fma roundings).
  fp32 D is held to those bounds; bf16 D to 1 bf16 ulp of fp64 plus the same bound as the floor (the fp32 error that the
  final rounding may amplify into a different bf16 neighbour). Neither bound has a sqrt(K) term.

Every output is a view into a NaN-filled buffer with guard rows and columns (tests/guards.py).

What notices a wrong term. The library was rebuilt with each of these one-line defects (wrong values only, nothing out of
bounds) and the older kernel tests of the same family (test_kernels_gpu / test_gemm_edges_gpu; test_attention_gpu /
test_attention_edges_gpu; test_int4_gpu / test_int8_gpu) and the exact tests were run against it, on an NVIDIA H100 80GB HBM3
(700 W limit):

| defect | older tests | exact test that fails, and what it says |
|---|---|---|
| attention_fwd: `col <= kmax` becomes `col < kmax` where col % 128 == 0 | fail (row 0 loses its only key: max abs(O - ref) = 3.9) | test_ramp_causal_with_padding, every S: "causal ramp S=1024 D=64 edge 0: O 1798/524288 elements differ; first at [b, s, h, d] = (0, 0, 0, 0): got 0.0, want -7.0"; also the padding ramp, causal ties and causal selector |
| attention_fwd: bias row `brow` one entry on | fail (abs(O - ref) up to 4.6 with random biases) | test_rel_bias_selects_one_offset: "selector S=300 D=64: O 250332/422400 elements differ; first at (0, 0, 5, 0): got 0.0, want -2.0"; test_rel_bias_gradient_exact |
| attention_bwd dKV: `qi < kv_row` becomes `qi <= kv_row` where qi % 64 == 0 | fail (dv err 2.8 against tol 0.16) | test_ramp_causal_with_padding: "causal ramp S=1024 D=64 edge 0 dv: max err 1 beyond 2^-18 max(grad); 228/524288 elements differ; first at (0, 0, 0, 36): got 0.0, want 1.0"; causal ties; drel causal |
| attention_bwd dKV: `i_start` one query tile late for kv0 >= 256 | fail (only the S = 1024 cases: dk err 2.1) | test_ramp_causal_with_padding S = 1024 and 2048 + 77: "dv: 5228/524288 elements differ; first at (0, 256, 0, 9): got 0.0, want -1.0" (the first key of the first affected tile); causal ties at S = 1024 |
| gemm k_range: the last split loses its last k-block | fail (split-K cases: max err 9 to 21) | test_position_coded_gemm[TN]: "TN split-K 8x768x8192 reserved 0: 384/6144 elements differ; first at row 0, column 15: k-block 127 (k 8128..8191) reads 0, want 3"; test_int_gemm_splitk, all four shapes |
| gemm: A&S coefficient 1.421413741 written 1.421913741 | PASS (65 passed) | test_gelu_epilogue_sweep[erf-*]: "fp32 D: 32686/34304 beyond the bound; worst at x = -0.00032806396484375: got -0.00016407109797000885, want -0.00016398904587472607, bound 1.03e-10" |
| gemm_w8 int4: the last k16 step of a group takes the next group's scale | fail (error 0.08 to 0.27 beyond the bound) | test_weight_only_gemm_exact[*-w4a16] and every w4a16 Ziya shape: "w4a16 m=1 n=200 k=384 (one pass): 199/200 elements differ; first at (0, 0): got 16.375, want 50.5" |

So the older tests do see six of the seven as specified (those defects shift a whole row or a whole split); only the exact
tests see the coefficient, and only they name the row, key, k-block or column that is wrong.
"""
import pytest
import torch

import exact_inputs as X
import int4_ref
from guards import Guarded, assert_ulp_close, bits, guarded_2d

pytestmark = pytest.mark.gpu

from fsb200 import lib as L, ops  # noqa: E402

DEV = "cuda"
LAYOUTS = [L.GEMM_NT, L.GEMM_NN, L.GEMM_TN]
_NAME = {L.GEMM_NT: "NT", L.GEMM_NN: "NN", L.GEMM_TN: "TN"}
BF16, F32 = torch.bfloat16, torch.float32


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _dev(t):
    """bf16 copy on the device as a strided view (ld a multiple of 8 beyond the width), so that any M or N is legal in any
    layout and every operand is read through a row stride."""
    rows, cols = t.shape
    ld = (cols + 8 + 7) // 8 * 8
    buf = torch.full((rows, ld), 7.0, dtype=BF16, device=DEV)
    buf[:, :cols] = t.to(BF16)
    return buf[:, :cols]


def _operands(layout, A, B):
    a, b = X.to_layout(layout, A, B)
    return _dev(a), _dev(b)


def _want(exact, dt):
    e = exact.to(DEV)
    return e.float() if dt == F32 else X.bf16_of(e)


def _first_diff(got, want):
    bad = (bits(got.contiguous()) != bits(want.contiguous())).nonzero()
    return f"{len(bad)}/{got.numel()} elements differ; first at {tuple(int(v) for v in bad[0])}: got " \
           f"{got[tuple(bad[0])].item()!r}, want {want[tuple(bad[0])].item()!r}"


def _assert_bits(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    if not torch.equal(bits(got.contiguous()), bits(want.contiguous())):
        raise AssertionError(f"{what}: {_first_diff(got, want)}")


def _run_exact(layout, A, B, what, dts=(BF16, F32), **kw):
    a, b = _operands(layout, A, B)
    exact = A.to(DEV) @ B.to(DEV)
    M, N = exact.shape
    for dt in dts:
        d = guarded_2d(M, N, dt)
        ops.gemm(layout, a, b, out=d.view, **kw)
        d.check(f"{what} {dt}")
        _assert_bits(d.view, _want(exact, dt), f"{what} {dt}")
    return exact


# ------------------------------------------------------------------------------------------------- A.1 integer operands
EDGE_M = [127, 128, 129, 255, 256, 257]
EDGE_N = [120, 128, 136, 248, 256, 264]   # N is a multiple of 8 by the ABI (test_gemm_rejects_n_that_ends_inside_a_16_byte_chunk)


@pytest.mark.parametrize("layout", LAYOUTS)
def test_int_gemm_tile_edges(layout):
    """M and N on either side of the 128 / 256 tile edges, K short, ragged and long (4096 + 8)."""
    for i, M in enumerate(EDGE_M):
        for jn, N in enumerate(EDGE_N):
            Ks = (8, 16, 56, 64, 72, 200) if (i + jn) % 3 else (64, 200, 4096 + 8)
            for K in Ks:
                A, B = X.int_operands(M, N, K, seed=M * 7 + N * 3 + K)
                _run_exact(layout, A, B, f"{_NAME[layout]} {M}x{N}x{K}")


@pytest.mark.parametrize("layout", LAYOUTS)
def test_int_gemm_ragged_two_wave_and_many_tiles(layout):
    """The ragged 1096 x 4008 of the epilogue matrix at K in {192, 4096 + 8} and a shape of 325 tiles (more than two waves of
    132 SMs), the latter also with 16 and 64 SMs reserved (the grid and tile width change; the result must not)."""
    for K in (192, 4096 + 8):
        A, B = X.int_operands(1096, 4008, K, seed=K)
        _run_exact(layout, A, B, f"{_NAME[layout]} 1096x4008x{K}")
    A, B = X.int_operands(1543, 6152, 72, seed=5)
    try:
        for n in (0, 16, 64):
            ops.set_reserved_sms(n)
            _run_exact(layout, A, B, f"{_NAME[layout]} 1543x6152x72 reserved {n}")
    finally:
        ops.set_reserved_sms(0)


SPLITK = [(8, 768, 8192), (256, 128, 8192), (384, 256, 6144), (384, 256, 8192)]


@pytest.mark.parametrize("M,N,K", SPLITK)
def test_int_gemm_splitk(M, N, K):
    """The split-K weight-gradient shapes (TN), plain and accumulating onto an integer D, with 0, 16 and 64 SMs reserved: the
    split plan changes with the SM count, and with exact inputs every plan must give the same bits."""
    lib = L.load()
    A, B = X.int_operands(M, N, K, seed=K + M)
    a, b = _operands(L.GEMM_TN, A, B)
    exact = A.to(DEV) @ B.to(DEV)
    old = X.int_vector(M * N, seed=3, amax=100).view(M, N).to(DEV)
    try:
        for n in (0, 16, 64):
            ops.set_reserved_sms(n)
            if n == 0:
                assert lib.fsb_gemm_workspace_bytes(L.GEMM_TN, M, N, K) > 0, "shape meant to split K"
            for dt in (BF16, F32):
                d = guarded_2d(M, N, dt)
                ops.gemm(L.GEMM_TN, a, b, out=d.view)
                d.check(f"split-K {M}x{N}x{K} reserved {n} {dt}")
                _assert_bits(d.view, _want(exact, dt), f"split-K {M}x{N}x{K} reserved {n} {dt}")
                acc = guarded_2d(M, N, dt, fill=0.0, init=old.to(dt), pad_cols=16)
                ops.gemm(L.GEMM_TN, a, b, out=acc.view, accumulate=True)
                acc.check(f"split-K accumulate reserved {n} {dt}")
                _assert_bits(acc.view, _want(exact + old, dt), f"split-K accumulate {M}x{N}x{K} reserved {n} {dt}")
    finally:
        ops.set_reserved_sms(0)


@pytest.mark.parametrize("layout", LAYOUTS)
def test_int_gemm_strided_and_batched(layout):
    """D written into a column slice of a live buffer and accumulated into every second row of another; then the raw ABI with
    batch = 3 and gapped strides. Exact, and everything around the outputs unchanged."""
    M, N, K = 264, 200, 136
    A, B = X.int_operands(M, N, K, seed=60 + layout)
    a, b = _operands(layout, A, B)
    exact = A.to(DEV) @ B.to(DEV)
    for dt in (BF16, F32):
        live = X.int_vector((M + 6) * (N + 80), seed=1).view(M + 6, N + 80).to(DEV).to(dt)
        col = Guarded(live, lambda t: t[3:3 + M, 8:8 + N])
        ops.gemm(layout, a, b, out=col.view)
        col.check(f"column slice {dt}")
        _assert_bits(col.view, _want(exact, dt), f"{_NAME[layout]} column slice {dt}")
        rows = X.int_vector(2 * M * (N + 8), seed=2).view(2 * M, N + 8).to(DEV).to(dt)
        strided = Guarded(rows, lambda t: t.view(M, 2, N + 8)[:, 0, :N])
        old = strided.view.double().clone()
        ops.gemm(layout, a, b, out=strided.view, accumulate=True)
        strided.check(f"row-strided accumulate {dt}", written=False)
        _assert_bits(strided.view, _want(exact + old, dt), f"{_NAME[layout]} row-strided accumulate {dt}")
    batch, gap = 3, 24
    mats = [X.int_operands(M, N, K, seed=70 + i) for i in range(batch)]
    mem = [X.to_layout(layout, Ai, Bi) for Ai, Bi in mats]
    (ar, ac), (br, bc) = mem[0][0].shape, mem[0][1].shape
    sa, sb = ar * ac + gap, br * bc + gap
    a_flat = torch.full((batch * sa,), 5.0, dtype=BF16, device=DEV)
    b_flat = torch.full((batch * sb,), 5.0, dtype=BF16, device=DEV)
    for i, (ai, bi) in enumerate(mem):
        a_flat[i * sa:i * sa + ar * ac] = ai.reshape(-1).to(BF16)
        b_flat[i * sb:i * sb + br * bc] = bi.reshape(-1).to(BF16)
    bias = X.int_vector(N, seed=9).float().to(DEV)
    ldd, ldaux = N + 8, N + 16
    sd, saux = M * ldd + gap, M * ldaux + 2 * gap
    d = Guarded(torch.full((batch * sd + gap,), float("nan"), dtype=BF16, device=DEV),
                lambda t: t[:batch * sd].view(batch, sd)[:, :M * ldd].reshape(batch, M, ldd)[:, :, :N])
    aux = Guarded(torch.full((batch * saux + gap,), float("nan"), dtype=BF16, device=DEV),
                  lambda t: t[:batch * saux].view(batch, saux)[:, :M * ldaux].reshape(batch, M, ldaux)[:, :, :N])
    rc = L.load().fsb_gemm_bf16(layout, M, N, K, a_flat.data_ptr(), ac, b_flat.data_ptr(), bc, d.buf.data_ptr(), ldd, L.BF16,
                                bias.data_ptr(), L.F32, L.EPI_NONE, 0, aux.buf.data_ptr(), ldaux, batch, sa, sb, sd, saux,
                                None, 0, _stream())
    assert rc == 0, L.last_error()
    d.check("batched D")
    aux.check("batched aux")
    for i, (Ai, Bi) in enumerate(mats):
        want = _want(Ai.to(DEV) @ Bi.to(DEV) + bias.double(), BF16)
        _assert_bits(d.view[i], want, f"{_NAME[layout]} batch {i}")
        _assert_bits(aux.view[i], want, f"{_NAME[layout]} batch {i} aux")


def test_gemm_rejects_n_that_ends_inside_a_16_byte_chunk():
    """D and aux leave through TMA stores that clip a ragged row end only at 16-byte granularity: with N = 129 the 7 bf16
    (3 fp32) columns after the view used to come back 0 in every row, in row padding or in live neighbour columns of a
    column slice. Such an N is refused (include/fsb200.h) and D is left untouched; N % 4 == 0 is enough for an fp32 D
    without aux, and is exact there."""
    for N, dt, with_aux in ((127, BF16, False), (129, BF16, False), (257, BF16, False), (132, BF16, False), (130, F32, False),
                            (257, F32, False), (132, F32, True)):
        A, B = X.int_operands(128, N, 64, seed=N)
        a, b = _operands(L.GEMM_NT, A, B)
        d = guarded_2d(128, N, dt)
        aux = guarded_2d(128, N, BF16) if with_aux else None
        with pytest.raises(RuntimeError, match="multiple of"):
            ops.gemm(L.GEMM_NT, a, b, out=d.view, aux=None if aux is None else aux.view)
        d.check(f"refused N={N} {dt}", written=False)
        assert torch.isnan(d.view.float()).all(), "a refused call must not write D"
    for N in (132, 252, 260):
        A, B = X.int_operands(129, N, 72, seed=N)
        _run_exact(L.GEMM_NT, A, B, f"NT 129x{N}x72", dts=(F32,))


# ---------------------------------------------------------------------------------------------- A.2 position-coded operands
def _check_position(layout, M, N, K, what):
    A, B = X.position_coded(M, N, K)
    a, b = _operands(layout, A, B)
    want = (A @ B).to(torch.int64)
    d = guarded_2d(M, N, F32)
    ops.gemm(layout, a, b, out=d.view)
    d.check(what)
    got = d.view.double().cpu()
    assert bool((got == got.round()).all()), f"{what}: a non-integer result"
    diff = X.position_decode(got.to(torch.int64), want)
    if diff is not None:
        m, n, fields, count = diff
        w0 = X.position_window_start(n, K)
        named = ", ".join(f"k-block {w0 + f} (k {64 * (w0 + f)}..{min(K, 64 * (w0 + f + 1)) - 1}) reads {g}, want {w}"
                          for f, g, w in fields)
        raise AssertionError(f"{what}: {count}/{M * N} elements differ; first at row {m}, column {n}: {named}")


@pytest.mark.parametrize("layout", LAYOUTS)
def test_position_coded_gemm(layout):
    """Each k-block contributes its own base-8 digit, so a failure names the k-block (and column) that was lost, doubled or
    read from the wrong place. One ragged-K shape per layout; for TN also the split-K shapes under three SM reservations."""
    _check_position(layout, 264, 392, 456, f"{_NAME[layout]} 264x392x456")
    _check_position(layout, 136, 264, 4096 + 8, f"{_NAME[layout]} 136x264x4104")
    if layout == L.GEMM_TN:
        try:
            for n in (0, 16, 64):
                ops.set_reserved_sms(n)
                for M, N, K in SPLITK:
                    _check_position(layout, M, N, K, f"TN split-K {M}x{N}x{K} reserved {n}")
        finally:
            ops.set_reserved_sms(0)


# ------------------------------------------------------------------------------------------------------------ A.3 copy GEMM
@pytest.mark.parametrize("layout", LAYOUTS)
def test_copy_gemm_reproduces_bit_patterns(layout):
    """A selects one row of B per output row, so D is a gather of B's rows: arbitrary normal bf16 patterns over the whole
    exponent range must come back bit for bit (bf16 D) or widened exactly (fp32 D). Pins the swizzle, the K-major / MN-major
    descriptors and the transpose bits independently of any arithmetic."""
    for M, N, K in ((129, 264, 72), (264, 392, 200), (520, 136, 1032)):
        A, sel = X.row_selector(M, K, seed=M)
        Bb = X.normal_bf16_patterns(K, N, seed=N)
        a, b = X.to_layout(layout, A, Bb)
        a, b = _dev(a), _dev(b)
        want = Bb.to(DEV)[sel.to(DEV)]
        for dt in (BF16, F32):
            d = guarded_2d(M, N, dt)
            ops.gemm(layout, a, b, out=d.view)
            d.check(f"copy {dt}")
            _assert_bits(d.view, want.to(dt), f"{_NAME[layout]} copy {M}x{N}x{K} {dt}")


# --------------------------------------------------------------------------------------------------- A.4 epilogue, exactly
@pytest.mark.parametrize("layout", LAYOUTS)
def test_epilogue_matrix_exact(layout):
    """{no bias, bf16 bias, fp32 bias} x {aux off, on} x {store, accumulate} x {bf16, fp32 D} without activation, on the ragged
    two-wave shape: D = bf16 / fp32 of (old D + A.B + bias) with one rounding, aux = bf16(A.B + bias), bit for bit."""
    M, N, K = 1096, 4008, 192
    A, B = X.int_operands(M, N, K, seed=40 + layout)
    a, b = _operands(layout, A, B)
    prod = A.to(DEV) @ B.to(DEV)
    bias_i = X.int_vector(N, seed=50)
    biases = {"none": None, "bf16": bias_i.to(BF16).to(DEV), "f32": (bias_i * 3 + 1).float().to(DEV)}
    old = {BF16: X.int_vector(M * N, seed=52, amax=200).view(M, N).to(DEV),
           F32: X.int_vector(M * N, seed=53, amax=5000).view(M, N).to(DEV)}
    for bname, bias in biases.items():
        pre = prod if bias is None else prod + bias.double()
        for with_aux in (False, True):
            for acc in (False, True):
                for dt in (BF16, F32):
                    what = f"{_NAME[layout]} bias={bname} aux={with_aux} acc={acc} {dt}"
                    d = guarded_2d(M, N, dt, fill=0.0 if acc else float("nan"), init=old[dt].to(dt) if acc else None)
                    aux = guarded_2d(M, N, BF16) if with_aux else None
                    ops.gemm(layout, a, b, out=d.view, bias=bias, accumulate=acc, aux=None if aux is None else aux.view)
                    d.check(what)
                    _assert_bits(d.view, _want(pre + old[dt] if acc else pre, dt), what)
                    if aux is not None:
                        aux.check(what + " aux")
                        _assert_bits(aux.view, _want(pre, BF16), what + " aux")


# ------------------------------------------------------------------------------------------------------ A.5 GELU sweep
def _gelu_bound(epi, x, ref):
    if epi == L.EPI_GELU_TANH:
        a = (2 * 0.7978845608028654 * 1.4426950408889634) * x * (1 + 0.044715 * x * x)
        return (2.0 ** -21 + 2.0 ** -22 * a.abs()) * ref.abs() + 2.0 ** -119
    return 0.75e-7 * x.abs() + 2.0 ** -21 * ref.abs()


@pytest.mark.parametrize("with_bias", [False, True], ids=["product", "product_plus_bias"])
@pytest.mark.parametrize("epi", [L.EPI_GELU_TANH, L.EPI_GELU_ERF], ids=["tanh", "erf"])
def test_gelu_epilogue_sweep(epi, with_bias):
    """Every normal bf16 x in [-128, 128] and zero reaches the epilogue as a pre-activation through the copy GEMM (A a
    permutation), once as the product alone and once as (x - base) + base with the bias carrying base (an exact sum).
    aux == x bit for bit; D against the bounds derived in the module docstring."""
    Xv, base = X.gelu_sweep_values()
    R, N = Xv.shape
    perm = torch.randperm(R, generator=torch.Generator().manual_seed(1))
    A = torch.zeros(R, R, dtype=torch.float64)
    A[torch.arange(R), perm] = 1.0
    Bm = Xv - base[None, :] if with_bias else Xv
    bias = base.float().to(DEV) if with_bias else None
    a, b = _operands(L.GEMM_NT, A, Bm)
    x = Xv[perm].to(DEV)
    ref = (X.gelu_tanh if epi == L.EPI_GELU_TANH else X.gelu_erf)(x)
    bound = _gelu_bound(epi, x, ref)
    for dt in (BF16, F32):
        d, aux = guarded_2d(R, N, dt), guarded_2d(R, N, BF16)
        ops.gemm(L.GEMM_NT, a, b, out=d.view, bias=bias, epilogue=epi, aux=aux.view)
        d.check(f"gelu {dt}")
        aux.check("gelu aux")
        _assert_bits(aux.view, x.to(BF16), f"epi {epi} bias={with_bias} {dt}: aux is not the pre-activation")
        if dt == F32:
            err = (d.view.double() - ref).abs()
            bad = ~(err <= bound)
            if bad.any():
                i = int((err / bound).reshape(-1).nan_to_num(0).argmax())
                raise AssertionError(f"epi {epi} bias={with_bias} fp32 D: {int(bad.sum())}/{bad.numel()} beyond the bound; worst "
                                     f"at x = {x.reshape(-1)[i].item()!r}: got {d.view.reshape(-1)[i].item()!r}, want "
                                     f"{ref.reshape(-1)[i].item()!r}, bound {bound.reshape(-1)[i].item():.3g}")
        else:
            assert_ulp_close(d.view, ref, f"epi {epi} bias={with_bias} bf16 D", ulps=1.0, floor=bound)


# ------------------------------------------------------------------------------------------------- B weight-only GEMMs
WQ_M = [1, 7, 8, 16, 33, 64, 129, 2048]
# ragged n, k that split K at small m (5120, 13824) and k that do not (256, 384), then the four Ziya-13B projections
WQ_SHAPES = [(200, 384), (1032, 256), (264, 5120)]
ZIYA = [(15360, 5120), (5120, 5120), (27648, 5120), (5120, 13824)]


def _wq_case(fmt, m, n, k, seed):
    qmax = 127 if fmt == 8 else 7
    A, Q = X.wq_int_operands(m, n, k, qmax, seed)
    lda = k + 64 if m % 2 else k
    abuf = torch.full((m, lda), 3.0, dtype=BF16, device=DEV)
    abuf[:, :k] = A.to(BF16)
    a = abuf[:, :k]
    if fmt == 8:
        s = X.w8_scales(n, seed + 1)
        exact = X.w8_exact(A.to(DEV), Q.to(DEV), s.to(DEV))
        q, sdev, op = Q.to(DEV), s.to(DEV), ops.gemm_w8a16
        ws = L.load().fsb_gemm_w8a16_workspace_bytes(m, n, k)
    else:
        s = X.w4_scales(n, k // 128, seed + 1)
        exact = X.w4_exact(A.to(DEV), Q.to(DEV), s.to(DEV))
        q = torch.from_numpy(int4_ref.pack(Q.numpy())).to(DEV)
        sdev, op = s.to(DEV), ops.gemm_w4a16
        ws = L.load().fsb_gemm_w4a16_workspace_bytes(m, n, k)
    d = guarded_2d(m, n, BF16, pad_cols=16)
    op(a, q, sdev, out=d.view)
    what = f"w{fmt}a16 m={m} n={n} k={k} ({'split-K' if ws else 'one pass'})"
    d.check(what)
    _assert_bits(d.view, X.bf16_of(exact), what)
    return ws


@pytest.mark.parametrize("fmt", [8, 4], ids=["w8a16", "w4a16"])
@pytest.mark.parametrize("m", WQ_M)
def test_weight_only_gemm_exact(fmt, m):
    """Integer activations, hand-built codes over the full range and power-of-two scales (per row for int8; per row and
    128-k group, never equal in neighbouring groups, for int4): D == bf16(exact) bit for bit, for every token-tile width
    (m <= 8, 16, 32, 64, 128), a ragged n, and k on both sides of the split-K plan."""
    split = []
    for n, k in WQ_SHAPES:
        if fmt == 4 and k % 128:
            continue
        split.append(_wq_case(fmt, m, n, k, seed=m * 31 + n) > 0)
    if m <= 8:
        assert any(split) and not all(split), "the shapes are meant to cover both the split-K and the single-pass path"


@pytest.mark.parametrize("fmt", [8, 4], ids=["w8a16", "w4a16"])
@pytest.mark.parametrize("m", [1, 32])
@pytest.mark.parametrize("nk", ZIYA, ids=[f"n{n}k{k}" for n, k in ZIYA])
def test_weight_only_gemm_exact_ziya(fmt, m, nk):
    _wq_case(fmt, m, nk[0], nk[1], seed=m + nk[0])
