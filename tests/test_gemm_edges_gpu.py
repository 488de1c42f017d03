"""GEMM parity at the edges the models reach: tiny and ragged operands, every fused-epilogue combination, strided and
batched outputs, the split-K plan, reserved SMs and the tensor-map memo.

Reference: the same formula in fp64 on the same bf16 inputs, D = D_old + act(A.B + bias) and aux = bf16(A.B + bias)
(include/fsb200.h). Tolerance model, as in test_kernels_gpu.py: the kernel accumulates in fp32 and rounds once, so a bf16
output is within 2^-8 relative of the exact value (rtol 1e-2) plus fp32 accumulation-order noise that grows with sqrt(K)
(atol 2e-2 sqrt(K/64)); an fp32 output has no final rounding to speak of (rtol 1e-4, atol 1e-3 sqrt(K/64)).
Every output is a view into a NaN-filled buffer with guard rows and columns (tests/guards.py): each element of the view
must be written and no guard element may change. Accumulating calls start from finite values instead of NaN.
"""
import math

import pytest
import torch

from guards import Guarded, bits, guarded_2d

pytestmark = pytest.mark.gpu

from fsb200 import lib as L, ops  # noqa: E402

DEV = "cuda"
LAYOUTS = [L.GEMM_NT, L.GEMM_NN, L.GEMM_TN]
_NAME = {L.GEMM_NT: "NT", L.GEMM_NN: "NN", L.GEMM_TN: "TN"}


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(DEV)


def _operands(layout, M, N, K, seed=0, scale_b=1.0):
    """bf16 operands in the layout's memory order and the exact product A.B in fp64."""
    if layout == L.GEMM_NT:
        a, b = _rand(M, K, seed=seed), _rand(N, K, seed=seed + 1, scale=scale_b)
        ref = a.double() @ b.double().t()
    elif layout == L.GEMM_NN:
        a, b = _rand(M, K, seed=seed), _rand(K, N, seed=seed + 1, scale=scale_b)
        ref = a.double() @ b.double()
    else:
        a, b = _rand(K, M, seed=seed), _rand(K, N, seed=seed + 1, scale=scale_b)
        ref = a.double().t() @ b.double()
    return a, b, ref


def _tol(K, dtype):
    s = math.sqrt(max(K, 1) / 64)
    return (2e-2 * s, 1e-2) if dtype == torch.bfloat16 else (1e-3 * s, 1e-4)


def _close(got, ref, K, dtype, what):
    atol, rtol = _tol(K, dtype)
    err = (got.double() - ref).abs()
    bad = err > atol + rtol * ref.abs()
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.numel()} elements off; max err {err.max().item():.4g}"


def _gelu_tanh(x):
    return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))


def _gelu_erf(x):
    return 0.5 * x * (1 + torch.special.erf(x / math.sqrt(2)))


_ACT = {L.EPI_NONE: lambda x: x, L.EPI_GELU_TANH: _gelu_tanh, L.EPI_GELU_ERF: _gelu_erf}


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------------------- A.1
@pytest.mark.parametrize("layout", LAYOUTS)
def test_gemm_tiny_and_ragged_shapes(layout):
    """M in {1, 3, 8, 33} x N in {8, 24, 72} x K in {8, 16, 40, 72}, bf16 and fp32 D (TN: lda = M, so M % 8 == 0).
    M < 8 is accepted and correct, so the LLaMA decode head would not need its rows padded to 8."""
    Ms = [8, 16, 40] if layout == L.GEMM_TN else [1, 3, 8, 33]
    for M in Ms:
        for N in (8, 24, 72):
            for K in (8, 16, 40, 72):
                a, b, ref = _operands(layout, M, N, K, seed=M * 1000 + N * 10 + K)
                for dt in (torch.bfloat16, torch.float32):
                    out = guarded_2d(M, N, dt)
                    ops.gemm(layout, a, b, out=out.view)
                    what = f"{_NAME[layout]} {M}x{N}x{K} {dt}"
                    out.check(what)
                    _close(out.view, ref, K, dt, what)


def test_gemm_nsp_head_shapes():
    """BERT's next-sentence head: NT with N = 8 plus bias (bert.py: pooled x W_nsp^T + b), and its weight gradient TN with
    M = 8, K = batch (tiny, not a multiple of 8), fp32 out."""
    for B in (2, 5, 32):
        pooled, w = _rand(B, 768, seed=B), _rand(8, 768, seed=B + 1, scale=0.05)
        for bias in (_rand(8, seed=3), _rand(8, seed=3).float()):
            out = guarded_2d(B, 8, torch.bfloat16)
            ops.gemm(L.GEMM_NT, pooled, w, out=out.view, bias=bias)
            out.check(f"nsp fwd B={B}")
            _close(out.view, pooled.double() @ w.double().t() + bias.double(), 768, torch.bfloat16, f"nsp fwd B={B}")
        dnsp = _rand(B, 8, seed=B + 2)
        dw = guarded_2d(8, 768, torch.float32)
        ops.gemm(L.GEMM_TN, dnsp, pooled, out=dw.view)
        dw.check(f"nsp wgrad B={B}")
        _close(dw.view, dnsp.double().t() @ pooled.double(), B, torch.float32, f"nsp wgrad B={B}")


# ------------------------------------------------------------------------------------------------------------- A.2
@pytest.mark.parametrize("layout", LAYOUTS)
def test_gemm_epilogue_matrix(layout):
    """bias {none, bf16, fp32} x epilogue {none, tanh, erf} x aux {off, on} x accumulate {off, on} x D {bf16, fp32} on one
    ragged two-wave shape (N % 32 != 0: the ragged tail falls inside a 64-column bf16 and a 32-column fp32 sub-tile)."""
    M, N, K = 1096, 4008, 192
    a, b, prod = _operands(layout, M, N, K, seed=40 + layout, scale_b=0.2)
    biases = {"none": None, "bf16": _rand(N, seed=50), "f32": (torch.randn(N, generator=torch.Generator().manual_seed(51)))
              .to(DEV)}
    d_old = {torch.bfloat16: _rand(M, N, seed=52), torch.float32: _rand(M, N, seed=53).float() + 0.25}
    for bname, bias in biases.items():
        pre = prod if bias is None else prod + bias.double()
        for epi in (L.EPI_NONE, L.EPI_GELU_TANH, L.EPI_GELU_ERF):
            act = _ACT[epi](pre)
            for with_aux in (False, True):
                for acc in (False, True):
                    for dt in (torch.bfloat16, torch.float32):
                        what = f"{_NAME[layout]} bias={bname} epi={epi} aux={with_aux} acc={acc} {dt}"
                        d = guarded_2d(M, N, dt, fill=0.0 if acc else float("nan"), init=d_old[dt] if acc else None)
                        aux = guarded_2d(M, N, torch.bfloat16) if with_aux else None
                        ops.gemm(layout, a, b, out=d.view, bias=bias, epilogue=epi, accumulate=acc,
                                 aux=None if aux is None else aux.view)
                        d.check(what)
                        want = act + d_old[dt].double() if acc else act
                        _close(d.view, want, K, dt, what)
                        if aux is not None:
                            aux.check(what + " aux")
                            _close(aux.view, pre, K, torch.bfloat16, what + " aux")


# ------------------------------------------------------------------------------------------------------------- A.3
@pytest.mark.parametrize("layout", LAYOUTS)
def test_gemm_strided_outputs(layout):
    """D and aux written into a column slice of a wider live buffer and into a row-strided view (ldd > N, the pooler /
    token-0 rows of bert.py): the ragged N edge is clipped right next to live neighbour columns, which must not change."""
    M, N, K = 264, 200, 136
    a, b, prod = _operands(layout, M, N, K, seed=60 + layout)
    bias = _rand(N, seed=61)
    pre = prod + bias.double()
    for dt in (torch.bfloat16, torch.float32):
        # column slice [M, 8 + N + 72) of live (finite, non-zero) data
        live = _rand(M + 6, N + 80, seed=62).to(dt)
        col = Guarded(live, lambda t: t[3:3 + M, 8:8 + N])
        aux_live = _rand(M + 6, N + 80, seed=63)
        aux = Guarded(aux_live, lambda t: t[3:3 + M, 8:8 + N])
        ops.gemm(layout, a, b, out=col.view, bias=bias, epilogue=L.EPI_GELU_ERF, aux=aux.view)
        col.check(f"{_NAME[layout]} column slice {dt}")
        aux.check(f"{_NAME[layout]} aux column slice")
        _close(col.view, _gelu_erf(pre), K, dt, "column slice")
        _close(aux.view, pre, K, torch.bfloat16, "aux column slice")
        # every second row of a [2M, N + 8] buffer (ldd = 2 (N + 8)), accumulated into like the token-0 rows of BERT
        rows = _rand(2 * M, N + 8, seed=64).to(dt)
        strided = Guarded(rows, lambda t: t.view(M, 2, N + 8)[:, 0, :N])
        old = strided.view.double().clone()
        ops.gemm(layout, a, b, out=strided.view, accumulate=True)
        strided.check(f"{_NAME[layout]} row-strided accumulate {dt}", written=False)
        _close(strided.view, old + prod, K, dt, "row-strided accumulate")


# ------------------------------------------------------------------------------------------------------------- A.4
def _call_raw(layout, M, N, K, a, lda, b, ldb, d, ldd, d_dtype, ws, ws_bytes, accumulate=0):
    return L.load().fsb_gemm_bf16(layout, M, N, K, a.data_ptr(), lda, b.data_ptr(), ldb, d.data_ptr(), ldd, d_dtype,
                                  None, L.BF16, L.EPI_NONE, accumulate, None, 0, 1, 0, 0, 0, 0,
                                  None if ws is None else ws.data_ptr(), ws_bytes, _stream())


@pytest.mark.parametrize("M,N,K", [(8, 768, 8192),      # BERT token-type weight gradient: TN, M = 8, K = B*S
                                   (256, 128, 8192),    # narrow N: 128-wide tiles
                                   (384, 256, 6144)])   # a split count that is not a power of two
def test_gemm_splitk_plan_edges(M, N, K):
    """Split-K weight gradients: the workspace the kernel needs is exactly fsb_gemm_workspace_bytes (a byte less is
    refused), the fp32 / bf16 results (and accumulation into a strided D, ldd > N) match fp64, and reruns are
    bit-identical (fixed reduction order)."""
    lib = L.load()
    nbytes = int(lib.fsb_gemm_workspace_bytes(L.GEMM_TN, M, N, K))
    splits = nbytes // (M * N * 4)
    assert nbytes == splits * M * N * 4 and 2 <= splits <= 16 and K % (splits * 64) == 0, (nbytes, splits)
    if K == 6144:
        assert splits & (splits - 1) != 0, f"shape meant to split a non-power-of-two number of ways, got {splits}"
    a, b, ref = _operands(L.GEMM_TN, M, N, K, seed=70, scale_b=0.5)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    for dt, code in ((torch.bfloat16, L.BF16), (torch.float32, L.F32)):
        d = guarded_2d(M, N, dt)
        assert _call_raw(L.GEMM_TN, M, N, K, a, M, b, N, d.view, d.buf.stride(0), code, ws, nbytes - 16) != 0
        assert "workspace" in L.last_error()
        d.check("refused call", written=False)
        assert _call_raw(L.GEMM_TN, M, N, K, a, M, b, N, d.view, d.buf.stride(0), code, ws, nbytes) == 0, L.last_error()
        d.check(f"split-K {splits} ways {dt}")
        _close(d.view, ref, K, dt, f"split-K {M}x{N}x{K} {dt}")
        first = d.view.clone()
        d.reset()
        ops.gemm(L.GEMM_TN, a, b, out=d.view)
        assert torch.equal(bits(first), bits(d.view)), "split-K is not deterministic"
        init = _rand(M, N, seed=71).to(dt)
        acc = guarded_2d(M, N, dt, fill=0.0, init=init, pad_cols=16)
        ops.gemm(L.GEMM_TN, a, b, out=acc.view, accumulate=True)
        acc.check(f"split-K accumulate {dt}")
        _close(acc.view, ref + init.double(), K, dt, f"split-K accumulate {dt}")


# ------------------------------------------------------------------------------------------------------------- A.5
def test_gemm_reserved_sms():
    """fsb_set_reserved_sms changes the persistent grid (and the tile width / split plan). A tile's K order does not depend
    on which CTA runs it, so unsplit GEMMs are bit-identical for every reservation; split-K ones stay within tolerance."""
    cases = [(L.GEMM_NT, 1096, 4008, 192), (L.GEMM_NN, 760, 2560, 256), (L.GEMM_TN, 760, 2560, 256)]
    split = (L.GEMM_TN, 384, 2816, 4096)
    results = {}
    try:
        for n in (0, 16, 64):
            ops.set_reserved_sms(n)
            for layout, M, N, K in cases:
                a, b, _ = _operands(layout, M, N, K, seed=80)
                d = guarded_2d(M, N, torch.bfloat16)
                ops.gemm(layout, a, b, out=d.view, epilogue=L.EPI_GELU_TANH)
                d.check(f"reserved {n} {_NAME[layout]}")
                results.setdefault((layout, M, N, K), []).append(d.view.clone())
            layout, M, N, K = split
            a, b, ref = _operands(layout, M, N, K, seed=81, scale_b=0.5)
            for dt in (torch.bfloat16, torch.float32):
                d = guarded_2d(M, N, dt)
                ops.gemm(layout, a, b, out=d.view)
                d.check(f"reserved {n} split-K {dt}")
                _close(d.view, ref, K, dt, f"reserved {n} split-K {dt}")
    finally:
        ops.set_reserved_sms(0)
    for key, outs in results.items():
        for o in outs[1:]:
            assert torch.equal(bits(outs[0]), bits(o)), f"{key}: result depends on the number of reserved SMs"


# ------------------------------------------------------------------------------------------------------------- A.6
def test_gemm_splitk_workspace_follows_reserved_sms():
    """A TN shape whose split count (and workspace) grows when fewer SMs are reserved: ops.gemm must size the workspace
    for the current reservation, not for the one in force at the shape's first call."""
    lib = L.load()
    found = None
    try:
        for tm in range(1, 12):
            for tn in range(1, 40):
                M, N, K = 128 * tm - 56, 256 * tn - 24, 4096
                lib.fsb_set_reserved_sms(16)
                hi = lib.fsb_gemm_workspace_bytes(L.GEMM_TN, M, N, K)
                lib.fsb_set_reserved_sms(0)
                lo = lib.fsb_gemm_workspace_bytes(L.GEMM_TN, M, N, K)
                if lo > hi:
                    found = (M, N, K)
                    break
            if found:
                break
        assert found, "no TN shape whose split-K workspace grows when the reservation drops"
        M, N, K = found
        a, b, ref = _operands(L.GEMM_TN, M, N, K, seed=90, scale_b=0.5)
        for n in (16, 0):
            ops.set_reserved_sms(n)
            d = guarded_2d(M, N, torch.float32)
            ops.gemm(L.GEMM_TN, a, b, out=d.view)
            d.check(f"reserved {n} {found}")
            _close(d.view, ref, K, torch.float32, f"reserved {n} {found}")
    finally:
        ops.set_reserved_sms(0)


# ------------------------------------------------------------------------------------------------------------- A.7
@pytest.mark.parametrize("layout", LAYOUTS)
def test_gemm_batched_abi(layout):
    """fsb_gemm_bf16 with batch = 3 and gapped strides for A, B, D and aux, with bias, aux and GELU: every batch matches
    its own product and the gaps between the batches are untouched."""
    batch, M, N, K = 3, 200, 136, 72
    gap = 24
    if layout == L.GEMM_NT:
        a_rows, a_cols, b_rows, b_cols = M, K, N, K
    elif layout == L.GEMM_NN:
        a_rows, a_cols, b_rows, b_cols = M, K, K, N
    else:
        a_rows, a_cols, b_rows, b_cols = K, M, K, N
    sa, sb = a_rows * a_cols + gap, b_rows * b_cols + gap
    a_flat, b_flat = _rand(batch * sa, seed=100), _rand(batch * sb, seed=101, scale=0.2)
    A = [a_flat[i * sa:i * sa + a_rows * a_cols].view(a_rows, a_cols) for i in range(batch)]
    B = [b_flat[i * sb:i * sb + b_rows * b_cols].view(b_rows, b_cols) for i in range(batch)]
    bias = _rand(N, seed=102).float()
    ldd, ldaux = N + 8, N + 16
    sd, saux = M * ldd + gap, M * ldaux + 2 * gap
    d = Guarded(torch.full((batch * sd + gap,), float("nan"), dtype=torch.bfloat16, device=DEV),
                lambda t: t[:batch * sd].view(batch, sd)[:, :M * ldd].reshape(batch, M, ldd)[:, :, :N])
    aux = Guarded(torch.full((batch * saux + gap,), float("nan"), dtype=torch.bfloat16, device=DEV),
                  lambda t: t[:batch * saux].view(batch, saux)[:, :M * ldaux].reshape(batch, M, ldaux)[:, :, :N])
    rc = L.load().fsb_gemm_bf16(layout, M, N, K, a_flat.data_ptr(), a_cols, b_flat.data_ptr(), b_cols, d.buf.data_ptr(), ldd,
                                L.BF16, bias.data_ptr(), L.F32, L.EPI_GELU_TANH, 0, aux.buf.data_ptr(), ldaux, batch, sa, sb,
                                sd, saux, None, 0, _stream())
    assert rc == 0, L.last_error()
    d.check("batched D")
    aux.check("batched aux")
    for i in range(batch):
        if layout == L.GEMM_NT:
            prod = A[i].double() @ B[i].double().t()
        elif layout == L.GEMM_NN:
            prod = A[i].double() @ B[i].double()
        else:
            prod = A[i].double().t() @ B[i].double()
        pre = prod + bias.double()
        _close(d.view[i], _gelu_tanh(pre), K, torch.bfloat16, f"batch {i}")
        _close(aux.view[i], pre, K, torch.bfloat16, f"batch {i} aux")


# ------------------------------------------------------------------------------------------------------------- A.8
def test_gemm_tensor_map_memo_distinguishes_geometry():
    """The host memoises tensor maps by (dtype, base, dims, strides, box). Reusing one base address for D with a different
    ld, row count, element type or box (aux vs D) must encode a new map each time: every result stays correct."""
    M, N, K = 136, 264, 64
    a, b, prod = _operands(L.GEMM_NT, 2 * M, N, K, seed=110)
    pool = torch.empty(4 * M * (N + 64) * 4, dtype=torch.uint8, device=DEV)

    def view(dtype, rows, ld):
        return pool.view(dtype)[:rows * ld].view(rows, ld)[:, :N]

    geoms = [(torch.bfloat16, M, N), (torch.bfloat16, M, N + 32), (torch.bfloat16, 2 * M, N), (torch.float32, M, N),
             (torch.float32, 2 * M, N + 8), (torch.bfloat16, M, N)]
    for rnd in range(2):
        for dt, rows, ld in geoms:
            pool.view(dt).fill_(float("nan"))
            out = view(dt, rows, ld)
            ops.gemm(L.GEMM_NT, a[:rows], b, out=out)
            what = f"round {rnd} {dt} rows={rows} ld={ld}"
            assert not torch.isnan(out.float()).any(), what
            _close(out, prod[:rows], K, dt, what)
        # the same base as the pre-activation copy (64 x 64 box) of another call, then again as D
        pool.view(torch.bfloat16).fill_(float("nan"))
        other = torch.empty(M, N, dtype=torch.float32, device=DEV)
        aux = view(torch.bfloat16, M, N)
        ops.gemm(L.GEMM_NT, a[:M], b, out=other, aux=aux, epilogue=L.EPI_GELU_ERF)
        _close(aux, prod[:M], K, torch.bfloat16, f"round {rnd} aux on a reused base")
        _close(other, _gelu_erf(prod[:M]), K, torch.float32, f"round {rnd} D beside it")
