"""Tensor-level wrappers over the C ABI: torch is used only for device memory and the current stream.

Each function validates what the C side cannot know (dtype, device, contiguity) and forwards raw pointers.
No function here has a PyTorch fallback path.
"""
import torch

from . import lib as L

_bf16 = torch.bfloat16
_ws_cache = {}


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _chk(t, dtype=None, name="tensor"):
    if not t.is_cuda:
        raise RuntimeError(f"fsb200: {name} must be a CUDA tensor (the hot path has no CPU fallback)")
    if dtype is not None and t.dtype != dtype:
        raise RuntimeError(f"fsb200: {name} must be {dtype}, got {t.dtype}")


def _rows2d(t, name):
    """View as [rows, cols] with unit inner stride; returns (rows, cols, ld)."""
    if t.dim() != 2 or t.stride(1) != 1:
        raise RuntimeError(f"fsb200: {name} must be 2-D with unit inner stride, got shape {tuple(t.shape)} "
                           f"strides {t.stride()}")
    return t.shape[0], t.shape[1], t.stride(0)


def _span(t, n, name, what):
    """Refuse t unless it is exactly the n contiguous elements the C entry addresses from its first element on."""
    if not t.is_contiguous() or t.numel() != n:
        raise RuntimeError(f"fsb200 {what}: {name} must be contiguous with {n} elements, got shape {tuple(t.shape)} "
                           f"strides {t.stride()}")


def workspace(nbytes, device, tag="default"):
    """Grow-only scratch buffer per (device, tag); caller-owned from the library's point of view."""
    key = (device, tag)
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(int(nbytes), 1 << 20), dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    return buf


# ------------------------------------------------------------------------------------------------------ GEMM
def gemm(layout, a, b, out=None, out_dtype=_bf16, bias=None, epilogue=L.EPI_NONE, accumulate=False, aux=None):
    """layout NT: a[M,K] b[N,K]; NN: a[M,K] b[K,N]; TN: a[K,M] b[K,N]. Returns out[M,N]."""
    _chk(a, _bf16, "a"); _chk(b, _bf16, "b")
    ar, ac, lda = _rows2d(a, "a")
    br, bc, ldb = _rows2d(b, "b")
    if layout == L.GEMM_NT:
        M, K, N = ar, ac, br
        if bc != K: raise RuntimeError(f"fsb200 gemm NT: K mismatch {ac} vs {bc}")
    elif layout == L.GEMM_NN:
        M, K, N = ar, ac, bc
        if br != K: raise RuntimeError(f"fsb200 gemm NN: K mismatch {ac} vs {br}")
    else:
        K, M, N = ar, ac, bc
        if br != K: raise RuntimeError(f"fsb200 gemm TN: K mismatch {ar} vs {br}")
    if out is None:
        if accumulate: raise RuntimeError("fsb200 gemm: accumulate needs an existing `out`")
        out = torch.empty((M, N), dtype=out_dtype, device=a.device)
    _chk(out, None, "out")
    if out.dtype not in (_bf16, torch.float32): raise RuntimeError("fsb200 gemm: out must be bf16 or fp32")
    orr, occ, ldd = _rows2d(out, "out")
    if (orr, occ) != (M, N): raise RuntimeError(f"fsb200 gemm: out shape {tuple(out.shape)} != ({M},{N})")
    bias_dt = L.BF16
    if bias is not None:
        _chk(bias, None, "bias")
        if bias.numel() != N or not bias.is_contiguous(): raise RuntimeError("fsb200 gemm: bias must be contiguous [N]")
        bias_dt = L.F32 if bias.dtype == torch.float32 else L.BF16
    ldaux = 0
    if aux is not None:
        _chk(aux, _bf16, "aux")
        if tuple(aux.shape) != (M, N): raise RuntimeError(f"fsb200 gemm: aux shape {tuple(aux.shape)} != ({M},{N})")
        _, _, ldaux = _rows2d(aux, "aux")
    ws, ws_bytes = None, 0
    if layout == L.GEMM_TN and bias is None and aux is None and epilogue == L.EPI_NONE:
        # asked on every call, not memoised per shape: the split plan follows fsb_set_reserved_sms
        ws_bytes = int(L.load().fsb_gemm_workspace_bytes(layout, M, N, K))
        if ws_bytes:
            ws = workspace(ws_bytes, a.device, "gemm_splitk")   # one stream issues the step's GEMMs: a shared scratch is safe
    prof = _profiler
    if prof is not None:
        ev0 = torch.cuda.Event(enable_timing=True); ev0.record()
    L.call("fsb_gemm_bf16", layout, M, N, K, _p(a), lda, _p(b), ldb, _p(out), ldd,
           L.F32 if out.dtype == torch.float32 else L.BF16, _p(bias), bias_dt, epilogue, int(bool(accumulate)),
           _p(aux), ldaux, 1, 0, 0, 0, 0, _p(ws), ws_bytes, _stream(),
           tag=(f"{('NT', 'NN', 'TN')[layout]} {M}x{N}x{K} epi{epilogue} acc{int(bool(accumulate))} "
                f"{'f32' if out.dtype == torch.float32 else 'bf16'}{' bias' if bias is not None else ''}"
                f"{' aux' if aux is not None else ''}") if L.call_profiler is not None else None)
    if prof is not None:
        ev1 = torch.cuda.Event(enable_timing=True); ev1.record()
        prof.add("gemm_bf16_kernel", ev0, ev1, 2.0 * M * N * K)
    return out


def quantize_w8(w, q=None, s=None):
    """Symmetric per-output-channel int8 quantisation of a bf16 weight w[n, k] (unit inner stride) -> (q int8 [n, k]
    contiguous, s fp32 [n]) with s = absmax / 127 and q = clamp(rint(w / s), -127, 127) (include/fsb200.h). q and s may be
    given (contiguous, e.g. row slices of a larger operand) to quantise in place of a new allocation."""
    _chk(w, _bf16, "w")
    n, k, ldw = _rows2d(w, "w")
    q = torch.empty((n, k), dtype=torch.int8, device=w.device) if q is None else q
    s = torch.empty((n,), dtype=torch.float32, device=w.device) if s is None else s
    _chk(q, torch.int8, "q"); _chk(s, torch.float32, "s")
    if tuple(q.shape) != (n, k) or not q.is_contiguous() or tuple(s.shape) != (n,) or not s.is_contiguous():
        raise RuntimeError(f"fsb200 quantize_w8: q must be contiguous [{n}, {k}] and s contiguous [{n}]")
    L.call("fsb_quantize_w8", _p(w), ldw, n, k, _p(q), _p(s), _stream())
    return q, s


def _wq_bias(what, bias, epilogue, n):
    """The bias / epilogue arguments of gemm_w8a16 / gemm_w4a16 checked: bias None (the plain GEMM: epilogue must be
    EPI_NONE) or a contiguous bf16 [n] tensor with epilogue EPI_NONE or EPI_GELU_TANH."""
    if bias is None:
        if epilogue != L.EPI_NONE:
            raise RuntimeError(f"fsb200 {what}: an epilogue needs a bias (the bias-free GEMM has none)")
        return
    _chk(bias, _bf16, "bias")
    if bias.numel() != n or not bias.is_contiguous():
        raise RuntimeError(f"fsb200 {what}: bias must be contiguous [{n}], got shape {tuple(bias.shape)}")
    if epilogue not in (L.EPI_NONE, L.EPI_GELU_TANH):
        raise RuntimeError(f"fsb200 {what}: epilogue {epilogue} unsupported (EPI_NONE or EPI_GELU_TANH)")


def _wq_call(what, m, n, k, a, lda, q, s, out, ldd, ws, ws_bytes, bias, epilogue):
    """fsb_<what> without a bias, fsb_<what>_bias with one."""
    tag = f"{m}x{n}x{k}{'' if bias is None else f' bias epi{epilogue}'}" if L.call_profiler is not None else None
    if bias is None:
        L.call(f"fsb_{what}", m, n, k, _p(a), lda, _p(q), _p(s), _p(out), ldd, _p(ws), ws_bytes, _stream(), tag=tag)
    else:
        L.call(f"fsb_{what}_bias", m, n, k, _p(a), lda, _p(q), _p(s), _p(bias), epilogue, _p(out), ldd, _p(ws), ws_bytes,
               _stream(), tag=tag)


def gemm_w8a16(a, q, s, out=None, bias=None, epilogue=L.EPI_NONE):
    """out[m, n] = bf16(s[n] * (a[m, k] @ q[n, k]^T)), fp32 accumulation: a bf16 (unit inner stride), q int8 [n, k]
    contiguous and s fp32 [n] as quantize_w8 returns them. `out` (bf16, unit inner stride) may be a strided view.
    bias (bf16 [n]): out = bf16(act(s[n] * (a @ q^T) + bias[n])), act by epilogue (EPI_NONE or EPI_GELU_TANH), through
    fsb_gemm_w8a16_bias; None makes the bias-free call."""
    _chk(a, _bf16, "a"); _chk(q, torch.int8, "q"); _chk(s, torch.float32, "s")
    m, k, lda = _rows2d(a, "a")
    if q.dim() != 2 or not q.is_contiguous(): raise RuntimeError("fsb200 gemm_w8a16: q must be contiguous [n, k]")
    n = q.shape[0]
    if q.shape[1] != k: raise RuntimeError(f"fsb200 gemm_w8a16: K mismatch {k} vs {q.shape[1]}")
    if tuple(s.shape) != (n,) or not s.is_contiguous(): raise RuntimeError("fsb200 gemm_w8a16: s must be contiguous [n]")
    if out is None:
        out = torch.empty((m, n), dtype=_bf16, device=a.device)
    _chk(out, _bf16, "out")
    orr, occ, ldd = _rows2d(out, "out")
    if (orr, occ) != (m, n): raise RuntimeError(f"fsb200 gemm_w8a16: out shape {tuple(out.shape)} != ({m},{n})")
    _wq_bias("gemm_w8a16", bias, epilogue, n)
    ws_bytes = int(L.load().fsb_gemm_w8a16_workspace_bytes(m, n, k))
    ws = workspace(ws_bytes, a.device, "gemm_w8a16") if ws_bytes else None
    _wq_call("gemm_w8a16", m, n, k, a, lda, q, s, out, ldd, ws, ws_bytes, bias, epilogue)
    return out


def quantize_w4(w, q=None, s=None):
    """Symmetric int4 quantisation of a bf16 weight w[n, k] (unit inner stride) with one scale per row and group of 128 k
    -> (q uint8 [n / 2, k] contiguous, two 4-bit codes per byte, s bf16 [n, k / 128] contiguous) with
    s = bf16(absmax / 7) and q = clamp(rint(w / s), -7, 7); include/fsb200.h gives the packed layout. q and s may be given
    (contiguous, e.g. row slices of a larger operand: an even number of rows) to quantise in place of a new allocation."""
    _chk(w, _bf16, "w")
    n, k, ldw = _rows2d(w, "w")
    if n % 2 or k % 128:
        raise RuntimeError(f"fsb200 quantize_w4: w [{n}, {k}] needs k a multiple of 128 and n a multiple of 8")
    q = torch.empty((n // 2, k), dtype=torch.uint8, device=w.device) if q is None else q
    s = torch.empty((n, k // 128), dtype=_bf16, device=w.device) if s is None else s
    _chk(q, torch.uint8, "q"); _chk(s, _bf16, "s")
    if tuple(q.shape) != (n // 2, k) or not q.is_contiguous() or tuple(s.shape) != (n, k // 128) or not s.is_contiguous():
        raise RuntimeError(f"fsb200 quantize_w4: q must be contiguous [{n // 2}, {k}] and s contiguous [{n}, {k // 128}]")
    L.call("fsb_quantize_w4", _p(w), ldw, n, k, _p(q), _p(s), _stream())
    return q, s


def gemm_w4a16(a, q, s, out=None, bias=None, epilogue=L.EPI_NONE):
    """out[m, n] = bf16(a[m, k] @ W^[n, k]^T), fp32 accumulation, W^ = bf16(q * s) the dequantised int4 weight: a bf16
    (unit inner stride), q uint8 [n / 2, k] and s bf16 [n, k / 128] contiguous as quantize_w4 returns them. `out` (bf16,
    unit inner stride) may be a strided view. bias / epilogue as gemm_w8a16 (fsb_gemm_w4a16_bias)."""
    _chk(a, _bf16, "a"); _chk(q, torch.uint8, "q"); _chk(s, _bf16, "s")
    m, k, lda = _rows2d(a, "a")
    if q.dim() != 2 or not q.is_contiguous(): raise RuntimeError("fsb200 gemm_w4a16: q must be contiguous [n / 2, k]")
    n = 2 * q.shape[0]
    if q.shape[1] != k: raise RuntimeError(f"fsb200 gemm_w4a16: K mismatch {k} vs {q.shape[1]}")
    if s.dim() != 2 or s.shape[0] != n or s.shape[1] * 128 != k or not s.is_contiguous():
        raise RuntimeError(f"fsb200 gemm_w4a16: s must be contiguous [{n}, k / 128] for k = {k}")
    if out is None:
        out = torch.empty((m, n), dtype=_bf16, device=a.device)
    _chk(out, _bf16, "out")
    orr, occ, ldd = _rows2d(out, "out")
    if (orr, occ) != (m, n): raise RuntimeError(f"fsb200 gemm_w4a16: out shape {tuple(out.shape)} != ({m},{n})")
    _wq_bias("gemm_w4a16", bias, epilogue, n)
    ws_bytes = int(L.load().fsb_gemm_w4a16_workspace_bytes(m, n, k))
    ws = workspace(ws_bytes, a.device, "gemm_w4a16") if ws_bytes else None
    _wq_call("gemm_w4a16", m, n, k, a, lda, q, s, out, ldd, ws, ws_bytes, bias, epilogue)
    return out


FP8_FORMATS = {"e4m3": (0, torch.float8_e4m3fn), "e5m2": (1, torch.float8_e5m2)}   # name -> (fsb_fp8_format, code dtype)
_FP8_CODE = {dt: code for code, dt in FP8_FORMATS.values()}


def fp8_quantize(x, fmt, rowwise=True, colwise=False):
    """Per-tensor FP8 quantisation of a bf16 x [rows, cols] (unit inner stride, row stride a multiple of 8; rows and cols
    multiples of 16) in format `fmt` ("e4m3" or "e5m2") -> (y [rows, cols] or None, yt [cols, rows] or None, scale_inv fp32
    [1]): the row-major codes if `rowwise`, the transposed codes if `colwise` (torch.float8_e4m3fn / float8_e5m2 tensors), and
    1 / scale, the scale being the power of two 2^floor(log2(fmax / amax)); include/fsb200.h gives the rule, the rounding and
    the NaN convention."""
    _chk(x, _bf16, "x")
    if fmt not in FP8_FORMATS:
        raise RuntimeError(f"fsb200 fp8_quantize: format {fmt!r} is not one of {sorted(FP8_FORMATS)}")
    code, dt = FP8_FORMATS[fmt]
    rows, cols, ldx = _rows2d(x, "x")
    y = torch.empty((rows, cols), dtype=dt, device=x.device) if rowwise else None
    yt = torch.empty((cols, rows), dtype=dt, device=x.device) if colwise else None
    sinv = torch.empty(2, dtype=torch.float32, device=x.device)   # [scale_inv, amax]
    L.call("fsb_fp8_quantize", _p(x), ldx, rows, cols, code, _p(y), _p(yt), _p(sinv), _p(sinv[1:]), _stream())
    return y, yt, sinv[:1]


def gemm_fp8(a, a_scale_inv, b, b_scale_inv, out=None, accumulate=False, bias=None, epilogue=L.EPI_NONE, aux=None,
             store_transposed=False):
    """out[m, n] (+)= bf16((a[m, k] @ b[n, k]^T) * a_scale_inv * b_scale_inv), fp32 accumulation: a and b contiguous FP8
    codes as fp8_quantize returns them, (e4m3, e4m3) or (e5m2, e4m3); the scales fp32 [1] device tensors. `out` (bf16, unit
    inner stride) may be a strided view; `accumulate` adds into it with one rounding. bias (bf16 [n], contiguous), epilogue
    and aux (bf16 [m, n], unit inner stride) as in `gemm`: scaled product (+ bias) -> aux -> activation -> (+ out).
    store_transposed: out is [n, m] and receives the result transposed, bit for bit (fsb_gemm_fp8_t, a GPT-2 Conv1D's
    [in, out] weight gradient from dy^T and x^T codes): (e5m2, e4m3) codes only, m a multiple of 8, any n; bias, epilogue
    and aux are refused."""
    op = "gemm_fp8_t" if store_transposed else "gemm_fp8"
    _chk(a_scale_inv, torch.float32, "a_scale_inv"); _chk(b_scale_inv, torch.float32, "b_scale_inv")
    for t, name in ((a, "a"), (b, "b")):
        _chk(t, None, name)
        if t.dtype not in _FP8_CODE: raise RuntimeError(f"fsb200 {op}: {name} must hold FP8 codes, got {t.dtype}")
        if t.dim() != 2 or not t.is_contiguous(): raise RuntimeError(f"fsb200 {op}: {name} must be contiguous 2-D")
    m, k = a.shape
    n = b.shape[0]
    if b.shape[1] != k: raise RuntimeError(f"fsb200 {op}: K mismatch {k} vs {b.shape[1]}")
    shape = (n, m) if store_transposed else (m, n)
    if out is None:
        if accumulate: raise RuntimeError(f"fsb200 {op}: accumulate needs an existing `out`")
        out = torch.empty(shape, dtype=_bf16, device=a.device)
    _chk(out, _bf16, "out")
    orr, occ, ldd = _rows2d(out, "out")
    if (orr, occ) != shape: raise RuntimeError(f"fsb200 {op}: out shape {tuple(out.shape)} != ({shape[0]},{shape[1]})")
    if bias is not None:
        _chk(bias, _bf16, "bias")
        if bias.numel() != n or not bias.is_contiguous(): raise RuntimeError(f"fsb200 {op}: bias must be contiguous [{n}]")
    ldaux = 0
    if aux is not None:
        _chk(aux, _bf16, "aux")
        if tuple(aux.shape) != (m, n): raise RuntimeError(f"fsb200 {op}: aux shape {tuple(aux.shape)} != ({m},{n})")
        _, _, ldaux = _rows2d(aux, "aux")
    L.call("fsb_" + op, m, n, k, _p(a), _FP8_CODE[a.dtype], _p(a_scale_inv), _p(b), _FP8_CODE[b.dtype], _p(b_scale_inv),
           _p(out), ldd, _p(bias), epilogue, int(bool(accumulate)), _p(aux), ldaux, _stream(),
           tag=(f"{m}x{n}x{k} epi{epilogue} acc{int(bool(accumulate))}{' bias' if bias is not None else ''}"
                f"{' aux' if aux is not None else ''}") if L.call_profiler is not None else None)
    return out


def set_reserved_sms(n):
    """Leave n SMs (2n for CTA-pair kernels) of every persistent GEMM grid to overlapping communication kernels."""
    L.call("fsb_set_reserved_sms", int(n))


class KernelProfiler:
    """CUDA-event timing of individual launches on the launching stream (bench.py's roofline block)."""

    def __init__(self):
        self.rec = {}

    def add(self, name, ev0, ev1, work):
        self.rec.setdefault(name, []).append((ev0, ev1, work))

    def summary(self):
        out = {}
        for name, items in self.rec.items():
            ms = sum(a.elapsed_time(b) for a, b, _ in items)
            out[name] = {"launches": len(items), "ms": ms, "work": sum(w for _, _, w in items)}
        return out


_profiler = None


def set_profiler(p):
    global _profiler
    _profiler = p


# ------------------------------------------------------------------------------------------------------ norms
def rmsnorm_fwd(x, scale, eps, residual=None, drop=None):
    """x [rows, cols] bf16. Returns (y, rstd, x_sum) where x_sum = x + residual (or x itself when residual is None).
    drop: optional Dropout (see `Dropout`): x_sum = dropout(x) + residual (the dropped branch of a residual block)."""
    _chk(x, _bf16, "x"); _chk(scale, _bf16, "scale")
    rows, cols = x.shape
    y = torch.empty_like(x)
    rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
    xs = torch.empty_like(x) if residual is not None else None
    if drop is None:
        L.call("fsb_rmsnorm_fwd", _p(x), _p(residual), _p(scale), _p(y), _p(xs), _p(rstd), rows, cols, float(eps), _stream())
    else:
        L.call("fsb_rmsnorm_fwd_dropout", _p(x), _p(residual), _p(scale), _p(y), _p(xs), _p(rstd), rows, cols, float(eps),
               *drop.args(), _stream())
    return y, rstd, (xs if residual is not None else x)


def rmsnorm_bwd(dy, x, scale, rstd, dscale_out, accumulate=False, dres=None):
    rows, cols = x.shape
    _span(dscale_out, cols, "dscale_out", "rmsnorm_bwd")
    dx = torch.empty_like(x)
    nbytes = L.load().fsb_norm_bwd_workspace_bytes(rows, cols, 0)
    ws = workspace(nbytes, x.device, "norm")
    L.call("fsb_rmsnorm_bwd", _p(dy), _p(x), _p(scale), _p(rstd), _p(dres), _p(dx), _p(dscale_out),
           L.F32 if dscale_out.dtype == torch.float32 else L.BF16, int(bool(accumulate)), _p(ws), ws.numel(), rows, cols,
           _stream())
    return dx


def rmsnorm_bwd_dropout(dy, x, scale, rstd, dscale_out, drop, accumulate=False, dres=None):
    """Backward of rmsnorm_fwd(..., residual, drop): returns (dx, dbranch) — the gradient of the sum (= of the residual)
    and the gradient of the dropped branch, dx * Z / (1 - p)."""
    rows, cols = x.shape
    _span(dscale_out, cols, "dscale_out", "rmsnorm_bwd")
    dx = torch.empty_like(x)
    dbranch = torch.empty_like(x)
    nbytes = L.load().fsb_norm_bwd_workspace_bytes(rows, cols, 0)
    ws = workspace(nbytes, x.device, "norm")
    L.call("fsb_rmsnorm_bwd_dropout", _p(dy), _p(x), _p(scale), _p(rstd), _p(dres), _p(dx), _p(dbranch), _p(dscale_out),
           L.F32 if dscale_out.dtype == torch.float32 else L.BF16, int(bool(accumulate)), _p(ws), ws.numel(), rows, cols,
           *drop.args(), _stream())
    return dx, dbranch


def layernorm_fwd(x, gamma, beta, eps, residual=None, drop=None):
    """drop: optional Dropout (see `Dropout`): x_sum = dropout(x) + residual (the dropped branch of a residual block)."""
    _chk(x, _bf16, "x"); _chk(gamma, _bf16, "gamma"); _chk(beta, _bf16, "beta")
    rows, cols = x.shape
    y = torch.empty_like(x)
    stats = torch.empty(rows, 2, dtype=torch.float32, device=x.device)
    xs = torch.empty_like(x) if residual is not None else None
    if drop is None:
        L.call("fsb_layernorm_fwd", _p(x), _p(residual), _p(gamma), _p(beta), _p(y), _p(xs), _p(stats), rows, cols,
               float(eps), _stream())
    else:
        L.call("fsb_layernorm_fwd_dropout", _p(x), _p(residual), _p(gamma), _p(beta), _p(y), _p(xs), _p(stats), rows, cols,
               float(eps), *drop.args(), _stream())
    return y, stats, (xs if residual is not None else x)


def layernorm_bwd(dy, x, gamma, stats, dgamma_out, dbeta_out, accumulate=False, dres=None):
    rows, cols = x.shape
    _span(dgamma_out, cols, "dgamma_out", "layernorm_bwd"); _span(dbeta_out, cols, "dbeta_out", "layernorm_bwd")
    dx = torch.empty_like(x)
    nbytes = L.load().fsb_norm_bwd_workspace_bytes(rows, cols, 1)
    ws = workspace(nbytes, x.device, "norm")
    L.call("fsb_layernorm_bwd", _p(dy), _p(x), _p(gamma), _p(stats), _p(dres), _p(dx), _p(dgamma_out), _p(dbeta_out),
           L.F32 if dgamma_out.dtype == torch.float32 else L.BF16, int(bool(accumulate)), _p(ws), ws.numel(), rows, cols,
           _stream())
    return dx


def layernorm_bwd_dropout(dy, x, gamma, stats, dgamma_out, dbeta_out, drop, accumulate=False, dres=None):
    """Backward of layernorm_fwd(..., residual, drop): returns (dx, dbranch) — the gradient of the sum (= of the residual)
    and the gradient of the dropped branch, dx * Z / (1 - p)."""
    rows, cols = x.shape
    _span(dgamma_out, cols, "dgamma_out", "layernorm_bwd"); _span(dbeta_out, cols, "dbeta_out", "layernorm_bwd")
    dx = torch.empty_like(x)
    dbranch = torch.empty_like(x)
    nbytes = L.load().fsb_norm_bwd_workspace_bytes(rows, cols, 1)
    ws = workspace(nbytes, x.device, "norm")
    L.call("fsb_layernorm_bwd_dropout", _p(dy), _p(x), _p(gamma), _p(stats), _p(dres), _p(dx), _p(dbranch), _p(dgamma_out),
           _p(dbeta_out), L.F32 if dgamma_out.dtype == torch.float32 else L.BF16, int(bool(accumulate)), _p(ws), ws.numel(),
           rows, cols, *drop.args(), _stream())
    return dx, dbranch


# ------------------------------------------------------------------------------------------------------ dropout
class Dropout:
    """One dropout site of one forward: probability p, the model's seed, the forward's stream base (int64 [1] on the
    device, from dropout_advance) and the site number. The keep mask is a function of these and of the element's coordinates
    only (include/fsb200.h), so the backward passes the same object."""
    __slots__ = ("p", "seed", "base", "site")

    def __init__(self, p, seed, base, site):
        if not 0.0 <= float(p) < 1.0:
            raise RuntimeError(f"fsb200 dropout: p = {p} outside [0, 1)")
        _chk(base, torch.int64, "dropout stream base")
        self.p, self.seed, self.base, self.site = float(p), int(seed), base, int(site)

    def args(self):
        return self.p, self.seed, _p(self.base), self.site


def dropout_advance(counter, n):
    """Advance the device stream counter (int64 [1]) by n streams, on the device; returns the base this forward uses (a new
    int64 [1] device tensor, saved with the activations for the backward)."""
    _chk(counter, torch.int64, "dropout counter")
    _span(counter, 1, "counter", "dropout_advance")
    saved = torch.empty(1, dtype=torch.int64, device=counter.device)
    L.call("fsb_dropout_advance", _p(counter), _p(saved), int(n), _stream())
    return saved


def dropout(x, drop, out=None):
    """out = x * Z / (1 - p) over bf16 [rows, cols]; also the backward (pass dy, get dx)."""
    _chk(x, _bf16, "x")
    rows, cols, ld = _rows2d(x, "x")
    if ld != cols:
        raise RuntimeError("fsb200 dropout: x must be contiguous")
    if out is None:
        out = torch.empty_like(x)
    _chk(out, _bf16, "out")
    _span(out, rows * cols, "out", "dropout")
    L.call("fsb_dropout", _p(x), _p(out), rows, cols, *drop.args(), _stream())
    return out


# ------------------------------------------------------------------------------------------------------ pointwise
def rope_inplace(x, cos, sin, positions, nheads, head_dim, row_stride, head_stride, backward=False, offset=0):
    """Rotate `nheads` heads per row in place. x is the flat packed buffer; `offset` (elements) selects q or k."""
    _chk(x, _bf16, "x")
    rows = positions.numel()
    end = offset + (rows - 1) * row_stride + (nheads - 1) * head_stride + head_dim
    if not x.is_contiguous() or offset < 0 or (rows > 0 and end > x.numel()):
        raise RuntimeError(f"fsb200 rope_inplace: the heads addressed (up to element {end}) must lie inside the contiguous "
                           f"x of {x.numel()} elements")
    L.call("fsb_rope_inplace", x.data_ptr() + 2 * offset, _p(cos), _p(sin), _p(positions), rows, nheads, head_dim,
           row_stride, head_stride, cos.shape[0], int(bool(backward)), _stream())


def glu_fwd(act, gate, up, drop=None):
    """out = act(gate) * up; drop: optional Dropout on out (out * Z / (1 - p))."""
    rows, cols, ldg = _rows2d(gate, "gate")
    _, _, ldu = _rows2d(up, "up")
    out = torch.empty((rows, cols), dtype=_bf16, device=gate.device)
    if drop is None:
        L.call("fsb_glu_fwd", act, _p(gate), _p(up), _p(out), rows, cols, ldg, ldu, cols, _stream())
    else:
        L.call("fsb_glu_fwd_dropout", act, _p(gate), _p(up), _p(out), rows, cols, ldg, ldu, cols, *drop.args(), _stream())
    return out


def glu_bwd(act, dout, gate, up, dgate, dup, drop=None):
    """drop: the forward's Dropout (the mask is applied to dout first)."""
    rows, cols, ldg = _rows2d(gate, "gate")
    _, _, ldu = _rows2d(up, "up")
    _, _, ldo = _rows2d(dout, "dout")
    _, _, ldg2 = _rows2d(dgate, "dgate")
    _, _, ldu2 = _rows2d(dup, "dup")
    for t, n in ((up, "up"), (dout, "dout"), (dgate, "dgate"), (dup, "dup")):
        if t.shape != gate.shape:
            raise RuntimeError(f"fsb200 glu_bwd: {n} shape {tuple(t.shape)} != gate shape {tuple(gate.shape)}")
    args = (act, _p(dout), _p(gate), _p(up), _p(dgate), _p(dup), rows, cols, ldo, ldg, ldu, ldg2, ldu2)
    if drop is None:
        L.call("fsb_glu_bwd", *args, _stream())
    else:
        L.call("fsb_glu_bwd_dropout", *args, *drop.args(), _stream())


def act_fwd(act, x):
    y = torch.empty_like(x)
    L.call("fsb_act_fwd", act, _p(x), _p(y), x.numel(), _stream())
    return y


def act_bwd(act, dy, x):
    dx = torch.empty_like(x)
    L.call("fsb_act_bwd", act, _p(dy), _p(x), _p(dx), x.numel(), _stream())
    return dx


def act_bwd_bias(act, dy, x, dbias, accumulate=False):
    """dx = dy * act'(x) and dbias[c] (+)= sum_r dx[r, c] in one pass (x, dy contiguous [rows, cols])."""
    _chk(x, _bf16, "x"); _chk(dy, _bf16, "dy")
    if not (x.is_contiguous() and dy.is_contiguous()) or x.dim() != 2 or dy.shape != x.shape:
        raise RuntimeError("fsb200 act_bwd_bias: x and dy must be contiguous [rows, cols] of the same shape")
    rows, cols = x.shape
    dx = torch.empty_like(x)
    _span(dbias, cols, "dbias", "act_bwd_bias")
    nbytes = L.load().fsb_act_bwd_bias_workspace_bytes(rows, cols)
    ws = workspace(nbytes, x.device, "act_bwd_bias")
    L.call("fsb_act_bwd_bias", act, _p(dy), _p(x), _p(dx), rows, cols, _p(dbias),
           L.F32 if dbias.dtype == torch.float32 else L.BF16, int(bool(accumulate)), _p(ws), ws.numel(), _stream())
    return dx


def add(a, b, out=None):
    if out is None: out = torch.empty_like(a)
    for t, n in ((a, "a"), (b, "b"), (out, "out")):
        _chk(t, _bf16, n); _span(t, a.numel(), n, "add")
    L.call("fsb_add", _p(a), _p(b), _p(out), a.numel(), _stream())
    return out


def accumulate(acc32, x16, scale=1.0, overwrite=False):
    """acc32 (fp32) = (0 if overwrite else acc32) + scale * x16 (bf16)."""
    _span(acc32, acc32.numel(), "acc32", "accumulate"); _span(x16, acc32.numel(), "x16", "accumulate")
    L.call("fsb_accumulate", _p(acc32), _p(x16), acc32.numel(), float(scale), int(bool(overwrite)), _stream())


def scale_inplace(x16, scale_dev):
    """x16 (bf16, contiguous) *= scale_dev (0-d fp32 CUDA tensor); free when the scalar is 1."""
    _span(x16, x16.numel(), "x16", "scale_inplace")
    if scale_dev.dtype != torch.float32 or not scale_dev.is_cuda:
        scale_dev = scale_dev.to(device=x16.device, dtype=torch.float32)
    L.call("fsb_scale_inplace", _p(x16), x16.numel(), _p(scale_dev), _stream())


def colsum(x, out, accumulate=False):
    """out[c] (+)= sum_r x[r, c]; x bf16 [rows, cols] (unit inner stride); out bf16 or fp32 [cols]."""
    rows, cols, ld = _rows2d(x, "x")
    _span(out, cols, "out", "colsum")
    nbytes = L.load().fsb_colsum_workspace_bytes(rows, cols)
    ws = workspace(nbytes, x.device, "colsum")
    L.call("fsb_colsum", _p(x), rows, cols, ld, _p(out), L.F32 if out.dtype == torch.float32 else L.BF16,
           int(bool(accumulate)), _p(ws), ws.numel(), _stream())


def embedding_fwd(ids, W, pos=None, P=None, token_type=None, T=None, seq_len=1):
    rows = ids.numel()
    cols = W.shape[1]
    out = torch.empty((rows, cols), dtype=_bf16, device=W.device)
    L.call("fsb_embedding_fwd", _p(ids), _p(pos), _p(token_type), _p(W), _p(P), _p(T), _p(out), rows, cols, seq_len,
           _stream())
    return out


def embedding_bwd(ids, dout, dW, idx_mod=0):
    """dW[ids[t]] += dout[t]. With ids: deterministic — the ids are sorted (torch.sort: integer index plumbing) and every
    distinct row is summed in fp32 in a fixed order, one bf16 rounding. ids=None: row t % idx_mod (bf16 atomics)."""
    rows, cols = dout.shape
    if dW.dim() != 2 or dW.shape[1] != cols or not dW.is_contiguous() or (ids is None and idx_mod > dW.shape[0]):
        raise RuntimeError(f"fsb200 embedding_bwd: dW must be contiguous [rows, {cols}] (and hold idx_mod rows), got "
                           f"{tuple(dW.shape)} strides {dW.stride()}")
    if ids is None:
        L.call("fsb_embedding_bwd", None, _p(dout), _p(dW), rows, cols, idx_mod, _stream())
        return
    ids_sorted, order = torch.sort(ids.view(-1), stable=True)
    L.call("fsb_embedding_bwd_sorted", _p(ids_sorted), _p(order), _p(dout), _p(dW), rows, cols, _stream())


def cast_f32_to_bf16(x32, out=None):
    if out is None:
        out = torch.empty(x32.shape, dtype=_bf16, device=x32.device)
    _chk(out, _bf16, "out")
    _span(x32, x32.numel(), "x32", "cast_f32_to_bf16"); _span(out, x32.numel(), "out", "cast_f32_to_bf16")
    L.call("fsb_cast_f32_to_bf16", _p(x32), _p(out), x32.numel(), _stream())
    return out


# ------------------------------------------------------------------------------------------------------ loss / optim
def softmax_xent(logits, labels, seq_len, shift=1, ignore_index=-100, grad_scale=1.0, dlogits="inplace"):
    """logits [rows, V] bf16 (rows = b*seq_len), labels int64 [rows]. Returns (loss scalar tensor, dlogits, n_valid).
    dlogits: "inplace" (into logits), None / "none" (not computed) or a bf16 [rows, V] tensor with the logits' row stride."""
    _chk(logits, _bf16, "logits")
    rows, V, ld = _rows2d(logits, "logits")
    dev = logits.device
    row_loss = torch.empty(rows, dtype=torch.float32, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    n_valid = torch.empty((), dtype=torch.int32, device=dev)
    if isinstance(dlogits, str):
        dl = logits if dlogits == "inplace" else None
    else:
        dl = dlogits
    if dl is not None and dl is not logits:   # the entry writes dlogits with the logits' row stride (include/fsb200.h)
        _chk(dl, _bf16, "dlogits")
        if tuple(dl.shape) != (rows, V) or dl.stride(1) != 1 or (rows > 1 and dl.stride(0) != ld):
            raise RuntimeError(f"fsb200 softmax_xent: dlogits must be bf16 [{rows}, {V}] with the logits' row stride {ld}, "
                               f"got shape {tuple(dl.shape)} strides {dl.stride()}")
    L.call("fsb_softmax_xent_fwd_bwd", _p(logits), _p(labels), _p(dl), _p(row_loss), _p(loss), _p(n_valid), rows, V, ld,
           seq_len, shift, ignore_index, float(grad_scale), _stream())
    return loss, dl, n_valid


def adamw_flat(master, m, v, grad, param16, lr, beta1, beta2, eps, weight_decay, step, grad_scale=None, hyper=None):
    """hyper: optional fp32 CUDA tensor [lr, 1 - beta1^t, sqrt(1 - beta2^t)] read by the kernel instead of lr / step."""
    n = master.numel()
    for t, name in ((master, "master"), (m, "m"), (v, "v"), (grad, "grad"), (param16, "param16")):
        if t is not None:
            _span(t, n, name, "adamw_flat")
    L.call("fsb_adamw_flat", _p(master), _p(m), _p(v), _p(grad), L.F32 if grad.dtype == torch.float32 else L.BF16,
           _p(param16), master.numel(), float(lr), float(beta1), float(beta2), float(eps), float(weight_decay), int(step),
           _p(grad_scale), _p(hyper), _stream())


def sumsq(x, out, accumulate=False):
    _span(x, x.numel(), "x", "sumsq"); _span(out, 1, "out", "sumsq")
    nbytes = L.load().fsb_sumsq_workspace_bytes()
    ws = workspace(nbytes, x.device, "sumsq")
    L.call("fsb_sumsq", _p(x), L.F32 if x.dtype == torch.float32 else L.BF16, x.numel(), _p(out), int(bool(accumulate)),
           _p(ws), ws.numel(), _stream())


def clip_coef(sumsq_t, max_norm, coef_out, norm_out=None):
    _span(coef_out, 1, "coef_out", "clip_coef")
    if norm_out is not None:
        _span(norm_out, 1, "norm_out", "clip_coef")
    L.call("fsb_clip_coef", _p(sumsq_t), float(max_norm), _p(coef_out), _p(norm_out), _stream())


# ------------------------------------------------------------------------------------------------------ attention
def _bshd(t, name):
    """[batch, seq, heads, dim] view with unit inner stride and batch stride == seq * row stride."""
    if t.dim() != 4 or t.stride(3) != 1:
        raise RuntimeError(f"fsb200: {name} must be [batch, seq, heads, dim] with unit inner stride")
    B, S, H, D = t.shape
    if B > 1 and t.stride(0) != S * t.stride(1):
        raise RuntimeError(f"fsb200: {name} batch stride {t.stride(0)} != seq*row_stride {S * t.stride(1)}")
    return B, S, H, D, t.stride(1), t.stride(2)


def _chk_rel(rel, H, Sq, Skv, name):
    _chk(rel, torch.float32, name)
    if tuple(rel.shape) != (H, Sq + Skv - 1) or not rel.is_contiguous():
        raise RuntimeError(f"fsb200: {name} must be contiguous fp32 [heads, seq_q + seq_kv - 1] = [{H}, {Sq + Skv - 1}], "
                           f"got {tuple(rel.shape)}")


def sdpa_fwd(q, k, v, scale, causal, kv_mask=None, out=None, rel_bias=None, drop=None):
    """q,k,v: strided [B,S,H,D] bf16 views (e.g. slices of the packed QKV projection). Returns (out [B,Sq,H,D], lse).
    causal: mask the keys after each query (seq_q == seq_kv); the key tiles wholly above the diagonal are skipped.
    kv_mask: optional uint8 [B, Skv] key-padding mask (0: masked). rel_bias: optional fp32 [H, Sq + Skv - 1] additive bias
    over the offset k - q (T5 relative-position bias). drop: optional Dropout on the attention probabilities, its keep mask
    the attention layout of include/fsb200.h. The causal flag, kv_mask, rel_bias and drop compose. head_dim 64 or 128; 96
    (GPT-2 3.5B) with causal=True and no rel_bias only."""
    return _sdpa_fwd(q, k, v, scale, causal, kv_mask, rel_bias, drop, out)


def _sdpa_fwd(q, k, v, scale, causal, kv_mask, rel_bias, drop, out, bounds=(None,) * 4):
    """The one fsb_sdpa_fwd call of sdpa_fwd and sdpa_segments_fwd. bounds: (seg_start, seg_end, q_start, q_end), each
    None or contiguous int32, the query-side pair [B, Sq] and the key-side pair [B, Skv]; the arguments select the form."""
    _chk(q, _bf16, "q"); _chk(k, _bf16, "k"); _chk(v, _bf16, "v")
    B, Sq, H, D, q_rs, q_hs = _bshd(q, "q")
    _, Skv, _, _, k_rs, k_hs = _bshd(k, "k")
    _, _, _, _, v_rs, v_hs = _bshd(v, "v")
    if out is None:
        out = torch.empty((B, Sq, H, D), dtype=_bf16, device=q.device)
    if tuple(out.shape) != (B, Sq, H, D): raise RuntimeError(f"fsb200: out shape {tuple(out.shape)} != {(B, Sq, H, D)}")
    _, _, _, _, o_rs, o_hs = _bshd(out, "out")
    lse = torch.empty((B, H, Sq), dtype=torch.float32, device=q.device)
    if kv_mask is not None:
        _chk(kv_mask, torch.uint8, "kv_mask")
        if tuple(kv_mask.shape) != (B, Skv) or not kv_mask.is_contiguous():
            raise RuntimeError("fsb200: kv_mask must be contiguous uint8 [batch, seq_kv]")
    if rel_bias is not None:
        _chk_rel(rel_bias, H, Sq, Skv, "rel_bias")
    _chk_bounds(bounds, B, Sq, Skv)
    L.call("fsb_sdpa_fwd", _p(q), _p(k), _p(v), _p(out), _p(lse), B, Sq, Skv, H, D, q_rs, k_rs, v_rs, o_rs, q_hs, k_hs,
           v_hs, o_hs, float(scale), int(bool(causal)), _p(kv_mask), _p(rel_bias), *map(_p, bounds),
           *(_NO_DROP if drop is None else drop.args()), _stream())
    return out, lse


def attn_decode(q, k_cache, v_cache, kv_len, scale, kv_mask=None, rel_bias=None, out=None):
    """One decode step: q [B, H, D] (the newest token, at cache slot kv_len - 1) against k_cache / v_cache [B, cap, H, D]
    (strided bf16 views, unit inner stride). kv_len: int32 CUDA scalar. kv_mask: uint8 [B, cap]. rel_bias: fp32
    [H, 2 cap - 1] (sdpa_fwd's convention with seq_q = seq_kv = cap). Returns (out [B, H, D], lse [B, H] log2 domain)."""
    for t, n in ((q, "q"), (k_cache, "k_cache"), (v_cache, "v_cache")):
        _chk(t, _bf16, n)
    if q.dim() != 3 or q.stride(2) != 1:
        raise RuntimeError("fsb200 attn_decode: q must be [batch, heads, dim] with unit inner stride")
    B, H, D = q.shape
    cap = _chk_cache(k_cache, v_cache, kv_mask, kv_len, B, H, D, "attn_decode")
    if out is None:
        out = torch.empty((B, H, D), dtype=_bf16, device=q.device)
    _chk(out, _bf16, "out")
    if tuple(out.shape) != (B, H, D) or out.stride(2) != 1:
        raise RuntimeError("fsb200 attn_decode: out must be [batch, heads, dim] with unit inner stride")
    if rel_bias is not None:
        _chk_rel(rel_bias, H, cap, cap, "rel_bias")
    lse = torch.empty((B, H), dtype=torch.float32, device=q.device)
    ws_bytes = int(L.load().fsb_attn_decode_workspace_bytes(B, H, D, cap))
    ws = workspace(ws_bytes, q.device, "attn_decode")
    L.call("fsb_attn_decode", _p(q), _p(k_cache), _p(v_cache), _p(out), _p(lse), B, H, D, cap, _p(kv_len),
           q.stride(0), q.stride(1), k_cache.stride(0), k_cache.stride(1), k_cache.stride(2),
           v_cache.stride(0), v_cache.stride(1), v_cache.stride(2), out.stride(0), out.stride(1), float(scale),
           _p(kv_mask), _p(rel_bias), _p(ws), ws_bytes, _stream())
    return out, lse


def _chk_kv_len(kv_len, what):
    _chk(kv_len, torch.int32, "kv_len")
    if kv_len.numel() != 1:
        raise RuntimeError(f"fsb200 {what}: kv_len must be a one-element int32 tensor")


def _chk_cache(k_cache, v_cache, kv_mask, kv_len, B, H, D, what):
    """The decode ops' cache operands: k_cache / v_cache [B, cap, H, D] (unit inner stride), kv_mask None or contiguous
    uint8 [B, cap], kv_len a one-element int32 tensor. Returns cap."""
    for t, n in ((k_cache, "k_cache"), (v_cache, "v_cache")):
        if t.dim() != 4 or t.stride(3) != 1 or (t.shape[0], t.shape[2], t.shape[3]) != (B, H, D):
            raise RuntimeError(f"fsb200 {what}: {n} must be [{B}, cap, {H}, {D}] with unit inner stride, "
                               f"got {tuple(t.shape)} strides {t.stride()}")
    cap = k_cache.shape[1]
    if v_cache.shape[1] != cap:
        raise RuntimeError(f"fsb200 {what}: k_cache and v_cache capacities differ")
    _chk_kv_len(kv_len, what)
    if kv_mask is not None:
        _chk(kv_mask, torch.uint8, "kv_mask")
        if tuple(kv_mask.shape) != (B, cap) or not kv_mask.is_contiguous():
            raise RuntimeError(f"fsb200 {what}: kv_mask must be contiguous uint8 [{B}, {cap}]")
    return cap


def kv_append(k_new, v_new, k_cache, v_cache, kv_len, kv_mask=None):
    """Write the newest token's keys / values k_new, v_new [B, H, D] (strided bf16 views, unit inner stride) into slot
    kv_len - 1 of k_cache / v_cache [B, cap, H, D] (strided views, e.g. the K and V halves of a [B, cap, 2, H, D] cache).
    kv_len: int32 CUDA scalar (read on the device). kv_mask: optional uint8 [B, cap]; its bit at that slot is set to 1.
    A slot outside [0, cap) writes nothing."""
    for t, n in ((k_new, "k_new"), (v_new, "v_new"), (k_cache, "k_cache"), (v_cache, "v_cache")):
        _chk(t, _bf16, n)
    if k_new.dim() != 3 or k_new.stride(2) != 1:
        raise RuntimeError("fsb200 kv_append: k_new must be [batch, heads, dim] with unit inner stride")
    B, H, D = k_new.shape
    if tuple(v_new.shape) != (B, H, D) or v_new.stride(2) != 1:
        raise RuntimeError(f"fsb200 kv_append: v_new must be [{B}, {H}, {D}] with unit inner stride")
    cap = _chk_cache(k_cache, v_cache, kv_mask, kv_len, B, H, D, "kv_append")
    L.call("fsb_kv_append", _p(k_new), _p(v_new), _p(k_cache), _p(v_cache), _p(kv_mask), B, H, D, cap, _p(kv_len),
           k_new.stride(0), k_new.stride(1), v_new.stride(0), v_new.stride(1), k_cache.stride(0), k_cache.stride(1),
           k_cache.stride(2), v_cache.stride(0), v_cache.stride(1), v_cache.stride(2), _stream())


def kv_reorder(src, dst, index, kv_len):
    """Beam-search gather of the caches of every layer, one launch: dst[l, r, s] = src[l, index[r], s] for the live slots
    s < kv_len (device int32 scalar); slots at or beyond it are neither read nor written. src / dst: contiguous bf16
    [layers, rows, cap, ...], distinct buffers. index: int64 [rows] on the device."""
    _chk(src, _bf16, "src"); _chk(dst, _bf16, "dst")
    if src.dim() < 3 or not src.is_contiguous() or not dst.is_contiguous() or src.shape != dst.shape:
        raise RuntimeError(f"fsb200 kv_reorder: src and dst must be contiguous bf16 [layers, rows, cap, ...] of one shape, "
                           f"got {tuple(src.shape)} and {tuple(dst.shape)}")
    layers, rows, cap = src.shape[:3]
    _chk(index, torch.int64, "index")
    if tuple(index.shape) != (rows,) or not index.is_contiguous():
        raise RuntimeError(f"fsb200 kv_reorder: index must be contiguous int64 [{rows}]")
    _chk_kv_len(kv_len, "kv_reorder")
    slot = src[0, 0, 0].numel()
    L.call("fsb_kv_reorder", _p(src), _p(dst), _p(index), layers, rows, cap, slot, _p(kv_len), _stream())


def _chk_grads(q, k, dq, dk, dv):
    """dq has q's shape and dk / dv have k's: the backward writes every element of each."""
    for t, ref, n in ((dq, q, "dq"), (dk, k, "dk"), (dv, k, "dv")):
        if t.shape != ref.shape:
            raise RuntimeError(f"fsb200: {n} shape {tuple(t.shape)} != {tuple(ref.shape)}")


def sdpa_bwd(q, k, v, out, dout, lse, scale, causal, dq, dk, dv, kv_mask=None, rel_bias=None, drel_bias=None, drop=None):
    """All tensors strided [B,S,H,D] bf16 views; dq/dk/dv are written (e.g. slices of a packed dQKV buffer).
    causal, kv_mask and rel_bias as in sdpa_fwd; drel_bias (fp32 [H, Sq + Skv - 1]) is accumulated into (+=),
    deterministically. drop: the forward's Dropout (same seed, base and site). head_dim as in sdpa_fwd."""
    _sdpa_bwd(q, k, v, out, dout, lse, scale, causal, dq, dk, dv, kv_mask, rel_bias, drel_bias, drop)


def _sdpa_bwd(q, k, v, out, dout, lse, scale, causal, dq, dk, dv, kv_mask, rel_bias, drel_bias, drop, bounds=(None,) * 4):
    """The one fsb_sdpa_bwd call of sdpa_bwd and sdpa_segments_bwd (bounds as in _sdpa_fwd)."""
    B, Sq, H, D, q_rs, q_hs = _bshd(q, "q")
    _, Skv, _, _, k_rs, k_hs = _bshd(k, "k")
    _, _, _, _, v_rs, v_hs = _bshd(v, "v")
    _, _, _, _, o_rs, o_hs = _bshd(out, "out")
    _, _, _, _, do_rs, do_hs = _bshd(dout, "dout")
    _, _, _, _, dq_rs, dq_hs = _bshd(dq, "dq")
    _, _, _, _, dk_rs, dk_hs = _bshd(dk, "dk")
    _, _, _, _, dv_rs, dv_hs = _bshd(dv, "dv")
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out"), (dout, "dout"), (dq, "dq"), (dk, "dk"), (dv, "dv")):
        _chk(t, _bf16, n)
    _chk_grads(q, k, dq, dk, dv)
    _chk_bounds(bounds, B, Sq, Skv)
    delta = torch.empty((B, H, Sq), dtype=torch.float32, device=q.device)
    ws, ws_bytes = None, 0
    if rel_bias is not None:
        _chk_rel(rel_bias, H, Sq, Skv, "rel_bias")
    if drel_bias is not None:
        _chk_rel(drel_bias, H, Sq, Skv, "drel_bias")
        ws_bytes = int(L.load().fsb_sdpa_bwd_workspace_bytes(B, Sq, Skv, H))
        ws = workspace(ws_bytes, q.device, "sdpa_dbias")
    L.call("fsb_sdpa_bwd", _p(q), _p(k), _p(v), _p(out), _p(dout), _p(lse), _p(delta), _p(dq), _p(dk), _p(dv), B, Sq, Skv,
           H, D, q_rs, k_rs, v_rs, o_rs, do_rs, dq_rs, dk_rs, dv_rs, q_hs, k_hs, v_hs, o_hs, do_hs, dq_hs, dk_hs, dv_hs,
           float(scale), int(bool(causal)), _p(kv_mask), _p(rel_bias), _p(drel_bias), _p(ws), ws_bytes, *map(_p, bounds),
           *(_NO_DROP if drop is None else drop.args()), _stream())


# ------------------------------------------------------------------------------------------------- packed sequences
def segment_bounds(segment_ids):
    """segment_ids: integer [B, S] (any device). A segment is a maximal run of equal consecutive values in a row, so every
    integer tensor is valid. Returns (seg_start, seg_end), contiguous int32 [B, S] on segment_ids' device: the row position of
    the first token of each token's segment and one past its last (include/fsb200.h, the segment forms of fsb_sdpa_fwd). Torch ops
    only, no host synchronisation: capturable in a CUDA graph."""
    if segment_ids.dim() != 2 or segment_ids.dtype.is_floating_point or segment_ids.dtype.is_complex or \
            segment_ids.dtype == torch.bool:
        raise RuntimeError(f"fsb200: segment_ids must be an integer [batch, seq] tensor, got {segment_ids.dtype} "
                           f"{tuple(segment_ids.shape)}")
    B, S = segment_ids.shape
    pos = torch.arange(S, dtype=torch.int32, device=segment_ids.device).expand(B, S)
    first = torch.ones((B, S), dtype=torch.bool, device=segment_ids.device)   # token starts a segment
    first[:, 1:] = segment_ids[:, 1:] != segment_ids[:, :-1]
    last = torch.ones_like(first)                                              # token ends one
    last[:, :-1] = first[:, 1:]
    start = torch.cummax(torch.where(first, pos, 0), dim=1).values
    end = torch.where(last, pos + 1, S).flip(1).cummin(dim=1).values.flip(1)
    return start.to(torch.int32).contiguous(), end.to(torch.int32).contiguous()


_NO_DROP = (0.0, 0, None, 0)   # p, seed, stream_base, site of an attention call without dropout


def _chk_bounds(bounds, B, Sq, Skv):
    """(seg_start, seg_end, q_start, q_end): each pair None or contiguous int32, [B, Sq] and [B, Skv]."""
    for t, n, S in zip(bounds, ("seg_start", "seg_end", "q_start", "q_end"), (Sq, Sq, Skv, Skv)):
        if t is None:
            continue
        _chk(t, torch.int32, n)
        if tuple(t.shape) != (B, S) or not t.is_contiguous():
            raise RuntimeError(f"fsb200: {n} must be contiguous int32 [batch, seq] = [{B}, {S}], got {tuple(t.shape)}")


def _segment_bounds_arg(seg_start, seg_end, rel_bias, kv_bounds, causal):
    """The bounds of sdpa_segments_fwd / _bwd; the cross form (kv_bounds) takes no rel_bias and has no causal mask."""
    if kv_bounds is None:
        return seg_start, seg_end, None, None
    if rel_bias is not None:
        raise RuntimeError("fsb200: the cross-attention segment form (kv_bounds) takes no rel_bias")
    if causal:
        raise RuntimeError("fsb200: the cross-attention segment form (kv_bounds) has no causal mask: pass causal=False")
    return seg_start, seg_end, kv_bounds[0], kv_bounds[1]


def sdpa_segments_fwd(q, k, v, scale, seg_start, seg_end, out=None, drop=None, causal=True, rel_bias=None, kv_bounds=None):
    """sdpa_fwd over rows that pack several sequences: causal inside each segment, nothing across segments. q, k, v as in
    sdpa_fwd (seq_q == seq_kv); seg_start / seg_end from segment_bounds. Key / query tiles outside a tile's segments are
    skipped. head_dim 64, 96 or 128. drop: optional Dropout on the attention probabilities, as in sdpa_fwd (head_dim 64 or
    96 when p > 0).
    causal=False: bidirectional inside each segment (packed encoder rows: query q sees seg_start[q] <= k < seg_end[q]),
    head_dim 64 only.
    rel_bias: the T5 relative-position bias of sdpa_fwd (fp32 [H, 2 S - 1]) added inside either segment form, head_dim 64
    only.
    kv_bounds=(q_start, q_end): cross-attention from packed decoder rows to packed encoder rows (seq_q and seq_kv may
    differ, causal=False): seg_start / seg_end are then the query side's key ranges [B, Sq] and kv_bounds the key side's
    query ranges [B, Skv] (models/base.py cross_segment_bounds), head_dim 64 only. The forms are those of fsb_sdpa_fwd
    (include/fsb200.h). Returns (out [B, Sq, H, D], lse)."""
    bounds = _segment_bounds_arg(seg_start, seg_end, rel_bias, kv_bounds, causal)
    return _sdpa_fwd(q, k, v, scale, causal, None, rel_bias, drop, out, bounds)


def sdpa_segments_bwd(q, k, v, out, dout, lse, scale, seg_start, seg_end, dq, dk, dv, drop=None, causal=True,
                      rel_bias=None, drel_bias=None, kv_bounds=None):
    """Backward of sdpa_segments_fwd (the forward's seg_start / seg_end, drop, causal, rel_bias and kv_bounds); dq / dk / dv
    are written as in sdpa_bwd. drel_bias (with rel_bias): fp32 [H, 2 S - 1], accumulated into (+=) deterministically, as in
    sdpa_bwd."""
    bounds = _segment_bounds_arg(seg_start, seg_end, rel_bias, kv_bounds, causal)
    if drel_bias is not None and rel_bias is None:
        raise RuntimeError("fsb200: drel_bias needs rel_bias")
    _sdpa_bwd(q, k, v, out, dout, lse, scale, causal, dq, dk, dv, None, rel_bias, drel_bias, drop, bounds)
