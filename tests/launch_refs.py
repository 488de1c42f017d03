"""One fp64 reference and one elementwise bound per public `fsb200.ops` entry point the training step calls.

`CHECKERS[name](real, bound, *args, **kwargs)` snapshots what the call modifies in place or accumulates into, runs the
real call `real(*args, **kwargs)`, recomputes the result in fp64 with plain torch on the operands' device (in row or batch
chunks sized so that all fp64 temporaries of one chunk together stay within about 2 GB) and checks every output element against a bound derived from the
kernel's rounding steps. It returns what `real` returned. `bound` (a `Bound`) raises on the first element out of bound and
keeps the worst err / bound ratio seen. The `verify_*` functions are the reference-and-bound halves: they take the inputs,
the values the kernel produced and the snapshots, and need no GPU (tests/test_launch_refs_cpu.py runs them on the CPU).

Notation in the docstrings: u16 = 2^-8 is the unit roundoff of bf16 (8 significant bits), u32 = 2^-24 that of fp32,
ulp(r) the bf16 spacing at |r| (guards.bf16_ulp); a value rounded to bf16 once is within 1/2 ulp of what was rounded, and
the bounds allow a whole ulp, as guards.assert_ulp_close does. A sum of n fp32 terms in any order is within
(n - 1) u32 sum|terms| of the exact sum; where a kernel reduces in a tree, test_layer_ops_gpu's ACC_REL = 2e-6 of
sum|terms| is used (`_sum_close` there). A K-deep fp32 dot product is bounded by the bf16-ulp + K 2^-23 |A||B| form of
test_fp8_gpu / test_int8_gpu.
"""
import math
from typing import NamedTuple

import numpy as np
import torch

import fp8_ref
import int4_ref
import int8_ref
import philox_ref
from guards import bf16_ulp, bits

U16 = 2.0 ** -8
U32 = 2.0 ** -24
ACC_REL = 2e-6          # fp32 tree-reduction noise relative to sum|terms| (test_layer_ops_gpu.ACC_REL)
ACT_FLOOR = 2.0 ** -18  # fp32 cancellation in an activation or its derivative (test_layer_ops_gpu.ACT_FLOOR)
GELU_SLOPE = 1.13       # max |d gelu / dx| over the reals (1.1289 at x = 1.5 for tanh- and erf-GeLU)
CHUNK_BYTES = 2 << 30   # fp64 working set of one chunk: all of its row- or batch-sized temporaries together
BF16, F32 = torch.bfloat16, torch.float32
ACT_SILU, ACT_GELU_TANH, ACT_GELU_ERF, ACT_TANH = 0, 1, 2, 3
EPI_NONE, EPI_GELU_TANH, EPI_GELU_ERF = 0, 1, 2
GEMM_NT, GEMM_NN, GEMM_TN = 0, 1, 2


class Bound:
    """Elementwise |got - ref| <= tol checks; remembers the largest err / tol ratio (0 when every err is 0)."""

    def __init__(self, what=""):
        self.what, self.worst = what, 0.0

    def close(self, name, got, ref, tol):
        ref = ref.double()
        err = (got.double() - ref).abs()
        tol = torch.as_tensor(tol, dtype=torch.float64, device=ref.device).expand_as(ref)
        bad = ~(err <= tol)
        if bad.any():
            i = int(bad.reshape(-1).nonzero()[0])
            raise AssertionError(
                f"{self.what} {name}: {int(bad.sum())}/{bad.numel()} elements out of bound; first at flat index {i}: got "
                f"{got.reshape(-1)[i].item():.6g}, want {ref.reshape(-1)[i].item():.6g} +- {tol.reshape(-1)[i].item():.3g}")
        if err.numel():
            r = (err / tol.clamp_min(1e-300)).max().item()
            self.worst = max(self.worst, r)

    def exact(self, name, got, want):
        if got.shape != want.shape or got.dtype != want.dtype or not torch.equal(bits(got), bits(want)):
            diff = (bits(got) != bits(want)) if got.shape == want.shape and got.dtype == want.dtype else None
            n = int(diff.sum()) if diff is not None else "shape/dtype"
            raise AssertionError(f"{self.what} {name}: {n} elements differ from the exact copy")

    def equal(self, name, got, want):
        if not torch.equal(got, want):
            raise AssertionError(f"{self.what} {name}: got {got.tolist() if got.numel() < 8 else '...'}, want "
                                 f"{want.tolist() if want.numel() < 8 else '...'}")


def _chunks(n, bytes_per_item):
    step = max(1, int(CHUNK_BYTES // max(1, bytes_per_item)))
    for s in range(0, n, step):
        yield slice(s, min(n, s + step))


def _ulp_tol(ref, dtype):
    """The storage rounding of a value computed in fp32: 1 bf16 ulp, or 2 u32 relative for an fp32 result."""
    return bf16_ulp(ref) if dtype == BF16 else 2 * U32 * ref.abs()


# ----------------------------------------------------------------------------------------------------------- dropout
class DropSpec(NamedTuple):
    """What a dropout mask is a function of (include/fsb200.h): the rate, the model's seed and the stream number
    s = *stream_base + site."""
    p: float
    seed: int
    stream: int


def drop_spec(drop):
    """The DropSpec of an ops.Dropout: its base is read from the device."""
    return None if drop is None else DropSpec(drop.p, drop.seed, int(drop.base.item()) + drop.site)


def keep_scale(p):
    """1 / (1 - p) as the kernels form it: fp32 p, fp32 subtraction and IEEE division (philox.cuh make_drop_args)."""
    one = torch.tensor(1.0, dtype=F32)
    return float(one / (one - torch.tensor(p, dtype=F32)))


def hidden_mult(d, rows, cols, device):
    """Z / (1 - p) of the hidden layout for the rows in range `rows`: fp64 [len(rows), cols] (0 where dropped)."""
    keep = philox_ref.hidden_keep_t(d.seed, d.stream, rows, cols, d.p, device)
    return keep.double() * keep_scale(d.p)


def attn_mult(d, batches, nheads, seq_q, seq_kv, device):
    """Z / (1 - p) of the attention layout for the batch rows in range `batches`: fp64 [nb, nheads, seq_q, seq_kv]."""
    keep = philox_ref.attn_keep_t(d.seed, d.stream, batches, nheads, seq_q, seq_kv, d.p, device)
    return keep.double() * keep_scale(d.p)


def _range(sl):
    return range(sl.start, sl.stop)


def verify_dropout(bound, x, d, out):
    """out = bf16(fp32(x) * fp32(1 / (1 - p))) where the hidden mask keeps, +0 where it drops: one fp32 product rounded
    once, bit for bit."""
    rows, cols = x.shape
    ks = torch.tensor(keep_scale(d.p), dtype=F32)
    for rs in _chunks(rows, cols * 8 * 6):
        keep = philox_ref.hidden_keep_t(d.seed, d.stream, _range(rs), cols, d.p, x.device)
        want = torch.where(keep, x[rs].float() * ks.to(x.device), torch.zeros((), dtype=F32, device=x.device)).to(BF16)
        bound.exact("x * Z / (1 - p)", out[rs], want)


def check_dropout(real, bound, x, drop, out=None):
    x0 = x.clone() if out is not None else x        # out may alias x
    d = drop_spec(drop)
    ret = real(x, drop, out=out)
    verify_dropout(bound, x0, d, ret)
    return ret


def verify_dropout_advance(bound, old, n, saved, counter):
    """saved = the old counter and counter = old + n, exactly."""
    bound.equal("saved stream base", saved.reshape(-1).cpu(), torch.tensor([old]))
    bound.equal("advanced counter", counter.reshape(-1).cpu(), torch.tensor([old + n]))


def check_dropout_advance(real, bound, counter, n):
    old = int(counter.item())
    saved = real(counter, n)
    verify_dropout_advance(bound, old, int(n), saved, counter)
    return saved


# ------------------------------------------------------------------------------------------------------- activations
def act64(act, x):
    if act == ACT_SILU:
        return x * torch.sigmoid(x)
    if act == ACT_GELU_TANH:
        return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))
    if act == ACT_GELU_ERF:
        return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))
    if act == ACT_TANH:
        return torch.tanh(x)
    raise ValueError(f"activation {act}")


def dact64(act, x):
    if act == ACT_SILU:
        s = torch.sigmoid(x)
        return s * (1.0 + x * (1.0 - s))
    if act == ACT_GELU_TANH:
        c = math.sqrt(2.0 / math.pi)
        t = torch.tanh(c * (x + 0.044715 * x ** 3))
        return 0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * c * (1.0 + 3 * 0.044715 * x * x)
    if act == ACT_GELU_ERF:
        return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)
    if act == ACT_TANH:
        return 1.0 - torch.tanh(x) ** 2
    raise ValueError(f"activation {act}")


_EPI_ACT = {EPI_GELU_TANH: ACT_GELU_TANH, EPI_GELU_ERF: ACT_GELU_ERF}


# ------------------------------------------------------------------------------------------------------------- GEMM
def _gemm_operands(layout, a, b):
    """(A [M, K], B [K, N]) views of the call's operands."""
    if layout == GEMM_NT:
        return a, b.t()
    if layout == GEMM_NN:
        return a, b
    return a.t(), b


def verify_gemm(bound, layout, a, b, out, bias=None, epilogue=EPI_NONE, old=None, aux=None, aux_plain=None):
    """D = act(A B + bias) (+ D_old), fp32 accumulation, one rounding to D's dtype; aux = bf16(A B + bias).

    Bound per element: K 2^-23 (|A||B|)_mn for the fp32 accumulation (times GELU_SLOPE through a GeLU epilogue), 2 u32
    |bias| for the bias add, ACT_FLOOR (1 + |x|) for the fp32 GeLU (erf by Abramowitz-Stegun 7.1.26, 1.5e-7 absolute), 2 u32
    |D_old| for the accumulate add, and the final rounding (1 ulp in bf16, 2 u32 relative in fp32).
    aux: when `aux_plain` is given (the same GEMM with the same bias and no epilogue, stored bf16: the same fp32 value rounded
    the same way) aux must equal it bit for bit; otherwise aux is held to the bound of a bf16 D without activation."""
    A, B = _gemm_operands(layout, a, b)
    M, K = A.shape
    N = B.shape[1]
    act = _EPI_ACT.get(epilogue)
    for cs in _chunks(N, 8 * 2 * K):                     # B's columns and |B| (K deep)
        B64 = B[:, cs].double()
        Babs = B64.abs()
        n = cs.stop - cs.start
        bias64 = None if bias is None else bias[cs].double().view(1, n)
        for rs in _chunks(M, 8 * (2 * K + 14 * n)):      # A's rows and |A| (K wide), 14 temporaries as wide as the block
            A64 = A[rs].double()
            pre = A64 @ B64
            mag = K * 2.0 ** -23 * (A64.abs() @ Babs)
            del A64
            if bias64 is not None:
                pre = pre + bias64
                mag = mag + 2 * U32 * bias64.abs()
            if aux is not None:
                if aux_plain is not None:
                    bound.exact("aux (pre-activation) against the plain GEMM", aux[rs, cs], aux_plain[rs, cs])
                else:
                    bound.close("aux", aux[rs, cs], pre, mag + bf16_ulp(pre))
            if act is not None:
                ref = act64(act, pre)
                tol = GELU_SLOPE * mag + ACT_FLOOR * (1.0 + pre.abs())
            else:
                ref, tol = pre, mag
            if old is not None:
                o = old[rs, cs].double()
                ref = ref + o
                tol = tol + 2 * U32 * o.abs()
            bound.close("D", out[rs, cs], ref, tol + _ulp_tol(ref, out.dtype))
            del pre, mag, ref, tol
        del B64, Babs


def check_gemm(real, bound, layout, a, b, out=None, out_dtype=BF16, bias=None, epilogue=EPI_NONE, accumulate=False,
               aux=None):
    old = out.clone() if accumulate else None
    ret = real(layout, a, b, out=out, out_dtype=out_dtype, bias=bias, epilogue=epilogue, accumulate=accumulate, aux=aux)
    aux_plain = None
    # a TN call without bias, aux or epilogue may split K; with a bias it runs the same unsplit plan as the epilogue call
    if aux is not None and not (layout == GEMM_TN and bias is None):
        aux_plain = real(layout, a, b, out_dtype=BF16, bias=bias)
    verify_gemm(bound, layout, a, b, ret, bias, epilogue, old, aux, aux_plain)
    return ret


# ------------------------------------------------------------------------------------------------------------ norms
def _sum_tol(abs_sum, ref, dtype):
    """test_layer_ops_gpu._sum_close: ACC_REL sum|terms| (+ 1 ulp when the sum is stored in bf16)."""
    tol = ACC_REL * abs_sum + 1e-30
    return tol + bf16_ulp(ref) if dtype == BF16 else tol


def verify_norm_fwd(bound, layer, x, residual, w, beta, eps, y, stats, xsum, drop=None):
    """x_sum = bf16(x + residual): the fp32 sum of two bf16 values rounded once, compared bit for bit. With dropout (a
    DropSpec) x_sum = bf16(t + residual), t = fp32(x * fp32(1 / (1 - p))) where the hidden mask keeps and 0 where it drops
    (norm.cu's apply_keep8 before the add), bit for bit.
    Statistics against fp64 on x_sum: rstd within 1e-5 relative (rsqrtf, 2 ulp, and a per-row fp32 sum of at most
    8 VPT + log2 TPR <= 72 levels: (72 u32 / 2 + 2^-22) < 1e-5); LayerNorm's mean within 72 u32 mean|x| + 1e-30.
    RMSNorm: y = bf16(bf16(x rstd) * scale) with the kernel's rstd, bit for bit (norms.py casts before the scale multiply).
    LayerNorm: y = bf16((x - mean) rstd gamma + beta) with the kernel's statistics: four fp32 roundings, 2^-22
    (|xhat gamma| + |beta|), and 1 ulp."""
    rows, cols = x.shape
    xs = xsum
    for rs in _chunks(rows, cols * 8 * 10):
        if residual is not None:
            xf = x[rs].float()
            if drop is not None:
                keep = philox_ref.hidden_keep_t(drop.seed, drop.stream, _range(rs), cols, drop.p, x.device)
                ks = torch.tensor(keep_scale(drop.p), dtype=F32, device=x.device)
                xf = torch.where(keep, xf * ks, torch.zeros((), dtype=F32, device=x.device))
            bound.exact("x + residual", xsum[rs], (xf + residual[rs].float()).to(BF16))
        xd = xs[rs].double()
        if layer:
            mean_g, rstd_g = stats[rs, 0].double(), stats[rs, 1].double()
            mean = xd.mean(1)
            bound.close("mean", mean_g, mean, 72 * U32 * xd.abs().mean(1) + 1e-30)
            rstd = 1.0 / torch.sqrt((xd - mean[:, None]).pow(2).mean(1) + eps)
            bound.close("rstd", rstd_g, rstd, 1e-5 * rstd)
            xh = (xd - mean_g[:, None]) * rstd_g[:, None]
            core = xh * w.double()
            ref = core + beta.double()
            bound.close("y", y[rs], ref, 2.0 ** -22 * (core.abs() + beta.double().abs()) + bf16_ulp(ref))
        else:
            rstd_g = stats[rs].double()
            rstd = 1.0 / torch.sqrt(xd.pow(2).mean(1) + eps)
            bound.close("rstd", rstd_g, rstd, 1e-5 * rstd)
            want = (xs[rs].float() * stats[rs].float()[:, None]).to(BF16) * w
            bound.exact("y = scale * bf16(x rstd)", y[rs], want)


def check_rmsnorm_fwd(real, bound, x, scale, eps, residual=None, drop=None):
    d = drop_spec(drop)
    y, rstd, xs = ret = real(x, scale, eps, residual=residual, drop=drop)
    verify_norm_fwd(bound, False, x, residual, scale, None, eps, y, rstd, xs, d)
    return ret


def check_layernorm_fwd(real, bound, x, gamma, beta, eps, residual=None, drop=None):
    d = drop_spec(drop)
    y, stats, xs = ret = real(x, gamma, beta, eps, residual=residual, drop=drop)
    verify_norm_fwd(bound, True, x, residual, gamma, beta, eps, y, stats, xs, d)
    return ret


def verify_norm_bwd(bound, layer, dy, x, w, stats, dres, dx, dw, dw_old, db=None, db_old=None, drop=None, dbranch=None):
    """With the forward's statistics (the call's own operands): xhat = (x - mean) rstd, g = dy w,
    dx = rstd (g - [mean(g)] - xhat mean(g xhat)) (+ dres), rounded once: 1 ulp plus test_layer_ops_gpu's floor
    1e-5 max_row |rstd (g - ...)| for the fp32 row sums inside the means.
    dw = sum_rows dy * xhat (RMSNorm: dy * bf16(x rstd), the rounded value the forward multiplied), db = sum_rows dy, each
    (+ the old value when accumulating): ACC_REL of sum|terms| (+ 1 ulp in bf16).
    With dropout (a DropSpec): dbranch = bf16(dx32 Z / (1 - p)) from the kernel's unrounded fp32 dx (norm.cu applies the
    mask after dx is stored): M = Z / (1 - p) times dx's bound, plus 1 ulp of the product."""
    rows, cols = x.shape
    wd = w.double()
    gw = torch.zeros(cols, dtype=torch.float64, device=x.device)
    aw = torch.zeros_like(gw)
    gb, ab = torch.zeros_like(gw), torch.zeros_like(gw)
    for rs in _chunks(rows, cols * 8 * 16):
        xd, dyd = x[rs].double(), dy[rs].double()
        if layer:
            mean, rstd = stats[rs, 0].double()[:, None], stats[rs, 1].double()[:, None]
            xh = (xd - mean) * rstd
            xw = xh
        else:
            rstd = stats[rs].double()[:, None]
            xh = xd * rstd
            xw = (x[rs].float() * stats[rs].float()[:, None]).to(BF16).double()
        g = dyd * wd
        core = g - xh * (g * xh).mean(1, keepdim=True)
        if layer:
            core = core - g.mean(1, keepdim=True)
        core = rstd * core
        ref = core + (dres[rs].double() if dres is not None else 0.0)
        tol = 1e-5 * core.abs().amax(1, keepdim=True) + bf16_ulp(ref)
        bound.close("dx", dx[rs], ref, tol)
        if drop is not None:
            m = hidden_mult(drop, _range(rs), cols, x.device)
            bound.close("dbranch", dbranch[rs], m * ref, m * tol + bf16_ulp(m * ref))
        t = dyd * xw
        gw += t.sum(0); aw += t.abs().sum(0)
        if layer:
            gb += dyd.sum(0); ab += dyd.abs().sum(0)
    for name, got, s, a, old in (("dweight", dw, gw, aw, dw_old), ("dbias", db, gb, ab, db_old)):
        if got is None:
            continue
        if old is not None:
            s, a = s + old.double(), a + old.double().abs()
        bound.close(name, got, s, _sum_tol(a, s, got.dtype))


def check_rmsnorm_bwd(real, bound, dy, x, scale, rstd, dscale_out, accumulate=False, dres=None):
    old = dscale_out.clone() if accumulate else None
    dx = real(dy, x, scale, rstd, dscale_out, accumulate=accumulate, dres=dres)
    verify_norm_bwd(bound, False, dy, x, scale, rstd, dres, dx, dscale_out, old)
    return dx


def check_rmsnorm_bwd_dropout(real, bound, dy, x, scale, rstd, dscale_out, drop, accumulate=False, dres=None):
    old = dscale_out.clone() if accumulate else None
    d = drop_spec(drop)
    dx, dbr = ret = real(dy, x, scale, rstd, dscale_out, drop, accumulate=accumulate, dres=dres)
    verify_norm_bwd(bound, False, dy, x, scale, rstd, dres, dx, dscale_out, old, drop=d, dbranch=dbr)
    return ret


def check_layernorm_bwd_dropout(real, bound, dy, x, gamma, stats, dgamma_out, dbeta_out, drop, accumulate=False,
                                dres=None):
    og = dgamma_out.clone() if accumulate else None
    ob = dbeta_out.clone() if accumulate else None
    d = drop_spec(drop)
    dx, dbr = ret = real(dy, x, gamma, stats, dgamma_out, dbeta_out, drop, accumulate=accumulate, dres=dres)
    verify_norm_bwd(bound, True, dy, x, gamma, stats, dres, dx, dgamma_out, og, dbeta_out, ob, drop=d, dbranch=dbr)
    return ret


def check_layernorm_bwd(real, bound, dy, x, gamma, stats, dgamma_out, dbeta_out, accumulate=False, dres=None):
    og = dgamma_out.clone() if accumulate else None
    ob = dbeta_out.clone() if accumulate else None
    dx = real(dy, x, gamma, stats, dgamma_out, dbeta_out, accumulate=accumulate, dres=dres)
    verify_norm_bwd(bound, True, dy, x, gamma, stats, dres, dx, dgamma_out, og, dbeta_out, ob)
    return dx


# ------------------------------------------------------------------------------------------------------------- rope
def rope_view(x, rows, nheads, head_dim, row_stride, head_stride, offset):
    return torch.as_strided(x, (rows, nheads, head_dim), (row_stride, head_stride, 1), x.storage_offset() + offset)


def verify_rope(bound, before, after, cos, sin, positions, nheads, head_dim, row_stride, head_stride, backward, offset):
    """Rotate-half rotation of the selected heads on the fp32 tables (backward: the transposed rotation), in fp64: 1 ulp
    plus test_layer_ops_gpu's 1e-6 max|ref| for the fp32 cancellation in x1 cos - x2 sin. Every element outside the
    rotated heads is unchanged, bit for bit."""
    rows = positions.numel()
    sel = lambda t: rope_view(t, rows, nheads, head_dim, row_stride, head_stride, offset)   # noqa: E731
    mask = torch.zeros(before.shape, dtype=torch.bool, device=before.device)
    sel(mask).fill_(True)
    bound.exact("elements outside the rotated heads", after[~mask], before[~mask])
    h = head_dim // 2
    pos = positions.view(-1)
    for rs in _chunks(rows, nheads * head_dim * 8 * 12):
        v = sel(before)[rs].double()
        c = torch.cat([cos[pos[rs]], cos[pos[rs]]], -1).double()[:, None, :]
        s = torch.cat([sin[pos[rs]], sin[pos[rs]]], -1).double()[:, None, :]
        rot = torch.cat([v[..., h:], -v[..., :h]], -1) if backward else torch.cat([-v[..., h:], v[..., :h]], -1)
        ref = v * c + rot * s
        bound.close("rotated heads", sel(after)[rs], ref, bf16_ulp(ref) + 1e-6 * ref.abs().max())


def check_rope_inplace(real, bound, x, cos, sin, positions, nheads, head_dim, row_stride, head_stride, backward=False,
                       offset=0):
    before = x.clone()
    ret = real(x, cos, sin, positions, nheads, head_dim, row_stride, head_stride, backward=backward, offset=offset)
    verify_rope(bound, before, x, cos, sin, positions, nheads, head_dim, row_stride, head_stride, bool(backward), offset)
    return ret


# ------------------------------------------------------------------------------------------------------ activations
def verify_glu_fwd(bound, act, gate, up, out, drop=None):
    """out = act(gate) * up rounded once: 1 ulp plus ACT_FLOOR |up|. With dropout (a DropSpec) the fp32 product is
    multiplied by M = Z / (1 - p) of the hidden layout before the rounding: M ACT_FLOOR |up| plus 2 u32 |ref| for the extra
    fp32 product."""
    cols = gate.shape[1]
    for rs in _chunks(gate.shape[0], cols * 8 * 12):
        g, u = gate[rs].double(), up[rs].double()
        ref = act64(act, g) * u
        tol = ACT_FLOOR * u.abs()
        if drop is not None:
            m = hidden_mult(drop, _range(rs), cols, gate.device)
            ref, tol = ref * m, tol * m + 2 * U32 * (ref * m).abs()
        bound.close("out", out[rs], ref, bf16_ulp(ref) + tol)


def check_glu_fwd(real, bound, act, gate, up, drop=None):
    d = drop_spec(drop)
    out = real(act, gate, up, drop=drop)
    verify_glu_fwd(bound, act, gate, up, out, d)
    return out


def verify_glu_bwd(bound, act, dout, gate, up, dgate, dup, drop=None):
    """dgate = dout * up * act'(gate), dup = dout * act(gate), each rounded once: 1 ulp plus ACT_FLOOR |dout up| and
    ACT_FLOOR |dout|. With dropout (a DropSpec) dout is first multiplied by M = Z / (1 - p) in fp32 (elementwise.cu):
    the same bounds on M dout, plus 2 u32 |ref| for that product."""
    cols = gate.shape[1]
    for rs in _chunks(gate.shape[0], cols * 8 * 18):
        d, g, u = dout[rs].double(), gate[rs].double(), up[rs].double()
        extra = 0.0
        if drop is not None:
            d = d * hidden_mult(drop, _range(rs), cols, gate.device)
            extra = 2 * U32
        rg = d * u * dact64(act, g)
        ru = d * act64(act, g)
        bound.close("dgate", dgate[rs], rg, bf16_ulp(rg) + ACT_FLOOR * (d * u).abs() + extra * rg.abs())
        bound.close("dup", dup[rs], ru, bf16_ulp(ru) + ACT_FLOOR * d.abs() + extra * ru.abs())


def check_glu_bwd(real, bound, act, dout, gate, up, dgate, dup, drop=None):
    d0, g0, u0 = dout.clone(), gate.clone(), up.clone()     # dgate / dup may overwrite them
    d = drop_spec(drop)
    ret = real(act, dout, gate, up, dgate, dup, drop=drop)
    verify_glu_bwd(bound, act, d0, g0, u0, dgate, dup, d)
    return ret


def verify_act_fwd(bound, act, x, y):
    """y = act(x) rounded once: 1 ulp plus ACT_FLOOR."""
    xf, yf = x.reshape(-1), y.reshape(-1)
    for rs in _chunks(xf.numel(), 8 * 10):
        ref = act64(act, xf[rs].double())
        bound.close("y", yf[rs], ref, bf16_ulp(ref) + ACT_FLOOR)


def check_act_fwd(real, bound, act, x):
    y = real(act, x)
    verify_act_fwd(bound, act, x, y)
    return y


def verify_act_bwd(bound, act, dy, x, dx, dbias=None, dbias_old=None):
    """dx = dy * act'(x) rounded once: 1 ulp plus ACT_FLOOR |dy|. dbias (+)= sum_rows dx over the bf16 dx the kernel
    stored (elementwise.cu's act_bwd_colsum_kernel adds up what it wrote, as a separate colsum over dx would; dx itself is
    held to fp64 above): ACC_REL of sum|terms| (+ 1 ulp in bf16)."""
    x2, dy2, dx2 = (t.reshape(-1, x.shape[-1]) for t in (x, dy, dx))
    s = torch.zeros(x2.shape[1], dtype=torch.float64, device=x.device)
    a = torch.zeros_like(s)
    for rs in _chunks(x2.shape[0], x2.shape[1] * 8 * 12):
        d = dy2[rs].double()
        ref = d * dact64(act, x2[rs].double())
        bound.close("dx", dx2[rs], ref, bf16_ulp(ref) + ACT_FLOOR * d.abs())
        t = dx2[rs].double()
        s += t.sum(0); a += t.abs().sum(0)
    if dbias is not None:
        if dbias_old is not None:
            s, a = s + dbias_old.double(), a + dbias_old.double().abs()
        bound.close("dbias", dbias, s, _sum_tol(a, s, dbias.dtype))


def check_act_bwd(real, bound, act, dy, x):
    dx = real(act, dy, x)
    verify_act_bwd(bound, act, dy, x, dx)
    return dx


def check_act_bwd_bias(real, bound, act, dy, x, dbias, accumulate=False):
    old = dbias.clone() if accumulate else None
    dx = real(act, dy, x, dbias, accumulate=accumulate)
    verify_act_bwd(bound, act, dy, x, dx, dbias, old)
    return dx


def verify_colsum(bound, x, out, old=None):
    """out[c] (+)= sum_r x[r, c]: ACC_REL of sum|terms| (+ 1 ulp in bf16)."""
    s = torch.zeros(x.shape[1], dtype=torch.float64, device=x.device)
    a = torch.zeros_like(s)
    for rs in _chunks(x.shape[0], x.shape[1] * 8 * 3):
        t = x[rs].double()
        s += t.sum(0); a += t.abs().sum(0)
    if old is not None:
        s, a = s + old.double(), a + old.double().abs()
    bound.close("column sums", out, s, _sum_tol(a, s, out.dtype))


def check_colsum(real, bound, x, out, accumulate=False):
    old = out.clone() if accumulate else None
    ret = real(x, out, accumulate=accumulate)
    verify_colsum(bound, x, out, old)
    return ret


# ------------------------------------------------------------------------------------------------------ elementwise
def verify_add(bound, a, b, out):
    """out = bf16(a + b): one rounding of the fp32 sum, 1 ulp plus 2 u32 |a + b|."""
    af, bf, of = a.reshape(-1), b.reshape(-1), out.reshape(-1)
    for rs in _chunks(af.numel(), 8 * 10):
        ref = af[rs].double() + bf[rs].double()
        bound.close("a + b", of[rs], ref, bf16_ulp(ref) + 2 * U32 * ref.abs())


def check_add(real, bound, a, b, out=None):
    ret = real(a, b, out=out)
    verify_add(bound, a, b, ret)
    return ret


def verify_accumulate(bound, old, x16, scale, overwrite, acc):
    """acc = (0 if overwrite else acc_old) + scale * x16 in fp32: two roundings, 2 u32 (|acc_old| + |scale x| + |ref|)."""
    s = float(torch.tensor(scale, dtype=F32))
    af, xf, of = acc.reshape(-1), x16.reshape(-1), None if overwrite else old.reshape(-1)
    for rs in _chunks(af.numel(), 8 * 10):
        sx = s * xf[rs].double()
        base = 0.0 if overwrite else of[rs].double()
        ref = base + sx
        tol = 2 * U32 * ((base.abs() if not overwrite else 0.0) + sx.abs() + ref.abs())
        bound.close("acc", af[rs], ref, tol)


def check_accumulate(real, bound, acc32, x16, scale=1.0, overwrite=False):
    old = None if overwrite else acc32.clone()
    ret = real(acc32, x16, scale=scale, overwrite=overwrite)
    verify_accumulate(bound, old, x16, scale, overwrite, acc32)
    return ret


def verify_scale(bound, before, s, after):
    """x * s rounded once (a scalar of 1 leaves x unchanged): 1 ulp."""
    bf, af = before.reshape(-1), after.reshape(-1)
    for rs in _chunks(bf.numel(), 8 * 10):
        ref = bf[rs].double() * float(s)
        bound.close("x * s", af[rs], ref, bf16_ulp(ref))


def check_scale_inplace(real, bound, x16, scale_dev):
    before = x16.clone()
    ret = real(x16, scale_dev)
    verify_scale(bound, before, float(scale_dev.float().item()), x16)
    return ret


def verify_cast(bound, x32, out):
    """out = bf16(x32), round to nearest even: bit for bit what torch's cast gives."""
    bound.exact("bf16(x)", out, x32.to(BF16))


def check_cast_f32_to_bf16(real, bound, x32, out=None):
    ret = real(x32, out=out)
    verify_cast(bound, x32, ret)
    return ret


# -------------------------------------------------------------------------------------------------------- embedding
def verify_embedding_fwd(bound, ids, W, pos, P, token_type, T, seq_len, out):
    """out[t] = W[ids[t]] (+ P[pos[t] or t % seq_len] + T[token_type[t]]): a gather alone is a copy, bit for bit; with the
    added tables, the fp32 sum rounded once: 1 ulp plus 2 u32 sum|terms|."""
    rows = ids.numel()
    idx = ids.reshape(-1)
    if P is None and T is None:
        bound.exact("gathered rows", out, W[idx])
        return
    t = torch.arange(rows, device=ids.device)
    for rs in _chunks(rows, W.shape[1] * 8 * 10):
        ref = W[idx[rs]].double()
        mag = ref.abs()
        if P is not None:
            p = (pos.reshape(-1)[rs] if pos is not None else t[rs] % seq_len)
            ref = ref + P[p].double(); mag = mag + P[p].double().abs()
        if T is not None:
            ref = ref + T[token_type.reshape(-1)[rs]].double(); mag = mag + T[token_type.reshape(-1)[rs]].double().abs()
        bound.close("embedding sum", out[rs], ref, bf16_ulp(ref) + 2 * U32 * mag)


def check_embedding_fwd(real, bound, ids, W, pos=None, P=None, token_type=None, T=None, seq_len=1):
    out = real(ids, W, pos=pos, P=P, token_type=token_type, T=T, seq_len=seq_len)
    verify_embedding_fwd(bound, ids, W, pos, P, token_type, T, seq_len, out)
    return out


def verify_embedding_bwd(bound, ids, dout, before, after, idx_mod=0):
    """dW[ids[t]] += dout[t]. Rows no token maps to are unchanged, bit for bit. With ids (sorted form): every row's terms
    summed in fp32 and added onto the old row with one rounding: ACC_REL (|old| + sum|terms|) + 1 ulp. ids = None (row
    t % idx_mod, bf16 atomics): each of the c adds onto a row rounds to bf16, c u16 (|old| + sum|terms|) + 1 ulp."""
    rows, cols = dout.shape
    idx = ids.reshape(-1) if ids is not None else torch.arange(rows, device=dout.device) % idx_mod
    touched = torch.zeros(before.shape[0], dtype=torch.bool, device=before.device)
    touched[idx] = True
    bound.exact("rows without tokens", after[~touched], before[~touched])
    uniq, inv = torch.unique(idx, return_inverse=True)
    counts = torch.bincount(inv, minlength=uniq.numel()).double()[:, None]
    for us in _chunks(uniq.numel(), cols * 8 * 10):
        sel = (inv >= us.start) & (inv < us.stop)
        k = inv[sel] - us.start
        n = us.stop - us.start
        s = torch.zeros((n, cols), dtype=torch.float64, device=dout.device)
        a = torch.zeros_like(s)
        d = dout[sel].double()
        s.index_add_(0, k, d); a.index_add_(0, k, d.abs())
        old = before[uniq[us]].double()
        ref = old + s
        mag = old.abs() + a
        rel = ACC_REL if ids is not None else counts[us] * U16
        bound.close("accumulated rows", after[uniq[us]], ref, rel * mag + bf16_ulp(ref))


def check_embedding_bwd(real, bound, ids, dout, dW, idx_mod=0):
    before = dW.clone()
    ret = real(ids, dout, dW, idx_mod=idx_mod)
    verify_embedding_bwd(bound, ids, dout, before, dW, idx_mod)
    return ret


# --------------------------------------------------------------------------------------------------------- the loss
def xent_valid(labels, rows, seq_len, shift, ignore_index):
    """(valid [rows] bool, label index [rows]) of fsb_softmax_xent_fwd_bwd's causal shift."""
    t = torch.arange(rows, device=labels.device)
    lab = labels.reshape(-1)
    in_range = (t % seq_len) + shift < seq_len
    tgt = torch.where(in_range, lab[(t + shift).clamp_max(lab.numel() - 1)], torch.full_like(t, ignore_index))
    valid = in_range & (tgt != ignore_index)
    return valid, torch.where(valid, tgt, torch.zeros_like(tgt))


def verify_softmax_xent(bound, logits, labels, seq_len, shift, ignore_index, grad_scale, loss, dl, n_valid):
    """n_valid exact. Row loss lse - x[label] of a valid row: the fp32 sum of V exponentials (ex2.approx, 2^-22 relative
    each) is within (V u32 + 2^-22) relative, so the log is within that absolutely, plus 2 u32 |lse| for the log and the
    subtraction: e_r = V u32 + 2^-21 + 2 u32 (|lse| + |x[label]|). loss = sum / n_valid, n_valid terms of an fp32 sum:
    mean(e_r) + n_valid u32 mean|row loss| + u32 |loss|. dlogits = (softmax - onehot) grad_scale / n_valid rounded once:
    1 ulp plus softmax * e_r * grad_scale / n_valid; ignored rows get exact zeros."""
    rows, V = logits.shape
    valid, tgt = xent_valid(labels, rows, seq_len, shift, ignore_index)
    n = int(valid.sum())
    bound.equal("n_valid", n_valid.reshape(()).to(torch.int64).cpu(), torch.tensor(n))
    gs = float(torch.tensor(grad_scale, dtype=F32)) / max(n, 1)
    tot = torch.zeros((), dtype=torch.float64, device=logits.device)
    err = torch.zeros_like(tot)
    absl = torch.zeros_like(tot)
    for rs in _chunks(rows, V * 8 * 16):
        x = logits[rs].double()
        lse = torch.logsumexp(x, 1)
        xl = x.gather(1, tgt[rs, None])[:, 0]
        v = valid[rs]
        rl = torch.where(v, lse - xl, torch.zeros_like(lse))
        e_r = V * U32 + 2.0 ** -21 + 2 * U32 * (lse.abs() + xl.abs())
        tot += rl.sum(); absl += rl.abs().sum(); err += torch.where(v, e_r, torch.zeros_like(e_r)).sum()
        if dl is not None:
            p = torch.exp(x - lse[:, None])
            ref = p.clone()
            ref.scatter_add_(1, tgt[rs, None], -torch.ones_like(lse)[:, None])
            ref = torch.where(v[:, None], ref * gs, torch.zeros_like(ref))
            tol = bf16_ulp(ref) + torch.where(v[:, None], p * e_r[:, None] * gs, torch.zeros_like(ref))
            bound.close("dlogits", dl[rs], ref, tol)
        del x
    m = max(n, 1)
    ref_loss = tot / m
    tol = err / m + n * U32 * absl / m + U32 * ref_loss.abs()
    bound.close("loss", loss.reshape(()), ref_loss, tol)


def check_softmax_xent(real, bound, logits, labels, seq_len, shift=1, ignore_index=-100, grad_scale=1.0, dlogits="inplace"):
    x = logits.clone() if isinstance(dlogits, str) and dlogits == "inplace" else logits
    ret = real(logits, labels, seq_len, shift=shift, ignore_index=ignore_index, grad_scale=grad_scale, dlogits=dlogits)
    loss, dl, nv = ret
    verify_softmax_xent(bound, x, labels, seq_len, shift, ignore_index, grad_scale, loss, dl, nv)
    return ret


# ---------------------------------------------------------------------------------------------------- the optimizer
def _f32(v):
    return float(torch.tensor(float(v), dtype=F32))


def verify_adamw(bound, master0, m0, v0, grad, master, m, v, param16, lr, beta1, beta2, eps, wd, step, grad_scale=None,
                 hyper=None):
    """torch.optim.AdamW's order on fp32 scalars as the C side receives them: g = grad * coef; p *= 1 - lr wd;
    m = b1 m + (1 - b1) g; v = b2 v + (1 - b2) g^2; p -= (lr / bc1) m / (sqrt(v) / sqrt(bc2) + eps), bc1 = 1 - b1^t and
    sqrt(bc2) = sqrt(1 - b2^t) formed in double and rounded to fp32 (or read from `hyper`).
    m: three fp32 roundings, 2^-22 (b1 |m0| + (1 - b1) |g|) + 2 u32 |m|; v likewise with g^2. The step u = m / denom has
    relative error under 2^-19 (m and v's, sqrt, the division); master: 2^-22 |p0| + lr / bc1 |u| 2^-19 + 2 u32 |p|.
    param16 = bf16(master) of the kernel's own new master, bit for bit."""
    if hyper is not None:
        lr_, bc1, bc2s = (float(x) for x in hyper.double().cpu())
    else:
        lr_ = _f32(lr)
        b1d, b2d = _f32(beta1), _f32(beta2)
        bc1 = _f32(1.0 - b1d ** step)
        bc2s = _f32(math.sqrt(1.0 - b2d ** step))
    b1, b2, e, w = _f32(beta1), _f32(beta2), _f32(eps), _f32(wd)
    coef = 1.0 if grad_scale is None else float(grad_scale.double().reshape(-1)[0])
    step_sz = lr_ / bc1
    decay = 1.0 - lr_ * w
    n = master.numel()
    for rs in _chunks(n, 8 * 24):
        g = grad.reshape(-1)[rs].double() * coef
        mo, vo, po = m0.reshape(-1)[rs].double(), v0.reshape(-1)[rs].double(), master0.reshape(-1)[rs].double()
        mr = b1 * mo + (1 - b1) * g
        vr = b2 * vo + (1 - b2) * g * g
        u = mr / (torch.sqrt(vr) / bc2s + e)
        pr = po * decay - step_sz * u
        bound.close("exp_avg", m.reshape(-1)[rs], mr, 2.0 ** -22 * (b1 * mo.abs() + (1 - b1) * g.abs()) + 2 * U32 * mr.abs())
        bound.close("exp_avg_sq", v.reshape(-1)[rs], vr, 2.0 ** -22 * (b2 * vo + (1 - b2) * g * g) + 2 * U32 * vr)
        bound.close("master", master.reshape(-1)[rs], pr,
                    2.0 ** -22 * po.abs() + step_sz * u.abs() * 2.0 ** -19 + 2 * U32 * pr.abs() + 1e-45)
        if param16 is not None:
            bound.exact("param16 = bf16(master)", param16.reshape(-1)[rs], master.reshape(-1)[rs].to(BF16))


def check_adamw_flat(real, bound, master, m, v, grad, param16, lr, beta1, beta2, eps, weight_decay, step, grad_scale=None,
                     hyper=None):
    p0, m0, v0 = master.clone(), m.clone(), v.clone()
    g0 = grad.clone()                    # the engine never aliases grad with the state, but a check must not assume it
    ret = real(master, m, v, grad, param16, lr, beta1, beta2, eps, weight_decay, step, grad_scale=grad_scale, hyper=hyper)
    verify_adamw(bound, p0, m0, v0, g0, master, m, v, param16, lr, beta1, beta2, eps, weight_decay, step, grad_scale,
                 hyper)
    return ret


def verify_sumsq(bound, x, out, old=None):
    """out (+)= sum x^2 in fp32 (squares of bf16 or fp32 values): ACC_REL of the sum (all terms non-negative)."""
    xf = x.reshape(-1)
    s = torch.zeros((), dtype=torch.float64, device=x.device)
    for rs in _chunks(xf.numel(), 8 * 3):
        s += xf[rs].double().pow(2).sum()
    if old is not None:
        s = s + old.double().reshape(())
    bound.close("sum of squares", out.reshape(()), s, ACC_REL * s + 1e-45)


def check_sumsq(real, bound, x, out, accumulate=False):
    old = out.clone() if accumulate else None
    ret = real(x, out, accumulate=accumulate)
    verify_sumsq(bound, x, out, old)
    return ret


def verify_clip_coef(bound, sumsq, max_norm, coef, norm=None):
    """torch.nn.utils.clip_grad_norm_: norm = sqrt(sumsq), coef = min(1, max_norm / (norm + 1e-6)), fp32: 2^-22
    relative each."""
    s = sumsq.double().reshape(())
    nr = torch.sqrt(s)
    cr = torch.clamp(_f32(max_norm) / (nr + 1e-6), max=1.0)
    bound.close("clip coefficient", coef.reshape(()), cr, 2.0 ** -22 * cr)
    if norm is not None:
        bound.close("gradient norm", norm.reshape(()), nr, 2.0 ** -22 * nr)


def check_clip_coef(real, bound, sumsq_t, max_norm, coef_out, norm_out=None):
    ret = real(sumsq_t, max_norm, coef_out, norm_out=norm_out)
    verify_clip_coef(bound, sumsq_t, max_norm, coef_out, norm_out)
    return ret


# -------------------------------------------------------------------------------------------------------- attention
def _bhsd(t):
    return t.permute(0, 2, 1, 3)


def _scores(q, k, scale, causal, kv_mask, rel_bias, bs):
    """fp64 scores [nb, H, Sq, Skv] in natural-log units (masked: -inf) and the fp32 score error e_s of each: the D-deep
    fp32 dot product, D 2^-23 scale (|q||k|), plus 2^-22 (|scale q.k| + |bias|) for the scale, the bias fma and the
    conversion to the log2 domain."""
    qd, kd = _bhsd(q[bs]).double(), _bhsd(k[bs]).double()
    D, Sq, Skv = q.shape[3], q.shape[1], k.shape[1]
    s = scale * (qd @ kd.transpose(-1, -2))
    e = D * 2.0 ** -23 * scale * (qd.abs() @ kd.abs().transpose(-1, -2)) + 2.0 ** -22 * s.abs()
    keep = torch.ones((1, 1, Sq, Skv), dtype=torch.bool, device=q.device)
    if rel_bias is not None:
        qi = torch.arange(Sq, device=q.device)[:, None]
        ki = torch.arange(Skv, device=q.device)[None, :]
        bias = rel_bias.double()[:, ki - qi + Sq - 1]           # [H, Sq, Skv]
        s = s + bias
        e = e + 2.0 ** -22 * bias.abs()
    if causal:
        keep = keep & torch.ones((Sq, Skv), dtype=torch.bool, device=q.device).tril()
    if kv_mask is not None:
        keep = keep & (kv_mask[bs] != 0)[:, None, None, :]
    s = s.masked_fill(~keep, float("-inf"))
    e = e.masked_fill(~keep, 0.0)
    return s, e, keep


def _softmax(s):
    m = s.amax(-1, keepdim=True)
    m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    p = torch.exp(s - m)
    l = p.sum(-1, keepdim=True)
    p = torch.where(l > 0, p / l.clamp_min(1e-300), torch.zeros_like(p))
    lse = torch.where(l[..., 0] > 0, m[..., 0] + torch.log(l[..., 0].clamp_min(1e-300)), torch.full_like(l[..., 0], math.inf))
    return p, lse


def _batch_chunks(q, k):
    B, Sq, H, _ = q.shape
    return _chunks(B, H * Sq * k.shape[1] * 8 * 16)


def verify_sdpa_fwd(bound, q, k, v, scale, causal, kv_mask, rel_bias, out, lse, drop=None):
    """O = softmax(scale q k^T + bias) V. The kernel rounds each unnormalised probability exp2(x - m) <= 1 to bf16 before
    the PV MMA and O once at the end, dividing by the fp32 sum of the unrounded probabilities. With the per-row score error
    E = max_k e_s (see _scores) + (2 + Skv / 64) 2^-22 (ex2.approx per probability and per online-softmax rescale), each
    probability is within E relative before the bf16 rounding, so
    |O - O_ref| <= (u16 + 2 E + Skv 2^-23) (P |V|) + 1 ulp(O) (u16 for the rounded P, 2 E through numerator and
    denominator, the Skv-deep fp32 PV accumulation). P |V| <= max|V|: the issue's 2^-8 max|V| + 1 ulp, per element.
    lse (log2 domain) within (E + 2^-22 (1 + |lse|)) / ln 2. Rows with no key attended: O = 0, lse = +inf.
    With dropout (a DropSpec): O = (P M) V, M = Z / (1 - p) of the attention layout; the kernel multiplies each fp32
    probability by the fp32 1 / (1 - p) before the bf16 rounding (2^-23 more in E); the lse is that of the undropped P."""
    B, Sq, H, _ = q.shape
    Skv = k.shape[1]
    ln2 = math.log(2.0)
    for bs in _batch_chunks(q, k):
        s, e, keep = _scores(q, k, scale, causal, kv_mask, rel_bias, bs)
        p, lse_ref = _softmax(s)
        E = e.amax(-1, keepdim=True) + (2 + Skv / 64) * 2.0 ** -22
        if drop is not None:
            p = p * attn_mult(drop, _range(bs), H, Sq, Skv, q.device)
            E = E + 2.0 ** -23
        vd = _bhsd(v[bs]).double()
        ref = p @ vd
        mag = p @ vd.abs()
        tol = (U16 + 2 * E + Skv * 2.0 ** -23) * mag + bf16_ulp(ref)
        bound.close("O", _bhsd(out[bs]), ref, tol)
        lg = lse[bs].double()
        fin = torch.isfinite(lse_ref)
        bound.equal("rows without keys (lse = inf)", torch.isinf(lg) & (lg > 0), ~fin)
        ltol = (E[..., 0] + 2.0 ** -22 * (1 + lse_ref.abs())) / ln2
        bound.close("lse", torch.where(fin, lg, 0.0), torch.where(fin, lse_ref / ln2, 0.0), torch.where(fin, ltol, 0.0))


def check_sdpa_fwd(real, bound, q, k, v, scale, causal, kv_mask=None, out=None, rel_bias=None, drop=None):
    d = drop_spec(drop)
    o, lse = ret = real(q, k, v, scale, causal, kv_mask=kv_mask, out=out, rel_bias=rel_bias, drop=drop)
    verify_sdpa_fwd(bound, q, k, v, scale, causal, kv_mask, rel_bias, o, lse, d)
    return ret


def _diag_sums(m, Sq):
    """[nb, H, Sq, Skv] -> [H, Sq + Skv - 1]: sum over (b, q) of m[b, h, q, q + r - (Sq - 1)]."""
    nb, H, _, Skv = m.shape
    qi = torch.arange(Sq, device=m.device)[:, None]
    ki = torch.arange(Skv, device=m.device)[None, :]
    idx = (ki - qi + Sq - 1).expand(Sq, Skv).reshape(-1)
    out = torch.zeros((H, Sq + Skv - 1), dtype=torch.float64, device=m.device)
    out.index_add_(1, idx, m.sum(0).reshape(H, -1))
    return out


def verify_sdpa_bwd(bound, q, k, v, out, dout, lse, scale, causal, dq, dk, dv, kv_mask=None, rel_bias=None,
                    drel_bias=None, drel_old=None, drop=None):
    """The exact gradients of O = softmax(scale q k^T + bias) V for the given dO, in fp64: dV = P^T dO, dS = P (dP - delta)
    with dP = dO V^T and delta = rowsum(dO O), dQ = scale dS K, dK = scale dS^T Q, dbias[h, r] += sum over (b, q) of dS on
    diagonal r.
    The kernel recomputes P = exp2(x - lse) from the forward's lse and takes delta from the forward's bf16 O, so each P is
    within eps_P = |lse - lse_ref| ln 2 + max_k e_s + 3 2^-22 relative, delta within
    e_delta = sum_d |dO| |O - O_ref| + D 2^-23 sum_d |dO O|, dP within e_dP = D 2^-23 (|dO| |V|^T) (all computable from
    the call's own operands). Hence the fp32 dS is within E = P (eps_P |dP - delta| + (1 + eps_P)(e_dP + e_delta)).
    dQ, dK multiply bf16(dS) (u16 relative): |dQ - ref| <= scale ((u16 + Skv 2^-23)(|dS| + E) + E) |K| + 1 ulp, dK the
    same with Sq and |Q|; dV multiplies bf16(P): ((1 + u16)(eps_P + u16) + Sq 2^-23) P^T |dO| + 1 ulp. dbias sums the fp32
    dS: diagonal sums of E + B Sq 2^-23 |dS|, plus 2 u32 |dbias| for the add onto the old value.
    With dropout (a DropSpec, M = Z / (1 - p)): O = (P M) V, so dV = (P M)^T dO and dS = P (M dP - delta), delta still
    rowsum(dO O) of the dropped O (attention_bwd.cu multiplies dP by the fp32 M before subtracting delta): the bounds above
    with P M in dV's and M dP, M e_dP in dS's, and 2^-23 more in eps_P for the fp32 products with 1 / (1 - p)."""
    B, Sq, H, D = q.shape
    Skv = k.shape[1]
    ln2 = math.log(2.0)
    dsum = None if drel_bias is None else torch.zeros((H, Sq + Skv - 1), dtype=torch.float64, device=q.device)
    etot, atot = (torch.zeros_like(dsum), torch.zeros_like(dsum)) if dsum is not None else (None, None)
    for bs in _batch_chunks(q, k):
        s, e, keep = _scores(q, k, scale, causal, kv_mask, rel_bias, bs)
        p, lse_ref = _softmax(s)
        del s
        vd, dod, qd, kd = (_bhsd(t[bs]).double() for t in (v, dout, q, k))
        od = _bhsd(out[bs]).double()
        m = None if drop is None else attn_mult(drop, _range(bs), H, Sq, Skv, q.device)
        o_ref = (p if m is None else p * m) @ vd
        delta = (dod * o_ref).sum(-1, keepdim=True)
        e_delta = (dod.abs() * (od - o_ref).abs()).sum(-1, keepdim=True) + D * 2.0 ** -23 * (dod * od).abs().sum(-1, keepdim=True)
        del o_ref
        lg = lse[bs].double()
        dl = torch.where(torch.isfinite(lse_ref), (lg * ln2 - lse_ref).abs(), torch.zeros_like(lse_ref))
        eps_p = (dl[..., None] + e.amax(-1, keepdim=True) + 3 * 2.0 ** -22 + (0.0 if m is None else 2.0 ** -23))
        del e
        dP = dod @ vd.transpose(-1, -2)
        e_dp = D * 2.0 ** -23 * (dod.abs() @ vd.abs().transpose(-1, -2))
        if m is not None:
            dP, e_dp = dP * m, e_dp * m
        dS = p * (dP - delta)
        E = p * (eps_p * (dP - delta).abs() + (1 + eps_p) * (e_dp + e_delta))
        del dP, e_dp
        aS = dS.abs()
        ref = scale * (dS @ kd)
        tol = scale * (((U16 + Skv * 2.0 ** -23) * (aS + E) + E) @ kd.abs()) + bf16_ulp(ref)
        bound.close("dQ", _bhsd(dq[bs]), ref, tol)
        ref = scale * (dS.transpose(-1, -2) @ qd)
        tol = scale * (((U16 + Sq * 2.0 ** -23) * (aS + E) + E).transpose(-1, -2) @ qd.abs()) + bf16_ulp(ref)
        bound.close("dK", _bhsd(dk[bs]), ref, tol)
        pm = p if m is None else p * m
        del m
        ref = pm.transpose(-1, -2) @ dod
        w = ((1 + U16) * (eps_p + U16) + Sq * 2.0 ** -23) * pm
        del pm
        tol = w.transpose(-1, -2) @ dod.abs() + bf16_ulp(ref)
        bound.close("dV", _bhsd(dv[bs]), ref, tol)
        if dsum is not None:
            dsum += _diag_sums(dS, Sq)
            etot += _diag_sums(E, Sq)
            atot += _diag_sums(aS, Sq)
        del p, dS, E, aS
    if dsum is not None:
        ref = drel_old.double() + dsum
        tol = etot + B * Sq * 2.0 ** -23 * atot + 2 * U32 * (drel_old.double().abs() + ref.abs())
        bound.close("drel_bias", drel_bias, ref, tol)


def check_sdpa_bwd(real, bound, q, k, v, out, dout, lse, scale, causal, dq, dk, dv, kv_mask=None, rel_bias=None,
                   drel_bias=None, drop=None):
    old = None if drel_bias is None else drel_bias.clone()
    d = drop_spec(drop)
    ret = real(q, k, v, out, dout, lse, scale, causal, dq, dk, dv, kv_mask=kv_mask, rel_bias=rel_bias, drel_bias=drel_bias,
               drop=drop)
    verify_sdpa_bwd(bound, q, k, v, out, dout, lse, scale, causal, dq, dk, dv, kv_mask, rel_bias, drel_bias, old, d)
    return ret


# ------------------------------------------------------------------------------------------------ weight-only int8 / int4
def verify_quantize_w8(bound, w, q, s):
    """q and s bit for bit as int8_ref.quantize (the numpy float32 restatement of include/fsb200.h) gives them."""
    n, k = w.shape
    for rs in _chunks(n, k * 4 * 8):
        qn, sn = int8_ref.quantize(w[rs].float().cpu().numpy())
        bound.equal("int8 codes", q[rs].cpu(), torch.from_numpy(qn))
        bound.equal("row scales (bits)", s[rs].cpu().view(torch.int32), torch.from_numpy(sn).view(torch.int32))


def check_quantize_w8(real, bound, w, q=None, s=None):
    ret = real(w, q=q, s=s)
    verify_quantize_w8(bound, w, *ret)
    return ret


def verify_quantize_w4(bound, w, q, s):
    """The packed codes and the bf16 group scales bit for bit as int4_ref.quantize and int4_ref.pack give them."""
    n, k = w.shape
    for rs in _chunks(n // 2, 2 * k * 4 * 8):
        rows = slice(2 * rs.start, 2 * rs.stop)
        qn, sn = int4_ref.quantize(w[rows].float().cpu().numpy())
        bound.equal("packed int4 codes", q[rs].cpu(), torch.from_numpy(int4_ref.pack(qn)))
        bound.exact("group scales", s[rows].cpu(), torch.from_numpy(sn).to(BF16))


def check_quantize_w4(real, bound, w, q=None, s=None):
    ret = real(w, q=q, s=s)
    verify_quantize_w4(bound, w, *ret)
    return ret


def unpack_w4(q, s):
    """W^ = bf16(q * s) [n, k] from the packed codes and the group scales (int4_ref.unpack / dequantize in torch, so it
    runs on the operands' device)."""
    p2, k = q.shape
    b = q.reshape(p2, k // 16, 4, 2, 2).to(torch.int16)                        # [p, block, t, b, h]
    u = torch.stack([b & 0xF, b >> 4], -1) - 8                                 # [p, block, t, b, h, row]
    codes = u.permute(0, 5, 1, 4, 2, 3).reshape(2 * p2, k)
    return (codes.float() * s.float().repeat_interleave(int4_ref.GROUP, 1)).to(BF16)


def _verify_scaled_gemm(bound, what, a64_of, b64_of, m, n, k, out, old=None, acc_rel=None):
    """out[m, n] = bf16(A B^T (+ old)), fp32 accumulation of exact products: 2^-8 |ref| for the rounding (and the scale
    products), K 2^-23 (|A||B|^T) for the accumulation, 2 u32 |old| for the add (test_fp8_gpu / test_int8_gpu's bound).
    `acc_rel` replaces K 2^-23 where the accumulation is not plain fp32."""
    for cs in _chunks(n, 8 * 2 * k):
        B64 = b64_of(cs)
        Babs = B64.abs()
        for rs in _chunks(m, 8 * (2 * k + 6 * (cs.stop - cs.start))):
            A64 = a64_of(rs)
            ref = A64 @ B64.t()
            tol = (k * 2.0 ** -23 if acc_rel is None else acc_rel) * (A64.abs() @ Babs.t())
            del A64
            if old is not None:
                o = old[rs, cs].double()
                ref, tol = ref + o, tol + 2 * U32 * o.abs()
            bound.close(what, out[rs, cs], ref, tol + 2.0 ** -8 * ref.abs())
            del ref, tol
        del B64, Babs


def verify_gemm_w8a16(bound, a, q, s, out):
    """out = bf16(s[n] (A q^T)): the fp64 product with the dequantised weight q s, at the bound of test_int8_gpu."""
    m, k = a.shape
    _verify_scaled_gemm(bound, "W8A16 D", lambda rs: a[rs].double(), lambda cs: q[cs].double() * s[cs].double()[:, None],
                        m, q.shape[0], k, out)


def check_gemm_w8a16(real, bound, a, q, s, out=None):
    ret = real(a, q, s, out=out)
    verify_gemm_w8a16(bound, a, q, s, ret)
    return ret


def verify_gemm_w4a16(bound, a, q, s, out):
    """out = bf16(A W^T), W^ = bf16(q s) the dequantised int4 weight: fp64 over W^ at the bound of test_int4_gpu."""
    m, k = a.shape
    n = 2 * q.shape[0]

    def b64(cs):
        lines = slice(cs.start // 2, (cs.stop + 1) // 2)
        w = unpack_w4(q[lines], s[2 * lines.start:2 * lines.stop]).double()
        return w[cs.start - 2 * lines.start:cs.stop - 2 * lines.start]
    _verify_scaled_gemm(bound, "W4A16 D", lambda rs: a[rs].double(), b64, m, n, k, out)


def check_gemm_w4a16(real, bound, a, q, s, out=None):
    ret = real(a, q, s, out=out)
    verify_gemm_w4a16(bound, a, q, s, ret)
    return ret


# ------------------------------------------------------------------------------------------------------------- FP8
def verify_fp8_quantize(bound, x, fmt, y, yt, scale_inv):
    """The codes (row-major and transposed) and 1 / scale bit for bit as tests/fp8_ref.py gives them: amax over the whole
    tensor, scale = 2^e, each code the satfinite round-to-nearest-even cast of x scale."""
    rows, cols = x.shape
    amax = float(x.float().abs().max()) if x.numel() else 0.0
    e, sinv = fp8_ref.scale_exp(amax, fmt)
    bound.equal("scale_inv (bits)", scale_inv.reshape(-1).cpu().view(torch.int32),
                torch.tensor([sinv], dtype=torch.float32).view(torch.int32))
    sc = np.float32(np.ldexp(1.0, e))
    for rs in _chunks(rows, cols * 8 * 16):
        codes = torch.from_numpy(fp8_ref.encode(x[rs].float().cpu().numpy() * sc, fmt))
        if y is not None:
            bound.equal("row-major codes", y[rs].view(torch.uint8).cpu(), codes)
        if yt is not None:
            bound.equal("transposed codes", yt[:, rs].view(torch.uint8).cpu(), codes.t())


def check_fp8_quantize(real, bound, x, fmt, rowwise=True, colwise=False):
    ret = real(x, fmt, rowwise=rowwise, colwise=colwise)
    verify_fp8_quantize(bound, x, fmt, *ret)
    return ret


FP8_MMA_REL = 2.0 ** -9    # the FP8 tensor-core accumulation error of one 128-deep block, relative to its sum |A||B|


def verify_gemm_fp8(bound, a, a_scale_inv, b, b_scale_inv, out, old=None):
    """out (+)= bf16((A B^T) a_scale_inv b_scale_inv) over the decoded codes, on the scaled operands: 2^-8 |ref| for the
    rounding, 2 u32 |old| for the accumulate add, and (FP8_MMA_REL + K / 128 2^-23) (|A||B|^T) for the accumulation.
    The FP8 wgmma does not accumulate in full fp32: inside the tensor core the sum keeps about 14 significant bits (the
    DeepSeek-V3 report, section 3.3.2, measured it on Hopper), which is why gemm_fp8.cu promotes the partial of every
    128-deep block into an fp32 accumulator (K / 128 fp32 adds, 2^-23 each). NVIDIA does not document how the tensor core
    aligns and truncates, so the in-block term is not derived: FP8_MMA_REL = 2^-9 allows each of a block's four k32 wgmma
    steps to lose 2^-11 of the block's sum |A||B|. On one H100 80GB HBM3 the census's weight-gradient GEMMs (K = 1024
    tokens) measured up to 8e-4 = 2^-10.3 of sum |A||B| beyond the bf16 rounding, more than an fp32 sum of 1024 terms can
    lose (1024 2^-24 = 6e-5); test_fp8_gpu.test_gemm_vs_fp64's fp32 bound K 2^-23 (|A||B|^T) fails there."""
    sa, sb = float(a_scale_inv.double()), float(b_scale_inv.double())
    m, k = a.shape
    _verify_scaled_gemm(bound, "FP8 D", lambda rs: a[rs].float().double() * sa, lambda cs: b[cs].float().double() * sb,
                        m, b.shape[0], k, out, old, acc_rel=FP8_MMA_REL + -(-k // 128) * 2.0 ** -23)


def check_gemm_fp8(real, bound, a, a_scale_inv, b, b_scale_inv, out=None, accumulate=False):
    old = out.clone() if accumulate else None
    ret = real(a, a_scale_inv, b, b_scale_inv, out=out, accumulate=accumulate)
    verify_gemm_fp8(bound, a, a_scale_inv, b, b_scale_inv, ret, old)
    return ret


# --------------------------------------------------------------------------------------------------------- decoding
def verify_attn_decode(bound, q, k_cache, v_cache, kv_len, scale, kv_mask, rel_bias, out, lse):
    """One query per (batch, head) against the slots [0, kv_len) only: scores scale q.k + rel_bias[h, k - (kv_len - 1) +
    cap - 1], masked where kv_mask is 0 (or the bias -inf), softmax and P V in fp64. The kernel keeps every probability in
    fp32 (no bf16 rounding of P) and merges the split partials in fp32, so with E = max_k e_s (_scores' error) +
    (3 + cap / 32) 2^-22 (ex2.approx per probability, per rescale and per merged split)
    |O - O_ref| <= (2 E + kv_len 2^-23) (P |V|) + 1 ulp(O); lse (log2 domain) within (E + 2^-22 (1 + |lse|)) / ln 2. A row
    that sees no key: O = 0, lse = +inf."""
    B, H, D = q.shape
    cap = k_cache.shape[1]
    L = max(0, min(int(kv_len), cap))
    ln2 = math.log(2.0)
    for bs in _chunks(B, H * max(L, 1) * 8 * (12 + 4 * D)):
        qd = q[bs].double()                                         # [b, H, D]
        kd = k_cache[bs, :L].double().permute(0, 2, 1, 3)           # [b, H, L, D]
        vd = v_cache[bs, :L].double().permute(0, 2, 1, 3)
        s = scale * torch.einsum("bhd,bhld->bhl", qd, kd)
        e = D * 2.0 ** -23 * scale * torch.einsum("bhd,bhld->bhl", qd.abs(), kd.abs()) + 2.0 ** -22 * s.abs()
        keep = torch.ones_like(s, dtype=torch.bool)
        if rel_bias is not None:
            bias = rel_bias.double()[:, torch.arange(L, device=q.device) - (L - 1) + cap - 1][None]   # [1, H, L]
            fin = torch.isfinite(bias)
            bias = torch.where(fin, bias, 0.0)
            s, e, keep = s + bias, e + 2.0 ** -22 * bias.abs(), keep & fin
        if kv_mask is not None:
            keep = keep & (kv_mask[bs, :L] != 0)[:, None, :]
        s = s.masked_fill(~keep, float("-inf"))
        e = e.masked_fill(~keep, 0.0)
        p, lse_ref = _softmax(s)
        E = (e.amax(-1, keepdim=True) if L else torch.zeros_like(s[..., :1])) + (3 + cap / 32) * 2.0 ** -22
        ref = torch.einsum("bhl,bhld->bhd", p, vd)
        mag = torch.einsum("bhl,bhld->bhd", p, vd.abs())
        bound.close("O", out[bs], ref, (2 * E + L * 2.0 ** -23) * mag + bf16_ulp(ref))
        if lse is not None:
            lg = lse[bs].double()
            fin = torch.isfinite(lse_ref)
            bound.equal("rows without keys (lse = inf)", torch.isinf(lg) & (lg > 0), ~fin)
            ltol = (E[..., 0] + 2.0 ** -22 * (1 + lse_ref.abs())) / ln2
            bound.close("lse", torch.where(fin, lg, 0.0), torch.where(fin, lse_ref / ln2, 0.0), torch.where(fin, ltol, 0.0))


def check_attn_decode(real, bound, q, k_cache, v_cache, kv_len, scale, kv_mask=None, rel_bias=None, out=None):
    o, lse = ret = real(q, k_cache, v_cache, kv_len, scale, kv_mask=kv_mask, rel_bias=rel_bias, out=out)
    verify_attn_decode(bound, q, k_cache, v_cache, int(kv_len.item()), scale, kv_mask, rel_bias, o, lse)
    return ret


def verify_kv_append(bound, k_new, v_new, kv_len, k_before, v_before, m_before, k_cache, v_cache, kv_mask):
    """Slot kv_len - 1 of both caches holds k_new / v_new bit for bit and its kv_mask bit is 1; every other element of both
    caches and of the mask is unchanged (a slot outside the cache: nothing changes)."""
    cap = k_cache.shape[1]
    slot = int(kv_len) - 1
    for name, new, before, after in (("K cache", k_new, k_before, k_cache), ("V cache", v_new, v_before, v_cache)):
        want = before.clone()
        if 0 <= slot < cap:
            want[:, slot] = new
        bound.exact(name, after, want)
    if kv_mask is not None:
        want = m_before.clone()
        if 0 <= slot < cap:
            want[:, slot] = 1
        bound.equal("kv_mask", kv_mask, want)


def check_kv_append(real, bound, k_new, v_new, k_cache, v_cache, kv_len, kv_mask=None):
    kb, vb = k_cache.clone(), v_cache.clone()
    mb = None if kv_mask is None else kv_mask.clone()
    ret = real(k_new, v_new, k_cache, v_cache, kv_len, kv_mask=kv_mask)
    verify_kv_append(bound, k_new, v_new, int(kv_len.item()), kb, vb, mb, k_cache, v_cache, kv_mask)
    return ret


def verify_kv_reorder(bound, src, index, kv_len, dst_before, dst):
    """dst[l, r, :kv_len] = src[l, index[r], :kv_len] bit for bit; dst's slots at or beyond kv_len are unchanged."""
    cap = src.shape[2]
    L = max(0, min(int(kv_len), cap))
    want = dst_before.clone()
    want[:, :, :L] = src[:, index.to(src.device), :L]
    bound.exact("reordered cache", dst, want)


def check_kv_reorder(real, bound, src, dst, index, kv_len):
    before = dst.clone()
    ret = real(src, dst, index, kv_len)
    verify_kv_reorder(bound, src, index, int(kv_len.item()), before, dst)
    return ret


CHECKERS = {
    "gemm": check_gemm,
    "rmsnorm_fwd": check_rmsnorm_fwd, "rmsnorm_bwd": check_rmsnorm_bwd,
    "layernorm_fwd": check_layernorm_fwd, "layernorm_bwd": check_layernorm_bwd,
    "rope_inplace": check_rope_inplace,
    "glu_fwd": check_glu_fwd, "glu_bwd": check_glu_bwd,
    "act_fwd": check_act_fwd, "act_bwd": check_act_bwd, "act_bwd_bias": check_act_bwd_bias,
    "colsum": check_colsum,
    "embedding_fwd": check_embedding_fwd, "embedding_bwd": check_embedding_bwd,
    "sdpa_fwd": check_sdpa_fwd, "sdpa_bwd": check_sdpa_bwd,
    "softmax_xent": check_softmax_xent,
    "accumulate": check_accumulate, "scale_inplace": check_scale_inplace, "cast_f32_to_bf16": check_cast_f32_to_bf16,
    "add": check_add,
    "sumsq": check_sumsq, "clip_coef": check_clip_coef, "adamw_flat": check_adamw_flat,
    "dropout": check_dropout, "dropout_advance": check_dropout_advance,
    "layernorm_bwd_dropout": check_layernorm_bwd_dropout, "rmsnorm_bwd_dropout": check_rmsnorm_bwd_dropout,
    "fp8_quantize": check_fp8_quantize, "gemm_fp8": check_gemm_fp8,
    "quantize_w8": check_quantize_w8, "quantize_w4": check_quantize_w4,
    "gemm_w8a16": check_gemm_w8a16, "gemm_w4a16": check_gemm_w4a16,
    "attn_decode": check_attn_decode, "kv_append": check_kv_append, "kv_reorder": check_kv_reorder,
}
