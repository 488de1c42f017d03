"""fp64 references of the W8A16 / W4A16 GEMMs with a bias / GELU epilogue (ops.gemm_w8a16 / ops.gemm_w4a16 with `bias`,
include/fsb200.h fsb_gemm_w8a16_bias / fsb_gemm_w4a16_bias), in the form of tests/launch_refs.py's checkers, and
`CHECKERS`: launch_refs.CHECKERS with the two GEMM entries replaced by these, for launch censuses of int8 / int4 GPT-2.
A call without a bias is held to the bound launch_refs gives the bias-free GEMM. tests/test_gpt2_int8_cpu.py pins these
references to an independent torch computation."""
import launch_refs as R

EPI_NONE, EPI_GELU_TANH = R.EPI_NONE, R.EPI_GELU_TANH


def _verify(bound, what, a64_of, b64_of, m, n, k, out, bias, epilogue):
    """out[m, n] = bf16(act(A B^T + bias)), fp32 accumulation of exact products. The bound is launch_refs'
    _verify_scaled_gemm's (K 2^-23 (|A||B|^T) for the accumulation, 2^-8 |ref| for the rounding and the scale products),
    plus 2 u32 |bias| for the fp32 bias add; a GELU epilogue scales the accumulated bound by GELU_SLOPE and adds
    ACT_FLOOR (1 + |pre-activation|), as launch_refs.verify_gemm does for the bf16 GEMM's epilogue."""
    act = R._EPI_ACT.get(epilogue)
    for cs in R._chunks(n, 8 * 2 * k):
        B64 = b64_of(cs)
        Babs = B64.abs()
        bias64 = None if bias is None else bias[cs].double().view(1, -1)
        for rs in R._chunks(m, 8 * (2 * k + 6 * (cs.stop - cs.start))):
            A64 = a64_of(rs)
            ref = A64 @ B64.t()
            tol = k * 2.0 ** -23 * (A64.abs() @ Babs.t())
            del A64
            if bias64 is not None:
                ref, tol = ref + bias64, tol + 2 * R.U32 * bias64.abs()
            if act is not None:
                ref, tol = R.act64(act, ref), R.GELU_SLOPE * tol + R.ACT_FLOOR * (1.0 + ref.abs())
            bound.close(what, out[rs, cs], ref, tol + 2.0 ** -8 * ref.abs())
            del ref, tol
        del B64, Babs


def verify_gemm_w8a16(bound, a, q, s, out, bias=None, epilogue=EPI_NONE):
    """out = bf16(act(s[n] (A q^T) + bias)) against the fp64 product with the dequantised weight q s."""
    m, k = a.shape
    _verify(bound, "W8A16 D", lambda rs: a[rs].double(), lambda cs: q[cs].double() * s[cs].double()[:, None],
            m, q.shape[0], k, out, bias, epilogue)


def verify_gemm_w4a16(bound, a, q, s, out, bias=None, epilogue=EPI_NONE):
    """out = bf16(act(A W^T + bias)), W^ = bf16(q s) the dequantised int4 weight, against fp64 over W^."""
    m, k = a.shape
    n = 2 * q.shape[0]

    def b64(cs):
        lines = slice(cs.start // 2, (cs.stop + 1) // 2)
        w = R.unpack_w4(q[lines], s[2 * lines.start:2 * lines.stop]).double()
        return w[cs.start - 2 * lines.start:cs.stop - 2 * lines.start]
    _verify(bound, "W4A16 D", lambda rs: a[rs].double(), b64, m, n, k, out, bias, epilogue)


def check_gemm_w8a16(real, bound, a, q, s, out=None, bias=None, epilogue=EPI_NONE):
    if bias is None and epilogue == EPI_NONE:   # the bias-free call: launch_refs' checker, unchanged
        return R.check_gemm_w8a16(real, bound, a, q, s, out=out)
    ret = real(a, q, s, out=out, bias=bias, epilogue=epilogue)
    verify_gemm_w8a16(bound, a, q, s, ret, bias, epilogue)
    return ret


def check_gemm_w4a16(real, bound, a, q, s, out=None, bias=None, epilogue=EPI_NONE):
    if bias is None and epilogue == EPI_NONE:
        return R.check_gemm_w4a16(real, bound, a, q, s, out=out)
    ret = real(a, q, s, out=out, bias=bias, epilogue=epilogue)
    verify_gemm_w4a16(bound, a, q, s, ret, bias, epilogue)
    return ret


CHECKERS = dict(R.CHECKERS, gemm_w8a16=check_gemm_w8a16, gemm_w4a16=check_gemm_w4a16)
