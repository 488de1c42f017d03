"""fp64 reference for fsb_gemm_fp8 with its epilogue (bias, GELU, aux), on top of tests/launch_refs.py's FP8 GEMM bound.
Used by the BERT / MegatronBERT FP8 tests (tests/test_bert_fp8_{cpu,gpu}.py) and by their launch censuses, whose FP8 GEMM
calls carry bias / epilogue / aux keywords; calls without them are exactly launch_refs.verify_gemm_fp8."""
import launch_refs as R


def verify_gemm_fp8(bound, a, a_scale_inv, b, b_scale_inv, out, old=None, bias=None, epilogue=R.EPI_NONE, aux=None):
    """out (+)= act((A B^T) a_scale_inv b_scale_inv + bias) over the decoded codes, aux = bf16 of the pre-activation.
    Without bias, epilogue or aux this is launch_refs.verify_gemm_fp8. With them, the epilogue is launch_refs.verify_gemm's
    on the FP8 accumulation bound: (FP8_MMA_REL + K / 128 2^-23) (|A||B|^T), plus 2 u32 |bias| for the bias add; aux within
    that plus 2^-8 |pre|; D = act(pre) (+ old) within GELU_SLOPE times the bound, ACT_FLOOR (1 + |pre|) for the fp32 GELU,
    2 u32 |old| for the accumulate add, and 2^-8 |ref| for the rounding."""
    if bias is None and epilogue == R.EPI_NONE and aux is None:
        R.verify_gemm_fp8(bound, a, a_scale_inv, b, b_scale_inv, out, old)
        return
    sa, sb = float(a_scale_inv.double()), float(b_scale_inv.double())
    m, k = a.shape
    n = b.shape[0]
    acc_rel = R.FP8_MMA_REL + -(-k // 128) * 2.0 ** -23
    act = R._EPI_ACT.get(epilogue)
    for cs in R._chunks(n, 8 * 2 * k):
        B64 = b[cs].float().double() * sb
        Babs = B64.abs()
        bias64 = None if bias is None else bias.reshape(-1)[cs].double().view(1, -1)
        for rs in R._chunks(m, 8 * (2 * k + 14 * (cs.stop - cs.start))):
            A64 = a[rs].float().double() * sa
            pre = A64 @ B64.t()
            mag = acc_rel * (A64.abs() @ Babs.t())
            del A64
            if bias64 is not None:
                pre, mag = pre + bias64, mag + 2 * R.U32 * bias64.abs()
            if aux is not None:
                bound.close("FP8 aux (pre-activation)", aux[rs, cs], pre, mag + 2.0 ** -8 * pre.abs())
            if act is not None:
                ref, tol = R.act64(act, pre), R.GELU_SLOPE * mag + R.ACT_FLOOR * (1.0 + pre.abs())
            else:
                ref, tol = pre, mag
            if old is not None:
                o = old[rs, cs].double()
                ref, tol = ref + o, tol + 2 * R.U32 * o.abs()
            bound.close("FP8 D", out[rs, cs], ref, tol + 2.0 ** -8 * ref.abs())
            del pre, mag, ref, tol
        del B64, Babs


def check_gemm_fp8(real, bound, a, a_scale_inv, b, b_scale_inv, out=None, accumulate=False, bias=None, epilogue=R.EPI_NONE,
                   aux=None):
    """launch_census checker for ops.gemm_fp8 calls with any of its keywords."""
    old = out.clone() if accumulate else None
    ret = real(a, a_scale_inv, b, b_scale_inv, out=out, accumulate=accumulate, bias=bias, epilogue=epilogue, aux=aux)
    verify_gemm_fp8(bound, a, a_scale_inv, b, b_scale_inv, ret, old, bias, epilogue, aux)
    return ret
