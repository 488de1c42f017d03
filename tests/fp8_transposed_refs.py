"""The fp64 reference of the FP8 GEMM's transposed store (`ops.gemm_fp8(..., store_transposed=True)`, fsb_gemm_fp8_t), for
the launch censuses of FP8 GPT-2 steps: the result is the plain call's D transposed, so it is verified with
tests/launch_refs.py's verify_gemm_fp8 through the transposed views of out and of the old out."""
import launch_refs as R


def check_gemm_fp8_t(real, bound, a, a_scale_inv, b, b_scale_inv, out=None, accumulate=False, store_transposed=True):
    assert store_transposed
    old = out.clone() if accumulate else None
    ret = real(a, a_scale_inv, b, b_scale_inv, out=out, accumulate=accumulate, store_transposed=True)
    R.verify_gemm_fp8(bound, a, a_scale_inv, b, b_scale_inv, ret.t(), None if old is None else old.t())
    return ret
