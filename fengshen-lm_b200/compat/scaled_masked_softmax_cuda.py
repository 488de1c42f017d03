"""Drop-in for the reference's pybind module `scaled_masked_softmax_cuda`
(fengshen/models/megatron/fused_kernels/scaled_masked_softmax.cpp:70-83): same three functions, same tensor contract
(input [b, np, sq, sk] half-precision, mask [b|1, 1, sq, sk] uint8/bool with 1 = masked, float scale; backward returns the
gradient written IN PLACE over `output_grads`), executed by libfsb200.so. Only bf16 is implemented (the GPU path trains in
bf16); an fp16 tensor raises instead of silently falling back."""
import torch

from fsb200 import lib as _L


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _check(t, name):
    if not t.is_cuda or t.dtype != torch.bfloat16 or not t.is_contiguous():
        raise RuntimeError(f"{name} must be a contiguous CUDA bfloat16 tensor (got {t.dtype}, cuda={t.is_cuda})")


def forward(input, mask, scale_factor):
    _check(input, "input")
    if input.dim() != 4:
        raise RuntimeError("expected 4D tensor")                        # scaled_masked_softmax.cpp:35
    b, np_, sq, sk = input.shape
    if mask.dim() != 4 or mask.size(1) != 1 or mask.size(2) != sq or mask.size(3) != sk or mask.size(0) not in (1, b):
        raise RuntimeError("mask must be [b or 1, 1, sq, sk]")          # scaled_masked_softmax_cuda.cu:46-49
    m = mask.to(torch.uint8).contiguous()
    out = torch.empty_like(input)
    _L.call("fsb_scaled_masked_softmax_fwd", input.data_ptr(), m.data_ptr(), out.data_ptr(), b, np_, sq, sk, m.size(0),
            float(scale_factor), _stream())
    return out


def backward(output_grads, softmax_results, scale_factor):
    _check(output_grads, "output_grads"); _check(softmax_results, "softmax_results")
    sk = output_grads.shape[-1]
    _L.call("fsb_scaled_masked_softmax_bwd", output_grads.data_ptr(), softmax_results.data_ptr(),
            output_grads.numel() // sk, sk, float(scale_factor), _stream())
    return output_grads                                                  # in place, like the reference


def get_batch_per_block(query_seq_len, key_seq_len, batches, attn_heads):
    return _L.load().fsb_softmax_get_batch_per_block(query_seq_len, key_seq_len, batches, attn_heads)
