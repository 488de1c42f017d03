"""ctypes binding of libfsb200.so (C ABI declared in include/fsb200.h).

The library is the product; this module only marshals pointers. There is NO fallback: if the shared object is
missing or a call fails, a RuntimeError is raised (the reference prints and exit()s when its fused kernels are
missing, fengshen/models/megatron/fused_kernels/__init__.py:32-44).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libfsb200.so")

c_void_p = ctypes.c_void_p
c_int = ctypes.c_int
c_i64 = ctypes.c_int64
c_f32 = ctypes.c_float
c_size = ctypes.c_size_t
c_u64 = ctypes.c_uint64

BF16, F32, U32, U64 = 0, 1, 2, 3
GEMM_NT, GEMM_NN, GEMM_TN = 0, 1, 2
EPI_NONE, EPI_GELU_TANH, EPI_GELU_ERF = 0, 1, 2
ACT_SILU, ACT_GELU_TANH, ACT_GELU_ERF, ACT_TANH = 0, 1, 2, 3

# name -> (restype, [argtypes])  — must mirror include/fsb200.h exactly (tests/test_abi.py checks the symbol list)
SIGNATURES = {
    "fsb_version": (c_int, []),
    "fsb_last_error": (ctypes.c_char_p, []),
    "fsb_num_sms": (c_int, []),
    "fsb_gemm_bf16": (c_int, [c_int, c_i64, c_i64, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_int,
                              c_void_p, c_int, c_int, c_int, c_void_p, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64,
                              c_void_p, c_size, c_void_p]),
    "fsb_gemm_workspace_bytes": (c_size, [c_int, c_i64, c_i64, c_i64]),
    "fsb_set_reserved_sms": (c_int, [c_int]),
    "fsb_quantize_w8": (c_int, [c_void_p, c_i64, c_i64, c_i64, c_void_p, c_void_p, c_void_p]),
    "fsb_gemm_w8a16_workspace_bytes": (c_size, [c_i64, c_i64, c_i64]),
    "fsb_gemm_w8a16": (c_int, [c_i64, c_i64, c_i64, c_void_p, c_i64, c_void_p, c_void_p, c_void_p, c_i64, c_void_p, c_size,
                               c_void_p]),
    "fsb_quantize_w4": (c_int, [c_void_p, c_i64, c_i64, c_i64, c_void_p, c_void_p, c_void_p]),
    "fsb_gemm_w4a16_workspace_bytes": (c_size, [c_i64, c_i64, c_i64]),
    "fsb_gemm_w4a16": (c_int, [c_i64, c_i64, c_i64, c_void_p, c_i64, c_void_p, c_void_p, c_void_p, c_i64, c_void_p, c_size,
                               c_void_p]),
    "fsb_gemm_w8a16_bias": (c_int, [c_i64, c_i64, c_i64, c_void_p, c_i64, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                    c_i64, c_void_p, c_size, c_void_p]),
    "fsb_gemm_w4a16_bias": (c_int, [c_i64, c_i64, c_i64, c_void_p, c_i64, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                    c_i64, c_void_p, c_size, c_void_p]),
    "fsb_fp8_quantize": (c_int, [c_void_p, c_i64, c_i64, c_i64, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fsb_gemm_fp8": (c_int, [c_i64, c_i64, c_i64, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_i64,
                             c_void_p, c_int, c_int, c_void_p, c_i64, c_void_p]),
    "fsb_gemm_fp8_t": (c_int, [c_i64, c_i64, c_i64, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_i64,
                               c_void_p, c_int, c_int, c_void_p, c_i64, c_void_p]),
    "fsb_norm_bwd_workspace_bytes": (c_size, [c_i64, c_i64, c_int]),
    "fsb_rmsnorm_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_f32,
                                c_void_p]),
    "fsb_rmsnorm_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                c_void_p, c_size, c_i64, c_i64, c_void_p]),
    "fsb_layernorm_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64,
                                  c_f32, c_void_p]),
    "fsb_layernorm_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_int, c_int, c_void_p, c_size, c_i64, c_i64, c_void_p]),
    "fsb_rope_inplace": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_int, c_int, c_i64, c_i64, c_i64,
                                 c_int, c_void_p]),
    "fsb_glu_fwd": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_i64, c_void_p]),
    "fsb_glu_bwd": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64,
                            c_i64, c_i64, c_i64, c_void_p]),
    "fsb_act_fwd": (c_int, [c_int, c_void_p, c_void_p, c_i64, c_void_p]),
    "fsb_act_bwd": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_i64, c_void_p]),
    "fsb_act_bwd_bias_workspace_bytes": (c_size, [c_i64, c_i64]),
    "fsb_act_bwd_bias": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_void_p, c_int, c_int, c_void_p, c_size,
                                 c_void_p]),
    "fsb_add": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_void_p]),
    "fsb_accumulate": (c_int, [c_void_p, c_void_p, c_i64, c_f32, c_int, c_void_p]),
    "fsb_scale_inplace": (c_int, [c_void_p, c_i64, c_void_p, c_void_p]),
    "fsb_colsum_workspace_bytes": (c_size, [c_i64, c_i64]),
    "fsb_colsum": (c_int, [c_void_p, c_i64, c_i64, c_i64, c_void_p, c_int, c_int, c_void_p, c_size, c_void_p]),
    "fsb_embedding_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64,
                                  c_i64, c_void_p]),
    "fsb_embedding_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_void_p]),
    "fsb_embedding_bwd_sorted": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_void_p]),
    "fsb_cast_f32_to_bf16": (c_int, [c_void_p, c_void_p, c_i64, c_void_p]),
    "fsb_softmax_xent_fwd_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64,
                                         c_i64, c_i64, c_int, c_int, c_f32, c_void_p]),
    "fsb_adamw_flat": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_i64, c_f32, c_f32, c_f32,
                               c_f32, c_f32, c_i64, c_void_p, c_void_p, c_void_p]),
    "fsb_sumsq_workspace_bytes": (c_size, []),
    "fsb_sumsq": (c_int, [c_void_p, c_int, c_i64, c_void_p, c_int, c_void_p, c_size, c_void_p]),
    "fsb_clip_coef": (c_int, [c_void_p, c_f32, c_void_p, c_void_p, c_void_p]),
    "fsb_scaled_masked_softmax_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_i64, c_f32,
                                              c_void_p]),
    "fsb_scaled_masked_softmax_bwd": (c_int, [c_void_p, c_void_p, c_i64, c_i64, c_f32, c_void_p]),
    "fsb_scaled_upper_triang_masked_softmax_fwd": (c_int, [c_void_p, c_void_p, c_i64, c_i64, c_f32, c_void_p]),
    "fsb_scaled_upper_triang_masked_softmax_bwd": (c_int, [c_void_p, c_void_p, c_i64, c_i64, c_f32, c_void_p]),
    "fsb_softmax_get_batch_per_block": (c_int, [c_i64, c_i64, c_i64, c_i64]),
    "fsb_comm_unique_id": (c_int, [c_void_p]),
    "fsb_comm_init": (c_int, [c_void_p, c_void_p, c_int, c_int]),
    "fsb_comm_destroy": (c_int, [c_void_p]),
    "fsb_comm_reduce_scatter": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_int, c_void_p]),
    "fsb_comm_all_gather": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_int, c_void_p]),
    "fsb_comm_all_reduce": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_int, c_void_p]),
    "fsb_index_build_sample_idx": (c_int, [c_void_p, c_void_p, c_i64, ctypes.c_int32, ctypes.c_int32, c_i64, c_void_p, c_i64]),
    "fsb_index_build_mapping": (c_i64, [c_void_p, c_i64, c_void_p, ctypes.c_int32, ctypes.c_uint64, ctypes.c_int32,
                                        ctypes.c_double, ctypes.c_int32, ctypes.c_int32, c_int, c_void_p, c_i64]),
    "fsb_index_build_blocks_mapping": (c_i64, [c_void_p, c_i64, c_void_p, c_void_p, ctypes.c_int32, ctypes.c_uint64,
                                               ctypes.c_int32, ctypes.c_int32, c_int, c_int, c_void_p, c_i64]),
    "fsb_index_build_blending_indices": (c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_int32, c_i64]),
    "fsb_bert_collate": (c_i64, [c_void_p, c_void_p, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64] + [ctypes.c_int32] * 5 +
                         [ctypes.c_double, c_void_p, ctypes.c_int32, c_void_p, c_void_p] + [c_void_p] * 5),
    "fsb_sdpa_fwd": (c_int, [c_void_p] * 5 + [c_i64, c_i64, c_i64, c_int, c_int] + [c_i64] * 8 +
                     [c_f32, c_int, c_void_p, c_void_p] + [c_void_p] * 4 + [c_f32, c_u64, c_void_p, c_i64, c_void_p]),
    "fsb_sdpa_bwd_workspace_bytes": (c_size, [c_i64, c_i64, c_i64, c_int]),
    "fsb_sdpa_bwd": (c_int, [c_void_p] * 10 + [c_i64, c_i64, c_i64, c_int, c_int] + [c_i64] * 16 +
                     [c_f32, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_size] + [c_void_p] * 4 +
                     [c_f32, c_u64, c_void_p, c_i64, c_void_p]),
    "fsb_layernorm_fwd_dropout": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64,
                                          c_f32, c_f32, c_u64, c_void_p, c_i64, c_void_p]),
    "fsb_layernorm_bwd_dropout": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p, c_int, c_int, c_void_p, c_size, c_i64, c_i64,
                                          c_f32, c_u64, c_void_p, c_i64, c_void_p]),
    "fsb_rmsnorm_fwd_dropout": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_f32,
                                        c_f32, c_u64, c_void_p, c_i64, c_void_p]),
    "fsb_rmsnorm_bwd_dropout": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_int, c_int, c_void_p, c_size, c_i64, c_i64,
                                        c_f32, c_u64, c_void_p, c_i64, c_void_p]),
    "fsb_glu_fwd_dropout": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_i64,
                                    c_f32, c_u64, c_void_p, c_i64, c_void_p]),
    "fsb_glu_bwd_dropout": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64,
                                    c_i64, c_i64, c_i64, c_f32, c_u64, c_void_p, c_i64, c_void_p]),
    "fsb_dropout": (c_int, [c_void_p, c_void_p, c_i64, c_i64, c_f32, c_u64, c_void_p, c_i64, c_void_p]),
    "fsb_dropout_advance": (c_int, [c_void_p, c_void_p, c_i64, c_void_p]),
    "fsb_attn_decode_workspace_bytes": (c_size, [c_i64, c_int, c_int, c_i64]),
    "fsb_attn_decode": (c_int, [c_void_p] * 5 + [c_i64, c_int, c_int, c_i64, c_void_p] + [c_i64] * 10 +
                        [c_f32, c_void_p, c_void_p, c_void_p, c_size, c_void_p]),
    "fsb_kv_append": (c_int, [c_void_p] * 5 + [c_i64, c_int, c_int, c_i64, c_void_p] + [c_i64] * 10 + [c_void_p]),
    "fsb_kv_reorder": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_void_p, c_void_p]),
}

_lib = None
launch_count = 0  # number of fsb_* compute calls issued (bench.py reports kernel launches from this)


def load():
    """Load libfsb200.so (once). Raises RuntimeError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"fsb200: {LIB_PATH} not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C fengshen-lm_b200/csrc`). There is no CPU/PyTorch fallback for the hot path.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise RuntimeError(f"fsb200: symbol {name} missing from {LIB_PATH}; rebuild the library") from e
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error():
    return load().fsb_last_error().decode("utf-8", "replace")


def check(rc, what):
    if rc != 0:
        raise RuntimeError(f"fsb200: {what} failed (status {rc}): {last_error()}")


kernel_launches = 0  # number of __global__ launches issued by the library on behalf of this process
# kernels launched per successful entry-point call (everything not listed launches exactly one)
_NO_KERNEL = {"fsb_set_reserved_sms", "fsb_comm_unique_id", "fsb_comm_init", "fsb_comm_destroy", "fsb_comm_reduce_scatter",
              "fsb_comm_all_gather", "fsb_comm_all_reduce", "fsb_index_build_sample_idx", "fsb_index_build_mapping",
              "fsb_index_build_blocks_mapping", "fsb_index_build_blending_indices", "fsb_bert_collate"}   # host-only calls / NCCL's kernels, not ours
_KERNELS_PER_CALL = {"fsb_rmsnorm_bwd": 2, "fsb_layernorm_bwd": 2, "fsb_softmax_xent_fwd_bwd": 3, "fsb_sdpa_bwd": 3,
                     "fsb_layernorm_bwd_dropout": 2, "fsb_rmsnorm_bwd_dropout": 2,
                     "fsb_sumsq": 2, "fsb_colsum": 2, "fsb_act_bwd_bias": 2, "fsb_attn_decode": 2, "fsb_fp8_quantize": 2}


call_profiler = None  # optional: object with .add(name, ev0, ev1, work); set by bench.py --breakdown (CUDA events per call)


def call(name, *args, tag=None):
    """Invoke a status-returning entry point and raise on error. `tag` refines the profiler key (e.g. the GEMM shape)."""
    global launch_count, kernel_launches
    if name not in _NO_KERNEL:
        launch_count += 1
        kernel_launches += _KERNELS_PER_CALL.get(name, 1)
    if call_profiler is not None:
        import torch
        ev0 = torch.cuda.Event(enable_timing=True); ev0.record()
        rc = getattr(load(), name)(*args)
        ev1 = torch.cuda.Event(enable_timing=True); ev1.record()
        call_profiler.add(name if tag is None else f"{name} {tag}", ev0, ev1, 0.0)
    else:
        rc = getattr(load(), name)(*args)
    if rc != 0:
        raise RuntimeError(f"fsb200: {name} failed (status {rc}): {last_error()}")
