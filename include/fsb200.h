/* fsb200 — C ABI of libfsb200.so, the H100 (sm_90a) backend for the Fengshen data-parallel pretraining step.
 *
 * This is the drop-in boundary (SURVEY.md §8b). The reference reaches its native code through pybind11
 * torch-extension modules that take torch::Tensor (fengshen/models/megatron/fused_kernels/
 * scaled_masked_softmax.cpp:70-83, scaled_upper_triang_masked_softmax.cpp:62-70) and through third-party
 * extensions (flash_attn_cuda, deepspeed.ops.adam.FusedAdam, cuBLAS via F.linear). Every entry below names the
 * reference call site it replaces. Conventions:
 *   - plain pointers + sizes only; all pointers are DEVICE pointers unless stated; caller owns every buffer;
 *   - the library never allocates device memory and never synchronises: work is enqueued on `stream`; every scratch
 *     buffer is a caller-owned `workspace` whose size a fsb_*_workspace_bytes() query returns;
 *   - row-major tensors; "ld*" are row strides in ELEMENTS;
 *   - bf16 activations/weights, fp32 statistics / optimizer state;
 *   - return 0 on success, negative fsb_status on error; fsb_last_error() gives a thread-local message;
 *   - no silent no-ops: an unsupported shape/dtype is an error (cf. the silent `default: break` at
 *     scaled_masked_softmax.h:448 in the reference).
 */
#ifndef FSB200_H_
#define FSB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* fsb_stream_t; /* cudaStream_t */

typedef enum {
  FSB_OK = 0,
  FSB_ERR_INVALID = -1,     /* bad shape / alignment / argument */
  FSB_ERR_CUDA = -2,        /* CUDA runtime / driver error      */
  FSB_ERR_UNSUPPORTED = -3  /* valid request this build does not implement */
} fsb_status;

typedef enum { FSB_BF16 = 0, FSB_F32 = 1, FSB_U32 = 2, FSB_U64 = 3 /* index builders only */ } fsb_dtype;

/* ---- library ---------------------------------------------------------------------------------------------- */
int fsb_version(void);               /* 1000*major + minor */
const char* fsb_last_error(void);    /* thread-local, never NULL */
int fsb_num_sms(void);               /* SM count of the current device (132 on H100 SXM) */

/* ---- GEMM (wgmma + TMA) ------------------------------------------------------------------------------------
 * Replaces F.linear / torch.baddbmm / torch.bmm -> cuBLAS on the hot path:
 *   ColumnParallelLinear.forward  fengshen/models/megatron/mpu/layers.py:347-360  (Y = X W^T)
 *   RowParallelLinear.forward     fengshen/models/megatron/mpu/layers.py:451-470
 *   ParallelLinear (LM head)      fengshen/models/megatron/layers/transformer.py:136-172
 * and their autograd transposes (dgrad / wgrad).
 *
 *   FSB_GEMM_NT : D[M,N] = A[M,K] * B[N,K]^T      forward       (X W^T)
 *   FSB_GEMM_NN : D[M,N] = A[M,K] * B[K,N]        data grad     (dY W)
 *   FSB_GEMM_TN : D[M,N] = A[K,M]^T * B[K,N]      weight grad   (dY^T X)
 *
 * A, B bf16. D bf16 or fp32 (d_dtype). Optional fused epilogue, applied in this order:
 *   acc (+ bias[N]) -> activation -> (+ D_old if accumulate) -> store.
 * bias: fp32 or bf16 vector of length N (bias_dtype), may be NULL.
 * Requirements: pointers 16-byte aligned; lda/ldb/ldd multiples of 8 elements.
 * aux (bf16, may be NULL): receives acc + bias BEFORE the activation (saved for the activation's backward).
 * `batch` > 1 runs independent GEMMs with element strides stride_a/b/d between them (use 1 and 0 otherwise).
 * Kernel selection is internal: persistent 128 x 256 tiles, or 128 x 128 tiles when the wide ones would leave many SMs
 * idle. FSB_GEMM_TN calls whose output has few tiles and K >= 4096
 * (weight gradients of small models) split K: the chunks are accumulated in fp32 in the caller's `workspace`
 * (fsb_gemm_workspace_bytes(layout, M, N, K) bytes; 0 when the call does not split) and reduced in a fixed order — results
 * are deterministic; a split call with too small a workspace is an error. Other calls ignore `workspace` (may be NULL).
 * fsb_set_reserved_sms(n): persistent GEMM grids leave n SMs to communication kernels that
 * overlap them (the ZeRO engine's reduce-scatter / all-gather on the side stream); 0 restores the full grid.
 * FSB_EPI_GELU_ERF evaluates erf through Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7, below the bf16 rounding of the output).
 */
typedef enum { FSB_GEMM_NT = 0, FSB_GEMM_NN = 1, FSB_GEMM_TN = 2 } fsb_gemm_layout;
typedef enum {
  FSB_EPI_NONE = 0,
  FSB_EPI_GELU_TANH = 1, /* gelu_new / bias_gelu: layers/activations.py:60-77 */
  FSB_EPI_GELU_ERF = 2   /* erf_gelu: layers/activations.py:98-117; HF BERT hidden_act="gelu" */
} fsb_gemm_epilogue;

int fsb_gemm_bf16(int layout, int64_t M, int64_t N, int64_t K,
                  const void* A, int64_t lda, const void* B, int64_t ldb,
                  void* D, int64_t ldd, int d_dtype,
                  const void* bias, int bias_dtype, int epilogue, int accumulate,
                  void* aux, int64_t ldaux,
                  int64_t batch, int64_t stride_a, int64_t stride_b, int64_t stride_d, int64_t stride_aux,
                  void* workspace, size_t workspace_bytes, fsb_stream_t stream);
size_t fsb_gemm_workspace_bytes(int layout, int64_t M, int64_t N, int64_t K);
int fsb_set_reserved_sms(int n);

/* ---- RMSNorm / LayerNorm ------------------------------------------------------------------------------------
 * RMSNorm.forward fengshen/models/megatron/layers/norms.py:44-52 (y = scale * cast(x * rsqrt(mean(x^2) + eps)), the cast to
 * 16 bit happening BEFORE the scale multiply); LayerNorm = torch.nn.LayerNorm (norms.py:16; HF BERT/GPT-2 eps 1e-12/1e-5).
 * x, y, residual, sum_out, dy, dx, dres: bf16 [rows, cols] contiguous; cols % 8 == 0, cols <= 16384. scale/gamma/beta bf16.
 * residual != NULL fuses x_sum = x + residual (written to sum_out, which the norm then reads) — the residual adds of
 * ParallelTransformerLayer.forward (layers/transformer.py:775-788). dres != NULL fuses dx += dres in backward.
 * stats: fp32 [rows] (rstd) for RMSNorm, [rows][2] (mean, rstd) for LayerNorm. Weight gradients (bf16 or fp32 per
 * wgrad_dtype, optionally accumulated) are reduced deterministically through `workspace` (fsb_norm_bwd_workspace_bytes). */
size_t fsb_norm_bwd_workspace_bytes(int64_t rows, int64_t cols, int is_layernorm);
int fsb_rmsnorm_fwd(const void* x, const void* residual, const void* scale, void* y, void* sum_out, float* rstd,
                    int64_t rows, int64_t cols, float eps, fsb_stream_t stream);
int fsb_rmsnorm_bwd(const void* dy, const void* x, const void* scale, const float* rstd, const void* dres, void* dx,
                    void* dscale, int wgrad_dtype, int accumulate, void* workspace, size_t workspace_bytes,
                    int64_t rows, int64_t cols, fsb_stream_t stream);
int fsb_layernorm_fwd(const void* x, const void* residual, const void* gamma, const void* beta, void* y, void* sum_out,
                      float* mean_rstd, int64_t rows, int64_t cols, float eps, fsb_stream_t stream);
int fsb_layernorm_bwd(const void* dy, const void* x, const void* gamma, const float* mean_rstd, const void* dres,
                      void* dx, void* dgamma, void* dbeta, int wgrad_dtype, int accumulate, void* workspace,
                      size_t workspace_bytes, int64_t rows, int64_t cols, fsb_stream_t stream);

/* ---- rotary embedding, in place -----------------------------------------------------------------------------
 * apply_rotary_pos_emb / rotate_half, layers/positional_embeddings.py:71-87, applied to one of {q, k} inside the packed QKV
 * projection output (layers/transformer.py:488-523): head h of row t starts at x + t*row_stride + h*head_stride.
 * cos/sin: fp32 [max_pos, head_dim/2] (RotaryEmbedding cache, positional_embeddings.py:38-52); positions int64 [rows].
 * backward != 0 applies the transposed rotation (gradient). head_dim % 16 == 0. A position outside [0, max_pos) never
 * reads outside the tables: its row is filled with NaN (the reference regrows the cache instead, :54-68 — the host
 * wrapper sizes the tables to the sequence and validates position_ids). */
int fsb_rope_inplace(void* x, const float* cos_table, const float* sin_table, const int64_t* positions, int64_t rows,
                     int nheads, int head_dim, int64_t row_stride, int64_t head_stride, int64_t max_pos, int backward,
                     fsb_stream_t stream);

/* ---- gated / plain activations ------------------------------------------------------------------------------
 * act: 0 SiLU (LLaMAParallelMLP.forward layers/transformer.py:620-623: silu(w1 x) * w3 x), 1 tanh-GeLU (gelu_new /
 * bias_gelu layers/activations.py:60-94; MT5DenseGatedActDense), 2 erf-GeLU (activations.py:98-117; BERT).
 * glu: out[t,c] = act(gate[t,c]) * up[t,c] with independent row strides (gate|up are column halves of one GEMM output). */
int fsb_glu_fwd(int act, const void* gate, const void* up, void* out, int64_t rows, int64_t cols, int64_t ld_gate,
                int64_t ld_up, int64_t ld_out, fsb_stream_t stream);
int fsb_glu_bwd(int act, const void* dout, const void* gate, const void* up, void* dgate, void* dup, int64_t rows,
                int64_t cols, int64_t ld_dout, int64_t ld_gate, int64_t ld_up, int64_t ld_dgate, int64_t ld_dup,
                fsb_stream_t stream);
int fsb_act_fwd(int act, const void* x, void* y, int64_t n, fsb_stream_t stream);
int fsb_act_bwd(int act, const void* dy, const void* x, void* dx, int64_t n, fsb_stream_t stream);
/* dx = dy * act'(x) over contiguous [rows, cols] AND dbias[c] (+)= sum_r dx[r,c] in the same pass: the bias gradient of the
 * linear layer that produced x (HF GPT2MLP c_fc / BertIntermediate.dense) without a second pass over dx. act 1..3;
 * workspace: fsb_act_bwd_bias_workspace_bytes(rows, cols). Deterministic. */
size_t fsb_act_bwd_bias_workspace_bytes(int64_t rows, int64_t cols);
int fsb_act_bwd_bias(int act, const void* dy, const void* x, void* dx, int64_t rows, int64_t cols, void* dbias,
                     int dbias_dtype, int accumulate, void* workspace, size_t workspace_bytes, fsb_stream_t stream);
int fsb_add(const void* a, const void* b, void* out, int64_t n, fsb_stream_t stream);            /* bf16, n % 8 == 0 */
/* x (bf16, n % 8 == 0) *= *scale_dev; a no-op launch when the device scalar is 1 (upstream gradient of the loss) */
int fsb_scale_inplace(void* x, int64_t n, const float* scale_dev, fsb_stream_t stream);
/* acc (fp32) = (overwrite ? 0 : acc) + scale * x (bf16): ZeRO-2 per-micro-step gradient accumulation into the fp32 shard */
int fsb_accumulate(float* acc, const void* x, int64_t n, float scale, int overwrite, fsb_stream_t stream);
/* out[c] (+)= sum_r x[r,c]  (bias gradients; learned-position gradient as [B, S*h] column sum); deterministic */
size_t fsb_colsum_workspace_bytes(int64_t rows, int64_t cols);
int fsb_colsum(const void* x, int64_t rows, int64_t cols, int64_t ld, void* out, int out_dtype, int accumulate,
               void* workspace, size_t workspace_bytes, fsb_stream_t stream);

/* ---- embedding ----------------------------------------------------------------------------------------------
 * VocabParallelEmbedding.forward fengshen/models/megatron/mpu/layers.py:104-130 (TP = 1): out[t] = W[ids[t]]
 * (+ P[pos[t]] learned positions, pos == NULL -> t % seq_len; + T[token_type[t]]) — HF BertEmbeddings / GPT-2 wte + wpe.
 * Backward: fsb_embedding_bwd_sorted is the deterministic form — `ids_sorted` (ascending, stable) and `order` (token index of
 * each sorted position) come from a sort of the ids; every distinct id's rows are summed in fp32 in a fixed order and added
 * onto dW[id] with ONE bf16 rounding (torch's embedding backward, which the reference runs, accumulates in fp32 too).
 * fsb_embedding_bwd scatter-adds with bf16x2 atomics (kept for ids == NULL -> row t % idx_mod, learned positions).
 * fsb_cast_f32_to_bf16: out = bf16(in), n % 8 == 0 (fp32 gradient accumulators handed back to bf16 kernels). */
int fsb_embedding_fwd(const int64_t* ids, const int64_t* pos, const int64_t* token_type, const void* W, const void* P,
                      const void* T, void* out, int64_t rows, int64_t cols, int64_t seq_len, fsb_stream_t stream);
int fsb_embedding_bwd(const int64_t* ids, const void* dout, void* dW, int64_t rows, int64_t cols, int64_t idx_mod,
                      fsb_stream_t stream);
int fsb_embedding_bwd_sorted(const int64_t* ids_sorted, const int64_t* order, const void* dout, void* dW, int64_t rows,
                             int64_t cols, fsb_stream_t stream);
int fsb_cast_f32_to_bf16(const float* in, void* out, int64_t n, fsb_stream_t stream);

/* ---- fused softmax cross-entropy, forward + backward ----------------------------------------------------------
 * torch.nn.CrossEntropyLoss()(shift_logits, shift_labels), fengshen/models/llama/modeling_llama.py:334-339: mean NLL over
 * labels != ignore_index. Row t = (b, s) uses labels[t + shift] and is ignored when s + shift >= seq_len (the
 * shift-by-one without the `.contiguous()` copy of :336). logits bf16 [rows, vocab] (row stride ld); dlogits (may alias
 * logits, may be NULL) receives (softmax - onehot) * grad_scale / n_valid. row_loss fp32 [rows], loss fp32 [1],
 * n_valid int32 [1] are device outputs (token-id side is bit-exact: n_valid and the one-hot index). */
int fsb_softmax_xent_fwd_bwd(const void* logits, const int64_t* labels, void* dlogits, float* row_loss, float* loss,
                             int* n_valid, int64_t rows, int64_t vocab, int64_t ld, int64_t seq_len, int shift,
                             int ignore_index, float grad_scale, fsb_stream_t stream);

/* ---- flat-shard AdamW, gradient norm, clip ------------------------------------------------------------------
 * deepspeed.ops.adam.FusedAdam(adam_w_mode=True) as selected at fengshen/models/model_utils.py:69-72, in
 * torch.optim.AdamW's operation order, on the rank's flat fp32 shard {master, exp_avg, exp_avg_sq}; grad bf16 or fp32;
 * param16 (bf16, may be NULL) receives the updated parameters. grad_scale: optional DEVICE scalar multiplied into the
 * gradient (clip coefficient). n % 4 == 0. fsb_sumsq / fsb_clip_coef give torch.nn.utils.clip_grad_norm_ semantics.
 * hyper: optional DEVICE array {lr, 1 - beta1^t, sqrt(1 - beta2^t)} that overrides `lr` / `step` — the per-step scalars then
 * live in device memory and the launch is byte-identical every step, which is what lets a whole training step be captured
 * in a CUDA graph and replayed (fsb200.trainer.PretrainStep(cuda_graph=True)). */
int fsb_adamw_flat(float* master, float* exp_avg, float* exp_avg_sq, const void* grad, int grad_dtype, void* param16,
                   int64_t n, float lr, float beta1, float beta2, float eps, float weight_decay, int64_t step,
                   const float* grad_scale, const float* hyper, fsb_stream_t stream);
size_t fsb_sumsq_workspace_bytes(void);
int fsb_sumsq(const void* x, int dtype, int64_t n, float* out, int accumulate, void* workspace, size_t workspace_bytes,
              fsb_stream_t stream);
int fsb_clip_coef(const float* sumsq, float max_norm, float* coef, float* norm_out, fsb_stream_t stream);

/* ---- the reference's own two CUDA ops (legacy non-flash attention path) -------------------------------------
 * scaled_masked_softmax_cuda.{forward, backward, get_batch_per_block}  fused_kernels/scaled_masked_softmax.cpp:70-83
 *   forward : y = softmax(mask == 1 ? -10000 : scale * x) over sk; x, y bf16 [batches, attn_heads, sq, sk];
 *             mask uint8 [mask_batches (1 or batches), 1, sq, sk] or NULL (scaled_masked_softmax.h:117-238).
 *   backward: dy <- scale * (dy*y - y*sum(dy*y)) IN PLACE (scaled_masked_softmax_cuda.cu:95-105); rows = b*np*sq.
 * scaled_upper_triang_masked_softmax_cuda.{forward, backward}          scaled_upper_triang_masked_softmax.cpp:62-70
 *   causal variant on [attn_batches, seq_len, seq_len]; zeros above the diagonal.
 * sk % 8 == 0, sk <= 4096 (the reference asserts sk <= 2048 and silently skips unsupported sizes, .h:448; here any
 * violation is an error). fsb_softmax_get_batch_per_block reproduces the reference's launch-geometry helper that
 * layers/fused_softmax.py:163-170 uses to gate the fused path. */
int fsb_scaled_masked_softmax_fwd(const void* x, const uint8_t* mask, void* y, int64_t batches, int64_t attn_heads,
                                  int64_t sq, int64_t sk, int64_t mask_batches, float scale, fsb_stream_t stream);
int fsb_scaled_masked_softmax_bwd(void* dy_inplace, const void* y, int64_t rows, int64_t sk, float scale,
                                  fsb_stream_t stream);
int fsb_scaled_upper_triang_masked_softmax_fwd(const void* x, void* y, int64_t attn_batches, int64_t seq_len,
                                               float scale, fsb_stream_t stream);
int fsb_scaled_upper_triang_masked_softmax_bwd(void* dy_inplace, const void* y, int64_t attn_batches, int64_t seq_len,
                                               float scale, fsb_stream_t stream);
int fsb_softmax_get_batch_per_block(int64_t sq, int64_t sk, int64_t batches, int64_t attn_heads);

/* ---- fused scaled-dot-product attention (wgmma, flash-style online softmax) ----------------------------------
 * Replaces ParallelSelfAttention.flash_attention (fengshen/models/megatron/layers/transformer.py:410-456; 3P
 * flash_attn_cuda.fwd/bwd, layers/flash_attention.py:31-47,81-101) and the legacy baddbmm -> FusedScaleMaskSoftmax ->
 * bmm path (transformer.py:307-408). q/k/v are read in place from the packed QKV projection output:
 *   element (b, s, head, d) of X lives at X + ((b*seq + s)*x_row_stride + head*x_head_stride + d)  (elements).
 * o: same addressing with o_*_stride. lse: fp32 [batch, nheads, seq_q], log2 domain (internal, consumed by bwd).
 * kv_mask: optional uint8 [batch, seq_kv], 1 = attend (HF additive padding mask), NULL = none.
 * causal=1 masks key > query (requires seq_q == seq_kv). head_dim in {64, 128}.
 * rel_bias: optional fp32 [nheads, seq_q + seq_kv - 1], natural-log units, added to scale * q.k before the softmax:
 *   bias(h, q, k) = rel_bias[h][k - q + seq_q - 1]  — the T5 / mT5 relative-position bias (transformers
 *   mt5/modeling_mt5.py:181-235,:320: an embedding over bucket(k - q), shared by every layer of a stack), used by
 *   fengshen/examples/pretrain_t5/pretrain_t5.py:57-59 (scale = 1: T5 attention is unscaled, :300). NULL = none.
 */
int fsb_sdpa_fwd(const void* q, const void* k, const void* v, void* o, float* lse,
                 int64_t batch, int64_t seq_q, int64_t seq_kv, int nheads, int head_dim,
                 int64_t q_row_stride, int64_t k_row_stride, int64_t v_row_stride, int64_t o_row_stride,
                 int64_t q_head_stride, int64_t k_head_stride, int64_t v_head_stride, int64_t o_head_stride,
                 float scale, int causal, const uint8_t* kv_mask, const float* rel_bias, fsb_stream_t stream);

/* Backward of fsb_sdpa_fwd. o/lse are the forward outputs; delta: fp32 scratch [batch, nheads, seq_q] (written here);
 * dq/dk/dv are written with their own strides (e.g. the three slices of a packed dQKV buffer). Deterministic.
 * rel_bias as in the forward; drel_bias (fp32 [nheads, seq_q + seq_kv - 1], may be NULL) is ACCUMULATED into:
 *   drel_bias[h][r] += sum over (batch, q) of dS[q, q + r - (seq_q - 1)]   (gradient w.r.t. the bias vector; the
 * [buckets, heads] table gradient is its scatter over bucket(r), autograd of T5Attention.compute_bias). It needs a workspace of
 * fsb_sdpa_bwd_workspace_bytes(batch, seq_q, seq_kv, nheads) bytes: per-step diagonal sums written by the dQ kernel and
 * reduced in a fixed order (no atomics). */
size_t fsb_sdpa_bwd_workspace_bytes(int64_t batch, int64_t seq_q, int64_t seq_kv, int nheads);
int fsb_sdpa_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout,
                 const float* lse, float* delta, void* dq, void* dk, void* dv,
                 int64_t batch, int64_t seq_q, int64_t seq_kv, int nheads, int head_dim,
                 int64_t q_row_stride, int64_t k_row_stride, int64_t v_row_stride, int64_t o_row_stride,
                 int64_t do_row_stride, int64_t dq_row_stride, int64_t dk_row_stride, int64_t dv_row_stride,
                 int64_t q_head_stride, int64_t k_head_stride, int64_t v_head_stride, int64_t o_head_stride,
                 int64_t do_head_stride, int64_t dq_head_stride, int64_t dk_head_stride, int64_t dv_head_stride,
                 float scale, int causal, const uint8_t* kv_mask, const float* rel_bias, float* drel_bias,
                 void* workspace, size_t workspace_bytes, fsb_stream_t stream);

/* ---- communication (NCCL over NVLink / NVSwitch) --------------------------------------------------------------
 * The three exchange steps of the ZeRO-1/2 data path (SURVEY.md §8e) — the collectives the reference delegates to DeepSpeed
 * (fengshen/strategies/megatron_deepspeed.py:302-320; Appendix D): bucketed gradient reduce-scatter (SUM), the fp32 scalar
 * all-reduce of the squared gradient norm, and the in-place parameter all-gather. One communicator per process (= per GPU);
 * rank 0 creates the 128-byte id with fsb_comm_unique_id and the host distributes it out of band (MPI, a file, a TCP store).
 * All calls are asynchronous on `stream` (the engine issues them on a dedicated side stream, fenced with events against
 * the compute stream). In-place forms are allowed where NCCL allows them (all_gather: send == recv + rank * send_count).
 * NCCL is loaded at run time (dlopen "libnccl.so.2"); if it is absent every fsb_comm_* call fails with FSB_ERR_INVALID. */
typedef void* fsb_comm_t;
int fsb_comm_unique_id(void* id128);
int fsb_comm_init(fsb_comm_t* comm, const void* id128, int world, int rank);
int fsb_comm_destroy(fsb_comm_t comm);
int fsb_comm_reduce_scatter(fsb_comm_t comm, const void* send, void* recv, int64_t recv_count, int dtype, fsb_stream_t stream);
int fsb_comm_all_gather(fsb_comm_t comm, const void* send, void* recv, int64_t send_count, int dtype, fsb_stream_t stream);
int fsb_comm_all_reduce(fsb_comm_t comm, const void* send, void* recv, int64_t count, int dtype, fsb_stream_t stream);

/* ---- index builders of the Megatron indexed datasets (HOST functions: no device, no stream) -----------------------
 * Replace the pybind11 module `helpers` (fengshen/data/megatron_dataloader/helpers.cpp:788-793, built by its Makefile:1-9 and
 * called from blendable_dataset.py:51 and dataset_utils.py). Integer outputs are bit-identical to the reference's, including its
 * pseudo-random sequence (std::mt19937(seed) for the short-sequence draws, std::mt19937_64(seed + 1) for the row shuffle), so
 * an index cached by one implementation is valid for the other. All arrays are caller-owned, C-contiguous.
 *
 * fsb_index_build_sample_idx  (helpers.cpp:101-195): GPT-style flattened stream. sizes[doc] = tokens per document, doc_idx
 *   [n_doc_idx] = document order over all epochs. out: int32 [num_samples + 1, 2] rows (index into doc_idx, token offset), with
 *   num_samples = (num_epochs * tokens_per_epoch - 1) / seq_length and out_rows == num_samples + 1.
 * fsb_index_build_mapping     (helpers.cpp:213-516): BERT-style sentence spans. docs[n_docs + 1] = first sentence of each
 *   document, sizes[sentence] = tokens. Rows (first sentence, end sentence, target length), dtype FSB_U32 or FSB_U64 (the
 *   reference switches to uint64 when there are more than 2^32-1 sentences). Call with out == NULL to get the row count, then
 *   with out_rows == that count; the filled rows are shuffled. Returns the row count, or -1 with fsb_last_error() set.
 * fsb_index_build_blocks_mapping (helpers.cpp:518-786): as above with a per-document title length subtracted from the target and
 *   rows (first sentence, end sentence, document, block id within the epoch).
 * fsb_index_build_blending_indices (helpers.cpp:34-99): for `size` samples pick, greedily, the dataset whose sample count lags
 *   its weight the most; dataset_index uint8 [size], dataset_sample_index int64 [size]. */
int fsb_index_build_sample_idx(const int32_t* sizes, const int32_t* doc_idx, int64_t n_doc_idx, int32_t seq_length,
                               int32_t num_epochs, int64_t tokens_per_epoch, int32_t* out, int64_t out_rows);
int64_t fsb_index_build_mapping(const int64_t* docs, int64_t n_docs, const int32_t* sizes, int32_t num_epochs,
                                uint64_t max_num_samples, int32_t max_seq_length, double short_seq_prob, int32_t seed,
                                int32_t min_num_sent, int dtype, void* out, int64_t out_rows);
int64_t fsb_index_build_blocks_mapping(const int64_t* docs, int64_t n_docs, const int32_t* sizes, const int32_t* titles_sizes,
                                       int32_t num_epochs, uint64_t max_num_samples, int32_t max_seq_length, int32_t seed,
                                       int use_one_sent_blocks, int dtype, void* out, int64_t out_rows);
int fsb_index_build_blending_indices(uint8_t* dataset_index, int64_t* dataset_sample_index, const double* weights,
                                     int32_t num_datasets, int64_t size);

/* ---- MegatronBERT sample assembly (HOST function) --------------------------------------------------------------------
 * The per-document work of `ErLangShenCollator` (fengshen/examples/pretrain_erlangshen_bert/pretrain_erlangshen.py:57-123 ->
 * data_utils/sop_utils.py:2-32, truncate_utils.py:2-19, token_type_utils.py:1-25, mask_utils.py:19-285 with its defaults:
 * whole-word n-gram masking, 'bert' style) over a batch of TOKENISED documents:
 *   tokens[sent_offsets[s] .. sent_offsets[s+1]) is sentence s; document d holds sentences [doc_offsets[d], doc_offsets[d+1]).
 * continuation[id] != 0 marks WordPiece continuation pieces ("##..."); vocab_ids[n_vocab_ids] is the list random replacements are
 * drawn from; ngram_cdf[max_ngrams] the normalised cumulative weights of n-gram sizes 1..max_ngrams as numpy computes them
 * (cumsum(p) / cumsum(p)[-1] with p ~ 1/n).
 * mt_key[624] / mt_pos are numpy's legacy MT19937 state (`RandomState.get_state()[1:3]`), read and UPDATED: the rows and the state
 * left behind are bit-identical to running the Python collator on the same generator.
 * Outputs are int64 [n_docs, max_seq_length] (next_sentence_label: [n_docs]); documents that yield no sample (no sentence, empty
 * first segment) are skipped, the return value is the number of rows written (-1 + fsb_last_error() on a bad argument). */
int64_t fsb_bert_collate(const int32_t* tokens, const int64_t* sent_offsets, const int64_t* doc_offsets, int64_t n_docs,
                         const uint8_t* continuation, int64_t vocab_table_len, const int32_t* vocab_ids, int64_t n_vocab_ids,
                         int32_t cls_id, int32_t sep_id, int32_t mask_id, int32_t pad_id, int32_t max_seq_length,
                         double masked_lm_prob, const double* ngram_cdf, int32_t max_ngrams, uint32_t* mt_key, int32_t* mt_pos,
                         int64_t* input_ids, int64_t* attention_mask, int64_t* token_type_ids, int64_t* labels,
                         int64_t* next_sentence_label);

#ifdef __cplusplus
}
#endif
#endif /* FSB200_H_ */
