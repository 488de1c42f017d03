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
 * Requirements: pointers 16-byte aligned; lda/ldb/ldd multiples of 8 elements; N a multiple of 8 (of 4 for an fp32 D
 * without aux): D and aux are stored in whole 16-byte chunks, so a row may not end inside one. M and K are free.
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

/* ---- int8 weight-only inference (W8A16) ------------------------------------------------------------------------
 * Stand in for `from_pretrained(..., load_in_8bit=True)` (fengshen/examples/ziya_inference/hf_quantizatin_inference.py:20-22),
 * whose Linear layers bitsandbytes replaces with Linear8bitLt (third party). Weight-only: activations stay bf16, there is
 * no outlier decomposition, so results are not bit-comparable with bitsandbytes.
 *
 * fsb_quantize_w8: symmetric per-output-channel quantisation of W bf16 [n, k] (row stride ldw >= k):
 *   s[r] = absmax(W[r, :]) / 127.0f (IEEE fp32 division); q[r, c] = clamp(rint(W[r, c] / s[r]), -127, 127), rint rounding
 *   half to even, the division IEEE fp32. A zero row gives s = 0, q = 0. q: int8 [n, k] row-major contiguous; s: fp32 [n].
 * fsb_gemm_w8a16: D[m, n] = bf16(s[n] * sum_k A[m, k] q[n, k]), fp32 accumulation. A bf16 [m, k] (row stride lda), q / s as
 *   fsb_quantize_w8 writes them, D bf16 [m, n] (row stride ldd); rows of D at or beyond m and columns beyond n are not
 *   written. Requirements: k % 16 == 0, n % 8 == 0, lda >= k and ldd >= n multiples of 8, a / q / s / d 16-byte aligned.
 *   Any m >= 1; one kernel serves decode (m of 1-32) and prefill. Calls whose output tiles leave SMs idle split K: fp32
 *   partials go to the caller's `workspace` (fsb_gemm_w8a16_workspace_bytes(m, n, k) bytes, 0 when the call does not split)
 *   and are summed in a fixed order. The plan depends on (m, n, k) and the SM count only: results are deterministic. A
 *   split call with too small a workspace is an error. */
int fsb_quantize_w8(const void* w, int64_t ldw, int64_t n, int64_t k, int8_t* q, float* s, fsb_stream_t stream);
size_t fsb_gemm_w8a16_workspace_bytes(int64_t m, int64_t n, int64_t k);
int fsb_gemm_w8a16(int64_t m, int64_t n, int64_t k, const void* a, int64_t lda, const int8_t* q, const float* s,
                   void* d, int64_t ldd, void* workspace, size_t workspace_bytes, fsb_stream_t stream);

/* ---- int4 weight-only inference (W4A16) ------------------------------------------------------------------------
 * Stand in for `from_pretrained(..., load_in_4bit=True)` (fengshen/examples/ziya_inference/hf_quantizatin_inference.py:3,16).
 * Symmetric round-to-nearest with one scale per output row and group of 128 consecutive k, no calibration and no zero
 * point: results are not bit-comparable with bitsandbytes NF4/FP4 or llama.cpp q4_*.
 *
 * fsb_quantize_w4: W bf16 [n, k] (row stride ldw >= k). For row r and group g (columns 128g .. 128g + 127):
 *   a = absmax(W[r, group]) over the fp32 values; s[r, g] = bf16_rne(a / 7.0f), the division IEEE fp32;
 *   q[r, c] = clamp(rint(W[r, c] / float(s[r, g])), -7, 7), rint rounding half to even, the division IEEE fp32; where
 *   s == 0 (a zero group, or an underflow) q = 0. The dequantised weight is W^[r, c] = bf16_rne(q[r, c] * s[r, g]), the
 *   exact product rounded once.
 *   s: bf16 [n, k / 128] row-major contiguous.
 *   q: n * k / 2 bytes, packed as [n / 2, k] bytes, row-major contiguous. Byte line p holds rows 2p and 2p + 1: row 2p in
 *   the low nibble, row 2p + 1 in the high nibble, each as the 4-bit code q + 8 (1 .. 15). Along the line, k runs in blocks
 *   of 16; inside block j (bytes 16j .. 16j + 15) the byte at 16j + 4t + 2b + h (t < 4, b < 2, h < 2) holds
 *   k = 16j + 8h + 2t + b. Each 32-bit word is then one thread's wgmma register-A fragment for one k16 step.
 *   Requirements: k % 128 == 0, n % 8 == 0, w 2-byte, q 4-byte and s 2-byte aligned. fsb_quantize_w4 is the only writer of
 *   this layout.
 * fsb_gemm_w4a16: D[m, n] = bf16(sum_k A[m, k] W^[n, k]), fp32 accumulation. A bf16 [m, k] (row stride lda), q / s as
 *   fsb_quantize_w4 writes them, D bf16 [m, n] (row stride ldd). Requirements: k % 128 == 0 and otherwise as fsb_gemm_w8a16
 *   (n % 8 == 0, lda >= k and ldd >= n multiples of 8, a / q / s / d 16-byte aligned). Tiles, K-split plan, workspace
 *   (fsb_gemm_w4a16_workspace_bytes) and determinism as fsb_gemm_w8a16. */
int fsb_quantize_w4(const void* w, int64_t ldw, int64_t n, int64_t k, uint8_t* q, void* s, fsb_stream_t stream);
size_t fsb_gemm_w4a16_workspace_bytes(int64_t m, int64_t n, int64_t k);
int fsb_gemm_w4a16(int64_t m, int64_t n, int64_t k, const void* a, int64_t lda, const uint8_t* q, const void* s,
                   void* d, int64_t ldd, void* workspace, size_t workspace_bytes, fsb_stream_t stream);

/* ---- weight-only GEMMs with a bias / GELU epilogue (int8 / int4 GPT-2: Conv1D projections carry a bias) ----------
 * fsb_gemm_w8a16_bias: D[m, n] = bf16(act(s[n] * sum_k A[m, k] q[n, k] + bias[n])).
 * fsb_gemm_w4a16_bias: D[m, n] = bf16(act(sum_k A[m, k] W^[n, k] + bias[n])).
 *   fp32 throughout: the sum (times s[n] for int8), + bias[n], then act, rounded once to bf16 — the order of
 *   fsb_gemm_bf16's epilogue. bias: bf16 [n], non-NULL, 16-byte aligned. epilogue: FSB_EPI_NONE (act = identity) or
 *   FSB_EPI_GELU_TANH (act = gelu_new, fsb_gemm_bf16's device code: the same fp32 pre-activation gives the same bits);
 *   anything else is an error. Operands, requirements, plan and workspace (fsb_gemm_w8a16_workspace_bytes /
 *   fsb_gemm_w4a16_workspace_bytes) as fsb_gemm_w8a16 / fsb_gemm_w4a16. A call that splits K sums the fp32 partials in
 *   order first and applies scale, bias and act once per element after. */
int fsb_gemm_w8a16_bias(int64_t m, int64_t n, int64_t k, const void* a, int64_t lda, const int8_t* q, const float* s,
                        const void* bias, int epilogue, void* d, int64_t ldd, void* workspace, size_t workspace_bytes,
                        fsb_stream_t stream);
int fsb_gemm_w4a16_bias(int64_t m, int64_t n, int64_t k, const void* a, int64_t lda, const uint8_t* q, const void* s,
                        const void* bias, int epilogue, void* d, int64_t ldd, void* workspace, size_t workspace_bytes,
                        fsb_stream_t stream);

/* ---- FP8 training GEMM (opt-in `fp8=True`: LLaMA, BERT, MegatronBERT, mT5, GPT-2) -----------------------------------
 * The "hybrid" recipe with just-in-time ("current") per-tensor scaling: activations and weights are e4m3 (largest finite
 * value 448), gradients e5m2 (57344); accumulation is fp32, outputs bf16.
 *
 * fsb_fp8_quantize: x bf16 [rows, cols] (row stride ldx >= cols, a multiple of 8) -> FP8 codes in format `fmt`.
 *   amax = max |x| over the whole tensor, written to the caller's device fp32 scalar `amax` (scratch and output).
 *   scale = 2^e with e = floor(log2(fmax / amax)) clamped to [-126, 126], so that scale and 1 / scale are normal fp32 numbers;
 *   amax == 0 gives scale = 1. code = cvt.rn.satfinite(x * scale): round to nearest even, magnitudes beyond fmax (and inf)
 *   saturate to +-fmax, NaN stays NaN. scale_inv = 1 / scale, except when amax is not finite (a NaN or inf in x): then
 *   scale_inv = NaN, so everything computed from the codes is NaN rather than a clipped finite value.
 *   Outputs, each optional (NULL: not written): y uint8 [rows, cols] row-major contiguous; yt uint8 [cols, rows], the
 *   transposed codes, contiguous; scale_inv one device fp32. Requirements: rows % 16 == 0 and cols % 16 == 0 (both layouts
 *   need 16-byte row strides for TMA), x / y / yt 16-byte aligned. Two kernel launches (amax, then cast and transpose) after
 *   an asynchronous clear of amax; deterministic (the maximum does not depend on order).
 * fsb_gemm_fp8: D[m, n] = bf16((sum_k A[m, k] B[n, k]) * a_scale_inv * b_scale_inv), the product accumulated in fp32 and
 *   promoted into a separate fp32 accumulator after every 128 k; with `accumulate`, D[m, n] = bf16(that fp32 value + D[m, n])
 *   with one rounding. The epilogue is fsb_gemm_bf16's, in the same order:
 *     acc * a_scale_inv * b_scale_inv (+ bias[n]) -> aux = bf16(that value) -> activation -> (+ D_old if accumulate) -> store,
 *   with one rounding of D. bias: bf16 [n], may be NULL. epilogue: FSB_EPI_NONE / FSB_EPI_GELU_TANH / FSB_EPI_GELU_ERF,
 *   evaluated with fsb_gemm_bf16's device code (the same fp32 pre-activation gives the same bits). aux: bf16 [m, n] with row
 *   stride ldaux, may be NULL; receives the pre-activation. A uint8 codes [m, k] and B uint8 codes [n, k], both contiguous (K-major), as fsb_fp8_quantize writes y
 *   or yt; a_scale_inv / b_scale_inv: device fp32 scalars (read by the kernel, so a captured graph stays valid). Format pairs
 *   (a_fmt, b_fmt): (E4M3, E4M3) forward, (E5M2, E4M3) data and weight gradients; any other pair is an error.
 *   D bf16 [m, n], row stride ldd >= n a multiple of 8. Requirements: k % 16 == 0, n % 8 == 0, a / b / d / bias / aux
 *   16-byte aligned, ldaux >= n a multiple of 8;
 *   any m >= 1; rows of D at or beyond m and columns beyond n are not written. Persistent 128 x 128 tiles on the SMs that
 *   fsb_set_reserved_sms leaves to GEMMs, no K-split: deterministic (the result does not depend on the grid).
 * fsb_gemm_fp8_t: D[n, m] (+)= bf16((sum_k A[m, k] B[n, k]) * a_scale_inv * b_scale_inv), the transpose of what fsb_gemm_fp8
 *   writes for the same operands, bit for bit (same main loop, promotion, tile schedule and device-memory scales; with
 *   `accumulate`, the fp32 sum with the old D[n, m] is rounded once). It is the weight gradient of a GPT-2 Conv1D, whose
 *   weight is stored [in, out]: D = dW = x^T dy = (dy^T x)^T from A = dy^T, e5m2 codes [out, tokens], and B = x^T, e4m3
 *   codes [in, tokens]. Only the pair (a_fmt, b_fmt) = (E5M2, E4M3); bias and aux must be NULL and epilogue FSB_EPI_NONE
 *   (ldaux is ignored); anything else is an error. D bf16 [n, m], row stride ldd >= m a multiple of 8, so m % 8 == 0; any
 *   n >= 1 (fsb_gemm_fp8's bounds swapped). k % 16 == 0, a / b / d 16-byte aligned. Ragged tile edges on both axes are
 *   clipped: nothing outside D[:n, :m] of the strided view is read or written. */
typedef enum { FSB_FP8_E4M3 = 0, FSB_FP8_E5M2 = 1 } fsb_fp8_format;
int fsb_fp8_quantize(const void* x, int64_t ldx, int64_t rows, int64_t cols, int fmt, void* y, void* yt, float* scale_inv,
                     float* amax, fsb_stream_t stream);
int fsb_gemm_fp8(int64_t m, int64_t n, int64_t k, const void* a, int a_fmt, const float* a_scale_inv, const void* b,
                 int b_fmt, const float* b_scale_inv, void* d, int64_t ldd, const void* bias, int epilogue, int accumulate,
                 void* aux, int64_t ldaux, fsb_stream_t stream);
int fsb_gemm_fp8_t(int64_t m, int64_t n, int64_t k, const void* a, int a_fmt, const float* a_scale_inv, const void* b,
                   int b_fmt, const float* b_scale_inv, void* d, int64_t ldd, const void* bias, int epilogue, int accumulate,
                   void* aux, int64_t ldaux, fsb_stream_t stream);

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
 * logits, may be NULL) receives (softmax - onehot) * grad_scale / n_valid as bf16 [rows, vocab] with the SAME row stride ld
 * (an ignored row gets zeros): a separate dlogits must span (rows - 1) * ld + vocab elements. row_loss fp32 [rows], loss fp32 [1],
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
 * causal=1 masks key > query (requires seq_q == seq_kv); the key / query tiles wholly above the diagonal are skipped.
 * rel_bias: optional fp32 [nheads, seq_q + seq_kv - 1], natural-log units, added to scale * q.k before the softmax:
 *   bias(h, q, k) = rel_bias[h][k - q + seq_q - 1]  — the T5 / mT5 relative-position bias (transformers
 *   mt5/modeling_mt5.py:181-235,:320: an embedding over bucket(k - q), shared by every layer of a stack), used by
 *   fengshen/examples/pretrain_t5/pretrain_t5.py:57-59 (scale = 1: T5 attention is unscaled, :300). NULL = none.
 * seg_start / seg_end, q_start / q_end: segment bounds of packed rows (below); all NULL = unsegmented.
 * p, seed, stream_base, site: dropout on the attention probabilities (the dropout section), O = (P * Z / (1 - p)) V; the
 *   LSE is that of the un-dropped P, the backward's delta is unchanged. p == 0 runs the dropout-free kernels and does not
 *   read stream_base. Z of an element is a function of its row-relative (q, k) only, so it is the same whichever tiles a
 *   launch visits: the tiles that the causal rule or the segment bounds skip draw no bit another element needs, and a
 *   masked element has P = 0 whatever its bit. The backward must get the forward's seed, stream_base value and site.
 *
 * The arguments select the form, and with it the kernels (p composes with every form):
 *   form                    selected by                          head_dim                     causal kv_mask  rel_bias seq_q, seq_kv
 *   dense                   no bounds                            64, 128; 96 causal, no bias  0 / 1  optional optional equal if causal
 *   causal segments         seg_*, causal = 1, no rel_bias, q_*  64, 96, 128 (p > 0: 64, 96)  1      -        -        equal
 *   bidirectional segments  seg_*, causal = 0, no rel_bias, q_*  64                           0      -        -        equal
 *   biased segments         seg_* + rel_bias                     64                           0 / 1  -        required equal
 *   cross segments          seg_* + q_start / q_end              64                           0      -        -        may differ
 * head_dim 96 is GPT-2 3.5B's (32 heads x 96): the kernels stage 128 columns and store 96.
 * With p > 0 every form refuses sequences longer than 65536. Refused as well: only one of seg_start / seg_end or of
 * q_start / q_end, q_* without seg_*, and a kv_mask with segment bounds.
 *
 * Segment bounds: int32 arrays, contiguous, indices relative to the row. Self-attention (seq_q == seq_kv), two [batch, seq]:
 *   seg_start[b][t] : the position of the first token of t's segment;
 *   seg_end[b][t]   : one past the position of its last token.
 * The bounds are valid when every row is cut into contiguous segments [s, e) covering [0, seq) in order and both arrays hold
 * each token's own segment. Invalid bounds give unspecified results but never an out-of-bounds access: the tile ranges
 * are clamped into the sequence.
 *   causal segments: key k is visible to query q iff seg_start[q] <= k <= q (equivalently k <= q < seg_end[k]), nothing
 *     across segments. The key / query tiles wholly outside a tile's segments are never loaded: the forward and dQ pass start
 *     at the key tile of seg_start[first query of the tile], the dK / dV pass stops after the query tile of seg_end[last key
 *     of the tile]. The forward reads seg_start only; the backward needs the forward's seg_start and the matching seg_end.
 *     Dropout: an element keeps the bit it has in an unsegmented causal launch.
 *   bidirectional segments (packed BERT / MegatronBERT encoder rows): key k is visible to query q iff
 *     seg_start[q] <= k < seg_end[q] (equivalently seg_start[k] <= q < seg_end[k]); both bounds are read by the forward as
 *     well as the backward. With valid bounds the forward and dQ pass visit the key tiles from the one of seg_start[first
 *     query of the tile] to the one of seg_end[last query of the tile] - 1, and the dK / dV pass the query tiles from
 *     seg_start[first key of the tile] to seg_end[last key of the tile] - 1; a step masks only where it crosses a row's
 *     lower or upper bound. The ranges are clamped into the sequence and always hold the tile's diagonal tile. Dropout: the
 *     keep mask of an element is its bit at the row-relative (q, k) of an unsegmented non-causal launch.
 *   biased segments (packed mT5 / T5 self-attention): the causal (causal = 1, the decoder) or bidirectional (causal = 0, the
 *     encoder) segment rule plus rel_bias (fp32 [nheads, 2 seq - 1] over the offset k - q). The bias depends on (q, k)
 *     through k - q only, so inside a segment the scores are those of the segment run alone and no position ids are needed.
 *     Tile skipping and clamping as in the unbiased rule. The backward accumulates the bias gradient into drel_bias (or
 *     skips it when NULL) with the workspace of the dense form: the reduction reads exactly the per-step slots the dQ pass
 *     wrote (the steps the segment bounds skip are neither written nor read), so the workspace needs no clearing.
 *   cross segments (packed encoder-decoder cross-attention): row b of the queries (seq_q decoder tokens) attends to row b of
 *     the keys (seq_kv encoder tokens), seq_q and seq_kv may differ. Four arrays:
 *       seg_start[b][q], seg_end[b][q] ([batch, seq_q])  : query q sees the keys seg_start[q] <= k < seg_end[q];
 *       q_start[b][k],   q_end[b][k]   ([batch, seq_kv]) : key k is seen by the queries q_start[k] <= q < q_end[k].
 *     They must describe the same visibility, and each array must be non-decreasing along the row (segments paired in
 *     order, e.g. by equal segment id). Then the forward and dQ pass visit the key tiles from the one of seg_start[first
 *     query of the tile] to the one of seg_end[last query of the tile] - 1, the dK / dV pass the query tiles from
 *     q_start[first key] to q_end[last key] - 1, clamped into the sequence. An empty range is legal: a query that sees no
 *     key writes O = 0 and LSE = +inf (which makes its dQ and its share of dK / dV exactly 0), and a key no query sees gets
 *     dK = dV = 0; every output element is written. Dropout: an element's keep bit is that of its row-relative (q, k) in an
 *     unsegmented non-causal launch. The forward reads seg_start / seg_end only.
 */
int fsb_sdpa_fwd(const void* q, const void* k, const void* v, void* o, float* lse,
                 int64_t batch, int64_t seq_q, int64_t seq_kv, int nheads, int head_dim,
                 int64_t q_row_stride, int64_t k_row_stride, int64_t v_row_stride, int64_t o_row_stride,
                 int64_t q_head_stride, int64_t k_head_stride, int64_t v_head_stride, int64_t o_head_stride,
                 float scale, int causal, const uint8_t* kv_mask, const float* rel_bias,
                 const int32_t* seg_start, const int32_t* seg_end, const int32_t* q_start, const int32_t* q_end,
                 float p, uint64_t seed, const int64_t* stream_base, int64_t site, fsb_stream_t stream);

/* Backward of fsb_sdpa_fwd, with the forward's form arguments. o/lse are the forward outputs; delta: fp32 scratch
 * [batch, nheads, seq_q] (written here); dq/dk/dv are written with their own strides (e.g. the three slices of a packed
 * dQKV buffer). Deterministic.
 * drel_bias (fp32 [nheads, seq_q + seq_kv - 1], may be NULL, needs rel_bias) is ACCUMULATED into:
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
                 void* workspace, size_t workspace_bytes,
                 const int32_t* seg_start, const int32_t* seg_end, const int32_t* q_start, const int32_t* q_end,
                 float p, uint64_t seed, const int64_t* stream_base, int64_t site, fsb_stream_t stream);

/* ---- dropout (GPT-2 / BERT / MegatronBERT / mT5 training) -----------------------------------------------------------
 * torch.nn.functional.dropout semantics: an element is dropped with probability p and every kept element is scaled by
 * 1 / (1 - p). The keep bit is a pure function of (seed, stream, coordinates) through Philox4x32-10 (Random123; key =
 * (seed & 0xffffffff, seed >> 32)), so no mask is stored: the backward kernels regenerate it.
 *   threshold : thr = floor(p * 256 + 0.5) (fp32 arithmetic); an element whose 8-bit random value r < thr is dropped. The
 *               effective rate thr / 256 is within 2^-9 of p. p outside [0, 1) is an error; p == 0 runs the kernels without
 *               dropout (fsb_sdpa_fwd, fsb_layernorm_fwd, ...) and does not read the stream counter.
 *   stream    : s = *stream_base + site (int64 read on the device; per-site stream numbers of one forward).
 *   hidden    : element (row, col): counter (col / 16, row, s & 0xffffffff, s >> 32); r = byte (col % 16) % 4 (bits 8 (col % 4))
 *               of output word (col % 16) / 4.
 *   attention : element (b, head, q, k) with q = 16 qa + 8 qh + 2 qs + qp and k = 16 ka + 8 kh + 2 ks + kp:
 *               counter ((4 ka + ks) | (4 qa + qs) << 16, b * nheads + head, s & 0xffffffff, s >> 32); r = byte 2 qh + kh of
 *               output word 2 qp + kp. seq_q, seq_kv <= 65536.
 * fsb_layernorm_fwd_dropout: fsb_layernorm_fwd with sum_out = x * Z / (1 - p) + residual (residual required when p > 0): the
 *   dropped branch of a residual block. With p > 0 both LayerNorm entries take cols <= 12288. fsb_layernorm_bwd_dropout: fsb_layernorm_bwd that also writes dbranch = dx * Z / (1 - p)
 *   (dx already includes dres), the gradient of the branch x, beside dx, the gradient of the sum (and of the residual).
 * fsb_rmsnorm_fwd_dropout / fsb_rmsnorm_bwd_dropout: the same contract over fsb_rmsnorm_fwd / fsb_rmsnorm_bwd.
 * fsb_glu_fwd_dropout: fsb_glu_fwd with out = act(gate) * up * Z / (1 - p), Z the hidden mask at (row, col) of out
 *   (rows < 2^31 when p > 0). fsb_glu_bwd_dropout: fsb_glu_bwd with the same mask applied to dout first.
 * fsb_dropout: y = x * Z / (1 - p) over bf16 [rows, cols] (cols % 8 == 0, rows < 2^32); also the backward (dx = dy * Z / (1 - p)).
 *   x == y is allowed.
 * fsb_dropout_advance: *saved = *stream_base; *stream_base += n (one thread on the device). A training forward calls it once
 *   and hands `saved` to every dropout call of that forward and of its backward, so a replayed CUDA graph draws new masks. */
int fsb_layernorm_fwd_dropout(const void* x, const void* residual, const void* gamma, const void* beta, void* y,
                              void* sum_out, float* mean_rstd, int64_t rows, int64_t cols, float eps,
                              float p, uint64_t seed, const int64_t* stream_base, int64_t site, fsb_stream_t stream);
int fsb_layernorm_bwd_dropout(const void* dy, const void* x, const void* gamma, const float* mean_rstd, const void* dres,
                              void* dx, void* dbranch, void* dgamma, void* dbeta, int wgrad_dtype, int accumulate,
                              void* workspace, size_t workspace_bytes, int64_t rows, int64_t cols,
                              float p, uint64_t seed, const int64_t* stream_base, int64_t site, fsb_stream_t stream);
int fsb_rmsnorm_fwd_dropout(const void* x, const void* residual, const void* scale, void* y, void* sum_out, float* rstd,
                            int64_t rows, int64_t cols, float eps,
                            float p, uint64_t seed, const int64_t* stream_base, int64_t site, fsb_stream_t stream);
int fsb_rmsnorm_bwd_dropout(const void* dy, const void* x, const void* scale, const float* rstd, const void* dres, void* dx,
                            void* dbranch, void* dscale, int wgrad_dtype, int accumulate, void* workspace,
                            size_t workspace_bytes, int64_t rows, int64_t cols,
                            float p, uint64_t seed, const int64_t* stream_base, int64_t site, fsb_stream_t stream);
int fsb_glu_fwd_dropout(int act, const void* gate, const void* up, void* out, int64_t rows, int64_t cols, int64_t ld_gate,
                        int64_t ld_up, int64_t ld_out,
                        float p, uint64_t seed, const int64_t* stream_base, int64_t site, fsb_stream_t stream);
int fsb_glu_bwd_dropout(int act, const void* dout, const void* gate, const void* up, void* dgate, void* dup, int64_t rows,
                        int64_t cols, int64_t ld_dout, int64_t ld_gate, int64_t ld_up, int64_t ld_dgate, int64_t ld_dup,
                        float p, uint64_t seed, const int64_t* stream_base, int64_t site, fsb_stream_t stream);
int fsb_dropout(const void* x, void* y, int64_t rows, int64_t cols, float p, uint64_t seed, const int64_t* stream_base,
                int64_t site, fsb_stream_t stream);
int fsb_dropout_advance(int64_t* stream_base, int64_t* saved, int64_t n, fsb_stream_t stream);

/* ---- decode attention over a KV cache (split-KV) -------------------------------------------------------------------
 * One query row per (batch, head) — the newest token of a generation step, at cache slot *kv_len - 1 — attends to the cache
 * slots [0, *kv_len):  O = softmax(scale * q.K^T + bias + mask) V. kv_len is a DEVICE int32 scalar, clamped to [0, kv_cap];
 * no slot at or beyond it is ever read. Element addressing (elements, 16-byte aligned bases, strides multiples of 8):
 *   q (b, head, d)       at q + b*q_batch_stride + head*q_head_stride + d        (o likewise with o_*_stride)
 *   k (b, slot, head, d) at k + b*k_batch_stride + slot*k_row_stride + head*k_head_stride + d   (v likewise)
 * lse: optional fp32 [batch, nheads], log2 domain as in fsb_sdpa_fwd. kv_mask: optional uint8 [batch, kv_cap], 1 = attend.
 * rel_bias: optional fp32 [nheads, 2*kv_cap - 1] in fsb_sdpa_fwd's convention with seq_q = seq_kv = kv_cap, i.e. the bias of key
 *   k is rel_bias[head][k - (*kv_len - 1) + kv_cap - 1] (T5 / mT5 decoder self-attention). A row that sees no key gets O = 0
 *   and lse = +inf. head_dim in {64, 128}. The keys are split into chunks planned from (batch, nheads, kv_cap) alone; the fp32
 * partials go to `workspace` (fsb_attn_decode_workspace_bytes bytes, 16-byte aligned) and are merged in a fixed order, so the
 * result is deterministic. Two kernel launches. */
size_t fsb_attn_decode_workspace_bytes(int64_t batch, int nheads, int head_dim, int64_t kv_cap);
int fsb_attn_decode(const void* q, const void* k, const void* v, void* o, float* lse,
                    int64_t batch, int nheads, int head_dim, int64_t kv_cap, const int32_t* kv_len,
                    int64_t q_batch_stride, int64_t q_head_stride,
                    int64_t k_batch_stride, int64_t k_row_stride, int64_t k_head_stride,
                    int64_t v_batch_stride, int64_t v_row_stride, int64_t v_head_stride,
                    int64_t o_batch_stride, int64_t o_head_stride,
                    float scale, const uint8_t* kv_mask, const float* rel_bias,
                    void* workspace, size_t workspace_bytes, fsb_stream_t stream);

/* ---- KV-cache maintenance of a decode step (device-side position) ------------------------------------------------------
 * Both entries read the cache length from the same DEVICE int32 scalar `kv_len` as fsb_attn_decode and take no host-side
 * slot, so a decode step built from them issues identical launches at every position and can be captured in a CUDA graph.
 *
 * fsb_kv_append: copies the newest token's keys and values into cache slot *kv_len - 1, for every row and head (16-byte
 *   vector accesses). It replaces the per-step concatenation of the new key / value onto the layer's past (transformers'
 *   cache update, `layer_past` in the reference) and a slot copy at a host index. Element addressing (elements; 16-byte
 *   aligned bases; strides multiples of 8; head_dim a multiple of 8):
 *     new key   (row, head, d)       at k_new + row*k_new_row_stride + head*k_new_head_stride + d        (v_new likewise)
 *     cache key (row, slot, head, d) at k_cache + row*k_batch_stride + slot*k_row_stride + head*k_head_stride + d
 *                                                                                                          (v_cache likewise)
 *   e.g. GPT-2 / mT5: the new keys are the K third of the packed [t, {q,k,v}, heads, d] projection and the cache is
 *   [rows, kv_cap, {k,v}, heads, d]; LLaMA: the K slice of the interleaved [t, heads, {q,k,v}, d] projection into a separate
 *   [rows, kv_cap, heads, d] K cache. kv_mask: optional contiguous uint8 [rows, kv_cap]; kv_mask[row, slot] is set to 1.
 *   A slot outside [0, kv_cap) writes nothing. One kernel launch.
 *
 * fsb_kv_reorder: the beam-search gather dst[l, r, s, :] = src[l, index[r], s, :] over the caches of all `layers` in one
 *   launch, for the live slots s < *kv_len only (clamped to [0, kv_cap]); slots at or beyond it are neither read nor written.
 *   It replaces transformers' `_reorder_cache` (an index_select of every layer's full capacity). src and dst are contiguous
 *   bf16 [layers, rows, kv_cap, slot_elems] (slot_elems = the elements of one slot of one row, a multiple of 8, e.g.
 *   2 * heads * head_dim), 16-byte aligned and disjoint. index: int64 [rows] on the device; a row whose index lies outside
 *   [0, rows) is left untouched. One kernel launch. */
int fsb_kv_append(const void* k_new, const void* v_new, void* k_cache, void* v_cache, uint8_t* kv_mask,
                  int64_t rows, int nheads, int head_dim, int64_t kv_cap, const int32_t* kv_len,
                  int64_t k_new_row_stride, int64_t k_new_head_stride, int64_t v_new_row_stride, int64_t v_new_head_stride,
                  int64_t k_batch_stride, int64_t k_row_stride, int64_t k_head_stride,
                  int64_t v_batch_stride, int64_t v_row_stride, int64_t v_head_stride, fsb_stream_t stream);
int fsb_kv_reorder(const void* src, void* dst, const int64_t* index, int64_t layers, int64_t rows, int64_t kv_cap,
                   int64_t slot_elems, const int32_t* kv_len, fsb_stream_t stream);

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
