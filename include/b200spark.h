/*
 * b200spark C ABI — the drop-in boundary for DashInfer's quantized decode hot path on H100 (sm_90a).
 *
 * Everything here is `extern "C"`, takes plain pointers / sizes / POD structs and returns an `int`
 * status (b2_status); nothing throws, nothing synchronises the device, every call is ordered on the
 * `stream` it is given (a `cudaStream_t` passed as `void*`).  Enum values on the wire are the
 * reference's own (allspark.proto DataType / UnaryType, span::QuantMode), so the C++ operator shims
 * (dash-infer_b200/host/) forward attributes unchanged.
 *
 * Reference interfaces replaced (paths relative to modelscope/dash-infer @ f3cca8e):
 *   b2_gemm_wq_*          cuda::GemmA16W4Launcher::Run / GetWorkSpaceSize
 *                           csrc/core/kernel/cuda/gemm_lowp/gemm_a16w4_kernel.h:133-273
 *                         cuda::GemmA16W8Launcher::Run
 *                           csrc/core/kernel/cuda/gemm_lowp/gemm_a16w8_kernel.h:229-330
 *                         weight re-layout at op init (GemmA16W8GPU::B_I8_Reorder...)
 *                           csrc/core/operator/general/gemm_lowp/gemm_a16w8_gpu.cpp:422-473
 *                         dense Gemm (lm_head): cuda::GemmWraper  csrc/core/kernel/cuda/gemm.cu:596-615
 *   b2_span_bytes         CacheUtils::GetSpanSizeInBytes  csrc/runtime/cache/virtual_cache.cpp:202-232
 *   b2_span_cache_append  cuda::DecoderCacheAppendLauncher
 *                           csrc/core/kernel/cuda/cache/decoder_cache_append.cuh:102-185
 *   b2_span_context_copy  cuda::ContextSpanCopyLauncher  csrc/core/kernel/cuda/cache/context_span_copy.cuh:220-245
 *   b2_span_attn_*        span::CreateHandle/GetDeviceWorkspaceSize/Run/DestroyHandle
 *                           span-attention/include/spanattn/span_attn.h:108-175
 *   b2_comm_*, b2_allreduce, b2_allgather, b2_gemm_wq_run_allreduce
 *                         AllReduceOp::Forward  csrc/core/operator/nccl/allreduce/allreduce_op.cpp:73-115
 *   b2_rmsnorm, b2_rotary, b2_binary, b2_embedding, b2_argmax ("next" rows, SURVEY.md §8f)
 *                         LayerNormNoBeta / Rotary / Binary / EmbeddingT5 / GenerateOp(top_k=1)
 *                           csrc/core/kernel/cuda/layernorm.cu:86, rotary.cu:23, binary.cu
 */
#ifndef B200SPARK_H_
#define B200SPARK_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes (map 1:1 onto span::SaStatus, span_attn.h:53-70; AsStatus in the shims) ---- */
typedef enum {
  B2_OK = 0,
  B2_ERR_CUDA = 1,
  B2_ERR_RUNTIME = 2,
  B2_ERR_PARAM = 3,
  B2_ERR_LIMIT = 4,
  B2_ERR_INTERNAL = 5,
  B2_ERR_UNSUPPORTED = 6
} b2_status;

const char* b2_status_string(int status);
/* Last CUDA error text recorded by a failing call on this thread (empty string if none). */
const char* b2_last_error(void);
/* "b200spark <ver> sm_90a" */
const char* b2_version(void);

/* ---- allspark.proto wire enums (csrc/proto/allspark.proto:35-76) ---- */
enum { B2_DT_F32 = 1, B2_DT_F16 = 2, B2_DT_I8 = 3, B2_DT_BF16 = 9, B2_DT_U8 = 10 };
enum { B2_ACT_NONE = 0, B2_ACT_TANH = 1, B2_ACT_GELU_ERF = 2, B2_ACT_GELU_TANH = 3, B2_ACT_RELU = 4,
       B2_ACT_SILU = 5, B2_ACT_SIGMOID = 6 };
enum { B2_BIN_ADD = 1, B2_BIN_MUL = 2 };
/* extension (not a reference UnaryType): fused SwiGLU epilogue of a gate/up weight pair, see b2_gemm_wq_prepare_swiglu */
enum { B2_ACT_SWIGLU = 100 };
/* span::QuantMode (span_attn.h:41-48) */
enum { B2_KV_NONE = 0, B2_KV_I8 = 1, B2_KV_U4 = 2 };
/* extension (not a span::QuantMode value): fp8-e4m3fn KV cache, head 128 only.  Same span layout as B2_KV_I8 (one byte
 * per element, then {f32 zero, f32 scale} per row) with zero always 0: per (token, kv-head) row
 * scale = max(max|x|, 1e-12) / 448, code = e4m3(x * (1 / scale)) rounded to nearest even, saturating (IEEE fp32 steps). */
enum { B2_KV_FP8 = 3 };

/* =====================================================================================
 * Weight-only quantized GEMV/GEMM:  C[M,N] = act(alpha * A[M,K] x dequant(W)[K,N] + bias) (+ residual)
 *   wbits 4 : qdata uint8 [K, ceil(N/2)], lo nibble = even column   (GemmA16W4, gemm_a16w4.h:14-33)
 *   wbits 8 : qdata int8/uint8 [K, N]                               (GemmA16W8)
 *   wbits 16: unquantized FT weights [K, N] (dense Gemm / lm_head), scales/zeros ignored
 *   dequant(W)[k,n] = (q[k,n] - zero[k/group, n]) * scale[k/group, n];  group_size -1 = per channel.
 * The handle owns an init-time re-laid-out copy of the weights (the reference re-lays out at op init
 * too); the caller's [K,N] buffers are only read during prepare and may be freed afterwards.
 * ===================================================================================== */
typedef struct b2_gemm_wq* b2_gemm_wq_t;

typedef struct {
  int32_t K;
  int32_t N;
  int32_t wbits;      /* 4, 8 or 16 */
  int32_t group_size; /* -1 per-channel; otherwise a multiple of 64 (int4: any multiple of 8 >= 32) */
  int32_t ft;         /* B2_DT_BF16 or B2_DT_F16 (activations, scales, zeros, bias, residual, output) */
  int32_t qtype;      /* B2_DT_U8 (uint4x2 or uint8) or B2_DT_I8 (wbits 8) */
  int32_t max_m;      /* largest M this handle will be run with (sizes persistent buffers) */
  int32_t reserved;
} b2_gemm_wq_desc;

int b2_gemm_wq_create(b2_gemm_wq_t* handle, const b2_gemm_wq_desc* desc);
int b2_gemm_wq_destroy(b2_gemm_wq_t handle);
/* Bytes of the re-laid-out weight image. */
size_t b2_gemm_wq_packed_bytes(b2_gemm_wq_t handle);
/* Re-layout device tensors qdata/scales/zeros (reference layouts above) into the handle's image.
 * If packed_dst != NULL the image is written there (caller-owned, >= packed_bytes, 128B aligned)
 * instead of handle-owned memory — this is how two op instances share one image. */
int b2_gemm_wq_prepare_weights(b2_gemm_wq_t handle, const void* qdata, const void* scales,
                               const void* zeros, void* packed_dst, void* stream);
/* Fusion of the reference's three ops  GemmA16Wx(gate, SiLU) -> GemmA16Wx(up) -> Binary MUL  (qwen_v15.py:330-360)
 * into one weight stream: the handle is created with N = intermediate size and desc.reserved = 1; both [K,N] weight
 * sets are re-laid-out into one image (64 gate + 64 up channels per 128-row tile) and _run with
 * activation = B2_ACT_SWIGLU writes C[m,n] = silu(alpha * a.Wg[:,n]) * (alpha * a.Wu[:,n]), C is [M, N].  No bias. */
int b2_gemm_wq_prepare_swiglu(b2_gemm_wq_t handle, const void* q_gate, const void* s_gate, const void* z_gate,
                              const void* q_up, const void* s_up, const void* z_up, void* stream);
/* Use an image prepared by another handle with an identical desc (prefill/decode sharing). */
int b2_gemm_wq_attach_packed(b2_gemm_wq_t handle, const void* packed, const void* scales_f32,
                             const void* zeros_f32);
/* Scratch the caller must provide to _run for this M (split-K partials); may be 0. */
size_t b2_gemm_wq_workspace_bytes(b2_gemm_wq_t handle, int M);
/* A: [M, lda] FT, C: [M, ldc] FT, bias: [N] FT or NULL, residual: [M, ldc] FT or NULL (added after
 * the activation).  workspace: >= workspace_bytes(M), 16B aligned, contents undefined on entry/exit. */
int b2_gemm_wq_run(b2_gemm_wq_t handle, const void* A, int64_t lda, void* C, int64_t ldc, int M,
                   const void* bias, const void* residual, int activation, float alpha,
                   void* workspace, size_t workspace_bytes, void* stream);
/* RMSNorm fusion ("next" row f2 of SURVEY.md §8), two forms named by the fields that are set; any other combination
 * (norm_sumsq with norm_gamma, sumsq_out without xg_out, a form on the other kernel's batches) is B2_ERR_UNSUPPORTED.
 * Self-contained form, batches <= 16 (norm_gamma only, norm_hidden == K): the GEMV needs nothing from its producer — it
 * stages bf16(A[m,k] * gamma[k]), collects sum_k A[m,k]^2 over its own k-slice in the same pass (the split-K reducer adds
 * the slices), and multiplies the reduced fp32 tile by rsqrt(sum / K + eps) before alpha / bias / activation:
 *   C = act(alpha * inv_rms[m] * sum_k bf16(A[m,k] gamma[k]) W[k,n] + bias)   — one bf16 rounding per activation, like the
 * stand-alone norm, at a different point of the product.  Every CTA repeats the normalisation of its k-slice of every live
 * row, so it pays at tiny batches only: the decode stack uses it at batches <= 2 (FT(x) stands for bf16 or fp16).
 * Hand-off form, batches >= 17 (int4 group sizes that are not a multiple of 64: every batch): see the struct.
 * Range: both forms stage FT(x * gamma) before normalising.  In fp16 a row with max|x * gamma| > 65504 stages inf, where
 * b2_rmsnorm stays finite; keep fp16 rows below that.  On N(0,1) rows with one channel at 64 sigma, both forms stay inside the
 * fp64 RMSNorm -> GEMM envelope wherever checked: RMS 2^-16 (the lowest checked) up to 2^12 in bf16, up to that overflow in
 * fp16 (H100 SXM, tests/test_norm_exact_gpu.py). */
typedef struct {
  const float* norm_sumsq; /* hand-off consumer: [norm_parts][M], or NULL */
  const void* norm_gamma;  /* self-contained form: [K] FT, or NULL */
  int32_t norm_parts;
  int32_t norm_hidden;
  float norm_eps;
  int32_t reserved;
  float* sumsq_out;        /* hand-off producer: [b2_gemm_wq_sumsq_parts(handle)][M], or NULL */
  /* Hand-off form (wgmma path).  The producer (o_proj / down_proj with residual) writes, besides C, per-tile row sums of
   * squares (sumsq_out) and xg_out[m, n] = FT(C[m, n] * gamma_out[n]) — the next RMSNorm's input already scaled by its gamma;
   * the consumer (A = xg, norm_sumsq = the producer's sumsq_out, norm_gamma = NULL) multiplies its fp32 result rows by
   * rsqrt(sum_p norm_sumsq[p][m] / norm_hidden + eps).  A call may be both.  Two RMSNorm launches per layer disappear; the
   * statistics are taken from the values as stored (FT), like the stand-alone norm reads them. */
  void* xg_out;            /* [M, ldxg] FT or NULL (requires sumsq_out and gamma_out) */
  const void* gamma_out;   /* [N] FT */
  int64_t ldxg;
} b2_gemm_fuse;
int b2_gemm_wq_sumsq_parts(b2_gemm_wq_t handle);
int b2_gemm_wq_run_fused(b2_gemm_wq_t handle, const void* A, int64_t lda, void* C, int64_t ldc, int M,
                         const void* bias, const void* residual, int activation, float alpha,
                         void* workspace, size_t workspace_bytes, const b2_gemm_fuse* fuse, void* stream);
/* FP8 activations ("next" row f3; BASELINE config "GPTQ-int4, fp8 activations"): fp8-e4m3 activations x int4 weights on
 * the Hopper warpgroup tensor cores (e4m3 wgmma, K = 32 per MMA).  Beyond the reference (its FP8 operator is per-tensor A8W8 through
 * cuBLASLt, csrc/core/operator/general/gemm_lowp/gemm_fp8_a8w8_gpu.cpp:325-395), so the accuracy contract is its own:
 *   C[m,n] = act(alpha * scale_a[m] * s_n * (sum_k a8[m,k] q[k,n] - z_n sum_k a8[m,k]) + bias) (+ residual)
 * exact products (e4m3 x e4m3) and fp32 accumulation: the only loss is the activation quantization itself.
 * b2_quant_fp8 produces the operands: y = e4m3(x / scale[r]) with scale[r] = max|x[r,:]| / 448 (optionally after a fused
 * RMSNorm: gamma != NULL), stored in the "b2 fp8 activation layout" (inside every aligned group of 8 k the bytes hold
 * k = 0,2,4,6,1,3,5,7), plus tile_sums[r][ceil(cols/64)] = per-64-k sums of the quantized values.  ldy in bytes (>= cols,
 * multiple of 16).  b2_gemm_wq_run_fp8: int4 per-channel weights only (B2_ERR_UNSUPPORTED otherwise); workspace as for
 * b2_gemm_wq_run at M >= 17. */
int b2_quant_fp8(void* y, int64_t ldy, float* scale, float* tile_sums, const void* x, const void* gamma, int rows, int cols,
                 float eps, void* stream);
int b2_gemm_wq_run_fp8(b2_gemm_wq_t handle, const void* A8, int64_t lda_bytes, const float* a_scale, const float* tile_sums,
                       void* C, int64_t ldc, int M, const void* bias, const void* residual, int activation, float alpha,
                       void* workspace, size_t workspace_bytes, void* stream);
/* Algorithmic bytes one run at this M must read from HBM (weights + params + A + C). */
size_t b2_gemm_wq_algo_bytes(b2_gemm_wq_t handle, int M);

/* =====================================================================================
 * SpanAttention: paged KV cache (spans) append + single-query attention, GQA, KV in FT / int8 / uint4 / fp8-e4m3.
 * Span wire format (decoder_cache_append.cuh:33-92): [n_groups, span_len, head_size] of QT followed,
 * for I8/U4/FP8, by [n_groups, span_len] of {float zero, float scale} (FP8: zero = 0).
 * Span tables: device arrays [batch, max_spans_per_seq] of device pointers.
 * ===================================================================================== */
typedef struct {
  int32_t ft;                /* B2_DT_BF16 or B2_DT_F16: Q, the output, an unquantized cache (head 64: bf16 only) */
  int32_t quant_mode;        /* B2_KV_NONE / B2_KV_I8 / B2_KV_U4 / B2_KV_FP8 (head 128 only) */
  int32_t n_heads;           /* query heads on this rank */
  int32_t n_groups;          /* kv heads on this rank; n_heads % n_groups == 0, n_heads/n_groups <= 16 */
  int32_t head_size;         /* 128 */
  int32_t span_len;          /* 16, 32, 64 or 128 */
  int32_t max_spans_per_seq; /* row stride of the span pointer tables */
  int32_t reserved;
} b2_span_cfg;

size_t b2_span_bytes(const b2_span_cfg* cfg);

/* Gather Q and append this step's K,V rows (one new token per sequence).
 *   qkv      [batch, (n_heads + 2*n_groups) * head_size] FT (post-RoPE unless rope != NULL)
 *   q_out    [batch, n_heads * head_size] FT
 *   old_lens [batch] int32 device: tokens already cached (= write position)
 * rope: optional fused rotary (NeoX rotate-half over rotary_dim, position = old_lens[b]); pass NULL
 * when the graph has a separate Rotary op.  Quantised modes follow QuantParam<I8/U4>::Builder
 * (span-attention/src/cache_quant/impl_i8.cuh:106-140, impl_u4.cuh:146-182) with IEEE division; B2_KV_FP8 quantizes as
 * described at its enum. */
typedef struct {
  float base;          /* e.g. 1e6 for Qwen2 */
  int32_t rotary_dim;  /* <= head_size, even */
  int32_t reserved;
} b2_rope_cfg;
int b2_span_cache_append(const b2_span_cfg* cfg, void* const* k_spans, void* const* v_spans,
                         void* q_out, const void* qkv, const int32_t* old_lens, int batch,
                         const b2_rope_cfg* rope, void* stream);

/* Prefill side of the cache ("next" row f4): slice one sequence's contiguous K (or V) rows into its spans, quantizing like
 * the append does (replaces cuda::ContextSpanCopyLauncher, csrc/core/kernel/cuda/cache/context_span_copy.cuh:47-106,220-245).
 *   spans        device array of this sequence's span pointers (one row of a span table), K or V
 *   src          [seq_len][token_stride] FT, the n_groups * head_size values of a token contiguous at its start
 *                (token_stride = n_groups * head_size for a packed [seq, nG, head] tensor; a larger stride reads K or V
 *                straight out of a fused qkv activation)
 * Tokens 0 .. seq_len-1 are written; unlike the reference (which quantizes whole spans and so reads src up to the next span
 * multiple) rows >= seq_len are left untouched. */
int b2_span_context_copy(const b2_span_cfg* cfg, void* const* spans, const void* src, int64_t token_stride, int seq_len,
                         void* stream);

/* Attention handle (replaces span::CreateHandle/DestroyHandle, span_attn.h:108-133).  Unlike the
 * reference it is created ONCE per op (not per layer per step): tile scheduling happens on the
 * device from new_lens, so nothing is rebuilt or copied host->device per step.  Owns only a small
 * self-resetting counter array. */
typedef struct b2_span_attn* b2_span_attn_t;
int b2_span_attn_create(b2_span_attn_t* handle, const b2_span_cfg* cfg, int max_batch);
int b2_span_attn_destroy(b2_span_attn_t handle);
size_t b2_span_attn_workspace_bytes(b2_span_attn_t handle, int batch, int max_len);

/* out [batch, n_heads*head_size] FT = softmax(qk_scale * q K^T) V over the first new_lens[b] tokens.
 * I8 / U4 / FP8: the MMAs run in fp16, so |q| < 65504 after Q's conversion to fp16, and each probability times its
 * token's V scale is rounded to fp16 with a per-mode power of two folded in.  Accuracy window: for V rows (before
 * quantization) with per-row max|v| in [2^-12, 2^12] the output meets the attention error envelope (probabilities far
 * below the row's maximum may still round as fp16 subnormals; their error stays inside the envelope).  Above per-row
 * max|v| ~ 2^12.8 the rounded products can overflow to inf and the output is undefined.
 * new_lens: device int32 [batch] (including the token appended this step).  max_len bounds every
 * new_lens[b] (only sizes the workspace check; a loose bound is fine).
 * workspace >= workspace_bytes(batch,max_len), 16B aligned, contents undefined on entry/exit. */
int b2_span_attn_run(b2_span_attn_t handle, void* out, const void* q, const void* const* k_spans,
                     const void* const* v_spans, const int32_t* new_lens, int batch, int max_len,
                     void* workspace, size_t workspace_bytes, float qk_scale, void* stream);
/* Algorithmic KV bytes for a given total token count (sum of lens): 2 * n_groups * (row + param). */
size_t b2_span_attn_algo_bytes(const b2_span_cfg* cfg, int64_t total_tokens);

/* ---- Multi-token decode steps (speculative decoding: verify up to 16 drafted tokens per sequence in one step).
 * Layout: with q_len = T, row b*T + t of every activation (qkv, q, out) holds token t of sequence b.  Head 128 only
 * (B2_ERR_UNSUPPORTED otherwise); 1 <= q_len <= 16 (B2_ERR_LIMIT otherwise).
 *
 * Append: row (b, t) of qkv [batch*q_len, (n_heads + 2*n_groups) * 128] is written at position old_lens[b] + t (fused rotary
 * at that position) and its q heads go to q_out [batch*q_len, n_heads * 128].  The span bytes and {zero, scale} equal those
 * of q_len successive b2_span_cache_append calls. */
int b2_span_cache_append_tokens(const b2_span_cfg* cfg, void* const* k_spans, void* const* v_spans, void* q_out,
                                const void* qkv, const int32_t* old_lens, int batch, int q_len, const b2_rope_cfg* rope,
                                void* stream);
/* Attention: q, out [batch*q_len, n_heads*128]; row (b, t) attends to tokens 0 .. new_lens[b] - q_len + t (itself and the
 * tokens before it).  Precondition new_lens[b] >= q_len.  batch * q_len <= the handle's max_batch (B2_ERR_LIMIT).  The
 * q-heads of whole tokens share the 16 rows of one MMA tile (floor(16 / (n_heads/n_groups)) tokens per row block), so K and
 * V are read once per row block. */
size_t b2_span_attn_tokens_workspace_bytes(b2_span_attn_t handle, int batch, int q_len, int max_len);
int b2_span_attn_run_tokens(b2_span_attn_t handle, void* out, const void* q, const void* const* k_spans,
                            const void* const* v_spans, const int32_t* new_lens, int batch, int q_len, int max_len,
                            void* workspace, size_t workspace_bytes, float qk_scale, void* stream);

/* ---- Tree-structured verification (Medusa / EAGLE-style draft trees).  The q_len rows of a sequence are the nodes of a
 * draft tree; the layout, limits and handle rules of the multi-token entry points above apply.
 * Tree format: parents [batch][q_len] int32, device-resident, filled by the caller before each step like the tokens.
 *   Node 0 is the root (the last emitted token); parents[b][0] is ignored.  For t >= 1, parents[b][t] lies in [0, t): nodes
 *   are in topological order.  Trees may differ per sequence.
 *   depth(t) = the parent steps from t to node 0; anc(t) = the 16-bit mask of t and its ancestors.  Both are derived on the
 *   device (a walk of at most q_len - 1 steps).
 *   A chain (parents[b][t] = t - 1: depth t, anc bits 0..t) reproduces the multi-token entry points bit for bit.
 *   Malformed parents are a caller error: results are unspecified, but no kernel reads or writes out of bounds or loops
 *   without bound, for any int32 input.
 *
 * Append: row (b, t) is written at slot old_lens[b] + t, with fused rotary at position old_lens[b] + depth(t). */
int b2_span_cache_append_tree(const b2_span_cfg* cfg, void* const* k_spans, void* const* v_spans, void* q_out, const void* qkv,
                              const int32_t* old_lens, const int32_t* parents, int batch, int q_len, const b2_rope_cfg* rope,
                              void* stream);
/* Attention: row (b, t) attends to the prefix (tokens < new_lens[b] - q_len) and to the slots new_lens[b] - q_len + j for
 * every j in anc(t).  Workspace: b2_span_attn_tokens_workspace_bytes. */
int b2_span_attn_run_tree(b2_span_attn_t handle, void* out, const void* q, const void* const* k_spans,
                          const void* const* v_spans, const int32_t* new_lens, const int32_t* parents, int batch, int q_len,
                          int max_len, void* workspace, size_t workspace_bytes, float qk_scale, void* stream);

/* =====================================================================================
 * Glue ops of the decode graph ("next" rows): element-wise / norm / lookup, FT = bf16.
 * ===================================================================================== */
/* Every glue op below that takes 16-bit tensors moves them in vectors: y, x, gamma (rmsnorm), out, a, b (binary) and out, table
 * (embedding) must be 16-byte aligned, qkv (rotary) 8-byte aligned; a misaligned pointer is B2_ERR_UNSUPPORTED. */
/* y[r,:] = x[r,:] * rsqrt(mean(x^2) + eps) * gamma   (LayerNormNoBeta, layernorm.cu:86).  y may be x.  Finite x with
 * sum(x[r,:]^2) < 2^127 (the kernel sums the squares in fp32 before it divides by cols); non-finite x is out of contract. */
int b2_rmsnorm(void* y, const void* x, const void* gamma, int rows, int cols, float eps, void* stream);
/* The glue ops with an explicit 16-bit type (ft = B2_DT_BF16 or B2_DT_F16); the unsuffixed entry points are the bf16 forms. */
int b2_rmsnorm_ft(void* y, const void* x, const void* gamma, int rows, int cols, float eps, int ft, void* stream);
int b2_binary_ft(void* out, const void* a, const void* b, int64_t n, int op, int ft, void* stream);
int b2_argmax_ft(int64_t* ids_out, float* vals_out /* or NULL */, const void* logits, int batch, int n, int64_t ld, int64_t id_offset,
                 int ft, void* stream);
/* in-place NeoX rotary on the q and k heads of qkv [batch, (nH+2nG)*head]; position = pos[b] */
int b2_rotary(void* qkv, const int32_t* pos, int batch, int n_heads, int n_groups, int head_size,
              const b2_rope_cfg* rope, void* stream);
/* out = a (op) b, n elements; op = B2_BIN_ADD / B2_BIN_MUL */
int b2_binary(void* out, const void* a, const void* b, int64_t n, int op, void* stream);
/* out[b,:] = table[ids[b],:] */
int b2_embedding(void* out, const void* table, const int64_t* ids, int batch, int hidden, void* stream);
/* ids_out[b] = argmax_n logits[b,n] (lowest index on ties); logits FT [batch, ld], ld >= n (else B2_ERR_PARAM).
 * The order is torch.argmax's: NaN ranks above every number (+inf included), so a row holding a NaN yields the index of
 * its first NaN, and ids_out[b] always lies in [id_offset, id_offset + n) (the _ft / _shard forms' offset; 0 here).  An
 * all -inf row yields its first index.  vals_out[b] (the _ft / _shard forms) = the winner's value widened to fp32. */
int b2_argmax(int64_t* ids_out, const void* logits, int batch, int n, int64_t ld, void* stream);
/* vocab-sharded lm_head (tensor parallel): per-rank argmax of its shard, ids offset by the shard start, plus the max
 * value (fp32) so the ranks can pick the global winner with a B-element all-gather instead of all-reducing logits. */
int b2_argmax_shard(int64_t* ids_out, float* vals_out, const void* logits, int batch, int n, int64_t ld,
                    int64_t id_offset, void* stream);
/* ids_out[b] = all_ids[r*][b] with r* = the rank of the largest all_vals[r][b] under b2_argmax's order (NaN above every
 * number; lowest rank among equal values or among NaNs): the second half of the vocab-split argmax after the (max, argmax)
 * pairs were all-gathered ([nranks][batch] each).  With rank r holding vocab ids [r*n, (r+1)*n), it equals b2_argmax of the
 * whole row. */
int b2_argmax_merge(int64_t* ids_out, const float* all_vals, const int64_t* all_ids, int nranks, int batch, void* stream);
/* lens[b] += delta for b < batch (keeps sequence lengths device-resident under CUDA graphs) */
int b2_lens_add(int32_t* lens, int batch, int delta, void* stream);
/* Greedy verification of a multi-token step, on the device (CUDA-graph replayable).  tokens [batch][q_len] int64: column 0
 * is the last emitted token, columns 1.. the draft; pred [batch][q_len] = argmax of the step's rows.
 *   n_b = 1 + the number of leading i >= 1 with tokens[b][i] == pred[b][i-1]
 * writes accepted[b] = n_b (int32), next_ids[b] = pred[b][n_b-1] (may be NULL) and tokens[b][0] = pred[b][n_b-1] (the last
 * emitted token of the next step); old_lens[b] += n_b, new_lens[b] = old_lens[b] + q_len.  The emitted tokens of the step are
 * pred[b][0 .. n_b-1].  Rows of rejected drafts stay in the cache; the next step overwrites them. */
int b2_spec_accept(int32_t* accepted, int64_t* next_ids, int32_t* old_lens, int32_t* new_lens, int64_t* tokens,
                   const int64_t* pred, int batch, int q_len, void* stream);
/* Greedy verification of a draft tree (tree format: b2_span_cache_append_tree).  From u = 0: while some child c of u has
 * tokens[b][c] == pred[b][u], take the lowest-index such c, append it to the path and set u = c.  Writes accepted[b] = n (the
 * path length, >= 1), path[b][0 .. n-1] (int32 [batch][q_len], path[b][0] = 0; later entries untouched), next_ids[b] (may be
 * NULL) = tokens[b][0] = pred[b][u]; old_lens[b] += n, new_lens[b] = old_lens[b] + q_len.  The emitted tokens of the step
 * are pred[b][path[b][i]], i < n.  A chain gives b2_spec_accept's results. */
int b2_spec_accept_tree(int32_t* accepted, int32_t* path, int64_t* next_ids, int32_t* old_lens, int32_t* new_lens,
                        int64_t* tokens, const int64_t* pred, const int32_t* parents, int batch, int q_len, void* stream);
/* Move the accepted path's K/V rows to consecutive slots, in every layer with one launch.  k_tables / v_tables: device
 * arrays of n_layers span-table pointers (each table [batch][max_spans_per_seq], as for the other span entry points).  With
 * base = old_lens[b] - accepted[b] (the lengths as b2_spec_accept_tree left them), slot base + path[b][i] is copied to slot
 * base + i for 1 <= i < accepted[b] where path[b][i] != i: the row bytes of every kv-head of K and V, and their {zero,
 * scale} in the quantized modes.  A node at depth i carries rotary position base + i already, so the copy is exact.  All
 * source rows of a (sequence, layer, kv-head) are read before any is written (path [0, 2, 3] reads slot 2 while slot 2 is
 * written).  Rows of rejected nodes stay; the next step overwrites them.  Head 128 only. */
int b2_span_cache_compact(const b2_span_cfg* cfg, void* const* const* k_tables, void* const* const* v_tables, int n_layers,
                          const int32_t* old_lens, const int32_t* accepted, const int32_t* path, int batch, int q_len,
                          void* stream);

/* =====================================================================================
 * Tensor-parallel exchange over NVLink peer memory (replaces AllReduceOp / ncclAllReduce for the decode step's
 * activations, csrc/core/operator/nccl/allreduce/allreduce_op.cpp:73-115).  One communicator per rank, one process per
 * GPU.  Every rank owns an exchange buffer; the peers map it (CUDA IPC handles exchanged by the caller, or any table of
 * peer pointers).  All calls are stream-ordered, never synchronise the host and are CUDA-graph replayable; every rank
 * must issue the same sequence of exchanges on a communicator.  FT = bf16; sums are fp32 in rank order (deterministic).
 * ===================================================================================== */
typedef struct b2_comm* b2_comm_t;
#define B2_COMM_HANDLE_BYTES 64 /* sizeof(cudaIpcMemHandle_t) */
/* max_bytes: largest payload of one exchange (per rank).  Allocates and zeroes this rank's exchange buffer. */
int b2_comm_create(b2_comm_t* comm, int rank, int nranks, size_t max_bytes);
int b2_comm_destroy(b2_comm_t comm);
size_t b2_comm_buffer_bytes(int nranks, size_t max_bytes);
/* IPC route: export this rank's handle (B2_COMM_HANDLE_BYTES), all-gather the handles on the host (any transport), then
 * connect with the nranks handles in rank order. */
int b2_comm_export(b2_comm_t comm, void* handle_out);
int b2_comm_connect(b2_comm_t comm, const void* all_handles);
/* Pointer route: peer_buffers[r] = rank r's exchange buffer as addressable from this process (b2_comm_local_buffer of
 * that rank's communicator: same process with peer access, symmetric memory, ...).  peer_buffers[rank] is ignored. */
int b2_comm_connect_pointers(b2_comm_t comm, void* const* peer_buffers);
void* b2_comm_local_buffer(b2_comm_t comm);
/* B2_OK, or B2_ERR_RUNTIME when a kernel gave up waiting for a peer (B2_COMM_TIMEOUT_MS, default 5000); synchronises. */
int b2_comm_error(b2_comm_t comm);
/* out[i] = sum over ranks of in[i] (+ residual[i], added once after the sum), count elements of FT (count % 8 == 0,
 * 16-byte aligned pointers).  out may alias in or residual. */
int b2_allreduce(b2_comm_t comm, void* out, const void* in, const void* residual, int64_t count, int ft, void* stream);
/* out[r * bytes_per_rank ...] = rank r's `in` (small payloads: the vocab-split lm_head's per-rank (max, argmax)). */
int b2_allgather(b2_comm_t comm, void* out, const void* in, int bytes_per_rank, void* stream);
/* Row-parallel projection fused with its all-reduce: b2_gemm_wq_run where the partial sums of each 128-channel tile are
 * pushed into the peers' exchange buffers by the tile's last CTA, which then waits for the peers' tiles, sums the nranks
 * partials in rank order, adds `residual` once and writes C — one kernel instead of GEMV + all-reduce (+ copy), the
 * exchange of a tile overlapping the weight streaming of the others.  M <= 16 (the GEMV path), activation NONE, no bias
 * on ranks != 0 (pass bias only on rank 0).  Returns B2_ERR_UNSUPPORTED otherwise: call b2_gemm_wq_run + b2_allreduce. */
int b2_gemm_wq_run_allreduce(b2_gemm_wq_t handle, const void* A, int64_t lda, void* C, int64_t ldc, int M, const void* bias,
                             const void* residual, float alpha, void* workspace, size_t workspace_bytes, b2_comm_t comm,
                             void* stream);

/* Programmatic dependent launch (PDL) for every kernel launched by this library on this thread:
 * 1 = on (default), 0 = off. */
void b2_set_pdl(int enabled);

#ifdef __cplusplus
}
#endif
#endif /* B200SPARK_H_ */
