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
 *   b2_qk_rmsnorm, b2_span_cache_append_qknorm
 *                         QKLayerNormNoBeta (Qwen3, qwen_v30.py)  csrc/core/kernel/cuda/layernorm.cu:259-304
 *   b2_rotary_table, b2_span_cache_append_rope_table
 *                         Rotary with a [batch, head/2] inverse-frequency table  kernel/cuda/rotary.cu:24-80 (static tables)
 *   b2_sample             gen_sample_gpu (top-k, top-p, temperature, Philox draw)
 *                           csrc/core/operator/generate_opt/generate/generate_impl_gpu.hpp:116-191
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
/* CTAs per thread-block cluster of the batch 17..64 path's k-slices (planned on first use): S when the slices of an
 * n-group sum their partial tiles in distributed shared memory, 1 when they go through the workspace or there are none. */
int b2_gemm_wq_tc_cluster(b2_gemm_wq_t handle);

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
 * rope: optional fused rotary (over the first rotary_dim dims, position = old_lens[b], pairing as rope->style); pass NULL
 * when the graph has a separate Rotary op.  Quantised modes follow QuantParam<I8/U4>::Builder
 * (span-attention/src/cache_quant/impl_i8.cuh:106-140, impl_u4.cuh:146-182) with IEEE division; B2_KV_FP8 quantizes as
 * described at its enum. */
typedef struct {
  float base;          /* e.g. 1e6 for Qwen2 */
  int32_t rotary_dim;  /* <= head_size, even */
  int32_t style;       /* B2_ROPE_NEOX or B2_ROPE_INTERLEAVED */
} b2_rope_cfg;
/* Pairing styles of the rotary (b2_rope_cfg.style).  Dims d >= rotary_dim are never touched.
 *   B2_ROPE_NEOX (0): rotate-half (Qwen2, Llama).  With half = rotary_dim / 2, dim d < rotary_dim uses frequency index
 *     f = d % half and partner d + half (d < half: the "first half" expression) or d - half ("second half").  Computed
 *     frequencies: inv = exp2f(-log2f(base) * (2f / rotary_dim)), ang = fl32(pos * inv), sn, cs = sincosf(ang),
 *     first half: y = FT(x[d] cs - x[partner] sn), second half: y = FT(x[d] cs + x[partner] sn), one FT rounding
 *     (whether the products fuse into an fma is the compiler's choice, the same in both styles).
 *   B2_ROPE_INTERLEAVED (1): GPT-J / ChatGLM "half_inner" pairs (x[2i], x[2i+1]) at frequency i.  Dim d < rotary_dim uses
 *     f = d / 2 and partner d ^ 1; even d takes the "first half" expression, odd d the "second half" one.  Every other
 *     instruction is that of the NeoX form of the same entry point (angle, sincosf, attn_factor, products, fma, rounding),
 *     so with P the permutation that de-interleaves the first rotary_dim dims of a head (evens, then odds) and keeps the
 *     rest: interleaved(x) = P^-1 neox(P x), bit for bit (q_out, span rows, and quantized {zero, scale} and codes after P^-1).
 *     A lane of the append holds 4 consecutive dims, so the pair is in one lane: no shuffle.
 * Every entry point that takes a b2_rope_cfg honours style; a style outside {0, 1} is B2_ERR_PARAM and B2_ROPE_INTERLEAVED
 * on the head-64 append is B2_ERR_UNSUPPORTED, before any launch. */
enum { B2_ROPE_NEOX = 0, B2_ROPE_INTERLEAVED = 1 };
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

/* ---- Per-head Q/K RMSNorm (Qwen3: the reference's QKLayerNormNoBeta operator, qwen_v30.py; arithmetic of its
 * batch_layernorm_nobeta_kernel, layernorm.cu:259-304).  Head 128 only.  For each q head and each k head of a row, with x
 * the 128 stored FT values of that head:
 *   ss = sum x^2 in fp32: each lane of a warp sums its 4 consecutive squares in order, then an xor butterfly over
 *        16, 8, 4, 2, 1 (a fixed order, so results are deterministic);
 *   rs = rsqrtf(ss * (1/128) + eps);   y = FT((x * rs) * gamma), one FT rounding.
 * q heads use q_gamma, k heads k_gamma (both shared by all heads of their kind). */
typedef struct {
  const void* q_gamma; /* [head_size] FT, 8-byte aligned */
  const void* k_gamma; /* [head_size] FT, 8-byte aligned */
  float eps;
  int32_t reserved;
} b2_qk_norm;
/* b2_span_cache_append / _tokens / _tree with the per-head norm applied to the q and k rows as they are loaded, before the
 * fused rotary (which rounds to FT again, as without the norm); V rows are stored as given.  parents == NULL: the
 * single-token form (q_len 1) or the chain form (q_len > 1); otherwise the tree form.  The span bytes, {zero, scale} and
 * q_out equal those of b2_qk_rmsnorm followed by the matching entry point without the norm, bit for bit.  NULL norm or
 * gamma: B2_ERR_PARAM; a misaligned gamma or head_size != 128: B2_ERR_UNSUPPORTED; q_len and batch as the other appends. */
int b2_span_cache_append_qknorm(const b2_span_cfg* cfg, void* const* k_spans, void* const* v_spans, void* q_out,
                                const void* qkv, const int32_t* old_lens, const int32_t* parents, int batch, int q_len,
                                const b2_rope_cfg* rope, const b2_qk_norm* norm, void* stream);

/* ---- Scaled rotary (YaRN, Llama-3.1 "llama3", linear, or any other per-frequency scaling): the rotary reads its inverse
 * frequencies from a caller-given table instead of computing base^(-2f / rotary_dim).  The table IS the caller's definition
 * of the scaling: the library never computes frequencies for this form (b200spark.ops.rope_table builds the published
 * Hugging Face tables on the host).  Head 128 only.  With half = rotary_dim / 2 and, for row b, inv = inv_freq + b * stride
 * (stride 0: one row shared by every sequence; otherwise one row per sequence, the [batch, rotary_dim / 2] layout of the
 * reference's Rotary op), each q and k head dim d < rotary_dim, f = d % half, is computed in fp32 as
 *   ang = fl32(pos * inv[f]);  sn, cs = sincosf(ang);  c = fl32(cs * attn_factor);  s = fl32(sn * attn_factor);
 *   d < half:  t = fl32(x[d + half] * s),  y = FT(fma(x[d], c, -t));
 *   d >= half: t = fl32(x[d - half] * s),  y = FT(fma(x[d], c, t)),   one FT rounding.
 * B2_ROPE_INTERLEAVED: f = d / 2; even d: t = fl32(x[d + 1] * s), y = FT(fma(x[d], c, -t)); odd d: t = fl32(x[d - 1] * s),
 * y = FT(fma(x[d], c, t)) (the pairing rule at b2_rope_cfg).
 * attn_factor is YaRN's mscale (Hugging Face scales the cos / sin caches, so both q and k); 1.0 leaves cs and sn unchanged. */
typedef struct {
  const float* inv_freq; /* fp32 [rows][stride] (>= rotary_dim / 2 per row), device, 16-byte aligned, stride % 4 == 0 */
  int64_t stride;        /* floats between the rows of consecutive sequences; 0 = one shared row */
  float attn_factor;
  int32_t reserved;
} b2_rope_table;
/* b2_span_cache_append / _tokens / _tree (parents and q_len as b2_span_cache_append_qknorm) with the rotary at the same
 * positions (old_lens[b] + t, or old_lens[b] + depth(t) in the tree form) computed from the table; the row of token (b, t)
 * is the table row of sequence b.  norm: the per-head Q/K RMSNorm before the rotary, or NULL.  The span bytes, {zero, scale}
 * and q_out equal those of b2_rotary_table (same table, per-token rows) followed by the entry point without rotary, bit for
 * bit.  Errors: NULL rope, table or inv_freq, stride < 0, or 0 < stride < rotary_dim / 2: B2_ERR_PARAM; inv_freq not
 * 16-byte aligned or stride % 4 != 0, rotary_dim other than 128 or 64, head_size != 128: B2_ERR_UNSUPPORTED; norm as in
 * b2_span_cache_append_qknorm; q_len and batch as the other appends.  rope->base is not read. */
int b2_span_cache_append_rope_table(const b2_span_cfg* cfg, void* const* k_spans, void* const* v_spans, void* q_out,
                                    const void* qkv, const int32_t* old_lens, const int32_t* parents, int batch, int q_len,
                                    const b2_rope_cfg* rope, const b2_rope_table* table, const b2_qk_norm* norm,
                                    void* stream);

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
/* in-place rotary (pairing rope->style) on the q and k heads of qkv [batch, (nH+2nG)*head]; position = pos[b] */
int b2_rotary(void* qkv, const int32_t* pos, int batch, int n_heads, int n_groups, int head_size,
              const b2_rope_cfg* rope, void* stream);
/* b2_rotary with the frequencies of a b2_rope_table (arithmetic and errors there; row b of qkv uses inv_freq + b * stride),
 * in place, ft = B2_DT_BF16 or B2_DT_F16 (else B2_ERR_UNSUPPORTED); V heads and dims >= rotary_dim are left as they are. */
int b2_rotary_table(void* qkv, const int32_t* pos, int batch, int n_heads, int n_groups, int head_size,
                    const b2_rope_cfg* rope, const b2_rope_table* table, int ft, void* stream);
/* QKLayerNormNoBeta (arithmetic: b2_qk_norm): x, y [rows, ld] FT.  Per row, heads [0, n_heads) and [n_heads,
 * n_heads + n_groups) are normalised; the V heads [n_heads + n_groups, n_heads + 2 n_groups) are copied unless y == x; the
 * columns beyond are untouched.  y may be x (any other overlap is undefined).  head_size 128 and ft B2_DT_BF16 / B2_DT_F16
 * (else B2_ERR_UNSUPPORTED); ld >= (n_heads + 2 n_groups) * 128 (else B2_ERR_PARAM); x, y and the gammas 8-byte aligned and
 * ld a multiple of 4 (else B2_ERR_UNSUPPORTED). */
int b2_qk_rmsnorm(void* y, const void* x, int rows, int64_t ld, int n_heads, int n_groups, int head_size,
                  const b2_qk_norm* norm, int ft, void* stream);
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
/* Log-probabilities of the decode step (logprobs / top_logprobs of a greedy step), on the device, CUDA-graph replayable.
 * A row runs on one CTA, or on a cluster of 8 CTAs when n > 32768 (a function of n alone: the same bits at every batch).
 * logits FT [rows, ld] (ft = B2_DT_BF16 / B2_DT_F16), the first n columns of each row; columns n .. ld-1 are ignored.  Per
 * row, with every value widened to fp32 exactly:
 *   m = the row maximum;  s = sum_i expf(x_i - m) in fp32;  lp_i = (x_i - m) - logf(s)  (lse = m + logf(s)).
 *   top_ids[r][k], top_lp[r][k] (k < n_top, 0 <= n_top <= B2_MAX_TOP_LOGPROBS): the first n_top entries in argmax order (NaN
 *   first, then descending value, the lower index on ties), so top_ids[r][0] == ids_out[r] == b2_argmax's id bit for bit.
 *   When n_top > n the slots past n hold id -1 and lp -inf.
 *   tok_lp[r] = lp at tok_ids[r] when tok_ids is given, else at the top-1.  An id outside [0, n) gives NaN (never read).
 * Non-finite rows follow torch.log_softmax(x.double()) cast to fp32: a NaN or a +inf anywhere makes every lp of the row NaN,
 * an all -inf row gives NaN, -inf entries of a row with a finite maximum give -inf.  The ids follow argmax order all the same.
 * Accuracy, per element against log_softmax of the widened row in fp64, for a row of finite maximum:
 *   |lp_i - exact| <= (1 + u)(u |x_i - m| + dL) + u |exact|,  u = 2^-24,
 *   dL = -log(1 - e_s) + 2^-23 (|L| - log(1 - e_s)),  L = log(sum_i exp(x_i - m)),
 *   e_s = (sum_i t_i ((1 + 2^-22) exp(u |x_i - m|) (1 + u)^d - 1) + n 2^-148 (1 + u)^d) / sum_i t_i,  t_i = exp(x_i - m),
 * with d = ceil(n / (1024 C)) + 8 + C additions on a term's way into s, C the CTAs of the row (expf's 2 ulp, the
 * rounding of x_i - m, the sum, logf's ulp and the final subtraction); the merge adds, per rank, the rounding of m_q - M
 * and expf's 2 ulp on that rank's scale, and its
 * fused multiply-add.  A result beyond the fp32 range is -inf.  The reduction order is fixed and there are no atomics:
 * results are bitwise repeatable.  Unlike the reference, whose logprobs are rounded to FT before its top-k
 * (generate_impl_gpu.hpp:46-64), these are fp32.
 * n_top outside [0, 10], n < 1, ld < n, top_ids / top_lp NULL with n_top > 0 or given with n_top == 0, or no output at all:
 * B2_ERR_PARAM, before any launch. */
#define B2_MAX_TOP_LOGPROBS 10 /* the reference's engine_max_top_logprobs */
int b2_logprobs(int64_t* ids_out /* [rows] or NULL */, float* tok_lp /* [rows] or NULL */, int64_t* top_ids, float* top_lp,
                const int64_t* tok_ids /* [rows] or NULL */, const void* logits, int rows, int n, int64_t ld, int n_top, int ft,
                void* stream);
/* Vocab-split form (tensor parallel).  b2_logprobs_shard writes one record of b2_logprobs_partial_bytes(n_top) bytes per row
 * (partials [rows][bytes], 4-byte aligned): the shard's m and s, its top max(n_top, 1) (value, id + id_offset) padded with
 * (-inf, INT_MAX), and the token's logit when tok_ids[r] lies in [id_offset, id_offset + n).  The records are opaque bytes
 * (b2_allgather moves them unchanged).  id_offset >= 0 and id_offset + n < INT_MAX (else B2_ERR_PARAM).
 * b2_logprobs_merge takes all_partials [nranks][rows][bytes] and writes b2_logprobs' outputs over the whole vocabulary:
 *   M = max_q m_q,  S = sum_q s_q expf(m_q - M) in rank order (shards with m_q = -inf add nothing),  lp = (x - M) - logf(S);
 * the top list is taken over the nranks x max(n_top, 1) candidates in argmax order (the lowest id, i.e. the lowest rank, on
 * ties).  One shard of the whole row followed by the merge equals b2_logprobs bit for bit. */
size_t b2_logprobs_partial_bytes(int n_top); /* 0 for n_top outside [0, 10] */
int b2_logprobs_shard(void* partials, const int64_t* tok_ids /* or NULL */, const void* logits, int rows, int n, int64_t ld,
                      int64_t id_offset, int n_top, int ft, void* stream);
int b2_logprobs_merge(int64_t* ids_out, float* tok_lp, int64_t* top_ids, float* top_lp, const void* all_partials, int nranks,
                      int rows, int n_top, void* stream);
/* Sampling of the decode step (temperature, top-k, top-p; gen_sample_gpu, generate_impl_gpu.hpp:116-191), on the device,
 * CUDA-graph replayable.  ids_out[r] = a token drawn from row r of logits [rows, ld] FT (ft = B2_DT_BF16 / B2_DT_F16, the
 * first n columns).  temperature, top_p: fp32 [rows]; top_k: int32 [rows]; seeds, offsets: uint64 [rows]; all
 * device-resident, so a captured graph picks up values the caller writes between replays.  offsets[r] += 1 for every row,
 * every call.  Per row, with every logit widened to fp32 exactly:
 *   1. Greedy rows take b2_argmax's id bit for bit: the row maximum m not finite (a NaN, a +inf, or every entry -inf),
 *      temperature NaN or <= 0, or c = __fdiv_rn(LOG2E_F32, temperature) not finite (LOG2E_F32 = 0x3FB8AA3B).  The ids
 *      always lie in [0, n).
 *   2. Order: by value, highest first, the lower id first among equal values; -0 and +0 are equal.
 *   3. Weights: W_i = 0 for x_i = -inf, else W_i = __float2ull_rn(ex2.approx.ftz(fl32(fl32(x_i - m) c)) 2^40), an integer
 *      <= 2^40; the maximum has W = 2^40.  temperature = +inf gives c = 0: uniform over the finite entries.  A token below
 *      about 2^-41 of the maximum's probability has weight 0 and is never drawn.
 *   4. Top-k: k = top_k[r] (k <= 0 or k > n: n); the kept set is the first k elements in the order (ties at the boundary
 *      split by id); S_k = the sum of their W (< 2^58).
 *   5. Top-p: p24 = clamp(__float2uint_rn(top_p 2^24), 0, 2^24) (NaN or >= 1: 2^24); Pt = max(1, ceil(p24 S_k / 2^24)) in
 *      exact 128-bit arithmetic; the nucleus is the shortest prefix of the kept set, in the order, whose W sum is at least
 *      Pt (it always holds the maximum); S_p = its sum.
 *   6. Draw: (r0, r1, r2, r3) = Philox4x32-10(counter = (lo32(off), hi32(off), 0, 0), key = (lo32(seed), hi32(seed))),
 *      off = offsets[r] before the increment; u24 = r0 >> 8; U = floor(u24 S_p / 2^24) (0 <= U < S_p).  The drawn id is the
 *      first element of the nucleus, in the order, at which the running W sum exceeds U (zero-weight elements are never
 *      drawn).  The row index is not part of the counter: equal seeds, offsets and logits draw the same token at any batch
 *      position and batch size.
 * Everything after step 3 is integer arithmetic, so no summation order can change a result.  A row runs on one CTA, or on
 * a cluster of 8 when n > 32768.
 * n < 1, ld < n, rows < 0, a NULL pointer, ft other than bf16 / fp16: B2_ERR_PARAM; n > B2_SAMPLE_MAX_N: B2_ERR_LIMIT; all
 * before any launch.  No workspace. */
#define B2_SAMPLE_MAX_N 262144
int b2_sample(int64_t* ids_out, const void* logits, int rows, int n, int64_t ld, const float* temperature,
              const int32_t* top_k, const float* top_p, const uint64_t* seeds, uint64_t* offsets, int ft, void* stream);
/* The step form of b2_sample, for sampled verification of a multi-token or tree step.  logits [batch q_len, ld] FT; row
 * r = b q_len + t is draft node t of sequence b (tree format: b2_span_cache_append_tree; parents NULL: a chain).  Row r is
 * drawn by b2_sample's steps 1-6 with sequence b's parameters temperature[b], top_k[b], top_p[b], seeds[b] (all [batch])
 * and the counter off = offsets[b] + depth(t), depth(t) the parent steps from node t to the root (t for a chain): ids_out[r]
 * equals b2_sample's id for that row at offsets[b] = off, bit for bit.  The offsets are read, not written; q_len = 1 gives
 * b2_sample's ids without advancing them.  Same per-row decomposition as b2_sample (one CTA, or a cluster of 8 above 32768
 * columns).  A NULL required pointer, n < 1, ld < n, batch < 0, ft other than bf16 / fp16: B2_ERR_PARAM; q_len outside
 * [1, 16] or n > B2_SAMPLE_MAX_N: B2_ERR_LIMIT; all before any launch.  batch = 0 launches nothing. */
int b2_sample_tokens(int64_t* ids_out, const void* logits, int batch, int q_len, const int32_t* parents /* NULL: chain */,
                     int n, int64_t ld, const float* temperature, const int32_t* top_k, const float* top_p,
                     const uint64_t* seeds, const uint64_t* offsets, int ft, void* stream);
/* b2_sample under tensor parallelism: the rows' columns are split over the ranks of a vocab-split lm_head, and every rank
 * draws b2_sample's id of the whole row by exchanging small per-row records instead of the logits.  Rank q of P
 * (1 <= P <= 8) holds columns [id_offset_q, id_offset_q + n_q) of a row of n_total columns (n_q >= 1): the ranges are
 * contiguous, ascend with the rank and together cover [0, n_total); they may be unequal.  Every rank passes the same
 * temperature, top_k, top_p, seeds and offsets ([rows] each, its own device copies); top_k is read against n_total
 * (k <= 0 or k > n_total: n_total).
 * Result: ids_out[r] on every rank equals b2_sample's id of the concatenated row at the same offset, bit for bit (all of
 * its steps 1-6, greedy rows included, whose id is b2_argmax's of the whole row), and every rank's offsets[r] advances by
 * exactly 1.
 * Protocol, per row: phases p = 0 .. B2_SAMPLE_SHARD_PHASES - 1 in order, each followed by an all-gather of its records
 * (record_out [rows][b2_sample_shard_record_bytes(p)] on each rank -> all_records [nranks][rows][bytes] in rank order,
 * opaque bytes: b2_allgather or an NCCL all-gather moves them unchanged), then b2_sample_shard_merge.  Phase p >= 1 reads
 * the all-gathered records of phase p - 1 (all_records; NULL for phase 0).  state [rows][b2_sample_shard_state_bytes()]
 * is this rank's own memory, written and read by the phases in turn and never exchanged: every rank derives the same
 * values from the same records.
 *   0  reads the shard: its argmax under b2_argmax's order (value, global id)                        record 8 B
 *   1  the row's m, c, greedy predicate and argmax; the shard's level-1 histogram (high byte of the key: counts and
 *      weight sums at the row's m and c)                                                            record 3072 B
 *   2  the row's level 1; with k < n_total the k-th element's high byte; the shard's level-2 counts in it   1024 B
 *   3  S_k; the top-p target Pt and its high byte; the shard's level-2 counts in it                        1024 B
 *   4  S_p; the draw's U (offsets[r] read here) and its high byte; the shard's level-2 counts in it        1024 B
 *   5  the drawn key K and its rank j among K's elements; the rank holding the j-th writes its id, the others -1   8 B
 *   merge: ids_out[r] = the holder's id (the argmax for a greedy row); offsets[r] += 1.
 * A greedy row, or one without a top-k or top-p limit, passes through the phases with an empty record, so the launch
 * sequence is static (a CUDA graph captures it).  The records depend only on the row, the parameters and the split.
 * Errors, all before any launch: a NULL pointer (all_records may be NULL for phase 0 only), nranks outside [1, 8],
 * rows < 0, n < 1, ld < n, id_offset < 0, id_offset + n > n_total, ft other than bf16 / fp16, or a phase out of range:
 * B2_ERR_PARAM; n_total > B2_SAMPLE_MAX_N: B2_ERR_LIMIT.  rows = 0 launches nothing.  One 1024-thread CTA per row and
 * phase; the merge reads state and offsets of its own rank. */
#define B2_SAMPLE_SHARD_PHASES 6
size_t b2_sample_shard_record_bytes(int phase); /* bytes per row; 0 for a phase out of range */
size_t b2_sample_shard_state_bytes(void);       /* bytes per row of the rank-local state */
int b2_sample_shard(int phase, void* record_out, void* state, const void* all_records /* NULL for phase 0 */, int nranks,
                    const void* logits, int rows, int n, int64_t ld, int64_t id_offset, int64_t n_total,
                    const float* temperature, const int32_t* top_k, const float* top_p, const uint64_t* seeds,
                    const uint64_t* offsets, int ft, void* stream);
int b2_sample_shard_merge(int64_t* ids_out, const void* all_records, const void* state, int nranks, int rows,
                          uint64_t* offsets, void* stream);
/* Per-sequence token history on the device (the in_ids / cur_len / input_len of the reference's logits processor).  Every
 * array has `rows` slots (row r of a step uses slot r); all pointers are device memory, zero-initialised before first use.
 *   tokens     int32 [rows][max_len]  the sequence, prompt first; an id outside [0, vocab) is stored as -1
 *   len        int32 [rows]           cur_len: the tokens held (prompt included)
 *   prompt_len int32 [rows]           input_len: positions < prompt_len are the prompt
 *   table      int32 [rows][vocab]    per id: bit 30 = occurs in the prompt, bits 0..29 = occurrences at positions
 *                                     >= prompt_len (the generated count); 0 for an id that does not occur
 *   distinct   int32 [rows][max_len]  the ids whose table entry is not 0, each once, in no particular order
 *   n_distinct int32 [rows]
 * max_len < 2^30.  The processor reads the table and the distinct list, so its work per row follows the distinct ids, not
 * the vocabulary. */
typedef struct b2_token_history {
  int32_t* tokens;
  int32_t* len;
  int32_t* prompt_len;
  int32_t* table;
  int32_t* distinct;
  int32_t* n_distinct;
  int32_t max_len;
  int32_t vocab;
} b2_token_history;
/* Load slot `slot` with ids[0 .. n_ids) (device int32, each in [0, vocab), n_ids <= max_len), the first prompt_len of them
 * the prompt (0 <= prompt_len <= n_ids).  The table entries of the slot's previous ids are cleared first, through its
 * distinct list (no vocab-wide clear).  n_ids = 0 empties the slot.  One CTA; the other slots are untouched. */
int b2_history_load(const b2_token_history* hist, int slot, const int32_t* ids, int n_ids, int prompt_len, void* stream);
/* Append ids[r] (int64, device) to slot r for r < rows, on the device (CUDA-graph replayable: each replay appends once).  A
 * slot that holds max_len tokens is left as it is.  An id outside [0, vocab) is stored as -1 and counted nowhere. */
int b2_history_append(const b2_token_history* hist, const int64_t* ids, int rows, void* stream);
/* Append the emitted tokens of a verify step (b2_spec_accept / _tree / _sampled) to slot b for b < batch, in order:
 * pred[b][path[b][i]] (chain, path NULL: pred[b][i]) for i < accepted[b].  pred int64 [batch][q_len], accepted int32
 * [batch], path int32 [batch][q_len], all device memory.  Every array of the history ends as accepted[b] successive
 * b2_history_append calls leave it, the order of the distinct list included; a slot stops at max_len like there.
 * accepted[b] is clamped to [0, q_len] and a path entry outside [0, q_len) is read as 0, so no input reads out of bounds.
 * One thread per sequence, CUDA-graph replayable (each replay appends once).  A NULL required pointer, batch < 0 or a
 * history b2_history_append refuses: B2_ERR_PARAM; q_len outside [1, 16]: B2_ERR_LIMIT; before any launch.  batch = 0
 * launches nothing. */
int b2_history_append_tokens(const b2_token_history* hist, const int64_t* pred, const int32_t* accepted,
                             const int32_t* path /* NULL: chain */, int batch, int q_len, void* stream);
/* N-gram (prompt-lookup) drafting of a verify step from the token history, on the device (CUDA-graph replayable): the
 * drafts continue the most recent earlier occurrences of the sequence's last tokens.  For sequence b, S = hist.tokens[b][0
 * .. L), L = hist.len[b]; S[L-1] is the last emitted token, which the caller keeps equal to tokens[b][0] (DecodeStack does
 * so by construction).  tokens int64 [batch][q_len]: column 0 is read, never written.
 *   m(e), for an end position e in [0, L-2]: the number of leading i < n_max with e - i >= 0 and S[e-i] == S[L-1-i]
 *        (-1 entries compare like any id, as in b2_penalize's n-gram step).  n* = max_e m(e); n* < n_min: no match.
 *   Candidates: the `width` largest e with m(e) >= n*, most recent first.  Candidate e has period p = L-1-e and
 *        continuation c_k = S[e+1 + (k mod p)], k < q_len-1: the tokens that followed the match and, past the end of the
 *        history, the same period again, so a loop keeps being predicted.  A match therefore always fills all q_len-1
 *        drafts (prompt lookup that truncates at the end of the history drafts fewer): a verify step runs q_len rows
 *        whether they hold drafts or not.
 *   Chain (parents NULL, width == 1): tokens[b][1+k] = c_k of the candidate.
 *   Tree (parents int32 [batch][q_len], tree format: b2_span_cache_append_tree): the trie of the candidates'
 *        continuations, a node per distinct prefix, node 0 the root (the empty prefix).  Nodes are numbered breadth first;
 *        within a level by parent index, then by the rank of the first candidate that has the prefix.  The first q_len
 *        nodes are kept: tokens[b][t] = the last token of node t's prefix, parents[b][t] = its parent (always < t),
 *        parents[b][0] = 0.  Identical continuations merge, so an exact loop drafts a chain and distinct continuations
 *        branch; a candidate whose continuation equals a more recent one's still takes one of the `width` slots.
 *   Padding: drafts or nodes that no candidate fills (all of them without a match) get token tokens[b][0] and parent 0; a
 *        draft that would be -1 is written as tokens[b][0] too.  n_draft[b] (int32 [batch], may be NULL) = the drafts a
 *        candidate fills: q_len-1 for a matched chain, the kept nodes minus the root for a tree, 0 without a match.
 * Integer arithmetic only: the results are exact.  One CTA per sequence.  A NULL required pointer, batch < 0, n_min < 1,
 * n_min > n_max, width < 1, width > q_len-1 or a chain with width != 1: B2_ERR_PARAM; q_len outside [2, 16] or n_max >
 * 16: B2_ERR_LIMIT; before any launch.  batch = 0 launches nothing. */
int b2_ngram_draft(int64_t* tokens, int32_t* parents /* NULL: chain */, int32_t* n_draft /* or NULL */,
                   const b2_token_history* hist, int batch, int q_len, int n_min, int n_max, int width, void* stream);
/* Per-row parameters of b2_penalize, device arrays [rows], read at every call (a captured step uses the values last
 * written).  The neutral values repetition 1, presence 0, frequency 0, no_repeat_ngram 0, min_length 0 change nothing. */
typedef struct b2_penalty_params {
  const float* repetition;
  const float* presence;
  const float* frequency;
  const int32_t* no_repeat_ngram;
  const int32_t* min_length;
  const int32_t* eos_id;    /* < 0: none */
  const int32_t* suppress;  /* suppress_repetition_in_generation: != 0 counts only generated positions for repetition */
  const void* reserved;     /* NULL */
} b2_penalty_params;
/* The logits processor of the reference's sampling step (LogitsProcessor, beam_search.cu), in place, CUDA-graph
 * replayable.  logits FT [rows, ld] (ft = B2_DT_BF16 / B2_DT_F16) hold vocabulary ids [id_offset, id_offset + n) of the
 * rows (a vocab-split lm_head passes its shard); columns n .. ld-1 are never written, and an id outside the shard is skipped.
 * Row r reads slot r of hist: L = len[r], P = prompt_len[r], the table entry e_t of id t, c_t = its generated count.  FT(v)
 * is round-to-nearest-even of fp32 v to FT.  For every id t with e_t != 0 (the ids occurring at positions < L), once,
 * from its value x:
 *   1. Repetition (when suppress[r] == 0, or c_t > 0): with R = FT(repetition[r]),  x < 0 ? x * R : x / R  in FT
 *      arithmetic: the product is __hmul (correctly rounded); the quotient is CUDA's __hdiv of the FT type, the same
 *      instructions the reference's fast-math build runs: bf16 div.approx.f32 of the widened values (operands scaled by
 *      1/4 when |R| >= 2^126) rounded to bf16, fp16 the widened x times rcp.approx.ftz.f32(R) rounded to fp16 (one fma
 *      correction step when that result is a nonzero value below 0x008F).  Both equal the correctly rounded FT quotient
 *      except within about 2^-22 relative of a rounding midpoint.  0 and NaN take the quotient.  Skipped when R == 1.
 *   2. Frequency and presence: x = x - FT(s) (__hsub, correctly rounded), s = fl32(c_t frequency[r]) + (c_t > 0 ?
 *      presence[r] : 0), products and sums in fp32 with subnormals flushed (the reference's mul.ftz / add.ftz).  Skipped
 *      when FT(s) is +0.  Repetition comes first, as in the reference; an id is penalised once however often it occurs.
 * Then the bans, which write FT(-1e9f) (bf16 0xCE6E; fp16 -inf):
 *   3. No-repeat n-gram, g = no_repeat_ngram[r] > 0: for every j <= L - g with tokens[j + i] == tokens[L - g + 1 + i] for
 *      all i < g - 1, the id tokens[j + g - 1] (g == 1: every id of the history).  The comparison is of the stored
 *      tokens, so positions that held ids outside [0, vocab) compare as -1, equal to one another (the reference compares
 *      the raw ids); the front end never appends such an id.
 *   4. Min-length: eos_id[r] when L < min_length[r] and eos_id[r] >= 0 (L counts the prompt, as in the reference).
 * Differences from the reference, none visible to b2_argmax, b2_sample or b2_logprobs: the reference subtracts
 * FT(0 * frequency) from every column of the row, so with frequency < 0 it turns -0 into +0 in columns outside the
 * history (a non-finite frequency turns them into NaN); it writes canonical NaNs where this kernel leaves a NaN's bits
 * as they are (steps 1 and 2 are skipped at neutral values, so neutral parameters leave the row bit-identical).
 * Parameter ranges (the reference accepts repetition in [0, 2], presence and frequency in [-2, 2]) are the caller's to
 * check; the arithmetic is as stated for any value.  One CTA per row.  rows < 0, n < 1, ld < n, id_offset < 0,
 * id_offset + n > vocab, a NULL pointer or an ft other than bf16 / fp16: B2_ERR_PARAM, before any launch. */
int b2_penalize(void* logits, int rows, int n, int64_t ld, int64_t id_offset, const b2_token_history* hist,
                const b2_penalty_params* params, int ft, void* stream);
/* The logits processor of a verify step (b2_spec_accept / _tree / _sampled), in place, CUDA-graph replayable.  logits FT
 * [batch * q_len, ld]: row r = b * q_len + t is draft node t of sequence b (tree format: b2_span_cache_append_tree;
 * parents NULL: a chain).  tokens int64 [batch][q_len] is the array the append and accept kernels read; column 0 is never
 * read.  History slot b and parameter row b are sequence b's (params [batch], as in b2_sample_tokens).
 *   V(b, t): slot b (length L, prompt length P) followed by tokens[b][a_1 .. a_d], where a_1 < ... < a_d = t are the
 *   non-root nodes on the path from the root to t (d = depth(t); a chain has a_i = i; a parent outside [0, t) is read as
 *   the root), appended as b2_history_append appends: an id outside [0, vocab) is stored as -1 and counted nowhere, the
 *   appends stop at max_len (L' = min(L + d, max_len)), and the prompt length stays P, so every path token counts as
 *   generated.
 * Row (b, t) is exactly, bit for bit, b2_penalize's result for that row with slot b holding V(b, t): repetition (with
 * suppress), presence and frequency over the counts of V, the no-repeat n-gram over V (its tail may lie in the path) and
 * min-length against L'.  So a verify row is processed as the single-token step with the same context would be, and a
 * penalised speculative loop emits exactly the tokens of single-token penalised decoding.  q_len = 1 is b2_penalize on
 * batch rows.  The history is only read; columns n .. ld-1 and ids outside the shard are never written (id_offset as in
 * b2_penalize); neutral parameters leave the rows bit-identical.  One CTA per row.  A NULL required pointer, batch < 0,
 * n < 1, ld < n, id_offset < 0, id_offset + n > vocab or an ft other than bf16 / fp16: B2_ERR_PARAM; q_len outside
 * [1, 16] (or batch * q_len >= 2^31): B2_ERR_LIMIT; before any launch.  batch = 0 launches nothing. */
int b2_penalize_tokens(void* logits, int batch, int q_len, const int32_t* parents /* NULL: chain */, const int64_t* tokens,
                       int n, int64_t ld, int64_t id_offset, const b2_token_history* hist, const b2_penalty_params* params,
                       int ft, void* stream);
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
/* Sampled verification of a chain (parents and path NULL) or a draft tree.  pred [batch][q_len] = b2_sample_tokens' draws
 * of the step's rows.  The walk, the outputs and the lengths are b2_spec_accept's (chain) or b2_spec_accept_tree's (tree)
 * over these draws; then offsets[b] += accepted[b].  The step emits pred[b][0 .. n_b-1] (pred[b][path[b][i]] in a tree).
 * Exactness: a node at depth d of the accepted path is drawn at counter offsets[b] + d after the accepted prefix and the d
 * tokens drawn before it, which is the context and the counter of single-token step d.  So when every row's logits equal
 * those of the single-token steps, the emitted tokens are exactly the next n_b tokens b2_sample would draw from the same
 * seed, and the offsets end where those n_b steps leave them.  The drafts decide only how many tokens a step emits, never
 * which, so the output distribution is single-token sampling's for any drafter; a draft token of weight 0 is never
 * accepted.  With every temperature <= 0 the draws are argmax ids, and every output but the offsets equals greedy
 * verification's.  A NULL required pointer, path NULL while parents is not (or the reverse), batch < 0: B2_ERR_PARAM;
 * q_len outside [1, 16]: B2_ERR_LIMIT; before any launch.  batch = 0 launches nothing. */
int b2_spec_accept_sampled(int32_t* accepted, int32_t* path /* NULL iff parents is NULL */, int64_t* next_ids /* or NULL */,
                           int32_t* old_lens, int32_t* new_lens, int64_t* tokens, const int64_t* pred,
                           const int32_t* parents /* NULL: chain */, uint64_t* offsets, int batch, int q_len, void* stream);
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
