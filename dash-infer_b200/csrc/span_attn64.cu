// b200spark — SpanAttention for head_size 64 (bf16 KV): the geometry of BASELINE.json's parity anchor C0 (Qwen2-0.5B: 14
// q-heads / 2 kv-heads of 64).  The reference's GPU library supports head_size 128 only (span_attention.hpp:203-208); its CPU
// path (csrc/core/kernel/cpu/mha.cpp:595-829) runs any head size, and C0 is the CPU-parity configuration — so this path exists
// for parity, not for speed: one CTA per (sequence, kv-head), one warp per q-head, 32 tokens per step (lane = token for the
// scores, lane = 2 dims for the output), online softmax in fp32, CUDA cores only.  Small models at short context are
// launch-bound anyway (SURVEY.md §8d: C0 is "parity only").
#include "b2_common.cuh"

namespace b2 {

struct Attn64Params {
  __nv_bfloat16* out;
  const __nv_bfloat16* q;
  const void* const* k_spans;
  const void* const* v_spans;
  const int32_t* lens;
  int n_heads, n_groups, hpg, span_len, span_shift, max_spans;
  float scale_log2;
};

__global__ void __launch_bounds__(128) span_attn64_kernel(const Attn64Params p) {
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.x / p.n_groups, g = blockIdx.x - b * p.n_groups;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int len = p.lens[b];
  const void* const* ktab = p.k_spans + (size_t)b * p.max_spans;
  const void* const* vtab = p.v_spans + (size_t)b * p.max_spans;
  for (int hh = warp; hh < p.hpg; hh += 4) {
    const int h = g * p.hpg + hh;
    const __nv_bfloat16* qr = p.q + ((size_t)b * p.n_heads + h) * 64;
    float qv[64];
#pragma unroll
    for (int d = 0; d < 64; d += 2) {
      const uint32_t w = *reinterpret_cast<const uint32_t*>(qr + d);
      qv[d] = bf16_lo(w);
      qv[d + 1] = bf16_hi(w);
    }
    float m = -INFINITY, l = 0.f, o0 = 0.f, o1 = 0.f;
    for (int t0 = 0; t0 < len; t0 += 32) {
      const int tok = t0 + lane;
      float s = -INFINITY;
      if (tok < len) {
        const __nv_bfloat16* kr = reinterpret_cast<const __nv_bfloat16*>(ktab[tok >> p.span_shift]) +
                                  ((size_t)g * p.span_len + (tok & (p.span_len - 1))) * 64;
        float acc = 0.f;
#pragma unroll
        for (int d = 0; d < 64; d += 8) {
          const uint4 kv = *reinterpret_cast<const uint4*>(kr + d);
          acc += qv[d] * bf16_lo(kv.x) + qv[d + 1] * bf16_hi(kv.x) + qv[d + 2] * bf16_lo(kv.y) + qv[d + 3] * bf16_hi(kv.y) +
                 qv[d + 4] * bf16_lo(kv.z) + qv[d + 5] * bf16_hi(kv.z) + qv[d + 6] * bf16_lo(kv.w) + qv[d + 7] * bf16_hi(kv.w);
        }
        s = acc * p.scale_log2;
      }
      float mx = s;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      const float mnew = fmaxf(m, mx);
      const float corr = exp2f(m - mnew);
      const float pr = tok < len ? exp2f(s - mnew) : 0.f;
      float ps = pr;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, o);
      l = l * corr + ps;
      o0 *= corr;
      o1 *= corr;
      m = mnew;
      const int nt = min(32, len - t0);
      for (int j = 0; j < nt; ++j) {  // lane owns output dims 2*lane, 2*lane+1: the V row read is one coalesced 128 bytes
        const float pj = __shfl_sync(0xffffffffu, pr, j);
        const int tj = t0 + j;
        const __nv_bfloat16* vr = reinterpret_cast<const __nv_bfloat16*>(vtab[tj >> p.span_shift]) +
                                  ((size_t)g * p.span_len + (tj & (p.span_len - 1))) * 64;
        const uint32_t w = *reinterpret_cast<const uint32_t*>(vr + 2 * lane);
        o0 += pj * bf16_lo(w);
        o1 += pj * bf16_hi(w);
      }
    }
    const float inv = 1.f / l;
    *reinterpret_cast<uint32_t*>(p.out + ((size_t)b * p.n_heads + h) * 64 + 2 * lane) = pack_bf16x2(o0 * inv, o1 * inv);
  }
}

struct Append64Params {
  void* const* k_spans;
  void* const* v_spans;
  __nv_bfloat16* q_out;
  const __nv_bfloat16* qkv;
  const int32_t* old_lens;
  int batch, n_heads, n_groups, span_len, span_shift, max_spans;
  int rope, rotary_dim;
  float log2_base;
};

// one warp per (sequence, head slot), 2 values per lane; NeoX rotate-half over the first rotary_dim (64 or 32) dims
__global__ void __launch_bounds__(128) cache_append64_kernel(const Append64Params p) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int slots = p.n_heads + 2 * p.n_groups;
  const int wid = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (wid >= p.batch * slots) return;
  const int b = wid / slots, slot = wid - b * slots;
  const uint32_t raw = *reinterpret_cast<const uint32_t*>(p.qkv + ((size_t)b * slots + slot) * 64 + lane * 2);
  float x[2] = {bf16_lo(raw), bf16_hi(raw)};
  const int pos = p.old_lens[b];
  const bool is_v = slot >= p.n_heads + p.n_groups;
  if (p.rope && !is_v) {
    const int half = p.rotary_dim >> 1;  // 32 or 16 dims = 16 or 8 lanes
    float other[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) other[i] = __shfl_xor_sync(0xffffffffu, x[i], half >> 1);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int d = lane * 2 + i;
      if (d < p.rotary_dim) {
        const int fi = d % half;
        const float inv = exp2f(-p.log2_base * (2.0f * fi / (float)p.rotary_dim));
        float sn, cs;
        sincosf((float)pos * inv, &sn, &cs);
        x[i] = __bfloat162float(__float2bfloat16(d < half ? x[i] * cs - other[i] * sn : x[i] * cs + other[i] * sn));
      }
    }
  }
  const uint32_t pk = pack_bf16x2(x[0], x[1]);
  if (slot < p.n_heads) {
    *reinterpret_cast<uint32_t*>(p.q_out + ((size_t)b * p.n_heads + slot) * 64 + lane * 2) = pk;
    return;
  }
  const int g = is_v ? slot - p.n_heads - p.n_groups : slot - p.n_heads;
  void* const* tab = (is_v ? p.v_spans : p.k_spans) + (size_t)b * p.max_spans;
  __nv_bfloat16* span = reinterpret_cast<__nv_bfloat16*>(tab[pos >> p.span_shift]);
  *reinterpret_cast<uint32_t*>(span + ((size_t)g * p.span_len + (pos & (p.span_len - 1))) * 64 + lane * 2) = pk;
}

int span_attn64_run(const b2_span_cfg* c, void* out, const void* q, const void* const* k_spans, const void* const* v_spans,
                    const int32_t* lens, int batch, float qk_scale, cudaStream_t stream) {
  Attn64Params p;
  p.out = (__nv_bfloat16*)out; p.q = (const __nv_bfloat16*)q; p.k_spans = k_spans; p.v_spans = v_spans; p.lens = lens;
  p.n_heads = c->n_heads; p.n_groups = c->n_groups; p.hpg = c->n_heads / c->n_groups;
  p.span_len = c->span_len; p.span_shift = ilog2(c->span_len); p.max_spans = c->max_spans_per_seq;
  p.scale_log2 = qk_scale * 1.4426950408889634f;
  cudaError_t e = launch(span_attn64_kernel, dim3(batch * c->n_groups), dim3(128), 0, stream, true, p);
  if (e != cudaSuccess) {
    set_last_error("span_attn64 launch", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

int span_append64_run(const b2_span_cfg* c, void* const* k_spans, void* const* v_spans, void* q_out, const void* qkv,
                      const int32_t* old_lens, int batch, const b2_rope_cfg* rope, cudaStream_t stream) {
  if (rope && rope->rotary_dim != 64 && rope->rotary_dim != 32) return B2_ERR_UNSUPPORTED;
  Append64Params p;
  p.k_spans = k_spans; p.v_spans = v_spans; p.q_out = (__nv_bfloat16*)q_out; p.qkv = (const __nv_bfloat16*)qkv; p.old_lens = old_lens;
  p.batch = batch; p.n_heads = c->n_heads; p.n_groups = c->n_groups; p.span_len = c->span_len; p.span_shift = ilog2(c->span_len);
  p.max_spans = c->max_spans_per_seq;
  p.rope = rope ? 1 : 0; p.rotary_dim = rope ? rope->rotary_dim : 0; p.log2_base = rope ? log2f(rope->base) : 0.f;
  const int warps = batch * (c->n_heads + 2 * c->n_groups);
  cudaError_t e = launch(cache_append64_kernel, dim3((warps + 3) / 4), dim3(128), 0, stream, true, p);
  if (e != cudaSuccess) {
    set_last_error("cache_append64 launch", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

}  // namespace b2
