// b200spark — glue ops of the decode graph ("next" rows, SURVEY.md §8f): RMSNorm, rotary, binary,
// embedding lookup, greedy argmax, device-resident sequence lengths.  All bandwidth-trivial at decode;
// they exist so that a whole decode step runs without leaving the library (and the CUDA graph).
// Reference counterparts: csrc/core/kernel/cuda/layernorm.cu:86 (LayerNormNoBeta), rotary.cu:23,
// binary.cu, embedding.cu, and GenerateOp with top_k=1 (generate_impl_cpu.hpp:153-165 = argmax).
#include "b2_common.cuh"

namespace b2 {

template <bool H>
__global__ void __launch_bounds__(256) rmsnorm_kernel(__nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ x,
                                                      const __nv_bfloat16* __restrict__ gamma, int cols, float eps) {
  using F = Ft<H>;
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float red[8];
  const int row = blockIdx.x;
  const __nv_bfloat16* xr = x + (size_t)row * cols;
  float ss = 0.f;
  for (int i = threadIdx.x * 8; i < cols; i += 256 * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(xr + i);
    const float f[8] = {F::lo(v.x), F::hi(v.x), F::lo(v.y), F::hi(v.y), F::lo(v.z), F::hi(v.z), F::lo(v.w), F::hi(v.w)};
#pragma unroll
    for (int j = 0; j < 8; ++j) ss += f[j] * f[j];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  const float inv = rsqrtf(tot / (float)cols + eps);
  for (int i = threadIdx.x * 8; i < cols; i += 256 * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(xr + i);
    const uint4 gv = *reinterpret_cast<const uint4*>(gamma + i);
    uint4 o;
    o.x = F::pack(F::lo(v.x) * inv * F::lo(gv.x), F::hi(v.x) * inv * F::hi(gv.x));
    o.y = F::pack(F::lo(v.y) * inv * F::lo(gv.y), F::hi(v.y) * inv * F::hi(gv.y));
    o.z = F::pack(F::lo(v.z) * inv * F::lo(gv.z), F::hi(v.z) * inv * F::hi(gv.z));
    o.w = F::pack(F::lo(v.w) * inv * F::lo(gv.w), F::hi(v.w) * inv * F::hi(gv.w));
    *reinterpret_cast<uint4*>(y + (size_t)row * cols + i) = o;
  }
}

// ---- fp8 activations for the e4m3 wgmma GEMM (b2_gemm_wq_run_fp8): per-token dynamic scale
//   scale[r] = max(|x[r,:]|, tiny) / 448 ;  y = e4m3(x / scale) (round to nearest even, saturating)
// optional fused RMSNorm (gamma != NULL): x is first normalised exactly like rmsnorm_kernel (result rounded to bf16).
// Layout of y ("b2 fp8 activation layout"): inside every aligned group of 8 k the bytes hold k = (0,2,4,6,1,3,5,7) — the
// order in which the int4 weight image yields its nibbles (the in-word k order, wq_gemm_shared.cuh), so the GEMM's dequant needs no final byte shuffle (a dot product
// is invariant under a common permutation of k).  tile_sums[r][kt] = sum of the QUANTIZED values of k-tile kt (64 k), the
// zero-point term of the affine dequantisation (exact in fp32: multiples of 2^-9 below 2^15).
__global__ void __launch_bounds__(256) quant_fp8_kernel(uint8_t* __restrict__ y, float* __restrict__ scale, float* __restrict__ tile_sums,
                                                        const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ gamma,
                                                        int cols, int64_t ldy, int kt_count, float eps) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float red[8];
  __shared__ float red2[8];
  const int row = blockIdx.x;
  const __nv_bfloat16* xr = x + (size_t)row * cols;
  float ss = 0.f, amax = 0.f;
  for (int i = threadIdx.x * 8; i < cols; i += 256 * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(xr + i);
    const float f[8] = {bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y), bf16_lo(v.z), bf16_hi(v.z), bf16_lo(v.w), bf16_hi(v.w)};
#pragma unroll
    for (int j = 0; j < 8; ++j) { ss += f[j] * f[j]; amax = fmaxf(amax, fabsf(f[j])); }
  }
  float inv = 1.f;
  if (gamma) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) tot += red[i];
    inv = rsqrtf(tot / (float)cols + eps);
    amax = 0.f;  // the maximum of the NORMALISED row: second pass below
    for (int i = threadIdx.x * 8; i < cols; i += 256 * 8) {
      const uint4 v = *reinterpret_cast<const uint4*>(xr + i);
      const uint4 gv = *reinterpret_cast<const uint4*>(gamma + i);
      const uint32_t vv[4] = {v.x, v.y, v.z, v.w}, gg[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t o2 = pack_bf16x2(bf16_lo(vv[j]) * inv * bf16_lo(gg[j]), bf16_hi(vv[j]) * inv * bf16_hi(gg[j]));
        amax = fmaxf(amax, fmaxf(fabsf(bf16_lo(o2)), fabsf(bf16_hi(o2))));
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if ((threadIdx.x & 31) == 0) red2[threadIdx.x >> 5] = amax;
  __syncthreads();
  amax = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) amax = fmaxf(amax, red2[i]);
  const float sc = fmaxf(amax, 1e-12f) / 448.f;
  const float rs = 1.f / sc;
  if (threadIdx.x == 0) scale[row] = sc;
  // one thread per aligned group of 8 k; 8 consecutive threads = one 64-k tile
  const int kend = (kt_count * 64 + 255) & ~255;  // whole warps stay in the loop (shuffles below)
  for (int i = threadIdx.x * 8; i < kend; i += 256 * 8) {
    float f[8];
    if (i < cols) {
      const uint4 v = *reinterpret_cast<const uint4*>(xr + i);
      const uint32_t vv[4] = {v.x, v.y, v.z, v.w};
      if (gamma) {
        const uint4 gv = *reinterpret_cast<const uint4*>(gamma + i);
        const uint32_t gg[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t o2 = pack_bf16x2(bf16_lo(vv[j]) * inv * bf16_lo(gg[j]), bf16_hi(vv[j]) * inv * bf16_hi(gg[j]));
          f[2 * j] = bf16_lo(o2); f[2 * j + 1] = bf16_hi(o2);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) { f[2 * j] = bf16_lo(vv[j]); f[2 * j + 1] = bf16_hi(vv[j]); }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = 0.f;
    }
    // e4m3 pairs: cvt packs (hi, lo) -> 16 bits; byte order (0,2,4,6,1,3,5,7)
    uint16_t p02, p46, p13, p57;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(p02) : "f"(f[2] * rs), "f"(f[0] * rs));
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(p46) : "f"(f[6] * rs), "f"(f[4] * rs));
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(p13) : "f"(f[3] * rs), "f"(f[1] * rs));
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(p57) : "f"(f[7] * rs), "f"(f[5] * rs));
    const uint32_t w0 = (uint32_t)p02 | ((uint32_t)p46 << 16), w1 = (uint32_t)p13 | ((uint32_t)p57 << 16);
    if (i < cols) *reinterpret_cast<uint2*>(y + (size_t)row * ldy + i) = make_uint2(w0, w1);
    // sum of the quantized values (decode them back: the GEMM multiplies exactly these)
    float qs = 0.f;
    {
      const uint16_t pp[4] = {p02, p46, p13, p57};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint32_t h2;
        asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"(pp[j]));
        const __half2 hh = *reinterpret_cast<const __half2*>(&h2);
        qs += __low2float(hh) + __high2float(hh);
      }
    }
    qs += __shfl_xor_sync(0xffffffffu, qs, 1);
    qs += __shfl_xor_sync(0xffffffffu, qs, 2);
    qs += __shfl_xor_sync(0xffffffffu, qs, 4);
    if ((threadIdx.x & 7) == 0 && (i >> 6) < kt_count) tile_sums[(size_t)row * kt_count + (i >> 6)] = qs;
  }
}

// in-place rotary on the q and k heads: one warp per (sequence, head); RS: the pairing style (b2_rope_cfg.style)
template <int RS>
__device__ __forceinline__ void rotary_row(__nv_bfloat16* __restrict__ qkv, const int32_t* __restrict__ pos, int batch,
                                           int n_heads, int n_groups, int rotary_dim, float log2_base) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int rot_heads = n_heads + n_groups;
  const int slots = n_heads + 2 * n_groups;
  const int wid = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (wid >= batch * rot_heads) return;
  const int b = wid / rot_heads, h = wid - b * rot_heads;
  __nv_bfloat16* ptr = qkv + ((size_t)b * slots + h) * 128 + lane * 4;
  const uint2 raw = *reinterpret_cast<const uint2*>(ptr);
  float x[4] = {bf16_lo(raw.x), bf16_hi(raw.x), bf16_lo(raw.y), bf16_hi(raw.y)};
  const int half = rotary_dim >> 1;
  float other[4];
  rope_partners<RS>(x, other, half);
  const int ps = pos[b];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int d = lane * 4 + i;
    if (d < rotary_dim) {
      const int fi = RS == B2_ROPE_NEOX ? d % half : d >> 1;
      const bool first = RS == B2_ROPE_NEOX ? d < half : (d & 1) == 0;
      x[i] = rope_rotate(x[i], other[i], fi, first, ps, log2_base, rotary_dim);
    }
  }
  *reinterpret_cast<uint2*>(ptr) = make_uint2(pack_bf16x2(x[0], x[1]), pack_bf16x2(x[2], x[3]));
}

__global__ void __launch_bounds__(128) rotary_kernel(__nv_bfloat16* __restrict__ qkv, const int32_t* __restrict__ pos, int batch,
                                                     int n_heads, int n_groups, int rotary_dim, float log2_base) {
  rotary_row<B2_ROPE_NEOX>(qkv, pos, batch, n_heads, n_groups, rotary_dim, log2_base);
}

__global__ void __launch_bounds__(128) rotary_il_kernel(__nv_bfloat16* __restrict__ qkv, const int32_t* __restrict__ pos,
                                                        int batch, int n_heads, int n_groups, int rotary_dim, float log2_base) {
  rotary_row<B2_ROPE_INTERLEAVED>(qkv, pos, batch, n_heads, n_groups, rotary_dim, log2_base);
}

// in-place rotary from a caller-given frequency table (b2_rotary_table): one warp per (row, q or k head); row b reads
// the table row inv + b * stride (rope_from_table)
template <bool H, int RS>
__device__ __forceinline__ void rotary_table_row(__nv_bfloat16* __restrict__ qkv, const int32_t* __restrict__ pos, int batch,
                                                 int n_heads, int n_groups, int rotary_dim, const float* __restrict__ inv,
                                                 int64_t stride, float af) {
  using F = Ft<H>;
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int rot_heads = n_heads + n_groups;
  const int slots = n_heads + 2 * n_groups;
  const int wid = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (wid >= batch * rot_heads) return;
  const int b = wid / rot_heads, h = wid - b * rot_heads;
  __nv_bfloat16* ptr = qkv + ((size_t)b * slots + h) * 128 + lane * 4;
  const uint2 raw = *reinterpret_cast<const uint2*>(ptr);
  float x[4] = {F::lo(raw.x), F::hi(raw.x), F::lo(raw.y), F::hi(raw.y)};
  rope_from_table<H, RS>(x, pos[b], inv + (size_t)b * stride, af, rotary_dim, lane);
  *reinterpret_cast<uint2*>(ptr) = make_uint2(F::pack(x[0], x[1]), F::pack(x[2], x[3]));
}

template <bool H>
__global__ void __launch_bounds__(128) rotary_table_kernel(__nv_bfloat16* __restrict__ qkv, const int32_t* __restrict__ pos,
                                                           int batch, int n_heads, int n_groups, int rotary_dim,
                                                           const float* __restrict__ inv, int64_t stride, float af) {
  rotary_table_row<H, B2_ROPE_NEOX>(qkv, pos, batch, n_heads, n_groups, rotary_dim, inv, stride, af);
}

template <bool H>
__global__ void __launch_bounds__(128) rotary_table_il_kernel(__nv_bfloat16* __restrict__ qkv, const int32_t* __restrict__ pos,
                                                              int batch, int n_heads, int n_groups, int rotary_dim,
                                                              const float* __restrict__ inv, int64_t stride, float af) {
  rotary_table_row<H, B2_ROPE_INTERLEAVED>(qkv, pos, batch, n_heads, n_groups, rotary_dim, inv, stride, af);
}

// QKLayerNormNoBeta (b2_qk_rmsnorm): one warp per (row, head) of x [rows, ld]; heads [0, n_heads) normalised with q_gamma,
// [n_heads, n_heads + n_groups) with k_gamma (head_rmsnorm), the V heads copied unless y == x
template <bool H>
__global__ void __launch_bounds__(128) qk_rmsnorm_kernel(__nv_bfloat16* y, const __nv_bfloat16* x, int64_t ld, int64_t warps,
                                                         int n_heads, int n_groups, const __nv_bfloat16* q_gamma,
                                                         const __nv_bfloat16* k_gamma, float eps) {
  using F = Ft<H>;
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int slots = n_heads + 2 * n_groups;
  const int64_t wid = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
  if (wid >= warps) return;
  const int64_t row = wid / slots;
  const int h = (int)(wid - row * slots);
  const size_t off = (size_t)row * ld + (size_t)h * 128 + lane * 4;
  const uint2 raw = *reinterpret_cast<const uint2*>(x + off);
  if (h >= n_heads + n_groups) {
    if (y != x) *reinterpret_cast<uint2*>(y + off) = raw;
    return;
  }
  float v[4] = {F::lo(raw.x), F::hi(raw.x), F::lo(raw.y), F::hi(raw.y)};
  head_rmsnorm<H>(v, h < n_heads ? q_gamma : k_gamma, eps, lane);
  *reinterpret_cast<uint2*>(y + off) = make_uint2(F::pack(v[0], v[1]), F::pack(v[2], v[3]));
}

template <bool H>
__global__ void __launch_bounds__(256) binary_kernel(__nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ a,
                                                     const __nv_bfloat16* __restrict__ b, int64_t n, int op) {
  using F = Ft<H>;
  pdl_wait();
  pdl_launch_dependents();
  const int64_t i = ((int64_t)blockIdx.x * 256 + threadIdx.x) * 8;
  if (i + 8 <= n) {
    const uint4 va = *reinterpret_cast<const uint4*>(a + i), vb = *reinterpret_cast<const uint4*>(b + i);
    const uint32_t wa[4] = {va.x, va.y, va.z, va.w}, wb[4] = {vb.x, vb.y, vb.z, vb.w};
    uint32_t wo[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float l = op == B2_BIN_ADD ? F::lo(wa[j]) + F::lo(wb[j]) : F::lo(wa[j]) * F::lo(wb[j]);
      const float h = op == B2_BIN_ADD ? F::hi(wa[j]) + F::hi(wb[j]) : F::hi(wa[j]) * F::hi(wb[j]);
      wo[j] = F::pack(l, h);
    }
    *reinterpret_cast<uint4*>(out + i) = make_uint4(wo[0], wo[1], wo[2], wo[3]);
  } else {
    for (int64_t j = i; j < n; ++j) {
      const float x = F::to_f(a[j]), y = F::to_f(b[j]);
      out[j] = F::from_f(op == B2_BIN_ADD ? x + y : x * y);
    }
  }
}

__global__ void __launch_bounds__(128) embedding_kernel(__nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ table,
                                                        const int64_t* __restrict__ ids, int hidden) {
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.x;
  const int64_t id = ids[b];
  for (int i = threadIdx.x * 8; i < hidden; i += 128 * 8)
    *reinterpret_cast<uint4*>(out + (size_t)b * hidden + i) = *reinterpret_cast<const uint4*>(table + (size_t)id * hidden + i);
}

// greedy sampling: lowest index among the maxima (bit-exact index contract)
template <bool H>
__global__ void __launch_bounds__(1024) argmax_kernel(int64_t* __restrict__ ids_out, float* __restrict__ vals_out,
                                                      const __nv_bfloat16* __restrict__ logits, int n, int64_t ld, int64_t id_offset) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float sv[32];
  __shared__ int si[32];
  const int b = blockIdx.x;
  const __nv_bfloat16* row = logits + (size_t)b * ld;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < n; i += 1024) {
    const float v = Ft<H>::to_f(row[i]);
    if (argmax_beats(v, i, best, bi)) { best = v; bi = i; }
  }
  warp_argmax(best, bi);
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x < 32) {
    best = sv[threadIdx.x];
    bi = si[threadIdx.x];
    warp_argmax(best, bi);
    if (threadIdx.x == 0) {
      ids_out[b] = bi + id_offset;
      if (vals_out) vals_out[b] = best;
    }
  }
}

__global__ void lens_add_kernel(int32_t* lens, int batch, int delta) {
  pdl_wait();
  pdl_launch_dependents();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < batch) lens[i] += delta;
}

// greedy verification of a multi-token step: row t of sequence b predicted pred[b][t] after tokens[b][0..t] (a draft tree:
// after t's path from the root).  From the root u = 0, step to the lowest-index child c of u with tokens[b][c] == pred[b][u]
// while there is one.  Children have larger indices than their parent, so one pass over c finds the path.  A chain
// (TREE = false) has the parent of c at c - 1, so its drafts tokens[b][1..] are accepted while each equals the prediction
// before it, and it records no path.
template <bool TREE>
__device__ __forceinline__ int spec_accept_seq(int b, int32_t* accepted, int32_t* path, int64_t* next_ids, int32_t* old_lens,
                                               int32_t* new_lens, int64_t* tokens, const int64_t* pred, const int32_t* parents,
                                               int q_len) {
  const int64_t* tk = tokens + (size_t)b * q_len;
  const int64_t* pr = pred + (size_t)b * q_len;
  int n = 1, u = 0;
  if (TREE) path[(size_t)b * q_len] = 0;
  for (int c = 1; c < q_len; ++c) {
    const int parent = TREE ? tree_parent(parents + (size_t)b * q_len, c) : c - 1;
    if (parent == u && tk[c] == pr[u]) {
      if (TREE) path[(size_t)b * q_len + n] = c;
      ++n;
      u = c;
    }
  }
  const int64_t next = pr[u];
  accepted[b] = n;
  if (next_ids) next_ids[b] = next;
  tokens[(size_t)b * q_len] = next;  // the last emitted token of the next step
  const int ol = old_lens[b] + n;
  old_lens[b] = ol;
  new_lens[b] = ol + q_len;
  return n;
}

template <bool TREE>
__global__ void spec_accept_kernel(int32_t* accepted, int32_t* path, int64_t* next_ids, int32_t* old_lens, int32_t* new_lens,
                                   int64_t* tokens, const int64_t* pred, const int32_t* parents, int batch, int q_len) {
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  spec_accept_seq<TREE>(b, accepted, path, next_ids, old_lens, new_lens, tokens, pred, parents, q_len);
}

// sampled verification: the same walk over the step's draws (b2_sample_tokens), then the sequence's draw counter advances by
// the tokens emitted, as that many single-token b2_sample steps would advance it
template <bool TREE>
__global__ void spec_accept_sampled_kernel(int32_t* accepted, int32_t* path, int64_t* next_ids, int32_t* old_lens,
                                           int32_t* new_lens, int64_t* tokens, const int64_t* pred, const int32_t* parents,
                                           uint64_t* offsets, int batch, int q_len) {
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  offsets[b] += spec_accept_seq<TREE>(b, accepted, path, next_ids, old_lens, new_lens, tokens, pred, parents, q_len);
}

// vocab-split lm_head: pick the global winner among the ranks' (max, argmax) pairs under argmax_beats' order; ties (equal
// values, or NaN on several ranks) -> lowest rank == lowest vocab id
__global__ void argmax_merge_kernel(int64_t* ids_out, const float* vals, const int64_t* ids, int nranks, int batch) {
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  float best = vals[b];
  int64_t bid = ids[b];
  for (int r = 1; r < nranks; ++r) {
    const float v = vals[(size_t)r * batch + b];
    if (argmax_beats(v, 0, best, 0)) { best = v; bid = ids[(size_t)r * batch + b]; }
  }
  ids_out[b] = bid;
}

}  // namespace b2

using namespace b2;

// the vector loads and stores of the kernels above: 16 bytes (uint4) for rmsnorm / binary / embedding, 8 (uint2) for rotary
static bool aligned(const void* p, uintptr_t bytes) { return ((uintptr_t)p & (bytes - 1)) == 0; }

#define B2_LAUNCH_CHECK(name, call)            \
  do {                                         \
    cudaError_t _e = (call);                   \
    if (_e != cudaSuccess) {                   \
      set_last_error(name, _e);                \
      return B2_ERR_CUDA;                      \
    }                                          \
  } while (0)

// path and parents: the tree form's
static int spec_accept(int32_t* accepted, int32_t* path, int64_t* next_ids, int32_t* old_lens, int32_t* new_lens, int64_t* tokens,
                       const int64_t* pred, const int32_t* parents, bool tree, int batch, int q_len, void* stream) {
  if (!accepted || !old_lens || !new_lens || !tokens || !pred || (tree && (!path || !parents)) || batch <= 0) return B2_ERR_PARAM;
  if (q_len < 1 || q_len > kMaxQLen) return B2_ERR_LIMIT;
  B2_LAUNCH_CHECK(tree ? "spec_accept_tree" : "spec_accept",
                  launch(tree ? spec_accept_kernel<true> : spec_accept_kernel<false>, dim3((batch + 127) / 128), dim3(128), 0,
                         (cudaStream_t)stream, true, accepted, path, next_ids, old_lens, new_lens, tokens, pred, parents, batch, q_len));
  return B2_OK;
}

extern "C" {

int b2_rmsnorm_ft(void* y, const void* x, const void* gamma, int rows, int cols, float eps, int ft, void* stream) {
  if (!y || !x || !gamma || rows <= 0 || cols <= 0) return B2_ERR_PARAM;
  if (cols % 8 || (ft != B2_DT_BF16 && ft != B2_DT_F16)) return B2_ERR_UNSUPPORTED;
  if (!aligned(y, 16) || !aligned(x, 16) || !aligned(gamma, 16)) return B2_ERR_UNSUPPORTED;
  if (ft == B2_DT_F16)
    B2_LAUNCH_CHECK("rmsnorm", launch(rmsnorm_kernel<true>, dim3(rows), dim3(256), 0, (cudaStream_t)stream, true, (__nv_bfloat16*)y,
                                      (const __nv_bfloat16*)x, (const __nv_bfloat16*)gamma, cols, eps));
  else
    B2_LAUNCH_CHECK("rmsnorm", launch(rmsnorm_kernel<false>, dim3(rows), dim3(256), 0, (cudaStream_t)stream, true, (__nv_bfloat16*)y,
                                      (const __nv_bfloat16*)x, (const __nv_bfloat16*)gamma, cols, eps));
  return B2_OK;
}
int b2_rmsnorm(void* y, const void* x, const void* gamma, int rows, int cols, float eps, void* stream) {
  return b2_rmsnorm_ft(y, x, gamma, rows, cols, eps, B2_DT_BF16, stream);
}

int b2_quant_fp8(void* y, int64_t ldy, float* scale, float* tile_sums, const void* x, const void* gamma, int rows, int cols,
                 float eps, void* stream) {
  if (!y || !scale || !tile_sums || !x || rows <= 0 || cols <= 0) return B2_ERR_PARAM;
  if (cols % 8 || ldy < cols || (ldy & 15) || ((uintptr_t)y & 15)) return B2_ERR_UNSUPPORTED;
  B2_LAUNCH_CHECK("quant_fp8", launch(quant_fp8_kernel, dim3(rows), dim3(256), 0, (cudaStream_t)stream, true, (uint8_t*)y, scale,
                                      tile_sums, (const __nv_bfloat16*)x, (const __nv_bfloat16*)gamma, cols, ldy, (cols + 63) / 64, eps));
  return B2_OK;
}

int b2_rotary(void* qkv, const int32_t* pos, int batch, int n_heads, int n_groups, int head_size, const b2_rope_cfg* rope,
              void* stream) {
  if (!qkv || !pos || !rope || batch <= 0) return B2_ERR_PARAM;
  if (int st = rope_style_check(rope)) return st;
  if (head_size != 128 || (rope->rotary_dim != 128 && rope->rotary_dim != 64) || !aligned(qkv, 8)) return B2_ERR_UNSUPPORTED;
  const int warps = batch * (n_heads + n_groups);
  const auto kern = rope->style == B2_ROPE_INTERLEAVED ? rotary_il_kernel : rotary_kernel;
  B2_LAUNCH_CHECK("rotary", launch(kern, dim3((warps + 3) / 4), dim3(128), 0, (cudaStream_t)stream, true,
                                   (__nv_bfloat16*)qkv, pos, batch, n_heads, n_groups, rope->rotary_dim, log2f(rope->base)));
  return B2_OK;
}

int b2_rotary_table(void* qkv, const int32_t* pos, int batch, int n_heads, int n_groups, int head_size, const b2_rope_cfg* rope,
                    const b2_rope_table* table, int ft, void* stream) {
  if (!qkv || !pos || batch <= 0 || n_heads <= 0 || n_groups <= 0) return B2_ERR_PARAM;
  if (int st = rope_table_check(rope, table)) return st;
  if (head_size != 128 || (ft != B2_DT_BF16 && ft != B2_DT_F16) || !aligned(qkv, 8)) return B2_ERR_UNSUPPORTED;
  const int warps = batch * (n_heads + n_groups);
  const bool il = rope->style == B2_ROPE_INTERLEAVED;
  const auto kern = ft == B2_DT_F16 ? (il ? rotary_table_il_kernel<true> : rotary_table_kernel<true>)
                                    : (il ? rotary_table_il_kernel<false> : rotary_table_kernel<false>);
  B2_LAUNCH_CHECK("rotary_table", launch(kern, dim3((warps + 3) / 4), dim3(128), 0, (cudaStream_t)stream, true, (__nv_bfloat16*)qkv,
                                         pos, batch, n_heads, n_groups, rope->rotary_dim, table->inv_freq, table->stride,
                                         table->attn_factor));
  return B2_OK;
}

int b2_qk_rmsnorm(void* y, const void* x, int rows, int64_t ld, int n_heads, int n_groups, int head_size, const b2_qk_norm* norm,
                  int ft, void* stream) {
  if (!y || !x || !norm || !norm->q_gamma || !norm->k_gamma || rows <= 0 || n_heads <= 0 || n_groups <= 0) return B2_ERR_PARAM;
  if (head_size != 128 || (ft != B2_DT_BF16 && ft != B2_DT_F16)) return B2_ERR_UNSUPPORTED;
  if (ld < (int64_t)(n_heads + 2 * n_groups) * 128) return B2_ERR_PARAM;
  if ((ld & 3) || !aligned(y, 8) || !aligned(x, 8) || !aligned(norm->q_gamma, 8) || !aligned(norm->k_gamma, 8)) return B2_ERR_UNSUPPORTED;
  const int64_t warps = (int64_t)rows * (n_heads + 2 * n_groups);
  if (warps > (int64_t)1 << 31) return B2_ERR_LIMIT;
  const dim3 grid((unsigned)((warps + 3) / 4)), block(128);
  const auto kern = ft == B2_DT_F16 ? qk_rmsnorm_kernel<true> : qk_rmsnorm_kernel<false>;
  B2_LAUNCH_CHECK("qk_rmsnorm", launch(kern, grid, block, 0, (cudaStream_t)stream, true, (__nv_bfloat16*)y, (const __nv_bfloat16*)x,
                                       ld, warps, n_heads, n_groups, (const __nv_bfloat16*)norm->q_gamma,
                                       (const __nv_bfloat16*)norm->k_gamma, norm->eps));
  return B2_OK;
}

int b2_binary_ft(void* out, const void* a, const void* b, int64_t n, int op, int ft, void* stream) {
  if (!out || !a || !b || n <= 0) return B2_ERR_PARAM;
  if ((op != B2_BIN_ADD && op != B2_BIN_MUL) || (ft != B2_DT_BF16 && ft != B2_DT_F16)) return B2_ERR_UNSUPPORTED;
  if (!aligned(out, 16) || !aligned(a, 16) || !aligned(b, 16)) return B2_ERR_UNSUPPORTED;
  const int64_t blocks = (n + 2047) / 2048;
  if (ft == B2_DT_F16)
    B2_LAUNCH_CHECK("binary", launch(binary_kernel<true>, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, true,
                                     (__nv_bfloat16*)out, (const __nv_bfloat16*)a, (const __nv_bfloat16*)b, n, op));
  else
    B2_LAUNCH_CHECK("binary", launch(binary_kernel<false>, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, true,
                                     (__nv_bfloat16*)out, (const __nv_bfloat16*)a, (const __nv_bfloat16*)b, n, op));
  return B2_OK;
}
int b2_binary(void* out, const void* a, const void* b, int64_t n, int op, void* stream) {
  return b2_binary_ft(out, a, b, n, op, B2_DT_BF16, stream);
}

int b2_embedding(void* out, const void* table, const int64_t* ids, int batch, int hidden, void* stream) {
  if (!out || !table || !ids || batch <= 0 || hidden <= 0) return B2_ERR_PARAM;
  if (hidden % 8 || !aligned(out, 16) || !aligned(table, 16)) return B2_ERR_UNSUPPORTED;
  B2_LAUNCH_CHECK("embedding", launch(embedding_kernel, dim3(batch), dim3(128), 0, (cudaStream_t)stream, true, (__nv_bfloat16*)out,
                                      (const __nv_bfloat16*)table, ids, hidden));
  return B2_OK;
}

int b2_argmax_ft(int64_t* ids_out, float* vals_out, const void* logits, int batch, int n, int64_t ld, int64_t id_offset, int ft,
                 void* stream) {
  if (!ids_out || !logits || batch <= 0 || n <= 0 || ld < n) return B2_ERR_PARAM;
  if (ft != B2_DT_BF16 && ft != B2_DT_F16) return B2_ERR_UNSUPPORTED;
  if (ft == B2_DT_F16)
    B2_LAUNCH_CHECK("argmax", launch(argmax_kernel<true>, dim3(batch), dim3(1024), 0, (cudaStream_t)stream, true, ids_out, vals_out,
                                     (const __nv_bfloat16*)logits, n, ld, id_offset));
  else
    B2_LAUNCH_CHECK("argmax", launch(argmax_kernel<false>, dim3(batch), dim3(1024), 0, (cudaStream_t)stream, true, ids_out, vals_out,
                                     (const __nv_bfloat16*)logits, n, ld, id_offset));
  return B2_OK;
}

int b2_argmax(int64_t* ids_out, const void* logits, int batch, int n, int64_t ld, void* stream) {
  return b2_argmax_ft(ids_out, nullptr, logits, batch, n, ld, 0, B2_DT_BF16, stream);
}

int b2_argmax_shard(int64_t* ids_out, float* vals_out, const void* logits, int batch, int n, int64_t ld, int64_t id_offset,
                    void* stream) {
  if (!vals_out) return B2_ERR_PARAM;
  return b2_argmax_ft(ids_out, vals_out, logits, batch, n, ld, id_offset, B2_DT_BF16, stream);
}

int b2_argmax_merge(int64_t* ids_out, const float* all_vals, const int64_t* all_ids, int nranks, int batch, void* stream) {
  if (!ids_out || !all_vals || !all_ids || nranks <= 0 || batch <= 0) return B2_ERR_PARAM;
  B2_LAUNCH_CHECK("argmax_merge", launch(argmax_merge_kernel, dim3((batch + 127) / 128), dim3(128), 0, (cudaStream_t)stream, true,
                                         ids_out, all_vals, all_ids, nranks, batch));
  return B2_OK;
}

int b2_lens_add(int32_t* lens, int batch, int delta, void* stream) {
  if (!lens || batch <= 0) return B2_ERR_PARAM;
  B2_LAUNCH_CHECK("lens_add", launch(lens_add_kernel, dim3((batch + 127) / 128), dim3(128), 0, (cudaStream_t)stream, true, lens,
                                     batch, delta));
  return B2_OK;
}

int b2_spec_accept(int32_t* accepted, int64_t* next_ids, int32_t* old_lens, int32_t* new_lens, int64_t* tokens, const int64_t* pred,
                   int batch, int q_len, void* stream) {
  return spec_accept(accepted, nullptr, next_ids, old_lens, new_lens, tokens, pred, nullptr, false, batch, q_len, stream);
}

int b2_spec_accept_tree(int32_t* accepted, int32_t* path, int64_t* next_ids, int32_t* old_lens, int32_t* new_lens, int64_t* tokens,
                        const int64_t* pred, const int32_t* parents, int batch, int q_len, void* stream) {
  return spec_accept(accepted, path, next_ids, old_lens, new_lens, tokens, pred, parents, true, batch, q_len, stream);
}

int b2_spec_accept_sampled(int32_t* accepted, int32_t* path, int64_t* next_ids, int32_t* old_lens, int32_t* new_lens,
                           int64_t* tokens, const int64_t* pred, const int32_t* parents, uint64_t* offsets, int batch, int q_len,
                           void* stream) {
  if (!accepted || !old_lens || !new_lens || !tokens || !pred || !offsets || !path != !parents || batch < 0) return B2_ERR_PARAM;
  if (q_len < 1 || q_len > kMaxQLen) return B2_ERR_LIMIT;
  if (batch == 0) return B2_OK;
  B2_LAUNCH_CHECK("spec_accept_sampled",
                  launch(parents ? spec_accept_sampled_kernel<true> : spec_accept_sampled_kernel<false>, dim3((batch + 127) / 128),
                         dim3(128), 0, (cudaStream_t)stream, true, accepted, path, next_ids, old_lens, new_lens, tokens, pred,
                         parents, offsets, batch, q_len));
  return B2_OK;
}

}  // extern "C"
