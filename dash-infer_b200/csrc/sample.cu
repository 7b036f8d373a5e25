// b200spark — sampling of the decode step (b2_sample): temperature, top-k and top-p with a per-sequence Philox draw, on the
// device.  Reference counterpart: gen_sample_gpu, generate_impl_gpu.hpp:116-191 (radix top-k, TopPSoftmaxLauncher,
// SampleKernelLauncher with Philox states).  The contract is in include/b200spark.h; every quantity that decides the token
// is an integer, the only floating-point step being one ex2.approx per weight.
//
// One CTA per row, or a cluster of 8 for rows longer than 32768; CTA c holds the contiguous ids [c chunk, (c + 1) chunk) and
// stages its 16-bit logits in shared memory once (at most 32768 x 2 bytes).  The row's order is that of a 16-bit key
// (the FT bits made order-preserving, -0 mapped to +0), highest first, the lower id first among equal keys.  A weight
// depends on the key alone, so each of the three selections (the k-th element, the nucleus end, the draw point) is a
// position (key K, j-th element of key K in id order), found by a descent over the key: a 256-bin histogram of the high
// byte (counts and weight sums, built once) then one of the low byte within the selected high byte (counts only; the
// weight of a bin is its count times the weight of its key).  The CTAs of a cluster add their histograms over distributed
// shared memory: integer sums, so the result does not depend on the split.  Only the draw needs an id: the j-th element
// of key K in id order, by a prefix count over the CTAs, then the warps of the holding CTA.
//
// Level-1 atomics: the high byte of a bf16 logit is its sign and 7 exponent bits, so the logits of a real model fall into a
// handful of bins and plain per-lane shared atomics would serialise on them.  Each warp sums its lanes per distinct bin
// (a leader's bin, the ballot of its peers, two 32-bit warp reductions of the weights) and issues one atomic pair per bin.
//
// The arithmetic shared with the vocab-split form (sample_tp.cu) is in sample_shared.cuh.
#include <climits>

#include "sample_shared.cuh"

namespace b2 {

constexpr int kSmpThreads = 1024;
constexpr int kSmpCtas = 8;
constexpr int kSmpSplitMin = 32768;
__host__ __device__ constexpr int smp_ctas(int n) { return n > kSmpSplitMin ? kSmpCtas : 1; }
__host__ __device__ constexpr int smp_chunk(int n) { return (n + smp_ctas(n) - 1) / smp_ctas(n); }

struct SmpShared {
  uint32_t cnt1[256];   // this CTA's level-1 histogram: counts and weight sums per high byte
  u64 mass1[256];
  uint32_t cnt2[3][256];  // this CTA's level-2 histograms (low byte), one per selection
  uint32_t tot1[256];   // the cluster's level-1 sums
  u64 totm1[256];
  uint32_t tot2[256];   // the cluster's level-2 counts of the current selection
  uint32_t wcnt[32];    // elements of the drawn key per warp
  float bv;             // this CTA's argmax winner
  int bi;
  uint32_t tie;         // this CTA's elements of the drawn key
  uint32_t hb, key;     // a selection's high byte, then its key
  u64 j, acnt, amass;   // ... its rank among the key's elements (from 1) and the counts / weights before the key
  int wsel;
  u64 wrank;
};

__device__ __forceinline__ uint32_t ld_dsmem_u32(const void* p, uint32_t cta) {
  uint32_t v;
  asm volatile("ld.shared::cluster.u32 %0, [%1];" : "=r"(v) : "r"(dsmem_addr(smem_u32(p), cta)) : "memory");
  return v;
}
__device__ __forceinline__ u64 ld_dsmem_u64(const void* p, uint32_t cta) {
  u64 v;
  asm volatile("ld.shared::cluster.u64 %0, [%1];" : "=l"(v) : "r"(dsmem_addr(smem_u32(p), cta)) : "memory");
  return v;
}
__device__ __forceinline__ void cluster_sync() {
  cluster_arrive();
  cluster_wait();
}

// One selection (all threads of every CTA of the cluster): the first position in the row's order at which the running sum
// of q reaches T, as (sh.key, sh.j) with sh.acnt / sh.amass the counts / weights of the keys above sh.key.
template <bool H>
__device__ __forceinline__ void smp_select(SmpShared& sh, const uint16_t* st, int len, int q, bool by_mass, u64 T, float m,
                                           float c, int nc) {
  const int tid = threadIdx.x, lane = tid & 31;
  __syncthreads();  // every thread has read the previous selection's results
  if (tid < 32) {
    u64 ac, am;
    const int hb = smp_scan(sh.tot1, [&](int b) { return sh.totm1[b]; }, by_mass, T, lane, ac, am);
    if (lane == 0) { sh.hb = hb; sh.acnt = ac; sh.amass = am; }
  }
  __syncthreads();
  const uint32_t hb = sh.hb;
  uint32_t* cnt2 = sh.cnt2[q];
  for (int i = tid; i < len; i += kSmpThreads) {
    const uint32_t k = smp_key(st[i]);
    if ((k >> 8) == hb) atomicAdd(&cnt2[k & 255], 1u);
  }
  cluster_sync();
  if (tid < 256) {
    uint32_t s = 0;
    for (int x = 0; x < nc; ++x) s += ld_dsmem_u32(&cnt2[tid], x);
    sh.tot2[tid] = s;
  }
  __syncthreads();
  if (tid < 32) {
    const u64 a1c = sh.acnt, a1m = sh.amass;
    auto wkey = [&](int b) { return smp_weight(smp_val<H>(smp_unkey((hb << 8) | (uint32_t)b)), m, c); };
    u64 ac, am;
    const int lo = smp_scan(sh.tot2, [&](int b) { return (u64)sh.tot2[b] * wkey(b); }, by_mass, T - (by_mass ? a1m : a1c), lane,
                            ac, am);
    if (lane == 0) {
      ac += a1c;
      am += a1m;
      const u64 w = wkey(lo);
      sh.key = (hb << 8) | (uint32_t)lo;
      sh.j = !by_mass ? T - ac : w ? (T - am + w - 1) / w : 1;  // the selected key's bin holds weight: w > 0
      sh.acnt = ac;
      sh.amass = am;
    }
  }
  __syncthreads();
}

// The draw of one row, by all threads of every CTA of the row's cluster.  Row r of logits takes the parameters at index q
// and the Philox counter off: q = r and off = offsets[r] (b2_sample, which then advances offsets[r]), or, for STEP (row r =
// b q_len + t of a verify step, b2_sample_tokens), q = b and off = offsets[b] + depth(t), with the offsets only read.
// STEP selects nothing but that mapping.
template <bool H, bool STEP>
__device__ __forceinline__ void smp_rows(int64_t* ids_out, const __nv_bfloat16* logits, int n, int64_t ld,
                                         const float* temperature, const int32_t* top_k, const float* top_p,
                                         const uint64_t* seeds, uint64_t* offsets, int q_len, const int32_t* parents) {
  extern __shared__ __align__(16) uint16_t st[];
  __shared__ SmpShared sh;
  pdl_wait();
  pdl_launch_dependents();
  const int nc = smp_ctas(n), chunk = smp_chunk(n);
  const int r = blockIdx.x / nc, cta = blockIdx.x - r * nc;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int start = cta * chunk, len = min(chunk, n - start);
  const uint16_t* row = reinterpret_cast<const uint16_t*>(logits) + (size_t)r * ld + start;
  const int q = STEP ? r / q_len : r;
  int depth = 0;
  if (STEP) {
    depth = r - q * q_len;
    if (parents) tree_walk(parents + (size_t)q * q_len, r - q * q_len, depth);
  }
  const float t = temperature[q];
  const int32_t k_in = top_k[q];
  const float p = top_p[q];
  const u64 seed = seeds[q], off = offsets[q] + (u64)depth;  // read by every CTA before the first cluster barrier

  for (int i = tid; i < 256; i += kSmpThreads) {
    sh.cnt1[i] = 0;
    sh.mass1[i] = 0;
    sh.cnt2[0][i] = sh.cnt2[1][i] = sh.cnt2[2][i] = 0;
  }
  // stage the chunk; the argmax under argmax_beats on the way
  float bv = -INFINITY;
  int bi = INT_MAX;
  int i = tid;
  for (; i + 3 * kSmpThreads < len; i += 4 * kSmpThreads) {
    uint16_t b[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) b[u] = row[i + u * kSmpThreads];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      st[i + u * kSmpThreads] = b[u];
      const float x = smp_val<H>(b[u]);
      if (argmax_beats(x, start + i + u * kSmpThreads, bv, bi)) { bv = x; bi = start + i + u * kSmpThreads; }
    }
  }
  for (; i < len; i += kSmpThreads) {
    const uint16_t b = row[i];
    st[i] = b;
    const float x = smp_val<H>(b);
    if (argmax_beats(x, start + i, bv, bi)) { bv = x; bi = start + i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (argmax_beats(ov, oi, bv, bi)) { bv = ov; bi = oi; }
  }
  __shared__ float wv[32];
  __shared__ int wi[32];
  if (lane == 0) { wv[w] = bv; wi[w] = bi; }
  __syncthreads();
  if (w == 0) {
    bv = wv[lane];
    bi = wi[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (argmax_beats(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { sh.bv = bv; sh.bi = bi; }
  }
  cluster_sync();
  // the row's winner, in every CTA: lane x holds CTA x's
  if (w == 0) {
    bv = lane < nc ? __uint_as_float(ld_dsmem_u32(&sh.bv, lane)) : -INFINITY;
    bi = lane < nc ? (int)ld_dsmem_u32(&sh.bi, lane) : INT_MAX;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (argmax_beats(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { wv[0] = bv; wi[0] = bi; }  // wv / wi were last read before the cluster barrier
  }
  __syncthreads();
  const float m = wv[0];
  const float c = __fdiv_rn(__uint_as_float(kLog2eF32), t);
  const bool greedy = !(fabsf(m) <= 3.402823466e38f) || !(t > 0.f) || !(fabsf(c) <= 3.402823466e38f);
  if (greedy) {
    if (cta == 0 && tid == 0) ids_out[r] = wi[0];
  } else {
    // level 1: counts and weight sums per high byte, one atomic pair per distinct bin of a warp
    const int steps = (len + kSmpThreads - 1) / kSmpThreads;
    for (int s = 0; s < steps; ++s) {
      const int e = s * kSmpThreads + tid;
      const bool valid = e < len;
      uint32_t hb = 0;
      u64 wt = 0;
      if (valid) {
        const uint32_t b = st[e];
        hb = smp_key(b) >> 8;
        wt = smp_weight(smp_val<H>(b), m, c);
      }
      uint32_t todo = __ballot_sync(0xffffffffu, valid);
      while (todo) {
        const int lead = __ffs(todo) - 1;
        const uint32_t h = __shfl_sync(0xffffffffu, hb, lead);
        const bool mine = valid && hb == h;
        const uint32_t grp = __ballot_sync(0xffffffffu, mine);
        const uint32_t slo = __reduce_add_sync(0xffffffffu, mine ? (uint32_t)(wt & 0xffffffu) : 0u);  // < 2^29
        const uint32_t shi = __reduce_add_sync(0xffffffffu, mine ? (uint32_t)(wt >> 24) : 0u);         // <= 2^21
        if (lane == lead) {
          atomicAdd(&sh.cnt1[h], (uint32_t)__popc(grp));
          atomicAdd(&sh.mass1[h], ((u64)shi << 24) + slo);
        }
        todo &= ~grp;
      }
    }
    cluster_sync();
    if (tid < 256) {
      uint32_t sc = 0;
      u64 sm = 0;
      for (int x = 0; x < nc; ++x) {
        sc += ld_dsmem_u32(&sh.cnt1[tid], x);
        sm += ld_dsmem_u64(&sh.mass1[tid], x);
      }
      sh.tot1[tid] = sc;
      sh.totm1[tid] = sm;
    }
    __syncthreads();
    // top-k: the kept set ends at the k-th element; S_k its weight
    const int k = (k_in <= 0 || k_in > n) ? n : k_in;
    u64 Sk = 0;
    if (k == n) {
      if (tid < 32) {
        u64 s = 0;
#pragma unroll
        for (int b = 0; b < 8; ++b) s += sh.totm1[lane * 8 + b];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) sh.amass = s;
      }
      __syncthreads();
      Sk = sh.amass;
    } else {
      smp_select<H>(sh, st, len, 0, false, (u64)k, m, c, nc);
      Sk = sh.amass + sh.j * smp_weight(smp_val<H>(smp_unkey(sh.key)), m, c);
    }
    // top-p: the shortest prefix whose weight reaches Pt; S_p its weight
    const uint32_t p24 = !(p < 1.f) ? (1u << 24) : min(__float2uint_rn(__fmul_rn(p, 16777216.f)), 1u << 24);
    u64 Sp = Sk;
    if (p24 < (1u << 24)) {
      const u64 Pt = max(mul_shr24(p24, Sk, true), (u64)1);
      smp_select<H>(sh, st, len, 1, true, Pt, m, c, nc);
      Sp = sh.amass + sh.j * smp_weight(smp_val<H>(smp_unkey(sh.key)), m, c);
    }
    // the draw: the first element at which the running weight exceeds U
    const uint32_t u24 = philox_r0((uint32_t)off, (uint32_t)(off >> 32), 0, 0, (uint32_t)seed, (uint32_t)(seed >> 32)) >> 8;
    const u64 U = mul_shr24(u24, Sp, false);
    smp_select<H>(sh, st, len, 2, true, U + 1, m, c, nc);
    // the j-th element of the drawn key in id order: counts per warp (warp w holds a contiguous range), per CTA, then the
    // prefix over the CTAs
    const uint32_t key = sh.key;
    const u64 j = sh.j;
    const int seg = ((len + kSmpThreads - 1) / kSmpThreads) * 32;
    uint32_t cnt = 0;
    for (int e = w * seg + lane; e < (w + 1) * seg; e += 32)
      cnt += __popc(__ballot_sync(0xffffffffu, e < len && smp_key(st[e]) == key));
    if (lane == 0) sh.wcnt[w] = cnt;
    __syncthreads();
    if (tid == 0) {
      uint32_t s = 0;
      for (int x = 0; x < 32; ++x) s += sh.wcnt[x];
      sh.tie = s;
    }
    cluster_sync();
    if (tid == 0) {
      u64 pre = 0;
      for (int x = 0; x < cta; ++x) pre += ld_dsmem_u32(&sh.tie, x);
      sh.wsel = -1;
      if (pre < j && j <= pre + sh.tie) {
        u64 jl = j - pre;
        for (int x = 0; x < 32; ++x) {
          if (jl <= sh.wcnt[x]) { sh.wsel = x; sh.wrank = jl; break; }
          jl -= sh.wcnt[x];
        }
      }
    }
    __syncthreads();
    if (w == sh.wsel) {
      const uint32_t want = (uint32_t)sh.wrank;
      uint32_t seen = 0;
      for (int e = w * seg + lane; e < (w + 1) * seg; e += 32) {
        const bool hit = e < len && smp_key(st[e]) == key;
        const uint32_t bal = __ballot_sync(0xffffffffu, hit);
        if (seen + __popc(bal) >= want) {
          if (hit && seen + __popc(bal & ((1u << lane) - 1)) + 1 == want) ids_out[r] = start + e;
          break;
        }
        seen += __popc(bal);
      }
    }
  }
  cluster_sync();  // no CTA leaves while another reads its shared memory; every CTA has read offsets[q]
  if (!STEP && cta == 0 && tid == 0) offsets[r] = off + 1;
}

template <bool H>
__global__ void __launch_bounds__(kSmpThreads) sample_kernel(int64_t* ids_out, const __nv_bfloat16* __restrict__ logits, int n,
                                                             int64_t ld, const float* temperature, const int32_t* top_k,
                                                             const float* top_p, const uint64_t* seeds, uint64_t* offsets) {
  smp_rows<H, false>(ids_out, logits, n, ld, temperature, top_k, top_p, seeds, offsets, 1, nullptr);
}

template <bool H>
__global__ void __launch_bounds__(kSmpThreads) sample_tokens_kernel(int64_t* ids_out, const __nv_bfloat16* __restrict__ logits,
                                                                    int n, int64_t ld, int q_len, const int32_t* parents,
                                                                    const float* temperature, const int32_t* top_k,
                                                                    const float* top_p, const uint64_t* seeds,
                                                                    const uint64_t* offsets) {
  // STEP never writes offsets
  smp_rows<H, true>(ids_out, logits, n, ld, temperature, top_k, top_p, seeds, const_cast<uint64_t*>(offsets), q_len, parents);
}

}  // namespace b2

using namespace b2;

extern "C" {

int b2_sample(int64_t* ids_out, const void* logits, int rows, int n, int64_t ld, const float* temperature, const int32_t* top_k,
              const float* top_p, const uint64_t* seeds, uint64_t* offsets, int ft, void* stream) {
  if (!ids_out || !logits || !temperature || !top_k || !top_p || !seeds || !offsets || rows < 0 || n < 1 || ld < n)
    return B2_ERR_PARAM;
  if (ft != B2_DT_BF16 && ft != B2_DT_F16) return B2_ERR_PARAM;
  if (n > B2_SAMPLE_MAX_N || (int64_t)rows * smp_ctas(n) > INT_MAX) return B2_ERR_LIMIT;
  if (rows == 0) return B2_OK;
  const int nc = smp_ctas(n);
  const size_t smem = ((size_t)smp_chunk(n) * 2 + 15) & ~(size_t)15;
  const cudaError_t e = with_flag(ft == B2_DT_F16, [&](auto h) {
    constexpr bool H = decltype(h)::value;
    static const cudaError_t attr = cudaFuncSetAttribute(sample_kernel<H>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                         kSmpSplitMin * 2);
    if (attr != cudaSuccess) return attr;
    return launch_cluster(sample_kernel<H>, dim3((unsigned)rows * nc), dim3(kSmpThreads), smem, (cudaStream_t)stream, true,
                          (unsigned)nc, ids_out, (const __nv_bfloat16*)logits, n, ld, temperature, top_k, top_p, seeds, offsets);
  });
  if (e != cudaSuccess) {
    set_last_error("sample", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

int b2_sample_tokens(int64_t* ids_out, const void* logits, int batch, int q_len, const int32_t* parents, int n, int64_t ld,
                     const float* temperature, const int32_t* top_k, const float* top_p, const uint64_t* seeds,
                     const uint64_t* offsets, int ft, void* stream) {
  if (!ids_out || !logits || !temperature || !top_k || !top_p || !seeds || !offsets || batch < 0 || n < 1 || ld < n)
    return B2_ERR_PARAM;
  if (ft != B2_DT_BF16 && ft != B2_DT_F16) return B2_ERR_PARAM;
  if (q_len < 1 || q_len > kMaxQLen || n > B2_SAMPLE_MAX_N || (int64_t)batch * q_len * smp_ctas(n) > INT_MAX) return B2_ERR_LIMIT;
  if (batch == 0) return B2_OK;
  const int nc = smp_ctas(n);
  const size_t smem = ((size_t)smp_chunk(n) * 2 + 15) & ~(size_t)15;
  const cudaError_t e = with_flag(ft == B2_DT_F16, [&](auto h) {
    constexpr bool H = decltype(h)::value;
    static const cudaError_t attr = cudaFuncSetAttribute(sample_tokens_kernel<H>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                         kSmpSplitMin * 2);
    if (attr != cudaSuccess) return attr;
    return launch_cluster(sample_tokens_kernel<H>, dim3((unsigned)(batch * q_len * nc)), dim3(kSmpThreads), smem,
                          (cudaStream_t)stream, true, (unsigned)nc, ids_out, (const __nv_bfloat16*)logits, n, ld, q_len, parents,
                          temperature, top_k, top_p, seeds, offsets);
  });
  if (e != cudaSuccess) {
    set_last_error("sample_tokens", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

}  // extern "C"
