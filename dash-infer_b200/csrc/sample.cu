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
// Each step of the draw is one function of sample_shared.cuh, which the vocab-split form (sample_tp.cu) calls between its
// phases too; this file adds the cluster's meeting points.
#include <climits>

#include "sample_shared.cuh"

namespace b2 {

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
  float wv[32];         // the warps' argmax winners, then the row's
  int wi[32];
  float bv;             // this CTA's argmax winner
  int bi;
  uint32_t tie;         // this CTA's elements of the drawn key
  uint32_t hb, key;     // a selection's high byte; the drawn key
  u64 j;                // ... and its rank among the key's elements (from 1)
};

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
  // stage the chunk and take its argmax; the row's argmax over the cluster (lane x holds CTA x's)
  float bv;
  int bi;
  smp_argmax<H, true>(row, len, start, st, sh.wv, sh.wi, bv, bi);
  if (tid == 0) { sh.bv = bv; sh.bi = bi; }
  cluster_sync();
  if (w == 0) {
    bv = lane < nc ? __uint_as_float(ld_dsmem_u32(&sh.bv, lane)) : -INFINITY;
    bi = lane < nc ? (int)ld_dsmem_u32(&sh.bi, lane) : INT_MAX;
    warp_argmax(bv, bi);
    if (lane == 0) { sh.wv[0] = bv; sh.wi[0] = bi; }  // wv / wi were last read before the cluster barrier
  }
  __syncthreads();
  const SmpRow R = smp_row_setup(sh.wv[0], t, k_in, n);
  const float m = R.m, c = R.c;
  if (R.greedy) {
    if (cta == 0 && tid == 0) ids_out[r] = sh.wi[0];
  } else {
    smp_level1<H>(sh.cnt1, sh.mass1, st, len, m, c);
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
    // the three selections: top-k, top-p, the draw.  Warp 0 runs the scans and keeps a selection's state and the kept
    // weight S (S_k, then S_p) in registers; the other threads learn only the high byte to count in.
    u64 S = 0;
    SmpSel sel{};
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      const SmpTarget tg = smp_target(s, R.k, n, p, seed, off, S);
      if (!tg.sel) {
        if (s == 0 && w == 0) S = smp_total_mass(sh.totm1, lane);
        continue;
      }
      uint32_t hb = 0;
      u64 a1c = 0, a1m = 0;
      if (w == 0) {
        hb = (uint32_t)smp_scan(sh.tot1, [&](int b) { return sh.totm1[b]; }, tg.by_mass, tg.T, lane, a1c, a1m);
        if (lane == 0) sh.hb = hb;
      }
      __syncthreads();
      smp_level2(sh.cnt2[s], st, len, sh.hb);
      cluster_sync();
      if (tid < 256) {
        uint32_t sc = 0;
        for (int x = 0; x < nc; ++x) sc += ld_dsmem_u32(&sh.cnt2[s][tid], x);
        sh.tot2[tid] = sc;
      }
      __syncthreads();
      if (w == 0) {
        sel = smp_select_end<H>(sh.tot2, hb, tg.T, a1c, a1m, tg.by_mass, m, c, lane);
        S = smp_kept<H>(sel, m, c);
      }
    }
    // the j-th element of the drawn key in id order: counts per warp and per CTA, the prefix over the lower CTAs, then the
    // holding warp's walk
    if (tid == 0) { sh.key = sel.key; sh.j = sel.j; }
    __syncthreads();
    const uint32_t key = sh.key;
    smp_key_counts(st, len, key, sh.wcnt);
    __syncthreads();
    if (w == 0) {
      const uint32_t tie = __reduce_add_sync(0xffffffffu, sh.wcnt[lane]);
      if (lane == 0) sh.tie = tie;
    }
    cluster_sync();
    const uint32_t pre = __reduce_add_sync(0xffffffffu, lane < cta ? ld_dsmem_u32(&sh.tie, lane) : 0u);
    const int e = smp_pick(st, len, key, sh.wcnt, sh.j - pre);
    if (e >= 0) ids_out[r] = start + e;
  }
  cluster_sync();  // no CTA leaves while another reads its shared memory; every CTA has read offsets[q]
  if (!STEP && cta == 0 && tid == 0) offsets[r] = off + 1;
}

// The two kernels take the same parameters, so one launcher serves both; sample_kernel reads neither q_len nor parents.
// Both ask ptxas for one resident CTA per SM, not two: without that bound it fits sample_kernel in 32 registers so that two
// CTAs share an SM, which shortened the kernel alone but slowed the Qwen2-7B decode step at batch 8 by 2 % (H100 80GB HBM3,
// 700 W).
template <bool H>
__global__ void __launch_bounds__(kSmpThreads, 1) sample_kernel(int64_t* ids_out, const __nv_bfloat16* __restrict__ logits, int n,
                                                             int64_t ld, int q_len, const int32_t* parents, const float* temperature,
                                                             const int32_t* top_k, const float* top_p, const uint64_t* seeds,
                                                             uint64_t* offsets) {
  smp_rows<H, false>(ids_out, logits, n, ld, temperature, top_k, top_p, seeds, offsets, q_len, parents);
}

template <bool H>
__global__ void __launch_bounds__(kSmpThreads, 1) sample_tokens_kernel(int64_t* ids_out, const __nv_bfloat16* __restrict__ logits,
                                                                    int n, int64_t ld, int q_len, const int32_t* parents,
                                                                    const float* temperature, const int32_t* top_k,
                                                                    const float* top_p, const uint64_t* seeds, uint64_t* offsets) {
  smp_rows<H, true>(ids_out, logits, n, ld, temperature, top_k, top_p, seeds, offsets, q_len, parents);  // never writes offsets
}

// b2_sample (STEP false: q_len = 1, no parents) and b2_sample_tokens: batch * q_len rows, one CTA or cluster per row
template <bool STEP>
static int smp_launch(const char* what, int64_t* ids_out, const void* logits, int batch, int q_len, const int32_t* parents, int n,
                      int64_t ld, const float* temperature, const int32_t* top_k, const float* top_p, const uint64_t* seeds,
                      uint64_t* offsets, int ft, void* stream) {
  if (!ids_out || !logits || !temperature || !top_k || !top_p || !seeds || !offsets || batch < 0 || n < 1 || ld < n)
    return B2_ERR_PARAM;
  if (ft != B2_DT_BF16 && ft != B2_DT_F16) return B2_ERR_PARAM;
  if (q_len < 1 || q_len > kMaxQLen || n > B2_SAMPLE_MAX_N || (int64_t)batch * q_len * smp_ctas(n) > INT_MAX) return B2_ERR_LIMIT;
  if (batch == 0) return B2_OK;
  const int nc = smp_ctas(n);
  const size_t smem = ((size_t)smp_chunk(n) * 2 + 15) & ~(size_t)15;
  const cudaError_t e = with_flag(ft == B2_DT_F16, [&](auto h) {
    constexpr bool H = decltype(h)::value;
    const auto kernel = STEP ? sample_tokens_kernel<H> : sample_kernel<H>;
    static const cudaError_t attr = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmpSplitMin * 2);
    if (attr != cudaSuccess) return attr;
    return launch_cluster(kernel, dim3((unsigned)(batch * q_len * nc)), dim3(kSmpThreads), smem, (cudaStream_t)stream, true,
                          (unsigned)nc, ids_out, (const __nv_bfloat16*)logits, n, ld, q_len, parents, temperature, top_k, top_p,
                          seeds, offsets);
  });
  if (e != cudaSuccess) {
    set_last_error(what, e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

}  // namespace b2

using namespace b2;

extern "C" {

int b2_sample(int64_t* ids_out, const void* logits, int rows, int n, int64_t ld, const float* temperature, const int32_t* top_k,
              const float* top_p, const uint64_t* seeds, uint64_t* offsets, int ft, void* stream) {
  return smp_launch<false>("sample", ids_out, logits, rows, 1, nullptr, n, ld, temperature, top_k, top_p, seeds, offsets, ft,
                           stream);
}

int b2_sample_tokens(int64_t* ids_out, const void* logits, int batch, int q_len, const int32_t* parents, int n, int64_t ld,
                     const float* temperature, const int32_t* top_k, const float* top_p, const uint64_t* seeds,
                     const uint64_t* offsets, int ft, void* stream) {
  return smp_launch<true>("sample_tokens", ids_out, logits, batch, q_len, parents, n, ld, temperature, top_k, top_p, seeds,
                          const_cast<uint64_t*>(offsets), ft, stream);
}

}  // extern "C"
