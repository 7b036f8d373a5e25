// b200spark — log-probabilities of the decode step (b2_logprobs, b2_logprobs_shard, b2_logprobs_merge): the emitted
// token's logprob and the top-N alternatives, for whole and vocab-split logits, on the device.  Reference counterpart:
// generate_impl_gpu.hpp:33-79 (StridedLogSoftmax, SelectBatchTokenLogprob, then a top-k of the log-probabilities); the
// logprobs here stay fp32 (the reference rounds them to FT before its top-k).
//
// One CTA per row, or a cluster of 8 for rows longer than 32768.  Pass 1 is the argmax traversal: the row maximum m and a
// threshold per CTA that every top-list entry reaches.  Pass 2 sums expf(x_i - m) and keeps a per-thread top-K in
// registers, fed only by the elements at the threshold or above; warps, then the block, then the cluster merge the lists.  The row's statistics and candidates form a
// partial record (LpHead + candidates): the shard form writes it out, the whole-row form finishes it in place with the
// same function the merge runs over all ranks' records, so one shard + the merge is the whole-row form bit for bit.
#include <climits>

#include "b2_common.cuh"

namespace b2 {

constexpr int kLpThreads = 1024;

// A row's partial record: this head, then K = max(n_top, 1) candidate values (fp32) and K candidate ids (int32, the
// shard's id_offset added) in argmax_beats order.  Slots the shard cannot fill hold (-inf, INT_MAX), argmax_beats' start,
// which loses to every real entry.
struct LpHead {
  float m;            // the maximum under argmax_beats (NaN when the row holds one)
  float s;            // sum of expf(x_i - m), in the kernel's order
  float tok;          // the token's logit when tok_where == 1
  int32_t tok_where;  // -1: no token ids given (the token is the top-1), 0: the id is not in this shard, 1: it is
};
constexpr int lp_k(int n_top) { return n_top > 1 ? n_top : 1; }
constexpr size_t lp_rec_bytes(int n_top) { return sizeof(LpHead) + 8 * (size_t)lp_k(n_top); }

// insert (x, i) into a thread's list, kept sorted under argmax_beats; static indices only, so the list stays in registers
template <int K>
__device__ __forceinline__ void lp_insert(float (&v)[K], int (&id)[K], float x, int i) {
  if (!argmax_beats(x, i, v[K - 1], id[K - 1])) return;
  bool placed = false;
#pragma unroll
  for (int j = K - 1; j > 0; --j) {
    if (!placed) {
      if (argmax_beats(x, i, v[j - 1], id[j - 1])) {
        v[j] = v[j - 1];
        id[j] = id[j - 1];
      } else {
        v[j] = x;
        id[j] = i;
        placed = true;
      }
    }
  }
  if (!placed) {
    v[0] = x;
    id[0] = i;
  }
}

// Rows longer than kLpSplitMin run on a cluster of kLpCtas CTAs, CTA c taking the elements c * 1024 + t + 1024 kLpCtas j
// (a function of n alone, so a row gives the same bits at every batch size).
constexpr int kLpCtas = 8;
constexpr int kLpSplitMin = 32768;
__host__ __device__ constexpr int lp_ctas(int n) { return n > kLpSplitMin ? kLpCtas : 1; }

// The per-row reduction shared by the whole-row and the shard kernels: the `nc` CTAs of a cluster (nc = lp_ctas(n)) fill the
// record `rec` (shared memory of the cluster's CTA 0) of row r.
// Pass 1 is the argmax traversal.  Each CTA's 32 warp winners give its best and a threshold tau (the max(n_top, 1)-th best
// of them: that many distinct elements of the CTA are at least as good, so every CTA element of the row's top list is too);
// the CTAs' bests give m.  Pass 2 sums the terms and inserts into the thread's list only the elements tau does not beat.
// The lists are merged by warps (max(n_top, 1) butterfly rounds, no block barrier), the 32 warp lists by warp 0 the same
// way; CTA 0 reads the nc CTA lists through distributed shared memory in one round, and each candidate takes the slot
// given by its rank (the number of candidates that beat it).
// The sum: each thread adds its terms in index order from 0, then an xor butterfly over the 32 lanes and one over the 32
// warp partials; CTA 0 adds the nc CTA partials in CTA order.
template <bool H, int K>
__device__ __forceinline__ void lp_row(LpHead* rec, const __nv_bfloat16* __restrict__ row, int n, int64_t id_offset,
                                       const int64_t* __restrict__ tok_ids, int r, int n_top, int nc, int c) {
  using F = Ft<H>;
  __shared__ float sv[32];
  __shared__ int si[32];
  __shared__ float wl_v[32][K];  // the warps' lists
  __shared__ int wl_i[32][K];
  __shared__ float cl_v[K];      // this CTA's list, read by CTA 0
  __shared__ int cl_i[K];
  __shared__ float ml_v[kLpCtas * K], ml_s[kLpCtas];  // CTA 0: the cluster's lists and partial sums, fetched in one round
  __shared__ int ml_i[kLpCtas * K];
  __shared__ float cb_v, tv, m_sh, cs;
  __shared__ int cb_i, ti;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int kk = lp_k(n_top);
  const int stride = kLpThreads * nc;
  float* vals = reinterpret_cast<float*>(rec + 1);
  int32_t* ids = reinterpret_cast<int32_t*>(vals + kk);

  float bv = -INFINITY;
  int bi = INT_MAX;
  int i = c * kLpThreads + tid;
  for (; i + 3 * stride < n; i += 4 * stride) {
    float x[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) x[u] = F::to_f(row[i + u * stride]);
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (argmax_beats(x[u], i + u * stride, bv, bi)) { bv = x[u]; bi = i + u * stride; }
  }
  for (; i < n; i += stride) {
    const float x = F::to_f(row[i]);
    if (argmax_beats(x, i, bv, bi)) { bv = x; bi = i; }
  }
  warp_argmax(bv, bi);
  if (lane == 0) { sv[w] = bv; si[w] = bi; }
  __syncthreads();
  if (w == 0) {
    const float cv = sv[lane];
    const int ci = si[lane];
    int rank = 0;  // the warp winners that beat this one (the winners are distinct elements, or padding)
#pragma unroll 8
    for (int j = 0; j < 32; ++j) rank += argmax_beats(__shfl_sync(0xffffffffu, cv, j), __shfl_sync(0xffffffffu, ci, j), cv, ci);
    if (lane == 0) { tv = -INFINITY; ti = INT_MAX; }  // fewer than kk real winners: every element passes
    __syncwarp();
    if (rank == 0) { cb_v = cv; cb_i = ci; }
    if (rank == kk - 1 && ci != INT_MAX) { tv = cv; ti = ci; }
  }
  cluster_sync();  // the CTAs' bests are visible cluster-wide after it (it also orders the block)
  if (w == 0) {
    float mv = lane < nc ? __uint_as_float(ld_dsmem_u32(&cb_v, lane)) : -INFINITY;
    int mi = lane < nc ? (int)ld_dsmem_u32(&cb_i, lane) : INT_MAX;
    warp_argmax(mv, mi);
    if (lane == 0) m_sh = mv;
  }
  __syncthreads();
  const float m = m_sh;

  float v[K];
  int id[K];
#pragma unroll
  for (int j = 0; j < K; ++j) { v[j] = -INFINITY; id[j] = INT_MAX; }
  const float tau = tv;
  const int taui = ti;
  float s = 0.f;
  i = c * kLpThreads + tid;
  for (; i + 3 * stride < n; i += 4 * stride) {
    float x[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) x[u] = F::to_f(row[i + u * stride]);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      s += expf(x[u] - m);
      if (K > 1 && !argmax_beats(tau, taui, x[u], i + u * stride)) lp_insert<K>(v, id, x[u], i + u * stride);
    }
  }
  for (; i < n; i += stride) {
    const float x = F::to_f(row[i]);
    s += expf(x - m);
    if (K > 1 && !argmax_beats(tau, taui, x, i)) lp_insert<K>(v, id, x, i);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) sv[w] = s;  // sv was last read before the cluster barrier

  if (K == 1) {
    if (tid == 0) { cl_v[0] = cb_v; cl_i[0] = cb_i; }
  } else {
    for (int k = 0; k < kk; ++k) {  // the warp's list: kk rounds of "pop the best head" over its lanes
      float hv = v[0];
      int hi = id[0];
      warp_argmax(hv, hi);
      if (lane == 0) { wl_v[w][k] = hv; wl_i[w][k] = hi; }
      if (hi != INT_MAX && id[0] == hi) {
#pragma unroll
        for (int j = 0; j + 1 < K; ++j) { v[j] = v[j + 1]; id[j] = id[j + 1]; }
        v[K - 1] = -INFINITY;
        id[K - 1] = INT_MAX;
      }
    }
  }
  __syncthreads();
  if (w == 0) {
    float t = sv[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (lane == 0) cs = t;
    if (K > 1) {  // the CTA's list from the 32 warp lists (lane l walks warp l's)
      int p = 0;
      for (int k = 0; k < kk; ++k) {
        float hv = p < kk ? wl_v[lane][p] : -INFINITY;
        int hi = p < kk ? wl_i[lane][p] : INT_MAX;
        const int mine = hi;
        warp_argmax(hv, hi);
        if (lane == 0) { cl_v[k] = hv; cl_i[k] = hi; }
        if (hi != INT_MAX && mine == hi) ++p;
      }
    }
  }
  cluster_sync();  // every CTA's list and partial sum are ready
  if (c == 0) {  // the row's list from the nc CTA lists, the sum in CTA order
    if (tid < nc * kk) {
      ml_v[tid] = __uint_as_float(ld_dsmem_u32(&cl_v[tid % kk], tid / kk));
      ml_i[tid] = (int)ld_dsmem_u32(&cl_i[tid % kk], tid / kk);
    }
    if (tid < nc) ml_s[tid] = __uint_as_float(ld_dsmem_u32(&cs, tid));
    if (tid < kk) { vals[tid] = -INFINITY; ids[tid] = INT_MAX; }
    __syncthreads();
    if (tid < nc * kk) {
      const float cv = ml_v[tid];
      const int ci = ml_i[tid];
      int rank = 0;
      for (int q = 0; q < nc * kk; ++q) rank += argmax_beats(ml_v[q], ml_i[q], cv, ci);
      if (ci != INT_MAX && rank < kk) { vals[rank] = cv; ids[rank] = (int32_t)(ci + id_offset); }
    }
    if (tid == 0) {
      float st = ml_s[0];
      for (int q = 1; q < nc; ++q) st += ml_s[q];
      rec->m = m;
      rec->s = st;
      rec->tok = NAN;
      rec->tok_where = -1;
      if (tok_ids) {
        const int64_t t = tok_ids[r] - id_offset;  // never dereferenced outside [0, n)
        rec->tok_where = t >= 0 && t < n;
        if (t >= 0 && t < n) rec->tok = F::to_f(row[t]);
      }
    }
  }
  cluster_sync();  // no CTA leaves while CTA 0 reads its shared memory
}

// Finish row r from the records of nranks shards (rank q's at recs + q * rank_stride), one thread:
//   M = max_q m_q under argmax_beats;  S = sum over q with m_q != -inf of s_q expf(m_q - M), fused multiply-adds in rank
//   order from 0;  lp(x) = (x - M) - logf(S).
// The top list is picked from the nranks x K candidates under argmax_beats (ids are global, so ties go to the lowest id,
// i.e. the lowest rank); a slot no real candidate fills gets id -1 and lp -inf.
__device__ __forceinline__ void lp_finish(const uint8_t* recs, size_t rank_stride, int nranks, int n_top, int r,
                                          int64_t* ids_out, float* tok_lp, int64_t* top_ids, float* top_lp) {
  const int kk = lp_k(n_top);
  float M = reinterpret_cast<const LpHead*>(recs)->m;
  for (int q = 1; q < nranks; ++q) {
    const float mq = reinterpret_cast<const LpHead*>(recs + q * rank_stride)->m;
    if (argmax_beats(mq, 0, M, 0)) M = mq;
  }
  float S = 0.f, tok = NAN;
  bool tok_top = false, tok_found = false;
  for (int q = 0; q < nranks; ++q) {
    const LpHead* h = reinterpret_cast<const LpHead*>(recs + q * rank_stride);
    if (h->m != -INFINITY) S = __fmaf_rn(h->s, expf(h->m - M), S);
    if (h->tok_where < 0) tok_top = true;
    if (h->tok_where > 0 && !tok_found) { tok = h->tok; tok_found = true; }
  }
  const float ls = logf(S);
  float lv = 0.f;
  int li = 0;
  for (int k = 0; k < kk; ++k) {
    float bv = -INFINITY;
    int bi = INT_MAX;
    for (int q = 0; q < nranks; ++q) {
      const float* vals = reinterpret_cast<const float*>(recs + q * rank_stride + sizeof(LpHead));
      const int32_t* ids = reinterpret_cast<const int32_t*>(vals + kk);
      for (int j = 0; j < kk; ++j) {
        const float cv = vals[j];
        const int ci = ids[j];
        if ((k == 0 || argmax_beats(lv, li, cv, ci)) && argmax_beats(cv, ci, bv, bi)) { bv = cv; bi = ci; }
      }
    }
    lv = bv;
    li = bi;
    const bool real = bi != INT_MAX;
    if (k == 0) {
      if (ids_out) ids_out[r] = bi;
      if (tok_top) tok = bv;
    }
    if (k < n_top) {
      top_ids[(size_t)r * n_top + k] = real ? bi : -1;
      top_lp[(size_t)r * n_top + k] = real ? (bv - M) - ls : -INFINITY;
    }
  }
  if (tok_lp) tok_lp[r] = (tok - M) - ls;
}

// partials == NULL: the whole-row form (outputs written here); else the shard form (the record of row r written to
// partials + r * lp_rec_bytes(n_top)).
template <bool H, int K>
__global__ void __launch_bounds__(kLpThreads) logprobs_kernel(int64_t* ids_out, float* tok_lp, int64_t* top_ids, float* top_lp,
                                                              uint32_t* partials, const int64_t* __restrict__ tok_ids,
                                                              const __nv_bfloat16* __restrict__ logits, int n, int64_t ld,
                                                              int64_t id_offset, int n_top) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ __align__(16) uint32_t rec[lp_rec_bytes(B2_MAX_TOP_LOGPROBS) / 4];
  const int nc = lp_ctas(n);  // the cluster's size: blockIdx.x = r * nc + (the CTA's rank in it)
  const int r = blockIdx.x / nc, c = blockIdx.x - r * nc;
  lp_row<H, K>(reinterpret_cast<LpHead*>(rec), logits + (size_t)r * ld, n, id_offset, tok_ids, r, n_top, nc, c);
  if (c != 0) return;
  const int words = (int)(lp_rec_bytes(n_top) / 4);
  if (partials) {
    for (int j = threadIdx.x; j < words; j += kLpThreads) partials[(size_t)r * words + j] = rec[j];
  } else if (threadIdx.x == 0) {
    lp_finish(reinterpret_cast<const uint8_t*>(rec), 0, 1, n_top, r, ids_out, tok_lp, top_ids, top_lp);
  }
}

__global__ void __launch_bounds__(128) logprobs_merge_kernel(int64_t* ids_out, float* tok_lp, int64_t* top_ids, float* top_lp,
                                                             const uint8_t* all_partials, int nranks, int rows, int n_top) {
  pdl_wait();
  pdl_launch_dependents();
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const size_t rb = lp_rec_bytes(n_top);
  lp_finish(all_partials + r * rb, rows * rb, nranks, n_top, r, ids_out, tok_lp, top_ids, top_lp);
}

}  // namespace b2

using namespace b2;

static int logprobs_launch(int64_t* ids_out, float* tok_lp, int64_t* top_ids, float* top_lp, void* partials, const int64_t* tok_ids,
                           const void* logits, int rows, int n, int64_t ld, int64_t id_offset, int n_top, int ft, void* stream) {
  if (ft != B2_DT_BF16 && ft != B2_DT_F16) return B2_ERR_UNSUPPORTED;
  const cudaError_t e = with_flag(ft == B2_DT_F16, [&](auto h) {
    constexpr bool H = decltype(h)::value;
    auto kern = n_top > 1 ? logprobs_kernel<H, B2_MAX_TOP_LOGPROBS> : logprobs_kernel<H, 1>;
    const int nc = lp_ctas(n);
    return launch_cluster(kern, dim3((unsigned)rows * nc), dim3(kLpThreads), 0, (cudaStream_t)stream, true, (unsigned)nc, ids_out,
                          tok_lp, top_ids, top_lp, (uint32_t*)partials, tok_ids, (const __nv_bfloat16*)logits, n, ld, id_offset,
                          n_top);
  });
  if (e != cudaSuccess) {
    set_last_error(partials ? "logprobs_shard" : "logprobs", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

extern "C" {

size_t b2_logprobs_partial_bytes(int n_top) {
  return n_top < 0 || n_top > B2_MAX_TOP_LOGPROBS ? 0 : lp_rec_bytes(n_top);
}

int b2_logprobs(int64_t* ids_out, float* tok_lp, int64_t* top_ids, float* top_lp, const int64_t* tok_ids, const void* logits, int rows,
                int n, int64_t ld, int n_top, int ft, void* stream) {
  if (n_top < 0 || n_top > B2_MAX_TOP_LOGPROBS || !logits || rows <= 0 || n < 1 || ld < n) return B2_ERR_PARAM;
  if (n >= INT_MAX) return B2_ERR_PARAM;  // INT_MAX marks padding
  if ((n_top > 0) != (top_ids != nullptr) || (n_top > 0) != (top_lp != nullptr) || (!ids_out && !tok_lp && n_top == 0))
    return B2_ERR_PARAM;
  if ((int64_t)rows * lp_ctas(n) > INT_MAX) return B2_ERR_LIMIT;
  return logprobs_launch(ids_out, tok_lp, top_ids, top_lp, nullptr, tok_ids, logits, rows, n, ld, 0, n_top, ft, stream);
}

int b2_logprobs_shard(void* partials, const int64_t* tok_ids, const void* logits, int rows, int n, int64_t ld, int64_t id_offset,
                      int n_top, int ft, void* stream) {
  if (n_top < 0 || n_top > B2_MAX_TOP_LOGPROBS || !partials || !logits || rows <= 0 || n < 1 || ld < n) return B2_ERR_PARAM;
  if (id_offset < 0 || id_offset + n >= (int64_t)INT_MAX) return B2_ERR_PARAM;  // global ids are int32; INT_MAX marks padding
  if ((uintptr_t)partials & 3) return B2_ERR_UNSUPPORTED;
  if ((int64_t)rows * lp_ctas(n) > INT_MAX) return B2_ERR_LIMIT;
  return logprobs_launch(nullptr, nullptr, nullptr, nullptr, partials, tok_ids, logits, rows, n, ld, id_offset, n_top, ft, stream);
}

int b2_logprobs_merge(int64_t* ids_out, float* tok_lp, int64_t* top_ids, float* top_lp, const void* all_partials, int nranks,
                      int rows, int n_top, void* stream) {
  if (n_top < 0 || n_top > B2_MAX_TOP_LOGPROBS || !all_partials || nranks < 1 || rows <= 0) return B2_ERR_PARAM;
  if ((n_top > 0) != (top_ids != nullptr) || (n_top > 0) != (top_lp != nullptr) || (!ids_out && !tok_lp && n_top == 0))
    return B2_ERR_PARAM;
  if ((uintptr_t)all_partials & 3) return B2_ERR_UNSUPPORTED;
  const cudaError_t e = launch(logprobs_merge_kernel, dim3((rows + 127) / 128), dim3(128), 0, (cudaStream_t)stream, true, ids_out,
                               tok_lp, top_ids, top_lp, (const uint8_t*)all_partials, nranks, rows, n_top);
  if (e != cudaSuccess) {
    set_last_error("logprobs_merge", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

}  // extern "C"
