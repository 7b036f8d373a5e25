// b200spark — n-gram (prompt-lookup) drafting of speculative tokens from the per-sequence token history (b2_ngram_draft).
// The contract is in include/b200spark.h; DESIGN.md §3.3 gives the reasons.
//
// One CTA per sequence.  Pass 1 computes the match length m(e) of every end position e (each thread 8 consecutive
// positions, all loads issued before any compare; almost every position fails its first compare, so the pass is about one
// read of the history) and reduces n* = max m(e).  Pass 2 walks e downwards in block-sized chunks, collects the `width`
// most recent positions with m(e) >= n* by per-thread counts and a block prefix sum, and stops at the chunk that completes
// them.  Warp 0 then builds the trie of the candidates' continuations level by level (at most 16 nodes are kept, so at
// most 15 levels of at most 15 candidates) and writes the outputs.
#include "b2_common.cuh"

namespace b2 {

constexpr int kDraftThreads = 1024;
constexpr int kDraftRun = 8;  // consecutive end positions per thread and chunk
constexpr int kDraftChunk = kDraftThreads * kDraftRun;
constexpr int kMaxNgram = 16;

// m(e) for e = hi, hi - 1, ..., hi - kDraftRun + 1 (0 for e < 0); tail[i] = S[L-1-i], read for i <= e < L - 1 only
__device__ __forceinline__ void match_run(const int32_t* S, int hi, const int32_t* tail, int n_max, int (&m)[kDraftRun]) {
  int32_t x[kDraftRun];
#pragma unroll
  for (int u = 0; u < kDraftRun; ++u) x[u] = hi - u >= 0 ? S[hi - u] : 0;
  const int32_t t0 = tail[0];
#pragma unroll
  for (int u = 0; u < kDraftRun; ++u) {
    const int e = hi - u;
    int i = 0;
    if (e >= 0 && x[u] == t0) {
      i = 1;
      while (i < n_max && i <= e && S[e - i] == tail[i]) ++i;
    }
    m[u] = i;
  }
}

// (kDraftThreads, 1): with the block size alone ptxas holds the kernel to 32 registers and spills
__global__ void __launch_bounds__(kDraftThreads, 1) ngram_draft_kernel(int64_t* tokens, int32_t* parents, int32_t* n_draft,
                                                                    b2_token_history h, int q_len, int n_min, int n_max,
                                                                    int width) {
  __shared__ int32_t s_tail[kMaxNgram];
  __shared__ int s_warp[kDraftThreads / 32];
  __shared__ int s_cand[kMaxQLen];
  __shared__ int32_t s_tok[kMaxQLen];
  __shared__ int s_par[kMaxQLen];
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int L = min(h.len[b], h.max_len);
  const int32_t* S = h.tokens + (size_t)b * h.max_len;
  int64_t* tok = tokens + (size_t)b * q_len;
  if (tid < n_max && tid < L) s_tail[tid] = S[L - 1 - tid];
  __syncthreads();

  int m[kDraftRun];
  int best = 0;
  for (int hi = L - 2 - tid * kDraftRun; hi >= 0; hi -= kDraftChunk) {
    match_run(S, hi, s_tail, n_max, m);
#pragma unroll
    for (int u = 0; u < kDraftRun; ++u) best = max(best, m[u]);
  }
  best = __reduce_max_sync(0xffffffffu, best);
  if (lane == 0) s_warp[warp] = best;
  __syncthreads();
  int nstar = 0;
#pragma unroll 8
  for (int w = 0; w < kDraftThreads / 32; ++w) nstar = max(nstar, s_warp[w]);
  __syncthreads();  // s_warp is reused below

  int found = 0;
  if (nstar >= n_min) {
    for (int base = L - 2; base >= 0 && found < width; base -= kDraftChunk) {
      const int hi = base - tid * kDraftRun;
      match_run(S, hi, s_tail, n_max, m);
      unsigned hits = 0;
#pragma unroll
      for (int u = 0; u < kDraftRun; ++u) hits |= (unsigned)(m[u] >= nstar) << u;
      const int cnt = __popc(hits);
      int incl = cnt;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= off) incl += v;
      }
      if (lane == 31) s_warp[warp] = incl;
      __syncthreads();
      int pre = 0, total = 0;
#pragma unroll 8
      for (int w = 0; w < kDraftThreads / 32; ++w) {
        const int v = s_warp[w];
        pre += w < warp ? v : 0;
        total += v;
      }
      int r = found + pre + incl - cnt;  // rank of this thread's first hit, most recent first
#pragma unroll
      for (int u = 0; u < kDraftRun; ++u) {
        if ((hits >> u & 1) && r < width) s_cand[r] = hi - u;
        r += hits >> u & 1;
      }
      found += total;
      __syncthreads();  // s_warp is rewritten by the next chunk; s_cand is complete when the loop ends
    }
  }
  if (warp != 0) return;

  const int64_t t0 = tok[0];
  const int nc = min(found, width);
  const bool have = lane < nc;
  const int e = have ? s_cand[lane] : 0;
  const int p = L - 1 - e;  // the period of this candidate's continuation
  if (parents == nullptr) {  // chain: width 1
    if (lane >= 1 && lane < q_len) {
      int64_t v = t0;
      if (nc > 0) {
        const int e0 = s_cand[0];
        const int32_t s = S[e0 + 1 + (lane - 1) % (L - 1 - e0)];
        if (s >= 0) v = s;
      }
      tok[lane] = v;
    }
    if (n_draft != nullptr && lane == 0) n_draft[b] = nc > 0 ? q_len - 1 : 0;
    return;
  }

  // tree: level k + 1 of the trie holds the distinct prefixes of length k + 1.  Candidate j (lane j) sits at node `node`
  // of level k; its child is (node, c_k).  The leader of a child is the first candidate (lowest rank) that reaches it, and
  // the children of a level are numbered by (parent node, leader rank).  Every child of a level outranks every node of the
  // level before it, so once q_len nodes are numbered no later node can be kept.
  int node = 0, count = 1;
  for (int k = 0; k < q_len - 1 && count < q_len && nc > 0; ++k) {
    const int32_t c = have ? S[e + 1 + k % p] : 0;
    int leader = lane;
    for (int i = 0; i < nc; ++i) {
      const int ni = __shfl_sync(0xffffffffu, node, i);
      const int32_t ci = __shfl_sync(0xffffffffu, c, i);
      if (i < leader && ni == node && ci == c) leader = i;
    }
    const unsigned leads = __ballot_sync(0xffffffffu, have && leader == lane);
    int rank = 0;  // the leaders numbered before this lane's child, were this lane a leader
    for (int i = 0; i < nc; ++i) {
      const int ni = __shfl_sync(0xffffffffu, node, i);
      rank += (leads >> i & 1) && (ni < node || (ni == node && i < lane));
    }
    const int n_level = __popc(leads);
    const int child = count + __shfl_sync(0xffffffffu, rank, leader);
    if (have && leader == lane && child < q_len) {
      s_tok[child] = c;
      s_par[child] = node;
    }
    node = child;
    count += n_level;
  }
  __syncwarp();
  const int nodes = min(count, q_len);
  if (lane < q_len) {
    const bool real = lane >= 1 && lane < nodes;
    if (lane >= 1) tok[lane] = real && s_tok[lane] >= 0 ? (int64_t)s_tok[lane] : t0;
    parents[(size_t)b * q_len + lane] = real ? s_par[lane] : 0;
  }
  if (n_draft != nullptr && lane == 0) n_draft[b] = nodes - 1;
}

}  // namespace b2

using namespace b2;

extern "C" {

int b2_ngram_draft(int64_t* tokens, int32_t* parents, int32_t* n_draft, const b2_token_history* hist, int batch, int q_len,
                   int n_min, int n_max, int width, void* stream) {
  if (!tokens || !hist || !hist->tokens || !hist->len || hist->max_len <= 0 || batch < 0) return B2_ERR_PARAM;
  if (n_min < 1 || n_min > n_max || width < 1 || (!parents && width != 1)) return B2_ERR_PARAM;
  if (q_len < 2 || q_len > kMaxQLen || n_max > kMaxNgram) return B2_ERR_LIMIT;
  if (width > q_len - 1) return B2_ERR_PARAM;
  if (batch == 0) return B2_OK;
  B2_CUDA_TRY(launch(ngram_draft_kernel, dim3((unsigned)batch), dim3(kDraftThreads), 0, (cudaStream_t)stream, true, tokens,
                     parents, n_draft, *hist, q_len, n_min, n_max, width));
  return B2_OK;
}

}  // extern "C"
