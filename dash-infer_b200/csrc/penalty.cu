// b200spark — the logits processor of the sampling step (b2_penalize: repetition, presence and frequency penalties,
// no-repeat n-grams, min-length) and of a verify step's rows (b2_penalize_tokens) over a per-sequence token history kept
// on the device (b2_history_load / _append / _append_tokens).
// Reference counterpart: LogitsProcessor, beam_search.cu:329-539, called from GenerateOp::RunSample.  The contract is in
// include/b200spark.h.
//
// The reference copies the whole [B, vocab] row, clears a [B, vocab] count table, re-counts the [B, max_len] history with
// atomics and subtracts a penalty from every column, every step.  Here the history keeps its per-id state (a generated
// count and an in-prompt bit) and the list of its distinct ids, updated once per appended token, so a row's work is one
// visit per distinct id plus the n-gram scan.  Visiting each distinct id once also removes the read-after-write hazard
// between duplicate ids that the reference avoids with its copy of the row.
//
// One CTA per row: the penalty phase writes each distinct id once; after a barrier, the ban phase writes the constant
// FT(-1e9f) (several threads may write it to one id).
#include "b2_common.cuh"

namespace b2 {

constexpr int kPenThreads = 512;
constexpr int kLoadThreads = 1024;
constexpr int32_t kInPrompt = 1 << 30;
constexpr int32_t kCountMask = kInPrompt - 1;

template <bool H>
struct PenFt {
  using T = __nv_bfloat16;
  static __device__ __forceinline__ T from_f(float v) { return __float2bfloat16(v); }  // cvt.rn.bf16.f32
};
template <>
struct PenFt<true> {
  using T = __half;
  static __device__ __forceinline__ T from_f(float v) { return __float2half_rn(v); }  // cvt.rn.f16.f32
};

// The reference's fp32 penalty sum, compiled with --use_fast_math: mul.ftz, then add.ftz (no contraction: the add is
// conditional).
__device__ __forceinline__ float mul_ftz(float a, float b) {
  float d;
  asm("mul.rn.ftz.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
  return d;
}
__device__ __forceinline__ float add_ftz(float a, float b) {
  float d;
  asm("add.rn.ftz.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
  return d;
}

// Slot `slot` := ids[0 .. n_ids), the first prompt_len the prompt.  The old entries are cleared through the old distinct
// list; the new list is built with atomics (the first thread to move an entry off 0 appends the id).
__global__ void __launch_bounds__(kLoadThreads) history_load_kernel(b2_token_history h, int slot, const int32_t* ids, int n_ids,
                                                                    int prompt_len) {
  __shared__ int s_nd;
  pdl_wait();
  pdl_launch_dependents();
  const size_t so = (size_t)slot;
  int32_t* tab = h.table + so * h.vocab;
  int32_t* tok = h.tokens + so * h.max_len;
  int32_t* dl = h.distinct + so * h.max_len;
  const int nd_old = h.n_distinct[slot];
  for (int i = threadIdx.x; i < nd_old; i += blockDim.x) tab[dl[i]] = 0;
  if (threadIdx.x == 0) s_nd = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n_ids; i += blockDim.x) {
    const int32_t t = ids[i];
    const bool ok = t >= 0 && t < h.vocab;
    tok[i] = ok ? t : -1;
    if (!ok) continue;
    const int32_t old = i < prompt_len ? atomicOr(&tab[t], kInPrompt) : atomicAdd(&tab[t], 1);
    if (old == 0) dl[atomicAdd(&s_nd, 1)] = t;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    h.len[slot] = n_ids;
    h.prompt_len[slot] = prompt_len;
    h.n_distinct[slot] = s_nd;
  }
}

// Append id *id to slot r: the token, its table entry, the distinct list (an id whose entry leaves 0 goes to its end) and
// len.  A full slot is left as it is.  Every append of the history goes through here.  The id is passed by address and
// read after the full-slot check, as history_append_kernel always read it; that keeps its machine code what it was.
__device__ __forceinline__ void history_push(const b2_token_history& h, int r, const int64_t* id) {
  const int L = h.len[r];
  if (L >= h.max_len) return;
  const int64_t t = *id;
  const bool ok = t >= 0 && t < h.vocab;
  h.tokens[(size_t)r * h.max_len + L] = ok ? (int32_t)t : -1;
  if (ok) {
    int32_t* e = h.table + (size_t)r * h.vocab + t;
    const int32_t old = *e;
    if (old == 0) {
      const int nd = h.n_distinct[r];
      h.distinct[(size_t)r * h.max_len + nd] = (int32_t)t;
      h.n_distinct[r] = nd + 1;
    }
    *e = old + 1;
  }
  h.len[r] = L + 1;
}

__global__ void history_append_kernel(b2_token_history h, const int64_t* ids, int rows) {
  pdl_wait();
  pdl_launch_dependents();
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  history_push(h, r, ids + r);
}

// The emitted tokens of a verify step, in order, one thread per sequence (appends to one slot are sequential).
__global__ void history_append_tokens_kernel(b2_token_history h, const int64_t* pred, const int32_t* accepted,
                                             const int32_t* path, int batch, int q_len) {
  pdl_wait();
  pdl_launch_dependents();
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= batch) return;
  const int64_t* row = pred + (size_t)r * q_len;
  const int n = min(max(accepted[r], 0), q_len);
  for (int i = 0; i < n; ++i) {
    int u = i;
    if (path != nullptr) {
      u = path[(size_t)r * q_len + i];
      u = (unsigned)u < (unsigned)q_len ? u : 0;
    }
    history_push(h, r, row + u);
  }
}

// Steps 1 and 2 of the contract for one id of generated count cnt, from its value v: penalize_kernel's loop body, which
// keeps its own copy (calling this from it changes its register allocation).
template <bool H>
__device__ __forceinline__ typename PenFt<H>::T pen_value(typename PenFt<H>::T v, int cnt, typename PenFt<H>::T R, bool rep,
                                                          bool sup, float freq, float pres) {
  using F = PenFt<H>;
  using T = typename F::T;
  if (rep && (!sup || cnt > 0)) v = __hlt(v, F::from_f(0.f)) ? __hmul(v, R) : __hdiv(v, R);
  float s = mul_ftz(__int2float_rn(cnt), freq);
  if (cnt > 0) s = add_ftz(s, pres);
  const T pen = F::from_f(s);
  if (*reinterpret_cast<const unsigned short*>(&pen) != 0) v = __hsub(v, pen);
  return v;
}

template <bool H>
__global__ void __launch_bounds__(kPenThreads) penalize_kernel(__nv_bfloat16* logits, int n, int64_t ld, int64_t id_offset,
                                                               b2_token_history h, b2_penalty_params p) {
  using F = PenFt<H>;
  using T = typename F::T;
  pdl_wait();
  pdl_launch_dependents();
  const int r = blockIdx.x;
  T* x = reinterpret_cast<T*>(logits + (size_t)r * ld);
  const int L = h.len[r];
  const int nd = h.n_distinct[r];
  const int32_t* tab = h.table + (size_t)r * h.vocab;
  const int32_t* dl = h.distinct + (size_t)r * h.max_len;
  const int32_t* tok = h.tokens + (size_t)r * h.max_len;
  const T R = F::from_f(p.repetition[r]);
  const bool rep = !__heq(R, F::from_f(1.f));
  const bool sup = p.suppress[r] != 0;
  const float freq = p.frequency[r], pres = p.presence[r];
  const int g = p.no_repeat_ngram[r];
  // the column of vocabulary id t, or -1 outside the shard
  auto col = [&](int32_t t) { return (uint64_t)((int64_t)t - id_offset) < (uint64_t)n ? (int)((int64_t)t - id_offset) : -1; };

  for (int i = threadIdx.x; i < nd; i += blockDim.x) {
    const int32_t t = dl[i];
    const int c = col(t);
    if (c < 0) continue;
    const int cnt = tab[t] & kCountMask;
    T v = x[c];
    if (rep && (!sup || cnt > 0)) v = __hlt(v, F::from_f(0.f)) ? __hmul(v, R) : __hdiv(v, R);
    float s = mul_ftz(__int2float_rn(cnt), freq);
    if (cnt > 0) s = add_ftz(s, pres);
    const T pen = F::from_f(s);
    if (*reinterpret_cast<const unsigned short*>(&pen) != 0) v = __hsub(v, pen);
    x[c] = v;
  }
  __syncthreads();  // every penalty write lands before a ban may overwrite it
  const T ban = F::from_f(-1e9f);
  if (g == 1) {  // every id of the history
    for (int i = threadIdx.x; i < nd; i += blockDim.x) {
      const int c = col(dl[i]);
      if (c >= 0) x[c] = ban;
    }
  } else if (g > 1) {
    const int32_t* tail = tok + (L - g + 1);  // the last g - 1 tokens
    for (int j = threadIdx.x; j <= L - g; j += blockDim.x) {
      int i = 0;
      while (i < g - 1 && tok[j + i] == tail[i]) ++i;
      if (i == g - 1) {
        const int c = col(tok[j + g - 1]);
        if (c >= 0) x[c] = ban;
      }
    }
  }
  if (threadIdx.x == 0 && L < p.min_length[r] && p.eos_id[r] >= 0) {
    const int c = col(p.eos_id[r]);
    if (c >= 0) x[c] = ban;
  }
}

// Row r = b * q_len + t of a verify step: penalize_kernel's row over the virtual history V = slot b followed by the
// drafts on the path from the root to node t (the set bits of anc(t) above bit 0, ascending), appended as
// history_push would append them.  The slot is only read; the path's d tokens sit in shared memory, and a path token
// counts as one more generated occurrence of its id.  Distinct ids of V: the slot's list, then the path ids whose table
// entry is 0 at their first path position; the two sets are disjoint, so each column is still written once before the
// barrier.
template <bool H>
__global__ void __launch_bounds__(kPenThreads) penalize_tokens_kernel(__nv_bfloat16* logits, int n, int64_t ld, int64_t id_offset,
                                                                      b2_token_history h, b2_penalty_params p,
                                                                      const int64_t* tokens, const int32_t* parents, int q_len) {
  using F = PenFt<H>;
  using T = typename F::T;
  __shared__ int32_t s_path[kMaxQLen - 1];
  __shared__ int s_d;
  pdl_wait();
  pdl_launch_dependents();
  const int r = blockIdx.x;
  const int b = r / q_len, node = r - b * q_len;
  T* x = reinterpret_cast<T*>(logits + (size_t)r * ld);
  const int L = h.len[b];
  const int nd = h.n_distinct[b];
  const int32_t* tab = h.table + (size_t)b * h.vocab;
  const int32_t* dl = h.distinct + (size_t)b * h.max_len;
  const int32_t* tok = h.tokens + (size_t)b * h.max_len;
  if (threadIdx.x == 0) {
    int depth;
    unsigned anc = parents != nullptr ? tree_walk(parents + (size_t)b * q_len, node, depth) : (2u << node) - 1u;
    const int room = max(h.max_len - L, 0);
    int d = 0;
    for (anc &= ~1u; anc != 0 && d < room; anc &= anc - 1u) {
      const int64_t v = tokens[(size_t)b * q_len + (__ffs(anc) - 1)];
      s_path[d++] = v >= 0 && v < h.vocab ? (int32_t)v : -1;
    }
    s_d = d;
  }
  __syncthreads();
  const int d = s_d, Lv = L + d;
  const T R = F::from_f(p.repetition[b]);
  const bool rep = !__heq(R, F::from_f(1.f));
  const bool sup = p.suppress[b] != 0;
  const float freq = p.frequency[b], pres = p.presence[b];
  const int g = p.no_repeat_ngram[b];
  auto col = [&](int32_t t) { return (uint64_t)((int64_t)t - id_offset) < (uint64_t)n ? (int)((int64_t)t - id_offset) : -1; };
  auto on_path = [&](int32_t t, int end) {
    int k = 0;
    for (int j = 0; j < end; ++j) k += s_path[j] == t;
    return k;
  };
  auto token = [&](int q) { return q < L ? tok[q] : s_path[q - L]; };

  for (int i = threadIdx.x; i < nd; i += blockDim.x) {
    const int32_t t = dl[i];
    const int c = col(t);
    if (c < 0) continue;
    x[c] = pen_value<H>(x[c], (tab[t] & kCountMask) + on_path(t, d), R, rep, sup, freq, pres);
  }
  if (threadIdx.x < d) {
    const int32_t t = s_path[threadIdx.x];
    const int c = col(t);
    if (c >= 0 && tab[t] == 0 && on_path(t, threadIdx.x) == 0) x[c] = pen_value<H>(x[c], on_path(t, d), R, rep, sup, freq, pres);
  }
  __syncthreads();  // every penalty write lands before a ban may overwrite it
  const T ban = F::from_f(-1e9f);
  if (g == 1) {  // every id of V
    for (int i = threadIdx.x; i < nd; i += blockDim.x) {
      const int c = col(dl[i]);
      if (c >= 0) x[c] = ban;
    }
    if (threadIdx.x < d) {
      const int c = col(s_path[threadIdx.x]);
      if (c >= 0) x[c] = ban;
    }
  } else if (g > 1) {
    const int tail = Lv - g + 1;  // the last g - 1 tokens of V start here
    for (int j = threadIdx.x; j <= Lv - g; j += blockDim.x) {
      int i = 0;
      while (i < g - 1 && token(j + i) == token(tail + i)) ++i;
      if (i == g - 1) {
        const int c = col(token(j + g - 1));
        if (c >= 0) x[c] = ban;
      }
    }
  }
  if (threadIdx.x == 0 && Lv < p.min_length[b] && p.eos_id[b] >= 0) {
    const int c = col(p.eos_id[b]);
    if (c >= 0) x[c] = ban;
  }
}

static bool history_ok(const b2_token_history* h) {
  return h && h->tokens && h->len && h->prompt_len && h->table && h->distinct && h->n_distinct && h->max_len > 0 &&
         h->max_len < kInPrompt && h->vocab > 0;
}

}  // namespace b2

using namespace b2;

extern "C" {

int b2_history_load(const b2_token_history* hist, int slot, const int32_t* ids, int n_ids, int prompt_len, void* stream) {
  if (!history_ok(hist) || slot < 0 || n_ids < 0 || n_ids > hist->max_len || prompt_len < 0 || prompt_len > n_ids ||
      (n_ids > 0 && !ids))
    return B2_ERR_PARAM;
  B2_CUDA_TRY(launch(history_load_kernel, dim3(1), dim3(kLoadThreads), 0, (cudaStream_t)stream, true, *hist, slot, ids,
                     n_ids, prompt_len));
  return B2_OK;
}

int b2_history_append(const b2_token_history* hist, const int64_t* ids, int rows, void* stream) {
  if (!history_ok(hist) || !ids || rows < 0) return B2_ERR_PARAM;
  if (rows == 0) return B2_OK;
  B2_CUDA_TRY(launch(history_append_kernel, dim3((rows + 127) / 128), dim3(128), 0, (cudaStream_t)stream, true, *hist,
                     ids, rows));
  return B2_OK;
}

int b2_history_append_tokens(const b2_token_history* hist, const int64_t* pred, const int32_t* accepted, const int32_t* path,
                             int batch, int q_len, void* stream) {
  if (!history_ok(hist) || !pred || !accepted || batch < 0) return B2_ERR_PARAM;
  if (q_len < 1 || q_len > kMaxQLen) return B2_ERR_LIMIT;
  if (batch == 0) return B2_OK;
  B2_CUDA_TRY(launch(history_append_tokens_kernel, dim3((batch + 127) / 128), dim3(128), 0, (cudaStream_t)stream, true,
                     *hist, pred, accepted, path, batch, q_len));
  return B2_OK;
}

int b2_penalize(void* logits, int rows, int n, int64_t ld, int64_t id_offset, const b2_token_history* hist,
                const b2_penalty_params* params, int ft, void* stream) {
  if (!logits || !history_ok(hist) || !params || !params->repetition || !params->presence || !params->frequency ||
      !params->no_repeat_ngram || !params->min_length || !params->eos_id || !params->suppress)
    return B2_ERR_PARAM;
  if (rows < 0 || n < 1 || ld < n || id_offset < 0 || id_offset + n > hist->vocab) return B2_ERR_PARAM;
  if (ft != B2_DT_BF16 && ft != B2_DT_F16) return B2_ERR_PARAM;
  if (rows == 0) return B2_OK;
  const cudaError_t e = with_flag(ft == B2_DT_F16, [&](auto h) {
    constexpr bool H = decltype(h)::value;
    return launch(penalize_kernel<H>, dim3((unsigned)rows), dim3(kPenThreads), 0, (cudaStream_t)stream, true,
                  (__nv_bfloat16*)logits, n, ld, id_offset, *hist, *params);
  });
  if (e != cudaSuccess) {
    set_last_error("penalize", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

int b2_penalize_tokens(void* logits, int batch, int q_len, const int32_t* parents, const int64_t* tokens, int n, int64_t ld,
                       int64_t id_offset, const b2_token_history* hist, const b2_penalty_params* params, int ft, void* stream) {
  if (!logits || !tokens || !history_ok(hist) || !params || !params->repetition || !params->presence || !params->frequency ||
      !params->no_repeat_ngram || !params->min_length || !params->eos_id || !params->suppress)
    return B2_ERR_PARAM;
  if (batch < 0 || n < 1 || ld < n || id_offset < 0 || id_offset + n > hist->vocab) return B2_ERR_PARAM;
  if (ft != B2_DT_BF16 && ft != B2_DT_F16) return B2_ERR_PARAM;
  if (q_len < 1 || q_len > kMaxQLen || (int64_t)batch * q_len > INT32_MAX) return B2_ERR_LIMIT;
  if (batch == 0) return B2_OK;
  const cudaError_t e = with_flag(ft == B2_DT_F16, [&](auto h) {
    constexpr bool H = decltype(h)::value;
    return launch(penalize_tokens_kernel<H>, dim3((unsigned)(batch * q_len)), dim3(kPenThreads), 0, (cudaStream_t)stream, true,
                  (__nv_bfloat16*)logits, n, ld, id_offset, *hist, *params, tokens, parents, q_len);
  });
  if (e != cudaSuccess) {
    set_last_error("penalize_tokens", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

}  // extern "C"
