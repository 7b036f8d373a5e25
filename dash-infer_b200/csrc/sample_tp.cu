// b200spark — b2_sample under tensor parallelism (b2_sample_shard, b2_sample_shard_merge): each rank holds a contiguous
// vocab range of the rows, and the ranks draw b2_sample's id of the whole row by exchanging small per-row records.  The
// contract is in include/b200spark.h.
//
// b2_sample's cluster form already splits a long row into contiguous chunks that meet at six points (the argmax, the
// level-1 histogram, three level-2 selections, the tie prefix).  Here each meeting point is a record all-gathered between
// two launches, and what a CTA of the cluster keeps in shared memory across a meeting point is the per-row state, kept in
// each rank's own memory and derived by every rank from the same records.  Every rank weighs its elements with
// smp_weight at the same global maximum m and the same c, so every sum after that is an integer and neither the split nor
// the rank order can change a result.
//
// One 1024-thread CTA per row and phase.  The shard is read from global memory in every phase that needs it (it stays in
// L2 between the phases: 9.7 MB at B = 64 on two ranks of a 152064-column row).
#include <climits>

#include "sample_shared.cuh"

namespace b2 {

constexpr int kStThreads = 1024;
constexpr uint32_t kNoSel = 0xffffffffu;  // the state's hb when no selection is pending

struct StArgRec {  // phase 0: the shard's argmax under argmax_beats, its global id
  float v;
  int32_t id;
};
struct StHist1Rec {  // phase 1: the shard's level-1 histogram
  u64 mass[256];
  uint32_t cnt[256];
};
// phases 2-4: uint32_t[256], the shard's level-2 counts within the pending selection's high byte;  phase 5: int64_t, the
// drawn id on the rank that holds it, else -1

struct StState {  // per row, rank-local
  u64 totm1[256];  // the row's level-1 histogram (phase 2 on)
  uint32_t tot1[256];
  u64 T, acnt, amass;  // the pending selection: its target, the counts / weights of the high bytes above its bin
  u64 Sk, Sp;
  float m, c;
  int32_t gid;   // the row's argmax id (greedy rows take it)
  int32_t rank;  // this rank's index among the ranks
  int32_t k;     // top-k against n_total
  int32_t greedy;
  uint32_t hb;   // the pending selection's high byte, or kNoSel
  uint32_t pad;
};

// bytes per row of phase `phase`'s record (0 <= phase < B2_SAMPLE_SHARD_PHASES)
__host__ __device__ constexpr size_t st_rec_bytes(int phase) {
  return phase == 0 ? sizeof(StArgRec) : phase == 1 ? sizeof(StHist1Rec) : phase == 5 ? sizeof(int64_t) : 256 * sizeof(uint32_t);
}

struct StArgs {
  void* rec_out;
  StState* state;
  const uint8_t* all_rec;
  const uint16_t* logits;
  const float* temperature;
  const int32_t* top_k;
  const float* top_p;
  const uint64_t* seeds;
  const uint64_t* offsets;
  int64_t ld;
  int nranks, rows, n, id_offset, n_total;
};

__device__ __forceinline__ const uint8_t* st_rec(const StArgs& a, int phase, int q, int r) {
  return a.all_rec + ((size_t)q * a.rows + r) * st_rec_bytes(phase);
}

// Level 1 of one element per lane (the whole warp calls it): sample.cu's warp-aggregated atomic pair per distinct bin.
// (sample.cu keeps its copy of this loop inline, so its kernels compile as they did.)
__device__ __forceinline__ void st_level1_add(uint32_t* cnt1, u64* mass1, bool valid, uint32_t hb, u64 wt, int lane) {
  uint32_t todo = __ballot_sync(0xffffffffu, valid);
  while (todo) {
    const int lead = __ffs(todo) - 1;
    const uint32_t h = __shfl_sync(0xffffffffu, hb, lead);
    const bool mine = valid && hb == h;
    const uint32_t grp = __ballot_sync(0xffffffffu, mine);
    const uint32_t slo = __reduce_add_sync(0xffffffffu, mine ? (uint32_t)(wt & 0xffffffu) : 0u);  // < 2^29
    const uint32_t shi = __reduce_add_sync(0xffffffffu, mine ? (uint32_t)(wt >> 24) : 0u);         // <= 2^21
    if (lane == lead) {
      atomicAdd(&cnt1[h], (uint32_t)__popc(grp));
      atomicAdd(&mass1[h], ((u64)shi << 24) + slo);
    }
    todo &= ~grp;
  }
}

struct StShared {
  uint32_t cnt[256];  // the shard's histogram of this phase (level 1 or level 2)
  u64 mass[256];
  uint32_t tot1[256];  // the row's level-1 histogram
  u64 totm1[256];
  uint32_t tot2[256];  // the row's level-2 counts of the selection that ends in this phase
  uint32_t wcnt[32];
  float wv[32];
  int wi[32];
  uint32_t hb, key;
  u64 j, acnt, amass;
  int wsel;
  uint32_t wrank;
  long long id;
};

// the shard's level-2 counts within high byte hb, written as this phase's record (all threads)
template <bool H>
__device__ __forceinline__ void st_level2(StShared& sh, const uint16_t* row, int n, uint32_t hb, uint32_t* rec) {
  const int tid = threadIdx.x;
  if (tid < 256) sh.cnt[tid] = 0;
  __syncthreads();
  if (hb != kNoSel) {
    for (int i = tid; i < n; i += kStThreads) {
      const uint32_t k = smp_key(row[i]);
      if ((k >> 8) == hb) atomicAdd(&sh.cnt[k & 255], 1u);
    }
  }
  __syncthreads();
  if (tid < 256) rec[tid] = sh.cnt[tid];
}

// Warp 0: the end of a selection begun at high byte hb (target T, a1c / a1m above hb) from the row's level-2 counts
// sh.tot2, as smp_select ends it: sh.key, sh.j, sh.acnt, sh.amass (written by lane 0).
template <bool H>
__device__ __forceinline__ void st_finish(StShared& sh, uint32_t hb, u64 T, u64 a1c, u64 a1m, bool by_mass, float m, float c,
                                          int lane) {
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

// the row's level-2 counts: the sum over the ranks of the previous phase's records (threads < 256)
__device__ __forceinline__ void st_sum_level2(StShared& sh, const StArgs& a, int phase, int r) {
  const int tid = threadIdx.x;
  if (tid < 256) {
    uint32_t s = 0;
    for (int q = 0; q < a.nranks; ++q) s += reinterpret_cast<const uint32_t*>(st_rec(a, phase, q, r))[tid];
    sh.tot2[tid] = s;
  }
}

template <bool H, int PH>
__global__ void __launch_bounds__(kStThreads) sample_shard_kernel(const StArgs a) {
  __shared__ StShared sh;
  pdl_wait();
  pdl_launch_dependents();
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const uint16_t* row = a.logits + (size_t)r * a.ld;
  const int n = a.n;
  uint8_t* out = reinterpret_cast<uint8_t*>(a.rec_out) + (size_t)r * st_rec_bytes(PH);
  StState& S = a.state[r];

  if (PH == 0) {  // the shard's argmax
    float bv = -INFINITY;
    int bi = INT_MAX;
    int i = tid;
    for (; i + 3 * kStThreads < n; i += 4 * kStThreads) {
      uint16_t b[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) b[u] = row[i + u * kStThreads];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float x = smp_val<H>(b[u]);
        if (argmax_beats(x, a.id_offset + i + u * kStThreads, bv, bi)) { bv = x; bi = a.id_offset + i + u * kStThreads; }
      }
    }
    for (; i < n; i += kStThreads) {
      const float x = smp_val<H>(row[i]);
      if (argmax_beats(x, a.id_offset + i, bv, bi)) { bv = x; bi = a.id_offset + i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (argmax_beats(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { sh.wv[w] = bv; sh.wi[w] = bi; }
    __syncthreads();
    if (w == 0) {
      bv = sh.wv[lane];
      bi = sh.wi[lane];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (argmax_beats(ov, oi, bv, bi)) { bv = ov; bi = oi; }
      }
      if (lane == 0) *reinterpret_cast<StArgRec*>(out) = StArgRec{bv, bi};
    }
    return;
  }

  if (PH == 1) {  // the row's m, c, greedy predicate and argmax from the ranks' argmaxes (lane q holds rank q's); then the
                  // shard's level-1 histogram
    if (w == 0) {
      const StArgRec* rec = lane < a.nranks ? reinterpret_cast<const StArgRec*>(st_rec(a, 0, lane, r)) : nullptr;
      float bv = rec ? rec->v : -INFINITY;
      int bi = rec ? rec->id : INT_MAX;
      const uint32_t mine = __ballot_sync(0xffffffffu, rec && bi >= a.id_offset && bi < a.id_offset + n);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (argmax_beats(ov, oi, bv, bi)) { bv = ov; bi = oi; }
      }
      if (lane == 0) {
        const float t = a.temperature[r];
        const int32_t k_in = a.top_k[r];
        const float c = __fdiv_rn(__uint_as_float(kLog2eF32), t);
        const bool greedy = !(fabsf(bv) <= 3.402823466e38f) || !(t > 0.f) || !(fabsf(c) <= 3.402823466e38f);
        S.m = bv;
        S.c = c;
        S.gid = bi;
        S.rank = mine ? __ffs(mine) - 1 : 0;
        S.k = (k_in <= 0 || k_in > a.n_total) ? a.n_total : k_in;
        S.greedy = greedy;
        S.hb = kNoSel;
        sh.wv[0] = bv;
        sh.wv[1] = c;
        sh.wi[0] = greedy;
      }
    }
    if (tid < 256) {
      sh.cnt[tid] = 0;
      sh.mass[tid] = 0;
    }
    __syncthreads();
    const float m = sh.wv[0], c = sh.wv[1];
    if (!sh.wi[0]) {
      const int steps = (n + kStThreads - 1) / kStThreads;
      for (int s = 0; s < steps; ++s) {
        const int e = s * kStThreads + tid;
        const bool valid = e < n;
        uint32_t hb = 0;
        u64 wt = 0;
        if (valid) {
          const uint32_t b = row[e];
          hb = smp_key(b) >> 8;
          wt = smp_weight(smp_val<H>(b), m, c);
        }
        st_level1_add(sh.cnt, sh.mass, valid, hb, wt, lane);
      }
    }
    __syncthreads();
    StHist1Rec* rec = reinterpret_cast<StHist1Rec*>(out);
    if (tid < 256) {
      rec->mass[tid] = sh.mass[tid];
      rec->cnt[tid] = sh.cnt[tid];
    }
    return;
  }

  if (PH == 5) {  // the drawn key K, its rank j, the ranks' counts of K: the holding rank finds its element
    if (S.greedy) {
      if (tid == 0) *reinterpret_cast<long long*>(out) = -1;
      return;
    }
    const float m = S.m, c = S.c;
    const uint32_t hb = S.hb;
    st_sum_level2(sh, a, 4, r);
    if (tid == 0) sh.id = -1;
    __syncthreads();
    if (w == 0) st_finish<H>(sh, hb, S.T, S.acnt, S.amass, true, m, c, lane);
    __syncthreads();
    const uint32_t key = sh.key, lo = key & 255;
    const u64 j = sh.j;
    const int rank = S.rank;
    u64 pre = 0;
    for (int q = 0; q < rank; ++q) pre += reinterpret_cast<const uint32_t*>(st_rec(a, 4, q, r))[lo];
    const u64 mine = reinterpret_cast<const uint32_t*>(st_rec(a, 4, rank, r))[lo];
    if (pre < j && j <= pre + mine) {  // uniform over the CTA: the j-th element of K in id order is here
      const int seg = ((n + kStThreads - 1) / kStThreads) * 32;  // warp w holds [w seg, (w + 1) seg)
      uint32_t cnt = 0;
      for (int e = w * seg + lane; e < (w + 1) * seg; e += 32)
        cnt += __popc(__ballot_sync(0xffffffffu, e < n && smp_key(row[e]) == key));
      if (lane == 0) sh.wcnt[w] = cnt;
      __syncthreads();
      if (tid == 0) {
        u64 jl = j - pre;
        sh.wsel = -1;
        for (int x = 0; x < 32; ++x) {
          if (jl <= sh.wcnt[x]) { sh.wsel = x; sh.wrank = (uint32_t)jl; break; }
          jl -= sh.wcnt[x];
        }
      }
      __syncthreads();
      if (w == sh.wsel) {
        const uint32_t want = sh.wrank;
        uint32_t seen = 0;
        for (int e = w * seg + lane; e < (w + 1) * seg; e += 32) {
          const bool hit = e < n && smp_key(row[e]) == key;
          const uint32_t bal = __ballot_sync(0xffffffffu, hit);
          if (seen + __popc(bal) >= want) {
            if (hit && seen + __popc(bal & ((1u << lane) - 1)) + 1 == want) sh.id = (long long)a.id_offset + e;
            break;
          }
          seen += __popc(bal);
        }
      }
      __syncthreads();
    }
    if (tid == 0) *reinterpret_cast<long long*>(out) = sh.id;
    return;
  }

  // phases 2-4: end the pending selection (if any), begin the next one, count the shard's level 2 within its high byte
  uint32_t* rec = reinterpret_cast<uint32_t*>(out);
  if (S.greedy) {
    if (tid < 256) rec[tid] = 0;
    return;
  }
  const float m = S.m, c = S.c;
  if (PH == 2) {  // the row's level 1 from the ranks' records; kept in the state for the later selections
    if (tid < 256) {
      uint32_t sc = 0;
      u64 sm = 0;
      for (int q = 0; q < a.nranks; ++q) {
        const StHist1Rec* h = reinterpret_cast<const StHist1Rec*>(st_rec(a, 1, q, r));
        sc += h->cnt[tid];
        sm += h->mass[tid];
      }
      sh.tot1[tid] = S.tot1[tid] = sc;
      sh.totm1[tid] = S.totm1[tid] = sm;
    }
  } else {
    if (tid < 256) {
      sh.tot1[tid] = S.tot1[tid];
      sh.totm1[tid] = S.totm1[tid];
    }
    if (S.hb != kNoSel) st_sum_level2(sh, a, PH - 1, r);
  }
  __syncthreads();
  if (w == 0) {
    const uint32_t phb = S.hb;
    u64 T = 0;
    bool by_mass = true, sel = true;
    if (PH == 2) {  // top-k: the kept set ends at the k-th element; without a limit S_k is the whole weight
      const int k = S.k;
      if (k == a.n_total) {
        u64 s = 0;
#pragma unroll
        for (int b = 0; b < 8; ++b) s += sh.totm1[lane * 8 + b];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) S.Sk = s;
        sel = false;
      } else {
        T = (u64)k;
        by_mass = false;
      }
    } else if (PH == 3) {  // S_k; top-p: the shortest prefix whose weight reaches Pt
      u64 Sk = S.Sk;
      if (phb != kNoSel) {
        st_finish<H>(sh, phb, S.T, S.acnt, S.amass, false, m, c, lane);
        __syncwarp();
        Sk = sh.amass + sh.j * smp_weight(smp_val<H>(smp_unkey(sh.key)), m, c);
      }
      const float p = a.top_p[r];
      const uint32_t p24 = !(p < 1.f) ? (1u << 24) : min(__float2uint_rn(__fmul_rn(p, 16777216.f)), 1u << 24);
      if (lane == 0) S.Sk = Sk;
      if (p24 < (1u << 24)) {
        T = max(mul_shr24(p24, Sk, true), (u64)1);
      } else {
        if (lane == 0) S.Sp = Sk;
        sel = false;
      }
    } else {  // S_p; the draw: the first element at which the running weight exceeds U
      u64 Sp = S.Sp;
      if (phb != kNoSel) {
        st_finish<H>(sh, phb, S.T, S.acnt, S.amass, true, m, c, lane);
        __syncwarp();
        Sp = sh.amass + sh.j * smp_weight(smp_val<H>(smp_unkey(sh.key)), m, c);
      }
      const u64 seed = a.seeds[r], off = a.offsets[r];
      const uint32_t u24 = philox_r0((uint32_t)off, (uint32_t)(off >> 32), 0, 0, (uint32_t)seed, (uint32_t)(seed >> 32)) >> 8;
      T = mul_shr24(u24, Sp, false) + 1;
      if (lane == 0) S.Sp = Sp;
    }
    uint32_t hb = kNoSel;
    if (sel) {
      u64 ac, am;
      hb = (uint32_t)smp_scan(sh.tot1, [&](int b) { return sh.totm1[b]; }, by_mass, T, lane, ac, am);
      if (lane == 0) {
        S.T = T;
        S.acnt = ac;
        S.amass = am;
      }
    }
    if (lane == 0) {
      S.hb = hb;
      sh.hb = hb;
    }
  }
  __syncthreads();
  st_level2<H>(sh, row, n, sh.hb, rec);
}

// ids_out[r]: the holder's id, or the argmax of a greedy row; offsets[r] += 1
__global__ void __launch_bounds__(128) sample_shard_merge_kernel(int64_t* ids_out, const long long* all_rec, const StState* state,
                                                                 int nranks, int rows, uint64_t* offsets) {
  pdl_wait();
  pdl_launch_dependents();
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  long long id = state[r].gid;
  if (!state[r].greedy) {
    for (int q = nranks - 1; q >= 0; --q) {
      const long long v = all_rec[(size_t)q * rows + r];
      if (v >= 0) id = v;
    }
  }
  ids_out[r] = id;
  offsets[r] += 1;
}

}  // namespace b2

using namespace b2;

extern "C" {

size_t b2_sample_shard_record_bytes(int phase) {
  return (phase >= 0 && phase < B2_SAMPLE_SHARD_PHASES) ? st_rec_bytes(phase) : 0;
}

size_t b2_sample_shard_state_bytes(void) { return sizeof(StState); }

int b2_sample_shard(int phase, void* record_out, void* state, const void* all_records, int nranks, const void* logits, int rows,
                    int n, int64_t ld, int64_t id_offset, int64_t n_total, const float* temperature, const int32_t* top_k,
                    const float* top_p, const uint64_t* seeds, const uint64_t* offsets, int ft, void* stream) {
  if (phase < 0 || phase >= B2_SAMPLE_SHARD_PHASES || !record_out || !state || (phase > 0 && !all_records) || !logits ||
      !temperature || !top_k || !top_p || !seeds || !offsets)
    return B2_ERR_PARAM;
  if (nranks < 1 || nranks > 8 || rows < 0 || n < 1 || ld < n || id_offset < 0 || id_offset + n > n_total) return B2_ERR_PARAM;
  if (ft != B2_DT_BF16 && ft != B2_DT_F16) return B2_ERR_PARAM;
  if (n_total > B2_SAMPLE_MAX_N) return B2_ERR_LIMIT;
  if (rows == 0) return B2_OK;
  StArgs a{record_out, (StState*)state, (const uint8_t*)all_records, (const uint16_t*)logits, temperature, top_k, top_p,
           seeds, offsets, ld, nranks, rows, n, (int)id_offset, (int)n_total};
  const cudaError_t e = with_flag(ft == B2_DT_F16, [&](auto h) {
    constexpr bool H = decltype(h)::value;
    const dim3 g((unsigned)rows), b(kStThreads);
    const cudaStream_t s = (cudaStream_t)stream;
    switch (phase) {
      case 0: return launch(sample_shard_kernel<H, 0>, g, b, 0, s, true, a);
      case 1: return launch(sample_shard_kernel<H, 1>, g, b, 0, s, true, a);
      case 2: return launch(sample_shard_kernel<H, 2>, g, b, 0, s, true, a);
      case 3: return launch(sample_shard_kernel<H, 3>, g, b, 0, s, true, a);
      case 4: return launch(sample_shard_kernel<H, 4>, g, b, 0, s, true, a);
      default: return launch(sample_shard_kernel<H, 5>, g, b, 0, s, true, a);
    }
  });
  if (e != cudaSuccess) {
    set_last_error("sample_shard", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

int b2_sample_shard_merge(int64_t* ids_out, const void* all_records, const void* state, int nranks, int rows, uint64_t* offsets,
                          void* stream) {
  if (!ids_out || !all_records || !state || !offsets || nranks < 1 || nranks > 8 || rows < 0) return B2_ERR_PARAM;
  if (rows == 0) return B2_OK;
  const cudaError_t e = launch(sample_shard_merge_kernel, dim3((unsigned)((rows + 127) / 128)), dim3(128), 0,
                               (cudaStream_t)stream, true, ids_out, (const long long*)all_records, (const StState*)state, nranks,
                               rows, offsets);
  if (e != cudaSuccess) {
    set_last_error("sample_shard_merge", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

}  // extern "C"
