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
// Each phase runs the steps of sample_shared.cuh that the cluster form runs between the same two meeting points, on the
// shard in global memory.  One 1024-thread CTA per row and phase.  The shard is read from global memory in every phase
// that needs it (it stays in L2 between the phases: 9.7 MB at B = 64 on two ranks of a 152064-column row).
#include "sample_shared.cuh"

namespace b2 {

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
  u64 S;               // the kept weight before the pending selection: S_k, then S_p
  u64 unused;          // keeps the state's size
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
  u64 j;
  long long id;
};

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
__global__ void __launch_bounds__(kSmpThreads) sample_shard_kernel(const StArgs a) {
  __shared__ StShared sh;
  pdl_wait();
  pdl_launch_dependents();
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const uint16_t* row = a.logits + (size_t)r * a.ld;
  const int n = a.n;
  uint8_t* out = reinterpret_cast<uint8_t*>(a.rec_out) + (size_t)r * st_rec_bytes(PH);
  StState& S = a.state[r];

  if (PH == 0) {  // the shard's argmax
    float bv;
    int bi;
    smp_argmax<H, false>(row, n, a.id_offset, nullptr, sh.wv, sh.wi, bv, bi);
    if (tid == 0) *reinterpret_cast<StArgRec*>(out) = StArgRec{bv, bi};
    return;
  }

  if (PH == 1) {  // the row's argmax and parameters from the ranks' argmaxes (lane q holds rank q's); the shard's level 1
    if (w == 0) {
      const StArgRec* rec = lane < a.nranks ? reinterpret_cast<const StArgRec*>(st_rec(a, 0, lane, r)) : nullptr;
      float bv = rec ? rec->v : -INFINITY;
      int bi = rec ? rec->id : INT_MAX;
      const uint32_t mine = __ballot_sync(0xffffffffu, rec && bi >= a.id_offset && bi < a.id_offset + n);
      warp_argmax(bv, bi);
      if (lane == 0) {
        const SmpRow R = smp_row_setup(bv, a.temperature[r], a.top_k[r], a.n_total);
        S.m = R.m;
        S.c = R.c;
        S.gid = bi;
        S.rank = mine ? __ffs(mine) - 1 : 0;
        S.k = R.k;
        S.greedy = R.greedy;
        S.hb = kNoSel;
        sh.wv[0] = R.m;
        sh.wv[1] = R.c;
        sh.wi[0] = R.greedy;
      }
    }
    if (tid < 256) {
      sh.cnt[tid] = 0;
      sh.mass[tid] = 0;
    }
    __syncthreads();
    if (!sh.wi[0]) smp_level1<H>(sh.cnt, sh.mass, row, n, sh.wv[0], sh.wv[1]);
    __syncthreads();
    StHist1Rec* rec = reinterpret_cast<StHist1Rec*>(out);
    if (tid < 256) {
      rec->mass[tid] = sh.mass[tid];
      rec->cnt[tid] = sh.cnt[tid];
    }
    return;
  }

  // phases 2-5: end selection PH - 3 if one is pending; phases 2-4: begin selection PH - 2 and count the shard's level 2
  // within its high byte; phase 5: the rank holding the drawn element finds it
  if (S.greedy) {
    if (PH == 5 && tid == 0) *reinterpret_cast<long long*>(out) = -1;
    if (PH < 5 && tid < 256) reinterpret_cast<uint32_t*>(out)[tid] = 0;
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
    if (PH < 5 && tid < 256) {
      sh.tot1[tid] = S.tot1[tid];
      sh.totm1[tid] = S.totm1[tid];
    }
    if (S.hb != kNoSel) st_sum_level2(sh, a, PH - 1, r);
  }
  if (PH < 5 && tid < 256) sh.cnt[tid] = 0;
  if (PH == 5 && tid == 0) sh.id = -1;
  __syncthreads();
  if (w == 0) {
    u64 Sv = S.S;  // the kept weight entering selection PH - 2 (phase 2: not read)
    if (PH > 2 && S.hb != kNoSel) {  // selection 0 (top-k) counts elements, the later ones weigh them
      const SmpSel sel = smp_select_end<H>(sh.tot2, S.hb, S.T, S.acnt, S.amass, PH > 3, m, c, lane);
      Sv = smp_kept<H>(sel, m, c);
      if (PH == 5 && lane == 0) { sh.key = sel.key; sh.j = sel.j; }
    }
    if (PH < 5) {
      const SmpTarget tg = smp_target(PH - 2, S.k, a.n_total, a.top_p[r], a.seeds[r], a.offsets[r], Sv);
      if (PH == 2 && !tg.sel) Sv = smp_total_mass(sh.totm1, lane);
      uint32_t hb = kNoSel;
      u64 ac = 0, am = 0;
      if (tg.sel) hb = (uint32_t)smp_scan(sh.tot1, [&](int b) { return sh.totm1[b]; }, tg.by_mass, tg.T, lane, ac, am);
      if (lane == 0) {
        S.T = tg.T;
        S.acnt = ac;
        S.amass = am;
        S.S = Sv;
        S.hb = sh.hb = hb;
      }
    }
  }
  __syncthreads();
  if (PH < 5) {
    uint32_t* rec = reinterpret_cast<uint32_t*>(out);
    if (sh.hb != kNoSel) smp_level2(sh.cnt, row, n, sh.hb);
    __syncthreads();
    if (tid < 256) rec[tid] = sh.cnt[tid];
    return;
  }
  // the drawn key K and its rank j; each rank's count of K is its phase-4 record at K's low byte
  const uint32_t key = sh.key;
  const u64 j = sh.j;
  const int rank = S.rank;
  u64 pre = 0;
  for (int q = 0; q < rank; ++q) pre += reinterpret_cast<const uint32_t*>(st_rec(a, 4, q, r))[key & 255];
  const u64 mine = reinterpret_cast<const uint32_t*>(st_rec(a, 4, rank, r))[key & 255];
  if (pre < j && j <= pre + mine) {  // uniform over the CTA: the j-th element of K in id order is here
    smp_key_counts(row, n, key, sh.wcnt);
    __syncthreads();
    const int e = smp_pick(row, n, key, sh.wcnt, j - pre);
    if (e >= 0) sh.id = (long long)a.id_offset + e;
    __syncthreads();
  }
  if (tid == 0) *reinterpret_cast<long long*>(out) = sh.id;
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
    const dim3 g((unsigned)rows), b(kSmpThreads);
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
