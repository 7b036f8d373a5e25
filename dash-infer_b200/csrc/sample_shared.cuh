// b200spark — the steps of b2_sample's draw, shared by its whole-row kernels (sample.cu, a CTA or a cluster meeting over
// distributed shared memory) and its vocab-split form (sample_tp.cu, b2_sample_shard, phases meeting over all-gathered
// records).  Each step reads its source as (pointer, length): the staged chunk in shared memory or the shard in global
// memory.  Both forms call the same functions between their meeting points, so a shard of a row is weighed, ordered,
// counted and selected exactly as the whole row is; only the transport of the partial sums differs.
#pragma once
#include <climits>

#include "b2_common.cuh"

namespace b2 {

constexpr int kSmpThreads = 1024;  // threads per CTA of every sampling kernel
constexpr uint32_t kLog2eF32 = 0x3FB8AA3Bu;
typedef unsigned long long u64;

// The order-preserving key of the FT bits b (-0 mapped to +0 first), and its inverse.
__device__ __forceinline__ uint32_t smp_key(uint32_t b) {
  if (b == 0x8000u) b = 0;
  return (b & 0x8000u) ? (~b & 0xffffu) : (b | 0x8000u);
}
__device__ __forceinline__ uint32_t smp_unkey(uint32_t k) { return (k & 0x8000u) ? (k & 0x7fffu) : (~k & 0xffffu); }

template <bool H>
__device__ __forceinline__ float smp_val(uint32_t b) {
  return Ft<H>::to_f(__ushort_as_bfloat16((unsigned short)b));
}

// W = 0 for -inf, else round(ex2.approx.ftz(fl32(fl32(x - m) c)) 2^40): at most 2^40, exactly 2^40 at x = m.
__device__ __forceinline__ u64 smp_weight(float x, float m, float c) {
  if (x == -INFINITY) return 0;
  const float y = __fmul_rn(__fsub_rn(x, m), c);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(y));
  return __float2ull_rn(__fmul_rn(e, 1099511627776.f));
}

// Philox4x32-10 (Salmon et al., SC'11; the Random123 constants), r0 of the result.
__device__ __forceinline__ uint32_t philox_r0(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c0;
}

// floor(a b / 2^24) and ceil(a b / 2^24) for a <= 2^24, b < 2^58, in 128-bit integer arithmetic
__device__ __forceinline__ u64 mul_shr24(u64 a, u64 b, bool up) {
  const u64 lo = a * b, hi = __umul64hi(a, b);
  return ((hi << 40) | (lo >> 24)) + (up && (lo & 0xffffffu) != 0);
}

// Warp 0: the first of the 256 bins, from bin 255 down, at which the running sum of q (the weights if by_mass, else the
// counts) reaches T (1 <= T <= the total).  Returns the bin and the counts / weights of the bins above it (all lanes).
template <class MassF>
__device__ __forceinline__ int smp_scan(const uint32_t* cnt, MassF mass, bool by_mass, u64 T, int lane, u64& acnt, u64& amass) {
  u64 lc = 0, lm = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int b = 255 - 8 * lane - i;
    lc += cnt[b];
    lm += mass(b);
  }
  u64 ic = lc, im = lm;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const u64 tc = __shfl_up_sync(0xffffffffu, ic, o), tm = __shfl_up_sync(0xffffffffu, im, o);
    if (lane >= o) { ic += tc; im += tm; }
  }
  u64 ec = ic - lc, em = im - lm;
  const uint32_t hit = __ballot_sync(0xffffffffu, (by_mass ? em : ec) < T && T <= (by_mass ? im : ic));
  const int src = hit ? __ffs(hit) - 1 : 31;
  int bin = 0;
  if (lane == src) {  // walk the lane's 8 bins (the last one if T exceeds the total, which the callers rule out)
    for (int i = 0; i < 8; ++i) {
      bin = 255 - 8 * lane - i;
      const uint32_t cb = cnt[bin];
      const u64 mb = mass(bin);
      if ((by_mass ? em + mb : ec + cb) >= T || i == 7) break;
      ec += cb;
      em += mb;
    }
  }
  acnt = __shfl_sync(0xffffffffu, ec, src);
  amass = __shfl_sync(0xffffffffu, em, src);
  return __shfl_sync(0xffffffffu, bin, src);
}

// All threads: the argmax under argmax_beats of src[0, len), ids from id0; with STAGE, src is also copied to stage.  The
// warps' winners pass through wv / wi (shared, 32 each); warp 0 returns the CTA's winner in every lane.
template <bool H, bool STAGE>
__device__ __forceinline__ void smp_argmax(const uint16_t* src, int len, int id0, uint16_t* stage, float* wv, int* wi, float& bv,
                                           int& bi) {
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  bv = -INFINITY;
  bi = INT_MAX;
  int i = tid;
  for (; i + 3 * kSmpThreads < len; i += 4 * kSmpThreads) {
    uint16_t b[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) b[u] = src[i + u * kSmpThreads];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (STAGE) stage[i + u * kSmpThreads] = b[u];
      const float x = smp_val<H>(b[u]);
      if (argmax_beats(x, id0 + i + u * kSmpThreads, bv, bi)) { bv = x; bi = id0 + i + u * kSmpThreads; }
    }
  }
  for (; i < len; i += kSmpThreads) {
    const uint16_t b = src[i];
    if (STAGE) stage[i] = b;
    const float x = smp_val<H>(b);
    if (argmax_beats(x, id0 + i, bv, bi)) { bv = x; bi = id0 + i; }
  }
  warp_argmax(bv, bi);
  if (lane == 0) { wv[w] = bv; wi[w] = bi; }
  __syncthreads();
  if (w == 0) {
    bv = wv[lane];
    bi = wi[lane];
    warp_argmax(bv, bi);
  }
}

// The row's parameters from its maximum m (the argmax's value), temperature t and top-k k_in over n elements.  A greedy row
// (m not finite, t NaN or <= 0, or c not finite) takes the argmax's id; k = n sets no limit.
struct SmpRow {
  float m, c;
  int k;
  bool greedy;
};
__device__ __forceinline__ SmpRow smp_row_setup(float m, float t, int32_t k_in, int n) {
  const float c = __fdiv_rn(__uint_as_float(kLog2eF32), t);
  const bool greedy = !(fabsf(m) <= 3.402823466e38f) || !(t > 0.f) || !(fabsf(c) <= 3.402823466e38f);
  return {m, c, (k_in <= 0 || k_in > n) ? n : k_in, greedy};
}

// All threads: level 1 of src[0, len), added to cnt1 / mass1 (shared): counts and weight sums per high byte.  The high
// byte of a bf16 logit is its sign and 7 exponent bits, so a real row falls into a handful of bins and per-lane atomics
// would serialise on them: each warp sums its lanes per distinct bin (the leader's bin, the ballot of its peers, two
// 32-bit warp reductions of the split weight) and issues one atomic pair per bin.
template <bool H>
__device__ __forceinline__ void smp_level1(uint32_t* cnt1, u64* mass1, const uint16_t* src, int len, float m, float c) {
  const int lane = threadIdx.x & 31;
  const int steps = (len + kSmpThreads - 1) / kSmpThreads;
  for (int s = 0; s < steps; ++s) {
    const int e = s * kSmpThreads + threadIdx.x;
    const bool valid = e < len;
    uint32_t hb = 0;
    u64 wt = 0;
    if (valid) {
      const uint32_t b = src[e];
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
        atomicAdd(&cnt1[h], (uint32_t)__popc(grp));
        atomicAdd(&mass1[h], ((u64)shi << 24) + slo);
      }
      todo &= ~grp;
    }
  }
}

// Warp 0: the whole weight of the row's level-1 weight sums totm1, in every lane (S_k when k sets no limit).
__device__ __forceinline__ u64 smp_total_mass(const u64* totm1, int lane) {
  u64 s = 0;
#pragma unroll
  for (int b = 0; b < 8; ++b) s += totm1[lane * 8 + b];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

// Selection q's target: the first position in the row's order at which the running sum of the counts (q = 0, top-k: the
// k-th element) or of the weights (q = 1, top-p: Pt = max(1, ceil(p24 S / 2^24)) with S = S_k; q = 2, the draw: U + 1 with
// U = floor(u24 S / 2^24), S = S_p and u24 = Philox4x32-10(counter = off, key = seed).r0 >> 8) reaches T.  sel is false
// when q sets no limit.
struct SmpTarget {
  u64 T;
  bool by_mass, sel;
};
__device__ __forceinline__ SmpTarget smp_target(int q, int k, int n, float p, u64 seed, u64 off, u64 S) {
  if (q == 0) return {(u64)k, false, k < n};
  if (q == 1) {
    const uint32_t p24 = !(p < 1.f) ? (1u << 24) : min(__float2uint_rn(__fmul_rn(p, 16777216.f)), 1u << 24);
    return {max(mul_shr24(p24, S, true), (u64)1), true, p24 < (1u << 24)};
  }
  const uint32_t u24 = philox_r0((uint32_t)off, (uint32_t)(off >> 32), 0, 0, (uint32_t)seed, (uint32_t)(seed >> 32)) >> 8;
  return {mul_shr24(u24, S, false) + 1, true, true};
}

// All threads: the level-2 counts of src[0, len) within high byte hb, added to cnt2 (shared, by low byte).
__device__ __forceinline__ void smp_level2(uint32_t* cnt2, const uint16_t* src, int len, uint32_t hb) {
  for (int i = threadIdx.x; i < len; i += kSmpThreads) {
    const uint32_t k = smp_key(src[i]);
    if ((k >> 8) == hb) atomicAdd(&cnt2[k & 255], 1u);
  }
}

// A selection's position: key K and the rank j (from 1) of its element among K's in id order; acnt / amass are the counts
// / weights of the keys above K.
struct SmpSel {
  uint32_t key;
  u64 j, acnt, amass;
};

// Warp 0: the end of a selection (target T, by_mass) that began at high byte hb with a1c / a1m above it (smp_scan over
// the row's level 1), from the row's level-2 counts tot2 within hb.  Every lane returns the position.
template <bool H>
__device__ __forceinline__ SmpSel smp_select_end(const uint32_t* tot2, uint32_t hb, u64 T, u64 a1c, u64 a1m, bool by_mass, float m,
                                                 float c, int lane) {
  auto wkey = [&](int b) { return smp_weight(smp_val<H>(smp_unkey((hb << 8) | (uint32_t)b)), m, c); };
  u64 ac, am;
  const int lo = smp_scan(tot2, [&](int b) { return (u64)tot2[b] * wkey(b); }, by_mass, T - (by_mass ? a1m : a1c), lane, ac,
                          am);
  ac += a1c;
  am += a1m;
  const u64 w = wkey(lo);
  const u64 j = !by_mass ? T - ac : w ? (T - am + w - 1) / w : 1;  // the selected key's bin holds weight: w > 0
  return {(hb << 8) | (uint32_t)lo, j, ac, am};
}

// The weight kept up to and including a selection's position: S_k after top-k, S_p after top-p.
template <bool H>
__device__ __forceinline__ u64 smp_kept(const SmpSel& s, float m, float c) {
  return s.amass + s.j * smp_weight(smp_val<H>(smp_unkey(s.key)), m, c);
}

// Warp w owns the contiguous range [w seg, (w + 1) seg) of a source of len elements, so its elements are in id order.
__device__ __forceinline__ int smp_seg(int len) { return ((len + kSmpThreads - 1) / kSmpThreads) * 32; }

// All threads: each warp's count of key in its range of src[0, len), written to wcnt[w] (shared).
__device__ __forceinline__ void smp_key_counts(const uint16_t* src, int len, uint32_t key, uint32_t* wcnt) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, seg = smp_seg(len);
  uint32_t cnt = 0;
  for (int e = w * seg + lane; e < (w + 1) * seg; e += 32)
    cnt += __popc(__ballot_sync(0xffffffffu, e < len && smp_key(src[e]) == key));
  if (lane == 0) wcnt[w] = cnt;
}

// All threads, after smp_key_counts' wcnt is visible: the index in src of the jl-th element (from 1) of key in id order,
// on the one thread that finds it; -1 on every other thread, and on all of them when jl is not in [1, sum of wcnt].
__device__ __forceinline__ int smp_pick(const uint16_t* src, int len, uint32_t key, const uint32_t* wcnt, u64 jl) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, seg = smp_seg(len);
  u64 pre = 0;  // the key's elements in the lower warps' ranges
  for (int x = 0; x < w; ++x) pre += wcnt[x];
  if (!(pre < jl && jl <= pre + wcnt[w])) return -1;
  const uint32_t want = (uint32_t)(jl - pre);
  uint32_t seen = 0;
  for (int e = w * seg + lane; e < (w + 1) * seg; e += 32) {
    const bool hit = e < len && smp_key(src[e]) == key;
    const uint32_t bal = __ballot_sync(0xffffffffu, hit);
    if (seen + __popc(bal) >= want) return hit && seen + __popc(bal & ((1u << lane) - 1)) + 1 == want ? e : -1;
    seen += __popc(bal);
  }
  return -1;
}

}  // namespace b2
