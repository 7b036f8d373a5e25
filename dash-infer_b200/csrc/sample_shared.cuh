// b200spark — the integer arithmetic of b2_sample shared by its whole-row kernels (sample.cu) and the vocab-split form
// (sample_tp.cu, b2_sample_shard): the order key, the weights, the Philox draw, the 128-bit scaling and the 256-bin scan.
// Both files call these functions, so a shard of a row is weighed and ordered exactly as the whole row is.
#pragma once
#include "b2_common.cuh"

namespace b2 {

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

}  // namespace b2
