// b200spark — weight-only quantized (int4 / int8) and dense bf16 GEMM for decode batches 17..64 on the Hopper warpgroup
// tensor cores (wgmma), sm_90a.
//
// Replaces the reference's "dequantize the whole weight to a [K,N] bf16 workspace, then cuBLAS" fallback
// (csrc/core/operator/general/gemm_lowp/gemm_a16w4_gpu.cpp:193-210, gemm_a16w8_gpu.cpp:210-237): 4.5 B of HBM
// traffic per weight there, 0.5 B (int4) / 1 B (int8) here.
//
//   C^T[128 n x NM m] (fp32, registers) += W^T[128 n x 16 k] (bf16, registers) * A^T[16 k x NM m] (bf16, shared memory)
//
//   warps 0..7  : two consumer warpgroups, 64 output channels each.  Every thread dequantizes the weights of its wgmma
//                 A-operand fragment (rows g and g + 8 of its warp's 16, the k pairs 2t and 2t + 8 of every k16 step):
//                 LDS.128 of the row's image chunk -> shf/lop3 -> exact bf16 integers (16+q) in registers, which
//                 wgmma.mma_async reads directly (the dequantized weights never touch shared memory: its bandwidth could
//                 not carry 2 B/weight at HBM rate).  One commit group per 64-k tile, at most two in flight, so the
//                 dequantization of tile t+1 overlaps the MMAs of tile t; the accumulators stay in registers.
//   warp 8      : TMA producer — int4/int8/bf16 weight tiles (same init-time image as the mma.sync kernel) stream
//                 HBM -> shared memory with cp.async.bulk (16 KB stages), ahead of the previous kernel's completion (PDL)
//   warp 9      : activation tiles (64 k x NM m) by TMA tensor-map loads into the 128B-swizzled K-major layout the wgmma
//                 B descriptor reads (out-of-range rows/columns are zero-filled by the TMA unit)
//   warps 10..11: per-row sums sum_k a[m][k] needed by the zero-point term, read from the landed tiles
//   epilogue    : the consumers apply s * (acc - (16+z) * sum a) to their accumulators and park the fp32 tile in the drained
//                 activation ring; then ALL 384 threads do the split-K partial store / last-CTA reduction and the final
//                 alpha/bias/activation/residual (or SwiGLU) with 16-byte reads and 8-byte bf16x4 stores.
//   schedule    : one CTA per SM; the launch's tiles are spread evenly over them (TcSched, wq_gemm_shared.cuh): whole
//                 n-groups in rounds while there are more n-groups than CTAs (MULTI instantiation: gate+up pair, lm_head),
//                 each n-group left over cut in two k-ordered halves on two CTAs, the second starting from the first's
//                 accumulators; else equal k-slices.  A CTA walks its segments with the barriers and ring phases carried
//                 over; the next segment's first weight stages are issued before the epilogue.
//
//   variants    : GROUPED (sub-channel int4: the scale is applied to the weights at dequantization; group sizes that do not
//                 divide the 64-k tile look their params up per 8-k word), A8 (fp8 activations, e4m3 wgmma), H (fp16
//                 instead of bf16 activations / outputs), the RMSNorm hand-off (row statistics + gamma-scaled copy out, 1/rms in).
//
// Roofline: HBM-bound up to M ~ 64 (~300 FLOP/B is the H100 tensor/HBM ridge); report both.
#include <type_traits>

#include "b2_common.cuh"
#include "wq_gemm_shared.cuh"

namespace b2 {

constexpr int kTcThreads = 384;      // warps 0-7 two consumer warpgroups, 8 weights TMA, 9 activation TMA, 10-11 row sums;
                                     // every warp joins the epilogue
constexpr int kTcNM = 64;            // batch columns per MMA (wgmma N)
constexpr int kTcNSW = 6;            // weight stages (16 KB each): ~2 us of HBM latency x 25 GB/s/SM needs >= 50 KB in flight
constexpr int kTcNSX = 3;            // activation stages (32 or 16 KB each)
constexpr int kTcXTile = kTcNM * 128;  // bytes: NM rows x 64 k bf16

// ---- wgmma wrappers (PTX ISA 8.0, sm_90a): A from registers, B from a shared-memory descriptor, D in registers ----
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
__device__ __forceinline__ void wg_fence_acc(float (&d)[32]) {
#pragma unroll
  for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// K-major operand, 128-byte swizzle, 8-row groups 1024 B apart; a k16 (bf16) or k32 (e4m3) step inside the swizzle atom is
// +32 B, i.e. +2 in the start-address field
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

#define B2_WG_D16 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}"
#define B2_WG_D32                                                                                                          \
  "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}"
#define B2_WG_ACC16(d)                                                                                                       \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), \
      "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
#define B2_WG_ACC32(d)                                                                                                       \
  B2_WG_ACC16(d), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
      "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])

// D[64 x NM] += A[64 x k] (registers) * B[k x NM] (smem): KIND 0 = bf16 (k16), 1 = fp16 (k16), 2 = e4m3 (k32).  NM = 32 uses
// d[0..15] only.  The width is a template argument: with a runtime choice every MMA is a basic block of its own, and ptxas
// then fences each one with a warpgroup.arrive and waits for it alone, so no MMA overlaps the next tile's dequantization.
template <int KIND, bool N32>
__device__ __forceinline__ void wg_mma(float (&d)[32], const uint32_t (&a)[4], uint64_t desc) {
  if constexpr (N32) {
    if (KIND == 0)
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
                   "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 " B2_WG_D16 ", {%16,%17,%18,%19}, %20, p, 1, 1, 0;\n\t}"
                   : B2_WG_ACC16(d) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
    else if (KIND == 1)
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
                   "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 " B2_WG_D16 ", {%16,%17,%18,%19}, %20, p, 1, 1, 0;\n\t}"
                   : B2_WG_ACC16(d) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
    else
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
                   "wgmma.mma_async.sync.aligned.m64n32k32.f32.e4m3.e4m3 " B2_WG_D16 ", {%16,%17,%18,%19}, %20, p, 1, 1;\n\t}"
                   : B2_WG_ACC16(d) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
  } else {
    if (KIND == 0)
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                   "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " B2_WG_D32 ", {%32,%33,%34,%35}, %36, p, 1, 1, 0;\n\t}"
                   : B2_WG_ACC32(d) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
    else if (KIND == 1)
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                   "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " B2_WG_D32 ", {%32,%33,%34,%35}, %36, p, 1, 1, 0;\n\t}"
                   : B2_WG_ACC32(d) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
    else
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                   "wgmma.mma_async.sync.aligned.m64n64k32.f32.e4m3.e4m3 " B2_WG_D32 ", {%32,%33,%34,%35}, %36, p, 1, 1;\n\t}"
                   : B2_WG_ACC32(d) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
  }
}

__device__ __forceinline__ uint32_t tc_prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
  return d;
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
// 4 of the 8 int4 codes of one image word -> 4 e4m3 bytes (exact: 0..15 are e4m3 values): half 0 = codes of k (0,2,4,6),
// half 1 = codes of k (1,3,5,7) of the word's 8 consecutive k (the in-word k order of the image, wq_gemm_shared.cuh) — the
// byte order of the b2 fp8 activation layout (glue.cu quant_fp8_kernel).  Byte-permute look-ups: codes 0..7 from one 8-byte
// table, 8..15 are 0x50 | (q & 7) from a second one, the choice by a sign-replicating permute of bit 3 of every nibble.
// qsh = 16 * half, msel = half ? 0xFBEA : 0xD9C8.
__device__ __forceinline__ uint32_t nib4_to_e4m3(uint32_t w_rot3, uint32_t qsh, uint32_t msel) {
  const uint32_t word = __funnelshift_r(w_rot3, w_rot3, 3);  // the image stores words rotated left by 3 (bf16 path)
  const uint32_t sel = (word & 0x77777777u) >> qsh;
  const uint32_t T0 = 0x44403800u, T1 = 0x4E4C4A48u, H0 = 0x53525150u, H1 = 0x57565554u;
  const uint32_t lo = tc_prmt(T0, T1, sel), hi = tc_prmt(H0, H1, sel);
  const uint32_t m = tc_prmt(word << 4, word, msel);  // 0xFF where the nibble is >= 8
  uint32_t r;
  asm("lop3.b32 %0, %1, %2, %3, 0xD8;" : "=r"(r) : "r"(lo), "r"(hi), "r"(m));  // m ? hi : lo
  return r;
}

// MULTI: more n-groups than CTAs, a CTA walks whole n-groups and at most one head and one tail; else one k-slice
// A8: fp8-e4m3 activations (b2_gemm_wq_run_fp8, int4 weights only): the int4 codes become exact e4m3 bytes, the MMAs are
// e4m3 x e4m3 with K = 32 (half the MMAs of the bf16 path), an activation tile is 128 k wide.
// GROUPED: sub-channel weights (GPTQ g128 ...): the (scale, zero) of a channel changes every group_tiles k-tiles, so the affine
// dequantisation cannot wait for the accumulator.  The consumers apply it to the weights instead — exact integer (q - 8)
// in bf16, then ONE fused multiply-add per two weights: w = (q - 8) * s + (8 - z) * s, rounded to bf16 once — which is what
// the reference's kernels (dequant in FT, gemm_lowp_utils.cuh:28-47) and its CPU path (weights stored in the model dtype)
// feed their GEMMs with; the accumulator then needs no zero-point term and no row sums.
// H: fp16 activations / outputs (the exact-integer constants are 128 + q instead of 16 + q).
template <int WBITS, bool MULTI, bool A8 = false, bool GROUPED = false, bool H = false>
__global__ void __launch_bounds__(kTcThreads, 1) wq_gemm_tc_kernel(const TcParams p, const __grid_constant__ CUtensorMap amap) {
  using I = Image<WBITS>;
  constexpr int TILE_BYTES = I::kTileBytes;
  constexpr int NSW = WBITS == 16 ? 4 : kTcNSW;               // weight stages (bf16: 32 KB each)
  // k-tiles per pipeline stage (k256 for W4, k128 for W8): one stage = 16 KB of weights per barrier round trip
  constexpr int TPS = WBITS == 4 ? 4 : 2;
  constexpr int KIND = A8 ? 2 : (H ? 1 : 0);
  static_assert(!A8 || WBITS == 4, "fp8 activations: int4 weights only");
  static_assert(!H || !A8, "fp8 activations come with bf16 outputs");
  using F = Ft<H>;
  static_assert(!GROUPED || (!A8 && WBITS != 16), "sub-channel weights: bf16 activations, int4 / int8");
  const int XTILE_LD = p.nm * 128;             // bytes the TMA writes per activation tile (the tile slot stays 64 rows)
  constexpr int XTPS = A8 ? TPS / 2 : TPS;     // activation tiles per stage (fp8: 128 k per 128-byte row)
  constexpr int WSTAGE = TPS * TILE_BYTES;     // 16 KB
  constexpr int XSTAGE = XTPS * kTcXTile;      // 32 KB / 16 KB
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* xring = smem;                                   // NSX x XSTAGE, 1024B aligned (SWIZZLE_128B atoms)
  uint8_t* wring = xring + kTcNSX * XSTAGE;                // NSW x WSTAGE
  float* suma = reinterpret_cast<float*>(wring + NSW * WSTAGE);  // [NM]
  uint64_t* bars = reinterpret_cast<uint64_t*>(suma + kTcNM);
  uint64_t* wfull = bars;                 // [NSW] weights landed (TMA tx)
  uint64_t* wfree = wfull + kTcNSW;       // [NSW] consumer warps done reading the smem stage (8 arrivals)
  uint64_t* afull = wfree + kTcNSW;       // [NSX] activation tiles landed (TMA tx)
  uint64_t* xsum = afull + kTcNSX;        // [NSX] row sums done with the stage (2 arrivals)
  uint64_t* xfree = xsum + kTcNSX;        // [NSX] the MMAs reading the stage completed (8 consumer-warp arrivals)
  float* ascale = reinterpret_cast<float*>(bars) + 64;  // [NM] per-token activation scales (A8) or 1/rms, 256 B into the barrier block
  __shared__ int s_is_last;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const TcSched sch(p.NG, p.KT, (int)gridDim.x, p.rounds, p.S, p.h, (int)blockIdx.x);
  const int nseg = MULTI ? sch.count() : 1;  // MULTI: whole n-groups, a head first / a tail last; else one k-slice
  auto segment = [&](int i) { return sch.seg(i); };
  __shared__ unsigned s_carry;

  if (tid == 0) {
    for (int i = 0; i < NSW; ++i) { mbar_init(&wfull[i], 1); mbar_init(&wfree[i], 8); }
    for (int i = 0; i < kTcNSX; ++i) { mbar_init(&afull[i], 1); mbar_init(&xsum[i], 2); mbar_init(&xfree[i], 8); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  // The CTA walks its segments (TcSched).  Barriers and the ring phases carry over; g = gbase + st is the stage index since
  // kernel start.  Stage g uses weight slot g % NSW and X slot g % NSX.
  int w_pre = 0;  // weight stages of the current segment already issued during the previous one's tail (producer thread only)
  // The MMA width (N32: m64n32 for batches <= 32) is fixed once per launch: the whole segment loop is compiled once per width.
  // A width chosen inside it would leave two main loops in one segment loop, and ptxas then serializes the MMAs of the
  // persistent instantiations for lack of registers.
  auto body = [&](auto n32) {
  constexpr bool N32 = decltype(n32)::value;
  int gbase = 0;  // stages of the earlier segments
  for (int si = 0; si < nseg; ++si) {
  const TcSeg sg = segment(si);
  const int ng = sg.ng, kt1 = sg.kt1;
  // a tail starts from its head's parked accumulators if they are there (the head's arrival makes the count 1), else it runs
  // the whole n-group.  Counters and workspace belong to the previous kernels until pdl_wait.
  bool carry_in = false;
  if (MULTI && sg.carry == 2) {
    pdl_wait();
    if (tid == 0) {
      s_carry = atomicAdd(&p.counters[ng], 1u);
      if (s_carry == 1u) p.counters[ng] = 0;  // both have arrived: re-arm for the next launch / graph replay
      __threadfence();
    }
    __syncthreads();
    carry_in = s_carry == 1u;
  }
  const int kt0 = sg.carry == 2 && !carry_in ? 0 : sg.kt0;
  const float* carry_src = p.ws + (size_t)(ng - sch.nfull) * kTcCarryFloats;
  const int nt = kt1 - kt0;
  const int nst = (nt + TPS - 1) / TPS;  // pipeline stages of this segment
  if (warp == 8) {
    // ===================== weight producer (does not wait for the previous kernel) =====================
    if (lane == 0) {
      auto issue = [&](int g, const uint8_t* src, uint32_t bytes) {
        const int slot = g % NSW;
        if (g >= NSW) mbar_wait_backoff(&wfree[slot], ((g / NSW) & 1) ^ 1);
        mbar_arrive_expect_tx(&wfull[slot], bytes);
        bulk_g2s(wring + slot * WSTAGE, src, bytes, &wfull[slot]);
      };
      const uint8_t* wsrc = p.packed + ((size_t)ng * p.KT + kt0) * TILE_BYTES;
      for (int st = w_pre; st < nst; ++st) issue(gbase + st, wsrc + (size_t)st * WSTAGE, min(TPS, nt - st * TPS) * TILE_BYTES);
      // head of the next segment: its first stages stream in while this one drains and runs its epilogue
      w_pre = 0;
      if (si + 1 < nseg && segment(si + 1).carry != 2) {  // a tail's first k-tile is only known when it starts
        const TcSeg s2 = segment(si + 1);
        const int nt2 = s2.kt1 - s2.kt0, nst2 = (nt2 + TPS - 1) / TPS;
        const uint8_t* wsrc2 = p.packed + ((size_t)s2.ng * p.KT + s2.kt0) * TILE_BYTES;
        w_pre = min(NSW, nst2);
        for (int st = 0; st < w_pre; ++st)
          issue(gbase + nst + st, wsrc2 + (size_t)st * WSTAGE, min(TPS, nt2 - st * TPS) * TILE_BYTES);
      }
    }
  } else if (warp == 9) {
    // ===================== activation producer: TMA tensor-map loads (zero fill outside [M, K]) =====================
    if (lane == 0) {
      pdl_wait();  // A is the previous kernel's output
      for (int st = 0; st < nst; ++st) {
        const int g = gbase + st;
        const int slot = g % kTcNSX;
        if (g >= kTcNSX) {
          const uint32_t par = ((g / kTcNSX) & 1) ^ 1;
          mbar_wait_backoff(&xfree[slot], par);
          mbar_wait_backoff(&xsum[slot], par);
        }
        const int wtiles = min(TPS, nt - st * TPS);
        const int tiles = A8 ? (wtiles + 1) / 2 : wtiles;     // activation tiles (fp8: one per two 64-k weight tiles)
        mbar_arrive_expect_tx(&afull[slot], tiles * XTILE_LD);
        for (int ti = 0; ti < tiles; ++ti)
          asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                       ::"r"(smem_u32(xring + slot * XSTAGE + ti * kTcXTile)), "l"(reinterpret_cast<uint64_t>(&amap)),
                         "r"((kt0 + st * TPS + (A8 ? 2 * ti : ti)) * kBK), "r"(0), "r"(smem_u32(&afull[slot]))
                       : "memory");
      }
    }
  } else if (warp >= 10) {
    // ===================== row sums of the landed activation tiles (row = xt) =====================
    const int xt = tid - 320;  // 0..63
    float r0 = 0.f, r1 = 0.f, r2 = 0.f, r3 = 0.f;
    if (carry_in) {
      const float4 r = __ldcg(reinterpret_cast<const float4*>(carry_src + 256 * 32) + xt);
      r0 = r.x; r1 = r.y; r2 = r.z; r3 = r.w;
    }
    if (A8) {  // the quantizer already summed every 64-k tile of every row: add this unit's tiles; stage the token scales
      pdl_wait();
      if (xt < p.M) {
        const float* ts = p.tile_sums + (size_t)xt * p.KT;
        for (int kt = kt0; kt < kt1; ++kt) r0 += ts[kt];
        ascale[xt] = p.a_scale[xt];
      } else {
        ascale[xt] = 0.f;
      }
    }
    if (!A8 && p.norm_sumsq) {  // the producer's per-tile row statistics -> 1/rms per row, applied at the accumulator read-out
      pdl_wait();
      float ss = 0.f;
      if (xt < p.M)
        for (int i = 0; i < p.norm_parts; ++i) ss += __ldcg(p.norm_sumsq + (size_t)i * p.norm_ld + xt);
      ascale[xt] = rsqrtf(ss * p.norm_inv_hidden + p.norm_eps);
    }
    for (int st = 0; st < nst; ++st) {
      const int g = gbase + st;
      const int slot = g % kTcNSX;
      mbar_wait(&afull[slot], (g / kTcNSX) & 1);  // activation tiles landed
      const int tiles = (WBITS == 16 || A8 || GROUPED || xt >= p.nm) ? 0 : min(TPS, nt - st * TPS);  // (no zero-point term)
      for (int ti = 0; ti < tiles; ++ti) {
        const uint32_t rbase = smem_u32(xring + slot * XSTAGE + ti * kTcXTile) + xt * 128;
#pragma unroll
        for (int c = 0; c < 8; c += 2) {
          const uint4 v = lds128(rbase + ((c ^ (xt & 7)) << 4));
          const uint4 w = lds128(rbase + (((c + 1) ^ (xt & 7)) << 4));
          r0 += (F::lo(v.x) + F::hi(v.x)) + (F::lo(v.y) + F::hi(v.y));
          r1 += (F::lo(v.z) + F::hi(v.z)) + (F::lo(v.w) + F::hi(v.w));
          r2 += (F::lo(w.x) + F::hi(w.x)) + (F::lo(w.y) + F::hi(w.y));
          r3 += (F::lo(w.z) + F::hi(w.z)) + (F::lo(w.w) + F::hi(w.w));
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&xsum[slot]);
    }
    suma[xt] = (r0 + r1) + (r2 + r3);
    asm volatile("bar.sync 3, 320;" ::: "memory");  // hand the sums to the consumers
    if (MULTI && sg.carry == 1)  // a head parks its running sums behind the accumulators (the ring is drained now)
      reinterpret_cast<float4*>(xring)[256 * 32 / 4 + xt] = make_float4(r0, r1, r2, r3);
  } else {
    // ===================== consumers: dequantize into wgmma A fragments, MMA, accumulators -> smem tile =====================
    const int wg = warp >> 2, g8 = lane >> 2, t4 = lane & 3;
    const int rr0 = wg * 64 + (warp & 3) * 16 + g8, rr1 = rr0 + 8;  // the two output channels (tile rows) of this thread
    // per-channel (scale, zero + bias constant): immutable, read before the waits
    const float2 sz0 = (WBITS == 16 || GROUPED) ? make_float2(1.f, 0.f) : p.sz[ng * kBN + rr0];
    const float2 sz1 = (WBITS == 16 || GROUPED) ? make_float2(1.f, 0.f) : p.sz[ng * kBN + rr1];
    const uint32_t wring_u = smem_u32(wring), xring_u = smem_u32(xring);
    uint32_t off0[I::kChunks], off1[I::kChunks];
#pragma unroll
    for (int c = 0; c < I::kChunks; ++c) {
      off0[c] = I::chunk_offset(rr0, c);
      off1[c] = I::chunk_offset(rr1, c);
    }
    // W4: the nibble of k pair 2t of a word; W8 / A8: which word of a 16-byte chunk, which half of it
    const uint32_t sh4 = 4 * t4, sh8 = 8 * (t4 & 1), qsh = 16 * (t4 & 1), msel = (t4 & 1) ? 0xFBEAu : 0xD9C8u;
    const int wa = t4 >> 1;
    auto word = [](const uint4& v, int j) { return j == 0 ? v.x : (j == 1 ? v.y : (j == 2 ? v.z : v.w)); };

    // fp8 MMAs accumulate with less than fp32 precision on Hopper: A8 runs them into dt and adds dt to the fp32 accumulator
    // d every 128 k (two weight tiles)
    float d[32], dt[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) d[i] = dt[i] = 0.f;
    if (carry_in) {
#pragma unroll
      for (int i = 0; i < 32; i += 4) {
        const float4 v = __ldcg(reinterpret_cast<const float4*>(carry_src + tid * 32 + i));
        d[i] = v.x; d[i + 1] = v.y; d[i + 2] = v.z; d[i + 3] = v.w;
      }
    }
    int prev_xs = -1;
    for (int st = 0; st < nst; ++st) {
      const int g = gbase + st;
      const int slot = g % NSW, xs = g % kTcNSX;
      // sub-channel weights: this stage's per-(group, channel) params are requested before the wait on the weights
      uint32_t gs2[TPS][2], gc2[TPS][2];
      if (GROUPED && p.group_k == 0) {
#pragma unroll
        for (int ti = 0; ti < TPS; ++ti) {
          const int kt = min(kt0 + st * TPS + ti, kt1 - 1);
          const float2 z0 = __ldg(p.sz + (size_t)(kt / p.group_tiles) * p.Np + ng * kBN + rr0);  // (scale, zero + 16)
          const float2 z1 = __ldg(p.sz + (size_t)(kt / p.group_tiles) * p.Np + ng * kBN + rr1);
          const float c0 = (F::kBias + 8.f - z0.y) * z0.x, c1 = (F::kBias + 8.f - z1.y) * z1.x;  // (8 - zero) * scale
          gs2[ti][0] = F::pack(z0.x, z0.x); gs2[ti][1] = F::pack(z1.x, z1.x);
          gc2[ti][0] = F::pack(c0, c0); gc2[ti][1] = F::pack(c1, c1);
        }
      }
      mbar_wait(&wfull[slot], (g / NSW) & 1);
      mbar_wait(&afull[xs], (g / kTcNSX) & 1);
      const int tiles = min(TPS, nt - st * TPS);
#pragma unroll
      for (int ti = 0; ti < TPS; ++ti) {
        if (ti < tiles) {
          const uint32_t wt = wring_u + slot * WSTAGE + ti * TILE_BYTES;
          if (A8) {  // activation tile ti / 2 holds 128 k; this weight tile is its half ti & 1 = two K=32 steps
            const uint64_t bd = wg_desc(xring_u + xs * XSTAGE + (ti >> 1) * kTcXTile) + (uint64_t)(4 * (ti & 1));
            uint32_t a[2][4];
#pragma unroll
            for (int c = 0; c < 2; ++c) {  // chunk c = 32 k = one K=32 step
              const uint4 v0 = lds128(wt + off0[c]), v1 = lds128(wt + off1[c]);
              a[c][0] = nib4_to_e4m3(word(v0, wa), qsh, msel);
              a[c][1] = nib4_to_e4m3(word(v1, wa), qsh, msel);
              a[c][2] = nib4_to_e4m3(word(v0, 2 + wa), qsh, msel);
              a[c][3] = nib4_to_e4m3(word(v1, 2 + wa), qsh, msel);
            }
            wg_fence();
#pragma unroll
            for (int c = 0; c < 2; ++c) wg_mma<KIND, N32>(dt, a[c], bd + (uint64_t)(2 * c));
          } else {
            const uint64_t bd = wg_desc(xring_u + xs * XSTAGE + ti * kTcXTile);
            if (WBITS == 4) {
              uint32_t a[4][4];
#pragma unroll
              for (int c = 0; c < 2; ++c) {
                const uint4 v0 = lds128(wt + off0[c]), v1 = lds128(wt + off1[c]);
#pragma unroll
                for (int h = 0; h < 2; ++h) {  // k16 step kk = 2c + h: words 2h (k pair 2t), 2h + 1 (k pair 2t + 8)
                  uint32_t* f = a[2 * c + h];
                  f[0] = lop3_and_or(__funnelshift_r(word(v0, 2 * h), word(v0, 2 * h), sh4), kMask4, F::kMagic);
                  f[1] = lop3_and_or(__funnelshift_r(word(v1, 2 * h), word(v1, 2 * h), sh4), kMask4, F::kMagic);
                  f[2] = lop3_and_or(__funnelshift_r(word(v0, 2 * h + 1), word(v0, 2 * h + 1), sh4), kMask4, F::kMagic);
                  f[3] = lop3_and_or(__funnelshift_r(word(v1, 2 * h + 1), word(v1, 2 * h + 1), sh4), kMask4, F::kMagic);
                  if (GROUPED) {  // (16 + q) - 24 = q - 8 exactly, then one fused multiply-add: (q - 8) s + (8 - z) s
                    uint32_t sw[4], cw[4];  // per fragment register: rows r0, r1, r0, r1
                    if (p.group_k > 0) {  // word j of chunk c holds k = 64 kt + 32 c + 8 j + (0..7): one group per word
#pragma unroll
                      for (int e = 0; e < 4; ++e) {
                        const int k0 = (kt0 + st * TPS + ti) * kBK + 32 * c + 8 * (2 * h + (e >> 1));
                        const float2 z = __ldg(p.sz + (size_t)min(k0 / p.group_k, p.ngroups - 1) * p.Np + ng * kBN + ((e & 1) ? rr1 : rr0));
                        sw[e] = F::pack(z.x, z.x);
                        const float cc = (F::kBias + 8.f - z.y) * z.x;
                        cw[e] = F::pack(cc, cc);
                      }
                    } else {
#pragma unroll
                      for (int e = 0; e < 4; ++e) { sw[e] = gs2[ti][e & 1]; cw[e] = gc2[ti][e & 1]; }
                    }
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                      uint32_t t2;
                      if (H) {  // (128 + q) - 136
                        asm("add.rn.f16x2 %0, %1, %2;" : "=r"(t2) : "r"(f[e]), "r"(0xD840D840u));
                        asm("fma.rn.f16x2 %0, %1, %2, %3;" : "=r"(f[e]) : "r"(t2), "r"(sw[e]), "r"(cw[e]));
                      } else {
                        asm("add.rn.bf16x2 %0, %1, %2;" : "=r"(t2) : "r"(f[e]), "r"(0xC1C0C1C0u));
                        asm("fma.rn.bf16x2 %0, %1, %2, %3;" : "=r"(f[e]) : "r"(t2), "r"(sw[e]), "r"(cw[e]));
                      }
                    }
                  }
                }
              }
              wg_fence();
#pragma unroll
              for (int kk = 0; kk < 4; ++kk) wg_mma<KIND, N32>(d, a[kk], bd + (uint64_t)(2 * kk));
            } else if (WBITS == 16) {  // bf16 weights: k16 step kk = chunks 2kk (k pair 2t), 2kk + 1 (k pair 2t + 8)
              uint32_t a[4][4];
#pragma unroll
              for (int kk = 0; kk < 4; ++kk) {
                a[kk][0] = lds32(wt + off0[2 * kk] + 4 * t4);
                a[kk][1] = lds32(wt + off1[2 * kk] + 4 * t4);
                a[kk][2] = lds32(wt + off0[2 * kk + 1] + 4 * t4);
                a[kk][3] = lds32(wt + off1[2 * kk + 1] + 4 * t4);
              }
              wg_fence();
#pragma unroll
              for (int kk = 0; kk < 4; ++kk) wg_mma<KIND, N32>(d, a[kk], bd + (uint64_t)(2 * kk));
            } else {  // W8: chunk c = k16 step c; the low and high nibble planes are two MMAs (16 + lo, 16 (16 + hi))
              uint32_t lo[4][4], hi[4][4];
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                const uint4 v0 = lds128(wt + off0[c]), v1 = lds128(wt + off1[c]);
                const uint32_t w[4] = {word(v0, wa), word(v1, wa), word(v0, 2 + wa), word(v1, 2 + wa)};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  lo[c][e] = lop3_and_or(__funnelshift_r(w[e], w[e], sh8), kMask4, F::kMagic);
                  hi[c][e] = lop3_and_or(__funnelshift_r(w[e], w[e], sh8 + 4), kMask4, F::kMagicHi);
                }
              }
              wg_fence();
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                wg_mma<KIND, N32>(d, lo[c], bd + (uint64_t)(2 * c));
                wg_mma<KIND, N32>(d, hi[c], bd + (uint64_t)(2 * c));
              }
            }
          }
          wg_commit();
          wg_wait<1>();  // the previous tile's MMAs completed (their fragment registers and, at a stage start, X slot are free)
          if (ti == 0 && prev_xs >= 0) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&xfree[prev_xs]);
            prev_xs = -1;
          }
          if (A8 && ((ti & 1) || ti + 1 == tiles)) {
            wg_wait<0>();
            wg_fence_acc(dt);
#pragma unroll
            for (int i = 0; i < 32; ++i) { d[i] += dt[i]; dt[i] = 0.f; }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&wfree[slot]);  // the weights are in registers: the smem stage is free
      prev_xs = xs;
    }
    wg_wait<0>();
    wg_fence_acc(d);
    __syncwarp();
    if (prev_xs >= 0 && lane == 0) mbar_arrive(&xfree[prev_xs]);

    // ---------------- accumulators -> fp32 tile in shared memory: [m][128 n] over the drained activation ring ----------------
    asm volatile("bar.sync 3, 320;" ::: "memory");  // row sums ready; every MMA of both warpgroups has completed
    float* fs = reinterpret_cast<float*>(xring);
    if (MULTI && sg.carry == 1) {  // a head parks its raw accumulators
#pragma unroll
      for (int i = 0; i < 32; i += 4)
        reinterpret_cast<float4*>(fs + tid * 32)[i / 4] = make_float4(d[i], d[i + 1], d[i + 2], d[i + 3]);
    } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) {  // n8 block j of the accumulator: batch rows m = 8j + 2t (+1), channels rr0 / rr1
      const int m = 8 * j + 2 * t4;
      float s0 = 1.f, s1 = 1.f;
      if (A8 || p.norm_sumsq) { s0 = ascale[m]; s1 = ascale[m + 1]; }
      const float zz0 = A8 ? sz0.y - 16.f : sz0.y, zz1 = A8 ? sz1.y - 16.f : sz1.y;
      const float sa0 = suma[m], sa1 = suma[m + 1];
      fs[m * kBN + rr0] = sz0.x * s0 * (d[4 * j + 0] - zz0 * sa0);
      fs[(m + 1) * kBN + rr0] = sz0.x * s1 * (d[4 * j + 1] - zz0 * sa1);
      fs[m * kBN + rr1] = sz1.x * s0 * (d[4 * j + 2] - zz1 * sa0);
      fs[(m + 1) * kBN + rr1] = sz1.x * s1 * (d[4 * j + 3] - zz1 * sa1);
    }
    }
  }

  // ======================= epilogue: all threads =======================
  pdl_wait();  // workspace / counters / C belong to the previous kernels until here
  __syncthreads();  // tile parked
  {
    constexpr int T = kTcThreads;
    const float4* fs4 = reinterpret_cast<const float4*>(xring);
    float4* fs4w = reinterpret_cast<float4*>(xring);
    const int units = p.M * (kBN / 4);  // float4 units, index = m * 32 + nq
    constexpr int MPK4 = kTcNM * kBN / 4;
    bool finalize = true;
    if (MULTI && sg.carry == 1) {  // a head: accumulators and row sums to the workspace, then count its arrival
      float4* dst = reinterpret_cast<float4*>(p.ws + (size_t)(ng - sch.nfull) * kTcCarryFloats);
      for (int i = tid; i < kTcCarryFloats / 4; i += T) dst[i] = fs4[i];
      __threadfence();
      __syncthreads();
      if (tid == 0 && atomicAdd(&p.counters[ng], 1u) == 1u) p.counters[ng] = 0;  // the tail ran whole already: re-arm
      finalize = false;
    } else if (sg.parts > 1) {  // k-slice sg.part of sg.parts: partial tile to slot ng * S + part
      const size_t slots = (size_t)ng * p.S;
      float4* wsu = reinterpret_cast<float4*>(p.ws) + (slots + sg.part) * MPK4;
      for (int i = tid; i < units; i += T) wsu[i] = fs4[i];
      __threadfence();
      __syncthreads();
      if (tid == 0) {
        const unsigned prev = atomicAdd(&p.counters[ng], 1u);
        s_is_last = (prev == (unsigned)(sg.parts - 1));
      }
      __syncthreads();
      finalize = s_is_last != 0;
      if (finalize) {
        __threadfence();
        // fixed-order sum over the partials in k order (deterministic, whichever CTA arrives last); 2 units x 8 partials =
        // 16 independent 16-byte loads in flight per thread, so the reduction is a few L2 round trips
        const float4* wsg = reinterpret_cast<const float4*>(p.ws) + slots * MPK4;
        for (int i0 = tid; i0 < units; i0 += 2 * T) {
          float4 a[2];
          a[0] = a[1] = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int s0 = 0; s0 < sg.parts; s0 += 8) {
            float4 b[2][8];
#pragma unroll
            for (int g = 0; g < 2; ++g)
#pragma unroll
              for (int u = 0; u < 8; ++u) {
                const int i = i0 + g * T;
                b[g][u] = (s0 + u < sg.parts && i < units) ? __ldcg(wsg + (size_t)(s0 + u) * MPK4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
              }
#pragma unroll
            for (int g = 0; g < 2; ++g)
#pragma unroll
              for (int u = 0; u < 8; ++u) { a[g].x += b[g][u].x; a[g].y += b[g][u].y; a[g].z += b[g][u].z; a[g].w += b[g][u].w; }
          }
#pragma unroll
          for (int g = 0; g < 2; ++g) {
            const int i = i0 + g * T;
            if (i < units) fs4w[i] = a[g];
          }
        }
        if (tid == 0) p.counters[ng] = 0;  // re-arm for the next launch / graph replay
        __syncthreads();
      }
    }
    if (finalize) {
      const bool vec_ok = (p.ldc & 3) == 0 && (reinterpret_cast<uintptr_t>(p.C) & 7) == 0;
      if (p.act == B2_ACT_SWIGLU) {
        // tile = [64 gate | 64 up] channels: out[m, 64*ng + c] = silu(gate) * up; unit = 4 outputs
        const int su = p.M * 16;
#pragma unroll 1
        for (int i = tid; i < su; i += T) {
          const int m = i >> 4, nq = i & 15;
          const int nn = ng * 64 + nq * 4;
          if (nn >= p.N) continue;
          const float4 gv = fs4[m * 32 + nq], uv = fs4[m * 32 + 16 + nq];
          float v[4];
          v[0] = apply_act<B2_ACT_SILU>(gv.x * p.alpha) * (uv.x * p.alpha);
          v[1] = apply_act<B2_ACT_SILU>(gv.y * p.alpha) * (uv.y * p.alpha);
          v[2] = apply_act<B2_ACT_SILU>(gv.z * p.alpha) * (uv.z * p.alpha);
          v[3] = apply_act<B2_ACT_SILU>(gv.w * p.alpha) * (uv.w * p.alpha);
          __nv_bfloat16* cp = p.C + (int64_t)m * p.ldc + nn;
          if (vec_ok && nn + 3 < p.N) {
            *reinterpret_cast<uint2*>(cp) = make_uint2(F::pack(v[0], v[1]), F::pack(v[2], v[3]));
          } else {
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if (nn + e < p.N) cp[e] = F::from_f(v[e]);
          }
        }
      } else if (p.act == B2_ACT_NONE && vec_ok && (p.N & 3) == 0 &&
                 (!p.residual || (reinterpret_cast<uintptr_t>(p.residual) & 7) == 0) &&
                 (!p.bias || (reinterpret_cast<uintptr_t>(p.bias) & 7) == 0)) {
        // the decode-path case: no activation; all residual loads of a thread are issued before the first use
        constexpr int UPT = (kTcNM * (kBN / 4) + T - 1) / T;  // units per thread (6)
        uint2 res[UPT];
#pragma unroll
        for (int j = 0; j < UPT; ++j) {
          const int i = tid + j * T;
          const int m = i >> 5, nn = ng * kBN + (i & 31) * 4;
          res[j] = make_uint2(0u, 0u);
          if (p.residual && i < units && nn < p.N) res[j] = __ldg(reinterpret_cast<const uint2*>(p.residual + (int64_t)m * p.ldc + nn));
        }
#pragma unroll
        for (int j = 0; j < UPT; ++j) {
          const int i = tid + j * T;
          const int m = i >> 5, nn = ng * kBN + (i & 31) * 4;
          float ssq = 0.f;
          if (i < units && nn < p.N) {
            const float4 a = fs4[i];
            float v0 = a.x * p.alpha, v1 = a.y * p.alpha, v2 = a.z * p.alpha, v3 = a.w * p.alpha;
            if (p.bias) {
              const uint2 bv = __ldg(reinterpret_cast<const uint2*>(p.bias + nn));
              v0 += F::lo(bv.x); v1 += F::hi(bv.x); v2 += F::lo(bv.y); v3 += F::hi(bv.y);
            }
            v0 += F::lo(res[j].x); v1 += F::hi(res[j].x); v2 += F::lo(res[j].y); v3 += F::hi(res[j].y);
            const uint2 st2 = make_uint2(F::pack(v0, v1), F::pack(v2, v3));
            *reinterpret_cast<uint2*>(p.C + (int64_t)m * p.ldc + nn) = st2;
            if (p.xg_out) {  // the next RMSNorm's scaled input and row statistics, from the values as stored (bf16)
              const float r0 = F::lo(st2.x), r1 = F::hi(st2.x), r2 = F::lo(st2.y), r3 = F::hi(st2.y);
              const uint2 gv = __ldg(reinterpret_cast<const uint2*>(p.gamma_out + nn));
              *reinterpret_cast<uint2*>(p.xg_out + (int64_t)m * p.ldxg + nn) =
                  make_uint2(F::pack(r0 * F::lo(gv.x), r1 * F::hi(gv.x)), F::pack(r2 * F::lo(gv.y), r3 * F::hi(gv.y)));
              ssq = (r0 * r0 + r1 * r1) + (r2 * r2 + r3 * r3);
            }
          }
          if (p.xg_out) {  // a warp holds the 32 four-column units of one row (384 = 12 x 32): fixed-order lane reduction
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) ssq += __shfl_xor_sync(0xffffffffu, ssq, o);
            if (lane == 0 && i < units) p.sumsq_out[(size_t)ng * p.norm_ld + m] = ssq;
          }
        }
      } else {
        // generic: any activation / alignment (rolled on purpose: the inlined activation switch is large)
        const float* fs = reinterpret_cast<const float*>(xring);
#pragma unroll 1
        for (int i = tid; i < p.M * (kBN / 2); i += T) {
          const int m = i >> 6, np = i & 63;
          const int nn = ng * kBN + np * 2;
          if (nn >= p.N) continue;
          float v0 = fs[m * kBN + np * 2] * p.alpha, v1 = fs[m * kBN + np * 2 + 1] * p.alpha;
          const bool has1 = (nn + 1) < p.N;
          if (p.bias) {
            v0 += F::to_f(p.bias[nn]);
            if (has1) v1 += F::to_f(p.bias[nn + 1]);
          }
          v0 = apply_act_rt(v0, p.act);
          v1 = apply_act_rt(v1, p.act);
          __nv_bfloat16* cp = p.C + (int64_t)m * p.ldc + nn;
          if (p.residual) {
            const __nv_bfloat16* rp = p.residual + (int64_t)m * p.ldc + nn;
            v0 += F::to_f(rp[0]);
            if (has1) v1 += F::to_f(rp[1]);
          }
          if (has1 && ((reinterpret_cast<uintptr_t>(cp) & 3) == 0)) {
            *reinterpret_cast<uint32_t*>(cp) = F::pack(v0, v1);
          } else {
            cp[0] = F::from_f(v0);
            if (has1) cp[1] = F::from_f(v1);
          }
        }
      }
    }
  }

  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy tile writes before the next segment's TMA writes
  __syncthreads();  // the tile in the X ring is free again
  gbase += nst;
  }  // segment loop
  };
  if (p.nm == 32)
    body(std::true_type{});
  else
    body(std::false_type{});
}

template <int WBITS>
static int tc_smem_bytes() {
  const int tps = WBITS == 4 ? 4 : 2;
  const int wstage = tps * Image<WBITS>::kTileBytes;
  const int nsw = WBITS == 16 ? 4 : kTcNSW;
  return 1024 + kTcNSX * tps * kTcXTile + nsw * wstage + kTcNM * 4 + 96 * 8 + 64;  // barrier block: 21 barriers, 64 scales
}

EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

cudaError_t tc_launch(int wbits, bool fp16, TcParams p, cudaStream_t stream) {
  EncodeTiledFn enc = encode_tiled();
  if (!enc) return cudaErrorNotSupported;
  // activations A[M, K] bf16, row stride lda: box = 64 k x 64 rows, 128B swizzle, zero fill outside [M, K]
  alignas(64) CUtensorMap amap;
  const bool a8 = p.a_scale != nullptr;  // fp8 activations: bytes, 128 k per 128-byte swizzle row
  const cuuint64_t gdim[2] = {(cuuint64_t)p.K, (cuuint64_t)p.M};
  const cuuint64_t gstride[1] = {(cuuint64_t)p.lda * (a8 ? 1 : 2)};
  // batches <= 32 run the MMAs with N = 32 and load 32-row activation tiles (B2_GEMM_TC_N32=0: always 64)
  static const int n32 = env_int("B2_GEMM_TC_N32", 1);
  p.nm = (n32 && p.M <= 32) ? 32 : kTcNM;
  const cuuint32_t box[2] = {(cuuint32_t)(a8 ? 2 * kBK : kBK), (cuuint32_t)p.nm};
  const cuuint32_t estr[2] = {1, 1};
  if (enc(&amap, a8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<__nv_bfloat16*>(p.A), gdim, gstride, box, estr,
          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return cudaErrorInvalidValue;

  const int grid = p.grid;
  const bool grouped = p.group_tiles > 0 || p.group_k > 0;
  // instantiations: fp8 activations with int4 weights and bf16 outputs; sub-channel weights with int4 only
  if ((a8 && (wbits != 4 || fp16)) || (grouped && !a8 && wbits != 4)) return cudaErrorNotSupported;
  return with_wbits(wbits, [&](auto W) {
    const size_t smem = (size_t)tc_smem_bytes<W>();
    auto go = [&](auto kern) {
      const cudaError_t e = raise_smem_limit((const void*)kern, (int)smem);
      return e != cudaSuccess ? e : launch(kern, dim3(grid), dim3(kTcThreads), smem, stream, true, p, amap);
    };
    return with_flag(p.NG > grid, [&](auto MULTI) {
      if constexpr (W == 4) {
        if (a8) return go(wq_gemm_tc_kernel<4, MULTI, true>);
      }
      return with_flag(grouped, [&](auto G) {
        return with_flag(fp16, [&](auto H) { return go(wq_gemm_tc_kernel<W, MULTI, false, G && W == 4, H>); });
      });
    });
  });
}

}  // namespace b2
