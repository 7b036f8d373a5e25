// b200spark — weight-only quantized GEMV/GEMM for the decode step (small M), sm_90a.
//
// Replaces the reference's K1/K2/K3/K6/K7/K8 kernels and the dequant+cuBLAS fallbacks
// (csrc/core/kernel/cuda/gemm_lowp/gemm_a16w4_{perc,subc}_kernel.cu, gemm_a16w8_*_kernel.cu,
//  gemm_lowp_utils.cuh:582-604 reduce_sum) with ONE weight-streaming kernel family:
//
//   * init time: the reference [K,N/2] nibble / [K,N] int8 / [K,N] bf16 weights are re-laid-out into
//     tiles of (128 n x 64 k) such that each CTA's K-slice is ONE contiguous byte range and each
//     lane's 16-byte shared-memory word is exactly the mma.m16n8k16 A-fragments it needs.
//   * run time: a producer lane streams the CTA's slice HBM -> shared memory with TMA 1-D bulk copies
//     (cp.async.bulk + mbarrier ring).  The producer does NOT wait for the previous kernel
//     (programmatic dependent launch): weights of op i+1 stream in while op i drains.
//   * 8 consumer warps (one n16 tile each) expand nibbles to exact bf16 integers (16+q) with
//     lop3/shf only, run C^T[n16 x m8] += W^T[n16 x k16] * A^T[k16 x m8] on the tensor cores
//     (weights = A operand, activations = B operand: batch 1..8 fills the n8 side, no wasted rows),
//     and apply the affine dequant on the fp32 accumulators:  s * (acc - (16+z) * sum_k a).
//   * split-K across CTAs.  Default: the S in {2, 4, 8} k-slices of a tile form a thread-block cluster, the partial tiles stay
//     in shared memory and every CTA sums and finishes its share of the tile through distributed shared memory (slice order:
//     deterministic).  Fallback (narrow shapes, forced splits, the fused all-reduce): fp32 partials in the caller's workspace,
//     the last CTA of an n-group (device counter) sums them in fixed order.  Either way: fused bias / activation / residual /
//     SwiGLU, optionally a self-contained RMSNorm (b2_gemm_fuse): the kernel normalises its own activations, nothing comes
//     from the producer (the RMSNorm hand-off of batches >= 17 belongs to the wgmma kernel, wq_gemm_tc.cu).
//   * the 16-bit type of activations / outputs / scales is a template parameter (Ft<H>: bf16 or fp16; fp16 uses 128 + q).
//
// Roofline: HBM-bound; algorithmic bytes/launch = K*N*wbits/8 + 4*G*N + 2*M*(K+N).
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <new>

#include "b2_common.cuh"
#include "comm_shared.cuh"
#include "wq_gemm_shared.cuh"

namespace b2 {

constexpr int kWarps = 8;                  // consumer warps per CTA
constexpr int kThreads = kWarps * 32 + 32; // + producer warp
constexpr int kStageBytes = 8192;
static_assert(kBN == kWarps * 16, "one n16 tile per consumer warp");

struct GemmParams {
  const uint8_t* packed;
  const float2* sz;  // [G][Np] (scale, zero + bias-constant)
  const __nv_bfloat16* A;
  int64_t lda;
  __nv_bfloat16* C;
  int64_t ldc;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* residual;
  float* ws;
  unsigned* counters;
  int M, N, K, Np, KT, NG, S;
  int group_tiles;  // k-tiles per quant group (GROUPED) else 0
  int quanta;       // number of split quanta (KT / max(group_tiles,1))
  int xt;           // k-tiles per activation chunk (multiple of TPS and of the quant group)
  int nst_log2;     // log2(pipeline stages)
  int act;
  float alpha;
  int cluster;    // 1: the S k-slices of a tile are one thread-block cluster; partial tiles are summed through distributed
                  //    shared memory (no workspace, no counters)
  // optional self-contained RMSNorm (b2_gemm_fuse): the kernel takes the row statistics itself while staging the
  // activations (K == hidden)
  int norm_self;
  const __nv_bfloat16* norm_gamma;
  float norm_inv_hidden, norm_eps;
  // optional fused all-reduce of the output over tensor-parallel ranks (b2_gemm_wq_run_allreduce)
  int comm_on;
  CommDev comm;
};

template <int WBITS>
struct WTraits {
  static constexpr int TILE_BYTES = Image<WBITS>::kTileBytes;
  static constexpr int TPS = kStageBytes / TILE_BYTES > 0 ? kStageBytes / TILE_BYTES : 1;  // tiles per stage
  static constexpr int STAGE_BYTES = TPS * TILE_BYTES;
};

__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// One k-tile (64 k x 16 n per warp) of tensor-core work for this warp.  woff0/woff1: byte offsets of this thread's
// row g / row g+8 data inside the tile; xaddr: this thread's 32 bytes of activations (16 consecutive k).
template <int WBITS, int MT, bool H>
__device__ __forceinline__ void tile_mma(float (&acc)[MT][4], uint32_t wtile, uint32_t woff0, uint32_t woff1, uint32_t xaddr,
                                         int XS8) {
  uint4 xb[MT][2];
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    xb[m][0] = lds128(xaddr + m * XS8);
    xb[m][1] = lds128(xaddr + m * XS8 + 16);
  }
  if (WBITS == 4) {
    const uint2 w0 = lds64(wtile + woff0), w1 = lds64(wtile + woff1);
    const uint32_t r0w[2] = {w0.x, w0.y}, r1w[2] = {w1.x, w1.y};
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const uint32_t u = r0w[j], v = r1w[j];
      const uint32_t p0 = lop3_and_or(u, kMask4, Ft<H>::kMagic), q0 = lop3_and_or(v, kMask4, Ft<H>::kMagic);
      const uint32_t p1 = lop3_and_or(__funnelshift_r(u, u, 4), kMask4, Ft<H>::kMagic), q1 = lop3_and_or(__funnelshift_r(v, v, 4), kMask4, Ft<H>::kMagic);
      const uint32_t p2 = lop3_and_or(__funnelshift_r(u, u, 8), kMask4, Ft<H>::kMagic), q2 = lop3_and_or(__funnelshift_r(v, v, 8), kMask4, Ft<H>::kMagic);
      const uint32_t p3 = lop3_and_or(__funnelshift_r(u, u, 12), kMask4, Ft<H>::kMagic), q3 = lop3_and_or(__funnelshift_r(v, v, 12), kMask4, Ft<H>::kMagic);
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        Ft<H>::mma(acc[m], p0, q0, p1, q1, xb[m][j].x, xb[m][j].y);
        Ft<H>::mma(acc[m], p2, q2, p3, q3, xb[m][j].z, xb[m][j].w);
      }
    }
  } else if (WBITS == 8) {
    const uint4 w0 = lds128(wtile + woff0), w1 = lds128(wtile + woff1);
    const uint32_t r0w[4] = {w0.x, w0.y, w0.z, w0.w}, r1w[4] = {w1.x, w1.y, w1.z, w1.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t u = r0w[j], v = r1w[j];
      const uint32_t l0 = lop3_and_or(u, kMask4, Ft<H>::kMagic), m0 = lop3_and_or(v, kMask4, Ft<H>::kMagic);
      const uint32_t h0 = lop3_and_or(__funnelshift_r(u, u, 4), kMask4, Ft<H>::kMagicHi), n0 = lop3_and_or(__funnelshift_r(v, v, 4), kMask4, Ft<H>::kMagicHi);
      const uint32_t l1 = lop3_and_or(__funnelshift_r(u, u, 8), kMask4, Ft<H>::kMagic), m1 = lop3_and_or(__funnelshift_r(v, v, 8), kMask4, Ft<H>::kMagic);
      const uint32_t h1 = lop3_and_or(__funnelshift_r(u, u, 12), kMask4, Ft<H>::kMagicHi), n1 = lop3_and_or(__funnelshift_r(v, v, 12), kMask4, Ft<H>::kMagicHi);
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        const uint32_t b0 = (j & 1) ? xb[m][j >> 1].z : xb[m][j >> 1].x;
        const uint32_t b1 = (j & 1) ? xb[m][j >> 1].w : xb[m][j >> 1].y;
        Ft<H>::mma(acc[m], l0, m0, l1, m1, b0, b1);   // low nibbles:  16 + lo
        Ft<H>::mma(acc[m], h0, n0, h1, n1, b0, b1);   // high nibbles: 16 * (16 + hi)
      }
    }
  } else {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const uint4 w0 = lds128(wtile + woff0 + u * Image<16>::kChunkBytes), w1 = lds128(wtile + woff1 + u * Image<16>::kChunkBytes);
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        Ft<H>::mma(acc[m], w0.x, w1.x, w0.y, w1.y, xb[m][u].x, xb[m][u].y);
        Ft<H>::mma(acc[m], w0.z, w1.z, w0.w, w1.w, xb[m][u].z, xb[m][u].w);
      }
    }
  }
}

B2_TRACE_DECL(g_gemv_tr)
#ifdef B2_TRACE
extern "C" int b2_debug_trace_gemv(unsigned long long* host_out) { return (int)cudaMemcpyFromSymbol(host_out, g_gemv_tr, sizeof(g_gemv_tr)); }
#endif

// CTAs per SM each instantiation is compiled for (registers <= 65536 / (kThreads * n)).  make_plan sizes the split-K from
// the occupancy, so this fixes the plans, and with them the summation order of every result; left to ptxas, the register
// budget (and the occupancy) moves with unrelated edits of the kernel body.
template <int W, int MT, bool G, bool H>
constexpr int kMinCtasPerSm = MT == 1 ? ((W == 8 && (G || H)) || (W == 4 && G) ? 3 : 4)
                                      : (W == 16 ? (H ? 3 : 4) : W == 4 && !H ? (G ? 2 : 4) : 3);

template <int WBITS, int MT, bool GROUPED, bool H>
__global__ void __launch_bounds__(kThreads, (kMinCtasPerSm<WBITS, MT, GROUPED, H>)) wq_gemm_kernel(const GemmParams p) {
  using T = WTraits<WBITS>;
  using F = Ft<H>;  // bf16 / fp16 activations, outputs, bias, residual
  constexpr int MP = 8 * MT;
  const int NST = 1 << p.nst_log2;
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;

  const int ng = blockIdx.x / p.S;
  const int s = blockIdx.x - ng * p.S;
  const int gt = GROUPED ? p.group_tiles : 1;
  const int q0 = (int)((int64_t)s * p.quanta / p.S), q1 = (int)((int64_t)(s + 1) * p.quanta / p.S);
  const int kt0 = q0 * gt, kt1 = q1 * gt;
  const int nt = kt1 - kt0;

  // ---- shared memory carve-up
  uint8_t* ring = smem;
  const int ring_bytes = NST * T::STAGE_BYTES;
  const int XS = p.xt * 128 + 16;  // activation row stride (bytes), == 16 mod 128: conflict-free LDS.128
  uint8_t* xs = ring + ring_bytes;
  uint8_t* grow = xs + MP * XS;                               // [xt*64] gamma slice of the chunk (self-contained norm)
  float* fs = reinterpret_cast<float*>(grow + XS);           // [MP][kBN] partial tile
  float* suma = fs + MP * kBN;                                // [MP][groups per chunk] (or [MP])
  const int gpc = GROUPED ? p.xt / gt : 1;                    // groups per chunk
  float* sumsq = suma + MP * gpc;  // [MP] self-contained norm: sum x^2 of the rows over this CTA's k-slice (all of K once
                                   //      the workspace reducer has added the slices)
  float* srs = sumsq + MP;         // [MP] self-contained norm: 1/rms of the rows
  uint64_t* full = reinterpret_cast<uint64_t*>((reinterpret_cast<uintptr_t>(srs + MP + 4) + 7) & ~uintptr_t(7));
  uint64_t* empty = full + NST;
  uint64_t* xbar = empty + NST;  // activation rows of a chunk landed (bulk copies)
  uint64_t* gbar = xbar + 1;     // gamma slice of a chunk landed
  __shared__ int s_is_last;

  const bool tr0 = blockIdx.x == 0 && tid == 0;
  if (tr0) B2_TR(g_gemv_tr, 0);
  if (tid == 0) {
    for (int i = 0; i < NST; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], kWarps);
    }
    mbar_init(xbar, 1);
    mbar_init(gbar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();  // let the next kernel start streaming ITS weights as soon as SM resources free up
  if (tr0) B2_TR(g_gemv_tr, 1);

  if (warp == kWarps) {
    // ===================== producer: TMA bulk copies, independent of the previous kernel ==========
    if (lane == 0) {
      const uint8_t* wsrc = p.packed + ((size_t)ng * p.KT + kt0) * T::TILE_BYTES;
      const int nstages_total = (nt + T::TPS - 1) / T::TPS;
      for (int i = 0; i < nstages_total; ++i) {
        const int slot = i & (NST - 1);
        if (i >= NST) mbar_wait(&empty[slot], ((i >> p.nst_log2) & 1) ^ 1);
        const int tiles = min(T::TPS, nt - i * T::TPS);
        const uint32_t bytes = tiles * T::TILE_BYTES;
        mbar_arrive_expect_tx(&full[slot], bytes);
        bulk_g2s(ring + slot * T::STAGE_BYTES, wsrc + (size_t)i * T::STAGE_BYTES, bytes, &full[slot]);
        if (blockIdx.x == 0 && i == 0) B2_TR(g_gemv_tr, 2);
      }
    }
    return;
  }

  // ===================== consumers =====================
  const int n0 = ng * kBN + warp * 16 + g;  // this thread's two output channels: n0, n0+8
  float2 sz0 = make_float2(1.f, 0.f), sz1 = make_float2(1.f, 0.f);
  if (!GROUPED && WBITS != 16) {  // immutable after prepare: safe to read before the dependency wait
    sz0 = p.sz[n0];
    sz1 = p.sz[n0 + 8];
  }

  float acc[MT][4], facc[MT][4];
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[m][c] = facc[m][c] = 0.f;

  // rows M..MP-1 of the MMA's batch dimension stay zero for the whole kernel
  for (int i = p.M * XS + tid * 16; i < MP * XS; i += kWarps * 32 * 16) *reinterpret_cast<uint4*>(xs + i) = make_uint4(0, 0, 0, 0);
  const int64_t k_first = (int64_t)kt0 * kBK;
  if (p.norm_self && tid == 0) {  // gamma is immutable: its first slice travels ahead of the dependency wait
    const int64_t left = ((int64_t)p.K - k_first) * 2;
    const uint32_t gb = (uint32_t)max((int64_t)0, min((int64_t)min(p.xt, nt) * 128, left));
    mbar_arrive_expect_tx(gbar, gb);
    if (gb) bulk_g2s(grow, p.norm_gamma + k_first, gb, gbar);
  }

  pdl_wait();  // activations / workspace / counters belong to the previous kernels from here on
  if (tr0) B2_TR(g_gemv_tr, 3);

  const uint32_t w_ring = smem_u32(ring);
  // this thread's rows (16*warp + g, +8) inside the [chunk][row ^ swz][16B] tile image
  const int wc = WBITS == 4 ? (t >> 1) : (WBITS == 8 ? t : 2 * t);
  const int wr = warp * 16 + g;
  const uint32_t woff0 = Image<WBITS>::chunk_offset(wr, wc) + (WBITS == 4 ? 8 * (t & 1) : 0);
  const uint32_t woff1 = Image<WBITS>::chunk_offset(wr + 8, wc) + (WBITS == 4 ? 8 * (t & 1) : 0);
  const uint32_t x_thr = smem_u32(xs) + g * XS + t * 32;
  const int XS8 = 8 * XS;
  int stage_i = 0;

  for (int xc0 = 0; xc0 < nt; xc0 += p.xt) {  // p.xt is a multiple of TPS and of the quant group
    const int xn = min(p.xt, nt - xc0);
    if (xc0 > 0) named_bar_sync(1, kWarps * 32);  // previous chunk fully consumed
    // ---- stage activations A[m][k-chunk] (bf16) -> xs (zero-fill m >= M, k >= K) and, in the same pass, sum_k a[m][k] per
    //      (row, quant group): the zero-point term of the affine dequant.  Two forms: plain loads by all eight warps (the
    //      default: measured faster than bulk copies as soon as several rows are live — Qwen2-72B TP=2 batch 16: 946 vs 894
    //      tok/s), and for batches <= 2 / the self-contained RMSNorm one bulk copy per live row plus one pass over shared
    //      memory that also scales by gamma and collects the row statistics (batch 1: 445 -> 462 tok/s with the norm fused).
    if (!(p.norm_self || p.M <= 2)) {
      const int64_t kbase = (int64_t)(kt0 + xc0) * kBK;
      const int nvec = xn * 8;
      const int gvec = GROUPED ? gt * 8 : nvec;  // 16B vectors per quant group
      for (int m = warp; m < MP; m += kWarps) {
        const __nv_bfloat16* arow = p.A + (int64_t)m * p.lda + kbase;
        uint8_t* xrow = xs + m * XS;
        const bool mrow = m < p.M;
        for (int v0 = 0, gi = 0; v0 < nvec; v0 += gvec, ++gi) {
          float sacc = 0.f;
          for (int v = v0 + lane; v < v0 + gvec; v += 32) {
            uint4 val = make_uint4(0, 0, 0, 0);
            if (mrow && kbase + v * 8 < p.K) val = *reinterpret_cast<const uint4*>(arow + v * 8);
            *reinterpret_cast<uint4*>(xrow + v * 16) = val;
            sacc += (F::lo(val.x) + F::hi(val.x)) + (F::lo(val.y) + F::hi(val.y)) +
                    (F::lo(val.z) + F::hi(val.z)) + (F::lo(val.w) + F::hi(val.w));
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) sacc += __shfl_xor_sync(0xffffffffu, sacc, o);
          if (lane == 0) {
            if (GROUPED) suma[m * gpc + gi] = sacc;
            else suma[m] = (xc0 == 0 ? 0.f : suma[m]) + sacc;
          }
        }
      }
    } else
    {
      const int64_t kbase = (int64_t)(kt0 + xc0) * kBK;
      const int chunk = xc0 / p.xt;
      const uint32_t rb = (uint32_t)max((int64_t)0, min((int64_t)xn * 128, ((int64_t)p.K - kbase) * 2));  // live bytes per row
      if (warp == 0) {  // lane m issues row m's copy: one issue slot for the whole chunk instead of M serial ones
        if (lane == 0) {
          fence_proxy_async();  // the previous chunk was read / rewritten through the generic proxy
          if (p.norm_self && xc0 > 0) {
            mbar_arrive_expect_tx(gbar, rb);
            if (rb) bulk_g2s(grow, p.norm_gamma + kbase, rb, gbar);
          }
          mbar_arrive_expect_tx(xbar, rb * p.M);
        }
        __syncwarp();
        if (rb && lane < p.M) bulk_g2s(xs + lane * XS, p.A + (int64_t)lane * p.lda + kbase, rb, xbar);
      }
      if (tr0 && xc0 == 0) B2_TR(g_gemv_tr, 12);
      mbar_wait(xbar, chunk & 1);
      if (p.norm_self) mbar_wait(gbar, chunk & 1);
      if (tr0 && xc0 == 0) B2_TR(g_gemv_tr, 13);
      const int nvec = xn * 8;
      const int gvec = GROUPED ? gt * 8 : nvec;  // 16B vectors per quant group
      const int lvec = rb >> 4;                  // live vectors per row
      for (int m = warp; m < MP; m += kWarps) {
        uint8_t* xrow = xs + m * XS;
        const bool mrow = m < p.M;
        float ssq = 0.f;
        for (int v0 = 0, gi = 0; v0 < nvec; v0 += gvec, ++gi) {
          float sacc = 0.f;
          if (mrow) {
            for (int v = v0 + lane; v < v0 + gvec; v += 32) {
              uint4 val = make_uint4(0, 0, 0, 0);
              if (v < lvec) {
                val = *reinterpret_cast<const uint4*>(xrow + v * 16);
                if (p.norm_self) {
                  // self-contained RMSNorm: bf16(x * gamma) feeds the MMAs, sum x^2 of this CTA's k-slice is collected on
                  // the way; the 1/rms factor is linear in the row and is applied to the reduced fp32 tile in the epilogue
                  const uint4 gv = *reinterpret_cast<const uint4*>(grow + v * 16);
                  const float x0 = F::lo(val.x), x1 = F::hi(val.x), x2 = F::lo(val.y), x3 = F::hi(val.y);
                  const float x4 = F::lo(val.z), x5 = F::hi(val.z), x6 = F::lo(val.w), x7 = F::hi(val.w);
                  ssq += (x0 * x0 + x1 * x1) + (x2 * x2 + x3 * x3) + (x4 * x4 + x5 * x5) + (x6 * x6 + x7 * x7);
                  val.x = F::pack(x0 * F::lo(gv.x), x1 * F::hi(gv.x));
                  val.y = F::pack(x2 * F::lo(gv.y), x3 * F::hi(gv.y));
                  val.z = F::pack(x4 * F::lo(gv.z), x5 * F::hi(gv.z));
                  val.w = F::pack(x6 * F::lo(gv.w), x7 * F::hi(gv.w));
                  *reinterpret_cast<uint4*>(xrow + v * 16) = val;
                }
              } else {
                *reinterpret_cast<uint4*>(xrow + v * 16) = val;  // k >= K
              }
              sacc += (F::lo(val.x) + F::hi(val.x)) + (F::lo(val.y) + F::hi(val.y)) +
                      (F::lo(val.z) + F::hi(val.z)) + (F::lo(val.w) + F::hi(val.w));
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) sacc += __shfl_xor_sync(0xffffffffu, sacc, o);
          }
          if (lane == 0) {
            if (GROUPED) suma[m * gpc + gi] = sacc;
            else suma[m] = (xc0 == 0 ? 0.f : suma[m]) + sacc;
          }
        }
        if (p.norm_self) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) ssq += __shfl_xor_sync(0xffffffffu, ssq, o);
          if (lane == 0) sumsq[m] = (xc0 == 0 ? 0.f : sumsq[m]) + ssq;
        }
      }
    }
    if (tr0 && xc0 == 0) B2_TR(g_gemv_tr, 14);
    named_bar_sync(1, kWarps * 32);
    if (tr0 && xc0 == 0) B2_TR(g_gemv_tr, 4);

    // ---- main loop: one pipeline stage (TPS k-tiles) per iteration
    int gcount = 0;  // tiles into the current quant group
    for (int xs0 = 0; xs0 < xn; xs0 += T::TPS, ++stage_i) {
      const int slot = stage_i & (NST - 1);
      mbar_wait(&full[slot], (stage_i >> p.nst_log2) & 1);
      if (tr0 && stage_i == 0) B2_TR(g_gemv_tr, 5);
      const uint32_t wst = w_ring + slot * T::STAGE_BYTES;
#pragma unroll
      for (int ti = 0; ti < T::TPS; ++ti) {
        if (T::TPS > 1 && xs0 + ti >= xn) break;
        if (GROUPED && gcount == 0) {  // prefetch this group's (scale, zero) — consumed at group end
          const int grp = (kt0 + xc0 + xs0 + ti) / gt;
          sz0 = p.sz[(size_t)grp * p.Np + n0];
          sz1 = p.sz[(size_t)grp * p.Np + n0 + 8];
        }
        tile_mma<WBITS, MT, H>(acc, wst + ti * T::TILE_BYTES, woff0, woff1, x_thr + (xs0 + ti) * 128, XS8);
        if (GROUPED && ++gcount == gt) {  // fold this quant group into the fp32 result
          gcount = 0;
          const int gi = (xs0 + ti) / gt;
#pragma unroll
          for (int m = 0; m < MT; ++m) {
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const float2 z = (c < 2) ? sz0 : sz1;
              const float sa = suma[(m * 8 + 2 * t + (c & 1)) * gpc + gi];
              facc[m][c] += z.x * (acc[m][c] - z.y * sa);
              acc[m][c] = 0.f;
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[slot]);
    }
  }

  if (tr0) B2_TR(g_gemv_tr, 6);
  // ---- dequant epilogue on the accumulators (per-channel) and park the tile in shared memory
#pragma unroll
  for (int m = 0; m < MT; ++m) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float v;
      if (WBITS == 16) v = acc[m][c];
      else if (GROUPED) v = facc[m][c];
      else {
        const float2 z = (c < 2) ? sz0 : sz1;
        const float sa = suma[m * 8 + 2 * t + (c & 1)];
        v = z.x * (acc[m][c] - z.y * sa);
      }
      fs[(m * 8 + 2 * t + (c & 1)) * kBN + warp * 16 + g + (c >> 1) * 8] = v;
    }
  }
  named_bar_sync(1, kWarps * 32);

  const int ctid = tid;
  const int MPK = MP * kBN;
  if (p.cluster) {
    // ---- split-K inside a thread-block cluster: every k-slice's partial tile (and row statistics) stays in its CTA's shared
    // memory; after one cluster barrier each CTA sums its share of the tile's 16-byte granules over the S slices in slice
    // order (deterministic) through distributed shared memory and finishes them — no workspace round trip, no fence, no
    // atomic ticket, and the epilogue of one tile is spread over S SMs.
    if (tr0) B2_TR(g_gemv_tr, 7);
    cluster_arrive();
    cluster_wait();
    if (tr0) B2_TR(g_gemv_tr, 8);
    const uint32_t fs_a = smem_u32(fs), sumsq_a = smem_u32(sumsq);
    if (p.norm_self) {
      if (ctid < MP) {
        float ss = 0.f;
        for (int r = 0; r < p.S; ++r) ss += ld_dsmem_f(dsmem_addr(sumsq_a + ctid * 4, r));
        srs[ctid] = rsqrtf(ss * p.norm_inv_hidden + p.norm_eps);
      }
      named_bar_sync(1, kWarps * 32);
    }
    auto slice_sum = [&](int elem) {  // sum over the S slices of the 4 floats at fs[elem .. elem+3], slice order
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int r0 = 0; r0 < p.S; r0 += 4) {
        float4 b[4];
#pragma unroll
        for (int r = 0; r < 4; ++r)
          b[r] = r0 + r < p.S ? ld_dsmem_f4(dsmem_addr(fs_a + elem * 4, r0 + r)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int r = 0; r < 4; ++r) { a.x += b[r].x; a.y += b[r].y; a.z += b[r].z; a.w += b[r].w; }
      }
      return a;
    };
    if (!p.comm_on) {  // the fused all-reduce needs the whole tile in one CTA: gathered below
      if (p.act == B2_ACT_SWIGLU) {
        for (int i = s + p.S * ctid; i < p.M * 16; i += p.S * kWarps * 32) {
          const int m = i >> 4, cg = i & 15;
          const int n = ng * 64 + cg * 4;
          if (n >= p.N) continue;
          const float4 gq = slice_sum(m * kBN + cg * 4), uq = slice_sum(m * kBN + 64 + cg * 4);
          const float ra = p.norm_self ? p.alpha * srs[m] : p.alpha;
          const float v[4] = {apply_act<B2_ACT_SILU>(gq.x * ra) * (uq.x * ra), apply_act<B2_ACT_SILU>(gq.y * ra) * (uq.y * ra),
                              apply_act<B2_ACT_SILU>(gq.z * ra) * (uq.z * ra), apply_act<B2_ACT_SILU>(gq.w * ra) * (uq.w * ra)};
          __nv_bfloat16* cp = p.C + (int64_t)m * p.ldc + n;
          if (n + 3 < p.N && (reinterpret_cast<uintptr_t>(cp) & 7) == 0) {
            *reinterpret_cast<uint2*>(cp) = make_uint2(F::pack(v[0], v[1]), F::pack(v[2], v[3]));
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (n + j < p.N) cp[j] = F::from_f(v[j]);
          }
        }
      } else {
        for (int i = s + p.S * ctid; i < p.M * 32; i += p.S * kWarps * 32) {
          const int m = i >> 5, c = (i & 31) * 4;
          const int n = ng * kBN + c;
          if (n >= p.N) continue;
          const float4 q = slice_sum(m * kBN + c);
          const float ra = p.norm_self ? p.alpha * srs[m] : p.alpha;
          float v[4] = {q.x * ra, q.y * ra, q.z * ra, q.w * ra};
          __nv_bfloat16* cp = p.C + (int64_t)m * p.ldc + n;
          const __nv_bfloat16* rp = p.residual ? p.residual + (int64_t)m * p.ldc + n : nullptr;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (n + j < p.N) {
              if (p.bias) v[j] += F::to_f(p.bias[n + j]);
              v[j] = apply_act_rt(v[j], p.act);
              if (rp) v[j] += F::to_f(rp[j]);
            }
          }
          if (n + 3 < p.N && (reinterpret_cast<uintptr_t>(cp) & 7) == 0) {
            *reinterpret_cast<uint2*>(cp) = make_uint2(F::pack(v[0], v[1]), F::pack(v[2], v[3]));
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (n + j < p.N) cp[j] = F::from_f(v[j]);
          }
        }
      }
      if (tr0) B2_TR(g_gemv_tr, 10);
      cluster_arrive();  // peers may still be reading this CTA's tile: stay resident until everybody is done
      cluster_wait();
      if (tr0) B2_TR(g_gemv_tr, 11);
      return;
    }
    // fused all-reduce: slice 0 collects the whole tile and runs the exchange below
    if (s == 0) {
      for (int i = ctid; i < p.M * 32; i += kWarps * 32) {
        const float4 q = slice_sum(i * 4);
        *reinterpret_cast<float4*>(fs + i * 4) = q;
      }
    }
    cluster_arrive();
    cluster_wait();
    if (s != 0) return;
  } else if (p.S > 1) {
    float* wsu = p.ws + ((size_t)ng * p.S + s) * MPK;
    for (int i = ctid * 4; i < p.M * kBN; i += kWarps * 32 * 4)
      *reinterpret_cast<float4*>(wsu + i) = *reinterpret_cast<const float4*>(fs + i);
    float* wsq = p.ws + (size_t)p.NG * p.S * MPK;  // [NG][S][MP] sum x^2 of each k-slice (self-contained norm)
    if (p.norm_self && ctid < p.M) wsq[((size_t)ng * p.S + s) * MP + ctid] = sumsq[ctid];
    __threadfence();
    named_bar_sync(1, kWarps * 32);
    if (tr0) B2_TR(g_gemv_tr, 7);
    if (ctid == 0) {
      const unsigned prev = atomicAdd(&p.counters[ng], 1u);
      s_is_last = (prev == (unsigned)(p.S - 1));
    }
    named_bar_sync(1, kWarps * 32);
    if (tr0) B2_TR(g_gemv_tr, 8);
    if (!s_is_last) return;
    __threadfence();
    if (ng == 0 && ctid == 0) B2_TR(g_gemv_tr, 9);
    // fixed-order sum over the S partials (deterministic); loads are issued 8 at a time so the L2 round
    // trips overlap instead of serialising behind the adds
    const float* wsg = p.ws + (size_t)ng * p.S * MPK;
    float ssq_l = 0.f;  // lane s holds slice s of row (warp, warp + 8): one round trip, overlapped with the tile loads below
    float ssq_h = 0.f;
    if (p.norm_self) {
      if (lane < p.S && warp < p.M) ssq_l = __ldcg(wsq + ((size_t)ng * p.S + lane) * MP + warp);
      if (lane < p.S && warp + kWarps < p.M) ssq_h = __ldcg(wsq + ((size_t)ng * p.S + lane) * MP + warp + kWarps);
    }
    for (int i = ctid * 4; i < p.M * kBN; i += kWarps * 32 * 4) {
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int s0 = 0; s0 < p.S; s0 += 8) {
        float4 b[8];
#pragma unroll
        for (int u = 0; u < 8; ++u)
          b[u] = (s0 + u < p.S) ? __ldcg(reinterpret_cast<const float4*>(wsg + (size_t)(s0 + u) * MPK + i))
                                : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int u = 0; u < 8; ++u) { a.x += b[u].x; a.y += b[u].y; a.z += b[u].z; a.w += b[u].w; }
      }
      *reinterpret_cast<float4*>(fs + i) = a;
    }
    if (p.norm_self) {  // S <= 32 slices, MP <= 16 rows
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        ssq_l += __shfl_xor_sync(0xffffffffu, ssq_l, o);
        ssq_h += __shfl_xor_sync(0xffffffffu, ssq_h, o);
      }
      if (lane == 0) {
        sumsq[warp] = ssq_l;
        if (MP > kWarps) sumsq[warp + kWarps] = ssq_h;
      }
    }
    if (ctid == 0) p.counters[ng] = 0;  // re-arm for the next launch / graph replay
    named_bar_sync(1, kWarps * 32);
    if (ng == 0 && ctid == 0) B2_TR(g_gemv_tr, 10);
  }

  if (p.norm_self && !p.cluster) {  // sum x^2 -> 1/rms, one thread per row (the cluster path already has it)
    if (ctid < MP) srs[ctid] = rsqrtf(sumsq[ctid] * p.norm_inv_hidden + p.norm_eps);
    named_bar_sync(1, kWarps * 32);
  }
  // ---- final: alpha (x 1/rms of the row), bias, activation, residual, bf16 store (coalesced along n)
  if (p.act == B2_ACT_SWIGLU) {  // tile = [64 gate | 64 up] channels of n in [64*ng, 64*ng+64): out = silu(gate) * up
    for (int i = ctid; i < p.M * 32; i += kWarps * 32) {
      const int m = i >> 5, np = i & 31;
      const int n = ng * 64 + np * 2;
      if (n >= p.N) continue;
      const float ra = p.norm_self ? p.alpha * srs[m] : p.alpha;
      const float g0 = fs[m * kBN + np * 2] * ra, g1 = fs[m * kBN + np * 2 + 1] * ra;
      const float u0 = fs[m * kBN + 64 + np * 2] * ra, u1 = fs[m * kBN + 64 + np * 2 + 1] * ra;
      const float v0 = apply_act<B2_ACT_SILU>(g0) * u0, v1 = apply_act<B2_ACT_SILU>(g1) * u1;
      __nv_bfloat16* cp = p.C + (int64_t)m * p.ldc + n;
      if ((n + 1) < p.N && ((reinterpret_cast<uintptr_t>(cp) & 3) == 0)) *reinterpret_cast<uint32_t*>(cp) = F::pack(v0, v1);
      else {
        cp[0] = F::from_f(v0);
        if ((n + 1) < p.N) cp[1] = F::from_f(v1);
      }
    }
    return;
  }
  if (p.comm_on) {
    // ---- fused all-reduce over the tensor-parallel ranks (row-parallel o_proj / down_proj): this CTA holds the final
    // partial sums of tile `ng` of THIS rank.  Push them (bf16, like the reference's partial outputs) into slot[rank] of
    // every rank's exchange buffer, raise the tile's flag there, wait for the other ranks' tiles in local memory, sum the
    // nranks partials in rank order in fp32, add the residual once, round once.  Tiles are independent: the exchange of
    // this tile overlaps the weight streaming of the n-groups still running.  N is even (checked on the host).
    const CommDev& cd = p.comm;
    const unsigned epoch = *reinterpret_cast<volatile unsigned*>(cd.epoch);
    const unsigned want = epoch + 1;
    const int par = epoch & 1;
    const size_t my_slot = comm_slot_offset(cd, par, cd.rank);
    for (int i = ctid; i < p.M * (kBN / 2); i += kWarps * 32) {
      const int m = i >> 6, np = i & 63;
      const int n = ng * kBN + np * 2;
      if (n >= p.N) continue;
      float v0 = fs[m * kBN + np * 2] * p.alpha, v1 = fs[m * kBN + np * 2 + 1] * p.alpha;
      if (p.bias) {
        v0 += F::to_f(p.bias[n]);
        v1 += F::to_f(p.bias[n + 1]);
      }
      const uint32_t pk = F::pack(v0, v1);
      const size_t off = my_slot + ((size_t)m * p.N + n) * 2;
      for (int r = 0; r < cd.nranks; ++r) *reinterpret_cast<uint32_t*>(cd.peer[(cd.rank + r) % cd.nranks] + off) = pk;
    }
    __threadfence_system();
    named_bar_sync(1, kWarps * 32);
    __shared__ int s_comm_ok;
    if (ctid == 0) s_comm_ok = 1;
    if (ctid < cd.nranks) {
      unsigned* f = reinterpret_cast<unsigned*>(cd.peer[ctid] + comm_flag_offset(cd, par, cd.rank, ng));
      asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(f), "r"(want) : "memory");
    }
    named_bar_sync(1, kWarps * 32);
    if (ctid < cd.nranks) {
      const unsigned* f = reinterpret_cast<const unsigned*>(cd.peer[cd.rank] + comm_flag_offset(cd, par, ctid, ng));
      if (!wait_flag(f, want, cd.timeout_ns, cd.error)) s_comm_ok = 0;
    }
    named_bar_sync(1, kWarps * 32);
    if (s_comm_ok) {
      const uint8_t* base = cd.peer[cd.rank];
      for (int i = ctid; i < p.M * (kBN / 2); i += kWarps * 32) {
        const int m = i >> 6, np = i & 63;
        const int n = ng * kBN + np * 2;
        if (n >= p.N) continue;
        const size_t eo = ((size_t)m * p.N + n) * 2;
        float a0 = 0.f, a1 = 0.f;
        for (int r = 0; r < cd.nranks; ++r) {
          const uint32_t v = __ldcg(reinterpret_cast<const uint32_t*>(base + comm_slot_offset(cd, par, r) + eo));
          a0 += F::lo(v);
          a1 += F::hi(v);
        }
        if (p.residual) {
          const uint32_t v = *reinterpret_cast<const uint32_t*>(p.residual + (int64_t)m * p.ldc + n);
          a0 += F::lo(v);
          a1 += F::hi(v);
        }
        *reinterpret_cast<uint32_t*>(p.C + (int64_t)m * p.ldc + n) = F::pack(a0, a1);
      }
    }
    named_bar_sync(1, kWarps * 32);
    if (ctid == 0) {  // the last tile of the launch advances the communicator's epoch
      __threadfence();
      if (atomicAdd(cd.done, 1u) == (unsigned)(p.NG - 1)) {
        *cd.done = 0;
        __threadfence();
        *reinterpret_cast<volatile unsigned*>(cd.epoch) = want;
      }
    }
    return;
  }
  for (int i = ctid; i < p.M * (kBN / 2); i += kWarps * 32) {
    const int m = i >> 6, np = i & 63;
    const int n = ng * kBN + np * 2;
    if (n >= p.N) continue;
    const float ra = p.norm_self ? p.alpha * srs[m] : p.alpha;
    float v0 = fs[m * kBN + np * 2] * ra, v1 = fs[m * kBN + np * 2 + 1] * ra;
    const bool has1 = (n + 1) < p.N;
    if (p.bias) {
      v0 += F::to_f(p.bias[n]);
      if (has1) v1 += F::to_f(p.bias[n + 1]);
    }
    v0 = apply_act_rt(v0, p.act);
    v1 = apply_act_rt(v1, p.act);
    __nv_bfloat16* cp = p.C + (int64_t)m * p.ldc + n;
    if (p.residual) {
      const __nv_bfloat16* rp = p.residual + (int64_t)m * p.ldc + n;
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
  if (ng == 0 && ctid == 0) B2_TR(g_gemv_tr, 11);
}

// ------------------------------------------------------------------------------------------------
// init-time re-layout (reference layouts -> tile image, wq_gemm_shared.cuh).  One thread per 32-bit word of the image:
// word index -> (tile, chunk, stored row, word j) -> logical row / k run.  Sources: int4 [K, ceil(N/2)] (low nibble = even
// column), int8 / uint8 [K, N] (int8 stored with the sign bit flipped: 128 + q), bf16 [K, N]; k >= K and n >= N pack as 0.
// pair != 0: rows 0..63 of every 128-row tile come from q (gate), rows 64..127 from q2 (up).
// ------------------------------------------------------------------------------------------------
template <int WBITS>
__global__ void pack_image_kernel(uint32_t* __restrict__ dst, const void* __restrict__ q, const void* __restrict__ q2, int pair, int K,
                                  int N, int KT, int NG, int is_signed) {
  using I = Image<WBITS>;
  const int64_t total = (int64_t)NG * KT * I::kTileWords;
  const uint32_t flip = (WBITS == 8 && is_signed) ? 0x80u : 0u;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int j = i & 3;
    const int rs = (i >> 2) & (kBN - 1);
    const int c = (i / (4 * kBN)) & (I::kChunks - 1);
    const int64_t tile = i / I::kTileWords;
    const int kt = tile % KT, ng = tile / KT;
    const int r = rs ^ I::swz(c);
    const int n = pair ? ng * 64 + (r & 63) : ng * kBN + r;
    const void* src = (pair && r >= 64) ? q2 : q;
    uint32_t word = 0;
    for (int e = 0; e < I::kKPerWord; ++e) {  // k run of the word: even k in the low half, odd k in the high half
      const int k = kt * kBK + I::kKPerChunk * c + I::kKPerWord * j + e;
      uint32_t v = 0;
      if (n < N && k < K) {
        if (WBITS == 4) {
          const uint8_t b = static_cast<const uint8_t*>(src)[(int64_t)k * ((N + 1) / 2) + (n >> 1)];
          v = (n & 1) ? (b >> 4) : (b & 0xF);
        } else if (WBITS == 8) {
          v = static_cast<const uint8_t*>(src)[(int64_t)k * N + n];
        } else {
          v = static_cast<const uint16_t*>(src)[(int64_t)k * N + n];
        }
      }
      word |= (v ^ flip) << (WBITS * ((e >> 1) + (e & 1) * I::kKPerWord / 2));
    }
    dst[i] = I::kRotated ? (word << 3) | (word >> 29) : word;
  }
}

// (scale, zero) bf16 [G][N] -> float2 [G][Np] with the integer-bias constant folded into the zero
__global__ void pack_sz_kernel(float2* __restrict__ dst, const __nv_bfloat16* __restrict__ scales,
                               const __nv_bfloat16* __restrict__ zeros, const __nv_bfloat16* __restrict__ scales2,
                               const __nv_bfloat16* __restrict__ zeros2, int pair, int G, int N, int Np, float zbias, int fp16) {
  const int64_t total = (int64_t)G * Np;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int np = i % Np, gi = i / Np;
    const int r = np & (kBN - 1), ng = np / kBN;
    const int n = pair ? ng * 64 + (r & 63) : np;
    const __nv_bfloat16* sc = (pair && r >= 64) ? scales2 : scales;
    const __nv_bfloat16* zr = (pair && r >= 64) ? zeros2 : zeros;
    float2 v = make_float2(0.f, 0.f);
    if (n < N) {
      const __nv_bfloat16 sv = sc[(int64_t)gi * N + n], zv = zr[(int64_t)gi * N + n];
      v = fp16 ? make_float2(Ft<true>::to_f(sv), Ft<true>::to_f(zv) + zbias) : make_float2(Ft<false>::to_f(sv), Ft<false>::to_f(zv) + zbias);
    }
    dst[i] = v;
  }
}

}  // namespace b2

// ================================================================================================
// host side
// ================================================================================================
using namespace b2;

struct Plan {
  bool valid = false;
  int S = 1, xt = 1, smem = 0, quanta = 1, nst_log2 = 2;
  bool cluster = false;  // the S k-slices of a tile form a thread-block cluster (DSMEM reduction)
};

struct b2_gemm_wq {
  b2_gemm_wq_desc d;
  int Kp = 0, Np = 0, KT = 0, NG = 0, G = 1, group_tiles = 0;
  int group_k = 0;  // > 0: quantization group size that is not a multiple of 64 (params looked up per 8-k word)
  size_t packed_bytes = 0;
  void* packed = nullptr;
  bool own_packed = false;
  float2* sz = nullptr;
  bool own_sz = false;
  unsigned* counters = nullptr;
  Plan plans[2];  // MT = 1, 2
  int tc_grid = 0, tc_rounds = 0, tc_S = 1, tc_h = 0;  // schedule of the wgmma path (TcSched; tc_grid 0 = not planned)
  bool pair = false;  // gate/up pair image (SwiGLU epilogue): physical channels = 2 * N
  int device = 0;
};

typedef void (*gemm_kernel_t)(const GemmParams);

// bf16 weights carry no sub-channel params: one instantiation whatever `grouped` says
static gemm_kernel_t pick_kernel(int wbits, bool grouped, int mt, bool fp16) {
  return with_wbits(wbits, [&](auto W) {
    return with_flag(grouped, [&](auto G) {
      return with_flag(mt == 1, [&](auto MT1) {
        return with_flag(fp16, [&](auto H) { return wq_gemm_kernel<W, MT1 ? 1 : 2, G && W != 16, H>; });
      });
    });
  });
}
static int stage_bytes_of(int wbits) { return with_wbits(wbits, [](auto W) { return WTraits<W>::STAGE_BYTES; }); }

cudaError_t b2::raise_smem_limit(const void* kern, int smem) {
  static std::mutex mu;
  static std::map<const void*, int> limit;
  std::lock_guard<std::mutex> lk(mu);
  int& cur = limit[kern];
  if (smem <= cur) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e == cudaSuccess) cur = smem;
  return e;
}

static int make_plan(b2_gemm_wq* h, int mti) {
  Plan& pl = h->plans[mti];
  if (pl.valid) return B2_OK;
  const int mt = 1 << mti, MP = 8 * mt;
  const bool grouped = h->group_tiles > 0;
  const int gt = grouped ? h->group_tiles : 1;
  const int quanta = h->KT / gt;
  const int sms = sm_count();
  gemm_kernel_t kern = pick_kernel(h->d.wbits, grouped, mt, h->d.ft == B2_DT_F16);
  const int ring_kb = env_int("B2_GEMM_RING_KB", 32);
  auto log2_stages = [&](int kb) {
    int l = 1;
    while ((2 << l) * stage_bytes_of(h->d.wbits) <= kb * 1024) ++l;
    return l;
  };
  int nst_log2 = log2_stages(ring_kb);
  const int tps = with_wbits(h->d.wbits, [](auto W) { return WTraits<W>::TPS; });
  const int xq = gt > tps ? gt : tps;  // chunk granularity (gt and tps are powers of two)
  const int x_budget = env_int("B2_GEMM_XBYTES", 20 * 1024);
  // activation chunk: as many k-tiles as fit the budget, a multiple of the quant group
  int xt_cap = (x_budget / (MP + 1) - 16) / 128;  // MP activation rows + the gamma slice
  xt_cap = xt_cap / xq * xq;
  if (xt_cap < xq) xt_cap = xq;
  auto smem_for = [&](int xt, int nl2) {
    const int gpc = grouped ? xt / gt : 1;
    return (1 << nl2) * stage_bytes_of(h->d.wbits) + (MP + 1) * (xt * 128 + 16) + MP * kBN * 4 + MP * gpc * 4 + 2 * MP * 4 + 16 + 8 +
           (1 << nl2) * 16 + 16 + 64;
  };
  // first guess occupancy with the cap, derive S, then shrink xt to what a unit really needs
  int smem = smem_for(xt_cap, nst_log2);
  B2_CUDA_TRY(raise_smem_limit((const void*)kern, smem));
  int occ = 1;
  B2_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kThreads, smem));
  if (occ < 1) occ = 1;
  const int want = env_int("B2_GEMM_CTAS_PER_SM", 4);  // leave room for the NEXT kernel's CTAs (PDL overlap)
  if (want > 0 && occ > want) occ = want;
  const int slots = occ * sms;
  int S = slots / h->NG;
  const int min_quanta = (2 + gt - 1) / gt;  // at least ~2 k-tiles per unit
  if (S > quanta / (min_quanta > 0 ? min_quanta : 1)) S = quanta / (min_quanta > 0 ? min_quanta : 1);
  const int smax = env_int("B2_GEMM_MAX_SPLIT", 32);
  if (S > smax) S = smax;
  if (S < 1) S = 1;
  const int force = env_int("B2_GEMM_FORCE_SPLIT", 0);
  if (force > 0) S = force < quanta ? force : quanta;
  if (S > 32) S = 32;  // the reducer reads one k-slice statistic per lane
  // ---- split-K inside thread-block clusters (the default when it keeps enough CTAs in flight): S in {2, 4, 8} slices of a
  // tile form one cluster, the partial tiles meet in distributed shared memory.  Fewer, fatter CTAs than the global
  // split (<= 8 slices), so the ring grows to keep the same number of weight bytes in flight.  8 is the portable cluster size
  // limit; the non-portable 16 measured no better (o_proj 7.3 vs 6.4 us).
  bool cluster = false;
  if (env_int("B2_GEMM_CLUSTER", 1) && force <= 0 && S > 1) {
    int sc = 2;
    while (sc * 2 <= S && sc * 2 <= 8) sc *= 2;
    while (sc > 1 && !cluster) {
      if (h->NG * sc * 4 < sms * 3) break;  // too few CTAs to pull the HBM bandwidth: keep the wide global split
      const int nl2 = h->NG * sc <= 2 * sms ? log2_stages(env_int("B2_GEMM_CLUSTER_RING_KB", 64)) : nst_log2;
      const int sm_c = smem_for(xt_cap, nl2);
      B2_CUDA_TRY(raise_smem_limit((const void*)kern, sm_c));
      cudaLaunchConfig_t cfg{};
      cfg.gridDim = dim3(h->NG * sc);
      cfg.blockDim = dim3(kThreads);
      cfg.dynamicSmemBytes = sm_c;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = sc;
      at[0].val.clusterDim.y = 1;
      at[0].val.clusterDim.z = 1;
      cfg.attrs = at;
      cfg.numAttrs = 1;
      int ncl = 0;
      if (cudaOccupancyMaxActiveClusters(&ncl, kern, &cfg) == cudaSuccess && ncl >= h->NG) {  // one wave
        cluster = true;
        S = sc;
        nst_log2 = nl2;
      } else {
        (void)cudaGetLastError();
        sc >>= 1;
      }
    }
  }
  const int unit_tiles = ((quanta + S - 1) / S) * gt;
  int xt = unit_tiles < xt_cap ? unit_tiles : xt_cap;
  xt = (xt + xq - 1) / xq * xq;
  pl.S = S;
  pl.xt = xt;
  pl.nst_log2 = nst_log2;
  pl.cluster = cluster;
  pl.smem = smem_for(xt, nst_log2);
  pl.quanta = quanta;
  pl.valid = true;
  return B2_OK;
}

extern "C" {

int b2_gemm_wq_create(b2_gemm_wq_t* out, const b2_gemm_wq_desc* d) {
  if (!out || !d) return B2_ERR_PARAM;
  if (d->K <= 0 || d->N <= 0 || d->max_m <= 0) return B2_ERR_PARAM;
  if (d->wbits != 4 && d->wbits != 8 && d->wbits != 16) return B2_ERR_PARAM;
  if (d->ft != B2_DT_BF16 && d->ft != B2_DT_F16) return B2_ERR_UNSUPPORTED;
  if (d->wbits == 4 && d->qtype != B2_DT_U8) return B2_ERR_PARAM;  // gemm_a16w4.cpp:104-110: uint8(uint4x2) only
  if (d->wbits == 8 && d->qtype != B2_DT_U8 && d->qtype != B2_DT_I8) return B2_ERR_PARAM;
  if (d->K % 8 != 0) return B2_ERR_UNSUPPORTED;
  bool general_groups = false;  // group sizes that do not divide the 64-k tile (reference: any multiple of 8 >= 32 through its
                                // dequantize + cuBLAS path, gemm_a16w4.cpp:57-63): int4 only, wgmma kernel at every batch
  if (d->wbits != 16 && d->group_size != -1) {
    if (d->group_size <= 0) return B2_ERR_UNSUPPORTED;
    if (d->group_size % kBK != 0) {
      if (d->wbits != 4 || d->group_size % 8 != 0 || d->group_size < 32 || d->reserved == 1) return B2_ERR_UNSUPPORTED;
      general_groups = true;
    }
  }
  b2_gemm_wq* h = new (std::nothrow) b2_gemm_wq();
  if (!h) return B2_ERR_RUNTIME;
  h->d = *d;
  const bool grouped = d->wbits != 16 && d->group_size != -1;
  const int kq = (grouped && !general_groups) ? d->group_size : kBK;
  h->Kp = (d->K + kq - 1) / kq * kq;
  h->pair = d->reserved == 1;
  h->Np = h->pair ? (d->N + 63) / 64 * kBN : (d->N + kBN - 1) / kBN * kBN;  // pair: 64 gate + 64 up channels per tile
  h->KT = h->Kp / kBK;
  h->NG = h->Np / kBN;
  h->group_tiles = (grouped && !general_groups) ? d->group_size / kBK : 0;
  h->group_k = general_groups ? d->group_size : 0;
  h->G = grouped ? (general_groups ? (d->K + d->group_size - 1) / d->group_size : h->Kp / d->group_size) : 1;
  h->packed_bytes = (size_t)h->NG * h->KT * with_wbits(d->wbits, [](auto W) { return Image<W>::kTileBytes; });
  cudaGetDevice(&h->device);
  cudaError_t e = cudaMalloc(&h->counters, sizeof(unsigned) * h->NG);
  if (e == cudaSuccess) e = cudaMemset(h->counters, 0, sizeof(unsigned) * h->NG);
  if (e != cudaSuccess) {
    set_last_error("b2_gemm_wq_create", e);
    delete h;
    return B2_ERR_CUDA;
  }
  *out = h;
  return B2_OK;
}

int b2_gemm_wq_destroy(b2_gemm_wq_t h) {
  if (!h) return B2_OK;
  if (h->own_packed && h->packed) cudaFree(h->packed);
  if (h->own_sz && h->sz) cudaFree(h->sz);
  if (h->counters) cudaFree(h->counters);
  delete h;
  return B2_OK;
}

size_t b2_gemm_wq_packed_bytes(b2_gemm_wq_t h) { return h ? h->packed_bytes : 0; }

static int prepare_impl(b2_gemm_wq_t h, const void* qdata, const void* scales, const void* zeros, const void* qdata2,
                        const void* scales2, const void* zeros2, void* packed_dst, void* stream_) {
  if (!h || !qdata) return B2_ERR_PARAM;
  cudaStream_t stream = (cudaStream_t)stream_;
  const b2_gemm_wq_desc& d = h->d;
  const int pair = h->pair ? 1 : 0;
  if (pair && !qdata2) return B2_ERR_PARAM;
  if (d.wbits != 16 && (!scales || !zeros || (pair && (!scales2 || !zeros2)))) return B2_ERR_PARAM;
  if (packed_dst) {
    if (h->own_packed && h->packed) cudaFree(h->packed);
    h->packed = packed_dst;
    h->own_packed = false;
  } else if (!h->packed || !h->own_packed) {
    B2_CUDA_TRY(cudaMalloc(&h->packed, h->packed_bytes));
    h->own_packed = true;
  }
  const int threads = 256;
  const int64_t words = (int64_t)h->packed_bytes / 4;
  const int blocks = (int)((words + threads - 1) / threads > 65535 * 8 ? 65535 * 8 : (words + threads - 1) / threads);
  with_wbits(d.wbits, [&](auto W) {
    pack_image_kernel<W><<<blocks, threads, 0, stream>>>((uint32_t*)h->packed, qdata, qdata2, pair, d.K, d.N, h->KT, h->NG,
                                                         d.qtype == B2_DT_I8);
  });
  if (int st = launch_failed("pack_weights")) return st;
  if (d.wbits != 16) {
    if (!h->sz || !h->own_sz) {
      B2_CUDA_TRY(cudaMalloc(&h->sz, sizeof(float2) * (size_t)h->G * h->Np));
      h->own_sz = true;
    }
    // 16+q trick: W4 raw = sum a*(16+q); W8 raw = 16*sum a*(16+hi) + sum a*(16+lo) = sum a*(272+u), u = q (+128 if int8)
    // (fp16 handles: 128 + q, so 128 and 17 * 128 = 2176)
    const float b0 = d.ft == B2_DT_F16 ? 128.f : 16.f;
    const float zbias = d.wbits == 4 ? b0 : (d.qtype == B2_DT_I8 ? 17.f * b0 + 128.f : 17.f * b0);
    const int64_t tot = (int64_t)h->G * h->Np;
    pack_sz_kernel<<<(int)((tot + 255) / 256), 256, 0, stream>>>(h->sz, (const __nv_bfloat16*)scales, (const __nv_bfloat16*)zeros,
                                                                 (const __nv_bfloat16*)scales2, (const __nv_bfloat16*)zeros2, pair,
                                                                 h->G, d.N, h->Np, zbias, d.ft == B2_DT_F16 ? 1 : 0);
    if (int st = launch_failed("pack_sz")) return st;
  }
  return B2_OK;
}

int b2_gemm_wq_prepare_weights(b2_gemm_wq_t h, const void* qdata, const void* scales, const void* zeros,
                               void* packed_dst, void* stream_) {
  if (h && h->pair) return B2_ERR_PARAM;  // a paired handle takes two weight sets (b2_gemm_wq_prepare_swiglu)
  return prepare_impl(h, qdata, scales, zeros, nullptr, nullptr, nullptr, packed_dst, stream_);
}

int b2_gemm_wq_prepare_swiglu(b2_gemm_wq_t h, const void* q_gate, const void* s_gate, const void* z_gate, const void* q_up,
                              const void* s_up, const void* z_up, void* stream_) {
  if (!h || !h->pair) return B2_ERR_PARAM;
  return prepare_impl(h, q_gate, s_gate, z_gate, q_up, s_up, z_up, nullptr, stream_);
}

int b2_gemm_wq_attach_packed(b2_gemm_wq_t h, const void* packed, const void* scales_f32, const void* zeros_f32) {
  (void)zeros_f32;
  if (!h || !packed) return B2_ERR_PARAM;
  if (h->own_packed && h->packed) cudaFree(h->packed);
  h->packed = const_cast<void*>(packed);
  h->own_packed = false;
  if (scales_f32) {
    if (h->own_sz && h->sz) cudaFree(h->sz);
    h->sz = (float2*)const_cast<void*>(scales_f32);
    h->own_sz = false;
  }
  return B2_OK;
}

static int mt_index_for(int M) { return M <= 8 ? 0 : 1; }

// Batches from kTcMinM up take the wgmma kernel: int4 / int8 per-channel, dense bf16 (lm_head), and int4 sub-channel (the scale
// is applied to the weights in the dequant warps).  Sub-channel int8 weights have no wgmma path yet: at M > 16 they run on the
// mma.sync kernel in passes of kGemvMaxM rows (MT = 2, two CTAs per SM) and stream the weights once per pass.
constexpr int kTcMinM = 17;

static bool use_tc(const b2_gemm_wq* h, int M) {
  if (h->group_k > 0) return true;  // general group sizes exist on the wgmma kernel only
  return M >= kTcMinM && (h->group_tiles == 0 || h->d.wbits == 4);
}

// The wgmma path's schedule (TcSched), once per handle.  At most as many n-groups as SMs: S = min(SMs / n-groups, KT / 4,
// B2_GEMM_TC_MAX_SPLIT) equal k-slices per n-group, one CTA each (B2_GEMM_TC_PERSIST=0: also above that, S = 1).  More
// n-groups than SMs: one CTA per SM, whole n-groups in rounds, and the NR left over each cut in two at a multiple of 4 k-tiles
// near KT / 2, a head on CTA b < NR and a tail on CTA NR + b: the gate+up pair's 296 n-groups (132 SMs) run 2 rounds plus
// 28 tiles on 64 CTAs instead of 3 rounds on 32.  The tail continues the head's accumulator chain, so the results are those
// of whole n-groups bit for bit.  B2_GEMM_TC_MAX_SPLIT=1 splits no n-group.
static void make_tc_plan(b2_gemm_wq* h) {
  if (h->tc_grid > 0) return;
  const int sms = sm_count(), NG = h->NG, KT = h->KT;
  const int smax = std::max(1, env_int("B2_GEMM_TC_MAX_SPLIT", 6));
  if (NG <= sms || !env_int("B2_GEMM_TC_PERSIST", 1)) {
    h->tc_S = std::max(1, std::min({sms / NG, KT / 4, smax}));
    h->tc_grid = NG * h->tc_S;
    h->tc_rounds = 0;
    h->tc_h = 0;
    return;
  }
  const int NR = NG % sms;
  h->tc_S = 1;
  h->tc_grid = sms;
  h->tc_rounds = NG / sms;
  h->tc_h = (NR > 0 && smax > 1 && 2 * NR <= sms) ? KT / 2 / 4 * 4 : 0;
}

// workspace of the wgmma path: the k-slices' partial tiles, or the parked heads, of one launch (kTcMaxM rows)
static size_t tc_workspace_bytes(b2_gemm_wq* h) {
  make_tc_plan(h);
  if (h->tc_S > 1) return (size_t)h->NG * h->tc_S * kTcMaxM * kBN * sizeof(float) + 16;
  if (h->tc_h > 0) return (size_t)(h->NG - h->tc_rounds * h->tc_grid) * kTcCarryFloats * sizeof(float) + 16;
  return 16;
}

// The wgmma kernel over M rows, kTcMaxM per launch.  p holds the caller's operands for row 0 (A, C, residual and the per-row
// fp8 / RMSNorm arrays, offset here for every launch); the image, its params and the split-K plan come from the handle.
static int run_tc(b2_gemm_wq* h, TcParams p, int M, cudaStream_t stream) {
  make_tc_plan(h);
  if ((h->tc_S > 1 || h->tc_h > 0) && !p.ws) return B2_ERR_PARAM;
  p.packed = (const uint8_t*)h->packed; p.sz = h->sz; p.counters = h->counters;
  p.N = h->d.N; p.K = h->d.K; p.Np = h->Np; p.KT = h->KT; p.NG = h->NG;
  p.grid = h->tc_grid; p.rounds = h->tc_rounds; p.S = h->tc_S; p.h = h->tc_h;
  const int64_t a_row = p.a_scale ? p.lda : 2 * p.lda;  // bytes per activation row (fp8: lda counts bytes)
  for (int m0 = 0; m0 < M; m0 += kTcMaxM) {
    TcParams q = p;
    q.M = (M - m0) > kTcMaxM ? kTcMaxM : (M - m0);
    q.A = reinterpret_cast<const __nv_bfloat16*>(reinterpret_cast<const uint8_t*>(p.A) + m0 * a_row);
    q.C = p.C + (int64_t)m0 * p.ldc;
    if (p.residual) q.residual = p.residual + (int64_t)m0 * p.ldc;
    if (p.a_scale) {
      q.a_scale = p.a_scale + m0;
      q.tile_sums = p.tile_sums + (size_t)m0 * p.KT;
    }
    if (p.norm_sumsq) q.norm_sumsq = p.norm_sumsq + m0;
    if (p.xg_out) {
      q.sumsq_out = p.sumsq_out + m0;
      q.xg_out = p.xg_out + (int64_t)m0 * p.ldxg;
    }
    cudaError_t e = tc_launch(h->d.wbits, h->d.ft == B2_DT_F16, q, stream);
    if (e != cudaSuccess) {
      set_last_error(p.a_scale ? "wq_gemm_tc (fp8) launch" : "wq_gemm_tc launch", e);
      return B2_ERR_CUDA;
    }
  }
  return B2_OK;
}

size_t b2_gemm_wq_workspace_bytes(b2_gemm_wq_t h, int M) {
  if (!h || M <= 0) return 0;
  if (use_tc(h, M)) return tc_workspace_bytes(h);
  const int mc = M > kGemvMaxM ? kGemvMaxM : M;
  const int mti = mt_index_for(mc);
  if (make_plan(h, mti) != B2_OK) return 0;
  const Plan& pl = h->plans[mti];
  if (pl.S <= 1 || pl.cluster) return 16;
  return (size_t)h->NG * pl.S * (8 << mti) * (kBN + 1) * sizeof(float) + 16;  // partial tiles + per-slice sum x^2
}

size_t b2_gemm_wq_algo_bytes(b2_gemm_wq_t h, int M) {
  if (!h) return 0;
  const b2_gemm_wq_desc& d = h->d;
  const size_t mul = h->pair ? 2 : 1;
  size_t w = mul * (size_t)d.K * d.N * d.wbits / 8;
  size_t prm = d.wbits == 16 ? 0 : mul * (size_t)2 * 2 * h->G * d.N;
  return w + prm + (size_t)2 * M * ((size_t)d.K + d.N);
}

int b2_gemm_wq_sumsq_parts(b2_gemm_wq_t h) { return h ? h->NG : 0; }

int b2_gemm_wq_run(b2_gemm_wq_t h, const void* A, int64_t lda, void* C, int64_t ldc, int M, const void* bias,
                   const void* residual, int activation, float alpha, void* workspace, size_t workspace_bytes,
                   void* stream_) {
  return b2_gemm_wq_run_fused(h, A, lda, C, ldc, M, bias, residual, activation, alpha, workspace, workspace_bytes, nullptr, stream_);
}

extern "C" const void* b2_comm_device_view(b2_comm_t c);

static int run_impl(b2_gemm_wq_t h, const void* A, int64_t lda, void* C, int64_t ldc, int M, const void* bias,
                    const void* residual, int activation, float alpha, void* workspace, size_t workspace_bytes,
                    const b2_gemm_fuse* fuse, const CommDev* comm, void* stream_);

int b2_gemm_wq_run_fused(b2_gemm_wq_t h, const void* A, int64_t lda, void* C, int64_t ldc, int M, const void* bias,
                         const void* residual, int activation, float alpha, void* workspace, size_t workspace_bytes,
                         const b2_gemm_fuse* fuse, void* stream_) {
  return run_impl(h, A, lda, C, ldc, M, bias, residual, activation, alpha, workspace, workspace_bytes, fuse, nullptr, stream_);
}

int b2_gemm_wq_run_fp8(b2_gemm_wq_t h, const void* A8, int64_t lda_bytes, const float* a_scale, const float* tile_sums, void* C,
                       int64_t ldc, int M, const void* bias, const void* residual, int activation, float alpha, void* workspace,
                       size_t workspace_bytes, void* stream_) {
  if (!h || !A8 || !a_scale || !tile_sums || !C || M <= 0) return B2_ERR_PARAM;
  if (!h->packed) return B2_ERR_RUNTIME;
  if (M > h->d.max_m) return B2_ERR_LIMIT;
  if (h->d.wbits != 4 || h->group_tiles > 0 || h->group_k > 0 || h->d.ft != B2_DT_BF16) return B2_ERR_UNSUPPORTED;  // int4 per-channel weights (the IQ default), bf16 outputs
  if (h->pair != (activation == B2_ACT_SWIGLU)) return B2_ERR_PARAM;
  if (activation != B2_ACT_SWIGLU && (activation < 0 || activation > B2_ACT_SIGMOID)) return B2_ERR_PARAM;
  if (h->pair && (bias || residual)) return B2_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(A8) & 15) || (lda_bytes % 16) != 0 || lda_bytes < h->d.K) return B2_ERR_UNSUPPORTED;
  if (workspace_bytes < tc_workspace_bytes(h)) return B2_ERR_PARAM;
  TcParams p;
  p.A = (const __nv_bfloat16*)A8; p.lda = lda_bytes;
  p.C = (__nv_bfloat16*)C; p.ldc = ldc;
  p.bias = (const __nv_bfloat16*)bias;
  p.residual = (const __nv_bfloat16*)residual;
  p.ws = (float*)workspace;
  p.act = activation; p.alpha = alpha;
  p.a_scale = a_scale; p.tile_sums = tile_sums;
  return run_tc(h, p, M, (cudaStream_t)stream_);
}

int b2_gemm_wq_run_allreduce(b2_gemm_wq_t h, const void* A, int64_t lda, void* C, int64_t ldc, int M, const void* bias,
                             const void* residual, float alpha, void* workspace, size_t workspace_bytes, b2_comm_t comm,
                             void* stream_) {
  const CommDev* cd = static_cast<const CommDev*>(b2_comm_device_view(comm));
  if (!h || !cd) return B2_ERR_PARAM;
  for (int r = 0; r < cd->nranks; ++r)
    if (!cd->peer[r]) return B2_ERR_RUNTIME;  // communicator not connected
  // the GEMV path only (one launch, M <= 16), even N, plain [M, N] output, every tile has a flag, payload fits a slot
  if (M > 16 || h->pair || (h->d.N & 1) || ldc != h->d.N || h->NG > kCommMaxChunks) return B2_ERR_UNSUPPORTED;
  if ((size_t)M * h->d.N * 2 > cd->max_bytes) return B2_ERR_LIMIT;
  if (((uintptr_t)C & 3) || (residual && ((uintptr_t)residual & 3))) return B2_ERR_UNSUPPORTED;
  return run_impl(h, A, lda, C, ldc, M, bias, residual, B2_ACT_NONE, alpha, workspace, workspace_bytes, nullptr, cd, stream_);
}

static int run_impl(b2_gemm_wq_t h, const void* A, int64_t lda, void* C, int64_t ldc, int M, const void* bias,
                    const void* residual, int activation, float alpha, void* workspace, size_t workspace_bytes,
                    const b2_gemm_fuse* fuse, const CommDev* comm, void* stream_) {
  if (!h || !A || !C || M <= 0) return B2_ERR_PARAM;
  const bool tc = use_tc(h, M) && !comm;  // wgmma path, 64 rows per launch (else the mma.sync GEMV, 16 rows per launch)
  // ---- RMSNorm fusion: the fields of b2_gemm_fuse that are set name one of two forms, each checked here once; every other
  //      combination is B2_ERR_UNSUPPORTED.
  //        self-contained: norm_gamma alone, on the mma.sync GEMV (M <= 16)
  //        hand-off, on the wgmma path: consumer norm_sumsq (no norm_gamma) and / or producer xg_out + sumsq_out + gamma_out
  bool norm_self = false, handoff = false;
  if (fuse) {
    const bool cons = fuse->norm_sumsq != nullptr, prod = fuse->xg_out != nullptr;
    norm_self = fuse->norm_gamma && !cons;
    handoff = cons || prod || fuse->sumsq_out;
    if (norm_self) {
      if (tc || M > kGemvMaxM || handoff) return B2_ERR_UNSUPPORTED;
      if (fuse->norm_hidden != h->d.K) return B2_ERR_PARAM;  // the row statistics span exactly this GEMM's K
      if (reinterpret_cast<uintptr_t>(fuse->norm_gamma) & 15) return B2_ERR_UNSUPPORTED;  // bulk-copied by slices
    } else if (handoff) {
      if (!tc || fuse->norm_gamma || (fuse->sumsq_out && !prod)) return B2_ERR_UNSUPPORTED;
      if (cons && (fuse->norm_parts <= 0 || fuse->norm_hidden <= 0)) return B2_ERR_PARAM;
      if (prod) {
        if (!fuse->sumsq_out || !fuse->gamma_out || h->pair || activation != B2_ACT_NONE) return B2_ERR_PARAM;
        // the statistics come out of the vectorised residual epilogue: 8-byte aligned rows everywhere
        if ((h->d.N & 3) || (ldc & 3) || (fuse->ldxg & 3) || (reinterpret_cast<uintptr_t>(C) & 7) ||
            (reinterpret_cast<uintptr_t>(fuse->xg_out) & 7) || (reinterpret_cast<uintptr_t>(fuse->gamma_out) & 7) ||
            (residual && (reinterpret_cast<uintptr_t>(residual) & 7)) || (bias && (reinterpret_cast<uintptr_t>(bias) & 7)))
          return B2_ERR_UNSUPPORTED;
      }
    }
  }
  if (!h->packed) return B2_ERR_RUNTIME;
  if (M > h->d.max_m) return B2_ERR_LIMIT;
  if (h->group_k > 0 && comm) return B2_ERR_UNSUPPORTED;
  if (h->pair != (activation == B2_ACT_SWIGLU)) return B2_ERR_PARAM;  // paired image <=> SwiGLU epilogue
  if (activation != B2_ACT_SWIGLU && (activation < 0 || activation > B2_ACT_SIGMOID)) return B2_ERR_PARAM;
  if (h->pair && (bias || residual)) return B2_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(A) & 15) || (lda % 8) != 0) return B2_ERR_UNSUPPORTED;
  if (workspace_bytes < b2_gemm_wq_workspace_bytes(h, M)) return B2_ERR_PARAM;
  cudaStream_t stream = (cudaStream_t)stream_;
  const bool grouped = h->group_tiles > 0;
  if (tc) {
    TcParams p;
    p.A = (const __nv_bfloat16*)A; p.lda = lda;
    p.C = (__nv_bfloat16*)C; p.ldc = ldc;
    p.bias = (const __nv_bfloat16*)bias;
    p.residual = (const __nv_bfloat16*)residual;
    p.ws = (float*)workspace;
    p.act = activation; p.alpha = alpha;
    p.group_tiles = h->group_tiles;
    p.group_k = h->group_k; p.ngroups = h->G;
    if (handoff) {
      p.norm_ld = M;
      if (fuse->norm_sumsq) {
        p.norm_sumsq = fuse->norm_sumsq; p.norm_parts = fuse->norm_parts;
        p.norm_inv_hidden = 1.0f / (float)fuse->norm_hidden; p.norm_eps = fuse->norm_eps;
      }
      if (fuse->xg_out) {
        p.sumsq_out = fuse->sumsq_out;
        p.xg_out = (__nv_bfloat16*)fuse->xg_out;
        p.gamma_out = (const __nv_bfloat16*)fuse->gamma_out; p.ldxg = fuse->ldxg;
      }
    }
    return run_tc(h, p, M, stream);
  }
  // ---- dense bf16 weights at batches <= 16: no global split-K (wq_gemv2.cu), unless a fusion only the split-K kernel
  //      implements is asked for (fp16 handles: the split-K kernel)
  if (h->d.wbits == 16 && M <= kGemvMaxM && !norm_self && !comm && h->d.ft == B2_DT_BF16) {
    Gemv2Params p;
    p.packed = (const uint8_t*)h->packed;
    p.A = (const __nv_bfloat16*)A; p.lda = lda;
    p.C = (__nv_bfloat16*)C; p.ldc = ldc;
    p.bias = (const __nv_bfloat16*)bias;
    p.residual = (const __nv_bfloat16*)residual;
    p.M = M; p.N = h->d.N; p.K = h->d.K; p.KT = h->KT; p.NG = h->NG;
    p.pair = h->pair ? 1 : 0; p.act = activation; p.alpha = alpha;
    Gemv2Plan pl;
    if (gemv2_plan(p, &pl)) {
      cudaError_t e = gemv2_launch(p, pl, stream);
      if (e != cudaSuccess) {
        set_last_error("wq_gemv2 launch", e);
        return B2_ERR_CUDA;
      }
      return B2_OK;
    }
  }
  for (int m0 = 0; m0 < M; m0 += kGemvMaxM) {
    const int mc = (M - m0) > kGemvMaxM ? kGemvMaxM : (M - m0);
    const int mti = mt_index_for(mc);
    if (int st = make_plan(h, mti)) return st;
    const Plan& pl = h->plans[mti];
    if (pl.S > 1 && !pl.cluster && !workspace) return B2_ERR_PARAM;
    GemmParams p;
    p.packed = (const uint8_t*)h->packed;
    p.sz = h->sz;
    p.A = (const __nv_bfloat16*)A + (int64_t)m0 * lda;
    p.lda = lda;
    p.C = (__nv_bfloat16*)C + (int64_t)m0 * ldc;
    p.ldc = ldc;
    p.bias = (const __nv_bfloat16*)bias;
    p.residual = residual ? (const __nv_bfloat16*)residual + (int64_t)m0 * ldc : nullptr;
    p.ws = (float*)workspace;
    p.counters = h->counters;
    p.M = mc; p.N = h->d.N; p.K = h->d.K; p.Np = h->Np; p.KT = h->KT; p.NG = h->NG; p.S = pl.S;
    p.group_tiles = h->group_tiles;
    p.quanta = pl.quanta;
    p.xt = pl.xt;
    p.nst_log2 = pl.nst_log2;
    p.act = activation;
    p.alpha = alpha;
    p.cluster = pl.cluster ? 1 : 0;
    p.norm_self = norm_self ? 1 : 0;
    p.norm_gamma = norm_self ? (const __nv_bfloat16*)fuse->norm_gamma : nullptr;
    p.norm_inv_hidden = norm_self ? 1.0f / (float)fuse->norm_hidden : 0.f;
    p.norm_eps = norm_self ? fuse->norm_eps : 0.f;
    p.comm_on = comm ? 1 : 0;
    if (comm) p.comm = *comm;
    else memset(&p.comm, 0, sizeof(p.comm));
    gemm_kernel_t kern = pick_kernel(h->d.wbits, grouped, 1 << mti, h->d.ft == B2_DT_F16);
    cudaError_t e = pl.cluster ? launch_cluster(kern, dim3(h->NG * pl.S), dim3(kThreads), (size_t)pl.smem, stream, true, (unsigned)pl.S, p)
                               : launch(kern, dim3(h->NG * pl.S), dim3(kThreads), (size_t)pl.smem, stream, true, p);
    if (e != cudaSuccess) {
      set_last_error("wq_gemm launch", e);
      return B2_ERR_CUDA;
    }
  }
  return B2_OK;
}

}  // extern "C"
