// b200spark — weight-only quantized GEMV/GEMM for decode batches 1..16 (per-channel and sub-channel) WITHOUT global split-K,
// sm_90a.  Same weight image, same tensor-core math and the same results (up to fp32 summation order) as wq_gemm.cu.
//
// Why a second decomposition: at batch 1 most of the split-K kernel's time after the weight stream is its split-K tail —
// partials to the workspace, __threadfence, atomic ticket, waiting for the sibling CTAs, re-reading the partial tiles from
// L2.  A 16-way K split across CTAs is what it takes to fill 132 SMs with 128-channel tiles of a 4608-channel
// projection, so the split has to move INSIDE the CTA:
//
//   * a CTA owns CB in {128, 64, 32, 16} output channels of one 128-channel n-group and the FULL K range;
//     grid = N / CB CTAs (CB is chosen so that the grid covers the SMs at least ~1.5 times);
//   * its 8 consumer warps form WN = CB/16 n16-tiles x WK = 128/CB k-slices; a pipeline stage carries WK quanta of q k-tiles
//     (q = 2, or one quantization group) and warp (wn, wk) takes quantum wk of every stage — all warps always work on the
//     stage that just landed, and a sub-channel group is never split between warps;
//   * the producer lane fetches a whole stage with ONE TMA tensor request: the tile image is described as a 4-D tensor
//     [tile][chunk][half: rows 0-63 | 64-127][64 rows x 16 B] and the CTA's box is {its rows, 1 or 2 halves, all chunks, the
//     stage's tiles} (a gate/up pair image takes the 16 gate rows and the 16 matching up rows with the half dimension) —
//     the TMA unit spends ~46 clocks per REQUEST whatever its size, so row-run bulk copies of 256 B could not exceed 10 GB/s
//     per SM (measured: 83 us for down_proj).  Issued ahead of the previous kernel's completion (PDL);
//   * the WK partial accumulators meet in shared memory (fixed order => deterministic): no workspace, no fence, no atomics,
//     no second wave of L2 reads.  The dequantisation s * (acc - (16+z) * sum a) is linear, so it is applied once, after
//     the k-slices are summed.
//   * only the M live batch rows are staged (the split-K kernel zero-fills all 8 / 16 rows of the MMA's n side).
//
// Roofline: HBM-bound; algorithmic bytes/launch = K*N*wbits/8 + 4*G*N + 2*M*(K+N).
#include <cuda.h>  // CUtensorMap (types only; the encoder is fetched with cudaGetDriverEntryPoint)

#include <cstdlib>

#include "b2_common.cuh"
#include "wq_gemm_shared.cuh"

namespace b2 {

constexpr int kV2Warps = 8;
constexpr int kV2Threads = kV2Warps * 32 + 32;  // + producer warp

struct Gemv2Params {
  const uint8_t* packed;
  const float2* sz;  // [G][Np] (scale, zero + bias-constant)
  const __nv_bfloat16* A;
  int64_t lda;
  __nv_bfloat16* C;
  int64_t ldc;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* residual;
  int M, N, K, Np, KT, NG;
  int cb_log2;      // log2(CB)
  int q;            // k-tiles per quantum (= per warp per stage): 2, or the quantization group in tiles
  int grouped_gt;   // k-tiles per quantization group (GROUPED) else 0
  int xt;           // k-tiles per activation chunk (multiple of the stage: WK * q)
  int nst_log2;     // log2(pipeline stages)
  int pair;         // gate/up pair image (SwiGLU epilogue)
  int act;
  float alpha;
};

__device__ __forceinline__ void v2_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// One k-tile (64 k x 16 n) of tensor-core work for this warp.  woff0/woff1: byte offsets of this thread's row g / g+8
// inside the CTA's sub-tile [chunk][CB rows][16 B] (CS = CB * 16 bytes per chunk); xaddr: this thread's 32 bytes of
// activations of batch row g (16 consecutive k); live[m]: batch row g + 8m exists.
template <int WBITS, int MT>
__device__ __forceinline__ void v2_tile_mma(float (&acc)[MT][4], uint32_t wtile, uint32_t woff0, uint32_t woff1, uint32_t CS,
                                            uint32_t xaddr, int XS8, const bool (&live)[MT]) {
  uint4 xb[MT][2];
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    if (live[m]) {
      xb[m][0] = lds128(xaddr + m * XS8);
      xb[m][1] = lds128(xaddr + m * XS8 + 16);
    } else {
      xb[m][0] = xb[m][1] = make_uint4(0u, 0u, 0u, 0u);
    }
  }
  if (WBITS == 4) {
    const uint2 w0 = lds64(wtile + woff0), w1 = lds64(wtile + woff1);
    const uint32_t r0w[2] = {w0.x, w0.y}, r1w[2] = {w1.x, w1.y};
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const uint32_t u = r0w[j], v = r1w[j];
      const uint32_t p0 = lop3_and_or(u, kMask4, kMagic), q0 = lop3_and_or(v, kMask4, kMagic);
      const uint32_t p1 = lop3_and_or(__funnelshift_r(u, u, 4), kMask4, kMagic), q1 = lop3_and_or(__funnelshift_r(v, v, 4), kMask4, kMagic);
      const uint32_t p2 = lop3_and_or(__funnelshift_r(u, u, 8), kMask4, kMagic), q2 = lop3_and_or(__funnelshift_r(v, v, 8), kMask4, kMagic);
      const uint32_t p3 = lop3_and_or(__funnelshift_r(u, u, 12), kMask4, kMagic), q3 = lop3_and_or(__funnelshift_r(v, v, 12), kMask4, kMagic);
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        mma_bf16_16816(acc[m], p0, q0, p1, q1, xb[m][j].x, xb[m][j].y);
        mma_bf16_16816(acc[m], p2, q2, p3, q3, xb[m][j].z, xb[m][j].w);
      }
    }
  } else if (WBITS == 8) {
    const uint4 w0 = lds128(wtile + woff0), w1 = lds128(wtile + woff1);
    const uint32_t r0w[4] = {w0.x, w0.y, w0.z, w0.w}, r1w[4] = {w1.x, w1.y, w1.z, w1.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t u = r0w[j], v = r1w[j];
      const uint32_t l0 = lop3_and_or(u, kMask4, kMagic), m0 = lop3_and_or(v, kMask4, kMagic);
      const uint32_t h0 = lop3_and_or(__funnelshift_r(u, u, 4), kMask4, kMagicHi), n0 = lop3_and_or(__funnelshift_r(v, v, 4), kMask4, kMagicHi);
      const uint32_t l1 = lop3_and_or(__funnelshift_r(u, u, 8), kMask4, kMagic), m1 = lop3_and_or(__funnelshift_r(v, v, 8), kMask4, kMagic);
      const uint32_t h1 = lop3_and_or(__funnelshift_r(u, u, 12), kMask4, kMagicHi), n1 = lop3_and_or(__funnelshift_r(v, v, 12), kMask4, kMagicHi);
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        const uint32_t b0 = (j & 1) ? xb[m][j >> 1].z : xb[m][j >> 1].x;
        const uint32_t b1 = (j & 1) ? xb[m][j >> 1].w : xb[m][j >> 1].y;
        mma_bf16_16816(acc[m], l0, m0, l1, m1, b0, b1);   // low nibbles:  16 + lo
        mma_bf16_16816(acc[m], h0, n0, h1, n1, b0, b1);   // high nibbles: 16 * (16 + hi)
      }
    }
  } else {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const uint4 w0 = lds128(wtile + woff0 + u * CS), w1 = lds128(wtile + woff1 + u * CS);
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        mma_bf16_16816(acc[m], w0.x, w1.x, w0.y, w1.y, xb[m][u].x, xb[m][u].y);
        mma_bf16_16816(acc[m], w0.z, w1.z, w0.w, w1.w, xb[m][u].z, xb[m][u].w);
      }
    }
  }
}

template <int WBITS, int MT, bool GROUPED>
__global__ void __launch_bounds__(kV2Threads) wq_gemv2_kernel(const Gemv2Params p, const __grid_constant__ CUtensorMap wmap) {
  constexpr int MP = 8 * MT;
  constexpr int NCH = WBITS == 4 ? 2 : (WBITS == 8 ? 4 : 8);        // 16-byte chunks per row per k-tile
  constexpr int TILE_BYTES = 128 * NCH * 16;                        // one (128 n x 64 k) tile of the image
  const int NST = 1 << p.nst_log2;
  const int CB = 1 << p.cb_log2;                                    // channels (image rows) of this CTA
  const int SUBS = kBN >> p.cb_log2;                                // CTAs per n-group == k-slices per CTA (WK)
  const int WK = SUBS, WN = CB >> 4;
  const uint32_t CS = (uint32_t)CB * 16u;                           // bytes per chunk of the CTA's sub-tile
  const int sub_tile_bytes = NCH * (int)CS;                         // bytes per k-tile in shared memory
  const int stage_tiles = WK * p.q;
  const int stage_bytes = stage_tiles * sub_tile_bytes;             // == q * TILE_BYTES
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int ng = blockIdx.x / SUBS, sub = blockIdx.x - ng * SUBS;

  // ---- shared memory carve-up
  uint8_t* ring = smem;
  const int XS = p.xt * 128 + 16;                                   // activation row stride (bytes), == 16 mod 128
  uint8_t* xs = ring + NST * stage_bytes;
  float* fs2 = reinterpret_cast<float*>(xs + MP * XS);              // [WK][MP][CB] partial tiles of the k-slices
  const int gpc = GROUPED ? p.xt / p.grouped_gt : 1;                // quantization groups per activation chunk
  float* suma = fs2 + WK * MP * CB;                                 // [MP][gpc] (GROUPED) or [MP]
  uint64_t* full = reinterpret_cast<uint64_t*>((reinterpret_cast<uintptr_t>(suma + MP * gpc + 4) + 7) & ~uintptr_t(7));
  uint64_t* empty = full + NST;

  if (tid == 0) {
    for (int i = 0; i < NST; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], kV2Warps);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  const int nstages = (p.KT + stage_tiles - 1) / stage_tiles;
  // image rows of this CTA: plain: [sub*CB, +CB); pair: gate rows [sub*CB/2, +CB/2) and the matching up rows (+64)
  const int nruns = p.pair ? 2 : 1;
  const int run_rows = CB / nruns;

  if (warp == kV2Warps) {
    // ===================== producer: one tensor request per stage, independent of the previous kernel ==========
    if (lane == 0) {
      // box origin inside a tile: d0 = 8-byte element inside a 64-row half, d1 = half
      const int rows_per_half_box = p.pair ? run_rows : min(CB, 64);
      const int c0 = p.pair ? sub * run_rows * 2 : ((sub * CB) & 63) * 2;
      const int c1 = p.pair ? 0 : (sub * CB) >> 6;
      (void)rows_per_half_box;
      for (int i = 0; i < nstages; ++i) {
        const int slot = i & (NST - 1);
        if (i >= NST) mbar_wait(&empty[slot], ((i >> p.nst_log2) & 1) ^ 1);
        // the box always has stage_tiles tiles: tiles past this n-group's K range belong to the next n-group (or are
        // zero-filled past the end of the image) and are simply not consumed
        mbar_arrive_expect_tx(&full[slot], (uint32_t)stage_bytes);
        asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
                     ::"r"(smem_u32(ring + (size_t)slot * stage_bytes)), "l"(reinterpret_cast<uint64_t>(&wmap)), "r"(c0), "r"(c1), "r"(0),
                       "r"(ng * p.KT + i * stage_tiles), "r"(smem_u32(&full[slot]))
                     : "memory");
      }
    }
    return;
  }

  // ===================== consumers =====================
  const int wn = warp % WN, wk = warp / WN;
  const int lr0 = wn * 16 + g, lr1 = lr0 + 8;                       // this thread's rows inside the CTA's sub-tile
  // physical row (position in the 128-row image tile) of a local row: scale/zero are stored per physical row
  auto phys = [&](int lr) { return p.pair ? (lr < run_rows ? sub * run_rows + lr : 64 + sub * run_rows + (lr - run_rows)) : sub * CB + lr; };
  const int pr0 = ng * kBN + phys(lr0), pr1 = ng * kBN + phys(lr1);
  float2 sz0 = make_float2(1.f, 0.f), sz1 = make_float2(1.f, 0.f);
  if (GROUPED) {
    // consumed at every group end
  }

  float acc[MT][4], facc[MT][4];
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[m][c] = facc[m][c] = 0.f;
  bool live[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) live[m] = (g + 8 * m) < p.M;

  pdl_wait();  // activations belong to the previous kernel from here on

  const uint32_t w_ring = smem_u32(ring);
  const int wc = WBITS == 4 ? (t >> 1) : (WBITS == 8 ? t : 2 * t);
  // the image stores row r of chunk c at r ^ swz(c): swz < 8 and the CTA's row runs are 16-aligned, so the XOR stays local
  const uint32_t woff0 = wc * CS + ((lr0 ^ tile_swz(WBITS, wc)) << 4) + (WBITS == 4 ? 8 * (t & 1) : 0);
  const uint32_t woff1 = wc * CS + ((lr1 ^ tile_swz(WBITS, wc)) << 4) + (WBITS == 4 ? 8 * (t & 1) : 0);
  const uint32_t x_thr = smem_u32(xs) + g * XS + t * 32;
  const int XS8 = 8 * XS;
  int stage_i = 0;

  for (int xc0 = 0; xc0 < p.KT; xc0 += p.xt) {   // p.xt is a multiple of stage_tiles (and so of the quantization group)
    const int xn = min(p.xt, p.KT - xc0);
    if (xc0 > 0) v2_bar_sync(1, kV2Warps * 32);  // previous chunk fully consumed
    // ---- stage the M live activation rows of this k-chunk and their per-(row, group) sums (zero-point term)
    {
      const int64_t kbase = (int64_t)xc0 * kBK;
      const int nvec = xn * 8;
      const int gvec = GROUPED ? p.grouped_gt * 8 : nvec;  // 16-byte vectors per quantization group
      for (int m = warp; m < p.M; m += kV2Warps) {
        const __nv_bfloat16* arow = p.A + (int64_t)m * p.lda + kbase;
        uint8_t* xrow = xs + m * XS;
        for (int v0 = 0, gi = 0; v0 < nvec; v0 += gvec, ++gi) {
          float sacc = 0.f;
          for (int v = v0 + lane; v < v0 + gvec; v += 32) {
            uint4 val = make_uint4(0, 0, 0, 0);
            if (kbase + v * 8 < p.K) val = *reinterpret_cast<const uint4*>(arow + v * 8);
            *reinterpret_cast<uint4*>(xrow + v * 16) = val;
            sacc += (bf16_lo(val.x) + bf16_hi(val.x)) + (bf16_lo(val.y) + bf16_hi(val.y)) +
                    (bf16_lo(val.z) + bf16_hi(val.z)) + (bf16_lo(val.w) + bf16_hi(val.w));
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) sacc += __shfl_xor_sync(0xffffffffu, sacc, o);
          if (lane == 0) {
            if (GROUPED) suma[m * gpc + gi] = sacc;
            else suma[m] = (xc0 == 0 ? 0.f : suma[m]) + sacc;
          }
        }
      }
    }
    v2_bar_sync(1, kV2Warps * 32);

    // ---- main loop: one pipeline stage per iteration; this warp takes quantum wk of it
    for (int xs0 = 0; xs0 < xn; xs0 += stage_tiles, ++stage_i) {
      const int slot = stage_i & (NST - 1);
      mbar_wait(&full[slot], (stage_i >> p.nst_log2) & 1);
      const uint32_t wst = w_ring + slot * stage_bytes;
      const int tq0 = wk * p.q;                                     // first tile of this warp's quantum inside the stage
#pragma unroll 2
      for (int u = 0; u < p.q; ++u) {
        const int tis = tq0 + u;                                    // tile index inside the stage
        if (xc0 + xs0 + tis >= p.KT) break;
        v2_tile_mma<WBITS, MT>(acc, wst + tis * sub_tile_bytes, woff0, woff1, CS, x_thr + (xs0 + tis) * 128, XS8, live);
      }
      if (GROUPED && xc0 + xs0 + tq0 < p.KT) {  // the quantum was one quantization group: fold it into the fp32 result
        const int grp = (xc0 + xs0 + tq0) / p.grouped_gt;
        const int gi = (xs0 + tq0) / p.grouped_gt;
        sz0 = p.sz[(size_t)grp * p.Np + pr0];
        sz1 = p.sz[(size_t)grp * p.Np + pr1];
#pragma unroll
        for (int m = 0; m < MT; ++m) {
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float2 z = (c < 2) ? sz0 : sz1;
            const int row = m * 8 + 2 * t + (c & 1);
            const float sa = row < p.M ? suma[row * gpc + gi] : 0.f;
            facc[m][c] += z.x * (acc[m][c] - z.y * sa);
            acc[m][c] = 0.f;
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[slot]);
    }
  }

  // ---- park this warp's partial tile (raw accumulators for per-channel weights: the dequantisation is linear)
#pragma unroll
  for (int m = 0; m < MT; ++m) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int row = m * 8 + 2 * t + (c & 1);
      fs2[(wk * MP + row) * CB + wn * 16 + g + (c >> 1) * 8] = GROUPED ? facc[m][c] : acc[m][c];
    }
  }
  v2_bar_sync(1, kV2Warps * 32);

  // ---- sum the k-slices in fixed order, dequantise, alpha / bias / activation / residual (or SwiGLU), bf16 store
  const int ctid = tid;
  if (p.act == B2_ACT_SWIGLU) {  // local rows [0, CB/2) gate, [CB/2, CB) up of output channels ng*64 + sub*CB/2 + i
    const int half = CB >> 1;
    for (int i = ctid; i < p.M * half; i += kV2Warps * 32) {
      const int m = i / half, c = i - m * half;
      const int n = ng * 64 + sub * half + c;
      if (n >= p.N) continue;
      float gv = 0.f, uv = 0.f;
      for (int k = 0; k < WK; ++k) {
        gv += fs2[(k * MP + m) * CB + c];
        uv += fs2[(k * MP + m) * CB + half + c];
      }
      if (!GROUPED && WBITS != 16) {
        const float2 zg = p.sz[ng * kBN + sub * half + c], zu = p.sz[ng * kBN + 64 + sub * half + c];
        gv = zg.x * (gv - zg.y * suma[m]);
        uv = zu.x * (uv - zu.y * suma[m]);
      }
      gv *= p.alpha;
      uv *= p.alpha;
      p.C[(int64_t)m * p.ldc + n] = __float2bfloat16(apply_act<B2_ACT_SILU>(gv) * uv);
    }
    return;
  }
  for (int i = ctid; i < p.M * CB; i += kV2Warps * 32) {
    const int m = i >> p.cb_log2, c = i & (CB - 1);
    const int n = ng * kBN + sub * CB + c;
    if (n >= p.N) continue;
    float v = 0.f;
    for (int k = 0; k < WK; ++k) v += fs2[(k * MP + m) * CB + c];
    if (!GROUPED && WBITS != 16) {
      const float2 z = p.sz[n];
      v = z.x * (v - z.y * suma[m]);
    }
    v *= p.alpha;
    if (p.bias) v += __bfloat162float(p.bias[n]);
    v = apply_act_rt(v, p.act);
    if (p.residual) v += __bfloat162float(p.residual[(int64_t)m * p.ldc + n]);
    p.C[(int64_t)m * p.ldc + n] = __float2bfloat16(v);
  }
}

typedef void (*gemv2_kernel_t)(const Gemv2Params, const CUtensorMap);

template <int WBITS, bool GROUPED>
static gemv2_kernel_t v2_pick_mt(int mt) {
  switch (mt) {
    case 1: return wq_gemv2_kernel<WBITS, 1, GROUPED>;
    case 2: return wq_gemv2_kernel<WBITS, 2, GROUPED>;
    default: return wq_gemv2_kernel<WBITS, 4, GROUPED>;
  }
}
static gemv2_kernel_t v2_pick(int wbits, bool grouped, int mt) {
  if (wbits == 4) return grouped ? v2_pick_mt<4, true>(mt) : v2_pick_mt<4, false>(mt);
  if (wbits == 8) return grouped ? v2_pick_mt<8, true>(mt) : v2_pick_mt<8, false>(mt);
  return v2_pick_mt<16, false>(mt);
}

static int v2_env(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}

// Channels per CTA: the largest of 128/64/32/16 whose grid still covers the SMs ~twice (more CTAs = more independent TMA
// rings = more bytes in flight per SM); a pair image needs >= 32 (16 gate + 16 up rows per CTA).
bool gemv2_plan(const Gemv2Launch& a, Gemv2Plan* pl) {
  // With the 128-row tile image a CTA that owns fewer than 128 channels reads 256..1024-byte row runs at a 2 KB stride and
  // eight CTAs revisit every DRAM page, which starves quantized shapes; 128-channel blocks of dense bf16 weights (lm_head)
  // stream whole tiles.
  // Default policy (B2_GEMV2=1): dense bf16 weights only; B2_GEMV2=2 takes every shape (tests), 0 none.
  const int mode = v2_env("B2_GEMV2", 1);
  if (mode == 0 || (mode == 1 && a.wbits != 16)) return false;
  const int sms = sm_count();
  const int rows = a.NG * kBN;
  const int want = v2_env("B2_GEMV2_MIN_CTAS", 2 * sms);
  int cb = 128;
  const int cb_min = a.pair ? 32 : 16;
  const int forced = v2_env("B2_GEMV2_CB", 0);
  if (forced) cb = forced;
  else
    while (cb > cb_min && rows / cb < want) cb >>= 1;
  if (cb < cb_min || cb > 128 || (cb & (cb - 1))) return false;
  if (!forced && rows / cb < v2_env("B2_GEMV2_FLOOR_CTAS", sms / 2)) return false;  // too small even at 16 channels: split-K kernel
  const int wk = kBN / cb;
  const int q = a.group_tiles > 0 ? a.group_tiles : 2;
  const int stage_tiles = wk * q;
  const int tile_bytes = a.wbits == 4 ? 4096 : (a.wbits == 8 ? 8192 : 16384);
  const int stage_bytes = q * tile_bytes;
  if (stage_bytes > 64 * 1024) return false;  // very large quantization groups: split-K kernel
  const int ring_kb = v2_env("B2_GEMV2_RING_KB", 32);
  int nst_log2 = 1;
  while ((2 << nst_log2) * stage_bytes <= ring_kb * 1024) ++nst_log2;
  const int mt = a.M <= 8 ? 1 : (a.M <= 16 ? 2 : 4);
  const int MP = 8 * mt;
  const int x_budget = v2_env("B2_GEMV2_XBYTES", 24 * 1024);
  int xt = (x_budget / MP - 16) / 128;
  xt = xt / stage_tiles * stage_tiles;
  if (xt < stage_tiles) xt = stage_tiles;
  const int kt_round = (a.KT + stage_tiles - 1) / stage_tiles * stage_tiles;
  if (xt > kt_round) xt = kt_round;
  const int gpc = a.group_tiles > 0 ? xt / a.group_tiles : 1;
  pl->cb_log2 = cb == 128 ? 7 : (cb == 64 ? 6 : (cb == 32 ? 5 : 4));
  pl->q = q;
  pl->xt = xt;
  pl->nst_log2 = nst_log2;
  pl->mt = mt;
  pl->grid = a.NG * wk;
  pl->smem = (1 << nst_log2) * stage_bytes + MP * (xt * 128 + 16) + wk * MP * cb * 4 + MP * gpc * 4 + 16 + 8 + (1 << nst_log2) * 16 + 64;
  return pl->smem <= 200 * 1024;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn v2_encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

cudaError_t gemv2_launch(const Gemv2Launch& a, const Gemv2Plan& pl, cudaStream_t stream) {
  gemv2_kernel_t kern = v2_pick(a.wbits, a.group_tiles > 0, pl.mt);
  // the opt-in shared-memory limit is only ever raised (the instantiation is shared by handles with different plans)
  static int limit[3][2][3] = {};
  int& cur = limit[a.wbits == 4 ? 0 : (a.wbits == 8 ? 1 : 2)][a.group_tiles > 0][pl.mt == 1 ? 0 : (pl.mt == 2 ? 1 : 2)];
  if (pl.smem > cur) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, pl.smem);
    if (e != cudaSuccess) return e;
    cur = pl.smem;
  }
  // the tile image as a 4-D tensor of 8-byte elements: [tile (NG*KT)][chunk][half: rows 0-63 | 64-127][64 rows x 16 B = 128 el]
  EncodeTiledFn enc = v2_encode_tiled();
  if (!enc) return cudaErrorNotSupported;
  const int nch = a.wbits == 4 ? 2 : (a.wbits == 8 ? 4 : 8);
  const int cb = 1 << pl.cb_log2, wk = kBN / cb;
  const int run_rows = a.pair ? cb / 2 : (cb < 64 ? cb : 64);
  alignas(64) CUtensorMap wmap;
  const cuuint64_t gdim[4] = {128, 2, (cuuint64_t)nch, (cuuint64_t)a.NG * a.KT};
  const cuuint64_t gstride[3] = {1024, 2048, (cuuint64_t)nch * 2048};
  const cuuint32_t box[4] = {(cuuint32_t)run_rows * 2, (cuuint32_t)((a.pair || cb == 128) ? 2 : 1), (cuuint32_t)nch, (cuuint32_t)(wk * pl.q)};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  if (enc(&wmap, CU_TENSOR_MAP_DATA_TYPE_UINT64, 4, const_cast<uint8_t*>(a.packed), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
          CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return cudaErrorInvalidValue;
  Gemv2Params p;
  p.packed = a.packed; p.sz = a.sz; p.A = a.A; p.lda = a.lda; p.C = a.C; p.ldc = a.ldc; p.bias = a.bias; p.residual = a.residual;
  p.M = a.M; p.N = a.N; p.K = a.K; p.Np = a.Np; p.KT = a.KT; p.NG = a.NG;
  p.cb_log2 = pl.cb_log2; p.q = pl.q; p.grouped_gt = a.group_tiles; p.xt = pl.xt; p.nst_log2 = pl.nst_log2;
  p.pair = a.pair ? 1 : 0; p.act = a.act; p.alpha = a.alpha;
  return launch(kern, dim3(pl.grid), dim3(kV2Threads), (size_t)pl.smem, stream, true, p, wmap);
}

}  // namespace b2
