// b200spark — GEMV for dense bf16 weights at decode batches 1..16 WITHOUT global split-K, sm_90a.  Same weight image, same
// tensor-core math and the same results (up to fp32 summation order) as the split-K kernel of wq_gemm.cu.
//
// Why a second decomposition: at batch 1 most of the split-K kernel's time after the weight stream is its split-K tail —
// partials to the workspace, __threadfence, atomic ticket, waiting for the sibling CTAs, re-reading the partial tiles from
// L2.  A 16-way K split across CTAs is what it takes to fill 132 SMs with 128-channel tiles of a 4608-channel
// projection, so the split has to move INSIDE the CTA:
//
//   * a CTA owns CB in {128, 64, 32, 16} output channels of one 128-channel n-group and the FULL K range;
//     grid = N / CB CTAs (CB is chosen so that the grid covers the SMs at least ~1.5 times);
//   * its 8 consumer warps form WN = CB/16 n16-tiles x WK = 128/CB k-slices; a pipeline stage carries WK quanta of 2 k-tiles
//     and warp (wn, wk) takes quantum wk of every stage — all warps always work on the stage that just landed;
//   * the producer lane fetches a whole stage with ONE TMA tensor request: the tile image is described as a 4-D tensor
//     [tile][chunk][half: rows 0-63 | 64-127][64 rows x 16 B] and the CTA's box is {its rows, 1 or 2 halves, all chunks, the
//     stage's tiles} (a gate/up pair image takes the 16 gate rows and the 16 matching up rows with the half dimension) —
//     the TMA unit spends ~46 clocks per REQUEST whatever its size, so row-run bulk copies of 256 B could not exceed 10 GB/s
//     per SM (measured: 83 us for down_proj).  Issued ahead of the previous kernel's completion (PDL);
//   * the WK partial accumulators meet in shared memory (fixed order => deterministic): no workspace, no fence, no atomics,
//     no second wave of L2 reads;
//   * only the M live batch rows are staged (the split-K kernel zero-fills all 8 / 16 rows of the MMA's n side).
//
// Quantized weights stay on the split-K kernel: with the 128-row tile image a CTA that owns fewer than 128 channels reads
// 256..1024-byte row runs at a 2 KB stride and eight CTAs revisit every DRAM page, which starves quantized shapes;
// 128-channel blocks of dense bf16 weights (lm_head) stream whole tiles.
//
// Roofline: HBM-bound; algorithmic bytes/launch = 2*K*N + 2*M*(K+N).
#include "b2_common.cuh"
#include "wq_gemm_shared.cuh"

namespace b2 {

using V2Image = Image<16>;
constexpr int kV2Warps = 8;
constexpr int kV2Threads = kV2Warps * 32 + 32;  // + producer warp
constexpr int kV2Q = 2;                         // k-tiles per quantum (= per warp per stage)

__device__ __forceinline__ void v2_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// One k-tile (64 k x 16 n) of tensor-core work for this warp.  woff0/woff1: byte offsets of this thread's row g / g+8
// inside the CTA's sub-tile [chunk][CB rows][16 B] (CS = CB * 16 bytes per chunk); xaddr: this thread's 32 bytes of
// activations of batch row g (16 consecutive k); live[m]: batch row g + 8m exists.
template <int MT>
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

template <int MT>
__global__ void __launch_bounds__(kV2Threads) wq_gemv2_kernel(const Gemv2Params p, const __grid_constant__ CUtensorMap wmap) {
  constexpr int MP = 8 * MT;
  const int NST = 1 << p.nst_log2;
  const int CB = 1 << p.cb_log2;                                    // channels (image rows) of this CTA
  const int SUBS = kBN >> p.cb_log2;                                // CTAs per n-group == k-slices per CTA (WK)
  const int WK = SUBS, WN = CB >> 4;
  const uint32_t CS = (uint32_t)CB * 16u;                           // bytes per chunk of the CTA's sub-tile
  const int sub_tile_bytes = V2Image::kChunks * (int)CS;            // bytes per k-tile in shared memory
  const int stage_tiles = WK * kV2Q;
  const int stage_bytes = stage_tiles * sub_tile_bytes;             // == kV2Q * V2Image::kTileBytes
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int ng = blockIdx.x / SUBS, sub = blockIdx.x - ng * SUBS;

  // ---- shared memory carve-up
  // (the partial tiles sit between the ring and the activations: with them last, ptxas spills their address around the
  // main loop of the MT = 2 instantiation)
  uint8_t* ring = smem;
  const int XS = p.xt * 128 + 16;                                   // activation row stride (bytes), == 16 mod 128
  float* fs2 = reinterpret_cast<float*>(ring + NST * stage_bytes);  // [WK][MP][CB] partial tiles of the k-slices
  uint8_t* xs = reinterpret_cast<uint8_t*>(fs2 + WK * MP * CB);     // 128-byte aligned: WK * CB == 128
  uint64_t* full = reinterpret_cast<uint64_t*>((reinterpret_cast<uintptr_t>(xs + MP * XS + 16) + 7) & ~uintptr_t(7));
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
      const int c0 = p.pair ? sub * run_rows * 2 : ((sub * CB) & 63) * 2;
      const int c1 = p.pair ? 0 : (sub * CB) >> 6;
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

  float acc[MT][4];
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[m][c] = 0.f;
  bool live[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) live[m] = (g + 8 * m) < p.M;

  pdl_wait();  // activations belong to the previous kernel from here on

  const uint32_t w_ring = smem_u32(ring);
  const int wc = 2 * t;
  // the image stores row r of chunk c at r ^ swz(c): swz < 8 and the CTA's row runs are 16-aligned, so the XOR stays local
  const uint32_t woff0 = wc * CS + V2Image::row_offset(lr0, wc);
  const uint32_t woff1 = wc * CS + V2Image::row_offset(lr1, wc);
  const uint32_t x_thr = smem_u32(xs) + g * XS + t * 32;
  const int XS8 = 8 * XS;
  int stage_i = 0;

  for (int xc0 = 0; xc0 < p.KT; xc0 += p.xt) {   // p.xt is a multiple of stage_tiles
    const int xn = min(p.xt, p.KT - xc0);
    if (xc0 > 0) v2_bar_sync(1, kV2Warps * 32);  // previous chunk fully consumed
    // ---- stage the M live activation rows of this k-chunk
    {
      const int64_t kbase = (int64_t)xc0 * kBK;
      const int nvec = xn * 8;
      for (int m = warp; m < p.M; m += kV2Warps) {
        const __nv_bfloat16* arow = p.A + (int64_t)m * p.lda + kbase;
        uint8_t* xrow = xs + m * XS;
        for (int v = lane; v < nvec; v += 32) {
          uint4 val = make_uint4(0, 0, 0, 0);
          if (kbase + v * 8 < p.K) val = *reinterpret_cast<const uint4*>(arow + v * 8);
          *reinterpret_cast<uint4*>(xrow + v * 16) = val;
        }
      }
    }
    v2_bar_sync(1, kV2Warps * 32);

    // ---- main loop: one pipeline stage per iteration; this warp takes quantum wk of it
    for (int xs0 = 0; xs0 < xn; xs0 += stage_tiles, ++stage_i) {
      const int slot = stage_i & (NST - 1);
      mbar_wait(&full[slot], (stage_i >> p.nst_log2) & 1);
      const uint32_t wst = w_ring + slot * stage_bytes;
      const int tq0 = wk * kV2Q;                                    // first tile of this warp's quantum inside the stage
#pragma unroll
      for (int u = 0; u < kV2Q; ++u) {
        const int tis = tq0 + u;                                    // tile index inside the stage
        if (xc0 + xs0 + tis >= p.KT) break;
        v2_tile_mma<MT>(acc, wst + tis * sub_tile_bytes, woff0, woff1, CS, x_thr + (xs0 + tis) * 128, XS8, live);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[slot]);
    }
  }

  // ---- park this warp's partial tile
#pragma unroll
  for (int m = 0; m < MT; ++m) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int row = m * 8 + 2 * t + (c & 1);
      fs2[(wk * MP + row) * CB + wn * 16 + g + (c >> 1) * 8] = acc[m][c];
    }
  }
  v2_bar_sync(1, kV2Warps * 32);

  // ---- sum the k-slices in fixed order, alpha / bias / activation / residual (or SwiGLU), bf16 store
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
    v *= p.alpha;
    if (p.bias) v += __bfloat162float(p.bias[n]);
    v = apply_act_rt(v, p.act);
    if (p.residual) v += __bfloat162float(p.residual[(int64_t)m * p.ldc + n]);
    p.C[(int64_t)m * p.ldc + n] = __float2bfloat16(v);
  }
}

// Channels per CTA: the largest of 128/64/32/16 whose grid still covers the SMs ~twice (more CTAs = more independent TMA
// rings = more bytes in flight per SM); a pair image needs >= 32 (16 gate + 16 up rows per CTA).  B2_GEMV2=0: never.
bool gemv2_plan(Gemv2Params& p, Gemv2Plan* pl) {
  if (!env_int("B2_GEMV2", 1) || p.M > kGemvMaxM) return false;
  const int sms = sm_count();
  const int rows = p.NG * kBN;
  const int want = env_int("B2_GEMV2_MIN_CTAS", 2 * sms);
  int cb = 128;
  const int cb_min = p.pair ? 32 : 16;
  const int forced = env_int("B2_GEMV2_CB", 0);
  if (forced) cb = forced;
  else
    while (cb > cb_min && rows / cb < want) cb >>= 1;
  if (cb < cb_min || cb > 128 || (cb & (cb - 1))) return false;
  if (!forced && rows / cb < env_int("B2_GEMV2_FLOOR_CTAS", sms / 2)) return false;  // too small even at 16 channels: split-K kernel
  const int wk = kBN / cb;
  const int stage_tiles = wk * kV2Q;
  const int stage_bytes = kV2Q * V2Image::kTileBytes;
  const int ring_kb = env_int("B2_GEMV2_RING_KB", 32);
  int nst_log2 = 1;
  while ((2 << nst_log2) * stage_bytes <= ring_kb * 1024) ++nst_log2;
  const int mt = p.M <= 8 ? 1 : 2;
  const int MP = 8 * mt;
  const int x_budget = env_int("B2_GEMV2_XBYTES", 24 * 1024);
  int xt = (x_budget / MP - 16) / 128;
  xt = xt / stage_tiles * stage_tiles;
  if (xt < stage_tiles) xt = stage_tiles;
  const int kt_round = (p.KT + stage_tiles - 1) / stage_tiles * stage_tiles;
  if (xt > kt_round) xt = kt_round;
  p.cb_log2 = cb == 128 ? 7 : (cb == 64 ? 6 : (cb == 32 ? 5 : 4));
  p.xt = xt;
  p.nst_log2 = nst_log2;
  pl->mt = mt;
  pl->grid = p.NG * wk;
  pl->smem = (1 << nst_log2) * stage_bytes + wk * MP * cb * 4 + MP * (xt * 128 + 16) + 16 + 8 + (1 << nst_log2) * 16 + 64;
  return pl->smem <= 200 * 1024;
}

cudaError_t gemv2_launch(const Gemv2Params& p, const Gemv2Plan& pl, cudaStream_t stream) {
  auto kern = pl.mt == 1 ? wq_gemv2_kernel<1> : wq_gemv2_kernel<2>;
  cudaError_t e = raise_smem_limit((const void*)kern, pl.smem);
  if (e != cudaSuccess) return e;
  // the tile image as a 4-D tensor of 8-byte elements: [tile (NG*KT)][chunk][half: rows 0-63 | 64-127][64 rows x 16 B = 128 el]
  EncodeTiledFn enc = encode_tiled();
  if (!enc) return cudaErrorNotSupported;
  const int cb = 1 << p.cb_log2, wk = kBN / cb;
  const int run_rows = p.pair ? cb / 2 : (cb < 64 ? cb : 64);
  alignas(64) CUtensorMap wmap;
  const cuuint64_t gdim[4] = {V2Image::kChunkBytes / 16, 2, (cuuint64_t)V2Image::kChunks, (cuuint64_t)p.NG * p.KT};
  const cuuint64_t gstride[3] = {V2Image::kChunkBytes / 2, V2Image::kChunkBytes, V2Image::kTileBytes};
  const cuuint32_t box[4] = {(cuuint32_t)run_rows * 2, (cuuint32_t)((p.pair || cb == 128) ? 2 : 1), (cuuint32_t)V2Image::kChunks,
                             (cuuint32_t)(wk * kV2Q)};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  if (enc(&wmap, CU_TENSOR_MAP_DATA_TYPE_UINT64, 4, const_cast<uint8_t*>(p.packed), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
          CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return cudaErrorInvalidValue;
  return launch(kern, dim3(pl.grid), dim3(kV2Threads), (size_t)pl.smem, stream, true, p, wmap);
}

}  // namespace b2
