// b200spark — definitions shared by the two weight-only GEMM kernels (mma.sync small-M, wgmma medium-M).
#pragma once
#include "b2_common.cuh"

namespace b2 {

constexpr int kBN = 128;                   // output channels per CTA tile
constexpr int kBK = 64;                    // k per tile
constexpr uint32_t kMask4 = 0x00780078u;   // nibble at mantissa bits 3..6 of each bf16 half
constexpr uint32_t kMagic = 0x41804180u;   // bf16 16.0 in both halves: 16 + q exactly
constexpr uint32_t kMagicHi = 0x43804380u; // bf16 256.0: 16 * (16 + q) exactly (hi nibble plane of W8)

// ---- weight image layout (one image serves both kernels) ----
// tile(ng, kt) = 128 output channels x 64 k, stored as [chunk c][row r ^ swz(c)][16 bytes]:
//   W4 : 2 chunks, chunk = 32 k of one row as 4 words; word j nibble i <-> k = 32c+8j+2i, nibble i+4 <-> k+1
//   W8 : 4 chunks, chunk = 16 k of one row as 4 words; word j bytes (b0,b2,b1,b3) <-> k = 16c+4j+(0,1,2,3)
//   W16: 8 chunks, chunk = 8 k of one row, natural order
// every word of W4/W8 is rotated left by 3 so that (w >> 4i) & 0x00780078 | magic yields two exact bf16 integers.
__host__ __device__ __forceinline__ int tile_swz(int wbits, int c) {
  return wbits == 4 ? 4 * (c & 1) : (wbits == 8 ? 2 * (c & 3) : 2 * ((c >> 1) & 3));
}

// wgmma kernel entry (wq_gemm_tc.cu)
struct TcLaunch {
  const uint8_t* packed;
  const float2* sz;
  const __nv_bfloat16* A;
  int64_t lda;
  __nv_bfloat16* C;
  int64_t ldc;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* residual;
  float* ws;
  unsigned* counters;
  int M, N, K, Np, KT, NG, S;
  int act;
  float alpha;
  const float* a_scale = nullptr;    // != NULL: A is fp8-e4m3 in the b2 fp8 activation layout (lda in bytes)
  const float* tile_sums = nullptr;  // [M][KT] sums of the quantized activations per 64-k tile
  int group_tiles = 0;               // > 0: sub-channel weights, k-tiles per quantization group (sz is [G][Np])
  int group_k = 0, ngroups = 1;      // group_k > 0: group size not a multiple of 64 (a multiple of 8): params per 8-k word
  bool fp16 = false;                 // activations / outputs / bias / residual are fp16 (else bf16)
  bool dual = false;                 // two CTAs per SM (int4 weights, bf16 activations): half-depth stages
  // RMSNorm hand-off between GEMMs (b2_gemm_fuse, batches >= 17).  Consumer: A holds bf16(x * gamma); the result rows are
  // scaled by rsqrt(sum_p norm_sumsq[p * norm_ld + m] / hidden + eps).  Producer: besides C it writes xg = bf16(C * gamma_out)
  // and, per 128-channel tile, the sum of squares of every stored row.
  const float* norm_sumsq = nullptr;
  int norm_parts = 0, norm_ld = 0;
  float norm_inv_hidden = 0.f, norm_eps = 0.f;
  float* sumsq_out = nullptr;        // [NG][norm_ld]
  __nv_bfloat16* xg_out = nullptr;   // [M, ldxg]
  const __nv_bfloat16* gamma_out = nullptr;
  int64_t ldxg = 0;
};
// GEMV without global split-K (wq_gemv2.cu)
struct Gemv2Launch {
  const uint8_t* packed;
  const float2* sz;
  const __nv_bfloat16* A;
  int64_t lda;
  __nv_bfloat16* C;
  int64_t ldc;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* residual;
  int M, N, K, Np, KT, NG;
  int wbits, group_tiles;  // group_tiles: k-tiles per quantization group, 0 = per channel
  bool pair;
  int act;
  float alpha;
};
struct Gemv2Plan {
  int cb_log2, q, xt, nst_log2, mt, grid, smem;
};
bool gemv2_plan(const Gemv2Launch& a, Gemv2Plan* plan);   // false: use the split-K kernel
cudaError_t gemv2_launch(const Gemv2Launch& a, const Gemv2Plan& plan, cudaStream_t stream);

constexpr int kTcMaxM = 64;  // batch rows per wgmma launch
int tc_smem_bytes(int wbits, bool dual);
cudaError_t tc_configure(int wbits);
cudaError_t tc_launch(int wbits, const TcLaunch& a, cudaStream_t stream);

}  // namespace b2
