// b200spark — definitions shared by the weight-only GEMM kernels (mma.sync small-M: wq_gemm.cu, wq_gemv2.cu; wgmma
// medium-M: wq_gemm_tc.cu).
#pragma once
#include <cuda.h>  // CUtensorMap (types only; the encoder is fetched with cudaGetDriverEntryPoint)

#include <type_traits>

#include "b2_common.cuh"

namespace b2 {

constexpr int kBN = 128;                   // output channels per CTA tile
constexpr int kBK = 64;                    // k per tile
constexpr uint32_t kMask4 = 0x00780078u;   // nibble at mantissa bits 3..6 of each bf16 half
constexpr uint32_t kMagic = 0x41804180u;   // bf16 16.0 in both halves: 16 + q exactly
constexpr uint32_t kMagicHi = 0x43804380u; // bf16 256.0: 16 * (16 + q) exactly (hi nibble plane of W8)

// ---- weight image layout (one image serves every weight-only GEMM kernel) ----
// image[n_group][k_tile] = tile of 128 output channels x 64 k, stored as [chunk c][row r ^ swz(c)][16 bytes]:
//   W4 : 2 chunks, chunk = 32 k of one row as 4 words; word j nibble i <-> k = 32c+8j+2i, nibble i+4 <-> k+1
//   W8 : 4 chunks, chunk = 16 k of one row as 4 words; word j bytes (b0,b2,b1,b3) <-> k = 16c+4j+(0,1,2,3)
//   W16: 8 chunks, chunk = 8 k of one row as 4 words; word j halves (h0,h1) <-> k = 8c+2j+(0,1)
// i.e. the even k of a word fill its low half and the odd k its high half, each in k order.  Every word of W4/W8 is rotated
// left by 3 so that (w >> 4i) & 0x00780078 | magic yields two exact bf16 integers.  A gate/up pair image (SwiGLU) takes rows
// 0..63 of every tile from the gate weights and rows 64..127 from the up weights.
template <int WBITS>
struct Image {
  static constexpr int kChunks = WBITS == 4 ? 2 : (WBITS == 8 ? 4 : 8);  // 16-byte chunks per tile row
  static constexpr int kKPerChunk = kBK / kChunks;                       // 32 / 16 / 8
  static constexpr int kKPerWord = kKPerChunk / 4;                       // 8 / 4 / 2
  static constexpr int kChunkBytes = kBN * 16;                           // 2048
  static constexpr int kTileBytes = kChunks * kChunkBytes;               // 4096 / 8192 / 16384
  static constexpr int kTileWords = kTileBytes / 4;
  static constexpr bool kRotated = WBITS != 16;                          // words stored rotated left by 3
  __host__ __device__ __forceinline__ static int swz(int c) {
    return WBITS == 4 ? 4 * (c & 1) : (WBITS == 8 ? 2 * (c & 3) : 2 * ((c >> 1) & 3));
  }
  // byte offset of (row, chunk c) inside a chunk of rows / inside a tile.  chunk_offset takes the row by reference: by value
  // it is an argument when the helper is simplified on its own, the XOR's operands come out swapped, and ptxas schedules the
  // mma.sync GEMV kernel's address arithmetic differently.
  __host__ __device__ __forceinline__ static int row_offset(int row, int c) { return (row ^ swz(c)) << 4; }
  __host__ __device__ __forceinline__ static int chunk_offset(const int& row, int c) { return c * kChunkBytes + ((row ^ swz(c)) << 4); }
};

// Runtime weight width -> template argument: f(std::integral_constant<int, WBITS>)  (flags: with_flag, b2_common.cuh)
template <typename F>
inline auto with_wbits(int wbits, F&& f) {
  if (wbits == 4) return f(std::integral_constant<int, 4>{});
  if (wbits == 8) return f(std::integral_constant<int, 8>{});
  return f(std::integral_constant<int, 16>{});
}

// wgmma kernel entry (wq_gemm_tc.cu)
struct TcParams {
  const uint8_t* packed;
  const float2* sz;
  const __nv_bfloat16* A;
  int64_t lda;
  __nv_bfloat16* C;
  int64_t ldc;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* residual;
  float* ws;              // [NG][S] partial tiles of the k-slices, or [NR][kTcCarryFloats] parked heads (TcSched)
  unsigned* counters;
  int M, N, K, Np, KT, NG;
  int grid, rounds, S, h;  // the work schedule (TcSched)
  int cluster = 0;         // 1: the S k-slices of an n-group are one thread-block cluster and sum their partial tiles over
                           // distributed shared memory (rounds == 0 only; launched by tc_launch as clusters of S CTAs)
  int act;
  float alpha;
  // fp8 activations (A8 instantiation): A is fp8-e4m3 in the b2 fp8 activation layout (lda in bytes), per-token scale [M] and
  // per-(row, 64-k tile) sums of the quantized values [M][KT]
  const float* a_scale = nullptr;
  const float* tile_sums = nullptr;
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
  int nm;                 // MMA N (batch columns): 64, or 32 when M <= 32 (half the tensor-pipe time and activation traffic)
  int group_tiles = 0;    // > 0: sub-channel weights (GROUPED instantiation), k-tiles per quantization group; sz is [G][Np]
  int group_k = 0, ngroups = 1;  // group_k > 0: a group size that is no multiple of 64 (a multiple of 8, >= 32): 8 consecutive
                                 // k — one word of the image — never straddle a group, so the params are looked up per word
};

// The wgmma kernel's work schedule (planned by make_tc_plan, walked by wq_gemm_tc_kernel).  While there are at most as many
// n-groups as CTAs, CTA b takes k-slice b % S of n-group b / S (S equal slices; the partials are summed in slice order by
// the last slice to arrive, or, when the S slices are one cluster, by every slice for its share of the rows).  Otherwise each of the grid CTAs takes `rounds` whole n-groups, b + j * grid, and each of the NR = NG - nfull
// n-groups left over is cut in two at k-tile h: CTA b < NR runs the head [0, h) of n-group nfull + b first and parks its
// raw accumulators; CTA NR + b runs the tail [h, KT) last, starting from them, so every output is the one k-ordered fp32
// chain of a whole n-group, bit for bit.  A tail that starts before its head has parked runs the whole n-group instead: no
// CTA waits for another.  h = 0: CTA b < NR runs leftover n-group nfull + b whole.
struct TcSeg {
  int ng, kt0, kt1;  // k-tiles [kt0, kt1) of n-group ng
  int part, parts;   // k-slice `part` of `parts` (parts == 1: the CTA finishes the n-group)
  int carry;         // 1: head (parks its accumulators), 2: tail (starts from them if they are there)
};
constexpr int kTcCarryFloats = 256 * 32 + 64 * 4;  // a parked head: 32 accumulators per consumer thread, 4 row sums per row
struct TcSched {
  int NG, KT, grid, rounds, S, h, b, nfull, NR;
  __host__ __device__ TcSched(int NG_, int KT_, int grid_, int rounds_, int S_, int h_, int b_)
      : NG(NG_), KT(KT_), grid(grid_), rounds(rounds_), S(S_), h(h_), b(b_), nfull(rounds_ * grid_), NR(NG_ - rounds_ * grid_) {}
  __host__ __device__ int count() const {
    return rounds == 0 ? 1 : rounds + (b < NR ? 1 : 0) + (h > 0 && b >= NR && b < 2 * NR ? 1 : 0);
  }
  __host__ __device__ TcSeg seg(int i) const {
    if (rounds == 0) {
      const int ng = b / S, s = b - ng * S;
      return TcSeg{ng, s * KT / S, (s + 1) * KT / S, s, S, 0};
    }
    const int head = b < NR ? 1 : 0;
    if (head && i == 0) return TcSeg{nfull + b, 0, h > 0 ? h : KT, 0, 1, h > 0 ? 1 : 0};
    const int j = i - head;
    if (j < rounds) return TcSeg{j * grid + b, 0, KT, 0, 1, 0};
    return TcSeg{nfull + b - NR, h, KT, 0, 1, 2};
  }
};

// GEMV for dense bf16 weights without global split-K (wq_gemv2.cu)
struct Gemv2Params {
  const uint8_t* packed;
  const __nv_bfloat16* A;
  int64_t lda;
  __nv_bfloat16* C;
  int64_t ldc;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* residual;
  int M, N, K, KT, NG;
  int cb_log2;      // log2(CB)
  int xt;           // k-tiles per activation chunk (multiple of the stage: WK * kV2Q)
  int nst_log2;     // log2(pipeline stages)
  int pair;         // gate/up pair image (SwiGLU epilogue)
  int act;
  float alpha;
};
struct Gemv2Plan {
  int mt, grid, smem;
};
bool gemv2_plan(Gemv2Params& p, Gemv2Plan* plan);   // fills cb_log2, xt, nst_log2; false: use the split-K kernel
cudaError_t gemv2_launch(const Gemv2Params& p, const Gemv2Plan& plan, cudaStream_t stream);

constexpr int kGemvMaxM = 16;  // batch rows per launch of the mma.sync GEMV kernels (MT <= 2)
constexpr int kTcMaxM = 64;    // batch rows per wgmma launch
// sets p.nm; fp16: activations / outputs / bias / residual are fp16 (else bf16)
cudaError_t tc_launch(int wbits, bool fp16, TcParams p, cudaStream_t stream);
// whether `clusters` thread-block clusters of S wgmma CTAs are resident at once (one wave) on this device
bool tc_clusters_fit(int wbits, int S, int clusters);

// Raise a kernel's dynamic shared-memory opt-in to smem, never lower it: an instantiation is shared by handles whose plans
// need different amounts, and a later handle with a smaller need must not lower the limit under an earlier one's launches.
cudaError_t raise_smem_limit(const void* kern, int smem);

// cuTensorMapEncodeTiled, fetched from the driver through the runtime (nullptr if unavailable)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled();

}  // namespace b2
