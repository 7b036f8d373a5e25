// b200spark — SpanAttention decode: paged KV (spans) single-query attention, GQA, sm_90a.
//
// Replaces the reference's three-kernel pipeline with a materialised score matrix
// (span-attention/src/attn/qk/qk_gemv.cuh, softmax/block_softmax.cuh, qkv/qkv_gemv.cuh + reduce)
// and its per-layer-per-step host staging (span_attention.hpp:36-176) with ONE persistent kernel:
//
//   * work items (sequence, kv-head, token-chunk) are derived ON THE DEVICE from new_lens — no host
//     tile mapping, no H2D copies, CUDA-graph replayable while sequences grow;
//   * each CTA streams 64-token K and V tiles of its item through a cp.async ring into XOR-swizzled
//     shared memory straight from the span pages (page table walked per 16-byte chunk);
//   * all q-heads of the kv-group ride in the 16 rows of one mma.m16n8k16 tile, so K and V are read
//     once per group: S = Q K^T on tensor cores, online softmax in fp32 (exp2), O += P V on tensor cores;
//   * split-KV partials (fp32, unnormalised) go to the caller's workspace; the last CTA of a
//     (sequence, kv-head) — device counter, self-resetting — merges them in fixed order.
//
// Roofline: HBM-bound; algorithmic bytes = sum_b len_b * 2 * n_groups * (128*elem + 8[quant]).
#include <cstdlib>
#include <new>

#include "b2_common.cuh"

namespace b2 {

constexpr int kAttnThreads = 128;  // 4 warps, 16 tokens of each 64-token tile per warp
constexpr int kTile = 64;
constexpr int kHead = 128;
constexpr int kMaxBatch = 1024;
constexpr int kMergeRS = 136;  // padded fp32 row stride of the merge buffer (conflict-free float2 stores)
constexpr int kMergeDirect = 16;  // up to this many pieces per (sequence, kv-head): the last CTA merges them all
constexpr int kMergeFan = 8;      // above: groups of 8 pieces are merged by their last CTA, the last group merges the groups

struct AttnParams {
  __nv_bfloat16* out;
  const __nv_bfloat16* q;
  const void* const* k_spans;
  const void* const* v_spans;
  const int32_t* lens;
  float* ws_o;       // [slots][hpg][128]   level-0 partials (one or two per CTA)
  float* ws_ml;      // [slots][hpg][2]
  float* ws2_o;      // [slots][hpg][128]   level-1 partials (merged groups of kMergeFan pieces), indexed by the group's first slot
  float* ws2_ml;     // [slots][hpg][2]
  unsigned* counters;  // [batch * n_groups]  arrivals per (sequence, kv-head): pieces (direct merge) or groups (two-level)
  unsigned* counters1; // [slots]             arrivals per level-1 group
  int max_pieces;      // upper bound on pieces per (sequence, kv-head) (B2_ATTN_MAX_PIECES; effectively unbounded by default)
  int batch, n_heads, n_groups, hpg, span_len, span_shift, max_spans;
  int nstage;
  float scale_log2;
};

template <int QM>
struct KVTraits;
template <>
struct KVTraits<B2_KV_NONE> {
  static constexpr int ROW = 256;                   // bytes per token row
  static constexpr int TILE = kTile * ROW;          // 16 KB
  static constexpr int PARAM = 0;
};
template <>
struct KVTraits<B2_KV_I8> {
  static constexpr int ROW = 128;
  static constexpr int TILE = kTile * ROW;
  static constexpr int PARAM = kTile * 8;
};
template <>
struct KVTraits<B2_KV_U4> {
  static constexpr int ROW = 64;
  static constexpr int TILE = kTile * ROW;
  static constexpr int PARAM = kTile * 8;
};

// Issue the cp.async copies of one 64-token tile (K and V) of (sequence b, kv-head g) into a stage.
// Thread tid owns 16-byte chunk column (tid & (CPR-1)) of rows (tid / CPR) + i * (128 / CPR): the swizzled
// destination and the in-span source offset are per-thread constants, so one tile costs ~4 instructions per copy.
template <int QM>
__device__ __forceinline__ void load_tile(const AttnParams& p, uint8_t* stage, const void* const* ktab,
                                          const void* const* vtab, int g, int tok_base, int tok_end) {
  using T = KVTraits<QM>;
  constexpr int CPR = T::ROW / 16;            // 16B chunks per row: 16 / 8 / 4
  constexpr int RPI = kAttnThreads / CPR;     // rows covered per iteration: 8 / 16 / 32
  constexpr int ITERS = kTile / RPI;          // 8 / 4 / 2
  const int tid = threadIdx.x;
  const int row0 = tid / CPR, c = tid % CPR;
  const int nvalid = tok_end - tok_base;      // rows of this tile that hold live tokens (>= 1)
  const int sw = (QM == B2_KV_U4) ? (c ^ ((row0 >> 1) & 3)) : (c ^ (row0 & 7));
  uint8_t* dk = stage + row0 * T::ROW + sw * 16;
  uint8_t* dv = dk + T::TILE;
  const int pos0 = tok_base & (p.span_len - 1);  // tile offset inside its first span (0 unless span_len > 64)
  const int si0 = tok_base >> p.span_shift;
  const uint8_t* ks = nullptr;
  const uint8_t* vs = nullptr;
  int cur = -1;
#pragma unroll
  for (int i = 0; i < ITERS; ++i) {
    const int row = row0 + i * RPI;
    const bool valid = row < nvalid;
    const int sj = valid ? ((pos0 + row) >> p.span_shift) : 0;  // span of this row relative to si0
    if (sj != cur) {  // uniform per (i, span_len): 1, 2 or 4 table lookups per tile
      cur = sj;
      ks = reinterpret_cast<const uint8_t*>(ktab[si0 + sj]);
      vs = reinterpret_cast<const uint8_t*>(vtab[si0 + sj]);
    }
    const int pos = valid ? ((pos0 + row) & (p.span_len - 1)) : (pos0 & (p.span_len - 1));
    const size_t off = ((size_t)g * p.span_len + pos) * T::ROW + c * 16;
    cp_async16_zfill(dk + i * RPI * T::ROW, ks + off, valid);
    cp_async16_zfill(dv + i * RPI * T::ROW, vs + off, valid);
  }
  if (QM != B2_KV_NONE) {
    // per-token {zero, scale} for K and V: 64 x 8 B each = 32 x 16 B chunks each
    if (tid < 64) {
      const int which = tid >> 5, cc = tid & 31;  // 0: K, 1: V
      const int row = cc * 2;
      const bool valid = row < nvalid;
      const int rr = valid ? row : 0;
      const int sj = (pos0 + rr) >> p.span_shift, pos = (pos0 + rr) & (p.span_len - 1);
      const uint8_t* sp = reinterpret_cast<const uint8_t*>((which ? vtab : ktab)[si0 + sj]);
      const size_t poff = (size_t)p.n_groups * p.span_len * T::ROW + ((size_t)g * p.span_len + pos) * 8;
      cp_async16_zfill(stage + 2 * T::TILE + which * T::PARAM + cc * 16, sp + poff, valid);
    }
  }
}

// One 64-token tile of attention math for this warp's 16-token slice (cache in the 16-bit type FT: bf16, or fp16 when H).
template <bool H>
__device__ __forceinline__ void tile_compute_bf16(const uint8_t* st, int warp, int lane, int wtok, int tok1, float scale_log2,
                                                  const uint32_t (&qa)[8][4], float (&o)[16][4], float (&mrow)[2],
                                                  float (&lrow)[2]) {
  using T = KVTraits<B2_KV_NONE>;
  const int t = lane & 3;
  const uint32_t kb = smem_u32(st), vb = kb + T::TILE;
  // ---------- S = Q K^T : 2 n8 token tiles x 8 k16 steps
  float sc[2][4];
#pragma unroll
  for (int nt = 0; nt < 2; ++nt) sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 8; ks += 2) {
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      const int row = warp * 16 + nt * 8 + (lane & 7);
      const int chunk = 2 * ks + (lane >> 3);
      uint32_t r[4];
      ldmatrix_x4(r, kb + row * T::ROW + ((chunk ^ (row & 7)) << 4));
      Ft<H>::mma(sc[nt], qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3], r[0], r[1]);
      Ft<H>::mma(sc[nt], qa[ks + 1][0], qa[ks + 1][1], qa[ks + 1][2], qa[ks + 1][3], r[2], r[3]);
    }
  }
  // ---------- online softmax (base 2), rows gq and gq+8
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int cc = 0; cc < 4; ++cc) {
      const int tok = wtok + nt * 8 + 2 * t + (cc & 1);
      const float v = tok < tok1 ? sc[nt][cc] * scale_log2 : -INFINITY;
      sc[nt][cc] = v;
      mx[cc >> 1] = fmaxf(mx[cc >> 1], v);
    }
#pragma unroll
  for (int r2 = 0; r2 < 2; ++r2) {
    mx[r2] = fmaxf(mx[r2], __shfl_xor_sync(0xffffffffu, mx[r2], 1));
    mx[r2] = fmaxf(mx[r2], __shfl_xor_sync(0xffffffffu, mx[r2], 2));
  }
  float corr[2], psum[2] = {0.f, 0.f};
#pragma unroll
  for (int r2 = 0; r2 < 2; ++r2) {
    const float mnew = fmaxf(mrow[r2], mx[r2]);  // finite: the warp's first token is always live
    corr[r2] = exp2f(mrow[r2] - mnew);
    mrow[r2] = mnew;
  }
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int cc = 0; cc < 4; ++cc) {
      const float pv = exp2f(sc[nt][cc] - mrow[cc >> 1]);
      sc[nt][cc] = pv;
      psum[cc >> 1] += pv;
    }
#pragma unroll
  for (int r2 = 0; r2 < 2; ++r2) {
    psum[r2] += __shfl_xor_sync(0xffffffffu, psum[r2], 1);
    psum[r2] += __shfl_xor_sync(0xffffffffu, psum[r2], 2);
    lrow[r2] = lrow[r2] * corr[r2] + psum[r2];
  }
  if (corr[0] != 1.f || corr[1] != 1.f) {
#pragma unroll
    for (int dt = 0; dt < 16; ++dt) {
      o[dt][0] *= corr[0]; o[dt][1] *= corr[0];
      o[dt][2] *= corr[1]; o[dt][3] *= corr[1];
    }
  }
  const uint32_t pa0 = Ft<H>::pack(sc[0][0], sc[0][1]), pa1 = Ft<H>::pack(sc[0][2], sc[0][3]);
  const uint32_t pa2 = Ft<H>::pack(sc[1][0], sc[1][1]), pa3 = Ft<H>::pack(sc[1][2], sc[1][3]);
  // ---------- O += P V : 16 d-tiles, k16 = this warp's 16 tokens
#pragma unroll
  for (int dt = 0; dt < 16; dt += 2) {
    const int mi = lane >> 3;
    const int row = warp * 16 + 8 * (mi & 1) + (lane & 7);
    const int chunk = dt + (mi >> 1);
    uint32_t r[4];
    ldmatrix_x4_trans(r, vb + row * T::ROW + ((chunk ^ (row & 7)) << 4));
    Ft<H>::mma(o[dt], pa0, pa1, pa2, pa3, r[0], r[1]);
    Ft<H>::mma(o[dt + 1], pa0, pa1, pa2, pa3, r[2], r[3]);
  }
}

// ---- quantized KV (I8 / U4): the tensor cores run on the RAW cache integers converted exactly to fp16
// (1024 + u by byte/nibble permutes, no arithmetic); scale and zero are applied to the fp32 scores / folded into P:
//   score[h,tok] = s_k[tok] * ( sum_d Q[h,d]*(BIAS+u[tok,d]) - (BIAS + z_k[tok]) * sum_d Q[h,d] )
//   O[h,d]       = sum_tok P'[h,tok]*(BIAS+u[tok,d]) - sum_tok P'[h,tok]*(BIAS + z_v[tok]),   P' = P * s_v[tok]
// with BIAS = 1024+128 (int8, u = q+128) or 1024 (uint4).  Same math as QuantParam::Dequant
// (span-attention/src/cache_quant/impl_i8.cuh:66-70, impl_u4.cuh:97-106) without ever rounding a dequantized value.
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
  return d;
}

template <int QM>
__device__ __forceinline__ void tile_compute_q(const uint8_t* st, int warp, int lane, int wtok, int tok1, float scale_log2,
                                               const uint32_t (&qa)[8][4], const float (&sq)[2], float (&o)[16][4],
                                               float (&mrow)[2], float (&lrow)[2], float (&cacc)[2]) {
  using T = KVTraits<QM>;
  constexpr float BIAS = QM == B2_KV_I8 ? 1152.f : 1024.f;
  const int gq = lane >> 2, t = lane & 3;
  const uint32_t kb = smem_u32(st), vb = kb + T::TILE;
  const float2* kprm = reinterpret_cast<const float2*>(st + 2 * T::TILE);             // {zero, scale} per token
  const float2* vprm = reinterpret_cast<const float2*>(st + 2 * T::TILE + T::PARAM);
  // ---------- raw S = Q (BIAS + u)^T
  float sc[2][4];
#pragma unroll
  for (int nt = 0; nt < 2; ++nt) {
    sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
    const int row = warp * 16 + nt * 8 + gq;  // this thread's token for the B fragments
    if (QM == B2_KV_I8) {
#pragma unroll
      for (int c2 = 0; c2 < 2; ++c2) {  // chunks 2t, 2t+1: d = 32t + 16*c2 + (0..15)
        const uint4 kv = lds128(kb + row * T::ROW + ((((2 * t + c2) ^ (row & 7))) << 4));
        const uint32_t kw[4] = {kv.x ^ 0x80808080u, kv.y ^ 0x80808080u, kv.z ^ 0x80808080u, kv.w ^ 0x80808080u};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int ks = 4 * c2 + j;
          const uint32_t b0 = prmt(kw[j], 0x64646464u, 0x5140u), b1 = prmt(kw[j], 0x64646464u, 0x7362u);
          mma_f16_16816(sc[nt], qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3], b0, b1);
        }
      }
    } else {
      const uint4 kv = lds128(kb + row * T::ROW + ((t ^ ((row >> 1) & 3)) << 4));  // d = 32t + (0..31)
      const uint32_t kw[4] = {kv.x, kv.y, kv.z, kv.w};
#pragma unroll
      for (int wj = 0; wj < 4; ++wj) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int ks = 2 * wj + h;
          const uint32_t b0 = ((kw[wj] >> (8 * h)) & 0x000f000fu) | 0x64006400u;
          const uint32_t b1 = ((kw[wj] >> (8 * h + 4)) & 0x000f000fu) | 0x64006400u;
          mma_f16_16816(sc[nt], qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3], b0, b1);
        }
      }
    }
  }
  // ---------- dequantize the scores, online softmax (base 2)
  float mx[2] = {-INFINITY, -INFINITY};
  float vz[2][2], vs[2][2];  // V params of this thread's 4 tokens
#pragma unroll
  for (int nt = 0; nt < 2; ++nt) {
    const int tl = warp * 16 + nt * 8 + 2 * t;  // tile-local token of column 2t
    const float4 kp = *reinterpret_cast<const float4*>(kprm + tl);  // {z0, s0, z1, s1}
    const float4 vp = *reinterpret_cast<const float4*>(vprm + tl);
    // tokens at or beyond tok1 carry whatever the span memory held (the reference's span manager never zeroes frames,
    // and the 16-byte param chunk of an odd-length tail covers one unwritten token): their V params must not reach
    // the arithmetic (0 * NaN), so they are forced to zero exactly like the scores are forced to -inf
    const bool live0 = wtok + nt * 8 + 2 * t < tok1, live1 = wtok + nt * 8 + 2 * t + 1 < tok1;
    vz[nt][0] = live0 ? vp.x : 0.f; vs[nt][0] = live0 ? vp.y : 0.f;
    vz[nt][1] = live1 ? vp.z : 0.f; vs[nt][1] = live1 ? vp.w : 0.f;
#pragma unroll
    for (int cc = 0; cc < 4; ++cc) {
      const int tok = wtok + nt * 8 + 2 * t + (cc & 1);
      const float kz = (cc & 1) ? kp.z : kp.x, ksc = (cc & 1) ? kp.w : kp.y;
      const float raw = ksc * (sc[nt][cc] - (BIAS + kz) * sq[cc >> 1]);
      const float v = tok < tok1 ? raw * scale_log2 : -INFINITY;
      sc[nt][cc] = v;
      mx[cc >> 1] = fmaxf(mx[cc >> 1], v);
    }
  }
#pragma unroll
  for (int r2 = 0; r2 < 2; ++r2) {
    mx[r2] = fmaxf(mx[r2], __shfl_xor_sync(0xffffffffu, mx[r2], 1));
    mx[r2] = fmaxf(mx[r2], __shfl_xor_sync(0xffffffffu, mx[r2], 2));
  }
  float corr[2], psum[2] = {0.f, 0.f}, csum[2] = {0.f, 0.f};
#pragma unroll
  for (int r2 = 0; r2 < 2; ++r2) {
    const float mnew = fmaxf(mrow[r2], mx[r2]);
    corr[r2] = exp2f(mrow[r2] - mnew);
    mrow[r2] = mnew;
  }
  uint32_t pa[4];
#pragma unroll
  for (int nt = 0; nt < 2; ++nt) {
    float pq[4];
#pragma unroll
    for (int cc = 0; cc < 4; ++cc) {
      const float pv = exp2f(sc[nt][cc] - mrow[cc >> 1]);
      psum[cc >> 1] += pv;
      pq[cc] = pv * vs[nt][cc & 1];  // fold the V scale into the probability
    }
    pa[2 * nt] = pack_f16x2(pq[0], pq[1]);
    pa[2 * nt + 1] = pack_f16x2(pq[2], pq[3]);
    // zero-point term with the SAME fp16-rounded probabilities the tensor core sees
    const __half2 h01 = *reinterpret_cast<const __half2*>(&pa[2 * nt]), h23 = *reinterpret_cast<const __half2*>(&pa[2 * nt + 1]);
    csum[0] += __low2float(h01) * (BIAS + vz[nt][0]) + __high2float(h01) * (BIAS + vz[nt][1]);
    csum[1] += __low2float(h23) * (BIAS + vz[nt][0]) + __high2float(h23) * (BIAS + vz[nt][1]);
  }
#pragma unroll
  for (int r2 = 0; r2 < 2; ++r2) {
    psum[r2] += __shfl_xor_sync(0xffffffffu, psum[r2], 1);
    psum[r2] += __shfl_xor_sync(0xffffffffu, psum[r2], 2);
    lrow[r2] = lrow[r2] * corr[r2] + psum[r2];
    cacc[r2] = cacc[r2] * corr[r2] + csum[r2];  // per-thread partial (its 4 tokens); reduced over the quad at the end
  }
  if (corr[0] != 1.f || corr[1] != 1.f) {
#pragma unroll
    for (int dt = 0; dt < 16; ++dt) {
      o[dt][0] *= corr[0]; o[dt][1] *= corr[0];
      o[dt][2] *= corr[1]; o[dt][3] *= corr[1];
    }
  }
  // ---------- raw O += P' (BIAS + u): ldmatrix.trans on 16-bit units of the raw rows
  const int mi = lane >> 3;
  const int vrow = warp * 16 + 8 * (mi & 1) + (lane & 7);
  if (QM == B2_KV_I8) {
#pragma unroll
    for (int c = 0; c < 8; c += 2) {
      uint32_t r[4];
      ldmatrix_x4_trans(r, vb + vrow * T::ROW + (((c + (mi >> 1)) ^ (vrow & 7)) << 4));
#pragma unroll
      for (int u = 0; u < 2; ++u) {  // chunk c+u: bytes {V[2t][2g], V[2t][2g+1], V[2t+1][2g], V[2t+1][2g+1]}
        const uint32_t lo = r[2 * u] ^ 0x80808080u, hi = r[2 * u + 1] ^ 0x80808080u;
        mma_f16_16816(o[2 * (c + u)], pa[0], pa[1], pa[2], pa[3], prmt(lo, 0x64646464u, 0x6240u), prmt(hi, 0x64646464u, 0x6240u));
        mma_f16_16816(o[2 * (c + u) + 1], pa[0], pa[1], pa[2], pa[3], prmt(lo, 0x64646464u, 0x7351u), prmt(hi, 0x64646464u, 0x7351u));
      }
    }
  } else {
#pragma unroll
    for (int c = 0; c < 4; c += 2) {
      uint32_t r[4];
      ldmatrix_x4_trans(r, vb + vrow * T::ROW + (((c + (mi >> 1)) ^ ((vrow >> 1) & 3)) << 4));
#pragma unroll
      for (int u = 0; u < 2; ++u) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const uint32_t b0 = ((r[2 * u] >> (4 * i)) & 0x000f000fu) | 0x64006400u;
          const uint32_t b1 = ((r[2 * u + 1] >> (4 * i)) & 0x000f000fu) | 0x64006400u;
          mma_f16_16816(o[4 * (c + u) + i], pa[0], pa[1], pa[2], pa[3], b0, b1);
        }
      }
    }
  }
}

// Merge n split-KV partials of one (sequence, kv-head): source i lives in slot `slot0 + i * stride2 (+ par0 for i == 0)`
// of (src_o, src_ml).  All 128 threads take part; a thread owns (head row, 4 consecutive d) units and the sources are
// visited in index order with fp32 arithmetic only => deterministic.  The partials sit in L2 (other CTAs wrote them), so the
// cost is L2 round trips: the (max, sum) pairs of ALL sources and the first 8 sources' rows are requested together, i.e. a
// merge of up to 8 sources (every level-1 group, most final merges) is ONE round trip; longer lists take one more per 8.
// FINAL writes softmax-normalised bf16 rows of `out`; otherwise the merged, still unnormalised partial goes to slot
// `dst_slot` of (dst_o, dst_ml).  s_w: shared scratch [kMergeMaxSrc][16] floats (weights), s_ML: [16][2].
constexpr int kMergeMaxSrc = 96;  // sources of one merge call (final level: ceil(pieces / kMergeFan)); more -> looped M pass
template <bool FINAL, bool H>
__device__ __forceinline__ void merge_partials(const float* src_o, const float* src_ml, int slot0, int stride2, int par0, int n,
                                               int hpg, __nv_bfloat16* out_rows, float* dst_o, float* dst_ml, int dst_slot,
                                               float* s_w, float* s_ML) {
  const int tid = threadIdx.x;
  auto slot_of = [&](int i) { return slot0 + i * stride2 + (i == 0 ? par0 : 0); };
  const int nunits = hpg * 32;  // (row, float4) units
  // ---- request the first batch of rows and every (m, l) pair before waiting for anything
  float4 v[2][8];
#pragma unroll
  for (int uu = 0; uu < 2; ++uu) {
    const int u = tid + uu * kAttnThreads;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      v[uu][i] = (u < nunits && i < n) ? __ldcg(reinterpret_cast<const float4*>(src_o + ((size_t)slot_of(i) * hpg + (u >> 5)) * kHead) + (u & 31))
                                       : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int k = tid; k < n * hpg; k += kAttnThreads) {  // k = i * hpg + r
    const int i = k / hpg, r = k - i * hpg;
    const float2 ml = __ldcg(reinterpret_cast<const float2*>(src_ml + ((size_t)slot_of(i) * hpg + r) * 2));
    if (i < kMergeMaxSrc) { s_w[i * 16 + r] = ml.x; s_w[(kMergeMaxSrc + i) * 16 + r] = ml.y; }
  }
  __syncthreads();
  const int nn = min(n, kMergeMaxSrc);  // (n > kMergeMaxSrc cannot happen: pieces <= grid, fan-in 8, grid <= 8 * kMergeMaxSrc)
  if (tid < hpg) {  // per row: global max, weights, denominator (fixed source order)
    float M = -INFINITY;
    for (int i = 0; i < nn; ++i) M = fmaxf(M, s_w[i * 16 + tid]);
    float L = 0.f;
    for (int i = 0; i < nn; ++i) {
      const float m = s_w[i * 16 + tid];
      const float w = m == -INFINITY ? 0.f : exp2f(m - M);
      L += w * s_w[(kMergeMaxSrc + i) * 16 + tid];
      s_w[i * 16 + tid] = w;
    }
    s_ML[tid * 2] = M;
    s_ML[tid * 2 + 1] = L;
  }
  __syncthreads();
  float4 acc[2];
#pragma unroll
  for (int uu = 0; uu < 2; ++uu) {
    const int r = (tid + uu * kAttnThreads) >> 5;
    acc[uu] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float w = (i < nn && r < hpg) ? s_w[i * 16 + r] : 0.f;
      acc[uu].x += w * v[uu][i].x; acc[uu].y += w * v[uu][i].y; acc[uu].z += w * v[uu][i].z; acc[uu].w += w * v[uu][i].w;
    }
  }
  for (int i0 = 8; i0 < nn; i0 += 8) {  // longer lists: one more round trip per 8 sources
#pragma unroll
    for (int uu = 0; uu < 2; ++uu) {
      const int u = tid + uu * kAttnThreads;
#pragma unroll
      for (int i = 0; i < 8; ++i)
        v[uu][i] = (u < nunits && i0 + i < nn) ? __ldcg(reinterpret_cast<const float4*>(src_o + ((size_t)slot_of(i0 + i) * hpg + (u >> 5)) * kHead) + (u & 31))
                                               : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int uu = 0; uu < 2; ++uu) {
      const int r = (tid + uu * kAttnThreads) >> 5;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float w = (i0 + i < nn && r < hpg) ? s_w[(i0 + i) * 16 + r] : 0.f;
        acc[uu].x += w * v[uu][i].x; acc[uu].y += w * v[uu][i].y; acc[uu].z += w * v[uu][i].z; acc[uu].w += w * v[uu][i].w;
      }
    }
  }
  // hpg <= 16: up to 512 units, two per thread cover 8 rows; the remaining rows (hpg > 8) take a second sweep
  for (int sweep = 0; sweep < 2; ++sweep) {
    if (sweep == 1) {
      if (hpg <= 8) break;
#pragma unroll
      for (int uu = 0; uu < 2; ++uu) {
        const int u = tid + (uu + 2) * kAttnThreads;
        acc[uu] = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int i = 0; i < nn; ++i) {
          if (u < nunits) {
            const float4 x = __ldcg(reinterpret_cast<const float4*>(src_o + ((size_t)slot_of(i) * hpg + (u >> 5)) * kHead) + (u & 31));
            const float w = s_w[i * 16 + (u >> 5)];
            acc[uu].x += w * x.x; acc[uu].y += w * x.y; acc[uu].z += w * x.z; acc[uu].w += w * x.w;
          }
        }
      }
    }
#pragma unroll
    for (int uu = 0; uu < 2; ++uu) {
      const int u = tid + (uu + 2 * sweep) * kAttnThreads;
      if (u >= nunits) continue;
      const int r = u >> 5, c4 = u & 31;
      if (FINAL) {
        const float inv = 1.f / s_ML[r * 2 + 1];
        *reinterpret_cast<uint2*>(out_rows + (size_t)r * kHead + c4 * 4) =
            make_uint2(Ft<H>::pack(acc[uu].x * inv, acc[uu].y * inv), Ft<H>::pack(acc[uu].z * inv, acc[uu].w * inv));
      } else {
        const size_t row = (size_t)dst_slot * hpg + r;
        *(reinterpret_cast<float4*>(dst_o + row * kHead) + c4) = acc[uu];
        if (c4 == 0) *reinterpret_cast<float2*>(dst_ml + row * 2) = make_float2(s_ML[r * 2], s_ML[r * 2 + 1]);
      }
    }
  }
  __syncthreads();  // s_w / s_ML are reused by the next merge of this CTA
}

// Work decomposition: the flat list of (sequence, kv-head, tile) is cut into equal ranges of Tc tiles, one per CTA
// (stream-K style): every CTA moves the same number of bytes whatever the batch/length mix.  A (sequence, kv-head)
// covered by several CTAs is merged by the last CTA to finish it (device counter, fixed order => deterministic).
B2_TRACE_DECL(g_attn_tr)
#ifdef B2_TRACE
extern "C" int b2_debug_trace_attn(unsigned long long* host_out) { return (int)cudaMemcpyFromSymbol(host_out, g_attn_tr, sizeof(g_attn_tr)); }
#endif

template <int QM, bool H>
__global__ void __launch_bounds__(kAttnThreads) span_attn_kernel(const AttnParams p) {
  using F = Ft<H>;  // the 16-bit type of Q, the output and an unquantized cache
  using T = KVTraits<QM>;
  constexpr int STAGE = 2 * T::TILE + 2 * T::PARAM;
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ int s_prefix[kMaxBatch + 1];  // flat tile index of each sequence's first tile (x n_groups)
  __shared__ int s_red[8];
  __shared__ int s_is_last;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int gq = lane >> 2, t = lane & 3;

  const bool tr0 = blockIdx.x == 0 && threadIdx.x == 0;
  if (tr0) B2_TR(g_attn_tr, 0);
  const unsigned long long t_entry = 0;
  (void)t_entry;
  pdl_wait();  // the newest token's K/V (and q) come from the preceding append kernel
  pdl_launch_dependents();
  if (tr0) B2_TR(g_attn_tr, 1);

  // ---------------- device-side work decomposition (ONE global round trip: the lengths) ----------------
  {
    int my_tiles = 0, my_max = 0;
    for (int b = tid; b < p.batch; b += kAttnThreads) {
      const int tl = (p.lens[b] + kTile - 1) / kTile;
      s_prefix[b] = tl;  // tile count for now; warp 0 turns it into the exclusive scan below
      my_tiles += tl;
      my_max = max(my_max, tl);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      my_tiles += __shfl_xor_sync(0xffffffffu, my_tiles, o);
      my_max = max(my_max, __shfl_xor_sync(0xffffffffu, my_max, o));
    }
    if (lane == 0) { s_red[warp] = my_tiles; s_red[4 + warp] = my_max; }
  }
  __syncthreads();
  const int total = (s_red[0] + s_red[1] + s_red[2] + s_red[3]) * p.n_groups;
  const int max_tiles = max(max(s_red[4], s_red[5]), max(s_red[6], s_red[7]));
  int Tc = (total + (int)gridDim.x - 1) / (int)gridDim.x;
  Tc = max(Tc, (max_tiles + p.max_pieces - 1) / p.max_pieces);  // optional bound on pieces per (sequence, kv-head)
  Tc = max(Tc, 1);
  const int lo = blockIdx.x * Tc, hi = min(total, lo + Tc);
  if (lo >= hi) return;
  if (warp == 0) {  // exclusive scan of tiles*n_groups per sequence
    int carry = 0;
    for (int b0 = 0; b0 < p.batch; b0 += 32) {
      const int b = b0 + lane;
      int v = b < p.batch ? s_prefix[b] * p.n_groups : 0, x = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      if (b < p.batch) s_prefix[b] = carry + x - v;
      carry += __shfl_sync(0xffffffffu, x, 31);
    }
    if (lane == 0) s_prefix[p.batch] = carry;
  }
  __syncthreads();

  if (tr0) B2_TR(g_attn_tr, 2);
  float* mrg = reinterpret_cast<float*>(smem);                 // [4][16][kMergeRS] after the ring is drained
  float* mrg_ml = mrg + 4 * 16 * kMergeRS;                      // [4][16][2]
  // scratch of the cross-CTA partial merge: (m -> weight, l) per (source, head row).  It aliases the warp-merge buffer, which
  // is dead by then (its result went to the workspace before the arrival counter was bumped)
  float* s_w = mrg;                                             // [2][kMergeMaxSrc][16]
  float* s_ML = mrg + 2 * kMergeMaxSrc * 16;                    // [16][2]

  int pos = lo;
  while (pos < hi) {
    // ---- locate (b, g, first tile) of the piece starting at flat index pos
    int blo = 0, bhi = p.batch - 1;
    while (blo < bhi) {
      const int mid = (blo + bhi + 1) >> 1;
      if (s_prefix[mid] <= pos) blo = mid; else bhi = mid - 1;
    }
    const int b = blo;
    const int len = p.lens[b];
    const int tiles_b = (len + kTile - 1) / kTile;
    const int within = pos - s_prefix[b];
    const int g = within / tiles_b, t0 = within - g * tiles_b;
    const int bg_start = s_prefix[b] + g * tiles_b, bg_end = bg_start + tiles_b;
    const int pend = min(hi, bg_end);
    const int ntiles = pend - pos;
    const int tok0 = t0 * kTile;
    const int tok1 = min(len, (t0 + ntiles) * kTile);
    const int k0 = bg_start / Tc;
    const int npieces = (bg_end - 1) / Tc - k0 + 1;
    const void* const* ktab = p.k_spans + (size_t)b * p.max_spans;
    const void* const* vtab = p.v_spans + (size_t)b * p.max_spans;

    // ---- start streaming: the piece's first nstage-1 tiles are requested NOW (span-table lookups + cp.async), so their
    //      HBM latency overlaps the load of the query rows below
    for (int i = 0; i < p.nstage - 1; ++i) {
      if (i < ntiles) load_tile<QM>(p, smem + i * STAGE, ktab, vtab, g, tok0 + i * kTile, tok1);
      cp_async_commit();
    }

    // ---- Q fragments (A operand, rows = q-heads of this kv-group).  The head-dim order each thread uses is free as
    //      long as Q and K agree, so it follows how that thread reads K: natural for bf16 (ldmatrix), per-thread
    //      contiguous 32-d slices for the quantized modes.  Quantized modes run the MMAs in fp16.
    uint32_t qa[8][4];
    float sq[2] = {0.f, 0.f};  // sum_d Q[row][d] over this thread's d-slice, then over the quad (quantized modes)
    {
      // quantized modes: stage the group's hpg x 128 query rows through shared memory with 16-byte loads (one global round
      // trip; their fragment orders would otherwise need 64 scalar loads per thread: 3.3 us measured at ctx 32768)
      // [16][128] in the LAST ring stage: the only one the prefetch above does not write (it is first filled at iteration 0)
      __nv_bfloat16* qs = reinterpret_cast<__nv_bfloat16*>(smem + (p.nstage - 1) * STAGE);
      const __nv_bfloat16* qb = p.q + ((size_t)b * p.n_heads + (size_t)g * p.hpg) * kHead;
      if (QM != B2_KV_NONE) {
        for (int i = tid; i < 16 * (kHead / 8); i += kAttnThreads) {
          const int row = i >> 4;
          *reinterpret_cast<uint4*>(qs + row * kHead + (i & 15) * 8) =
              row < p.hpg ? *reinterpret_cast<const uint4*>(qb + row * kHead + (i & 15) * 8) : make_uint4(0, 0, 0, 0);
        }
        __syncthreads();
      }
      const bool r0 = gq < p.hpg, r1 = (gq + 8) < p.hpg;
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        if (QM == B2_KV_NONE) {  // natural d order: 32 independent 4-byte loads per thread straight from global memory
          const int d0 = 16 * ks + 2 * t;
          qa[ks][0] = r0 ? *reinterpret_cast<const uint32_t*>(qb + gq * kHead + d0) : 0u;
          qa[ks][1] = r1 ? *reinterpret_cast<const uint32_t*>(qb + (gq + 8) * kHead + d0) : 0u;
          qa[ks][2] = r0 ? *reinterpret_cast<const uint32_t*>(qb + gq * kHead + d0 + 8) : 0u;
          qa[ks][3] = r1 ? *reinterpret_cast<const uint32_t*>(qb + (gq + 8) * kHead + d0 + 8) : 0u;
        } else {
          int da[2], db[2];  // d of (reg lo, reg hi) for the k-columns (2t,2t+1) and (2t+8,2t+9)
          if (QM == B2_KV_I8) {
            da[0] = 32 * t + 4 * ks; da[1] = da[0] + 1; db[0] = da[0] + 2; db[1] = da[0] + 3;
          } else {
            const int base = 32 * t + 8 * (ks >> 1) + 2 * (ks & 1);
            da[0] = base; da[1] = base + 4; db[0] = base + 1; db[1] = base + 5;
          }
          float f[2][4];
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const __nv_bfloat16* qr = qs + (gq + 8 * rr) * kHead;
            f[rr][0] = F::to_f(qr[da[0]]);
            f[rr][1] = F::to_f(qr[da[1]]);
            f[rr][2] = F::to_f(qr[db[0]]);
            f[rr][3] = F::to_f(qr[db[1]]);
          }
          qa[ks][0] = pack_f16x2(f[0][0], f[0][1]);
          qa[ks][1] = pack_f16x2(f[1][0], f[1][1]);
          qa[ks][2] = pack_f16x2(f[0][2], f[0][3]);
          qa[ks][3] = pack_f16x2(f[1][2], f[1][3]);
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {  // sums of exactly the fp16 values the tensor core multiplies
            const __half2 ha = *reinterpret_cast<const __half2*>(&qa[ks][rr]), hb = *reinterpret_cast<const __half2*>(&qa[ks][2 + rr]);
            sq[rr] += (__low2float(ha) + __high2float(ha)) + (__low2float(hb) + __high2float(hb));
          }
        }
      }
      if (QM != B2_KV_NONE) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          sq[rr] += __shfl_xor_sync(0xffffffffu, sq[rr], 1);
          sq[rr] += __shfl_xor_sync(0xffffffffu, sq[rr], 2);
        }
      }
      if (QM != B2_KV_NONE) __syncthreads();  // the ring's last stage may be filled now
    }
    float cacc[2] = {0.f, 0.f};
    if (tr0) B2_TR(g_attn_tr, 3);

    float o[16][4];
#pragma unroll
    for (int i = 0; i < 16; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};

    // ---- cp.async ring over the piece's tiles (its first nstage-1 tiles were requested before the Q fragments were built)
    int slot = 0, pslot = p.nstage - 1;
    for (int i = 0; i < ntiles; ++i) {
      const int pf = i + p.nstage - 1;
      if (pf < ntiles) load_tile<QM>(p, smem + pslot * STAGE, ktab, vtab, g, tok0 + pf * kTile, tok1);
      cp_async_commit();
      // all groups except the newest (nstage-1) are complete -> tile i has landed
      if (p.nstage == 2) cp_async_wait<1>(); else if (p.nstage == 3) cp_async_wait<2>(); else cp_async_wait<3>();
      __syncthreads();
      if (tr0 && i == 0) B2_TR(g_attn_tr, 4);
      const int wtok = tok0 + i * kTile + warp * 16;  // first token of this warp's slice
      if (wtok < tok1) {
        if (QM == B2_KV_NONE) tile_compute_bf16<H>(smem + slot * STAGE, warp, lane, wtok, tok1, p.scale_log2, qa, o, mrow, lrow);
        else tile_compute_q<QM == B2_KV_NONE ? B2_KV_I8 : QM>(smem + slot * STAGE, warp, lane, wtok, tok1, p.scale_log2, qa, sq, o, mrow, lrow, cacc);
      }
      __syncthreads();  // this stage may be refilled by the next iteration's prefetch
      slot = slot + 1 == p.nstage ? 0 : slot + 1;
      pslot = pslot + 1 == p.nstage ? 0 : pslot + 1;
    }
    cp_async_wait<0>();
    if (tr0) B2_TR(g_attn_tr, 5);

    // ---------------- merge the 4 warps (each saw a disjoint token slice) ----------------
    if (QM != B2_KV_NONE) {  // subtract the zero-point term (quad-reduced) before leaving registers
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        cacc[rr] += __shfl_xor_sync(0xffffffffu, cacc[rr], 1);
        cacc[rr] += __shfl_xor_sync(0xffffffffu, cacc[rr], 2);
      }
#pragma unroll
      for (int dt = 0; dt < 16; ++dt) {
        o[dt][0] -= cacc[0]; o[dt][1] -= cacc[0];
        o[dt][2] -= cacc[1]; o[dt][3] -= cacc[1];
      }
    }
    {
      float* m0 = mrg + (warp * 16 + gq) * kMergeRS;
      float* m1 = mrg + (warp * 16 + gq + 8) * kMergeRS;
      if (QM == B2_KV_NONE) {
#pragma unroll
        for (int dt = 0; dt < 16; ++dt) {
          const int d = 8 * dt + 2 * t;
          *reinterpret_cast<float2*>(m0 + d) = make_float2(o[dt][0], o[dt][1]);
          *reinterpret_cast<float2*>(m1 + d) = make_float2(o[dt][2], o[dt][3]);
        }
      } else if (QM == B2_KV_I8) {  // o[2c] <-> d = 16c+4t+{0,2}, o[2c+1] <-> d = 16c+4t+{1,3}
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const int d = 16 * c + 4 * t;
          *reinterpret_cast<float4*>(m0 + d) = make_float4(o[2 * c][0], o[2 * c + 1][0], o[2 * c][1], o[2 * c + 1][1]);
          *reinterpret_cast<float4*>(m1 + d) = make_float4(o[2 * c][2], o[2 * c + 1][2], o[2 * c][3], o[2 * c + 1][3]);
        }
      } else {  // o[4c+i] <-> d = 32c+8t+i and 32c+8t+4+i
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int d = 32 * c + 8 * t;
          *reinterpret_cast<float4*>(m0 + d) = make_float4(o[4 * c][0], o[4 * c + 1][0], o[4 * c + 2][0], o[4 * c + 3][0]);
          *reinterpret_cast<float4*>(m0 + d + 4) = make_float4(o[4 * c][1], o[4 * c + 1][1], o[4 * c + 2][1], o[4 * c + 3][1]);
          *reinterpret_cast<float4*>(m1 + d) = make_float4(o[4 * c][2], o[4 * c + 1][2], o[4 * c + 2][2], o[4 * c + 3][2]);
          *reinterpret_cast<float4*>(m1 + d + 4) = make_float4(o[4 * c][3], o[4 * c + 1][3], o[4 * c + 2][3], o[4 * c + 3][3]);
        }
      }
    }
    if (t == 0) {
      mrg_ml[(warp * 16 + gq) * 2] = mrow[0];
      mrg_ml[(warp * 16 + gq) * 2 + 1] = lrow[0];
      mrg_ml[(warp * 16 + gq + 8) * 2] = mrow[1];
      mrg_ml[(warp * 16 + gq + 8) * 2 + 1] = lrow[1];
    }
    __syncthreads();
    // thread d = tid handles column d of every head row
    const int cnt_idx = b * p.n_groups + g;
    const int my_slot = 2 * blockIdx.x + (pos != lo ? 1 : 0);
    for (int r = 0; r < p.hpg; ++r) {
      float M = -INFINITY;
#pragma unroll
      for (int w = 0; w < 4; ++w) M = fmaxf(M, mrg_ml[(w * 16 + r) * 2]);
      float L = 0.f, acc = 0.f;
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const float mw = mrg_ml[(w * 16 + r) * 2];
        const float f = mw == -INFINITY ? 0.f : exp2f(mw - M);
        L += f * mrg_ml[(w * 16 + r) * 2 + 1];
        acc += f * mrg[(w * 16 + r) * kMergeRS + tid];
      }
      if (npieces == 1) {
        p.out[((size_t)b * p.n_heads + (size_t)g * p.hpg + r) * kHead + tid] = F::from_f(acc / L);
      } else {
        p.ws_o[((size_t)my_slot * p.hpg + r) * kHead + tid] = acc;
        if (tid == 0) {
          p.ws_ml[((size_t)my_slot * p.hpg + r) * 2] = M;
          p.ws_ml[((size_t)my_slot * p.hpg + r) * 2 + 1] = L;
        }
      }
    }
    if (tr0) B2_TR(g_attn_tr, 6);
    if (npieces > 1) {
      __threadfence();
      __syncthreads();
      if (tr0) B2_TR(g_attn_tr, 7);
      // pieces of this (sequence, kv-head) come from CTAs k0 .. k0+npieces-1 (one each); only CTA k0's piece can start
      // inside its range (slot parity 1)
      const int first_par = bg_start > k0 * Tc ? 1 : 0;
      __nv_bfloat16* out_rows = p.out + ((size_t)b * p.n_heads + (size_t)g * p.hpg) * kHead;
      if (npieces <= kMergeDirect) {
        if (tid == 0) s_is_last = atomicAdd(&p.counters[cnt_idx], 1u) == (unsigned)(npieces - 1);
        __syncthreads();
        if (s_is_last) {
          __threadfence();
          if (tid == 0 && cnt_idx == 0) B2_TR(g_attn_tr, 10);
          merge_partials<true, H>(p.ws_o, p.ws_ml, 2 * k0, 2, first_par, npieces, p.hpg, out_rows, nullptr, nullptr, 0, s_w, s_ML);
          if (tid == 0) p.counters[cnt_idx] = 0;  // re-arm
          if (tid == 0 && cnt_idx == 0) B2_TR(g_attn_tr, 11);
        }
      } else {
        // two-level: the last CTA of each group of kMergeFan consecutive pieces merges the group into a level-1 partial;
        // the last group to finish merges the level-1 partials.  The merge work of a long sequence is spread over
        // npieces / kMergeFan CTAs instead of serialising behind one.
        const int j = (int)blockIdx.x - k0;
        const int q = j / kMergeFan;
        const int gsize = min(kMergeFan, npieces - q * kMergeFan);
        const int ngroups = (npieces + kMergeFan - 1) / kMergeFan;
        const int lead = 2 * (k0 + q * kMergeFan) + (q == 0 ? first_par : 0);  // slot of the group's first piece
        if (tid == 0) s_is_last = atomicAdd(&p.counters1[lead], 1u) == (unsigned)(gsize - 1);
        __syncthreads();
        if (s_is_last) {
          __threadfence();
          if (tid == 0 && cnt_idx == 0 && q == 0) B2_TR(g_attn_tr, 8);
          merge_partials<false, H>(p.ws_o, p.ws_ml, 2 * (k0 + q * kMergeFan), 2, q == 0 ? first_par : 0, gsize, p.hpg, nullptr,
                                p.ws2_o, p.ws2_ml, lead, s_w, s_ML);
          if (tid == 0 && cnt_idx == 0 && q == 0) B2_TR(g_attn_tr, 9);
          if (tid == 0) p.counters1[lead] = 0;
          __threadfence();
          __syncthreads();
          if (tid == 0) s_is_last = atomicAdd(&p.counters[cnt_idx], 1u) == (unsigned)(ngroups - 1);
          __syncthreads();
          if (s_is_last) {
            __threadfence();
            if (tid == 0 && cnt_idx == 0) B2_TR(g_attn_tr, 10);
            merge_partials<true, H>(p.ws2_o, p.ws2_ml, 2 * k0, 2 * kMergeFan, first_par, ngroups, p.hpg, out_rows, nullptr, nullptr, 0, s_w, s_ML);
            if (tid == 0) p.counters[cnt_idx] = 0;
            if (tid == 0 && cnt_idx == 0) B2_TR(g_attn_tr, 11);
          }
        }
      }
    }
    __syncthreads();  // merge buffer aliases the ring
    pos = pend;
  }
}

// ---- QuantParam<I8/U4>::Builder + Quant (impl_i8.cuh:54-61,106-140, impl_u4.cuh:146-182) with the arithmetic the
// reference's kernels really execute: the span-cache writers are built with --use_fast_math, which turns
//   Div(maxVal - minVal, RANGE)   into a multiply by the constant fl(1/RANGE),
//   Div(x, qs) = __fdividef(x,qs) into x * MUFU.RCP(qs), contracted with the following add into one FFMA,
//   rintf + static_cast           into one round-to-nearest-even conversion,
// all flush-to-zero (SASS of QuantCacheAppendKernel / QuantSpanCopyKernel: FADD, FMUL 0x3b808081 / 0x3d888889, FMNMX 1e-5,
// MUFU.RCP, FFMA, FMNMX, FRND, FFMA x4, FMNMX, F2I).  Repeating exactly that sequence makes the span bytes and the stored
// {zero, scale} bit-identical to the reference's on the same GPU (tests/test_ref_pin_gpu.py); an IEEE division differs
// from it on the rows whose zero point is an exact tie (max == -min: ~0.5 % of N(0,1) bf16 rows).
// One warp per 128-wide row, 4 consecutive values per lane.
template <int QM>
__device__ __forceinline__ void quant_row(const float (&x)[4], float& qz, float& qs, int (&qv)[4]) {
  float mx = fmaxf(fmaxf(x[0], x[1]), fmaxf(x[2], x[3])), mn = fminf(fminf(x[0], x[1]), fminf(x[2], x[3]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
  }
  const float INV_RANGE = QM == B2_KV_I8 ? __uint_as_float(0x3b808081u) : __uint_as_float(0x3d888889u);  // fl(1/255), fl(1/15)
  const float ORIGIN = QM == B2_KV_I8 ? -128.f : 0.f, QMAX = QM == B2_KV_I8 ? 127.f : 15.f;
  float rq;
  asm("{\n\t.reg .f32 d;\n\t"
      "sub.rn.ftz.f32 d, %3, %4;\n\t"
      "mul.rn.ftz.f32 d, d, %5;\n\t"
      "max.ftz.f32 %0, d, 0f3727C5AC;\n\t"       // EPS = 1e-5f
      "rcp.approx.ftz.f32 %1, %0;\n\t"
      "neg.ftz.f32 d, %4;\n\t"
      "fma.rn.ftz.f32 %2, d, %1, %6;\n\t}"
      : "=&f"(qs), "=&f"(rq), "=&f"(qz)
      : "f"(mx), "f"(mn), "f"(INV_RANGE), "f"(ORIGIN));
  qz = fminf(qz, QMAX);
  if (QM == B2_KV_I8) qz = fmaxf(qz, -128.f);
  asm("cvt.rni.ftz.f32.f32 %0, %0;" : "+f"(qz));
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float tq;
    asm("fma.rn.ftz.f32 %0, %1, %2, %3;" : "=f"(tq) : "f"(x[i]), "f"(rq), "f"(qz));
    tq = fminf(tq, QMAX);
    if (QM == B2_KV_I8) {
      tq = fmaxf(tq, -128.f);
      asm("cvt.rni.ftz.s32.f32 %0, %1;" : "=r"(qv[i]) : "f"(tq));
    } else {
      asm("cvt.rni.ftz.u32.f32 %0, %1;" : "=r"(qv[i]) : "f"(tq));  // saturates negatives to 0
    }
  }
}

// store one (possibly quantized) 128-wide row at row index rowi of a span ([n_rows][row] data, then [n_rows] {zero, scale})
template <int QM, bool H>
__device__ __forceinline__ void store_row(uint8_t* span, size_t rowi, int n_rows, int lane, const float (&x)[4]) {
  if (QM == B2_KV_NONE) {
    *reinterpret_cast<uint2*>(span + rowi * 256 + lane * 8) = make_uint2(Ft<H>::pack(x[0], x[1]), Ft<H>::pack(x[2], x[3]));
    return;
  }
  float qz, qs;
  int qv[4];
  quant_row<QM == B2_KV_NONE ? B2_KV_I8 : QM>(x, qz, qs, qv);
  if (QM == B2_KV_I8) {
    const uint32_t w = (qv[0] & 0xff) | ((qv[1] & 0xff) << 8) | ((qv[2] & 0xff) << 16) | ((uint32_t)(qv[3] & 0xff) << 24);
    *reinterpret_cast<uint32_t*>(span + rowi * 128 + lane * 4) = w;
    if (lane == 0) *reinterpret_cast<float2*>(span + (size_t)n_rows * 128 + rowi * 8) = make_float2(qz, qs);
  } else {
    const uint16_t w = (uint16_t)((qv[0] & 0xf) | ((qv[1] & 0xf) << 4) | ((qv[2] & 0xf) << 8) | ((qv[3] & 0xf) << 12));
    *reinterpret_cast<uint16_t*>(span + rowi * 64 + lane * 2) = w;
    if (lane == 0) *reinterpret_cast<float2*>(span + (size_t)n_rows * 64 + rowi * 8) = make_float2(qz, qs);
  }
}

// ------------------------------------------------------------------------------------------------
// prefill: contiguous K (or V) rows of one sequence -> its spans (ContextSpanCopyLauncher,
// csrc/core/kernel/cuda/cache/context_span_copy.cuh:47-106): one warp per (token, kv-head) row
// ------------------------------------------------------------------------------------------------
struct ContextCopyParams {
  void* const* spans;
  const __nv_bfloat16* src;
  int64_t token_stride;  // elements between consecutive tokens of src
  int seq_len, n_groups, span_len, span_shift;
};

template <int QM, bool H>
__global__ void __launch_bounds__(128) context_span_copy_kernel(const ContextCopyParams p) {
  using F = Ft<H>;
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int64_t wid = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
  if (wid >= (int64_t)p.seq_len * p.n_groups) return;
  const int tok = (int)(wid / p.n_groups), g = (int)(wid - (int64_t)tok * p.n_groups);
  const uint2 raw = *reinterpret_cast<const uint2*>(p.src + (int64_t)tok * p.token_stride + g * kHead + lane * 4);
  const float x[4] = {F::lo(raw.x), F::hi(raw.x), F::lo(raw.y), F::hi(raw.y)};
  uint8_t* span = reinterpret_cast<uint8_t*>(p.spans[tok >> p.span_shift]);
  store_row<QM, H>(span, (size_t)g * p.span_len + (tok & (p.span_len - 1)), p.n_groups * p.span_len, lane, x);
}

// ------------------------------------------------------------------------------------------------
// cache append (+ optional fused rotary): one warp per (sequence, head slot)
// ------------------------------------------------------------------------------------------------
struct AppendParams {
  void* const* k_spans;
  void* const* v_spans;
  __nv_bfloat16* q_out;
  const __nv_bfloat16* qkv;
  const int32_t* old_lens;
  int batch, n_heads, n_groups, span_len, span_shift, max_spans;
  int rope;        // 0/1
  int rotary_dim;
  float log2_base;
};

template <int QM, bool H>
__global__ void __launch_bounds__(128) cache_append_kernel(const AppendParams p) {
  using F = Ft<H>;
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int slots = p.n_heads + 2 * p.n_groups;
  const int wid = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (wid >= p.batch * slots) return;
  const int b = wid / slots, slot = wid - b * slots;
  const __nv_bfloat16* src = p.qkv + ((size_t)b * slots + slot) * kHead + lane * 4;
  const uint2 raw = *reinterpret_cast<const uint2*>(src);
  float x[4] = {F::lo(raw.x), F::hi(raw.x), F::lo(raw.y), F::hi(raw.y)};
  const int pos = p.old_lens[b];
  const bool is_v = slot >= p.n_heads + p.n_groups;

  if (p.rope && !is_v) {
    // NeoX rotate-half over the first rotary_dim dims: out[i] = x[i]cos - x[i+h]sin ; out[i+h] = x[i+h]cos + x[i]sin
    const int half = p.rotary_dim >> 1;
    float other[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) other[i] = __shfl_xor_sync(0xffffffffu, x[i], half == 64 ? 16 : 8);
    if (half == 64 || half == 32) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int d = lane * 4 + i;
        if (d < p.rotary_dim) {
          const int fi = d % half;
          const float inv = exp2f(-p.log2_base * (2.0f * fi / (float)p.rotary_dim));
          float sn, cs;
          sincosf((float)pos * inv, &sn, &cs);
          // round to bf16 like the reference's Rotary op output (it feeds the cache through an FT tensor)
          x[i] = F::to_f(F::from_f(d < half ? x[i] * cs - other[i] * sn : x[i] * cs + other[i] * sn));
        }
      }
    }
  }

  if (slot < p.n_heads) {
    *reinterpret_cast<uint2*>(p.q_out + ((size_t)b * p.n_heads + slot) * kHead + lane * 4) =
        make_uint2(F::pack(x[0], x[1]), F::pack(x[2], x[3]));
    return;
  }
  const int g = is_v ? slot - p.n_heads - p.n_groups : slot - p.n_heads;
  void* const* tab = (is_v ? p.v_spans : p.k_spans) + (size_t)b * p.max_spans;
  const int si = pos >> p.span_shift, ps = pos & (p.span_len - 1);
  uint8_t* span = reinterpret_cast<uint8_t*>(tab[si]);
  const size_t rowi = (size_t)g * p.span_len + ps;
  store_row<QM, H>(span, rowi, p.n_groups * p.span_len, lane, x);
}

int span_attn64_run(const b2_span_cfg* c, void* out, const void* q, const void* const* k_spans, const void* const* v_spans,
                    const int32_t* lens, int batch, float qk_scale, cudaStream_t stream);
int span_append64_run(const b2_span_cfg* c, void* const* k_spans, void* const* v_spans, void* q_out, const void* qkv,
                      const int32_t* old_lens, int batch, const b2_rope_cfg* rope, cudaStream_t stream);

static int ilog2(int x) {
  int s = 0;
  while ((1 << s) < x) ++s;
  return s;
}

static int check_cfg(const b2_span_cfg* c) {
  if (!c) return B2_ERR_PARAM;
  if (c->ft != B2_DT_BF16 && c->ft != B2_DT_F16) return B2_ERR_UNSUPPORTED;
  if (c->ft == B2_DT_F16 && c->head_size != kHead) return B2_ERR_UNSUPPORTED;  // the head-64 kernels are bf16 only
  // 128: the reference GPU library's only head size (span_attention.hpp:203-208).  64: bf16 KV only — the parity anchor C0
  // (Qwen2-0.5B) that the reference runs on its CPU path; span_attn64.cu
  if (c->head_size != kHead && !(c->head_size == 64 && c->quant_mode == B2_KV_NONE)) return B2_ERR_UNSUPPORTED;
  if (c->quant_mode < B2_KV_NONE || c->quant_mode > B2_KV_U4) return B2_ERR_PARAM;
  if (c->span_len != 16 && c->span_len != 32 && c->span_len != 64 && c->span_len != 128) return B2_ERR_PARAM;
  if (c->n_groups <= 0 || c->n_heads <= 0 || c->n_heads % c->n_groups) return B2_ERR_PARAM;
  if (c->n_heads / c->n_groups > 16) return B2_ERR_UNSUPPORTED;
  if (c->max_spans_per_seq <= 0) return B2_ERR_PARAM;
  return B2_OK;
}

}  // namespace b2

using namespace b2;

struct b2_span_attn {
  b2_span_cfg cfg;
  int max_batch = 0;
  unsigned* counters = nullptr;   // [max_batch * n_groups] + [2 * grid] (level-1 groups), self-resetting
  int grid = 0, nstage = 2, smem = 0, max_pieces = 1 << 20;
};

template <int QM>
static int stage_bytes() { return 2 * KVTraits<QM>::TILE + 2 * KVTraits<QM>::PARAM; }

typedef void (*attn_kernel_t)(const AttnParams);
static attn_kernel_t attn_kernel_for(int qm, bool fp16 = false);
static attn_kernel_t attn_kernel_for_cfg(const b2_span_cfg* c) { return attn_kernel_for(c->quant_mode, c->ft == B2_DT_F16); }
static attn_kernel_t attn_kernel_for(int qm, bool fp16) {
  if (fp16) {
    switch (qm) {
      case B2_KV_NONE: return span_attn_kernel<B2_KV_NONE, true>;
      case B2_KV_I8: return span_attn_kernel<B2_KV_I8, true>;
      default: return span_attn_kernel<B2_KV_U4, true>;
    }
  }
  switch (qm) {
    case B2_KV_NONE: return span_attn_kernel<B2_KV_NONE, false>;
    case B2_KV_I8: return span_attn_kernel<B2_KV_I8, false>;
    default: return span_attn_kernel<B2_KV_U4, false>;
  }
}

extern "C" {

size_t b2_span_bytes(const b2_span_cfg* c) {
  if (check_cfg(c) != B2_OK) return 0;
  const size_t rows = (size_t)c->span_len * c->n_groups;
  switch (c->quant_mode) {  // csrc/runtime/cache/virtual_cache.cpp:202-232
    case B2_KV_NONE: return rows * c->head_size * 2;
    case B2_KV_I8: return rows * c->head_size + 2 * rows * 4;
    default: return rows * c->head_size / 2 + 2 * rows * 4;
  }
}

size_t b2_span_attn_algo_bytes(const b2_span_cfg* c, int64_t total_tokens) {
  if (check_cfg(c) != B2_OK) return 0;
  const size_t row = c->quant_mode == B2_KV_NONE ? (size_t)c->head_size * 2 : (c->quant_mode == B2_KV_I8 ? 128 + 8 : 64 + 8);
  return (size_t)total_tokens * 2 * c->n_groups * row;
}

int b2_span_attn_create(b2_span_attn_t* out, const b2_span_cfg* cfg, int max_batch) {
  if (!out) return B2_ERR_PARAM;
  if (int st = check_cfg(cfg)) return st;
  if (max_batch <= 0 || max_batch > kMaxBatch) return B2_ERR_LIMIT;
  b2_span_attn* h = new (std::nothrow) b2_span_attn();
  if (!h) return B2_ERR_RUNTIME;
  h->cfg = *cfg;
  h->max_batch = max_batch;
  attn_kernel_t kern = attn_kernel_for_cfg(cfg);
  const int sb = cfg->quant_mode == B2_KV_NONE ? stage_bytes<B2_KV_NONE>()
                                                : (cfg->quant_mode == B2_KV_I8 ? stage_bytes<B2_KV_I8>() : stage_bytes<B2_KV_U4>());
  const char* env = getenv("B2_ATTN_STAGES");
  h->nstage = env ? atoi(env) : (cfg->quant_mode == B2_KV_NONE ? 2 : (cfg->quant_mode == B2_KV_I8 ? 3 : 4));
  if (h->nstage < 2) h->nstage = 2;
  if (h->nstage > 4) h->nstage = 4;
  const int merge = (4 * 16 * kMergeRS + 4 * 16 * 2) * 4;
  h->smem = h->nstage * sb > merge ? h->nstage * sb : merge;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem);
  int occ = 1;
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kAttnThreads, h->smem);
  if (e != cudaSuccess) {
    set_last_error("b2_span_attn_create(occupancy)", e);
    delete h;
    return B2_ERR_CUDA;
  }
  if (occ < 1) occ = 1;
  const char* envo = getenv("B2_ATTN_CTAS_PER_SM");
  if (envo && atoi(envo) > 0 && atoi(envo) < occ) occ = atoi(envo);
  h->grid = occ * sm_count();
  if (const char* envp = getenv("B2_ATTN_MAX_PIECES")) h->max_pieces = atoi(envp) > 0 ? atoi(envp) : h->max_pieces;
  const size_t nb = sizeof(unsigned) * ((size_t)max_batch * cfg->n_groups + (size_t)2 * h->grid);
  e = cudaMalloc(&h->counters, nb);
  if (e == cudaSuccess) e = cudaMemset(h->counters, 0, nb);
  if (e != cudaSuccess) {
    set_last_error("b2_span_attn_create", e);
    delete h;
    return B2_ERR_CUDA;
  }
  *out = h;
  return B2_OK;
}

int b2_span_attn_destroy(b2_span_attn_t h) {
  if (!h) return B2_OK;
  if (h->counters) cudaFree(h->counters);
  delete h;
  return B2_OK;
}

// split-KV partials: at most two per CTA (its first and its last piece), independent of batch and length
static size_t partial_slots(const b2_span_attn* h) { return (size_t)2 * h->grid; }

size_t b2_span_attn_workspace_bytes(b2_span_attn_t h, int batch, int max_len) {
  if (!h || batch <= 0 || max_len <= 0) return 0;
  const int hpg = h->cfg.n_heads / h->cfg.n_groups;
  return 2 * partial_slots(h) * hpg * (kHead + 2) * sizeof(float) + 256;  // level-0 and level-1 partials
}

int b2_span_attn_run(b2_span_attn_t h, void* out, const void* q, const void* const* k_spans, const void* const* v_spans,
                     const int32_t* new_lens, int batch, int max_len, void* workspace, size_t workspace_bytes,
                     float qk_scale, void* stream_) {
  if (!h || !out || !q || !k_spans || !v_spans || !new_lens) return B2_ERR_PARAM;
  if (batch <= 0 || batch > h->max_batch) return B2_ERR_LIMIT;
  if (max_len <= 0 || (int64_t)(max_len + h->cfg.span_len - 1) / h->cfg.span_len > h->cfg.max_spans_per_seq) return B2_ERR_LIMIT;
  if (!workspace || workspace_bytes < b2_span_attn_workspace_bytes(h, batch, max_len)) return B2_ERR_PARAM;
  if (h->cfg.head_size == 64) return span_attn64_run(&h->cfg, out, q, k_spans, v_spans, new_lens, batch, qk_scale, (cudaStream_t)stream_);
  const int hpg = h->cfg.n_heads / h->cfg.n_groups;
  AttnParams p;
  p.out = (__nv_bfloat16*)out;
  p.q = (const __nv_bfloat16*)q;
  p.k_spans = k_spans;
  p.v_spans = v_spans;
  p.lens = new_lens;
  const size_t items = partial_slots(h);
  p.ws_o = (float*)(((uintptr_t)workspace + 127) & ~(uintptr_t)127);
  p.ws_ml = p.ws_o + items * hpg * kHead;
  p.ws2_o = p.ws_ml + items * hpg * 2;
  p.ws2_ml = p.ws2_o + items * hpg * kHead;
  p.counters = h->counters;
  p.counters1 = h->counters + (size_t)h->max_batch * h->cfg.n_groups;
  p.max_pieces = h->max_pieces;
  p.batch = batch; p.n_heads = h->cfg.n_heads; p.n_groups = h->cfg.n_groups; p.hpg = hpg;
  p.span_len = h->cfg.span_len; p.span_shift = ilog2(h->cfg.span_len); p.max_spans = h->cfg.max_spans_per_seq;
  p.nstage = h->nstage;
  p.scale_log2 = qk_scale * 1.4426950408889634f;
  attn_kernel_t kern = attn_kernel_for_cfg(&h->cfg);
  cudaError_t e = launch(kern, dim3(h->grid), dim3(kAttnThreads), (size_t)h->smem, (cudaStream_t)stream_, true, p);
  if (e != cudaSuccess) {
    set_last_error("span_attn launch", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

int b2_span_context_copy(const b2_span_cfg* cfg, void* const* spans, const void* src, int64_t token_stride, int seq_len,
                         void* stream_) {
  if (int st = check_cfg(cfg)) return st;
  if (cfg->head_size != kHead) return B2_ERR_UNSUPPORTED;
  if (!spans || !src || seq_len <= 0) return B2_ERR_PARAM;
  if (token_stride < (int64_t)cfg->n_groups * kHead || (token_stride & 3) || ((uintptr_t)src & 7)) return B2_ERR_PARAM;
  if ((int64_t)(seq_len + cfg->span_len - 1) / cfg->span_len > cfg->max_spans_per_seq) return B2_ERR_LIMIT;
  ContextCopyParams p;
  p.spans = spans; p.src = (const __nv_bfloat16*)src; p.token_stride = token_stride;
  p.seq_len = seq_len; p.n_groups = cfg->n_groups; p.span_len = cfg->span_len; p.span_shift = ilog2(cfg->span_len);
  const int64_t warps = (int64_t)seq_len * cfg->n_groups;
  const dim3 grid((unsigned)((warps + 3) / 4)), block(128);
  cudaError_t e;
  cudaStream_t stream = (cudaStream_t)stream_;
  const bool h16 = cfg->ft == B2_DT_F16;
  if (cfg->quant_mode == B2_KV_NONE) e = h16 ? launch(context_span_copy_kernel<B2_KV_NONE, true>, grid, block, 0, stream, true, p)
                                             : launch(context_span_copy_kernel<B2_KV_NONE, false>, grid, block, 0, stream, true, p);
  else if (cfg->quant_mode == B2_KV_I8) e = h16 ? launch(context_span_copy_kernel<B2_KV_I8, true>, grid, block, 0, stream, true, p)
                                                : launch(context_span_copy_kernel<B2_KV_I8, false>, grid, block, 0, stream, true, p);
  else e = h16 ? launch(context_span_copy_kernel<B2_KV_U4, true>, grid, block, 0, stream, true, p)
               : launch(context_span_copy_kernel<B2_KV_U4, false>, grid, block, 0, stream, true, p);
  if (e != cudaSuccess) {
    set_last_error("context_span_copy launch", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

int b2_span_cache_append(const b2_span_cfg* cfg, void* const* k_spans, void* const* v_spans, void* q_out,
                         const void* qkv, const int32_t* old_lens, int batch, const b2_rope_cfg* rope, void* stream_) {
  if (int st = check_cfg(cfg)) return st;
  if (!k_spans || !v_spans || !q_out || !qkv || !old_lens || batch <= 0) return B2_ERR_PARAM;
  if (cfg->head_size == 64) return span_append64_run(cfg, k_spans, v_spans, q_out, qkv, old_lens, batch, rope, (cudaStream_t)stream_);
  if (rope && (rope->rotary_dim != 128 && rope->rotary_dim != 64)) return B2_ERR_UNSUPPORTED;
  AppendParams p;
  p.k_spans = k_spans; p.v_spans = v_spans;
  p.q_out = (__nv_bfloat16*)q_out; p.qkv = (const __nv_bfloat16*)qkv; p.old_lens = old_lens;
  p.batch = batch; p.n_heads = cfg->n_heads; p.n_groups = cfg->n_groups;
  p.span_len = cfg->span_len; p.span_shift = ilog2(cfg->span_len); p.max_spans = cfg->max_spans_per_seq;
  p.rope = rope ? 1 : 0;
  p.rotary_dim = rope ? rope->rotary_dim : 0;
  p.log2_base = rope ? log2f(rope->base) : 0.f;
  const int warps = batch * (cfg->n_heads + 2 * cfg->n_groups);
  const dim3 grid((warps + 3) / 4), block(128);
  cudaError_t e;
  cudaStream_t stream = (cudaStream_t)stream_;
  const bool h16 = cfg->ft == B2_DT_F16;
  if (cfg->quant_mode == B2_KV_NONE) e = h16 ? launch(cache_append_kernel<B2_KV_NONE, true>, grid, block, 0, stream, true, p)
                                             : launch(cache_append_kernel<B2_KV_NONE, false>, grid, block, 0, stream, true, p);
  else if (cfg->quant_mode == B2_KV_I8) e = h16 ? launch(cache_append_kernel<B2_KV_I8, true>, grid, block, 0, stream, true, p)
                                                : launch(cache_append_kernel<B2_KV_I8, false>, grid, block, 0, stream, true, p);
  else e = h16 ? launch(cache_append_kernel<B2_KV_U4, true>, grid, block, 0, stream, true, p)
               : launch(cache_append_kernel<B2_KV_U4, false>, grid, block, 0, stream, true, p);
  if (e != cudaSuccess) {
    set_last_error("cache_append launch", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

}  // extern "C"
