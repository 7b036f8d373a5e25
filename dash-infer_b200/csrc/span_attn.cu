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
// The span format and its shared-memory tile are described once, by KVTraits below; how the 16 MMA rows of a piece map to
// sequences, tokens, heads and visible tokens (single-token, chain and tree steps) once, by QueryRows.
// Roofline: HBM-bound; algorithmic bytes = sum_b len_b * 2 * n_groups * KVTraits<QM>::SPAN_ROW.
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
// The multi-token form (span_attn_kernel<..., MT = true>) takes these fields on top.  They are not members of AttnParams
// because a kernel parameter larger than 128 bytes changes the code of the single-token kernels.
// q / out rows b*q_len + t; the 16 MMA rows hold the heads of one kv-group for tpb consecutive tokens of one sequence (a
// row block), nrb row blocks per sequence; partial slots hold rstride = tpb * hpg rows.
struct AttnTokParams : AttnParams {
  int q_len, tpb, nrb, rstride;
};
// Tree form (span_attn_kernel<..., MT = true, TREE = true>): the q_len rows of a sequence are the nodes of a draft tree.
//   parents [batch][q_len] int32: node t >= 1 hangs below parents[b][t] in [0, t) (topological order); node 0 is the
//   root (the last emitted token) and parents[b][0] is ignored.  depth(t) = parent steps from t to 0; anc(t) = the 16-bit
//   mask of t and its ancestors (tree_walk in b2_common.cuh, shared with the append and the accept kernels).
//   Node t sits in slot lens[b] - q_len + t and carries rotary position lens[b] - q_len + depth(t); row t attends to the
//   prefix (tokens < lens[b] - q_len) and to the slots lens[b] - q_len + j, j in anc(t).  A chain (parents[t] = t - 1) is
//   the plain multi-token step.  Malformed parents read as the root (tree_parent): results unspecified, accesses in bounds.
// A node's ancestors have smaller indices, so a row block streams the same tiles as in the chain form.
struct AttnTreeParams : AttnTokParams {
  const int32_t* parents;
};
template <bool MT, bool TREE = false>
using AttnArgs = std::conditional_t<TREE, AttnTreeParams, std::conditional_t<MT, AttnTokParams, AttnParams>>;

// ---- span format (one description for the writers, the tile loader, the tile math and the host sizes) ----
// A span holds span_len tokens of one sequence for all n_groups kv-heads (the wire format of decoder_cache_append.cuh:33-92):
//   [n_groups][span_len] rows of ROW bytes, then, for the quantized modes, [n_groups][span_len] of {f32 zero, f32 scale}:
//   NONE: 128 bf16 / fp16 values                                   ROW 256, no {zero, scale}
//   I8  : 128 int8 codes q, value = (q - zero) * scale              ROW 128
//   FP8 : 128 e4m3fn codes, value = e4m3(q) * scale, zero = 0      ROW 128 (the I8 layout)
//   U4  : 128 uint4 codes, element 2i in the low nibble of byte i   ROW 64
// SPAN_ROW = ROW + 8 (quantized) is both the span bytes per token row and what attention reads per token and kv-head.
// A ring stage holds one 64-token tile: K rows [64][ROW], V rows [64][ROW], then K's and V's {zero, scale} [64] each.
// 16-byte chunk c of tile row r is stored at chunk swz(r, c) of that row, so the 8 rows an ldmatrix / LDS.128 phase reads
// start in different bank groups: 8 or 16 chunks per row XOR with r & 7; U4's 4 chunks (two rows per 128 bytes) with (r >> 1) & 3.
// All quantized modes run the MMAs in fp16 on the raw codes converted exactly (tile_compute_q); I8 and U4 also carry a
// zero-point term there, FP8 does not.
template <int QM>
struct KVTraits {
  static constexpr bool kCodesF16 = QM != B2_KV_NONE;                  // quantized: MMAs on fp16-converted codes
  static constexpr bool kZeroPoint = QM == B2_KV_I8 || QM == B2_KV_U4;  // scores / O carry a zero-point term
  static constexpr int ROW = QM == B2_KV_NONE ? 256 : (QM == B2_KV_U4 ? 64 : 128);  // bytes per token row
  static constexpr int PARAM_ROW = kCodesF16 ? 8 : 0;                  // {f32 zero, f32 scale} per token row
  static constexpr int SPAN_ROW = ROW + PARAM_ROW;                     // 256 / 136 / 72 / 136
  static constexpr int TILE = kTile * ROW;                             // K (or V) rows of a stage
  static constexpr int PARAM = kTile * PARAM_ROW;                      // K (or V) {zero, scale} of a stage
  static constexpr int STAGE = 2 * TILE + 2 * PARAM;
  static constexpr int kStages = QM == B2_KV_NONE ? 2 : (QM == B2_KV_U4 ? 4 : 3);  // default ring depth (B2_ATTN_STAGES)
  // tile_compute_q rounds P' = P * s_v * 2^kPExp to fp16.  Without the power of two a small V scale puts P' among the fp16
  // subnormals (spacing 2^-24), whose error relative to the output grows as V shrinks.  The exponent keeps s_v 2^kPExp
  // below 65504 for per-row max|v| <= 4096 (u4: s_v <= 8192 / 15, i8: 8192 / 255, fp8: 4096 / 448); l carries the same
  // factor, so o / l is what it would be without it, bit for bit.
  static constexpr int kPExp = QM == B2_KV_U4 ? 6 : (QM == B2_KV_I8 ? 10 : (QM == B2_KV_FP8 ? 12 : 0));
  static constexpr float kPScale = static_cast<float>(1 << kPExp);
  // byte offset of row rowi's {zero, scale} in a span of n_rows = n_groups * span_len rows
  __device__ __forceinline__ static size_t param_offset(size_t n_rows, size_t rowi) { return n_rows * ROW + rowi * PARAM_ROW; }
  __device__ __forceinline__ static int swz(int row, int c) { return QM == B2_KV_U4 ? c ^ ((row >> 1) & 3) : c ^ (row & 7); }
};

// ---- d-order of the quantized modes: which head dims a thread's Q fragment registers and o[] elements hold.  The order
// of Q is free as long as Q and K agree, and it follows how a thread reads K: whole 16-byte chunks of codes (I8 / FP8: the
// 32 d of chunks 2t, 2t+1; U4: the 32 d of chunk t).  The order of o[] is the one the V codes give the PV MMAs' columns.
//   q(t, ks, j): d of column {2t, 2t+1, 2t+8, 2t+9}[j] of k-step ks      o(t, dt, e): d of o[dt][e] and o[dt][2 + e]
template <int QM>
struct DOrder {
  __device__ __forceinline__ static int q(int t, int ks, int j) {
    if constexpr (QM == B2_KV_U4) return 32 * t + 8 * (ks >> 1) + 2 * (ks & 1) + 4 * (j & 1) + (j >> 1);
    else return 32 * t + 4 * ks + j;
  }
  __device__ __forceinline__ static int o(int t, int dt, int e) {
    if constexpr (QM == B2_KV_U4) return 32 * (dt >> 2) + 8 * t + (dt & 3) + 4 * e;
    else return 16 * (dt >> 1) + 4 * t + (dt & 1) + 2 * e;
  }
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
  uint8_t* dk = stage + row0 * T::ROW + T::swz(row0, c) * 16;
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
  if constexpr (T::kCodesF16) {
    // per-token {zero, scale} for K and V: 64 x 8 B each = 32 x 16 B chunks each
    if (tid < 64) {
      const int which = tid >> 5, cc = tid & 31;  // 0: K, 1: V
      const int row = cc * 2;
      const bool valid = row < nvalid;
      const int rr = valid ? row : 0;
      const int sj = (pos0 + rr) >> p.span_shift, pos = (pos0 + rr) & (p.span_len - 1);
      const uint8_t* sp = reinterpret_cast<const uint8_t*>((which ? vtab : ktab)[si0 + sj]);
      const size_t poff = T::param_offset((size_t)p.n_groups * p.span_len, (size_t)g * p.span_len + pos);
      cp_async16_zfill(stage + 2 * T::TILE + which * T::PARAM + cc * 16, sp + poff, valid);
    }
  }
}

// ---- online softmax (base 2) of the tile functions: a thread holds scores of rows gq and gq+8, its quad the row's 16 tokens
__device__ __forceinline__ void quad_max(float& x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
}
__device__ __forceinline__ void quad_sum(float& x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  x += __shfl_xor_sync(0xffffffffu, x, 2);
}
// running max of both rows after this tile (mx: the thread's tile max); corr rescales what was summed under the old max;
// msub is what the tile's scores are reduced by before exp2
template <bool MT>
__device__ __forceinline__ void softmax_max(float (&mx)[2], float (&mrow)[2], float (&corr)[2], float (&msub)[2]) {
#pragma unroll
  for (int r2 = 0; r2 < 2; ++r2) quad_max(mx[r2]);
#pragma unroll
  for (int r2 = 0; r2 < 2; ++r2) {
    // single token: finite, the warp's first token is always live.  Multi-token: a row whose limit lies before this
    // warp's slice has seen no live token yet (mnew = -inf); it subtracts 0 so that corr and its probabilities are 0, not NaN
    const float mnew = fmaxf(mrow[r2], mx[r2]);
    msub[r2] = MT && mnew == -INFINITY ? 0.f : mnew;
    corr[r2] = exp2f(mrow[r2] - msub[r2]);
    mrow[r2] = mnew;
  }
}
// l = l * corr + the row's tile probabilities (psum: the thread's share), o *= corr
__device__ __forceinline__ void softmax_sum(float (&psum)[2], float (&lrow)[2], const float (&corr)[2], float (&o)[16][4]) {
#pragma unroll
  for (int r2 = 0; r2 < 2; ++r2) {
    quad_sum(psum[r2]);
    lrow[r2] = lrow[r2] * corr[r2] + psum[r2];
  }
  if (corr[0] != 1.f || corr[1] != 1.f) {
#pragma unroll
    for (int dt = 0; dt < 16; ++dt) {
      o[dt][0] *= corr[0]; o[dt][1] *= corr[0];
      o[dt][2] *= corr[1]; o[dt][3] *= corr[1];
    }
  }
}

// ---- the query rows of a piece: the one place that knows how the 16 MMA rows of a work item map to sequences, tokens and
// heads, and which cached tokens each row may see.  Three step forms (span_attn_kernel<QM, H, MT, TREE>):
//   single token   item = sequence b; row r = head r of kv-group g; every row sees the item's len = lens[b] tokens.
//   chain (MT)     item = (sequence b, row block rb): tokens qt0 = rb*tpb .. qt0+ntok-1 of the step's q_len, row r = token
//                  qt0 + r / hpg, head r % hpg.  Token t sees the first lens[b] - q_len + t + 1 tokens, so the item streams the
//                  len tiles its last token sees and each row is masked at its own limit.
//   tree (TREE)    the chain's rows; row r sees the prefix (tokens < lens[b] - q_len) and the draft slots of node qt0 + r / hpg
//                  and its ancestors (AttnTreeParams).  Ancestors have smaller indices: the same tiles as the chain.
// The scheduler treats every item alike: counters and partials are per (item, kv-head), a partial slot holds rstride rows.

// What the calling thread's rows gq (rr = 0) and gq + 8 (rr = 1) may see.  tok1, the end of the piece, bounds every row.
template <bool MT, bool TREE>
struct RowMask {
  int tok1;
  int lim[2] = {0, 0};        // chain: the row's own end (<= tok1).  Tree: the prefix end.  A dead row: the item's len
  unsigned am[2] = {0u, 0u};  // tree: tree_walk's ancestor mask of the row's node (a dead row: 0)
  __device__ __forceinline__ bool visible(int tok, int rr) const {
    // tree: past the prefix, the token's draft slot tok - lim must be an ancestor's (tok < tok1 keeps the shift below 16)
    if constexpr (TREE) return tok < lim[rr] || (tok < tok1 && ((am[rr] >> (tok - lim[rr])) & 1u));
    else if constexpr (MT) return tok < lim[rr];
    else return tok < tok1;
  }
};

template <bool MT, bool TREE>
struct QueryRows;

// Single token.  (A specialisation of its own, not `MT ? :` expressions: these kernels are the decode hot path and must see
// no multi-token arithmetic.)
template <>
struct QueryRows<false, false> {
  __device__ __forceinline__ static int n_items(const AttnParams& p) { return p.batch; }
  __device__ __forceinline__ static int seq(const AttnParams&, int item) { return item; }
  __device__ __forceinline__ static int item_len(const AttnParams& p, int item) { return p.lens[item]; }  // tokens attended to

  int nrows, rstride;  // live MMA rows; rows of a partial slot
  size_t row0;
  RowMask<false, false> mask;

  // the piece of `item` (sequence b, len tokens) for kv-head g that ends at token tok1; gq = lane / 4
  __device__ __forceinline__ QueryRows(const AttnParams& p, int item, int b, int g, int len, int tok1, int gq) {
    row0 = ((size_t)b * p.n_heads + (size_t)g * p.hpg) * kHead;
    nrows = rstride = p.hpg;
    mask.tok1 = tok1;
  }
  // MMA row r in q or in out (same layout)
  template <class E>
  __device__ __forceinline__ E* at(E* base, int r) const { return base + row0 + r * kHead; }
};

// Chain and tree: the same members for a row block.
template <bool TREE>
struct QueryRows<true, TREE> {
  using Params = AttnArgs<true, TREE>;
  __device__ __forceinline__ static int n_items(const Params& p) { return p.batch * p.nrb; }
  __device__ __forceinline__ static int seq(const Params& p, int item) { return item / p.nrb; }
  __device__ __forceinline__ static int item_len(const Params& p, int item) {
    const int b = item / p.nrb, rb = item - b * p.nrb;
    return p.lens[b] - p.q_len + min(p.q_len, (rb + 1) * p.tpb);
  }

  const Params& p;
  int b, g, qt0;
  int nrows, rstride;
  RowMask<true, TREE> mask;

  __device__ __forceinline__ QueryRows(const Params& p_, int item, int b_, int g_, int len, int tok1, int gq) : p(p_), b(b_), g(g_) {
    qt0 = (item - b * p.nrb) * p.tpb;
    const int ntok = min(p.tpb, p.q_len - qt0);
    nrows = ntok * p.hpg;
    rstride = p.rstride;
    mask.tok1 = tok1;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int r = gq + 8 * rr;
      if constexpr (TREE) {
        int depth;
        mask.am[rr] = r < nrows ? tree_walk(p.parents + (size_t)b * p.q_len, qt0 + r / p.hpg, depth) : 0u;
        mask.lim[rr] = r < nrows ? len - ntok - qt0 : len;
      } else {
        mask.lim[rr] = r < nrows ? len - ntok + 1 + r / p.hpg : len;
      }
    }
  }
  template <class E>
  __device__ __forceinline__ E* at(E* base, int r) const {
    return base + ((size_t)b * p.q_len + qt0 + r / p.hpg) * p.n_heads * kHead + ((size_t)g * p.hpg + r % p.hpg) * kHead;
  }
};

// One 64-token tile of attention math for this warp's 16-token slice (cache in the 16-bit type FT: bf16, or fp16 when H).
// mask says which tokens the thread's rows gq and gq+8 see.
template <bool H, bool MT, bool TREE>
__device__ __forceinline__ void tile_compute_bf16(const uint8_t* st, int warp, int lane, int wtok, const RowMask<MT, TREE>& mask,
                                                  float scale_log2, const uint32_t (&qa)[8][4],
                                                  float (&o)[16][4], float (&mrow)[2], float (&lrow)[2]) {
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
      ldmatrix_x4(r, kb + row * T::ROW + (T::swz(row, chunk) << 4));
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
      const float v = mask.visible(tok, cc >> 1) ? sc[nt][cc] * scale_log2 : -INFINITY;
      sc[nt][cc] = v;
      mx[cc >> 1] = fmaxf(mx[cc >> 1], v);
    }
  float corr[2], psum[2] = {0.f, 0.f}, msub[2];
  softmax_max<MT>(mx, mrow, corr, msub);
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int cc = 0; cc < 4; ++cc) {
      const float pv = exp2f(sc[nt][cc] - msub[cc >> 1]);
      sc[nt][cc] = pv;
      psum[cc >> 1] += pv;
    }
  softmax_sum(psum, lrow, corr, o);
  const uint32_t pa0 = Ft<H>::pack(sc[0][0], sc[0][1]), pa1 = Ft<H>::pack(sc[0][2], sc[0][3]);
  const uint32_t pa2 = Ft<H>::pack(sc[1][0], sc[1][1]), pa3 = Ft<H>::pack(sc[1][2], sc[1][3]);
  // ---------- O += P V : 16 d-tiles, k16 = this warp's 16 tokens
#pragma unroll
  for (int dt = 0; dt < 16; dt += 2) {
    const int mi = lane >> 3;
    const int row = warp * 16 + 8 * (mi & 1) + (lane & 7);
    const int chunk = dt + (mi >> 1);
    uint32_t r[4];
    ldmatrix_x4_trans(r, vb + row * T::ROW + (T::swz(row, chunk) << 4));
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
// FP8 shares the I8 tile layout and d-order; its codes are converted with cvt (e4m3 -> fp16 exact) and have no zero point.
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
  return d;
}

// ---- FP8 KV: the e4m3 codes convert EXACTLY to fp16 (one F2FP.F16.E4M3.UNPACK_B per pair), so the same fp16 MMAs run on
// the codes themselves and only the per-token scale remains (no zero point):
//   score[h,tok] = s_k[tok] * sum_d Q[h,d] * e4m3(k[tok,d]),   O[h,d] = sum_tok (P[h,tok] * s_v[tok]) * e4m3(v[tok,d])
// Byte HALF (0: bytes 0,1; 1: bytes 2,3) of w -> fp16x2 {lower byte, upper byte}.
template <int HALF>
__device__ __forceinline__ uint32_t e4m3x2_to_f16x2(uint32_t w) {
  uint32_t d;
  if (HALF == 0)
    asm("{\n\t.reg .b16 lo, hi;\n\tmov.b32 {lo, hi}, %1;\n\tcvt.rn.f16x2.e4m3x2 %0, lo;\n\t}" : "=r"(d) : "r"(w));
  else
    asm("{\n\t.reg .b16 lo, hi;\n\tmov.b32 {lo, hi}, %1;\n\tcvt.rn.f16x2.e4m3x2 %0, hi;\n\t}" : "=r"(d) : "r"(w));
  return d;
}

template <int QM, bool MT, bool TREE>
__device__ __forceinline__ void tile_compute_q(const uint8_t* st, int warp, int lane, int wtok, const RowMask<MT, TREE>& mask,
                                               float scale_log2, const uint32_t (&qa)[8][4], const float (&sq)[2],
                                               float (&o)[16][4], float (&mrow)[2], float (&lrow)[2], float (&cacc)[2]) {
  using T = KVTraits<QM>;
  constexpr float BIAS = QM == B2_KV_I8 ? 1152.f : 1024.f;
  const int gq = lane >> 2, t = lane & 3;
  const uint32_t kb = smem_u32(st), vb = kb + T::TILE;
  const float2* kprm = reinterpret_cast<const float2*>(st + 2 * T::TILE);             // {zero, scale} per token
  const float2* vprm = reinterpret_cast<const float2*>(st + 2 * T::TILE + T::PARAM);
  // ---------- raw S = Q (BIAS + u)^T: the thread's 32 d of a token are CPT 16-byte chunks of codes
  constexpr int CPT = T::ROW / 64;
  float sc[2][4];
#pragma unroll
  for (int nt = 0; nt < 2; ++nt) {
    sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
    const int row = warp * 16 + nt * 8 + gq;  // this thread's token for the B fragments
#pragma unroll
    for (int c2 = 0; c2 < CPT; ++c2) {  // chunk CPT*t + c2: d = 32t + 16*c2 + (0..15) (U4: d = 32t + (0..31))
      const uint4 kv = lds128(kb + row * T::ROW + (T::swz(row, CPT * t + c2) << 4));
      uint32_t kw[4] = {kv.x, kv.y, kv.z, kv.w};
      if constexpr (QM == B2_KV_I8) {
#pragma unroll
        for (int j = 0; j < 4; ++j) kw[j] ^= 0x80808080u;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if constexpr (QM == B2_KV_I8) {
          const int ks = 4 * c2 + j;
          const uint32_t b0 = prmt(kw[j], 0x64646464u, 0x5140u), b1 = prmt(kw[j], 0x64646464u, 0x7362u);
          mma_f16_16816(sc[nt], qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3], b0, b1);
        } else if constexpr (QM == B2_KV_FP8) {  // the I8 d-order: the two halves of a word pair like prmt 0x5140 / 0x7362
          const int ks = 4 * c2 + j;
          mma_f16_16816(sc[nt], qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3], e4m3x2_to_f16x2<0>(kw[j]), e4m3x2_to_f16x2<1>(kw[j]));
        } else {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int ks = 2 * j + h;
            const uint32_t b0 = ((kw[j] >> (8 * h)) & 0x000f000fu) | 0x64006400u;
            const uint32_t b1 = ((kw[j] >> (8 * h + 4)) & 0x000f000fu) | 0x64006400u;
            mma_f16_16816(sc[nt], qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3], b0, b1);
          }
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
    const bool live0 = wtok + nt * 8 + 2 * t < mask.tok1, live1 = wtok + nt * 8 + 2 * t + 1 < mask.tok1;
    vz[nt][0] = live0 ? vp.x : 0.f; vs[nt][0] = live0 ? vp.y * T::kPScale : 0.f;
    vz[nt][1] = live1 ? vp.z : 0.f; vs[nt][1] = live1 ? vp.w * T::kPScale : 0.f;
#pragma unroll
    for (int cc = 0; cc < 4; ++cc) {
      const int tok = wtok + nt * 8 + 2 * t + (cc & 1);
      const float kz = (cc & 1) ? kp.z : kp.x, ksc = (cc & 1) ? kp.w : kp.y;
      const float raw = T::kZeroPoint ? ksc * (sc[nt][cc] - (BIAS + kz) * sq[cc >> 1]) : ksc * sc[nt][cc];
      const float v = mask.visible(tok, cc >> 1) ? raw * scale_log2 : -INFINITY;
      sc[nt][cc] = v;
      mx[cc >> 1] = fmaxf(mx[cc >> 1], v);
    }
  }
  float corr[2], psum[2] = {0.f, 0.f}, csum[2] = {0.f, 0.f}, msub[2];
  softmax_max<MT>(mx, mrow, corr, msub);
  uint32_t pa[4];
#pragma unroll
  for (int nt = 0; nt < 2; ++nt) {
    float pq[4];
#pragma unroll
    for (int cc = 0; cc < 4; ++cc) {
      const float pv = exp2f(sc[nt][cc] - msub[cc >> 1]);
      psum[cc >> 1] += pv;
      pq[cc] = pv * vs[nt][cc & 1];  // fold the V scale (times 2^kPExp) into the probability
    }
    pa[2 * nt] = pack_f16x2(pq[0], pq[1]);
    pa[2 * nt + 1] = pack_f16x2(pq[2], pq[3]);
    if constexpr (T::kZeroPoint) {
      // zero-point term with the SAME fp16-rounded probabilities the tensor core sees
      const __half2 h01 = *reinterpret_cast<const __half2*>(&pa[2 * nt]), h23 = *reinterpret_cast<const __half2*>(&pa[2 * nt + 1]);
      csum[0] += __low2float(h01) * (BIAS + vz[nt][0]) + __high2float(h01) * (BIAS + vz[nt][1]);
      csum[1] += __low2float(h23) * (BIAS + vz[nt][0]) + __high2float(h23) * (BIAS + vz[nt][1]);
    }
  }
  if constexpr (T::kZeroPoint) {
#pragma unroll
    for (int r2 = 0; r2 < 2; ++r2) cacc[r2] = cacc[r2] * corr[r2] + csum[r2];  // per-thread partial (its 4 tokens); reduced over the quad at the end
  }
  softmax_sum(psum, lrow, corr, o);
  // ---------- raw O += P' (BIAS + u): ldmatrix.trans on 16-bit units of the raw rows
  const int mi = lane >> 3;
  const int vrow = warp * 16 + 8 * (mi & 1) + (lane & 7);
#pragma unroll
  for (int c = 0; c < T::ROW / 16; c += 2) {
    uint32_t r[4];
    ldmatrix_x4_trans(r, vb + vrow * T::ROW + (T::swz(vrow, c + (mi >> 1)) << 4));
#pragma unroll
    for (int u = 0; u < 2; ++u) {  // chunk c+u: bytes {V[2t][2g], V[2t][2g+1], V[2t+1][2g], V[2t+1][2g+1]}
      if constexpr (QM == B2_KV_I8) {
        const uint32_t lo = r[2 * u] ^ 0x80808080u, hi = r[2 * u + 1] ^ 0x80808080u;
        mma_f16_16816(o[2 * (c + u)], pa[0], pa[1], pa[2], pa[3], prmt(lo, 0x64646464u, 0x6240u), prmt(hi, 0x64646464u, 0x6240u));
        mma_f16_16816(o[2 * (c + u) + 1], pa[0], pa[1], pa[2], pa[3], prmt(lo, 0x64646464u, 0x7351u), prmt(hi, 0x64646464u, 0x7351u));
      } else if constexpr (QM == B2_KV_FP8) {  // -> {even d pair, odd d pair}
        const uint32_t lo = prmt(r[2 * u], 0u, 0x3120u), hi = prmt(r[2 * u + 1], 0u, 0x3120u);
        mma_f16_16816(o[2 * (c + u)], pa[0], pa[1], pa[2], pa[3], e4m3x2_to_f16x2<0>(lo), e4m3x2_to_f16x2<0>(hi));
        mma_f16_16816(o[2 * (c + u) + 1], pa[0], pa[1], pa[2], pa[3], e4m3x2_to_f16x2<1>(lo), e4m3x2_to_f16x2<1>(hi));
      } else {
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
// A slot holds rows.rstride rows of which the first rows.nrows are live; FINAL puts row r at out + rows.row(r).
constexpr int kMergeMaxSrc = 96;  // sources of one merge call (final level: ceil(pieces / kMergeFan)); more -> looped M pass
template <bool FINAL, bool H, class Rows>
__device__ __forceinline__ void merge_partials(const float* src_o, const float* src_ml, int slot0, int stride2, int par0, int n,
                                               const Rows& rows, __nv_bfloat16* out, float* dst_o, float* dst_ml, int dst_slot,
                                               float* s_w, float* s_ML) {
  const int tid = threadIdx.x;
  auto slot_of = [&](int i) { return slot0 + i * stride2 + (i == 0 ? par0 : 0); };
  const int R = rows.nrows, hpg = rows.rstride;  // rows merged, rows of a slot
  const int nunits = R * 32;  // (row, float4) units
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
  for (int k = tid; k < n * R; k += kAttnThreads) {  // k = i * R + r
    const int i = k / R, r = k - i * R;
    const float2 ml = __ldcg(reinterpret_cast<const float2*>(src_ml + ((size_t)slot_of(i) * hpg + r) * 2));
    if (i < kMergeMaxSrc) { s_w[i * 16 + r] = ml.x; s_w[(kMergeMaxSrc + i) * 16 + r] = ml.y; }
  }
  __syncthreads();
  const int nn = min(n, kMergeMaxSrc);  // (n > kMergeMaxSrc cannot happen: pieces <= grid, fan-in 8, grid <= 8 * kMergeMaxSrc)
  if (tid < R) {  // per row: global max, weights, denominator (fixed source order)
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
      const float w = (i < nn && r < R) ? s_w[i * 16 + r] : 0.f;
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
        const float w = (i0 + i < nn && r < R) ? s_w[(i0 + i) * 16 + r] : 0.f;
        acc[uu].x += w * v[uu][i].x; acc[uu].y += w * v[uu][i].y; acc[uu].z += w * v[uu][i].z; acc[uu].w += w * v[uu][i].w;
      }
    }
  }
  // R <= 16: up to 512 units, two per thread cover 8 rows; the remaining rows (R > 8) take a second sweep
  for (int sweep = 0; sweep < 2; ++sweep) {
    if (sweep == 1) {
      if (R <= 8) break;
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
        *reinterpret_cast<uint2*>(rows.at(out, r) + c4 * 4) =
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

template <int QM, bool H, bool MT = false, bool TREE = false>
__global__ void __launch_bounds__(kAttnThreads) span_attn_kernel(const AttnArgs<MT, TREE> p) {
  using F = Ft<H>;  // the 16-bit type of Q, the output and an unquantized cache
  using T = KVTraits<QM>;
  using Rows = QueryRows<MT, TREE>;
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ int s_prefix[kMaxBatch + 1];  // flat tile index of each sequence's first tile (x n_groups)
  __shared__ int s_red[8];
  __shared__ int s_is_last;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int gq = lane >> 2, t = lane & 3;

  const bool tr0 = blockIdx.x == 0 && threadIdx.x == 0;
  if (tr0) B2_TR(g_attn_tr, 0);
  pdl_wait();  // the newest token's K/V (and q) come from the preceding append kernel
  pdl_launch_dependents();
  if (tr0) B2_TR(g_attn_tr, 1);

  // ---------------- device-side work decomposition (ONE global round trip: the lengths) ----------------
  // items: sequences, or (sequence, row block)s (QueryRows)
  {
    int my_tiles = 0, my_max = 0;
    for (int b = tid; b < Rows::n_items(p); b += kAttnThreads) {
      const int tl = (Rows::item_len(p, b) + kTile - 1) / kTile;
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
    for (int b0 = 0; b0 < Rows::n_items(p); b0 += 32) {
      const int b = b0 + lane;
      int v = b < Rows::n_items(p) ? s_prefix[b] * p.n_groups : 0, x = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      if (b < Rows::n_items(p)) s_prefix[b] = carry + x - v;
      carry += __shfl_sync(0xffffffffu, x, 31);
    }
    if (lane == 0) s_prefix[Rows::n_items(p)] = carry;
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
    int blo = 0, bhi = Rows::n_items(p) - 1;
    while (blo < bhi) {
      const int mid = (blo + bhi + 1) >> 1;
      if (s_prefix[mid] <= pos) blo = mid; else bhi = mid - 1;
    }
    const int item = blo;
    const int b = Rows::seq(p, item), len = Rows::item_len(p, item);  // the sequence, the tokens the item attends to
    const int tiles_b = (len + kTile - 1) / kTile;
    const int within = pos - s_prefix[item];
    const int g = within / tiles_b, t0 = within - g * tiles_b;
    const int bg_start = s_prefix[item] + g * tiles_b, bg_end = bg_start + tiles_b;
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
      if (i < ntiles) load_tile<QM>(p, smem + i * T::STAGE, ktab, vtab, g, tok0 + i * kTile, tok1);
      cp_async_commit();
    }

    // ---- Q fragments (A operand, rows = q-heads of this kv-group).  The head-dim order each thread uses is free as
    //      long as Q and K agree, so it follows how that thread reads K: natural for bf16 (ldmatrix), per-thread
    //      contiguous 32-d slices for the quantized modes.  Quantized modes run the MMAs in fp16.
    const Rows rows(p, item, b, g, len, tok1, gq);  // after the prefetch: a tree's ancestor walk reads global memory
    uint32_t qa[8][4];
    float sq[2] = {0.f, 0.f};  // sum_d Q[row][d] over this thread's d-slice, then over the quad (quantized modes)
    {
      // quantized modes: stage the group's hpg x 128 query rows through shared memory with 16-byte loads (one global round
      // trip; their fragment orders would otherwise need 64 scalar loads per thread: 3.3 us measured at ctx 32768)
      // [16][128] in the LAST ring stage: the only one the prefetch above does not write (it is first filled at iteration 0)
      __nv_bfloat16* qs = reinterpret_cast<__nv_bfloat16*>(smem + (p.nstage - 1) * T::STAGE);
      if (QM != B2_KV_NONE) {
        for (int i = tid; i < 16 * (kHead / 8); i += kAttnThreads) {
          const int row = i >> 4;
          *reinterpret_cast<uint4*>(qs + row * kHead + (i & 15) * 8) =
              row < rows.nrows ? *reinterpret_cast<const uint4*>(rows.at(p.q, row) + (i & 15) * 8) : make_uint4(0, 0, 0, 0);
        }
        __syncthreads();
      }
      const bool r0 = gq < rows.nrows, r1 = (gq + 8) < rows.nrows;
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        if (QM == B2_KV_NONE) {  // natural d order: 32 independent 4-byte loads per thread straight from global memory
          const int d0 = 16 * ks + 2 * t;
          const __nv_bfloat16 *q0 = rows.at(p.q, gq), *q1 = rows.at(p.q, gq + 8);
          qa[ks][0] = r0 ? *reinterpret_cast<const uint32_t*>(q0 + d0) : 0u;
          qa[ks][1] = r1 ? *reinterpret_cast<const uint32_t*>(q1 + d0) : 0u;
          qa[ks][2] = r0 ? *reinterpret_cast<const uint32_t*>(q0 + d0 + 8) : 0u;
          qa[ks][3] = r1 ? *reinterpret_cast<const uint32_t*>(q1 + d0 + 8) : 0u;
        } else {
          float f[2][4];
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const __nv_bfloat16* qr = qs + (gq + 8 * rr) * kHead;
#pragma unroll
            for (int j = 0; j < 4; ++j) f[rr][j] = F::to_f(qr[DOrder<QM>::q(t, ks, j)]);
          }
          qa[ks][0] = pack_f16x2(f[0][0], f[0][1]);
          qa[ks][1] = pack_f16x2(f[1][0], f[1][1]);
          qa[ks][2] = pack_f16x2(f[0][2], f[0][3]);
          qa[ks][3] = pack_f16x2(f[1][2], f[1][3]);
#pragma unroll
          for (int rr = 0; rr < 2 && QM != B2_KV_FP8; ++rr) {  // sums of exactly the fp16 values the tensor core multiplies
            const __half2 ha = *reinterpret_cast<const __half2*>(&qa[ks][rr]), hb = *reinterpret_cast<const __half2*>(&qa[ks][2 + rr]);
            sq[rr] += (__low2float(ha) + __high2float(ha)) + (__low2float(hb) + __high2float(hb));
          }
        }
      }
      if (QM != B2_KV_NONE && QM != B2_KV_FP8) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) quad_sum(sq[rr]);
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
      if (pf < ntiles) load_tile<QM>(p, smem + pslot * T::STAGE, ktab, vtab, g, tok0 + pf * kTile, tok1);
      cp_async_commit();
      // all groups except the newest (nstage-1) are complete -> tile i has landed
      if (p.nstage == 2) cp_async_wait<1>(); else if (p.nstage == 3) cp_async_wait<2>(); else cp_async_wait<3>();
      __syncthreads();
      if (tr0 && i == 0) B2_TR(g_attn_tr, 4);
      const int wtok = tok0 + i * kTile + warp * 16;  // first token of this warp's slice
      if (wtok < tok1) {
        if constexpr (!T::kCodesF16)
          tile_compute_bf16<H>(smem + slot * T::STAGE, warp, lane, wtok, rows.mask, p.scale_log2, qa, o, mrow, lrow);
        else tile_compute_q<QM>(smem + slot * T::STAGE, warp, lane, wtok, rows.mask, p.scale_log2, qa, sq, o, mrow, lrow, cacc);
      }
      __syncthreads();  // this stage may be refilled by the next iteration's prefetch
      slot = slot + 1 == p.nstage ? 0 : slot + 1;
      pslot = pslot + 1 == p.nstage ? 0 : pslot + 1;
    }
    cp_async_wait<0>();
    if (tr0) B2_TR(g_attn_tr, 5);

    // ---------------- merge the 4 warps (each saw a disjoint token slice) ----------------
    if (T::kZeroPoint) {  // subtract the zero-point term (quad-reduced) before leaving registers
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) quad_sum(cacc[rr]);
#pragma unroll
      for (int dt = 0; dt < 16; ++dt) {
        o[dt][0] -= cacc[0]; o[dt][1] -= cacc[0];
        o[dt][2] -= cacc[1]; o[dt][3] -= cacc[1];
      }
    }
    {
      // quantized: one float4 store per 4 consecutive d of DOrder, at the d of its first element.  Scalar stores per o[]
      // element are not merged back into float4s, and `if constexpr` here makes ptxas allocate registers differently.
      using D = DOrder<QM>;
      float* m0 = mrg + (warp * 16 + gq) * kMergeRS;
      float* m1 = mrg + (warp * 16 + gq + 8) * kMergeRS;
      if (!T::kCodesF16) {
#pragma unroll
        for (int dt = 0; dt < 16; ++dt) {
          const int d = 8 * dt + 2 * t;
          *reinterpret_cast<float2*>(m0 + d) = make_float2(o[dt][0], o[dt][1]);
          *reinterpret_cast<float2*>(m1 + d) = make_float2(o[dt][2], o[dt][3]);
        }
      } else if (QM != B2_KV_U4) {  // d + {0, 1, 2, 3} = o[2c][0], o[2c+1][0], o[2c][1], o[2c+1][1]
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const int d = D::o(t, 2 * c, 0);
          *reinterpret_cast<float4*>(m0 + d) = make_float4(o[2 * c][0], o[2 * c + 1][0], o[2 * c][1], o[2 * c + 1][1]);
          *reinterpret_cast<float4*>(m1 + d) = make_float4(o[2 * c][2], o[2 * c + 1][2], o[2 * c][3], o[2 * c + 1][3]);
        }
      } else {  // d + {0, 1, 2, 3} = o[4c + {0, 1, 2, 3}][e]
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int d = D::o(t, 4 * c, 0), d1 = D::o(t, 4 * c, 1);
          *reinterpret_cast<float4*>(m0 + d) = make_float4(o[4 * c][0], o[4 * c + 1][0], o[4 * c + 2][0], o[4 * c + 3][0]);
          *reinterpret_cast<float4*>(m0 + d1) = make_float4(o[4 * c][1], o[4 * c + 1][1], o[4 * c + 2][1], o[4 * c + 3][1]);
          *reinterpret_cast<float4*>(m1 + d) = make_float4(o[4 * c][2], o[4 * c + 1][2], o[4 * c + 2][2], o[4 * c + 3][2]);
          *reinterpret_cast<float4*>(m1 + d1) = make_float4(o[4 * c][3], o[4 * c + 1][3], o[4 * c + 2][3], o[4 * c + 3][3]);
        }
      }
    }
    if (t == 0) {  // quantized: o carries the 2^kPExp folded into P', and l takes it here (exact), so o / l is unchanged
      mrg_ml[(warp * 16 + gq) * 2] = mrow[0];
      mrg_ml[(warp * 16 + gq) * 2 + 1] = T::kCodesF16 ? lrow[0] * T::kPScale : lrow[0];
      mrg_ml[(warp * 16 + gq + 8) * 2] = mrow[1];
      mrg_ml[(warp * 16 + gq + 8) * 2 + 1] = T::kCodesF16 ? lrow[1] * T::kPScale : lrow[1];
    }
    __syncthreads();
    // thread d = tid handles column d of every head row
    const int cnt_idx = item * p.n_groups + g;
    const int my_slot = 2 * blockIdx.x + (pos != lo ? 1 : 0);
    for (int r = 0; r < rows.nrows; ++r) {
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
        rows.at(p.out, r)[tid] = F::from_f(acc / L);
      } else {
        p.ws_o[((size_t)my_slot * rows.rstride + r) * kHead + tid] = acc;
        if (tid == 0) {
          p.ws_ml[((size_t)my_slot * rows.rstride + r) * 2] = M;
          p.ws_ml[((size_t)my_slot * rows.rstride + r) * 2 + 1] = L;
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
      if (npieces <= kMergeDirect) {
        if (tid == 0) s_is_last = atomicAdd(&p.counters[cnt_idx], 1u) == (unsigned)(npieces - 1);
        __syncthreads();
        if (s_is_last) {
          __threadfence();
          if (tid == 0 && cnt_idx == 0) B2_TR(g_attn_tr, 10);
          merge_partials<true, H>(p.ws_o, p.ws_ml, 2 * k0, 2, first_par, npieces, rows, p.out, nullptr, nullptr, 0, s_w, s_ML);
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
          merge_partials<false, H>(p.ws_o, p.ws_ml, 2 * (k0 + q * kMergeFan), 2, q == 0 ? first_par : 0, gsize, rows, nullptr,
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
            merge_partials<true, H>(p.ws2_o, p.ws2_ml, 2 * k0, 2 * kMergeFan, first_par, ngroups, rows, p.out, nullptr, nullptr, 0,
                                    s_w, s_ML);
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

// FP8 row quantizer (B2_KV_FP8, the convention of b2_quant_fp8): scale = max(amax, 1e-12) / 448 and r = 1 / scale, both
// IEEE fp32 (this library is built without fast math), code = e4m3(x * r), round to nearest even, saturating to +-448 —
// a finite input never becomes 0x7F / 0xFF (the two e4m3fn NaNs).  Returns the lane's 4 codes, element 0 in the low byte.
__device__ __forceinline__ uint32_t quant_row_fp8(const float (&x)[4], float& qs) {
  float amax = fmaxf(fmaxf(fabsf(x[0]), fabsf(x[1])), fmaxf(fabsf(x[2]), fabsf(x[3])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  qs = fmaxf(amax, 1e-12f) / 448.f;
  const float r = 1.f / qs;
  uint16_t p01, p23;  // cvt puts its FIRST source in the UPPER byte
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(p01) : "f"(x[1] * r), "f"(x[0] * r));
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(p23) : "f"(x[3] * r), "f"(x[2] * r));
  return (uint32_t)p01 | ((uint32_t)p23 << 16);
}

// store one (possibly quantized) 128-wide row at row index rowi of a span of n_rows rows (format: KVTraits)
template <int QM, bool H>
__device__ __forceinline__ void store_row(uint8_t* span, size_t rowi, int n_rows, int lane, const float (&x)[4]) {
  using T = KVTraits<QM>;
  if constexpr (QM == B2_KV_NONE) {
    *reinterpret_cast<uint2*>(span + rowi * T::ROW + lane * 8) = make_uint2(Ft<H>::pack(x[0], x[1]), Ft<H>::pack(x[2], x[3]));
  } else if constexpr (QM == B2_KV_FP8) {
    float s;
    *reinterpret_cast<uint32_t*>(span + rowi * T::ROW + lane * 4) = quant_row_fp8(x, s);
    if (lane == 0) *reinterpret_cast<float2*>(span + T::param_offset(n_rows, rowi)) = make_float2(0.f, s);
  } else {
    float qz, qs;
    int qv[4];
    quant_row<QM>(x, qz, qs, qv);
    if constexpr (QM == B2_KV_I8) {
      const uint32_t w = (qv[0] & 0xff) | ((qv[1] & 0xff) << 8) | ((qv[2] & 0xff) << 16) | ((uint32_t)(qv[3] & 0xff) << 24);
      *reinterpret_cast<uint32_t*>(span + rowi * T::ROW + lane * 4) = w;
    } else {
      const uint16_t w = (uint16_t)((qv[0] & 0xf) | ((qv[1] & 0xf) << 4) | ((qv[2] & 0xf) << 8) | ((qv[3] & 0xf) << 12));
      *reinterpret_cast<uint16_t*>(span + rowi * T::ROW + lane * 2) = w;
    }
    if (lane == 0) *reinterpret_cast<float2*>(span + T::param_offset(n_rows, rowi)) = make_float2(qz, qs);
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
  int q_len;       // multi-token forms: rows per sequence
  const int32_t* parents;  // tree form: the draft tree of each sequence (format: AttnTreeParams)
};

// Where row `row` of qkv / q_out goes: its sequence b, the slot it is written to and its rotary position.
// MT = false: row b is sequence b, at position old_lens[b].  MT = true: row b*q_len + t is token t of sequence b, at position
// old_lens[b] + t.  TREE (with MT): at slot old_lens[b] + t, rotary position old_lens[b] + depth(t).
template <bool MT, bool TREE>
__device__ __forceinline__ void append_row(const AppendParams& p, int row, int& b, int& slot, int& pos) {
  b = MT ? row / p.q_len : row;
  slot = pos = MT ? p.old_lens[b] + (row - b * p.q_len) : p.old_lens[b];
  if constexpr (TREE) {
    int depth;
    tree_walk(p.parents + (size_t)b * p.q_len, row - b * p.q_len, depth);
    pos = p.old_lens[b] + depth;
  }
}

template <int QM, bool H, bool MT = false, bool TREE = false>
__global__ void __launch_bounds__(128) cache_append_kernel(const AppendParams p) {
  using F = Ft<H>;
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int slots = p.n_heads + 2 * p.n_groups;
  const int wid = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (wid >= (MT ? p.batch * p.q_len : p.batch) * slots) return;
  const int row = wid / slots, slot = wid - row * slots;
  const __nv_bfloat16* src = p.qkv + ((size_t)row * slots + slot) * kHead + lane * 4;
  const uint2 raw = *reinterpret_cast<const uint2*>(src);
  float x[4] = {F::lo(raw.x), F::hi(raw.x), F::lo(raw.y), F::hi(raw.y)};
  int b, wpos, pos;
  append_row<MT, TREE>(p, row, b, wpos, pos);
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
    *reinterpret_cast<uint2*>(p.q_out + ((size_t)row * p.n_heads + slot) * kHead + lane * 4) =
        make_uint2(F::pack(x[0], x[1]), F::pack(x[2], x[3]));
    return;
  }
  const int g = is_v ? slot - p.n_heads - p.n_groups : slot - p.n_heads;
  void* const* tab = (is_v ? p.v_spans : p.k_spans) + (size_t)b * p.max_spans;
  const int si = wpos >> p.span_shift, ps = wpos & (p.span_len - 1);
  uint8_t* span = reinterpret_cast<uint8_t*>(tab[si]);
  const size_t rowi = (size_t)g * p.span_len + ps;
  store_row<QM, H>(span, rowi, p.n_groups * p.span_len, lane, x);
}

// ------------------------------------------------------------------------------------------------
// compaction after tree acceptance: the accepted path's rows (slots base + path[i]) move to slots base + i, for every layer.
// One warp per (layer, sequence, K or V, kv-head) reads all of its source rows (and their {zero, scale}) before it writes
// any: path[j] == i for j < i is possible (path [0, 2, 3] reads slot 2 while slot 2 is being written).  A row carries RoPE at
// base + depth = base + i already, so the copy is exact bytes.
// ------------------------------------------------------------------------------------------------
struct CompactParams {
  void* const* const* k_tables;  // [n_layers] -> span table [batch][max_spans]
  void* const* const* v_tables;
  const int32_t* old_lens;       // as b2_spec_accept_tree left them: base = old_lens[b] - accepted[b]
  const int32_t* accepted;
  const int32_t* path;           // [batch][q_len]
  int n_layers, batch, q_len, n_groups, span_len, span_shift, max_spans;
};

template <int QM>
__global__ void __launch_bounds__(128) cache_compact_kernel(const CompactParams p) {
  using T = KVTraits<QM>;
  constexpr int BPL = T::ROW / 32;  // row bytes per lane: 8 / 4 / 2
  using Chunk = std::conditional_t<BPL == 8, uint2, std::conditional_t<BPL == 4, uint32_t, uint16_t>>;
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int wid = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (wid >= p.n_layers * p.batch * 2 * p.n_groups) return;
  const int g = wid % p.n_groups, which = (wid / p.n_groups) & 1;
  const int b = (wid / (2 * p.n_groups)) % p.batch, layer = wid / (2 * p.n_groups * p.batch);
  const int n = min(max(p.accepted[b], 1), p.q_len);
  const int base = p.old_lens[b] - n;
  const int32_t* path = p.path + (size_t)b * p.q_len;
  void* const* tab = (which ? p.v_tables : p.k_tables)[layer] + (size_t)b * p.max_spans;
  const size_t n_rows = (size_t)p.n_groups * p.span_len;
  auto row_of = [&](int s, uint8_t*& span) {  // span and row index of slot s
    span = reinterpret_cast<uint8_t*>(tab[s >> p.span_shift]);
    return (size_t)g * p.span_len + (s & (p.span_len - 1));
  };
  Chunk buf[kMaxQLen];
  float2 prm = make_float2(0.f, 0.f);
  int src[kMaxQLen];
#pragma unroll
  for (int i = 1; i < kMaxQLen; ++i) {
    const int j = i < n ? path[i] : i;
    src[i] = (unsigned)j < (unsigned)p.q_len ? j : i;  // a malformed path entry: no move
    if (src[i] != i) {
      uint8_t* span;
      const size_t r = row_of(base + src[i], span);
      buf[i] = *reinterpret_cast<const Chunk*>(span + r * T::ROW + lane * BPL);
      if (T::kCodesF16 && lane == i) prm = *reinterpret_cast<const float2*>(span + T::param_offset(n_rows, r));
    }
  }
  __syncwarp();
#pragma unroll
  for (int i = 1; i < kMaxQLen; ++i) {
    if (src[i] != i) {
      uint8_t* span;
      const size_t r = row_of(base + i, span);
      *reinterpret_cast<Chunk*>(span + r * T::ROW + lane * BPL) = buf[i];
      if (T::kCodesF16 && lane == i) *reinterpret_cast<float2*>(span + T::param_offset(n_rows, r)) = prm;
    }
  }
}

int span_attn64_run(const b2_span_cfg* c, void* out, const void* q, const void* const* k_spans, const void* const* v_spans,
                    const int32_t* lens, int batch, float qk_scale, cudaStream_t stream);
int span_append64_run(const b2_span_cfg* c, void* const* k_spans, void* const* v_spans, void* q_out, const void* qkv,
                      const int32_t* old_lens, int batch, const b2_rope_cfg* rope, cudaStream_t stream);

static int check_cfg(const b2_span_cfg* c) {
  if (!c) return B2_ERR_PARAM;
  if (c->ft != B2_DT_BF16 && c->ft != B2_DT_F16) return B2_ERR_UNSUPPORTED;
  if (c->ft == B2_DT_F16 && c->head_size != kHead) return B2_ERR_UNSUPPORTED;  // the head-64 kernels are bf16 only
  // 128: the reference GPU library's only head size (span_attention.hpp:203-208).  64: bf16 KV only — the parity anchor C0
  // (Qwen2-0.5B) that the reference runs on its CPU path; span_attn64.cu
  if (c->head_size != kHead && !(c->head_size == 64 && c->quant_mode == B2_KV_NONE)) return B2_ERR_UNSUPPORTED;
  if (c->quant_mode < B2_KV_NONE || c->quant_mode > B2_KV_FP8) return B2_ERR_PARAM;
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

// The step forms of the attention and append kernels: 0 single token, 1 chain (MT), 2 tree (MT, TREE).
// form -> template arguments: f(std::bool_constant<MT>, std::bool_constant<TREE>)
template <typename F>
static auto with_step_form(int form, F&& f) {
  if (form == 2) return f(std::true_type{}, std::true_type{});
  if (form == 1) return f(std::true_type{}, std::false_type{});
  return f(std::false_type{}, std::false_type{});
}

template <bool MT, bool TREE>
static auto attn_kernel_for(const b2_span_cfg* c) {
  using kernel_t = void (*)(const AttnArgs<MT, TREE>);
  return with_kv_mode(c->quant_mode, [&](auto QM) {
    return with_flag(c->ft == B2_DT_F16, [&](auto H) -> kernel_t { return span_attn_kernel<QM, H, MT, TREE>; });
  });
}

// multi-token row blocks: whole tokens per block of 16 MMA rows
static int tokens_per_block(const b2_span_cfg* c, int q_len) {
  const int tpb = 16 / (c->n_heads / c->n_groups);
  return q_len < tpb ? q_len : tpb;
}

// bytes of one token row of one kv-head in a span (KVTraits::SPAN_ROW; head 64 is bf16 only)
static size_t span_row_bytes(const b2_span_cfg* c) {
  if (c->head_size != kHead) return (size_t)c->head_size * 2;
  return with_kv_mode(c->quant_mode, [](auto QM) { return (size_t)KVTraits<QM>::SPAN_ROW; });
}

extern "C" {

size_t b2_span_bytes(const b2_span_cfg* c) {
  if (check_cfg(c) != B2_OK) return 0;
  return (size_t)c->span_len * c->n_groups * span_row_bytes(c);  // csrc/runtime/cache/virtual_cache.cpp:202-232
}

size_t b2_span_attn_algo_bytes(const b2_span_cfg* c, int64_t total_tokens) {
  if (check_cfg(c) != B2_OK) return 0;
  return (size_t)total_tokens * 2 * c->n_groups * span_row_bytes(c);
}

int b2_span_attn_create(b2_span_attn_t* out, const b2_span_cfg* cfg, int max_batch) {
  if (!out) return B2_ERR_PARAM;
  if (int st = check_cfg(cfg)) return st;
  if (max_batch <= 0 || max_batch > kMaxBatch) return B2_ERR_LIMIT;
  b2_span_attn* h = new (std::nothrow) b2_span_attn();
  if (!h) return B2_ERR_RUNTIME;
  h->cfg = *cfg;
  h->max_batch = max_batch;
  const auto kern = attn_kernel_for<false, false>(cfg);
  int sb = 0;
  with_kv_mode(cfg->quant_mode, [&](auto QM) {
    sb = KVTraits<QM>::STAGE;
    h->nstage = env_int("B2_ATTN_STAGES", KVTraits<QM>::kStages);
  });
  if (h->nstage < 2) h->nstage = 2;
  if (h->nstage > 4) h->nstage = 4;
  const int merge = (4 * 16 * kMergeRS + 4 * 16 * 2) * 4;
  h->smem = h->nstage * sb > merge ? h->nstage * sb : merge;
  cudaError_t e = cudaSuccess;
  for (int form = 0; form < (cfg->head_size == kHead ? 3 : 1) && e == cudaSuccess; ++form)  // head 64 has the single-token form only
    e = with_step_form(form, [&](auto MT, auto TREE) {
      return cudaFuncSetAttribute(attn_kernel_for<MT, TREE>(cfg), cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem);
    });
  int occ = 1;
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kAttnThreads, h->smem);
  if (e != cudaSuccess) {
    set_last_error("b2_span_attn_create(occupancy)", e);
    delete h;
    return B2_ERR_CUDA;
  }
  if (occ < 1) occ = 1;
  const int want = env_int("B2_ATTN_CTAS_PER_SM", 0);  // ignored when <= 0
  if (want > 0 && want < occ) occ = want;
  // the multi-token kernel launches the same grid (and so the same partial slots): its merges are done by the last CTA to
  // arrive and never wait for another, so any grid is correct; its register count (162-168 against 160) leaves the
  // occupancy of these 128-thread CTAs unchanged
  h->grid = occ * sm_count();
  const int max_pieces = env_int("B2_ATTN_MAX_PIECES", 0);  // ignored when <= 0
  if (max_pieces > 0) h->max_pieces = max_pieces;
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

}  // extern "C"

// split-KV partials: at most two per CTA (its first and its last piece), independent of batch and length
static size_t partial_slots(const b2_span_attn* h) { return (size_t)2 * h->grid; }

// level-0 and level-1 partials of `rows` rows per slot
static size_t attn_workspace_bytes(const b2_span_attn* h, int rows) {
  return 2 * partial_slots(h) * rows * (kHead + 2) * sizeof(float) + 256;
}

// the workspace of a step of q_len tokens per sequence (1: the single-token form)
static size_t attn_step_workspace_bytes(const b2_span_attn* h, int q_len) {
  return attn_workspace_bytes(h, tokens_per_block(&h->cfg, q_len) * (h->cfg.n_heads / h->cfg.n_groups));
}

// The checks of the attention entry points, in the order their callers observe.  ptrs_ok: no required pointer is NULL.
static int attn_check(b2_span_attn_t h, bool ptrs_ok, int form, int batch, int q_len, int max_len, const void* workspace,
                      size_t workspace_bytes) {
  if (!h || !ptrs_ok) return B2_ERR_PARAM;
  if (form != 0 && h->cfg.head_size != kHead) return B2_ERR_UNSUPPORTED;
  if (q_len < 1 || q_len > kMaxQLen || batch <= 0 || (int64_t)batch * q_len > h->max_batch) return B2_ERR_LIMIT;
  if (max_len <= 0 || (int64_t)(max_len + h->cfg.span_len - 1) / h->cfg.span_len > h->cfg.max_spans_per_seq) return B2_ERR_LIMIT;
  if (!workspace || workspace_bytes < attn_step_workspace_bytes(h, q_len)) return B2_ERR_PARAM;
  return B2_OK;
}

// q_len tokens per sequence (1 in the single-token form); parents: the tree form's
static int attn_launch(b2_span_attn_t h, void* out, const void* q, const void* const* k_spans, const void* const* v_spans,
                       const int32_t* new_lens, const int32_t* parents, int form, int batch, int q_len, void* workspace,
                       float qk_scale, void* stream_) {
  const int hpg = h->cfg.n_heads / h->cfg.n_groups;
  AttnTreeParams p;  // each form's kernel takes the base it needs (AttnArgs)
  p.parents = parents;
  p.q_len = q_len;
  p.tpb = tokens_per_block(&h->cfg, q_len);
  p.nrb = (q_len + p.tpb - 1) / p.tpb;
  p.rstride = p.tpb * hpg;
  const size_t rows = p.rstride;
  p.out = (__nv_bfloat16*)out;
  p.q = (const __nv_bfloat16*)q;
  p.k_spans = k_spans;
  p.v_spans = v_spans;
  p.lens = new_lens;
  const size_t items = partial_slots(h);
  p.ws_o = (float*)(((uintptr_t)workspace + 127) & ~(uintptr_t)127);
  p.ws_ml = p.ws_o + items * rows * kHead;
  p.ws2_o = p.ws_ml + items * rows * 2;
  p.ws2_ml = p.ws2_o + items * rows * kHead;
  p.counters = h->counters;
  p.counters1 = h->counters + (size_t)h->max_batch * h->cfg.n_groups;
  p.max_pieces = h->max_pieces;
  p.batch = batch; p.n_heads = h->cfg.n_heads; p.n_groups = h->cfg.n_groups; p.hpg = hpg;
  p.span_len = h->cfg.span_len; p.span_shift = ilog2(h->cfg.span_len); p.max_spans = h->cfg.max_spans_per_seq;
  p.nstage = h->nstage;
  p.scale_log2 = qk_scale * 1.4426950408889634f;
  const cudaError_t e = with_step_form(form, [&](auto MT, auto TREE) {
    return launch(attn_kernel_for<MT, TREE>(&h->cfg), dim3(h->grid), dim3(kAttnThreads), (size_t)h->smem, (cudaStream_t)stream_, true, p);
  });
  if (e != cudaSuccess) {
    set_last_error("span_attn launch", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

extern "C" {

size_t b2_span_attn_workspace_bytes(b2_span_attn_t h, int batch, int max_len) {
  if (!h || batch <= 0 || max_len <= 0) return 0;
  return attn_step_workspace_bytes(h, 1);
}

int b2_span_attn_run(b2_span_attn_t h, void* out, const void* q, const void* const* k_spans, const void* const* v_spans,
                     const int32_t* new_lens, int batch, int max_len, void* workspace, size_t workspace_bytes,
                     float qk_scale, void* stream_) {
  if (int st = attn_check(h, out && q && k_spans && v_spans && new_lens, 0, batch, 1, max_len, workspace, workspace_bytes)) return st;
  if (h->cfg.head_size == 64) return span_attn64_run(&h->cfg, out, q, k_spans, v_spans, new_lens, batch, qk_scale, (cudaStream_t)stream_);
  return attn_launch(h, out, q, k_spans, v_spans, new_lens, nullptr, 0, batch, 1, workspace, qk_scale, stream_);
}

size_t b2_span_attn_tokens_workspace_bytes(b2_span_attn_t h, int batch, int q_len, int max_len) {
  if (!h || batch <= 0 || q_len < 1 || q_len > kMaxQLen || max_len <= 0) return 0;
  return attn_step_workspace_bytes(h, q_len);
}

int b2_span_attn_run_tokens(b2_span_attn_t h, void* out, const void* q, const void* const* k_spans, const void* const* v_spans,
                            const int32_t* new_lens, int batch, int q_len, int max_len, void* workspace, size_t workspace_bytes,
                            float qk_scale, void* stream_) {
  if (int st = attn_check(h, out && q && k_spans && v_spans && new_lens, 1, batch, q_len, max_len, workspace, workspace_bytes)) return st;
  return attn_launch(h, out, q, k_spans, v_spans, new_lens, nullptr, 1, batch, q_len, workspace, qk_scale, stream_);
}

int b2_span_attn_run_tree(b2_span_attn_t h, void* out, const void* q, const void* const* k_spans, const void* const* v_spans,
                          const int32_t* new_lens, const int32_t* parents, int batch, int q_len, int max_len, void* workspace,
                          size_t workspace_bytes, float qk_scale, void* stream_) {
  if (int st = attn_check(h, out && q && k_spans && v_spans && new_lens && parents, 2, batch, q_len, max_len, workspace, workspace_bytes))
    return st;
  return attn_launch(h, out, q, k_spans, v_spans, new_lens, parents, 2, batch, q_len, workspace, qk_scale, stream_);
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
  const cudaError_t e = with_kv_mode(cfg->quant_mode, [&](auto QM) {
    return with_flag(cfg->ft == B2_DT_F16, [&](auto H) {
      return launch(context_span_copy_kernel<QM, H>, grid, block, 0, (cudaStream_t)stream_, true, p);
    });
  });
  if (e != cudaSuccess) {
    set_last_error("context_span_copy launch", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

}  // extern "C"

// The checks of the append and compaction entry points, in the order their callers observe.  args_ok: no required pointer
// is NULL and every count is positive.
static int append_check(const b2_span_cfg* cfg, bool args_ok, int form, int q_len) {
  if (int st = check_cfg(cfg)) return st;
  if (form != 0 && cfg->head_size != kHead) return B2_ERR_UNSUPPORTED;
  if (!args_ok) return B2_ERR_PARAM;
  if (q_len < 1 || q_len > kMaxQLen) return B2_ERR_LIMIT;
  return B2_OK;
}

// q_len rows per sequence (1 in the single-token form), the nodes of the draft tree `parents` in the tree form
static int cache_append_launch(const b2_span_cfg* cfg, void* const* k_spans, void* const* v_spans, void* q_out, const void* qkv,
                               const int32_t* old_lens, const int32_t* parents, int form, int batch, int q_len,
                               const b2_rope_cfg* rope, void* stream_) {
  if (rope && (rope->rotary_dim != 128 && rope->rotary_dim != 64)) return B2_ERR_UNSUPPORTED;
  AppendParams p;
  p.parents = parents;
  p.k_spans = k_spans; p.v_spans = v_spans;
  p.q_out = (__nv_bfloat16*)q_out; p.qkv = (const __nv_bfloat16*)qkv; p.old_lens = old_lens;
  p.batch = batch; p.n_heads = cfg->n_heads; p.n_groups = cfg->n_groups;
  p.span_len = cfg->span_len; p.span_shift = ilog2(cfg->span_len); p.max_spans = cfg->max_spans_per_seq;
  p.rope = rope ? 1 : 0;
  p.rotary_dim = rope ? rope->rotary_dim : 0;
  p.log2_base = rope ? log2f(rope->base) : 0.f;
  p.q_len = q_len;
  const int warps = batch * q_len * (cfg->n_heads + 2 * cfg->n_groups);
  const dim3 grid((warps + 3) / 4), block(128);
  const cudaError_t e = with_kv_mode(cfg->quant_mode, [&](auto QM) {
    return with_flag(cfg->ft == B2_DT_F16, [&](auto H) {
      return with_step_form(form, [&](auto MT, auto TREE) {
        return launch(cache_append_kernel<QM, H, MT, TREE>, grid, block, 0, (cudaStream_t)stream_, true, p);
      });
    });
  });
  if (e != cudaSuccess) {
    set_last_error("cache_append launch", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

extern "C" {

int b2_span_cache_append(const b2_span_cfg* cfg, void* const* k_spans, void* const* v_spans, void* q_out,
                         const void* qkv, const int32_t* old_lens, int batch, const b2_rope_cfg* rope, void* stream_) {
  if (int st = append_check(cfg, k_spans && v_spans && q_out && qkv && old_lens && batch > 0, 0, 1)) return st;
  if (cfg->head_size == 64) return span_append64_run(cfg, k_spans, v_spans, q_out, qkv, old_lens, batch, rope, (cudaStream_t)stream_);
  return cache_append_launch(cfg, k_spans, v_spans, q_out, qkv, old_lens, nullptr, 0, batch, 1, rope, stream_);
}

int b2_span_cache_append_tokens(const b2_span_cfg* cfg, void* const* k_spans, void* const* v_spans, void* q_out, const void* qkv,
                                const int32_t* old_lens, int batch, int q_len, const b2_rope_cfg* rope, void* stream_) {
  if (int st = append_check(cfg, k_spans && v_spans && q_out && qkv && old_lens && batch > 0, 1, q_len)) return st;
  return cache_append_launch(cfg, k_spans, v_spans, q_out, qkv, old_lens, nullptr, 1, batch, q_len, rope, stream_);
}

int b2_span_cache_append_tree(const b2_span_cfg* cfg, void* const* k_spans, void* const* v_spans, void* q_out, const void* qkv,
                              const int32_t* old_lens, const int32_t* parents, int batch, int q_len, const b2_rope_cfg* rope,
                              void* stream_) {
  if (int st = append_check(cfg, k_spans && v_spans && q_out && qkv && old_lens && parents && batch > 0, 2, q_len)) return st;
  return cache_append_launch(cfg, k_spans, v_spans, q_out, qkv, old_lens, parents, 2, batch, q_len, rope, stream_);
}

int b2_span_cache_compact(const b2_span_cfg* cfg, void* const* const* k_tables, void* const* const* v_tables, int n_layers,
                          const int32_t* old_lens, const int32_t* accepted, const int32_t* path, int batch, int q_len,
                          void* stream_) {
  if (int st = append_check(cfg, k_tables && v_tables && old_lens && accepted && path && n_layers > 0 && batch > 0, 2, q_len)) return st;
  CompactParams p;
  p.k_tables = k_tables; p.v_tables = v_tables;
  p.old_lens = old_lens; p.accepted = accepted; p.path = path;
  p.n_layers = n_layers; p.batch = batch; p.q_len = q_len; p.n_groups = cfg->n_groups;
  p.span_len = cfg->span_len; p.span_shift = ilog2(cfg->span_len); p.max_spans = cfg->max_spans_per_seq;
  const int64_t warps = (int64_t)n_layers * batch * 2 * cfg->n_groups;
  if (warps > (int64_t)1 << 30) return B2_ERR_LIMIT;
  const dim3 grid((unsigned)((warps + 3) / 4)), block(128);
  const cudaError_t e = with_kv_mode(cfg->quant_mode, [&](auto QM) {
    return launch(cache_compact_kernel<QM>, grid, block, 0, (cudaStream_t)stream_, true, p);
  });
  if (e != cudaSuccess) {
    set_last_error("cache_compact launch", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

}  // extern "C"
