// b200spark — shared device helpers (sm_90a): mbarrier, TMA bulk copy, cp.async, mma.sync,
// ldmatrix, programmatic dependent launch, error plumbing.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/b200spark.h"

namespace b2 {

// ------------------------------------------------------------------ host-side error plumbing
void set_last_error(const char* what, cudaError_t e);
int launch_failed(const char* what);  // returns B2_OK or B2_ERR_CUDA after checking cudaGetLastError
bool pdl_enabled();
int sm_count();
int max_smem_optin();
int env_int(const char* name, int dflt);  // integer value of environment variable `name`, dflt if unset

inline int ilog2(int x) {  // ceil(log2(x)); the shift of a power-of-two span length
  int s = 0;
  while ((1 << s) < x) ++s;
  return s;
}

// Runtime flag / KV-cache mode -> template argument: f(std::bool_constant<b>) / f(std::integral_constant<int, QM>).
// Modes above B2_KV_FP8 are rejected before dispatch; they would run as B2_KV_U4.
template <typename F>
inline auto with_flag(bool b, F&& f) {
  return b ? f(std::true_type{}) : f(std::false_type{});
}
template <typename F>
inline auto with_kv_mode(int qm, F&& f) {
  if (qm == B2_KV_NONE) return f(std::integral_constant<int, B2_KV_NONE>{});
  if (qm == B2_KV_I8) return f(std::integral_constant<int, B2_KV_I8>{});
  if (qm == B2_KV_FP8) return f(std::integral_constant<int, B2_KV_FP8>{});
  return f(std::integral_constant<int, B2_KV_U4>{});
}

#define B2_CUDA_TRY(expr)                         \
  do {                                            \
    cudaError_t _e = (expr);                      \
    if (_e != cudaSuccess) {                      \
      ::b2::set_last_error(#expr, _e);            \
      return B2_ERR_CUDA;                         \
    }                                             \
  } while (0)

// Launch with optional PDL attribute.
template <typename... KArgs, typename... Args>
inline cudaError_t launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                          bool pdl, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = (pdl && pdl_enabled()) ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// Same, as thread-block clusters of `cluster_x` consecutive CTAs (distributed shared memory between the k-slices of a tile).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl,
                                  unsigned cluster_x, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster_x;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = (pdl && pdl_enabled()) ? 2 : 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// ------------------------------------------------------------------ device helpers
#ifdef __CUDACC__

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- thread-block clusters: barrier + distributed shared memory reads
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t dsmem_addr(uint32_t local_smem_addr, uint32_t cta_rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(cta_rank));
  return r;
}
__device__ __forceinline__ float4 ld_dsmem_f4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ float ld_dsmem_f(uint32_t addr) {
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}

// ---- optional timeline instrumentation (-DB2_TRACE): globaltimer stamps into a per-translation-unit buffer
#ifdef B2_TRACE
#define B2_TRACE_DECL(name) static __device__ unsigned long long name[32];
#define B2_TR(name, ev) do { unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); name[ev] = t_; } while (0)
#else
#define B2_TRACE_DECL(name)
#define B2_TR(name, ev) do {} while (0)
#endif

// ---- programmatic dependent launch
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---- draft trees of speculative verification (tree format: include/b200spark.h, "Tree-structured verification").
// par = parents[b][0 .. q_len-1]: node t >= 1 hangs below par[t] in [0, t); par[0] is ignored.  A parent outside [0, t) is
// a caller error; it is read as the root, so every walk stays inside the row and ends within t steps.
constexpr int kMaxQLen = 16;  // tokens per sequence of a multi-token step (draft-tree nodes: tree_walk's 16-bit ancestor mask)
__device__ __forceinline__ int tree_parent(const int32_t* par, int t) {
  const int p = par[t];
  return (unsigned)p < (unsigned)t ? p : 0;
}
// anc(t): bit j set for t and each of its ancestors j; depth: the parent steps from t to node 0 (the root).  A chain
// (par[t] = t - 1) gives bits 0..t and depth t.
__device__ __forceinline__ unsigned tree_walk(const int32_t* par, int t, int& depth) {
  unsigned anc = 1u << t;
  depth = 0;
  for (int u = t; u > 0; ++depth) {
    u = tree_parent(par, u);
    anc |= 1u << u;
  }
  return anc;
}

// ---- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)  // no suspend-time hint: ptxas lowers it to NANOSLEEP polling (measured: +2 us per wait)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// for roles with slack (producers): poll with back-off so the spin does not steal issue slots from the math warps
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) __nanosleep(40);
}

// ---- TMA 1D bulk copy global -> shared, completion on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- cp.async 16B (SASS: LDGSTS)
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async16_zfill(void* smem_dst, const void* gmem_src, bool valid) {
  uint32_t n = valid ? 16u : 0u;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(n)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// ---- shared-memory vector load
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}

__device__ __forceinline__ uint2 lds64(uint32_t addr) {
  uint2 v;
  asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
  return v;
}

// ---- streaming global loads (read-once data: bypass L1 allocation)
__device__ __forceinline__ uint4 ldg_stream128(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

// ---- warp-level tensor core MMA m16n8k16, fp32 accumulate (SASS: HMMA)
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_f16_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                              uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// ---- ldmatrix
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

__device__ __forceinline__ uint32_t lop3_and_or(uint32_t a, uint32_t mask, uint32_t orv) {
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(a), "r"(mask), "r"(orv));  // (a & mask) | orv
  return d;
}

__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  __half2 v = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// ---- the 16-bit activation type of a GEMM handle (FT): bf16 (H = false) or fp16 (H = true).  Pointers stay `__nv_bfloat16*`
// (16-bit storage); everything that interprets the bits goes through this trait.  kMagic / kMagicHi: the "exact integer"
// dequantisation constants — a 4-bit code OR-ed into mantissa bits 3..6 of {16.0, 256.0} (bf16: 16 + q, 16 (16 + q)) or of
// {128.0, 2048.0} (fp16, three more mantissa bits: 128 + q, 16 (128 + q)); kBias is the additive constant that comes with it.
template <bool H>
struct Ft;
template <>
struct Ft<false> {
  static constexpr uint32_t kMagic = 0x41804180u, kMagicHi = 0x43804380u;
  static constexpr float kBias = 16.f;
  static __device__ __forceinline__ float lo(uint32_t v) { return __uint_as_float(v << 16); }
  static __device__ __forceinline__ float hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
  static __device__ __forceinline__ uint32_t pack(float a, float b) { return pack_bf16x2(a, b); }
  static __device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16(v); }
  static __device__ __forceinline__ void mma(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    mma_bf16_16816(d, a0, a1, a2, a3, b0, b1);
  }
};
template <>
struct Ft<true> {
  static constexpr uint32_t kMagic = 0x58005800u, kMagicHi = 0x68006800u;
  static constexpr float kBias = 128.f;
  static __device__ __forceinline__ float lo(uint32_t v) { return __half2float(__ushort_as_half((unsigned short)(v & 0xffffu))); }
  static __device__ __forceinline__ float hi(uint32_t v) { return __half2float(__ushort_as_half((unsigned short)(v >> 16))); }
  static __device__ __forceinline__ uint32_t pack(float a, float b) { return pack_f16x2(a, b); }
  static __device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __half2float(__ushort_as_half(__bfloat16_as_ushort(v))); }
  static __device__ __forceinline__ __nv_bfloat16 from_f(float v) { return __ushort_as_bfloat16(__half_as_ushort(__float2half_rn(v))); }
  static __device__ __forceinline__ void mma(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    mma_f16_16816(d, a0, a1, a2, a3, b0, b1);
  }
};

template <int ACT>
__device__ __forceinline__ float apply_act(float x) {
  // csrc/core/kernel/cuda/hie/cuda_activation.hpp (reference formulas, fp32)
  if (ACT == B2_ACT_RELU) return x < 0.f ? 0.f : x;
  if (ACT == B2_ACT_TANH) return tanhf(x);
  if (ACT == B2_ACT_GELU_ERF) return x * 0.5f * (1.0f + erff(x * 0.70710678f));
  if (ACT == B2_ACT_GELU_TANH) return x * 0.5f * (1.0f + tanhf(0.7978845608028654f * (x + 0.044715f * x * x * x)));
  if (ACT == B2_ACT_SILU) return x / (1.0f + __expf(-x));
  if (ACT == B2_ACT_SIGMOID) return 1.0f / (1.0f + __expf(-x));
  return x;
}
__device__ __forceinline__ float apply_act_rt(float x, int act) {
  switch (act) {
    case B2_ACT_RELU: return apply_act<B2_ACT_RELU>(x);
    case B2_ACT_TANH: return apply_act<B2_ACT_TANH>(x);
    case B2_ACT_GELU_ERF: return apply_act<B2_ACT_GELU_ERF>(x);
    case B2_ACT_GELU_TANH: return apply_act<B2_ACT_GELU_TANH>(x);
    case B2_ACT_SILU: return apply_act<B2_ACT_SILU>(x);
    case B2_ACT_SIGMOID: return apply_act<B2_ACT_SIGMOID>(x);
    default: return x;
  }
}

#endif  // __CUDACC__
}  // namespace b2
