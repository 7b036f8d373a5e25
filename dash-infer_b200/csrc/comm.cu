// b200spark — tensor-parallel exchange over NVLink peer memory, sm_90a.
//
// Replaces the reference's AllReduceOp (csrc/core/operator/nccl/allreduce/allreduce_op.cpp:73-115: ncclAllReduce on the
// op's stream preceded by a ctx_->Synchronize() of the whole device) for the decode step's exchanges: [batch, hidden]
// bf16 partial sums after o_proj and down_proj (<= 512 KB), and the per-rank (max, argmax) of the vocab-split lm_head.
//
//   * one process per GPU; every rank owns one EXCHANGE BUFFER in its own HBM, mapped into the peers (CUDA IPC, or any
//     other way the caller obtains peer pointers: b2_comm_connect_pointers takes a plain table);
//   * ONE-SHOT all-reduce: a rank pushes its partial into slot[rank] of every peer's buffer (16-byte stores over NVLink /
//     NVSwitch), raises a per-chunk flag there, waits for the other ranks' flags in ITS OWN memory and sums the nranks
//     slots in rank order in fp32 (deterministic; the residual and the bf16 rounding happen once, after the sum).
//     (nranks-1) x bytes leave every GPU, in one latency hop — the right trade below ~1 MB; NCCL's ring / LL protocols pay
//     2 (nranks-1) hops.
//   * stream-ordered and CUDA-graph replayable: the epoch that flags are compared against lives in device memory and is
//     advanced by the kernel itself; two buffer parities make a slot reusable while a slower peer still reads the other.
//   * no host synchronisation, no NCCL, no staging copy.  The same push/flag/sum sequence is fused into the epilogue of
//     the row-parallel GEMV (wq_gemm.cu, b2_gemm_wq_run_allreduce) so the exchange of one 128-channel tile overlaps the
//     weight streaming of the others.
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

#include "b2_common.cuh"
#include "comm_shared.cuh"

namespace b2 {

// grid = comm chunks (<= kCommMaxChunks); chunk c of every rank covers the same element range
__global__ void __launch_bounds__(256) allreduce_oneshot_kernel(const CommDev cd, __nv_bfloat16* out, const __nv_bfloat16* in,
                                                                const __nv_bfloat16* residual, int64_t count, int64_t per_chunk) {
  pdl_wait();  // `in` is the previous kernel's output; the previous exchange on this stream has fully completed
  pdl_launch_dependents();
  const unsigned epoch = *reinterpret_cast<volatile unsigned*>(cd.epoch);
  const unsigned want = epoch + 1;
  const int par = epoch & 1;
  const int c = blockIdx.x;
  const int64_t e0 = (int64_t)c * per_chunk, e1 = min(count, e0 + per_chunk);
  const int64_t nvec = (e1 - e0 + 7) / 8;  // 16-byte vectors (count is padded to 8 elements by the host)
  // ---- push my partial of this chunk into slot[rank] of every rank (mine included: the sum reads local memory only)
  const uint4* src = reinterpret_cast<const uint4*>(in + e0);
  for (int r = 0; r < cd.nranks; ++r) {
    const int peer = (cd.rank + r) % cd.nranks;  // start with myself, stagger the peers
    uint4* dst = reinterpret_cast<uint4*>(cd.peer[peer] + comm_slot_offset(cd, par, cd.rank)) + e0 / 8;
    for (int64_t i = threadIdx.x; i < nvec; i += blockDim.x) dst[i] = src[i];
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x < cd.nranks) {
    unsigned* f = reinterpret_cast<unsigned*>(cd.peer[threadIdx.x] + comm_flag_offset(cd, par, cd.rank, c));
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(f), "r"(want) : "memory");
  }
  // ---- wait for every rank's chunk c in my memory
  __shared__ int s_ok;
  if (threadIdx.x == 0) s_ok = 1;
  __syncthreads();
  if (threadIdx.x < cd.nranks) {
    const unsigned* f = reinterpret_cast<const unsigned*>(cd.peer[cd.rank] + comm_flag_offset(cd, par, threadIdx.x, c));
    if (!wait_flag(f, want, cd.timeout_ns, cd.error)) s_ok = 0;
  }
  __syncthreads();
  if (s_ok) {
    // ---- sum the slots in rank order (fp32), add the residual, round once
    const uint8_t* base = cd.peer[cd.rank];
    for (int64_t i = threadIdx.x; i < nvec; i += blockDim.x) {
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int r = 0; r < cd.nranks; ++r) {
        const uint4 v = __ldcg(reinterpret_cast<const uint4*>(base + comm_slot_offset(cd, par, r)) + e0 / 8 + i);
        acc[0] += bf16_lo(v.x); acc[1] += bf16_hi(v.x); acc[2] += bf16_lo(v.y); acc[3] += bf16_hi(v.y);
        acc[4] += bf16_lo(v.z); acc[5] += bf16_hi(v.z); acc[6] += bf16_lo(v.w); acc[7] += bf16_hi(v.w);
      }
      if (residual) {
        const uint4 v = *(reinterpret_cast<const uint4*>(residual + e0) + i);
        acc[0] += bf16_lo(v.x); acc[1] += bf16_hi(v.x); acc[2] += bf16_lo(v.y); acc[3] += bf16_hi(v.y);
        acc[4] += bf16_lo(v.z); acc[5] += bf16_hi(v.z); acc[6] += bf16_lo(v.w); acc[7] += bf16_hi(v.w);
      }
      uint4 o;
      o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
      o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
      *(reinterpret_cast<uint4*>(out + e0) + i) = o;
    }
  }
  // ---- the last chunk to finish advances the epoch for the next exchange on this stream
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(cd.done, 1u) == gridDim.x - 1) {
      *cd.done = 0;
      __threadfence();
      *reinterpret_cast<volatile unsigned*>(cd.epoch) = want;
    }
  }
}

// all-gather of a few bytes per rank (the vocab-split lm_head's per-rank (max, argmax) pairs): same push / flag / wait
__global__ void __launch_bounds__(256) allgather_small_kernel(const CommDev cd, uint8_t* out, const uint8_t* in, int bytes) {
  pdl_wait();
  pdl_launch_dependents();
  const unsigned epoch = *reinterpret_cast<volatile unsigned*>(cd.epoch);
  const unsigned want = epoch + 1;
  const int par = epoch & 1;
  for (int r = 0; r < cd.nranks; ++r) {
    uint8_t* dst = cd.peer[r] + comm_slot_offset(cd, par, cd.rank);
    for (int i = threadIdx.x; i < bytes; i += blockDim.x) dst[i] = in[i];
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x < cd.nranks) {
    unsigned* f = reinterpret_cast<unsigned*>(cd.peer[threadIdx.x] + comm_flag_offset(cd, par, cd.rank, 0));
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(f), "r"(want) : "memory");
  }
  __shared__ int s_ok;
  if (threadIdx.x == 0) s_ok = 1;
  __syncthreads();
  if (threadIdx.x < cd.nranks) {
    const unsigned* f = reinterpret_cast<const unsigned*>(cd.peer[cd.rank] + comm_flag_offset(cd, par, threadIdx.x, 0));
    if (!wait_flag(f, want, cd.timeout_ns, cd.error)) s_ok = 0;
  }
  __syncthreads();
  if (s_ok) {
    const uint8_t* base = cd.peer[cd.rank];
    for (int r = 0; r < cd.nranks; ++r)
      for (int i = threadIdx.x; i < bytes; i += blockDim.x)
        out[(size_t)r * bytes + i] = *reinterpret_cast<const volatile uint8_t*>(base + comm_slot_offset(cd, par, r) + i);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    *reinterpret_cast<volatile unsigned*>(cd.epoch) = want;
  }
}

}  // namespace b2

using namespace b2;

struct b2_comm {
  CommDev dev{};
  int rank = 0, nranks = 1;
  size_t max_bytes = 0, buf_bytes = 0;
  void* local = nullptr;          // this rank's exchange buffer (cudaMalloc), first bytes = [epoch, done, error]
  bool own_local = false;
  std::vector<void*> opened;      // peers mapped with cudaIpcOpenMemHandle
};

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

static void layout(b2_comm* c) {
  c->dev.rank = c->rank;
  c->dev.nranks = c->nranks;
  c->dev.max_bytes = c->max_bytes;
  c->dev.slot_bytes = align_up(c->max_bytes, 256);
  c->dev.data_off = 256;                                                     // after the control words
  c->dev.flag_off = c->dev.data_off + 2 * (size_t)c->nranks * c->dev.slot_bytes;
  c->buf_bytes = c->dev.flag_off + 2 * (size_t)c->nranks * kCommMaxChunks * kCommFlagStride;
  const char* t = getenv("B2_COMM_TIMEOUT_MS");
  c->dev.timeout_ns = (unsigned long long)(t ? atoll(t) : 5000) * 1000000ull;
}

extern "C" {

size_t b2_comm_buffer_bytes(int nranks, size_t max_bytes) {
  if (nranks < 1 || nranks > kCommMaxRanks || max_bytes == 0) return 0;
  b2_comm c;
  c.nranks = nranks;
  c.max_bytes = max_bytes;
  layout(&c);
  return c.buf_bytes;
}

int b2_comm_create(b2_comm_t* out, int rank, int nranks, size_t max_bytes) {
  if (!out || nranks < 1 || nranks > kCommMaxRanks || rank < 0 || rank >= nranks || max_bytes == 0) return B2_ERR_PARAM;
  b2_comm* c = new (std::nothrow) b2_comm();
  if (!c) return B2_ERR_RUNTIME;
  c->rank = rank; c->nranks = nranks; c->max_bytes = max_bytes;
  layout(c);
  cudaError_t e = cudaMalloc(&c->local, c->buf_bytes);
  if (e == cudaSuccess) e = cudaMemset(c->local, 0, c->buf_bytes);
  if (e != cudaSuccess) {
    set_last_error("b2_comm_create", e);
    delete c;
    return B2_ERR_CUDA;
  }
  c->own_local = true;
  for (int r = 0; r < kCommMaxRanks; ++r) c->dev.peer[r] = nullptr;
  c->dev.peer[rank] = (uint8_t*)c->local;
  c->dev.epoch = (unsigned*)c->local;
  c->dev.done = (unsigned*)c->local + 1;
  c->dev.error = (int*)c->local + 2;
  *out = c;
  return B2_OK;
}

int b2_comm_export(b2_comm_t c, void* handle_out) {
  if (!c || !handle_out || !c->local) return B2_ERR_PARAM;
  static_assert(sizeof(cudaIpcMemHandle_t) == B2_COMM_HANDLE_BYTES, "handle size");
  cudaIpcMemHandle_t h;
  B2_CUDA_TRY(cudaIpcGetMemHandle(&h, c->local));
  memcpy(handle_out, &h, sizeof(h));
  return B2_OK;
}

int b2_comm_connect(b2_comm_t c, const void* all_handles) {
  if (!c || !all_handles) return B2_ERR_PARAM;
  for (int r = 0; r < c->nranks; ++r) {
    if (r == c->rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, (const char*)all_handles + (size_t)r * B2_COMM_HANDLE_BYTES, sizeof(h));
    void* p = nullptr;
    B2_CUDA_TRY(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    c->opened.push_back(p);
    c->dev.peer[r] = (uint8_t*)p;
  }
  return B2_OK;
}

int b2_comm_connect_pointers(b2_comm_t c, void* const* peer_buffers) {
  if (!c || !peer_buffers) return B2_ERR_PARAM;
  for (int r = 0; r < c->nranks; ++r) {
    if (r == c->rank) continue;
    if (!peer_buffers[r]) return B2_ERR_PARAM;
    c->dev.peer[r] = (uint8_t*)peer_buffers[r];
  }
  return B2_OK;
}

void* b2_comm_local_buffer(b2_comm_t c) { return c ? c->local : nullptr; }

int b2_comm_destroy(b2_comm_t c) {
  if (!c) return B2_OK;
  for (void* p : c->opened) cudaIpcCloseMemHandle(p);
  if (c->own_local && c->local) cudaFree(c->local);
  delete c;
  return B2_OK;
}

int b2_comm_error(b2_comm_t c) {
  if (!c) return B2_ERR_PARAM;
  int e = 0;
  if (cudaMemcpy(&e, c->dev.error, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return B2_ERR_CUDA;
  return e ? B2_ERR_RUNTIME : B2_OK;
}

static int comm_ready(const b2_comm* c) {
  if (!c) return B2_ERR_PARAM;
  for (int r = 0; r < c->nranks; ++r)
    if (!c->dev.peer[r]) return B2_ERR_RUNTIME;  // not connected
  return B2_OK;
}

int b2_allreduce(b2_comm_t c, void* out, const void* in, const void* residual, int64_t count, int ft, void* stream_) {
  if (int st = comm_ready(c)) return st;
  if (!out || !in || count <= 0) return B2_ERR_PARAM;
  if (ft != B2_DT_BF16) return B2_ERR_UNSUPPORTED;
  if ((size_t)count * 2 > c->max_bytes) return B2_ERR_LIMIT;
  if ((count % 8) != 0 || ((uintptr_t)in & 15) || ((uintptr_t)out & 15) || (residual && ((uintptr_t)residual & 15))) return B2_ERR_UNSUPPORTED;
  // chunks of >= 8 KB, at most kCommMaxChunks: the flags are per chunk so a chunk's sum starts as soon as ITS pieces landed
  int64_t chunks = (count * 2 + 8191) / 8192;
  if (chunks > kCommMaxChunks) chunks = kCommMaxChunks;
  int64_t per = (count + chunks - 1) / chunks;
  per = (per + 7) / 8 * 8;
  chunks = (count + per - 1) / per;
  cudaError_t e = launch(allreduce_oneshot_kernel, dim3((unsigned)chunks), dim3(256), 0, (cudaStream_t)stream_, true, c->dev,
                         (__nv_bfloat16*)out, (const __nv_bfloat16*)in, (const __nv_bfloat16*)residual, count, per);
  if (e != cudaSuccess) {
    set_last_error("b2_allreduce launch", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

int b2_allgather(b2_comm_t c, void* out, const void* in, int bytes_per_rank, void* stream_) {
  if (int st = comm_ready(c)) return st;
  if (!out || !in || bytes_per_rank <= 0) return B2_ERR_PARAM;
  if ((size_t)bytes_per_rank > c->max_bytes) return B2_ERR_LIMIT;
  cudaError_t e = launch(allgather_small_kernel, dim3(1), dim3(256), 0, (cudaStream_t)stream_, true, c->dev, (uint8_t*)out,
                         (const uint8_t*)in, bytes_per_rank);
  if (e != cudaSuccess) {
    set_last_error("b2_allgather launch", e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

// the device view of a communicator, for kernels in other translation units (wq_gemm.cu's fused epilogue)
const void* b2_comm_device_view(b2_comm_t c) { return c ? &c->dev : nullptr; }

}  // extern "C"
