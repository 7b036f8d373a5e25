// oracle/_ref shim — TEST INFRASTRUCTURE ONLY (never linked into the product libraries).
//
// A plain-C door into the UNMODIFIED reference GPU code that oracle/build_ref.py compiles from where it lies under
// /root/reference (span-attention/src + csrc/core/kernel/cuda/cache): the span-attention library
// (span::CreateHandle / Run, span-attention/include/spanattn/span_attn.h:108-175) and the cache writers
// (DecoderCacheAppendLauncher, ContextSpanCopyLauncher, csrc/core/kernel/cuda/cuda_kernel_span_cache.h:11-27).
// tests/golden/make_ref_pin.py uses it on a GPU to pin oracle/kvcache_ref.py and the b200spark kernels against what the reference
// itself computes (append bytes, quant params, attention output).
#include <cuda_runtime.h>
#include <span_attn.h>
#include <stdint.h>

#include <exception>
#include <vector>

#include "cuda/cuda_kernel_span_cache.h"
#ifdef ENABLE_BF16
#include "hie_bfloat16.hpp"
#endif
#ifdef ENABLE_FP16
#include <cuda_fp16.h>
#endif

extern "C" {

// dtype: span::DataType (0 fp32, 1 fp16, 2 bf16); qmode: span::QuantMode (0 none, 1 i8, 2 u4).  Returns SaStatus or -1 (CUDA).
int ref_span_attn(void* out, const void* q, const void* const* k_spans, const void* const* v_spans, const int* host_lens,
                  int batch, int n_heads, int n_groups, int head_size, int span_len, int n_spans, int qmode, int dtype,
                  float qk_scale, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  cudaDeviceProp prop;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return -1;
  span::SpanAttnHandle_t h = nullptr;
  span::SaStatus st = span::CreateHandle(&h, (span::DataType)dtype, (span::QuantMode)qmode, batch, n_heads, n_groups, head_size,
                                         span_len, n_spans, host_lens, prop);
  if (st != span::SaStatus::SUCCESS) return (int)st;
  size_t dws = 0, hws = 0;
  span::GetDeviceWorkspaceSize(&dws, h);
  span::GetHostWorkspaceSize(&hws, h);
  void *dbuf = nullptr, *hbuf = nullptr;
  int rc = 0;
  if (cudaMalloc(&dbuf, dws ? dws : 16) != cudaSuccess || cudaMallocHost(&hbuf, hws ? hws : 16) != cudaSuccess) rc = -1;
  if (rc == 0) {
    st = span::Run(out, q, k_spans, v_spans, dbuf, dws, hbuf, hws, qk_scale, h, stream);
    rc = (int)st;
    if (cudaStreamSynchronize(stream) != cudaSuccess) rc = -1;
  }
  if (dbuf) cudaFree(dbuf);
  if (hbuf) cudaFreeHost(hbuf);
  span::DestroyHandle(h);
  return rc;
}

int ref_cache_append(void* const* k_spans, void* const* v_spans, void* q_out, const void* src, const uint32_t* old_lens,
                     int batch, int n_heads, int n_groups, int head_size, int span_len, int n_spans, int qmode, int dtype,
                     void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  try {
#ifdef ENABLE_BF16
    if (dtype == 2) {
      allspark::cuda::DecoderCacheAppendLauncher(k_spans, v_spans, (hie::bfloat16*)q_out, (const hie::bfloat16*)src, old_lens,
                                                 batch, n_heads, n_groups, head_size, span_len, n_spans,
                                                 (span::QuantMode)qmode, stream);
      return 0;
    }
#endif
#ifdef ENABLE_FP16
    if (dtype == 1) {
      allspark::cuda::DecoderCacheAppendLauncher(k_spans, v_spans, (half*)q_out, (const half*)src, old_lens, batch, n_heads,
                                                 n_groups, head_size, span_len, n_spans, (span::QuantMode)qmode, stream);
      return 0;
    }
#endif
  } catch (const std::exception&) {
    return -2;
  }
  return 3;
}

// src: [seq_len, n_groups, head] contiguous; spans: device array of span pointers for ONE sequence (K or V)
int ref_context_span_copy(void* const* spans, const void* src, int n_groups, int head_size, int span_len, int seq_len,
                          int qmode, int dtype, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  try {
#ifdef ENABLE_BF16
    if (dtype == 2) {
      allspark::cuda::ContextSpanCopyLauncher(spans, (const hie::bfloat16*)src, n_groups, head_size, span_len, seq_len,
                                              (span::QuantMode)qmode, stream);
      return 0;
    }
#endif
#ifdef ENABLE_FP16
    if (dtype == 1) {
      allspark::cuda::ContextSpanCopyLauncher(spans, (const half*)src, n_groups, head_size, span_len, seq_len,
                                              (span::QuantMode)qmode, stream);
      return 0;
    }
#endif
  } catch (const std::exception&) {
    return -2;
  }
  return 3;
}

const char* ref_version(void) { return "dash-infer f3cca8e span-attention + cache kernels, built for sm_90 by oracle/build_ref.py"; }
}
