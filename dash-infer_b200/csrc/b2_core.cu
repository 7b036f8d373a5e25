// b200spark — library plumbing: status strings, last-error text, device queries, PDL switch.
#include <cstdio>
#include <cstring>

#include "b2_common.cuh"

namespace b2 {

static thread_local char g_last_error[512] = {0};
static thread_local int g_pdl = 1;

void set_last_error(const char* what, cudaError_t e) {
  snprintf(g_last_error, sizeof(g_last_error), "%s: %s", what, cudaGetErrorString(e));
}

int launch_failed(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error(what, e);
    return B2_ERR_CUDA;
  }
  return B2_OK;
}

bool pdl_enabled() { return g_pdl != 0; }

int sm_count() {
  static thread_local int cached_dev = -1, cached = 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev != cached_dev) {
    cudaDeviceGetAttribute(&cached, cudaDevAttrMultiProcessorCount, dev);
    cached_dev = dev;
  }
  return cached > 0 ? cached : 132;
}

int max_smem_optin() {
  int dev = 0, v = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  return v;
}

}  // namespace b2

extern "C" {

const char* b2_status_string(int s) {
  switch (s) {
    case B2_OK: return "B2_OK";
    case B2_ERR_CUDA: return "B2_ERR_CUDA";
    case B2_ERR_RUNTIME: return "B2_ERR_RUNTIME";
    case B2_ERR_PARAM: return "B2_ERR_PARAM";
    case B2_ERR_LIMIT: return "B2_ERR_LIMIT";
    case B2_ERR_INTERNAL: return "B2_ERR_INTERNAL";
    case B2_ERR_UNSUPPORTED: return "B2_ERR_UNSUPPORTED";
    default: return "B2_ERR_UNKNOWN";
  }
}

const char* b2_last_error(void) { return b2::g_last_error; }

const char* b2_version(void) { return "b200spark 0.1 sm_90a"; }

void b2_set_pdl(int enabled) { b2::g_pdl = enabled ? 1 : 0; }

}  // extern "C"
