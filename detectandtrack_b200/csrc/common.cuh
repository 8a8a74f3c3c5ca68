// Shared helpers for the DetectAndTrack C-ABI library (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace dt {

// Last error text, one per host thread (dt_last_error()).
char* last_error_buf();
void set_error(const char* fmt, ...);

#define DT_CHECK_ARG(cond, ...)                         \
  do {                                                  \
    if (!(cond)) {                                      \
      ::dt::set_error(__VA_ARGS__);                     \
      return 1;                                         \
    }                                                   \
  } while (0)

#define DT_CHECK_CUDA(expr)                                                    \
  do {                                                                         \
    cudaError_t _e = (expr);                                                   \
    if (_e != cudaSuccess) {                                                   \
      ::dt::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),  \
                      __FILE__, __LINE__);                                     \
      return 2;                                                                \
    }                                                                          \
  } while (0)

#define DT_CHECK_LAUNCH() DT_CHECK_CUDA(cudaGetLastError())

// cudaFuncAttributeMaxDynamicSharedMemorySize is a PER-DEVICE attribute: remember, per launch site and device, the
// largest size already granted (a process may use the library on several GPUs and from several threads).
struct DynSmemGrant {
  int granted[64];                     // bytes set so far on device i (0 = never); races only repeat the call
};
template <typename K>
static inline cudaError_t grant_dyn_smem(K kernel, int bytes, DynSmemGrant* g) {
  int dev = -1;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev >= 0 && dev < 64 && __atomic_load_n(&g->granted[dev], __ATOMIC_ACQUIRE) >= bytes) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess && dev >= 0 && dev < 64) __atomic_store_n(&g->granted[dev], bytes, __ATOMIC_RELEASE);
  return e;
}

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// SM count of the current device (grid sizing of persistent / split-K launches); 132 on an H100 SXM
static inline int num_sms() {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms < 1)
    return 132;
  return sms;
}
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

}  // namespace dt
