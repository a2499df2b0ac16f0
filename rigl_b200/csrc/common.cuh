// Shared helpers for the rigl_b200 C-ABI library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>

#include "../../include/rigl_b200.h"

namespace rigl {

// SM count of an H100 SXM: sizes grids before (or without) a device query.  Grid-size heuristics only; the
// persistent tensor-core kernels size their grids from the device's own count.
constexpr int kNumSmsHint = 132;

void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;

inline int cuda_fail(cudaError_t e, const char* what) {
  set_error("%s: %s", what, cudaGetErrorString(e));
  return RIGL_ERR_CUDA;
}

#define RIGL_CUDA(...)                                                \
  do {                                                                \
    cudaError_t _e = (__VA_ARGS__);                                   \
    if (_e != cudaSuccess) return ::rigl::cuda_fail(_e, #__VA_ARGS__); \
  } while (0)

#define RIGL_LAUNCH_CHECK(name)                                 \
  do {                                                          \
    ::rigl::g_launches.fetch_add(1, std::memory_order_relaxed); \
    cudaError_t _e = cudaGetLastError();                        \
    if (_e != cudaSuccess) return ::rigl::cuda_fail(_e, name);  \
  } while (0)

#define RIGL_REQUIRE(cond, ...)          \
  do {                                   \
    if (!(cond)) {                       \
      ::rigl::set_error(__VA_ARGS__);    \
      return RIGL_ERR_INVALID_ARG;       \
    }                                    \
  } while (0)

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Order-preserving map float32 -> uint32 (larger float <=> larger key);
// -0.0 is canonicalised to +0.0 so that it ties with +0.0 like a float compare.
__device__ __forceinline__ uint32_t ord_key(float s) {
  s = __fadd_rn(s, 0.0f);
  uint32_t u = __float_as_uint(s);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

}  // namespace rigl
