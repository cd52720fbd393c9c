// Shared host/device helpers for libpulse_b200.so (sm_90a, H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "pulse_b200.h"

namespace pulse {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define PULSE_REQUIRE(cond, ...)                 \
  do {                                           \
    if (!(cond)) {                               \
      ::pulse::set_error(__VA_ARGS__);           \
      return PULSE_ERR_ARG;                      \
    }                                            \
  } while (0)

#define PULSE_CUDA_OK(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      ::pulse::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return PULSE_ERR_CUDA;                                                             \
    }                                                                                    \
  } while (0)

#define PULSE_LAUNCH_OK(name)                                                            \
  do {                                                                                   \
    cudaError_t _e = cudaGetLastError();                                                 \
    if (_e != cudaSuccess) {                                                             \
      ::pulse::set_error("launch of %s failed: %s", name, cudaGetErrorString(_e));       \
      return PULSE_ERR_CUDA;                                                             \
    }                                                                                    \
    ::pulse::count_launch();                                                             \
  } while (0)

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

constexpr int kWarp = 32;
// SM count of the H100 SXM: sizes the grid caps of the grid-stride element-wise / reduction kernels (the persistent GEMM
// queries the device instead).
constexpr int kNumSMs = 132;
constexpr unsigned kFull = 0xffffffffu;

}  // namespace pulse

struct pulse_motionlib {
  pulse_motionlib_desc_t d;
};
