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

// Blocks for `items` work items at `per_block` per block, capped at `waves` blocks per SM: the kernels grid-stride over the rest.
inline unsigned grid_for(long long items, int per_block, int waves = 8) {
  long long b = (items + per_block - 1) / per_block;
  const long long cap = static_cast<long long>(kNumSMs) * waves;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return static_cast<unsigned>(b);
}

// Sum over the 32 lanes of a full warp (float or double), the result in every lane.
template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

}  // namespace pulse

struct pulse_motionlib {
  pulse_motionlib_desc_t d;
};

struct pulse_smplx_motionlib {
  pulse_smplx_motionlib_desc_t d;
};
