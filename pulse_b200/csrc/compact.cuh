// The ordered block-wide compaction shared by the reset entry points (reset.cu, getup_reset.cu, ztask_reset.cu): a reset mask or an
// id list becomes an ascending env list with a device-side count, by ballot and prefix scan, without atomics, so the order is
// deterministic.
#pragma once
#include "pulse_common.cuh"

namespace pulse {
namespace {

constexpr int kCompactThreads = 1024;

// One round of an ordered compaction over a CTA of kCompactThreads threads, called by all of them together: a thread with `take`
// gets slot *base + (takers before it in thread order), -1 otherwise; *base (shared) then advances by the round's takers.
__device__ __forceinline__ int compact_slot(bool take, int* warp_cnt, int* base) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const unsigned m = __ballot_sync(kFull, take);
  if (lane == 0) warp_cnt[wid] = __popc(m);
  __syncthreads();
  int before = 0, total = 0;
#pragma unroll 1
  for (int w = 0; w < kCompactThreads / 32; ++w) {
    const int c = warp_cnt[w];
    if (w < wid) before += c;
    total += c;
  }
  const int pos = take ? *base + before + __popc(m & ((1u << lane) - 1u)) : -1;
  __syncthreads();
  if (tid == 0) *base += total;
  __syncthreads();
  return pos;
}

}  // namespace
}  // namespace pulse
