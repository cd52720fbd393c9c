// Gradient averaging + norm clip + Adam in ONE kernel over NVLink peer memory (SURVEY 8e: the path's only exchange step).
//
// Replaces, on G GPUs of one NVSwitch domain, the sequence  ncclAllReduce(AVG, flat gradients)  ->  sum_squares  ->  adam_kernel
// (Horovod's DistributedOptimizer + clip_grad_norm_ + torch.optim.Adam in the reference, amp_agent.py:725-750):
//
//   phase 0  every rank announces "my gradients are final" to its peers (a flag store into their signal blocks).
//   phase 1  rank r PULLS slice r of every rank's gradient buffer through the peer mappings (or lets the switch add them:
//            multimem.ld_reduce on the multicast alias), averages in rank order, keeps the averaged slice in its own buffer and its
//            sum of squares -- a reduce-scatter whose output never exists as a full tensor.  The G slice norms are exchanged as
//            8-byte stores; every rank adds them in rank order, so all ranks clip with the bit-identical global norm.
//   phase 2  rank r runs Adam on slice r only (moments are sharded: 1/G of the optimizer traffic per GPU) and PUSHES the new fp32
//            masters and the bf16 GEMM operands of its slice into every rank's buffers (peer stores, or one multimem.st the switch
//            replicates); it also clears its whole gradient buffer -- every peer has finished reading it by then.
//   phase 3  a last flag round: a rank's kernel ends only when all slices of ITS operand copy have landed.
//
// Each byte crosses NVLink once per direction; nothing is staged, no second kernel reads the reduced gradients back.  All waits are
// bounded (timeout_ms, default 30 min: a lost peer surfaces as a launch failure, never as a GPU hung for good).  Flags are monotonic epoch numbers kept on the device, so
// the launch is CUDA-graph replayable.
#include <cuda_bf16.h>

#include "pulse_common.cuh"

namespace pulse {
namespace {

constexpr int kPeerThreads = 512;
// Default bound of a wait on a peer.  Ranks legitimately drift far apart in a training run -- rl_games checkpoints, logs and runs the
// minutes-long evaluation pass on rank 0 only while the other ranks already sit in their next optimizer step -- so the default is the
// order of a collective-library watchdog, not of a kernel; tests and probes pass seconds.
constexpr unsigned kDefaultTimeoutMs = 30u * 60u * 1000u;

__device__ __forceinline__ unsigned long long now_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;\n" : "=l"(t));
  return t;
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;\n" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_gpu64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];\n" : "=l"(v) : "l"(p) : "memory");
  return v;
}
// gradients another GPU wrote: never served from this SM's L1
__device__ __forceinline__ float4 ld_peer_f4(const float* p) {
  float4 v;
  asm volatile("ld.volatile.global.v4.f32 {%0, %1, %2, %3}, [%4];\n" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float4 mc_ld_reduce_f4(const float* p) {   // the switch adds the G replicas
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];\n"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void mc_st_f4(float* p, float4 v) {        // the switch replicates the store into every rank's buffer
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void mc_st_u2(void* p, uint2 v) {
  asm volatile("multimem.st.relaxed.sys.global.v2.bf16x2 [%0], {%1, %2};\n" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}

// Wait until the epoch flags of all ranks in row `phase` of the LOCAL signal block have reached `target` (threads 0..world-1 poll one
// flag each), then the whole CTA proceeds.
__device__ __forceinline__ void wait_flags(const unsigned* my_signals, int phase, int world, unsigned target, unsigned long long kSpinNs) {
  if (threadIdx.x < static_cast<unsigned>(world)) {
    const unsigned* f = my_signals + phase * PULSE_PEER_MAX + threadIdx.x;
    const unsigned long long t0 = now_ns();
    while (static_cast<int>(ld_acquire_sys(f) - target) < 0) {
      if (now_ns() - t0 > kSpinNs) __trap();
      __nanosleep(64);
    }
  }
  __syncthreads();
}

// All CTAs of this launch (co-resident: grid <= SM count, nothing this kernel waits on can be queued behind it).
__device__ __forceinline__ void grid_sync(unsigned long long* counter, unsigned long long target, unsigned long long kSpinNs) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1ull);
    const unsigned long long t0 = now_ns();
    while (ld_acquire_gpu64(counter) < target) {
      if (now_ns() - t0 > kSpinNs) __trap();
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kPeerThreads, 1) peer_reduce_adam_kernel(const pulse_peer_adam_args_t a) {
  const int me = a.rank, W = a.world;
  const unsigned epoch = *a.epoch;              // calls completed so far; this call's flags carry epoch + 1
  const unsigned tag = epoch + 1u;
  const unsigned G = gridDim.x;
  const unsigned long long spin_ns = static_cast<unsigned long long>(a.timeout_ms ? a.timeout_ms : kDefaultTimeoutMs) * 1000000ull;
  const unsigned long long bar_base = static_cast<unsigned long long>(epoch) * 2ull * G;
  unsigned* my_sig = a.signals[me];
  double* my_norms = reinterpret_cast<double*>(my_sig + 3 * PULSE_PEER_MAX);
  const long long n4 = a.count / 4;
  const long long per = (n4 + W - 1) / W;
  const long long s0 = per * me < n4 ? per * me : n4, s1 = (s0 + per) < n4 ? (s0 + per) : n4;
  const long long T = static_cast<long long>(G) * blockDim.x, t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  float* g_loc = a.grads[me];

  // ---- phase 0: "my gradients are final" ----------------------------------------------------------------------------------------
  if (blockIdx.x == 0 && threadIdx.x < static_cast<unsigned>(W)) st_release_sys(a.signals[threadIdx.x] + 0 * PULSE_PEER_MAX + me, tag);
  wait_flags(my_sig, 0, W, tag, spin_ns);

  // ---- phase 1: reduce-scatter by pulling, slice norm -------------------------------------------------------------------------------
  const float inv_w = 1.0f / static_cast<float>(W);
  double sq = 0.0;
  for (long long i = s0 + t; i < s1; i += T) {
    float4 acc;
    if (a.mc_grads != nullptr) {
      acc = mc_ld_reduce_f4(a.mc_grads + 4 * i);
    } else {
      float4 v[PULSE_PEER_MAX];
#pragma unroll
      for (int p = 0; p < PULSE_PEER_MAX; ++p)
        if (p < W) v[p] = ld_peer_f4(a.grads[p] + 4 * i);     // all loads in flight before the first add
      acc = v[0];
#pragma unroll
      for (int p = 1; p < PULSE_PEER_MAX; ++p)
        if (p < W) { acc.x += v[p].x; acc.y += v[p].y; acc.z += v[p].z; acc.w += v[p].w; }   // rank order: every run adds alike
    }
    acc.x *= inv_w; acc.y *= inv_w; acc.z *= inv_w; acc.w *= inv_w;
    reinterpret_cast<float4*>(g_loc)[i] = acc;               // slice `me` of MY buffer is read by no peer
    sq += static_cast<double>(fmaf(acc.x, acc.x, fmaf(acc.y, acc.y, fmaf(acc.z, acc.z, acc.w * acc.w))));
  }
  __shared__ double red[kPeerThreads / 32];
  sq = warp_sum(sq);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sq;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int k = 0; k < kPeerThreads / 32; ++k) s += red[k];
    a.cta_partials[blockIdx.x] = s;
  }
  grid_sync(a.grid_bar, bar_base + G, spin_ns);
  if (blockIdx.x == 0) {
    __shared__ double slice_norm;
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (unsigned k = 0; k < G; ++k) s += __ldcg(a.cta_partials + k);
      slice_norm = s;
    }
    __syncthreads();
    if (threadIdx.x < static_cast<unsigned>(W)) {   // thread p: norm, then flag, to peer p -- "slice norm ready, and I am done reading your gradients"
      double* dst = reinterpret_cast<double*>(a.signals[threadIdx.x] + 3 * PULSE_PEER_MAX) + me;
      *reinterpret_cast<volatile double*>(dst) = slice_norm;
      __threadfence_system();
      st_release_sys(a.signals[threadIdx.x] + 1 * PULSE_PEER_MAX + me, tag);
    }
  }
  wait_flags(my_sig, 1, W, tag, spin_ns);
  double total = 0.0;
  for (int p = 0; p < W; ++p) total += *reinterpret_cast<volatile double*>(my_norms + p);   // rank order: identical on every rank

  // ---- phase 2: Adam on my slice, push the new parameters everywhere, clear my gradient buffer ---------------------------------
  const float step = static_cast<float>(*a.step + 1);
  const float bc1 = 1.0f - powf(a.beta1, step), bc2 = 1.0f - powf(a.beta2, step);
  float scale = 1.0f;
  if (a.max_norm > 0.0f) scale = fminf(1.0f, a.max_norm / (static_cast<float>(sqrt(total)) + 1e-6f));   // torch.nn.utils.clip_grad_norm_
  const float lr1 = a.lr / bc1, rs2 = sqrtf(bc2), b1 = a.beta1, b2 = a.beta2, eps = a.eps;
  auto upd = [&](float gi, float& mi, float& vi, float& pi) {   // same expressions as adam_kernel (mlp_ops.cu)
    gi *= scale;
    mi = b1 * mi + (1.0f - b1) * gi;
    vi = b2 * vi + (1.0f - b2) * gi * gi;
    pi = pi - lr1 * mi / (sqrtf(vi) / rs2 + eps);
  };
  float* p_loc = a.params[me];
  const float4 zero4 = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  for (long long i = s0 + t; i < s1; i += T) {
    const float4 g4 = __ldcg(reinterpret_cast<const float4*>(g_loc) + i);
    reinterpret_cast<float4*>(g_loc)[i] = zero4;             // consumed (by the thread that read it)
    float4 m4 = reinterpret_cast<float4*>(a.exp_avg)[i], v4 = reinterpret_cast<float4*>(a.exp_avg_sq)[i];
    float4 p4 = reinterpret_cast<const float4*>(p_loc)[i];
    upd(g4.x, m4.x, v4.x, p4.x);
    upd(g4.y, m4.y, v4.y, p4.y);
    upd(g4.z, m4.z, v4.z, p4.z);
    upd(g4.w, m4.w, v4.w, p4.w);
    reinterpret_cast<float4*>(a.exp_avg)[i] = m4;
    reinterpret_cast<float4*>(a.exp_avg_sq)[i] = v4;
    __nv_bfloat162 lo = __floats2bfloat162_rn(p4.x, p4.y), hi = __floats2bfloat162_rn(p4.z, p4.w);
    uint2 u;
    u.x = *reinterpret_cast<unsigned*>(&lo);
    u.y = *reinterpret_cast<unsigned*>(&hi);
    if (a.mc_params != nullptr) {
      mc_st_f4(a.mc_params + 4 * i, p4);
      mc_st_u2(reinterpret_cast<uint2*>(a.mc_params_bf16) + i, u);
    } else {
#pragma unroll
      for (int p = 0; p < PULSE_PEER_MAX; ++p)
        if (p < W) {
          reinterpret_cast<float4*>(a.params[p])[i] = p4;
          reinterpret_cast<uint2*>(a.params_bf16[p])[i] = u;
        }
    }
  }
  // the other slices: every peer finished reading them before it raised its phase-1 flag -- the next minibatch accumulates from zero
  for (long long i = t; i < n4; i += T)
    if (i < s0 || i >= s1) reinterpret_cast<float4*>(g_loc)[i] = zero4;
  for (long long i = n4 * 4 + t; i < a.count; i += T) g_loc[i] = 0.0f;
  __threadfence_system();                         // my pushes are performed at system scope before the barrier publishes them
  grid_sync(a.grid_bar, bar_base + 2ull * G, spin_ns);

  // ---- phase 3: "my slice has landed in your buffers" -------------------------------------------------------------------------------
  if (blockIdx.x == 0) {
    if (threadIdx.x < static_cast<unsigned>(W)) {
      __threadfence_system();
      st_release_sys(a.signals[threadIdx.x] + 2 * PULSE_PEER_MAX + me, tag);
    }
    wait_flags(my_sig, 2, W, tag, spin_ns);
    if (threadIdx.x == 0) {
      *a.step = static_cast<int>(step);
      *a.epoch = tag;
      __threadfence();
    }
  }
}

}  // namespace
}  // namespace pulse

extern "C" int pulse_peer_reduce_adam(const pulse_peer_adam_args_t* args, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_peer_reduce_adam: null args");
  const pulse_peer_adam_args_t& a = *args;
  PULSE_REQUIRE(a.world >= 1 && a.world <= PULSE_PEER_MAX && a.rank >= 0 && a.rank < a.world, "pulse_peer_reduce_adam: rank %d / world %d (max %d)",
                a.rank, a.world, PULSE_PEER_MAX);
  PULSE_REQUIRE(a.count > 0 && a.count % 4 == 0, "pulse_peer_reduce_adam: count %lld must be a positive multiple of 4", (long long)a.count);
  for (int p = 0; p < a.world; ++p) {
    PULSE_REQUIRE(a.grads[p] && a.params[p] && a.params_bf16[p] && a.signals[p], "pulse_peer_reduce_adam: null peer buffer of rank %d", p);
    PULSE_REQUIRE(aligned16(a.grads[p]) && aligned16(a.params[p]) && (reinterpret_cast<uintptr_t>(a.params_bf16[p]) & 7u) == 0 &&
                      aligned16(a.signals[p]), "pulse_peer_reduce_adam: misaligned peer buffer of rank %d", p);
  }
  PULSE_REQUIRE(a.exp_avg && a.exp_avg_sq && aligned16(a.exp_avg) && aligned16(a.exp_avg_sq), "pulse_peer_reduce_adam: null / misaligned moments");
  PULSE_REQUIRE(a.step && a.epoch && a.cta_partials && a.grid_bar, "pulse_peer_reduce_adam: null counter / scratch");
  PULSE_REQUIRE((a.mc_params == nullptr) == (a.mc_params_bf16 == nullptr), "pulse_peer_reduce_adam: mc_params and mc_params_bf16 go together");
  PULSE_REQUIRE((a.mc_grads == nullptr || aligned16(a.mc_grads)) && (a.mc_params == nullptr || aligned16(a.mc_params)),
                "pulse_peer_reduce_adam: misaligned multicast alias");
  int dev = 0, sms = 0;
  PULSE_CUDA_OK(cudaGetDevice(&dev));
  PULSE_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  int grid = a.grid > 0 ? a.grid : sms;
  if (grid > sms) grid = sms;               // co-residency of the software grid barrier
  if (grid > PULSE_PEER_MAX_GRID) grid = PULSE_PEER_MAX_GRID;
  peer_reduce_adam_kernel<<<grid, kPeerThreads, 0, static_cast<cudaStream_t>(stream)>>>(a);
  PULSE_LAUNCH_OK("peer_reduce_adam_kernel");
  return PULSE_OK;
}
