// The AMP demo and replay rings (learning/replay_buffer.py ReplayBuffer, AMPAgent._update_amp_demos / _store_replay_amp_obs and the
// buffer samples of train_epoch, phc/learning/amp_agent.py:476-484, :988-1057) on device-side counters:
//   demo_fetch_kernel    one warp per (row, history step): clip and t0 draws, the motion at t0 - k dt, the AMP row straight into the ring
//                        (SMPL, and SMPL-X through pulse_smplx_amp_demo_fetch);
//   keep_compact_kernel  one CTA: the Bernoulli keep mask (once total_count > capacity) and the ordered compaction of the kept rows;
//   ring_store_kernel    one warp per stored row: the kept row (or the subset's pick of it) into the ring at head, with wrap;
//   ring_sample_kernel   one warp per gathered row: the permuted ring position (or the fallback row);
//   ring_*_done_kernel   one thread: the counter updates, after the kernels that read the old values.
// The counters, Philox planes and the Feistel permutation are documented in include/pulse_b200.h.
#include "compact.cuh"
#include "motion_amp.cuh"
#include "philox.cuh"

namespace pulse {
namespace {

constexpr int kRingWarps = 8;
constexpr unsigned long long kPlane = 1ull << 32;

__device__ __forceinline__ unsigned fmix32(unsigned h) {
  h ^= h >> 16;
  h *= 0x85EBCA6Bu;
  h ^= h >> 13;
  h *= 0xC2B2AE35u;
  h ^= h >> 16;
  return h;
}

// The keyed bijection of [0, m): a four-round balanced Feistel network on 2h bits, cycle-walked back into the domain.
struct Feistel {
  unsigned k[4];
  int half;
  unsigned mask;
  long long m;
  __device__ Feistel(unsigned long long seed, unsigned long long plane, unsigned long long counter, long long domain) : m(domain) {
    const Philox4 r = philox4x32_10(seed, plane * kPlane, counter);
    k[0] = r.x; k[1] = r.y; k[2] = r.z; k[3] = r.w;
    int bits = 2;
    while (bits < 62 && (1ll << bits) < domain) ++bits;
    bits += bits & 1;
    half = bits >> 1;
    mask = (1u << half) - 1u;
  }
  __device__ long long operator()(long long x) const {
    if (m <= 1) return 0;
    do {
      unsigned l = static_cast<unsigned>(x >> half), r = static_cast<unsigned>(x) & mask;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const unsigned t = l ^ (fmix32(r * 0x9E3779B1u ^ k[i]) & mask);
        l = r;
        r = t;
      }
      x = (static_cast<long long>(l) << half) | r;
    } while (x >= m);
    return x;
  }
};

__device__ __forceinline__ void copy_row(float* __restrict__ dst, const float* __restrict__ src, int n, int lane) {
  for (int c = lane; c < n; c += 32) __stcs(dst + c, __ldcs(src + c));
}

// ---- demo fetch -------------------------------------------------------------------------------------------------------------------
template <class L, class Desc>
__global__ void __launch_bounds__(kRingWarps * 32) demo_fetch_kernel(const Desc lib, const pulse_amp_demo_args_t a) {
  __shared__ float stage_all[kRingWarps][L::kAmpObs];
  float* stage = stage_all[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  const long long items = a.num_samples * a.num_steps;
  const long long warp0 = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const long long* ctr = reinterpret_cast<const long long*>(a.ring.ctr);
  const unsigned long long off = static_cast<unsigned long long>(ctr[PULSE_RING_DRAWS]);
  const long long head = ctr[PULSE_RING_HEAD];
  for (long long it = warp0; it < items; it += nwarps) {
    const long long i = it / a.num_steps;
    const int k = static_cast<int>(it - i * a.num_steps);
    const Philox4 rc = philox4x32_10(a.ring.seed, PULSE_PLANE_DEMO_CLIP * kPlane + static_cast<unsigned long long>(i), off);
    const Philox4 rt = philox4x32_10(a.ring.seed, PULSE_PLANE_DEMO_TIME * kPlane + static_cast<unsigned long long>(i), off);
    const long long mid = pick_motion(a.sampling_cdf, lib.num_motions, u01(rc.x));
    const float mlen = lib.lengths[mid];
    const float t0 = sample_time_interval(u01(rt.x), mlen);
    if (k == 0 && lane == 0) {
      if (a.motion_ids_out != nullptr) a.motion_ids_out[i] = mid;
      if (a.times_out != nullptr) a.times_out[i] = t0;
    }
    const float t = __fadd_rn(t0, __fmul_rn(-a.dt, static_cast<float>(k)));   // motion_times0 + (-dt * arange(num_steps))
    long long i0, i1;
    float b;
    frame_blend_rn(t, mlen, lib.num_frames[mid], lib.dt[mid], i0, i1, b);
    const long long f0 = i0 + lib.length_starts[mid], f1 = i1 + lib.length_starts[mid];
    const long long slot = (head + i) % a.ring.capacity;
    store_motion_amp_row<L>(b, lib.frame_rec + f0 * L::kFrameRec, lib.frame_rec + f1 * L::kFrameRec, lib.aux_rec + f0 * L::kAuxRec,
                            lib.aux_rec + f1 * L::kAuxRec, a.ring.rows + slot * a.ring.row_floats + k * a.amp_width, a.amp_width, stage, lane,
                            a.upright != 0);
  }
}

// store(): head = (head + n) % capacity, total_count += n; and the draw counter moves on.
__global__ void ring_store_done_kernel(long long* ctr, long long capacity, long long n_fixed) {
  long long n = n_fixed >= 0 ? n_fixed : ctr[PULSE_RING_LAST_COUNT];
  if (n > capacity) n = capacity;   // a replay store keeps at most capacity rows (the subset)
  ctr[PULSE_RING_HEAD] = (ctr[PULSE_RING_HEAD] + n) % capacity;
  ctr[PULSE_RING_TOTAL] += n;
  ctr[PULSE_RING_DRAWS] += 1;
}

// ---- replay store -----------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kCompactThreads) keep_compact_kernel(const pulse_amp_store_args_t a) {
  __shared__ int warp_cnt[kCompactThreads / 32];
  __shared__ int base;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  long long* ctr = reinterpret_cast<long long*>(a.ring.ctr);
  const bool masked = ctr[PULSE_RING_TOTAL] > a.ring.capacity;   // _store_replay_amp_obs: buf_total_count > buf_size
  const unsigned long long off = static_cast<unsigned long long>(ctr[PULSE_RING_DRAWS]);
  for (long long c0 = 0; c0 < a.num_rows; c0 += kCompactThreads) {
    const long long r = c0 + threadIdx.x;
    bool keep = r < a.num_rows;
    if (keep && masked)
      keep = u01(philox4x32_10(a.ring.seed, PULSE_PLANE_REPLAY_KEEP * kPlane + static_cast<unsigned long long>(r), off).x) < a.keep_prob;
    const int pos = compact_slot(keep, warp_cnt, &base);
    if (pos >= 0) a.kept[pos] = static_cast<int>(r);
  }
  if (threadIdx.x == 0) ctr[PULSE_RING_LAST_COUNT] = base;
}

__global__ void __launch_bounds__(kRingWarps * 32) ring_store_kernel(const pulse_amp_store_args_t a, long long upper) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const long long* ctr = reinterpret_cast<const long long*>(a.ring.ctr);
  const long long m = ctr[PULSE_RING_LAST_COUNT], cap = a.ring.capacity, head = ctr[PULSE_RING_HEAD];
  const long long stored = m < cap ? m : cap;
  const Feistel subset(a.ring.seed, PULSE_PLANE_REPLAY_SUBSET, static_cast<unsigned long long>(ctr[PULSE_RING_DRAWS]), m);
  for (long long i = warp0; i < upper; i += nwarps) {
    if (i >= stored) {
      if (a.src_rows_out != nullptr && lane == 0) a.src_rows_out[i] = -1;
      continue;
    }
    const long long src = a.kept[m > cap ? subset(i) : i];   // amp_obs[randperm(m)[:buf_size]] once more than buf_size rows are kept
    if (a.src_rows_out != nullptr && lane == 0) a.src_rows_out[i] = src;
    copy_row(a.ring.rows + ((head + i) % cap) * a.ring.row_floats, a.src + src * a.ring.row_floats, a.ring.row_floats, lane);
  }
}

// ---- sample -----------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRingWarps * 32) ring_sample_kernel(const pulse_amp_sample_args_t a, long long rows) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const long long* ctr = reinterpret_cast<const long long*>(a.ring.ctr);
  const long long cap = a.ring.capacity, total = ctr[PULSE_RING_TOTAL], head = ctr[PULSE_RING_HEAD], sh = ctr[PULSE_RING_SAMPLE_HEAD];
  const Feistel perm(a.ring.seed, PULSE_PLANE_RING_PERM, static_cast<unsigned long long>(ctr[PULSE_RING_PERM_KEY]), cap);
  for (long long o = warp0; o < rows; o += nwarps) {
    const long long j = (o / a.take) * a.block + o % a.take;
    float* dst = a.out + o * a.ring.row_floats;
    if (total == 0) {   // train_epoch: amp_obs_replay = amp_obs while the replay buffer is empty
      if (a.ring_rows_out != nullptr && lane == 0) a.ring_rows_out[o] = -1;
      if (a.fallback != nullptr) copy_row(dst, a.fallback + j * a.ring.row_floats, a.ring.row_floats, lane);
      else for (int c = lane; c < a.ring.row_floats; c += 32) dst[c] = 0.0f;
      continue;
    }
    long long r = perm((sh + j) % cap);
    if (total < cap) r %= head;
    if (a.ring_rows_out != nullptr && lane == 0) a.ring_rows_out[o] = r;
    copy_row(dst, a.ring.rows + r * a.ring.row_floats, a.ring.row_floats, lane);
  }
}

__global__ void ring_sample_done_kernel(long long* ctr, long long capacity, long long n) {
  if (ctr[PULSE_RING_TOTAL] == 0) return;
  const long long sh = ctr[PULSE_RING_SAMPLE_HEAD] + n;
  if (sh >= capacity) {   // _reset_sample_idx
    ctr[PULSE_RING_SAMPLE_HEAD] = 0;
    ctr[PULSE_RING_PERM_KEY] += 1;
  } else {
    ctr[PULSE_RING_SAMPLE_HEAD] = sh;
  }
}

int check_ring(const pulse_amp_ring_t& r, const char* who) {
  PULSE_REQUIRE(r.rows != nullptr && r.ctr != nullptr, "%s: null ring rows / counters", who);
  PULSE_REQUIRE(r.capacity >= 1 && r.capacity < (1ll << 31), "%s: capacity %lld outside [1, 2^31)", who, (long long)r.capacity);
  PULSE_REQUIRE(r.row_floats >= 1, "%s: row_floats %d", who, r.row_floats);
  return PULSE_OK;
}

// The checks of a demo fetch over a MotionLib descriptor `d` whose AMP rows are `full` floats (`full - 1` without the root height),
// then the fetch kernel in layout L and store()'s counter update.
template <class L, class Desc>
int demo_fetch(const Desc& d, const pulse_amp_demo_args_t& a, void* stream, const char* who) {
  if (const int s = check_ring(a.ring, who)) return s;
  constexpr int full = L::kAmpObs;
  PULSE_REQUIRE(a.sampling_cdf != nullptr && d.num_motions >= 1, "%s: null sampling_cdf", who);
  PULSE_REQUIRE(d.aux_rec != nullptr, "%s: the MotionLib handle has no aux records (dof_pos / dof_vel)", who);
  PULSE_REQUIRE(a.num_steps >= 1 && a.num_steps <= 16, "%s: num_steps %d outside [1,16]", who, a.num_steps);
  PULSE_REQUIRE(a.amp_width == full || a.amp_width == full - 1, "%s: amp_width %d is neither %d nor %d", who, a.amp_width, full, full - 1);
  PULSE_REQUIRE(L::kUpright || a.upright == 0, "%s: the SMPL-X rows take the heading of remove_base_rot(q0) (upright 0)", who);
  PULSE_REQUIRE(a.ring.row_floats == a.num_steps * a.amp_width, "%s: ring rows of %d floats, the demo rows have %d", who,
                a.ring.row_floats, a.num_steps * a.amp_width);
  PULSE_REQUIRE(a.num_samples >= 0 && a.num_samples <= a.ring.capacity, "%s: num_samples %lld outside [0, capacity]", who,
                (long long)a.num_samples);
  if (a.num_samples == 0) return PULSE_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  demo_fetch_kernel<L><<<grid_for(a.num_samples * a.num_steps, kRingWarps), kRingWarps * 32, 0, st>>>(d, a);
  PULSE_LAUNCH_OK("demo_fetch_kernel");
  ring_store_done_kernel<<<1, 1, 0, st>>>(reinterpret_cast<long long*>(a.ring.ctr), (long long)a.ring.capacity, (long long)a.num_samples);
  PULSE_LAUNCH_OK("ring_store_done_kernel");
  return PULSE_OK;
}

}  // namespace
}  // namespace pulse

extern "C" int pulse_amp_demo_fetch(const pulse_motionlib_t* lib, const pulse_amp_demo_args_t* args, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(lib != nullptr && args != nullptr, "pulse_amp_demo_fetch: null lib/args");
  return demo_fetch<SmplLayout>(lib->d, *args, stream, "pulse_amp_demo_fetch");
}

extern "C" int pulse_smplx_amp_demo_fetch(const pulse_smplx_motionlib_t* lib, const pulse_amp_demo_args_t* args, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(lib != nullptr && args != nullptr, "pulse_smplx_amp_demo_fetch: null lib/args");
  return demo_fetch<SmplxLayout>(lib->d, *args, stream, "pulse_smplx_amp_demo_fetch");
}

extern "C" int pulse_amp_replay_store(const pulse_amp_store_args_t* args, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_amp_replay_store: null args");
  const pulse_amp_store_args_t& a = *args;
  if (const int s = check_ring(a.ring, "pulse_amp_replay_store")) return s;
  PULSE_REQUIRE(a.src != nullptr && a.kept != nullptr, "pulse_amp_replay_store: null src / kept");
  PULSE_REQUIRE(a.num_rows >= 0 && a.num_rows < (1ll << 31), "pulse_amp_replay_store: num_rows %lld outside [0, 2^31)", (long long)a.num_rows);
  PULSE_REQUIRE(a.keep_prob >= 0.0f && a.keep_prob <= 1.0f, "pulse_amp_replay_store: keep_prob %g outside [0, 1]", a.keep_prob);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  keep_compact_kernel<<<1, kCompactThreads, 0, st>>>(a);
  PULSE_LAUNCH_OK("keep_compact_kernel");
  const long long upper = a.num_rows < a.ring.capacity ? a.num_rows : a.ring.capacity;
  if (upper > 0) {
    ring_store_kernel<<<grid_for(upper, kRingWarps), kRingWarps * 32, 0, st>>>(a, upper);
    PULSE_LAUNCH_OK("ring_store_kernel");
  }
  ring_store_done_kernel<<<1, 1, 0, st>>>(reinterpret_cast<long long*>(a.ring.ctr), (long long)a.ring.capacity, -1ll);
  PULSE_LAUNCH_OK("ring_store_done_kernel");
  return PULSE_OK;
}

extern "C" int pulse_amp_ring_sample(const pulse_amp_sample_args_t* args, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_amp_ring_sample: null args");
  const pulse_amp_sample_args_t& a = *args;
  if (const int s = check_ring(a.ring, "pulse_amp_ring_sample")) return s;
  PULSE_REQUIRE(a.out != nullptr, "pulse_amp_ring_sample: null out");
  PULSE_REQUIRE(a.block >= 1 && a.take >= 1 && a.take <= a.block, "pulse_amp_ring_sample: need 1 <= take <= block");
  PULSE_REQUIRE(a.n >= 0 && a.n % a.block == 0, "pulse_amp_ring_sample: n %lld is not a multiple of block %lld", (long long)a.n, (long long)a.block);
  const long long rows = a.n / a.block * a.take;
  if (rows == 0) return PULSE_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ring_sample_kernel<<<grid_for(rows, kRingWarps), kRingWarps * 32, 0, st>>>(a, rows);
  PULSE_LAUNCH_OK("ring_sample_kernel");
  ring_sample_done_kernel<<<1, 1, 0, st>>>(reinterpret_cast<long long*>(a.ring.ctr), (long long)a.ring.capacity, (long long)a.n);
  PULSE_LAUNCH_OK("ring_sample_done_kernel");
  return PULSE_OK;
}
