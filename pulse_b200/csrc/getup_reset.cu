// Getup reset of HumanoidImGetup on the device (humanoid_im_getup.py:135-196), no host synchronisation.  Five launches:
//   getup_classify_kernel   one CTA: releases the assignments of the reset envs, counts the free fall states, then splits the reset
//                           set into ascending union / reference-state / fall / recovery lists with device-side counts (the ordered
//                           compaction of reset_state.cuh) and sets the recovery counters;
//   getup_keys_kernel       one sort key (key, state id) per fall state, all ones for the held ones;
//   getup_select_kernel     rank of every free state among the free ones (one warp per state): the state of rank i goes to the
//                           i-th fall env;
//   getup_apply_kernel      one warp per union env (counters, contact forces) and per fall env (fall-pool copy, assignment);
//   reset_ref_state_kernel  (reset_state.cuh) the reference-state envs, exactly as pulse_reset_ref_state.
// pulse_getup_amp_init writes the AMP history of the fall / recovery envs after the simulator's refresh.
#include "reset_state.cuh"

namespace pulse {
namespace {

constexpr uint64_t kHeldKey = ~0ull;

__global__ void __launch_bounds__(kCompactThreads) getup_classify_kernel(const pulse_getup_reset_args_t g, long long num_envs) {
  const pulse_reset_args_t& a = g.base;
  __shared__ int warp_cnt[kCompactThreads / 32];
  __shared__ int base[4];   // union, reference state, fall, recovery
  __shared__ int num_free;
  const int tid = threadIdx.x;
  if (tid < 4) base[tid] = 0;
  if (tid == 0) num_free = 0;
  const long long n = a.env_ids_in != nullptr ? a.num_ids : num_envs;
  // 1. release (humanoid_im_getup.py:136): the assignment as it stands, even when another env has taken that state since
  for (long long i = tid; i < n; i += kCompactThreads) {
    const long long env = reset_candidate(a, i, n);
    if (env >= 0) g.available_fall_states[g.fall_id_assignments[env]] = 0;
  }
  __syncthreads();
  int free_here = 0;
  for (long long s = tid; s < g.num_fall_states; s += kCompactThreads) free_here += g.available_fall_states[s] == 0;
  free_here = warp_sum(free_here);
  if ((tid & 31) == 0) atomicAdd(&num_free, free_here);
  __syncthreads();
  const int free_states = num_free;
  const unsigned long long off = a.offset + (a.offset_dev != nullptr ? *a.offset_dev : 0ull);
  // 2.-4. classification in ascending env order
  for (long long c0 = 0; c0 < n; c0 += kCompactThreads) {
    const long long env = reset_candidate(a, c0 + tid, n);
    bool rec = false, fall = false;
    if (env >= 0) {
      Philox4 r{0u, 0u, 0u, 0u};
      if (g.recovery_u == nullptr || g.fall_u == nullptr) r = philox4x32_10(a.seed, static_cast<unsigned long long>(env), off);
      const float ur = g.recovery_u != nullptr ? g.recovery_u[env] : u01(r.y);
      const float uf = g.fall_u != nullptr ? g.fall_u[env] : u01(r.z);
      rec = ur < g.recovery_prob && a.terminate_buf[env] == 1;
      fall = !rec && uf < g.fall_prob;
    }
    const int upos = compact_slot(env >= 0, warp_cnt, &base[0]);
    const int fpos = compact_slot(fall, warp_cnt, &base[2]);
    fall = fall && fpos < free_states;          // the surplus of an exhausted pool takes a reference-state episode
    const bool ref = env >= 0 && !rec && !fall;
    const int rpos = compact_slot(ref, warp_cnt, &base[1]);
    const int cpos = compact_slot(rec, warp_cnt, &base[3]);
    if (env < 0) continue;
    a.env_list[upos] = env;
    if (a.actor_list != nullptr) a.actor_list[upos] = a.actor_ids != nullptr ? a.actor_ids[env] : static_cast<int>(env);
    if (ref) g.ref_list[rpos] = env;
    if (fall) g.fall_list[fpos] = env;
    if (rec) g.recovery_list[cpos] = env;
    g.recovery_counter[env] = ref ? 0 : g.recovery_steps;
    if (g.env_class != nullptr) g.env_class[env] = ref ? PULSE_GETUP_REF : (fall ? PULSE_GETUP_FALL : PULSE_GETUP_RECOVERY);
  }
  if (tid == 0) {
    const int falls = base[2] < free_states ? base[2] : free_states;
    *a.count = base[0];
    g.class_counts[0] = base[1];
    g.class_counts[1] = falls;
    g.class_counts[2] = base[3];
    if (base[2] > falls) *g.error += base[2] - falls;
  }
}

// (key bits, state id): distinct for every state, ordered by key first.  A non-negative float key orders like its bit pattern.
__global__ void __launch_bounds__(256) getup_keys_kernel(const pulse_getup_reset_args_t g) {
  const pulse_reset_args_t& a = g.base;
  const unsigned long long off = a.offset + (a.offset_dev != nullptr ? *a.offset_dev : 0ull);
  for (long long s = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; s < g.num_fall_states;
       s += static_cast<long long>(gridDim.x) * blockDim.x) {
    uint64_t k = kHeldKey;
    if (g.available_fall_states[s] == 0) {
      const unsigned bits = g.fall_keys != nullptr ? __float_as_uint(g.fall_keys[s]) : philox4x32_10(a.seed, static_cast<unsigned long long>(s), off).w;
      k = (static_cast<unsigned long long>(bits) << 32) | static_cast<unsigned long long>(s);
    }
    g.fall_key_scratch[s] = k;
  }
}

// Rank of each free state = number of smaller keys, one warp per state: every lane compares one key of a 32-key chunk and a ballot
// counts the chunk.  A state stops counting once its rank reaches the number of fall envs, so only the chosen states scan the whole
// pool; the others stop after about falls * P / rank keys.
__global__ void __launch_bounds__(256) getup_select_kernel(const pulse_getup_reset_args_t g) {
  const int falls = g.class_counts[1];
  if (falls == 0) return;
  const int lane = threadIdx.x & 31;
  const long long warp0 = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const uint64_t* key = g.fall_key_scratch;
  const long long P = g.num_fall_states;
  for (long long s = warp0; s < P; s += nwarps) {
    const uint64_t mine = key[s];
    if (mine == kHeldKey) continue;
    int rank = 0;
    for (long long t0 = 0; t0 < P && rank < falls; t0 += 4 * 32) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const long long t = t0 + 32 * j + lane;
        rank += __popc(__ballot_sync(kFull, t < P && key[t] < mine));
      }
    }
    if (lane == 0 && rank < falls) g.fall_pick[rank] = s;
  }
}

__global__ void __launch_bounds__(256) getup_apply_kernel(const pulse_getup_reset_args_t g) {
  const pulse_reset_args_t& a = g.base;
  const int lane = threadIdx.x & 31;
  const long long warp0 = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const long long num_union = *a.count;
  const long long items = num_union + g.class_counts[1];
  for (long long it = warp0; it < items; it += nwarps) {
    if (it < num_union) {   // _reset_env_tensors (humanoid.py:603-606)
      const long long e = a.env_list[it];
      if (a.contact_forces != nullptr)
        for (int c = lane; c < a.contact_bodies * 3; c += 32) a.contact_forces[e * a.contact_env_stride + c] = 0.0f;
      if (lane == 0) {
        a.progress_buf[e] = 0;
        if (a.reset_buf != nullptr) a.reset_buf[e] = 0;
        a.terminate_buf[e] = 0;
      }
      continue;
    }
    // _reset_fall_episode (humanoid_im_getup.py:174-182): plain copies of the fall pool
    const long long r = it - num_union;
    const long long e = g.fall_list[r], s = g.fall_pick[r];
    if (lane < PULSE_BODY_STATE_W) a.root_states[e * a.root_env_stride + lane] = g.fall_root_states[s * g.fall_root_stride + lane];
    for (int c = lane; c < PULSE_NUM_DOF; c += 32) {
      const long long src = s * g.fall_dof_env_stride + c * g.fall_dof_elem_stride, dst = e * a.dof_env_stride + c * a.dof_elem_stride;
      a.dof_pos[dst] = g.fall_dof_pos[src];
      a.dof_vel[dst] = g.fall_dof_vel[src];
    }
    if (lane == 0) {
      g.available_fall_states[s] = 1;
      g.fall_id_assignments[e] = s;
    }
  }
}

__global__ void __launch_bounds__(256) getup_amp_init_kernel(const pulse_getup_amp_args_t a) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const long long falls = a.class_counts[1];
  const long long items = falls + a.class_counts[2];
  for (long long it = warp0; it < items; it += nwarps) {
    const bool fall = it < falls;
    const long long e = fall ? a.fall_list[it] : a.recovery_list[it - falls];
    float* row0 = a.amp_obs_buf + e * static_cast<long long>(a.num_steps) * PULSE_AMP_OBS;
    store_amp_obs_sim(row0, lane, a, e);   // _compute_amp_observations(env_ids) (humanoid_amp.py:520)
    if (!fall) continue;
    __syncwarp();
    for (int k = 1; k < a.num_steps; ++k)  // _init_amp_obs_default (humanoid_amp.py:530-533)
      for (int c = lane; c < PULSE_AMP_OBS; c += 32) row0[k * PULSE_AMP_OBS + c] = row0[c];
  }
}

}  // namespace
}  // namespace pulse

extern "C" int pulse_reset_getup(const pulse_motionlib_t* lib, const pulse_getup_reset_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(lib != nullptr && args != nullptr, "pulse_reset_getup: null lib/args");
  const pulse_getup_reset_args_t& g = *args;
  const pulse_reset_args_t& a = g.base;
  const int rc = check_ref_state_args(lib, a, num_envs, "pulse_reset_getup");
  if (rc != PULSE_OK) return rc;
  PULSE_REQUIRE(a.terminate_buf != nullptr, "pulse_reset_getup: terminate_buf is required (it selects the recovery envs)");
  PULSE_REQUIRE(g.recovery_counter && g.available_fall_states && g.fall_id_assignments, "pulse_reset_getup: null getup buffer");
  PULSE_REQUIRE(g.ref_list && g.fall_list && g.recovery_list && g.class_counts && g.error, "pulse_reset_getup: null output list / count");
  PULSE_REQUIRE(g.fall_pick && g.fall_key_scratch, "pulse_reset_getup: null scratch");
  PULSE_REQUIRE(g.num_fall_states >= 1 && g.num_fall_states < (1ll << 31), "pulse_reset_getup: num_fall_states %lld outside [1, 2^31)",
                (long long)g.num_fall_states);
  PULSE_REQUIRE(g.fall_root_states && g.fall_dof_pos && g.fall_dof_vel, "pulse_reset_getup: null fall-state pool");
  PULSE_REQUIRE(g.fall_root_stride >= PULSE_BODY_STATE_W && g.fall_dof_elem_stride >= 1 &&
                g.fall_dof_env_stride >= PULSE_NUM_DOF * g.fall_dof_elem_stride, "pulse_reset_getup: bad fall-state strides");
  PULSE_REQUIRE(g.recovery_steps >= 0, "pulse_reset_getup: negative recovery_steps");
  if (num_envs == 0) return PULSE_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long upper = a.env_ids_in != nullptr ? a.num_ids : num_envs;
  getup_classify_kernel<<<1, kCompactThreads, 0, st>>>(g, (long long)num_envs);
  PULSE_LAUNCH_OK("getup_classify_kernel");
  getup_keys_kernel<<<grid_for(g.num_fall_states, 256), 256, 0, st>>>(g);
  PULSE_LAUNCH_OK("getup_keys_kernel");
  getup_select_kernel<<<grid_for(g.num_fall_states, 8), 256, 0, st>>>(g);
  PULSE_LAUNCH_OK("getup_select_kernel");
  getup_apply_kernel<<<grid_for(2 * upper, 8), 256, 0, st>>>(g);
  PULSE_LAUNCH_OK("getup_apply_kernel");
  pulse_reset_args_t r = a;   // the reference-state envs: pulse_reset_ref_state's kernel over their list
  r.env_list = g.ref_list;
  r.count = g.class_counts;
  r.actor_list = nullptr;
  return launch_ref_state(lib, r, upper, st);
}

extern "C" int pulse_getup_amp_init(const pulse_getup_amp_args_t* args, int64_t num_envs, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_getup_amp_init: null args");
  PULSE_REQUIRE(num_envs >= 0, "pulse_getup_amp_init: negative num_envs");
  const pulse_getup_amp_args_t& a = *args;
  PULSE_REQUIRE(a.body_state && a.dof_pos && a.dof_vel && a.amp_obs_buf, "pulse_getup_amp_init: null buffer");
  PULSE_REQUIRE(a.fall_list && a.recovery_list && a.class_counts, "pulse_getup_amp_init: null list / count");
  PULSE_REQUIRE(a.num_steps >= 1 && a.num_steps <= 16, "pulse_getup_amp_init: num_steps %d outside [1,16]", a.num_steps);
  PULSE_REQUIRE(a.body_env_stride >= PULSE_NUM_BODIES * PULSE_BODY_STATE_W, "pulse_getup_amp_init: body_env_stride too small");
  if (num_envs == 0) return PULSE_OK;
  getup_amp_init_kernel<<<grid_for(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  PULSE_LAUNCH_OK("getup_amp_init_kernel");
  return PULSE_OK;
}
