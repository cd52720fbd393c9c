// Fused HumanoidIm post-physics step kernel: reward(t) -> reset(t) -> observation(t+dt).
//
// One persistent, warp-specialised CTA per SM (20 warps), looping over groups of 8 envs:
//   planner   (1 warp, lane = env, 4 groups per pass): per-env task scalars, per-motion constants, the
//             two motion times and frame indices in the reference's exact fp32 order; deduplicates the
//             four frame rows of the two queries into <= 3 copy slots (at 30 fps the reward query's
//             second frame IS the observation query's first).  Runs up to two passes (8 groups) ahead
//             through a plan ring.
//   issuer    (1 warp): the moment a data stage is free, launches the group's bulk async copies
//             (cp.async.bulk: 1248-byte packed frame records + the 24x13 rigid-body state) onto the
//             stage's "full" mbarrier -- the dependent chain scalars -> motion constants -> rows is
//             already resolved, so every stage that is not being computed on has loads in flight.
//   consumers (3 teams x 6 warps; a team = 8 envs x 24 bodies, one thread per (env, body), no idle
//             lanes): blend the reference pose (lerp / slerp), per-body reward errors and termination
//             distance into shared partials, observation pieces into registers; the 934-float row is
//             then staged in the bytes the env's records occupied and leaves with ONE bulk async store
//             per env (16-byte aligned middle; <= 3 ragged floats at either end stored directly).  Teams
//             take groups round-robin; five data stages keep two groups loading while three compute.  The
//             power-term operands |tau . qdot| of a team's next group ride in registers across its math.
//
// HBM-bound by design: algorithmic traffic is 9 396 B per env-step (SURVEY.md 8d), nothing is
// re-read from DRAM.  References: humanoid_im.py:853-919, :1119-1192, :677-851, :1328-1378,
// :1543-1628; humanoid.py:1675-1731; motion_lib_base.py:434-517, :546-556.
#include "humanoid_obs.cuh"

namespace pulse {
namespace {

constexpr int kNB = PULSE_NUM_BODIES;
constexpr int kEnvs = 8;                   // envs per group
constexpr int kTeam = kEnvs * kNB;         // 192 threads: one per (env, body)
#ifndef PULSE_STEP_TEAMS
#define PULSE_STEP_TEAMS 3    // A/B knob (tools/build_variant.sh): 2 teams = 448 threads, register cap 146 instead of 96
#endif
#ifndef PULSE_STEP_STAGES
#define PULSE_STEP_STAGES 5
#endif
constexpr int kTeams = PULSE_STEP_TEAMS;   // consumer teams per CTA
constexpr int kConsumers = kTeam * kTeams; // 576
constexpr int kThreads = kConsumers + 64;  // + issuer warp + planner warp (20 warps: register cap 102)
constexpr int kStages = PULSE_STEP_STAGES; // data stages
constexpr int kBatch = 4;                  // groups planned per planner pass (4 x 8 envs = 32 lanes)
constexpr int kPlanSlots = 2;              // plan ring: planner passes in flight
constexpr int kFrame = PULSE_FRAME_REC;    // 312 floats = 1248 B
constexpr int kSlots = 3;                  // frame-record copy slots per env
constexpr int kObs = PULSE_IM_OBS;         // 934
constexpr int kRed = 6;                    // pos, rot, vel, ang-vel, distance (mean criterion), power
constexpr unsigned kFrameBytes = kFrame * 4;
constexpr unsigned kDirect = 3;            // slot id of a 4th distinct row: read straight from global / L2
static_assert(kTeam % 32 == 0, "a team must fill whole warps");

struct EnvParams {           // issuer -> consumers (copied into the stage)
  long long env;             // env index after the env_ids indirection
  long long prog;            // progress_buf
  long long aux0, aux1;      // rows of the observation query (aux records for ref_dof_pos)
  long long direct_row;      // row that did not get a copy slot (rare), else -1
  float b_rew, b_obs;
  float gx, gy, gz;
  float t_rew, mlen;
  int cyc;
  int rec;                   // recovery_counter > 0 (getup task)
  int valid;
  int body_bulk;
  unsigned char sl[4];       // copy slot (0..2, or kDirect) of logical rows: rew f0, rew f1, obs f0, obs f1
};

struct PlanEntry {           // planner -> issuer
  EnvParams prm;
  long long slot_row[kSlots];
  const float* body_src;
  int nslots;
};

// Per env: three frame-record slots (936 floats) and, in a SEPARATE array, the rigid-body state (312 floats); the obs row is staged over
// the frame slots once they are consumed.  Round 1 kept [slot0 | slot1 | slot2 | body] in one 1248-float block: 1248 = 0 (mod 32 banks), so
// the 8 lanes of a warp that belong to the next env hit the banks of the first env's lanes on EVERY record read (ncu: 1.93 M conflicts,
// 46 % of the stall cycles on shared-memory scoreboards).  With lane = (env k, body j) a stride-3 read of a frame record is conflict-free
// across the env boundary iff the env stride is 8 (mod 32) -- 936 is; the stride-13 body-state read needs 24 (mod 32) -- 312 is.
constexpr int kFrameBlock = kSlots * kFrame;   // 936
struct __align__(16) Stage {
  float fr[kEnvs][kFrameBlock];
  float body[kEnvs][kFrame];
  EnvParams prm[kEnvs];
};
static_assert((kObs + 2) <= kFrameBlock, "obs staging (alignment phase <= 2) must fit inside the frame slots");
static_assert(kFrameBlock % 32 == 8 && kFrame % 32 == 24, "bank-conflict-free env strides");

struct __align__(16) CtaSmem {
  Stage stage[kStages];
  float red[kTeams][kEnvs][kRed][kNB + 1];  // per-body partials, column kNB = sum
  float root[kTeams][kEnvs][8];             // root position / rotation of the team's envs
  PlanEntry plan[kPlanSlots][kBatch][kEnvs];
  unsigned fallen[kTeams][kEnvs];
  unsigned long long full[kStages];           // issuer -> consumers: records landed (tx bytes)
  unsigned long long empty[kStages];          // consumers -> issuer: stage may be overwritten
  unsigned long long plan_full[kPlanSlots];   // planner -> issuer
  unsigned long long plan_empty[kPlanSlots];  // issuer -> planner
};

// ---- mbarrier / bulk-copy PTX ----------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return static_cast<unsigned>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void team_sync(int team) { asm volatile("bar.sync %0, %1;\n" ::"r"(team + 1), "n"(kTeam) : "memory"); }
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, unsigned parity) {
  unsigned ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  // bounded: a byte-count bug must surface as a launch error, never as a hung GPU
  for (int spin = 0; spin < (1 << 24); ++spin)
    if (mbar_try_wait(bar, parity)) return;
  __trap();
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gmem_dst, const void* smem_src, unsigned bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;\n" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;\n" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

// Reference pose of body j blended between two frame records.
struct RefPose {
  Vec3 p, v, w;
  Quat q;
};
__device__ __forceinline__ RefPose blend_pose(const float* f0, const float* f1, int j, float b, float gx, float gy, float gz) {
  RefPose r;
  // position feeds the reset mask: reproduce ((1-b)*p0 + b*p1) + off without contraction
  r.p.x = __fadd_rn(lerp_rn(f0[3 * j + 0], f1[3 * j + 0], b), gx);
  r.p.y = __fadd_rn(lerp_rn(f0[3 * j + 1], f1[3 * j + 1], b), gy);
  r.p.z = __fadd_rn(lerp_rn(f0[3 * j + 2], f1[3 * j + 2], b), gz);
  r.q = slerp(ldq4(f0 + 72 + 4 * j), ldq4(f1 + 72 + 4 * j), b);
  const float a = 1.0f - b;
  const float* v0 = f0 + 168 + 3 * j;
  const float* v1 = f1 + 168 + 3 * j;
  r.v = {a * v0[0] + b * v1[0], a * v0[1] + b * v1[1], a * v0[2] + b * v1[2]};
  const float* w0 = f0 + 240 + 3 * j;
  const float* w1 = f1 + 240 + 3 * j;
  r.w = {a * w0[0] + b * w1[0], a * w0[1] + b * w1[1], a * w0[2] + b * w1[2]};
  return r;
}

// yaw_rot of a difference of the blended reference position, with the y and z products fused the way the full row's code compiles
// them (fma(s, v.y, wz2 * v.x), fma(s, v.z, zz2 * v.z)).  Which product of a * b + c * d the compiler fuses follows the code around
// it; the tracked row pins it with intrinsics so its columns stay the full row's bit for bit.
__device__ __forceinline__ Vec3 yaw_rot_pinned(Yaw y, Vec3 v) {
  return {v.x * y.s - y.wz2 * v.y, __fmaf_rn(y.s, v.y, __fmul_rn(y.wz2, v.x)), __fmaf_rn(y.s, v.z, __fmul_rn(y.zz2, v.z))};
}

// ---- planner: one pass plans kBatch groups (lane = group-in-batch * 8 + env slot) ----------------------
__device__ __forceinline__ void plan_batch(const pulse_motionlib_desc_t& lib, const pulse_im_step_args_t& a, long long num_envs,
                                           long long ngroups, long long first_group, long long group_stride,
                                           PlanEntry (*slot)[kEnvs], int lane, bool need_t, bool do_obs, bool do_reset) {
  const int gb = lane / kEnvs, ks = lane - gb * kEnvs;
  const long long group = first_group + gb * group_stride;
  const long long widx = group * kEnvs + ks;
  PlanEntry& E = slot[gb][ks];
  if (group < ngroups && widx < num_envs) {
    const long long e = a.env_ids != nullptr ? a.env_ids[widx] : widx;
    long long prog = a.progress_buf[e];
    // HumanoidImGetup._compute_reset (humanoid_im_getup.py:203-210): a recovering env does not advance its progress counter, so its
    // observation is taken at (prog - 1) + 1
    const int rec = (do_reset && a.recovery_counter != nullptr) ? (a.recovery_counter[e] > 0 ? 1 : 0) : 0;
    if (a.flags & PULSE_STEP_ADVANCE) {   // `self.progress_buf += 1` of post_physics_step (humanoid.py:1317) done here
      prog += 1;
      if (!rec) a.progress_rw[e] = prog;  // a recovering env's counter is written once, by the reset epilogue (prog - 1)
    }
    const long long mid = a.motion_ids[e];
    const float t_start = a.motion_start_times[e];
    const float t_off = a.motion_start_offset[e];
    const float mlen = lib.lengths[mid];
    const float mdt = lib.dt[mid];
    const long long nf = lib.num_frames[mid];
    const long long row0 = lib.length_starts[mid];
    const float t_rew = motion_time_rn(prog, a.dt, t_start, t_off);
    const float t_obs = motion_time_rn(prog + 1 - rec, a.dt, t_start, t_off);
    long long i0r, i1r, i0o, i1o;
    float b_rew, b_obs;
    frame_blend_rn(t_rew, mlen, nf, mdt, i0r, i1r, b_rew);
    frame_blend_rn(t_obs, mlen, nf, mdt, i0o, i1o, b_obs);
    const long long rows[4] = {row0 + i0r, row0 + i1r, row0 + i0o, row0 + i1o};
    // <= 3 copy slots for the (up to) four rows; a 4th distinct row is fetched by the consumers directly
    long long srow[kSlots] = {-1, -1, -1};
    long long direct = -1;
    int ns = 0;
    unsigned char sl[4] = {0, 0, 0, 0};
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const bool wanted = (r < 2) ? need_t : do_obs;
      if (!wanted) continue;
      int found = -1;
#pragma unroll
      for (int m = 0; m < kSlots; ++m)
        if (m < ns && srow[m] == rows[r]) found = m;
      if (found < 0) {
        if (ns < kSlots) {
          found = ns;
#pragma unroll
          for (int m = 0; m < kSlots; ++m)
            if (m == ns) srow[m] = rows[r];
          ++ns;
        } else {
          found = kDirect;
          direct = rows[r];
        }
      }
      sl[r] = static_cast<unsigned char>(found);
    }
    const float* bsrc = a.body_state + e * a.body_env_stride;
#pragma unroll
    for (int m = 0; m < kSlots; ++m) E.slot_row[m] = srow[m];
    E.nslots = ns;
    E.body_src = bsrc;
    EnvParams& P = E.prm;
    P.env = e;
    P.prog = prog;
    P.aux0 = rows[2];
    P.aux1 = rows[3];
    P.direct_row = direct;
    P.b_rew = b_rew;
    P.b_obs = b_obs;
    P.gx = a.global_offset[3 * e + 0];
    P.gy = a.global_offset[3 * e + 1];
    P.gz = a.global_offset[3 * e + 2];
    P.t_rew = t_rew;
    P.mlen = mlen;
    P.cyc = (do_reset && a.cycle_counter != nullptr) ? a.cycle_counter[e] : 0;
    P.rec = rec;
    P.valid = 1;
    P.body_bulk = (reinterpret_cast<uintptr_t>(bsrc) & 15u) == 0 ? 1 : 0;
#pragma unroll
    for (int r = 0; r < 4; ++r) P.sl[r] = sl[r];
  } else {
    E.prm.valid = 0;
    E.prm.body_bulk = 0;
    E.nslots = 0;
  }
}

// ---- issuer: launch one planned group's bulk copies into a free stage (warp-collective) -------------------
__device__ __forceinline__ void issue_group(const pulse_motionlib_desc_t& lib, const PlanEntry* plan, Stage& sg,
                                            unsigned long long* full, int lane) {
  unsigned bytes = 0;
  const bool mine = lane < kEnvs;
  bool v = false;
  int ns = 0, body_bulk = 0;
  if (mine) {
    const PlanEntry& E = plan[lane];
    sg.prm[lane] = E.prm;
    v = E.prm.valid != 0;
    ns = E.nslots;
    body_bulk = E.prm.body_bulk;
    if (v) bytes = static_cast<unsigned>(ns + (body_bulk ? 1 : 0)) * kFrameBytes;
  }
  const unsigned total = __reduce_add_sync(kFull, bytes);  // REDUX also orders the prm[] writes before lane 0's arrive
  __syncwarp();
  if (lane == 0) mbar_arrive_expect_tx(full, total);
  __syncwarp();                                    // the expectation is posted before any copy can complete
  if (v) {
    const PlanEntry& E = plan[lane];
    float* blk = sg.fr[lane];
#pragma unroll
    for (int m = 0; m < kSlots; ++m)
      if (m < ns) bulk_g2s(blk + m * kFrame, lib.frame_rec + E.slot_row[m] * kFrame, kFrameBytes, full);
    if (body_bulk) bulk_g2s(sg.body[lane], E.body_src, kFrameBytes, full);
  }
}

// raw dof force / velocity operands of the power term (humanoid_im.py:910-912) for (env slot k of `group`, body j)
struct PowerOps {
  float f[3], v[3];
};
__device__ __forceinline__ PowerOps power_load(const pulse_im_step_args_t& a, long long num_envs, long long group, int k, int j) {
  PowerOps o;
#pragma unroll
  for (int m = 0; m < 3; ++m) o.f[m] = o.v[m] = 0.0f;
  const long long widx = group * kEnvs + k;
  if (widx < num_envs) {
    const long long e = a.env_ids != nullptr ? a.env_ids[widx] : widx;
    const float* fr = a.dof_force + e * a.dof_force_stride;
    const float* dv = a.dof_vel + e * a.dof_env_stride;
#pragma unroll
    for (int m = 0; m < 3; ++m) {
      const int d = j + kNB * m;
      if (d < PULSE_NUM_DOF) {
        o.f[m] = __ldg(fr + d);
        o.v[m] = __ldg(dv + d * a.dof_elem_stride);
      }
    }
  }
  return o;
}

// kTrack: the observation row is [self | task observation of the tracked bodies] (pulse_im_track_t) instead of the 934-float row
template <bool kTrack>
__global__ void __launch_bounds__(kThreads, 1) im_step_kernel(const pulse_motionlib_desc_t lib, const pulse_im_step_args_t a,
                                                              long long num_envs, const pulse_im_track_t tr) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  CtaSmem& sm = *reinterpret_cast<CtaSmem*>(smem_raw);
  const int tid = threadIdx.x;
  const bool do_rew = a.flags & PULSE_STEP_REWARD;
  const bool do_reset = a.flags & PULSE_STEP_RESET;
  const bool do_obs = a.flags & PULSE_STEP_OBS;
  const bool need_t = do_rew || do_reset;
  const bool do_power = do_rew && a.dof_force != nullptr;
  if (a.env_count != nullptr) {   // device-side length of the env list (pulse_reset_ref_state): no host read of the count
    const long long c = *a.env_count;
    num_envs = c < num_envs ? (c < 0 ? 0 : c) : num_envs;
  }
  const long long ngroups = (num_envs + kEnvs - 1) / kEnvs;

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], kTeam);  // every thread of the consuming team hands the stage back itself
    }
#pragma unroll
    for (int s = 0; s < kPlanSlots; ++s) {
      mbar_init(&sm.plan_full[s], 1);
      mbar_init(&sm.plan_empty[s], 1);
    }
  }
  __syncthreads();
  // this CTA handles groups blockIdx.x + n * gridDim.x, n = 0 .. my_groups-1
  const long long my_groups = (ngroups - blockIdx.x + gridDim.x - 1) / gridDim.x;

  if (tid >= kConsumers + 32) {
    // ================================ planner warp: runs up to kPlanSlots passes ahead =================
    const int lane = tid - (kConsumers + 32);
    for (long long b = 0; b * kBatch < my_groups; ++b) {
      const int ps = static_cast<int>(b % kPlanSlots);
      if (b >= kPlanSlots) mbar_wait(&sm.plan_empty[ps], ((b / kPlanSlots) - 1) & 1);
      plan_batch(lib, a, num_envs, ngroups, blockIdx.x + b * kBatch * gridDim.x, gridDim.x, sm.plan[ps], lane, need_t, do_obs,
                 do_reset);
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.plan_full[ps]);
    }
    return;
  }
  if (tid >= kConsumers) {
    // ================================ issuer warp: bulk copies as soon as a stage is free ===============
    const int lane = tid - kConsumers;
    for (long long n = 0; n < my_groups; ++n) {
      const long long b = n / kBatch;
      const int ps = static_cast<int>(b % kPlanSlots), gb = static_cast<int>(n % kBatch);
      const int s = static_cast<int>(n % kStages);
      mbar_wait(&sm.plan_full[ps], (b / kPlanSlots) & 1);
      if (n >= kStages) mbar_wait(&sm.empty[s], ((n / kStages) - 1) & 1);  // consumers released this stage
      issue_group(lib, sm.plan[ps][gb], sm.stage[s], &sm.full[s], lane);
      if (gb == kBatch - 1 || n == my_groups - 1) {
        __syncwarp();                                  // every lane has read its plan entry
        if (lane == 0) mbar_arrive(&sm.plan_empty[ps]);
      }
    }
    return;
  }

  // ================================== consumers: team x (env slot k, body j) ==========================
  const int team = tid / kTeam;
  const int ttid = tid - team * kTeam;
  const int k = ttid / kNB;
  const int j = ttid - k * kNB;
  const float term_j = do_reset ? a.termination_distances[j] : 0.0f;
  float(*red)[kRed][kNB + 1] = sm.red[team];
  unsigned* fallen = sm.fallen[team];
  const int rank = kTrack ? tr.rank[j] : -1;   // body j's place in the tracked row, -1 = untracked
  PowerOps pw_ops = {};
  if (do_power && team < my_groups) pw_ops = power_load(a, num_envs, blockIdx.x + team * (long long)gridDim.x, k, j);
  for (long long n = team; n < my_groups; n += kTeams) {
    const int s = static_cast<int>(n % kStages);
    Stage& sg = sm.stage[s];
    const float pw = fabsf(pw_ops.f[0] * pw_ops.v[0]) + fabsf(pw_ops.f[1] * pw_ops.v[1]) + fabsf(pw_ops.f[2] * pw_ops.v[2]);
    // operands of this team's NEXT group stay in flight (registers) across this group's math
    if (do_power && n + kTeams < my_groups) pw_ops = power_load(a, num_envs, blockIdx.x + (n + kTeams) * gridDim.x, k, j);
    mbar_wait(&sm.full[s], (n / kStages) & 1);  // frame records + body state have landed, prm[] visible

    const EnvParams P = sg.prm[k];
    const bool valid = P.valid != 0;
    float* blk = sg.fr[k];
    // rigid-body state: shared memory when it came through the bulk path, else straight from global
    const float* body = (P.body_bulk || !valid) ? sg.body[k] : a.body_state + P.env * a.body_env_stride;
    const float* bj = body + j * PULSE_BODY_STATE_W;
    const Vec3 p = {bj[0], bj[1], bj[2]};
    const Quat q = {bj[3], bj[4], bj[5], bj[6]};
    const Vec3 v = {bj[7], bj[8], bj[9]};
    const Vec3 w = {bj[10], bj[11], bj[12]};
    if (j == 0) {  // the env's root state, needed by every body thread of the env in the obs part
      float* rt = sm.root[team][k];
      rt[0] = p.x; rt[1] = p.y; rt[2] = p.z;
      rt[3] = q.x; rt[4] = q.y; rt[5] = q.z; rt[6] = q.w;
    }
    if (ttid < kEnvs) fallen[ttid] = 0u;  // OR-ed after the first team_sync, read after the second
    const float* direct = (valid && P.direct_row >= 0) ? lib.frame_rec + P.direct_row * kFrame : blk;

    // ---- reward + reset partials at t -----------------------------------------------------------------
    RefPose r2;
    bool is_fallen = false;
    if (valid && need_t) {
      const float* f0 = P.sl[0] < kDirect ? blk + P.sl[0] * kFrame : direct;
      const float* f1 = P.sl[1] < kDirect ? blk + P.sl[1] * kFrame : direct;
      const RefPose r = blend_pose(f0, f1, j, P.b_rew, P.gx, P.gy, P.gz);
      if (do_rew) {
        const float th = quat_angle(qmul(r.q, qconj(q)));
        red[k][0][j] = sq3(r.p - p);
        red[k][1][j] = th * th;
        red[k][2][j] = sq3(r.v - v);
        red[k][3][j] = sq3(r.w - w);
        red[k][5][j] = pw;
      }
      if (do_reset) {
        const bool in_mask = (a.reset_body_mask >> j) & 1u;
        const float dist = norm3_rn(__fsub_rn(p.x, r.p.x), __fsub_rn(p.y, r.p.y), __fsub_rn(p.z, r.p.z));
        red[k][4][j] = in_mask ? dist : 0.0f;
        is_fallen = in_mask && dist > term_j;
      }
    }
    // ---- observation at t + dt: fold the frames into registers --------------------------------------------
    if (valid && do_obs) {
      const float* f0 = P.sl[2] < kDirect ? blk + P.sl[2] * kFrame : direct;
      const float* f1 = P.sl[3] < kDirect ? blk + P.sl[3] * kFrame : direct;
      r2 = blend_pose(f0, f1, j, P.b_obs, P.gx, P.gy, P.gz);
    }
    team_sync(team);  // the env blocks are consumed: their bytes become the obs rows; partials complete

    float* orow = nullptr;
    int ophase = 0;
    if (valid && do_obs) {
      const float* rt = sm.root[team][k];
      const Vec3 p_root = {rt[0], rt[1], rt[2]};
      const Quat q_root = {rt[3], rt[4], rt[5], rt[6]};
      float hs, hc;
      heading_half(q_root, hs, hc);
      const Yaw yr = make_yaw(Quat{0.0f, 0.0f, -hs, hc});
      orow = a.obs_buf + P.env * a.obs_stride;
      ophase = static_cast<int>((reinterpret_cast<uintptr_t>(orow) >> 2) & 3);
      // global 16-byte boundaries coincide with shared ones; a row starting 3 floats past a boundary would need 937 staging floats:
      // it is written straight to global memory instead (never the case for [N, 934]-strided buffers: 934 k = 0 or 2 mod 4; every
      // fourth row of a tracked v7 row with odd K, 358 + 9 K floats wide)
      float* o = ophase == 3 ? orow : blk + ophase;
      // self observation, store_self_obs's layout written out: through the helper ptxas fuses the other product of yaw_rot's
      // a * b - c * d, which moves the result by an ulp
      if (j == 0) o[0] = p_root.z;
      else stv(o + 1 + 3 * (j - 1), yaw_rot(yr, p - p_root));
      qsix(yaw_mul_left(-hs, hc, q), o + 70 + 6 * j);
      stv(o + 214 + 3 * j, yaw_rot(yr, v));
      stv(o + 286 + 3 * j, yaw_rot(yr, w));
      // task observation v6 (humanoid_im.py:1328-1378), block-major
      float* t = o + PULSE_SELF_OBS;
      if constexpr (kTrack) {
        // the tracked subset: the full row's pieces, each block K bodies wide, body j at its rank in _track_bodies_id (v7, :1381-1413,
        // keeps dp | dv | R(p_ref - p_root)).  Every thread computes all six pieces in this block, without a branch, as the full row
        // does, so the compiler orders and fuses their products as there; for the two pieces rotated from the blended reference
        // position it still picks the other product of y and z to fuse, and yaw_rot_pinned fixes that.  The columns are then the full
        // row's bit for bit (the PTX expression trees of the six pieces match; tests/test_gpu_imz_rollout.py checks the values).
        // What is not part of the row goes to a 24-float sink at the end of the env's frame slots, past the staged row (the row
        // reaches it only at K = 24, when every body is tracked); nothing reads the sink.
        const int K = tr.num_track;
        const bool v6 = tr.version == 6, on = rank >= 0;
        float* sink = blk + (kFrameBlock - 24);
        float* const d[6] = {on ? t + 3 * rank : sink,
                             on && v6 ? t + 3 * K + 6 * rank : sink + 3,
                             on ? t + (v6 ? 9 : 3) * K + 3 * rank : sink + 9,
                             on && v6 ? t + 12 * K + 3 * rank : sink + 12,
                             on ? t + (v6 ? 15 : 6) * K + 3 * rank : sink + 15,
                             on && v6 ? t + 18 * K + 6 * rank : sink + 18};
        stv(d[0], yaw_rot_pinned(yr, r2.p - p));
        qsix(yaw_mul_right(yaw_mul_left(-hs, hc, qmul(r2.q, qconj(q))), hs, hc), d[1]);
        stv(d[2], yaw_rot(yr, r2.v - v));
        stv(d[3], yaw_rot(yr, r2.w - w));
        stv(d[4], yaw_rot_pinned(yr, r2.p - p_root));
        qsix(yaw_mul_left(-hs, hc, r2.q), d[5]);
      } else {
        stv(t + 3 * j, yaw_rot(yr, r2.p - p));
        qsix(yaw_mul_right(yaw_mul_left(-hs, hc, qmul(r2.q, qconj(q))), hs, hc), t + 72 + 6 * j);
        stv(t + 216 + 3 * j, yaw_rot(yr, r2.v - v));
        stv(t + 288 + 3 * j, yaw_rot(yr, r2.w - w));
        stv(t + 360 + 3 * j, yaw_rot(yr, r2.p - p_root));
        qsix(yaw_mul_left(-hs, hc, r2.q), t + 432 + 6 * j);
      }
      // reference-pose side buffers (humanoid_im.py:835-848)
      if (a.ref_body_pos != nullptr) stv(a.ref_body_pos + P.env * (kNB * 3) + 3 * j, r2.p);
      if (a.ref_body_vel != nullptr) stv(a.ref_body_vel + P.env * (kNB * 3) + 3 * j, r2.v);
      if (a.ref_body_rot != nullptr) {
        float* d = a.ref_body_rot + P.env * (kNB * 4) + 4 * j;
        d[0] = r2.q.x; d[1] = r2.q.y; d[2] = r2.q.z; d[3] = r2.q.w;
      }
      if (a.ref_dof_pos != nullptr && j >= 1) {
        // dof_pos = exp_map(slerp(lrs[f0, j], lrs[f1, j], blend)), joints 1..23 (motion_lib_base.py:489-490)
        const float* x0 = lib.aux_rec + P.aux0 * PULSE_AUX_REC + 4 * j;
        const float* x1 = lib.aux_rec + P.aux1 * PULSE_AUX_REC + 4 * j;
        stv(a.ref_dof_pos + P.env * PULSE_NUM_DOF + 3 * (j - 1), quat_exp_map(slerp(ldq4(x0), ldq4(x1), P.b_obs)));
      }
    }
    // column sums of the partials: thread (kk, c) adds 24 values; fallen flags OR-ed per env
    if (need_t && ttid < kEnvs * kRed) {
      const int kk = ttid / kRed, c = ttid - kk * kRed;
      float sum = 0.0f;
#pragma unroll
      for (int b = 0; b < kNB; ++b) sum += red[kk][c][b];
      red[kk][c][kNB] = sum;
    }
    if (is_fallen) atomicOr(&fallen[k], 1u);
    fence_proxy_async();  // generic-proxy writes of the obs rows -> visible to the bulk (async proxy) store
    team_sync(team);

    // ---- epilogue ---------------------------------------------------------------------------------------------
    if (valid && do_obs) {
      const int width = kTrack ? PULSE_SELF_OBS + (tr.version == 6 ? 24 : 9) * tr.num_track : kObs;   // floats in the row
      const int head = (4 - ophase) & 3;          // floats before the first 16-byte boundary
      const int nmid = ((width - head) / 4) * 4;  // floats in the aligned middle
      const float* o = ophase == 3 ? orow : blk + ophase;
      if (ophase != 3) {
        if (j == 0) {
          bulk_s2g(orow + head, o + head, static_cast<unsigned>(nmid) * 4u);
          bulk_commit();
        } else if (j <= 3) {
          if (j - 1 < head) orow[j - 1] = o[j - 1];
        } else if (j <= 6) {
          const int i = head + nmid + (j - 4);
          if (i < width) orow[i] = o[i];
        }
      }
      if (a.self_obs_buf != nullptr) {
        float* srow = a.self_obs_buf + P.env * PULSE_SELF_OBS;
        for (int i = j; i < PULSE_SELF_OBS; i += kNB) srow[i] = o[i];
      }
    }
    if (ttid < kEnvs && sg.prm[ttid].valid && need_t) {  // lane = env slot: finish reward / reset
      const EnvParams& Q = sg.prm[ttid];
      const long long ee = Q.env;
      const bool pass_time = a.cycle_motion ? (Q.prog >= a.max_episode_length - 1) : (Q.t_rew >= Q.mlen);
      if (do_rew) {
        const float e_pos = red[ttid][0][kNB] * (1.0f / (3.0f * kNB));
        const float e_rot = red[ttid][1][kNB] * (1.0f / kNB);
        const float e_vel = red[ttid][2][kNB] * (1.0f / (3.0f * kNB));
        const float e_ang = red[ttid][3][kNB] * (1.0f / (3.0f * kNB));
        const float r_pos = expf(-a.k_pos * e_pos);
        const float r_rot = expf(-a.k_rot * e_rot);
        const float r_vel = expf(-a.k_vel * e_vel);
        const float r_ang = expf(-a.k_ang_vel * e_ang);
        float rew = a.w_pos * r_pos + a.w_rot * r_rot + a.w_vel * r_vel + a.w_ang_vel * r_ang;
        float p_rew = 0.0f;
        if (do_power) {
          p_rew = (Q.prog <= 3) ? 0.0f : -a.power_coefficient * red[ttid][5][kNB];
          rew += p_rew;
        }
        a.rew_buf[ee] = rew;
        if (a.reward_raw != nullptr) {
          float* rr = a.reward_raw + ee * a.raw_stride;
          rr[0] = r_pos; rr[1] = r_rot; rr[2] = r_vel; rr[3] = r_ang;
          if (do_power) rr[4] = p_rew;
        }
      }
      if (do_reset) {
        bool fell;
        if (a.use_mean_reset) {
          // mean over the reset bodies vs the first reset body's distance (humanoid_im.py:1606)
          const unsigned m = a.reset_body_mask & 0xffffffu;
          fell = (red[ttid][4][kNB] / static_cast<float>(__popc(m))) > a.termination_distances[__ffs(m) - 1];
        } else {
          fell = fallen[ttid] != 0u;
        }
        fell = fell && (Q.prog > 1) && a.enable_early_termination;
        long long terminated = fell ? 1 : 0;
        long long reset = pass_time ? 1 : terminated;
        if (!pass_time && Q.cyc > 0) {  // recovering envs: humanoid_im.py:1188-1190
          reset = 0;
          terminated = 0;
        }
        if (Q.rec) {                    // humanoid_im_getup.py:203-210
          reset = 0;
          terminated = 0;
          a.progress_rw[ee] = Q.prog - 1;
        }
        a.reset_buf[ee] = reset;
        a.terminate_buf[ee] = terminated;
        if (a.fdones_out != nullptr) a.fdones_out[ee] = static_cast<float>(reset);
      }
      if (a.pass_time != nullptr) a.pass_time[ee] = (Q.t_rew >= Q.mlen) ? 1 : 0;
    }
    if (valid && do_obs && j == 0 && ophase != 3) bulk_wait_read();  // the stage's bytes are free once the store has read them
    // No third team barrier: each thread releases the stage when IT is done with it.  red[] columns 0..23,
    // fallen[] and root[] are next written only after this thread passed the second team_sync above, and the
    // column sums / flags are next overwritten only after the next group's first team_sync.
    mbar_arrive(&sm.empty[s]);
  }
}


// Argument checks and launch shared by both entry points; `who` names the entry point in the messages, `width` is the row's float count.
template <bool kTrack>
int im_step_launch(const char* who, const pulse_motionlib_t* lib, const pulse_im_step_args_t& a, const pulse_im_track_t& tr, int width,
                   int64_t num_envs, void* stream) {
  PULSE_REQUIRE(num_envs >= 0, "%s: negative num_envs", who);
  if (num_envs == 0) return PULSE_OK;
  PULSE_REQUIRE(a.env_count == nullptr || a.env_ids != nullptr, "%s: env_count limits an env_ids list", who);
  PULSE_REQUIRE((a.flags & PULSE_STEP_ALL) != 0 && (a.flags & ~(PULSE_STEP_ALL | PULSE_STEP_ADVANCE)) == 0, "%s: bad flags 0x%x", who, a.flags);
  PULSE_REQUIRE(!(a.flags & PULSE_STEP_ADVANCE) || a.progress_rw != nullptr, "%s: PULSE_STEP_ADVANCE needs the writable progress_rw", who);
  PULSE_REQUIRE(a.body_state && a.progress_buf && a.motion_ids && a.motion_start_times && a.motion_start_offset &&
                    a.global_offset, "%s: null state/task buffer", who);
  PULSE_REQUIRE(a.body_env_stride >= PULSE_NUM_BODIES * PULSE_BODY_STATE_W, "%s: body_env_stride %lld < 312", who,
                (long long)a.body_env_stride);
  PULSE_REQUIRE((reinterpret_cast<uintptr_t>(a.body_state) & 3u) == 0, "%s: body_state not 4-byte aligned", who);
  PULSE_REQUIRE(aligned16(lib->d.frame_rec), "%s: frame records not 16-byte aligned", who);
  if (a.flags & PULSE_STEP_REWARD) {
    PULSE_REQUIRE(a.rew_buf != nullptr, "%s: rew_buf is null", who);
    if (a.dof_force) {
      PULSE_REQUIRE(a.dof_vel != nullptr, "%s: dof_force given without dof_vel", who);
      PULSE_REQUIRE(!a.reward_raw || a.raw_stride >= 5, "%s: raw_stride must be >= 5 with the power term", who);
    } else {
      PULSE_REQUIRE(!a.reward_raw || a.raw_stride >= 4, "%s: raw_stride must be >= 4", who);
    }
  }
  if (a.flags & PULSE_STEP_RESET) {
    PULSE_REQUIRE(a.reset_buf && a.terminate_buf && a.termination_distances, "%s: null reset buffer", who);
    PULSE_REQUIRE(a.recovery_counter == nullptr || a.progress_rw != nullptr, "%s: recovery_counter needs the writable progress_rw", who);
    PULSE_REQUIRE((a.reset_body_mask & 0xffffffu) != 0, "%s: empty reset_body_mask", who);
  }
  if (a.flags & PULSE_STEP_OBS) {
    PULSE_REQUIRE(a.obs_buf != nullptr && a.obs_stride >= width, "%s: obs_buf null or obs_stride < %d", who, width);
    PULSE_REQUIRE((reinterpret_cast<uintptr_t>(a.obs_buf) & 3u) == 0, "%s: obs_buf misaligned", who);
    PULSE_REQUIRE(!a.ref_dof_pos || lib->d.aux_rec, "%s: ref_dof_pos needs the aux records", who);
  }
  static bool attr_set = false;
  const size_t smem = sizeof(CtaSmem);
  if (!attr_set) {
    PULSE_CUDA_OK(cudaFuncSetAttribute(im_step_kernel<kTrack>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set = true;
  }
  static int max_ctas = 0;
  if (max_ctas == 0) {
    int dev = 0, sms = 0, per_sm = 0;
    PULSE_CUDA_OK(cudaGetDevice(&dev));
    PULSE_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    PULSE_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, im_step_kernel<kTrack>, kThreads, smem));
    PULSE_REQUIRE(per_sm >= 1, "%s: kernel does not fit on this device (smem %zu B)", who, smem);
    max_ctas = sms * per_sm;  // persistent: one resident wave
  }
  const long long ngroups = (num_envs + kEnvs - 1) / kEnvs;
  const unsigned grid = static_cast<unsigned>(ngroups < max_ctas ? ngroups : max_ctas);
  im_step_kernel<kTrack><<<grid, kThreads, smem, static_cast<cudaStream_t>(stream)>>>(lib->d, a, (long long)num_envs, tr);
  PULSE_LAUNCH_OK("im_step_kernel");
  return PULSE_OK;
}

}  // namespace
}  // namespace pulse

extern "C" int pulse_im_step(const pulse_motionlib_t* lib, const pulse_im_step_args_t* args, int64_t num_envs,
                             void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(lib != nullptr && args != nullptr, "pulse_im_step: null lib/args");
  return im_step_launch<false>("pulse_im_step", lib, *args, pulse_im_track_t{}, kObs, num_envs, stream);
}

extern "C" int pulse_im_track_step(const pulse_motionlib_t* lib, const pulse_im_step_args_t* args, const pulse_im_track_t* track,
                                   int64_t num_envs, void* stream) {
  using namespace pulse;
  const char* who = "pulse_im_track_step";
  PULSE_REQUIRE(lib != nullptr && args != nullptr, "%s: null lib/args", who);
  PULSE_REQUIRE(track != nullptr, "%s: null track", who);
  const pulse_im_track_t& tr = *track;
  PULSE_REQUIRE(tr.num_track >= 1 && tr.num_track <= kNB, "%s: num_track %d outside [1, 24]", who, tr.num_track);
  PULSE_REQUIRE(tr.version == 6 || tr.version == 7, "%s: version %d (the tracked row is built for 6 and 7)", who, tr.version);
  unsigned seen = 0u;
  for (int j = 0; j < kNB; ++j) {
    const int r = tr.rank[j];
    if (r < 0) continue;
    PULSE_REQUIRE(r < tr.num_track && !((seen >> r) & 1u), "%s: rank is not a permutation of 0..num_track-1 (body %d has rank %d)", who, j, r);
    seen |= 1u << r;
  }
  PULSE_REQUIRE(__builtin_popcount(seen) == tr.num_track, "%s: rank is not a permutation of 0..num_track-1 (%d of %d ranks given)", who,
                __builtin_popcount(seen), tr.num_track);
  const int width = PULSE_SELF_OBS + (tr.version == 6 ? 24 : 9) * tr.num_track;
  return im_step_launch<true>(who, lib, *args, tr, width, num_envs, stream);
}
