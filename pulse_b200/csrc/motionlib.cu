// MotionLib tables on the device: packing into per-frame records, and the general
// get_motion_state query (motion_lib_base.py:434-517) used by the reset path and AMP demo sampling.
#include <stdarg.h>
#include <stdlib.h>

#include <atomic>

#include "pulse_common.cuh"
#include "quat_math.cuh"

namespace pulse {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

namespace {

// One thread per (frame, float4 chunk) of the two packed records.
__global__ void pack_tables_kernel(pulse_motionlib_desc_t d) {
  const long long total = d.total_frames * (PULSE_FRAME_REC + PULSE_AUX_REC);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long f = i / (PULSE_FRAME_REC + PULSE_AUX_REC);
    const int c = static_cast<int>(i - f * (PULSE_FRAME_REC + PULSE_AUX_REC));
    if (c < PULSE_FRAME_REC) {
      float v;
      if (c < 72) v = d.gts[f * 72 + c];
      else if (c < 168) v = d.grs[f * 96 + (c - 72)];
      else if (c < 240) v = d.gvs[f * 72 + (c - 168)];
      else v = d.gavs[f * 72 + (c - 240)];
      d.frame_rec[f * PULSE_FRAME_REC + c] = v;
    } else if (d.aux_rec != nullptr) {
      const int k = c - PULSE_FRAME_REC;
      float v = 0.0f;
      if (k < 96) v = d.lrs[f * 96 + k];
      else if (k < 165) v = d.dvs[f * 69 + (k - 96)];
      else if (k < 237) v = d.motion_aa ? d.motion_aa[f * 72 + (k - 165)] : 0.0f;
      d.aux_rec[f * PULSE_AUX_REC + k] = v;
    }
  }
}

// One warp per query, lane j = body j.  Everything is read straight from the packed records (L2).
__global__ void __launch_bounds__(128) motion_state_kernel(const pulse_motionlib_desc_t lib, const pulse_motion_query_t q,
                                                           long long n) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  const long long mid = q.motion_ids[i];
  const float t = q.motion_times[i];
  long long i0, i1;
  float b;
  frame_blend_rn(t, lib.lengths[mid], lib.num_frames[mid], lib.dt[mid], i0, i1, b);
  const long long f0 = i0 + lib.length_starts[mid];
  const long long f1 = i1 + lib.length_starts[mid];
  if (lane == 0) {
    if (q.frame_idx0) q.frame_idx0[i] = i0;
    if (q.frame_idx1) q.frame_idx1[i] = i1;
    if (q.blend) q.blend[i] = b;
  }
  const float* r0 = lib.frame_rec + f0 * PULSE_FRAME_REC;
  const float* r1 = lib.frame_rec + f1 * PULSE_FRAME_REC;
  Vec3 off = {0.f, 0.f, 0.f};
  if (q.offset) off = {q.offset[3 * i], q.offset[3 * i + 1], q.offset[3 * i + 2]};
  if (lane < PULSE_NUM_BODIES) {
    const int j = lane;
    Vec3 p;
    p.x = lerp_rn(r0[3 * j], r1[3 * j], b);
    p.y = lerp_rn(r0[3 * j + 1], r1[3 * j + 1], b);
    p.z = lerp_rn(r0[3 * j + 2], r1[3 * j + 2], b);
    if (q.offset) p = {__fadd_rn(p.x, off.x), __fadd_rn(p.y, off.y), __fadd_rn(p.z, off.z)};
    Vec3 v, w;
    v.x = lerp_rn(r0[168 + 3 * j], r1[168 + 3 * j], b);
    v.y = lerp_rn(r0[169 + 3 * j], r1[169 + 3 * j], b);
    v.z = lerp_rn(r0[170 + 3 * j], r1[170 + 3 * j], b);
    w.x = lerp_rn(r0[240 + 3 * j], r1[240 + 3 * j], b);
    w.y = lerp_rn(r0[241 + 3 * j], r1[241 + 3 * j], b);
    w.z = lerp_rn(r0[242 + 3 * j], r1[242 + 3 * j], b);
    const Quat rq = slerp(ldq4(r0 + 72 + 4 * j), ldq4(r1 + 72 + 4 * j), b);
    if (q.rg_pos) { float* d = q.rg_pos + i * 72 + 3 * j; d[0] = p.x; d[1] = p.y; d[2] = p.z; }
    if (q.body_vel) { float* d = q.body_vel + i * 72 + 3 * j; d[0] = v.x; d[1] = v.y; d[2] = v.z; }
    if (q.body_ang_vel) { float* d = q.body_ang_vel + i * 72 + 3 * j; d[0] = w.x; d[1] = w.y; d[2] = w.z; }
    if (q.rb_rot) { float* d = q.rb_rot + i * 96 + 4 * j; d[0] = rq.x; d[1] = rq.y; d[2] = rq.z; d[3] = rq.w; }
    if (j == 0) {
      if (q.root_pos) { q.root_pos[3 * i] = p.x; q.root_pos[3 * i + 1] = p.y; q.root_pos[3 * i + 2] = p.z; }
      if (q.root_vel) { q.root_vel[3 * i] = v.x; q.root_vel[3 * i + 1] = v.y; q.root_vel[3 * i + 2] = v.z; }
      if (q.root_ang_vel) { q.root_ang_vel[3 * i] = w.x; q.root_ang_vel[3 * i + 1] = w.y; q.root_ang_vel[3 * i + 2] = w.z; }
      if (q.root_rot) { float* d = q.root_rot + 4 * i; d[0] = rq.x; d[1] = rq.y; d[2] = rq.z; d[3] = rq.w; }
    }
  }
  if (lib.aux_rec != nullptr && (q.dof_pos || q.dof_vel || q.motion_aa)) {
    const float* x0 = lib.aux_rec + f0 * PULSE_AUX_REC;
    const float* x1 = lib.aux_rec + f1 * PULSE_AUX_REC;
    if (q.dof_pos && lane >= 1 && lane < PULSE_NUM_BODIES) {
      Vec3 em = quat_exp_map(slerp(ldq4(x0 + 4 * lane), ldq4(x1 + 4 * lane), b));
      float* d = q.dof_pos + i * PULSE_NUM_DOF + 3 * (lane - 1);
      d[0] = em.x; d[1] = em.y; d[2] = em.z;
    }
    if (q.dof_vel) {
      for (int k = lane; k < PULSE_NUM_DOF; k += 32) q.dof_vel[i * PULSE_NUM_DOF + k] = lerp_rn(x0[96 + k], x1[96 + k], b);
    }
    if (q.motion_aa) {
      for (int k = lane; k < 72; k += 32) q.motion_aa[i * 72 + k] = x0[165 + k];
    }
  }
}

// The SMPL-X records: one thread per (frame, float) of the frame record and the aux record (pad floats zero).
__global__ void smplx_pack_kernel(pulse_smplx_motionlib_desc_t d) {
  constexpr int B = PULSE_SMPLX_BODIES, FR = PULSE_SMPLX_FRAME_REC, AR = PULSE_SMPLX_AUX_REC;
  const long long total = d.total_frames * (FR + AR);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long f = i / (FR + AR);
    const int c = static_cast<int>(i - f * (FR + AR));
    if (c < FR) {
      float v;
      if (c < 3 * B) v = d.gts[f * 3 * B + c];
      else if (c < 7 * B) v = d.grs[f * 4 * B + (c - 3 * B)];
      else if (c < 10 * B) v = d.gvs[f * 3 * B + (c - 7 * B)];
      else v = d.gavs[f * 3 * B + (c - 10 * B)];
      d.frame_rec[f * FR + c] = v;
    } else {
      const int k = c - FR;
      float v = 0.0f;
      if (k < 4 * B) v = d.lrs[f * 4 * B + k];
      else if (k < 4 * B + PULSE_SMPLX_DOF) v = d.dvs[f * PULSE_SMPLX_DOF + (k - 4 * B)];
      d.aux_rec[f * AR + k] = v;
    }
  }
}

// get_motion_state over the SMPL-X records: motion_state_kernel's arithmetic, one warp per query, lane l = bodies l and l + 32.
__global__ void __launch_bounds__(128) smplx_motion_state_kernel(const pulse_smplx_motionlib_desc_t lib, const pulse_smplx_motion_query_t q,
                                                                 long long n) {
  constexpr int B = PULSE_SMPLX_BODIES;
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  const long long mid = q.motion_ids[i];
  long long i0, i1;
  float b;
  frame_blend_rn(q.motion_times[i], lib.lengths[mid], lib.num_frames[mid], lib.dt[mid], i0, i1, b);
  const long long f0 = i0 + lib.length_starts[mid], f1 = i1 + lib.length_starts[mid];
  const float* r0 = lib.frame_rec + f0 * PULSE_SMPLX_FRAME_REC;
  const float* r1 = lib.frame_rec + f1 * PULSE_SMPLX_FRAME_REC;
  const float* x0 = lib.aux_rec + f0 * PULSE_SMPLX_AUX_REC;
  const float* x1 = lib.aux_rec + f1 * PULSE_SMPLX_AUX_REC;
  const auto blend3 = [&](int o) { return Vec3{lerp_rn(r0[o], r1[o], b), lerp_rn(r0[o + 1], r1[o + 1], b), lerp_rn(r0[o + 2], r1[o + 2], b)}; };
  for (int j = lane; j < B; j += 32) {
    Vec3 p = blend3(3 * j);
    if (q.offset) p = {__fadd_rn(p.x, q.offset[3 * i]), __fadd_rn(p.y, q.offset[3 * i + 1]), __fadd_rn(p.z, q.offset[3 * i + 2])};
    const Vec3 v = blend3(7 * B + 3 * j), w = blend3(10 * B + 3 * j);
    const Quat rq = slerp(ldq4(r0 + 3 * B + 4 * j), ldq4(r1 + 3 * B + 4 * j), b);
    if (q.rg_pos) stv(q.rg_pos + (i * B + j) * 3, p);
    if (q.body_vel) stv(q.body_vel + (i * B + j) * 3, v);
    if (q.body_ang_vel) stv(q.body_ang_vel + (i * B + j) * 3, w);
    if (q.rb_rot) { float* d = q.rb_rot + (i * B + j) * 4; d[0] = rq.x; d[1] = rq.y; d[2] = rq.z; d[3] = rq.w; }
    if (j == 0) {
      if (q.root_pos) stv(q.root_pos + 3 * i, p);
      if (q.root_vel) stv(q.root_vel + 3 * i, v);
      if (q.root_ang_vel) stv(q.root_ang_vel + 3 * i, w);
      if (q.root_rot) { float* d = q.root_rot + 4 * i; d[0] = rq.x; d[1] = rq.y; d[2] = rq.z; d[3] = rq.w; }
    } else if (q.dof_pos) {
      stv(q.dof_pos + i * PULSE_SMPLX_DOF + 3 * (j - 1), quat_exp_map(slerp(ldq4(x0 + 4 * j), ldq4(x1 + 4 * j), b)));
    }
  }
  if (q.dof_vel)
    for (int k = lane; k < PULSE_SMPLX_DOF; k += 32) q.dof_vel[i * PULSE_SMPLX_DOF + k] = lerp_rn(x0[4 * B + k], x1[4 * B + k], b);
}

}  // namespace
}  // namespace pulse

extern "C" int pulse_abi_version(void) { return PULSE_ABI_VERSION; }
extern "C" const char* pulse_last_error(void) { return pulse::g_err; }
extern "C" int64_t pulse_launch_count(void) { return pulse::g_launches.load(); }

extern "C" int pulse_motionlib_create(const pulse_motionlib_desc_t* desc, void* stream, pulse_motionlib_t** out) {
  using namespace pulse;
  PULSE_REQUIRE(desc != nullptr && out != nullptr, "pulse_motionlib_create: null argument");
  const pulse_motionlib_desc_t& d = *desc;
  PULSE_REQUIRE(d.gts && d.grs && d.gvs && d.gavs && d.lengths && d.dt && d.num_frames && d.length_starts,
                "pulse_motionlib_create: null table pointer");
  PULSE_REQUIRE(d.total_frames > 0 && d.num_motions > 0, "pulse_motionlib_create: empty tables (F=%lld, M=%lld)",
                (long long)d.total_frames, (long long)d.num_motions);
  PULSE_REQUIRE(d.frame_rec != nullptr && aligned16(d.frame_rec), "pulse_motionlib_create: frame_rec null or not 16-byte aligned");
  PULSE_REQUIRE(d.aux_rec == nullptr || (aligned16(d.aux_rec) && d.lrs && d.dvs),
                "pulse_motionlib_create: aux_rec needs 16-byte alignment and the lrs/dvs tables");
  const long long total = d.total_frames * (PULSE_FRAME_REC + PULSE_AUX_REC);
  pack_tables_kernel<<<grid_for(total, 256, 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(d);
  PULSE_LAUNCH_OK("pack_tables_kernel");
  pulse_motionlib* h = static_cast<pulse_motionlib*>(malloc(sizeof(pulse_motionlib)));
  PULSE_REQUIRE(h != nullptr, "pulse_motionlib_create: host allocation failed");
  h->d = d;
  *out = h;
  return PULSE_OK;
}

extern "C" int pulse_motionlib_destroy(pulse_motionlib_t* lib) {
  if (lib) free(lib);
  return PULSE_OK;
}

extern "C" int pulse_motion_state(const pulse_motionlib_t* lib, const pulse_motion_query_t* q, int64_t n, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(lib != nullptr && q != nullptr, "pulse_motion_state: null lib/query");
  PULSE_REQUIRE(n >= 0, "pulse_motion_state: negative n");
  if (n == 0) return PULSE_OK;
  PULSE_REQUIRE(q->motion_ids && q->motion_times, "pulse_motion_state: null ids/times");
  PULSE_REQUIRE(lib->d.aux_rec || !(q->dof_pos || q->dof_vel || q->motion_aa),
                "pulse_motion_state: dof_pos/dof_vel/motion_aa need the aux records");
  const long long threads = n * 32;
  const unsigned grid = static_cast<unsigned>((threads + 127) / 128);
  motion_state_kernel<<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(lib->d, *q, (long long)n);
  PULSE_LAUNCH_OK("motion_state_kernel");
  return PULSE_OK;
}

extern "C" int pulse_smplx_motionlib_create(const pulse_smplx_motionlib_desc_t* desc, void* stream, pulse_smplx_motionlib_t** out) {
  using namespace pulse;
  PULSE_REQUIRE(desc != nullptr && out != nullptr, "pulse_smplx_motionlib_create: null argument");
  const pulse_smplx_motionlib_desc_t& d = *desc;
  PULSE_REQUIRE(d.gts && d.grs && d.lrs && d.gvs && d.gavs && d.dvs && d.lengths && d.dt && d.num_frames && d.length_starts,
                "pulse_smplx_motionlib_create: null table pointer");
  PULSE_REQUIRE(d.total_frames > 0 && d.num_motions > 0, "pulse_smplx_motionlib_create: empty tables (F=%lld, M=%lld)",
                (long long)d.total_frames, (long long)d.num_motions);
  PULSE_REQUIRE(d.frame_rec != nullptr && aligned16(d.frame_rec) && d.aux_rec != nullptr && aligned16(d.aux_rec),
                "pulse_smplx_motionlib_create: frame_rec / aux_rec null or not 16-byte aligned");
  const long long total = d.total_frames * (PULSE_SMPLX_FRAME_REC + PULSE_SMPLX_AUX_REC);
  smplx_pack_kernel<<<grid_for(total, 256, 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(d);
  PULSE_LAUNCH_OK("smplx_pack_kernel");
  pulse_smplx_motionlib* h = static_cast<pulse_smplx_motionlib*>(malloc(sizeof(pulse_smplx_motionlib)));
  PULSE_REQUIRE(h != nullptr, "pulse_smplx_motionlib_create: host allocation failed");
  h->d = d;
  *out = h;
  return PULSE_OK;
}

extern "C" int pulse_smplx_motionlib_destroy(pulse_smplx_motionlib_t* lib) {
  if (lib) free(lib);
  return PULSE_OK;
}

extern "C" int pulse_smplx_motion_state(const pulse_smplx_motionlib_t* lib, const pulse_smplx_motion_query_t* q, int64_t n, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(lib != nullptr && q != nullptr, "pulse_smplx_motion_state: null lib/query");
  PULSE_REQUIRE(n >= 0, "pulse_smplx_motion_state: negative n");
  if (n == 0) return PULSE_OK;
  PULSE_REQUIRE(q->motion_ids && q->motion_times, "pulse_smplx_motion_state: null ids/times");
  smplx_motion_state_kernel<<<static_cast<unsigned>((n * 32 + 127) / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(lib->d, *q, (long long)n);
  PULSE_LAUNCH_OK("smplx_motion_state_kernel");
  return PULSE_OK;
}
