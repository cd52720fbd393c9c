// MotionLib LOADER on the device (SURVEY 8f-1): the per-clip work MotionLibBase.load_motions does on the host every
// `shape_resampling_interval` epochs (motion_lib_base.py:179-323 -> motion_lib_smpl.py:101-174 -> poselib skeleton3d.py
// :389-462 forward kinematics, :1100-1118 velocity estimation -> motion_lib_base.py:47-70 dof velocities): ~60 ms of Python
// loops per clip in the reference, three streaming kernels here.  Inputs are the on-disk clip arrays as they are
// (float64 global rotations and root translation, convert_amass_isaac.py:127-136) concatenated over clips; outputs are the
// six fp32 tables `pulse_motionlib_create` packs.
//
// Precision follows the reference stage by stage (oracle.pulse_oracle.loader_clip): heading rotation, local rotations and
// the consecutive-frame rotation differences in float64; forward kinematics, linear and dof velocities in float32.
//
// STATUS: parity against the reference's tables is checked by tests/test_gpu_loader.py; not yet timed, and the
// bench still builds its synthetic tables directly.
#include "pulse_common.cuh"
#include "quat_math.cuh"

namespace pulse {
namespace {

constexpr int kJ = PULSE_NUM_BODIES;
constexpr int kRadius = 8;   // scipy gaussian_filter1d(sigma = 2, truncate = 4): radius int(4 * 2 + 0.5)

struct Qd {
  double x, y, z, w;
};
__device__ __forceinline__ Qd qd_mul(Qd a, Qd b) {  // poselib rotation3d.quat_mul (:15-27)
  return {a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
          a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
__device__ __forceinline__ Qd qd_conj(Qd a) { return {-a.x, -a.y, -a.z, a.w}; }
__device__ __forceinline__ Qd qd_normalize(Qd q) {  // quat_normalize (:93-98): w >= 0, unit length
  if (q.w < 0.0) q = {-q.x, -q.y, -q.z, -q.w};
  double n = sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  n = n < 1e-9 ? 1e-9 : n;
  return {q.x / n, q.y / n, q.z / n, q.w / n};
}
__device__ __forceinline__ Qd qd_load(const double* p) { return {p[0], p[1], p[2], p[3]}; }
// heading randomisation (motion_lib_smpl.py:131-140): R_z(h) (x) normalize(q)  (scipy's from_quat normalises its input)
__device__ __forceinline__ Qd qd_heading(Qd q, double sh, double ch) {
  double n = sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  q = {q.x / n, q.y / n, q.z / n, q.w / n};
  return qd_mul(Qd{0.0, 0.0, sh, ch}, q);
}

struct Qf {
  float x, y, z, w;
};
__device__ __forceinline__ Qf qf_mul(Qf a, Qf b) {
  return {a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
          a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
__device__ __forceinline__ Qf qf_normalize(Qf q) {
  if (q.w < 0.0f) q = {-q.x, -q.y, -q.z, -q.w};
  float n = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  n = n < 1e-9f ? 1e-9f : n;
  return {q.x / n, q.y / n, q.z / n, q.w / n};
}
// quat_rotate (:206-211): imaginary part of q (x) (v, 0) (x) conj(q)
__device__ __forceinline__ void qf_rotate(Qf q, float vx, float vy, float vz, float& ox, float& oy, float& oz) {
  const Qf t = qf_mul(qf_mul(q, Qf{vx, vy, vz, 0.0f}), Qf{-q.x, -q.y, -q.z, q.w});
  ox = t.x; oy = t.y; oz = t.z;
}

// ---- pass 1: one thread per frame -- global rotations after the heading step, local rotations, forward kinematics ----------
__global__ void __launch_bounds__(128) loader_pose_kernel(const pulse_loader_args_t a) {
  const long long f = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (f >= a.total_frames) return;
  const int clip = a.frame_clip[f];
  double sh = 0.0, ch = 1.0;
  if (a.headings != nullptr) sincos(0.5 * a.headings[clip], &sh, &ch);
  Qd g[kJ];
  Qf rot_fk[kJ];
  float px[kJ], py[kJ], pz[kJ];
#pragma unroll 1
  for (int j = 0; j < kJ; ++j) {
    g[j] = qd_load(a.pose_quat_global + (f * kJ + j) * 4);
    if (a.headings != nullptr) g[j] = qd_heading(g[j], sh, ch);
    float* gr = a.grs + (f * kJ + j) * 4;
    gr[0] = static_cast<float>(g[j].x); gr[1] = static_cast<float>(g[j].y); gr[2] = static_cast<float>(g[j].z); gr[3] = static_cast<float>(g[j].w);
    const int p = a.parents[j];
    // local rotation in float64, kept in float32 (skeleton3d.py:444-462 assigns into a float32 identity tensor)
    const Qd l = p < 0 ? g[j] : qd_normalize(qd_mul(qd_conj(g[p]), g[j]));
    const Qf lf = {static_cast<float>(l.x), static_cast<float>(l.y), static_cast<float>(l.z), static_cast<float>(l.w)};
    float* lr = a.lrs + (f * kJ + j) * 4;
    lr[0] = lf.x; lr[1] = lf.y; lr[2] = lf.z; lr[3] = lf.w;
    // forward kinematics in float32 (:389-407)
    if (p < 0) {
      rot_fk[j] = lf;
      double tx = a.root_trans[f * 3 + 0], ty = a.root_trans[f * 3 + 1];
      const double tz = a.root_trans[f * 3 + 2];
      if (a.headings != nullptr) {  // trans @ R^T with R = R_z(h): cos h = ch^2 - sh^2, sin h = 2 sh ch
        const double c = ch * ch - sh * sh, s = 2.0 * sh * ch;
        const double nx = c * tx - s * ty, ny = s * tx + c * ty;
        tx = nx; ty = ny;
      }
      px[j] = static_cast<float>(tx); py[j] = static_cast<float>(ty); pz[j] = static_cast<float>(tz);
    } else {
      rot_fk[j] = qf_normalize(qf_mul(rot_fk[p], lf));
      float ox, oy, oz;
      qf_rotate(rot_fk[p], a.local_translation[j * 3 + 0], a.local_translation[j * 3 + 1], a.local_translation[j * 3 + 2], ox, oy, oz);
      px[j] = ox + px[p]; py[j] = oy + py[p]; pz[j] = oz + pz[p];
    }
    float* gt = a.gts + (f * kJ + j) * 3;
    gt[0] = px[j]; gt[1] = py[j]; gt[2] = pz[j];
  }
}

// ---- pass 2: one thread per (frame, joint) -- raw finite-difference velocities and the dof velocities -------------------
__global__ void __launch_bounds__(256) loader_velocity_kernel(const pulse_loader_args_t a) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= a.total_frames * kJ) return;
  const long long f = i / kJ;
  const int j = static_cast<int>(i - f * kJ);
  const int clip = a.frame_clip[f];
  const long long f0 = a.clip_start[clip], f1 = a.clip_start[clip + 1];   // [f0, f1)
  const float fps = a.fps[clip];
  const double dt = 1.0 / static_cast<double>(fps);
  // np.gradient along time (:1101): one-sided at the ends, central inside
  const long long fa = f > f0 ? f - 1 : f, fb = f + 1 < f1 ? f + 1 : f;
  const float inv = 1.0f / static_cast<float>(static_cast<double>(fb - fa) * dt);
#pragma unroll
  for (int c = 0; c < 3; ++c)
    a.tmp_vel[i * 3 + c] = fb > fa ? (a.gts[(fb * kJ + j) * 3 + c] - a.gts[(fa * kJ + j) * 3 + c]) * inv : 0.0f;
  // angular velocity from consecutive GLOBAL rotations in float64 (:1110-1115); the last frame of a clip gets the identity
  float wx = 0.0f, wy = 0.0f, wz = 0.0f;
  if (f + 1 < f1) {
    double sh = 0.0, ch = 1.0;
    if (a.headings != nullptr) sincos(0.5 * a.headings[clip], &sh, &ch);
    Qd q0 = qd_load(a.pose_quat_global + (f * kJ + j) * 4), q1 = qd_load(a.pose_quat_global + ((f + 1) * kJ + j) * 4);
    if (a.headings != nullptr) {
      q0 = qd_heading(q0, sh, ch);
      q1 = qd_heading(q1, sh, ch);
    }
    const Qd d = qd_normalize(qd_mul(q1, qd_conj(q0)));
    double s = 2.0 * d.w * d.w - 1.0;
    s = s < -1.0 ? -1.0 : (s > 1.0 ? 1.0 : s);
    const double angle = acos(s);
    double n = sqrt(d.x * d.x + d.y * d.y + d.z * d.z);
    n = n < 1e-9 ? 1e-9 : n;
    const double k = angle / (n * dt);
    wx = static_cast<float>(d.x * k); wy = static_cast<float>(d.y * k); wz = static_cast<float>(d.z * k);
  }
  a.tmp_ang[i * 3 + 0] = wx; a.tmp_ang[i * 3 + 1] = wy; a.tmp_ang[i * 3 + 2] = wz;
  // dof velocity of joints 1..23 from consecutive LOCAL rotations in float32 (motion_lib_base.py:47-70), last frame repeats
  if (j >= 1) {
    long long fs = f + 1 < f1 ? f : f - 1;   // the pair (fs, fs + 1)
    float ox = 0.0f, oy = 0.0f, oz = 0.0f;
    if (fs >= f0 && fs + 1 < f1) {
      const float* l0 = a.lrs + (fs * kJ + j) * 4;
      const float* l1 = a.lrs + ((fs + 1) * kJ + j) * 4;
      const Quat d = qmul(qconj(Quat{l0[0], l0[1], l0[2], l0[3]}), Quat{l1[0], l1[1], l1[2], l1[3]});
      const Vec3 e = quat_exp_map(d);   // angle * axis (torch_utils.quat_to_angle_axis semantics)
      const float r = static_cast<float>(1.0 / dt);
      ox = e.x * r; oy = e.y * r; oz = e.z * r;
    }
    float* dv = a.dvs + (f * (kJ - 1) + (j - 1)) * 3;
    dv[0] = ox; dv[1] = oy; dv[2] = oz;
  }
}

// ---- pass 3: sigma = 2 gaussian along time inside each clip, `nearest` boundary (:1103, :1117) ------------------------------
__global__ void __launch_bounds__(256) loader_filter_kernel(const pulse_loader_args_t a) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= a.total_frames * kJ) return;
  const long long f = i / kJ;
  const int j = static_cast<int>(i - f * kJ);
  const int clip = a.frame_clip[f];
  const long long f0 = a.clip_start[clip], f1 = a.clip_start[clip + 1];
  float w[kRadius + 1];
  float wsum = 0.0f;
#pragma unroll
  for (int k = 0; k <= kRadius; ++k) {
    w[k] = expf(-0.5f * static_cast<float>(k * k) / 4.0f);
    wsum += k == 0 ? w[k] : 2.0f * w[k];
  }
  float v[3] = {0.0f, 0.0f, 0.0f}, o[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll 1
  for (int k = -kRadius; k <= kRadius; ++k) {
    long long t = f + k;
    t = t < f0 ? f0 : (t >= f1 ? f1 - 1 : t);
    const float wk = w[k < 0 ? -k : k] / wsum;
    const long long r = (t * kJ + j) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      v[c] = fmaf(wk, a.tmp_vel[r + c], v[c]);
      o[c] = fmaf(wk, a.tmp_ang[r + c], o[c]);
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    a.gvs[i * 3 + c] = v[c];
    a.gavs[i * 3 + c] = o[c];
  }
}

}  // namespace
}  // namespace pulse

using namespace pulse;

extern "C" int pulse_motionlib_load_clips(const pulse_loader_args_t* args, void* stream) {
  PULSE_REQUIRE(args, "pulse_motionlib_load_clips: null args");
  const pulse_loader_args_t& a = *args;
  PULSE_REQUIRE(a.pose_quat_global && a.root_trans && a.frame_clip && a.clip_start && a.fps && a.parents && a.local_translation,
                "pulse_motionlib_load_clips: null input");
  PULSE_REQUIRE(a.gts && a.grs && a.lrs && a.gvs && a.gavs && a.dvs && a.tmp_vel && a.tmp_ang, "pulse_motionlib_load_clips: null output / workspace");
  PULSE_REQUIRE(a.total_frames > 0 && a.num_clips > 0, "pulse_motionlib_load_clips: empty input");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long fj = a.total_frames * kJ;
  loader_pose_kernel<<<static_cast<unsigned>((a.total_frames + 127) / 128), 128, 0, st>>>(a);
  PULSE_LAUNCH_OK("loader_pose_kernel");
  loader_velocity_kernel<<<static_cast<unsigned>((fj + 255) / 256), 256, 0, st>>>(a);
  PULSE_LAUNCH_OK("loader_velocity_kernel");
  loader_filter_kernel<<<static_cast<unsigned>((fj + 255) / 256), 256, 0, st>>>(a);
  PULSE_LAUNCH_OK("loader_filter_kernel");
  return PULSE_OK;
}
