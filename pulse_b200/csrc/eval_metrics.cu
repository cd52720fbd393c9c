// Evaluation metrics on the device (SURVEY 8f-2): one launch pair per evaluation step replaces the reference's per-step host work --
// `.cpu().numpy()` copies of all body positions, Python lists of frames, and compute_metrics_lite over them at the end
// (phc/learning/im_amp.py:244-363, humanoid_im.py:664-673, smpl_sim compute_metrics_lite [3P-memory]).
//
//   eval_accumulate_kernel  one warp per env, lane = body: termination state (im_amp.py:249-251), and for every COUNTED frame
//                           (frame s of a sequence with n steps counts iff s < n - 1, the reference's `[:(n - 1)]` slices, and the chunk
//                           has not ended) the per-frame global / root-relative / Procrustes-aligned MPJPE and the velocity /
//                           acceleration errors, added to per-env fp64 sums.  Procrustes: Horn's quaternion form -- the largest
//                           eigenpair of a 4x4 symmetric matrix (cyclic Jacobi) gives the optimal proper rotation and the trace term at
//                           once; equal to the SVD form with the determinant sign fix.
//   eval_advance_kernel     one thread: the reference's `curr_max` stopping rule (im_amp.py:252-268, :275) incl. the wrapped last
//                           chunk, step counter, `finished` flag -- the host polls the flag instead of synchronising every step.
#include "pulse_common.cuh"

namespace pulse {
namespace {

constexpr int kEvalBodies = PULSE_NUM_BODIES;

// Largest eigenvalue / eigenvector of a symmetric 4x4 matrix by cyclic Jacobi rotations (every lane runs the same scalars).
__device__ __forceinline__ void jacobi4_max(float A[4][4], float q[4], float& lambda) {
  float V[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
#pragma unroll 1
  for (int sweep = 0; sweep < 10; ++sweep) {
    float off = 0.0f;
#pragma unroll
    for (int p = 0; p < 3; ++p)
#pragma unroll
      for (int r = p + 1; r < 4; ++r) off += A[p][r] * A[p][r];
    if (off < 1e-30f) break;
#pragma unroll
    for (int p = 0; p < 3; ++p) {
#pragma unroll
      for (int r = p + 1; r < 4; ++r) {
        const float apq = A[p][r];
        if (fabsf(apq) < 1e-30f) continue;
        const float theta = (A[r][r] - A[p][p]) / (2.0f * apq);
        const float t = copysignf(1.0f, theta) / (fabsf(theta) + sqrtf(theta * theta + 1.0f));
        const float c = rsqrtf(t * t + 1.0f), s = t * c;
#pragma unroll
        for (int k = 0; k < 4; ++k) {   // A <- A J (columns p, r)
          const float akp = A[k][p], akr = A[k][r];
          A[k][p] = c * akp - s * akr;
          A[k][r] = s * akp + c * akr;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {   // A <- J^T A (rows p, r)
          const float apk = A[p][k], ark = A[r][k];
          A[p][k] = c * apk - s * ark;
          A[r][k] = s * apk + c * ark;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float vkp = V[k][p], vkr = V[k][r];
          V[k][p] = c * vkp - s * vkr;
          V[k][r] = s * vkp + c * vkr;
        }
      }
    }
  }
  int best = 0;
  lambda = A[0][0];
#pragma unroll
  for (int k = 1; k < 4; ++k)
    if (A[k][k] > lambda) { lambda = A[k][k]; best = k; }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float v = V[k][0];
    if (best == 1) v = V[k][1];
    if (best == 2) v = V[k][2];
    if (best == 3) v = V[k][3];
    q[k] = v;
  }
}

__global__ void __launch_bounds__(128) eval_accumulate_kernel(const pulse_eval_args_t a) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= a.num_envs) return;
  const int e = warp;
  const int step = a.ctrl[0];
  if (a.ctrl[1] != 0) return;                                  // the chunk has ended: later launches are no-ops until the host starts the next
  const int nsteps = a.num_steps[e];
  int term = a.terminate_state[e];
  if (step <= nsteps - 1 && a.terminate[e] != 0) term = 1;      // im_amp.py:249-251
  const bool body = lane < kEvalBodies;
  float px = 0, py = 0, pz = 0, gx = 0, gy = 0, gz = 0;
  if (body) {
    const float* p = a.body_pos + (long long)e * a.pos_env_stride + (long long)lane * a.pos_body_stride;
    const float* g = a.body_pos_gt + (long long)e * a.gt_env_stride + (long long)lane * a.gt_body_stride;
    px = p[0]; py = p[1]; pz = p[2];
    gx = g[0]; gy = g[1]; gz = g[2];
  }
  const float dx = px - gx, dy = py - gy, dz = pz - gz;
  const float inv_j = 1.0f / kEvalBodies;
  const float mg = warp_sum(body ? sqrtf(dx * dx + dy * dy + dz * dz) : 0.0f) * inv_j;     // extras['mpjpe'] (humanoid_im.py:671)
  if (a.mpjpe_out != nullptr && lane == 0) a.mpjpe_out[e] = mg;
  // history of (pred - gt): velocity / acceleration errors are finite differences of it
  float* h = a.hist + (long long)e * (2 * kEvalBodies * 3);
  float d1x = 0, d1y = 0, d1z = 0, d2x = 0, d2y = 0, d2z = 0;
  if (body) {
    d1x = h[lane * 3 + 0]; d1y = h[lane * 3 + 1]; d1z = h[lane * 3 + 2];
    d2x = h[(kEvalBodies + lane) * 3 + 0]; d2y = h[(kEvalBodies + lane) * 3 + 1]; d2z = h[(kEvalBodies + lane) * 3 + 2];
    h[(kEvalBodies + lane) * 3 + 0] = d1x; h[(kEvalBodies + lane) * 3 + 1] = d1y; h[(kEvalBodies + lane) * 3 + 2] = d1z;
    h[lane * 3 + 0] = dx; h[lane * 3 + 1] = dy; h[lane * 3 + 2] = dz;
  }
  if (step < nsteps - 1) {   // a counted frame of this sequence
    // root-relative
    const float prx = __shfl_sync(kFull, px, 0), pry = __shfl_sync(kFull, py, 0), prz = __shfl_sync(kFull, pz, 0);
    const float grx = __shfl_sync(kFull, gx, 0), gry = __shfl_sync(kFull, gy, 0), grz = __shfl_sync(kFull, gz, 0);
    const float yx = px - prx, yy = py - pry, yz = pz - prz;   // predicted, root-relative
    const float xx = gx - grx, xy = gy - gry, xz = gz - grz;   // target, root-relative
    const float lx = yx - xx, ly = yy - xy, lz = yz - xz;
    const float ml = warp_sum(body ? sqrtf(lx * lx + ly * ly + lz * lz) : 0.0f) * inv_j;
    // Procrustes alignment of the root-relative sets
    const float mxx = warp_sum(body ? xx : 0.0f) * inv_j, mxy = warp_sum(body ? xy : 0.0f) * inv_j, mxz = warp_sum(body ? xz : 0.0f) * inv_j;
    const float myx = warp_sum(body ? yx : 0.0f) * inv_j, myy = warp_sum(body ? yy : 0.0f) * inv_j, myz = warp_sum(body ? yz : 0.0f) * inv_j;
    const float X[3] = {body ? xx - mxx : 0.0f, body ? xy - mxy : 0.0f, body ? xz - mxz : 0.0f};
    const float Y[3] = {body ? yx - myx : 0.0f, body ? yy - myy : 0.0f, body ? yz - myz : 0.0f};
    const float ny2 = warp_sum(Y[0] * Y[0] + Y[1] * Y[1] + Y[2] * Y[2]);
    float S[3][3];   // S[a][b] = sum_j Y_a X_b: the correlation of Horn's method for the rotation taking Y onto X
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) S[r][c] = warp_sum(Y[r] * X[c]);
    float Nm[4][4];
    Nm[0][0] = S[0][0] + S[1][1] + S[2][2];
    Nm[1][1] = S[0][0] - S[1][1] - S[2][2];
    Nm[2][2] = -S[0][0] + S[1][1] - S[2][2];
    Nm[3][3] = -S[0][0] - S[1][1] + S[2][2];
    Nm[0][1] = Nm[1][0] = S[1][2] - S[2][1];
    Nm[0][2] = Nm[2][0] = S[2][0] - S[0][2];
    Nm[0][3] = Nm[3][0] = S[0][1] - S[1][0];
    Nm[1][2] = Nm[2][1] = S[0][1] + S[1][0];
    Nm[1][3] = Nm[3][1] = S[2][0] + S[0][2];
    Nm[2][3] = Nm[3][2] = S[1][2] + S[2][1];
    float q[4], lam;
    jacobi4_max(Nm, q, lam);
    const float qn = rsqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const float w = q[0] * qn, x = q[1] * qn, y = q[2] * qn, z = q[3] * qn;
    const float scale = lam / ny2;   // tr * normX / normY of the normalised form = lambda_max(raw) / |Y0|^2
    // Q(q) applied to Y
    const float r00 = 1 - 2 * (y * y + z * z), r01 = 2 * (x * y - w * z), r02 = 2 * (x * z + w * y);
    const float r10 = 2 * (x * y + w * z), r11 = 1 - 2 * (x * x + z * z), r12 = 2 * (y * z - w * x);
    const float r20 = 2 * (x * z - w * y), r21 = 2 * (y * z + w * x), r22 = 1 - 2 * (x * x + y * y);
    const float ax = scale * (r00 * Y[0] + r01 * Y[1] + r02 * Y[2]) - X[0];
    const float ay = scale * (r10 * Y[0] + r11 * Y[1] + r12 * Y[2]) - X[1];
    const float az = scale * (r20 * Y[0] + r21 * Y[1] + r22 * Y[2]) - X[2];
    const float mpa = warp_sum(body ? sqrtf(ax * ax + ay * ay + az * az) : 0.0f) * inv_j;
    const float vx = dx - d1x, vy = dy - d1y, vz = dz - d1z;
    const float mv = warp_sum(body ? sqrtf(vx * vx + vy * vy + vz * vz) : 0.0f) * inv_j;
    const float cx = dx - 2.0f * d1x + d2x, cy = dy - 2.0f * d1y + d2y, cz = dz - 2.0f * d1z + d2z;
    const float ma = warp_sum(body ? sqrtf(cx * cx + cy * cy + cz * cz) : 0.0f) * inv_j;
    if (lane == 0) {
      double* s = a.sums + (long long)e * 5;
      int* c = a.counts + (long long)e * 3;
      s[0] += mg; s[1] += ml; s[2] += mpa;
      c[0] += 1;
      if (step >= 1) { s[3] += mv; c[1] += 1; }
      if (step >= 2) { s[4] += ma; c[2] += 1; }
    }
  }
  if (lane == 0) {
    a.terminate_state[e] = term;
    if (!term) {
      atomicAdd(&a.ctrl[3], 1);                                   // envs still running
      if (e < a.bound) {
        atomicAdd(&a.ctrl[4], 1);
        atomicMax(&a.ctrl[2], nsteps);                            // longest sequence still running
      }
    }
  }
}

__global__ void eval_advance_kernel(const pulse_eval_args_t a) {
  int* c = a.ctrl;
  if (c[1] != 0) return;
  const int s = c[0], running = c[3], running_bound = c[4], longest = c[2];
  int curr_max;
  if (running > 0) {                                              // im_amp.py:252-266
    curr_max = running_bound > 0 ? longest : s - 1;
    if (s >= curr_max) curr_max = s + 1;
  } else {
    curr_max = a.max_steps_all;                                   // :268
  }
  c[0] = s + 1;                                                   // :273
  if (s + 1 >= curr_max || running == 0) c[1] = 1;                // :275
  c[2] = 0; c[3] = 0; c[4] = 0;
}

}  // namespace
}  // namespace pulse

extern "C" int pulse_eval_step(const pulse_eval_args_t* args, void* stream) {
  using namespace pulse;
  PULSE_REQUIRE(args != nullptr, "pulse_eval_step: null args");
  const pulse_eval_args_t& a = *args;
  PULSE_REQUIRE(a.num_envs > 0 && a.bound >= 0 && a.bound <= a.num_envs, "pulse_eval_step: num_envs %d / bound %d", a.num_envs, a.bound);
  PULSE_REQUIRE(a.body_pos && a.body_pos_gt && a.terminate && a.num_steps, "pulse_eval_step: null input");
  PULSE_REQUIRE(a.pos_body_stride >= 3 && a.gt_body_stride >= 3, "pulse_eval_step: body strides must be >= 3 floats");
  PULSE_REQUIRE(a.ctrl && a.terminate_state && a.hist && a.sums && a.counts, "pulse_eval_step: null state buffer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int warps_per_cta = 4;
  eval_accumulate_kernel<<<(a.num_envs + warps_per_cta - 1) / warps_per_cta, warps_per_cta * 32, 0, st>>>(a);
  PULSE_LAUNCH_OK("eval_accumulate_kernel");
  eval_advance_kernel<<<1, 1, 0, st>>>(a);
  PULSE_LAUNCH_OK("eval_advance_kernel");
  return PULSE_OK;
}
