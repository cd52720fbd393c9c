// Row-wise kernels of the PULSE VAE distillation path (SURVEY K17-K19), the Z-task action decode (K20), the reach task
// (K21) and the PD-target map (K22).  The dense layers between them run on the wgmma GEMM; everything here is
// HBM-bound streaming work: one warp per row (lane = latent dimension / body), fp64 atomics for the scalar statistics.
#include <cuda_bf16.h>

#include "pulse_common.cuh"
#include "quat_math.cuh"

namespace pulse {
namespace {

constexpr int kSMs = kNumSMs;

inline unsigned warp_grid(long long rows, int warps_per_block, int waves = 8) {
  long long blocks = (rows + warps_per_block - 1) / warps_per_block;
  const long long cap = static_cast<long long>(kSMs) * waves;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<unsigned>(blocks);
}

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

// ---- normalise a column window -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) normalize_cols_kernel(const float* __restrict__ x, long long ldx, long long rows, long long cols,
                                                             const float* __restrict__ mean, const float* __restrict__ rstd, float clamp,
                                                             __nv_bfloat16* __restrict__ out, long long ld_out, long long zero_to) {
  const long long width = zero_to > cols ? zero_to : cols;
  const long long total = rows * width;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += 256ll * gridDim.x) {
    const long long r = i / width, c = i - r * width;
    float y = 0.0f;
    if (c < cols) {
      y = x[r * ldx + c];
      if (mean != nullptr) y = (y - mean[c]) * rstd[c];
      if (clamp > 0.0f) y = fminf(fmaxf(y, -clamp), clamp);
    }
    out[r * ld_out + c] = __float2bfloat16(y);
  }
}

__global__ void __launch_bounds__(256) copy_cols_kernel(const __nv_bfloat16* __restrict__ src, long long ld_src, long long rows, long long cols,
                                                        __nv_bfloat16* __restrict__ d1, long long ld1, __nv_bfloat16* __restrict__ d2,
                                                        long long ld2) {
  // two bf16 per thread (cols and all leading dimensions are even: checked by the host)
  const long long pairs = cols / 2;
  const long long total = rows * pairs;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += 256ll * gridDim.x) {
    const long long r = i / pairs, c = (i - r * pairs) * 2;
    const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(src + r * ld_src + c);
    *reinterpret_cast<__nv_bfloat162*>(d1 + r * ld1 + c) = v;
    if (d2 != nullptr) *reinterpret_cast<__nv_bfloat162*>(d2 + r * ld2 + c) = v;
  }
}

// ---- latent sample ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) vae_reparam_kernel(const float* __restrict__ head, long long ld_head, const float* __restrict__ noise,
                                                          long long ld_noise, long long rows, int latent, int mode, int clamp, float lo, float hi,
                                                          __nv_bfloat16* __restrict__ zb, long long ld_z, float* __restrict__ zf, long long ld_zf) {
  const long long total = rows * latent;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += 256ll * gridDim.x) {
    const long long r = i / latent;
    const int j = static_cast<int>(i - r * latent);
    const float mu = head[r * ld_head + j];
    float z = mu;
    if (mode == PULSE_Z_SAMPLE) {
      float lv = head[r * ld_head + latent + j];
      if (clamp) lv = fminf(fmaxf(lv, lo), hi);
      z = mu + expf(0.5f * lv) * noise[r * ld_noise + j];
    } else if (mode == PULSE_Z_RESIDUAL) {
      z = mu + noise[r * ld_noise + j];
    }
    if (zb != nullptr) zb[r * ld_z + j] = __float2bfloat16(z);
    if (zf != nullptr) zf[r * ld_zf + j] = z;
  }
}

// ---- action loss --------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) vae_action_loss_kernel(const float* __restrict__ pred, long long ld_pred, const float* __restrict__ gt,
                                                              long long ld_gt, long long rows, int A, __nv_bfloat16* __restrict__ dpred,
                                                              long long ld_d, long long zero_to, double* __restrict__ stats) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float inv_rows = 1.0f / static_cast<float>(rows);
  double acc = 0.0;
  for (long long r = blockIdx.x * 8ll + warp; r < rows; r += 8ll * gridDim.x) {
    float d[4];  // up to 128 actions per row
    float ss = 0.0f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int c = lane + 32 * q;
      d[q] = c < A ? pred[r * ld_pred + c] - gt[r * ld_gt + c] : 0.0f;
      ss = fmaf(d[q], d[q], ss);
    }
    ss = wsum(ss);
    const float nrm = sqrtf(ss);
    const float scale = nrm > 0.0f ? inv_rows / nrm : 0.0f;  // torch.norm backward: 0 at the origin
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int c = lane + 32 * q;
      if (c < A) dpred[r * ld_d + c] = __float2bfloat16(d[q] * scale);
      else if (c < zero_to) dpred[r * ld_d + c] = __float2bfloat16(0.0f);
    }
    acc += static_cast<double>(nrm);
  }
  if (lane == 0 && acc != 0.0) atomicAdd(stats, acc);
}

// ---- latent losses + head gradients -----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) vae_latent_kernel(const pulse_vae_latent_args_t a, long long rows) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int E = a.latent, T = a.horizon;
  const bool on = lane < E;
  __nv_bfloat16* d_enc = reinterpret_cast<__nv_bfloat16*>(a.d_enc_head);      // pulse_bf16_t is a 16-bit integer in the C header
  __nv_bfloat16* d_pri = reinterpret_cast<__nv_bfloat16*>(a.d_prior_head);
  const float inv_rows = 1.0f / static_cast<float>(rows);
  const bool ar1 = a.progress != nullptr && a.ar1_coef != 0.0f && T > 1;
  const float inv_pairs = ar1 ? 1.0f / static_cast<float>((rows / T) * (T - 1)) : 0.0f;
  const float regu_g = a.regu_coef * 0.001f * 2.0f * inv_rows / static_cast<float>(E);  // d/dx of regu_coef * 0.001 * mean(x^2)
  double s_kl = 0.0, s_ar = 0.0, s_pm = 0.0, s_qm = 0.0, s_pv = 0.0, s_qv = 0.0;
  for (long long r = blockIdx.x * 8ll + warp; r < rows; r += 8ll * gridDim.x) {
    float qm = 0.0f, qv_raw = 0.0f, pm = 0.0f, pv_raw = 0.0f, eps = 0.0f, dz = 0.0f;
    if (on) {
      qm = a.enc_head[r * a.ld_enc + lane];
      qv_raw = a.enc_head[r * a.ld_enc + E + lane];
      pm = a.prior_head[r * a.ld_prior + lane];
      pv_raw = a.prior_head[r * a.ld_prior + E + lane];
      eps = a.noise[r * a.ld_noise + lane];
      if (a.dz != nullptr) dz = a.dz[r * a.ld_dz + lane];
    }
    float qv = qv_raw, pv = pv_raw;
    bool qgate = true, pgate = true;  // torch.clamp passes the gradient where lo <= x <= hi
    if (a.clamp) {
      qv = fminf(fmaxf(qv_raw, a.clamp_lo), a.clamp_hi);
      pv = fminf(fmaxf(pv_raw, a.clamp_lo), a.clamp_hi);
      qgate = qv_raw >= a.clamp_lo && qv_raw <= a.clamp_hi;
      pgate = pv_raw >= a.clamp_lo && pv_raw <= a.clamp_hi;
    }
    // KL(q || p), loss_functions.py:9
    const float ipv = expf(-pv), ratio = expf(qv - pv), dm = qm - pm;
    const float kl = on ? 0.5f * (pv - qv + ratio + dm * dm * ipv - 1.0f) : 0.0f;
    const float kc = a.kld_coef * inv_rows;
    float g_qm = kc * dm * ipv;
    float g_qv = kc * 0.5f * (ratio - 1.0f);
    float g_pm = -g_qm;
    float g_pv = kc * 0.5f * (1.0f - ratio - dm * dm * ipv);
    // reparameterisation: z = qm + exp(0.5 qv) eps
    g_qm += dz;
    g_qv += dz * 0.5f * expf(0.5f * qv) * eps;
    // AR(1) prior on the posterior means of consecutive steps of the same env (amp_agent.py:792-808)
    float ar_row = 0.0f;
    if (ar1) {
      const long long t = r % T;
      const long long pr = a.progress[r];
      if (t > 0) {  // pair (t-1, t): this row is the "next" step
        const long long pp = a.progress[r - 1];
        const bool keep = (pr - pp == 1) && !(pr <= 2 || pp <= 2);
        if (keep) {
          const float prev = on ? a.enc_head[(r - 1) * a.ld_enc + lane] : 0.0f;
          const float e = on ? qm - a.phi * prev : 0.0f;
          const float nrm = sqrtf(wsum(e * e));
          if (nrm > 0.0f) g_qm += a.ar1_coef * inv_pairs * e / nrm;
          ar_row = nrm;  // each pair is counted once, by its "next" row
        }
      }
      if (t < T - 1) {  // pair (t, t+1): this row is the "previous" step
        const long long pn = a.progress[r + 1];
        const bool keep = (pn - pr == 1) && !(pn <= 2 || pr <= 2);
        if (keep) {
          const float nxt = on ? a.enc_head[(r + 1) * a.ld_enc + lane] : 0.0f;
          const float e = on ? nxt - a.phi * qm : 0.0f;
          const float nrm = sqrtf(wsum(e * e));
          if (nrm > 0.0f) g_qm -= a.ar1_coef * inv_pairs * a.phi * e / nrm;
        }
      }
    }
    if (a.regu_coef != 0.0f) {
      g_qm += regu_g * qm;
      g_pm += regu_g * pm;
      g_qv += regu_g * qv;
      g_pv += regu_g * pv;
    }
    if (!qgate) g_qv = 0.0f;
    if (!pgate) g_pv = 0.0f;
    if (on) {
      d_enc[r * a.ld_de + lane] = __float2bfloat16(g_qm);
      d_enc[r * a.ld_de + E + lane] = __float2bfloat16(g_qv);
      d_pri[r * a.ld_dp + lane] = __float2bfloat16(g_pm);
      d_pri[r * a.ld_dp + E + lane] = __float2bfloat16(g_pv);
    }
    s_kl += static_cast<double>(wsum(kl));
    s_ar += static_cast<double>(ar_row);
    if (a.regu_coef != 0.0f) {
      s_pm += static_cast<double>(wsum(on ? pm * pm : 0.0f));
      s_qm += static_cast<double>(wsum(on ? qm * qm : 0.0f));
      s_pv += static_cast<double>(wsum(on ? pv * pv : 0.0f));
      s_qv += static_cast<double>(wsum(on ? qv * qv : 0.0f));
    }
  }
  if (lane == 0) {
    atomicAdd(a.stats + 0, s_kl);
    if (s_ar != 0.0) atomicAdd(a.stats + 1, s_ar);
    if (a.regu_coef != 0.0f) {
      atomicAdd(a.stats + 2, s_pm);
      atomicAdd(a.stats + 3, s_qm);
      atomicAdd(a.stats + 4, s_pv);
      atomicAdd(a.stats + 5, s_qv);
    }
  }
}

// ---- teacher: weighted sum of the primitive columns ---------------------------------------------------------------------
__global__ void __launch_bounds__(256) pnn_compose_kernel(const float* __restrict__ acts, long long prim_stride, long long ld_a,
                                                          const float* __restrict__ w, long long ld_w, int act, long long rows, int A, int K,
                                                          float* __restrict__ out, long long ld_out) {
  const long long total = rows * A;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += 256ll * gridDim.x) {
    const long long r = i / A;
    const int c = static_cast<int>(i - r * A);
    float s = 0.0f;
    for (int k = 0; k < K; ++k) {
      float wk = w[r * ld_w + k];
      if (act == PULSE_ACT_SILU) wk = wk / (1.0f + expf(-wk));
      else if (act == PULSE_ACT_RELU) wk = fmaxf(wk, 0.0f);
      s = fmaf(wk, acts[k * prim_stride + r * ld_a + c], s);
    }
    out[r * ld_out + c] = s;
  }
}

__global__ void __launch_bounds__(256) pd_targets_kernel(const float* __restrict__ action, long long ld_a, const float* __restrict__ offset,
                                                         const float* __restrict__ scale, const uint8_t* __restrict__ freeze, long long rows,
                                                         int dofs, float* __restrict__ out, long long ld_out) {
  const long long total = rows * dofs;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += 256ll * gridDim.x) {
    const long long r = i / dofs;
    const int d = static_cast<int>(i - r * dofs);
    const float v = __fadd_rn(offset[d], __fmul_rn(scale[d], action[r * ld_a + d]));  // the reference's two roundings
    out[r * ld_out + d] = (freeze != nullptr && freeze[d]) ? 0.0f : v;
  }
}

// ---- reach task --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) reach_update_task_kernel(const long long* __restrict__ progress, long long* __restrict__ change,
                                                                float* __restrict__ tar, const float* __restrict__ u,
                                                                const long long* __restrict__ steps, float dist_max, float h_min, float h_max,
                                                                long long n) {
  for (long long e = blockIdx.x * 256ll + threadIdx.x; e < n; e += 256ll * gridDim.x) {
    if (progress[e] >= change[e]) {
      tar[3 * e + 0] = dist_max * (2.0f * u[3 * e + 0] - 1.0f);
      tar[3 * e + 1] = dist_max * (2.0f * u[3 * e + 1] - 1.0f);
      tar[3 * e + 2] = (h_max - h_min) * u[3 * e + 2] + h_min;
      change[e] = progress[e] + steps[e];
    }
  }
}

constexpr int kNB = 24;

__global__ void __launch_bounds__(256) reach_step_kernel(const pulse_reach_step_args_t a, long long n) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long e = blockIdx.x * 8ll + warp; e < n; e += 8ll * gridDim.x) {
    const int j = lane;
    const bool body = j < kNB;
    const float* bs = a.body_state + e * a.body_env_stride + (body ? j : 0) * 13;
    Vec3 p = {bs[0], bs[1], bs[2]}, v = {bs[7], bs[8], bs[9]}, w = {bs[10], bs[11], bs[12]};
    Quat q = {bs[3], bs[4], bs[5], bs[6]};
    const Vec3 p_root = {__shfl_sync(kFull, p.x, 0), __shfl_sync(kFull, p.y, 0), __shfl_sync(kFull, p.z, 0)};
    const Quat q_root = {__shfl_sync(kFull, q.x, 0), __shfl_sync(kFull, q.y, 0), __shfl_sync(kFull, q.z, 0), __shfl_sync(kFull, q.w, 0)};
    float hs, hc;
    heading_half(q_root, hs, hc);
    const Yaw yr = make_yaw(Quat{0.0f, 0.0f, -hs, hc});
    float* o = a.obs_buf + e * a.obs_stride;
    if (body) {  // compute_humanoid_observations_smpl_max (humanoid.py:1675-1731), same layout as the imitation step kernel
      if (j == 0) o[0] = p_root.z;
      else {
        const Vec3 lp = yaw_rot(yr, p - p_root);
        o[1 + 3 * (j - 1)] = lp.x; o[2 + 3 * (j - 1)] = lp.y; o[3 + 3 * (j - 1)] = lp.z;
      }
      float six[6];
      qsix(yaw_mul_left(-hs, hc, q), six);
#pragma unroll
      for (int i = 0; i < 6; ++i) o[70 + 6 * j + i] = six[i];
      const Vec3 lv = yaw_rot(yr, v), lw = yaw_rot(yr, w);
      o[214 + 3 * j] = lv.x; o[215 + 3 * j] = lv.y; o[216 + 3 * j] = lv.z;
      o[286 + 3 * j] = lw.x; o[287 + 3 * j] = lw.y; o[288 + 3 * j] = lw.z;
    }
    const Vec3 tar = {a.tar_pos[3 * e], a.tar_pos[3 * e + 1], a.tar_pos[3 * e + 2]};
    // early termination (humanoid.py:1573-1608)
    bool fall_contact = false, fall_height = false;
    if (a.enable_early_termination && body && !((a.contact_body_mask >> j) & 1u)) {
      if (a.contact_forces != nullptr) {
        const float* cf = a.contact_forces + e * a.contact_env_stride + j * 3;
        fall_contact = fabsf(cf[0]) > 0.1f || fabsf(cf[1]) > 0.1f || fabsf(cf[2]) > 0.1f;
      }
      fall_height = p.z < a.termination_heights[j];
    }
    const bool any_contact = __any_sync(kFull, fall_contact), any_height = __any_sync(kFull, fall_height);
    // the reach body's position, broadcast
    const int rb = a.reach_body_id;
    const Vec3 pr = {__shfl_sync(kFull, p.x, rb), __shfl_sync(kFull, p.y, rb), __shfl_sync(kFull, p.z, rb)};
    if (lane == 0) {
      const Vec3 lt = yaw_rot(yr, tar - p_root);  // compute_location_observations (humanoid_reach.py:224-236)
      o[PULSE_SELF_OBS + 0] = lt.x; o[PULSE_SELF_OBS + 1] = lt.y; o[PULSE_SELF_OBS + 2] = lt.z;
      const Vec3 d = tar - pr;                    // compute_reach_reward (:238-250)
      a.rew_buf[e] = expf(-4.0f * (d.x * d.x + d.y * d.y + d.z * d.z));
      const long long prog = a.progress_buf[e];
      const long long term = (any_contact && any_height && prog > 1) ? 1 : 0;
      a.terminate_buf[e] = term;
      a.reset_buf[e] = prog >= a.max_episode_length - 1 ? 1 : term;
    }
  }
}

inline unsigned elem_grid(long long total) {
  long long b = (total + 255) / 256;
  const long long cap = static_cast<long long>(kSMs) * 8;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return static_cast<unsigned>(b);
}

}  // namespace
}  // namespace pulse

using namespace pulse;

extern "C" int pulse_normalize_cols(const float* x, int64_t ldx, int64_t rows, int64_t cols, const float* mean, const float* rstd, float clamp,
                                    pulse_bf16_t* out, int64_t ld_out, int64_t zero_to, void* stream) {
  PULSE_REQUIRE(x && out, "pulse_normalize_cols: null buffer");
  PULSE_REQUIRE(rows > 0 && cols > 0 && ldx >= cols && ld_out >= cols && zero_to <= ld_out, "pulse_normalize_cols: bad shape");
  PULSE_REQUIRE((mean == nullptr) == (rstd == nullptr), "pulse_normalize_cols: mean and rstd go together");
  const long long width = zero_to > cols ? zero_to : cols;
  normalize_cols_kernel<<<elem_grid(rows * width), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, ldx, rows, cols, mean, rstd, clamp, reinterpret_cast<__nv_bfloat16*>(out), ld_out, zero_to);
  PULSE_LAUNCH_OK("normalize_cols_kernel");
  return PULSE_OK;
}

extern "C" int pulse_copy_cols_bf16(const pulse_bf16_t* src, int64_t ld_src, int64_t rows, int64_t cols, pulse_bf16_t* dst1, int64_t ld1,
                                    pulse_bf16_t* dst2, int64_t ld2, void* stream) {
  PULSE_REQUIRE(src && dst1, "pulse_copy_cols_bf16: null buffer");
  PULSE_REQUIRE(rows > 0 && cols > 0 && cols % 2 == 0 && ld_src % 2 == 0 && ld1 % 2 == 0 && (dst2 == nullptr || ld2 % 2 == 0),
                "pulse_copy_cols_bf16: cols and leading dimensions must be even");
  PULSE_REQUIRE((reinterpret_cast<uintptr_t>(src) & 3) == 0 && (reinterpret_cast<uintptr_t>(dst1) & 3) == 0 &&
                    (reinterpret_cast<uintptr_t>(dst2) & 3) == 0, "pulse_copy_cols_bf16: 4-byte alignment required");
  copy_cols_kernel<<<elem_grid(rows * (cols / 2)), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(src), ld_src, rows, cols, reinterpret_cast<__nv_bfloat16*>(dst1), ld1,
      reinterpret_cast<__nv_bfloat16*>(dst2), ld2);
  PULSE_LAUNCH_OK("copy_cols_kernel");
  return PULSE_OK;
}

extern "C" int pulse_vae_reparam(const float* head, int64_t ld_head, const float* noise, int64_t ld_noise, int64_t rows, int32_t latent,
                                 int32_t mode, int32_t clamp, float clamp_lo, float clamp_hi, pulse_bf16_t* z_bf16, int64_t ld_z, float* z_f32,
                                 int64_t ld_zf, void* stream) {
  PULSE_REQUIRE(head && (z_bf16 || z_f32), "pulse_vae_reparam: null buffer");
  PULSE_REQUIRE(rows > 0 && latent > 0, "pulse_vae_reparam: bad shape");
  PULSE_REQUIRE(mode == PULSE_Z_MEAN || noise != nullptr, "pulse_vae_reparam: noise required unless mode is PULSE_Z_MEAN");
  PULSE_REQUIRE(mode == PULSE_Z_SAMPLE || mode == PULSE_Z_MEAN || mode == PULSE_Z_RESIDUAL, "pulse_vae_reparam: unknown mode %d", mode);
  PULSE_REQUIRE(ld_head >= (mode == PULSE_Z_SAMPLE ? 2 * latent : latent), "pulse_vae_reparam: head too narrow");
  vae_reparam_kernel<<<elem_grid(rows * latent), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      head, ld_head, noise, ld_noise, rows, latent, mode, clamp, clamp_lo, clamp_hi, reinterpret_cast<__nv_bfloat16*>(z_bf16), ld_z, z_f32, ld_zf);
  PULSE_LAUNCH_OK("vae_reparam_kernel");
  return PULSE_OK;
}

extern "C" int pulse_vae_action_loss(const float* pred, int64_t ld_pred, const float* gt, int64_t ld_gt, int64_t rows, int32_t num_actions,
                                     pulse_bf16_t* dpred, int64_t ld_d, int64_t zero_to, double* stats, void* stream) {
  PULSE_REQUIRE(pred && gt && dpred && stats, "pulse_vae_action_loss: null buffer");
  PULSE_REQUIRE(rows > 0 && num_actions > 0 && num_actions <= 128 && zero_to <= 128 && zero_to <= ld_d && ld_d >= num_actions,
                "pulse_vae_action_loss: bad shape (num_actions <= 128)");
  vae_action_loss_kernel<<<warp_grid(rows, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      pred, ld_pred, gt, ld_gt, rows, num_actions, reinterpret_cast<__nv_bfloat16*>(dpred), ld_d, zero_to, stats);
  PULSE_LAUNCH_OK("vae_action_loss_kernel");
  return PULSE_OK;
}

extern "C" int pulse_vae_latent_loss(const pulse_vae_latent_args_t* args, int64_t rows, void* stream) {
  PULSE_REQUIRE(args, "pulse_vae_latent_loss: null args");
  const pulse_vae_latent_args_t& a = *args;
  PULSE_REQUIRE(a.enc_head && a.prior_head && a.noise && a.d_enc_head && a.d_prior_head && a.stats, "pulse_vae_latent_loss: null buffer");
  PULSE_REQUIRE(rows > 0 && a.latent > 0 && a.latent <= 32, "pulse_vae_latent_loss: latent must be in [1, 32]");
  PULSE_REQUIRE(a.ld_enc >= 2 * a.latent && a.ld_prior >= 2 * a.latent && a.ld_de >= 2 * a.latent && a.ld_dp >= 2 * a.latent,
                "pulse_vae_latent_loss: head buffers narrower than 2*latent");
  PULSE_REQUIRE(a.progress == nullptr || a.ar1_coef == 0.0f || (a.horizon > 0 && rows % a.horizon == 0),
                "pulse_vae_latent_loss: rows must be a multiple of horizon for the AR(1) term");
  vae_latent_kernel<<<warp_grid(rows, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, rows);
  PULSE_LAUNCH_OK("vae_latent_kernel");
  return PULSE_OK;
}

extern "C" int pulse_pnn_compose(const float* acts, int64_t prim_stride, int64_t ld_a, const float* w, int64_t ld_w, int32_t act, int64_t rows,
                                 int32_t num_actions, int32_t num_prim, float* out, int64_t ld_out, void* stream) {
  PULSE_REQUIRE(acts && w && out, "pulse_pnn_compose: null buffer");
  PULSE_REQUIRE(rows > 0 && num_actions > 0 && num_prim > 0 && ld_a >= num_actions && ld_w >= num_prim && ld_out >= num_actions,
                "pulse_pnn_compose: bad shape");
  pnn_compose_kernel<<<elem_grid(rows * num_actions), 256, 0, static_cast<cudaStream_t>(stream)>>>(acts, prim_stride, ld_a, w, ld_w, act, rows,
                                                                                                    num_actions, num_prim, out, ld_out);
  PULSE_LAUNCH_OK("pnn_compose_kernel");
  return PULSE_OK;
}

extern "C" int pulse_pd_targets(const float* action, int64_t ld_a, const float* offset, const float* scale, const uint8_t* freeze, int64_t rows,
                                int32_t dofs, float* out, int64_t ld_out, void* stream) {
  PULSE_REQUIRE(action && offset && scale && out, "pulse_pd_targets: null buffer");
  PULSE_REQUIRE(rows > 0 && dofs > 0 && ld_a >= dofs && ld_out >= dofs, "pulse_pd_targets: bad shape");
  pd_targets_kernel<<<elem_grid(rows * dofs), 256, 0, static_cast<cudaStream_t>(stream)>>>(action, ld_a, offset, scale, freeze, rows, dofs, out,
                                                                                           ld_out);
  PULSE_LAUNCH_OK("pd_targets_kernel");
  return PULSE_OK;
}

extern "C" int pulse_reach_update_task(const int64_t* progress, int64_t* tar_change_steps, float* tar_pos, const float* rand01,
                                       const int64_t* steps, float dist_max, float h_min, float h_max, int64_t num_envs, void* stream) {
  PULSE_REQUIRE(progress && tar_change_steps && tar_pos && rand01 && steps, "pulse_reach_update_task: null buffer");
  PULSE_REQUIRE(num_envs > 0, "pulse_reach_update_task: num_envs <= 0");
  reach_update_task_kernel<<<elem_grid(num_envs), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(progress), reinterpret_cast<long long*>(tar_change_steps), tar_pos, rand01,
      reinterpret_cast<const long long*>(steps), dist_max, h_min, h_max, num_envs);
  PULSE_LAUNCH_OK("reach_update_task_kernel");
  return PULSE_OK;
}

extern "C" int pulse_reach_step(const pulse_reach_step_args_t* args, int64_t num_envs, void* stream) {
  PULSE_REQUIRE(args, "pulse_reach_step: null args");
  const pulse_reach_step_args_t& a = *args;
  PULSE_REQUIRE(a.body_state && a.tar_pos && a.progress_buf && a.obs_buf && a.rew_buf && a.reset_buf && a.terminate_buf,
                "pulse_reach_step: null buffer");
  PULSE_REQUIRE(num_envs > 0 && a.body_env_stride >= 24 * 13 && a.obs_stride >= PULSE_REACH_OBS, "pulse_reach_step: bad strides");
  PULSE_REQUIRE(a.reach_body_id >= 0 && a.reach_body_id < 24, "pulse_reach_step: reach_body_id out of range");
  PULSE_REQUIRE(!a.enable_early_termination || a.termination_heights != nullptr, "pulse_reach_step: termination_heights required");
  PULSE_REQUIRE(a.contact_forces == nullptr || a.contact_env_stride >= 24 * 3, "pulse_reach_step: bad contact stride");
  reach_step_kernel<<<warp_grid(num_envs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, num_envs);
  PULSE_LAUNCH_OK("reach_step_kernel");
  return PULSE_OK;
}
