// Row-wise kernels of the PULSE VAE distillation path (SURVEY K17-K19), the Z-task action decode (K20) and the PD-target map
// (K22).  The dense layers between them run on the wgmma GEMM; everything here is HBM-bound streaming work: element-wise
// grid-stride loops, or one warp per row (lane = action / latent dimension) with fp64 atomics for the scalar statistics.
#include <cuda_bf16.h>

#include "philox.cuh"
#include "pulse_common.cuh"

namespace pulse {
namespace {

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

// z = mu + exp(0.5 clamp(logvar)) eps with eps drawn here (the reparameterisation of the distillation rollout): one thread per latent PAIR,
// one Philox4x32-10 call keyed (seed, row * 64 + pair, offset) whose first two words give the pair's two Box-Muller normals -- the
// indexing of policy_post_kernel.  The arithmetic after the draw is vae_reparam_kernel's PULSE_Z_SAMPLE path.
__global__ void __launch_bounds__(256) vae_reparam_philox_kernel(const float* __restrict__ head, long long ld_head, long long rows, int latent,
                                                                 int clamp, float lo, float hi, unsigned long long seed,
                                                                 const unsigned long long* __restrict__ offset_dev, unsigned long long step,
                                                                 __nv_bfloat16* __restrict__ zb, long long ld_z, float* __restrict__ noise_out,
                                                                 long long ld_noise) {
  const int pairs = (latent + 1) / 2;
  const long long total = rows * pairs;
  const unsigned long long off = offset_dev != nullptr ? *offset_dev + step : step;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += 256ll * gridDim.x) {
    const long long r = i / pairs;
    const int p = static_cast<int>(i - r * pairs);
    const Philox4 w = philox4x32_10(seed, static_cast<unsigned long long>(r) * 64ull + static_cast<unsigned long long>(p), off);
    float e[2];
    box_muller(w.x, w.y, e[0], e[1]);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = 2 * p + h;
      if (j >= latent) break;
      const float mu = head[r * ld_head + j];
      float lv = head[r * ld_head + latent + j];
      if (clamp) lv = fminf(fmaxf(lv, lo), hi);
      const float z = mu + expf(0.5f * lv) * e[h];
      zb[r * ld_z + j] = __float2bfloat16(z);
      if (noise_out != nullptr) noise_out[r * ld_noise + j] = e[h];
    }
  }
}

// ---- pre-physics step of the distillation rollout ---------------------------------------------------------------------------
// pd_out = freeze ? 0 : offset + scale * mus (pd_targets_kernel's two roundings), the progress record kin_progress[r] = progress[r] and
// HumanoidImGetup._update_recovery_count's recovery_counter = max(recovery_counter - 1, 0), in one launch: the row-wise outputs are
// written by the thread of column 0.
__global__ void __launch_bounds__(256) distill_pre_physics_kernel(const float* __restrict__ mus, long long ld_mus, const float* __restrict__ offset,
                                                                  const float* __restrict__ scale, const uint8_t* __restrict__ freeze,
                                                                  long long rows, int dofs, float* __restrict__ pd_out, long long ld_pd,
                                                                  const long long* __restrict__ progress, long long* __restrict__ kin_progress,
                                                                  long long ld_kp, int* __restrict__ recovery_counter) {
  const long long total = rows * dofs;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += 256ll * gridDim.x) {
    const long long r = i / dofs;
    const int d = static_cast<int>(i - r * dofs);
    const float v = __fadd_rn(offset[d], __fmul_rn(scale[d], mus[r * ld_mus + d]));
    pd_out[r * ld_pd + d] = (freeze != nullptr && freeze[d]) ? 0.0f : v;
    if (d == 0) {
      kin_progress[r * ld_kp] = progress[r];
      const int rc = recovery_counter[r];
      recovery_counter[r] = rc > 1 ? rc - 1 : 0;
    }
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
    ss = warp_sum(ss);
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
          const float nrm = sqrtf(warp_sum(e * e));
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
          const float nrm = sqrtf(warp_sum(e * e));
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
    s_kl += static_cast<double>(warp_sum(kl));
    s_ar += static_cast<double>(ar_row);
    if (a.regu_coef != 0.0f) {
      s_pm += static_cast<double>(warp_sum(on ? pm * pm : 0.0f));
      s_qm += static_cast<double>(warp_sum(on ? qm * qm : 0.0f));
      s_pv += static_cast<double>(warp_sum(on ? pv * pv : 0.0f));
      s_qv += static_cast<double>(warp_sum(on ? qv * qv : 0.0f));
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

}  // namespace
}  // namespace pulse

using namespace pulse;

extern "C" int pulse_normalize_cols(const float* x, int64_t ldx, int64_t rows, int64_t cols, const float* mean, const float* rstd, float clamp,
                                    pulse_bf16_t* out, int64_t ld_out, int64_t zero_to, void* stream) {
  PULSE_REQUIRE(x && out, "pulse_normalize_cols: null buffer");
  PULSE_REQUIRE(rows > 0 && cols > 0 && ldx >= cols && ld_out >= cols && zero_to <= ld_out, "pulse_normalize_cols: bad shape");
  PULSE_REQUIRE((mean == nullptr) == (rstd == nullptr), "pulse_normalize_cols: mean and rstd go together");
  const long long width = zero_to > cols ? zero_to : cols;
  normalize_cols_kernel<<<grid_for(rows * width, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
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
  copy_cols_kernel<<<grid_for(rows * (cols / 2), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
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
  vae_reparam_kernel<<<grid_for(rows * latent, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      head, ld_head, noise, ld_noise, rows, latent, mode, clamp, clamp_lo, clamp_hi, reinterpret_cast<__nv_bfloat16*>(z_bf16), ld_z, z_f32, ld_zf);
  PULSE_LAUNCH_OK("vae_reparam_kernel");
  return PULSE_OK;
}

extern "C" int pulse_vae_reparam_philox(const float* head, int64_t ld_head, int64_t rows, int32_t latent, int32_t clamp, float clamp_lo,
                                        float clamp_hi, uint64_t seed, const uint64_t* offset_dev, uint64_t step, pulse_bf16_t* z_bf16,
                                        int64_t ld_z, float* noise_out, int64_t ld_noise, void* stream) {
  PULSE_REQUIRE(head && z_bf16, "pulse_vae_reparam_philox: null head / z_bf16");
  PULSE_REQUIRE(rows >= 0, "pulse_vae_reparam_philox: negative rows");
  PULSE_REQUIRE(latent >= 1 && latent <= 32, "pulse_vae_reparam_philox: latent %d outside [1, 32]", latent);
  PULSE_REQUIRE(ld_head >= 2 * latent && ld_z >= latent, "pulse_vae_reparam_philox: head or z row stride too small");
  PULSE_REQUIRE(noise_out == nullptr || ld_noise >= latent, "pulse_vae_reparam_philox: noise_out row stride too small");
  if (rows == 0) return PULSE_OK;
  vae_reparam_philox_kernel<<<grid_for(rows * ((latent + 1) / 2), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      head, ld_head, rows, latent, clamp, clamp_lo, clamp_hi, seed, reinterpret_cast<const unsigned long long*>(offset_dev), step,
      reinterpret_cast<__nv_bfloat16*>(z_bf16), ld_z, noise_out, ld_noise);
  PULSE_LAUNCH_OK("vae_reparam_philox_kernel");
  return PULSE_OK;
}

extern "C" int pulse_distill_pre_physics(const float* mus, int64_t ld_mus, const float* pd_offset, const float* pd_scale, const uint8_t* freeze,
                                         int64_t rows, int32_t dofs, float* pd_out, int64_t ld_pd, const int64_t* progress_buf,
                                         int64_t* kin_progress, int64_t ld_progress, int32_t* recovery_counter, void* stream) {
  PULSE_REQUIRE(mus && pd_offset && pd_scale && pd_out, "pulse_distill_pre_physics: null mus / pd_offset / pd_scale / pd_out");
  PULSE_REQUIRE(progress_buf && kin_progress && recovery_counter, "pulse_distill_pre_physics: null progress_buf / kin_progress / recovery_counter");
  PULSE_REQUIRE(rows >= 0, "pulse_distill_pre_physics: negative rows");
  PULSE_REQUIRE(dofs >= 1, "pulse_distill_pre_physics: dofs %d < 1", dofs);
  PULSE_REQUIRE(ld_mus >= dofs && ld_pd >= dofs && ld_progress >= 1, "pulse_distill_pre_physics: row strides too small");
  if (rows == 0) return PULSE_OK;
  distill_pre_physics_kernel<<<grid_for(rows * dofs, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      mus, ld_mus, pd_offset, pd_scale, freeze, rows, dofs, pd_out, ld_pd, reinterpret_cast<const long long*>(progress_buf),
      reinterpret_cast<long long*>(kin_progress), ld_progress, recovery_counter);
  PULSE_LAUNCH_OK("distill_pre_physics_kernel");
  return PULSE_OK;
}

extern "C" int pulse_vae_action_loss(const float* pred, int64_t ld_pred, const float* gt, int64_t ld_gt, int64_t rows, int32_t num_actions,
                                     pulse_bf16_t* dpred, int64_t ld_d, int64_t zero_to, double* stats, void* stream) {
  PULSE_REQUIRE(pred && gt && dpred && stats, "pulse_vae_action_loss: null buffer");
  PULSE_REQUIRE(rows > 0 && num_actions > 0 && num_actions <= 128 && zero_to <= 128 && zero_to <= ld_d && ld_d >= num_actions,
                "pulse_vae_action_loss: bad shape (num_actions <= 128)");
  vae_action_loss_kernel<<<grid_for(rows, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
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
  vae_latent_kernel<<<grid_for(rows, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, rows);
  PULSE_LAUNCH_OK("vae_latent_kernel");
  return PULSE_OK;
}

extern "C" int pulse_pnn_compose(const float* acts, int64_t prim_stride, int64_t ld_a, const float* w, int64_t ld_w, int32_t act, int64_t rows,
                                 int32_t num_actions, int32_t num_prim, float* out, int64_t ld_out, void* stream) {
  PULSE_REQUIRE(acts && w && out, "pulse_pnn_compose: null buffer");
  PULSE_REQUIRE(rows > 0 && num_actions > 0 && num_prim > 0 && ld_a >= num_actions && ld_w >= num_prim && ld_out >= num_actions,
                "pulse_pnn_compose: bad shape");
  pnn_compose_kernel<<<grid_for(rows * num_actions, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(acts, prim_stride, ld_a, w, ld_w, act, rows,
                                                                                                    num_actions, num_prim, out, ld_out);
  PULSE_LAUNCH_OK("pnn_compose_kernel");
  return PULSE_OK;
}

extern "C" int pulse_pd_targets(const float* action, int64_t ld_a, const float* offset, const float* scale, const uint8_t* freeze, int64_t rows,
                                int32_t dofs, float* out, int64_t ld_out, void* stream) {
  PULSE_REQUIRE(action && offset && scale && out, "pulse_pd_targets: null buffer");
  PULSE_REQUIRE(rows > 0 && dofs > 0 && ld_a >= dofs && ld_out >= dofs, "pulse_pd_targets: bad shape");
  pd_targets_kernel<<<grid_for(rows * dofs, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(action, ld_a, offset, scale, freeze, rows, dofs, out,
                                                                                           ld_out);
  PULSE_LAUNCH_OK("pd_targets_kernel");
  return PULSE_OK;
}
