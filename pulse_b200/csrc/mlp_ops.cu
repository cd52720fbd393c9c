// Element-wise and reduction kernels around the wgmma GEMMs: observation normalisation, Gaussian
// policy head, PPO losses + output gradients, bias-gradient column sums, split-K slab reduction,
// gradient-norm clip + Adam, bf16 operand refresh.  All HBM-bound streaming kernels: 16-byte accesses
// where the layout allows, grid-stride loops sized to a multiple of the SM count.
#include <cuda_bf16.h>

#include "pulse_common.cuh"

namespace pulse {
namespace {

constexpr int kSMs = kNumSMs;

// ---- RunningMeanStd normalise + clamp -> bf16 (and transposed bf16) -------------------------------------------
// One CTA handles a 32-row x 32-col tile so the transposed copy can go through a padded shared tile.
__global__ void __launch_bounds__(256) normalize_kernel(const float* __restrict__ x, long long ldx, long long rows, long long cols,
                                                        const float* __restrict__ mean, const float* __restrict__ rstd,
                                                        __nv_bfloat16* __restrict__ out, long long ld_out,
                                                        __nv_bfloat16* __restrict__ out_t, long long ld_t, float pad_one) {
  __shared__ float tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const long long col_tiles = (ld_out + 31) / 32;
  const long long row_tiles = (rows + 31) / 32;
  for (long long t = blockIdx.x; t < col_tiles * row_tiles; t += gridDim.x) {
    const long long rt = t / col_tiles, ct = t - rt * col_tiles;
    const long long c = ct * 32 + tx;
    float m = 0.0f, rs = 1.0f;
    if (mean != nullptr && c < cols) {
      m = mean[c];
      rs = rstd[c];
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const long long r = rt * 32 + ty + 8 * i;
      float y = c == cols ? pad_one : 0.0f;   // first pad column: the "ones" column of a bias-augmented operand (else zero fill)
      if (r < rows && c < cols) {
        y = (x[r * ldx + c] - m) * rs;
        if (mean != nullptr) y = fminf(fmaxf(y, -5.0f), 5.0f);
      }
      if (r < rows && c < ld_out && out != nullptr) out[r * ld_out + c] = __float2bfloat16(y);
      tile[ty + 8 * i][tx] = y;
    }
    if (out_t != nullptr) {
      __syncthreads();
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const long long cc = ct * 32 + ty + 8 * i;  // transposed: row index of out_t
        const long long rr = rt * 32 + tx;
        if (cc < ld_out && rr < rows) out_t[cc * ld_t + rr] = __float2bfloat16(tile[tx][ty + 8 * i]);
      }
      __syncthreads();
    }
  }
}

// ---- per-column sum / sum of squares in fp64 --------------------------------------------------------------------
__global__ void __launch_bounds__(256) column_moments_kernel(const float* __restrict__ x, long long ldx, long long rows, long long cols,
                                                             double* __restrict__ sums) {
  // blockIdx.y: row chunk; each thread owns columns c = blockIdx.x*256 + threadIdx.x (coalesced across the warp)
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  const long long chunk = (rows + gridDim.y - 1) / gridDim.y;
  const long long r0 = blockIdx.y * chunk, r1 = min(rows, r0 + chunk);
  double s = 0.0, q = 0.0;
  for (long long r = r0; r < r1; ++r) {
    const double v = x[r * ldx + c];
    s += v;
    q += v * v;
  }
  atomicAdd(sums + c, s);
  atomicAdd(sums + cols + c, q);
}

// ---- fused normalise + moments: ONE pass over x ---------------------------------------------------------------------
// PHC's RunningMeanStd normalises with the statistics from BEFORE the batch and merges the batch moments afterwards
// (running_mean_std.py:91-107), so both consume the same fp32 rows: each thread owns a column PAIR (8-byte load,
// 4-byte bf16x2 store), walks a row chunk with 8 rows in flight, and finishes with four fp64 atomics.
// Rows [r0, r1) of source columns (c, c+1) of x -> destination columns (oc, oc+1) of out; sums[2*cols] += their moments.
__device__ __forceinline__ void normalize_pair_rows(const float* __restrict__ x, long long ldx, long long cols, long long c, long long r0,
                                                    long long r1, const float* __restrict__ mean, const float* __restrict__ rstd,
                                                    __nv_bfloat16* __restrict__ out, long long ld_out, long long oc,
                                                    double* __restrict__ sums) {
  const float2 m = *reinterpret_cast<const float2*>(mean + c), rs = *reinterpret_cast<const float2*>(rstd + c);
  double s0 = 0.0, s1 = 0.0, q0 = 0.0, q1 = 0.0;
  long long r = r0;
  for (; r + 8 <= r1; r += 8) {
    float2 v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = __ldcs(reinterpret_cast<const float2*>(x + (r + i) * ldx + c));
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float y0 = fminf(fmaxf((v[i].x - m.x) * rs.x, -5.0f), 5.0f), y1 = fminf(fmaxf((v[i].y - m.y) * rs.y, -5.0f), 5.0f);
      *reinterpret_cast<__nv_bfloat162*>(out + (r + i) * ld_out + oc) = __floats2bfloat162_rn(y0, y1);
      const double d0 = v[i].x, d1 = v[i].y;
      s0 += d0;
      s1 += d1;
      q0 += d0 * d0;
      q1 += d1 * d1;
    }
  }
  for (; r < r1; ++r) {
    const float2 v = *reinterpret_cast<const float2*>(x + r * ldx + c);
    const float y0 = fminf(fmaxf((v.x - m.x) * rs.x, -5.0f), 5.0f), y1 = fminf(fmaxf((v.y - m.y) * rs.y, -5.0f), 5.0f);
    *reinterpret_cast<__nv_bfloat162*>(out + r * ld_out + oc) = __floats2bfloat162_rn(y0, y1);
    const double d0 = v.x, d1 = v.y;
    s0 += d0;
    s1 += d1;
    q0 += d0 * d0;
    q1 += d1 * d1;
  }
  if (sums == nullptr) return;  // normalise-only launch (rollout side)
  atomicAdd(sums + c, s0);
  atomicAdd(sums + c + 1, s1);
  atomicAdd(sums + cols + c, q0);
  atomicAdd(sums + cols + c + 1, q1);
}

// (first, 0) into destination columns (oc, oc+1) of rows [r0, r1): zero padding, or the ones column of a bias-augmented operand
__device__ __forceinline__ void fill_pair_rows(__nv_bfloat16* __restrict__ out, long long ld_out, long long oc, long long r0, long long r1,
                                               float first) {
  const __nv_bfloat162 fill = __floats2bfloat162_rn(first, 0.0f);
  for (long long r = r0; r < r1; ++r) *reinterpret_cast<__nv_bfloat162*>(out + r * ld_out + oc) = fill;
}

__global__ void __launch_bounds__(256) normalize_moments_kernel(const float* __restrict__ x, long long ldx, long long rows, long long cols,
                                                                const float* __restrict__ mean, const float* __restrict__ rstd,
                                                                __nv_bfloat16* __restrict__ out, long long ld_out,
                                                                double* __restrict__ sums, float pad_one) {
  const long long c = 2 * ((long long)blockIdx.x * blockDim.x + threadIdx.x);
  if (c >= ld_out) return;
  const long long chunk = (rows + gridDim.y - 1) / gridDim.y;
  const long long r0 = blockIdx.y * chunk, r1 = min(rows, r0 + chunk);
  if (c < cols)  // cols is even on this path: a pair is either fully inside or fully padding
    normalize_pair_rows(x, ldx, cols, c, r0, r1, mean, rstd, out, ld_out, c, sums);
  else
    fill_pair_rows(out, ld_out, c, r0, r1, c == cols ? pad_one : 0.0f);   // (ones column | 0) on the first pad pair
}

// ---- split normalise for the task network of amp_sept (pulse_b200/sept.py) --------------------------------------------
// The observation [self | task] (self_cols even) feeds two bias-augmented first layers: the policy operand
// P = [embedding (p_off columns, written by the task network's top GEMM, not touched here) | self | 1 | 0...] and the task
// operand T = [task | 1 | 0...].  Thread j owns destination pair j of the concatenation P[:, p_off:ldp) ++ T[:, 0:ldt); every live pair
// maps to ONE source pair (the split is even), so this is normalize_moments_kernel with a remapped store and the same fp64 moments.
__global__ void __launch_bounds__(256) normalize_split_kernel(const float* __restrict__ x, long long ldx, long long rows, long long cols,
                                                              long long self_cols, const float* __restrict__ mean,
                                                              const float* __restrict__ rstd, __nv_bfloat16* __restrict__ p, long long ldp,
                                                              long long p_off, __nv_bfloat16* __restrict__ t, long long ldt,
                                                              double* __restrict__ sums) {
  const long long j = 2 * ((long long)blockIdx.x * blockDim.x + threadIdx.x);
  const long long pw = ldp - p_off;
  if (j >= pw + ldt) return;
  const long long chunk = (rows + gridDim.y - 1) / gridDim.y;
  const long long r0 = blockIdx.y * chunk, r1 = min(rows, r0 + chunk);
  const bool in_p = j < pw;
  __nv_bfloat16* out = in_p ? p : t;
  const long long ld = in_p ? ldp : ldt;
  const long long oc = in_p ? p_off + j : j - pw;
  const long long width = in_p ? self_cols : cols - self_cols;   // live columns of this operand
  const long long k = in_p ? j : j - pw;                         // column within this operand's live block
  if (k < width)
    normalize_pair_rows(x, ldx, cols, in_p ? k : self_cols + k, r0, r1, mean, rstd, out, ld, oc, sums);
  else
    fill_pair_rows(out, ld, oc, r0, r1, k == width ? 1.0f : 0.0f);
}

// ---- Gaussian head ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) gaussian_sample_kernel(const float* __restrict__ mu, long long ld_mu, const float* __restrict__ eps,
                                                              const float* __restrict__ logstd, long long rows, int A,
                                                              float* __restrict__ actions, float* __restrict__ neglogp) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float acc = 0.0f, ls = 0.0f;
  for (int k = lane; k < A; k += 32) {
    const float l = logstd[k];
    const float sg = expf(l);
    const float e = eps[row * A + k];
    const float m = mu[row * ld_mu + k];
    const float a = m + sg * e;
    actions[row * A + k] = a;
    const float z = (a - m) / sg;
    acc += z * z;
    ls += l;
  }
  acc = warp_sum(acc);
  ls = warp_sum(ls);
  if (lane == 0) neglogp[row] = 0.5f * acc + 0.5f * 1.8378770664093453f * A + ls;  // log(2*pi)
}

// ---- PPO losses + gradients w.r.t. mu / value ---------------------------------------------------------------------
// kPer actions per lane: 4 for A <= 128, 8 for A <= 256 (the SMPL-X dof-space policy's 153)
template <int kPer>
__global__ void __launch_bounds__(256) ppo_loss_kernel(const pulse_ppo_loss_args_t a, long long rows) {
  // Warps stride over the rows (a few rows each on a one-wave grid): the per-action constants are computed once per lane, the loss
  // statistics stay in registers until ONE set of fp64 atomics per block (six per 128-thread block serialise on six addresses).
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  __shared__ double s_stats[8][6];
  const int A = a.num_actions;
  float sg[kPer], inv_sg2[kPer], lsum = 0.0f;
#pragma unroll
  for (int q = 0; q < kPer; ++q) {
    const int k = lane + 32 * q;
    const float l = k < A ? a.logstd[k] : 0.0f;
    sg[q] = expf(l);
    inv_sg2[q] = 1.0f / (sg[q] * sg[q]);
    lsum += k < A ? l : 0.0f;
  }
  lsum = warp_sum(lsum);
  const float inv_rows = 1.0f / static_cast<float>(rows);
  double st[6] = {0, 0, 0, 0, 0, 0};
  for (long long row = warp0; row < rows; row += nwarps) {
    float m[kPer], act[kPer];
    float z2 = 0.0f, bl = 0.0f, kl = 0.0f;
    const float adv = a.advantages[row], old_nlp = a.old_neglogp[row], v = a.value[row * a.ld_value], ret = a.returns[row];   // in flight with the row
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      const int k = lane + 32 * q;
      if (k < A) {
        m[q] = a.mu[row * a.ld_mu + k];
        act[q] = a.actions[row * A + k];
        const float z = (act[q] - m[q]) / sg[q];
        z2 += z * z;
        const float hi = fmaxf(m[q] - 1.0f, 0.0f), lo = fminf(m[q] + 1.0f, 0.0f);
        bl += hi * hi + lo * lo;
        if (a.old_mu != nullptr) {
          // policy_kl(p0 = current, p1 = old) with equal sigma: log(s1/s0 + 1e-5) + (s0^2 + (mu1-mu0)^2)/(2(s1^2+1e-5)) - 0.5
          const float d = a.old_mu[row * A + k] - m[q];
          kl += logf(1.0f + 1e-5f) + (sg[q] * sg[q] + d * d) / (2.0f * (sg[q] * sg[q] + 1e-5f)) - 0.5f;
        }
      }
    }
    z2 = warp_sum(z2);
    bl = warp_sum(bl);
    kl = warp_sum(kl);
    const float nlp = 0.5f * z2 + 0.5f * 1.8378770664093453f * A + lsum;
    const float ratio = expf(old_nlp - nlp);
    const float rc = fminf(fmaxf(ratio, 1.0f - a.e_clip), 1.0f + a.e_clip);
    const float s1 = -adv * ratio, s2 = -adv * rc;
    const float a_loss = fmaxf(s1, s2);
    // d a_loss / d nlp: the unclipped branch is active when s1 >= s2 (torch.max sends the gradient there on ties);
    // the clipped branch has zero gradient unless ratio is inside the clip range, where both coincide.
    const float da_dnlp = (s1 >= s2) ? adv * ratio : 0.0f;
    const float c_loss = (ret - v) * (ret - v);
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      const int k = lane + 32 * q;
      if (k < A) {
        const float dnlp_dmu = -(act[q] - m[q]) * inv_sg2[q];
        const float hi = fmaxf(m[q] - 1.0f, 0.0f), lo = fminf(m[q] + 1.0f, 0.0f);
        const float g = (da_dnlp * dnlp_dmu + a.bounds_coef * 2.0f * (hi + lo)) * inv_rows;
        const __nv_bfloat16 gb = __float2bfloat16(g);
        if (a.dmu != nullptr) reinterpret_cast<__nv_bfloat16*>(a.dmu)[row * a.ld_dmu + k] = gb;
        if (a.dmu_t != nullptr) reinterpret_cast<__nv_bfloat16*>(a.dmu_t)[k * a.ld_dmu_t + row] = gb;
      }
    }
    if (lane == 0) {
      const __nv_bfloat16 gv = __float2bfloat16(-2.0f * (ret - v) * a.critic_coef * inv_rows);
      if (a.dvalue != nullptr) reinterpret_cast<__nv_bfloat16*>(a.dvalue)[row * a.ld_dv] = gv;
      if (a.dvalue_t != nullptr) reinterpret_cast<__nv_bfloat16*>(a.dvalue_t)[row] = gv;
      st[0] += a_loss;
      st[1] += c_loss;
      st[2] += bl;
      st[3] += kl;
      st[4] += fabsf(ratio - 1.0f) > a.e_clip ? 1.0 : 0.0;
      st[5] += nlp;
    }
  }
  if (lane == 0)
    for (int i = 0; i < 6; ++i) s_stats[warp][i] = st[i];
  __syncthreads();
  if (threadIdx.x < 6 && a.stats != nullptr) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += s_stats[w][threadIdx.x];
    atomicAdd(a.stats + threadIdx.x, t);
  }
}


// ---- column sums of a bf16 matrix (bias gradients) ------------------------------------------------------------------
// Block = 16 column groups (8 columns each, one 16-byte load) x 16 row lanes; blockIdx.y strides over row chunks.
__global__ void __launch_bounds__(256) column_sum_bf16_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, long long rows,
                                                              long long cols, float* __restrict__ out) {
  __shared__ float part[16][129];
  const int cg = threadIdx.x & 15, rl = threadIdx.x >> 4;
  const long long c0 = (long long)blockIdx.x * 128 + cg * 8;
  const long long chunk = (rows + gridDim.y - 1) / gridDim.y;
  const long long r0 = blockIdx.y * chunk, r1 = min(rows, r0 + chunk);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const bool vec = (ldx & 7) == 0 && c0 + 8 <= cols;
  if (c0 < cols) {
    for (long long r = r0 + rl; r < r1; r += 16) {
      const __nv_bfloat16* p = x + r * ldx + c0;
      if (vec) {
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 f = __bfloat1622float2(h[q]);
          acc[2 * q] += f.x;
          acc[2 * q + 1] += f.y;
        }
      } else {
        for (int q = 0; q < 8; ++q)
          if (c0 + q < cols) acc[q] += __bfloat162float(p[q]);
      }
    }
  }
#pragma unroll
  for (int q = 0; q < 8; ++q) part[rl][cg * 8 + q] = acc[q];
  __syncthreads();
  if (threadIdx.x < 128) {
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < 16; ++k) s += part[k][threadIdx.x];
    const long long c = (long long)blockIdx.x * 128 + threadIdx.x;
    if (c < cols) atomicAdd(out + c, s);
  }
}

// ---- RunningMeanStd training-mode merge (running_mean_std.py:54-66, :96-107), one CTA ----------------------------------
__global__ void __launch_bounds__(1024) rms_merge_kernel(double* __restrict__ sums, long long n, int size, double* __restrict__ mean,
                                                         double* __restrict__ var, double* __restrict__ count, float eps,
                                                         float* __restrict__ mean_f32, float* __restrict__ rstd_f32) {
  const double cnt = *count;
  const double tot = cnt + (double)n;
  for (int c = threadIdx.x; c < size; c += blockDim.x) {
    const double bm = sums[c] / (double)n;
    const double bv = (sums[size + c] - (double)n * bm * bm) / (double)(n - 1);  // unbiased, torch.var default
    const double delta = bm - mean[c];
    const double m2 = var[c] * cnt + bv * (double)n + delta * delta * cnt * (double)n / tot;
    const double nm = mean[c] + delta * (double)n / tot;
    const double nv = m2 / tot;
    mean[c] = nm;
    var[c] = nv;
    mean_f32[c] = (float)nm;
    rstd_f32[c] = 1.0f / sqrtf((float)nv + eps);
    sums[c] = 0.0;  // consumed: the accumulator is left zeroed for the next batch (no separate memset launch)
    sums[size + c] = 0.0;
  }
  __syncthreads();
  if (threadIdx.x == 0) *count = tot;
}

__global__ void __launch_bounds__(256) reduce_slabs_kernel(const float* __restrict__ slabs, long long slab_stride, int num_slabs,
                                                           long long count, float* __restrict__ dst) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
    float s = 0.0f;
    for (int k = 0; k < num_slabs; ++k) s += slabs[k * slab_stride + i];
    dst[i] = s;
  }
}

__global__ void __launch_bounds__(256) sum_squares_kernel(const float* __restrict__ x, long long count, double* __restrict__ out) {
  // fp64 multiplies run at a small fraction of the fp32 rate on this part: square in fp32 (exact enough: 24-bit operands, the sum of
  // eight products is then widened), accumulate the groups in fp64
  double s = 0.0;
  const long long n4 = ((reinterpret_cast<uintptr_t>(x) & 15u) == 0) ? count / 4 : 0;
  const float4* x4 = reinterpret_cast<const float4*>(x);
  const long long stride = (long long)gridDim.x * blockDim.x;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + stride < n4; i += 2 * stride) {
    const float4 a = __ldg(x4 + i), b = __ldg(x4 + i + stride);
    const float p = fmaf(a.x, a.x, fmaf(a.y, a.y, fmaf(a.z, a.z, a.w * a.w))) + fmaf(b.x, b.x, fmaf(b.y, b.y, fmaf(b.z, b.z, b.w * b.w)));
    s += static_cast<double>(p);
  }
  for (; i < n4; i += stride) {
    const float4 a = __ldg(x4 + i);
    s += static_cast<double>(fmaf(a.x, a.x, fmaf(a.y, a.y, fmaf(a.z, a.z, a.w * a.w))));
  }
  for (long long k = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; k < count; k += stride) s += static_cast<double>(x[k] * x[k]);
  s = warp_sum(s);
  __shared__ double ws[8];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < 8; ++k) t += ws[k];
    atomicAdd(out, t);
  }
}

__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
                                                   float* __restrict__ v, long long count, const double* __restrict__ sumsq, float max_norm,
                                                   float lr, float b1, float b2, float eps, const int* __restrict__ step_ptr,
                                                   __nv_bfloat16* __restrict__ p_bf16, int zero_grads, int* __restrict__ step_rw,
                                                   unsigned* __restrict__ block_counter, double* __restrict__ sumsq_rw) {
  // self-contained mode (block_counter != NULL): this launch IS optimizer step *step_ptr + 1; the last block to finish stores the new
  // step, re-zeroes the gradient-norm accumulator and its own counter -- no bump / memset launches around the update
  const float step = static_cast<float>(*step_ptr + (block_counter != nullptr ? 1 : 0));
  const float bc1 = 1.0f - powf(b1, step), bc2 = 1.0f - powf(b2, step);
  float scale = 1.0f;
  if (sumsq != nullptr && max_norm > 0.0f) {
    const float norm = static_cast<float>(sqrt(*sumsq));
    scale = fminf(1.0f, max_norm / (norm + 1e-6f));  // torch.nn.utils.clip_grad_norm_
  }
  const float lr1 = lr / bc1, rs2 = sqrtf(bc2);
  auto upd = [&](float gi, float& mi, float& vi, float& pi) {
    gi *= scale;
    mi = b1 * mi + (1.0f - b1) * gi;
    vi = b2 * vi + (1.0f - b2) * gi * gi;
    // torch.optim.Adam: p -= lr/bc1 * m / (sqrt(v)/sqrt(bc2) + eps)
    pi = pi - lr1 * mi / (sqrtf(vi) / rs2 + eps);
  };
  const long long n4 = count / 4;   // the flat buffers are 256-byte aligned and padded to multiples of 64 elements
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 g4 = reinterpret_cast<const float4*>(g)[i];
    float4 m4 = reinterpret_cast<float4*>(m)[i], v4 = reinterpret_cast<float4*>(v)[i], p4 = reinterpret_cast<float4*>(p)[i];
    upd(g4.x, m4.x, v4.x, p4.x);
    upd(g4.y, m4.y, v4.y, p4.y);
    upd(g4.z, m4.z, v4.z, p4.z);
    upd(g4.w, m4.w, v4.w, p4.w);
    reinterpret_cast<float4*>(m)[i] = m4;
    reinterpret_cast<float4*>(v)[i] = v4;
    reinterpret_cast<float4*>(p)[i] = p4;
    if (zero_grads) reinterpret_cast<float4*>(g)[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);   // consumed: the next minibatch accumulates from zero
    if (p_bf16 != nullptr) {  // the GEMM operand copy shares the flat layout
      __nv_bfloat162 lo = __floats2bfloat162_rn(p4.x, p4.y), hi = __floats2bfloat162_rn(p4.z, p4.w);
      uint2 u;
      u.x = *reinterpret_cast<unsigned*>(&lo);
      u.y = *reinterpret_cast<unsigned*>(&hi);
      reinterpret_cast<uint2*>(p_bf16)[i] = u;
    }
  }
  for (long long i = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
    float mi = m[i], vi = v[i], pi = p[i];
    upd(g[i], mi, vi, pi);
    m[i] = mi; v[i] = vi; p[i] = pi;
    if (zero_grads) g[i] = 0.0f;
    if (p_bf16 != nullptr) p_bf16[i] = __float2bfloat16(pi);
  }
  if (block_counter != nullptr) {
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      if (atomicAdd(block_counter, 1u) == gridDim.x - 1) {   // every block has read *step_ptr / *sumsq by now
        *step_rw = static_cast<int>(step);
        if (sumsq_rw != nullptr) *sumsq_rw = 0.0;
        *block_counter = 0u;
        __threadfence();
      }
    }
  }
}

__global__ void bump_step_kernel(int* step) { *step += 1; }

// ---- AMP discriminator: BCE-with-logits gradients (amp_agent.py:895-920, :935-952) -------------------------------------
// rows [0, n_agent) are agent / replay samples (target 0), rows [n_agent, n_agent + n_demo) demo samples (target 1).
// dlogit = scale * 0.5 * d/dl mean BCE;  stats: [sum softplus(l) agent, sum softplus(-l) demo, #agent l<0, #demo l>0].
__global__ void __launch_bounds__(256) disc_loss_kernel(const float* __restrict__ logits, long long ld, long long n_agent, long long n_demo,
                                                        float scale, __nv_bfloat16* __restrict__ dlogit, long long ld_d,
                                                        double* __restrict__ stats) {
  double st[4] = {0, 0, 0, 0};
  const long long n = n_agent + n_demo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float l = logits[i * ld];
    const float sg = 1.0f / (1.0f + expf(-l));
    const float sp = fmaxf(l, 0.0f) + log1pf(expf(-fabsf(l)));  // softplus(l), stable
    float g;
    if (i < n_agent) {
      g = 0.5f * scale * sg / static_cast<float>(n_agent);
      st[0] += sp;
      st[2] += l < 0.0f ? 1.0 : 0.0;
    } else {
      g = 0.5f * scale * (sg - 1.0f) / static_cast<float>(n_demo);
      st[1] += sp - l;  // softplus(-l)
      st[3] += l > 0.0f ? 1.0 : 0.0;
    }
    dlogit[i * ld_d] = __float2bfloat16(g);
  }
  __shared__ double ws[8][4];
#pragma unroll
  for (int k = 0; k < 4; ++k) st[k] = warp_sum(st[k]);
  if ((threadIdx.x & 31) == 0)
    for (int k = 0; k < 4; ++k) ws[threadIdx.x >> 5][k] = st[k];
  __syncthreads();
  if (threadIdx.x < 4 && stats != nullptr) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += ws[w][threadIdx.x];
    atomicAdd(stats + threadIdx.x, t);
  }
}

// out[r, c] = h[r, c] > 0 ? w[c] : 0   (first step of the analytic input gradient of a ReLU MLP: m2 * w_logit)
__global__ void __launch_bounds__(256) relu_mask_scale_kernel(const __nv_bfloat16* __restrict__ h, long long ldh, long long rows, long long cols,
                                                              const float* __restrict__ w, __nv_bfloat16* __restrict__ out, long long ldo) {
  const bool vec = (cols % 8) == 0 && (ldh % 8) == 0 && (ldo % 8) == 0 && (reinterpret_cast<uintptr_t>(h) % 16) == 0 &&
                   (reinterpret_cast<uintptr_t>(out) % 16) == 0;
  if (vec) {   // thread = (row, group of 8 columns): one 16-byte load and store
    const long long groups = cols / 8, total = rows * groups;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
      const long long r = i / groups, c = (i - r * groups) * 8;
      const uint4 u = *reinterpret_cast<const uint4*>(h + r * ldh + c);
      const unsigned wd[4] = {u.x, u.y, u.z, u.w};
      uint4 o;
      unsigned* od = reinterpret_cast<unsigned*>(&o);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        // bf16 > 0  <=>  sign clear and magnitude non-zero
        const bool p0 = (wd[q] & 0x8000u) == 0 && (wd[q] & 0x7fffu) != 0, p1 = (wd[q] & 0x80000000u) == 0 && (wd[q] & 0x7fff0000u) != 0;
        const __nv_bfloat162 v = __floats2bfloat162_rn(p0 ? w[c + 2 * q] : 0.0f, p1 ? w[c + 2 * q + 1] : 0.0f);
        od[q] = *reinterpret_cast<const unsigned*>(&v);
      }
      *reinterpret_cast<uint4*>(out + r * ldo + c) = o;
    }
    return;
  }
  const long long total = rows * cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols, c = i - r * cols;
    out[r * ldo + c] = __float2bfloat16(__bfloat162float(h[r * ldh + c]) > 0.0f ? w[c] : 0.0f);
  }
}
__global__ void __launch_bounds__(256) axpy_kernel(float a, const float* __restrict__ x, float* __restrict__ y, long long count) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) y[i] += a * x[i];
}

__global__ void __launch_bounds__(256) refresh_weight_kernel(const float* __restrict__ w, long long n, long long k,
                                                             __nv_bfloat16* __restrict__ wb, long long ld_k,
                                                             __nv_bfloat16* __restrict__ wt, long long ld_n) {
  __shared__ float tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const long long kt = (max(k, ld_k) + 31) / 32, nt = (max(n, ld_n) + 31) / 32;
  for (long long t = blockIdx.x; t < kt * nt; t += gridDim.x) {
    const long long rn = t / kt, ck = t - rn * kt;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const long long r = rn * 32 + ty + 8 * i, c = ck * 32 + tx;
      const float val = (r < n && c < k) ? w[r * k + c] : 0.0f;
      if (wb != nullptr && r < n && c < ld_k) wb[r * ld_k + c] = __float2bfloat16(val);
      tile[ty + 8 * i][tx] = val;
    }
    __syncthreads();
    if (wt != nullptr) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const long long c = ck * 32 + ty + 8 * i, r = rn * 32 + tx;  // wt[c][r]
        if (c < k && r < ld_n) wt[c * ld_n + r] = __float2bfloat16(tile[tx][ty + 8 * i]);
      }
    }
    __syncthreads();
  }
}

// ---- single-output head (critic value, discriminator logit): GEMV forward and ONE fused backward pass ---------------
// A [M,K] x [K,1] product has no tensor-core shape: a 128 x 128 MMA tile would be 127/128 padding and the three
// backward GEMMs (K = 1 dgrad, M = 1 wgrad) are pure epilogue / pure reduction.  Both directions are HBM streams
// over the last hidden activation h [M,K] bf16: forward reads it once; backward reads it once and writes dh once.
__global__ void __launch_bounds__(256) head1_forward_kernel(const __nv_bfloat16* __restrict__ h, long long ldh, long long rows, int K,
                                                            const __nv_bfloat16* __restrict__ w, const float* __restrict__ bias,
                                                            float* __restrict__ out, long long ldo) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const float b = bias != nullptr ? __ldg(bias) : 0.0f;
  constexpr int R = 4;                            // rows in flight per warp: the loads of all four are issued before any is consumed
  for (long long r0 = warp0 * R; r0 < rows; r0 += nwarps * R) {
    float acc[R] = {0.0f, 0.0f, 0.0f, 0.0f};
    for (int k = lane * 8; k < K; k += 256) {
      uint4 u[R];
#pragma unroll
      for (int i = 0; i < R; ++i)
        u[i] = (r0 + i < rows) ? __ldcs(reinterpret_cast<const uint4*>(h + (r0 + i) * ldh + k)) : make_uint4(0u, 0u, 0u, 0u);
      const uint4 wu = __ldg(reinterpret_cast<const uint4*>(w + k));
      const __nv_bfloat162* w2 = reinterpret_cast<const __nv_bfloat162*>(&wu);
#pragma unroll
      for (int i = 0; i < R; ++i) {
        const __nv_bfloat162* a2 = reinterpret_cast<const __nv_bfloat162*>(&u[i]);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 a = __bfloat1622float2(a2[q]), ww = __bfloat1622float2(w2[q]);
          acc[i] = fmaf(a.x, ww.x, acc[i]);
          acc[i] = fmaf(a.y, ww.y, acc[i]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const float t = warp_sum(acc[i]);
      if (lane == 0 && r0 + i < rows) out[(r0 + i) * ldo] = t + b;
    }
  }
}


// dh[m,k] = dv[m] * w[k] * (h[m,k] > 0);  dw[k] += sum_m dv[m] h[m,k];  db += sum_m dv[m];  dbias_prev[k] += sum_m dh[m,k].
// Thread = 8 columns (one 16-byte load / store); blockDim.x / (K/8) row lanes per CTA.  Each CTA writes its column sums to its own
// row of `partials` [gridDim.x][2K + 1]; ordered_sum_kernel then adds the rows in CTA order, so the sums do not depend on scheduling.
__global__ void __launch_bounds__(256) head1_backward_kernel(const __nv_bfloat16* __restrict__ h, long long ldh, long long rows, int K,
                                                             const __nv_bfloat16* __restrict__ dv, long long ld_dv,
                                                             const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ dh, long long ld_dh,
                                                             float* __restrict__ partials) {
  extern __shared__ float red[];  // [row lanes][2 * K + 1]
  const int groups = K >> 3;                     // column groups of 8
  const int lanes = blockDim.x / groups;         // row lanes per CTA (host guarantees >= 1)
  const int cg = threadIdx.x % groups, rl = threadIdx.x / groups;
  const long long chunk = (rows + gridDim.x - 1) / gridDim.x;
  const long long r0 = (long long)blockIdx.x * chunk, r1 = min(rows, r0 + chunk);
  float aw[8] = {0, 0, 0, 0, 0, 0, 0, 0}, ac[8] = {0, 0, 0, 0, 0, 0, 0, 0}, adb = 0.0f;
  if (rl < lanes) {
    float wf[8];
    {
      const uint4 wu = __ldg(reinterpret_cast<const uint4*>(w + cg * 8));
      const __nv_bfloat162* w2 = reinterpret_cast<const __nv_bfloat162*>(&wu);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 f = __bfloat1622float2(w2[q]);
        wf[2 * q] = f.x;
        wf[2 * q + 1] = f.y;
      }
    }
    constexpr int R = 4;   // rows in flight per thread: one 16-byte load each, all issued before the first is consumed
    for (long long rb = r0 + rl; rb < r1; rb += (long long)lanes * R) {
      uint4 u[R];
      float dd[R];
#pragma unroll
      for (int i = 0; i < R; ++i) {
        const long long r = rb + (long long)i * lanes;
        const bool ok = r < r1;
        u[i] = ok ? __ldcs(reinterpret_cast<const uint4*>(h + r * ldh + cg * 8)) : make_uint4(0u, 0u, 0u, 0u);
        dd[i] = ok ? __bfloat162float(dv[r * ld_dv]) : 0.0f;
      }
#pragma unroll
      for (int i = 0; i < R; ++i) {
        const long long r = rb + (long long)i * lanes;
        if (r >= r1) break;
        const float d = dd[i];
        const __nv_bfloat162* a2 = reinterpret_cast<const __nv_bfloat162*>(&u[i]);
        float o[8];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 a = __bfloat1622float2(a2[q]);
          aw[2 * q] = fmaf(d, a.x, aw[2 * q]);
          aw[2 * q + 1] = fmaf(d, a.y, aw[2 * q + 1]);
          o[2 * q] = a.x > 0.0f ? d * wf[2 * q] : 0.0f;
          o[2 * q + 1] = a.y > 0.0f ? d * wf[2 * q + 1] : 0.0f;
          ac[2 * q] += o[2 * q];
          ac[2 * q + 1] += o[2 * q + 1];
        }
        if (dh != nullptr) {
          __nv_bfloat162 p0 = __floats2bfloat162_rn(o[0], o[1]), p1 = __floats2bfloat162_rn(o[2], o[3]);
          __nv_bfloat162 p2 = __floats2bfloat162_rn(o[4], o[5]), p3 = __floats2bfloat162_rn(o[6], o[7]);
          uint4 st;
          st.x = *reinterpret_cast<unsigned*>(&p0);
          st.y = *reinterpret_cast<unsigned*>(&p1);
          st.z = *reinterpret_cast<unsigned*>(&p2);
          st.w = *reinterpret_cast<unsigned*>(&p3);
          *reinterpret_cast<uint4*>(dh + r * ld_dh + cg * 8) = st;
        }
        if (cg == 0) adb += d;
      }
    }
    float* mine = red + (long long)rl * (2 * K + 1);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      mine[cg * 8 + q] = aw[q];
      mine[K + cg * 8 + q] = ac[q];
    }
    if (cg == 0) mine[2 * K] = adb;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * K + 1; i += blockDim.x) {
    float t = 0.0f;
    for (int l = 0; l < lanes; ++l) t += red[(long long)l * (2 * K + 1) + i];
    partials[(long long)blockIdx.x * (2 * K + 1) + i] = t;
  }
}

// out[r, c] += sum_{s < n} x[s * stride_n + r * ld + c], the n terms added in the order s = 0, 1, ...: a reduction whose result does not
// depend on how the producing CTAs were scheduled (split-K slabs, per-CTA partial sums), so repeated runs compute identical bits.
__global__ void __launch_bounds__(256) ordered_sum_kernel(const float* __restrict__ x, long long n, long long stride_n, long long rows,
                                                          long long cols, long long ld, float* __restrict__ out, long long ldo) {
  const long long total = rows * cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols, c = i - r * cols;
    const float* p = x + r * ld + c;
    float s = 0.0f;
#pragma unroll 8
    for (long long k = 0; k < n; ++k) s += __ldg(p + k * stride_n);
    out[r * ldo + c] += s;
  }
}

}  // namespace
}  // namespace pulse

using namespace pulse;

extern "C" int pulse_normalize_to_bf16(const float* x, int64_t ldx, int64_t rows, int64_t cols, const float* mean, const float* rstd,
                                       pulse_bf16_t* out, int64_t ld_out, pulse_bf16_t* out_t, int64_t ld_t, float pad_one, void* stream) {
  PULSE_REQUIRE(x && (out || out_t), "pulse_normalize_to_bf16: null buffer");
  PULSE_REQUIRE(rows > 0 && cols > 0 && ld_out >= cols && ldx >= cols, "pulse_normalize_to_bf16: bad shape");
  PULSE_REQUIRE((mean == nullptr) == (rstd == nullptr), "pulse_normalize_to_bf16: mean and rstd go together");
  PULSE_REQUIRE(out_t == nullptr || ld_t >= rows, "pulse_normalize_to_bf16: ld_t < rows");
  const bool paired = mean != nullptr && out != nullptr && out_t == nullptr && (cols % 2 == 0) && (ldx % 2 == 0) && (ld_out % 2 == 0) &&
                      (reinterpret_cast<uintptr_t>(x) % 8 == 0) && (reinterpret_cast<uintptr_t>(out) % 4 == 0) &&
                      (reinterpret_cast<uintptr_t>(mean) % 8 == 0) && (reinterpret_cast<uintptr_t>(rstd) % 8 == 0);
  if (paired) {  // column-pair streaming kernel (8-byte loads, 8 rows in flight per thread)
    const unsigned gx = static_cast<unsigned>((ld_out / 2 + 255) / 256);
    unsigned gy = (2 * kSMs + gx - 1) / gx;
    if (gy > rows / 8) gy = static_cast<unsigned>(rows / 8);
    if (gy < 1) gy = 1;
    normalize_moments_kernel<<<dim3(gx, gy), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x, ldx, rows, cols, mean, rstd, reinterpret_cast<__nv_bfloat16*>(out), ld_out, nullptr, pad_one);
    PULSE_LAUNCH_OK("normalize_moments_kernel");
    return PULSE_OK;
  }
  const long long tiles = ((ld_out + 31) / 32) * ((rows + 31) / 32);
  normalize_kernel<<<grid_for(tiles, 1, 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, ldx, rows, cols, mean, rstd, reinterpret_cast<__nv_bfloat16*>(out), ld_out, reinterpret_cast<__nv_bfloat16*>(out_t), ld_t, pad_one);
  PULSE_LAUNCH_OK("normalize_kernel");
  return PULSE_OK;
}

extern "C" int pulse_column_moments(const float* x, int64_t ldx, int64_t rows, int64_t cols, double* sums, void* stream) {
  PULSE_REQUIRE(x && sums && rows > 0 && cols > 0, "pulse_column_moments: bad argument");
  dim3 grid(static_cast<unsigned>((cols + 255) / 256), static_cast<unsigned>(rows >= 4096 ? 128 : 1));
  column_moments_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, ldx, rows, cols, sums);
  PULSE_LAUNCH_OK("column_moments_kernel");
  return PULSE_OK;
}

extern "C" int pulse_normalize_moments(const float* x, int64_t ldx, int64_t rows, int64_t cols, const float* mean, const float* rstd,
                                       pulse_bf16_t* out, int64_t ld_out, double* sums, float pad_one, void* stream) {
  PULSE_REQUIRE(x && mean && rstd && out && sums, "pulse_normalize_moments: null buffer");
  PULSE_REQUIRE(rows > 0 && cols > 0 && ld_out >= cols && ldx >= cols, "pulse_normalize_moments: bad shape");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool paired = (cols % 2 == 0) && (ldx % 2 == 0) && (ld_out % 2 == 0) && (reinterpret_cast<uintptr_t>(x) % 8 == 0) &&
                      (reinterpret_cast<uintptr_t>(out) % 4 == 0) && (reinterpret_cast<uintptr_t>(mean) % 8 == 0) &&
                      (reinterpret_cast<uintptr_t>(rstd) % 8 == 0);
  if (!paired) {  // odd widths / unaligned views: the two single-purpose kernels (same results, two passes)
    const int rc = pulse_normalize_to_bf16(x, ldx, rows, cols, mean, rstd, out, ld_out, nullptr, 0, pad_one, stream);
    if (rc != PULSE_OK) return rc;
    return pulse_column_moments(x, ldx, rows, cols, sums, stream);
  }
  const unsigned gx = static_cast<unsigned>((ld_out / 2 + 255) / 256);
  unsigned gy = (2 * kSMs + gx - 1) / gx;  // two 256-thread CTAs per SM, 8 x 8-byte loads in flight per thread
  if (gy > rows / 8) gy = static_cast<unsigned>(rows / 8);
  if (gy < 1) gy = 1;
  normalize_moments_kernel<<<dim3(gx, gy), 256, 0, st>>>(x, ldx, rows, cols, mean, rstd, reinterpret_cast<__nv_bfloat16*>(out), ld_out, sums, pad_one);
  PULSE_LAUNCH_OK("normalize_moments_kernel");
  return PULSE_OK;
}

extern "C" int pulse_normalize_split(const float* x, int64_t ldx, int64_t rows, int64_t cols, int64_t self_cols, const float* mean,
                                     const float* rstd, pulse_bf16_t* p, int64_t ldp, int64_t p_off, pulse_bf16_t* t, int64_t ldt, double* sums,
                                     void* stream) {
  PULSE_REQUIRE(x && mean && rstd && p && t, "pulse_normalize_split: null buffer");
  PULSE_REQUIRE(rows > 0 && self_cols > 0 && cols > self_cols && ldx >= cols, "pulse_normalize_split: bad shape");
  PULSE_REQUIRE(p_off >= 0 && ldp > p_off + self_cols && ldt > cols - self_cols, "pulse_normalize_split: operands too narrow for the ones column");
  PULSE_REQUIRE(cols % 2 == 0 && self_cols % 2 == 0 && p_off % 2 == 0 && ldp % 2 == 0 && ldt % 2 == 0 && ldx % 2 == 0,
                "pulse_normalize_split: cols, self_cols, p_off, ldp, ldt and ldx must be even");
  PULSE_REQUIRE(reinterpret_cast<uintptr_t>(x) % 8 == 0 && reinterpret_cast<uintptr_t>(mean) % 8 == 0 && reinterpret_cast<uintptr_t>(rstd) % 8 == 0 &&
                    reinterpret_cast<uintptr_t>(p) % 4 == 0 && reinterpret_cast<uintptr_t>(t) % 4 == 0,
                "pulse_normalize_split: x / mean / rstd need 8-byte, p / t 4-byte alignment");
  const unsigned gx = static_cast<unsigned>(((ldp - p_off + ldt) / 2 + 255) / 256);
  unsigned gy = (2 * kSMs + gx - 1) / gx;  // as pulse_normalize_moments: two 256-thread CTAs per SM, 8 rows in flight per thread
  if (gy > rows / 8) gy = static_cast<unsigned>(rows / 8);
  if (gy < 1) gy = 1;
  normalize_split_kernel<<<dim3(gx, gy), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, ldx, rows, cols, self_cols, mean, rstd, reinterpret_cast<__nv_bfloat16*>(p), ldp, p_off, reinterpret_cast<__nv_bfloat16*>(t), ldt, sums);
  PULSE_LAUNCH_OK("normalize_split_kernel");
  return PULSE_OK;
}

extern "C" int pulse_head1_forward(const pulse_bf16_t* h, int64_t ldh, int64_t rows, int32_t k, const pulse_bf16_t* w, const float* bias,
                                   float* out, int64_t ldo, void* stream) {
  PULSE_REQUIRE(h && w && out && rows > 0 && k > 0 && ldo >= 1, "pulse_head1_forward: bad argument");
  PULSE_REQUIRE(k % 8 == 0 && ldh % 8 == 0 && reinterpret_cast<uintptr_t>(h) % 16 == 0 && reinterpret_cast<uintptr_t>(w) % 16 == 0,
                "pulse_head1_forward: K, ldh multiples of 8 and 16-byte aligned operands required");
  head1_forward_kernel<<<grid_for(rows, 8, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(h), ldh, rows, k, reinterpret_cast<const __nv_bfloat16*>(w), bias, out, ldo);
  PULSE_LAUNCH_OK("head1_forward_kernel");
  return PULSE_OK;
}

extern "C" int pulse_head1_backward(const pulse_bf16_t* h, int64_t ldh, int64_t rows, int32_t k, const pulse_bf16_t* dv, int64_t ld_dv,
                                    const pulse_bf16_t* w, pulse_bf16_t* dh, int64_t ld_dh, float* dw, float* db, float* dbias_prev,
                                    float* partials, void* stream) {
  PULSE_REQUIRE(h && dv && w && dw && partials && rows > 0 && k > 0 && ld_dv >= 1, "pulse_head1_backward: bad argument");
  PULSE_REQUIRE(k % 8 == 0 && k <= 2048 && ldh % 8 == 0 && (dh == nullptr || ld_dh % 8 == 0), "pulse_head1_backward: K <= 2048, K and lds multiples of 8");
  PULSE_REQUIRE(reinterpret_cast<uintptr_t>(h) % 16 == 0 && reinterpret_cast<uintptr_t>(w) % 16 == 0 && reinterpret_cast<uintptr_t>(dh) % 16 == 0,
                "pulse_head1_backward: 16-byte aligned operands required");
  const int groups = k / 8, lanes = 256 / groups;
  const size_t smem = static_cast<size_t>(lanes) * (2 * k + 1) * sizeof(float);
  long long blocks = (rows + 8LL * lanes - 1) / (8LL * lanes);  // >= 8 rows per row lane
  if (blocks > PULSE_HEAD1_MAX_CTAS) blocks = PULSE_HEAD1_MAX_CTAS;
  if (blocks < 1) blocks = 1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  head1_backward_kernel<<<static_cast<unsigned>(blocks), 256, smem, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(h), ldh, rows, k, reinterpret_cast<const __nv_bfloat16*>(dv), ld_dv,
      reinterpret_cast<const __nv_bfloat16*>(w), reinterpret_cast<__nv_bfloat16*>(dh), ld_dh, partials);
  PULSE_LAUNCH_OK("head1_backward_kernel");
  const long long row = 2LL * k + 1;
  ordered_sum_kernel<<<static_cast<unsigned>((k + 255) / 256), 256, 0, st>>>(partials, blocks, row, 1, k, 0, dw, 0);
  PULSE_LAUNCH_OK("ordered_sum_kernel");
  if (dbias_prev != nullptr) {
    ordered_sum_kernel<<<static_cast<unsigned>((k + 255) / 256), 256, 0, st>>>(partials + k, blocks, row, 1, k, 0, dbias_prev, 0);
    PULSE_LAUNCH_OK("ordered_sum_kernel");
  }
  if (db != nullptr) {
    ordered_sum_kernel<<<1, 32, 0, st>>>(partials + 2 * k, blocks, row, 1, 1, 0, db, 0);
    PULSE_LAUNCH_OK("ordered_sum_kernel");
  }
  return PULSE_OK;
}

extern "C" int pulse_ordered_sum_add(const float* x, int64_t n, int64_t stride_n, int64_t rows, int64_t cols, int64_t ld, float* out, int64_t ldo,
                                     void* stream) {
  PULSE_REQUIRE(x && out && n > 0 && rows > 0 && cols > 0 && (rows == 1 || (ld >= cols && ldo >= cols)), "pulse_ordered_sum_add: bad argument");
  ordered_sum_kernel<<<grid_for(rows * cols, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, n, stride_n, rows, cols, ld, out, ldo);
  PULSE_LAUNCH_OK("ordered_sum_kernel");
  return PULSE_OK;
}

extern "C" int pulse_gaussian_sample(const float* mu, int64_t ld_mu, const float* eps, const float* logstd, int64_t rows,
                                     int32_t num_actions, float* actions, float* neglogp, void* stream) {
  PULSE_REQUIRE(mu && eps && logstd && actions && neglogp && rows > 0 && num_actions > 0, "pulse_gaussian_sample: bad argument");
  gaussian_sample_kernel<<<static_cast<unsigned>((rows * 32 + 127) / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      mu, ld_mu, eps, logstd, rows, num_actions, actions, neglogp);
  PULSE_LAUNCH_OK("gaussian_sample_kernel");
  return PULSE_OK;
}

extern "C" int pulse_ppo_loss(const pulse_ppo_loss_args_t* args, int64_t rows, void* stream) {
  PULSE_REQUIRE(args != nullptr && rows > 0, "pulse_ppo_loss: bad argument");
  const pulse_ppo_loss_args_t& a = *args;
  PULSE_REQUIRE(a.mu && a.value && a.actions && a.old_neglogp && a.advantages && a.returns && a.logstd, "pulse_ppo_loss: null input");
  PULSE_REQUIRE(a.num_actions > 0 && a.num_actions <= 256, "pulse_ppo_loss: num_actions %d outside [1,256]", a.num_actions);
  PULSE_REQUIRE(a.ld_mu >= a.num_actions && a.ld_value >= 1 && (a.dmu == nullptr || a.ld_dmu >= a.num_actions),
                "pulse_ppo_loss: leading dimensions too small");
  // 8 warps per block, one row per warp at a time; 8 blocks per SM are all resident (2048 threads per SM)
  if (a.num_actions <= 128) {
    ppo_loss_kernel<4><<<grid_for(rows, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, rows);
    PULSE_LAUNCH_OK("ppo_loss_kernel<4>");
  } else {
    ppo_loss_kernel<8><<<grid_for(rows, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, rows);
    PULSE_LAUNCH_OK("ppo_loss_kernel<8>");
  }
  return PULSE_OK;
}

extern "C" int pulse_column_sum_bf16(const pulse_bf16_t* x, int64_t ldx, int64_t rows, int64_t cols, float* out, void* stream) {
  PULSE_REQUIRE(x && out && rows > 0 && cols > 0, "pulse_column_sum_bf16: bad argument");
  const unsigned gx = static_cast<unsigned>((cols + 127) / 128);
  unsigned gy = static_cast<unsigned>((rows + 31) / 32);  // >= 2 rows per lane: short chunks, many CTAs (latency-bound otherwise)
  const unsigned cap = (4 * kSMs + gx - 1) / gx;
  if (gy > cap) gy = cap;
  if (gy < 1) gy = 1;
  dim3 grid(gx, gy);
  column_sum_bf16_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const __nv_bfloat16*>(x), ldx, rows, cols, out);
  PULSE_LAUNCH_OK("column_sum_bf16_kernel");
  return PULSE_OK;
}

extern "C" int pulse_rms_merge(double* sums, int64_t n, int32_t size, double* mean, double* var, double* count, float eps,
                               float* mean_f32, float* rstd_f32, void* stream) {
  PULSE_REQUIRE(sums && mean && var && count && mean_f32 && rstd_f32 && n >= 2 && size > 0, "pulse_rms_merge: bad argument");
  rms_merge_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(sums, n, size, mean, var, count, eps, mean_f32, rstd_f32);
  PULSE_LAUNCH_OK("rms_merge_kernel");
  return PULSE_OK;
}

extern "C" int pulse_reduce_slabs(const float* slabs, int64_t slab_stride, int32_t num_slabs, int64_t count, float* dst, void* stream) {
  PULSE_REQUIRE(slabs && dst && num_slabs >= 1 && count > 0, "pulse_reduce_slabs: bad argument");
  reduce_slabs_kernel<<<grid_for(count, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(slabs, slab_stride, num_slabs, count, dst);
  PULSE_LAUNCH_OK("reduce_slabs_kernel");
  return PULSE_OK;
}

extern "C" int pulse_sum_squares(const float* x, int64_t count, double* sumsq, void* stream) {
  PULSE_REQUIRE(x && sumsq && count > 0, "pulse_sum_squares: bad argument");
  sum_squares_kernel<<<grid_for(count, 256 * 8, 4), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, count, sumsq);
  PULSE_LAUNCH_OK("sum_squares_kernel");
  return PULSE_OK;
}

extern "C" int pulse_adam_step(float* params, float* grads, float* exp_avg, float* exp_avg_sq, int64_t count,
                               double* grad_sumsq, float max_norm, float lr, float beta1, float beta2, float eps, int32_t* step,
                               pulse_bf16_t* params_bf16, uint32_t flags, uint32_t* block_counter, void* stream) {
  PULSE_REQUIRE(params && grads && exp_avg && exp_avg_sq && count > 0 && step != nullptr, "pulse_adam_step: bad argument");
  PULSE_REQUIRE((flags & ~3u) == 0, "pulse_adam_step: bad flags");
  PULSE_REQUIRE(!(flags & PULSE_ADAM_SELF_CONTAINED) || block_counter != nullptr, "pulse_adam_step: the self-contained mode needs block_counter");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool self = (flags & PULSE_ADAM_SELF_CONTAINED) != 0;
  if (!self) {
    bump_step_kernel<<<1, 1, 0, st>>>(step);
    PULSE_LAUNCH_OK("bump_step_kernel");
  }
  adam_kernel<<<grid_for(count, 256 * 4), 256, 0, st>>>(params, grads, exp_avg, exp_avg_sq, count, grad_sumsq, max_norm, lr, beta1, beta2, eps, step,
                                                        reinterpret_cast<__nv_bfloat16*>(params_bf16), (flags & PULSE_ADAM_ZERO_GRADS) ? 1 : 0, step,
                                                        self ? block_counter : nullptr, self ? grad_sumsq : nullptr);
  PULSE_LAUNCH_OK("adam_kernel");
  return PULSE_OK;
}

extern "C" int pulse_disc_loss(const float* logits, int64_t ld, int64_t n_agent, int64_t n_demo, float scale, pulse_bf16_t* dlogit,
                               int64_t ld_d, double* stats, void* stream) {
  PULSE_REQUIRE(logits && dlogit && n_agent > 0 && n_demo > 0 && ld >= 1 && ld_d >= 1, "pulse_disc_loss: bad argument");
  disc_loss_kernel<<<grid_for(n_agent + n_demo, 256, 2), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      logits, ld, n_agent, n_demo, scale, reinterpret_cast<__nv_bfloat16*>(dlogit), ld_d, stats);
  PULSE_LAUNCH_OK("disc_loss_kernel");
  return PULSE_OK;
}

extern "C" int pulse_relu_mask_scale(const pulse_bf16_t* h, int64_t ldh, int64_t rows, int64_t cols, const float* w, pulse_bf16_t* out,
                                     int64_t ldo, void* stream) {
  PULSE_REQUIRE(h && w && out && rows > 0 && cols > 0, "pulse_relu_mask_scale: bad argument");
  relu_mask_scale_kernel<<<grid_for(rows * cols, 256 * 4), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(h), ldh, rows, cols, w, reinterpret_cast<__nv_bfloat16*>(out), ldo);
  PULSE_LAUNCH_OK("relu_mask_scale_kernel");
  return PULSE_OK;
}

// Weight regularisers of the AMP discriminator (amp_agent.py:905-908, :932-937) for up to four weight blocks in ONE launch:
// g[r, c] += coef * w[r, c] over the [rows, cols] sub-block of a [rows, ld] matrix (the bias column / zero padding of an augmented
// layer stay out of it) and the fp64 sums of squares the logged loss terms need.
namespace pulse {
namespace {
__global__ void __launch_bounds__(256) weight_reg_kernel(const pulse_weight_reg_t d) {
  double sq = 0.0;
  const pulse_weight_block_t& b = d.block[blockIdx.y];
  const long long stride = (long long)gridDim.x * blockDim.x, t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool vec = (b.cols % 4) == 0 && (b.ld % 4) == 0 && (reinterpret_cast<uintptr_t>(b.w) % 16) == 0 &&
                   (b.g == nullptr || (reinterpret_cast<uintptr_t>(b.g) % 16) == 0);
  if (vec) {   // thread = (row, 4 columns): independent 16-byte read-modify-writes, many in flight per thread
    const long long c4 = b.cols / 4, total = b.rows * c4;
    for (long long i = t0; i < total; i += stride) {
      const long long r = i / c4, c = (i - r * c4) * 4;
      const float4 w = *reinterpret_cast<const float4*>(b.w + r * b.ld + c);
      if (b.g != nullptr) {
        float4 g = *reinterpret_cast<float4*>(b.g + r * b.ld + c);
        g.x += b.coef * w.x; g.y += b.coef * w.y; g.z += b.coef * w.z; g.w += b.coef * w.w;
        *reinterpret_cast<float4*>(b.g + r * b.ld + c) = g;
      }
      sq += static_cast<double>(fmaf(w.x, w.x, fmaf(w.y, w.y, fmaf(w.z, w.z, w.w * w.w))));
    }
  } else {
    const long long total = b.rows * b.cols;
    for (long long i = t0; i < total; i += stride) {
      const long long r = i / b.cols, c = i - r * b.cols;
      const float w = b.w[r * b.ld + c];
      if (b.g != nullptr) b.g[r * b.ld + c] += b.coef * w;
      sq += static_cast<double>(w * w);
    }
  }
  sq = warp_sum(sq);
  __shared__ double part_s[8];
  if ((threadIdx.x & 31) == 0) part_s[threadIdx.x >> 5] = sq;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < 8; ++k) t += part_s[k];
    if (b.sumsq != nullptr) atomicAdd(b.sumsq, t);
    if (b.sumsq2 != nullptr) atomicAdd(b.sumsq2, t);
  }
}
}  // namespace
}  // namespace pulse

extern "C" int pulse_weight_reg(const pulse_weight_reg_t* desc, void* stream) {
  PULSE_REQUIRE(desc != nullptr && desc->count >= 1 && desc->count <= 4, "pulse_weight_reg: 1..4 blocks");
  for (int i = 0; i < desc->count; ++i) {
    const pulse_weight_block_t& b = desc->block[i];
    PULSE_REQUIRE(b.w != nullptr && b.rows > 0 && b.cols > 0 && b.ld >= b.cols, "pulse_weight_reg: bad block %d", i);
  }
  weight_reg_kernel<<<dim3(4 * kSMs, static_cast<unsigned>(desc->count)), 256, 0, static_cast<cudaStream_t>(stream)>>>(*desc);
  PULSE_LAUNCH_OK("weight_reg_kernel");
  return PULSE_OK;
}

extern "C" int pulse_axpy(float a, const float* x, float* y, int64_t count, void* stream) {
  PULSE_REQUIRE(x && y && count > 0, "pulse_axpy: bad argument");
  axpy_kernel<<<grid_for(count, 256 * 4), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, x, y, count);
  PULSE_LAUNCH_OK("axpy_kernel");
  return PULSE_OK;
}

extern "C" int pulse_refresh_weight_bf16(const float* w, int64_t n, int64_t k, pulse_bf16_t* w_bf16, int64_t ld_k, pulse_bf16_t* wt_bf16,
                                         int64_t ld_n, void* stream) {
  PULSE_REQUIRE(w && (w_bf16 || wt_bf16) && n > 0 && k > 0, "pulse_refresh_weight_bf16: bad argument");
  PULSE_REQUIRE((!w_bf16 || ld_k >= k) && (!wt_bf16 || ld_n >= n), "pulse_refresh_weight_bf16: leading dimension too small");
  const long long tiles = ((std::max<long long>(k, ld_k) + 31) / 32) * ((std::max<long long>(n, ld_n) + 31) / 32);
  refresh_weight_kernel<<<grid_for(tiles, 1, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      w, n, k, reinterpret_cast<__nv_bfloat16*>(w_bf16), ld_k, reinterpret_cast<__nv_bfloat16*>(wt_bf16), ld_n);
  PULSE_LAUNCH_OK("refresh_weight_kernel");
  return PULSE_OK;
}
