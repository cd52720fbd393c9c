// The value de-normalisation shared by the rollout post kernels (rollout_ops.cu, ztask_rollout.cu).
#pragma once

namespace pulse {

// RunningMeanStd.forward(unnorm=True): clamp(y, -5, 5) * sqrt(var.float() + eps) + mean.float()
__device__ __forceinline__ float value_unnorm(float y, const double* mean, const double* var, float eps) {
  if (mean == nullptr) return y;
  const float sd = sqrtf(__fadd_rn(static_cast<float>(var[0]), eps));
  return __fadd_rn(__fmul_rn(fminf(fmaxf(y, -5.0f), 5.0f), sd), static_cast<float>(mean[0]));
}

}  // namespace pulse
