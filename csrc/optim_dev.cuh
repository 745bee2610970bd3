// Per-element local-optimizer math shared by the single-GPU fused optimizer (fused_ops.cu) and the fused
// reduce-scatter + optimizer + all-gather NVLink kernel (comm.cu).
#pragma once
#include "fused_ops.h"

namespace pb {

// kind 0 = ADOPT, 1 = DecoupledAdamW, 2 = SGD. gg is the (already clipped / unscaled) gradient.
__device__ __forceinline__ void optim_update4(float (&pp)[4], const float (&gg)[4], float (&mm)[4], float (&vv)[4], const OptimHyper& h) {
  if (h.kind == 2) {
#pragma unroll
    for (int k = 0; k < 4; ++k) pp[k] = pp[k] * h.decay - h.lr * gg[k];
  } else if (h.kind == 0) {  // ADOPT
    // coupled weight decay enters the gradient before anything reads it: the step-0 seed of v as well as the update
    float g[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) g[k] = h.wd != 0.f ? fmaf(h.wd, pp[k], gg[k]) : gg[k];
    if (h.first_step) {
#pragma unroll
      for (int k = 0; k < 4; ++k) vv[k] = g[k] * g[k];
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float ng = g[k] / fmaxf(sqrtf(vv[k]), h.eps);
        ng = fminf(fmaxf(ng, -h.clip), h.clip);
        mm[k] = mm[k] + (1.0f - h.beta1) * (ng - mm[k]);
        pp[k] = pp[k] * h.decay - h.lr * mm[k];
        vv[k] = h.beta2 * vv[k] + (1.0f - h.beta2) * g[k] * g[k];
      }
    }
  } else {  // DecoupledAdamW
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      pp[k] *= h.decay;
      mm[k] = mm[k] + (1.0f - h.beta1) * (gg[k] - mm[k]);
      vv[k] = h.beta2 * vv[k] + (1.0f - h.beta2) * gg[k] * gg[k];
      const float denom = sqrtf(vv[k]) * h.inv_sqrt_bc2 + h.eps;
      pp[k] -= h.step_size * mm[k] / denom;
    }
  }
}

}  // namespace pb
