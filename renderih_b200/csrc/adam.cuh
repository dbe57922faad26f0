// The per-element Adam / AdamW update shared by rih_adamw_step (token_ops.cu) and rih_ge_adam_step (ge_optim.cu).
#pragma once

namespace rih {

// torch.optim.AdamW's single-tensor update of one element (torch/optim/adamw.py); with decay == 1 (weight_decay = 0) it is Adam's.
// step_size = lr / (1 - beta1^t) and bc2_sqrt = sqrt(1 - beta2^t) are formed in double by the caller and rounded to float once.
__device__ __forceinline__ void adam_update(float& p, float& m, float& v, float g, float decay, float b1, float omb1, float b2, float omb2,
                                            float eps, float step_size, float bc2_sqrt) {
  float pi = p * decay;                          // decoupled weight decay: p *= 1 - lr * wd
  float mi = b1 * m + omb1 * g;                  // exp_avg.lerp_(grad, 1 - beta1)
  float vi = b2 * v + omb2 * g * g;              // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value = 1 - beta2)
  m = mi; v = vi;
  float denom = sqrtf(vi) / bc2_sqrt + eps;
  p = pi - step_size * (mi / denom);
}

}  // namespace rih
