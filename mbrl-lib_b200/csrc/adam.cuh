// torch.optim.Adam's element rule, shared by the fused training kernels (train.cu, sac.cu).  The rule and its order of
// operations are documented at the top of train.cu; t is the optimizer's step count after the step being applied.
#pragma once
#include <cuda_runtime.h>

struct AdamStep {
  float wd, omb1, b2, omb2, eps, bc2_sqrt, step_size;
};

static __device__ __forceinline__ AdamStep adam_scalars(double lr, double beta1, double beta2, double weight_decay, double eps,
                                                        long long t) {
  AdamStep s;
  s.wd = (float)weight_decay;
  s.omb1 = (float)(1.0 - beta1);
  s.b2 = (float)beta2;
  s.omb2 = (float)(1.0 - beta2);
  s.eps = (float)eps;
  const double bc1 = 1.0 - pow(beta1, (double)t), bc2 = 1.0 - pow(beta2, (double)t);
  s.step_size = (float)(-(lr / bc1));
  s.bc2_sqrt = (float)sqrt(bc2);
  return s;
}

static __device__ __forceinline__ void adam_update(float* p, float* mo, float* vo, float g, const AdamStep& s) {
  float pv = *p;
  if (s.wd != 0.0f) g = g + s.wd * pv;
  float mv = *mo;
  mv = mv + s.omb1 * (g - mv);
  float vv = *vo * s.b2;
  vv = vv + s.omb2 * g * g;
  const float den = sqrtf(vv) / s.bc2_sqrt + s.eps;
  pv = pv + s.step_size * (mv / den);
  *p = pv;
  *mo = mv;
  *vo = vv;
}
