// Host / device interface of the SAC update kernel (sac.cu) for the C entry points in api.cu.
#pragma once
#include "common.cuh"

#define SAC_MAX_ACTIONS 32  // the heads' row-wise phase holds one row's actions in one 32-column tile

// Indices into the parameter lists: the critic's QNetwork.parameters() order (linear1.weight, linear1.bias, ..,
// linear6.bias; net n, layer l: weight 6n + 2l, bias 6n + 2l + 1), then the policy's GaussianPolicy.parameters() order
// (linear1, linear2, mean_linear, log_std_linear; weight, bias).  Weights are nn.Linear's [out][in].
#define SAC_CRITIC_PARAMS 12
#define SAC_POLICY_PARAMS 8

// One SAC agent as the kernel sees it (kernel parameter).  All pointers are the caller's tensors, updated in place.
struct SacDev {
  int D, A, H;
  float* cp[SAC_CRITIC_PARAMS];  // critic parameters, exp_avg, exp_avg_sq
  float* cm[SAC_CRITIC_PARAMS];
  float* cv[SAC_CRITIC_PARAMS];
  float* ct[SAC_CRITIC_PARAMS];  // critic_target parameters
  float* pp[SAC_POLICY_PARAMS];  // policy parameters, exp_avg, exp_avg_sq
  float* pm[SAC_POLICY_PARAMS];
  float* pv[SAC_POLICY_PARAMS];
  float* log_alpha;              // [1] and its moments (automatic entropy tuning only)
  float* la_m;
  float* la_v;
  float scale[SAC_MAX_ACTIONS], bias[SAC_MAX_ACTIONS];
  float gamma;                   // as torch multiplies by a Python float: rounded to fp32
  float one_minus_tau, tau;      // soft_update's (1 - tau) and tau, each rounded to fp32
  float target_entropy;
  int tuning;
  double lr, beta1, beta2, eps;
};

// Per-call arguments of one update.
struct SacArgs {
  int B;
  int reverse_mask, soft_update;
  const float* trans;  // [B][2D + A + 2]: s, a, s', r, terminated
  const float* eps;    // [2][B][A] or NULL -> Philox
  unsigned long long seed, offset;
  long long step_c, step_p, step_a;  // Adam steps taken before this update (critic, policy, log_alpha)
  float* alpha;        // [1] read at the start, written with exp(log_alpha) when tuning
  float* stats;        // [8]
  float* ws;
};

size_t sac_workspace_floats(const SacDev& m, int batch);
int launch_sac_update(const SacDev& m, const SacArgs& a, cudaStream_t stream);
