// Host / device interface of the model-training kernels (train.cu) for the C entry points in api.cu.
#pragma once
#include "common.cuh"

// One ensemble GaussianMLP and its torch.optim.Adam state, as the training kernels see it (kernel parameter).
// Layer l = 0 .. L (L hidden layers, then mean_and_logvar): W[l] [E][K[l]][N[l]], b[l] [E][1][N[l]], the Adam moments in
// the same layout.  All pointers are the caller's tensors: the kernels update them in place.
struct TrainDev {
  int E, in, out, hid, L, nout;  // nout: out (deterministic) or 2 * out
  int act;
  float leaky;
  int deterministic, learn_bounds;
  int K[B200PETS_MAX_LAYERS], N[B200PETS_MAX_LAYERS];
  float* W[B200PETS_MAX_LAYERS];
  float* b[B200PETS_MAX_LAYERS];
  float* mW[B200PETS_MAX_LAYERS];  // exp_avg
  float* mb[B200PETS_MAX_LAYERS];
  float* vW[B200PETS_MAX_LAYERS];  // exp_avg_sq
  float* vb[B200PETS_MAX_LAYERS];
  float* lv[2];   // min_logvar, max_logvar [out] (probabilistic models)
  float* mlv[2];  // their moments (learn_bounds only)
  float* vlv[2];
  double lr, beta1, beta2, weight_decay, eps;
};

// Workspace of one train_epoch launch with minibatches of `batch` rows, in floats (see train_ws_layout in train.cu).
size_t train_workspace_floats(const TrainDev& m, int batch);
size_t eval_score_workspace_bytes(const TrainDev& m, long long rows);
int launch_train_epoch(const TrainDev& m, long long rows, const float* X, const float* Y, const int* idx, int steps, int batch,
                       int last_batch, long long adam_step, float* losses, float* ws, cudaStream_t stream);
int launch_eval_score(const TrainDev& m, long long rows, const float* X, const float* Y, float* scores, void* ws,
                      cudaStream_t stream);
// 0 when train_eval_kernel holds every layer's activations in shared memory on the current device, else the refusal
// (B200PETS_EUNSUPPORTED) launch_eval_score returns.  Reads only the sizes of m.
int eval_score_fits(const TrainDev& m);

struct PrepDesc {
  int D, A, Dp, in, out, obs_process, norm_mode, target_is_delta, learned_rewards;
  int f64;                // transitions stored as double (else float)
  uint32_t no_delta[32];  // bit j: observation column j is predicted as is (no_delta_list), D <= 1024
};
int launch_train_preprocess(const PrepDesc& d, long long rows, const void* obs, const void* act, const void* next_obs,
                            const void* reward, const void* norm_mean, const void* norm_std, float* X, float* Y,
                            cudaStream_t stream);
