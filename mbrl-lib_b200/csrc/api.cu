// C ABI of libb200pets: model staging (pack), rollout dispatch, fused CEM plan.  See include/b200pets.h.
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <cuda_bf16.h>

#include <new>
#include <vector>

#include "common.cuh"
#include "latent.cuh"
#include "sac.cuh"
#include "train.cuh"

// launchers defined in the kernel translation units
int launch_rollout_f32(const ModelDev& m, const RolloutArgs& a, cudaStream_t stream);
int launch_rollout_tc(const ModelDev& m, const RolloutArgs& a, cudaStream_t stream);
int launch_wgmma_selftest(int k, int n, const float* a, const float* b, float* d, cudaStream_t stream);
int launch_rollout_f32_batch(const ModelDev& m, const RolloutArgs& a, int num_problems, BatchArgs bt, cudaStream_t stream);
int launch_rollout_tc_batch(const ModelDev& m, const RolloutArgs& a, int num_problems, BatchArgs bt, cudaStream_t stream);
int launch_particle_mean(int N, int P, const float* total, float* returns, cudaStream_t stream);
bool cem_refit_sample_supported(int population, int dims, int elite_num);
int launch_cem_refit_sample_batch(int num_problems, int population, int dims, int elite_num, float alpha, int use_std,
                                  const float* row_totals, long long rows_stride, int particles, float* values, long long values_stride,
                                  float* mu, float* dispersion, float* best_solution, long long dims_stride, float* best_value,
                                  long long best_stride, void* workspace, long long ws_stride_bytes, size_t workspace_bytes, int refit,
                                  int sample, const float* lb, const float* ub, const float* z_next, long long z_stride,
                                  unsigned long long seed, unsigned long long offset, unsigned long long offset_step, int clipped,
                                  unsigned int tag, float* pop, long long pop_stride, void* stream);
int launch_cem_refit_sample(int population, int dims, int elite_num, float alpha, int use_std, const float* row_totals,
                            int particles, float* values, float* mu, float* dispersion, float* best_value, float* best_solution,
                            void* workspace, size_t workspace_bytes, int refit, int sample, const float* lb, const float* ub,
                            const float* z_next, unsigned long long seed, unsigned long long offset, int clipped, int seq0,
                            unsigned int* flag, unsigned int tag, float* pop, void* stream);
int launch_cem_update_rows(int population, int dims, int elite_num, float alpha, int unbiased, int use_std,
                           const float* population_in, const float* row_totals, int particles, float* values, float* mu,
                           float* dispersion, float* best_value, float* best_solution, void* workspace,
                           size_t workspace_bytes, void* stream);
int launch_mppi_sample_batch(int num_problems, int population, int horizon, int act_dim, float beta, const float* mean,
                             const float* past, const float* lower, const float* upper, const float* z, long long z_stride,
                             unsigned long long seed, unsigned long long offset, unsigned long long offset_step, float* pop,
                             cudaStream_t stream);
int launch_mppi_update_batch(int num_problems, int population, int dims, float gamma, const float* pop, float* values,
                             float* mean_out, float* workspace, long long ws_stride_floats, cudaStream_t stream);
bool tc_supported(const ModelDev& m);

// ---------------------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";

int b200pets_set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

// ---------------------------------------------------------------------------------------------------------
// model
// ---------------------------------------------------------------------------------------------------------
struct b200pets_model_s {
  b200pets_model_desc desc;
  ModelDev dev;
  unsigned char* blob = nullptr;
  size_t blob_bytes = 0;
  // offsets inside blob
  size_t off_W[B200PETS_MAX_LAYERS], off_b[B200PETS_MAX_LAYERS];
  size_t off_members, off_norm_d, off_norm_f, off_lv, off_nodelta, off_img;
  bool tc_ok = false;
};

static inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

namespace {

// gathered fp32 copy of the elite members: Wg[m][k][n] = W[members[m]][k][n]
__global__ void gather_members_kernel(const float* __restrict__ src, float* __restrict__ dst, const int* __restrict__ members,
                                      int M, long long per_member) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)M * per_member) return;
  const int m = (int)(idx / per_member);
  dst[idx] = src[(long long)members[m] * per_member + idx % per_member];
}

// bf16 tensor-core image of one layer for every member: [m][Kp/8][Np/8][8 n][8 k]; rows K, K+1 carry the split bias;
// the output layer's logvar columns are moved to start at column outp.
__global__ void pack_image_kernel(const float* __restrict__ Wg, const float* __restrict__ bg, unsigned char* __restrict__ img,
                                  unsigned member_stride, unsigned layer_off, int M, int K, int N, int Kp, int Np,
                                  int out, int outp, int is_last, int deterministic, float scale) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long per = (long long)Kp * Np;
  if (idx >= (long long)M * per) return;
  const int m = (int)(idx / per);
  const int rem = (int)(idx % per);
  const int n = rem % Np, k = rem / Np;
  int src_n = n;
  if (is_last) {
    if (n < outp) src_n = n < out ? n : -1;
    else src_n = (!deterministic && n - outp < out) ? out + (n - outp) : -1;
  } else if (n >= N) {
    src_n = -1;
  }
  float v = 0.f;
  if (src_n >= 0) {
    if (k < K) {
      v = Wg[((long long)m * K + k) * N + src_n];
    } else if (k == K || k == K + 1) {
      const float b = bg[(long long)m * N + src_n];
      const float hi = __bfloat162float(__float2bfloat16_rn(b));
      v = (k == K) ? hi : (b - hi);
    }
  }
  v *= scale;  // 0.5 for layers whose output feeds a SiLU (exact: a power of two commutes with bf16 rounding)
  const size_t off = (size_t)m * member_stride + layer_off + ((size_t)(k >> 3) * (Np >> 3) + (n >> 3)) * 128 + (n & 7) * 16 + (k & 7) * 2;
  *reinterpret_cast<__nv_bfloat16*>(img + off) = __float2bfloat16_rn(v);
}

// Last kernel of a staging call.  The rollout kernel is launched with programmatic stream serialisation and its weight
// producer reads the packed images BEFORE griddepcontrol.wait; a plain kernel boundary in between guarantees that the
// pack kernels above have completed and flushed before a dependent launch can even be considered (common.cuh, PDL).
__global__ void staging_fence_kernel() {}

}  // namespace

static int stage_model(b200pets_model_s* mdl, const float* const* weights, const float* const* biases,
                       const int32_t* members, const double* norm_mean, const double* norm_std, const float* min_lv,
                       const float* max_lv, const int32_t* no_delta, int num_no_delta, bool set_no_delta,
                       cudaStream_t stream) {
  const b200pets_model_desc& d = mdl->desc;
  ModelDev& v = mdl->dev;
  const int layers = d.num_hidden + 1;
  // small host-side arrays -> device (synchronous copies from pageable memory are fine: staging is not the hot path)
  CUDA_TRY(cudaMemcpyAsync(mdl->blob + mdl->off_members, members, sizeof(int32_t) * d.num_members, cudaMemcpyHostToDevice, stream));
  if (d.norm_mode) {
    if (!norm_mean || !norm_std) return b200pets_set_error(B200PETS_EINVAL, "norm_mode set but no statistics given");
    std::vector<float> f(3 * (size_t)d.in_size);
    for (int j = 0; j < d.in_size; ++j) {
      f[j] = (float)norm_mean[j];
      f[d.in_size + j] = (float)norm_std[j];
      f[2 * d.in_size + j] = (float)(1.0 / norm_std[j]);
    }
    CUDA_TRY(cudaMemcpyAsync(mdl->blob + mdl->off_norm_d, norm_mean, sizeof(double) * d.in_size, cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaMemcpyAsync(mdl->blob + mdl->off_norm_d + sizeof(double) * d.in_size, norm_std, sizeof(double) * d.in_size,
                             cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaMemcpyAsync(mdl->blob + mdl->off_norm_f, f.data(), sizeof(float) * f.size(), cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));  // f goes out of scope
  }
  if (!d.deterministic) {
    if (!min_lv || !max_lv) return b200pets_set_error(B200PETS_EINVAL, "probabilistic model needs min/max logvar");
    CUDA_TRY(cudaMemcpyAsync(mdl->blob + mdl->off_lv, min_lv, sizeof(float) * d.out_size, cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaMemcpyAsync(mdl->blob + mdl->off_lv + sizeof(float) * d.out_size, max_lv, sizeof(float) * d.out_size,
                             cudaMemcpyHostToDevice, stream));
  }
  if (set_no_delta) {
    std::vector<uint8_t> mask(d.obs_dim, 0);
    for (int i = 0; i < num_no_delta; ++i) {
      if (no_delta[i] < 0 || no_delta[i] >= d.obs_dim) return b200pets_set_error(B200PETS_EINVAL, "no_delta index %d out of range", no_delta[i]);
      mask[no_delta[i]] = 1;
    }
    CUDA_TRY(cudaMemcpyAsync(mdl->blob + mdl->off_nodelta, mask.data(), mask.size(), cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
  }
  const int* d_members = reinterpret_cast<const int*>(mdl->blob + mdl->off_members);
  for (int l = 0; l < layers; ++l) {
    const long long perW = (long long)v.K[l] * v.N[l], perB = v.N[l];
    float* Wg = reinterpret_cast<float*>(mdl->blob + mdl->off_W[l]);
    float* bg = reinterpret_cast<float*>(mdl->blob + mdl->off_b[l]);
    gather_members_kernel<<<(unsigned)((d.num_members * perW + 255) / 256), 256, 0, stream>>>(weights[l], Wg, d_members, d.num_members, perW);
    gather_members_kernel<<<(unsigned)((d.num_members * perB + 255) / 256), 256, 0, stream>>>(biases[l], bg, d_members, d.num_members, perB);
    if (mdl->tc_ok) {
      const long long tot = (long long)d.num_members * v.Kp[l] * v.Np[l];
      pack_image_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(
          Wg, bg, mdl->blob + mdl->off_img, v.img_member_stride, v.img_layer_off[l], d.num_members, v.K[l], v.N[l], v.Kp[l],
          v.Np[l], d.out_size, v.outp, l == layers - 1, d.deterministic,
          (l < layers - 1 && d.activation == B200PETS_ACT_SILU) ? 0.5f : 1.0f);
    }
  }
  if (mdl->tc_ok)
    for (int r = 1; r < v.img_replicas; ++r)
      CUDA_TRY(cudaMemcpyAsync(mdl->blob + mdl->off_img + (size_t)r * v.img_replica_stride, mdl->blob + mdl->off_img,
                               (size_t)v.img_member_stride * d.num_members, cudaMemcpyDeviceToDevice, stream));
  staging_fence_kernel<<<1, 1, 0, stream>>>();
  CUDA_TRY(cudaGetLastError());
  return B200PETS_OK;
}

extern "C" {

int b200pets_version(void) { return B200PETS_VERSION; }
const char* b200pets_last_error(void) { return g_err; }

int b200pets_device_info(int32_t* sm_count, int32_t* cc_major, int32_t* cc_minor) {
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  cudaDeviceProp p;
  CUDA_TRY(cudaGetDeviceProperties(&p, dev));
  if (sm_count) *sm_count = p.multiProcessorCount;
  if (cc_major) *cc_major = p.major;
  if (cc_minor) *cc_minor = p.minor;
  return B200PETS_OK;
}

int b200pets_model_create(const b200pets_model_desc* desc, const float* const* weights, const float* const* biases,
                          const int32_t* members, const double* norm_mean, const double* norm_std,
                          const float* min_logvar, const float* max_logvar, const int32_t* no_delta,
                          int32_t num_no_delta, void* stream, b200pets_model_t* out) {
  if (!desc || !weights || !biases || !members || !out) return b200pets_set_error(B200PETS_EINVAL, "model_create: null argument");
  const b200pets_model_desc& d = *desc;
  if (d.num_hidden < 1 || d.num_hidden + 1 > B200PETS_MAX_LAYERS)
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "model_create: %d hidden layers (supported: 1..%d)", d.num_hidden, B200PETS_MAX_LAYERS - 1);
  if (d.num_members < 1 || d.num_members > d.ensemble_size) return b200pets_set_error(B200PETS_EINVAL, "model_create: bad member count");
  for (int i = 0; i < d.num_members; ++i)
    if (members[i] < 0 || members[i] >= d.ensemble_size) return b200pets_set_error(B200PETS_EINVAL, "model_create: member index out of range");
  const int Dp = d.obs_dim + (d.obs_process == B200PETS_PROC_CARTPOLE ? 1 : 0);
  if (Dp + d.act_dim != d.in_size) return b200pets_set_error(B200PETS_EINVAL, "model_create: in_size %d != processed obs %d + act %d", d.in_size, Dp, d.act_dim);
  if (d.out_size != d.obs_dim + (d.learned_rewards ? 1 : 0))
    return b200pets_set_error(B200PETS_EINVAL, "model_create: out_size %d inconsistent with obs_dim %d / learned_rewards %d", d.out_size, d.obs_dim, d.learned_rewards);
  if (!d.learned_rewards && d.reward_fn == B200PETS_REWARD_LEARNED)
    return b200pets_set_error(B200PETS_EINVAL, "model_create: reward_fn required when rewards are not learned");

  b200pets_model_s* mdl = new b200pets_model_s();
  mdl->desc = d;
  ModelDev& v = mdl->dev;
  memset(&v, 0, sizeof(v));
  v.E = d.ensemble_size; v.M = d.num_members; v.D = d.obs_dim; v.A = d.act_dim; v.Dp = Dp; v.in = d.in_size;
  v.out = d.out_size; v.hid = d.hid_size; v.L = d.num_hidden; v.nout = d.deterministic ? d.out_size : 2 * d.out_size;
  v.act = d.activation; v.leaky = d.leaky_slope; v.obs_process = d.obs_process; v.learned_rewards = d.learned_rewards;
  v.target_is_delta = d.target_is_delta; v.deterministic = d.deterministic; v.reward_fn = d.reward_fn; v.term_fn = d.term_fn;
  v.norm_mode = d.norm_mode;
  v.outp = round_up(d.out_size, 16);
  const int layers = d.num_hidden + 1;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) & ~(size_t)255; return o; };
  uint32_t img_off = 0;
  for (int l = 0; l < layers; ++l) {
    v.K[l] = l == 0 ? d.in_size : d.hid_size;
    v.N[l] = l == layers - 1 ? v.nout : d.hid_size;
    v.Kp[l] = round_up(v.K[l] + 2, 16);
    v.Np[l] = l == layers - 1 ? (d.deterministic ? v.outp : 2 * v.outp) : round_up(d.hid_size, 16);
    v.img_layer_off[l] = img_off;
    img_off += (uint32_t)v.Kp[l] * v.Np[l] * 2;
    mdl->off_W[l] = take(sizeof(float) * d.num_members * v.K[l] * v.N[l]);
    mdl->off_b[l] = take(sizeof(float) * d.num_members * v.N[l]);
  }
  v.img_member_stride = (img_off + 127u) & ~127u;
  mdl->off_members = take(sizeof(int32_t) * d.num_members);
  mdl->off_norm_d = take(sizeof(double) * 2 * d.in_size);
  mdl->off_norm_f = take(sizeof(float) * 3 * d.in_size);
  mdl->off_lv = take(sizeof(float) * 2 * d.out_size);
  mdl->off_nodelta = take(d.obs_dim);
  v.img_replicas = 1;  // replicas at distinct addresses did not change streaming time (measured); keep the L2 footprint small
  v.img_replica_stride = ((v.img_member_stride * (uint32_t)d.num_members) + 255u) & ~255u;
  mdl->off_img = take((size_t)v.img_replica_stride * v.img_replicas);
  mdl->blob_bytes = off;
  cudaError_t e = cudaMalloc(&mdl->blob, mdl->blob_bytes);
  if (e != cudaSuccess) {
    delete mdl;
    return b200pets_set_error(B200PETS_ECUDA, "cudaMalloc(%zu) failed: %s", off, cudaGetErrorString(e));
  }
  for (int l = 0; l < layers; ++l) {
    v.W[l] = reinterpret_cast<const float*>(mdl->blob + mdl->off_W[l]);
    v.b[l] = reinterpret_cast<const float*>(mdl->blob + mdl->off_b[l]);
  }
  v.norm_mean_d = reinterpret_cast<const double*>(mdl->blob + mdl->off_norm_d);
  v.norm_std_d = v.norm_mean_d + d.in_size;
  v.norm_mean_f = reinterpret_cast<const float*>(mdl->blob + mdl->off_norm_f);
  v.norm_std_f = v.norm_mean_f + d.in_size;
  v.norm_istd_f = v.norm_std_f + d.in_size;
  v.min_lv = reinterpret_cast<const float*>(mdl->blob + mdl->off_lv);
  v.max_lv = v.min_lv + d.out_size;
  v.no_delta = mdl->blob + mdl->off_nodelta;
  v.img = mdl->blob + mdl->off_img;
  mdl->tc_ok = tc_supported(v);
  int rc = stage_model(mdl, weights, biases, members, norm_mean, norm_std, min_logvar, max_logvar, no_delta, num_no_delta,
                       true, (cudaStream_t)stream);
  if (rc != B200PETS_OK) {
    cudaFree(mdl->blob);
    delete mdl;
    return rc;
  }
  *out = mdl;
  return B200PETS_OK;
}

int b200pets_model_refresh(b200pets_model_t model, const float* const* weights, const float* const* biases,
                           const int32_t* members, const double* norm_mean, const double* norm_std,
                           const float* min_logvar, const float* max_logvar, void* stream) {
  if (!model || !weights || !biases || !members) return b200pets_set_error(B200PETS_EINVAL, "model_refresh: null argument");
  for (int i = 0; i < model->desc.num_members; ++i)
    if (members[i] < 0 || members[i] >= model->desc.ensemble_size) return b200pets_set_error(B200PETS_EINVAL, "model_refresh: member index out of range");
  return stage_model(model, weights, biases, members, norm_mean, norm_std, min_logvar, max_logvar, nullptr, 0, false,
                     (cudaStream_t)stream);
}

void b200pets_model_destroy(b200pets_model_t model) {
  if (!model) return;
  cudaFree(model->blob);
  delete model;
}

int b200pets_model_supports_tc(b200pets_model_t model) { return model && model->tc_ok ? 1 : 0; }

int b200pets_model_plan_info(b200pets_model_t model, int32_t propagation, int32_t info[4]) {
  if (!model || !info) return b200pets_set_error(B200PETS_EINVAL, "model_plan_info: null argument");
  if (propagation < B200PETS_PROP_RANDOM_MODEL || propagation > B200PETS_PROP_EXPECTATION)
    return b200pets_set_error(B200PETS_EINVAL, "model_plan_info: unknown propagation %d", propagation);
  int kslice = 0, nstages = 0, smem = 0;
  if (model->tc_ok) {
    int rc = tc_plan_info(model->dev, propagation == B200PETS_PROP_EXPECTATION, &kslice, &nstages, &smem);
    if (rc) return rc;
  }
  F32Plan fp;
  int rc = f32_tile_plan(model->dev, &fp);
  if (rc) return rc;
  info[0] = kslice;
  info[1] = nstages;
  info[2] = smem;
  info[3] = fp.rows;
  return B200PETS_OK;
}

// ---------------------------------------------------------------------------------------------------------
// rollouts
// ---------------------------------------------------------------------------------------------------------

static int shard_of(const b200pets_rollout_cfg* cfg, int* seq0, int* n_glob) {
  *seq0 = cfg->first_sequence;
  *n_glob = cfg->global_population > 0 ? cfg->global_population : cfg->population;
  if (*seq0 < 0 || (long long)*seq0 + cfg->population > (long long)*n_glob)
    return b200pets_set_error(B200PETS_EINVAL, "shard [%d, %d) outside the global population %d", *seq0,
                              *seq0 + cfg->population, *n_glob);
  return B200PETS_OK;
}

static int dispatch(const b200pets_model_s* mdl, int precision, const RolloutArgs& a_in, cudaStream_t stream) {
  RolloutArgs a = a_in;
  if (precision == B200PETS_PREC_BF16_TC) {
    if (!mdl->tc_ok) return b200pets_set_error(B200PETS_EUNSUPPORTED, "tensor-core path does not cover this model; use B200PETS_PREC_F32");
    return launch_rollout_tc(mdl->dev, a, stream);
  }
  if (precision == B200PETS_PREC_F32) return launch_rollout_f32(mdl->dev, a, stream);
  return b200pets_set_error(B200PETS_EINVAL, "unknown precision %d", precision);
}

// a batched launch (BatchArgs) of `num_problems` copies of `a_in`
static int dispatch_batch(const b200pets_model_s* mdl, int precision, const RolloutArgs& a, int num_problems, const BatchArgs& bt,
                          cudaStream_t stream) {
  if (precision == B200PETS_PREC_BF16_TC) {
    if (!mdl->tc_ok) return b200pets_set_error(B200PETS_EUNSUPPORTED, "tensor-core path does not cover this model; use B200PETS_PREC_F32");
    return launch_rollout_tc_batch(mdl->dev, a, num_problems, bt, stream);
  }
  if (precision == B200PETS_PREC_F32) return launch_rollout_f32_batch(mdl->dev, a, num_problems, bt, stream);
  return b200pets_set_error(B200PETS_EINVAL, "unknown precision %d", precision);
}

static size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

size_t b200pets_eval_workspace_bytes(b200pets_model_t model, const b200pets_rollout_cfg* cfg) {
  if (!model || !cfg) return 0;
  const size_t B = (size_t)cfg->population * cfg->particles;
  return al256(B * model->desc.obs_dim * sizeof(float)) + al256(B * sizeof(float)) + al256(B);
}

// checks shared by every evaluation entry point
static int check_eval(b200pets_model_t model, const b200pets_rollout_cfg* cfg, const char* what) {
  const b200pets_model_desc& d = model->desc;
  const int N = cfg->population, H = cfg->horizon, P = cfg->particles;
  if (N <= 0 || H <= 0 || P <= 0) return b200pets_set_error(B200PETS_EINVAL, "%s: population, horizon, particles must be positive", what);
  const long long B = (long long)N * P;
  if (B % d.num_members != 0)  // mbrl/models/gaussian_mlp.py:195-200
    return b200pets_set_error(B200PETS_EINVAL, "GaussianMLP ensemble requires batch size to be a multiple of the number of models. "
                                               "Current batch size is %lld for %d models.", B, d.num_members);
  return B200PETS_OK;
}

// Rollout launches for steps [t0, t1) of the evaluation `cfg` describes.  Between launches a row's observation is carried
// in obs_state [B][D] (stored when keep_obs, or when the window is split into per-step launches); its reward total and
// dead flag in total / dead when those are given (NULL: the kernel's own accumulation is not kept).  traj_* (or NULL)
// receive every step's next observation, reward and done at [t - t0][row].  bt (or NULL): the launches are batched over
// num_problems problems with these per-problem strides; every pointer is then problem 0's.
static int rollout_steps(b200pets_model_t model, const b200pets_rollout_cfg* cfg, int t0, int t1, bool keep_obs,
                         const float* obs0, const float* actions, const int64_t* perms, const float* eps, float* obs_state,
                         float* total, uint8_t* dead, float* traj_obs, float* traj_reward, uint8_t* traj_done,
                         cudaStream_t stream, int num_problems = 1, const BatchArgs* bt = nullptr) {
  const b200pets_model_desc& d = model->desc;
  const int N = cfg->population, H = cfg->horizon, P = cfg->particles;
  const long long B = (long long)N * P;
  RolloutArgs a{};
  a.N = N; a.H = H; a.P = P; a.B = B;
  a.propagation = cfg->propagation;
  a.sample = 1;
  a.seed = rng_key(cfg->seed, cfg->offset); a.offset = cfg->offset;
  { int rcs = shard_of(cfg, &a.seq0, &a.n_glob); if (rcs) return rcs; }
  a.act = actions; a.act_div = P; a.act_row_stride = (long long)H * d.act_dim; a.act_t_stride = d.act_dim;
  a.obs0 = obs0;
  a.total_state = total; a.dead_state = dead;
  int precision = cfg->precision;

  const bool ts1 = cfg->propagation == B200PETS_PROP_RANDOM_MODEL;
  if (ts1 && perms) {
    // reference TS1: a fresh permutation of all rows every step => rows change member (and tile) between steps;
    // one launch per step, state carried through the workspace
    for (int t = t0; t < t1; ++t) {
      RolloutArgs s = a;
      s.slot_mode = 0;
      s.perm = reinterpret_cast<const long long*>(perms) + (size_t)t * B;
      s.eps = eps ? eps + (size_t)t * B * d.out_size : nullptr;
      s.t0 = t; s.t1 = t + 1;
      s.init_from_obs0 = t == 0; s.load_state = t > 0 && total; s.store_state = 1;
      s.obs_in = obs_state; s.obs_out = obs_state;
      s.traj_obs = traj_obs ? traj_obs + (size_t)(t - t0) * B * d.obs_dim : nullptr;
      s.traj_reward = traj_reward ? traj_reward + (size_t)(t - t0) * B : nullptr;
      s.traj_done = traj_done ? traj_done + (size_t)(t - t0) * B : nullptr;
      int rc = bt ? dispatch_batch(model, precision, s, num_problems, *bt, stream) : dispatch(model, precision, s, stream);
      if (rc) return rc;
    }
  } else {
    a.t0 = t0; a.t1 = t1;
    a.eps = eps ? eps + (size_t)t0 * B * d.out_size : nullptr;
    a.init_from_obs0 = t0 == 0; a.load_state = t0 > 0 && total; a.store_state = 1;
    a.obs_in = t0 == 0 ? nullptr : obs_state; a.obs_out = keep_obs ? obs_state : nullptr;
    a.traj_obs = traj_obs; a.traj_reward = traj_reward; a.traj_done = traj_done;
    if (cfg->propagation == B200PETS_PROP_EXPECTATION) {
      a.slot_mode = 0; a.perm = nullptr;
    } else if (perms) {  // TSinf with the reset permutation
      a.slot_mode = 0; a.perm = reinterpret_cast<const long long*>(perms);
    } else {             // in-kernel member draw: per (tile, step) for TS1, per tile for TSinf
      a.slot_mode = ts1 ? 1 : 2; a.perm = nullptr;
    }
    int rc = bt ? dispatch_batch(model, precision, a, num_problems, *bt, stream) : dispatch(model, precision, a, stream);
    if (rc) return rc;
  }
  return B200PETS_OK;
}

// the rollout of one evaluation: per-row totals [B] (row r = n * P + p) in *totals_out, no particle mean
static int eval_rows(b200pets_model_t model, const b200pets_rollout_cfg* cfg, const float* obs0, const float* actions,
                     const int64_t* perms, const float* eps, float* row_returns, void* workspace, size_t workspace_bytes,
                     void* stream_, float** totals_out) {
  if (!model || !cfg || !obs0 || !actions || !workspace) return b200pets_set_error(B200PETS_EINVAL, "eval_sequences: null argument");
  const b200pets_model_desc& d = model->desc;
  { int rc = check_eval(model, cfg, "eval_sequences"); if (rc) return rc; }
  if (d.reward_fn == B200PETS_REWARD_EXTERNAL || d.term_fn == B200PETS_TERM_EXTERNAL)
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "eval_sequences: external reward/termination callables cannot run inside "
                                                     "this call; use b200pets_eval_trajectory, the callable, then b200pets_trajectory_returns");
  if (workspace_bytes < b200pets_eval_workspace_bytes(model, cfg)) return b200pets_set_error(B200PETS_EINVAL, "eval_sequences: workspace too small");
  const size_t B = (size_t)cfg->population * cfg->particles;
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  float* obs_state = reinterpret_cast<float*>(ws);
  const size_t o1 = al256(B * d.obs_dim * sizeof(float));
  float* total = row_returns ? row_returns : reinterpret_cast<float*>(ws + o1);
  uint8_t* dead = ws + o1 + al256(B * sizeof(float));
  int rc = rollout_steps(model, cfg, 0, cfg->horizon, false, obs0, actions, perms, eps, obs_state, total, dead, nullptr, nullptr,
                         nullptr, (cudaStream_t)stream_);
  if (rc) return rc;
  *totals_out = total;
  return B200PETS_OK;
}

namespace {
// model_env.py:183-188 over the steps of one window: a reward after termination is replaced (a select: NaN / inf
// cannot leak), then the row dies, then the reward is added.  Same order of operations as the rollout kernels.
__global__ void trajectory_returns_kernel(long long B, int T, int first, const float* __restrict__ reward,
                                          const uint8_t* __restrict__ done, float* total, uint8_t* dead,
                                          float* __restrict__ row_out) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= B) return;
  float tot = first ? 0.f : total[r];
  int dd = first ? 0 : (int)dead[r];
  for (int t = 0; t < T; ++t) {
    const float rew = reward[(size_t)t * B + r];
    tot += dd ? 0.f : rew;
    dd |= done[(size_t)t * B + r] != 0;
  }
  total[r] = tot;
  dead[r] = (uint8_t)dd;
  if (row_out) row_out[r] = tot;
}
}  // namespace

// trajectory workspace: reward totals [B], dead flags [B], then the carried observations [B][D] (the returns call does
// not know D, so the per-row scalars come first)
size_t b200pets_trajectory_workspace_bytes(b200pets_model_t model, const b200pets_rollout_cfg* cfg) {
  if (!model || !cfg) return 0;
  const size_t B = (size_t)cfg->population * cfg->particles;
  return al256(B * sizeof(float)) + al256(B) + al256(B * model->desc.obs_dim * sizeof(float));
}

int b200pets_eval_trajectory(b200pets_model_t model, const b200pets_rollout_cfg* cfg, int32_t t0, int32_t t1,
                             const float* obs0, const float* actions, const int64_t* perms, const float* eps,
                             float* next_obs, float* reward, uint8_t* done, void* workspace, size_t workspace_bytes,
                             void* stream) {
  if (!model || !cfg || !actions || !workspace || (t0 == 0 && !obs0))
    return b200pets_set_error(B200PETS_EINVAL, "eval_trajectory: null argument");
  { int rc = check_eval(model, cfg, "eval_trajectory"); if (rc) return rc; }
  if (t0 < 0 || t1 <= t0 || t1 > cfg->horizon)
    return b200pets_set_error(B200PETS_EINVAL, "eval_trajectory: steps [%d, %d) outside the horizon %d", t0, t1, cfg->horizon);
  if (workspace_bytes < b200pets_trajectory_workspace_bytes(model, cfg))
    return b200pets_set_error(B200PETS_EINVAL, "eval_trajectory: workspace too small");
  const size_t B = (size_t)cfg->population * cfg->particles;
  float* obs_state = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(workspace) + al256(B * sizeof(float)) + al256(B));
  return rollout_steps(model, cfg, t0, t1, t1 < cfg->horizon, obs0, actions, perms, eps, obs_state, nullptr, nullptr, next_obs,
                       reward, done, (cudaStream_t)stream);
}

int b200pets_trajectory_returns(const b200pets_rollout_cfg* cfg, int32_t t0, int32_t t1, const float* reward,
                                const uint8_t* done, float* returns, float* row_returns, void* workspace,
                                size_t workspace_bytes, void* stream_) {
  if (!cfg || !reward || !done || !workspace) return b200pets_set_error(B200PETS_EINVAL, "trajectory_returns: null argument");
  const int N = cfg->population, H = cfg->horizon, P = cfg->particles;
  if (N <= 0 || H <= 0 || P <= 0)
    return b200pets_set_error(B200PETS_EINVAL, "trajectory_returns: population, horizon, particles must be positive");
  if (t0 < 0 || t1 <= t0 || t1 > H)
    return b200pets_set_error(B200PETS_EINVAL, "trajectory_returns: steps [%d, %d) outside the horizon %d", t0, t1, H);
  const long long B = (long long)N * P;
  if (workspace_bytes < al256((size_t)B * sizeof(float)) + al256((size_t)B))
    return b200pets_set_error(B200PETS_EINVAL, "trajectory_returns: workspace too small");
  if (t1 == H && !returns) return b200pets_set_error(B200PETS_EINVAL, "trajectory_returns: null returns on the last window");
  cudaStream_t stream = (cudaStream_t)stream_;
  float* total = reinterpret_cast<float*>(workspace);
  uint8_t* dead = reinterpret_cast<unsigned char*>(workspace) + al256((size_t)B * sizeof(float));
  trajectory_returns_kernel<<<(unsigned)((B + 255) / 256), 256, 0, stream>>>(B, t1 - t0, t0 == 0, reward, done, total, dead,
                                                                             t1 == H ? row_returns : nullptr);
  CUDA_TRY(cudaGetLastError());
  if (t1 < H) return B200PETS_OK;
  return launch_particle_mean(N, P, total, returns, stream);  // model_env.py:190-191
}

int b200pets_eval_sequences(b200pets_model_t model, const b200pets_rollout_cfg* cfg, const float* obs0,
                            const float* actions, const int64_t* perms, const float* eps, float* returns,
                            float* row_returns, void* workspace, size_t workspace_bytes, void* stream_) {
  if (!returns) return b200pets_set_error(B200PETS_EINVAL, "eval_sequences: null argument");
  float* total = nullptr;
  int rc = eval_rows(model, cfg, obs0, actions, perms, eps, row_returns, workspace, workspace_bytes, stream_, &total);
  if (rc) return rc;
  return launch_particle_mean(cfg->population, cfg->particles, total, returns, (cudaStream_t)stream_);  // model_env.py:190-191
}

int b200pets_step(b200pets_model_t model, int32_t precision, int32_t propagation, int64_t batch, const float* obs,
                  const float* act, const int64_t* perm, const float* eps, uint64_t seed, uint64_t offset,
                  int32_t sample, float* next_obs, float* reward, uint8_t* done, void* stream_) {
  if (!model || !obs || !act || !next_obs) return b200pets_set_error(B200PETS_EINVAL, "step: null argument");
  const b200pets_model_desc& d = model->desc;
  if (batch <= 0) return b200pets_set_error(B200PETS_EINVAL, "step: empty batch");
  if (batch % d.num_members != 0)  // mbrl/models/gaussian_mlp.py:195-200 (checked for every propagation method)
    return b200pets_set_error(B200PETS_EINVAL, "GaussianMLP ensemble requires batch size to be a multiple of the number of models. "
                                               "Current batch size is %lld for %d models.", (long long)batch, d.num_members);
  if (propagation == B200PETS_PROP_FIXED_MODEL && !perm)  // gaussian_mlp.py:208-211
    return b200pets_set_error(B200PETS_EINVAL, "When using propagation='fixed_model', `propagation_indices` must be provided.");
  RolloutArgs a{};
  a.N = (int)batch; a.H = 1; a.P = 1; a.B = batch;
  a.t0 = 0; a.t1 = 1;
  a.propagation = propagation;
  a.sample = sample;
  a.seed = rng_key(seed, offset); a.offset = offset;
  a.seq0 = 0; a.n_glob = (int)batch;
  a.act = act; a.act_div = 1; a.act_row_stride = d.act_dim; a.act_t_stride = 0;
  a.eps = eps;
  a.init_from_obs0 = 0; a.load_state = 0; a.store_state = 1;
  a.obs_in = obs; a.obs_out = next_obs;
  a.reward_out = reward; a.done_out = done;
  if (propagation == B200PETS_PROP_EXPECTATION || perm || propagation == B200PETS_PROP_FIXED_MODEL) {
    a.slot_mode = 0; a.perm = reinterpret_cast<const long long*>(perm);
  } else {
    a.slot_mode = 1;
  }
  return dispatch(model, precision, a, (cudaStream_t)stream_);
}

// ---------------------------------------------------------------------------------------------------------
// fused CEM plan
// ---------------------------------------------------------------------------------------------------------
namespace {
__global__ void cem_init_kernel(int dims, const float* __restrict__ x0, const float* __restrict__ lb,
                                const float* __restrict__ ub, int clipped, float* mu, float* disp, float* best_value) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d == 0) {
    *best_value = -INFINITY;
    *reinterpret_cast<unsigned int*>(best_value + 2) = 0u;  // "refit done" tag of cem_refit_sample_kernel
  }
  if (d >= dims) return;
  mu[d] = x0[d];
  const float w = ub[d] - lb[d];
  disp[d] = clipped ? 1.0f : (w * w) / 16.0f;  // trajectory_opt.py:100-108
}
}  // namespace

size_t b200pets_cem_plan_workspace_bytes(b200pets_model_t model, const b200pets_rollout_cfg* rcfg, const b200pets_cem_cfg* ccfg) {
  if (!model || !rcfg || !ccfg) return 0;
  const size_t N = rcfg->population, dims = (size_t)rcfg->horizon * model->desc.act_dim;
  return al256(N * dims * 4) + al256(N * 4) + 3 * al256(dims * 4) + 256 +
         al256(b200pets_cem_update_workspace_bytes((int)N, (int)dims, ccfg->elite_num)) +
         al256(b200pets_eval_workspace_bytes(model, rcfg));
}

int b200pets_cem_plan(b200pets_model_t model, const b200pets_rollout_cfg* rcfg, const b200pets_cem_cfg* ccfg,
                      const float* obs0, const float* x0, const float* lower, const float* upper, const float* z,
                      const float* eps, const int64_t* perms, float* solution, float* values_out, void* workspace,
                      size_t workspace_bytes, void* stream_) {
  if (!model || !rcfg || !ccfg || !obs0 || !x0 || !lower || !upper || !solution || !workspace)
    return b200pets_set_error(B200PETS_EINVAL, "cem_plan: null argument");
  cudaStream_t stream = (cudaStream_t)stream_;
  const int N = rcfg->population, H = rcfg->horizon, P = rcfg->particles, A = model->desc.act_dim;
  const int dims = H * A;
  const long long B = (long long)N * P;
  if (workspace_bytes < b200pets_cem_plan_workspace_bytes(model, rcfg, ccfg)) return b200pets_set_error(B200PETS_EINVAL, "cem_plan: workspace too small");
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  float* pop = reinterpret_cast<float*>(ws); ws += al256((size_t)N * dims * 4);
  float* values = reinterpret_cast<float*>(ws); ws += al256((size_t)N * 4);
  float* mu = reinterpret_cast<float*>(ws); ws += al256((size_t)dims * 4);
  float* disp = reinterpret_cast<float*>(ws); ws += al256((size_t)dims * 4);
  float* best_sol = reinterpret_cast<float*>(ws); ws += al256((size_t)dims * 4);
  float* best_val = reinterpret_cast<float*>(ws); ws += 256;
  void* upd_ws = ws; const size_t upd_bytes = al256(b200pets_cem_update_workspace_bytes(N, dims, ccfg->elite_num)); ws += upd_bytes;
  void* eval_ws = ws; const size_t eval_bytes = al256(b200pets_eval_workspace_bytes(model, rcfg));

  cem_init_kernel<<<(dims + 255) / 256, 256, 0, stream>>>(dims, x0, lower, upper, ccfg->clipped_normal, mu, disp, best_val);
  CUDA_TRY(cudaGetLastError());
  // Per iteration: the rollout, then ONE kernel that refits (particle mean + top-k + mean / variance) and draws the next
  // iteration's population (cem.cu cem_refit_sample_kernel); the first population comes from the same kernel in
  // sample-only mode.  A population outside that kernel's single-CTA refit runs sample -> rollout -> refit instead.
  const bool merged = cem_refit_sample_supported(N, dims, ccfg->elite_num);
  unsigned int* refit_flag = reinterpret_cast<unsigned int*>(best_val + 2);
  auto next_pop = [&](int it_next, int refit, const float* totals) -> int {  // refit of it_next - 1 (if any) + population of it_next
    const int sample = it_next < ccfg->num_iterations;
    const unsigned long long off = rcfg->offset * 1024 + (unsigned long long)it_next;
    return launch_cem_refit_sample(N, dims, ccfg->elite_num, ccfg->alpha, ccfg->clipped_normal, totals, P, values, mu, disp,
                                   best_val, best_sol, upd_ws, upd_bytes, refit, sample, lower, upper,
                                   (z && sample) ? z + (size_t)it_next * N * dims : nullptr, rng_key(rcfg->seed, off), off,
                                   ccfg->clipped_normal, rcfg->first_sequence, refit_flag, (unsigned int)it_next, pop, stream);
  };
  if (merged) {
    int rc0 = next_pop(0, 0, nullptr);
    if (rc0) return rc0;
  }
  for (int it = 0; it < ccfg->num_iterations; ++it) {
    if (!merged) {
      int rcs = b200pets_cem_sample_shard(N, rcfg->first_sequence, dims, mu, disp, lower, upper,
                                          z ? z + (size_t)it * N * dims : nullptr, rcfg->seed, rcfg->offset * 1024 + it,
                                          ccfg->clipped_normal, pop, stream);
      if (rcs) return rcs;
    }
    b200pets_rollout_cfg rc_it = *rcfg;
    rc_it.offset = rcfg->offset * 1024 + it;
    const int nperm = rcfg->propagation == B200PETS_PROP_FIXED_MODEL ? 1 : H;
    float* totals = nullptr;
    int rc = eval_rows(model, &rc_it, obs0, pop, perms ? perms + (size_t)it * nperm * B : nullptr,
                       eps ? eps + (size_t)it * H * B * model->desc.out_size : nullptr, nullptr, eval_ws, eval_bytes, stream,
                       &totals);
    if (rc) return rc;
    if (merged)
      rc = next_pop(it + 1, 1, totals);
    else  // particle mean + NaN rule + top-k + refit in one kernel
      rc = launch_cem_update_rows(N, dims, ccfg->elite_num, ccfg->alpha, 1, ccfg->clipped_normal, pop, totals, P, values, mu,
                                  disp, best_val, best_sol, upd_ws, upd_bytes, stream);
    if (rc) return rc;
    // NB: values_out then holds the values AFTER the reference's in-place NaN rule (trajectory_opt.py:178)
    if (values_out) CUDA_TRY(cudaMemcpyAsync(values_out + (size_t)it * N, values, sizeof(float) * N, cudaMemcpyDeviceToDevice, stream));
  }
  CUDA_TRY(cudaMemcpyAsync(solution, ccfg->return_mean_elites ? mu : best_sol, sizeof(float) * dims, cudaMemcpyDeviceToDevice, stream));
  return B200PETS_OK;
}

// ---------------------------------------------------------------------------------------------------------
// batches of independent problems: one launch per rollout / refit for all of them
// ---------------------------------------------------------------------------------------------------------

// checks shared by the batched entry points
static int check_batch(b200pets_model_t model, const b200pets_rollout_cfg* cfg, int32_t num_problems, const char* what) {
  if (num_problems < 1) return b200pets_set_error(B200PETS_EINVAL, "%s: num_problems must be at least 1 (got %d)", what, num_problems);
  { int rc = check_eval(model, cfg, what); if (rc) return rc; }
  if (cfg->first_sequence != 0 || (cfg->global_population != 0 && cfg->global_population != cfg->population))
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "%s: a batch of problems cannot be sharded over GPUs "
                                                     "(first_sequence %d, global_population %d)", what, cfg->first_sequence,
                              cfg->global_population);
  const b200pets_model_desc& d = model->desc;
  if (d.reward_fn == B200PETS_REWARD_EXTERNAL || d.term_fn == B200PETS_TERM_EXTERNAL)
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "%s: external reward/termination callables cannot run inside this call; "
                                                     "evaluate the problems one at a time", what);
  return B200PETS_OK;
}

// evaluation workspace of a batch: observations [K][B][D], reward totals [K][B], dead flags [K][B]
size_t b200pets_eval_batch_workspace_bytes(b200pets_model_t model, const b200pets_rollout_cfg* cfg, int32_t num_problems) {
  if (!model || !cfg || num_problems < 1) return 0;
  const size_t KB = (size_t)num_problems * cfg->population * cfg->particles;
  return al256(KB * model->desc.obs_dim * sizeof(float)) + al256(KB * sizeof(float)) + al256(KB);
}

// The rollouts of K evaluations in batched launches: problem k starts from obs0 + k * D, reads actions + k * act_stride,
// perms + k * perm_stride, eps + k * eps_stride and draws with Philox offset cfg->offset + k * offset_step.  Per-row
// totals land in `total` [K][B].
static int eval_rows_batch(b200pets_model_t model, const b200pets_rollout_cfg* cfg, int K, const float* obs0, const float* actions,
                           long long act_stride, const int64_t* perms, long long perm_stride, const float* eps, long long eps_stride,
                           float* total, void* workspace, cudaStream_t stream, unsigned long long offset_step) {
  const b200pets_model_desc& d = model->desc;
  const size_t B = (size_t)cfg->population * cfg->particles, KB = (size_t)K * B;
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  float* obs_state = reinterpret_cast<float*>(ws);
  uint8_t* dead = ws + al256(KB * d.obs_dim * sizeof(float)) + al256(KB * sizeof(float));
  BatchArgs bt{};
  bt.obs0 = d.obs_dim;
  bt.obs_state = (long long)B * d.obs_dim;
  bt.act = act_stride;
  bt.rows = (long long)B;
  bt.perm = perm_stride;
  bt.eps = eps_stride;
  bt.seed = cfg->seed;
  bt.offset_step = offset_step;
  return rollout_steps(model, cfg, 0, cfg->horizon, false, obs0, actions, perms, eps, obs_state, total, dead, nullptr, nullptr,
                       nullptr, stream, K, &bt);
}

int b200pets_eval_sequences_batch(b200pets_model_t model, const b200pets_rollout_cfg* cfg, int32_t num_problems,
                                  const float* obs0, const float* actions, const int64_t* perms, const float* eps,
                                  float* returns, float* row_returns, void* workspace, size_t workspace_bytes, void* stream_) {
  if (!model || !cfg) return b200pets_set_error(B200PETS_EINVAL, "eval_sequences_batch: null argument");
  { int rc = check_batch(model, cfg, num_problems, "eval_sequences_batch"); if (rc) return rc; }
  if (!obs0 || !actions || !returns || !workspace) return b200pets_set_error(B200PETS_EINVAL, "eval_sequences_batch: null argument");
  if (workspace_bytes < b200pets_eval_batch_workspace_bytes(model, cfg, num_problems))
    return b200pets_set_error(B200PETS_EINVAL, "eval_sequences_batch: workspace too small");
  const b200pets_model_desc& d = model->desc;
  const int N = cfg->population, H = cfg->horizon;
  const size_t B = (size_t)N * cfg->particles, KB = (size_t)num_problems * B;
  const int nperm = cfg->propagation == B200PETS_PROP_FIXED_MODEL ? 1 : H;
  float* total = row_returns ? row_returns
                             : reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(workspace) + al256(KB * d.obs_dim * sizeof(float)));
  cudaStream_t stream = (cudaStream_t)stream_;
  int rc = eval_rows_batch(model, cfg, num_problems, obs0, actions, (long long)N * H * d.act_dim, perms, (long long)nperm * B, eps,
                           (long long)H * B * d.out_size, total, workspace, stream, 1024);
  if (rc) return rc;
  // problem k's totals are rows k * B .. k * B + B - 1: one particle mean over K * N sequences
  return launch_particle_mean(num_problems * N, cfg->particles, total, returns, stream);  // model_env.py:190-191
}

namespace {
__global__ void cem_init_batch_kernel(int K, int dims, const float* __restrict__ x0, const float* __restrict__ lb,
                                      const float* __restrict__ ub, int clipped, float* mu, float* disp, float* best_value) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)K * dims) return;
  const int k = (int)(idx / dims), d = (int)(idx % dims);
  if (d == 0) {  // per problem: best value, the refit flag of cem_refit_sample_batch_kernel
    best_value[(size_t)k * 64] = -INFINITY;
    *reinterpret_cast<unsigned int*>(best_value + (size_t)k * 64 + 2) = 0u;
  }
  mu[idx] = x0[idx];
  const float w = ub[d] - lb[d];
  disp[idx] = clipped ? 1.0f : (w * w) / 16.0f;  // trajectory_opt.py:100-108
}

// the workspace of a batched plan: per-problem arrays side by side, [K][...] each
struct PlanBatchLayout {
  size_t pop, values, mu, disp, best_sol, best_val, upd, eval, total;
  size_t upd_bytes;  // one problem's refit workspace
};
PlanBatchLayout plan_batch_layout(b200pets_model_t model, const b200pets_rollout_cfg* rcfg, const b200pets_cem_cfg* ccfg, int K) {
  const size_t N = rcfg->population, dims = (size_t)rcfg->horizon * model->desc.act_dim;
  PlanBatchLayout l{};
  l.upd_bytes = al256(b200pets_cem_update_workspace_bytes((int)N, (int)dims, ccfg->elite_num));
  size_t off = 0;
  l.pop = off; off += al256(K * N * dims * 4);
  l.values = off; off += al256(K * N * 4);
  l.mu = off; off += al256(K * dims * 4);
  l.disp = off; off += al256(K * dims * 4);
  l.best_sol = off; off += al256(K * dims * 4);
  l.best_val = off; off += (size_t)K * 256;  // per problem: best value, refit flag
  l.upd = off; off += (size_t)K * l.upd_bytes;
  l.eval = off; off += al256(b200pets_eval_batch_workspace_bytes(model, rcfg, K));
  l.total = off;
  return l;
}
}  // namespace

size_t b200pets_cem_plan_batch_workspace_bytes(b200pets_model_t model, const b200pets_rollout_cfg* rcfg, const b200pets_cem_cfg* ccfg,
                                               int32_t num_problems) {
  if (!model || !rcfg || !ccfg || num_problems < 1) return 0;
  return plan_batch_layout(model, rcfg, ccfg, num_problems).total;
}

int b200pets_cem_plan_batch(b200pets_model_t model, const b200pets_rollout_cfg* rcfg, const b200pets_cem_cfg* ccfg,
                            int32_t num_problems, const float* obs0, const float* x0, const float* lower, const float* upper,
                            const float* z, const float* eps, const int64_t* perms, float* solution, float* values_out,
                            void* workspace, size_t workspace_bytes, void* stream_) {
  if (!model || !rcfg || !ccfg) return b200pets_set_error(B200PETS_EINVAL, "cem_plan_batch: null argument");
  { int rc = check_batch(model, rcfg, num_problems, "cem_plan_batch"); if (rc) return rc; }
  if (!obs0 || !x0 || !lower || !upper || !solution || !workspace)
    return b200pets_set_error(B200PETS_EINVAL, "cem_plan_batch: null argument");
  const int K = num_problems;
  if (workspace_bytes < b200pets_cem_plan_batch_workspace_bytes(model, rcfg, ccfg, K))
    return b200pets_set_error(B200PETS_EINVAL, "cem_plan_batch: workspace too small");
  cudaStream_t stream = (cudaStream_t)stream_;
  const b200pets_model_desc& d = model->desc;
  const int N = rcfg->population, H = rcfg->horizon, P = rcfg->particles, A = d.act_dim, iters = ccfg->num_iterations;
  const int dims = H * A;
  const long long B = (long long)N * P;
  const PlanBatchLayout l = plan_batch_layout(model, rcfg, ccfg, K);
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  float* pop = reinterpret_cast<float*>(ws + l.pop);
  float* values = reinterpret_cast<float*>(ws + l.values);
  float* mu = reinterpret_cast<float*>(ws + l.mu);
  float* disp = reinterpret_cast<float*>(ws + l.disp);
  float* best_sol = reinterpret_cast<float*>(ws + l.best_sol);
  float* best_val = reinterpret_cast<float*>(ws + l.best_val);
  unsigned char* upd_ws = ws + l.upd;
  void* eval_ws = ws + l.eval;
  float* totals = reinterpret_cast<float*>(ws + l.eval + al256((size_t)K * B * d.obs_dim * sizeof(float)));
  const long long popk = (long long)N * dims;  // per-problem strides
  const int nperm = rcfg->propagation == B200PETS_PROP_FIXED_MODEL ? 1 : H;

  const long long tot = (long long)K * dims;
  cem_init_batch_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(K, dims, x0, lower, upper, ccfg->clipped_normal, mu, disp,
                                                                          best_val);
  CUDA_TRY(cudaGetLastError());
  // The default plan of b200pets_cem_plan for every problem: rollout, then one kernel that refits and draws the next
  // population (2 launches per iteration for the whole batch).  Outside the single-CTA refit, the sample and refit kernels
  // run once per problem around the batched rollout.
  const bool merged = cem_refit_sample_supported(N, dims, ccfg->elite_num);
  auto next_pop = [&](int it_next, int refit) -> int {  // refit of it_next - 1 (if any) + population of it_next
    const int sample = it_next < iters;
    return launch_cem_refit_sample_batch(K, N, dims, ccfg->elite_num, ccfg->alpha, ccfg->clipped_normal, refit ? totals : nullptr, B, P,
                                         values, N, mu, disp, best_sol, dims, best_val, 64, upd_ws, (long long)l.upd_bytes,
                                         l.upd_bytes, refit, sample, lower, upper,
                                         (z && sample) ? z + (size_t)it_next * N * dims : nullptr, (long long)iters * N * dims,
                                         rcfg->seed, rcfg->offset * 1024 + (unsigned long long)it_next, 1024, ccfg->clipped_normal,
                                         (unsigned int)it_next, pop, popk, stream);
  };
  if (merged) {
    int rc0 = next_pop(0, 0);
    if (rc0) return rc0;
  }
  for (int it = 0; it < iters; ++it) {
    if (!merged)
      for (int k = 0; k < K; ++k) {
        int rcs = b200pets_cem_sample_shard(N, 0, dims, mu + (size_t)k * dims, disp + (size_t)k * dims, lower, upper,
                                            z ? z + ((size_t)k * iters + it) * N * dims : nullptr, rcfg->seed,
                                            (rcfg->offset + k) * 1024 + it, ccfg->clipped_normal, pop + (size_t)k * popk, stream);
        if (rcs) return rcs;
      }
    b200pets_rollout_cfg rc_it = *rcfg;
    rc_it.offset = rcfg->offset * 1024 + it;
    int rc = eval_rows_batch(model, &rc_it, K, obs0, pop, popk, perms ? perms + (size_t)it * nperm * B : nullptr,
                             (long long)iters * nperm * B, eps ? eps + (size_t)it * H * B * d.out_size : nullptr,
                             (long long)iters * H * B * d.out_size, totals, eval_ws, stream, 1024);
    if (rc) return rc;
    if (merged) {
      rc = next_pop(it + 1, 1);
      if (rc) return rc;
    } else {
      for (int k = 0; k < K; ++k) {
        rc = launch_cem_update_rows(N, dims, ccfg->elite_num, ccfg->alpha, 1, ccfg->clipped_normal, pop + (size_t)k * popk,
                                    totals + (size_t)k * B, P, values + (size_t)k * N, mu + (size_t)k * dims,
                                    disp + (size_t)k * dims, best_val + (size_t)k * 64, best_sol + (size_t)k * dims,
                                    upd_ws + (size_t)k * l.upd_bytes, l.upd_bytes, stream);
        if (rc) return rc;
      }
    }
    if (values_out)  // problem k's values of iteration it -> values_out[k][it]
      CUDA_TRY(cudaMemcpy2DAsync(values_out + (size_t)it * N, sizeof(float) * iters * N, values, sizeof(float) * N, sizeof(float) * N,
                                 K, cudaMemcpyDeviceToDevice, stream));
  }
  CUDA_TRY(cudaMemcpyAsync(solution, ccfg->return_mean_elites ? mu : best_sol, sizeof(float) * K * dims, cudaMemcpyDeviceToDevice,
                           stream));
  return B200PETS_OK;
}

namespace {
// the start of MPPIOptimizer.optimize for each problem (trajectory_opt.py:257-258): mean[:-1] = mean[1:] in place, and the
// past action is the shifted mean[0].  One thread per (problem, action dim) walks its column forward.
__global__ void mppi_shift_batch_kernel(int K, int H, int A, float* __restrict__ mean, float* __restrict__ past) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)K * A) return;
  const long long k = idx / A;
  const int a = (int)(idx % A);
  float* m = mean + k * H * A;
  for (int t = 0; t + 1 < H; ++t) m[(size_t)t * A + a] = m[(size_t)(t + 1) * A + a];
  past[idx] = m[a];
}

// the workspace of a batched MPPI plan: per-problem arrays side by side, [K][...] each
struct MppiBatchLayout {
  size_t pop, values, past, upd, eval, total;
  long long upd_floats;  // one problem's update workspace (weights [N], per-warp partial sums [32][H*A])
};
MppiBatchLayout mppi_batch_layout(b200pets_model_t model, const b200pets_rollout_cfg* rcfg, int K) {
  const size_t N = rcfg->population, A = model->desc.act_dim, dims = (size_t)rcfg->horizon * A;
  MppiBatchLayout l{};
  l.upd_floats = (long long)(N + 32 * dims);
  size_t off = 0;
  l.pop = off; off += al256(K * N * dims * 4);
  l.values = off; off += al256(K * N * 4);
  l.past = off; off += al256(K * A * 4);
  l.upd = off; off += al256(K * (size_t)l.upd_floats * 4);
  l.eval = off; off += al256(b200pets_eval_batch_workspace_bytes(model, rcfg, K));
  l.total = off;
  return l;
}
}  // namespace

size_t b200pets_mppi_plan_batch_workspace_bytes(b200pets_model_t model, const b200pets_rollout_cfg* rcfg, const b200pets_mppi_cfg* mcfg,
                                                int32_t num_problems) {
  if (!model || !rcfg || !mcfg || num_problems < 1) return 0;
  return mppi_batch_layout(model, rcfg, num_problems).total;
}

int b200pets_mppi_plan_batch(b200pets_model_t model, const b200pets_rollout_cfg* rcfg, const b200pets_mppi_cfg* mcfg,
                             int32_t num_problems, const float* obs0, float* mean, const float* lower, const float* upper,
                             const float* z, const float* eps, const int64_t* perms, float* values_out, void* workspace,
                             size_t workspace_bytes, void* stream_) {
  if (!model || !rcfg || !mcfg) return b200pets_set_error(B200PETS_EINVAL, "mppi_plan_batch: null argument");
  { int rc = check_batch(model, rcfg, num_problems, "mppi_plan_batch"); if (rc) return rc; }
  if (!obs0 || !mean || !lower || !upper || !workspace) return b200pets_set_error(B200PETS_EINVAL, "mppi_plan_batch: null argument");
  if (mcfg->num_iterations < 0)
    return b200pets_set_error(B200PETS_EINVAL, "mppi_plan_batch: num_iterations must not be negative (got %d)", mcfg->num_iterations);
  const int K = num_problems;
  if (workspace_bytes < b200pets_mppi_plan_batch_workspace_bytes(model, rcfg, mcfg, K))
    return b200pets_set_error(B200PETS_EINVAL, "mppi_plan_batch: workspace too small");
  cudaStream_t stream = (cudaStream_t)stream_;
  const b200pets_model_desc& d = model->desc;
  const int N = rcfg->population, H = rcfg->horizon, P = rcfg->particles, A = d.act_dim, R = mcfg->num_iterations;
  const int dims = H * A;
  const long long B = (long long)N * P;
  const MppiBatchLayout l = mppi_batch_layout(model, rcfg, K);
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  float* pop = reinterpret_cast<float*>(ws + l.pop);
  float* values = reinterpret_cast<float*>(ws + l.values);
  float* past = reinterpret_cast<float*>(ws + l.past);
  float* upd_ws = reinterpret_cast<float*>(ws + l.upd);
  void* eval_ws = ws + l.eval;
  float* totals = reinterpret_cast<float*>(ws + l.eval + al256((size_t)K * B * d.obs_dim * sizeof(float)));
  const long long popk = (long long)N * dims;  // per-problem strides
  const int nperm = rcfg->propagation == B200PETS_PROP_FIXED_MODEL ? 1 : H;

  const long long tot = (long long)K * A;
  mppi_shift_batch_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(K, H, A, mean, past);
  CUDA_TRY(cudaGetLastError());
  // per refinement, for the whole batch: sample, rollout, particle mean, update.  Problem k's refinement r draws its
  // population with offset (sample_counter + k) * 1024 + r and rolls out with (offset + k * R + r) * 1024: the values
  // the k-th of K consecutive single plans takes.
  for (int r = 0; r < R; ++r) {
    int rc = launch_mppi_sample_batch(K, N, H, A, mcfg->beta, mean, past, lower, upper, z ? z + (size_t)r * popk : nullptr,
                                      (long long)R * popk, mcfg->sample_seed, mcfg->sample_counter * 1024 + (unsigned long long)r,
                                      1024, pop, stream);
    if (rc) return rc;
    b200pets_rollout_cfg rc_r = *rcfg;
    rc_r.offset = (rcfg->offset + (unsigned long long)r) * 1024;
    rc = eval_rows_batch(model, &rc_r, K, obs0, pop, popk, perms ? perms + (size_t)r * nperm * B : nullptr, (long long)R * nperm * B,
                         eps ? eps + (size_t)r * H * B * d.out_size : nullptr, (long long)R * H * B * d.out_size, totals, eval_ws,
                         stream, (unsigned long long)R * 1024);
    if (rc) return rc;
    rc = launch_particle_mean(K * N, P, totals, values, stream);  // model_env.py:190-191
    if (rc) return rc;
    rc = launch_mppi_update_batch(K, N, dims, mcfg->gamma, pop, values, mean, upd_ws, l.upd_floats, stream);
    if (rc) return rc;
    // NB: values_out then holds the values AFTER the reference's in-place NaN rule (trajectory_opt.py:297)
    if (values_out)  // problem k's values of refinement r -> values_out[k][r]
      CUDA_TRY(cudaMemcpy2DAsync(values_out + (size_t)r * N, sizeof(float) * R * N, values, sizeof(float) * N, sizeof(float) * N, K,
                                 cudaMemcpyDeviceToDevice, stream));
  }
  return B200PETS_OK;
}

namespace {
__global__ void member_map_kernel(RolloutArgs a, int M, int H, long long groups, int32_t* out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= groups * H) return;
  const int t = (int)(idx / groups);
  const long long g = idx % groups;
  const ShuffleGeom geom = shuffle_geom(a.seq0, a.N, a.n_glob);
  out[idx] = shuffle_member(a.seed, a.offset, a.slot_mode, shuffle_global_group(geom, g), t, M);
}
}  // namespace

int64_t b200pets_shuffle_num_groups(const b200pets_rollout_cfg* cfg) {
  if (!cfg || cfg->population <= 0 || cfg->particles <= 0) return 0;
  int seq0, n_glob;
  if (shard_of(cfg, &seq0, &n_glob)) return 0;
  return (int64_t)cfg->particles * shuffle_geom(seq0, cfg->population, n_glob).C_loc;
}

int b200pets_shuffle_member_map(const b200pets_rollout_cfg* cfg, int32_t num_members, int32_t* members_out, void* stream) {
  if (!cfg || !members_out || num_members < 1) return b200pets_set_error(B200PETS_EINVAL, "shuffle_member_map: bad argument");
  RolloutArgs a{};
  a.N = cfg->population; a.H = cfg->horizon; a.P = cfg->particles;
  int rc = shard_of(cfg, &a.seq0, &a.n_glob);
  if (rc) return rc;
  a.seed = rng_key(cfg->seed, cfg->offset); a.offset = cfg->offset;
  a.slot_mode = cfg->propagation == B200PETS_PROP_FIXED_MODEL ? 2 : 1;
  const long long groups = b200pets_shuffle_num_groups(cfg);
  const long long tot = groups * cfg->horizon;
  if (tot <= 0) return b200pets_set_error(B200PETS_EINVAL, "shuffle_member_map: empty configuration");
  member_map_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, num_members, cfg->horizon, groups, members_out);
  CUDA_TRY(cudaGetLastError());
  return B200PETS_OK;
}

int b200pets_selftest_wgmma(int32_t k, int32_t n, const float* a, const float* b, float* d, void* stream) {
  return launch_wgmma_selftest(k, n, a, b, d, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------------------
// training (train.cu)
// ---------------------------------------------------------------------------------------------------------
struct b200pets_trainer_s {
  TrainDev dev;
};

int b200pets_train_preprocess(const b200pets_prep_desc* desc, int64_t rows, const void* obs, const void* act,
                              const void* next_obs, const void* reward, const void* norm_mean, const void* norm_std,
                              const int32_t* no_delta, int32_t num_no_delta, float* inputs, float* targets, void* stream) {
  if (!desc || !obs || !act || !next_obs || !inputs || !targets || (desc->learned_rewards && !reward) ||
      (desc->norm_mode && (!norm_mean || !norm_std)) || (num_no_delta > 0 && !no_delta))
    return b200pets_set_error(B200PETS_EINVAL, "train_preprocess: NULL pointer");
  const b200pets_prep_desc& d = *desc;
  if (rows < 0 || d.obs_dim < 1 || d.act_dim < 0 || d.norm_mode < 0 || d.norm_mode > 2 || num_no_delta < 0)
    return b200pets_set_error(B200PETS_EINVAL, "train_preprocess: bad sizes");
  if (d.obs_process < B200PETS_PROC_NONE || d.obs_process > B200PETS_PROC_CARTPOLE)
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "train_preprocess: unknown obs_process %d", d.obs_process);
  if (d.dtype != B200PETS_DTYPE_F32 && d.dtype != B200PETS_DTYPE_F64)
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "train_preprocess: unknown dtype %d", d.dtype);
  if (d.obs_dim > 1024) return b200pets_set_error(B200PETS_EUNSUPPORTED, "train_preprocess: obs_dim %d > 1024", d.obs_dim);
  PrepDesc p{};
  p.D = d.obs_dim; p.A = d.act_dim; p.Dp = d.obs_dim + (d.obs_process == B200PETS_PROC_CARTPOLE ? 1 : 0);
  p.in = p.Dp + p.A; p.out = d.obs_dim + (d.learned_rewards ? 1 : 0);
  p.obs_process = d.obs_process; p.norm_mode = d.norm_mode; p.target_is_delta = d.target_is_delta;
  p.learned_rewards = d.learned_rewards;
  p.f64 = d.dtype == B200PETS_DTYPE_F64;
  for (int i = 0; i < num_no_delta; ++i) {
    const int c = no_delta[i];
    if (c < 0 || c >= d.obs_dim) return b200pets_set_error(B200PETS_EINVAL, "train_preprocess: no_delta index %d", c);
    p.no_delta[c >> 5] |= 1u << (c & 31);
  }
  return launch_train_preprocess(p, rows, obs, act, next_obs, reward, norm_mean, norm_std, inputs, targets,
                                 (cudaStream_t)stream);
}

// The descriptor checks of b200pets_trainer_create, and the sizes and hyper-parameters of its TrainDev (no pointers).
static int train_desc_to_dev(const b200pets_train_desc& d, const char* who, TrainDev* out) {
  if (d.num_hidden < 1 || d.num_hidden + 1 > B200PETS_MAX_LAYERS)
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "%s: %d hidden layers (1 .. %d)", who, d.num_hidden,
                              B200PETS_MAX_LAYERS - 1);
  if (d.activation != B200PETS_ACT_RELU && d.activation != B200PETS_ACT_SILU && d.activation != B200PETS_ACT_LEAKY_RELU)
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "%s: unknown activation %d", who, d.activation);
  if (d.ensemble_size < 1 || d.in_size < 1 || d.out_size < 1 || d.hid_size < 1)
    return b200pets_set_error(B200PETS_EINVAL, "%s: non-positive size", who);
  TrainDev v{};
  v.E = d.ensemble_size; v.in = d.in_size; v.out = d.out_size; v.hid = d.hid_size; v.L = d.num_hidden;
  v.nout = d.deterministic ? d.out_size : 2 * d.out_size;
  v.act = d.activation; v.leaky = d.leaky_slope; v.deterministic = d.deterministic ? 1 : 0;
  v.learn_bounds = !d.deterministic && d.learn_logvar_bounds ? 1 : 0;
  v.lr = d.lr; v.beta1 = d.beta1; v.beta2 = d.beta2; v.eps = d.eps; v.weight_decay = d.weight_decay;
  for (int l = 0; l <= d.num_hidden; ++l) {
    v.K[l] = l == 0 ? d.in_size : d.hid_size;
    v.N[l] = l == d.num_hidden ? v.nout : d.hid_size;
  }
  *out = v;
  return B200PETS_OK;
}

int b200pets_trainer_supported(const b200pets_train_desc* desc) {
  if (!desc) return b200pets_set_error(B200PETS_EINVAL, "trainer_supported: NULL pointer");
  TrainDev v;
  if (const int rc = train_desc_to_dev(*desc, "trainer_supported", &v)) return rc;
  return eval_score_fits(v);
}

int b200pets_trainer_create(const b200pets_train_desc* desc, float* const* params, float* const* exp_avg,
                            float* const* exp_avg_sq, b200pets_trainer_t* out) {
  if (!desc || !params || !exp_avg || !exp_avg_sq || !out) return b200pets_set_error(B200PETS_EINVAL, "trainer_create: NULL pointer");
  const b200pets_train_desc& d = *desc;
  TrainDev v;
  if (const int rc = train_desc_to_dev(d, "trainer_create", &v)) return rc;
  const int layers = d.num_hidden + 1;
  for (int l = 0; l < layers; ++l) {
    const int w = 2 * l, b = 2 * l + 1;
    if (!params[w] || !params[b] || !exp_avg[w] || !exp_avg[b] || !exp_avg_sq[w] || !exp_avg_sq[b])
      return b200pets_set_error(B200PETS_EINVAL, "trainer_create: NULL parameter or moment of layer %d", l);
    v.W[l] = params[w]; v.b[l] = params[b];
    v.mW[l] = exp_avg[w]; v.mb[l] = exp_avg[b];
    v.vW[l] = exp_avg_sq[w]; v.vb[l] = exp_avg_sq[b];
  }
  if (!d.deterministic) {
    for (int i = 0; i < 2; ++i) {
      const int k = 2 * layers + i;
      if (!params[k]) return b200pets_set_error(B200PETS_EINVAL, "trainer_create: NULL logvar bound");
      v.lv[i] = params[k];
      if (v.learn_bounds) {
        if (!exp_avg[k] || !exp_avg_sq[k]) return b200pets_set_error(B200PETS_EINVAL, "trainer_create: NULL logvar-bound moment");
        v.mlv[i] = exp_avg[k]; v.vlv[i] = exp_avg_sq[k];
      }
    }
  }
  b200pets_trainer_s* t = new (std::nothrow) b200pets_trainer_s;
  if (!t) return b200pets_set_error(B200PETS_ENOMEM, "trainer_create: out of host memory");
  t->dev = v;
  *out = t;
  return B200PETS_OK;
}

void b200pets_trainer_destroy(b200pets_trainer_t trainer) { delete trainer; }

size_t b200pets_train_workspace_bytes(b200pets_trainer_t trainer, int32_t batch) {
  if (!trainer || batch < 1) return 0;
  return train_workspace_floats(trainer->dev, batch) * sizeof(float);
}

int b200pets_train_epoch(b200pets_trainer_t trainer, int64_t rows, const float* inputs, const float* targets,
                         const int32_t* indices, int32_t steps, int32_t batch, int32_t last_batch, int64_t adam_step,
                         float* losses, void* workspace, size_t workspace_bytes, void* stream) {
  if (!trainer || !inputs || !targets || !indices || !losses || !workspace)
    return b200pets_set_error(B200PETS_EINVAL, "train_epoch: NULL pointer");
  if (rows < 1 || steps < 1 || batch < 1 || last_batch < 1 || last_batch > batch || adam_step < 0)
    return b200pets_set_error(B200PETS_EINVAL, "train_epoch: bad sizes (rows %lld, steps %d, batch %d, last_batch %d)",
                              (long long)rows, steps, batch, last_batch);
  const size_t need = b200pets_train_workspace_bytes(trainer, batch);
  if (workspace_bytes < need)
    return b200pets_set_error(B200PETS_EINVAL, "train_epoch: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  return launch_train_epoch(trainer->dev, rows, inputs, targets, indices, steps, batch, last_batch, adam_step, losses,
                            (float*)workspace, (cudaStream_t)stream);
}

size_t b200pets_eval_score_workspace_bytes(b200pets_trainer_t trainer, int64_t rows) {
  if (!trainer || rows < 1) return 0;
  return eval_score_workspace_bytes(trainer->dev, rows);
}

int b200pets_eval_score(b200pets_trainer_t trainer, int64_t rows, const float* inputs, const float* targets, float* scores,
                        void* workspace, size_t workspace_bytes, void* stream) {
  if (!trainer || !inputs || !targets || !scores || !workspace)
    return b200pets_set_error(B200PETS_EINVAL, "eval_score: NULL pointer");
  if (rows < 1) return b200pets_set_error(B200PETS_EINVAL, "eval_score: rows %lld < 1", (long long)rows);
  const size_t need = b200pets_eval_score_workspace_bytes(trainer, rows);
  if (workspace_bytes < need)
    return b200pets_set_error(B200PETS_EINVAL, "eval_score: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  return launch_eval_score(trainer->dev, rows, inputs, targets, scores, workspace, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------------------
// MBPO's SAC agent (sac.cu)
// ---------------------------------------------------------------------------------------------------------
struct b200pets_sac_s {
  SacDev dev;
  int interval;
};

// The descriptor checks of b200pets_sac_create, and the sizes and hyper-parameters of its SacDev (no pointers).
static int sac_desc_to_dev(const b200pets_sac_desc& d, const char* who, SacDev* out) {
  if (d.obs_dim < 1 || d.act_dim < 1 || d.hidden < 1)
    return b200pets_set_error(B200PETS_EINVAL, "%s: non-positive size (obs_dim %d, act_dim %d, hidden %d)", who, d.obs_dim,
                              d.act_dim, d.hidden);
  if (d.act_dim > SAC_MAX_ACTIONS)
    return b200pets_set_error(B200PETS_EUNSUPPORTED,
                              "%s: act_dim %d > %d (the policy heads' row-wise phase holds a row's actions in one tile)", who,
                              d.act_dim, SAC_MAX_ACTIONS);
  if (d.target_update_interval < 1)
    return b200pets_set_error(B200PETS_EINVAL, "%s: target_update_interval %d < 1", who, d.target_update_interval);
  SacDev v{};
  v.D = d.obs_dim; v.A = d.act_dim; v.H = d.hidden;
  for (int j = 0; j < d.act_dim; ++j) { v.scale[j] = d.action_scale[j]; v.bias[j] = d.action_bias[j]; }
  v.gamma = (float)d.gamma;
  v.one_minus_tau = (float)(1.0 - d.tau);
  v.tau = (float)d.tau;
  v.target_entropy = d.target_entropy;
  v.tuning = d.automatic_entropy_tuning ? 1 : 0;
  v.lr = d.lr; v.beta1 = d.beta1; v.beta2 = d.beta2; v.eps = d.eps;
  *out = v;
  return B200PETS_OK;
}

int b200pets_sac_supported(const b200pets_sac_desc* desc) {
  if (!desc) return b200pets_set_error(B200PETS_EINVAL, "sac_supported: NULL pointer");
  SacDev v;
  return sac_desc_to_dev(*desc, "sac_supported", &v);
}

int b200pets_sac_create(const b200pets_sac_desc* desc, float* const* params, float* const* target_params,
                        float* const* exp_avg, float* const* exp_avg_sq, float* log_alpha, float* log_alpha_exp_avg,
                        float* log_alpha_exp_avg_sq, b200pets_sac_t* out) {
  if (!desc || !params || !target_params || !exp_avg || !exp_avg_sq || !out)
    return b200pets_set_error(B200PETS_EINVAL, "sac_create: NULL pointer");
  SacDev v;
  if (const int rc = sac_desc_to_dev(*desc, "sac_create", &v)) return rc;
  for (int i = 0; i < B200PETS_SAC_NUM_PARAMS; ++i)
    if (!params[i] || !exp_avg[i] || !exp_avg_sq[i])
      return b200pets_set_error(B200PETS_EINVAL, "sac_create: NULL parameter or moment %d", i);
  for (int i = 0; i < SAC_CRITIC_PARAMS; ++i) {
    if (!target_params[i]) return b200pets_set_error(B200PETS_EINVAL, "sac_create: NULL target parameter %d", i);
    v.cp[i] = params[i]; v.cm[i] = exp_avg[i]; v.cv[i] = exp_avg_sq[i]; v.ct[i] = target_params[i];
  }
  for (int i = 0; i < SAC_POLICY_PARAMS; ++i) {
    const int k = SAC_CRITIC_PARAMS + i;
    v.pp[i] = params[k]; v.pm[i] = exp_avg[k]; v.pv[i] = exp_avg_sq[k];
  }
  if (v.tuning) {
    if (!log_alpha || !log_alpha_exp_avg || !log_alpha_exp_avg_sq)
      return b200pets_set_error(B200PETS_EINVAL, "sac_create: NULL log_alpha or moment with automatic entropy tuning");
    v.log_alpha = log_alpha; v.la_m = log_alpha_exp_avg; v.la_v = log_alpha_exp_avg_sq;
  }
  b200pets_sac_s* s = new (std::nothrow) b200pets_sac_s;
  if (!s) return b200pets_set_error(B200PETS_ENOMEM, "sac_create: out of host memory");
  s->dev = v;
  s->interval = desc->target_update_interval;
  *out = s;
  return B200PETS_OK;
}

void b200pets_sac_destroy(b200pets_sac_t sac) { delete sac; }

size_t b200pets_sac_workspace_bytes(b200pets_sac_t sac, int32_t batch) {
  if (!sac || batch < 1) return 0;
  return sac_workspace_floats(sac->dev, batch) * sizeof(float);
}

int b200pets_sac_update(b200pets_sac_t sac, int32_t batch, int64_t updates, int32_t reverse_mask,
                        const int64_t* adam_steps, const float* transitions, const float* eps, uint64_t seed,
                        uint64_t offset, float* alpha, float* stats, void* workspace, size_t workspace_bytes,
                        void* stream) {
  if (!sac || !adam_steps || !transitions || !alpha || !stats || !workspace)
    return b200pets_set_error(B200PETS_EINVAL, "sac_update: NULL pointer");
  if (batch < 1 || updates < 0 || adam_steps[0] < 0 || adam_steps[1] < 0 || adam_steps[2] < 0)
    return b200pets_set_error(B200PETS_EINVAL, "sac_update: bad sizes (batch %d, updates %lld)", batch, (long long)updates);
  const size_t need = b200pets_sac_workspace_bytes(sac, batch);
  if (workspace_bytes < need)
    return b200pets_set_error(B200PETS_EINVAL, "sac_update: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  SacArgs a{};
  a.B = batch;
  a.reverse_mask = reverse_mask ? 1 : 0;
  a.soft_update = updates % sac->interval == 0 ? 1 : 0;
  a.trans = transitions;
  a.eps = eps;
  a.seed = rng_key(seed, offset);
  a.offset = offset;
  a.step_c = adam_steps[0]; a.step_p = adam_steps[1]; a.step_a = adam_steps[2];
  a.alpha = alpha;
  a.stats = stats;
  a.ws = (float*)workspace;
  return launch_sac_update(sac->dev, a, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------------------
// PlaNet's latent model (latent.cu)
// ---------------------------------------------------------------------------------------------------------
}  // extern "C"

struct b200pets_latent_model_s {
  b200pets_latent_model_desc desc;
  LatentDev dev;
  float* blob = nullptr;
};

static int latent_check_params(const float* const* params, const char* who) {
  if (!params) return b200pets_set_error(B200PETS_EINVAL, "%s: null params", who);
  for (int i = 0; i < B200PETS_LATENT_NUM_PARAMS; ++i)
    if (!params[i]) return b200pets_set_error(B200PETS_EINVAL, "%s: parameter %d is NULL", who, i);
  return B200PETS_OK;
}

// checks of the latent evaluation and plan entry points: the fields of b200pets_rollout_cfg they read or constrain
static int latent_check_cfg(const b200pets_rollout_cfg* cfg, const char* who) {
  if (cfg->population <= 0 || cfg->horizon <= 0 || cfg->particles <= 0)
    return b200pets_set_error(B200PETS_EINVAL, "%s: population, horizon, particles must be positive", who);
  if (cfg->precision != B200PETS_PREC_F32)
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "%s: the latent model runs in fp32 only (precision %d)", who, cfg->precision);
  if (cfg->first_sequence != 0 || (cfg->global_population != 0 && cfg->global_population != cfg->population))
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "%s: the latent model's population cannot be sharded (first_sequence %d, "
                                                     "global_population %d)", who, cfg->first_sequence, cfg->global_population);
  return B200PETS_OK;
}

static void latent_rollout_args(const b200pets_rollout_cfg* cfg, unsigned long long offset, const float* latent0,
                                const float* belief0, const float* actions, const float* eps, float* totals, LatentArgs* a) {
  *a = LatentArgs{};
  a->B = (long long)cfg->population * cfg->particles;
  a->H = cfg->horizon;
  a->P = cfg->particles;
  a->latent0 = latent0;
  a->belief0 = belief0;
  a->act = actions;
  a->eps = eps;
  a->sample = 1;  // evaluate_action_sequences steps with sample=True (model_env.py:182-184)
  a->seed = rng_key(cfg->seed, offset);
  a->offset = offset;
  a->totals = totals;
}

extern "C" {

int b200pets_latent_model_create(const b200pets_latent_model_desc* desc, const float* const* params, void* stream,
                                 b200pets_latent_model_t* out) {
  if (!desc || !out) return b200pets_set_error(B200PETS_EINVAL, "latent_model_create: null argument");
  { int rc = latent_check_params(params, "latent_model_create"); if (rc) return rc; }
  const b200pets_latent_model_desc& d = *desc;
  if (d.action_size < 1 || d.latent_size < 1 || d.belief_size < 1 || d.hidden_size < 1)
    return b200pets_set_error(B200PETS_EINVAL, "latent_model_create: sizes must be positive (action %d, latent %d, belief %d, "
                                               "hidden %d)", d.action_size, d.latent_size, d.belief_size, d.hidden_size);
  LatentDev v{};
  v.A = d.action_size; v.L = d.latent_size; v.Hb = d.belief_size; v.Hf = d.hidden_size;
  v.A4 = round_up(v.A, 4); v.L4 = round_up(v.L, 4); v.Hb4 = round_up(v.Hb, 4); v.Hf4 = round_up(v.Hf, 4);
  v.min_std = d.min_std;
  LatentPlan plan;
  { int rc = latent_plan(v, 1, &plan); if (rc) return rc; }
  b200pets_latent_model_s* mdl = new (std::nothrow) b200pets_latent_model_s;
  if (!mdl) return b200pets_set_error(B200PETS_ENOMEM, "latent_model_create: out of host memory");
  mdl->desc = d;
  const size_t bytes = latent_blob_floats(v) * sizeof(float);
  cudaError_t e = cudaMalloc(&mdl->blob, bytes);
  if (e != cudaSuccess) {
    delete mdl;
    return b200pets_set_error(B200PETS_ECUDA, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
  }
  latent_bind(&v, mdl->blob);
  mdl->dev = v;
  int rc = latent_stage(mdl->dev, params, (cudaStream_t)stream);
  if (rc) {
    cudaFree(mdl->blob);
    delete mdl;
    return rc;
  }
  *out = mdl;
  return B200PETS_OK;
}

int b200pets_latent_model_refresh(b200pets_latent_model_t model, const float* const* params, void* stream) {
  if (!model) return b200pets_set_error(B200PETS_EINVAL, "latent_model_refresh: null model");
  { int rc = latent_check_params(params, "latent_model_refresh"); if (rc) return rc; }
  return latent_stage(model->dev, params, (cudaStream_t)stream);
}

void b200pets_latent_model_destroy(b200pets_latent_model_t model) {
  if (!model) return;
  cudaFree(model->blob);
  delete model;
}

int b200pets_latent_plan_info(b200pets_latent_model_t model, int64_t rows, int32_t info[4]) {
  if (!model || !info) return b200pets_set_error(B200PETS_EINVAL, "latent_plan_info: null argument");
  if (rows < 1) return b200pets_set_error(B200PETS_EINVAL, "latent_plan_info: rows %lld < 1", (long long)rows);
  LatentPlan p;
  { int rc = latent_plan(model->dev, rows, &p); if (rc) return rc; }
  info[0] = p.rows;
  info[1] = (int32_t)p.ctas;
  info[2] = (int32_t)p.smem;
  info[3] = (int32_t)p.row_bytes;
  return B200PETS_OK;
}

int b200pets_latent_step(b200pets_latent_model_t model, int64_t batch, const float* latent, const float* belief,
                         const float* act, const float* eps, uint64_t seed, uint64_t offset, int32_t sample,
                         float* next_latent, float* next_belief, float* reward, void* stream) {
  if (!model || !latent || !belief || !act) return b200pets_set_error(B200PETS_EINVAL, "latent_step: null argument");
  if (batch < 1) return b200pets_set_error(B200PETS_EINVAL, "latent_step: empty batch");
  LatentArgs a{};
  a.B = batch; a.H = 1; a.P = 1;
  a.latent_in = latent; a.belief_in = belief; a.act = act;
  a.eps = eps; a.sample = sample ? 1 : 0;
  a.seed = rng_key(seed, offset); a.offset = offset;
  a.latent_out = next_latent; a.belief_out = next_belief; a.reward_out = reward;
  return launch_latent_rollout(model->dev, a, (cudaStream_t)stream);
}

size_t b200pets_latent_eval_workspace_bytes(b200pets_latent_model_t model, const b200pets_rollout_cfg* cfg) {
  if (!model || !cfg) return 0;
  return al256((size_t)cfg->population * cfg->particles * sizeof(float));
}

int b200pets_latent_eval_sequences(b200pets_latent_model_t model, const b200pets_rollout_cfg* cfg, const float* latent0,
                                   const float* belief0, const float* actions, const float* eps, float* returns,
                                   float* row_returns, void* workspace, size_t workspace_bytes, void* stream_) {
  if (!model || !cfg || !latent0 || !belief0 || !actions || !returns || !workspace)
    return b200pets_set_error(B200PETS_EINVAL, "latent_eval_sequences: null argument");
  { int rc = latent_check_cfg(cfg, "latent_eval_sequences"); if (rc) return rc; }
  if (workspace_bytes < b200pets_latent_eval_workspace_bytes(model, cfg))
    return b200pets_set_error(B200PETS_EINVAL, "latent_eval_sequences: workspace too small");
  cudaStream_t stream = (cudaStream_t)stream_;
  float* totals = row_returns ? row_returns : reinterpret_cast<float*>(workspace);
  LatentArgs a;
  latent_rollout_args(cfg, cfg->offset, latent0, belief0, actions, eps, totals, &a);
  int rc = launch_latent_rollout(model->dev, a, stream);
  if (rc) return rc;
  return launch_particle_mean(cfg->population, cfg->particles, totals, returns, stream);  // model_env.py:190-191
}

size_t b200pets_latent_cem_plan_workspace_bytes(b200pets_latent_model_t model, const b200pets_rollout_cfg* rcfg,
                                                const b200pets_cem_cfg* ccfg) {
  if (!model || !rcfg || !ccfg) return 0;
  const size_t N = rcfg->population, dims = (size_t)rcfg->horizon * model->desc.action_size;
  return al256(N * dims * 4) + al256(N * 4) + 3 * al256(dims * 4) + 256 +
         al256(b200pets_cem_update_workspace_bytes((int)N, (int)dims, ccfg->elite_num)) +
         b200pets_latent_eval_workspace_bytes(model, rcfg);
}

// b200pets_cem_plan with the latent rollout: the same launches, offsets and buffers around a different model
int b200pets_latent_cem_plan(b200pets_latent_model_t model, const b200pets_rollout_cfg* rcfg, const b200pets_cem_cfg* ccfg,
                             const float* latent0, const float* belief0, const float* x0, const float* lower,
                             const float* upper, const float* z, const float* eps, float* solution, float* values_out,
                             void* workspace, size_t workspace_bytes, void* stream_) {
  if (!model || !rcfg || !ccfg || !latent0 || !belief0 || !x0 || !lower || !upper || !solution || !workspace)
    return b200pets_set_error(B200PETS_EINVAL, "latent_cem_plan: null argument");
  { int rc = latent_check_cfg(rcfg, "latent_cem_plan"); if (rc) return rc; }
  if (ccfg->num_iterations < 0 || ccfg->elite_num < 1 || ccfg->elite_num > rcfg->population)
    return b200pets_set_error(B200PETS_EINVAL, "latent_cem_plan: %d iterations, %d elites of %d", ccfg->num_iterations,
                              ccfg->elite_num, rcfg->population);
  if (workspace_bytes < b200pets_latent_cem_plan_workspace_bytes(model, rcfg, ccfg))
    return b200pets_set_error(B200PETS_EINVAL, "latent_cem_plan: workspace too small");
  cudaStream_t stream = (cudaStream_t)stream_;
  const int N = rcfg->population, H = rcfg->horizon, P = rcfg->particles, L = model->desc.latent_size;
  const int dims = H * model->desc.action_size;
  const long long B = (long long)N * P;
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  float* pop = reinterpret_cast<float*>(ws); ws += al256((size_t)N * dims * 4);
  float* values = reinterpret_cast<float*>(ws); ws += al256((size_t)N * 4);
  float* mu = reinterpret_cast<float*>(ws); ws += al256((size_t)dims * 4);
  float* disp = reinterpret_cast<float*>(ws); ws += al256((size_t)dims * 4);
  float* best_sol = reinterpret_cast<float*>(ws); ws += al256((size_t)dims * 4);
  float* best_val = reinterpret_cast<float*>(ws); ws += 256;
  void* upd_ws = ws; const size_t upd_bytes = al256(b200pets_cem_update_workspace_bytes(N, dims, ccfg->elite_num)); ws += upd_bytes;
  float* totals = reinterpret_cast<float*>(ws);

  cem_init_kernel<<<(dims + 255) / 256, 256, 0, stream>>>(dims, x0, lower, upper, ccfg->clipped_normal, mu, disp, best_val);
  CUDA_TRY(cudaGetLastError());
  const bool merged = cem_refit_sample_supported(N, dims, ccfg->elite_num);
  unsigned int* refit_flag = reinterpret_cast<unsigned int*>(best_val + 2);
  auto next_pop = [&](int it_next, int refit, const float* rows) -> int {  // refit of it_next - 1 (if any) + population of it_next
    const int sample = it_next < ccfg->num_iterations;
    const unsigned long long off = rcfg->offset * 1024 + (unsigned long long)it_next;
    return launch_cem_refit_sample(N, dims, ccfg->elite_num, ccfg->alpha, ccfg->clipped_normal, rows, P, values, mu, disp,
                                   best_val, best_sol, upd_ws, upd_bytes, refit, sample, lower, upper,
                                   (z && sample) ? z + (size_t)it_next * N * dims : nullptr, rng_key(rcfg->seed, off), off,
                                   ccfg->clipped_normal, 0, refit_flag, (unsigned int)it_next, pop, stream);
  };
  if (merged) {
    int rc0 = next_pop(0, 0, nullptr);
    if (rc0) return rc0;
  }
  for (int it = 0; it < ccfg->num_iterations; ++it) {
    const unsigned long long off = rcfg->offset * 1024 + it;
    if (!merged) {
      int rcs = b200pets_cem_sample_shard(N, 0, dims, mu, disp, lower, upper, z ? z + (size_t)it * N * dims : nullptr,
                                          rcfg->seed, off, ccfg->clipped_normal, pop, stream);
      if (rcs) return rcs;
    }
    LatentArgs a;
    latent_rollout_args(rcfg, off, latent0, belief0, pop, eps ? eps + (size_t)it * H * B * L : nullptr, totals, &a);
    int rc = launch_latent_rollout(model->dev, a, stream);
    if (rc) return rc;
    if (merged)
      rc = next_pop(it + 1, 1, totals);
    else  // particle mean + NaN rule + top-k + refit in one kernel
      rc = launch_cem_update_rows(N, dims, ccfg->elite_num, ccfg->alpha, 1, ccfg->clipped_normal, pop, totals, P, values, mu,
                                  disp, best_val, best_sol, upd_ws, upd_bytes, stream);
    if (rc) return rc;
    // values_out holds the values after the reference's in-place NaN rule (trajectory_opt.py:178), as b200pets_cem_plan's
    if (values_out) CUDA_TRY(cudaMemcpyAsync(values_out + (size_t)it * N, values, sizeof(float) * N, cudaMemcpyDeviceToDevice, stream));
  }
  CUDA_TRY(cudaMemcpyAsync(solution, ccfg->return_mean_elites ? mu : best_sol, sizeof(float) * dims, cudaMemcpyDeviceToDevice, stream));
  return B200PETS_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Training PlaNet's latent model: the recurrence's forward and backward passes (latent_train.cu)
// ---------------------------------------------------------------------------------------------------------
}  // extern "C"

static LatentTrainDev latent_train_dev(const b200pets_latent_train_desc& d, const float* const* params) {
  LatentTrainDev v{};
  v.m.A = d.action_size; v.m.L = d.latent_size; v.m.Hb = d.belief_size; v.m.Hf = d.hidden_size;
  v.m.A4 = round_up(v.m.A, 4); v.m.L4 = round_up(v.m.L, 4); v.m.Hb4 = round_up(v.m.Hb, 4); v.m.Hf4 = round_up(v.m.Hf, 4);
  v.m.min_std = d.min_std;
  v.E = d.encoding_size;
  if (params)
    for (int i = 0; i < B200PETS_LATENT_TRAIN_NUM_PARAMS; ++i) v.src[i] = params[i];
  return v;
}

static int latent_train_args(const b200pets_latent_train_desc* desc, const float* const* params, int32_t batch,
                             int32_t steps, const b200pets_latent_tape* tape, bool backward, const char* who) {
  if (!desc || !params) return b200pets_set_error(B200PETS_EINVAL, "%s: null argument", who);
  for (int i = 0; i < B200PETS_LATENT_TRAIN_NUM_PARAMS; ++i)
    if (!params[i]) return b200pets_set_error(B200PETS_EINVAL, "%s: parameter %d is NULL", who, i);
  if (batch < 1 || steps < 1)
    return b200pets_set_error(B200PETS_EINVAL, "%s: batch %d and steps %d must be positive", who, batch, steps);
  if (tape) {
    const float* f[6] = {tape->e, tape->gates, tape->q1, tape->p1, tape->pre_std, tape->eps};
    const float* g[6] = {tape->de, tape->dgi, tape->dghn, tape->dq, tape->dv, tape->dp};
    for (int i = 0; i < 6; ++i)
      if (!f[i] || (backward && !g[i])) return b200pets_set_error(B200PETS_EINVAL, "%s: a tape field is NULL", who);
  } else if (backward) {
    return b200pets_set_error(B200PETS_EINVAL, "%s: the backward pass needs the forward pass's tape", who);
  }
  return B200PETS_OK;
}

extern "C" {

int b200pets_latent_train_supported(const b200pets_latent_train_desc* desc) {
  if (!desc) return b200pets_set_error(B200PETS_EINVAL, "latent_train_supported: null argument");
  return latent_train_check(latent_train_dev(*desc, nullptr), "latent_train_supported");
}

size_t b200pets_latent_train_workspace_bytes(const b200pets_latent_train_desc* desc, int32_t batch, int32_t steps) {
  if (!desc || batch < 1 || steps < 1) return 0;
  return latent_train_blob_floats(latent_train_dev(*desc, nullptr)) * sizeof(float);
}

int b200pets_latent_seq_forward(const b200pets_latent_train_desc* desc, const float* const* params, int32_t batch,
                                int32_t steps, const float* P, const float* act, const float* eps_q, const float* eps_p,
                                uint64_t seed, uint64_t offset, float* beliefs, float* post_params, float* post_samples,
                                float* prior_params, float* prior_samples, const b200pets_latent_tape* tape,
                                void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = latent_train_args(desc, params, batch, steps, tape, false, "latent_seq_forward")) return rc;
  if (!P || !act || !beliefs || !post_params || !post_samples || !prior_params || !prior_samples || !workspace)
    return b200pets_set_error(B200PETS_EINVAL, "latent_seq_forward: null argument");
  if (!eps_q != !eps_p)
    return b200pets_set_error(B200PETS_EINVAL, "latent_seq_forward: inject both eps_q and eps_p or neither");
  LatentTrainDev d = latent_train_dev(*desc, params);
  if (int rc = latent_train_check(d, "latent_seq_forward")) return rc;
  const size_t need = b200pets_latent_train_workspace_bytes(desc, batch, steps);
  if (workspace_bytes < need)
    return b200pets_set_error(B200PETS_EINVAL, "latent_seq_forward: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  if (int rc = latent_train_stage(&d, (float*)workspace, (cudaStream_t)stream)) return rc;
  LatentSeqArgs a{};
  a.B = batch; a.T = steps;
  a.P = P; a.act = act; a.eps_q = eps_q; a.eps_p = eps_p;
  a.seed = rng_key(seed, offset); a.offset = offset;
  a.beliefs = beliefs; a.post_params = post_params; a.post_samples = post_samples;
  a.prior_params = prior_params; a.prior_samples = prior_samples;
  if (tape) a.tape = *tape;
  return launch_latent_seq_forward(d, a, (cudaStream_t)stream);
}

int b200pets_latent_seq_backward(const b200pets_latent_train_desc* desc, const float* const* params, int32_t batch,
                                 int32_t steps, const float* beliefs, const float* g_beliefs, const float* g_post_params,
                                 const float* g_post_samples, const float* g_prior_params, const float* g_prior_samples,
                                 const b200pets_latent_tape* tape, float* dP, void* stream) {
  if (int rc = latent_train_args(desc, params, batch, steps, tape, true, "latent_seq_backward")) return rc;
  if (!beliefs || !dP) return b200pets_set_error(B200PETS_EINVAL, "latent_seq_backward: null argument");
  const LatentTrainDev d = latent_train_dev(*desc, params);
  LatentSeqArgs a{};
  a.B = batch; a.T = steps;
  a.beliefs = const_cast<float*>(beliefs);
  a.g_beliefs = g_beliefs; a.g_post_params = g_post_params; a.g_post_samples = g_post_samples;
  a.g_prior_params = g_prior_params; a.g_prior_samples = g_prior_samples;
  a.dP = dP;
  a.tape = *tape;
  return launch_latent_seq_backward(d, a, (cudaStream_t)stream);
}

}  // extern "C"
