// C ABI of libb200pets: model staging (pack), rollout dispatch, fused CEM plan.  See include/b200pets.h.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cuda_bf16.h>

#include <vector>

#include "common.cuh"

// launchers defined in the kernel translation units
int launch_rollout_f32(const ModelDev& m, const RolloutArgs& a, cudaStream_t stream);
int launch_rollout_tc(const ModelDev& m, const RolloutArgs& a, cudaStream_t stream);
int launch_wgmma_selftest(int k, int n, const float* a, const float* b, float* d, cudaStream_t stream);
int launch_particle_mean(int N, int P, const float* total, float* returns, cudaStream_t stream);
bool cem_refit_sample_supported(int population, int dims, int elite_num);
int launch_cem_refit_sample(int population, int dims, int elite_num, float alpha, int use_std, const float* row_totals,
                            int particles, float* values, float* mu, float* dispersion, float* best_value, float* best_solution,
                            void* workspace, size_t workspace_bytes, int refit, int sample, const float* lb, const float* ub,
                            const float* z_next, unsigned long long seed, unsigned long long offset, int clipped, int seq0,
                            unsigned int* flag, unsigned int tag, float* pop, void* stream);
int launch_cem_update_rows(int population, int dims, int elite_num, float alpha, int unbiased, int use_std,
                           const float* population_in, const float* row_totals, int particles, float* values, float* mu,
                           float* dispersion, float* best_value, float* best_solution, void* workspace,
                           size_t workspace_bytes, void* stream);
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

size_t b200pets_eval_workspace_bytes(b200pets_model_t model, const b200pets_rollout_cfg* cfg) {
  if (!model || !cfg) return 0;
  const size_t B = (size_t)cfg->population * cfg->particles;
  return ((B * model->desc.obs_dim * sizeof(float) + 255) & ~(size_t)255) + ((B * sizeof(float) + 255) & ~(size_t)255) + ((B + 255) & ~(size_t)255);
}

// the rollout of one evaluation: per-row totals [B] (row r = n * P + p) in *totals_out, no particle mean
static int eval_rows(b200pets_model_t model, const b200pets_rollout_cfg* cfg, const float* obs0, const float* actions,
                     const int64_t* perms, const float* eps, float* row_returns, void* workspace, size_t workspace_bytes,
                     void* stream_, float** totals_out) {
  if (!model || !cfg || !obs0 || !actions || !workspace) return b200pets_set_error(B200PETS_EINVAL, "eval_sequences: null argument");
  cudaStream_t stream = (cudaStream_t)stream_;
  const b200pets_model_desc& d = model->desc;
  const int N = cfg->population, H = cfg->horizon, P = cfg->particles;
  if (N <= 0 || H <= 0 || P <= 0) return b200pets_set_error(B200PETS_EINVAL, "eval_sequences: population, horizon, particles must be positive");
  const long long B = (long long)N * P;
  if (B % d.num_members != 0)  // mbrl/models/gaussian_mlp.py:195-200
    return b200pets_set_error(B200PETS_EINVAL, "GaussianMLP ensemble requires batch size to be a multiple of the number of models. "
                                               "Current batch size is %lld for %d models.", B, d.num_members);
  if (d.reward_fn == B200PETS_REWARD_EXTERNAL || d.term_fn == B200PETS_TERM_EXTERNAL)
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "eval_sequences: external reward/termination callables need the per-step API");
  if (workspace_bytes < b200pets_eval_workspace_bytes(model, cfg)) return b200pets_set_error(B200PETS_EINVAL, "eval_sequences: workspace too small");
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  float* obs_state = reinterpret_cast<float*>(ws);
  size_t o1 = ((size_t)B * d.obs_dim * sizeof(float) + 255) & ~(size_t)255;
  float* total = row_returns ? row_returns : reinterpret_cast<float*>(ws + o1);
  uint8_t* dead = ws + o1 + (((size_t)B * sizeof(float) + 255) & ~(size_t)255);

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
    for (int t = 0; t < H; ++t) {
      RolloutArgs s = a;
      s.slot_mode = 0;
      s.perm = reinterpret_cast<const long long*>(perms) + (size_t)t * B;
      s.eps = eps ? eps + (size_t)t * B * d.out_size : nullptr;
      s.t0 = t; s.t1 = t + 1;
      s.init_from_obs0 = t == 0; s.load_state = t > 0; s.store_state = 1;
      s.obs_in = obs_state; s.obs_out = obs_state;
      int rc = dispatch(model, precision, s, stream);
      if (rc) return rc;
    }
  } else {
    a.t0 = 0; a.t1 = H;
    a.eps = eps;
    a.init_from_obs0 = 1; a.load_state = 0; a.store_state = 1;
    a.obs_in = nullptr; a.obs_out = nullptr;
    if (cfg->propagation == B200PETS_PROP_EXPECTATION) {
      a.slot_mode = 0; a.perm = nullptr;
    } else if (perms) {  // TSinf with the reset permutation
      a.slot_mode = 0; a.perm = reinterpret_cast<const long long*>(perms);
    } else {             // in-kernel member draw: per (tile, step) for TS1, per tile for TSinf
      a.slot_mode = ts1 ? 1 : 2; a.perm = nullptr;
    }
    int rc = dispatch(model, precision, a, stream);
    if (rc) return rc;
  }
  *totals_out = total;
  return B200PETS_OK;
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
    *reinterpret_cast<unsigned int*>(best_value + 1) = 0u;  // tail counter of the fused iteration kernel
    *reinterpret_cast<unsigned int*>(best_value + 2) = 0u;  // "refit done" tag of cem_refit_sample_kernel
  }
  if (d >= dims) return;
  mu[d] = x0[d];
  const float w = ub[d] - lb[d];
  disp[d] = clipped ? 1.0f : (w * w) / 16.0f;  // trajectory_opt.py:100-108
}
}  // namespace

static size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

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
  // Default: sample -> rollout -> refit (3 launches per iteration; the refit kernel fuses the particle mean).  B200PETS_CEM_FUSED=1 selects the fused variants (parity-tested, not the default): refit by the last CTA of the
  // rollout kernel (2 launches / iteration) and, with B200PETS_CEM_SAMPLE_IN_KERNEL=1, the population drawn inside the
  // rollout kernel too (1 launch / iteration: every particle row re-derives its sequence's actions).
  const char* env_fuse = getenv("B200PETS_CEM_FUSED");
  const bool fuse = (env_fuse && env_fuse[0] == '1') && rcfg->precision == B200PETS_PREC_BF16_TC && model->tc_ok && !z &&
                    !perms && N <= 2048 && dims <= 1024 && ccfg->elite_num >= 2 && ccfg->elite_num <= N &&
                    rcfg->propagation != B200PETS_PROP_EXPECTATION && B % model->desc.num_members == 0 &&
                    model->desc.reward_fn != B200PETS_REWARD_EXTERNAL && model->desc.term_fn != B200PETS_TERM_EXTERNAL;
  const char* env_sik = getenv("B200PETS_CEM_SAMPLE_IN_KERNEL");
  const bool sample_in_kernel = env_sik && env_sik[0] == '1';
  // Default: 2 launches per iteration -- rollout, then ONE kernel that refits (particle mean + top-k + mean / variance) and
  // draws the next iteration's population (cem.cu cem_refit_sample_kernel); the first population comes from the same
  // kernel in sample-only mode.  B200PETS_CEM_MERGED=0 (or a population outside the single-CTA refit) keeps the three
  // separate kernels.
  static const bool merged_env = [] { const char* e = getenv("B200PETS_CEM_MERGED"); return !(e && e[0] == '0'); }();
  const bool merged = merged_env && !fuse && cem_refit_sample_supported(N, dims, ccfg->elite_num);
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
    if (merged) {
      b200pets_rollout_cfg rc_it = *rcfg;
      rc_it.offset = rcfg->offset * 1024 + it;
      const int nperm = rcfg->propagation == B200PETS_PROP_FIXED_MODEL ? 1 : H;
      float* totals = nullptr;
      int rc = eval_rows(model, &rc_it, obs0, pop, perms ? perms + (size_t)it * nperm * B : nullptr,
                         eps ? eps + (size_t)it * H * B * model->desc.out_size : nullptr, nullptr, eval_ws, eval_bytes, stream,
                         &totals);
      if (rc) return rc;
      rc = next_pop(it + 1, 1, totals);
      if (rc) return rc;
      if (values_out) CUDA_TRY(cudaMemcpyAsync(values_out + (size_t)it * N, values, sizeof(float) * N, cudaMemcpyDeviceToDevice, stream));
      continue;
    }
    if (fuse) {
      // default: population drawn by cem_sample_kernel, rollout + refit in one kernel (2 launches per iteration);
      // B200PETS_CEM_SAMPLE_IN_KERNEL=1 also draws the population inside the rollout kernel (1 launch per iteration,
      // measured slower: every particle row re-derives its sequence's actions on the epilogue's critical path)
      if (!sample_in_kernel) {
        int rcs = b200pets_cem_sample_shard(N, rcfg->first_sequence, dims, mu, disp, lower, upper, nullptr, rcfg->seed,
                                            rcfg->offset * 1024 + it, ccfg->clipped_normal, pop, stream);
        if (rcs) return rcs;
      }
      unsigned char* ews = reinterpret_cast<unsigned char*>(eval_ws);
      const size_t o1 = ((size_t)B * model->desc.obs_dim * sizeof(float) + 255) & ~(size_t)255;
      RolloutArgs a{};
      a.N = N; a.H = H; a.P = P; a.B = B;
      a.t0 = 0; a.t1 = H;
      a.propagation = rcfg->propagation;
      a.slot_mode = rcfg->propagation == B200PETS_PROP_RANDOM_MODEL ? 1 : 2;
      a.sample = 1;
      a.offset = rcfg->offset * 1024 + it; a.seed = rng_key(rcfg->seed, a.offset);
      { int rcs = shard_of(rcfg, &a.seq0, &a.n_glob); if (rcs) return rcs; }
      a.eps = eps ? eps + (size_t)it * H * B * model->desc.out_size : nullptr;
      a.obs0 = obs0; a.init_from_obs0 = 1; a.store_state = 1;
      a.total_state = reinterpret_cast<float*>(ews + o1);
      a.dead_state = ews + o1 + (((size_t)B * sizeof(float) + 255) & ~(size_t)255);
      a.act = pop; a.act_div = P; a.act_row_stride = (long long)H * A; a.act_t_stride = A;
      if (sample_in_kernel) {
        a.cem_mu = mu; a.cem_disp = disp; a.cem_lb = lower; a.cem_ub = upper;
        a.cem_offset = rcfg->offset * 1024 + it;
      }
      a.cem_clipped = ccfg->clipped_normal;
      a.pop_out = pop;
      a.tail_counter = reinterpret_cast<unsigned int*>(best_val + 1);
      a.tail_values = values; a.tail_mu = mu; a.tail_disp = disp; a.tail_best_value = best_val; a.tail_best_solution = best_sol;
      a.tail_elite_num = ccfg->elite_num; a.tail_alpha = ccfg->alpha;
      int rc = dispatch(model, B200PETS_PREC_BF16_TC, a, stream);
      if (rc) return rc;
      if (values_out) CUDA_TRY(cudaMemcpyAsync(values_out + (size_t)it * N, values, sizeof(float) * N, cudaMemcpyDeviceToDevice, stream));
      continue;
    }
    int rc = b200pets_cem_sample_shard(N, rcfg->first_sequence, dims, mu, disp, lower, upper,
                                       z ? z + (size_t)it * N * dims : nullptr, rcfg->seed, rcfg->offset * 1024 + it,
                                       ccfg->clipped_normal, pop, stream);
    if (rc) return rc;
    b200pets_rollout_cfg rc_it = *rcfg;
    rc_it.offset = rcfg->offset * 1024 + it;
    const int nperm = rcfg->propagation == B200PETS_PROP_FIXED_MODEL ? 1 : H;
    float* totals = nullptr;
    rc = eval_rows(model, &rc_it, obs0, pop, perms ? perms + (size_t)it * nperm * B : nullptr,
                   eps ? eps + (size_t)it * H * B * model->desc.out_size : nullptr, nullptr, eval_ws, eval_bytes, stream,
                   &totals);
    if (rc) return rc;
    // particle mean + NaN rule + top-k + refit in ONE kernel (3 launches per iteration: sample, rollout, refit)
    rc = launch_cem_update_rows(N, dims, ccfg->elite_num, ccfg->alpha, 1, ccfg->clipped_normal, pop, totals, P, values, mu,
                                disp, best_val, best_sol, upd_ws, upd_bytes, stream);
    if (rc) return rc;
    // NB: values_out then holds the values AFTER the reference's in-place NaN rule (trajectory_opt.py:178)
    if (values_out) CUDA_TRY(cudaMemcpyAsync(values_out + (size_t)it * N, values, sizeof(float) * N, cudaMemcpyDeviceToDevice, stream));
  }
  CUDA_TRY(cudaMemcpyAsync(solution, ccfg->return_mean_elites ? mu : best_sol, sizeof(float) * dims, cudaMemcpyDeviceToDevice, stream));
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

}  // extern "C"
