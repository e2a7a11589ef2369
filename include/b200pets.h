/*
 * b200pets.h -- C ABI of the H100-native PETS planning hot path.
 *
 * The reference (facebookresearch/mbrl-lib) has no FFI: its plugin boundary is Python duck typing
 * (SURVEY.md section 8b).  This header is the boundary a native binding would target; every entry point
 * names the reference interface it stands in for (paths relative to the mbrl-lib tree).
 *
 * Conventions: every pointer marked [dev] is a CUDA device pointer owned by the caller, every pointer
 * marked [host] is host memory read during the call only.  `stream` is a cudaStream_t passed as void*
 * (NULL = legacy default stream).  Nothing allocates on the hot path: callers pass a workspace sized by the
 * matching *_workspace_bytes().  All functions return 0 on success and a negative B200PETS_E* code on
 * failure; b200pets_last_error() returns the message of the last failure on the calling thread.
 * No entry point synchronises the device.
 */
#ifndef B200PETS_H
#define B200PETS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200PETS_VERSION 2

/* error codes */
#define B200PETS_OK 0
#define B200PETS_EINVAL (-1)      /* bad argument / shape, mirrors the reference's assert / ValueError */
#define B200PETS_EUNSUPPORTED (-2) /* configuration outside what the kernels cover */
#define B200PETS_ECUDA (-3)       /* CUDA runtime error (no device, launch failure, ...) */
#define B200PETS_ENOMEM (-4)

/* activation of the hidden layers: mbrl/models/gaussian_mlp.py:89-111 */
#define B200PETS_ACT_RELU 0
#define B200PETS_ACT_SILU 1
#define B200PETS_ACT_LEAKY_RELU 2

/* obs_process_fn: mbrl/models/one_dim_tr_model.py:108-109 */
#define B200PETS_PROC_NONE 0
#define B200PETS_PROC_HALFCHEETAH 1 /* mbrl/env/pets_halfcheetah.py:91-113: [o1, sin o2, cos o2, o3:] */
#define B200PETS_PROC_CARTPOLE 2    /* mbrl/env/pets_cartpole.py:78-101:  [sin o1, cos o1, o0, o2:] */

/* reward_fn: mbrl/env/reward_fns.py */
#define B200PETS_REWARD_LEARNED 0 /* last model output column, one_dim_tr_model.py:287 */
#define B200PETS_REWARD_CARTPOLE 1
#define B200PETS_REWARD_CARTPOLE_PETS 2
#define B200PETS_REWARD_INVERTED_PENDULUM 3
#define B200PETS_REWARD_HALFCHEETAH 4
#define B200PETS_REWARD_PUSHER 5
#define B200PETS_REWARD_EXTERNAL 255 /* b200pets_step only: reward left to the caller's callable */

/* termination_fn: mbrl/env/termination_fns.py */
#define B200PETS_TERM_NONE 0
#define B200PETS_TERM_CARTPOLE 1
#define B200PETS_TERM_INVERTED_PENDULUM 2
#define B200PETS_TERM_HOPPER 3
#define B200PETS_TERM_WALKER2D 4
#define B200PETS_TERM_ANT 5
#define B200PETS_TERM_HUMANOID 6
#define B200PETS_TERM_EXTERNAL 255 /* b200pets_step only */

/* uncertainty propagation: mbrl/models/gaussian_mlp.py:179-216 */
#define B200PETS_PROP_RANDOM_MODEL 0 /* TS1   */
#define B200PETS_PROP_FIXED_MODEL 1  /* TSinf */
#define B200PETS_PROP_EXPECTATION 2

/* arithmetic of the ensemble MLP */
#define B200PETS_PREC_F32 0     /* fp32 SIMT: parity anchor (~1e-5 of the reference) */
#define B200PETS_PREC_BF16_TC 1 /* bf16 operands, fp32 accumulate on the tensor cores (wgmma) */

/* how TS1 assigns rows to members when no permutation is injected */
#define B200PETS_TS1_PERMS 0        /* explicit permutations (one per step), reference semantics */
#define B200PETS_TS1_TILE_SHUFFLE 1 /* in-kernel: a shuffle group = the particle-p copies of 128 consecutive (global)
                                       sequences; every (group, step) draws one member uniformly from Philox, so the
                                       particles of one sequence (different groups) draw independently, as rows do
                                       under the reference's randperm split (DESIGN.md "TS1 in production") */

typedef struct b200pets_model_s* b200pets_model_t;

/* Static description of OneDTransitionRewardModel(GaussianMLP): mbrl/models/one_dim_tr_model.py:84-101,
 * mbrl/models/gaussian_mlp.py:69-127. */
typedef struct {
  int32_t ensemble_size;   /* E, leading dim of the weight tensors */
  int32_t num_members;     /* M = len(elite_models) or E: members used for propagation */
  int32_t obs_dim;         /* D, raw observation size */
  int32_t act_dim;         /* A */
  int32_t in_size;         /* model input = processed obs + act */
  int32_t out_size;        /* D (+1 if learned_rewards) */
  int32_t hid_size;
  int32_t num_hidden;      /* hidden layers (num_layers) */
  int32_t activation;      /* B200PETS_ACT_* */
  float leaky_slope;
  int32_t obs_process;     /* B200PETS_PROC_* */
  int32_t learned_rewards;
  int32_t target_is_delta;
  int32_t deterministic;   /* GaussianMLP(deterministic=True): no logvar head */
  int32_t reward_fn;       /* B200PETS_REWARD_* */
  int32_t term_fn;         /* B200PETS_TERM_* */
  int32_t norm_mode;       /* 0 none, 1 fp32 stats, 2 fp64 stats (util/math.py:95-143) */
} b200pets_model_desc;

int b200pets_version(void);
const char* b200pets_last_error(void);
int b200pets_device_info(int32_t* sm_count, int32_t* cc_major, int32_t* cc_minor);

/* Stage a model for the kernels.  Replaces reading nn.Parameters on every forward
 * (mbrl/models/util.py:53-65 re-gathers weight[elite_models] per layer per step).
 *   weights[l] [dev] float [E][K_l][N_l], biases[l] [dev] float [E][1][N_l], l = 0..num_hidden
 *   members    [host] M ensemble indices in elite order (gaussian_mlp.py:377-379)
 *   norm_mean/norm_std [host] double[in_size] or NULL (norm_mode 0)
 *   min_logvar/max_logvar [host] float[out_size] or NULL (deterministic)
 *   no_delta   [host] indices of one_dim_tr_model.py:284-285 */
int b200pets_model_create(const b200pets_model_desc* desc, const float* const* weights,
                          const float* const* biases, const int32_t* members, const double* norm_mean,
                          const double* norm_std, const float* min_logvar, const float* max_logvar,
                          const int32_t* no_delta, int32_t num_no_delta, void* stream,
                          b200pets_model_t* out);
/* Re-stage after ModelTrainer.train / set_elite / update_normalizer (model_trainer.py:288-296). */
int b200pets_model_refresh(b200pets_model_t model, const float* const* weights, const float* const* biases,
                           const int32_t* members, const double* norm_mean, const double* norm_std,
                           const float* min_logvar, const float* max_logvar, void* stream);
void b200pets_model_destroy(b200pets_model_t model);
/* 1 if the tensor-core path covers this model's dimensions, else 0 (callers then use B200PETS_PREC_F32). */
int b200pets_model_supports_tc(b200pets_model_t model);

typedef struct {
  int32_t population;  /* N */
  int32_t horizon;     /* H */
  int32_t particles;   /* P */
  int32_t precision;   /* B200PETS_PREC_* */
  int32_t propagation; /* B200PETS_PROP_* */
  int32_t ts1_mode;    /* B200PETS_TS1_* (only read for PROP_RANDOM_MODEL with perms == NULL) */
  uint64_t seed;       /* Philox key of in-kernel draws */
  uint64_t offset;     /* Philox stream offset; callers advance it per call */
  /* population sharded over GPUs (SURVEY.md section 8e): this call evaluates global sequences
   * [first_sequence, first_sequence + population) of a population of global_population (0 = population, i.e. one GPU).
   * Every in-kernel draw (population noise, model noise, member per shuffle group) is keyed by GLOBAL sequence
   * index, so results do not depend on the number of GPUs. */
  int32_t first_sequence;
  int32_t global_population;
} b200pets_rollout_cfg;

/* ModelEnv.evaluate_action_sequences (mbrl/models/model_env.py:145-191).
 *   obs0    [dev] float[D]          initial_state (already cast to fp32, model_env.py:173)
 *   actions [dev] float[N][H][A]
 *   perms   [dev] int64: TS1 [H][B], TSinf [1][B]; NULL = draw in kernel (shuffle groups, see
 *           b200pets_shuffle_member_map: per step for TS1, once for TSinf)
 *   eps     [dev] float[H][B][out] injected N(0,1) model noise or NULL = Philox in kernel
 *   returns [dev] float[N]          mean over particles of the summed rewards
 *   row_returns [dev] float[B] or NULL: per-particle totals (row r = n*P + p) */
size_t b200pets_eval_workspace_bytes(b200pets_model_t model, const b200pets_rollout_cfg* cfg);
int b200pets_eval_sequences(b200pets_model_t model, const b200pets_rollout_cfg* cfg, const float* obs0,
                            const float* actions, const int64_t* perms, const float* eps, float* returns,
                            float* row_returns, void* workspace, size_t workspace_bytes, void* stream);

/* The member every shuffle group uses at every step when perms == NULL (exactly what the kernels draw; parity
 * tests feed it to the oracle as a per-row member assignment, gaussian_mlp.py:202-212 with the permutation replaced).
 * Group g of this shard = (particle p = g / C, chunk c = c_lo + g % C) with C = number of 128-aligned chunks of
 * global sequence indices that intersect the shard, c_lo = first_sequence / 128; its rows are the particle-p copies
 * of global sequences 128c .. 128c+127.  members_out [dev] int32[H][num_groups] (TSinf: all steps equal). */
int64_t b200pets_shuffle_num_groups(const b200pets_rollout_cfg* cfg);
int b200pets_shuffle_member_map(const b200pets_rollout_cfg* cfg, int32_t num_members, int32_t* members_out,
                                void* stream);

/* ModelEnv.step (mbrl/models/model_env.py:87-140) for a batch of B independent states.
 *   perm [dev] int64[B]; NULL is allowed for TS1 (tile shuffle) and expectation; TSinf requires the caller's
 *        propagation_indices and returns B200PETS_EINVAL without them (gaussian_mlp.py:208-211)
 *   eps  [dev] float[B][out] or NULL; sample == 0 returns the mean prediction (deterministic=True). */
int b200pets_step(b200pets_model_t model, int32_t precision, int32_t propagation, int64_t batch,
                  const float* obs, const float* act, const int64_t* perm, const float* eps, uint64_t seed,
                  uint64_t offset, int32_t sample, float* next_obs, float* reward, uint8_t* done,
                  void* stream);

/* ---- MBPO model rollouts kept on the device (mbrl/algorithms/mbpo.py:31-63) ------------------------------ */

/* The `accum_dones` bookkeeping of rollout_model_and_populate_sac_buffer (mbpo.py:44,51-62) for one step:
 *   alive[r] = !accum_dones[r]   (the rows of this step that go to sac_buffer.add_batch)
 *   accum_dones[r] |= done[r]
 * all [dev] uint8[batch]. */
int b200pets_mbpo_mask(int64_t batch, const uint8_t* done, uint8_t* accum_dones, uint8_t* alive, void* stream);

/* Ordered compaction of the alive transitions of `steps` model steps: replaces the per-step device->host copies and
 * numpy selections `obs[~accum_dones]`, ... of mbpo.py:53-60.  The outputs hold, packed and in (step, row) order -- the
 * order of the reference's add_batch calls --, the alive rows of every step:
 *   obs0     [dev] float[B][D]       observations before step 0 (the sampled start states)
 *   act      [dev] float[steps][B][A]
 *   next_obs [dev] float[steps][B][D] (the observation before step i > 0 is next_obs[i-1])
 *   reward   [dev] float[steps][B], done / alive [dev] uint8[steps][B]
 *   *_out    [dev] sized for steps * B rows
 *   counts   [dev] int64[steps + 1]: alive rows per step, counts[steps] = total */
size_t b200pets_mbpo_compact_workspace_bytes(int32_t steps, int64_t batch);
int b200pets_mbpo_compact(int32_t steps, int64_t batch, int32_t obs_dim, int32_t act_dim, const float* obs0,
                          const float* act, const float* next_obs, const float* reward, const uint8_t* done,
                          const uint8_t* alive, float* obs_out, float* act_out, float* next_obs_out,
                          float* reward_out, uint8_t* done_out, int64_t* counts, void* workspace,
                          size_t workspace_bytes, void* stream);

/* ---- CEM / iCEM building blocks (mbrl/planning/trajectory_opt.py) ------------------------------------ */

/* CEMOptimizer._sample_population (trajectory_opt.py:110-128) + util.math.truncated_normal_ (util/math.py
 * :69-92).  z [dev] float[N][H*A] injected draws or NULL = Philox (truncated by per-element rejection).
 * dims = H*A.  clipped_normal as in the reference ctor. */
int b200pets_cem_sample(int32_t population, int32_t dims, const float* mu, const float* dispersion,
                        const float* lower, const float* upper, const float* z, uint64_t seed,
                        uint64_t offset, int32_t clipped_normal, float* population_out, void* stream);
/* Same for one shard of a population split over GPUs: rows are global sequences first_sequence .. +population-1 and
 * the Philox draws are keyed by the global index (identical numbers whatever the number of shards). */
int b200pets_cem_sample_shard(int32_t population, int32_t first_sequence, int32_t dims, const float* mu,
                              const float* dispersion, const float* lower, const float* upper, const float* z,
                              uint64_t seed, uint64_t offset, int32_t clipped_normal, float* population_out,
                              void* stream);

/* One refit: NaN -> -1e-10, top-k, mean / variance of the elites, momentum, best-so-far
 * (trajectory_opt.py:130-140, 178-186; iCEM 474-486 with unbiased = 0).
 *   values [dev] float[N] (NaNs are overwritten in place, like the reference)
 *   mu, dispersion [dev] float[dims] updated in place
 *   best_value [dev] float[1], best_solution [dev] float[dims] updated in place
 *   elite_idx [dev] int32[elite_num] out (ascending index order; ties broken by lowest index)
 *   elites_out [dev] float[elite_num][dims] or NULL (iCEM keeps the elite set, trajectory_opt.py:476) */
size_t b200pets_cem_update_workspace_bytes(int32_t population, int32_t dims, int32_t elite_num);
int b200pets_cem_update(int32_t population, int32_t dims, int32_t elite_num, float alpha, int32_t unbiased,
                        int32_t use_std, const float* population_in, float* values, float* mu,
                        float* dispersion, float* best_value, float* best_solution, int32_t* elite_idx,
                        float* elites_out, void* workspace, size_t workspace_bytes, void* stream);

/* Sharded-population variant (SURVEY.md section 8e): each rank extracts its local top-k records
 * [value, sequence(dims)], ranks all-gather them (one NCCL collective), then every rank refits from the
 * gathered records.  records [dev] float[k][1+dims]. */
int b200pets_cem_local_topk(int32_t population, int32_t dims, int32_t k, const float* population_in,
                            float* values, float* records, void* workspace, size_t workspace_bytes,
                            void* stream);
int b200pets_cem_update_from_records(int32_t num_records, int32_t dims, int32_t elite_num, float alpha,
                                     int32_t unbiased, int32_t use_std, float* records, float* mu,
                                     float* dispersion, float* best_value, float* best_solution,
                                     float* elites_out, void* workspace, size_t workspace_bytes, void* stream);

/* Sharded population, exchange over NVLink peer memory fused into the select / refit kernels (no reference counterpart;
 * SURVEY.md section 8e "stretch": the gather issued from the kernel, and its threshold-first variant for large k).
 * Every rank allocates a buffer of b200pets_peer_buffer_bytes(world, local_population, dims, elite_num) with
 * b200pets_peer_alloc (cudaMalloc + its 64-byte cudaIpcMemHandle_t); ranks exchange the handles out of band and open each
 * other's with b200pets_peer_open; peer_bufs [host] void*[world] = this process's pointer to every rank's buffer (its own
 * included).  All ranks hold the same number of sequences (contiguous shards in rank order).  Per CEM iteration
 * (epoch = 1, 2, 3, ... never reused, the same on all ranks):
 *   b200pets_cem_values_push   NaN rule in place, this rank's values -> every rank's value table + flag
 *   b200pets_cem_elites_refit  waits for all values, selects the global top elite_num (ties: lowest global index), sends the
 *                              rows of the elites this rank owns to their (index-ordered) place in every rank's elite table,
 *                              waits for all of them, refits (mu, dispersion, best) with the arithmetic of
 *                              b200pets_cem_update (unbiased variance, sums in ascending global index order), then
 *                              (sample_next != 0) draws this rank's next population shard like b200pets_cem_sample_shard.
 *                              tag_word [dev] uint32 scratch. */
size_t b200pets_peer_buffer_bytes(int32_t world, int32_t local_population, int32_t dims, int32_t elite_num);
int b200pets_peer_alloc(size_t bytes, void** ptr, uint8_t* ipc_handle64);
int b200pets_peer_open(const uint8_t* ipc_handle64, void** ptr);
int b200pets_peer_close(void* ptr, int32_t owned);
int b200pets_cem_values_push(int32_t local_population, int32_t dims, int32_t elite_num, float* values, int32_t rank,
                             int32_t world, uint32_t epoch, void* const* peer_bufs, void* stream);
int b200pets_cem_elites_refit(int32_t local_population, int32_t first_sequence, int32_t dims, int32_t elite_num,
                              float alpha, int32_t use_std, int32_t rank, int32_t world, uint32_t epoch,
                              void* const* peer_bufs, const float* population_in, float* mu, float* dispersion,
                              float* best_value, float* best_solution, int32_t sample_next, const float* lower,
                              const float* upper, uint64_t seed, uint64_t offset, int32_t clipped_normal,
                              uint32_t* tag_word, float* population_out, void* stream);

/* iCEM sampling (trajectory_opt.py:433-441 + util/math.py:318-396): coloured noise along the horizon from
 * N(0,1) draws sr, si [dev] float[n][A][H/2+1] (or NULL = Philox), scaled by sqrt(var) + mu and clipped. */
int b200pets_icem_sample(int32_t n, int32_t horizon, int32_t act_dim, float exponent, const float* mu,
                         const float* var, const float* lower, const float* upper, const float* sr,
                         const float* si, uint64_t seed, uint64_t offset, float* population_out,
                         void* stream);
/* kept elites appended to the population (trajectory_opt.py:442-466): rows index[j] of `elite`
 * [elite_num][H][A]; shift != 0 drops the first action and appends mu[-1] + sqrt(var[-1]) * end_eps[j]. */
int b200pets_icem_append_elites(int32_t keep, int32_t horizon, int32_t act_dim, const float* elite,
                                const int64_t* index, int32_t shift, const float* mu, const float* var,
                                const float* end_eps, uint64_t seed, uint64_t offset, float* dst,
                                void* stream);

/* MPPIOptimizer building blocks (trajectory_opt.py:191-311).
 * sample: population[n][t] = clip(beta * (mean[t] + noise[n][t]) + (1 - beta) * population[n][t-1]), t = 0 uses
 *   past_action; noise = N(0,1) truncated to [-2, 2] (z [dev] float[N][H][A] injected or NULL = Philox).
 * update: NaN -> -1e-10, weights exp(gamma * (v - max v)), mean <- sum(w * population) / (sum w + 1e-10). */
int b200pets_mppi_sample(int32_t population, int32_t horizon, int32_t act_dim, float beta, const float* mean,
                         const float* past_action, const float* lower, const float* upper, const float* z,
                         uint64_t seed, uint64_t offset, float* population_out, void* stream);
size_t b200pets_mppi_update_workspace_bytes(int32_t population, int32_t dims);
int b200pets_mppi_update(int32_t population, int32_t dims, float gamma, const float* population_in, float* values,
                         float* mean_out, void* workspace, size_t workspace_bytes, void* stream);

/* TrajectoryOptimizer warm start (trajectory_opt.py:563-567): roll by -replan_freq, fill the tail. */
int b200pets_shift_solution(int32_t horizon, int32_t act_dim, int32_t replan_freq, const float* best,
                            const float* initial_row, float* previous_solution, void* stream);

/* Fused CEM plan over the model (CEMOptimizer.optimize driving evaluate_action_sequences,
 * trajectory_opt.py:142-188): enqueues num_iterations x (sample -> rollout -> refit) on `stream` with no
 * host round trip.  z / eps / perms as above with a leading [num_iterations] dimension, or NULL.
 *   x0 [dev] float[H*A]; lower/upper [dev] float[H*A]
 *   solution [dev] float[H*A]; values_out [dev] float[num_iterations][N] or NULL */
typedef struct {
  int32_t num_iterations;
  int32_t elite_num;
  float alpha;
  int32_t return_mean_elites;
  int32_t clipped_normal;
} b200pets_cem_cfg;
size_t b200pets_cem_plan_workspace_bytes(b200pets_model_t model, const b200pets_rollout_cfg* rcfg,
                                         const b200pets_cem_cfg* ccfg);
int b200pets_cem_plan(b200pets_model_t model, const b200pets_rollout_cfg* rcfg, const b200pets_cem_cfg* ccfg,
                      const float* obs0, const float* x0, const float* lower, const float* upper,
                      const float* z, const float* eps, const int64_t* perms, float* solution,
                      float* values_out, void* workspace, size_t workspace_bytes, void* stream);

/* Self test of the wgmma building block: D[128][n] = A[128][k] * B[n][k]^T with bf16 operands staged in the
 * no-swizzle canonical layouts, the weight ring and the accumulator fragments the rollout kernel uses.  a, b [dev] float
 * (rounded to bf16 inside), d [dev] float[128][n].  k, n multiples of 16, <= 256.  A negative k writes A as bf16 pairs
 * per thread and row (the hidden-layer epilogue's stores) with |k|. */
int b200pets_selftest_wgmma(int32_t k, int32_t n, const float* a, const float* b, float* d, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200PETS_H */
