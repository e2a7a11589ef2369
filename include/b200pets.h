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
#define B200PETS_REWARD_EXTERNAL 255 /* reward left to the caller's callable (b200pets_step, b200pets_eval_trajectory) */

/* termination_fn: mbrl/env/termination_fns.py */
#define B200PETS_TERM_NONE 0
#define B200PETS_TERM_CARTPOLE 1
#define B200PETS_TERM_INVERTED_PENDULUM 2
#define B200PETS_TERM_HOPPER 3
#define B200PETS_TERM_WALKER2D 4
#define B200PETS_TERM_ANT 5
#define B200PETS_TERM_HUMANOID 6
#define B200PETS_TERM_EXTERNAL 255 /* b200pets_step, b200pets_eval_trajectory */

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
/* Launch plans the rollout kernels choose for this model on the current device when running `propagation`
 * (B200PETS_PROP_*), computed by the same code as the launchers:
 *   info[0] tensor-core kernel: K steps (16 weight rows each) per ring slot, 1..4; 0 = no tensor-core plan
 *   info[1] tensor-core kernel: weight ring slots (0 when info[0] == 0)
 *   info[2] tensor-core kernel: dynamic shared memory in bytes (0 when info[0] == 0)
 *   info[3] fp32 kernel: rows per CTA tile, 64, 32 or 16; 0 = the model does not fit */
int b200pets_model_plan_info(b200pets_model_t model, int32_t propagation, int32_t info[4]);

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

/* evaluate_action_sequences with reward / termination callables the kernels do not know (B200PETS_REWARD_EXTERNAL /
 * B200PETS_TERM_EXTERNAL; b200pets_eval_sequences refuses those).  The observation trajectory does not depend on reward
 * or done (model_env.py:178-191), so the evaluation runs in windows of steps [t0, t1), in order, t0 = 0 first:
 *   1. b200pets_eval_trajectory rolls the model over the window and writes, for local step s = t - t0 and row
 *      r = n*P + p: next_obs [dev] float[t1-t0][B][D], reward [dev] float[t1-t0][B] (learned column or known function;
 *      0 for an external one), done [dev] uint8[t1-t0][B] (known function; 0 for an external one).  Each may be NULL.
 *   2. the caller overwrites reward / done with its callables' values on those rows;
 *   3. b200pets_trajectory_returns applies the reference's masking (a reward after termination counts 0) and
 *      accumulates per-row totals in the workspace; after the window with t1 == H it writes returns [dev] float[N]
 *      (particle mean) and row_returns [dev] float[B] (or NULL).
 * obs0 (read when t0 == 0), actions, perms, eps and cfg are those of b200pets_eval_sequences and are passed whole for
 * every window: Philox keys, shuffle groups and shards are the same, so how H is split into windows changes nothing.
 * One workspace of b200pets_trajectory_workspace_bytes carries the row state from window to window. */
size_t b200pets_trajectory_workspace_bytes(b200pets_model_t model, const b200pets_rollout_cfg* cfg);
int b200pets_eval_trajectory(b200pets_model_t model, const b200pets_rollout_cfg* cfg, int32_t t0, int32_t t1,
                             const float* obs0, const float* actions, const int64_t* perms, const float* eps,
                             float* next_obs, float* reward, uint8_t* done, void* workspace, size_t workspace_bytes,
                             void* stream);
int b200pets_trajectory_returns(const b200pets_rollout_cfg* cfg, int32_t t0, int32_t t1, const float* reward,
                                const uint8_t* done, float* returns, float* row_returns, void* workspace,
                                size_t workspace_bytes, void* stream);

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
 * N(0,1) draws sr, si [dev] float[n][A][H/2+1] (or NULL = Philox), scaled by sqrt(var) + mu and clipped.
 * horizon < 2 is refused (B200PETS_EINVAL): a one-sample series has no frequency to normalise the noise by. */
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
 * trajectory_opt.py:142-188): enqueues the first population, then per iteration the rollout and one kernel that refits
 * and draws the next population (two launches per iteration), on `stream` with no host round trip.  Outside that
 * kernel's single-CTA refit (more than 2048 sequences, fewer than 2 elites, or elite rows over 150 KB) the plan runs
 * sample -> rollout -> refit instead (three launches per iteration).  z / eps / perms as above with a leading
 * [num_iterations] dimension, or NULL.
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

/* Batches of independent problems (a vectorised environment, several episodes or seeds side by side): K evaluations or
 * K CEM plans that share the model, the action bounds and the configuration, each with its own initial observation,
 * warm start, sampling distribution, elites and solution, run in one launch per rollout / refit instead of K.  Problem k
 * gives, bit for bit, the single call's result for its inputs made with the Philox offset the batch assigns to it:
 *   b200pets_eval_sequences_batch: cfg->offset + k * 1024 (the offset of a single evaluation k ModelEnv calls later);
 *   b200pets_cem_plan_batch:       rcfg->offset + k (a single plan turns it into (offset + k) * 1024 + iteration).
 * Every array of a single call takes a leading [K] dimension (problem k's slice is the array its single call takes);
 * lower / upper are shared:
 *   obs0 [dev] float[K][D]; actions [dev] float[K][N][H][A]; perms [dev] int64[K][H or 1][B] or NULL;
 *   eps [dev] float[K][H][B][out] or NULL; returns [dev] float[K][N]; row_returns [dev] float[K][B] or NULL;
 *   plan: x0 [dev] float[K][H*A]; z [dev] float[K][it][N][H*A], eps [dev] float[K][it][H][B][out],
 *   perms [dev] int64[K][it][H or 1][B] (each or NULL); solution [dev] float[K][H*A];
 *   values_out [dev] float[K][it][N] or NULL.
 * The plan runs the default structure of b200pets_cem_plan (rollout, then refit + next population: two launches per
 * iteration for the whole batch).  Refused: num_problems < 1, a sharded cfg (first_sequence != 0 or global_population
 * other than 0 / population), external reward / termination callables. */
size_t b200pets_eval_batch_workspace_bytes(b200pets_model_t model, const b200pets_rollout_cfg* cfg, int32_t num_problems);
int b200pets_eval_sequences_batch(b200pets_model_t model, const b200pets_rollout_cfg* cfg, int32_t num_problems,
                                  const float* obs0, const float* actions, const int64_t* perms, const float* eps,
                                  float* returns, float* row_returns, void* workspace, size_t workspace_bytes,
                                  void* stream);
size_t b200pets_cem_plan_batch_workspace_bytes(b200pets_model_t model, const b200pets_rollout_cfg* rcfg,
                                               const b200pets_cem_cfg* ccfg, int32_t num_problems);
int b200pets_cem_plan_batch(b200pets_model_t model, const b200pets_rollout_cfg* rcfg, const b200pets_cem_cfg* ccfg,
                            int32_t num_problems, const float* obs0, const float* x0, const float* lower,
                            const float* upper, const float* z, const float* eps, const int64_t* perms,
                            float* solution, float* values_out, void* workspace, size_t workspace_bytes,
                            void* stream);

/* K MPPIOptimizer.optimize calls over ModelEnv.evaluate_action_sequences (trajectory_opt.py:239-311), one per
 * observation, each from its own carried mean.  The plan first shifts every problem's mean (mean[:-1] = mean[1:], past
 * action = the shifted mean[0]), then runs per refinement four launches for the whole batch: sample, rollout, particle
 * mean, update.  Problem k gives, bit for bit, the k-th of K consecutive single plans:
 *   population noise of refinement r: Philox key sample_seed (the optimiser's seed), offset
 *     (sample_counter + k) * 1024 + r;
 *   rollout of refinement r: key rcfg->seed (the environment's), offset (rcfg->offset + k * R + r) * 1024, R =
 *     num_iterations.  A batch therefore takes K optimiser and K * R environment counter values.
 * Arrays (problem k's slice is the array its single call takes; lower / upper are shared):
 *   obs0 [dev] float[K][D]; mean [dev] float[K][H][A]: the carried means in, the plans out;
 *   lower / upper [dev] float[H][A]; z [dev] float[K][R][N][H][A] or NULL (Philox);
 *   eps [dev] float[K][R][H][B][out] or NULL; perms [dev] int64[K][R][H or 1][B] or NULL (tile shuffle);
 *   values_out [dev] float[K][R][N] (after the NaN rule) or NULL.
 * num_iterations 0 returns the shifted means.  Refused: num_problems < 1, a sharded rcfg (first_sequence != 0 or
 * global_population other than 0 / population), external reward / termination callables, a negative num_iterations,
 * NULL obs0 / mean / lower / upper / workspace, a workspace smaller than b200pets_mppi_plan_batch_workspace_bytes. */
typedef struct {
  int32_t num_iterations; /* refinements R (0: the shift alone, as the single path does) */
  float gamma, beta;
  uint64_t sample_seed;    /* Philox key of the population noise: the optimiser's seed, not the environment's */
  uint64_t sample_counter; /* problem k, refinement r draws with offset (sample_counter + k) * 1024 + r */
} b200pets_mppi_cfg;
size_t b200pets_mppi_plan_batch_workspace_bytes(b200pets_model_t model, const b200pets_rollout_cfg* rcfg,
                                                const b200pets_mppi_cfg* mcfg, int32_t num_problems);
int b200pets_mppi_plan_batch(b200pets_model_t model, const b200pets_rollout_cfg* rcfg, const b200pets_mppi_cfg* mcfg,
                             int32_t num_problems, const float* obs0, float* mean, const float* lower,
                             const float* upper, const float* z, const float* eps, const int64_t* perms,
                             float* values_out, void* workspace, size_t workspace_bytes, void* stream);

/* ---- PlaNet's latent model (mbrl/models/planet.py, mbrl/algorithms/planet.py) --------------------------------
 * The prior transition and reward models PlaNet plans with, PlaNetModel.sample (planet.py:531-581), in fp32:
 *   e = relu(W_e [s, a] + b_e);  h' = GRUCell(e, h);  p = W_p2 relu(W_p1 h' + b_p1) + b_p2;
 *   s' = p[:L] + (softplus(p[L:]) + min_std) * eps  (s' = p[:L] when deterministic);
 *   reward = W_r3 relu(W_r2 relu(W_r1 [h', s'] + b_r1) + b_r2) + b_r3.
 * The encoder, the posterior and the decoder (update_posterior, training) stay with the caller. */
typedef struct b200pets_latent_model_s* b200pets_latent_model_t;
typedef struct {
  int32_t action_size;  /* A */
  int32_t latent_size;  /* L, latent_state_size */
  int32_t belief_size;  /* Hb */
  int32_t hidden_size;  /* Hf, hidden_size_fcs */
  float min_std;
} b200pets_latent_model_desc;

/* params [host] array of B200PETS_LATENT_NUM_PARAMS device pointers to contiguous fp32 tensors in torch's layout:
 *    0 W_e [Hb][L+A], 1 b_e [Hb]                                belief_model.embedding_layer[0]
 *    2 weight_ih [3Hb][Hb], 3 weight_hh [3Hb][Hb], 4 bias_ih [3Hb], 5 bias_hh [3Hb]   belief_model.rnn (gates r, z, n)
 *    6 W_p1 [Hf][Hb], 7 b_p1 [Hf]                               prior_transition_model[0]
 *    8 W_p2 [2L][Hf], 9 b_p2 [2L]                               prior_transition_model[2]
 *   10 W_r1 [Hf][Hb+L], 11 b_r1 [Hf]                            reward_model[0] (input: belief, then latent)
 *   12 W_r2 [Hf][Hf], 13 b_r2 [Hf]                              reward_model[2]
 *   14 W_r3 [1][Hf], 15 b_r3 [1]                                reward_model[4]
 * Staging packs transposed copies on `stream` (no host round trip); refresh re-packs them after the weights changed.
 * Refused (B200PETS_EUNSUPPORTED): a model whose per-row state needs more than an eighth of the device's opt-in shared
 * memory per CTA (29 056 bytes on an H100: about belief = hidden = 1200 at L 30, A 6); b200pets_latent_plan_info
 * reports the bytes per row. */
#define B200PETS_LATENT_NUM_PARAMS 16
int b200pets_latent_model_create(const b200pets_latent_model_desc* desc, const float* const* params, void* stream,
                                 b200pets_latent_model_t* out);
int b200pets_latent_model_refresh(b200pets_latent_model_t model, const float* const* params, void* stream);
void b200pets_latent_model_destroy(b200pets_latent_model_t model);
/* The rollout kernel's launch for `rows` rows on the current device:
 *   info[0] rows per CTA (1, 2, 4, 8, 16 or 32: enough CTAs to cover the SMs once, at most 32 rows)
 *   info[1] CTAs;  info[2] dynamic shared memory of one CTA in bytes;  info[3] shared memory bytes of one row */
int b200pets_latent_plan_info(b200pets_latent_model_t model, int64_t rows, int32_t info[4]);

/* ModelEnv.step over PlaNetModel.sample (model_env.py:87-140) for `batch` independent states, one launch:
 *   latent [dev] float[B][L], belief [dev] float[B][Hb], act [dev] float[B][A]
 *   eps [dev] float[B][L] injected N(0,1) draws or NULL = Philox (RNG_STREAM_LATENT, step 0, key seed / offset);
 *   sample == 0 returns the prior's mean (deterministic=True) and reads no draw
 *   next_latent [dev] float[B][L], next_belief [dev] float[B][Hb], reward [dev] float[B] (each may be NULL) */
int b200pets_latent_step(b200pets_latent_model_t model, int64_t batch, const float* latent, const float* belief,
                         const float* act, const float* eps, uint64_t seed, uint64_t offset, int32_t sample,
                         float* next_latent, float* next_belief, float* reward, void* stream);

/* ModelEnv.evaluate_action_sequences over PlaNetModel with no_termination (model_env.py:145-191): every row starts at
 * the posterior, row r = n * P + p follows sequence n, draws every step (sample=True), sums the rewards; returns the
 * particle mean.  One launch for the whole horizon, plus the particle mean.
 * The latent entry points read population, horizon, particles, seed and offset of b200pets_rollout_cfg; precision must
 * be B200PETS_PREC_F32, first_sequence 0 and global_population 0 or population (no sharding); propagation and ts1_mode
 * are not read.
 *   latent0 [dev] float[L], belief0 [dev] float[Hb]: the posterior (PlaNetModel.reset repeats it)
 *   actions [dev] float[N][H][A]; eps [dev] float[H][B][L] or NULL = Philox (row r, step t as in b200pets_latent_step)
 *   returns [dev] float[N]; row_returns [dev] float[B] or NULL */
size_t b200pets_latent_eval_workspace_bytes(b200pets_latent_model_t model, const b200pets_rollout_cfg* cfg);
int b200pets_latent_eval_sequences(b200pets_latent_model_t model, const b200pets_rollout_cfg* cfg, const float* latent0,
                                   const float* belief0, const float* actions, const float* eps, float* returns,
                                   float* row_returns, void* workspace, size_t workspace_bytes, void* stream);

/* CEMOptimizer.optimize over the latent model's evaluate_action_sequences as one call: the structure, Philox offsets
 * (offset * 1024 + iteration for the population and the rollout) and values_out of b200pets_cem_plan, with the latent
 * rollout in place of the ensemble's.  b200pets_cem_cfg is read whole.  z [dev] float[it][N][H*A] or NULL,
 * eps [dev] float[it][H][B][L] or NULL; x0, lower, upper, solution [dev] float[H*A]; values_out [dev] float[it][N] or
 * NULL. */
size_t b200pets_latent_cem_plan_workspace_bytes(b200pets_latent_model_t model, const b200pets_rollout_cfg* rcfg,
                                                const b200pets_cem_cfg* ccfg);
int b200pets_latent_cem_plan(b200pets_latent_model_t model, const b200pets_rollout_cfg* rcfg, const b200pets_cem_cfg* ccfg,
                             const float* latent0, const float* belief0, const float* x0, const float* lower,
                             const float* upper, const float* z, const float* eps, float* solution, float* values_out,
                             void* workspace, size_t workspace_bytes, void* stream);

/* ---- Training PlaNet's latent model: the recurrence of PlaNetModel.forward (planet.py:354-404) ------------------
 * The belief GRU, the posterior and the prior over T steps from s0 = 0, h0 = 0 (planet.py:364-367), in fp32 FFMA:
 *   e = relu(W_e [s, a_t] + b_e);  h = GRUCell(e, h);
 *   q = W_q2 relu(W_q1[:, :Hb] h + P_t) + b_q2;  s = q[:L] + (softplus(q[L:]) + min_std) * eps_q;
 *   p = W_p2 relu(W_p1 h + b_p1) + b_p2;        s_prior = p[:L] + (softplus(p[L:]) + min_std) * eps_p.
 * P_t = W_q1[:, Hb:] enc_t + b_q1 (the posterior's encoding half) comes in precomputed for every (b, t); the encoder,
 * the decoder, the reward model and the losses stay with the caller.  The backward pass runs t = T-1 .. 0 and writes
 * dP and every layer's pre-activation gradient for all (b, t) into the tape: the weight gradients are products of
 * those with the stored layer inputs over all B x T rows, which the caller forms.  Sums run in a fixed order, so both
 * calls are bit-identical from run to run. */
typedef struct {
  int32_t action_size;    /* A */
  int32_t latent_size;    /* L */
  int32_t belief_size;    /* Hb */
  int32_t hidden_size;    /* Hf */
  int32_t encoding_size;  /* E, obs_encoding_size */
  float min_std;
} b200pets_latent_train_desc;

/* params [host] array of B200PETS_LATENT_TRAIN_NUM_PARAMS device pointers to contiguous fp32 tensors in torch's layout:
 *    0 W_e [Hb][L+A], 1 b_e [Hb]                                belief_model.embedding_layer[0]
 *    2 weight_ih [3Hb][Hb], 3 weight_hh [3Hb][Hb], 4 bias_ih [3Hb], 5 bias_hh [3Hb]   belief_model.rnn (gates r, z, n)
 *    6 W_q1 [Hf][Hb+E] (only the belief columns are read)       posterior_transition_model[0] (input: belief, encoding)
 *    7 W_q2 [2L][Hf], 8 b_q2 [2L]                               posterior_transition_model[2]
 *    9 W_p1 [Hf][Hb], 10 b_p1 [Hf]                              prior_transition_model[0]
 *   11 W_p2 [2L][Hf], 12 b_p2 [2L]                              prior_transition_model[2] */
#define B200PETS_LATENT_TRAIN_NUM_PARAMS 13

/* What the backward pass needs from the forward pass, and the pre-activation gradients it writes: caller-owned device
 * arrays, each [B][T][width] fp32 (row b * T + t).  Forward: e [Hb] (the embedding after its ReLU), gates [4Hb]
 * (r, z, n, W_hn h + b_hn), q1 [Hf] and p1 [Hf] (the posterior's and the prior's hidden layer after its ReLU), pre_std
 * [2L] (q[L:], then p[L:]), eps [2L] (the posterior's draws, then the prior's).  Backward: de [Hb] (embedding
 * pre-activation), dgi [3Hb] (GRU input-side pre-activations r, z, n), dghn [Hb] (W_hn h + b_hn), dq [2L] (posterior
 * layer 2), dv [Hf] (prior layer 1), dp [2L] (prior layer 2).  The hidden-side gradients of r and z equal dgi's, and
 * the posterior's layer-1 pre-activation gradient is dP. */
typedef struct {
  float *e, *gates, *q1, *p1, *pre_std, *eps;
  float *de, *dgi, *dghn, *dq, *dv, *dp;
} b200pets_latent_tape;

/* 0 when the kernels cover `desc`, asked before anything is touched.  B200PETS_EINVAL for sizes below 1 or min_std
 * below 0; B200PETS_EUNSUPPORTED when a row of the forward or the backward kernel needs more than an eighth of the
 * device's opt-in shared memory per CTA (PlaNet's A 6, L 30, Hb = Hf = 200 needs 7 808 bytes; the limit is 29 056 on an
 * H100, which admits Hb = Hf up to 788 at A 6, L 30). */
int b200pets_latent_train_supported(const b200pets_latent_train_desc* desc);
/* Bytes of the workspace b200pets_latent_seq_forward re-packs the weights into (0 for bad arguments). */
size_t b200pets_latent_train_workspace_bytes(const b200pets_latent_train_desc* desc, int32_t batch, int32_t steps);
/* The forward pass (planet.py:370-402 without the decoder and the reward model), one re-pack and one launch:
 *   P [dev] float[B][T][Hf]; act [dev] float[B][T][A] (action[:, :-1]);
 *   eps_q, eps_p [dev] float[T][B][L] injected N(0,1) draws (both or neither), or NULL = Philox on RNG_STREAM_LATENT_TRAIN
 *   with key (seed, offset);
 *   beliefs [dev] float[B][T][Hb], post_params / prior_params [dev] float[B][T][2L] (mean, then std), post_samples /
 *   prior_samples [dev] float[B][T][L]: the five stacked outputs of PlaNetModel.forward;
 *   tape: every forward field set, or NULL when no backward pass follows (no_grad). */
int b200pets_latent_seq_forward(const b200pets_latent_train_desc* desc, const float* const* params, int32_t batch,
                                int32_t steps, const float* P, const float* act, const float* eps_q, const float* eps_p,
                                uint64_t seed, uint64_t offset, float* beliefs, float* post_params, float* post_samples,
                                float* prior_params, float* prior_samples, const b200pets_latent_tape* tape,
                                void* workspace, size_t workspace_bytes, void* stream);
/* The backward pass of the same call, after it on the same weights: the upstream gradients of the five outputs (each
 * may be NULL = zero), beliefs [dev] as the forward pass wrote them, the tape (every field set) in; dP [dev]
 * float[B][T][Hf] and the tape's backward fields out.  Reads torch's tensors directly: no workspace. */
int b200pets_latent_seq_backward(const b200pets_latent_train_desc* desc, const float* const* params, int32_t batch,
                                 int32_t steps, const float* beliefs, const float* g_beliefs, const float* g_post_params,
                                 const float* g_post_samples, const float* g_prior_params, const float* g_prior_samples,
                                 const b200pets_latent_tape* tape, float* dP, void* stream);

/* ---- Training the dynamics model (mbrl/models/model_trainer.py:70-262) ------------------------------------
 * OneDTransitionRewardModel(GaussianMLP) trained with torch.optim.Adam, fp32 throughout. */

/* element type of transition arrays */
#define B200PETS_DTYPE_F32 0
#define B200PETS_DTYPE_F64 1

/* Raw transitions -> model inputs and targets (one_dim_tr_model.py:103-136), for a whole dataset at once:
 *   inputs  [dev] float[rows][in_size]  = normalise(cat(obs_process_fn(obs), act)): norm_mode 1 (fp32 statistics, norm_mean /
 *           norm_std [dev] float[in_size]) or 2 (fp64, [dev] double[in_size], the result rounded to fp32), 0 = none
 *   targets [dev] float[rows][out_size] = next_obs - obs (next_obs for the no_delta columns, or for all of them when
 *           target_is_delta == 0), then reward as the last column when learned_rewards
 *   obs, next_obs [dev] [rows][obs_dim]; act [dev] [rows][act_dim]; reward [dev] [rows] (read only when learned_rewards),
 *   all of element type `dtype`: B200PETS_DTYPE_F32 (float) or B200PETS_DTYPE_F64 (double).  Float64 transitions are
 *   processed in double, as numpy processes them in the reference (obs_process_fn, delta, normaliser; fp32 statistics
 *   promoted to double), and rounded to float at the end;
 *   no_delta [host] int32[num_no_delta] observation columns, each < obs_dim <= 1024.
 * in_size = obs_dim (+1 for B200PETS_PROC_CARTPOLE) + act_dim, out_size = obs_dim + learned_rewards.
 * Refused: NULL pointers, an unknown dtype, obs_process or norm_mode, a no_delta column out of range. */
typedef struct {
  int32_t obs_dim, act_dim, obs_process, norm_mode, target_is_delta, learned_rewards;
  int32_t dtype; /* B200PETS_DTYPE_* of obs, act, next_obs, reward */
} b200pets_prep_desc;
int b200pets_train_preprocess(const b200pets_prep_desc* desc, int64_t rows, const void* obs, const void* act,
                              const void* next_obs, const void* reward, const void* norm_mean, const void* norm_std,
                              const int32_t* no_delta, int32_t num_no_delta, float* inputs, float* targets, void* stream);

/* A trainer: the caller's GaussianMLP parameters and torch.optim.Adam state (exp_avg, exp_avg_sq), updated in place by
 * the kernels; nothing is copied and no gradient buffer exists.  Entries of params / exp_avg / exp_avg_sq [host arrays of
 * dev pointers]: W_0, b_0, ..., W_L, b_L (L = num_hidden; W_l float[E][K_l][N_l], b_l float[E][1][N_l], N_L = out_size or
 * 2 * out_size), then, unless deterministic, min_logvar and max_logvar (float[1][out_size]); the moments of the bounds are
 * read only with learn_logvar_bounds (otherwise the bounds are constants, as with requires_grad=False) and may be NULL.
 * Adam hyper-parameters are torch's (lr, betas, eps, weight_decay as L2 added to the gradient).  Refused: NULL desc /
 * out / parameter or moment pointers, num_hidden < 1 or num_hidden + 1 > B200PETS_MAX_LAYERS (8), an unknown
 * activation, non-positive sizes. */
typedef struct b200pets_trainer_s* b200pets_trainer_t;
typedef struct {
  int32_t ensemble_size, in_size, out_size, hid_size, num_hidden;
  int32_t activation; /* B200PETS_ACT_* */
  float leaky_slope;
  int32_t deterministic;
  int32_t learn_logvar_bounds;
  double lr, beta1, beta2, eps, weight_decay;
} b200pets_train_desc;
int b200pets_trainer_create(const b200pets_train_desc* desc, float* const* params, float* const* exp_avg,
                            float* const* exp_avg_sq, b200pets_trainer_t* out);
void b200pets_trainer_destroy(b200pets_trainer_t trainer);
/* Whether the training kernels cover a model, asked before any tensor exists: 0 when b200pets_trainer_create accepts
 * desc (pointers aside) and b200pets_eval_score can evaluate its layers on the current device; otherwise the code and
 * b200pets_last_error() that the first of the two refusals gives (num_hidden > 7, or layers about 890 columns wide). */
int b200pets_trainer_supported(const b200pets_train_desc* desc);

/* One epoch of ModelTrainer.train (model_trainer.py:152-156): `steps` minibatch updates (model.update: loss, backward,
 * optimizer.step) enqueued on `stream` as one launch, with no host synchronisation.
 *   inputs / targets [dev] the dataset (b200pets_train_preprocess), rows rows
 *   indices [dev] int32[E][steps][batch]: rows of member e's minibatch at each step (a bootstrapped minibatch; give every
 *           member the same rows for a plain TransitionIterator batch); every step has `batch` rows except the last, which
 *           has last_batch (<= batch) and reads the first last_batch entries of its slice; entries must lie in [0, rows)
 *   adam_step the optimizer's step count before the epoch (bias correction of step s uses adam_step + s + 1)
 *   losses [dev] float[steps]: the loss of every step (loss.item() of the reference)
 * Refused: NULL pointers, steps < 1, batch < 1, last_batch not in [1, batch], a workspace smaller than
 * b200pets_train_workspace_bytes(trainer, batch). */
size_t b200pets_train_workspace_bytes(b200pets_trainer_t trainer, int32_t batch);
int b200pets_train_epoch(b200pets_trainer_t trainer, int64_t rows, const float* inputs, const float* targets,
                         const int32_t* indices, int32_t steps, int32_t batch, int32_t last_batch, int64_t adam_step,
                         float* losses, void* workspace, size_t workspace_bytes, void* stream);

/* ModelTrainer.evaluate (model_trainer.py:216-262) over a whole dataset in one launch: scores [dev] float[E], the mean
 * over rows and output columns of member e's squared error (OneDTransitionRewardModel.eval_score).  Refused: NULL
 * pointers, rows < 1, a workspace smaller than b200pets_eval_score_workspace_bytes(trainer, rows), layers wider than the
 * kernel's shared-memory tile (B200PETS_EUNSUPPORTED). */
size_t b200pets_eval_score_workspace_bytes(b200pets_trainer_t trainer, int64_t rows);
int b200pets_eval_score(b200pets_trainer_t trainer, int64_t rows, const float* inputs, const float* targets, float* scores,
                        void* workspace, size_t workspace_bytes, void* stream);

/* ---- Training MBPO's SAC agent (mbrl/third_party/pytorch_sac_pranz24/sac.py) ----------------------------------------
 * An agent: the caller's live tensors, updated in place by b200pets_sac_update; nothing is copied.
 *   params      [host array of 20 dev pointers] the critic's 12 parameters in QNetwork.parameters() order (linear1.weight,
 *               linear1.bias, .., linear6.bias), then the policy's 8 in GaussianPolicy.parameters() order (linear1,
 *               linear2, mean_linear, log_std_linear; weight, bias).  Weights are nn.Linear's float[out][in].
 *   target_params [12] critic_target's parameters, in the critic's order
 *   exp_avg, exp_avg_sq [20] the Adam moments of params, same order (critic_optim's, then policy_optim's)
 *   log_alpha, log_alpha_exp_avg, log_alpha_exp_avg_sq [dev] float[1]: read only with automatic_entropy_tuning (may be
 *               NULL otherwise)
 * Refused: NULL pointers, non-positive sizes, act_dim > 32 (the policy heads' row-wise phase holds a row's actions in
 * one 32-column tile: B200PETS_EUNSUPPORTED), target_update_interval < 1. */
#define B200PETS_SAC_MAX_ACTIONS 32
#define B200PETS_SAC_NUM_PARAMS 20
#define B200PETS_SAC_NUM_CRITIC_PARAMS 12
typedef struct b200pets_sac_s* b200pets_sac_t;
typedef struct {
  int32_t obs_dim, act_dim, hidden;
  float action_scale[B200PETS_SAC_MAX_ACTIONS], action_bias[B200PETS_SAC_MAX_ACTIONS]; /* first act_dim entries */
  double gamma, tau, lr, beta1, beta2, eps; /* one lr and one set of betas for the three optimizers, no weight decay */
  int32_t automatic_entropy_tuning;
  float target_entropy;
  int32_t target_update_interval;
} b200pets_sac_desc;
int b200pets_sac_supported(const b200pets_sac_desc* desc);
int b200pets_sac_create(const b200pets_sac_desc* desc, float* const* params, float* const* target_params,
                        float* const* exp_avg, float* const* exp_avg_sq, float* log_alpha, float* log_alpha_exp_avg,
                        float* log_alpha_exp_avg_sq, b200pets_sac_t* out);
void b200pets_sac_destroy(b200pets_sac_t sac);

/* One SAC.update_parameters (sac.py:76-173) after its memory.sample, enqueued on `stream` as one launch, with no host
 * synchronisation: the critic step, the policy step against the updated critic, the temperature step (with
 * automatic_entropy_tuning) and, when updates % target_update_interval == 0, the soft target update.
 *   updates       the reference's `updates` argument (>= 0)
 *   reverse_mask  nonzero: the target's mask is 1 - terminated (as MBPO calls it), else terminated
 *   adam_steps    [host] int64[3]: the step counts of critic_optim, policy_optim and alpha_optim before this update
 *   transitions   [dev] float[batch][2 * obs_dim + act_dim + 2]: s, a, s', r, terminated (0 or 1)
 *   eps           [dev] float[2][batch][act_dim]: the reparameterisation draws on s' and on s, or NULL for the in-kernel
 *                 Philox draws keyed by (seed, offset) (RNG_STREAM_SAC in csrc/common.cuh)
 *   alpha         [dev] float[1]: the temperature this update uses; written with exp(log_alpha) when tuning
 *   stats         [dev] float[8]: qf1 loss, qf2 loss, policy loss, alpha loss, alpha after the update, the batch's mean
 *                 reward, -mean(log pi), 0
 * Refused: NULL pointers, batch < 1, updates < 0, a workspace smaller than b200pets_sac_workspace_bytes(sac, batch). */
size_t b200pets_sac_workspace_bytes(b200pets_sac_t sac, int32_t batch);
int b200pets_sac_update(b200pets_sac_t sac, int32_t batch, int64_t updates, int32_t reverse_mask,
                        const int64_t* adam_steps, const float* transitions, const float* eps, uint64_t seed,
                        uint64_t offset, float* alpha, float* stats, void* workspace, size_t workspace_bytes,
                        void* stream);

/* Self test of the wgmma building block: D[128][n] = A[128][k] * B[n][k]^T with bf16 operands staged in the
 * no-swizzle canonical layouts, the weight ring and the accumulator fragments the rollout kernel uses.  a, b [dev] float
 * (rounded to bf16 inside), d [dev] float[128][n].  k, n multiples of 16, <= 256.  A negative k writes A as bf16 pairs
 * per thread and row (the hidden-layer epilogue's stores) with |k|. */
int b200pets_selftest_wgmma(int32_t k, int32_t n, const float* a, const float* b, float* d, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200PETS_H */
