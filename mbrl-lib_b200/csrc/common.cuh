// Shared device-side definitions of the PETS planning kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200pets.h"

#define B200PETS_MAX_LAYERS 8

// Everything a rollout kernel needs to know about the staged model; passed by value (kernel parameter).
struct ModelDev {
  int E, M, D, A, Dp, in, out, hid, L;  // L = hidden layers; layers = L + 1
  int nout;                             // width of the last layer: out (deterministic) or 2*out
  int act;
  float leaky;
  int obs_process, learned_rewards, target_is_delta, deterministic, reward_fn, term_fn, norm_mode;
  int K[B200PETS_MAX_LAYERS], N[B200PETS_MAX_LAYERS];
  const float* W[B200PETS_MAX_LAYERS];  // gathered elite members: [M][K][N]
  const float* b[B200PETS_MAX_LAYERS];  // [M][N]
  const double* norm_mean_d;            // [in]
  const double* norm_std_d;
  const float* norm_mean_f;
  const float* norm_std_f;
  const float* norm_istd_f;             // 1/std in fp32 (tensor-core path)
  const float* min_lv;                  // [out]
  const float* max_lv;
  const uint8_t* no_delta;              // [D] mask
  // tensor-core images (bf16, no-swizzle K-major canonical layout of wgmma), see rollout_tc.cu
  const uint8_t* img;                   // base of member 0
  uint32_t img_member_stride;           // bytes between members
  uint32_t img_replica_stride;          // bytes between replicas of the whole image set
  int img_replicas;                     // copies at distinct addresses: spreads simultaneous readers over L2 slices
  uint32_t img_layer_off[B200PETS_MAX_LAYERS];
  int Kp[B200PETS_MAX_LAYERS], Np[B200PETS_MAX_LAYERS];
  int outp;                             // padded out (multiple of 16): logvar columns start here
};

// One launch of a rollout kernel: steps [t0, t1) of every tile.
struct RolloutArgs {
  int N, H, P;          // population, horizon (stride of the action tensor), particles
  long long B;          // rows
  int t0, t1;
  int propagation;      // B200PETS_PROP_*
  int slot_mode;        // 0: rid = perm[slot] (or slot if perm == NULL), members own contiguous slot ranges
                        // 1: tile shuffle (see "tile shuffle" below): member drawn per (shuffle group, step)
                        // 2: as 1 but the member is drawn once per group (TSinf without an injected permutation)
  int seq0;             // tile shuffle: global index of this shard's first sequence (0 on one GPU)
  int n_glob;           // tile shuffle: global population (= N on one GPU); fixes the global group numbering
  const long long* perm;   // [B] for this launch or NULL
  // slot_mode 0 with per-row members (B200PETS_MEMBER_ROWS): [M+1] slot offsets of the members, perm = slot -> row
  // (member_slots_kernel); member m owns slots [member_off[m], member_off[m+1]).  NULL: the equal split above.
  const int* member_off;
  const float* eps;        // [t1-t0][B][out] for this launch (row-id indexed) or NULL -> Philox
  int sample;              // 0: mean prediction
  unsigned long long seed, offset;
  // action source: act + (rid / act_div) * act_row_stride + t * act_t_stride
  const float* act;
  long long act_row_stride;
  int act_div, act_t_stride;
  // state
  const float* obs0;       // [D] broadcast initial state (used when init_from_obs0)
  int init_from_obs0;
  const float* obs_in;     // [B][D] gather source when !init_from_obs0
  float* obs_out;          // [B][D] scatter target (NULL when the state is not needed after the launch)
  float* total_state;      // [B]
  uint8_t* dead_state;     // [B]
  int load_state, store_state;
  // step outputs (b200pets_step): next_obs = obs_out, reward, done
  float* reward_out;       // [B] or NULL
  uint8_t* done_out;       // [B] or NULL
  // trajectory outputs (b200pets_eval_trajectory): step t of the launch lands at [t - t0][rid]; NULL = not stored
  float* traj_obs;         // [t1-t0][B][D] next observation
  float* traj_reward;      // [t1-t0][B] the learned column or the known reward function, 0 for an external one
  uint8_t* traj_done;      // [t1-t0][B] the known termination function, 0 for an external one
};

// A batched launch: K independent evaluations of one configuration in one grid.  Tiles are problem-major (tile =
// k * tiles + local tile); problem k reads and writes base + k * stride of every per-problem array of RolloutArgs and
// draws with Philox offset `offset + k * offset_step` (keyed from the unkeyed `seed` as the C entry points do).  Every
// other field of RolloutArgs is shared, and a problem's rows do exactly what they do in a single launch.
struct BatchArgs {
  long long tiles;                 // tiles of one problem: the count a single launch of the configuration has
  long long obs0;                  // [D] initial observation
  long long obs_state;             // obs_in / obs_out [B][D]
  long long act;                   // action source
  long long rows;                  // total_state / dead_state [B]
  long long perm, eps;             // injected permutation / model noise
  unsigned long long seed, offset_step;
  long long member_off;            // member slot offsets (RolloutArgs::member_off)
};

// Launch plans, chosen on the host from the model's shape and the device's opt-in shared memory (the launchers and
// b200pets_model_plan_info call the same functions).
struct F32Plan {
  int rows;     // rows per CTA tile of rollout_f32_kernel: 64, 32 or 16 (0: no tile fits)
  int LD;       // row stride (floats) of the activation buffers
  int wmax;     // widest layer (input or output columns)
  size_t smem;  // dynamic shared memory of one CTA
};
int f32_tile_plan(const ModelDev& m, F32Plan* p);
// tensor-core kernel: K steps per ring slot (0: no plan for this propagation), ring slots, dynamic shared memory
int tc_plan_info(const ModelDev& m, bool expectation, int* kslice, int* nstages, int* smem_bytes);

// ------------------------------------------------------------------------------------------------------
// Philox4x32-10 counter RNG (Salmon et al. 2011).  key = seed, counter = (a, b, c, d).
// ------------------------------------------------------------------------------------------------------
struct U4 {
  uint32_t x, y, z, w;
};

__device__ __forceinline__ U4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                            uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return U4{c0, c1, c2, c3};
}

__device__ __forceinline__ float u32_to_unit(uint32_t x) {  // (0, 1)
  return ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f);
}

// four N(0,1) draws from one Philox block (not inlined: ~150 instructions, called from several cold places)
// Not inlined (code size), result returned BY VALUE in registers: an out-pointer would put the caller's array in
// local memory, which misses the small L1 left beside the shared-memory carve-out.
static __device__ __noinline__ float4 philox_normal4v(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                  unsigned long long seed) {
  U4 r = philox4x32_10(c0, c1, c2, c3, (uint32_t)seed, (uint32_t)(seed >> 32));
  float u0 = u32_to_unit(r.x), u1 = u32_to_unit(r.y), u2 = u32_to_unit(r.z), u3 = u32_to_unit(r.w);
  float r0 = sqrtf(-2.0f * __logf(u0)), r1 = sqrtf(-2.0f * __logf(u2));
  float s0, c0f, s1, c1f;
  __sincosf(6.283185307179586f * u1, &s0, &c0f);
  __sincosf(6.283185307179586f * u3, &s1, &c1f);
  return make_float4(r0 * c0f, r0 * s0, r1 * c1f, r1 * s1);
}
__device__ __forceinline__ void philox_normal4(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, unsigned long long seed,
                                               float out[4]) {
  const float4 v = philox_normal4v(c0, c1, c2, c3, seed);
  out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w;
}

// RNG stream tags (third counter word, high bits)
// rollout_f32.cu / rollout_tc.cu, the Gaussian output noise of column o (the learned-reward column o = out - 1 included)
// of row r at step t: philox_normal4(r, t, RNG_STREAM_EPS | (o >> 2), low word of off, rng_key(seed, off)), lane o & 3 (r: the
// global row (seq0 + n) * P + p, under an explicit permutation the row perm[slot] holds, not the slot; t: the step of the
// evaluation, 0 for b200pets_step, whose rows are r with P = 1; off: the call's offset, offset + k * offset_step for
// problem k of a batched launch).  Under expectation each (row, t, o) draws once, after the member passes.
#define RNG_STREAM_EPS 0x10000u
// shuffle_member below, the member of tile-shuffle group gt at step t: (x * M) >> 32, a position in the elite list, with
// x word 0 of philox4x32_10(gt, t, RNG_STREAM_MEMBER, low word of off, low word of s, high word of s ^ high word of gt),
// s = rng_key(seed, off) (gt = p * C_glob + global sequence / 128, see "tile shuffle" below; t = 0 when the member is
// drawn once per group (fixed_model); b200pets_step has gt = row / 128)
#define RNG_STREAM_MEMBER 0x20000u
#define RNG_STREAM_CEM 0x30000u
#define RNG_STREAM_ICEM 0x40000u
// latent.cu, the prior's draw of latent element j of row r at step t: philox_normal4(r, t, RNG_STREAM_LATENT | (j >> 2),
// offset, rng_key(seed, offset)), lane j & 3 (r: row of the call, n * P + p; t: step of the call, 0 for one step)
#define RNG_STREAM_LATENT 0x60000u
// latent_train.cu, the draw of latent element j of row b at step t of a training sequence, kind 0 for the posterior and
// 1 for the prior: philox_normal4(b, t, RNG_STREAM_LATENT_TRAIN | (kind << 15) | (j >> 2), offset, rng_key(seed, offset)),
// lane j & 3 (offset: the model's update counter)
#define RNG_STREAM_LATENT_TRAIN 0x80000u
// sac.cu, the reparameterisation draw of action j of row r in sample s (0: the policy on s', 1: on s) of one update:
// philox_normal4(r, s, RNG_STREAM_SAC | (j >> 2), offset, rng_key(seed, offset)), lane j & 3 (offset: the agent's update
// counter)
#define RNG_STREAM_SAC 0x70000u

// ------------------------------------------------------------------------------------------------------
// small math
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float softplus_f(float x) {  // torch F.softplus (beta 1, threshold 20)
  return x > 20.0f ? x : log1pf(expf(x));
}

__device__ __forceinline__ float activation_f(float x, int act, float slope) {
  if (act == B200PETS_ACT_SILU) return x / (1.0f + expf(-x));
  if (act == B200PETS_ACT_RELU) return fmaxf(x, 0.0f);
  return x > 0.0f ? x : x * slope;
}

// processed observation element j of the model input (obs_process_fn), obs points at one row [D]
static __device__ __noinline__ float proc_obs_elem(const float* obs, int j, int mode, int stride = 1) {
  if (mode == B200PETS_PROC_NONE) return obs[j * stride];
  if (mode == B200PETS_PROC_HALFCHEETAH) {  // [o1, sin o2, cos o2, o3:]  (D -> D)
    if (j == 0) return obs[1 * stride];
    if (j == 1) return sinf(obs[2 * stride]);
    if (j == 2) return cosf(obs[2 * stride]);
    return obs[j * stride];
  }
  // cartpole: [sin o1, cos o1, o0, o2:]  (D -> D + 1)
  if (j == 0) return sinf(obs[1 * stride]);
  if (j == 1) return cosf(obs[1 * stride]);
  if (j == 2) return obs[0];
  return obs[(j - 1) * stride];
}

// reward_fn(act, next_obs) -- mbrl/env/reward_fns.py
static __device__ __noinline__ bool term_eval(int fn, const float* o, int D, int os);

static __device__ __noinline__ float reward_eval(int fn, const float* a, int A, int as, const float* o, int D, int os) {
  switch (fn) {
    case B200PETS_REWARD_CARTPOLE:
      return term_eval(B200PETS_TERM_CARTPOLE, o, D, os) ? 0.0f : 1.0f;
    case B200PETS_REWARD_INVERTED_PENDULUM:
      return term_eval(B200PETS_TERM_INVERTED_PENDULUM, o, D, os) ? 0.0f : 1.0f;
    case B200PETS_REWARD_CARTPOLE_PETS: {
      float x0 = o[0], th = o[os];
      float ex = x0 - 0.6f * sinf(th) - 0.0f, ey = -0.6f * cosf(th) - 0.6f;
      float obs_cost = expf(-(ex * ex + ey * ey) / (0.6f * 0.6f));
      float s = 0.f;
      for (int i = 0; i < A; ++i) s += a[i * as] * a[i * as];
      return obs_cost + (-0.01f * s);
    }
    case B200PETS_REWARD_HALFCHEETAH: {
      float s = 0.f;
      for (int i = 0; i < A; ++i) s += a[i * as] * a[i * as];
      float run = o[0] - 0.0f * (o[2 * os] * o[2 * os]);
      return run + (-0.1f * s);
    }
    case B200PETS_REWARD_PUSHER: {
      const float g[3] = {0.45f, -0.05f, -0.323f};
      float d1 = 0.f, d2 = 0.f;
      for (int i = 0; i < 3; ++i) {
        d1 += fabsf(o[(14 + i) * os] - o[(17 + i) * os]);
        d2 += fabsf(g[i] - o[(17 + i) * os]);
      }
      float s = 0.f;
      for (int i = 0; i < A; ++i) s += a[i * as] * a[i * as];
      return -((0.5f * d1 + 1.25f * d2) + 0.1f * s);
    }
    default:
      return 0.0f;
  }
}

// termination_fn(act, next_obs) -- mbrl/env/termination_fns.py
static __device__ __noinline__ bool term_eval(int fn, const float* o, int D, int os) {
  switch (fn) {
    case B200PETS_TERM_CARTPOLE: {
      float x = o[0], th = o[2 * os];
      const float lim = (float)(12.0 * 2.0 * 3.141592653589793 / 360.0);
      bool ok = (x > -2.4f) && (x < 2.4f) && (th > -lim) && (th < lim);
      return !ok;
    }
    case B200PETS_TERM_INVERTED_PENDULUM: {
      bool fin = true;
      for (int i = 0; i < D; ++i) fin = fin && isfinite(o[i * os]);
      return !(fin && fabsf(o[os]) <= 0.2f);
    }
    case B200PETS_TERM_HOPPER: {
      bool ok = true;
      for (int i = 0; i < D; ++i) ok = ok && isfinite(o[i * os]);
      for (int i = 1; i < D; ++i) ok = ok && (fabsf(o[i * os]) < 100.0f);
      ok = ok && (o[0] > 0.7f) && (fabsf(o[os]) < 0.2f);
      return !ok;
    }
    case B200PETS_TERM_WALKER2D: {
      float h = o[0], an = o[os];
      return !((h > 0.8f) && (h < 2.0f) && (an > -1.0f) && (an < 1.0f));
    }
    case B200PETS_TERM_ANT: {
      bool fin = true;
      for (int i = 0; i < D; ++i) fin = fin && isfinite(o[i * os]);
      return !(fin && (o[0] >= 0.2f) && (o[0] <= 1.0f));
    }
    case B200PETS_TERM_HUMANOID:
      return (o[0] < 1.0f) || (o[0] > 2.0f);
    default:
      return false;
  }
}

// ------------------------------------------------------------------------------------------------------
// Row bookkeeping shared by both rollout kernels.
//
// slot_mode 0 (explicit permutation, the reference's rule gaussian_mlp.py:202-212): member m owns slots
// [m*B/M, (m+1)*B/M), row id = perm[slot].
//
// slot_mode >= 1 ("tile shuffle"): a shuffle GROUP is (particle p, 128-aligned chunk c of GLOBAL sequence
// indices): its rows are the particle-p copies of sequences 128c .. 128c+127.  Groups are numbered globally
// gt = p * C_glob + c (C_glob = ceil(global population / 128)), so that the member a row uses and its noise
// stream depend on (global sequence, particle, step, seed, offset) only -- not on how the population is sharded
// over GPUs.  A shard [seq0, seq0 + N) holds the chunks c_lo .. c_hi that intersect it; rows of a boundary chunk
// that belong to another shard are simply invalid here.  Local tile index = p * C_loc + (c - c_lo).
// Members: every (group, step) draws one member uniformly and independently from Philox keyed by (gt, t, seed,
// offset).  A row's member at a step is therefore uniform over the M elite members, and the 20 particles of one
// sequence (which sit in 20 different groups) draw independently of each other -- the law of the reference's rule for a
// row (randperm split, gaussian_mlp.py:202-206) up to its without-replacement coupling across the B rows, which is
// O(M / B) per pair of rows.  What is NOT reproduced: the exact balance (each member exactly B/M rows per step), and
// the 128 same-particle neighbours of a group share the draw (common random numbers across candidates).
// ------------------------------------------------------------------------------------------------------
#define B200PETS_GROUP_ROWS 128

struct ShuffleGeom {
  int c_lo, C_loc, C_glob;
};

__host__ __device__ __forceinline__ ShuffleGeom shuffle_geom(int seq0, int N, int n_glob) {
  ShuffleGeom g;
  g.c_lo = seq0 / B200PETS_GROUP_ROWS;
  g.C_loc = (seq0 + N - 1) / B200PETS_GROUP_ROWS - g.c_lo + 1;
  g.C_glob = (n_glob + B200PETS_GROUP_ROWS - 1) / B200PETS_GROUP_ROWS;
  return g;
}

// local group index -> global group number
__device__ __forceinline__ long long shuffle_global_group(const ShuffleGeom& g, long long group) {
  const long long p = group / g.C_loc;
  const int c = g.c_lo + (int)(group % g.C_loc);
  return p * g.C_glob + c;
}

// row `i` (0..127) of local group `group`: local row id (n_local * P + p), validity, global row id (RNG key)
__device__ __forceinline__ long long shuffle_row(const RolloutArgs& a, const ShuffleGeom& g, long long group, int i,
                                                 bool* valid, long long* rid_glob) {
  const long long p = group / g.C_loc;
  const int c = g.c_lo + (int)(group % g.C_loc);
  const long long ng = (long long)c * B200PETS_GROUP_ROWS + i;
  *valid = ng >= a.seq0 && ng < (long long)a.seq0 + a.N;
  *rid_glob = ng * a.P + p;
  return (ng - a.seq0) * a.P + p;
}

__device__ __forceinline__ long long slot_to_rid(const RolloutArgs& a, long long slot) {  // slot_mode 0 only
  return a.perm ? a.perm[slot] : slot;
}

// Per-row members (RolloutArgs::member_off = off): member m owns ceil(count_m / rows) tiles of `rows` rows, in member
// order, over its slots [off[m], off[m+1]).  Tile `tile` -> its member and first slot; returns its row count, 0 for a
// surplus tile of the bound ceil(B / rows) + M - 1 the grids are sized for.  Every role of a kernel that walks tiles
// derives its tile list from this one function.
__device__ __forceinline__ int member_tile(const int* off, int M, long long tile, int rows, int* member, long long* slot0) {
  long long rest = tile;
  for (int mm = 0; mm < M; ++mm) {
    const int cnt = off[mm + 1] - off[mm];
    const long long nt = (cnt + rows - 1) / rows;
    if (rest < nt) {
      *member = mm;
      *slot0 = off[mm] + rest * rows;
      return (int)min((long long)rows, cnt - rest * rows);
    }
    rest -= nt;
  }
  *member = 0;
  *slot0 = 0;
  return 0;
}

// member of global group `gt` at step t: an independent uniform draw per (group, step) from Philox
__device__ __forceinline__ int shuffle_member(unsigned long long seed, unsigned long long offset, int slot_mode,
                                              long long gt, int t, int M) {
  if (slot_mode == 2) t = 0;
  U4 r = philox4x32_10((uint32_t)gt, (uint32_t)t, RNG_STREAM_MEMBER, (uint32_t)offset, (uint32_t)seed,
                       (uint32_t)(seed >> 32) ^ (uint32_t)(gt >> 32));
  return (int)(((unsigned long long)r.x * (unsigned long long)M) >> 32);
}

// Kernels put the low 32 bits of the stream offset into a Philox counter word; the high 32 bits go into the key so
// that long runs (> 2^32 offsets) never replay a stream.  Applied once at every C entry point.
static __host__ __device__ inline unsigned long long rng_key(unsigned long long seed, unsigned long long offset) {
  return seed ^ (offset & 0xFFFFFFFF00000000ull);
}

// Problem k of a batched launch (BatchArgs, or latent.cuh's LatentBatch): the element offset of its slice of a per-problem
// array, its Philox offset and key.  With BATCH = false (single launches) these are 0, a.offset and a.seed, and `bt` is
// never read.
template <bool BATCH, class Batch>
__device__ __forceinline__ long long prob_off(const Batch* bt, long long k, long long Batch::*stride) {
  if constexpr (BATCH) return k * (bt->*stride);
  else return 0;
}
template <bool BATCH, class Args, class Batch>
__device__ __forceinline__ unsigned long long prob_offset(const Args& a, const Batch* bt, long long k) {
  if constexpr (BATCH) return a.offset + (unsigned long long)k * bt->offset_step;
  else return a.offset;
}
template <bool BATCH, class Args, class Batch>
__device__ __forceinline__ unsigned long long prob_seed(const Args& a, const Batch* bt, long long k) {
  if constexpr (BATCH) return rng_key(bt->seed, prob_offset<BATCH>(a, bt, k));
  else return a.seed;
}
template <bool BATCH>
__device__ __forceinline__ long long prob_rid(const RolloutArgs& a, const BatchArgs* bt, long long k, long long slot) {
  if constexpr (BATCH) return a.perm ? a.perm[k * bt->perm + slot] : slot;
  else return slot_to_rid(a, slot);
}

// ------------------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL).  The kernels of a plan form a chain  sample -> rollout -> refit -> sample ..
// on one stream.  Launched with the programmatic-stream-serialization attribute, a kernel may become resident as soon
// as its predecessor has executed pdl_trigger() in all its CTAs; it then runs its prologue (barrier set-up,
// constant tables, the first weight prefetches -- memory no kernel of the chain writes) and blocks in pdl_wait() until
// the predecessor grid has completed and flushed, BEFORE its first access to anything the chain produces.  Every
// kernel of the chain waits before it finishes, so completion is transitive along the chain.  Launch gaps and the
// rollout kernel's ~6 us prologue thereby overlap the tail of the previous kernel.
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

#ifdef __CUDACC__
#include <utility>
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                     Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}
#endif

// host-side error plumbing (api.cu)
int b200pets_set_error(int code, const char* fmt, ...);
#define CUDA_TRY(expr)                                                                            \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess)                                                                        \
      return b200pets_set_error(B200PETS_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                                __FILE__, __LINE__);                                              \
  } while (0)
