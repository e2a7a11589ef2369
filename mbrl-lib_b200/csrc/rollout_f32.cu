// fp32 SIMT rollout of the ensemble MLP: the parity anchor (same arithmetic as the reference's fp32 ATen
// path up to summation order).  One CTA owns a tile of TR rows of one member for steps [t0, t1).
//
// Reference path restated here (paths relative to mbrl-lib):
//   mbrl/models/model_env.py:145-191      evaluate_action_sequences loop, dead mask, accumulation
//   mbrl/models/one_dim_tr_model.py:103-116, 245-289   input build / normalise, delta add-back, reward split
//   mbrl/models/model.py:426-473          Gaussian sample  mean + sqrt(exp(logvar)) * eps
//   mbrl/models/gaussian_mlp.py:140-216   member MLP, logvar clamp, TS1/TSinf/expectation
//   mbrl/models/util.py:53-65             x @ W[e] + b[e]
#include "common.cuh"

namespace {

constexpr int kThreads = 256;

template <int TR>
__device__ __forceinline__ void dense_layer(const float* __restrict__ W, const float* __restrict__ bias,
                                            const float* __restrict__ in_s, float* __restrict__ out_s, int K,
                                            int N, int LD, int act, float slope, bool apply_act) {
  constexpr int RPT = TR / 4;
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const int r0 = ty * RPT;
  const int K4 = K & ~3;
  for (int c0 = 0; c0 < N; c0 += 256) {
    float acc[RPT][4];
#pragma unroll
    for (int r = 0; r < RPT; ++r)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[r][j] = 0.f;
    int col[4];
    bool ok[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      col[j] = c0 + tx + 64 * j;
      ok[j] = col[j] < N;
    }
    for (int k = 0; k < K4; k += 4) {
      float w[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int j = 0; j < 4; ++j) w[kk][j] = ok[j] ? __ldg(W + (size_t)(k + kk) * N + col[j]) : 0.f;
#pragma unroll
      for (int r = 0; r < RPT; ++r) {
        const float4 a = *reinterpret_cast<const float4*>(in_s + (r0 + r) * LD + k);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          acc[r][j] = fmaf(a.x, w[0][j], acc[r][j]);
          acc[r][j] = fmaf(a.y, w[1][j], acc[r][j]);
          acc[r][j] = fmaf(a.z, w[2][j], acc[r][j]);
          acc[r][j] = fmaf(a.w, w[3][j], acc[r][j]);
        }
      }
    }
    for (int k = K4; k < K; ++k) {
      float w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) w[j] = ok[j] ? __ldg(W + (size_t)k * N + col[j]) : 0.f;
#pragma unroll
      for (int r = 0; r < RPT; ++r) {
        const float a = in_s[(r0 + r) * LD + k];
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[r][j] = fmaf(a, w[j], acc[r][j]);
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (!ok[j]) continue;
      const float bv = __ldg(bias + col[j]);
#pragma unroll
      for (int r = 0; r < RPT; ++r) {
        float v = acc[r][j] + bv;
        if (apply_act) v = activation_f(v, act, slope);
        out_s[(r0 + r) * LD + col[j]] = v;
      }
    }
  }
  // zero the K-padding of the next layer's input (rows are read in float4 chunks)
  const int Nr = (N + 3) & ~3;
  for (int idx = threadIdx.x; idx < TR * (Nr - N); idx += kThreads) {
    int r = idx / (Nr - N), c = N + idx % (Nr - N);
    out_s[r * LD + c] = 0.f;
  }
}

// The kernels' body.  BATCH: K independent problems in one launch (common.cuh BatchArgs): CTA j runs local tile
// j % bt->tiles of problem j / bt->tiles, and everything after that decode is the single-problem code.
template <int TR, bool BATCH>
__device__ __forceinline__ void rollout_f32_body(const ModelDev& m, const RolloutArgs& a, int LD, const BatchArgs* bt) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* bufA = reinterpret_cast<float*>(smem_raw);
  float* bufB = bufA + TR * LD;
  float* obs_s = bufB + TR * LD;            // [TR][D]
  float* act_s = obs_s + TR * m.D;          // [TR][A]
  float* exp_s = act_s + TR * m.A;          // [TR][nout] (expectation only, else unused but allocated)
  float* tot_s = exp_s + TR * m.nout;       // [TR]
  float* rew_s = tot_s + TR;                // [TR]
  long long* rid_s = reinterpret_cast<long long*>(rew_s + TR);  // [TR] local row id (-1: no row)
  long long* gid_s = rid_s + TR;                                // [TR] global row id (Philox key)
  int* dead_s = reinterpret_cast<int*>(gid_s + TR);             // [TR]

  const int tid = threadIdx.x;
  int tile = blockIdx.x;
  long long kp = 0;  // problem of a batched launch
  if constexpr (BATCH) { kp = tile / bt->tiles; tile -= (int)(kp * bt->tiles); }
  const bool expectation = a.propagation == B200PETS_PROP_EXPECTATION;
  // nv: rows of this tile that may hold a row (row i is live iff rid_s[i] >= 0)
  int nv, member = 0;
  const bool shuffle = a.slot_mode >= 1 && !expectation;
  const ShuffleGeom geom = shuffle_geom(a.seq0, a.N, a.n_glob);
  constexpr int kSub = B200PETS_GROUP_ROWS / TR;  // tiles per shuffle group
  const long long group = tile / kSub;
  if (shuffle) {  // tile = TR consecutive rows of a shuffle group (common.cuh)
    nv = TR;
    for (int i = tid; i < TR; i += kThreads) {
      bool valid;
      long long gid;
      const long long rid = shuffle_row(a, geom, group, (tile % kSub) * TR + i, &valid, &gid);
      rid_s[i] = valid ? rid : -1;
      gid_s[i] = gid;
    }
  } else {
    long long slot0;
    if (expectation) {
      slot0 = (long long)tile * TR;
      nv = (int)min((long long)TR, a.B - slot0);
    } else if (a.member_off) {
      // per-row members: member m owns ceil(count_m / TR) tiles, in member order; the grid has the bound
      // ceil(B / TR) + M - 1 tiles, and tiles past the members' own have no rows
      nv = member_tile(a.member_off + prob_off<BATCH>(bt, kp, &BatchArgs::member_off), m.M, tile, TR, &member, &slot0);
      if (nv == 0) return;  // uniform over the CTA, before any barrier
    } else {
      const long long Bm = a.B / m.M;
      const int tpm = (int)((Bm + TR - 1) / TR);
      member = tile / tpm;
      const int c = tile % tpm;
      slot0 = (long long)member * Bm + (long long)c * TR;
      nv = (int)min((long long)TR, Bm - (long long)c * TR);
    }
    for (int i = tid; i < TR; i += kThreads) {
      rid_s[i] = i < nv ? prob_rid<BATCH>(a, bt, kp, slot0 + i) : -1;
      gid_s[i] = rid_s[i] + (long long)a.seq0 * a.P;
    }
  }
  __syncthreads();

  // ---- load state -------------------------------------------------------------------------------
  for (int idx = tid; idx < TR * m.D; idx += kThreads) {
    int i = idx / m.D, d = idx % m.D;
    float v = 0.f;
    if (rid_s[i] >= 0)
      v = a.init_from_obs0 ? a.obs0[prob_off<BATCH>(bt, kp, &BatchArgs::obs0) + d]
                           : a.obs_in[prob_off<BATCH>(bt, kp, &BatchArgs::obs_state) + rid_s[i] * m.D + d];
    obs_s[idx] = v;
  }
  for (int i = tid; i < TR; i += kThreads) {
    bool ld = a.load_state && rid_s[i] >= 0;
    tot_s[i] = ld ? a.total_state[prob_off<BATCH>(bt, kp, &BatchArgs::rows) + rid_s[i]] : 0.f;
    dead_s[i] = ld ? (int)a.dead_state[prob_off<BATCH>(bt, kp, &BatchArgs::rows) + rid_s[i]] : 0;
  }
  __syncthreads();

  const int nlayers = m.L + 1;
  for (int t = a.t0; t < a.t1; ++t) {
    if (shuffle)
      member = shuffle_member(prob_seed<BATCH>(a, bt, kp), prob_offset<BATCH>(a, bt, kp), a.slot_mode, shuffle_global_group(geom, group),
                              t, m.M);
    // ---- actions ------------------------------------------------------------------------------
    for (int idx = tid; idx < TR * m.A; idx += kThreads) {
      int i = idx / m.A, j = idx % m.A;
      float v = 0.f;
      if (rid_s[i] >= 0)
        v = a.act[prob_off<BATCH>(bt, kp, &BatchArgs::act) + (rid_s[i] / a.act_div) * a.act_row_stride + (long long)t * a.act_t_stride + j];
      act_s[idx] = v;
    }
    __syncthreads();
    const int passes = expectation ? m.M : 1;
    for (int pass = 0; pass < passes; ++pass) {
      const int mem = expectation ? pass : member;
      // ---- model input: normalise(cat(proc(obs), act)) -> bufA -----------------------------
      const int inr = (m.in + 3) & ~3;
      for (int idx = tid; idx < TR * inr; idx += kThreads) {
        int i = idx / inr, j = idx % inr;
        float v = 0.f;
        if (rid_s[i] >= 0 && j < m.in) {
          float x = j < m.Dp ? proc_obs_elem(obs_s + i * m.D, j, m.obs_process) : act_s[i * m.A + (j - m.Dp)];
          if (m.norm_mode == 2)
            x = (float)(((double)x - m.norm_mean_d[j]) / m.norm_std_d[j]);
          else if (m.norm_mode == 1)
            x = (x - m.norm_mean_f[j]) / m.norm_std_f[j];
          v = x;
        }
        bufA[i * LD + j] = v;
      }
      __syncthreads();
      float* cur = bufA;
      float* nxt = bufB;
      for (int l = 0; l < nlayers; ++l) {
        const float* W = m.W[l] + (size_t)mem * m.K[l] * m.N[l];
        const float* bias = m.b[l] + (size_t)mem * m.N[l];
        dense_layer<TR>(W, bias, cur, nxt, m.K[l], m.N[l], LD, m.act, m.leaky, l < nlayers - 1);
        __syncthreads();
        float* tmp = cur; cur = nxt; nxt = tmp;
      }
      if (expectation) {  // gaussian_mlp.py:213-215: average mean and (clamped) logvar over members
        for (int idx = tid; idx < TR * m.nout; idx += kThreads) {
          int i = idx / m.nout, c = idx % m.nout;
          float v = cur[i * LD + c];
          if (!m.deterministic && c >= m.out) {
            int o = c - m.out;
            v = m.max_lv[o] - softplus_f(m.max_lv[o] - v);
            v = m.min_lv[o] + softplus_f(v - m.min_lv[o]);
          }
          exp_s[idx] = pass == 0 ? v : exp_s[idx] + v;
        }
        __syncthreads();
      } else {
        // ---- prediction -> next observation (in place) ---------------------------------------
        for (int idx = tid; idx < nv * m.out; idx += kThreads) {
          int i = idx / m.out, o = idx % m.out;
          if (rid_s[i] < 0) continue;
          float mean = cur[i * LD + o];
          float pred = mean;
          if (!m.deterministic && a.sample) {
            float lv = cur[i * LD + m.out + o];
            lv = m.max_lv[o] - softplus_f(m.max_lv[o] - lv);
            lv = m.min_lv[o] + softplus_f(lv - m.min_lv[o]);
            float sd = sqrtf(expf(lv));
            float e;
            if (a.eps) {
              e = a.eps[prob_off<BATCH>(bt, kp, &BatchArgs::eps) + ((size_t)(t - a.t0) * a.B + rid_s[i]) * m.out + o];
            } else {
              float z[4];
              philox_normal4((uint32_t)gid_s[i], (uint32_t)t, RNG_STREAM_EPS | (uint32_t)(o >> 2), (uint32_t)prob_offset<BATCH>(a, bt, kp),
                             prob_seed<BATCH>(a, bt, kp), z);
              e = z[o & 3];
            }
            pred = mean + sd * e;
          }
          if (m.learned_rewards && o == m.out - 1) {
            rew_s[i] = pred;
          } else {
            float ob = obs_s[i * m.D + o];
            obs_s[i * m.D + o] = (m.target_is_delta && !m.no_delta[o]) ? pred + ob : pred;
          }
        }
        __syncthreads();
      }
    }
    if (expectation) {
      const float invM = 1.0f / (float)m.M;
      for (int idx = tid; idx < nv * m.out; idx += kThreads) {
        int i = idx / m.out, o = idx % m.out;
        if (rid_s[i] < 0) continue;
        float mean = exp_s[i * m.nout + o] / (float)m.M;
        float pred = mean;
        if (!m.deterministic && a.sample) {
          float lv = exp_s[i * m.nout + m.out + o] / (float)m.M;
          float sd = sqrtf(expf(lv));
          float e;
          if (a.eps) {
            e = a.eps[prob_off<BATCH>(bt, kp, &BatchArgs::eps) + ((size_t)(t - a.t0) * a.B + rid_s[i]) * m.out + o];
          } else {
            float z[4];
            philox_normal4((uint32_t)gid_s[i], (uint32_t)t, RNG_STREAM_EPS | (uint32_t)(o >> 2), (uint32_t)prob_offset<BATCH>(a, bt, kp),
                           prob_seed<BATCH>(a, bt, kp), z);
            e = z[o & 3];
          }
          pred = mean + sd * e;
        }
        if (m.learned_rewards && o == m.out - 1) {
          rew_s[i] = pred;
        } else {
          float ob = obs_s[i * m.D + o];
          obs_s[i * m.D + o] = (m.target_is_delta && !m.no_delta[o]) ? pred + ob : pred;
        }
      }
      (void)invM;
      __syncthreads();
    }
    // ---- reward, termination, accumulate (model_env.py:124-129, 186-188) ---------------------
    for (int i = tid; i < nv; i += kThreads) {
      if (rid_s[i] < 0) continue;
      // model_env.py:124-128: pred_rewards only when reward_fn is None, an explicit reward_fn always wins
      float rew = m.reward_fn == B200PETS_REWARD_LEARNED
                      ? rew_s[i]
                      : reward_eval(m.reward_fn, act_s + i * m.A, m.A, 1, obs_s + i * m.D, m.D, 1);
      bool done = term_eval(m.term_fn, obs_s + i * m.D, m.D, 1);
      if (a.reward_out) a.reward_out[rid_s[i]] = rew;
      if (a.done_out) a.done_out[rid_s[i]] = done ? 1 : 0;
      const size_t tr = (size_t)(t - a.t0) * a.B + rid_s[i];
      if (a.traj_reward) a.traj_reward[tr] = rew;
      if (a.traj_done) a.traj_done[tr] = done ? 1 : 0;
      if (dead_s[i]) rew = 0.f;
      dead_s[i] |= done ? 1 : 0;
      tot_s[i] += rew;
    }
    if (a.traj_obs)
      for (int idx = tid; idx < nv * m.D; idx += kThreads) {
        const int i = idx / m.D, d = idx % m.D;
        if (rid_s[i] >= 0) a.traj_obs[((size_t)(t - a.t0) * a.B + rid_s[i]) * m.D + d] = obs_s[idx];
      }
    __syncthreads();
  }
  // ---- store state ------------------------------------------------------------------------------
  if (a.store_state) {
    if (a.obs_out)
      for (int idx = tid; idx < nv * m.D; idx += kThreads) {
        int i = idx / m.D, d = idx % m.D;
        if (rid_s[i] >= 0) a.obs_out[prob_off<BATCH>(bt, kp, &BatchArgs::obs_state) + rid_s[i] * m.D + d] = obs_s[idx];
      }
    for (int i = tid; i < nv; i += kThreads) {
      if (rid_s[i] < 0) continue;
      if (a.total_state) a.total_state[prob_off<BATCH>(bt, kp, &BatchArgs::rows) + rid_s[i]] = tot_s[i];
      if (a.dead_state) a.dead_state[prob_off<BATCH>(bt, kp, &BatchArgs::rows) + rid_s[i]] = (uint8_t)dead_s[i];
    }
  }
}

template <int TR>
__global__ void __launch_bounds__(kThreads) rollout_f32_kernel(const ModelDev m, const RolloutArgs a, int LD) {
  rollout_f32_body<TR, false>(m, a, LD, nullptr);
}

// K independent evaluations in one launch
template <int TR>
__global__ void __launch_bounds__(kThreads) rollout_f32_batch_kernel(const __grid_constant__ ModelDev m,
                                                                     const __grid_constant__ RolloutArgs a, int LD,
                                                                     const __grid_constant__ BatchArgs bt) {
  rollout_f32_body<TR, true>(m, a, LD, &bt);
}

}  // namespace

// number of tiles for a launch (host side)
static long long f32_num_tiles(const ModelDev& m, const RolloutArgs& a, int TR) {
  if (a.propagation == B200PETS_PROP_EXPECTATION) return (a.B + TR - 1) / TR;
  if (a.slot_mode >= 1) return (long long)a.P * shuffle_geom(a.seq0, a.N, a.n_glob).C_loc * (B200PETS_GROUP_ROWS / TR);
  if (a.member_off) return (a.B + TR - 1) / TR + m.M - 1;
  long long Bm = a.B / m.M;
  return (long long)m.M * ((Bm + TR - 1) / TR);
}

// Tile of rollout_f32_kernel for a model on the current device: the most rows per CTA (64, 32 or 16) whose buffers fit
// in the opt-in shared memory.  p->rows = 0 when not even 16 rows fit.  Also what b200pets_model_plan_info reports.
int f32_tile_plan(const ModelDev& m, F32Plan* p) {
  int wmax = m.in;
  for (int l = 0; l <= m.L; ++l) wmax = max(wmax, m.N[l]);
  p->wmax = wmax;
  p->LD = ((wmax + 3) & ~3) + 4;
  int dev = 0, max_smem = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  CUDA_TRY(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  p->rows = 0;
  p->smem = 0;
  for (int TR = 64; TR >= 16; TR /= 2) {
    const size_t sm = (size_t)TR * (2 * p->LD + m.D + m.A + m.nout + 2) * sizeof(float) +
                      (size_t)TR * (2 * sizeof(long long) + sizeof(int));
    if (sm <= (size_t)max_smem) {
      p->rows = TR;
      p->smem = sm;
      break;
    }
  }
  return B200PETS_OK;
}

template <int TR>
static int launch_f32_rows(const ModelDev& m, const RolloutArgs& a, const F32Plan& p, int num_problems, BatchArgs bt,
                           cudaStream_t stream) {
  bt.tiles = f32_num_tiles(m, a, TR);
  if (num_problems == 1) {
    CUDA_TRY(cudaFuncSetAttribute(rollout_f32_kernel<TR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
    rollout_f32_kernel<TR><<<(unsigned)bt.tiles, kThreads, p.smem, stream>>>(m, a, p.LD);
  } else {
    CUDA_TRY(cudaFuncSetAttribute(rollout_f32_batch_kernel<TR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
    rollout_f32_batch_kernel<TR><<<(unsigned)(bt.tiles * num_problems), kThreads, p.smem, stream>>>(m, a, p.LD, bt);
  }
  CUDA_TRY(cudaGetLastError());
  return B200PETS_OK;
}

// `num_problems` evaluations of the launch `a` describes in one grid.  One problem runs rollout_f32_kernel and ignores
// bt; more run rollout_f32_batch_kernel with bt's per-problem strides (bt.tiles is set here).
int launch_rollout_f32(const ModelDev& m, const RolloutArgs& a, int num_problems, BatchArgs bt, cudaStream_t stream) {
  if (num_problems > 1 && (a.traj_obs || a.traj_reward || a.traj_done || a.reward_out || a.done_out))
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "batched rollout: evaluation outputs only");
  F32Plan p;
  int rc = f32_tile_plan(m, &p);
  if (rc) return rc;
  if (p.rows == 64) return launch_f32_rows<64>(m, a, p, num_problems, bt, stream);
  if (p.rows == 32) return launch_f32_rows<32>(m, a, p, num_problems, bt, stream);
  if (p.rows == 16) return launch_f32_rows<16>(m, a, p, num_problems, bt, stream);
  return b200pets_set_error(B200PETS_EUNSUPPORTED, "layer width %d needs more shared memory than a CTA has", p.wmax);
}
