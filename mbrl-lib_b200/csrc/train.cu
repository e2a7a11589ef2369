// Training of OneDTransitionRewardModel(GaussianMLP) on the device: ModelTrainer.train's inner loop
// (mbrl/models/model_trainer.py:146-177) with the model's update and eval_score (mbrl/models/model.py:129-167,
// gaussian_mlp.py:283-361, one_dim_tr_model.py:118-136).  fp32 throughout, FFMA only: the reference trains in fp32 and
// torch keeps TF32 matmuls off, so bf16 or TF32 operands would change what the model learns.
//
// Three kernels:
//   train_preprocess_kernel  raw transitions -> model inputs and targets for the whole dataset, once per train() (the
//                            normaliser does not change during train()): obs_process_fn, the fp32 / fp64 normaliser, delta
//                            targets with no_delta_list, the learned-reward column (one_dim_tr_model.py:103-136).
//   train_adam_kernel        every minibatch step of one epoch: forward, loss, backward and torch.optim.Adam on all E
//                            members, one launch for the whole epoch.
//   train_eval_kernel        eval_score (per-member MSE, OneDTransitionRewardModel.eval_score) over a whole dataset in
//                            one launch, replacing ModelTrainer.evaluate's per-batch loop (model_trainer.py:216-262).
//
// Structure of train_adam_kernel.  One step is a chain of small dependent matrix products (E x Bm rows, ~200 columns):
// far too little work for one product to fill an H100, and each depends on the previous one.  The kernel is a persistent
// cooperative grid (one 256-thread CTA per SM) that walks the chain phase by phase with a grid-wide barrier between
// phases.  Each phase is a list of independent 32 x 32 output tiles dealt round-robin to the CTAs; operands stream from
// L2 (the ~170 k parameters per member and both Adam moments, ~19 MB at E = 7, stay resident there).  Per step, with
// layers l = 0 .. L (L hidden, then mean_and_logvar), Z_l = A_{l-1} W_l + b_l, A_l = act(Z_l), A_{-1} = the gathered
// inputs, G_l = dloss/dZ_l:
//   forward l = 0 .. L                 Z_l (and A_l)                                   L + 1 phases
//   loss                               G_L per output element, loss terms, bound terms 1 phase
//   backward l = L .. 1                G_{l-1} = (G_l W_l^T) * act'(Z_{l-1}), and in the same phase the weight
//                                      gradient A_l^T G_{l+1} of layer l + 1 with its Adam update (layer l + 1 is
//                                      no longer read by anyone); at l = L instead the loss value and the
//                                      logvar-bound gradients and updates                 L phases
//   last                               gradients and Adam updates of layers 1 and 0     1 phase
// i.e. 2L + 3 barriers per step and one launch per epoch.  Every weight-gradient element is computed by exactly one
// thread, which applies Adam to it at once: gradients never go to memory.  Sums run in a fixed order, so a run is
// bit-reproducible.  The alternative, one launch per phase, pays a launch gap per phase; cuBLAS-shaped GEMMs per phase
// have the same gaps and use none of the fusion.
//
// Adam (torch.optim.Adam, weight_decay = L2 added to the gradient, no amsgrad, torch's foreach implementation and its
// order of operations; t = the step count after this step, scalars computed in double on the host side of torch and
// rounded to float where torch hands them to a float kernel):
//   g  = g + wd * p
//   m  = m + (1 - beta1) * (g - m)                      (lerp, weight 1 - beta1 < 0.5)
//   v  = v * beta2;  v = v + (1 - beta2) * g * g
//   p  = p + (-(lr / (1 - beta1^t))) * (m / (sqrt(v) / sqrt(1 - beta2^t) + eps))
#include <cooperative_groups.h>

#include "train.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int TT = 32;         // output tile edge and reduction chunk
constexpr int kThreads = 256;  // 8 warps: thread (ty, tx) owns rows ty, ty + 8, ty + 16, ty + 24 of column tx

// One matrix operand: element(x, y) = p[map(x) * s0 + map(y) * s1], x the outer (row or column) coordinate, y the
// reduction coordinate.  `idx` maps one of them (gathered minibatch rows); `ones_at` = x yields 1.0 (the bias row
// appended to a weight gradient's left operand).
struct Opnd {
  const float* p;
  const int* idx;
  long long s0, s1;
  int idx_on;   // 0: idx maps x, 1: idx maps y
  int ones_at;  // -1: none
};

__device__ __forceinline__ float opnd_load(const Opnd& o, int x, int y, int X, int Y) {
  if (y >= Y) return 0.0f;
  if (x == o.ones_at) return 1.0f;
  if (x >= X) return 0.0f;
  long long rx = x, ry = y;
  if (o.idx) {
    if (o.idx_on == 0) rx = o.idx[x];
    else ry = o.idx[y];
  }
  return o.p[rx * o.s0 + ry * o.s1];
}

// acc[q] = sum_k L(i0 + ty + 8q, k) * R(j0 + tx, k), k = 0 .. K-1 in ascending chunks of 32.
__device__ __forceinline__ void tile_mm(const Opnd& Lo, const Opnd& Ro, int M, int N, int K, int i0, int j0, float acc[4],
                                        float (*Ls)[TT + 1], float (*Rs)[TT + 1]) {
  const int tx = threadIdx.x % TT, ty = threadIdx.x / TT;
#pragma unroll
  for (int q = 0; q < 4; ++q) acc[q] = 0.0f;
  for (int k0 = 0; k0 < K; k0 += TT) {
    for (int e = threadIdx.x; e < TT * TT; e += kThreads) {
      // consecutive threads walk the operand's contiguous coordinate (coalesced loads)
      int a = e / TT, b = e % TT;
      if (Lo.s1 != 1) { a = e % TT; b = e / TT; }
      Ls[a][b] = opnd_load(Lo, i0 + a, k0 + b, M, K);
      a = e % TT; b = e / TT;
      if (Ro.s0 != 1) { a = e / TT; b = e % TT; }
      Rs[b][a] = opnd_load(Ro, j0 + a, k0 + b, N, K);
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < TT; ++kk) {
      const float r = Rs[kk][tx];
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[q] = fmaf(Ls[ty + 8 * q][kk], r, acc[q]);
    }
    __syncthreads();
  }
}

template <typename T>
__device__ __forceinline__ T block_sum(T v, T* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  const T r = red[0];
  __syncthreads();
  return r;
}

// torch's softplus backward: x > 20 ? 1 : e^x / (e^x + 1)
__device__ __forceinline__ float softplus_grad(float x) {
  if (x > 20.0f) return 1.0f;
  const float z = expf(x);
  return z / (z + 1.0f);
}

// d act(z) / dz, as torch's threshold / silu / leaky_relu backward
__device__ __forceinline__ float activation_grad(float g, float z, int act, float slope) {
  if (act == B200PETS_ACT_RELU) return z > 0.0f ? g : 0.0f;
  if (act == B200PETS_ACT_SILU) {
    const float s = 1.0f / (1.0f + expf(-z));
    return g * s * (1.0f + z * (1.0f - s));
  }
  return z > 0.0f ? g : g * slope;
}

struct AdamStep {
  float wd, omb1, b2, omb2, eps, bc2_sqrt, step_size;
};

__device__ __forceinline__ AdamStep adam_scalars(const TrainDev& m, long long t) {
  AdamStep s;
  s.wd = (float)m.weight_decay;
  s.omb1 = (float)(1.0 - m.beta1);
  s.b2 = (float)m.beta2;
  s.omb2 = (float)(1.0 - m.beta2);
  s.eps = (float)m.eps;
  const double bc1 = 1.0 - pow(m.beta1, (double)t), bc2 = 1.0 - pow(m.beta2, (double)t);
  s.step_size = (float)(-(m.lr / bc1));
  s.bc2_sqrt = (float)sqrt(bc2);
  return s;
}

__device__ __forceinline__ void adam_update(float* p, float* mo, float* vo, float g, const AdamStep& s) {
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

// Workspace of train_adam_kernel, offsets in floats.  Hidden layer l owns three consecutive [E][Bm][hid] blocks (Z, A,
// G), so their offsets are arithmetic in l (no per-layer offset table that a runtime index would put in local memory).
struct TrainWs {
  size_t scal;                                // [4]: bound term of the loss
  size_t hidden, hstride;                     // first hidden block, stride between blocks
  size_t out;                                 // [E][Bm][nout]: Z_L, then G_L in place
  size_t lossel, gmin, gmax;                  // [E][Bm][out]
  size_t total;
  __host__ __device__ size_t Z(int l) const { return hidden + (3 * (size_t)l) * hstride; }
  __host__ __device__ size_t A(int l) const { return hidden + (3 * (size_t)l + 1) * hstride; }
  __host__ __device__ size_t G(int l) const { return hidden + (3 * (size_t)l + 2) * hstride; }
};

__host__ __device__ inline TrainWs train_ws_layout(const TrainDev& m, int Bm) {
  TrainWs w;
  size_t off = 0;
  auto take = [&](size_t n) { size_t o = off; off += (n + 63) / 64 * 64; return o; };
  w.scal = take(4);
  const size_t h = (size_t)m.E * Bm * m.hid;
  w.hstride = (h + 63) / 64 * 64;
  w.hidden = off;
  off += 3 * (size_t)m.L * w.hstride;
  w.out = take((size_t)m.E * Bm * m.nout);
  const size_t o = (size_t)m.E * Bm * m.out;
  w.lossel = take(o);
  w.gmin = m.deterministic ? 0 : take(o);
  w.gmax = m.deterministic ? 0 : take(o);
  w.total = off;
  return w;
}

struct EpochArgs {
  const float* X;  // [rows][in]
  const float* Y;  // [rows][out]
  const int* idx;  // [E][steps][Bm]
  int steps, Bm, last_rows;
  long long adam_step;  // Adam steps taken before this launch
  float* losses;        // [steps]
  float* ws;
};

// ---- phases ---------------------------------------------------------------------------------------------------------

// Z_l = A_{l-1} W_l + b_l (matmul, then the bias, as EnsembleLinearLayer), A_l = act(Z_l)
__device__ void forward_job(const TrainDev& m, const EpochArgs& a, const TrainWs& w, int s, int B, int l, int job,
                            float (*Ls)[TT + 1], float (*Rs)[TT + 1]) {
  const int K = m.K[l], N = m.N[l];
  const int rt = (B + TT - 1) / TT, ct = (N + TT - 1) / TT;
  const int e = job / (rt * ct), r0 = (job / ct) % rt * TT, c0 = job % ct * TT;
  Opnd Lo, Ro;
  if (l == 0) Lo = Opnd{a.X, a.idx + ((long long)e * a.steps + s) * a.Bm, m.in, 1, 0, -1};
  else Lo = Opnd{a.ws + w.A(l - 1) + (size_t)e * a.Bm * K, nullptr, K, 1, 0, -1};
  Ro = Opnd{m.W[l] + (size_t)e * K * N, nullptr, 1, N, 0, -1};
  float acc[4];
  tile_mm(Lo, Ro, B, N, K, r0, c0, acc, Ls, Rs);
  const int tx = threadIdx.x % TT, ty = threadIdx.x / TT, c = c0 + tx;
  if (c >= N) return;
  const float bias = m.b[l][(size_t)e * N + c];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int r = r0 + ty + 8 * q;
    if (r >= B) continue;
    const float z = acc[q] + bias;
    const size_t o = ((size_t)e * a.Bm + r) * N + c;
    if (l < m.L) {
      a.ws[w.Z(l) + o] = z;
      a.ws[w.A(l) + o] = activation_f(z, m.act, m.leaky);
    } else {
      a.ws[w.out + o] = z;
    }
  }
}

// G_{l-1} = (G_l W_l^T) * act'(Z_{l-1})
__device__ void backdata_job(const TrainDev& m, const EpochArgs& a, const TrainWs& w, int B, int l, int job,
                             float (*Ls)[TT + 1], float (*Rs)[TT + 1]) {
  const int K = m.K[l], N = m.N[l];
  const int rt = (B + TT - 1) / TT, ct = (K + TT - 1) / TT;
  const int e = job / (rt * ct), r0 = (job / ct) % rt * TT, c0 = job % ct * TT;
  const float* G = a.ws + (l == m.L ? w.out : w.G(l)) + (size_t)e * a.Bm * N;
  const Opnd Lo{G, nullptr, N, 1, 0, -1};
  const Opnd Ro{m.W[l] + (size_t)e * K * N, nullptr, N, 1, 0, -1};
  float acc[4];
  tile_mm(Lo, Ro, B, K, N, r0, c0, acc, Ls, Rs);
  const int tx = threadIdx.x % TT, ty = threadIdx.x / TT, c = c0 + tx;
  if (c >= K) return;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int r = r0 + ty + 8 * q;
    if (r >= B) continue;
    const size_t o = ((size_t)e * a.Bm + r) * K + c;
    a.ws[w.G(l - 1) + o] = activation_grad(acc[q], a.ws[w.Z(l - 1) + o], m.act, m.leaky);
  }
}

// dW_l = A_{l-1}^T G_l, db_l = column sums of G_l (the ones row), then Adam on every element
__device__ void wgrad_job(const TrainDev& m, const EpochArgs& a, const TrainWs& w, int s, int B, int l, int job,
                          const AdamStep& st, float (*Ls)[TT + 1], float (*Rs)[TT + 1]) {
  const int K = m.K[l], N = m.N[l];
  const int it = (K + 1 + TT - 1) / TT, jt = (N + TT - 1) / TT;
  const int e = job / (it * jt), i0 = (job / jt) % it * TT, j0 = job % jt * TT;
  Opnd Lo;
  if (l == 0) Lo = Opnd{a.X, a.idx + ((long long)e * a.steps + s) * a.Bm, 1, m.in, 1, K};
  else Lo = Opnd{a.ws + w.A(l - 1) + (size_t)e * a.Bm * K, nullptr, 1, K, 0, K};
  const float* G = a.ws + (l == m.L ? w.out : w.G(l)) + (size_t)e * a.Bm * N;
  const Opnd Ro{G, nullptr, 1, N, 0, -1};
  float acc[4];
  tile_mm(Lo, Ro, K + 1, N, B, i0, j0, acc, Ls, Rs);
  const int tx = threadIdx.x % TT, ty = threadIdx.x / TT, c = j0 + tx;
  if (c >= N) return;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = i0 + ty + 8 * q;
    if (i > K) continue;
    if (i < K) {
      const size_t o = ((size_t)e * K + i) * N + c;
      adam_update(m.W[l] + o, m.mW[l] + o, m.vW[l] + o, acc[q], st);
    } else {
      const size_t o = (size_t)e * N + c;
      adam_update(m.b[l] + o, m.mb[l] + o, m.vb[l] + o, acc[q], st);
    }
  }
}

// Per output element: GaussianMLP._nll_loss (gaussian_nll(reduce=False).mean((1, 2)).sum() + bound term, through the
// soft logvar bounds) or _mse_loss, its value and its gradient w.r.t. the output layer's pre-activations.
__device__ void loss_elements(const TrainDev& m, const EpochArgs& a, const TrainWs& w, int s, int B) {
  float* ws = a.ws;
  if (blockIdx.x == 0 && threadIdx.x == 0 && !m.deterministic) {
    float smax = 0.f, smin = 0.f;
    for (int j = 0; j < m.out; ++j) {
      smax += m.lv[1][j];
      smin += m.lv[0][j];
    }
    ws[w.scal] = 0.01f * (smax - smin);
  }
  const long long total = (long long)m.E * B * m.out;
  const float invN = 1.0f / (float)((long long)B * m.out);
  for (long long t = (long long)blockIdx.x * kThreads + threadIdx.x; t < total; t += (long long)gridDim.x * kThreads) {
    const int j = (int)(t % m.out);
    const int r = (int)((t / m.out) % B);
    const int e = (int)(t / ((long long)m.out * B));
    const int row = a.idx[((long long)e * a.steps + s) * a.Bm + r];
    const float y = a.Y[(long long)row * m.out + j];
    float* o = ws + w.out + ((size_t)e * a.Bm + r) * m.nout;
    const size_t el = ((size_t)e * a.Bm + r) * m.out + j;
    const float d = o[j] - y;
    if (m.deterministic) {
      ws[w.lossel + el] = d * d;
      o[j] = 2.0f * d;
      continue;
    }
    const float mn = m.lv[0][j], mx = m.lv[1][j], lv0 = o[m.out + j];
    const float u = mx - lv0;
    const float ab = mx - softplus_f(u);
    const float wv = ab - mn;
    const float lv = mn + softplus_f(wv);
    const float l2 = d * d, iv = expf(-lv);
    ws[w.lossel + el] = l2 * iv + lv;
    const float gl = invN;
    const float glv = gl - gl * l2 * iv;  // through + lv and through l2 * exp(-lv)
    const float ga = glv * softplus_grad(wv);
    const float g0 = ga * softplus_grad(u);
    o[j] = 2.0f * d * (gl * iv);
    o[m.out + j] = g0;
    ws[w.gmin + el] = glv - ga;
    ws[w.gmax + el] = ga - g0;
  }
}

// Loss value of the step (job 0) and, with learned bounds, the min / max logvar gradients and updates (job 1 + j).
__device__ void reduce_job(const TrainDev& m, const EpochArgs& a, const TrainWs& w, int s, int B, int job,
                           const AdamStep& st, double* dred, float* fred) {
  const float* ws = a.ws;
  if (job == 0) {
    double loss = 0.0;
    for (int e = 0; e < m.E; ++e) {
      double part = 0.0;
      for (int t = threadIdx.x; t < B * m.out; t += kThreads)
        part += ws[w.lossel + (size_t)e * a.Bm * m.out + t];
      part = block_sum(part, dred);
      loss += m.deterministic ? part : part / ((double)B * m.out);
    }
    if (threadIdx.x == 0) a.losses[s] = (float)(m.deterministic ? loss : loss + (double)ws[w.scal]);
    return;
  }
  const int j = job - 1;
  float smin = 0.f, smax = 0.f;
  for (int t = threadIdx.x; t < m.E * B; t += kThreads) {
    const int e = t / B, r = t % B;
    const size_t el = ((size_t)e * a.Bm + r) * m.out + j;
    smin += ws[w.gmin + el];
    smax += ws[w.gmax + el];
  }
  smin = block_sum(smin, fred);
  smax = block_sum(smax, fred);
  if (threadIdx.x == 0) {
    adam_update(m.lv[0] + j, m.mlv[0] + j, m.vlv[0] + j, smin - 0.01f, st);
    adam_update(m.lv[1] + j, m.mlv[1] + j, m.vlv[1] + j, smax + 0.01f, st);
  }
}

__global__ void __launch_bounds__(kThreads) train_adam_kernel(const __grid_constant__ TrainDev m,
                                                              const __grid_constant__ EpochArgs a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ float Ls[TT][TT + 1], Rs[TT][TT + 1];
  __shared__ double dred[kThreads];
  __shared__ float fred[kThreads];
  const TrainWs w = train_ws_layout(m, a.Bm);
  for (int s = 0; s < a.steps; ++s) {
    const int B = s == a.steps - 1 ? a.last_rows : a.Bm;
    const AdamStep st = adam_scalars(m, a.adam_step + s + 1);
    const int rt = (B + TT - 1) / TT;
    for (int l = 0; l <= m.L; ++l) {
      const int jobs = m.E * rt * ((m.N[l] + TT - 1) / TT);
      for (int j = blockIdx.x; j < jobs; j += gridDim.x) forward_job(m, a, w, s, B, l, j, Ls, Rs);
      grid.sync();
    }
    loss_elements(m, a, w, s, B);
    grid.sync();
    for (int l = m.L; l >= 1; --l) {
      const int nb = m.E * rt * ((m.K[l] + TT - 1) / TT);
      int nx;
      if (l == m.L) nx = 1 + (m.deterministic || !m.learn_bounds ? 0 : m.out);
      else nx = m.E * ((m.K[l + 1] + 1 + TT - 1) / TT) * ((m.N[l + 1] + TT - 1) / TT);
      for (int j = blockIdx.x; j < nb + nx; j += gridDim.x) {
        if (j < nb) backdata_job(m, a, w, B, l, j, Ls, Rs);
        else if (l == m.L) reduce_job(m, a, w, s, B, j - nb, st, dred, fred);
        else wgrad_job(m, a, w, s, B, l + 1, j - nb, st, Ls, Rs);
      }
      grid.sync();
    }
    {
      const int n1 = m.L >= 1 ? m.E * ((m.K[1] + 1 + TT - 1) / TT) * ((m.N[1] + TT - 1) / TT) : 0;
      const int n0 = m.E * ((m.K[0] + 1 + TT - 1) / TT) * ((m.N[0] + TT - 1) / TT);
      for (int j = blockIdx.x; j < n1 + n0; j += gridDim.x) {
        if (j < n1) wgrad_job(m, a, w, s, B, 1, j, st, Ls, Rs);
        else wgrad_job(m, a, w, s, B, 0, j - n1, st, Ls, Rs);
      }
      grid.sync();
    }
  }
}

// ---- evaluation -----------------------------------------------------------------------------------------------------
// CTA (tile, member e): 32 dataset rows through every layer of member e with the activations in shared memory, then
// the rows' squared errors summed into partial[e][tile]; the last CTA to finish sums the partials of each member in
// tile order (double) and writes scores[e] = mean over rows and output columns.
constexpr int kEvalRows = 32;

__global__ void __launch_bounds__(kThreads) train_eval_kernel(const __grid_constant__ TrainDev m, long long rows, const float* __restrict__ X,
                                                              const float* __restrict__ Y, int LD, float* partial,
                                                              unsigned int* counter, float* scores) {
  extern __shared__ __align__(16) float ev_smem[];
  __shared__ float fred[kThreads];
  __shared__ bool last;
  float* bufA = ev_smem;
  float* bufB = ev_smem + kEvalRows * LD;
  const int tile = blockIdx.x, e = blockIdx.y, tiles = gridDim.x;
  const long long r0 = (long long)tile * kEvalRows;
  const int nr = (int)min((long long)kEvalRows, rows - r0);
  for (int t = threadIdx.x; t < kEvalRows * LD; t += kThreads) {
    const int i = t / LD, k = t % LD;
    bufA[t] = (i < nr && k < m.in) ? X[(r0 + i) * m.in + k] : 0.0f;
  }
  __syncthreads();
  const int tx = threadIdx.x % 32, ty = threadIdx.x / 32;  // column lane, rows ty * 4 .. ty * 4 + 3
  float* in = bufA;
  float* out = bufB;
  for (int l = 0; l <= m.L; ++l) {
    const int K = m.K[l], N = m.N[l];
    const int K4 = (K + 3) / 4 * 4;
    const float* W = m.W[l] + (size_t)e * K * N;
    const float* bias = m.b[l] + (size_t)e * N;
    for (int c = tx; c < N; c += 32) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int k = 0; k < K4; k += 4) {
        float wk[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) wk[u] = k + u < K ? W[(size_t)(k + u) * N + c] : 0.0f;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 x = *reinterpret_cast<const float4*>(in + (ty * 4 + q) * LD + k);
          acc[q] = fmaf(x.x, wk[0], acc[q]);
          acc[q] = fmaf(x.y, wk[1], acc[q]);
          acc[q] = fmaf(x.z, wk[2], acc[q]);
          acc[q] = fmaf(x.w, wk[3], acc[q]);
        }
      }
      const float b = bias[c];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float z = acc[q] + b;
        out[(ty * 4 + q) * LD + c] = l < m.L ? activation_f(z, m.act, m.leaky) : z;
      }
    }
    // zero the padding columns the next layer's float4 reads touch
    for (int t = threadIdx.x; t < kEvalRows * 4; t += kThreads) {
      const int i = t / 4, c = N + t % 4;
      if (c < LD) out[i * LD + c] = 0.0f;
    }
    __syncthreads();
    float* tmp = in;
    in = out;
    out = tmp;
  }
  float se = 0.0f;
  for (int t = threadIdx.x; t < nr * m.out; t += kThreads) {
    const int i = t / m.out, j = t % m.out;
    const float d = in[i * LD + j] - Y[(r0 + i) * m.out + j];
    se += d * d;
  }
  se = block_sum(se, fred);
  if (threadIdx.x == 0) {
    partial[(size_t)e * tiles + tile] = se;
    __threadfence();
    last = atomicAdd(counter, 1u) == (unsigned)(tiles * m.E) - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  __shared__ double dred[kThreads];
  for (int mem = 0; mem < m.E; ++mem) {
    double s = 0.0;
    for (int t = threadIdx.x; t < tiles; t += kThreads) s += (double)((volatile float*)partial)[(size_t)mem * tiles + t];
    s = block_sum(s, dred);
    if (threadIdx.x == 0) scores[mem] = (float)(s / ((double)rows * m.out));
  }
  if (threadIdx.x == 0) *counter = 0u;
}

// ---- preprocessing --------------------------------------------------------------------------------------------------
// Transitions stored as T (float or double), computed the way the reference's _process_batch computes them for that
// storage (one_dim_tr_model.py:118-136): numpy keeps float64 data in double through obs_process_fn, the delta targets
// and the normaliser (a float32 normaliser is promoted to double against float64 data), and .float() rounds at the end.

// proc_obs_elem (common.cuh) for float64 observations: the same columns, sin / cos in double as numpy computes them
__device__ __forceinline__ double proc_obs_elem_f64(const double* obs, int j, int mode) {
  if (mode == B200PETS_PROC_HALFCHEETAH) {  // [o1, sin o2, cos o2, o3:]
    if (j == 0) return obs[1];
    if (j == 1) return sin(obs[2]);
    if (j == 2) return cos(obs[2]);
    return obs[j];
  }
  if (mode == B200PETS_PROC_CARTPOLE) {  // [sin o1, cos o1, o0, o2:]
    if (j == 0) return sin(obs[1]);
    if (j == 1) return cos(obs[1]);
    if (j == 2) return obs[0];
    return obs[j - 1];
  }
  return obs[j];
}

__device__ __forceinline__ float model_input(const PrepDesc& d, const float* o, const float* act, long long r, int j,
                                             const void* norm_mean, const void* norm_std) {
  float x = j < d.Dp ? proc_obs_elem(o, j, d.obs_process) : act[r * d.A + (j - d.Dp)];
  if (d.norm_mode == 2) return (float)(((double)x - ((const double*)norm_mean)[j]) / ((const double*)norm_std)[j]);
  if (d.norm_mode == 1) return (x - ((const float*)norm_mean)[j]) / ((const float*)norm_std)[j];
  return x;
}

__device__ __forceinline__ float model_input(const PrepDesc& d, const double* o, const double* act, long long r, int j,
                                             const void* norm_mean, const void* norm_std) {
  double x = j < d.Dp ? proc_obs_elem_f64(o, j, d.obs_process) : act[r * d.A + (j - d.Dp)];
  if (d.norm_mode == 2) x = (x - ((const double*)norm_mean)[j]) / ((const double*)norm_std)[j];
  else if (d.norm_mode == 1) x = (x - (double)((const float*)norm_mean)[j]) / (double)((const float*)norm_std)[j];
  return (float)x;
}

// thread per (row, column) of [inputs | targets]
template <typename T>
__global__ void train_preprocess_kernel(const PrepDesc d, long long rows, const T* __restrict__ obs,
                                        const T* __restrict__ act, const T* __restrict__ next_obs,
                                        const T* __restrict__ reward, const void* norm_mean, const void* norm_std,
                                        float* __restrict__ X, float* __restrict__ Y) {
  const int width = d.in + d.out;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= rows * width) return;
  const long long r = t / width;
  const int j = (int)(t % width);
  const T* o = obs + r * d.D;
  if (j < d.in) {
    X[r * d.in + j] = model_input(d, o, act, r, j, norm_mean, norm_std);
    return;
  }
  const int c = j - d.in;
  float y;
  if (c < d.D) {
    const T nx = next_obs[r * d.D + c];
    const bool keep = !d.target_is_delta || ((d.no_delta[c >> 5] >> (c & 31)) & 1u);
    y = (float)(keep ? nx : nx - o[c]);
  } else {
    y = (float)reward[r];
  }
  Y[r * d.out + c] = y;
}

}  // namespace

size_t train_workspace_floats(const TrainDev& m, int batch) { return train_ws_layout(m, batch).total; }

static int eval_ld(const TrainDev& m) {
  int w = m.in;
  for (int l = 0; l <= m.L; ++l) w = max(w, m.N[l]);
  return (w + 3) / 4 * 4 + 4;  // float4 rows plus the zeroed padding
}

size_t eval_score_workspace_bytes(const TrainDev& m, long long rows) {
  const long long tiles = (rows + kEvalRows - 1) / kEvalRows;
  return 256 + (size_t)m.E * tiles * sizeof(float);
}

int launch_train_epoch(const TrainDev& m, long long rows, const float* X, const float* Y, const int* idx, int steps, int batch,
                       int last_batch, long long adam_step, float* losses, float* ws, cudaStream_t stream) {
  (void)rows;
  if (steps == 0) return 0;
  int dev, sms = 0, per_sm = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, train_adam_kernel, kThreads, 0));
  if (per_sm < 1) return b200pets_set_error(B200PETS_EUNSUPPORTED, "train_adam_kernel does not fit on an SM");
  EpochArgs a{X, Y, idx, steps, batch, last_batch, adam_step, losses, ws};
  TrainDev mm = m;
  void* args[] = {&mm, &a};
  // one CTA per SM: every CTA is co-resident, as the grid-wide barriers require
  CUDA_TRY(cudaLaunchCooperativeKernel((void*)train_adam_kernel, dim3(sms), dim3(kThreads), args, 0, stream));
  return 0;
}

int eval_score_fits(const TrainDev& m) {
  const int LD = eval_ld(m);
  const size_t smem = 2 * (size_t)kEvalRows * LD * sizeof(float);
  int dev, max_smem;
  cudaFuncAttributes fa;
  CUDA_TRY(cudaGetDevice(&dev));
  CUDA_TRY(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  CUDA_TRY(cudaFuncGetAttributes(&fa, train_eval_kernel));
  if (smem + fa.sharedSizeBytes > (size_t)max_smem)  // dynamic activations + the kernel's static reduction buffers
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "eval_score: layers of %d columns do not fit in shared memory", LD);
  return 0;
}

int launch_eval_score(const TrainDev& m, long long rows, const float* X, const float* Y, float* scores, void* ws,
                      cudaStream_t stream) {
  const long long tiles = (rows + kEvalRows - 1) / kEvalRows;
  if (tiles > 0x7fffffff) return b200pets_set_error(B200PETS_EINVAL, "eval_score: too many rows");
  if (const int rc = eval_score_fits(m)) return rc;
  const int LD = eval_ld(m);
  const size_t smem = 2 * (size_t)kEvalRows * LD * sizeof(float);
  CUDA_TRY(cudaFuncSetAttribute(train_eval_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  unsigned int* counter = (unsigned int*)ws;
  float* partial = (float*)((char*)ws + 256);
  CUDA_TRY(cudaMemsetAsync(counter, 0, sizeof(unsigned int), stream));
  train_eval_kernel<<<dim3((unsigned)tiles, m.E), kThreads, smem, stream>>>(m, rows, X, Y, LD, partial, counter, scores);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_train_preprocess(const PrepDesc& d, long long rows, const void* obs, const void* act, const void* next_obs,
                            const void* reward, const void* norm_mean, const void* norm_std, float* X, float* Y,
                            cudaStream_t stream) {
  const long long n = rows * (d.in + d.out);
  if (n == 0) return 0;
  const int threads = 256;
  const unsigned blocks = (unsigned)((n + threads - 1) / threads);
  if (d.f64)
    train_preprocess_kernel<double><<<blocks, threads, 0, stream>>>(d, rows, (const double*)obs, (const double*)act,
                                                                    (const double*)next_obs, (const double*)reward,
                                                                    norm_mean, norm_std, X, Y);
  else
    train_preprocess_kernel<float><<<blocks, threads, 0, stream>>>(d, rows, (const float*)obs, (const float*)act,
                                                                   (const float*)next_obs, (const float*)reward, norm_mean,
                                                                   norm_std, X, Y);
  CUDA_TRY(cudaGetLastError());
  return 0;
}
