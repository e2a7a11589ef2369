// One SAC update on the device: SAC.update_parameters of mbrl-lib's pytorch_sac_pranz24 agent
// (mbrl/third_party/pytorch_sac_pranz24/sac.py:76-173, networks in model.py:36-113) as one cooperative launch.  fp32
// FFMA throughout, for the reason train.cu's header gives: the reference trains in fp32 with TF32 off.
//
// Structure.  An update is a chain of small dependent products (B or 2B rows, hidden 256 .. 1024 columns), the same
// shape of work as train_adam_kernel's minibatch step, and it is run the same way: a persistent cooperative grid walks
// the chain phase by phase with a grid-wide barrier between phases; each phase is a list of independent 32 x 32 output
// tiles dealt round-robin to the CTAs; every weight-gradient element is computed by exactly one thread, which applies
// torch.optim.Adam (adam.cuh, the rule documented at the top of train.cu) to it at once.  Sums run in a fixed order, so
// two runs are bit-identical.  Rows of the policy are [s' ; s] (sample 0 on s', sample 1 on s); the twin networks of
// the critic are nets 0 (linear1-3) and 1 (linear4-6).
//
//   phase  work                                                                      reads the result of
//    0     policy layer 1 on s' and s;  critic layer 1 on (s, a)
//    1     policy layer 2;              critic layer 2 on (s, a)                      0
//    2     heads + sample (row-wise: a row's A <= 32 actions sit in one tile, so the
//          log-probability's sum over actions is a warp reduction): a', log pi', pi,
//          log pi                                                                     1
//    3     target critic layer 1 on (s', a')                                          2
//    4     target critic layer 2                                                      3
//    5     per row: both target Q, both Q(s, a), y_t, the MSE gradients, dL/dz of
//          critic layer 2                                                             1, 4
//    6     critic: dL/dz of layer 1;  Adam on linear3 / linear6                       5
//    7     critic: Adam on layers 2 and 1 (the critic step ends here)                 6
//    8     updated critic layer 1 on (s, pi);  the soft target update when due        7
//    9     critic layer 2 on (s, pi)                                                  8
//   10     per row: min(Q1, Q2)(s, pi) (ties give each side half the gradient), dL/dz
//          of critic layer 2                                                          9
//   11     critic: dL/dz of layer 1                                                   10
//   12     dL/d(action columns) through both critics, then through tanh, the
//          reparameterisation, log_prob and the clamp into both heads                 11
//   13     policy: dL/dz of layer 2 from both heads                                   12
//   14     policy: dL/dz of layer 1;  Adam on the heads                               13
//   15     policy: Adam on layers 2 and 1;  the temperature step and the statistics   14
// Critic gradients of the policy loss are computed only as far as the action columns: the reference discards them.
//
// At hidden 1024 (mbpo_ant, mbpo_humanoid) the parameters, the target copy and both Adam moments total about 48 MB,
// close to the H100's 50 MB L2; whether that costs anything has not been measured.
//
// In-kernel draws: see RNG_STREAM_SAC in common.cuh.
#include <cooperative_groups.h>

#include "adam.cuh"
#include "sac.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int TT = 32;         // output tile edge and reduction chunk
constexpr int kThreads = 256;  // 8 warps: thread (ty, tx) owns rows ty, ty + 8, ty + 16, ty + 24 of column tx
constexpr int kPhases = 16;
constexpr int kMaxCtasPerSm = 2;  // the launch bounds hold the kernel to 128 registers, which fits two
constexpr float kLogSqrt2Pi = 0.918938533204672742f;  // math.log(math.sqrt(2 * math.pi)) of torch's Normal.log_prob

// A [rows][features] matrix: features [0, split) from p (row stride ld), the rest from p2 (row stride ld2) -- the
// concatenations [s, a] / [s', a'] / [s, pi] of the critic's input without a copy.
struct Src {
  const float* p;
  long long ld;
  int split;
  const float* p2;
  long long ld2;
};

// One operand of a tile product, element (x, y): x the output coordinate, y the reduction coordinate.  x_row: x is the
// matrix's row and y its feature (else the reverse); ones_at = x yields 1.0 (the bias column of a weight gradient).
struct Opnd {
  Src s;
  int x_row;
  int ones_at;
};

__device__ __forceinline__ Src src(const float* p, long long ld) { return Src{p, ld, 1 << 30, nullptr, 0}; }
__device__ __forceinline__ Opnd rows_of(const Src& s) { return Opnd{s, 1, -1}; }
__device__ __forceinline__ Opnd cols_of(const Src& s, int ones_at = -1) { return Opnd{s, 0, ones_at}; }

__device__ __forceinline__ float opnd_at(const Opnd& o, int x, int y, int X, int Y) {
  if (y >= Y) return 0.0f;
  if (x == o.ones_at) return 1.0f;
  if (x >= X) return 0.0f;
  const long long r = o.x_row ? x : y;
  const int f = o.x_row ? y : x;
  return f < o.s.split ? o.s.p[r * o.s.ld + f] : o.s.p2[r * o.s.ld2 + (f - o.s.split)];
}

// acc[q] = sum_k L(i0 + ty + 8q, k) * R(j0 + tx, k), k = 0 .. K-1 in ascending chunks of 32.
__device__ __forceinline__ void tile_mm(const Opnd& Lo, const Opnd& Ro, int M, int N, int K, int i0, int j0, float acc[4],
                                        float (*Ls)[TT + 1], float (*Rs)[TT + 1]) {
  const int tx = threadIdx.x % TT, ty = threadIdx.x / TT;
#pragma unroll
  for (int q = 0; q < 4; ++q) acc[q] = 0.0f;
  for (int k0 = 0; k0 < K; k0 += TT) {
    for (int e = threadIdx.x; e < TT * TT; e += kThreads) {
      // consecutive threads walk the operand's feature coordinate (coalesced loads)
      int x = e / TT, y = e % TT;
      if (!Lo.x_row) { x = e % TT; y = e / TT; }
      Ls[x][y] = opnd_at(Lo, i0 + x, k0 + y, M, K);
      x = e % TT; y = e / TT;
      if (Ro.x_row) { x = e / TT; y = e % TT; }
      Rs[y][x] = opnd_at(Ro, j0 + x, k0 + y, N, K);
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

__device__ __forceinline__ double block_sum(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

// sum over the 32 lanes; every lane gets the same bits (each butterfly step adds the same two values on both sides)
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float warp_dot(const float* x, const float* w, int n) {
  float s = 0.0f;
  for (int k = threadIdx.x % 32; k < n; k += 32) s = fmaf(x[k], w[k], s);
  return warp_sum(s);
}

// Workspace, offsets in floats.  [2][B][H] blocks hold either both policy samples or both critic nets.
struct SacWs {
  size_t BH;
  size_t pA1, pA2;  // policy activations, samples 0 (s') and 1 (s)
  size_t cA1, cA2;  // critic activations of each net, on (s, a), then on (s, pi)
  size_t tA1, tA2;  // target critic activations on (s', a')
  size_t cG1, cG2;  // critic dL/dz, for the critic loss, then for the policy loss
  size_t pG1, pG2;  // [B][H] policy dL/dz (sample 1)
  size_t act;       // [2][B][A] a' and pi
  size_t y, eps, sd, xm, lsr, gmean, glsr;  // [B][A] of sample 1: tanh(x), the draw, std, x - mean, log_std before the
                                            // clamp, dL/dmean, dL/dlog_std before the clamp
  size_t logp;      // [2][B]
  size_t gq;        // [2][B] dL/dQ of each net (critic loss)
  size_t rows;      // [3][B] (Q1 - y_t)^2, (Q2 - y_t)^2, alpha log pi - min Q(s, pi)
  size_t total;
};

__host__ __device__ inline SacWs sac_ws_layout(const SacDev& m, int B) {
  SacWs w;
  size_t off = 0;
  auto take = [&](size_t n) { size_t o = off; off += (n + 63) / 64 * 64; return o; };
  w.BH = (size_t)B * m.H;
  w.pA1 = take(2 * w.BH); w.pA2 = take(2 * w.BH);
  w.cA1 = take(2 * w.BH); w.cA2 = take(2 * w.BH);
  w.tA1 = take(2 * w.BH); w.tA2 = take(2 * w.BH);
  w.cG1 = take(2 * w.BH); w.cG2 = take(2 * w.BH);
  w.pG1 = take(w.BH); w.pG2 = take(w.BH);
  const size_t BA = (size_t)B * m.A;
  w.act = take(2 * BA);
  w.y = take(BA); w.eps = take(BA); w.sd = take(BA); w.xm = take(BA); w.lsr = take(BA);
  w.gmean = take(BA); w.glsr = take(BA);
  w.logp = take(2 * (size_t)B);
  w.gq = take(2 * (size_t)B);
  w.rows = take(3 * (size_t)B);
  w.total = off;
  return w;
}

// ---- tasks: the units of a phase --------------------------------------------------------------------------------------
enum Kind { T_NONE, T_FWD, T_BWD, T_WGRAD, T_HEADS, T_ACTGRAD, T_ROWQ, T_ROWPI, T_STATS };

struct Task {
  int kind, M, N, K;  // tile products: out[M][N] = sum_k L(m, k) R(n, k)
  Opnd L, R, L2, R2;  // L2 R2^T: the second product of T_BWD (added), T_HEADS (log_std head), T_ACTGRAD (added)
  int two;
  const float* bias;  // T_FWD: out = relu?(acc + bias[n])
  int relu;
  float* out;
  const float* mask;  // T_BWD: out = acc * (mask > 0)
  float *w, *mw, *vw, *b, *mb, *vb;  // T_WGRAD: Adam on w[M][N - 1] and the bias column b[M]
  int opt;            // T_WGRAD: 0 critic, 1 policy (whose step count)
  int smp;            // T_HEADS: 0 on s', 1 on s
};

__device__ __forceinline__ int task_jobs(const Task& t) {
  if (t.kind == T_NONE) return 0;
  if (t.kind == T_ROWQ || t.kind == T_ROWPI) return (t.M + 7) / 8;
  if (t.kind == T_STATS) return 1;
  return ((t.M + TT - 1) / TT) * ((t.N + TT - 1) / TT);
}

// nn.Linear forward: out[M][N] = act(in[M][K] W[N][K]^T + b)
__device__ __forceinline__ Task fwd(const Src& in, int M, int K, int N, const float* W, const float* b, float* out,
                                    int relu) {
  Task t{};
  t.kind = T_FWD; t.M = M; t.N = N; t.K = K;
  t.L = rows_of(in); t.R = rows_of(src(W, K));
  t.bias = b; t.relu = relu; t.out = out;
  return t;
}

// backward through nn.Linear and the previous ReLU: out[M][Kw] = (G[M][Nw] W[Nw][Kw]) * (act[M][Kw] > 0)
__device__ __forceinline__ Task bwd(const float* G, int M, int Nw, int Kw, const float* W, const float* act, float* out) {
  Task t{};
  t.kind = T_BWD; t.M = M; t.N = Kw; t.K = Nw;
  t.L = rows_of(src(G, Nw)); t.R = cols_of(src(W, Kw));
  t.mask = act; t.out = out;
  return t;
}

// weight gradient G[B][Nw]^T X[B][Kw], bias gradient = column sums of G, then Adam on each element
__device__ __forceinline__ Task wgrad(const float* G, int B, int Nw, const Src& X, int Kw, float* const* p, float* const* m,
                                      float* const* v, int opt) {
  Task t{};
  t.kind = T_WGRAD; t.M = Nw; t.N = Kw + 1; t.K = B;
  t.L = cols_of(src(G, Nw)); t.R = cols_of(X, Kw);
  t.w = p[0]; t.b = p[1]; t.mw = m[0]; t.mb = m[1]; t.vw = v[0]; t.vb = v[1];
  t.opt = opt;
  return t;
}

// Task g of phase ph (kind T_NONE past the last one).  See the phase table at the top of the file.
__device__ __forceinline__ Task task(const SacDev& m, const SacArgs& a, const SacWs& w, int ph, int g) {
  const int B = a.B, D = m.D, A = m.A, H = m.H, TW = 2 * D + A + 2;
  float* ws = a.ws;
  const size_t BH = w.BH;
  const Src s_a = src(a.trans, TW);  // s, and [s, a] (contiguous columns 0 .. D + A - 1)
  const int n = g & 1;               // critic net / policy sample of a pair of tasks
  const int c = 6 * n;               // first critic parameter of net n
  Task t{};
  switch (ph) {
    case 0:
      if (g < 2) return fwd(g == 0 ? src(a.trans + D + A, TW) : s_a, B, D, H, m.pp[0], m.pp[1], ws + w.pA1 + g * BH, 1);
      if (g < 4) return fwd(s_a, B, D + A, H, m.cp[c], m.cp[c + 1], ws + w.cA1 + n * BH, 1);
      break;
    case 1:
      if (g < 2) return fwd(src(ws + w.pA1 + g * BH, H), B, H, H, m.pp[2], m.pp[3], ws + w.pA2 + g * BH, 1);
      if (g < 4) return fwd(src(ws + w.cA1 + n * BH, H), B, H, H, m.cp[c + 2], m.cp[c + 3], ws + w.cA2 + n * BH, 1);
      break;
    case 2:
      if (g < 2) {
        t.kind = T_HEADS; t.M = B; t.N = A; t.K = H; t.smp = g; t.two = 1;
        t.L = rows_of(src(ws + w.pA2 + g * BH, H));
        t.R = rows_of(src(m.pp[4], H));
        t.L2 = t.L;
        t.R2 = rows_of(src(m.pp[6], H));
        return t;
      }
      break;
    case 3:
      if (g < 2) {
        const Src in{a.trans + D + A, TW, D, ws + w.act, A};  // [s', a']
        return fwd(in, B, D + A, H, m.ct[c], m.ct[c + 1], ws + w.tA1 + n * BH, 1);
      }
      break;
    case 4:
      if (g < 2) return fwd(src(ws + w.tA1 + n * BH, H), B, H, H, m.ct[c + 2], m.ct[c + 3], ws + w.tA2 + n * BH, 1);
      break;
    case 5:
      if (g == 0) { t.kind = T_ROWQ; t.M = B; return t; }
      break;
    case 6:
      if (g < 2) return bwd(ws + w.cG2 + n * BH, B, H, H, m.cp[c + 2], ws + w.cA1 + n * BH, ws + w.cG1 + n * BH);
      if (g < 4) return wgrad(ws + w.gq + n * B, B, 1, src(ws + w.cA2 + n * BH, H), H, m.cp + c + 4, m.cm + c + 4,
                              m.cv + c + 4, 0);
      break;
    case 7:
      if (g < 2) return wgrad(ws + w.cG2 + n * BH, B, H, src(ws + w.cA1 + n * BH, H), H, m.cp + c + 2, m.cm + c + 2,
                              m.cv + c + 2, 0);
      if (g < 4) return wgrad(ws + w.cG1 + n * BH, B, H, s_a, D + A, m.cp + c, m.cm + c, m.cv + c, 0);
      break;
    case 8:
      if (g < 2) {
        const Src in{a.trans, TW, D, ws + w.act + (size_t)B * A, A};  // [s, pi]
        return fwd(in, B, D + A, H, m.cp[c], m.cp[c + 1], ws + w.cA1 + n * BH, 1);
      }
      break;
    case 9:
      if (g < 2) return fwd(src(ws + w.cA1 + n * BH, H), B, H, H, m.cp[c + 2], m.cp[c + 3], ws + w.cA2 + n * BH, 1);
      break;
    case 10:
      if (g == 0) { t.kind = T_ROWPI; t.M = B; return t; }
      break;
    case 11:
      if (g < 2) return bwd(ws + w.cG2 + n * BH, B, H, H, m.cp[c + 2], ws + w.cA1 + n * BH, ws + w.cG1 + n * BH);
      break;
    case 12:
      if (g == 0) {  // dL/dpi = sum over both nets of dL/dz1 W1[:, D:]
        t.kind = T_ACTGRAD; t.M = B; t.N = A; t.K = H; t.two = 1;
        t.L = rows_of(src(ws + w.cG1, H));
        t.R = cols_of(src(m.cp[0] + D, D + A));
        t.L2 = rows_of(src(ws + w.cG1 + BH, H));
        t.R2 = cols_of(src(m.cp[6] + D, D + A));
        return t;
      }
      break;
    case 13:
      if (g == 0) {  // both heads: dL/dmean Wm + dL/dlog_std Ws
        t = bwd(ws + w.gmean, B, A, H, m.pp[4], ws + w.pA2 + BH, ws + w.pG2);
        t.two = 1;
        t.L2 = rows_of(src(ws + w.glsr, A));
        t.R2 = cols_of(src(m.pp[6], H));
        return t;
      }
      break;
    case 14:
      if (g == 0) return bwd(ws + w.pG2, B, H, H, m.pp[2], ws + w.pA1 + BH, ws + w.pG1);
      if (g == 1) return wgrad(ws + w.gmean, B, A, src(ws + w.pA2 + BH, H), H, m.pp + 4, m.pm + 4, m.pv + 4, 1);
      if (g == 2) return wgrad(ws + w.glsr, B, A, src(ws + w.pA2 + BH, H), H, m.pp + 6, m.pm + 6, m.pv + 6, 1);
      break;
    case 15:
      if (g == 0) return wgrad(ws + w.pG2, B, H, src(ws + w.pA1 + BH, H), H, m.pp + 2, m.pm + 2, m.pv + 2, 1);
      if (g == 1) return wgrad(ws + w.pG1, B, H, s_a, D, m.pp, m.pm, m.pv, 1);
      if (g == 2) { t.kind = T_STATS; return t; }
      break;
  }
  t.kind = T_NONE;
  return t;
}

// ---- task bodies ------------------------------------------------------------------------------------------------------

// Row-wise head phase: mean, log_std (clamped to [-20, 2]), the reparameterised draw, tanh, the action and the
// log-probability of GaussianPolicy.sample, one row of A <= 32 actions per warp.
__device__ __forceinline__ void heads_epilogue(const SacDev& m, const SacArgs& a, const SacWs& w, int smp, int r, int j,
                                               float am, float as) {
  const bool valid = r < a.B && j < m.A;
  float lp = 0.0f;
  float* ws = a.ws;
  if (valid) {
    const float mean = am + m.pp[5][j];
    const float lsr = as + m.pp[7][j];
    const float ls = fminf(fmaxf(lsr, -20.0f), 2.0f);
    const float sd = expf(ls);
    float ep;
    if (a.eps) {
      ep = a.eps[((long long)smp * a.B + r) * m.A + j];
    } else {
      const float4 z = philox_normal4v((uint32_t)r, (uint32_t)smp, RNG_STREAM_SAC | (uint32_t)(j >> 2),
                                       (uint32_t)a.offset, a.seed);
      const int lane = j & 3;
      ep = lane == 0 ? z.x : lane == 1 ? z.y : lane == 2 ? z.z : z.w;
    }
    const float x = __fadd_rn(mean, __fmul_rn(ep, sd));  // loc + eps * scale
    const float y = tanhf(x);
    const float sc = m.scale[j];
    const float xm = __fsub_rn(x, mean);
    const float var = __fmul_rn(sd, sd);
    lp = -(xm * xm) / (2.0f * var) - logf(sd) - kLogSqrt2Pi;
    lp = lp - logf(sc * (1.0f - y * y) + 1e-6f);
    const size_t e = (size_t)r * m.A + j;
    ws[w.act + (size_t)smp * a.B * m.A + e] = __fadd_rn(__fmul_rn(y, sc), m.bias[j]);
    if (smp == 1) {
      ws[w.y + e] = y;
      ws[w.eps + e] = ep;
      ws[w.sd + e] = sd;
      ws[w.xm + e] = xm;
      ws[w.lsr + e] = lsr;
    }
  }
  lp = warp_sum(lp);
  if (r < a.B && j == 0) ws[w.logp + (size_t)smp * a.B + r] = lp;
}

// dL/dpi of the policy loss -> dL/dmean and dL/dlog_std (before the clamp) of one (row, action)
__device__ __forceinline__ void actgrad_epilogue(const SacDev& m, const SacArgs& a, const SacWs& w, float alpha, int r,
                                                 int j, float ga) {
  if (r >= a.B || j >= m.A) return;
  float* ws = a.ws;
  const size_t e = (size_t)r * m.A + j;
  const float y = ws[w.y + e], ep = ws[w.eps + e], sd = ws[w.sd + e], xm = ws[w.xm + e], lsr = ws[w.lsr + e];
  const float sc = m.scale[j];
  const float glogp = (1.0f / (float)a.B) * alpha;  // mean, then alpha * log_pi
  const float var = sd * sd;
  const float u = sc * (1.0f - y * y) + 1e-6f;
  const float gy = ga * sc + glogp * (2.0f * sc * y / u);  // action = y * scale + bias;  -log(scale (1 - y^2) + 1e-6)
  const float gx = gy * (1.0f - y * y) - glogp * (xm / var);                     // tanh;  log_prob through its value
  const float gmean = gx + glogp * (xm / var);                                    // x = mean + ...;  log_prob's loc
  const float gsd = gx * ep + glogp * (xm * xm / (var * sd) - 1.0f / sd);         // x = ... + eps std;  log_prob's scale
  const float gls = gsd * sd;                                                     // std = exp(log_std)
  ws[w.gmean + e] = gmean;
  ws[w.glsr + e] = (lsr >= -20.0f && lsr <= 2.0f) ? gls : 0.0f;                   // clamp: bounds pass gradient
}

__device__ __forceinline__ void mm_job(const SacDev& m, const SacArgs& a, const SacWs& w, const Task& t, int job,
                                       float alpha, float (*Ls)[TT + 1], float (*Rs)[TT + 1]) {
  const int ct = (t.N + TT - 1) / TT;
  const int i0 = job / ct * TT, j0 = job % ct * TT;
  const int tx = threadIdx.x % TT, ty = threadIdx.x / TT, c = j0 + tx;
  float acc[4], acc2[4];
  tile_mm(t.L, t.R, t.M, t.N, t.K, i0, j0, acc, Ls, Rs);
  if (t.two) tile_mm(t.L2, t.R2, t.M, t.N, t.K, i0, j0, acc2, Ls, Rs);
  if (t.kind == T_HEADS) {
#pragma unroll
    for (int q = 0; q < 4; ++q) heads_epilogue(m, a, w, t.smp, i0 + ty + 8 * q, c, acc[q], acc2[q]);
    return;
  }
  if (t.two) {
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[q] += acc2[q];
  }
  if (t.kind == T_ACTGRAD) {
#pragma unroll
    for (int q = 0; q < 4; ++q) actgrad_epilogue(m, a, w, alpha, i0 + ty + 8 * q, c, acc[q]);
    return;
  }
  if (c >= t.N) return;
  if (t.kind == T_WGRAD) {
    const AdamStep st = adam_scalars(m.lr, m.beta1, m.beta2, 0.0, m.eps, (t.opt ? a.step_p : a.step_c) + 1);
    const int Kw = t.N - 1;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = i0 + ty + 8 * q;
      if (i >= t.M) continue;
      if (c < Kw) {
        const size_t o = (size_t)i * Kw + c;
        adam_update(t.w + o, t.mw + o, t.vw + o, acc[q], st);
      } else {
        adam_update(t.b + i, t.mb + i, t.vb + i, acc[q], st);
      }
    }
    return;
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int r = i0 + ty + 8 * q;
    if (r >= t.M) continue;
    const size_t o = (size_t)r * t.N + c;
    if (t.kind == T_FWD) {
      const float z = acc[q] + t.bias[c];
      t.out[o] = t.relu ? fmaxf(z, 0.0f) : z;
    } else {  // T_BWD
      t.out[o] = t.mask[o] > 0.0f ? acc[q] : 0.0f;
    }
  }
}

// dL/dz of critic layer 2 of net n for row r: dL/dQ * linear3.weight through the ReLU
__device__ __forceinline__ void critic_out_grad(const SacDev& m, const SacWs& w, float* ws, int n, int r, float gq) {
  const float* h = ws + w.cA2 + n * w.BH + (size_t)r * m.H;
  const float* w3 = m.cp[6 * n + 4];
  float* out = ws + w.cG2 + n * w.BH + (size_t)r * m.H;
  for (int k = threadIdx.x % 32; k < m.H; k += 32) out[k] = h[k] > 0.0f ? gq * w3[k] : 0.0f;
}

// Critic loss, per row (one warp): y_t from the target critic, both Q(s, a), and dL/dQ.
__device__ __forceinline__ void rowq_job(const SacDev& m, const SacArgs& a, const SacWs& w, float alpha, int job) {
  const int r = job * 8 + threadIdx.x / 32;
  if (r >= a.B) return;
  float* ws = a.ws;
  const int H = m.H;
  const size_t o = (size_t)r * H;
  const float qt0 = warp_dot(ws + w.tA2 + o, m.ct[4], H) + m.ct[5][0];
  const float qt1 = warp_dot(ws + w.tA2 + w.BH + o, m.ct[10], H) + m.ct[11][0];
  const float q0 = warp_dot(ws + w.cA2 + o, m.cp[4], H) + m.cp[5][0];
  const float q1 = warp_dot(ws + w.cA2 + w.BH + o, m.cp[10], H) + m.cp[11][0];
  const float* tr = a.trans + (long long)r * (2 * m.D + m.A + 2);
  const float rew = tr[2 * m.D + m.A], term = tr[2 * m.D + m.A + 1];
  const float mk = a.reverse_mask ? (term == 0.0f ? 1.0f : 0.0f) : term;
  const float v = __fsub_rn(fminf(qt0, qt1), __fmul_rn(alpha, ws[w.logp + r]));
  const float yt = __fadd_rn(rew, __fmul_rn(__fmul_rn(mk, m.gamma), v));
  const float d0 = q0 - yt, d1 = q1 - yt;
  const float norm = 2.0f / (float)a.B;  // mse_loss backward
  const float g0 = norm * d0, g1 = norm * d1;
  if (threadIdx.x % 32 == 0) {
    ws[w.rows + r] = d0 * d0;
    ws[w.rows + a.B + r] = d1 * d1;
    ws[w.gq + r] = g0;
    ws[w.gq + a.B + r] = g1;
  }
  critic_out_grad(m, w, ws, 0, r, g0);
  critic_out_grad(m, w, ws, 1, r, g1);
}

// Policy loss, per row (one warp): min(Q1, Q2)(s, pi) of the updated critic and its gradient (torch.min gives each side
// half the gradient at a tie).
__device__ __forceinline__ void rowpi_job(const SacDev& m, const SacArgs& a, const SacWs& w, float alpha, int job) {
  const int r = job * 8 + threadIdx.x / 32;
  if (r >= a.B) return;
  float* ws = a.ws;
  const int H = m.H;
  const size_t o = (size_t)r * H;
  const float q0 = warp_dot(ws + w.cA2 + o, m.cp[4], H) + m.cp[5][0];
  const float q1 = warp_dot(ws + w.cA2 + w.BH + o, m.cp[10], H) + m.cp[11][0];
  const float g = -(1.0f / (float)a.B);
  const float g0 = q0 < q1 ? g : q0 == q1 ? 0.5f * g : 0.0f;
  const float g1 = q1 < q0 ? g : q0 == q1 ? 0.5f * g : 0.0f;
  if (threadIdx.x % 32 == 0) ws[w.rows + 2 * (size_t)a.B + r] = __fsub_rn(__fmul_rn(alpha, ws[w.logp + a.B + r]), fminf(q0, q1));
  critic_out_grad(m, w, ws, 0, r, g0);
  critic_out_grad(m, w, ws, 1, r, g1);
}

// The temperature step (automatic_entropy_tuning) and the statistics, in one CTA.
__device__ void stats_job(const SacDev& m, const SacArgs& a, const SacWs& w, float alpha, double* red) {
  const float* ws = a.ws;
  const int B = a.B;
  double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int r = threadIdx.x; r < B; r += kThreads) {
    s[0] += ws[w.rows + r];
    s[1] += ws[w.rows + B + r];
    s[2] += ws[w.rows + 2 * (size_t)B + r];
    s[3] += ws[w.logp + B + r];
    s[4] += a.trans[(long long)r * (2 * m.D + m.A + 2) + 2 * m.D + m.A];
  }
  double tot[5];
#pragma unroll
  for (int i = 0; i < 5; ++i) tot[i] = block_sum(s[i], red);
  if (threadIdx.x != 0) return;
  const double mean_logp = tot[3] / B;
  float alpha_loss = 0.0f, alpha_new = alpha;
  if (m.tuning) {
    const float la = *m.log_alpha;
    const double v = mean_logp + (double)m.target_entropy;  // mean(log_pi + target_entropy)
    alpha_loss = (float)(-(double)la * v);
    const AdamStep st = adam_scalars(m.lr, m.beta1, m.beta2, 0.0, m.eps, a.step_a + 1);
    adam_update(m.log_alpha, m.la_m, m.la_v, (float)(-v), st);
    alpha_new = expf(*m.log_alpha);
    *a.alpha = alpha_new;
  }
  a.stats[0] = (float)(tot[0] / B);
  a.stats[1] = (float)(tot[1] / B);
  a.stats[2] = (float)(tot[2] / B);
  a.stats[3] = alpha_loss;
  a.stats[4] = alpha_new;
  a.stats[5] = (float)(tot[4] / B);
  a.stats[6] = (float)(-mean_logp);
  a.stats[7] = 0.0f;
}

// critic_target = critic_target * (1 - tau) + critic * tau, element by element as torch's soft_update rounds it
__device__ __forceinline__ void soft_update(const SacDev& m) {
  const long long stride = (long long)gridDim.x * kThreads;
  const long long t0 = (long long)blockIdx.x * kThreads + threadIdx.x;
  for (int i = 0; i < SAC_CRITIC_PARAMS; ++i) {
    const int l = (i % 6) / 2;
    const long long rows = l == 2 ? 1 : m.H;
    const long long n = i % 2 ? rows : rows * (l == 0 ? m.D + m.A : m.H);
    float* t = m.ct[i];
    const float* p = m.cp[i];
    for (long long e = t0; e < n; e += stride) t[e] = __fadd_rn(__fmul_rn(t[e], m.one_minus_tau), __fmul_rn(p[e], m.tau));
  }
}

__global__ void __launch_bounds__(kThreads, 2) sac_update_kernel(const __grid_constant__ SacDev m,
                                                              const __grid_constant__ SacArgs a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ float Ls[TT][TT + 1], Rs[TT][TT + 1];
  __shared__ double red[kThreads];
  const SacWs w = sac_ws_layout(m, a.B);
  const float alpha = *a.alpha;  // the temperature of this update; written only in the last phase
  for (int ph = 0; ph < kPhases; ++ph) {
    int total = 0;
    for (int g = 0;; ++g) {
      const int n = task_jobs(task(m, a, w, ph, g));
      if (n == 0) break;
      total += n;
    }
    for (int j = blockIdx.x; j < total; j += gridDim.x) {
      int g = 0, jj = j;
      Task t = task(m, a, w, ph, 0);
      for (int n = task_jobs(t); jj >= n; n = task_jobs(t)) {
        jj -= n;
        t = task(m, a, w, ph, ++g);
      }
      if (t.kind == T_ROWQ) rowq_job(m, a, w, alpha, jj);
      else if (t.kind == T_ROWPI) rowpi_job(m, a, w, alpha, jj);
      else if (t.kind == T_STATS) stats_job(m, a, w, alpha, red);
      else mm_job(m, a, w, t, jj, alpha, Ls, Rs);
    }
    if (ph == 8 && a.soft_update) soft_update(m);
    if (ph + 1 < kPhases) grid.sync();
  }
}

}  // namespace

size_t sac_workspace_floats(const SacDev& m, int batch) { return sac_ws_layout(m, batch).total; }

int launch_sac_update(const SacDev& m, const SacArgs& a, cudaStream_t stream) {
  int dev, sms = 0, per_sm = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sac_update_kernel, kThreads, 0));
  if (per_sm < 1) return b200pets_set_error(B200PETS_EUNSUPPORTED, "sac_update_kernel does not fit on an SM");
  SacDev mm = m;
  SacArgs aa = a;
  void* args[] = {&mm, &aa};
  // every CTA co-resident, as the grid-wide barriers require
  const int blocks = sms * (per_sm < kMaxCtasPerSm ? per_sm : kMaxCtasPerSm);
  CUDA_TRY(cudaLaunchCooperativeKernel((void*)sac_update_kernel, dim3(blocks), dim3(kThreads), args, 0, stream));
  return 0;
}
