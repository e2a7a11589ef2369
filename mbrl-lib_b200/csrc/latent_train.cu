// Training PlaNet's latent model (mbrl/models/planet.py:354-519): the recurrence of PlaNetModel.forward and its backward
// pass, each one fp32 FFMA kernel that walks the whole sequence for a tile of rows.  Per step t and row:
//   e   = relu(W_e [s, a_t] + b_e);  h = GRUCell(e, h)      r, z = sigma(.), n = tanh(W_in e + b_in + r * (W_hn h + b_hn))
//   q   = W_q2 relu(W_q1h h + P_t) + b_q2;  s = q[:L] + (softplus(q[L:]) + min_std) * eps_q
//   p   = W_p2 relu(W_p1 h + b_p1) + b_p2;  s_prior = p[:L] + (softplus(p[L:]) + min_std) * eps_p
// The forward kernel is the rollout kernel's structure (latent.cu): state in shared memory, packed transposed weights
// read through L2.  The backward kernel runs t = T-1 .. 0 carrying dh and ds; its W^T dy products read torch's own
// [out][in] tensors down a column, so consecutive threads read consecutive addresses and no copy is needed.  Every sum
// runs in a fixed order.
#include "latent.cuh"

namespace {

enum { kWe, kBe, kWih, kWhh, kBih, kBhh, kWq1, kWq2, kBq2, kWp1, kBp1, kWp2, kBp2 };

// forward: V as the rollout's, G = gates, then a hidden layer [Hf4] and its head's output [2L]
__host__ __device__ inline int fwd_g_stride(const LatentDev& m) { return pad4(max(4 * m.Hb, m.Hf4 + 2 * m.L)); }
__host__ __device__ inline int fwd_row_floats(const LatentDev& m) { return latent_v_stride(m) + fwd_g_stride(m); }
// backward: dh (carried) [Hb4] | ds (carried) [L4] | dh' [Hb4] | de [Hb4] | [da_r, da_z, da_n | pad | dg_hn] | dq | dp |
// du | dv
__host__ __device__ inline int gg_hn(const LatentDev& m) { return pad4(3 * m.Hb); }
__host__ __device__ inline int bwd_row_floats(const LatentDev& m) {
  return 3 * m.Hb4 + m.L4 + gg_hn(m) + m.Hb4 + 2 * pad4(2 * m.L) + 2 * m.Hf4;
}

// acc[r] += sum_{k < K} in[r][k] * W[k][n] for W in torch's [out][in] layout (row k is ldw floats long): W^T dy
template <int R>
__device__ __forceinline__ void dense_t_col(const float* __restrict__ W, int ldw, int K, const float* in, int ld, int n,
                                            float (&acc)[R]) {
  const float* w = W + n;
  int k = 0;
#pragma unroll 2
  for (; k + 4 <= K; k += 4) {
    const float w0 = __ldg(w), w1 = __ldg(w + ldw), w2 = __ldg(w + 2 * ldw), w3 = __ldg(w + 3 * ldw);
    w += 4 * (size_t)ldw;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const float* x = in + r * ld + k;
      acc[r] = fmaf(x[0], w0, acc[r]);
      acc[r] = fmaf(x[1], w1, acc[r]);
      acc[r] = fmaf(x[2], w2, acc[r]);
      acc[r] = fmaf(x[3], w3, acc[r]);
    }
  }
  for (; k < K; ++k) {
    const float wk = __ldg(w);
    w += ldw;
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r] = fmaf(in[r * ld + k], wk, acc[r]);
  }
}

// torch's softplus backward (beta 1, threshold 20)
__device__ __forceinline__ float softplus_backward(float g, float x) {
  if (x > 20.0f) return g;
  const float z = expf(x);
  return g * z / (z + 1.0f);
}

template <int R>
__global__ void __launch_bounds__(kLatentThreads, 1) rssm_seq_forward_kernel(const LatentTrainDev d, const LatentSeqArgs a) {
  extern __shared__ float4 smem4[];
  float* smem = reinterpret_cast<float*>(smem4);
  const LatentDev& m = d.m;
  const int VS = latent_v_stride(m), GS = fwd_g_stride(m);
  float* V = smem;
  float* G = V + R * VS;
  const int oH = m.Hb4, oS = 2 * m.Hb4, oA = 2 * m.Hb4 + m.L4;  // the embedding sits at 0
  const int tid = threadIdx.x;
  const int b0 = blockIdx.x * R;
  const int A = m.A, L = m.L, Hb = m.Hb, Hf = m.Hf, T = a.T, B = a.B;
  const b200pets_latent_tape& tp = a.tape;
  const bool keep = tp.e != nullptr;
  auto at = [&](int r, int t) { return (long long)(b0 + r) * T + t; };  // output row of (b0 + r, t)

  // s0 = 0, h0 = 0 (planet.py:364-367); padding reads as zeros; rows past B run on zeros and store nothing
  for (int i = tid; i < R * (VS + GS); i += kLatentThreads) smem[i] = 0.f;
  __syncthreads();

  // s = mean + (softplus(pre) + min_std) * eps for the head output in G + Hf4; kind 0: posterior (also the next state)
  auto sample = [&](int t, int kind, const float* eps_in, float* params_out, float* samples_out) {
    for (int i = tid; i < R * L; i += kLatentThreads) {
      const int r = i / L, j = i % L;
      const int b = b0 + r;
      const float* q = G + r * GS + m.Hf4;
      float s = 0.f;
      if (b < B) {
        const float e = eps_in ? eps_in[((long long)t * B + b) * L + j]
                               : latent_draw((uint32_t)b, (uint32_t)t, RNG_STREAM_LATENT_TRAIN | ((uint32_t)kind << 15), j,
                                             (uint32_t)a.offset, a.seed);
        const float sd = softplus_f(q[L + j]) + m.min_std;
        s = q[j] + sd * e;
        const long long n = at(r, t);
        params_out[n * 2 * L + j] = q[j];
        params_out[n * 2 * L + L + j] = sd;
        samples_out[n * L + j] = s;
        if (keep) {
          tp.pre_std[n * 2 * L + kind * L + j] = q[L + j];
          tp.eps[n * 2 * L + kind * L + j] = e;
        }
      }
      if (kind == 0) V[r * VS + oS + j] = s;
    }
  };

  for (int t = 0; t < T; ++t) {
    for (int i = tid; i < R * A; i += kLatentThreads) {
      const int r = i / A, j = i % A;
      if (b0 + r < B) V[r * VS + oA + j] = a.act[at(r, t) * A + j];
    }
    __syncthreads();
    dense<R, true>(m.We, m.be, Hb, Hb, m.L4 + m.A4, V + oS, VS, V, VS);
    __syncthreads();
    // GRU pre-activations as in the rollout: [r | z] over [e, h], then W_in e + b_in, W_hn h + b_hn
    for (int j = tid; j < 4 * Hb; j += kLatentThreads) {
      float acc[R];
      const float* W;
      const float* in;
      int N, Kp, n;
      float bn;
      if (j < 2 * Hb) {
        W = m.Wrz; N = 2 * Hb; Kp = 2 * m.Hb4; in = V; n = j; bn = __ldg(m.brz + n);
      } else if (j < 3 * Hb) {
        W = m.Win; N = Hb; Kp = m.Hb4; in = V; n = j - 2 * Hb; bn = __ldg(m.bin + n);
      } else {
        W = m.Whn; N = Hb; Kp = m.Hb4; in = V + oH; n = j - 3 * Hb; bn = __ldg(m.bhn + n);
      }
#pragma unroll
      for (int r = 0; r < R; ++r) acc[r] = bn;
      dense_col<R>(W, N, Kp, in, VS, n, acc);
#pragma unroll
      for (int r = 0; r < R; ++r) G[r * GS + j] = acc[r];
    }
    __syncthreads();
    for (int i = tid; i < R * Hb; i += kLatentThreads) {
      const int r = i / Hb, c = i % Hb;
      const float* g = G + r * GS;
      const float rg = sigmoid_f(g[c]), zg = sigmoid_f(g[Hb + c]);
      const float ng = tanhf(g[2 * Hb + c] + rg * g[3 * Hb + c]);
      float* h = V + r * VS + oH + c;
      const float hn = (1.0f - zg) * ng + zg * *h;
      *h = hn;
      if (b0 + r < B) {
        const long long n = at(r, t);
        a.beliefs[n * Hb + c] = hn;
        if (keep) {
          tp.e[n * Hb + c] = V[r * VS + c];
          float* gt = tp.gates + n * 4 * Hb;
          gt[c] = rg;
          gt[Hb + c] = zg;
          gt[2 * Hb + c] = ng;
          gt[3 * Hb + c] = g[3 * Hb + c];
        }
      }
    }
    __syncthreads();
    // posterior: relu(W_q1h h + P_t) into G[0, Hf4), then its head into G[Hf4, Hf4 + 2L)
    for (int n = tid; n < m.Hf4; n += kLatentThreads) {
      float acc[R];
#pragma unroll
      for (int r = 0; r < R; ++r) acc[r] = (n < Hf && b0 + r < B) ? a.P[at(r, t) * Hf + n] : 0.f;
      if (n < Hf) dense_col<R>(d.Wq1, Hf, m.Hb4, V + oH, VS, n, acc);
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const float v = n < Hf ? fmaxf(acc[r], 0.f) : 0.f;
        G[r * GS + n] = v;
        if (keep && n < Hf && b0 + r < B) tp.q1[at(r, t) * Hf + n] = v;
      }
    }
    __syncthreads();
    dense<R, false>(d.Wq2, d.bq2, 2 * L, 2 * L, m.Hf4, G, GS, G + m.Hf4, GS);
    __syncthreads();
    sample(t, 0, a.eps_q, a.post_params, a.post_samples);
    __syncthreads();
    // prior: relu(W_p1 h + b_p1) into G[0, Hf4), then its head
    dense<R, true>(m.Wp1, m.bp1, Hf, m.Hf4, m.Hb4, V + oH, VS, G, GS);
    __syncthreads();
    if (keep)
      for (int i = tid; i < R * Hf; i += kLatentThreads) {
        const int r = i / Hf, c = i % Hf;
        if (b0 + r < B) tp.p1[at(r, t) * Hf + c] = G[r * GS + c];
      }
    dense<R, false>(m.Wp2, m.bp2, 2 * L, 2 * L, m.Hf4, G, GS, G + m.Hf4, GS);
    __syncthreads();
    sample(t, 1, a.eps_p, a.prior_params, a.prior_samples);
    __syncthreads();
  }
}

template <int R>
__global__ void __launch_bounds__(kLatentThreads, 1) rssm_seq_backward_kernel(const LatentTrainDev d, const LatentSeqArgs a) {
  extern __shared__ float4 smem4[];
  float* D = reinterpret_cast<float*>(smem4);
  const LatentDev& m = d.m;
  const int L = m.L, A = m.A, Hb = m.Hb, Hf = m.Hf, T = a.T, B = a.B, E = d.E;
  const int BS = bwd_row_floats(m), G3 = gg_hn(m);
  const int oDH = 0, oDS = m.Hb4, oDN = m.Hb4 + m.L4, oDE = 2 * m.Hb4 + m.L4, oGG = 3 * m.Hb4 + m.L4;
  const int oDQ = oGG + G3 + m.Hb4, oDP = oDQ + pad4(2 * L), oDU = oDP + pad4(2 * L), oDV = oDU + m.Hf4;
  const int tid = threadIdx.x;
  const int b0 = blockIdx.x * R;
  const b200pets_latent_tape& tp = a.tape;
  const float* const* W = d.src;  // the kernel parameter's own array
  auto at = [&](int r, int t) { return (long long)(b0 + r) * T + t; };

  for (int i = tid; i < R * BS; i += kLatentThreads) D[i] = 0.f;
  __syncthreads();

  for (int t = T - 1; t >= 0; --t) {
    // the reparameterisations and softplus: dq, dp (pre-activations of both heads)
    for (int i = tid; i < R * L; i += kLatentThreads) {
      const int r = i / L, j = i % L;
      if (b0 + r >= B) continue;
      const long long n = at(r, t);
      float* row = D + r * BS;
      const float dsq = (a.g_post_samples ? a.g_post_samples[n * L + j] : 0.f) + row[oDS + j];
      const float dsp = a.g_prior_samples ? a.g_prior_samples[n * L + j] : 0.f;
      const float gqm = a.g_post_params ? a.g_post_params[n * 2 * L + j] : 0.f;
      const float gqs = a.g_post_params ? a.g_post_params[n * 2 * L + L + j] : 0.f;
      const float gpm = a.g_prior_params ? a.g_prior_params[n * 2 * L + j] : 0.f;
      const float gps = a.g_prior_params ? a.g_prior_params[n * 2 * L + L + j] : 0.f;
      const float dqm = gqm + dsq, dpm = gpm + dsp;
      const float dqs = softplus_backward(gqs + dsq * tp.eps[n * 2 * L + j], tp.pre_std[n * 2 * L + j]);
      const float dps = softplus_backward(gps + dsp * tp.eps[n * 2 * L + L + j], tp.pre_std[n * 2 * L + L + j]);
      row[oDQ + j] = dqm;
      row[oDQ + L + j] = dqs;
      row[oDP + j] = dpm;
      row[oDP + L + j] = dps;
      tp.dq[n * 2 * L + j] = dqm;
      tp.dq[n * 2 * L + L + j] = dqs;
      tp.dp[n * 2 * L + j] = dpm;
      tp.dp[n * 2 * L + L + j] = dps;
    }
    __syncthreads();
    // through the heads and the hidden layers' ReLUs: du = (W_q2^T dq) [q1 > 0] (= dP), dv = (W_p2^T dp) [p1 > 0]
    for (int j = tid; j < 2 * Hf; j += kLatentThreads) {
      const bool prior = j >= Hf;
      const int c = prior ? j - Hf : j;
      float acc[R];
#pragma unroll
      for (int r = 0; r < R; ++r) acc[r] = 0.f;
      dense_t_col<R>(W[prior ? kWp2 : kWq2], Hf, 2 * L, D + (prior ? oDP : oDQ), BS, c, acc);
#pragma unroll
      for (int r = 0; r < R; ++r) {
        float v = 0.f;
        if (b0 + r < B) {
          const long long n = at(r, t);
          v = (prior ? tp.p1 : tp.q1)[n * Hf + c] > 0.f ? acc[r] : 0.f;
          if (prior) tp.dv[n * Hf + c] = v;
          else a.dP[n * Hf + c] = v;
        }
        D[r * BS + (prior ? oDV : oDU) + c] = v;
      }
    }
    __syncthreads();
    // dh' = g_belief + dh (from step t + 1) + W_q1h^T du + W_p1^T dv
    for (int c = tid; c < Hb; c += kLatentThreads) {
      float acc[R];
#pragma unroll
      for (int r = 0; r < R; ++r)
        acc[r] = D[r * BS + oDH + c] + ((a.g_beliefs && b0 + r < B) ? a.g_beliefs[at(r, t) * Hb + c] : 0.f);
      dense_t_col<R>(W[kWq1], Hb + E, Hf, D + oDU, BS, c, acc);
      dense_t_col<R>(W[kWp1], Hb, Hf, D + oDV, BS, c, acc);
#pragma unroll
      for (int r = 0; r < R; ++r) D[r * BS + oDN + c] = acc[r];
    }
    __syncthreads();
    // the GRU cell, elementwise: h' = (1 - z) n + z h
    for (int i = tid; i < R * Hb; i += kLatentThreads) {
      const int r = i / Hb, c = i % Hb;
      if (b0 + r >= B) continue;
      const long long n = at(r, t);
      float* row = D + r * BS;
      const float* g = tp.gates + n * 4 * Hb;
      const float rg = g[c], zg = g[Hb + c], ng = g[2 * Hb + c], ghn = g[3 * Hb + c];
      const float hp = t > 0 ? a.beliefs[(n - 1) * Hb + c] : 0.f;
      const float dh = row[oDN + c];
      const float dn = dh * (1.0f - zg), dz = dh * (hp - ng);
      const float dan = dn * (1.0f - ng * ng);
      const float dar = dan * ghn * (rg * (1.0f - rg));
      const float daz = dz * (zg * (1.0f - zg));
      const float dghn = dan * rg;
      row[oGG + c] = dar;
      row[oGG + Hb + c] = daz;
      row[oGG + 2 * Hb + c] = dan;
      row[oGG + G3 + c] = dghn;
      row[oDH + c] = dh * zg;
      tp.dgi[n * 3 * Hb + c] = dar;
      tp.dgi[n * 3 * Hb + Hb + c] = daz;
      tp.dgi[n * 3 * Hb + 2 * Hb + c] = dan;
      tp.dghn[n * Hb + c] = dghn;
    }
    __syncthreads();
    // dh (to step t - 1) += W_hh^T [da_r, da_z, dg_hn];  de = (W_ih^T [da_r, da_z, da_n]) [e > 0]
    for (int j = tid; j < 2 * Hb; j += kLatentThreads) {
      const bool emb = j >= Hb;
      const int c = emb ? j - Hb : j;
      float acc[R];
      if (!emb) {
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r] = D[r * BS + oDH + c];
        dense_t_col<R>(W[kWhh], Hb, 2 * Hb, D + oGG, BS, c, acc);
        dense_t_col<R>(W[kWhh] + (size_t)2 * Hb * Hb, Hb, Hb, D + oGG + G3, BS, c, acc);
#pragma unroll
        for (int r = 0; r < R; ++r) D[r * BS + oDH + c] = acc[r];
      } else {
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r] = 0.f;
        dense_t_col<R>(W[kWih], Hb, 3 * Hb, D + oGG, BS, c, acc);
#pragma unroll
        for (int r = 0; r < R; ++r) {
          float v = 0.f;
          if (b0 + r < B) {
            const long long n = at(r, t);
            v = tp.e[n * Hb + c] > 0.f ? acc[r] : 0.f;
            tp.de[n * Hb + c] = v;
          }
          D[r * BS + oDE + c] = v;
        }
      }
    }
    __syncthreads();
    // ds (to step t - 1) = W_e[:, :L]^T de
    for (int j = tid; j < L; j += kLatentThreads) {
      float acc[R];
#pragma unroll
      for (int r = 0; r < R; ++r) acc[r] = 0.f;
      dense_t_col<R>(W[kWe], L + A, Hb, D + oDE, BS, j, acc);
#pragma unroll
      for (int r = 0; r < R; ++r) D[r * BS + oDS + j] = acc[r];
    }
    __syncthreads();
  }
}

}  // namespace

int latent_train_check(const LatentTrainDev& d, const char* who) {
  const LatentDev& m = d.m;
  if (m.A < 1 || m.L < 1 || m.Hb < 1 || m.Hf < 1 || d.E < 1 || !(m.min_std >= 0.f))
    return b200pets_set_error(B200PETS_EINVAL, "%s: sizes must be positive and min_std non-negative (action %d, latent %d, "
                                               "belief %d, hidden %d, encoding %d, min_std %g)", who, m.A, m.L, m.Hb, m.Hf,
                              d.E, (double)m.min_std);
  int dev = 0, max_smem = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  CUDA_TRY(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const size_t fwd = (size_t)fwd_row_floats(m) * sizeof(float), bwd = (size_t)bwd_row_floats(m) * sizeof(float);
  const size_t limit = (size_t)max_smem / 8;
  if (fwd > limit || bwd > limit)
    return b200pets_set_error(B200PETS_EUNSUPPORTED,
                              "%s: one row of the sequence kernels needs %zu (forward) and %zu (backward) bytes of shared "
                              "memory (action %d, latent %d, belief %d, hidden %d); the limit is %zu bytes, an eighth of "
                              "the %d bytes a CTA can have", who, fwd, bwd, m.A, m.L, m.Hb, m.Hf, limit, max_smem);
  return B200PETS_OK;
}

// blob: We, be, Wrz, brz, Win, bin, Whn, bhn, Wp1, bp1, Wp2, bp2 (LatentDev's layouts), Wq1, Wq2, bq2; 256-byte aligned
static size_t train_sizes(const LatentTrainDev& d, size_t sz[15]) {
  const LatentDev& m = d.m;
  const size_t s[15] = {(size_t)(m.L4 + m.A4) * m.Hb, (size_t)m.Hb, (size_t)2 * m.Hb4 * 2 * m.Hb, (size_t)2 * m.Hb,
                        (size_t)m.Hb4 * m.Hb, (size_t)m.Hb, (size_t)m.Hb4 * m.Hb, (size_t)m.Hb, (size_t)m.Hb4 * m.Hf,
                        (size_t)m.Hf, (size_t)m.Hf4 * 2 * m.L, (size_t)2 * m.L, (size_t)m.Hb4 * m.Hf,
                        (size_t)m.Hf4 * 2 * m.L, (size_t)2 * m.L};
  size_t tot = 0;
  for (int i = 0; i < 15; ++i) {
    sz[i] = s[i];
    tot += (s[i] + 63) & ~(size_t)63;
  }
  return tot;
}

size_t latent_train_blob_floats(const LatentTrainDev& d) {
  size_t sz[15];
  return train_sizes(d, sz);
}

int latent_train_stage(LatentTrainDev* d, float* blob, cudaStream_t stream) {
  LatentDev& m = d->m;
  size_t sz[15];
  train_sizes(*d, sz);
  const float** f[15] = {&m.We, &m.be, &m.Wrz, &m.brz, &m.Win, &m.bin, &m.Whn, &m.bhn,
                         &m.Wp1, &m.bp1, &m.Wp2, &m.bp2, &d->Wq1, &d->Wq2, &d->bq2};
  size_t off = 0;
  for (int i = 0; i < 15; ++i) {
    *f[i] = blob + off;
    off += (sz[i] + 63) & ~(size_t)63;
  }
  const int L = m.L, A = m.A, Hb = m.Hb, Hf = m.Hf;
  const float* const* p = d->src;
  // as latent_stage packs the same modules (latent.cu), plus the posterior's belief columns and its head
  auto pack = [&](const float* dst, int Kp, int N, const float* s0, int ld0, int n0, int row_off) {
    latent_pack(const_cast<float*>(dst), Kp, N, s0, ld0, 0, n0, nullptr, 0, 0, 0, 0, row_off, stream);
  };
  auto bias = [&](const float* dst, int N, const float* b0, const float* b1, int off_) {
    latent_pack_bias(const_cast<float*>(dst), N, b0, b1, off_, stream);
  };
  latent_pack(const_cast<float*>(m.We), m.L4 + m.A4, Hb, p[kWe], L + A, 0, L, p[kWe], L + A, L, A, m.L4, 0, stream);
  bias(m.be, Hb, p[kBe], nullptr, 0);
  latent_pack(const_cast<float*>(m.Wrz), 2 * m.Hb4, 2 * Hb, p[kWih], Hb, 0, Hb, p[kWhh], Hb, 0, Hb, m.Hb4, 0, stream);
  bias(m.brz, 2 * Hb, p[kBih], p[kBhh], 0);
  pack(m.Win, m.Hb4, Hb, p[kWih], Hb, Hb, 2 * Hb);
  bias(m.bin, Hb, p[kBih], nullptr, 2 * Hb);
  pack(m.Whn, m.Hb4, Hb, p[kWhh], Hb, Hb, 2 * Hb);
  bias(m.bhn, Hb, p[kBhh], nullptr, 2 * Hb);
  pack(m.Wp1, m.Hb4, Hf, p[kWp1], Hb, Hb, 0);
  bias(m.bp1, Hf, p[kBp1], nullptr, 0);
  pack(m.Wp2, m.Hf4, 2 * L, p[kWp2], Hf, Hf, 0);
  bias(m.bp2, 2 * L, p[kBp2], nullptr, 0);
  pack(d->Wq1, m.Hb4, Hf, p[kWq1], Hb + d->E, Hb, 0);
  pack(d->Wq2, m.Hf4, 2 * L, p[kWq2], Hf, Hf, 0);
  bias(d->bq2, 2 * L, p[kBq2], nullptr, 0);
  CUDA_TRY(cudaGetLastError());
  return B200PETS_OK;
}

template <int R, bool FWD>
static int launch_seq(const LatentTrainDev& d, const LatentSeqArgs& a, size_t smem, int ctas, cudaStream_t stream) {
  auto kern = FWD ? rssm_seq_forward_kernel<R> : rssm_seq_backward_kernel<R>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<(unsigned)ctas, kLatentThreads, smem, stream>>>(d, a);
  CUDA_TRY(cudaGetLastError());
  return B200PETS_OK;
}

// Rows per CTA as latent_plan picks them: enough CTAs to cover the SMs once (at most 32 rows), halved while the tile
// does not fit in shared memory
template <bool FWD>
static int launch(const LatentTrainDev& d, const LatentSeqArgs& a, cudaStream_t stream) {
  if (int rc = latent_train_check(d, FWD ? "latent_seq_forward" : "latent_seq_backward")) return rc;
  int dev = 0, max_smem = 0, sms = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  CUDA_TRY(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const size_t row_bytes = (size_t)(FWD ? fwd_row_floats(d.m) : bwd_row_floats(d.m)) * sizeof(float);
  const int want = (a.B + sms - 1) / sms;
  int R = 1;
  while (R < want && R < 32) R *= 2;
  while (R > 1 && (size_t)R * row_bytes > (size_t)max_smem) R /= 2;
  const int ctas = (a.B + R - 1) / R;
  const size_t smem = ((size_t)R * row_bytes + 15) & ~(size_t)15;
  switch (R) {
    case 1: return launch_seq<1, FWD>(d, a, smem, ctas, stream);
    case 2: return launch_seq<2, FWD>(d, a, smem, ctas, stream);
    case 4: return launch_seq<4, FWD>(d, a, smem, ctas, stream);
    case 8: return launch_seq<8, FWD>(d, a, smem, ctas, stream);
    case 16: return launch_seq<16, FWD>(d, a, smem, ctas, stream);
    default: return launch_seq<32, FWD>(d, a, smem, ctas, stream);
  }
}

int launch_latent_seq_forward(const LatentTrainDev& d, const LatentSeqArgs& a, cudaStream_t stream) {
  return launch<true>(d, a, stream);
}

int launch_latent_seq_backward(const LatentTrainDev& d, const LatentSeqArgs& a, cudaStream_t stream) {
  return launch<false>(d, a, stream);
}
