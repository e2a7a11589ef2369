// PlaNet's latent model on the device (mbrl/models/planet.py:82-114, 231-264, 289-306, 531-581): one fp32 FFMA kernel
// runs a whole horizon for a tile of rows.  Per step and row:
//   e   = relu(W_e [s, a] + b_e)
//   h'  = GRUCell(e, h)                      r, z = sigma(.), n = tanh(W_in e + b_in + r * (W_hn h + b_hn))
//   p   = W_p2 relu(W_p1 h' + b_p1) + b_p2;  s' = p[:L] + (softplus(p[L:]) + min_std) * eps   (s' = p[:L] without a draw)
//   rew = W_r3 relu(W_r2 relu(W_r1 [h', s'] + b_r1) + b_r2) + b_r3
// Belief, latent, action, gates and hidden activations of the tile stay in shared memory; the weights are read through
// L2 (1.55 MB at PlaNet's sizes), each weight load feeding one FMA per row of the tile.
#include "latent.cuh"

namespace {

// The kernels' body.  BATCH: K problems in one launch (LatentBatch): CTA j runs local tile j % bt->tiles of problem
// j / bt->tiles, and everything after that decode is the single-problem code.
template <int R, bool BATCH>
__device__ __forceinline__ void latent_rollout_body(const LatentDev& m, const LatentArgs& a, const LatentBatch* bt) {
  extern __shared__ float4 smem4[];
  float* smem = reinterpret_cast<float*>(smem4);
  const int VS = latent_v_stride(m), GS = latent_g_stride(m);
  float* V = smem;
  float* G = V + R * VS;
  float* T = G + R * GS;
  const int oH = m.Hb4, oS = 2 * m.Hb4, oA = 2 * m.Hb4 + m.L4;  // the embedding sits at 0
  const int tid = threadIdx.x;
  long long kp = 0;  // problem of a batched launch
  long long row0 = (long long)blockIdx.x * R;
  if constexpr (BATCH) { kp = blockIdx.x / bt->tiles; row0 = (blockIdx.x - kp * bt->tiles) * R; }
  const int A = m.A, L = m.L, Hb = m.Hb, Hf = m.Hf;

  // padding must read as zeros (it meets zero weight rows); rows past B run on zeros and store nothing
  for (int i = tid; i < R * (VS + GS + 1); i += kLatentThreads) smem[i] = 0.f;
  __syncthreads();
  for (int i = tid; i < R * Hb; i += kLatentThreads) {
    const int r = i / Hb, c = i % Hb;
    const long long row = row0 + r;
    if (row < a.B)
      V[r * VS + oH + c] = a.belief0 ? (a.belief0 + prob_off<BATCH>(bt, kp, &LatentBatch::belief0))[c] : a.belief_in[row * Hb + c];
  }
  for (int i = tid; i < R * L; i += kLatentThreads) {
    const int r = i / L, c = i % L;
    const long long row = row0 + r;
    if (row < a.B)
      V[r * VS + oS + c] = a.latent0 ? (a.latent0 + prob_off<BATCH>(bt, kp, &LatentBatch::latent0))[c] : a.latent_in[row * L + c];
  }
  auto load_actions = [&](int t) {
    for (int i = tid; i < R * A; i += kLatentThreads) {
      const int r = i / A, j = i % A;
      const long long row = row0 + r;
      if (row < a.B)
        V[r * VS + oA + j] = (a.act + prob_off<BATCH>(bt, kp, &LatentBatch::act))[(row / a.P) * (long long)a.H * A + (long long)t * A + j];
    }
  };
  load_actions(0);
  __syncthreads();

  for (int t = 0; t < a.H; ++t) {
    // embedding of [s, a]
    dense<R, true>(m.We, m.be, Hb, Hb, m.L4 + m.A4, V + oS, VS, V, VS);
    __syncthreads();
    // GRU pre-activations: [r | z] over [e, h] (input and hidden sums in one), then W_in e + b_in, W_hn h + b_hn
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
    // h' = (1 - z) n + z h, in place
    for (int i = tid; i < R * Hb; i += kLatentThreads) {
      const int r = i / Hb, c = i % Hb;
      const float* g = G + r * GS;
      const float rg = sigmoid_f(g[c]), zg = sigmoid_f(g[Hb + c]);
      const float ng = tanhf(g[2 * Hb + c] + rg * g[3 * Hb + c]);
      float* h = V + r * VS + oH + c;
      *h = (1.0f - zg) * ng + zg * *h;
    }
    __syncthreads();
    // prior: hidden layer into G[0, Hf4), mean and pre-softplus std into G[Hf4, Hf4 + 2L)
    dense<R, true>(m.Wp1, m.bp1, Hf, m.Hf4, m.Hb4, V + oH, VS, G, GS);
    __syncthreads();
    dense<R, false>(m.Wp2, m.bp2, 2 * L, 2 * L, m.Hf4, G, GS, G + m.Hf4, GS);
    __syncthreads();
    // s' = mean + std * eps
    for (int i = tid; i < R * L; i += kLatentThreads) {
      const int r = i / L, j = i % L;
      const long long row = row0 + r;
      const float* p = G + r * GS + m.Hf4;
      float s = p[j];
      if (a.sample && row < a.B) {
        float e;
        if (a.eps) {
          e = (a.eps + prob_off<BATCH>(bt, kp, &LatentBatch::eps))[((long long)t * a.B + row) * L + j];
        } else {
          e = latent_draw((uint32_t)row, (uint32_t)t, RNG_STREAM_LATENT, j, (uint32_t)prob_offset<BATCH>(a, bt, kp),
                          prob_seed<BATCH>(a, bt, kp));
        }
        const float sd = softplus_f(p[L + j]) + m.min_std;
        s = s + sd * e;
      }
      V[r * VS + oS + j] = s;
    }
    __syncthreads();
    // reward head over [h', s']: G[0, Hf4) then G[Hf4, 2 Hf4), then one dot product per row
    dense<R, true>(m.Wr1, m.br1, Hf, m.Hf4, m.Hb4 + m.L4, V + oH, VS, G, GS);
    __syncthreads();
    dense<R, true>(m.Wr2, m.br2, Hf, m.Hf4, m.Hf4, G, GS, G + m.Hf4, GS);
    __syncthreads();
    const int warp = tid >> 5, lane = tid & 31;
    for (int r = warp; r < R; r += kLatentThreads / 32) {
      const float* x = G + r * GS + m.Hf4;
      float s = 0.f;
      for (int k = lane; k < Hf; k += 32) s = fmaf(x[k], __ldg(m.wr3 + k), s);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) {
        const float rew = s + __ldg(m.br3);
        T[r] += rew;  // no termination: every step counts (model_env.py:183-188 with no_termination)
        const long long row = row0 + r;
        if (a.reward_out && t == a.H - 1 && row < a.B) a.reward_out[row] = rew;
      }
    }
    if (t + 1 < a.H) load_actions(t + 1);
    __syncthreads();
  }

  float* totals = a.totals;
  if constexpr (BATCH) totals += prob_off<BATCH>(bt, kp, &LatentBatch::rows);
  for (int r = tid; r < R; r += kLatentThreads) {
    const long long row = row0 + r;
    if (totals && row < a.B) totals[row] = T[r];
  }
  if (a.latent_out)
    for (int i = tid; i < R * L; i += kLatentThreads) {
      const int r = i / L, c = i % L;
      const long long row = row0 + r;
      if (row < a.B) a.latent_out[row * L + c] = V[r * VS + oS + c];
    }
  if (a.belief_out)
    for (int i = tid; i < R * Hb; i += kLatentThreads) {
      const int r = i / Hb, c = i % Hb;
      const long long row = row0 + r;
      if (row < a.B) a.belief_out[row * Hb + c] = V[r * VS + oH + c];
    }
}

template <int R>
__global__ void __launch_bounds__(kLatentThreads, 1) latent_rollout_kernel(const LatentDev m, const LatentArgs a) {
  latent_rollout_body<R, false>(m, a, nullptr);
}

// K independent evaluations in one launch
template <int R>
__global__ void __launch_bounds__(kLatentThreads, 1)
    latent_rollout_batch_kernel(const __grid_constant__ LatentDev m, const __grid_constant__ LatentArgs a,
                                const __grid_constant__ LatentBatch bt) {
  latent_rollout_body<R, true>(m, a, &bt);
}

// dst[kp][n] (Kp x N) from torch's [out, in] weights: row kp < n0 is input column coff0 + kp of src0, rows
// row1 .. row1 + n1 - 1 are input columns coff1 .. of src1, every other row is zero; output column n is source row
// row_off + n
__global__ void latent_pack_kernel(float* __restrict__ dst, int Kp, int N, const float* __restrict__ src0, int ld0,
                                   int coff0, int n0, const float* __restrict__ src1, int ld1, int coff1, int n1, int row1,
                                   int row_off) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)Kp * N) return;
  const int kp = (int)(idx / N), n = (int)(idx % N);
  float v = 0.f;
  if (kp < n0) v = src0[(long long)(row_off + n) * ld0 + coff0 + kp];
  else if (src1 && kp >= row1 && kp < row1 + n1) v = src1[(long long)(row_off + n) * ld1 + coff1 + (kp - row1)];
  dst[idx] = v;
}

__global__ void latent_bias_kernel(float* __restrict__ dst, int N, const float* __restrict__ b0, const float* __restrict__ b1,
                                   int off) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  dst[n] = b1 ? b0[off + n] + b1[off + n] : b0[off + n];
}

// The last kernel of a staging call, as in api.cu: a plain kernel boundary between the packing and any rollout.
__global__ void latent_staging_fence_kernel() {}

}  // namespace

// blob: the 18 arrays of LatentDev back to back, each 256-byte aligned
static size_t latent_sizes(const LatentDev& m, size_t sz[18]) {
  const int A4 = m.A4, L4 = m.L4, Hb = m.Hb, Hb4 = m.Hb4, Hf = m.Hf, Hf4 = m.Hf4, L = m.L;
  const size_t s[18] = {(size_t)(L4 + A4) * Hb, (size_t)Hb, (size_t)2 * Hb4 * 2 * Hb, (size_t)2 * Hb, (size_t)Hb4 * Hb,
                        (size_t)Hb, (size_t)Hb4 * Hb, (size_t)Hb, (size_t)Hb4 * Hf, (size_t)Hf, (size_t)Hf4 * 2 * L,
                        (size_t)2 * L, (size_t)(Hb4 + L4) * Hf, (size_t)Hf, (size_t)Hf4 * Hf, (size_t)Hf, (size_t)Hf4, 1};
  size_t tot = 0;
  for (int i = 0; i < 18; ++i) {
    sz[i] = s[i];
    tot += (s[i] + 63) & ~(size_t)63;
  }
  return tot;
}

size_t latent_blob_floats(const LatentDev& m) {
  size_t sz[18];
  return latent_sizes(m, sz);
}

void latent_bind(LatentDev* m, float* blob) {
  size_t sz[18];
  latent_sizes(*m, sz);
  const float** f[18] = {&m->We, &m->be, &m->Wrz, &m->brz, &m->Win, &m->bin, &m->Whn, &m->bhn, &m->Wp1,
                         &m->bp1, &m->Wp2, &m->bp2, &m->Wr1, &m->br1, &m->Wr2, &m->br2, &m->wr3, &m->br3};
  size_t off = 0;
  for (int i = 0; i < 18; ++i) {
    *f[i] = blob + off;
    off += (sz[i] + 63) & ~(size_t)63;
  }
}

void latent_pack(float* dst, int Kp, int N, const float* src0, int ld0, int coff0, int n0, const float* src1, int ld1,
                 int coff1, int n1, int row1, int row_off, cudaStream_t stream) {
  const long long tot = (long long)Kp * N;
  latent_pack_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(dst, Kp, N, src0, ld0, coff0, n0, src1, ld1, coff1,
                                                                       n1, row1, row_off);
}

void latent_pack_bias(float* dst, int N, const float* b0, const float* b1, int off, cudaStream_t stream) {
  latent_bias_kernel<<<(N + 255) / 256, 256, 0, stream>>>(dst, N, b0, b1, off);
}

// params: the B200PETS_LATENT_NUM_PARAMS torch tensors in the order of include/b200pets.h
int latent_stage(const LatentDev& m, const float* const* params, cudaStream_t stream) {
  const int L = m.L, A = m.A, Hb = m.Hb, Hf = m.Hf;
  auto pack = [&](const float* dst, int Kp, int N, const float* s0, int ld0, int c0, int n0, const float* s1, int ld1, int c1,
                  int n1, int row1, int row_off) {
    latent_pack(const_cast<float*>(dst), Kp, N, s0, ld0, c0, n0, s1, ld1, c1, n1, row1, row_off, stream);
  };
  auto bias = [&](const float* dst, int N, const float* b0, const float* b1, int off) {
    latent_pack_bias(const_cast<float*>(dst), N, b0, b1, off, stream);
  };
  const float *We = params[0], *be = params[1], *Wih = params[2], *Whh = params[3], *bih = params[4], *bhh = params[5];
  pack(m.We, m.L4 + m.A4, Hb, We, L + A, 0, L, We, L + A, L, A, m.L4, 0);
  bias(m.be, Hb, be, nullptr, 0);
  pack(m.Wrz, 2 * m.Hb4, 2 * Hb, Wih, Hb, 0, Hb, Whh, Hb, 0, Hb, m.Hb4, 0);
  bias(m.brz, 2 * Hb, bih, bhh, 0);
  pack(m.Win, m.Hb4, Hb, Wih, Hb, 0, Hb, nullptr, 0, 0, 0, 0, 2 * Hb);
  bias(m.bin, Hb, bih, nullptr, 2 * Hb);
  pack(m.Whn, m.Hb4, Hb, Whh, Hb, 0, Hb, nullptr, 0, 0, 0, 0, 2 * Hb);
  bias(m.bhn, Hb, bhh, nullptr, 2 * Hb);
  pack(m.Wp1, m.Hb4, Hf, params[6], Hb, 0, Hb, nullptr, 0, 0, 0, 0, 0);
  bias(m.bp1, Hf, params[7], nullptr, 0);
  pack(m.Wp2, m.Hf4, 2 * L, params[8], Hf, 0, Hf, nullptr, 0, 0, 0, 0, 0);
  bias(m.bp2, 2 * L, params[9], nullptr, 0);
  pack(m.Wr1, m.Hb4 + m.L4, Hf, params[10], Hb + L, 0, Hb, params[10], Hb + L, Hb, L, m.Hb4, 0);
  bias(m.br1, Hf, params[11], nullptr, 0);
  pack(m.Wr2, m.Hf4, Hf, params[12], Hf, 0, Hf, nullptr, 0, 0, 0, 0, 0);
  bias(m.br2, Hf, params[13], nullptr, 0);
  pack(m.wr3, m.Hf4, 1, params[14], Hf, 0, Hf, nullptr, 0, 0, 0, 0, 0);
  bias(m.br3, 1, params[15], nullptr, 0);
  latent_staging_fence_kernel<<<1, 1, 0, stream>>>();
  CUDA_TRY(cudaGetLastError());
  return B200PETS_OK;
}

int latent_tile(size_t row_bytes, long long rows, LatentPlan* p) {
  int dev = 0, max_smem = 0, sms = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  CUDA_TRY(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const long long want = rows > 0 ? (rows + sms - 1) / sms : 1;
  int R = 1;
  while (R < want && R < 32) R *= 2;
  while (R > 1 && (size_t)R * row_bytes > (size_t)max_smem) R /= 2;
  p->rows = R;
  p->ctas = rows > 0 ? (rows + R - 1) / R : 0;
  p->smem = ((size_t)R * row_bytes + 15) & ~(size_t)15;
  p->row_bytes = row_bytes;
  p->row_limit = (size_t)max_smem / 8;
  return B200PETS_OK;
}

// The rollout's tile.  A model is refused when a row needs more than an eighth of the opt-in shared memory, so that the
// 8-row tile a 1000-row population takes on an H100 always fits.
int latent_plan(const LatentDev& m, long long rows, LatentPlan* p) {
  if (int rc = latent_tile((size_t)(latent_v_stride(m) + latent_g_stride(m) + 1) * sizeof(float), rows, p)) return rc;
  if (p->row_bytes > p->row_limit)
    return b200pets_set_error(B200PETS_EUNSUPPORTED,
                              "latent model: one row needs %zu bytes of shared memory (belief %d, hidden %d, latent %d, action "
                              "%d); the limit is %zu bytes, an eighth of the shared memory a CTA can have",
                              p->row_bytes, m.Hb, m.Hf, m.L, m.A, p->row_limit);
  return B200PETS_OK;
}

template <int R>
static int launch_rows(const LatentDev& m, const LatentArgs& a, const LatentPlan& p, int num_problems, LatentBatch bt,
                       cudaStream_t stream) {
  if (num_problems == 1) {
    CUDA_TRY(cudaFuncSetAttribute(latent_rollout_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
    latent_rollout_kernel<R><<<(unsigned)p.ctas, kLatentThreads, p.smem, stream>>>(m, a);
  } else {
    bt.tiles = (a.B + R - 1) / R;
    CUDA_TRY(cudaFuncSetAttribute(latent_rollout_batch_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
    latent_rollout_batch_kernel<R><<<(unsigned)(bt.tiles * num_problems), kLatentThreads, p.smem, stream>>>(m, a, bt);
  }
  CUDA_TRY(cudaGetLastError());
  return B200PETS_OK;
}

int launch_latent_rollout(const LatentDev& m, const LatentArgs& a, int num_problems, LatentBatch bt, cudaStream_t stream) {
  if (num_problems > 1 && (!a.latent0 || !a.belief0 || a.latent_out || a.belief_out || a.reward_out))
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "batched latent rollout: evaluations from a posterior only");
  LatentPlan p;
  int rc = latent_plan(m, (long long)num_problems * a.B, &p);
  if (rc) return rc;
  if (p.ctas == 0) return B200PETS_OK;
  switch (p.rows) {
    case 1: return launch_rows<1>(m, a, p, num_problems, bt, stream);
    case 2: return launch_rows<2>(m, a, p, num_problems, bt, stream);
    case 4: return launch_rows<4>(m, a, p, num_problems, bt, stream);
    case 8: return launch_rows<8>(m, a, p, num_problems, bt, stream);
    case 16: return launch_rows<16>(m, a, p, num_problems, bt, stream);
    default: return launch_rows<32>(m, a, p, num_problems, bt, stream);
  }
}
