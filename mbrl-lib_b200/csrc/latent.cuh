// The latent model of PlaNet (mbrl/models/planet.py) as the rollout kernel of latent.cu reads it.
#pragma once
#include "common.cuh"

// Staged copy: every nn.Linear / nn.GRUCell weight transposed to [K][N] (torch stores [out, in]), with K padded to a
// multiple of 4 by zero rows so that the kernel reads its inputs as float4.  The kernel's per-row input buffers use
// the same padding, so a concatenated input ([latent, action], [belief, latent]) is two padded segments.
struct LatentDev {
  int A, L, Hb, Hf;         // action, latent, belief, hidden sizes
  int A4, L4, Hb4, Hf4;     // the same rounded up to multiples of 4
  float min_std;
  const float *We, *be;     // embedding       [L4 + A4][Hb]  rows: latent, then action
  const float *Wrz, *brz;   // GRU r and z     [2 Hb4][2 Hb]  rows: embedding, then belief; bias b_ih + b_hh
  const float *Win, *bin;   // GRU n, input    [Hb4][Hb]
  const float *Whn, *bhn;   // GRU n, hidden   [Hb4][Hb]
  const float *Wp1, *bp1;   // prior layer 1   [Hb4][Hf]
  const float *Wp2, *bp2;   // prior layer 2   [Hf4][2 L]     columns: mean, then pre-softplus std
  const float *Wr1, *br1;   // reward layer 1  [Hb4 + L4][Hf] rows: belief, then latent
  const float *Wr2, *br2;   // reward layer 2  [Hf4][Hf]
  const float *wr3, *br3;   // reward layer 3  [Hf4], [1]
};

// One launch of the latent rollout: steps 0 .. H-1 of B rows (row r = n * P + p reads the actions of sequence n).
struct LatentArgs {
  long long B;
  int H, P;
  const float* latent0;     // [L] start of every row (the posterior), or NULL: latent_in [B][L]
  const float* belief0;     // [Hb] or NULL: belief_in [B][Hb]
  const float* latent_in;
  const float* belief_in;
  const float* act;         // row r, step t reads act[(r / P) * H * A + t * A ..]
  const float* eps;         // [H][B][L] injected N(0,1) draws, or NULL: Philox (RNG_STREAM_LATENT)
  int sample;               // 0: the prior's mean (deterministic=True)
  unsigned long long seed;  // Philox key (already through rng_key)
  unsigned long long offset;
  float* totals;            // [B] summed rewards, or NULL
  float* latent_out;        // [B][L] state after the last step, or NULL
  float* belief_out;        // [B][Hb] or NULL
  float* reward_out;        // [B] reward of the last step, or NULL
};

// A batched launch of the rollout: K evaluations of one LatentArgs in one grid (a.B rows each).  Tiles are
// problem-major (tile = k * tiles + local tile), so no tile holds two problems.  Problem k starts from
// latent0 + k * latent0 and belief0 + k * belief0, reads act + k * act and eps + k * eps, writes totals + k * rows and
// draws with Philox offset a.offset + k * offset_step under key rng_key(seed, that offset) (common.cuh prob_offset /
// prob_seed).  Its rows do exactly what they do in a single launch.
struct LatentBatch {
  long long tiles;          // tiles of one problem
  long long latent0, belief0, act, eps, rows;
  unsigned long long seed;  // unkeyed
  unsigned long long offset_step;
};

// Rows per CTA and shared memory, chosen from the row count and the device (launcher and b200pets_latent_plan_info).
struct LatentPlan {
  int rows;          // rows per CTA: 1, 2, 4, 8, 16 or 32
  long long ctas;
  size_t smem;       // dynamic shared memory of one CTA
  size_t row_bytes;  // shared memory one row needs
  size_t row_limit;  // the most a row may need: an 8-row tile must fit in the opt-in shared memory
};

// Device helpers shared by the rollout kernel (latent.cu) and the sequence kernels of training (latent_train.cu).
namespace {

constexpr int kLatentThreads = 256;

__host__ __device__ inline int pad4(int x) { return (x + 3) & ~3; }

// per-row shared memory (floats): V = [embedding | belief | latent | action], G = gates / hidden activations, total
__host__ __device__ inline int latent_v_stride(const LatentDev& m) { return 2 * m.Hb4 + m.L4 + m.A4; }
__host__ __device__ inline int latent_g_stride(const LatentDev& m) {
  return pad4(max(4 * m.Hb, max(m.Hf4 + 2 * m.L, 2 * m.Hf4)));
}

// acc[r] += sum_k in[r][k] * W[k][n] over k < Kp (a multiple of 4); in rows are ld floats apart
template <int R>
__device__ __forceinline__ void dense_col(const float* __restrict__ W, int N, int Kp, const float* in, int ld, int n,
                                          float (&acc)[R]) {
  const float* w = W + n;
#pragma unroll 2
  for (int k = 0; k < Kp; k += 4) {
    const float w0 = __ldg(w), w1 = __ldg(w + N), w2 = __ldg(w + 2 * N), w3 = __ldg(w + 3 * N);
    w += 4 * (size_t)N;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const float4 x = *reinterpret_cast<const float4*>(in + r * ld + k);
      acc[r] = fmaf(x.x, w0, acc[r]);
      acc[r] = fmaf(x.y, w1, acc[r]);
      acc[r] = fmaf(x.z, w2, acc[r]);
      acc[r] = fmaf(x.w, w3, acc[r]);
    }
  }
}

// out[r][n] = act(W[:, n] . in[r] + b[n]) for n < N4 (columns N .. N4-1 are written as zeros: they are the padding the
// next layer reads)
template <int R, bool RELU>
__device__ __forceinline__ void dense(const float* __restrict__ W, const float* __restrict__ b, int N, int N4, int Kp,
                                      const float* in, int ld_in, float* out, int ld_out) {
  for (int n = threadIdx.x; n < N4; n += kLatentThreads) {
    float acc[R];
    const float bn = n < N ? __ldg(b + n) : 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r] = bn;
    if (n < N) dense_col<R>(W, N, Kp, in, ld_in, n, acc);
#pragma unroll
    for (int r = 0; r < R; ++r) out[r * ld_out + n] = n < N ? (RELU ? fmaxf(acc[r], 0.f) : acc[r]) : 0.f;
  }
}

__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }

// Lane j & 3 of philox_normal4v at counter (row, t, stream | (j >> 2), offset) (common.cuh), computed inline: only the
// Box-Muller pair the lane belongs to, with the same operations, so the value is that of philox_normal4v
__device__ __forceinline__ float latent_draw(uint32_t row, uint32_t t, uint32_t stream, int j, uint32_t offset,
                                             unsigned long long key) {
  const U4 q = philox4x32_10(row, t, stream | (uint32_t)(j >> 2), offset, (uint32_t)key, (uint32_t)(key >> 32));
  const int lane = j & 3;
  const float ur = u32_to_unit(lane < 2 ? q.x : q.z), ua = u32_to_unit(lane < 2 ? q.y : q.w);
  const float rad = sqrtf(-2.0f * __logf(ur));
  float sn, cs;
  __sincosf(6.283185307179586f * ua, &sn, &cs);
  return rad * ((lane & 1) ? sn : cs);
}

}  // namespace

size_t latent_blob_floats(const LatentDev& m);  // m: sizes set
void latent_bind(LatentDev* m, float* blob);     // points the weight fields into blob
int latent_stage(const LatentDev& m, const float* const* params, cudaStream_t stream);
// The staging kernels on `stream`: dst[kp][n] (Kp x N) from torch's [out, in] weights -- row kp < n0 is input column
// coff0 + kp of src0, rows row1 .. row1 + n1 - 1 are input columns coff1 .. of src1, every other row is zero, output
// column n is source row row_off + n -- and dst[n] = b0[off + n] (+ b1[off + n])
void latent_pack(float* dst, int Kp, int N, const float* src0, int ld0, int coff0, int n0, const float* src1, int ld1,
                 int coff1, int n1, int row1, int row_off, cudaStream_t stream);
void latent_pack_bias(float* dst, int N, const float* b0, const float* b1, int off, cudaStream_t stream);
// The tile rule of every latent kernel (the rollout's and training's two): for `rows` rows of `row_bytes` bytes of
// shared memory each on the current device, enough CTAs to cover the SMs once (the smallest power of two >= rows / SMs,
// at most 32 rows), halved while the tile does not fit in the opt-in shared memory.  Sets every field of *p; rows < 1
// gives one row per CTA and no CTAs.
int latent_tile(size_t row_bytes, long long rows, LatentPlan* p);
int latent_plan(const LatentDev& m, long long rows, LatentPlan* p);
// `num_problems` copies of the launch `a` describes in one grid whose tile comes from latent_plan over all
// num_problems * a.B rows.  One problem runs latent_rollout_kernel and ignores bt; more (totals only, latent0 / belief0
// set) run latent_rollout_batch_kernel with bt's per-problem strides (bt.tiles is set here).
int launch_latent_rollout(const LatentDev& m, const LatentArgs& a, int num_problems, LatentBatch bt, cudaStream_t stream);

// ---- Training's sequence kernels (latent_train.cu): the RSSM of PlaNetModel.forward (planet.py:354-404) ------------
// The forward kernel reads packed transposed copies like the rollout's (LatentDev's embedding, GRU and prior fields; the
// reward fields are not read) plus the posterior's; the backward kernel reads torch's own [out][in] tensors.
struct LatentTrainDev {
  LatentDev m;
  int E;                              // encoding size: posterior_transition_model[0] takes [belief, encoding]
  const float *Wq1, *Wq2, *bq2;       // posterior layer 1, belief columns [Hb4][Hf]; layer 2 [Hf4][2 L], [2 L]
  const float* src[B200PETS_LATENT_TRAIN_NUM_PARAMS];  // torch's tensors (include/b200pets.h), by value: kernels read them
};

struct LatentSeqArgs {
  int B, T;
  const float* P;                     // [B][T][Hf]: W_q1e enc + b_q1
  const float* act;                   // [B][T][A]
  const float *eps_q, *eps_p;         // [T][B][L] injected draws, or NULL: Philox (RNG_STREAM_LATENT_TRAIN)
  unsigned long long seed, offset;    // Philox key (already through rng_key) and counter word
  float *beliefs, *post_params, *post_samples, *prior_params, *prior_samples;  // [B][T][Hb | 2L | L | 2L | L]
  const float *g_beliefs, *g_post_params, *g_post_samples, *g_prior_params, *g_prior_samples;  // or NULL = 0
  float* dP;                          // [B][T][Hf]
  b200pets_latent_tape tape;
};

// 0 when the kernels cover the sizes; B200PETS_EINVAL / B200PETS_EUNSUPPORTED (with the error message set) otherwise
int latent_train_check(const LatentTrainDev& d, const char* who);
size_t latent_train_blob_floats(const LatentTrainDev& d);
int latent_train_stage(LatentTrainDev* d, float* blob, cudaStream_t stream);  // binds the packed fields into blob
// The launch of the forward (or the backward) kernel for `batch` rows: latent_train_check, then latent_tile
int latent_train_plan(const LatentTrainDev& d, int batch, bool forward, const char* who, LatentPlan* p);
int launch_latent_seq_forward(const LatentTrainDev& d, const LatentSeqArgs& a, cudaStream_t stream);
int launch_latent_seq_backward(const LatentTrainDev& d, const LatentSeqArgs& a, cudaStream_t stream);
