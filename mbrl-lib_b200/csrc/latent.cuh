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

// Rows per CTA and shared memory, chosen from the row count and the device (launcher and b200pets_latent_plan_info).
struct LatentPlan {
  int rows;          // rows per CTA: 1, 2, 4, 8, 16 or 32
  long long ctas;
  size_t smem;       // dynamic shared memory of one CTA
  size_t row_bytes;  // shared memory one row needs
  size_t row_limit;  // the most a row may need: an 8-row tile must fit in the opt-in shared memory
};

size_t latent_blob_floats(const LatentDev& m);  // m: sizes set
void latent_bind(LatentDev* m, float* blob);     // points the weight fields into blob
int latent_stage(const LatentDev& m, const float* const* params, cudaStream_t stream);
int latent_plan(const LatentDev& m, long long rows, LatentPlan* p);
int launch_latent_rollout(const LatentDev& m, const LatentArgs& a, cudaStream_t stream);
