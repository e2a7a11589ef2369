// Tensor-core rollout of the ensemble MLP on sm_90a: bf16 operands, fp32 accumulation in registers (wgmma).
//
// Persistent CTAs walk row tiles through steps [t0, t1) of the horizon without leaving the chip.  A CTA has NWG consumer
// warpgroups and owns 64 * NWG rows.  NWG = 2: one CTA per SM, a whole 128-row tile.  NWG = 1: two CTAs per SM, each one
// half of a 128-row tile; the two interleave their MMAs, epilogues and barrier waits without an explicit schedule, but
// each streams its own copy of the weights.  NWG = 1 is used for launches with fewer 128-row tiles than SMs (the other
// shape would leave SMs idle) whose plan fits twice in an SM's shared memory:
//  * row state (observation, return, dead flag, actions) stays in shared memory / registers;
//  * each consumer warpgroup owns 64 rows.  A layer is a chain of wgmma.mma_async (M=64, K=16, N <= 128 per
//    instruction, two instructions per K step for layers wider than 128) that reads the warpgroup's activations from
//    its own shared-memory operand buffer; the accumulators stay in registers until the layer's last K step, then the
//    epilogue writes the activated, bf16-packed columns back into the same buffer (the next layer's A operand) or, for
//    the output layer, the fp32 accumulators into a staging area that aliases it;
//  * the B operand (weights) is streamed from the L2-resident packed image in K slices of up to 4 x 16 rows
//    by 1-D TMA bulk copies (cp.async.bulk + mbarrier expect_tx) into a ring of shared-memory slots: a producer warp
//    keeps the ring full across layers, steps and tiles, and a slot is released as soon as every warpgroup's MMAs that
//    read it have completed (wgmma.wait_group 1);
//  * propagation "expectation" runs M member passes per step.
//
// Warp roles (128 NWG + 32 threads): warps 0-3 = warpgroup 0 (CTA rows 0-63), warps 4-7 = warpgroup 1 (rows 64-127,
// NWG = 2 only), warp 4 * NWG (4 or 8) = weight producer (one lane).  Thread (row r, half h) of a warpgroup builds / samples half of the row's
// columns; half 0 owns the row's scalar state.
//
// Bias is folded into the GEMM: every A tile carries two constant-one columns after the real inputs and the
// packed weight image carries bf16(b) and bf16(b - bf16(b)) in the matching K rows (api.cu pack kernel).
//
// Reference semantics restated: see rollout_f32.cu header (same per-row maths, same file:line anchors).
#include <stdlib.h>

#include "common.cuh"
#include "sm90.cuh"

using namespace sm90;

struct TcPlan {
  int nwg;              // consumer warpgroups per CTA: 1 (64 rows, two CTAs per SM) or 2 (128 rows, one CTA per SM)
  int nlayers;
  int kp_max;           // widest layer input (K columns of the operand buffers)
  int kslice;           // K steps (16 rows of the weight image each) per ring slot
  uint32_t slot_bytes;  // one ring slot: kslice K steps of the widest layer
  int nstages;
  uint32_t wg_bytes;    // operand buffer / output staging of one warpgroup
  int stg_ld;           // row stride (floats) of the output staging
  uint32_t off_A, off_ring, off_obs, off_act, off_const, off_cout, off_bar;
  int obs_ld, act_ld;
  uint32_t smem_bytes;
  uint32_t off_exp;  // [rows][exp_ld] member sums of mean / log2-variance terms (propagation "expectation" launches only)
  int exp_ld;
};

namespace {

constexpr int kTileM = 128;  // rows of a tile: a shuffle group, a member's slot range chunk, an expectation chunk
template <int NWG>
constexpr int threads_of() { return 128 * NWG + 32; }
constexpr int kSliceK16 = 4;       // longest ring slot in K steps (16 rows of the weight image each)
constexpr int kMaxStages = 16;
constexpr int kActRegs = 8;  // models with up to this many actions load a step's action words in one round trip

__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float lg2_approx(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float sqrt_approx(float x) {  // one MUFU op, no slow-path fix-up (argument is in [1, inf))
  float y;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int ACT>
__device__ __forceinline__ float act_tc(float x, float slope) {
  // SiLU: x * sigmoid(x) = h + h * tanh(h) with h = x / 2 (one MUFU op).  The packed weight image of every layer that
  // feeds a SiLU is pre-scaled by 0.5 (api.cu pack_image_kernel), so the accumulator already holds h.
  if (ACT == B200PETS_ACT_SILU) return fmaf(x, tanh_approx(x), x);
  if (ACT == B200PETS_ACT_RELU) return fmaxf(x, 0.f);
  return x > 0.f ? x : x * slope;
}

// Byte offset of (row r, column k) in a warpgroup's operand buffer: 64 rows, K-major core matrices of 8 rows x 16 bytes,
// [k / 8][r / 8][r % 8][k % 8] -> LBO (K direction) = 1024 B, SBO (row direction) = 128 B.
__device__ __forceinline__ uint32_t a_off(int r, int k) {
  return (uint32_t)((k >> 3) * 1024 + (r >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2);
}

__device__ __forceinline__ void wg_bar(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

// One layer of one warpgroup: D (64 x np) = A (64 x 16 nk, shared memory) * W^T, W streamed through the ring in slices
// of kslice K steps.  The accumulator is split in two register chunks of W0 and W1 (0 or more) columns, np = W0 + W1.
// mode 0 (hidden layer): activation, bias-one columns n_true and n_true + 1, zero pad up to kp_next, bf16 pairs back into
// the operand buffer; mode 1 (output layer / self test): fp32 accumulators to the staging rows (stride stg_ld floats) that
// alias the operand buffer.  Returns the advanced ring position (stage | phase << 16).
struct LayerArgs {
  uint32_t a_addr;  // shared address of the warpgroup's operand buffer
  uint8_t* a_ptr;   // same, generic
  uint32_t ring_addr, slot_bytes;
  int nstages, kslice, nk, np, mode, n_true, kp_next, stg_ld;
  float leaky;
};

// One K slice: N K steps (kk0 .. kk0 + N - 1 of the layer) issued back to back as one wgmma group.  N is a compile-time
// constant so that the group is straight-line code: a loop with a runtime trip count is unrolled with a remainder whose
// branches sit between the MMAs, and ptxas then waits for each MMA to complete before it issues the next one
// (C7519 / C7520).  Only the layer's first K step overwrites the accumulators.
template <int N, int W0, int W1, int R0, int R1>
__device__ __forceinline__ void wg_slice(float (&d0)[R0], float (&d1)[R1], uint32_t a_addr, uint32_t slot, uint32_t b_lbo,
                                         int kk0) {
  const uint32_t b_kstep = 2u * b_lbo;  // bytes of one K step (16 rows) of the weight image
  wgmma_fence();
#pragma unroll
  for (int j = 0; j < N; ++j) {
    const uint64_t da = wgmma_desc(a_addr + (uint32_t)(kk0 + j) * 2048u, 1024u, 128u);
    const uint32_t b = slot + (uint32_t)j * b_kstep;
    const uint32_t acc = (j > 0 || kk0 > 0) ? 1u : 0u;
    Wgmma<W0>::mma(d0, da, wgmma_desc(b, b_lbo, 128u), acc);
    if constexpr (W1 > 0) Wgmma<W1>::mma(d1, da, wgmma_desc(b + (uint32_t)(W0 / 8) * 128u, b_lbo, 128u), acc);
  }
  wgmma_commit();
}

// Inlined into the kernel: ptxas also serialises wgmma chains in a function that is called (C7510).
template <int ACT, int W0, int W1>
__device__ __forceinline__ uint32_t wg_layer(const LayerArgs& la, uint32_t ring_pos, uint64_t* bar_full, uint64_t* bar_empty) {
  static_assert(kSliceK16 == 4, "wg_layer dispatches slices of 1 .. 4 K steps");
  constexpr int R1 = W1 > 0 ? W1 / 2 : 1;
  float d0[W0 / 2], d1[R1];
#pragma unroll
  for (int i = 0; i < W0 / 2; ++i) d0[i] = 0.f;
#pragma unroll
  for (int i = 0; i < R1; ++i) d1[i] = 0.f;
  const int wt = threadIdx.x & 127, lane = threadIdx.x & 31;
  int stage = (int)(ring_pos & 0xFFFFu);
  uint32_t phase = ring_pos >> 16;
  int prev = -1;
  const uint32_t b_lbo = (uint32_t)la.np * 16u;
  fence_operands(d0);
  fence_operands(d1);
  for (int k0 = 0; k0 < la.nk; k0 += la.kslice) {
    mbar_wait(&bar_full[stage], phase);
    const uint32_t slot = la.ring_addr + (uint32_t)stage * la.slot_bytes;
    switch (min(la.nk - k0, la.kslice)) {
      case 1: wg_slice<1, W0, W1>(d0, d1, la.a_addr, slot, b_lbo, k0); break;
      case 2: wg_slice<2, W0, W1>(d0, d1, la.a_addr, slot, b_lbo, k0); break;
      case 3: wg_slice<3, W0, W1>(d0, d1, la.a_addr, slot, b_lbo, k0); break;
      default: wg_slice<4, W0, W1>(d0, d1, la.a_addr, slot, b_lbo, k0); break;
    }
    if (prev >= 0) {  // the previous slice's MMAs are complete: hand its slot back to the producer
      wgmma_wait<1>();
      if (lane == 0) mbar_arrive(&bar_empty[prev]);
    }
    prev = stage;
    if (++stage == la.nstages) { stage = 0; phase ^= 1u; }
  }
  wgmma_wait<0>();
  fence_operands(d0);
  fence_operands(d1);
  if (lane == 0) mbar_arrive(&bar_empty[prev]);
  wg_bar((threadIdx.x >> 7) & 1);  // every MMA of the warpgroup has read its operand buffer: it may be overwritten

  const int r0 = 16 * (wt >> 5) + (lane >> 2);  // fragment rows r0 and r0 + 8
  const int cq = 2 * (lane & 3);
  if (la.mode == 0) {
    auto store = [&](float x0, float x1, float x2, float x3, int col) {
      float v[4] = {act_tc<ACT>(x0, la.leaky), act_tc<ACT>(x1, la.leaky), act_tc<ACT>(x2, la.leaky), act_tc<ACT>(x3, la.leaky)};
      if (col == la.n_true || col == la.n_true + 1) v[0] = v[2] = 1.f;
      if (col + 1 == la.n_true || col + 1 == la.n_true + 1) v[1] = v[3] = 1.f;
      *reinterpret_cast<uint32_t*>(la.a_ptr + a_off(r0, col)) = pack_bf16(v[0], v[1]);
      *reinterpret_cast<uint32_t*>(la.a_ptr + a_off(r0 + 8, col)) = pack_bf16(v[2], v[3]);
    };
#pragma unroll
    for (int j = 0; j < W0 / 8; ++j) store(d0[4 * j], d0[4 * j + 1], d0[4 * j + 2], d0[4 * j + 3], 8 * j + cq);
    if constexpr (W1 > 0) {
#pragma unroll
      for (int j = 0; j < W1 / 8; ++j) store(d1[4 * j], d1[4 * j + 1], d1[4 * j + 2], d1[4 * j + 3], W0 + 8 * j + cq);
    }
    // operand columns past the accumulator (np .. kp_next): bias ones / zero pad
    const int npad = la.kp_next - la.np;
    for (int idx = wt; idx < 64 * (npad >> 1); idx += 128) {
      const int r = idx & 63, col = la.np + 2 * (idx >> 6);
      const float v0 = (col == la.n_true || col == la.n_true + 1) ? 1.f : 0.f;
      const float v1 = (col + 1 == la.n_true || col + 1 == la.n_true + 1) ? 1.f : 0.f;
      *reinterpret_cast<uint32_t*>(la.a_ptr + a_off(r, col)) = pack_bf16(v0, v1);
    }
    fence_proxy_async_smem();
  } else {
    float* stg = reinterpret_cast<float*>(la.a_ptr);
#pragma unroll
    for (int j = 0; j < W0 / 8; ++j) {
      *reinterpret_cast<float2*>(stg + r0 * la.stg_ld + 8 * j + cq) = make_float2(d0[4 * j], d0[4 * j + 1]);
      *reinterpret_cast<float2*>(stg + (r0 + 8) * la.stg_ld + 8 * j + cq) = make_float2(d0[4 * j + 2], d0[4 * j + 3]);
    }
    if constexpr (W1 > 0) {
#pragma unroll
      for (int j = 0; j < W1 / 8; ++j) {
        *reinterpret_cast<float2*>(stg + r0 * la.stg_ld + W0 + 8 * j + cq) = make_float2(d1[4 * j], d1[4 * j + 1]);
        *reinterpret_cast<float2*>(stg + (r0 + 8) * la.stg_ld + W0 + 8 * j + cq) = make_float2(d1[4 * j + 2], d1[4 * j + 3]);
      }
    }
  }
  return (uint32_t)stage | (phase << 16);
}

// layer width -> register chunks: up to 128 columns in one, wider layers as 128 + the rest (np <= 256, multiple of 16)
template <int ACT>
__device__ __forceinline__ uint32_t run_layer(const LayerArgs& la, uint32_t ring_pos, uint64_t* bar_full, uint64_t* bar_empty) {
  switch (la.np) {
#define TC_W(N0, N1) \
  case N0 + N1: return wg_layer<ACT, N0, N1>(la, ring_pos, bar_full, bar_empty);
    TC_W(16, 0) TC_W(32, 0) TC_W(48, 0) TC_W(64, 0) TC_W(80, 0) TC_W(96, 0) TC_W(112, 0) TC_W(128, 0)
    TC_W(128, 16) TC_W(128, 32) TC_W(128, 48) TC_W(128, 64) TC_W(128, 80) TC_W(128, 96) TC_W(128, 112) TC_W(128, 128)
#undef TC_W
    default: __trap();  // tc_make_plan admits multiples of 16 up to 256 only
  }
  return ring_pos;
}

// The rollout kernels' body, inlined into each kernel (ptxas serialises wgmma chains in a called function, C7510).
// EXP: propagation "expectation" (member passes)
// TRAJ: per-step trajectory stores compiled in (b200pets_eval_trajectory); the other variants are compiled without them
//       so that their schedule stays what it was
// NWG: consumer warpgroups (TcPlan::nwg).  CTA tile u is half u % 2 of 128-row tile u / 2 when NWG = 1, tile u itself
//      when NWG = 2; either way a row keeps its member, keys, operands and K order.
// BATCH: K independent problems in one launch (common.cuh BatchArgs): 128-row tile j is local tile j % bt->tiles of
//      problem j / bt->tiles, and everything after that decode is the single-problem code.
template <int ACT, bool EXP, bool TRAJ, int NWG, bool BATCH>
__device__ __forceinline__ void rollout_tc_body(const ModelDev& m, const RolloutArgs& a, const TcPlan& p, const long long num_tiles,
                                                const BatchArgs* bt) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* ring = smem + p.off_ring;
  float* obs_s = reinterpret_cast<float*>(smem + p.off_obs);
  float* act_s = reinterpret_cast<float*>(smem + p.off_act);
  float2* c_norm = reinterpret_cast<float2*>(smem + p.off_const);  // [Kp0] {mean, 1/std}; (0, 1) past the real inputs
  // per-output constants of the output-layer maths, one 16-byte load per output (padded to a multiple of 4 outputs):
  //   x = max_logvar * log2(e), y = exp(max_logvar - min_logvar), z = exp(min_logvar / 2), w = 1 if the prediction is a
  //   delta to add to the old observation (0: keep the raw prediction -- no_delta columns, the learned-reward column, pad)
  const int outq = (m.out + 3) & ~3;
  float4* c_out = reinterpret_cast<float4*>(smem + p.off_cout);
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(smem + p.off_bar);
  uint64_t* bar_empty = bar_full + kMaxStages;

  constexpr int kThreads = threads_of<NWG>();
  constexpr int kSplit = 2 / NWG;  // CTA tiles per 128-row tile
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = p.nstages;
  // Programmatic dependent launch (common.cuh): let the next kernel of the chain become resident now; everything up
  // to the pdl_wait() below (barriers, constant tables, the producer's first weight copies) reads only the staged
  // model, which no kernel of a plan writes.
  pdl_trigger();

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&bar_full[s], 1);
      mbar_init(&bar_empty[s], 4 * NWG);  // one arrival per consumer warp
    }
    mbar_fence_init();
  }
  for (int j = threadIdx.x; j < m.Kp[0]; j += kThreads)
    c_norm[j] = (j < m.in && m.norm_mode) ? make_float2(m.norm_mean_f[j], m.norm_istd_f[j]) : make_float2(0.f, 1.f);
  // logvar clamp folded into two per-output constants (see the output-layer maths):
  //   var = exp(min + softplus(max - softplus(max - lv) - min)) = exp(min) * (1 + exp(max - min) / (1 + exp(max - lv)))
  for (int j = threadIdx.x; j < outq; j += kThreads) {
    const bool real = j < m.out;
    const float mn = (m.deterministic || !real) ? 0.f : m.min_lv[j], mx = (m.deterministic || !real) ? 0.f : m.max_lv[j];
    const bool delta = real && j < m.D && m.target_is_delta && !m.no_delta[j];
    c_out[j] = make_float4(mx * 1.4426950408889634f, expf(mx - mn), expf(0.5f * mn), delta ? 1.f : 0.f);
  }
  __syncthreads();

  // propagation "expectation" (gaussian_mlp.py:213-215): every row through every member, mean and clamped logvar averaged
  // over the members: `passes` = M forward passes per horizon step over the same layer-0 operand, member = pass
  constexpr bool expect = EXP;
  const int passes = expect ? m.M : 1;
  const bool shuffle = a.slot_mode >= 1 && !expect;
  const ShuffleGeom geom = shuffle_geom(a.seq0, a.N, a.n_glob);
  const long long Bm = shuffle ? 0 : (expect ? a.B : a.B / m.M);
  const int tpm = shuffle ? 1 : (int)((Bm + kTileM - 1) / kTileM);
  const int nlayers = p.nlayers;
  const int L = nlayers - 1;  // index of the output layer

  if (warp == 4 * NWG) {
    // =========================== weight producer ===========================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      // per-row members: the tile list comes from the bucketing kernel's offsets, the previous kernel's output
      if (!expect && a.member_off) pdl_wait();
      for (long long u = blockIdx.x; u < num_tiles; u += gridDim.x) {
        long long tile = u / kSplit;
        long long kp = 0;  // problem of a batched launch
        if constexpr (BATCH) { kp = tile / bt->tiles; tile -= kp * bt->tiles; }
        int member = (shuffle || expect) ? 0 : (int)(tile / tpm);
        if (!expect && a.member_off) {  // the consumers skip the same surplus tiles (member_tile)
          long long slot0;
          if (member_tile(a.member_off + prob_off<BATCH>(bt, kp, &BatchArgs::member_off), m.M, tile, kTileM, &member, &slot0) == 0)
            continue;
        }
        for (int t = a.t0; t < a.t1; ++t)
        for (int pass = 0; pass < passes; ++pass) {
          const int mem = expect ? pass : (shuffle ? shuffle_member(prob_seed<BATCH>(a, bt, kp), prob_offset<BATCH>(a, bt, kp), a.slot_mode,
                                                                    shuffle_global_group(geom, tile), t, m.M) : member);
          const uint8_t* base = m.img + (size_t)(blockIdx.x % m.img_replicas) * m.img_replica_stride + (size_t)mem * m.img_member_stride;
          for (int l = 0; l < nlayers; ++l) {
            // K steps are contiguous in the image (16 rows x Np columns each): a slice is one bulk copy
            const uint8_t* lsrc = base + m.img_layer_off[l];
            const int nk = m.Kp[l] >> 4;
            const uint32_t kstep = (uint32_t)m.Np[l] * 32u;
            for (int k0 = 0; k0 < nk; k0 += p.kslice) {
              const uint32_t bytes = (uint32_t)(min(nk, k0 + p.kslice) - k0) * kstep;
              mbar_wait(&bar_empty[stage], phase ^ 1u);
              mbar_arrive_expect_tx(&bar_full[stage], bytes);
              bulk_g2s(ring + (size_t)stage * p.slot_bytes, lsrc + (size_t)k0 * kstep, bytes, &bar_full[stage]);
              if (++stage == S) { stage = 0; phase ^= 1u; }
            }
          }
        }
      }
    }
    __syncwarp();
  } else {
    // =========================== consumer warpgroups ===========================
    const int wg = warp >> 2;
    const int wt = threadIdx.x & 127;
    const int r = wt & 63, h = wt >> 6;  // row of the warpgroup, half of the row's work
    const int i = wg * 64 + r;           // CTA row
    const bool owner = h == 0;           // the row's scalar state: observation / actions load, score, store
    uint8_t* abuf = smem + p.off_A + (size_t)wg * p.wg_bytes;
    const float* stg = reinterpret_cast<const float*>(abuf) + r * p.stg_ld;  // this row's output accumulators
    float* my_obs = obs_s + i * p.obs_ld;
    float* my_act = act_s + i * p.act_ld;
    const int ngroups = (m.out + 3) >> 2;
    const bool draw = !m.deterministic && a.sample;
    const int Kp0 = m.Kp[0];
    LayerArgs la;
    la.a_addr = smem_u32(abuf);
    la.a_ptr = abuf;
    la.ring_addr = smem_u32(ring);
    la.slot_bytes = p.slot_bytes;
    la.nstages = S;
    la.kslice = p.kslice;
    la.stg_ld = p.stg_ld;
    la.leaky = m.leaky;
    uint32_t ring_pos = 0;

    // layer-0 operand of one step: normalise(cat(proc(obs), act)), two constant-one bias columns, zero pad; the two
    // threads of a row take alternate column pairs
    auto build_input = [&]() {
      for (int jp = h; jp < (Kp0 >> 1); jp += 2) {
        float x[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int j = 2 * jp + e;
          float raw;
          if (j < m.Dp) raw = m.obs_process == B200PETS_PROC_NONE ? my_obs[j] : proc_obs_elem(my_obs, j, m.obs_process);
          else if (j < m.Dp + m.A) raw = my_act[j - m.Dp];
          else raw = j < m.Dp + m.A + 2 ? 1.f : 0.f;
          const float2 nm = c_norm[j];
          x[e] = (raw - nm.x) * nm.y;
        }
        *reinterpret_cast<uint32_t*>(abuf + a_off(r, 2 * jp)) = pack_bf16(x[0], x[1]);
      }
      fence_proxy_async_smem();
      wg_bar(wg);
    };

    pdl_wait();  // actions / observation / row state are the previous kernels' outputs; ours are written after this
    for (long long u = blockIdx.x; u < num_tiles; u += gridDim.x) {
      long long tile = u / kSplit;
      long long kp = 0;  // problem of a batched launch
      if constexpr (BATCH) { kp = tile / bt->tiles; tile -= kp * bt->tiles; }
      const int ti = i + 64 * (int)(u % kSplit);  // row of the 128-row tile
      bool valid;
      long long rid, rid_glob;  // local row id (n * P + p: indexes actions / state / injected noise), global one (RNG key)
      if (shuffle) {
        rid = shuffle_row(a, geom, tile, ti, &valid, &rid_glob);
        if (!valid) rid = 0;
      } else if (!expect && a.member_off) {  // per-row members: the producer's tile list (member_tile)
        int member;
        long long slot0;
        const int nv = member_tile(a.member_off + prob_off<BATCH>(bt, kp, &BatchArgs::member_off), m.M, tile, kTileM, &member, &slot0);
        if (nv == 0) continue;  // uniform over the CTA; the producer streams nothing for it
        valid = ti < nv;
        rid = valid ? prob_rid<BATCH>(a, bt, kp, slot0 + ti) : 0;
        rid_glob = rid + (long long)a.seq0 * a.P;
      } else {
        const int member = (int)(tile / tpm);
        const int c = (int)(tile % tpm);
        const long long slot0 = (long long)member * Bm + (long long)c * kTileM;
        valid = ti < (int)min((long long)kTileM, Bm - (long long)c * kTileM);
        rid = valid ? prob_rid<BATCH>(a, bt, kp, slot0 + ti) : 0;
        rid_glob = rid + (long long)a.seq0 * a.P;
      }
      float tot = 0.f;
      int dead = 0;
      const float* act_row = a.act + prob_off<BATCH>(bt, kp, &BatchArgs::act) + (rid / a.act_div) * a.act_row_stride;
      // this step's actions from the action tensor into the row's action words.  Up to kActRegs words are loaded into
      // registers first, so that the loads are in flight together (the word-by-word loop waits for each load before
      // it issues the next: one L2 round trip per word).
      auto load_actions = [&](int t) {
        if (owner) {
          const float* ap = act_row + (long long)t * a.act_t_stride;
          if (m.A <= kActRegs) {
            float v[kActRegs];
#pragma unroll
            for (int j = 0; j < kActRegs; ++j) v[j] = (j < m.A && valid) ? ap[j] : 0.f;
#pragma unroll
            for (int j = 0; j < kActRegs; ++j)
              if (j < m.A) my_act[j] = v[j];
          } else {
#pragma unroll 1
            for (int j = 0; j < m.A; ++j) my_act[j] = valid ? ap[j] : 0.f;
          }
        }
      };
      wg_bar(wg);  // previous tile fully consumed before its row state is overwritten
      if (owner) {
        if (a.load_state && valid) {
          tot = a.total_state[prob_off<BATCH>(bt, kp, &BatchArgs::rows) + rid];
          dead = a.dead_state[prob_off<BATCH>(bt, kp, &BatchArgs::rows) + rid];
        }
#pragma unroll 1
        for (int d = 0; d < m.D; ++d) {
          float v = 0.f;
          if (valid)
            v = a.init_from_obs0 ? a.obs0[prob_off<BATCH>(bt, kp, &BatchArgs::obs0) + d]
                                 : a.obs_in[prob_off<BATCH>(bt, kp, &BatchArgs::obs_state) + rid * m.D + d];
          my_obs[d] = v;
        }
      }
      load_actions(a.t0);
      wg_bar(wg);

      for (int t = a.t0; t < a.t1; ++t) {
        for (int pass = 0; pass < passes; ++pass) {
          const bool last_pass = pass == passes - 1;
          build_input();
          for (int l = 0; l < nlayers; ++l) {
            la.nk = m.Kp[l] >> 4;
            la.np = m.Np[l];
            la.mode = l < L ? 0 : 1;
            la.n_true = m.N[l];
            la.kp_next = l < L ? m.Kp[l + 1] : 0;
            ring_pos = run_layer<ACT>(la, ring_pos, bar_full, bar_empty);
            wg_bar(wg);  // hidden: next layer's operand complete; output: staged accumulators complete
          }
          // ---- output layer: groups of 4 outputs, the two threads of a row take alternate groups; Gaussian sample,
          //      delta add-back (branch-free inner maths) ----
          for (int gq = h; gq < ngroups; gq += 2) {
            float rm[4], rl[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              rm[e] = stg[4 * gq + e];
              if (!m.deterministic) rl[e] = stg[m.outp + 4 * gq + e];
            }
            // "expectation": member sums of the mean and of log2(1 + e2) (the clamped logvar is min + ln(1 + e2), see below)
            // in the row's scratch words; the last pass turns them into the averaged mean and sqrt(exp(averaged logvar))
            float sdv[4] = {0.f, 0.f, 0.f, 0.f};
            if (expect) {
              float* exm = reinterpret_cast<float*>(smem + p.off_exp) + i * p.exp_ld + 4 * gq;
              float* exl = exm + outq;
              const float inv_m = 1.0f / (float)passes;
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float4 ce = c_out[4 * gq + e];
                float l2 = 0.f;
                if (draw) {
                  const float e1 = ex2_approx(fmaf(rl[e], -1.4426950408889634f, ce.x));
                  l2 = lg2_approx(1.f + ce.y * rcp_approx(1.f + e1));
                }
                const float am = (pass ? exm[e] : 0.f) + rm[e];
                const float al = (pass ? exl[e] : 0.f) + l2;
                exm[e] = am;
                exl[e] = al;
                rm[e] = am * inv_m;
                sdv[e] = ce.z * ex2_approx(0.5f * al * inv_m);  // sqrt(exp(min + ln2 * mean_m log2(1 + e2)))
              }
              if (!last_pass) continue;
            }
            // Per output: one 16-byte constant load, 3 MUFU (ex2, rcp, sqrt), one LDS + FADD/FSEL + STS of the state.
            //   var = exp(min + softplus(max - softplus(max - lv) - min)) = e^min * (1 + e^(max-min) / (1 + e^(max-lv)))
            //   (gaussian_mlp.py:150-153 folded into two per-output constants), pred = mean + sqrt(var) * z
            //   (model.py:467-471), next = pred + keep * old (one_dim_tr_model.py:281-286).  Padded outputs (o >= out)
            //   land in the row's padding words; the learned-reward column is word D of the row.
            float z[4] = {0.f, 0.f, 0.f, 0.f};
            if (draw) {
              if (a.eps) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const int oc = min(4 * gq + e, m.out - 1);
                  z[e] = valid ? a.eps[prob_off<BATCH>(bt, kp, &BatchArgs::eps) + ((size_t)(t - a.t0) * a.B + rid) * m.out + oc] : 0.f;
                }
              } else {
                philox_normal4((uint32_t)rid_glob, (uint32_t)t, RNG_STREAM_EPS | (uint32_t)gq, (uint32_t)prob_offset<BATCH>(a, bt, kp),
                               prob_seed<BATCH>(a, bt, kp), z);
              }
            }
            const float4* cg = c_out + 4 * gq;
            float* og = my_obs + 4 * gq;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float4 ce = cg[e];
              float pv = rm[e];
              if (draw) {
                // exp(max - lv) (inf is fine); exp(max - min) / (1 + e1); sqrt(exp(clamped logvar))
                const float e1 = ex2_approx(fmaf(rl[e], -1.4426950408889634f, ce.x));
                const float e2 = ce.y * rcp_approx(1.f + e1);
                const float sd = expect ? sdv[e] : ce.z * sqrt_approx(1.f + e2);
                pv = fmaf(sd, z[e], pv);
              }
              // a select, not old * 0: a stale Inf / NaN word must not leak
              og[e] = ce.w != 0.f ? pv + og[e] : pv;
            }
          }
          wg_bar(wg);  // the row's words are complete; the staging area may be overwritten by the next operand
        }
        // ---- reward, termination, accumulate (model_env.py:124-129, 186-188) ----
        if (owner) {
          // model_env.py:124-128: pred_rewards only when reward_fn is None, an explicit reward_fn always wins
          float rew = m.reward_fn == B200PETS_REWARD_LEARNED ? my_obs[m.D] : reward_eval(m.reward_fn, my_act, m.A, 1, my_obs, m.D, 1);
          const bool done = term_eval(m.term_fn, my_obs, m.D, 1);
          if (valid) {
            if (a.reward_out) a.reward_out[rid] = rew;
            if (a.done_out) a.done_out[rid] = done ? 1 : 0;
          }
          if (TRAJ && valid) {
            const size_t tr = (size_t)(t - a.t0) * a.B + rid;
            if (a.traj_reward) a.traj_reward[tr] = rew;
            if (a.traj_done) a.traj_done[tr] = done ? 1 : 0;
            if (a.traj_obs) {
#pragma unroll 1
              for (int d = 0; d < m.D; ++d) a.traj_obs[tr * m.D + d] = my_obs[d];
            }
          }
          if (dead) rew = 0.f;
          dead |= done ? 1 : 0;
          tot += rew;
        }
        if (t + 1 < a.t1) {
          // the owner overwrites the action words its own score has just read: no barrier before
          load_actions(t + 1);
          wg_bar(wg);  // both threads of a row build the next operand from the action words one of them wrote
        }
      }
      // ---- store row state ----
      if (owner && a.store_state && valid) {
        if (a.obs_out) {
#pragma unroll 1
          for (int d = 0; d < m.D; ++d) a.obs_out[prob_off<BATCH>(bt, kp, &BatchArgs::obs_state) + rid * m.D + d] = my_obs[d];
        }
        if (a.total_state) a.total_state[prob_off<BATCH>(bt, kp, &BatchArgs::rows) + rid] = tot;
        if (a.dead_state) a.dead_state[prob_off<BATCH>(bt, kp, &BatchArgs::rows) + rid] = (uint8_t)dead;
      }
    }
  }

  __syncthreads();
}

template <int ACT, bool EXP, bool TRAJ, int NWG>
__global__ void __launch_bounds__(threads_of<NWG>(), NWG == 1 ? 2 : 1)
rollout_tc_kernel(const __grid_constant__ ModelDev m, const __grid_constant__ RolloutArgs a, const __grid_constant__ TcPlan p,
                  const long long num_tiles) {
  rollout_tc_body<ACT, EXP, TRAJ, NWG, false>(m, a, p, num_tiles, nullptr);
}

// K independent evaluations in one launch (plain and "expectation"; no trajectory variants)
template <int ACT, bool EXP, int NWG>
__global__ void __launch_bounds__(threads_of<NWG>(), NWG == 1 ? 2 : 1)
rollout_tc_batch_kernel(const __grid_constant__ ModelDev m, const __grid_constant__ RolloutArgs a, const __grid_constant__ TcPlan p,
                        const long long num_tiles, const __grid_constant__ BatchArgs bt) {
  rollout_tc_body<ACT, EXP, false, NWG, true>(m, a, p, num_tiles, &bt);
}

// ---------------------------------------------------------------------------------------------------------
// self test: one 128 x n x k GEMM through the rollout kernel's operand layouts, descriptors, weight ring and
// accumulator fragments: one warpgroup, rows 0-63 then rows 64-127 through the same operand buffer.  a_pairs = 1 writes
// A as bf16 pairs per thread and row, as the hidden-layer epilogue does; 0 as 16-byte core-matrix rows.
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128, 1) wgmma_selftest_kernel(int k, int n, int a_pairs, uint32_t wg_bytes, int stg_ld,
                                                                const float* __restrict__ A, const float* __restrict__ B,
                                                                float* __restrict__ D) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* A_s = smem;
  uint8_t* B_s = smem + wg_bytes;  // laid out as the weight ring would hold it: slice s of kSliceK16 K steps in slot s
  const int nsl = (k / 16 + kSliceK16 - 1) / kSliceK16;
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(B_s + (size_t)n * k * 2);  // [2][nsl]: one set per row half
  uint64_t* bar_empty = bar_full + 2 * nsl;
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < 2 * nsl; ++s) mbar_init(&bar_full[s], 1);
    for (int s = 0; s < nsl; ++s) mbar_init(&bar_empty[s], 8);  // (nobody waits for the slots to be released)
    mbar_fence_init();
  }
  // B: [n][k] row-major fp32 -> [k / 8][n / 8][n % 8][8]
  for (int idx = tid; idx < n * (k / 8); idx += 128) {
    int nn = idx % n, kc = idx / n;
    float x[8];
    for (int e = 0; e < 8; ++e) x[e] = B[nn * k + kc * 8 + e];
    *reinterpret_cast<uint4*>(B_s + (size_t)(kc * (n / 8) + (nn >> 3)) * 128 + (nn & 7) * 16) =
        make_uint4(pack_bf16(x[0], x[1]), pack_bf16(x[2], x[3]), pack_bf16(x[4], x[5]), pack_bf16(x[6], x[7]));
  }
  for (int half = 0; half < 2; ++half) {
    // A: rows 64 half .. 64 half + 63 of [128][k] row-major fp32
    if (a_pairs) {
      for (int idx = tid; idx < 64 * (k / 2); idx += 128) {
        const int r = idx & 63, c = 2 * (idx >> 6);
        const float* src = A + (64 * half + r) * k + c;
        *reinterpret_cast<uint32_t*>(A_s + a_off(r, c)) = pack_bf16(src[0], src[1]);
      }
    } else {
      for (int idx = tid; idx < 64 * (k / 8); idx += 128) {
        const int r = idx & 63, kc = idx >> 6;
        const float* src = A + (64 * half + r) * k + kc * 8;
        *reinterpret_cast<uint4*>(A_s + a_off(r, 8 * kc)) =
            make_uint4(pack_bf16(src[0], src[1]), pack_bf16(src[2], src[3]), pack_bf16(src[4], src[5]), pack_bf16(src[6], src[7]));
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
    if (tid == 0)  // the slots are already filled: complete this half's phase of them without a copy
      for (int s = 0; s < nsl; ++s) mbar_arrive(&bar_full[half * nsl + s]);
    LayerArgs la;
    la.a_addr = smem_u32(A_s);
    la.a_ptr = A_s;
    la.ring_addr = smem_u32(B_s);
    la.slot_bytes = (uint32_t)kSliceK16 * n * 32u;
    la.nstages = nsl;
    la.kslice = kSliceK16;
    la.nk = k / 16;
    la.np = n;
    la.mode = 1;
    la.n_true = n;
    la.kp_next = 0;
    la.stg_ld = stg_ld;
    la.leaky = 0.f;
    run_layer<B200PETS_ACT_RELU>(la, 0u, bar_full + half * nsl, bar_empty);
    wg_bar(0);
    const float* stg = reinterpret_cast<const float*>(A_s);
    for (int idx = tid; idx < 64 * n; idx += 128) {
      const int r = idx / n, c = idx % n;
      D[(64 * half + r) * n + c] = stg[r * stg_ld + c];
    }
    __syncthreads();
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
static int g_sm_count = 0, g_max_smem = 0, g_pair_smem = 0, g_limits_dev = -1;

static int tc_device_limits() {  // cached per device (a process may drive several)
  int dev = 0, sm_smem = 0, reserved = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  if (dev == g_limits_dev) return B200PETS_OK;
  CUDA_TRY(cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, dev));
  CUDA_TRY(cudaDeviceGetAttribute(&g_max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  CUDA_TRY(cudaDeviceGetAttribute(&sm_smem, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev));
  CUDA_TRY(cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev));
  // dynamic shared memory of a 64-row CTA that fits twice per SM: half the SM's, less the per-CTA reservation and the
  // static shared memory of the kernel (every 64-row variant, batched or not, has the same)
  cudaFuncAttributes fa;
  CUDA_TRY(cudaFuncGetAttributes(&fa, rollout_tc_kernel<B200PETS_ACT_SILU, false, false, 1>));
  g_pair_smem = min(g_max_smem, sm_smem / 2 - reserved - (int)fa.sharedSizeBytes);
  g_limits_dev = dev;
  return B200PETS_OK;
}

// smem plan for a model and CTA shape (nwg consumer warpgroups); returns false when the tensor-core path does not
// cover the dimensions or the plan does not fit in max_smem
static bool tc_make_plan(const ModelDev& m, int nwg, int max_smem, TcPlan* out, bool expectation) {
  TcPlan p{};
  p.nwg = nwg;
  const uint32_t rows = 64u * (uint32_t)nwg;
  p.nlayers = m.L + 1;
  if (m.in + 2 > 256 || m.hid + 2 > 256 || m.nout > 256 || m.D > 256) return false;
  int kp_max = 0;
  for (int l = 0; l < p.nlayers; ++l) {
    if (m.Np[l] > 256 || m.Kp[l] > 256) return false;
    kp_max = max(kp_max, m.Kp[l]);
  }
  p.kp_max = kp_max;
  const int npl = m.Np[p.nlayers - 1];
  p.stg_ld = npl + 4;
  p.wg_bytes = ((uint32_t)max(64 * kp_max * 2, 64 * p.stg_ld * 4) + 127u) & ~127u;
  const int outq = (m.out + 3) & ~3;
  p.obs_ld = max(m.D, outq) | 1;  // a row holds the D observation words, the learned-reward word and the output padding
  p.act_ld = m.A | 1;
  uint32_t off = 0;
  p.off_A = off; off += (uint32_t)nwg * p.wg_bytes;
  p.off_obs = off; off += rows * p.obs_ld * 4;
  p.off_act = off; off += rows * p.act_ld * 4;
  off = (off + 15u) & ~15u;
  p.off_const = off; off += (uint32_t)(2 * m.Kp[0]) * 4;
  off = (off + 15u) & ~15u;
  p.off_cout = off; off += (uint32_t)(4 * outq) * 4;
  off = (off + 15u) & ~15u;
  p.off_exp = off;
  p.exp_ld = (2 * outq) | 1;
  if (expectation) off += rows * p.exp_ld * 4;
  off = (off + 15u) & ~15u;
  p.off_bar = off; off += 2 * kMaxStages * 8;
  off = (off + 127u) & ~127u;
  p.off_ring = off;
  // longest slices that still leave three slots (one in use, two in flight); wide models get shorter slices
  int S = 0;
  for (p.kslice = kSliceK16;; --p.kslice) {
    uint32_t slot = 0;
    for (int l = 0; l < p.nlayers; ++l) slot = max(slot, (uint32_t)min(m.Kp[l] >> 4, p.kslice) * m.Np[l] * 32u);
    p.slot_bytes = (slot + 127u) & ~127u;
    S = ((int)max_smem - (int)off) / (int)p.slot_bytes;
    if (S >= 3 || p.kslice == 1) break;
  }
  if (S < 2) return false;
  p.nstages = min(S, kMaxStages);
  p.smem_bytes = off + (uint32_t)p.nstages * p.slot_bytes;
  if ((int)p.smem_bytes > max_smem) return false;
  *out = p;
  return true;
}

// The plan of a launch of `tiles` 128-row tiles.  Fewer tiles than SMs: 64-row CTAs two per SM when that plan fits in
// half an SM's shared memory, so that every SM gets work.  Otherwise 128-row CTAs one per SM with the whole opt-in shared
// memory: once every SM has a tile, two 64-row CTAs per SM measured slower than one 128-row CTA (they fetch the
// weights twice).  Every model with a 64-row plan also has a 128-row one.  Call after tc_device_limits().
static bool tc_choose_plan(const ModelDev& m, long long tiles, TcPlan* out, bool expectation = false) {
  if (tiles < g_sm_count && tc_make_plan(m, 1, g_pair_smem, out, expectation)) return true;
  return tc_make_plan(m, 2, g_max_smem, out, expectation);
}

bool tc_supported(const ModelDev& m) {
  if (tc_device_limits() != B200PETS_OK) return false;
  TcPlan p;
  return tc_choose_plan(m, g_sm_count, &p);
}

// the plan launch_rollout_tc uses for an evaluation / step with or without "expectation" that
// has a 128-row tile for every SM (launches with fewer tiles may run 64-row CTAs, see tc_choose_plan)
int tc_plan_info(const ModelDev& m, bool expectation, int* kslice, int* nstages, int* smem_bytes) {
  int rc = tc_device_limits();
  if (rc) return rc;
  TcPlan p;
  const bool ok = tc_choose_plan(m, g_sm_count, &p, expectation);
  *kslice = ok ? p.kslice : 0;
  *nstages = ok ? p.nstages : 0;
  *smem_bytes = ok ? (int)p.smem_bytes : 0;
  return B200PETS_OK;
}

using TcKernel = void (*)(const ModelDev, const RolloutArgs, const TcPlan, const long long);
using TcBatchKernel = void (*)(const ModelDev, const RolloutArgs, const TcPlan, const long long, const BatchArgs);

// The kernels of a launch: the single-problem kernel of its variant ("expectation", per-step trajectory stores for
// b200pets_eval_trajectory) and the batched kernel of the same activation and propagation.
struct TcKernels {
  TcKernel single;
  TcBatchKernel batch;
};

template <int ACT, bool EXPECT, int NWG>
static TcKernels tc_kernels(bool traj) {
  return {traj ? rollout_tc_kernel<ACT, EXPECT, true, NWG> : rollout_tc_kernel<ACT, EXPECT, false, NWG>,
          rollout_tc_batch_kernel<ACT, EXPECT, NWG>};
}

template <int NWG>
static TcKernels tc_kernels(int act, bool expect, bool traj) {
  if (act == B200PETS_ACT_SILU) return expect ? tc_kernels<B200PETS_ACT_SILU, true, NWG>(traj) : tc_kernels<B200PETS_ACT_SILU, false, NWG>(traj);
  if (act == B200PETS_ACT_RELU) return expect ? tc_kernels<B200PETS_ACT_RELU, true, NWG>(traj) : tc_kernels<B200PETS_ACT_RELU, false, NWG>(traj);
  return expect ? tc_kernels<B200PETS_ACT_LEAKY_RELU, true, NWG>(traj) : tc_kernels<B200PETS_ACT_LEAKY_RELU, false, NWG>(traj);
}

// 128-row tiles of one launch
static long long tc_launch_tiles(const ModelDev& m, const RolloutArgs& a) {
  if (a.propagation == B200PETS_PROP_EXPECTATION)  // every row through every member: plain 128-row tiles, no member binding
    return (a.B + kTileM - 1) / kTileM;
  if (a.slot_mode >= 1) return (long long)a.P * shuffle_geom(a.seq0, a.N, a.n_glob).C_loc;
  if (a.member_off) return (a.B + kTileM - 1) / kTileM + m.M - 1;  // per-row members: the bound of member_tile
  long long Bm = a.B / m.M;
  return (long long)m.M * ((Bm + kTileM - 1) / kTileM);
}

// `num_problems` evaluations of the launch `a` describes in one grid.  One problem runs rollout_tc_kernel and ignores
// bt; more run rollout_tc_batch_kernel with bt's per-problem strides (bt.tiles is set here).  The CTA shape follows the
// total tile count, as for a single launch of that many tiles.
int launch_rollout_tc(const ModelDev& m, const RolloutArgs& a, int num_problems, BatchArgs bt, cudaStream_t stream) {
  int rc = tc_device_limits();
  if (rc) return rc;
  if (num_problems > 1 && (a.traj_obs || a.traj_reward || a.traj_done || a.reward_out || a.done_out))
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "batched rollout: evaluation outputs only");
  const bool expect = a.propagation == B200PETS_PROP_EXPECTATION;
  const bool traj = a.traj_obs || a.traj_reward || a.traj_done;
  bt.tiles = tc_launch_tiles(m, a);
  const long long tiles = bt.tiles * num_problems;
  TcPlan p;
  if (!tc_choose_plan(m, tiles, &p, expect))
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "model dimensions outside the tensor-core path (in %d hid %d out %d)",
                              m.in, m.hid, m.out);
  const TcKernels kern = p.nwg == 1 ? tc_kernels<1>(m.act, expect, traj) : tc_kernels<2>(m.act, expect, traj);
  const int threads = p.nwg == 1 ? threads_of<1>() : threads_of<2>();
  const long long cta_tiles = tiles * (2 / p.nwg);
  // 64-row CTAs: fewer than two per SM, all resident (registers: tests/test_sass_occupancy.py; shared memory: the plan)
  const unsigned grid = (unsigned)min((long long)g_sm_count * (2 / p.nwg), cta_tiles);
  if (num_problems == 1) {
    CUDA_TRY(cudaFuncSetAttribute(kern.single, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem_bytes));
    CUDA_TRY(launch_pdl(kern.single, dim3(grid), dim3(threads), (size_t)p.smem_bytes, stream, m, a, p, cta_tiles));
  } else {
    CUDA_TRY(cudaFuncSetAttribute(kern.batch, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem_bytes));
    CUDA_TRY(launch_pdl(kern.batch, dim3(grid), dim3(threads), (size_t)p.smem_bytes, stream, m, a, p, cta_tiles, bt));
  }
  return B200PETS_OK;
}

int launch_wgmma_selftest(int k, int n, const float* a, const float* b, float* d, cudaStream_t stream) {
  const bool pairs = k < 0;  // negative k: A written as bf16 pairs per thread (the hidden-layer epilogue's stores)
  if (pairs) k = -k;
  if (k % 16 || n % 16 || n > 256 || k > 256 || k < 16 || n < 16)
    return b200pets_set_error(B200PETS_EINVAL, "selftest needs k, n multiples of 16, <= 256");
  const int stg_ld = n + 4;
  const uint32_t wg_bytes = ((uint32_t)max(64 * k * 2, 64 * stg_ld * 4) + 127u) & ~127u;
  const size_t smem = (size_t)wg_bytes + (size_t)n * k * 2 + 3 * 4 * 8;
  CUDA_TRY(cudaFuncSetAttribute(wgmma_selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  wgmma_selftest_kernel<<<1, 128, smem, stream>>>(k, n, pairs ? 1 : 0, wg_bytes, stg_ld, a, b, d);
  CUDA_TRY(cudaGetLastError());
  return B200PETS_OK;
}
