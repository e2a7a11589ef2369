// Sequence batches gathered from a device-resident mirror of a replay buffer (mbrl_lib_b200/replay.py): what
//   mbrl/util/replay_buffer.py:183-195  _sequence_getitem_impl          (rows start .. start + T - 1 of each sequence)
//   mbrl/models/planet.py:274-287       PlaNetModel._process_batch     (obs.float() / 256 - 0.5)
//   mbrl/models/planet.py:429-434       the loss's obs[:, 1:], action[:, :-1], rewards[:, :-1]
// compute on the host and copy over PCIe, as one launch that reads the mirror in HBM and writes only what the loss reads.
//
// The mirror keeps frames in chunks of 2^chunk_shift rows, each its own allocation, found through a device table of
// chunk pointers; actions and rewards are one float array each.  Pure byte movement: every CTA walks whole frames
// (grid-stride), its threads moving consecutive 16-byte pieces of a frame, so reads and writes coalesce.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kCtasPerSm = 8;  // 8 x 256 threads fill an SM; at B x (T-1) = 2450 frames each CTA walks 2 to 3 frames

struct GatherArgs {
  long long frame_elems, rows;
  int action_size, chunk_shift, batch, steps;  // steps = T: each sequence yields T - 1 frames
  const void* const* chunks;
  const float* act;
  const float* rew;
  const long long* starts;
  float *obs_out, *act_out, *rew_out;
};

// x / 256 - 0.5 in fp32, each operation rounded on its own: the division by a power of two is exact, so this is
// bit-identical to torch's `obs.float() / 256.0 - 0.5` whatever the compiler's contraction settings.
__device__ __forceinline__ float normalise(float x) { return __fsub_rn(__fmul_rn(x, 0x1p-8f), 0.5f); }

__device__ __forceinline__ float4 normalise4(float a, float b, float c, float d) {
  return make_float4(normalise(a), normalise(b), normalise(c), normalise(d));
}

// four uint8 pixels of a 32-bit word, lowest address first
__device__ __forceinline__ float4 normalise_bytes(uint32_t w) {
  return normalise4((float)(w & 0xff), (float)((w >> 8) & 0xff), (float)((w >> 16) & 0xff), (float)(w >> 24));
}

// one frame: 16-byte loads (16 uint8 pixels or 4 floats) and float4 stores.  A warp loads 32 consecutive 16-byte
// pieces (512 pixels) and stores their 128 float4 in 4 rounds of 32 consecutive float4: float4 o of the warp's span
// comes from 32-bit word o, held by lane o / 4 as component o % 4, and reaches its storing lane by a shuffle.  The
// loop bounds are the same for the whole warp (the caller runs this for the whole CTA), so every shuffle has all lanes.
__device__ __forceinline__ void frame_vec(const uint8_t* __restrict__ src, float* __restrict__ dst, long long n) {
  const uint4* s = reinterpret_cast<const uint4*>(src);
  float4* d = reinterpret_cast<float4*>(dst);
  const long long nv = n / 16, nout = n / 4;
  const int lane = threadIdx.x & 31, c = lane & 3;
  for (long long base = (threadIdx.x >> 5) * 32LL; base < nv; base += kThreads) {
    const long long i = base + lane;
    const uint4 v = i < nv ? __ldg(s + i) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int from = 8 * k + (lane >> 2);
      const uint32_t x = __shfl_sync(0xffffffffu, v.x, from), y = __shfl_sync(0xffffffffu, v.y, from),
                     z = __shfl_sync(0xffffffffu, v.z, from), w = __shfl_sync(0xffffffffu, v.w, from);
      const long long o = 4 * base + 32 * k + lane;
      if (o < nout) d[o] = normalise_bytes(c == 0 ? x : c == 1 ? y : c == 2 ? z : w);
    }
  }
}

__device__ __forceinline__ void frame_vec(const float* __restrict__ src, float* __restrict__ dst, long long n) {
  const float4* s = reinterpret_cast<const float4*>(src);
  float4* d = reinterpret_cast<float4*>(dst);
  const long long nv = n / 4;
#pragma unroll 4
  for (long long i = threadIdx.x; i < nv; i += kThreads) {
    const float4 v = __ldg(s + i);
    d[i] = normalise4(v.x, v.y, v.z, v.w);
  }
}

template <typename S>
__device__ __forceinline__ void frame_scalar(const S* __restrict__ src, float* __restrict__ dst, long long n) {
  for (long long i = threadIdx.x; i < n; i += kThreads) dst[i] = normalise((float)src[i]);
}

template <typename S>
__global__ void __launch_bounds__(kThreads) sequence_gather_kernel(const GatherArgs a) {
  constexpr long long kVec = 16 / sizeof(S);  // elements per 16-byte load
  const int per_seq = a.steps - 1;
  const int frames = a.batch * per_seq;  // below 2^31: the entry point refuses more
  const long long mask = (1LL << a.chunk_shift) - 1;
  // the 16-byte path needs whole 16-byte pieces per frame on both sides; chunk bases are checked per frame below
  const bool vec_rows = a.frame_elems % kVec == 0 && a.frame_elems % 4 == 0 &&
                        (reinterpret_cast<uintptr_t>(a.obs_out) & 15) == 0;
  for (int f = blockIdx.x; f < frames; f += gridDim.x) {
    const int b = f / per_seq, t = f - b * per_seq;
    const long long start = a.starts[b];
    if (start < 0 || start + a.steps > a.rows) continue;  // the host refuses these before upload; never read past the store
    // frame t + 1 of the sequence (the loss's obs[:, 1:]); action and reward t (action[:, :-1], rewards[:, :-1])
    const long long row = start + t + 1;
    const S* src = reinterpret_cast<const S*>(a.chunks[row >> a.chunk_shift]) + (row & mask) * a.frame_elems;
    float* dst = a.obs_out + (long long)f * a.frame_elems;
    if (vec_rows && (reinterpret_cast<uintptr_t>(src) & 15) == 0)
      frame_vec(src, dst, a.frame_elems);
    else
      frame_scalar(src, dst, a.frame_elems);
    const long long r = start + t;
    for (int j = threadIdx.x; j < a.action_size; j += kThreads)
      a.act_out[(long long)f * a.action_size + j] = a.act[r * a.action_size + j];
    if (threadIdx.x == 0) a.rew_out[f] = a.rew[r];
  }
}

// ---- MBPO's SAC transitions (mbrl_lib_b200/replay.py DeviceTransitionMirror) ---------------------------------------
// One packed float row per transition, [obs | action | next_obs | reward | terminated] (W = 2D + A + 2 floats), in
// chunks of 2^chunk_shift rows.  Both kernels move floats only: consecutive threads take consecutive floats of the
// flattened [rows][W] range, so a warp reads and writes whole rows.
struct TransitionArgs {
  long long rows;  // gather: indices outside [0, rows) are skipped; scatter: positions wrap at rows (the capacity)
  int W, D, A, chunk_shift;
  float* const* chunks;
};

__global__ void __launch_bounds__(kThreads) transition_gather_kernel(const TransitionArgs a, const long long* __restrict__ idx,
                                                                     int batch, float* __restrict__ out) {
  const long long n = (long long)batch * a.W, mask = (1LL << a.chunk_shift) - 1;
  for (long long e = (long long)blockIdx.x * kThreads + threadIdx.x; e < n; e += (long long)gridDim.x * kThreads) {
    const long long b = e / a.W, col = e - b * a.W;
    const long long row = idx[b];
    if (row < 0 || row >= a.rows) continue;  // the host draws indices below num_stored; never read past the store
    const float* chunk = a.chunks[row >> a.chunk_shift];
    if (chunk) out[e] = chunk[(row & mask) * a.W + col];
  }
}

// row j of the packed rollout output goes to position (first + j) mod rows, its columns from the five arrays
__global__ void __launch_bounds__(kThreads) transition_scatter_kernel(const TransitionArgs a, long long first, long long count,
                                                                      const float* __restrict__ obs, const float* __restrict__ act,
                                                                      const float* __restrict__ next_obs,
                                                                      const float* __restrict__ reward,
                                                                      const uint8_t* __restrict__ terminated) {
  const long long n = count * a.W, mask = (1LL << a.chunk_shift) - 1;
  for (long long e = (long long)blockIdx.x * kThreads + threadIdx.x; e < n; e += (long long)gridDim.x * kThreads) {
    const long long j = e / a.W;
    const int col = (int)(e - j * a.W);
    const long long pos = (first + j) % a.rows;
    float v;
    if (col < a.D) v = obs[j * a.D + col];
    else if (col < a.D + a.A) v = act[j * a.A + (col - a.D)];
    else if (col < 2 * a.D + a.A) v = next_obs[j * a.D + (col - a.D - a.A)];
    else if (col == 2 * a.D + a.A) v = reward[j];
    else v = terminated[j] ? 1.0f : 0.0f;
    float* chunk = a.chunks[pos >> a.chunk_shift];
    if (chunk) chunk[(pos & mask) * a.W + col] = v;
  }
}

int g_sms[64];  // SM count per device ordinal, read once

int sm_count(const char* who, int* out) {
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return b200pets_set_error(B200PETS_EUNSUPPORTED, "%s: device ordinal %d", who, dev);
  if (g_sms[dev] == 0) CUDA_TRY(cudaDeviceGetAttribute(&g_sms[dev], cudaDevAttrMultiProcessorCount, dev));
  *out = g_sms[dev];
  return B200PETS_OK;
}

int check_chunk_shift(int shift, const char* who) {
  if (shift >= 0 && shift <= B200PETS_REPLAY_MAX_CHUNK_SHIFT) return B200PETS_OK;
  return b200pets_set_error(B200PETS_EINVAL, "%s: chunk_shift %d outside [0, %d]", who, shift, B200PETS_REPLAY_MAX_CHUNK_SHIFT);
}

int transition_args(const b200pets_transition_desc* desc, float* const* chunks, const char* who, TransitionArgs* a) {
  if (desc->obs_dim < 1 || desc->act_dim < 1 || desc->rows < 1)
    return b200pets_set_error(B200PETS_EINVAL, "%s: obs_dim %d, act_dim %d and rows %lld must be positive", who,
                              desc->obs_dim, desc->act_dim, (long long)desc->rows);
  if (const int rc = check_chunk_shift(desc->chunk_shift, who)) return rc;
  if (desc->obs_dim > (1 << 24) || desc->act_dim > (1 << 24))
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "%s: rows wider than 2^26 floats", who);
  a->rows = desc->rows;
  a->D = desc->obs_dim;
  a->A = desc->act_dim;
  a->W = 2 * desc->obs_dim + desc->act_dim + 2;
  a->chunk_shift = desc->chunk_shift;
  a->chunks = chunks;
  return B200PETS_OK;
}

unsigned grid_for(long long elems, int sms) {
  const long long blocks = (elems + kThreads - 1) / kThreads, most = (long long)sms * kCtasPerSm;
  return (unsigned)(blocks < most ? blocks : most);
}

}  // namespace

extern "C" {

int b200pets_sequence_gather(const b200pets_replay_desc* desc, const void* const* obs_chunks, const float* act,
                             const float* rew, const int64_t* starts, int32_t batch, int32_t steps, float* obs_out,
                             float* act_out, float* rew_out, void* stream) {
  if (!desc || !obs_chunks || !act || !rew || !starts || !obs_out || !act_out || !rew_out)
    return b200pets_set_error(B200PETS_EINVAL, "sequence_gather: NULL argument");
  if (batch < 1 || steps < 2)
    return b200pets_set_error(B200PETS_EINVAL, "sequence_gather: needs batch >= 1 and steps >= 2 (batch %d, steps %d)",
                              batch, steps);
  if (desc->dtype != B200PETS_DTYPE_U8 && desc->dtype != B200PETS_DTYPE_F32)
    return b200pets_set_error(B200PETS_EINVAL, "sequence_gather: unknown storage dtype %d", desc->dtype);
  if (const int rc = check_chunk_shift(desc->chunk_shift, "sequence_gather")) return rc;
  if (desc->frame_elems < 1 || desc->action_size < 1 || desc->rows < steps)
    return b200pets_set_error(B200PETS_EINVAL,
                              "sequence_gather: frame_elems %lld and action_size %d must be positive and rows %lld at "
                              "least steps %d", (long long)desc->frame_elems, desc->action_size, (long long)desc->rows,
                              steps);
  if ((long long)batch * (steps - 1) > 0x7fffffffLL)
    return b200pets_set_error(B200PETS_EUNSUPPORTED, "sequence_gather: more than 2^31 - 1 frames (batch %d, steps %d)",
                              batch, steps);
  int sms = 0;
  if (const int rc = sm_count("sequence_gather", &sms)) return rc;
  GatherArgs a{};
  a.frame_elems = desc->frame_elems;
  a.rows = desc->rows;
  a.action_size = desc->action_size;
  a.chunk_shift = desc->chunk_shift;
  a.batch = batch;
  a.steps = steps;
  a.chunks = obs_chunks;
  a.act = act;
  a.rew = rew;
  a.starts = reinterpret_cast<const long long*>(starts);
  a.obs_out = obs_out;
  a.act_out = act_out;
  a.rew_out = rew_out;
  const long long frames = (long long)batch * (steps - 1);
  const unsigned grid = (unsigned)(frames < (long long)sms * kCtasPerSm ? frames : (long long)sms * kCtasPerSm);
  cudaStream_t s = (cudaStream_t)stream;
  if (desc->dtype == B200PETS_DTYPE_U8)
    sequence_gather_kernel<uint8_t><<<grid, kThreads, 0, s>>>(a);
  else
    sequence_gather_kernel<float><<<grid, kThreads, 0, s>>>(a);
  CUDA_TRY(cudaGetLastError());
  return B200PETS_OK;
}

int b200pets_transition_gather(const b200pets_transition_desc* desc, float* const* chunks, const int64_t* indices,
                               int32_t batch, float* out, void* stream) {
  if (!desc || !chunks || !indices || !out) return b200pets_set_error(B200PETS_EINVAL, "transition_gather: NULL argument");
  if (batch < 1) return b200pets_set_error(B200PETS_EINVAL, "transition_gather: batch %d < 1", batch);
  TransitionArgs a{};
  if (const int rc = transition_args(desc, chunks, "transition_gather", &a)) return rc;
  int sms = 0;
  if (const int rc = sm_count("transition_gather", &sms)) return rc;
  const long long elems = (long long)batch * a.W;
  transition_gather_kernel<<<grid_for(elems, sms), kThreads, 0, (cudaStream_t)stream>>>(
      a, reinterpret_cast<const long long*>(indices), batch, out);
  CUDA_TRY(cudaGetLastError());
  return B200PETS_OK;
}

int b200pets_transition_scatter(const b200pets_transition_desc* desc, float* const* chunks, int64_t first, int64_t count,
                                const float* obs, const float* act, const float* next_obs, const float* reward,
                                const uint8_t* terminated, void* stream) {
  if (!desc || !chunks || !obs || !act || !next_obs || !reward || !terminated)
    return b200pets_set_error(B200PETS_EINVAL, "transition_scatter: NULL argument");
  TransitionArgs a{};
  if (const int rc = transition_args(desc, chunks, "transition_scatter", &a)) return rc;
  if (count < 1 || count > a.rows || first < 0 || first >= a.rows)
    return b200pets_set_error(B200PETS_EINVAL, "transition_scatter: needs 1 <= count <= rows and 0 <= first < rows "
                              "(first %lld, count %lld, rows %lld)", (long long)first, (long long)count, a.rows);
  int sms = 0;
  if (const int rc = sm_count("transition_scatter", &sms)) return rc;
  transition_scatter_kernel<<<grid_for(count * a.W, sms), kThreads, 0, (cudaStream_t)stream>>>(
      a, first, count, obs, act, next_obs, reward, terminated);
  CUDA_TRY(cudaGetLastError());
  return B200PETS_OK;
}

}  // extern "C"
