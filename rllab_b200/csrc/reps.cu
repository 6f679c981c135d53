// REPS dual on the lane layout: the sample Bellman error delta = r + (phi(s') - phi(s)) . v, its maximum, and the sums
// behind the dual g(eta, v) and its gradient, plus the policy-step weights exp((delta - max delta) / eta).
//
// Replaces: rllab/algos/reps.py:101-102,164-197 (delta_v, the dual and theano.grad of it) and the per-path feat_diff
// construction of reps.py:227-238.  Nothing per sample is materialised: the features of (t, n) and of its successor
// (t + 1, n) are evaluated from obs / tstep inside the pass (lfb_features.cuh, the LinearFeatureBaseline map), with
// phi(s') = 0 after the last sample of a path (FLAG_END, which also marks a path cut by the end of the lane buffer).
// Both kernels stream 4 O + 7 bytes per sample (obs, rew, flags, tstep; the successor's observation is the next row,
// read again through L2), compute in float64, and reduce in two fixed-order stages: no atomics, bit-identical reruns.
#include "common.cuh"
#include "lfb_features.cuh"

namespace b200rl {

constexpr int REPS_THREADS = 256;
constexpr int REPS_BLOCKS_PER_SM = 4;

// A load the compiler may not merge with an earlier load of the same address (see reload() below).
__device__ __forceinline__ float ld_reload(const float* p) {
  float v;
  asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}

// One sample's inputs: its own observation, its successor's (zero features when `end`), the step index.
template <int OT>
struct RepsSample {
  float ov[OT], on[OT];
  unsigned short ts;
  bool end;
  double r;
  long long idx, nx;

  __device__ __forceinline__ void load(long long i, int N, int T, long long B, const float* __restrict__ obs,
                                       const float* __restrict__ rew, unsigned char f,
                                       const unsigned short* __restrict__ tstep) {
    idx = i;
    end = (f & B200RL_FLAG_END) || (idx / N) + 1 >= T;
    nx = end ? idx : idx + N;     // (no successor: a harmless in-bounds load, never used)
#pragma unroll
    for (int k = 0; k < OT; ++k) {
      ov[k] = obs[(size_t)k * B + idx];
      on[k] = obs[(size_t)k * B + nx];
    }
    ts = tstep[idx];
    r = (double)rew[idx];
  }
  // Read the two observations again (L1 hits) for the gradient sums: with 2 O + 6 float64 accumulators live, keeping
  // the 2 O floats (or their float64 features) alive from the Bellman error to the sums spilled at O = 20.
  __device__ __forceinline__ void reload(long long B, const float* __restrict__ obs) {
#pragma unroll
    for (int k = 0; k < OT; ++k) {
      ov[k] = ld_reload(obs + (size_t)k * B + idx);
      on[k] = ld_reload(obs + (size_t)k * B + nx);
    }
  }
  // feat_diff[j] = phi_j(s') - phi_j(s)
  __device__ __forceinline__ double dphi(int j) const {
    const double fn = end ? 0.0 : lfb_feature<OT>(on, (unsigned short)(ts + 1), j);
    return fn - lfb_feature<OT>(ov, ts, j);
  }
  __device__ __forceinline__ double delta(const double* __restrict__ v) const {
    double d = r;
#pragma unroll
    for (int j = 0; j < 2 * OT + 4; ++j) d += dphi(j) * v[j];
    return d;
  }
};

template <int OT>
__global__ void __launch_bounds__(REPS_THREADS)
    reps_delta_max_kernel(int N, int T, const float* __restrict__ obs, const float* __restrict__ rew,
                          const unsigned char* __restrict__ flags, const unsigned short* __restrict__ tstep, int masked,
                          const double* __restrict__ v, double* __restrict__ partial) {
  __shared__ double sv[2 * OT + 4];
  __shared__ double scratch[32];
  for (int i = threadIdx.x; i < 2 * OT + 4; i += blockDim.x) sv[i] = v[i];
  __syncthreads();
  const long long B = (long long)N * T;
  const long long stride = (long long)gridDim.x * blockDim.x;
  double m[1] = {-1.0e300};
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < B; idx += stride) {
    const unsigned char f = flags[idx];
    if (masked && (f & B200RL_FLAG_MASKED)) continue;
    RepsSample<OT> s;
    s.load(idx, N, T, B, obs, rew, f, tstep);
    m[0] = fmax(m[0], s.delta(sv));
  }
  block_reduce_store<1, true>(m, scratch, partial + blockIdx.x);
}

// out = [sum e, sum e (delta - M), sum e feat_diff (2 O + 4)] with e = exp((delta - M) / eta); w_out (optional) = e
template <int OT>
__global__ void __launch_bounds__(REPS_THREADS)
    reps_dual_sums_kernel(int N, int T, const float* __restrict__ obs, const float* __restrict__ rew,
                          const unsigned char* __restrict__ flags, const unsigned short* __restrict__ tstep, int masked,
                          const double* __restrict__ v, double eta, const double* __restrict__ M,
                          float* __restrict__ w_out, double* __restrict__ partial) {
  constexpr int D = 2 * OT + 4, K = D + 2;
  __shared__ double sv[D];
  __shared__ double scratch[K * 32];
  for (int i = threadIdx.x; i < D; i += blockDim.x) sv[i] = v[i];
  __syncthreads();
  const double Mv = *M;
  const long long B = (long long)N * T;
  const long long stride = (long long)gridDim.x * blockDim.x;
  double acc[K];
#pragma unroll
  for (int i = 0; i < K; ++i) acc[i] = 0.0;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < B; idx += stride) {
    const unsigned char f = flags[idx];
    if (masked && (f & B200RL_FLAG_MASKED)) {
      if (w_out != nullptr) w_out[idx] = 0.f;
      continue;
    }
    RepsSample<OT> s;
    s.load(idx, N, T, B, obs, rew, f, tstep);
    const double dm = s.delta(sv) - Mv;
    const double e = exp(dm / eta);
    acc[0] += e;
    acc[1] += e * dm;
    s.reload(B, obs);
#pragma unroll
    for (int j = 0; j < D; ++j) acc[2 + j] += e * s.dphi(j);
    if (w_out != nullptr) w_out[idx] = (float)e;
  }
  block_reduce_store<K>(acc, scratch, partial + (size_t)blockIdx.x * K);
}

static int reps_grid(long long B) { return partial_grid(REPS_BLOCKS_PER_SM, (B + REPS_THREADS - 1) / REPS_THREADS); }

static bool reps_obs_dim_ok(int O) { return O == 2 || O == 3 || O == 4 || O == 6 || O == 13 || O == 20; }

#define B200RL_REPS_DISPATCH(O, LAUNCH) \
  switch (O) {                          \
    case 2: LAUNCH(2); break;           \
    case 3: LAUNCH(3); break;           \
    case 4: LAUNCH(4); break;           \
    case 6: LAUNCH(6); break;           \
    case 13: LAUNCH(13); break;         \
    default: LAUNCH(20); break;         \
  }

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_reps_delta_max(int obs_dim, int N, int T, const float* obs, const float* rew, const unsigned char* flags,
                          const unsigned short* tstep, int masked, const double* v, double* out_max, double* ws,
                          void* stream) {
  B200RL_REQUIRE(obs && rew && flags && tstep && v && out_max && ws, "reps_delta_max: null buffer");
  B200RL_REQUIRE(N > 0 && T > 0, "reps_delta_max: bad sizes");
  if (!reps_obs_dim_ok(obs_dim)) {
    set_error("reps_delta_max: obs_dim %d is not compiled in (2, 3, 4, 6, 13, 20)", obs_dim);
    return B200RL_EUNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = reps_grid((long long)N * T);
#define B200RL_REPS_MAX(OT) \
  reps_delta_max_kernel<OT><<<grid, REPS_THREADS, 0, st>>>(N, T, obs, rew, flags, tstep, masked, v, ws)
  B200RL_REPS_DISPATCH(obs_dim, B200RL_REPS_MAX)
#undef B200RL_REPS_MAX
  B200RL_LAUNCH_CHECK("reps_delta_max_kernel");
  return launch_finalize_max(ws, grid, 1, out_max, st);
}

int b200rl_reps_dual_sums(int obs_dim, int N, int T, const float* obs, const float* rew, const unsigned char* flags,
                          const unsigned short* tstep, int masked, const double* v, double eta, const double* M,
                          double* out, float* w_out, double* ws, void* stream) {
  B200RL_REQUIRE(obs && rew && flags && tstep && v && M && out && ws, "reps_dual_sums: null buffer");
  B200RL_REQUIRE(N > 0 && T > 0, "reps_dual_sums: bad sizes");
  if (!reps_obs_dim_ok(obs_dim)) {
    set_error("reps_dual_sums: obs_dim %d is not compiled in (2, 3, 4, 6, 13, 20)", obs_dim);
    return B200RL_EUNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = reps_grid((long long)N * T);
  const int K = 2 * obs_dim + 6;
#define B200RL_REPS_SUMS(OT)                                                                                      \
  reps_dual_sums_kernel<OT><<<grid, REPS_THREADS, 0, st>>>(N, T, obs, rew, flags, tstep, masked, v, eta, M, w_out, \
                                                           ws)
  B200RL_REPS_DISPATCH(obs_dim, B200RL_REPS_SUMS)
#undef B200RL_REPS_SUMS
  B200RL_LAUNCH_CHECK("reps_dual_sums_kernel");
  return launch_finalize_sum(ws, grid, K, out, 1.0, st);
}
}
