// Lane rollout kernels: fused T-step rollout (policy forward + sample + env step + record, state in registers,
// policy parameters staged in shared memory), and the un-fused Env.reset / Env.step / Policy.get_actions
// entry points that mirror the reference API one call at a time.
//
// Replaces: rllab/algos/batch_polopt.py:22-34 (BatchSampler.obtain_samples), rllab/sampler/utils.py:6-43 (rollout),
// sandbox/rocky/tf/envs/vec_env_executor.py:14-26 (lock-step lanes with auto-reset),
// rllab/policies/gaussian_mlp_policy.py:125-137 (get_action/get_actions), rllab/envs/normalized_env.py:78-92.
#include "envs.cuh"
#include "mlp.cuh"

namespace b200rl {

constexpr int ROLLOUT_THREADS = 128;
// Register cap: the small classic-control kernels fit 128 registers (4 CTAs = 16 warps per SM: rollout 1.68 -> 1.46 ms
// on cfg2, A/B measured); the planar envs and 64-wide nets need the full 255.
template <class Env, int H>
constexpr int rollout_minblocks() { return (H == 32 && Env::S <= 4) ? 4 : 1; }

template <class Env>
__device__ __forceinline__ void draw_reset(float (&s)[Env::S], const float* __restrict__ reset_raw, int row, int N,
                                           int n, uint32_t seed, uint32_t iter, long long lane) {
  float raw[Env::K];
  if (reset_raw != nullptr) {
#pragma unroll
    for (int k = 0; k < Env::K; ++k) raw[k] = reset_raw[((size_t)row * Env::K + k) * N + n];
  } else {
#pragma unroll
    for (int c = 0; c < (Env::K + 3) / 4; ++c) {
      float q[4];
      noise4(Env::NOISE, seed, iter, 1, lane, row, c, q);
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (c * 4 + i < Env::K) raw[c * 4 + i] = q[i];
    }
  }
  Env::reset(s, raw);
}

template <int A>
__device__ __forceinline__ void draw_eps(float (&e)[A], const float* __restrict__ eps, int row, long long N,
                                         long long n, uint32_t seed, uint32_t iter, long long lane) {
  if (eps != nullptr) {
#pragma unroll
    for (int a = 0; a < A; ++a) e[a] = eps[((size_t)row * A + a) * N + n];
  } else {
    float q[4];
    noise4<(A + 1) / 2>(B200RL_NOISE_NORMAL, seed, iter, 0, lane, row, 0, q);
#pragma unroll
    for (int a = 0; a < A; ++a) e[a] = q[a];
  }
}

struct RolloutArgs {
  const float* params;
  float log_min_std;
  int N, T, max_path_length;
  const float* eps;
  const float* reset_raw;
  uint32_t seed, iter;
  long long lane0;
  float *obs, *act, *mean, *rew;
  unsigned char* flags;
  unsigned short* tstep;
  float* log_std_out;
};

// Policy weights of the 32-wide rollout through the CONSTANT bank: with theta in a __constant__ array the dense layers
// compile to FFMAs with a constant-bank operand (one load per warp, no LSU traffic) instead of LDS.128 + vector registers
// (the fully unrolled 32-wide layers index the weights with compile-time offsets).  The thread-per-sample update
// kernels keep theta in shared memory: their staging wants the registers.  theta is refreshed by one
// stream-ordered device-to-device cudaMemcpyToSymbolAsync (<= 7 KB) per rollout.
constexpr int ROLLOUT_CONST_MAXP = 2048;     // >= P of the largest 32-wide net (Hopper obs 20: 1 830)
__constant__ __align__(16) float c_theta[ROLLOUT_CONST_MAXP];
template <int H>
constexpr bool rollout_const_weights() { return H == 32; }

// One thread per lane; the whole T-step trajectory of a lane stays in that thread's registers.
template <class Env, int H>
__global__ void __launch_bounds__(ROLLOUT_THREADS, rollout_minblocks<Env, H>()) rollout_kernel(RolloutArgs a) {
  using N_ = Net<Env::O, H, H, Env::A>;
  // 32-wide: parameters in the constant bank; 64-wide: parameters in shared memory + one activation column per thread
  // for the rolled layer-2 loop
  constexpr int P4 = (N_::P + 3) & ~3;
  constexpr bool CW = rollout_const_weights<H>();
  extern __shared__ __align__(16) float rollout_smem[];
  const float* sp = CW ? c_theta : rollout_smem;
  float* hcol = (H > 32) ? rollout_smem + P4 + threadIdx.x : nullptr;
  if constexpr (!CW) {
    for (int i = threadIdx.x; i < N_::P; i += blockDim.x) rollout_smem[i] = a.params[i];
    __syncthreads();
  }
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  float std_[Env::A];
#pragma unroll
  for (int k = 0; k < Env::A; ++k) {
    float ls = clamp_log_std(sp[N_::ols + k], a.log_min_std);
    std_[k] = expf(ls);
    if (n == 0) a.log_std_out[k] = ls;
  }
  if (n >= a.N) return;
  const long long lane = a.lane0 + n;
  const size_t N = a.N, TN = (size_t)a.T * a.N;

  float s[Env::S];
  draw_reset<Env>(s, a.reset_raw, 0, a.N, n, a.seed, a.iter, lane);
  int plen = 0;
  for (int t = 0; t < a.T; ++t) {
    float o[Env::O], h1[H], h2[H], mu[Env::A], e[Env::A], act[Env::A], u[Env::A];
    // compiler barrier: without it the loop-invariant LDS of all P weights is hoisted out of the t loop and spilled
    asm volatile("" ::: "memory");
    Env::obs(s, o);
    mlp_forward_thread<N_>(sp, o, h1, h2, mu, hcol, ROLLOUT_THREADS);
    draw_eps<Env::A>(e, a.eps, t, a.N, n, a.seed, a.iter, lane);
    const size_t idx = (size_t)t * N + n;
#pragma unroll
    for (int k = 0; k < Env::O; ++k) a.obs[k * TN + idx] = o[k];
#pragma unroll
    for (int k = 0; k < Env::A; ++k) {
      act[k] = fmaf(std_[k], e[k], mu[k]);  // rnd * exp(log_std) + mean   (gaussian_mlp_policy.py:129)
      u[k] = scale_action(act[k], Env::lb(k), Env::ub(k));
      a.act[k * TN + idx] = act[k];
      a.mean[k * TN + idx] = mu[k];
    }
    float r;
    bool done;
    Env::step(s, u, r, done);
    a.tstep[idx] = (unsigned short)plen;
    ++plen;
    const bool whole = done || (plen >= a.max_path_length);
    const bool end = whole || (t == a.T - 1);
    a.rew[idx] = r;
    // FLAG_CUT: the path is cut by the end of the lane buffer, not by the env or max_path_length (process_samples drops
    // such paths when the caller asks for whole paths only, batch_polopt.py:30-34)
    a.flags[idx] = (unsigned char)((done ? B200RL_FLAG_DONE : 0) | (end ? B200RL_FLAG_END : 0) |
                                   ((end && !whole) ? B200RL_FLAG_CUT : 0));
    if (end) {
      draw_reset<Env>(s, a.reset_raw, t + 1, a.N, n, a.seed, a.iter, lane);
      plen = 0;
    }
  }
}

template <class Env>
__global__ void env_reset_kernel(int N, float* __restrict__ state, float* __restrict__ obs_out,
                                 const float* __restrict__ reset_raw, uint32_t seed, uint32_t iter, int row,
                                 long long lane0) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float s[Env::S], o[Env::O];
  // reset_raw here is a single [K][N] block: index it as row 0
  draw_reset<Env>(s, reset_raw, reset_raw ? 0 : row, N, n, seed, iter, lane0 + n);
  Env::obs(s, o);
#pragma unroll
  for (int k = 0; k < Env::S; ++k) state[(size_t)k * N + n] = s[k];
#pragma unroll
  for (int k = 0; k < Env::O; ++k) obs_out[(size_t)k * N + n] = o[k];
}

template <class Env>
__global__ void env_step_kernel(int N, int normalized, float* __restrict__ state, const float* __restrict__ actions,
                                float* __restrict__ obs_out, float* __restrict__ rew_out,
                                unsigned char* __restrict__ done_out) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float s[Env::S], o[Env::O], u[Env::A];
#pragma unroll
  for (int k = 0; k < Env::S; ++k) s[k] = state[(size_t)k * N + n];
#pragma unroll
  for (int k = 0; k < Env::A; ++k) {
    const float a = actions[(size_t)k * N + n];
    u[k] = normalized ? scale_action(a, Env::lb(k), Env::ub(k)) : a;
  }
  float r;
  bool done;
  Env::step(s, u, r, done);
  Env::obs(s, o);
#pragma unroll
  for (int k = 0; k < Env::S; ++k) state[(size_t)k * N + n] = s[k];
#pragma unroll
  for (int k = 0; k < Env::O; ++k) obs_out[(size_t)k * N + n] = o[k];
  rew_out[n] = r;
  done_out[n] = done ? 1 : 0;
}

template <class NetT>
__global__ void __launch_bounds__(ROLLOUT_THREADS)
    get_actions_kernel(const float* __restrict__ params, float log_min_std, const float* __restrict__ obs, long long n_,
                       const float* __restrict__ eps, uint32_t seed, uint32_t iter, int row, long long lane0,
                       float* __restrict__ act_out, float* __restrict__ mean_out, float* __restrict__ log_std_out) {
  __shared__ __align__(16) float sp[NetT::P];
  for (int i = threadIdx.x; i < NetT::P; i += blockDim.x) sp[i] = params[i];
  __syncthreads();
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  float std_[NetT::A];
#pragma unroll
  for (int k = 0; k < NetT::A; ++k) {
    float ls = clamp_log_std(sp[NetT::ols + k], log_min_std);
    std_[k] = expf(ls);
    if (n == 0) log_std_out[k] = ls;
  }
  if (n >= n_) return;
  float o[NetT::O], h1[NetT::H1], h2[NetT::H2], mu[NetT::A], e[NetT::A];
#pragma unroll
  for (int k = 0; k < NetT::O; ++k) o[k] = obs[(size_t)k * n_ + n];
  mlp_forward_thread<NetT>(sp, o, h1, h2, mu);
  if (eps != nullptr) {
#pragma unroll
    for (int k = 0; k < NetT::A; ++k) e[k] = eps[(size_t)k * n_ + n];
  } else {
    draw_eps<NetT::A>(e, nullptr, row, n_, n, seed, iter, lane0 + n);
  }
#pragma unroll
  for (int k = 0; k < NetT::A; ++k) {
    act_out[(size_t)k * n_ + n] = fmaf(std_[k], e[k], mu[k]);
    mean_out[(size_t)k * n_ + n] = mu[k];
  }
}

__global__ void fill_noise_kernel(float* __restrict__ out, int rows, int row0, int K, int N, long long lane0, int kind,
                                  uint32_t seed, uint32_t iter, int stream_id) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // over rows * chunks * N
  const int chunks = (K + 3) / 4;
  const long long total = (long long)rows * chunks * N;
  if (i >= total) return;
  const int n = (int)(i % N);
  const int c = (int)((i / N) % chunks);
  const int r = (int)(i / ((long long)N * chunks));
  float q[4];
  noise4(kind, seed, iter, stream_id, lane0 + n, row0 + r, c, q);
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (c * 4 + j < K) out[((size_t)r * K + c * 4 + j) * N + n] = q[j];
}

template <class Env>
static int launch_rollout(int h, const RolloutArgs& a, cudaStream_t st) {
  const int grid = (a.N + ROLLOUT_THREADS - 1) / ROLLOUT_THREADS;
  if (h == 32) {
    using N32 = Net<Env::O, 32, 32, Env::A>;
    static_assert(N32::P <= ROLLOUT_CONST_MAXP, "constant bank too small for this net");
    B200RL_CUDA_CHECK(cudaMemcpyToSymbolAsync(c_theta, a.params, (size_t)N32::P * sizeof(float), 0,
                                              cudaMemcpyDeviceToDevice, st));
    rollout_kernel<Env, 32><<<grid, ROLLOUT_THREADS, 0, st>>>(a);
  } else if (h == 64) {
    using N64 = Net<Env::O, 64, 64, Env::A>;
    const size_t smem = (((N64::P + 3) & ~3) + 64 * ROLLOUT_THREADS) * sizeof(float);
    B200RL_SET_MAX_SMEM((rollout_kernel<Env, 64>), smem);
    rollout_kernel<Env, 64><<<grid, ROLLOUT_THREADS, smem, st>>>(a);
  } else {
    set_error("hidden size %d not compiled in (32 or 64)", h);
    return B200RL_EUNSUPPORTED;
  }
  B200RL_LAUNCH_CHECK("rollout_kernel");
  return 0;
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_env_info(int env_kind, int* obs_dim, int* act_dim, int* state_dim, int* reset_dim, int* noise_kind,
                    float* lb_host, float* ub_host) {
  B200RL_DISPATCH_ENV(env_kind, {
    if (obs_dim) *obs_dim = Env::O;
    if (act_dim) *act_dim = Env::A;
    if (state_dim) *state_dim = Env::S;
    if (reset_dim) *reset_dim = Env::K;
    if (noise_kind) *noise_kind = Env::NOISE;
    for (int k = 0; k < Env::A; ++k) {
      if (lb_host) lb_host[k] = Env::lb(k);
      if (ub_host) ub_host[k] = Env::ub(k);
    }
  });
  return 0;
}

long long b200rl_policy_num_params(int obs_dim, int h1, int h2, int act_dim) {
  if (!net_supported(obs_dim, h1, h2, act_dim)) {
    set_error("network shape O=%d A=%d hidden=(%d,%d) is not compiled in", obs_dim, act_dim, h1, h2);
    return B200RL_EUNSUPPORTED;
  }
  return (long long)obs_dim * h1 + h1 + (long long)h1 * h2 + h2 + (long long)h2 * act_dim + act_dim + act_dim;
}

int b200rl_fill_noise(float* out, int rows, int row0, int K, int N, long long lane0, int noise_kind,
                      unsigned int seed, unsigned int iter, int stream_id, void* stream) {
  B200RL_REQUIRE(out && rows >= 0 && K > 0 && N > 0, "fill_noise: bad arguments");
  B200RL_REQUIRE(noise_kind == B200RL_NOISE_UNIFORM || noise_kind == B200RL_NOISE_NORMAL, "fill_noise: bad kind");
  if (rows == 0) return 0;
  const long long total = (long long)rows * ((K + 3) / 4) * N;
  const int bs = 256;
  fill_noise_kernel<<<(unsigned)((total + bs - 1) / bs), bs, 0, (cudaStream_t)stream>>>(
      out, rows, row0, K, N, lane0, noise_kind, seed, iter, stream_id);
  B200RL_LAUNCH_CHECK("fill_noise_kernel");
  return 0;
}

int b200rl_env_reset(int env_kind, int N, float* state, float* obs_out, const float* reset_raw, unsigned int seed,
                     unsigned int iter, int row, long long lane0, void* stream) {
  B200RL_REQUIRE(N > 0 && state && obs_out, "env_reset: bad arguments");
  B200RL_DISPATCH_ENV(env_kind, {
    env_reset_kernel<Env><<<(N + 127) / 128, 128, 0, (cudaStream_t)stream>>>(N, state, obs_out, reset_raw, seed,
                                                                              iter, row, lane0);
  });
  B200RL_LAUNCH_CHECK("env_reset_kernel");
  return 0;
}

int b200rl_env_step(int env_kind, int N, int normalized, float* state, const float* actions, float* obs_out,
                    float* rew_out, unsigned char* done_out, void* stream) {
  B200RL_REQUIRE(N > 0 && state && actions && obs_out && rew_out && done_out, "env_step: bad arguments");
  B200RL_DISPATCH_ENV(env_kind, {
    env_step_kernel<Env><<<(N + 127) / 128, 128, 0, (cudaStream_t)stream>>>(N, normalized, state, actions, obs_out,
                                                                             rew_out, done_out);
  });
  B200RL_LAUNCH_CHECK("env_step_kernel");
  return 0;
}

int b200rl_policy_get_actions(const float* params_f32, int obs_dim, int h1, int h2, int act_dim, float min_std,
                              const float* obs, long long n, const float* eps, unsigned int seed, unsigned int iter,
                              int row, long long lane0, float* act_out, float* mean_out, float* log_std_out,
                              void* stream) {
  B200RL_REQUIRE(params_f32 && obs && n > 0 && act_out && mean_out && log_std_out, "get_actions: bad arguments");
  const float lms = min_std > 0.f ? logf(min_std) : -INFINITY;
  const unsigned grid = (unsigned)((n + ROLLOUT_THREADS - 1) / ROLLOUT_THREADS);
  B200RL_DISPATCH_NET({
    get_actions_kernel<NetT><<<grid, ROLLOUT_THREADS, 0, (cudaStream_t)stream>>>(
        params_f32, lms, obs, n, eps, seed, iter, row, lane0, act_out, mean_out, log_std_out);
  });
  B200RL_LAUNCH_CHECK("get_actions_kernel");
  return 0;
}

int b200rl_rollout(int env_kind, const float* params_f32, int h1, int h2, float min_std, int N, int T,
                   int max_path_length, const float* eps, const float* reset_raw, unsigned int seed,
                   unsigned int iter, long long lane0, float* obs, float* act, float* mean, float* rew,
                   unsigned char* flags, unsigned short* tstep, float* log_std_out, void* stream) {
  B200RL_REQUIRE(params_f32 && obs && act && mean && rew && flags && tstep && log_std_out, "rollout: null buffer");
  B200RL_REQUIRE(N > 0 && T > 0 && max_path_length > 0, "rollout: N, T, max_path_length must be positive");
  B200RL_REQUIRE(max_path_length <= 65535, "rollout: max_path_length must fit uint16 tstep");
  B200RL_REQUIRE(h1 == h2, "rollout: hidden sizes must be equal (32,32) or (64,64)");
  RolloutArgs a;
  a.params = params_f32;
  a.log_min_std = min_std > 0.f ? logf(min_std) : -INFINITY;
  a.N = N; a.T = T; a.max_path_length = max_path_length;
  a.eps = eps; a.reset_raw = reset_raw;
  a.seed = seed; a.iter = iter; a.lane0 = lane0;
  a.obs = obs; a.act = act; a.mean = mean; a.rew = rew; a.flags = flags; a.tstep = tstep;
  a.log_std_out = log_std_out;
  B200RL_DISPATCH_ENV(env_kind, {
    int rc = launch_rollout<Env>(h1, a, (cudaStream_t)stream);
    if (rc) return rc;
  });
  return 0;
}
}
