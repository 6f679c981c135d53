// GaussianMLPRegressor passes (rllab/regressors/gaussian_mlp_regressor.py:20-244, the value function of
// GaussianMLPBaseline): a Net<O,32,32,1> with ReLU hidden units on normalised inputs, a Gaussian likelihood with a
// state-independent log_std, and the mean-KL trust region of PenaltyLbfgsOptimizer.
//
//   norm stats  per-column sums of obs / y over the valid samples, then sum (x - mean)^2 around the (all-reduced) mean,
//               both float64 (two passes, no sum x^2 - (sum x)^2 / n cancellation)
//   forward     thread per sample: mu(nx), normalised or denormalised (mu * y_std + y_mean)
//   loss_grad   thread per sample for forward / loss / backward (phase A), staged feature-major into the shared-memory
//               tile of tile_gram.cuh, whose TileGram accumulates the weight gradients (phase B) -- the FP32 formulation
//               of update_tile.cu with the regressor's loss in place of the surrogate
//
// Per sample, in normalised space (nx = (x - x_mean) / x_std, ny = (y - y_mean) / y_std, l = log_std, s2 = e^{2l}):
//   NLL = l + (ny - mu)^2 / (2 s2) + log(2 pi) / 2                         (diagonal_gaussian.py:58-69, A = 1)
//   KL  = ((mu_old - mu)^2 + s2_old - s2) / (2 s2 + 1e-8) + l - l_old     (diagonal_gaussian.py:14-34)
//   dNLL/dmu = -(ny - mu) / s2                 dNLL/dl = 1 - (ny - mu)^2 / s2
//   dKL/dmu  = -2 (mu_old - mu) / (2 s2 + 1e-8)
//   dKL/dl   = 1 - 2 s2 (2 s2 + 1e-8 + 2 ((mu_old - mu)^2 + s2_old - s2)) / (2 s2 + 1e-8)^2
// The objective of one evaluation is NLL + penalty * KL (penalty_lbfgs_optimizer.py:45-49).  ReLU derivative: 0 at a
// pre-activation <= 0 (h == 0), 1 above.
#include "tile_gram.cuh"

namespace b200rl {

constexpr int VF_THREADS = 128, VF_TILE = 128, VF_LD = VF_TILE + 4, VF_H = 32;
constexpr int VF_STATS_THREADS = 256;

struct VfArgs {
  long long B;
  const float *obs, *y;
  const unsigned char* flags;
  const double* stats;       // [2O+2]: x_mean (O), x_std (O), y_mean, y_std
  const float* params;       // [P] float32 shadow
  const float* mu_old;       // [B] normalised mean at theta_old, or NULL (no trust region)
  float ls_old;              // log_std at theta_old
  float penalty;
  int learn_std;
  double* partial;
};

__device__ __forceinline__ bool vf_valid(const unsigned char* flags, long long B, long long s) {
  return s < B && !(flags != nullptr && (flags[s] & B200RL_FLAG_MASKED));
}

// normalised input of sample s (float64 arithmetic, rounded once)
template <int O>
__device__ __forceinline__ void vf_load_x(const float* __restrict__ obs, const double* __restrict__ st, long long B,
                                          long long s, float (&x)[O]) {
#pragma unroll
  for (int o = 0; o < O; ++o) x[o] = (float)(((double)obs[(size_t)o * B + s] - st[o]) / st[O + o]);
}

template <int N>
__device__ __forceinline__ void relu_inplace(float (&v)[N]) {
#pragma unroll
  for (int j = 0; j < N; ++j) v[j] = fmaxf(v[j], 0.f);
}

// output unit in the canonical even/odd order of mlp.cuh
template <class N>
__device__ __forceinline__ float vf_out(const float* sp, const float (&h2)[N::H2]) {
  float s0 = sp[N::obo], s1 = 0.f;
#pragma unroll
  for (int j = 0; j < N::H2; j += 2) {
    s0 = fmaf(h2[j], sp[N::oWo + j], s0);
    s1 = fmaf(h2[j + 1], sp[N::oWo + j + 1], s1);
  }
  return s0 + s1;
}

// ---------------------------------------------------------------- normalisation statistics
// STAGE 0: partial[b][0..O] = sums of x_o and y, [O+1] = number of valid samples
// STAGE 1: partial[b][0..O] = sums of (x_o - mean_o)^2 and (y - mean_y)^2, means from acc[0..O+1]
template <int O, int STAGE>
__global__ void __launch_bounds__(VF_STATS_THREADS) vf_stats_kernel(long long B, const float* __restrict__ obs,
                                                                    const float* __restrict__ y,
                                                                    const unsigned char* __restrict__ flags,
                                                                    const double* __restrict__ acc,
                                                                    double* __restrict__ partial) {
  constexpr int K = (STAGE == 0) ? O + 2 : O + 1;
  __shared__ double scratch[K * 32];
  double v[K];
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = 0.0;
  double mean[O + 1];
  if (STAGE == 1) {
#pragma unroll
    for (int k = 0; k <= O; ++k) mean[k] = acc[k] / acc[O + 1];
  }
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < B; s += stride) {
    if (!vf_valid(flags, B, s)) continue;
#pragma unroll
    for (int k = 0; k <= O; ++k) {
      const double xv = (double)(k < O ? obs[(size_t)k * B + s] : y[s]);
      if (STAGE == 0) {
        v[k] += xv;
      } else {
        const double d = xv - mean[k];
        v[k] = fma(d, d, v[k]);
      }
    }
    if constexpr (STAGE == 0) v[O + 1] += 1.0;
  }
  block_reduce_store<K>(v, scratch, partial + (size_t)blockIdx.x * K);
}

// stats[2O+2] = [x_mean, x_std + 1e-8, y_mean, y_std + 1e-8] (population std, np.std) from the all-reduced acc
template <int O>
__global__ void vf_stats_finish_kernel(const double* __restrict__ acc, double* __restrict__ stats) {
  const int k = threadIdx.x;
  if (k > O) return;
  const double n = acc[O + 1];
  const double m = acc[k] / n, sd = sqrt(acc[O + 2 + k] / n) + 1e-8;
  if (k < O) {
    stats[k] = m;
    stats[O + k] = sd;
  } else {
    stats[2 * O] = m;
    stats[2 * O + 1] = sd;
  }
}

template <int O>
static int vf_norm_stats_run(long long B, const float* obs, const float* y, const unsigned char* flags, int stage,
                             double* acc, double* stats, double* ws, cudaStream_t st) {
  const int g = partial_grid(4, (B + VF_STATS_THREADS - 1) / VF_STATS_THREADS);
  if (stage == 0 || stage == 3) {
    vf_stats_kernel<O, 0><<<g, VF_STATS_THREADS, 0, st>>>(B, obs, y, flags, acc, ws);
    B200RL_LAUNCH_CHECK("vf_stats_kernel<0>");
    int rc = launch_finalize_sum(ws, g, O + 2, acc, 1.0, st);
    if (rc) return rc;
  }
  if (stage == 1 || stage == 3) {
    vf_stats_kernel<O, 1><<<g, VF_STATS_THREADS, 0, st>>>(B, obs, y, flags, acc, ws);
    B200RL_LAUNCH_CHECK("vf_stats_kernel<1>");
    int rc = launch_finalize_sum(ws, g, O + 1, acc + O + 2, 1.0, st);
    if (rc) return rc;
  }
  if (stage == 2 || stage == 3) {
    vf_stats_finish_kernel<O><<<1, 32, 0, st>>>(acc, stats);
    B200RL_LAUNCH_CHECK("vf_stats_finish_kernel");
  }
  return 0;
}

// ---------------------------------------------------------------- forward / predict
template <class N>
__global__ void __launch_bounds__(256) vf_forward_kernel(const float* __restrict__ params, long long B,
                                                         const float* __restrict__ obs, const double* __restrict__ stats,
                                                         int denorm, float* __restrict__ out) {
  constexpr int O = N::O, P = N::P;
  __shared__ __align__(16) float sp[(P + 3) & ~3];
  for (int i = threadIdx.x; i < P; i += blockDim.x) sp[i] = params[i];
  __syncthreads();
  const double y_mean = stats[2 * O], y_std = stats[2 * O + 1];
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < B; s += stride) {
    // compiler barriers: without them ptxas hoists the loop-invariant weight loads out of the loop and spills ~5 KB
    asm volatile("" ::: "memory");
    float x[O], h1[VF_H], h2[VF_H];
    vf_load_x<O>(obs, stats, B, s, x);
    dense_thread<O, VF_H>(sp + N::oW0, sp + N::ob0, x, h1);
    relu_inplace(h1);
    asm volatile("" ::: "memory");
    dense_thread<VF_H, VF_H>(sp + N::oW1, sp + N::ob1, h1, h2);
    relu_inplace(h2);
    const float mu = vf_out<N>(sp, h2);
    out[s] = denorm ? (float)((double)mu * y_std + y_mean) : mu;
  }
}

// ---------------------------------------------------------------- loss (+ gradient)
template <class N>
struct VfSmem {
  static constexpr int O = N::O, H = VF_H;
  static constexpr int rX = 0, rH1 = rX + O, rH2 = rH1 + H, rD1 = rH2 + H, rD2 = rD1 + H, rDM = rD2 + H, rDL = rDM + 1,
                       R = rDL + 1;
  static constexpr int P4 = (N::P + 3) & ~3;
  static constexpr int o_stage = P4;
  static constexpr int n_floats = o_stage + R * VF_LD;
  static constexpr int scratch_off = ((n_floats * 4 + 15) / 16) * 16;
  static constexpr size_t bytes = (size_t)scratch_off + 3 * 32 * 8;
  static_assert(2 * 64 * 16 * 8 <= R * VF_LD * 4, "stage region must hold the K-half combine scratch");
};

// GRAD = false: forward and loss sums only (no staging, no Gram phase)
template <class N, bool GRAD>
__global__ void __launch_bounds__(VF_THREADS, 2) vf_loss_grad_kernel(VfArgs a) {
  using SM = VfSmem<N>;
  constexpr int O = N::O, H = VF_H, P = N::P, LD = VF_LD;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* sp = reinterpret_cast<float*>(smem_raw);
  float* stage = sp + SM::o_stage;
  double* red_scratch = reinterpret_cast<double*>(smem_raw + SM::scratch_off);
  const int tid = threadIdx.x;
  for (int i = tid; i < P; i += VF_THREADS) sp[i] = a.params[i];
  __syncthreads();

  const double y_mean = a.stats[2 * O], y_std = a.stats[2 * O + 1];
  const float ls = sp[N::ols];
  const float var = expf(2.0f * ls), inv_var = 1.0f / var;
  const float var2 = 2.0f * var + 1e-8f;
  const float var_old = expf(2.0f * a.ls_old);
  const bool trust = a.mu_old != nullptr;
  const float half_log2pi = 0.5f * 1.8378770664093453f;

  TileGram<N, SM::rX, SM::rH1, SM::rH2, SM::rD1, SM::rD2, SM::rDM, LD> gram;
  if (GRAD) gram.init();
  double s_nll = 0.0, s_kl = 0.0, m_kl = -1.0e300;

  float* colX = stage + SM::rX * LD + tid;
  float* colH1 = stage + SM::rH1 * LD + tid;
  float* colH2 = stage + SM::rH2 * LD + tid;
  float* colD1 = stage + SM::rD1 * LD + tid;
  float* colD2 = stage + SM::rD2 * LD + tid;
  float* colDM = stage + SM::rDM * LD + tid;
  float* colDL = stage + SM::rDL * LD + tid;

  const long long ntiles = (a.B + VF_TILE - 1) / VF_TILE;
  for (long long ti = blockIdx.x; ti < ntiles; ti += gridDim.x) {
    asm volatile("" ::: "memory");
    const long long s_raw = ti * VF_TILE + tid;
    const bool valid = vf_valid(a.flags, a.B, s_raw);
    const long long s = s_raw < a.B ? s_raw : a.B - 1;
    // ================= phase A: forward, loss, output deltas, backward
    float mu;
    {
      float x[O], h1[H], h2[H];
      vf_load_x<O>(a.obs, a.stats, a.B, s, x);
      if (GRAD) {
#pragma unroll
        for (int o = 0; o < O; ++o) colX[o * LD] = x[o];
      }
      dense_thread<O, H>(sp + N::oW0, sp + N::ob0, x, h1);
      relu_inplace(h1);
      if (GRAD) {
#pragma unroll
        for (int j = 0; j < H; ++j) colH1[j * LD] = h1[j];
      }
      dense_thread<H, H>(sp + N::oW1, sp + N::ob1, h1, h2);
      relu_inplace(h2);
      if (GRAD) {
#pragma unroll
        for (int j = 0; j < H; ++j) colH2[j * LD] = h2[j];
      }
      mu = vf_out<N>(sp, h2);
    }
    asm volatile("" ::: "memory");   // keep the smem weights from staying live in registers
    const float ny = (float)(((double)a.y[s] - y_mean) / y_std);
    const float r = ny - mu;
    const float rsq = __fmul_rn(r, r);
    const float nll = ls + 0.5f * rsq * inv_var + half_log2pi;
    float dmu = -r * inv_var;
    float dls = 1.0f - rsq * inv_var;
    float kl = 0.f;
    if (trust) {
      const float dm = a.mu_old[s] - mu;
      const float num = __fmul_rn(dm, dm) + var_old - var;
      kl = num / var2 + ls - a.ls_old;
      dmu = fmaf(a.penalty, -2.0f * dm / var2, dmu);
      dls = fmaf(a.penalty, 1.0f - 2.0f * var * (var2 + 2.0f * num) / (var2 * var2), dls);
    }
    if (valid) {
      s_nll += (double)nll;
      if (trust) {
        s_kl += (double)kl;
        m_kl = fmax(m_kl, (double)kl);
      }
    } else {
      dmu = 0.f;
      dls = 0.f;
    }
    if (GRAD) {
      colDM[0] = dmu;
      colDL[0] = a.learn_std ? dls : 0.f;
      // backward: d2 = dmu Wout^T (h2 > 0); d1 = (d2 W1^T) (h1 > 0)
      float d2[H];
#pragma unroll
      for (int j = 0; j < H; ++j) {
        d2[j] = colH2[j * LD] > 0.f ? dmu * sp[N::oWo + j] : 0.f;
        colD2[j * LD] = d2[j];
      }
#pragma unroll
      for (int i = 0; i < H; ++i) {
        float2 acc = make_float2(0.f, 0.f);
#pragma unroll
        for (int j = 0; j < H; j += 4) {
          const float4 w = *reinterpret_cast<const float4*>(sp + N::oW1 + i * H + j);
          acc = ffma2(make_float2(d2[j], d2[j + 1]), make_float2(w.x, w.y), acc);
          acc = ffma2(make_float2(d2[j + 2], d2[j + 3]), make_float2(w.z, w.w), acc);
        }
        colD1[i * LD] = colH1[i * LD] > 0.f ? acc.x + acc.y : 0.f;
      }
      __syncthreads();
      // ================= phase B: Gram accumulation over the tile (tile_gram.cuh)
      gram.accumulate_a(stage, tid);
      gram.accumulate_b(stage, tid);
      __syncthreads();
    }
  }

  double* tri = a.partial + (GRAD ? (size_t)gridDim.x * P : 0) + (size_t)blockIdx.x * 3;
  if (GRAD) {
    gram.write(a.partial + (size_t)blockIdx.x * P, reinterpret_cast<double*>(stage), tid);
    __syncthreads();
  }
  double v[2] = {s_nll, s_kl};
  double mx[1] = {m_kl};
  block_reduce_store<2, false>(v, red_scratch, tri);
  block_reduce_store<1, true>(mx, red_scratch, tri + 2);
}

template <class N, bool GRAD>
static int vf_launch_loss_grad(const VfArgs& a, int* grid_out, cudaStream_t st) {
  using SM = VfSmem<N>;
  B200RL_SET_MAX_SMEM((vf_loss_grad_kernel<N, GRAD>), SM::bytes);
  int per_sm = (int)((228 * 1024) / (SM::bytes + 1024));
  if (per_sm < 1) per_sm = 1;
  if (per_sm > 2) per_sm = 2;
  const int grid = partial_grid(per_sm, (a.B + VF_TILE - 1) / VF_TILE);
  vf_loss_grad_kernel<N, GRAD><<<grid, VF_THREADS, SM::bytes, st>>>(a);
  B200RL_LAUNCH_CHECK("vf_loss_grad_kernel");
  *grid_out = grid;
  return 0;
}

// The regressor nets: the obs dims of the compiled envs, hidden (32,32), one output.
#define B200RL_VF_DISPATCH_O(O_, ...)                 \
  if (obs_dim == O_) {                                \
    using NetT = ::b200rl::Net<O_, 32, 32, 1>;        \
    __VA_ARGS__;                                      \
  } else
#define B200RL_VF_DISPATCH(...)                                                                        \
  B200RL_VF_DISPATCH_O(2, __VA_ARGS__)                                                                 \
  B200RL_VF_DISPATCH_O(3, __VA_ARGS__)                                                                 \
  B200RL_VF_DISPATCH_O(4, __VA_ARGS__)                                                                 \
  B200RL_VF_DISPATCH_O(6, __VA_ARGS__)                                                                 \
  B200RL_VF_DISPATCH_O(13, __VA_ARGS__)                                                                \
  B200RL_VF_DISPATCH_O(20, __VA_ARGS__)                                                                \
  {                                                                                                    \
    ::b200rl::set_error("regressor shape O=%d hidden=(%d,%d) is not compiled in", obs_dim, h1, h2);    \
    return B200RL_EUNSUPPORTED;                                                                        \
  }

}  // namespace b200rl

using namespace b200rl;

extern "C" {

long long b200rl_vf_num_params(int obs_dim, int h1, int h2) {
  if (h1 != 32 || h2 != 32) {
    set_error("regressor hidden sizes (%d,%d) are not compiled in (only (32,32))", h1, h2);
    return B200RL_EUNSUPPORTED;
  }
  B200RL_VF_DISPATCH({ return (long long)NetT::P; });
}

int b200rl_vf_norm_stats(int obs_dim, long long B, const float* obs, const float* y, const unsigned char* flags,
                         int stage, double* acc, double* stats_out, double* ws, void* stream) {
  B200RL_REQUIRE(obs && y && acc && ws && B > 0 && stage >= 0 && stage <= 3, "vf_norm_stats: bad arguments");
  B200RL_REQUIRE(stats_out || (stage != 2 && stage != 3), "vf_norm_stats: stats_out is NULL");
  const int h1 = 32, h2 = 32;
  cudaStream_t st = (cudaStream_t)stream;
  B200RL_VF_DISPATCH({ return vf_norm_stats_run<NetT::O>(B, obs, y, flags, stage, acc, stats_out, ws, st); });
}

int b200rl_vf_forward(const float* params_f32, int obs_dim, int h1, int h2, long long B, const float* obs,
                      const double* stats, int denormalize, float* out, void* stream) {
  B200RL_REQUIRE(params_f32 && obs && stats && out && B > 0, "vf_forward: bad arguments");
  B200RL_REQUIRE(h1 == 32 && h2 == 32, "vf_forward: hidden sizes must be (32,32)");
  cudaStream_t st = (cudaStream_t)stream;
  long long g = (B + 255) / 256;
  const long long cap = (long long)num_sms() * 8;
  if (g > cap) g = cap;
  B200RL_VF_DISPATCH({
    vf_forward_kernel<NetT><<<(unsigned)g, 256, 0, st>>>(params_f32, B, obs, stats, denormalize, out);
    B200RL_LAUNCH_CHECK("vf_forward_kernel");
  });
  return 0;
}

int b200rl_vf_loss_grad(const float* params_f32, int obs_dim, int h1, int h2, long long B, const float* obs,
                        const float* y, const unsigned char* flags, const double* stats, const float* mu_old,
                        float old_log_std, double penalty, int learn_std, double scale, const double* count,
                        double* g_out, double* loss_out, double* ws, void* stream) {
  B200RL_REQUIRE(params_f32 && obs && y && stats && ws && B > 0, "vf_loss_grad: bad arguments");
  B200RL_REQUIRE(g_out || loss_out, "vf_loss_grad: neither g_out nor loss_out");
  B200RL_REQUIRE(h1 == 32 && h2 == 32, "vf_loss_grad: hidden sizes must be (32,32)");
  cudaStream_t st = (cudaStream_t)stream;
  VfArgs a{};
  a.B = B; a.obs = obs; a.y = y; a.flags = flags; a.stats = stats; a.params = params_f32; a.mu_old = mu_old;
  a.ls_old = old_log_std; a.penalty = (float)penalty; a.learn_std = learn_std; a.partial = ws;
  int grid = 0, P = 0;
  B200RL_VF_DISPATCH({
    P = NetT::P;
    int rc = g_out ? vf_launch_loss_grad<NetT, true>(a, &grid, st) : vf_launch_loss_grad<NetT, false>(a, &grid, st);
    if (rc) return rc;
  });
  // the regressor has no log_std block: the gradient's min_std mask touches no entry
  return launch_finalize_update(fin_grad(ws, grid, g_out ? P : 0, g_out, loss_out, scale, count, {}), st);
}

}  // extern "C"
