// Policy-update passes over the sample batch: surrogate loss + KL (this file), surrogate gradient and Fisher-vector
// product (update_tile.cu for 32-wide nets, update_gemm.cu for 64-wide nets), and their C entry points.
//
// Replaces the Theano functions compiled by rllab/optimizers/conjugate_gradient_optimizer.py:184-215 (f_loss, f_grad,
// f_loss_constraint), :22-55 (PerlmutterHvp f_Hx_plain), rllab/optimizers/first_order_optimizer.py:62-76 (grad part
// of f_opt), rllab/algos/vpg.py:100-103 (f_kl), over rllab/algos/npo.py:72-82 / vpg.py:88-99 and
// rllab/distributions/diagonal_gaussian.py:14-34,58-69.
//
// Every pass is two launches: the sample kernel (per-block float64 partials) and ONE fused finalize
// (finalize_update_kernel, common.cu) that folds the partials in fixed block order, divides by the device-resident sample
// count, applies the min_std gradient mask / the reg + log_std block of the Fisher product, and reduces the
// (loss, sum KL, max KL) triple of the same pass.
#include "update_common.cuh"

namespace b200rl {

// Surrogate loss + KL, one THREAD per sample (forward only: no cross-sample reduction of per-weight quantities, so
// the thread-per-lane forward of the rollout kernel is the cheapest formulation; same canonical summation order).
constexpr int LOSS_THREADS = 128;
template <class N>
constexpr int loss_minblocks() { return (N::H1 == 32 && N::O <= 4) ? 4 : 1; }   // 128 registers: 1.47 -> 1.28 ms (A/B)
template <class N>
__global__ void __launch_bounds__(LOSS_THREADS, loss_minblocks<N>()) loss_thread_kernel(UpdArgs a) {
  constexpr int O = N::O, A = N::A;
  __shared__ __align__(16) float sp[N::P];
  __shared__ double red_scratch[3 * 32];
  for (int i = threadIdx.x; i < N::P; i += blockDim.x) sp[i] = a.params[i];
  __syncthreads();
  float ls_new[A], inv_std[A], var_new[A], var_new2[A], ls_old[A], inv_std_old[A], var_old[A];
  float sum_ls_new = 0.f, sum_ls_old = 0.f;
#pragma unroll
  for (int k = 0; k < A; ++k) {
    ls_new[k] = clamp_log_std(sp[N::ols + k], a.log_min_std);
    const float sd = expf(ls_new[k]);
    inv_std[k] = 1.0f / sd;
    var_new[k] = sd * sd;
    var_new2[k] = 2.0f * sd * sd + 1e-8f;
    ls_old[k] = a.old_log_std[k];
    const float so = expf(ls_old[k]);
    inv_std_old[k] = 1.0f / so;
    var_old[k] = so * so;
    sum_ls_new += ls_new[k];
    sum_ls_old += ls_old[k];
  }
  const float half_log2pi_A = 0.5f * (float)A * 1.8378770664093453f;
  double s_loss = 0.0, s_kl = 0.0, m_kl = -1.0e300;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < a.B; s += stride) {
    asm volatile("" ::: "memory");
    if (a.flags != nullptr && (a.flags[s] & B200RL_FLAG_MASKED)) continue;      // sample of a dropped (cut) path
    float x[O], h1[N::H1], h2[N::H2], mu[A];
#pragma unroll
    for (int o = 0; o < O; ++o) x[o] = a.obs[(size_t)o * a.B + s];
    mlp_forward_thread<N>(sp, x, h1, h2, mu);
    float zsq = 0.f, zsq_old = 0.f, kl = 0.f;
#pragma unroll
    for (int k = 0; k < A; ++k) {
      const float act = a.act[(size_t)k * a.B + s];
      const float om = a.old_mean[(size_t)k * a.B + s];
      const float z = (act - mu[k]) * inv_std[k];
      zsq += z * z;
      const float zo = (act - om) * inv_std_old[k];
      zsq_old += zo * zo;
      const float dm = om - mu[k];
      kl += (dm * dm + var_old[k] - var_new[k]) / var_new2[k] + ls_new[k] - ls_old[k];
    }
    const float adv_s = a.adv[s];
    const float logp_new = -sum_ls_new - 0.5f * zsq - half_log2pi_A;
    float term;
    if (a.loss_kind == B200RL_LOSS_TRPO) {
      const float logp_old = -sum_ls_old - 0.5f * zsq_old - half_log2pi_A;
      term = -expf(logp_new - logp_old) * adv_s;
    } else {
      term = -logp_new * adv_s;
    }
    s_loss += (double)term;
    s_kl += (double)kl;
    m_kl = fmax(m_kl, (double)kl);
  }
  double v[2] = {s_loss, s_kl};
  double mx[1] = {m_kl};
  block_reduce_store<2, false>(v, red_scratch, a.partial + (size_t)blockIdx.x * 3);
  block_reduce_store<1, true>(mx, red_scratch, a.partial + (size_t)blockIdx.x * 3 + 2);
}


// number of samples of the visited tiles that are not masked (the divisor of a sub-sampled Fisher product)
__global__ void __launch_bounds__(256) count_valid_kernel(long long B, const unsigned char* __restrict__ flags,
                                                          const int* __restrict__ tile_list, int n_list,
                                                          double* __restrict__ partial) {
  __shared__ double scratch[32];
  double c[1] = {0.0};
  const long long ntiles = tile_list ? (long long)n_list : (B + 127) / 128;
  for (long long i = blockIdx.x; i < ntiles; i += gridDim.x) {
    const long long tile = tile_list ? (long long)tile_list[i] : i;
    if (threadIdx.x < 128) {
      const long long s = tile * 128 + threadIdx.x;
      if (s < B && !(flags != nullptr && (flags[s] & B200RL_FLAG_MASKED))) c[0] += 1.0;
    }
  }
  block_reduce_store<1, false>(c, scratch, partial + blockIdx.x);
}

}  // namespace b200rl

using namespace b200rl;

static void fill_args(UpdArgs& a, const float* params, float min_std, long long B, const float* obs, const float* act,
                      const float* adv, const float* old_mean, const float* old_log_std, int loss_kind,
                      const unsigned char* flags, double* ws) {
  a.params = params; a.log_min_std = min_std > 0.f ? logf(min_std) : -INFINITY; a.B = B;
  a.obs = obs; a.act = act; a.adv = adv; a.old_mean = old_mean; a.old_log_std = old_log_std;
  a.loss_kind = loss_kind; a.flags = flags; a.partial = ws;
}

extern "C" {

int b200rl_loss_kl(int loss_kind, const float* params_f32, int obs_dim, int h1, int h2, int act_dim, float min_std,
                   long long B, const float* obs, const float* act, const float* adv, const float* old_mean,
                   const float* old_log_std, const unsigned char* flags, double scale, const double* count, double* out,
                   double* ws, void* stream) {
  B200RL_REQUIRE(params_f32 && obs && act && adv && old_mean && old_log_std && out && ws && B > 0,
                 "loss_kl: bad arguments");
  B200RL_REQUIRE(loss_kind == B200RL_LOSS_TRPO || loss_kind == B200RL_LOSS_VPG, "loss_kl: bad loss kind");
  cudaStream_t st = (cudaStream_t)stream;
  UpdArgs a{};
  fill_args(a, params_f32, min_std, B, obs, act, adv, old_mean, old_log_std, loss_kind, flags, ws);
  int grid = 0;
#ifndef B200RL_AB_TILE32
  if (h1 == 32 && h2 == 32) {
    // 32-wide nets: forward-only mode of the tensor-core kernel (update_umma32.cu) -- the same forward, instruction for
    // instruction, as the gradient pass, so (loss, KL) of the two passes agree bit for bit at equal theta
    int P = 0, ols = 0;
    int rc = update_umma32_launch(MODE_LOSS, obs_dim, act_dim, a, &grid, &P, &ols, st);
    if (rc) return rc;
  } else
#endif
  {
    long long g = (long long)num_sms() * 4;
    const long long need = (B + LOSS_THREADS - 1) / LOSS_THREADS;
    if (g > need) g = need;
    if (g > MAX_PARTIAL_BLOCKS) g = MAX_PARTIAL_BLOCKS;
    grid = (int)g;
    B200RL_DISPATCH_NET({ loss_thread_kernel<NetT><<<grid, LOSS_THREADS, 0, st>>>(a); });
    B200RL_LAUNCH_CHECK("loss_thread_kernel");
  }
  FinArgs f{};
  f.partial = nullptr; f.nblocks = grid; f.K = 0; f.vec_out = nullptr;
  f.tri_partial = ws; f.NT = 3; f.tri_out = out; f.scale = scale; f.count = count; f.post = FIN_NONE;
  if (peer_fused()) f.peer = peer_next();
  return launch_finalize_update(f, st);
}

int b200rl_grad(int loss_kind, const float* params_f32, int obs_dim, int h1, int h2, int act_dim, float min_std,
                long long B, const float* obs, const float* act, const float* adv, const float* old_mean,
                const float* old_log_std, const unsigned char* flags, double scale, const double* count, double* g_out,
                double* loss_out, float* h_cache_out, double* ws, void* stream) {
  B200RL_REQUIRE(params_f32 && obs && act && adv && old_mean && old_log_std && g_out && ws && B > 0,
                 "grad: bad arguments");
  B200RL_REQUIRE(loss_kind == B200RL_LOSS_TRPO || loss_kind == B200RL_LOSS_VPG, "grad: bad loss kind");
  B200RL_REQUIRE(h1 == h2 && (h1 == 32 || h1 == 64), "grad: hidden sizes must be (32,32) or (64,64)");
  cudaStream_t st = (cudaStream_t)stream;
  UpdArgs a{};
  fill_args(a, params_f32, min_std, B, obs, act, adv, old_mean, old_log_std, loss_kind, flags, ws);
  a.h_cache = h_cache_out;
  int grid = 0, P = 0, ols = 0;
#ifdef B200RL_AB_TILE32
  int rc = (h1 == 32) ? update_tile_launch(MODE_GRAD, obs_dim, act_dim, a, &grid, &P, &ols, st)
#else
  int rc = (h1 == 32) ? update_umma32_launch(MODE_GRAD, obs_dim, act_dim, a, &grid, &P, &ols, st)
#endif
#ifdef B200RL_AB_TILE32
                      : update_gemm_launch(MODE_GRAD, obs_dim, h1, act_dim, a, &grid, &P, &ols, st);
#else
                      : update_umma64_launch(MODE_GRAD, obs_dim, act_dim, a, &grid, &P, &ols, st);
#endif
  if (rc) return rc;
  FinArgs f{};
  f.partial = ws; f.nblocks = grid; f.K = P; f.vec_out = g_out;
  f.tri_partial = ws + (size_t)grid * P; f.NT = 3; f.tri_out = loss_out;   // per-block triples follow the [grid][P] partials
  f.scale = scale; f.count = count; f.post = FIN_GRAD; f.ols = ols; f.A = act_dim;
  f.params32 = params_f32; f.log_min_std = (double)a.log_min_std;
  if (peer_fused()) f.peer = peer_next();
  return launch_finalize_update(f, st);
}

int b200rl_fvp(const float* params_f32, int obs_dim, int h1, int h2, int act_dim, float min_std, long long B,
               const float* obs, const unsigned char* flags, const double* x, double scale, const double* count,
               double reg_coeff, double diag_scale, double* Hx_out, const float* h_cache, const int* tile_list,
               int n_list, double* ws, void* stream) {
  B200RL_REQUIRE(params_f32 && obs && x && Hx_out && ws && B > 0, "fvp: bad arguments");
  B200RL_REQUIRE(h1 == h2 && (h1 == 32 || h1 == 64), "fvp: hidden sizes must be (32,32) or (64,64)");
  B200RL_REQUIRE(tile_list == nullptr || n_list > 0, "fvp: empty tile list");
  cudaStream_t st = (cudaStream_t)stream;
  UpdArgs a{};
  fill_args(a, params_f32, min_std, B, obs, nullptr, nullptr, nullptr, nullptr, B200RL_LOSS_TRPO, flags, ws);
  a.xvec = x; a.h_cache = const_cast<float*>(h_cache); a.tile_list = tile_list; a.n_list = n_list;
  int grid = 0, P = 0, ols = 0;
  // 64-wide nets with cached activations: wgmma kernel (update_umma.cu); without a cache the FP32 tiled-GEMM kernel
  // 32-wide nets with cached activations: wgmma kernel (update_umma32.cu); without a cache the FP32 tile kernel
#ifdef B200RL_AB_TILE32
  int rc = (h1 == 32) ? update_tile_launch(MODE_FVP, obs_dim, act_dim, a, &grid, &P, &ols, st)
#else
  int rc = (h1 == 32) ? ((h_cache != nullptr) ? update_umma32_launch(MODE_FVP, obs_dim, act_dim, a, &grid, &P, &ols, st)
                                              : update_tile_launch(MODE_FVP, obs_dim, act_dim, a, &grid, &P, &ols, st))
#endif
           : (h_cache != nullptr) ? update_umma64_launch(MODE_FVP, obs_dim, act_dim, a, &grid, &P, &ols, st)
                                  : update_gemm_launch(MODE_FVP, obs_dim, h1, act_dim, a, &grid, &P, &ols, st);
  if (rc) return rc;
  FinArgs f{};
  f.partial = ws; f.nblocks = grid; f.K = P; f.vec_out = Hx_out; f.tri_out = nullptr;
  f.scale = scale; f.count = count; f.post = FIN_FVP; f.ols = ols; f.A = act_dim;
  f.params32 = params_f32; f.log_min_std = (double)a.log_min_std; f.x = x; f.reg = reg_coeff; f.diag_scale = diag_scale;
  if (peer_fused()) f.peer = peer_next();
  return launch_finalize_update(f, st);
}

int b200rl_count_valid(long long B, const unsigned char* flags, const int* tile_list, int n_list, double* count_out,
                       double* ws, void* stream) {
  B200RL_REQUIRE(B > 0 && count_out && ws, "count_valid: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const long long ntiles = tile_list ? (long long)n_list : (B + 127) / 128;
  long long g = (long long)num_sms() * 4;
  if (g > ntiles) g = ntiles;
  if (g < 1) g = 1;
  count_valid_kernel<<<(unsigned)g, 256, 0, st>>>(B, flags, tile_list, n_list, ws);
  B200RL_LAUNCH_CHECK("count_valid_kernel");
  return launch_finalize_sum(ws, (int)g, 1, count_out, 1.0, st);
}
}
