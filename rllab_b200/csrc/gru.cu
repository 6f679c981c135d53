// GaussianGRUPolicy on the lane batch (rllab/policies/gaussian_gru_policy.py, rllab/core/network.py:104-270 GRULayer /
// GRUNetwork, rllab/distributions/recurrent_diagonal_gaussian.py): the fused recurrent rollout, get_actions with an
// explicit hidden state, and the loss/KL, backpropagation-through-time gradient (+ KL penalty) and Fisher-vector passes,
// in float32 and in a float64 parity mode.
//
// Net (GRULayer.step, hidden_nonlinearity tanh, gate nonlinearity sigmoid):
//   x_t = [obs_t, prev_action_t] (state_include_action) or obs_t
//   r = sigma(x W_xr + h W_hr + b_r);  u = sigma(x W_xu + h W_hu + b_u);  c = tanh(x W_xc + r * (h W_hc) + b_c)
//   h' = (1 - u) h + u c;  mean = h' W_out + b_out;  log_std a state-independent parameter.
// h_0 = 0 (hidden_init_trainable=False) and prev_action_0 = 0 at every path start (tstep == 0); afterwards prev_action is
// the previous raw sampled action act[t-1] of the lane, before NormalizedEnv scales it.
// Flat layout (LasagnePowered over [l_mean, l_log_std], trainable parameters in add_param order):
//   [W_xr (I x H), W_hr (H x H), b_r, W_xu, W_hu, b_u, W_xc, W_hc, b_c, W_out (H x A), b_out (A), log_std (A)].
// Compiled for CartPole (obs 4, action 1), H = 32, state_include_action in {0, 1}.
//
// Lanes are time-major [T][N] (b200rl_rollout's planes).  The loss/KL pass runs one thread per lane over t = 0..T-1 with
// the rollout's own cell (gru_cell), so mean(theta_old) is bit-identical to the recorded one: likelihood ratio exactly 1,
// KL exactly 0.  The gradient and Fisher passes run a CTA of 128 lanes: a forward sweep writes h_t [H][T][N] (the
// activation cache), then a backward sweep over t = T-1..0 carries dh from step to step (cut where a path starts) and
// stages each step's 128 samples feature-major in shared memory; every weight-gradient entry is a Gram product over that
// tile, float32 inside the tile and float64 across tiles, each entry owned by one thread (fixed order, no atomics).
// Per-block partials go through launch_finalize_update, so the min_std mask, the log_std block of the Fisher product and
// the fused peer exchange are the Gaussian passes'.
#include "envs.cuh"
#include "update_common.cuh"

namespace b200rl {

constexpr int GRU_H = 32;

template <int O_, int A_, int INC>
struct GruNet {
  static constexpr int O = O_, A = A_, H = GRU_H, I = O_ + (INC ? A_ : 0);
  static constexpr int G = I * H + H * H + H;   // one gate block: W_x, W_h, b
  static constexpr int oWo = 3 * G, obo = oWo + H * A, ols = obo + A, P = ols + A, P4 = (P + 3) & ~3;
  __host__ __device__ static constexpr int oWx(int g) { return g * G; }
  __host__ __device__ static constexpr int oWh(int g) { return g * G + I * H; }
  __host__ __device__ static constexpr int ob(int g) { return g * G + I * H + H * H; }
};

inline bool gru_supported(int O, int H, int A) { return O == 4 && H == GRU_H && A == 1; }
#define B200RL_REQUIRE_GRU_SHAPE(O_, H_, A_, what)                                                                 \
  do {                                                                                                             \
    if (!gru_supported(O_, H_, A_)) {                                                                              \
      set_error("%s: GRU net obs_dim=%d hidden=%d act_dim=%d is not compiled in (only obs 4, hidden 32, act 1)", \
                what, (int)(O_), (int)(H_), (int)(A_));                                                            \
      return B200RL_EUNSUPPORTED;                                                                                  \
    }                                                                                                              \
  } while (0)
// dispatch on state_include_action for the one compiled (O, A)
#define B200RL_DISPATCH_GRU(inc, ...)                   \
  if (inc) {                                            \
    using NetG = ::b200rl::GruNet<4, 1, 1>;             \
    __VA_ARGS__;                                        \
  } else {                                              \
    using NetG = ::b200rl::GruNet<4, 1, 0>;             \
    __VA_ARGS__;                                        \
  }

__device__ __forceinline__ float sigm_f(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ double sigm_d(double x) { return 1.0 / (1.0 + exp(-x)); }

// One GRU step of one lane, column by column: for hidden unit j, the three pre-activations and (h W_hc)_j from the old
// h, then h'_j.  Shared by the rollout, get_actions and every float32 update pass (bit-identical h at equal theta).
template <class N>
__device__ __forceinline__ void gru_cell(const float* __restrict__ sp, const float (&x)[N::I], const float (&h)[N::H],
                                         float (&hn)[N::H]) {
  constexpr int I = N::I, H = N::H;
#pragma unroll
  for (int j = 0; j < H; ++j) {
    float ar = sp[N::ob(0) + j], au = sp[N::ob(1) + j], ac = sp[N::ob(2) + j], hc = 0.f;
#pragma unroll
    for (int i = 0; i < I; ++i) {
      ar = fmaf(x[i], sp[N::oWx(0) + i * H + j], ar);
      au = fmaf(x[i], sp[N::oWx(1) + i * H + j], au);
      ac = fmaf(x[i], sp[N::oWx(2) + i * H + j], ac);
    }
#pragma unroll
    for (int k = 0; k < H; ++k) {
      ar = fmaf(h[k], sp[N::oWh(0) + k * H + j], ar);
      au = fmaf(h[k], sp[N::oWh(1) + k * H + j], au);
      hc = fmaf(h[k], sp[N::oWh(2) + k * H + j], hc);
    }
    const float r = sigm_f(ar), u = sigm_f(au);
    const float c = tanh_f(fmaf(r, hc, ac));
    hn[j] = fmaf(u, c - h[j], h[j]);   // (1 - u) h + u c
  }
}

template <class N>
__device__ __forceinline__ void gru_mean(const float* __restrict__ sp, const float (&hn)[N::H], float (&mu)[N::A]) {
#pragma unroll
  for (int a = 0; a < N::A; ++a) {
    float s0 = sp[N::obo + a], s1 = 0.f;
#pragma unroll
    for (int j = 0; j < N::H; j += 2) {
      s0 = fmaf(hn[j], sp[N::oWo + j * N::A + a], s0);
      s1 = fmaf(hn[j + 1], sp[N::oWo + (j + 1) * N::A + a], s1);
    }
    mu[a] = s0 + s1;
  }
}

// x_t = [obs_t, prev_action_t]: prev_action is act[t-1] of the lane inside a path and 0 at its first step
template <class N>
__device__ __forceinline__ void gru_input(const float* __restrict__ obs, const float* __restrict__ act, size_t B,
                                          size_t idx, size_t N_, bool start, float (&x)[N::I]) {
#pragma unroll
  for (int o = 0; o < N::O; ++o) x[o] = obs[(size_t)o * B + idx];
#pragma unroll
  for (int a = 0; a < N::I - N::O; ++a) x[N::O + a] = start ? 0.f : act[(size_t)a * B + idx - N_];
}

// ------------------------------------------------------------------------------------------------ rollout / get_actions
// One thread per lane for all T steps (lane_rollout, envs.cuh): env state, h and prev_action in registers.
template <class Env, class N_>
__global__ void __launch_bounds__(128) gru_rollout_kernel(RolloutArgs a) {
  static_assert(Env::O == N_::O && Env::A == N_::A, "env and GRU net disagree");
  constexpr int H = N_::H, A = N_::A;
  __shared__ __align__(16) float sp[N_::P4];
  for (int i = threadIdx.x; i < N_::P; i += blockDim.x) sp[i] = a.params[i];
  __syncthreads();
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  float std_[A];
#pragma unroll
  for (int k = 0; k < A; ++k) {
    std_[k] = expf(sp[N_::ols + k]);
    if (n == 0) a.log_std_out[k] = sp[N_::ols + k];
  }
  if (n >= a.N) return;
  const long long lane = a.lane0 + n;
  float h[H], pa[A], hn[H], mu[A], e[A];
  lane_rollout<Env>(
      a, n,
      [&](int t, int plen, const float (&o)[Env::O]) {
        if (plen == 0) {   // path start: h_0 = 0, prev_action = 0
#pragma unroll
          for (int j = 0; j < H; ++j) h[j] = 0.f;
#pragma unroll
          for (int k = 0; k < A; ++k) pa[k] = 0.f;
        }
        float x[N_::I];
#pragma unroll
        for (int k = 0; k < Env::O; ++k) x[k] = o[k];
#pragma unroll
        for (int k = 0; k < N_::I - N_::O; ++k) x[N_::O + k] = pa[k];
        gru_cell<N_>(sp, x, h, hn);
        gru_mean<N_>(sp, hn, mu);
        draw_eps<A>(e, a.eps, t, a.N, n, a.seed, a.iter, lane);
      },
      [&](size_t idx, size_t TN, float (&u)[A]) {
#pragma unroll
        for (int k = 0; k < A; ++k) {
          pa[k] = fmaf(std_[k], e[k], mu[k]);   // rnd * exp(log_std) + mean (gaussian_gru_policy.py:get_action)
          u[k] = scale_action(pa[k], Env::lb(k), Env::ub(k));
          a.act[k * TN + idx] = pa[k];
          a.mean[k * TN + idx] = mu[k];
        }
#pragma unroll
        for (int j = 0; j < H; ++j) h[j] = hn[j];
      });
}

template <class N_>
__global__ void __launch_bounds__(128) gru_get_actions_kernel(const float* __restrict__ params,
                                                              const float* __restrict__ obs,
                                                              const float* __restrict__ prev_action,
                                                              const float* __restrict__ h_in, long long n_,
                                                              const float* __restrict__ eps, uint32_t seed,
                                                              uint32_t iter, int row, long long lane0,
                                                              float* __restrict__ act_out, float* __restrict__ mean_out,
                                                              float* __restrict__ h_out, float* __restrict__ log_std_out) {
  constexpr int H = N_::H, A = N_::A;
  __shared__ __align__(16) float sp[N_::P4];
  for (int i = threadIdx.x; i < N_::P; i += blockDim.x) sp[i] = params[i];
  __syncthreads();
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n == 0)
    for (int k = 0; k < A; ++k) log_std_out[k] = sp[N_::ols + k];
  if (n >= n_) return;
  float x[N_::I], h[H], hn[H], mu[A], e[A];
#pragma unroll
  for (int k = 0; k < N_::O; ++k) x[k] = obs[(size_t)k * n_ + n];
#pragma unroll
  for (int k = 0; k < N_::I - N_::O; ++k) x[N_::O + k] = prev_action ? prev_action[(size_t)k * n_ + n] : 0.f;
#pragma unroll
  for (int j = 0; j < H; ++j) h[j] = h_in ? h_in[(size_t)j * n_ + n] : 0.f;
  gru_cell<N_>(sp, x, h, hn);
  gru_mean<N_>(sp, hn, mu);
  if (eps != nullptr) {
#pragma unroll
    for (int k = 0; k < A; ++k) e[k] = eps[(size_t)k * n_ + n];
  } else {
    draw_eps<A>(e, nullptr, row, n_, n, seed, iter, lane0 + n);
  }
#pragma unroll
  for (int k = 0; k < A; ++k) {
    act_out[(size_t)k * n_ + n] = fmaf(expf(sp[N_::ols + k]), e[k], mu[k]);
    mean_out[(size_t)k * n_ + n] = mu[k];
  }
#pragma unroll
  for (int j = 0; j < H; ++j) h_out[(size_t)j * n_ + n] = hn[j];
}

// ------------------------------------------------------------------------------------------------ per-sample terms
struct GruArgs {
  const float* params;
  const double* xvec;         // FVP: tangent vector (float64, P)
  float* hbuf;                // [H][T][N] h_t after step t: written by the forward sweep, read back by the backward one
  int h_valid;                // FVP: hbuf already holds h at these params (written by the gradient pass)
  float* plane;               // FVP: [A][T][N] scratch, M * (J x) per sample
  int N, T;
  long long B;
  const float *obs, *act, *adv, *old_mean, *old_log_std;
  const unsigned short* tstep;
  int loss_kind;
  float penalty;
  const unsigned char* flags;
  double* partial;
};

template <int A>
struct GruDist {
  float ls_new[A], inv_std[A], var_new[A], var_new2[A], ls_old[A], inv_std_old[A], var_old[A], Mmu[A];
  float sum_ls_new, sum_ls_old, half_log2pi_A;
  __device__ void init(const float* ls_param, const float* old_log_std) {
    sum_ls_new = 0.f;
    sum_ls_old = 0.f;
#pragma unroll
    for (int k = 0; k < A; ++k) {
      ls_new[k] = ls_param[k];
      const float sd = expf(ls_new[k]);
      inv_std[k] = 1.0f / sd;
      var_new[k] = sd * sd;
      var_new2[k] = 2.0f * sd * sd + 1e-8f;
      Mmu[k] = 2.0f / var_new2[k];
      ls_old[k] = old_log_std ? old_log_std[k] : ls_new[k];
      const float so = expf(ls_old[k]);
      inv_std_old[k] = 1.0f / so;
      var_old[k] = so * so;
      sum_ls_new += ls_new[k];
      sum_ls_old += ls_old[k];
    }
    half_log2pi_A = 0.5f * (float)A * 1.8378770664093453f;
  }
};

// Surrogate term, KL and the output deltas (d term / d mean, d term / d log_std) of one sample: the arithmetic of
// loss_thread_kernel / tile_phase_a (npo.py:72-82, vpg.py:88-99 over diagonal_gaussian.py), + penalty * d kl.
template <int A>
__device__ __forceinline__ void gru_terms(const GruArgs& a, const GruDist<A>& D, size_t idx, const float (&mu)[A],
                                          float& term, float& kl, float (&dmu)[A], float (&dls)[A]) {
  float z[A], zsq = 0.f, zsq_old = 0.f, dm[A];
  kl = 0.f;
#pragma unroll
  for (int k = 0; k < A; ++k) {
    const float act = a.act[(size_t)k * a.B + idx];
    const float om = a.old_mean[(size_t)k * a.B + idx];
    z[k] = (act - mu[k]) * D.inv_std[k];
    zsq += z[k] * z[k];
    const float zo = (act - om) * D.inv_std_old[k];
    zsq_old += zo * zo;
    dm[k] = om - mu[k];
    kl += (dm[k] * dm[k] + D.var_old[k] - D.var_new[k]) / D.var_new2[k] + D.ls_new[k] - D.ls_old[k];
  }
  const float adv_s = a.adv[idx];
  const float logp_new = -D.sum_ls_new - 0.5f * zsq - D.half_log2pi_A;
  float w_s;
  if (a.loss_kind == B200RL_LOSS_TRPO) {
    const float logp_old = -D.sum_ls_old - 0.5f * zsq_old - D.half_log2pi_A;
    w_s = expf(logp_new - logp_old) * adv_s;
    term = -w_s;
  } else {
    w_s = adv_s;
    term = -logp_new * adv_s;
  }
#pragma unroll
  for (int k = 0; k < A; ++k) {
    dmu[k] = -w_s * z[k] * D.inv_std[k];
    dls[k] = -w_s * (z[k] * z[k] - 1.0f);
    if (a.penalty > 0.f) add_kl_penalty(a.penalty, dm[k], D.var_new[k], D.var_new2[k], D.var_old[k], dmu[k], dls[k]);
  }
}

__device__ __forceinline__ bool gru_masked(const GruArgs& a, size_t idx) {
  return a.flags != nullptr && (a.flags[idx] & B200RL_FLAG_MASKED);
}

// ------------------------------------------------------------------------------------------------ loss / KL
// One thread per lane over t = 0..T-1 (forward only); h_cache (optional) receives h_t.
template <class N_>
__global__ void __launch_bounds__(128) gru_loss_kernel(GruArgs a) {
  constexpr int H = N_::H, A = N_::A;
  __shared__ __align__(16) float sp[N_::P4];
  __shared__ double red_scratch[3 * 32];
  for (int i = threadIdx.x; i < N_::P; i += blockDim.x) sp[i] = a.params[i];
  __syncthreads();
  GruDist<A> D;
  D.init(sp + N_::ols, a.old_log_std);
  double s_loss = 0.0, s_kl = 0.0, m_kl = -1.0e300;
  const int stride = gridDim.x * blockDim.x;
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < a.N; n += stride) {
    float h[H];
    for (int t = 0; t < a.T; ++t) {
      asm volatile("" ::: "memory");
      const size_t idx = (size_t)t * a.N + n;
      const bool start = a.tstep[idx] == 0;
      if (start) {
#pragma unroll
        for (int j = 0; j < H; ++j) h[j] = 0.f;
      }
      float x[N_::I], hn[H], mu[A];
      gru_input<N_>(a.obs, a.act, a.B, idx, a.N, start, x);
      gru_cell<N_>(sp, x, h, hn);
      gru_mean<N_>(sp, hn, mu);
#pragma unroll
      for (int j = 0; j < H; ++j) {
        h[j] = hn[j];
        if (a.hbuf) a.hbuf[(size_t)j * a.B + idx] = hn[j];
      }
      if (gru_masked(a, idx)) continue;
      float term, kl, dmu[A], dls[A];
      gru_terms<A>(a, D, idx, mu, term, kl, dmu, dls);
      s_loss += (double)term;
      s_kl += (double)kl;
      m_kl = fmax(m_kl, (double)kl);
    }
  }
  double v[2] = {s_loss, s_kl};
  double mx[1] = {m_kl};
  block_reduce_store<2, false>(v, red_scratch, a.partial + (size_t)blockIdx.x * 3);
  block_reduce_store<1, true>(mx, red_scratch, a.partial + (size_t)blockIdx.x * 3 + 2);
}

// ------------------------------------------------------------------------------------------------ BPTT (float32)
constexpr int GT = 128, GLD = GT + 1;   // 128 lanes per CTA; odd stride: the Gram's row reads spread over the banks

template <class N_>
struct GruStage {
  static constexpr int I = N_::I, H = N_::H, A = N_::A;
  static constexpr int rX = 0, rHp = rX + I, rOne = rHp + H, rD = rOne + 1 /* Dr, Du, Dc */, rDhc = rD + 3 * H,
                       rHn = rDhc + H, rDM = rHn + H, rDL = rDM + A, R = rDL + A;
  static constexpr int o_sp = 0, o_sv = N_::P4, o_stage = 2 * N_::P4;
  static constexpr int acc_off = (((o_stage + R * GLD) * 4 + 15) / 16) * 16;   // bytes
  static constexpr int red_off = acc_off + N_::P * 8;
  static constexpr size_t bytes = (size_t)red_off + 3 * 32 * 8;

  // Gram operands of parameter entry e: dtheta_e = sum over the tile of stage[ra][s] * stage[rb][s]
  __device__ static void rows(int e, int& ra, int& rb) {
    if (e < 3 * N_::G) {
      const int g = e / N_::G, k = e - g * N_::G;
      if (k < I * H) {
        ra = rX + k / H; rb = rD + g * H + k % H;
      } else if (k < I * H + H * H) {
        const int kk = k - I * H;
        ra = rHp + kk / H; rb = (g == 2 ? rDhc : rD + g * H) + kk % H;
      } else {
        ra = rOne; rb = rD + g * H + (k - I * H - H * H);
      }
    } else if (e < N_::ols) {
      const int k = e - N_::oWo;
      if (k < H * A) { ra = rHn + k / A; rb = rDM + k % A; }
      else { ra = rOne; rb = rDM + (k - H * A); }
    } else {
      ra = rOne; rb = rDL + (e - N_::ols);
    }
  }
};

// Forward sweep of one lane: h_t into hbuf (unless FVP with a valid cache, which reads it), and per sample either the
// loss terms (gradient modes) or the tangent J x carried through h and M (J x) written to the plane (FVP).
template <class N_, int MODE>
__device__ __forceinline__ void gru_forward_lane(const GruArgs& a, const float* sp, const float* sv,
                                                 const GruDist<N_::A>& D, int n, double& s_loss, double& s_kl,
                                                 double& m_kl) {
  constexpr int H = N_::H, A = N_::A, I = N_::I;
  float h[H], th[H];
  for (int t = 0; t < a.T; ++t) {
    asm volatile("" ::: "memory");
    const size_t idx = (size_t)t * a.N + n;
    const bool start = a.tstep[idx] == 0;
    if (start) {
#pragma unroll
      for (int j = 0; j < H; ++j) { h[j] = 0.f; th[j] = 0.f; }
    }
    float x[I], hn[H];
    gru_input<N_>(a.obs, a.act, a.B, idx, a.N, start, x);
    if constexpr (MODE == MODE_FVP) {
      // tangent of the cell along x = sv:  with ar, au, ac = x W_x + h W_h + b and hc = h W_hc
      //   dr = r(1-r)(x V_xr + h V_hr + vb_r + th W_hr),  du likewise,  dhc = h V_hc + th W_hc
      //   dc = (1-c^2)(x V_xc + vb_c + dr hc + r dhc),  th' = (1-u) th + du (c - h) + u dc
      float tn[H];
#pragma unroll
      for (int j = 0; j < H; ++j) {
        float ar = sp[N_::ob(0) + j], au = sp[N_::ob(1) + j], ac = sp[N_::ob(2) + j], hc = 0.f;
        float tr = sv[N_::ob(0) + j], tu = sv[N_::ob(1) + j], tc = sv[N_::ob(2) + j], thc = 0.f;
#pragma unroll
        for (int i = 0; i < I; ++i) {
          ar = fmaf(x[i], sp[N_::oWx(0) + i * H + j], ar);
          au = fmaf(x[i], sp[N_::oWx(1) + i * H + j], au);
          ac = fmaf(x[i], sp[N_::oWx(2) + i * H + j], ac);
          tr = fmaf(x[i], sv[N_::oWx(0) + i * H + j], tr);
          tu = fmaf(x[i], sv[N_::oWx(1) + i * H + j], tu);
          tc = fmaf(x[i], sv[N_::oWx(2) + i * H + j], tc);
        }
#pragma unroll
        for (int k = 0; k < H; ++k) {
          ar = fmaf(h[k], sp[N_::oWh(0) + k * H + j], ar);
          au = fmaf(h[k], sp[N_::oWh(1) + k * H + j], au);
          hc = fmaf(h[k], sp[N_::oWh(2) + k * H + j], hc);
          tr = fmaf(h[k], sv[N_::oWh(0) + k * H + j], fmaf(th[k], sp[N_::oWh(0) + k * H + j], tr));
          tu = fmaf(h[k], sv[N_::oWh(1) + k * H + j], fmaf(th[k], sp[N_::oWh(1) + k * H + j], tu));
          thc = fmaf(h[k], sv[N_::oWh(2) + k * H + j], fmaf(th[k], sp[N_::oWh(2) + k * H + j], thc));
        }
        const float r = sigm_f(ar), u = sigm_f(au);
        const float c = tanh_f(fmaf(r, hc, ac));
        hn[j] = fmaf(u, c - h[j], h[j]);
        const float dr = r * (1.0f - r) * tr, du = u * (1.0f - u) * tu;
        const float dc = (1.0f - c * c) * (tc + dr * hc + r * thc);
        tn[j] = (1.0f - u) * th[j] + du * (c - h[j]) + u * dc;
      }
      if (a.h_valid) {   // the cache of the gradient pass: identical bits, but read back so that h is the cached one
#pragma unroll
        for (int j = 0; j < H; ++j) hn[j] = a.hbuf[(size_t)j * a.B + idx];
      } else {
#pragma unroll
        for (int j = 0; j < H; ++j) a.hbuf[(size_t)j * a.B + idx] = hn[j];
      }
      const bool valid = !gru_masked(a, idx);
#pragma unroll
      for (int k = 0; k < A; ++k) {
        float md = sv[N_::obo + k];
#pragma unroll
        for (int j = 0; j < H; ++j)
          md = fmaf(tn[j], sp[N_::oWo + j * A + k], fmaf(hn[j], sv[N_::oWo + j * A + k], md));
        a.plane[(size_t)k * a.B + idx] = valid ? md * D.Mmu[k] : 0.f;
      }
#pragma unroll
      for (int j = 0; j < H; ++j) { h[j] = hn[j]; th[j] = tn[j]; }
    } else {
      gru_cell<N_>(sp, x, h, hn);
#pragma unroll
      for (int j = 0; j < H; ++j) {
        a.hbuf[(size_t)j * a.B + idx] = hn[j];
        h[j] = hn[j];
      }
      if (gru_masked(a, idx)) continue;
      float mu[A], term, kl, dmu[A], dls[A];
      gru_mean<N_>(sp, hn, mu);
      gru_terms<A>(a, D, idx, mu, term, kl, dmu, dls);
      s_loss += (double)term;
      s_kl += (double)kl;
      m_kl = fmax(m_kl, (double)kl);
    }
  }
}

// Backward step t of one lane: gates recomputed from h_{t-1} (hbuf) and x_t, output deltas (surrogate [+ penalty KL], or
// the FVP plane), dh = carry + dmu W_out^T, gate deltas staged into this thread's tile column; returns the carry for t-1
// (zero when step t starts a path).
template <class N_, int MODE>
__device__ __forceinline__ void gru_backward_step(const GruArgs& a, const float* sp, const GruDist<N_::A>& D,
                                                  float* stage, int tid, int n, int t, float (&carry)[N_::H]) {
  using S = GruStage<N_>;
  constexpr int H = N_::H, A = N_::A, I = N_::I;
  // a thread past the last lane of a partial tile stages zeros and reads nothing: the lanes' hidden states are written
  // by their own threads' forward sweeps, which need not have finished, and a zero column adds nothing to the Gram
  const bool active = n < a.N;
  const size_t idx = (size_t)t * a.N + (active ? n : 0);
  const bool start = active ? a.tstep[idx] == 0 : true;
  float x[I], hp[H], ht[H], dmu[A], dls[A];
  if (active) {
    gru_input<N_>(a.obs, a.act, a.B, idx, a.N, start, x);
#pragma unroll
    for (int j = 0; j < H; ++j) {
      hp[j] = start ? 0.f : a.hbuf[(size_t)j * a.B + idx - a.N];
      ht[j] = a.hbuf[(size_t)j * a.B + idx];
    }
  } else {
#pragma unroll
    for (int i = 0; i < I; ++i) x[i] = 0.f;
#pragma unroll
    for (int j = 0; j < H; ++j) { hp[j] = 0.f; ht[j] = 0.f; }
  }
  const bool valid = active && !gru_masked(a, idx);
  if constexpr (MODE == MODE_FVP) {
#pragma unroll
    for (int k = 0; k < A; ++k) { dmu[k] = valid ? a.plane[(size_t)k * a.B + idx] : 0.f; dls[k] = 0.f; }
  } else {
    if (valid) {
      float mu[A], term, kl;
      gru_mean<N_>(sp, ht, mu);
      gru_terms<A>(a, D, idx, mu, term, kl, dmu, dls);
    } else {
#pragma unroll
      for (int k = 0; k < A; ++k) { dmu[k] = 0.f; dls[k] = 0.f; }
    }
  }
  float* col = stage + tid;
#pragma unroll
  for (int i = 0; i < I; ++i) col[(S::rX + i) * GLD] = x[i];
  col[S::rOne * GLD] = active ? 1.0f : 0.0f;
#pragma unroll
  for (int k = 0; k < A; ++k) {
    col[(S::rDM + k) * GLD] = dmu[k];
    col[(S::rDL + k) * GLD] = dls[k];
  }
  float dprev[H];
#pragma unroll
  for (int j = 0; j < H; ++j) {
    col[(S::rHp + j) * GLD] = hp[j];
    col[(S::rHn + j) * GLD] = ht[j];
    dprev[j] = 0.f;
  }
#pragma unroll
  for (int j = 0; j < H; ++j) {
    float ar = sp[N_::ob(0) + j], au = sp[N_::ob(1) + j], ac = sp[N_::ob(2) + j], hc = 0.f;
#pragma unroll
    for (int i = 0; i < I; ++i) {
      ar = fmaf(x[i], sp[N_::oWx(0) + i * H + j], ar);
      au = fmaf(x[i], sp[N_::oWx(1) + i * H + j], au);
      ac = fmaf(x[i], sp[N_::oWx(2) + i * H + j], ac);
    }
#pragma unroll
    for (int k = 0; k < H; ++k) {
      ar = fmaf(hp[k], sp[N_::oWh(0) + k * H + j], ar);
      au = fmaf(hp[k], sp[N_::oWh(1) + k * H + j], au);
      hc = fmaf(hp[k], sp[N_::oWh(2) + k * H + j], hc);
    }
    const float r = sigm_f(ar), u = sigm_f(au);
    const float c = tanh_f(fmaf(r, hc, ac));
    float dh = carry[j];
#pragma unroll
    for (int k = 0; k < A; ++k) dh = fmaf(dmu[k], sp[N_::oWo + j * A + k], dh);
    // dL/da_u = dh (c - h) u (1-u);  dL/da_c = dh u (1 - c^2);  dL/d(h W_hc) = da_c r;  dL/da_r = da_c hc r (1-r)
    const float du = dh * (c - hp[j]) * u * (1.0f - u);
    const float dc = dh * u * (1.0f - c * c);
    const float dhc = dc * r;
    const float dr = dc * hc * r * (1.0f - r);
    col[(S::rD + j) * GLD] = dr;
    col[(S::rD + H + j) * GLD] = du;
    col[(S::rD + 2 * H + j) * GLD] = dc;
    col[(S::rDhc + j) * GLD] = dhc;
    dprev[j] = fmaf(dh, 1.0f - u, dprev[j]);
#pragma unroll
    for (int k = 0; k < H; ++k)
      dprev[k] = fmaf(dr, sp[N_::oWh(0) + k * H + j],
                      fmaf(du, sp[N_::oWh(1) + k * H + j], fmaf(dhc, sp[N_::oWh(2) + k * H + j], dprev[k])));
  }
#pragma unroll
  for (int j = 0; j < H; ++j) carry[j] = start ? 0.f : dprev[j];   // the carried dh stops at the path start
}

template <class N_, int MODE>
__global__ void __launch_bounds__(GT, 1) gru_bptt_kernel(GruArgs a) {
  using S = GruStage<N_>;
  constexpr int P = N_::P, H = N_::H;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* sf = reinterpret_cast<float*>(smem_raw);
  float* sp = sf + S::o_sp;
  float* sv = sf + S::o_sv;
  float* stage = sf + S::o_stage;
  double* acc = reinterpret_cast<double*>(smem_raw + S::acc_off);
  double* red_scratch = reinterpret_cast<double*>(smem_raw + S::red_off);
  const int tid = threadIdx.x;
  for (int i = tid; i < P; i += GT) {
    sp[i] = a.params[i];
    if (MODE == MODE_FVP) sv[i] = (float)a.xvec[i];
    acc[i] = 0.0;
  }
  __syncthreads();
  GruDist<N_::A> D;
  D.init(sp + N_::ols, MODE == MODE_FVP ? nullptr : a.old_log_std);
  double s_loss = 0.0, s_kl = 0.0, m_kl = -1.0e300;
  const int ntiles = (a.N + GT - 1) / GT;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int n = tile * GT + tid;
    if (n < a.N) gru_forward_lane<N_, MODE>(a, sp, sv, D, n, s_loss, s_kl, m_kl);
    float carry[H];
#pragma unroll
    for (int j = 0; j < H; ++j) carry[j] = 0.f;
    for (int t = a.T - 1; t >= 0; --t) {
      gru_backward_step<N_, MODE>(a, sp, D, stage, tid, n, t, carry);
      __syncthreads();
      // Gram products of this step's 128-sample tile: entry e owned by thread e % 128, float32 over the tile
#pragma unroll 1
      for (int e = tid; e < P; e += GT) {
        int ra, rb;
        S::rows(e, ra, rb);
        const float* pa = stage + ra * GLD;
        const float* pb = stage + rb * GLD;
        float s0 = 0.f, s1 = 0.f;
#pragma unroll 8
        for (int s = 0; s < GT; s += 2) {
          s0 = fmaf(pa[s], pb[s], s0);
          s1 = fmaf(pa[s + 1], pb[s + 1], s1);
        }
        acc[e] += (double)(s0 + s1);
      }
      __syncthreads();
    }
  }
  double* out = a.partial + (size_t)blockIdx.x * P;
  for (int i = tid; i < P; i += GT) out[i] = acc[i];
  if constexpr (MODE != MODE_FVP) {
    double v[2] = {s_loss, s_kl};
    double mx[1] = {m_kl};
    double* sc = a.partial + (size_t)gridDim.x * P + (size_t)blockIdx.x * 3;
    block_reduce_store<2, false>(v, red_scratch, sc);
    block_reduce_store<1, true>(mx, red_scratch, sc + 2);
  }
}

template <class N_, int MODE>
static int launch_gru_bptt(const GruArgs& a, int* grid_out, cudaStream_t st) {
  using S = GruStage<N_>;
  B200RL_SET_MAX_SMEM((gru_bptt_kernel<N_, MODE>), S::bytes);
  const int grid = partial_grid(1, (a.N + GT - 1) / GT);
  gru_bptt_kernel<N_, MODE><<<grid, GT, S::bytes, st>>>(a);
  B200RL_LAUNCH_CHECK("gru_bptt_kernel");
  *grid_out = grid;
  return 0;
}

// ------------------------------------------------------------------------------------------------ float64 parity mode
// One thread per lane in plain float64 on the float64 master parameters; the lane's h history (and, for the Fisher
// product, M J x per sample) lives in the caller's float64 buffer h64 [H + A][T][N].  Weight gradients are summed with
// shared-memory float64 atomics (reruns agree to rounding).  MODE_GRAD with B200RL_LOSS_KL is the gradient of mean
// KL(old || new) (FiniteDifferenceHvp); MODE_FVP is J^T M J x, the exact Hessian of mean KL at theta_old (the KL's first
// derivative in the mean is zero there, and log_std enters linearly: its block is added by the finalize).
struct GruArgs64 {
  const double* params;
  const double* xvec;
  double* h64;
  int N, T;
  long long B;
  const float *obs, *act, *adv, *old_mean, *old_log_std;
  const unsigned short* tstep;
  int loss_kind;
  const unsigned char* flags;
  double* partial;
};

template <class N_>
__device__ __forceinline__ void gru_gates_d(const double* sp, const double (&x)[N_::I], const double (&h)[N_::H], int j,
                                            double& r, double& u, double& c, double& hc) {
  constexpr int I = N_::I, H = N_::H;
  double ar = sp[N_::ob(0) + j], au = sp[N_::ob(1) + j], ac = sp[N_::ob(2) + j];
  hc = 0.0;
  for (int i = 0; i < I; ++i) {
    ar = fma(x[i], sp[N_::oWx(0) + i * H + j], ar);
    au = fma(x[i], sp[N_::oWx(1) + i * H + j], au);
    ac = fma(x[i], sp[N_::oWx(2) + i * H + j], ac);
  }
  for (int k = 0; k < H; ++k) {
    ar = fma(h[k], sp[N_::oWh(0) + k * H + j], ar);
    au = fma(h[k], sp[N_::oWh(1) + k * H + j], au);
    hc = fma(h[k], sp[N_::oWh(2) + k * H + j], hc);
  }
  r = sigm_d(ar);
  u = sigm_d(au);
  c = tanh(fma(r, hc, ac));
}

template <class N_>
__device__ __forceinline__ void gru_input_d(const GruArgs64& a, size_t idx, bool start, double (&x)[N_::I]) {
  for (int o = 0; o < N_::O; ++o) x[o] = (double)a.obs[(size_t)o * a.B + idx];
  for (int k = 0; k < N_::I - N_::O; ++k) x[N_::O + k] = start ? 0.0 : (double)a.act[(size_t)k * a.B + idx - a.N];
}

template <class N_, int MODE>
__global__ void __launch_bounds__(64) gru_f64_kernel(GruArgs64 a) {
  constexpr int H = N_::H, A = N_::A, I = N_::I, P = N_::P;
  extern __shared__ __align__(16) double gru_sd[];
  double* sp = gru_sd;
  double* acc = gru_sd + P;
  double* sv = gru_sd + 2 * P;
  __shared__ double red_scratch[3 * 32];
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    sp[i] = a.params[i];
    acc[i] = 0.0;
    if (MODE == MODE_FVP) sv[i] = a.xvec[i];
  }
  __syncthreads();
  double ls_new[A], var_new[A], var_new2[A], ls_old[A], var_old[A], sum_ls_new = 0.0, sum_ls_old = 0.0;
  for (int k = 0; k < A; ++k) {
    ls_new[k] = sp[N_::ols + k];
    var_new[k] = exp(2.0 * ls_new[k]);
    var_new2[k] = 2.0 * var_new[k] + 1e-8;
    ls_old[k] = MODE == MODE_FVP ? ls_new[k] : (double)a.old_log_std[k];
    var_old[k] = exp(2.0 * ls_old[k]);
    sum_ls_new += ls_new[k];
    sum_ls_old += ls_old[k];
  }
  const double half_log2pi_A = 0.5 * A * 1.8378770664093453;
  double s_loss = 0.0, s_kl = 0.0, m_kl = -1.0e300;
  const int stride = gridDim.x * blockDim.x;
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < a.N; n += stride) {
    // forward sweep
    double h[H], th[H];
    for (int t = 0; t < a.T; ++t) {
      const size_t idx = (size_t)t * a.N + n;
      const bool start = a.tstep[idx] == 0;
      if (start)
        for (int j = 0; j < H; ++j) { h[j] = 0.0; th[j] = 0.0; }
      double x[I], hn[H], tn[H];
      gru_input_d<N_>(a, idx, start, x);
      for (int j = 0; j < H; ++j) {
        double r, u, c, hc;
        gru_gates_d<N_>(sp, x, h, j, r, u, c, hc);
        hn[j] = (1.0 - u) * h[j] + u * c;
        if (MODE == MODE_FVP) {
          double tr = sv[N_::ob(0) + j], tu = sv[N_::ob(1) + j], tc = sv[N_::ob(2) + j], thc = 0.0;
          for (int i = 0; i < I; ++i) {
            tr = fma(x[i], sv[N_::oWx(0) + i * H + j], tr);
            tu = fma(x[i], sv[N_::oWx(1) + i * H + j], tu);
            tc = fma(x[i], sv[N_::oWx(2) + i * H + j], tc);
          }
          for (int k = 0; k < H; ++k) {
            tr += h[k] * sv[N_::oWh(0) + k * H + j] + th[k] * sp[N_::oWh(0) + k * H + j];
            tu += h[k] * sv[N_::oWh(1) + k * H + j] + th[k] * sp[N_::oWh(1) + k * H + j];
            thc += h[k] * sv[N_::oWh(2) + k * H + j] + th[k] * sp[N_::oWh(2) + k * H + j];
          }
          const double dr = r * (1.0 - r) * tr, du = u * (1.0 - u) * tu;
          const double dc = (1.0 - c * c) * (tc + dr * hc + r * thc);
          tn[j] = (1.0 - u) * th[j] + du * (c - h[j]) + u * dc;
        }
      }
      for (int j = 0; j < H; ++j) {
        a.h64[(size_t)j * a.B + idx] = hn[j];
        h[j] = hn[j];
        if (MODE == MODE_FVP) th[j] = tn[j];
      }
      const bool valid = !(a.flags != nullptr && (a.flags[idx] & B200RL_FLAG_MASKED));
      if (MODE == MODE_FVP) {
        for (int k = 0; k < A; ++k) {
          double md = sv[N_::obo + k];
          for (int j = 0; j < H; ++j) md += th[j] * sp[N_::oWo + j * A + k] + h[j] * sv[N_::oWo + j * A + k];
          a.h64[(size_t)(H + k) * a.B + idx] = valid ? md * 2.0 / var_new2[k] : 0.0;
        }
        continue;
      }
      if (!valid) continue;
      double zsq = 0.0, zsq_old = 0.0, kl = 0.0;
      for (int k = 0; k < A; ++k) {
        double mu = sp[N_::obo + k];
        for (int j = 0; j < H; ++j) mu = fma(h[j], sp[N_::oWo + j * A + k], mu);
        const double act = a.act[(size_t)k * a.B + idx], om = a.old_mean[(size_t)k * a.B + idx];
        const double z = (act - mu) / exp(ls_new[k]), zo = (act - om) / exp(ls_old[k]), dm = om - mu;
        zsq += z * z;
        zsq_old += zo * zo;
        kl += (dm * dm + var_old[k] - var_new[k]) / var_new2[k] + ls_new[k] - ls_old[k];
      }
      const double adv_s = a.adv[idx];
      const double logp_new = -sum_ls_new - 0.5 * zsq - half_log2pi_A;
      s_loss += a.loss_kind == B200RL_LOSS_TRPO
                    ? -exp(logp_new - (-sum_ls_old - 0.5 * zsq_old - half_log2pi_A)) * adv_s
                    : -logp_new * adv_s;
      s_kl += kl;
      m_kl = fmax(m_kl, kl);
    }
    if constexpr (MODE == MODE_LOSS) continue;
    // backward sweep
    double carry[H];
    for (int j = 0; j < H; ++j) carry[j] = 0.0;
    for (int t = a.T - 1; t >= 0; --t) {
      const size_t idx = (size_t)t * a.N + n;
      const bool start = a.tstep[idx] == 0;
      const bool valid = !(a.flags != nullptr && (a.flags[idx] & B200RL_FLAG_MASKED));
      double x[I], hp[H], ht[H], dmu[A], dls[A];
      gru_input_d<N_>(a, idx, start, x);
      for (int j = 0; j < H; ++j) {
        hp[j] = start ? 0.0 : a.h64[(size_t)j * a.B + idx - a.N];
        ht[j] = a.h64[(size_t)j * a.B + idx];
      }
      for (int k = 0; k < A; ++k) {
        dmu[k] = 0.0;
        dls[k] = 0.0;
        if (!valid) continue;
        if (MODE == MODE_FVP) { dmu[k] = a.h64[(size_t)(H + k) * a.B + idx]; continue; }
        double mu = sp[N_::obo + k];
        for (int j = 0; j < H; ++j) mu = fma(ht[j], sp[N_::oWo + j * A + k], mu);
        const double act = a.act[(size_t)k * a.B + idx], om = a.old_mean[(size_t)k * a.B + idx];
        const double dm = om - mu;
        if (a.loss_kind == B200RL_LOSS_KL) {
          const double num = dm * dm + var_old[k] - var_new[k];
          dmu[k] = -2.0 * dm / var_new2[k];
          dls[k] = 1.0 - 2.0 * var_new[k] * (var_new2[k] + 2.0 * num) / (var_new2[k] * var_new2[k]);
        } else {
          double zsq = 0.0, zsq_old = 0.0;
          for (int q = 0; q < A; ++q) {
            double m2 = sp[N_::obo + q];
            for (int j = 0; j < H; ++j) m2 = fma(ht[j], sp[N_::oWo + j * A + q], m2);
            const double aq = a.act[(size_t)q * a.B + idx], oq = a.old_mean[(size_t)q * a.B + idx];
            zsq += (aq - m2) * (aq - m2) / var_new[q];
            zsq_old += (aq - oq) * (aq - oq) / var_old[q];
          }
          const double adv_s = a.adv[idx];
          const double w_s = a.loss_kind == B200RL_LOSS_TRPO ? exp(-sum_ls_new - 0.5 * zsq + sum_ls_old + 0.5 * zsq_old) * adv_s
                                                             : adv_s;
          const double z = (act - mu) / exp(ls_new[k]);
          dmu[k] = -w_s * z / exp(ls_new[k]);
          dls[k] = -w_s * (z * z - 1.0);
        }
      }
      for (int k = 0; k < A; ++k) {
        atomicAdd(&acc[N_::obo + k], dmu[k]);
        atomicAdd(&acc[N_::ols + k], dls[k]);
        for (int j = 0; j < H; ++j) atomicAdd(&acc[N_::oWo + j * A + k], ht[j] * dmu[k]);
      }
      double dprev[H];
      for (int j = 0; j < H; ++j) dprev[j] = 0.0;
      for (int j = 0; j < H; ++j) {
        double r, u, c, hc;
        gru_gates_d<N_>(sp, x, hp, j, r, u, c, hc);
        double dh = carry[j];
        for (int k = 0; k < A; ++k) dh += dmu[k] * sp[N_::oWo + j * A + k];
        const double du = dh * (c - hp[j]) * u * (1.0 - u);
        const double dc = dh * u * (1.0 - c * c);
        const double dhc = dc * r;
        const double dr = dc * hc * r * (1.0 - r);
        dprev[j] += dh * (1.0 - u);
        const double dg[3] = {dr, du, dc};
        for (int g = 0; g < 3; ++g) {
          atomicAdd(&acc[N_::ob(g) + j], dg[g]);
          for (int i = 0; i < I; ++i) atomicAdd(&acc[N_::oWx(g) + i * H + j], x[i] * dg[g]);
        }
        for (int k = 0; k < H; ++k) {
          atomicAdd(&acc[N_::oWh(0) + k * H + j], hp[k] * dr);
          atomicAdd(&acc[N_::oWh(1) + k * H + j], hp[k] * du);
          atomicAdd(&acc[N_::oWh(2) + k * H + j], hp[k] * dhc);
          dprev[k] += dr * sp[N_::oWh(0) + k * H + j] + du * sp[N_::oWh(1) + k * H + j] + dhc * sp[N_::oWh(2) + k * H + j];
        }
      }
      for (int j = 0; j < H; ++j) carry[j] = start ? 0.0 : dprev[j];
    }
  }
  __syncthreads();
  if (MODE != MODE_LOSS) {
    double* out = a.partial + (size_t)blockIdx.x * P;
    for (int i = threadIdx.x; i < P; i += blockDim.x) out[i] = acc[i];
  }
  if (MODE != MODE_FVP) {
    double v[2] = {s_loss, s_kl};
    double mx[1] = {m_kl};
    double* sc = (MODE == MODE_LOSS) ? a.partial + (size_t)blockIdx.x * 3
                                     : a.partial + (size_t)gridDim.x * P + (size_t)blockIdx.x * 3;
    block_reduce_store<2, false>(v, red_scratch, sc);
    block_reduce_store<1, true>(mx, red_scratch, sc + 2);
  }
}

template <class N_, int MODE>
static int launch_gru_f64(const GruArgs64& a, int* grid_out, cudaStream_t st) {
  const size_t smem = (size_t)3 * N_::P * sizeof(double);
  B200RL_SET_MAX_SMEM((gru_f64_kernel<N_, MODE>), smem);
  long long grid = (long long)num_sms() * 2;
  const long long need = (a.N + 63) / 64;
  if (grid > need) grid = need;
  gru_f64_kernel<N_, MODE><<<(unsigned)grid, 64, smem, st>>>(a);
  B200RL_LAUNCH_CHECK("gru_f64_kernel");
  *grid_out = (int)grid;
  return 0;
}

}  // namespace b200rl

using namespace b200rl;

static int gru_fill(GruArgs& a, const float* params, int N, int T, const float* obs, const float* act,
                    const unsigned short* tstep, const float* adv, const float* old_mean, const float* old_log_std,
                    int loss_kind, const unsigned char* flags, double* ws) {
  a.params = params; a.N = N; a.T = T; a.B = (long long)N * T;
  a.obs = obs; a.act = act; a.tstep = tstep; a.adv = adv; a.old_mean = old_mean; a.old_log_std = old_log_std;
  a.loss_kind = loss_kind; a.flags = flags; a.partial = ws;
  return 0;
}

extern "C" {

long long b200rl_gru_num_params(int obs_dim, int hidden, int act_dim, int include_action) {
  B200RL_REQUIRE_GRU_SHAPE(obs_dim, hidden, act_dim, "gru_num_params");
  long long P = 0;
  B200RL_DISPATCH_GRU(include_action, { P = NetG::P; });
  return P;
}

int b200rl_gru_get_actions(const float* params_f32, int obs_dim, int hidden, int act_dim, int include_action,
                           const float* obs, const float* prev_action, const float* h_in, long long n, const float* eps,
                           unsigned int seed, unsigned int iter, int row, long long lane0, float* act_out,
                           float* mean_out, float* h_out, float* log_std_out, void* stream) {
  B200RL_REQUIRE(params_f32 && obs && n > 0 && act_out && mean_out && h_out && log_std_out,
                 "gru_get_actions: bad arguments");
  B200RL_REQUIRE_GRU_SHAPE(obs_dim, hidden, act_dim, "gru_get_actions");
  const unsigned grid = (unsigned)((n + 127) / 128);
  B200RL_DISPATCH_GRU(include_action, {
    gru_get_actions_kernel<NetG><<<grid, 128, 0, (cudaStream_t)stream>>>(params_f32, obs, prev_action, h_in, n, eps,
                                                                         seed, iter, row, lane0, act_out, mean_out,
                                                                         h_out, log_std_out);
  });
  B200RL_LAUNCH_CHECK("gru_get_actions_kernel");
  return 0;
}

int b200rl_rollout_gru(int env_kind, const float* params_f32, int hidden, int include_action, int N, int T,
                       int max_path_length, const float* eps, const float* reset_raw, unsigned int seed,
                       unsigned int iter, long long lane0, float* obs, float* act, float* mean, float* rew,
                       unsigned char* flags, unsigned short* tstep, float* log_std_out, void* stream) {
  const RolloutArgs a{params_f32, 0.f, N, T, max_path_length, eps, reset_raw, seed, iter, lane0,
                      obs, act, mean, rew, flags, tstep, log_std_out};
  if (int rc = check_rollout_args("rollout_gru", a, true)) return rc;
  if (env_kind != B200RL_ENV_CARTPOLE) {
    set_error("rollout_gru: env kind %d is not compiled in for the GRU policy (only %d, CartpoleEnv)", env_kind,
              B200RL_ENV_CARTPOLE);
    return B200RL_EUNSUPPORTED;
  }
  B200RL_REQUIRE_GRU_SHAPE(CartPoleEnvD::O, hidden, CartPoleEnvD::A, "rollout_gru");
  B200RL_DISPATCH_GRU(include_action, {
    gru_rollout_kernel<CartPoleEnvD, NetG><<<(N + 127) / 128, 128, 0, (cudaStream_t)stream>>>(a);
  });
  B200RL_LAUNCH_CHECK("gru_rollout_kernel");
  return 0;
}

int b200rl_gru_loss_kl(int loss_kind, const float* params_f32, int obs_dim, int hidden, int act_dim,
                       int include_action, int N, int T, const float* obs, const float* act,
                       const unsigned short* tstep, const float* adv, const float* old_mean, const float* old_log_std,
                       const unsigned char* flags, double scale, const double* count, double* out, float* h_cache_out,
                       double* ws, void* stream) {
  B200RL_REQUIRE(params_f32 && obs && act && tstep && adv && old_mean && old_log_std && out && ws && N > 0 && T > 0,
                 "gru_loss_kl: bad arguments");
  if (int rc = check_loss_kind("gru_loss_kl", loss_kind)) return rc;
  B200RL_REQUIRE_GRU_SHAPE(obs_dim, hidden, act_dim, "gru_loss_kl");
  cudaStream_t st = (cudaStream_t)stream;
  GruArgs a{};
  gru_fill(a, params_f32, N, T, obs, act, tstep, adv, old_mean, old_log_std, loss_kind, flags, ws);
  a.hbuf = h_cache_out;
  const int grid = partial_grid(4, (N + 127) / 128);
  B200RL_DISPATCH_GRU(include_action, { gru_loss_kernel<NetG><<<grid, 128, 0, st>>>(a); });
  B200RL_LAUNCH_CHECK("gru_loss_kernel");
  return launch_finalize_update(fin_loss(ws, grid, out, scale, count), st);
}

int b200rl_gru_grad(int loss_kind, double penalty, const float* params_f32, int obs_dim, int hidden, int act_dim,
                    int include_action, int N, int T, const float* obs, const float* act, const unsigned short* tstep,
                    const float* adv, const float* old_mean, const float* old_log_std, const unsigned char* flags,
                    double scale, const double* count, double* g_out, double* loss_out, float* h_cache, double* ws,
                    void* stream) {
  B200RL_REQUIRE(params_f32 && obs && act && tstep && adv && old_mean && old_log_std && g_out && h_cache && ws &&
                 N > 0 && T > 0, "gru_grad: bad arguments");
  if (int rc = check_loss_kind("gru_grad", loss_kind)) return rc;
  B200RL_REQUIRE(penalty >= 0.0 && penalty <= 3.0e38, "gru_grad: penalty must be finite and >= 0");
  B200RL_REQUIRE_GRU_SHAPE(obs_dim, hidden, act_dim, "gru_grad");
  cudaStream_t st = (cudaStream_t)stream;
  GruArgs a{};
  gru_fill(a, params_f32, N, T, obs, act, tstep, adv, old_mean, old_log_std, loss_kind, flags, ws);
  a.hbuf = h_cache;
  a.penalty = (float)penalty;
  int grid = 0, P = 0, ols = 0;
  B200RL_DISPATCH_GRU(include_action, {
    P = NetG::P; ols = NetG::ols;
    int rc = launch_gru_bptt<NetG, MODE_GRAD>(a, &grid, st);
    if (rc) return rc;
  });
  return launch_finalize_update(
      fin_grad(ws, grid, P, g_out, loss_out, scale, count, {ols, act_dim, params_f32, nullptr, -INFINITY}), st);
}

int b200rl_gru_fvp(const float* params_f32, int obs_dim, int hidden, int act_dim, int include_action, int N, int T,
                   const float* obs, const float* act, const unsigned short* tstep, const unsigned char* flags,
                   const double* x, double scale, const double* count, double reg_coeff, double diag_scale,
                   double* Hx_out, float* h_cache, int h_valid, double* ws, void* stream) {
  B200RL_REQUIRE(params_f32 && obs && act && tstep && x && Hx_out && h_cache && ws && N > 0 && T > 0,
                 "gru_fvp: bad arguments");
  B200RL_REQUIRE_GRU_SHAPE(obs_dim, hidden, act_dim, "gru_fvp");
  cudaStream_t st = (cudaStream_t)stream;
  GruArgs a{};
  gru_fill(a, params_f32, N, T, obs, act, tstep, nullptr, nullptr, nullptr, B200RL_LOSS_TRPO, flags, ws);
  a.xvec = x; a.hbuf = h_cache; a.h_valid = h_valid ? 1 : 0;
  // the per-sample M J x plane follows the largest possible partials block in the workspace
  const size_t plane_off = (size_t)MAX_PARTIAL_BLOCKS * 4096;
  const size_t ws_doubles = (size_t)MAX_PARTIAL_BLOCKS * MAX_PARTIAL_K;
  B200RL_REQUIRE((size_t)act_dim * a.B <= 2 * (ws_doubles - plane_off),
                 "gru_fvp: %lld samples exceed the workspace's Fisher plane", (long long)a.B);
  a.plane = reinterpret_cast<float*>(ws + plane_off);
  int grid = 0, P = 0, ols = 0;
  B200RL_DISPATCH_GRU(include_action, {
    P = NetG::P; ols = NetG::ols;
    int rc = launch_gru_bptt<NetG, MODE_FVP>(a, &grid, st);
    if (rc) return rc;
  });
  return launch_finalize_update(fin_fvp(ws, grid, P, Hx_out, scale, count, {ols, act_dim, params_f32, nullptr, -INFINITY},
                                        x, reg_coeff, diag_scale),
                                st);
}

int b200rl_gru_update_f64(int mode, int loss_kind, const double* params_f64, int obs_dim, int hidden, int act_dim,
                          int include_action, int N, int T, const float* obs, const float* act,
                          const unsigned short* tstep, const float* adv, const float* old_mean,
                          const float* old_log_std, const unsigned char* flags, const double* x, double scale,
                          const double* count, double reg_coeff, double diag_scale, double* vec_out, double* loss_out,
                          double* h64, double* ws, void* stream) {
  B200RL_REQUIRE(params_f64 && obs && act && tstep && h64 && ws && N > 0 && T > 0, "gru_update_f64: bad arguments");
  if (int rc = check_f64_args("gru_update_f64", mode, loss_kind, adv && old_mean && old_log_std, x, vec_out, loss_out))
    return rc;
  B200RL_REQUIRE_GRU_SHAPE(obs_dim, hidden, act_dim, "gru_update_f64");
  cudaStream_t st = (cudaStream_t)stream;
  GruArgs64 a{};
  a.params = params_f64; a.xvec = x; a.h64 = h64; a.N = N; a.T = T; a.B = (long long)N * T;
  a.obs = obs; a.act = act; a.adv = adv; a.old_mean = old_mean; a.old_log_std = old_log_std; a.tstep = tstep;
  a.loss_kind = loss_kind; a.flags = flags; a.partial = ws;
  int grid = 0, P = 0, ols = 0;
  B200RL_DISPATCH_GRU(include_action, {
    P = NetG::P; ols = NetG::ols;
    int rc = (mode == MODE_LOSS) ? launch_gru_f64<NetG, MODE_LOSS>(a, &grid, st)
           : (mode == MODE_GRAD) ? launch_gru_f64<NetG, MODE_GRAD>(a, &grid, st)
                                 : launch_gru_f64<NetG, MODE_FVP>(a, &grid, st);
    if (rc) return rc;
  });
  // the gradient of mean KL is not masked where the min_std clamp would be active (the GRU's log_std is unclamped, and
  // with log_min_std = -inf the mask would still zero a NaN log_std entry): no log_std block for it
  const int A = (mode == MODE_GRAD && loss_kind == B200RL_LOSS_KL) ? 0 : act_dim;
  return launch_finalize_update(fin_f64(mode, ws, grid, P, vec_out, loss_out, scale, count,
                                        {ols, A, nullptr, params_f64, -INFINITY}, x, reg_coeff, diag_scale),
                                st);
}
}
