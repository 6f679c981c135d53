// CategoricalMLPPolicy on the lane batch (rllab/policies/categorical_mlp_policy.py, rllab/distributions/categorical.py):
// the fused discrete-action rollout, get_actions, and the loss/KL, gradient (+ KL penalty) and Fisher-vector passes of
// a softmax head, plus the entropy reduction behind the sampler's Entropy statistic.
//
// Net: h1 = tanh(x W0 + b0); h2 = tanh(h1 W1 + b1); z = h2 Wout + bout; prob = softmax(z).  The flat layout
// [W0, b0, W1, b1, Wout, bout] is the first Net<O, H, H, n>::ols entries of the Gaussian layout (no log_std), so the
// rollout's forward (mlp_forward_thread) runs on it unchanged and yields the logits.
// Compiled for one shape: obs_dim 4, hidden (32, 32), n = 2 (gym CartPole-v0).
//
// Arithmetic as the Gaussian passes (update.cu, update_tile.cu): float32 per sample and inside a 128-sample tile,
// float64 above; per-block partials folded in fixed order by launch_finalize_update.  Every pass computes the
// probabilities with cat_softmax() after the rollout's forward, so prob(theta_old) is bit-identical to the rollout's:
// the likelihood ratio is exactly 1 and the KL exactly 0 at theta_old.
#include "envs.cuh"
#include "tile_phase_a.cuh"   // TileGram, B200RL_SECTION_BARRIER

namespace b200rl {

constexpr int CAT_O = 4, CAT_H = 32, CAT_N = 2;
using CatNet = Net<CAT_O, CAT_H, CAT_H, CAT_N>;   // the Gaussian net of the same shape; the first ols entries are ours
constexpr int CAT_P = CatNet::ols;
constexpr float CAT_TINY = 1e-8f;                  // TINY of rllab/distributions/categorical.py

inline bool cat_supported(int O, int h1, int h2, int n) {
  return O == CAT_O && h1 == CAT_H && h2 == CAT_H && n == CAT_N;
}
#define B200RL_REQUIRE_CAT_SHAPE(O_, h1_, h2_, n_, what)                                                            \
  do {                                                                                                               \
    if (!cat_supported(O_, h1_, h2_, n_)) {                                                                          \
      set_error("%s: categorical net O=%d hidden=(%d,%d) n=%d is not compiled in (only O=4, (32,32), n=2)", what, \
                (int)(O_), (int)(h1_), (int)(h2_), (int)(n_));                                                     \
      return B200RL_EUNSUPPORTED;                                                                                    \
    }                                                                                                                \
  } while (0)

// softmax of Theano's nnet.softmax: e = exp(z - max z), p = e / sum e, the sum in ascending k
template <int NA>
__device__ __forceinline__ void cat_softmax(const float (&z)[NA], float (&p)[NA]) {
  float m = z[0];
#pragma unroll
  for (int k = 1; k < NA; ++k) m = fmaxf(m, z[k]);
  float e[NA], s = 0.f;
#pragma unroll
  for (int k = 0; k < NA; ++k) {
    e[k] = expf(__fsub_rn(z[k], m));
    s = __fadd_rn(s, e[k]);
  }
#pragma unroll
  for (int k = 0; k < NA; ++k) p[k] = __fdiv_rn(e[k], s);
}

// special.weighted_sample (rllab/misc/special.py:10-19): #{k : cumsum_k(p) < u}, clipped to n - 1
template <int NA>
__device__ __forceinline__ int cat_sample(const float (&p)[NA], float u) {
  float c = 0.f;
  int idx = 0;
#pragma unroll
  for (int k = 0; k < NA; ++k) {
    c = __fadd_rn(c, p[k]);
    idx += (c < u) ? 1 : 0;
  }
  return idx < NA - 1 ? idx : NA - 1;
}

// uniform u of lane `lane` at step `row`: u [row][N] (tests) or Philox stream 0, chunk 0, first word (b200rl_fill_noise
// with K = 1, kind uniform, stream 0)
__device__ __forceinline__ float cat_draw_u(const float* __restrict__ u, int row, long long N, long long n, uint32_t seed,
                                            uint32_t iter, long long lane) {
  if (u != nullptr) return u[(size_t)row * N + n];
  float q[4];
  noise4(B200RL_NOISE_UNIFORM, seed, iter, 0, lane, row, 0, q);
  return q[0];
}

// logits z = h2 Wout + bout in the rollout's summation order (mlp_forward_thread)
template <class N>
__device__ __forceinline__ void cat_logits(const float* __restrict__ sp, const float (&h2)[N::H2], float (&z)[N::A]) {
#pragma unroll
  for (int k = 0; k < N::A; ++k) {
    float s0 = sp[N::obo + k], s1 = 0.f;
#pragma unroll
    for (int j = 0; j < N::H2; j += 2) {
      s0 = fmaf(h2[j], sp[N::oWo + j * N::A + k], s0);
      s1 = fmaf(h2[j + 1], sp[N::oWo + (j + 1) * N::A + k], s1);
    }
    z[k] = s0 + s1;
  }
}

// Per-sample surrogate and KL (npo.py:72-82, vpg.py:91 over categorical.py):
//   pa = sum_k p_k x_k, qa = sum_k q_k x_k (x one-hot, q = old prob)
//   TRPO  term = -adv (pa + TINY) / (qa + TINY)     VPG  term = -adv log(pa + TINY)
//   kl = sum_k q_k (log(q_k + TINY) - log(p_k + TINY))
// c: the factor of the logit gradient d term / dz_j = -c p_j (x_j - pa) (TRPO: adv / (qa + TINY), VPG: adv / (pa + TINY)).
// Every operation is rounded on its own, so the loss pass and the gradient pass produce the same bits.
template <int NA>
__device__ __forceinline__ void cat_terms(int loss_kind, const float (&p)[NA], const float (&x)[NA],
                                          const float (&q)[NA], float adv, float& pa, float& term, float& kl,
                                          float& c) {
  pa = 0.f;
  float qa = 0.f;
  kl = 0.f;
#pragma unroll
  for (int k = 0; k < NA; ++k) {
    pa = __fadd_rn(pa, __fmul_rn(p[k], x[k]));
    qa = __fadd_rn(qa, __fmul_rn(q[k], x[k]));
    kl = __fadd_rn(kl, __fmul_rn(q[k], __fsub_rn(logf(__fadd_rn(q[k], CAT_TINY)), logf(__fadd_rn(p[k], CAT_TINY)))));
  }
  if (loss_kind == B200RL_LOSS_TRPO) {
    const float qt = __fadd_rn(qa, CAT_TINY);
    term = -__fmul_rn(__fdiv_rn(__fadd_rn(pa, CAT_TINY), qt), adv);
    c = __fdiv_rn(adv, qt);
  } else {
    const float pt = __fadd_rn(pa, CAT_TINY);
    term = -__fmul_rn(logf(pt), adv);
    c = __fdiv_rn(adv, pt);
  }
}

// Logit-space derivatives, float32 and float64, without differences of nearly equal numbers.  Softmax is shift-invariant,
// so each is a sum over pairs (k, j) of a term symmetric in (k, j) times a difference of the pair: 1 - p_a is never
// formed (it loses all accuracy in float32 once p_a rounds to 1, a logit gap of ~17), every product of probabilities
// keeps the relative accuracy of its factors, and each row sums to zero bit for bit (at n = 2, dz_1 = -dz_0 exactly),
// as the exact derivatives do.  The operations are rounded one by one so that the pair terms are computed alike.
__device__ __forceinline__ float cat_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float cat_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float cat_sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double cat_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double cat_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double cat_sub(double a, double b) { return __dsub_rn(a, b); }

// d term / dz_k = -c p_k (x_k - pa) = c sum_{j != k} (p_k p_j) (x_j - x_k)   (x one-hot, pa = sum_j p_j x_j)
template <int NA, class T>
__device__ __forceinline__ void cat_surr_logit_grad(T c, const T (&p)[NA], const T (&x)[NA], T (&dz)[NA]) {
#pragma unroll
  for (int k = 0; k < NA; ++k) {
    T d = T(0);
#pragma unroll
    for (int j = 0; j < NA; ++j)
      if (j != k) d = cat_add(d, cat_mul(cat_mul(p[k], p[j]), cat_sub(x[j], x[k])));
    dz[k] = cat_mul(c, d);
  }
}

// d kl(q || softmax(z)) / dz_k = -r_k + p_k sum_j r_j = sum_{j != k} (p_k r_j - r_k p_j),   r_j = q_j p_j / (p_j + TINY)
template <int NA, class T>
__device__ __forceinline__ void cat_kl_logit_grad(const T (&p)[NA], const T (&r)[NA], T (&g)[NA]) {
#pragma unroll
  for (int k = 0; k < NA; ++k) {
    T d = T(0);
#pragma unroll
    for (int j = 0; j < NA; ++j)
      if (j != k) d = cat_add(d, cat_sub(cat_mul(p[k], r[j]), cat_mul(r[k], p[j])));
    g[k] = d;
  }
}

// M tz, M = diag(R p - s) + s p^T + p s^T - (R + S) p p^T (the Hessian of kl(q || softmax(z)) in z at q = p; R = sum
// p_j^2 / (p_j + TINY), s_j = TINY p_j^2 / (p_j + TINY)^2, S = sum s_j).  M's rows sum to zero, so
//   (M tz)_k = sum_{j != k} W_kj (tz_k - tz_j),   W_kj = -M_kj = (R + S) p_k p_j - (s_k p_j + s_j p_k),
// and W_kj loses at most a quarter to cancellation (s_j <= p_j / 4).
template <int NA, class T>
__device__ __forceinline__ void cat_logit_hvp(const T (&p)[NA], const T (&tz)[NA], T (&m)[NA]) {
  constexpr T E = T(1e-8);   // TINY, exact in each type (float32: CAT_TINY)
  T s[NA], R = T(0), S = T(0);
#pragma unroll
  for (int k = 0; k < NA; ++k) {
    const T pe = p[k] + E;
    R += p[k] * p[k] / pe;
    s[k] = E * p[k] * p[k] / (pe * pe);
    S += s[k];
  }
  const T RS = cat_add(R, S);
#pragma unroll
  for (int k = 0; k < NA; ++k) {
    T d = T(0);
#pragma unroll
    for (int j = 0; j < NA; ++j) {
      if (j == k) continue;
      const T w = cat_sub(cat_mul(RS, cat_mul(p[k], p[j])), cat_add(cat_mul(s[k], p[j]), cat_mul(s[j], p[k])));
      d = cat_add(d, cat_mul(w, cat_sub(tz[k], tz[j])));
    }
    m[k] = d;
  }
}

// ------------------------------------------------------------------------------------------------ rollout / get_actions
// One thread per lane (lane_rollout, envs.cuh): the policy head draws action = weighted_sample(prob, u) with u from
// a.eps, and the env takes the index; act holds the one-hot action (the reference's flattened action,
// sampler/utils.py:23), the mean plane the probabilities.
template <class Env>
__global__ void __launch_bounds__(128, 4) cat_rollout_kernel(RolloutArgs a) {
  using N_ = CatNet;
  static_assert(Env::O == N_::O && EnvNumActions<Env>::value == N_::A, "env and categorical net disagree");
  __shared__ __align__(16) float sp[(CAT_P + 3) & ~3];
  for (int i = threadIdx.x; i < CAT_P; i += blockDim.x) sp[i] = a.params[i];
  __syncthreads();
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= a.N) return;
  const long long lane = a.lane0 + n;
  float p[CAT_N];
  int k_act;
  lane_rollout<Env>(
      a, n,
      [&](int t, int, const float (&o)[Env::O]) {
        float h1[CAT_H], h2[CAT_H], z[CAT_N];
        mlp_forward_thread<N_>(sp, o, h1, h2, z);
        cat_softmax(z, p);
        k_act = cat_sample(p, cat_draw_u(a.eps, t, a.N, n, a.seed, a.iter, lane));
      },
      [&](size_t idx, size_t TN, float (&u)[Env::A]) {
#pragma unroll
        for (int k = 0; k < CAT_N; ++k) {
          a.act[k * TN + idx] = (k == k_act) ? 1.0f : 0.0f;
          a.mean[k * TN + idx] = p[k];
        }
        u[0] = (float)k_act;
      });
}

__global__ void __launch_bounds__(128) cat_get_actions_kernel(const float* __restrict__ params,
                                                              const float* __restrict__ obs, long long n_,
                                                              const float* __restrict__ u, uint32_t seed, uint32_t iter,
                                                              int row, long long lane0, int* __restrict__ act_out,
                                                              float* __restrict__ prob_out) {
  __shared__ __align__(16) float sp[(CAT_P + 3) & ~3];
  for (int i = threadIdx.x; i < CAT_P; i += blockDim.x) sp[i] = params[i];
  __syncthreads();
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_) return;
  float o[CAT_O], h1[CAT_H], h2[CAT_H], z[CAT_N], p[CAT_N];
#pragma unroll
  for (int k = 0; k < CAT_O; ++k) o[k] = obs[(size_t)k * n_ + n];
  mlp_forward_thread<CatNet>(sp, o, h1, h2, z);
  cat_softmax(z, p);
  const float uu = (u != nullptr) ? u[n] : cat_draw_u(nullptr, row, n_, n, seed, iter, lane0 + n);
  act_out[n] = cat_sample(p, uu);
#pragma unroll
  for (int k = 0; k < CAT_N; ++k) prob_out[(size_t)k * n_ + n] = p[k];
}

// ------------------------------------------------------------------------------------------------ update passes
// UpdArgs fields used here: params, xvec, h_cache, B, obs, act (one-hot [n][B]), adv, old_mean (= old prob [n][B]),
// loss_kind, flags, tile_list, n_list, partial, penalty.

// Loss / KL, one thread per sample, forward only (the Gaussian loss_thread_kernel with the categorical head).
__global__ void __launch_bounds__(128, 3) cat_loss_kernel(UpdArgs a) {
  __shared__ __align__(16) float sp[(CAT_P + 3) & ~3];
  __shared__ double red_scratch[3 * 32];
  for (int i = threadIdx.x; i < CAT_P; i += blockDim.x) sp[i] = a.params[i];
  __syncthreads();
  double s_loss = 0.0, s_kl = 0.0, m_kl = -1.0e300;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < a.B; s += stride) {
    asm volatile("" ::: "memory");
    if (a.flags != nullptr && (a.flags[s] & B200RL_FLAG_MASKED)) continue;
    float x[CAT_O], h1[CAT_H], h2[CAT_H], z[CAT_N], p[CAT_N], xa[CAT_N], q[CAT_N];
#pragma unroll
    for (int o = 0; o < CAT_O; ++o) x[o] = a.obs[(size_t)o * a.B + s];
    mlp_forward_thread<CatNet>(sp, x, h1, h2, z);
    cat_softmax(z, p);
#pragma unroll
    for (int k = 0; k < CAT_N; ++k) {
      xa[k] = a.act[(size_t)k * a.B + s];
      q[k] = a.old_mean[(size_t)k * a.B + s];
    }
    float pa, term, kl, c;
    cat_terms(a.loss_kind, p, xa, q, a.adv[s], pa, term, kl, c);
    s_loss += (double)term;
    s_kl += (double)kl;
    m_kl = fmax(m_kl, (double)kl);
  }
  double v[2] = {s_loss, s_kl};
  double mx[1] = {m_kl};
  block_reduce_store<2, false>(v, red_scratch, a.partial + (size_t)blockIdx.x * 3);
  block_reduce_store<1, true>(mx, red_scratch, a.partial + (size_t)blockIdx.x * 3 + 2);
}

// Gradient / Fisher-vector product: the structure of update_tile_kernel (update_tile.cu) -- phase A per sample in one
// thread, staged feature-major into a 128-sample tile; phase B = TileGram (tile_gram.cuh) unchanged.  TileGram writes the
// Gaussian layout: the DL rows (log_std deltas) are zero here, and its log_std slots are dropped when the block's vector
// (staged in shared memory) is copied out with the categorical P.
constexpr int CT_THREADS = 128, CT_TILE = 128, CT_LD = CT_TILE + 4;

template <int MODE>
struct CatSmem {
  static constexpr int O = CAT_O, H = CAT_H, A = CAT_N;
  static constexpr int rX = 0, rH1 = rX + O, rH2 = rH1 + H, rD1 = rH2 + H, rD2 = rD1 + H, rDM = rD2 + H, rDL = rDM + A,
                       R = rDL + A;
  static constexpr int P4 = (CAT_P + 3) & ~3;
  static constexpr int o_sp = 0, o_sv = P4, o_stage = (MODE == MODE_FVP ? 2 : 1) * P4;
  static constexpr int n_floats = o_stage + R * CT_LD;
  static constexpr int scratch_off = ((n_floats * 4 + 15) / 16) * 16;
  static constexpr size_t bytes = (size_t)scratch_off + 3 * 32 * 8;
  // inside the (idle) stage region after the tile loop: TileGram's K-half scratch, then the block's Gaussian-layout vector
  static constexpr int scr_doubles = 2 * 64 * 16;
  static_assert((scr_doubles + CatNet::P) * 8 <= R * CT_LD * 4, "stage region must hold the write scratch + vector");
};

template <int MODE>
constexpr int cat_tile_minblocks() { return (CatSmem<MODE>::bytes + 1024) * 3 <= 228 * 1024 ? 3 : 2; }

template <int MODE, class SM>
__device__ __forceinline__ void cat_phase_a(const UpdArgs& a, const float* sp, const float* sv, float* stage,
                                            long long sl, bool inrange, bool valid, int tid, double& s_loss,
                                            double& s_kl, double& m_kl) {
  constexpr int O = CAT_O, H = CAT_H, A = CAT_N, LD = CT_LD;
  using N = CatNet;
  float* colX = stage + SM::rX * LD + tid;
  float* colH1 = stage + SM::rH1 * LD + tid;
  float* colH2 = stage + SM::rH2 * LD + tid;
  float* colD1 = stage + SM::rD1 * LD + tid;   // FVP: holds h1 V1 temporarily before d1 overwrites it
  float* colD2 = stage + SM::rD2 * LD + tid;
  float* colDM = stage + SM::rDM * LD + tid;
  float* colDL = stage + SM::rDL * LD + tid;
  float dz[A];
  {
    float x[O], h1[H];
#pragma unroll
    for (int o = 0; o < O; ++o) {
      x[o] = a.obs[(size_t)o * a.B + sl];
      colX[o * LD] = x[o];
    }
    const bool cached = (MODE == MODE_FVP) && (a.h_cache != nullptr);
    float* hc = a.h_cache ? a.h_cache + sl : nullptr;
    if (cached) {
#pragma unroll
      for (int j = 0; j < H; ++j) h1[j] = hc[(size_t)j * a.B];
    } else {
      dense_thread<O, H>(sp + N::oW0, sp + N::ob0, x, h1);
#pragma unroll
      for (int j = 0; j < H; ++j) h1[j] = tanh_f(h1[j]);
    }
#pragma unroll
    for (int j = 0; j < H; ++j) colH1[j * LD] = h1[j];
    if constexpr (MODE == MODE_FVP) {
      float p2b[H];
      dense_thread<H, H, false>(sv + N::oW1, nullptr, h1, p2b);
#pragma unroll
      for (int j = 0; j < H; ++j) colD1[j * LD] = p2b[j];
      B200RL_SECTION_BARRIER();
    }
    float h2[H];
    if (cached) {
#pragma unroll
      for (int j = 0; j < H; ++j) h2[j] = hc[(size_t)(H + j) * a.B];
    } else {
      dense_thread<H, H>(sp + N::oW1, sp + N::ob1, h1, h2);
#pragma unroll
      for (int j = 0; j < H; ++j) h2[j] = tanh_f(h2[j]);
    }
#pragma unroll
    for (int j = 0; j < H; ++j) colH2[j * LD] = h2[j];
    if (is_grad_mode(MODE) && hc != nullptr && inrange) {   // masked samples too: the FVP pass reads their rows back
#pragma unroll
      for (int j = 0; j < H; ++j) {
        hc[(size_t)j * a.B] = colH1[j * LD];
        hc[(size_t)(H + j) * a.B] = h2[j];
      }
    }
    B200RL_SECTION_BARRIER();
    float z[A], p[A];
    cat_logits<N>(sp, h2, z);
    cat_softmax(z, p);
    if constexpr (is_grad_mode(MODE)) {
      float xa[A], q[A];
#pragma unroll
      for (int k = 0; k < A; ++k) {
        xa[k] = a.act[(size_t)k * a.B + sl];
        q[k] = a.old_mean[(size_t)k * a.B + sl];
      }
      float pa, term, kl, c;
      cat_terms(a.loss_kind, p, xa, q, a.adv[sl], pa, term, kl, c);
      if (!valid) { c = 0.f; term = 0.f; }
      s_loss += (double)term;
      if (valid) { s_kl += (double)kl; m_kl = fmax(m_kl, (double)kl); }
      cat_surr_logit_grad(c, p, xa, dz);
      if (MODE == MODE_GRAD_KL && valid) {
        float r[A], g[A];
#pragma unroll
        for (int k = 0; k < A; ++k) r[k] = q[k] * p[k] / (p[k] + CAT_TINY);
        cat_kl_logit_grad(p, r, g);
#pragma unroll
        for (int k = 0; k < A; ++k) dz[k] = fmaf(a.penalty, g[k], dz[k]);
      }
    } else {
      // tangent forward J x (x = sv): t1 = (1-h1^2)(x V0 + vb0); t2 = (1-h2^2)(t1 W1 + h1 V1 + vb1); tz = t2 Wout + h2 Vout + vbout
      float t1[H];
      dense_thread<O, H>(sv + N::oW0, sv + N::ob0, x, t1);
#pragma unroll
      for (int j = 0; j < H; ++j) t1[j] *= (1.0f - h1[j] * h1[j]);
      B200RL_SECTION_BARRIER();
      float t2[H];
      dense_thread<H, H>(sp + N::oW1, sv + N::ob1, t1, t2);
      float tz[A];
#pragma unroll
      for (int k = 0; k < A; ++k) tz[k] = sv[N::obo + k];
#pragma unroll
      for (int j = 0; j < H; ++j) {
        const float h2j = colH2[j * LD];
        const float t2j = (t2[j] + colD1[j * LD]) * (1.0f - h2j * h2j);
#pragma unroll
        for (int k = 0; k < A; ++k) tz[k] = fmaf(t2j, sp[N::oWo + j * A + k], fmaf(h2j, sv[N::oWo + j * A + k], tz[k]));
      }
      // M tz, M = Hessian of kl(q || softmax(z)) in z at q = p (DESIGN.md section 5)
      float m[A];
      cat_logit_hvp(p, tz, m);
#pragma unroll
      for (int k = 0; k < A; ++k) dz[k] = valid ? m[k] : 0.f;
    }
#pragma unroll
    for (int k = 0; k < A; ++k) {
      colDM[k * LD] = dz[k];
      colDL[k * LD] = 0.f;
    }
  }
  B200RL_SECTION_BARRIER();
  // backward: d2 = (dz Wout^T) (1-h2^2); d1 = (d2 W1^T) (1-h1^2)
  float d2[H];
#pragma unroll
  for (int j = 0; j < H; ++j) {
    float sacc = 0.f;
#pragma unroll
    for (int k = 0; k < A; ++k) sacc = fmaf(dz[k], sp[N::oWo + j * A + k], sacc);
    const float h2j = colH2[j * LD];
    d2[j] = sacc * (1.0f - h2j * h2j);
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
    const float h1i = colH1[i * LD];
    colD1[i * LD] = (acc.x + acc.y) * (1.0f - h1i * h1i);
  }
}

template <int MODE>
__global__ void __launch_bounds__(CT_THREADS, cat_tile_minblocks<MODE>()) cat_tile_kernel(UpdArgs a) {
  using SM = CatSmem<MODE>;
  constexpr int LD = CT_LD;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* sf = reinterpret_cast<float*>(smem_raw);
  float* sp = sf + SM::o_sp;
  float* sv = sf + SM::o_sv;
  float* stage = sf + SM::o_stage;
  double* red_scratch = reinterpret_cast<double*>(smem_raw + SM::scratch_off);
  const int tid = threadIdx.x;
  for (int i = tid; i < CAT_P; i += CT_THREADS) sp[i] = a.params[i];
  if constexpr (MODE == MODE_FVP)
    for (int i = tid; i < CAT_P; i += CT_THREADS) sv[i] = (float)a.xvec[i];
  __syncthreads();

  TileGram<CatNet, SM::rX, SM::rH1, SM::rH2, SM::rD1, SM::rD2, SM::rDM, LD> gram;
  gram.init();
  double s_loss = 0.0, s_kl = 0.0, m_kl = -1.0e300;
  const long long ntiles = n_tiles_of(a, CT_TILE);
  for (long long ti_ = blockIdx.x; ti_ < ntiles; ti_ += gridDim.x) {
    asm volatile("" ::: "memory");
    const long long s = tile_at(a, ti_) * CT_TILE + tid;
    const bool inrange = s < a.B;
    const bool valid = sample_valid(a, s);
    cat_phase_a<MODE, SM>(a, sp, sv, stage, inrange ? s : a.B - 1, inrange, valid, tid, s_loss, s_kl, m_kl);
    __syncthreads();
    gram.accumulate_a(stage, tid);
    gram.accumulate_b(stage, tid);
    __syncthreads();
  }
  // the block's vector in the Gaussian layout, staged in shared memory; its first CAT_P entries are the partial
  double* scr = reinterpret_cast<double*>(stage);
  double* vec = scr + SM::scr_doubles;
  gram.write(vec, scr, tid);
  __syncthreads();
  double* out = a.partial + (size_t)blockIdx.x * CAT_P;
  for (int i = tid; i < CAT_P; i += CT_THREADS) out[i] = vec[i];
  if constexpr (is_grad_mode(MODE)) {
    __syncthreads();
    double v[2] = {s_loss, s_kl};
    double mx[1] = {m_kl};
    double* sc = a.partial + (size_t)gridDim.x * CAT_P + (size_t)blockIdx.x * 3;
    block_reduce_store<2, false>(v, red_scratch, sc);
    block_reduce_store<1, true>(mx, red_scratch, sc + 2);
  }
}

template <int MODE>
static int launch_cat_tile(const UpdArgs& a, int* grid_out, cudaStream_t st) {
  using SM = CatSmem<MODE>;
  B200RL_SET_MAX_SMEM((cat_tile_kernel<MODE>), SM::bytes);
  int per_sm = (int)((228 * 1024) / (SM::bytes + 1024));
  if (per_sm < 1) per_sm = 1;
  if (per_sm > cat_tile_minblocks<MODE>()) per_sm = cat_tile_minblocks<MODE>();
  const int grid = partial_grid(per_sm, host_n_tiles(a, CT_TILE));
  cat_tile_kernel<MODE><<<grid, CT_THREADS, SM::bytes, st>>>(a);
  B200RL_LAUNCH_CHECK("cat_tile_kernel");
  *grid_out = grid;
  return 0;
}

// Entropy of the recorded probabilities: sum over valid samples of -sum_k p_k log(p_k + TINY) (categorical.py:entropy),
// and the number of valid samples.
__global__ void __launch_bounds__(256) cat_entropy_kernel(long long B, const float* __restrict__ prob,
                                                          const unsigned char* __restrict__ flags,
                                                          double* __restrict__ partial) {
  __shared__ double scratch[2 * 32];
  double v[2] = {0.0, 0.0};
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < B; s += stride) {
    if (flags != nullptr && (flags[s] & B200RL_FLAG_MASKED)) continue;
    float e = 0.f;
#pragma unroll
    for (int k = 0; k < CAT_N; ++k) {
      const float p = prob[(size_t)k * B + s];
      e = __fadd_rn(e, __fmul_rn(p, logf(__fadd_rn(p, CAT_TINY))));
    }
    v[0] -= (double)e;
    v[1] += 1.0;
  }
  block_reduce_store<2, false>(v, scratch, partial + (size_t)blockIdx.x * 2);
}

// ------------------------------------------------------------------------------------------------ float64 parity mode
// The three passes in float64 on the float64 master parameters (the role of update_f64.cu for GaussianMLPPolicy): one
// thread per sample, weights in shared memory, weight gradients accumulated with shared-memory float64 atomics.
// MODE_GRAD with B200RL_LOSS_KL is the gradient of mean KL(old || new) (FiniteDifferenceHvp).  MODE_FVP is the exact
// Hessian-vector product of mean KL at theta_old, H x = J^T M J x + sum_j g_j (d^2 z_j)[x] with g = d kl / dz (O(TINY) at
// theta_old, DESIGN.md section 5): the second term is the tangent of the backward pass of g along x.
struct CatArgs64 {
  const double* params;
  const double* xvec;
  long long B;
  const float *obs, *act, *adv, *old_prob;
  int loss_kind;
  const unsigned char* flags;
  double* partial;
};

template <int NIN, int NOUT>
__device__ __forceinline__ void cat_dense_d(const double* W, const double* b, const double (&in)[NIN],
                                            double (&out)[NOUT]) {
#pragma unroll
  for (int j = 0; j < NOUT; ++j) out[j] = b ? b[j] : 0.0;
#pragma unroll 2
  for (int i = 0; i < NIN; ++i) {
#pragma unroll
    for (int j = 0; j < NOUT; ++j) out[j] = fma(in[i], W[i * NOUT + j], out[j]);
  }
}

template <int MODE>
__global__ void __launch_bounds__(128) cat_f64_kernel(CatArgs64 a) {
  using N = CatNet;
  constexpr int O = CAT_O, H = CAT_H, A = CAT_N, P = CAT_P;
  constexpr double E = 1e-8;
  extern __shared__ __align__(16) double cat_sd[];
  double* sp = cat_sd;
  double* acc = cat_sd + P;
  double* sv = cat_sd + 2 * P;
  __shared__ double red_scratch[3 * 32];
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    sp[i] = a.params[i];
    if (MODE != MODE_LOSS) acc[i] = 0.0;
    if (MODE == MODE_FVP) sv[i] = a.xvec[i];
  }
  __syncthreads();
  double s_loss = 0.0, s_kl = 0.0, m_kl = -1.0e300;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < a.B; s += stride) {
    if (a.flags != nullptr && (a.flags[s] & B200RL_FLAG_MASKED)) continue;
    double x[O], h1[H], h2[H], z[A], p[A], dz[A];
#pragma unroll
    for (int o = 0; o < O; ++o) x[o] = (double)a.obs[(size_t)o * a.B + s];
    cat_dense_d<O, H>(sp + N::oW0, sp + N::ob0, x, h1);
#pragma unroll
    for (int j = 0; j < H; ++j) h1[j] = tanh(h1[j]);
    cat_dense_d<H, H>(sp + N::oW1, sp + N::ob1, h1, h2);
#pragma unroll
    for (int j = 0; j < H; ++j) h2[j] = tanh(h2[j]);
#pragma unroll
    for (int k = 0; k < A; ++k) {
      double m = sp[N::obo + k];
#pragma unroll 4
      for (int j = 0; j < H; ++j) m = fma(h2[j], sp[N::oWo + j * A + k], m);
      z[k] = m;
    }
    double zm = z[0];
#pragma unroll
    for (int k = 1; k < A; ++k) zm = fmax(zm, z[k]);
    double es = 0.0;
#pragma unroll
    for (int k = 0; k < A; ++k) { p[k] = exp(z[k] - zm); es += p[k]; }
#pragma unroll
    for (int k = 0; k < A; ++k) p[k] /= es;
    // FVP: tangent (J x) and the extra operands of the curvature term
    double th1[H], th2[H], g[A];
    if (MODE != MODE_FVP) {
      double xa[A], q[A], pa = 0.0, qa = 0.0, kl = 0.0, r[A];
#pragma unroll
      for (int k = 0; k < A; ++k) {
        xa[k] = (double)a.act[(size_t)k * a.B + s];
        q[k] = (double)a.old_prob[(size_t)k * a.B + s];
        pa += p[k] * xa[k];
        qa += q[k] * xa[k];
        kl += q[k] * (log(q[k] + E) - log(p[k] + E));
        r[k] = q[k] * p[k] / (p[k] + E);
      }
      const double adv_s = (double)a.adv[s];
      double term, c;
      if (a.loss_kind == B200RL_LOSS_TRPO) {
        term = -(pa + E) / (qa + E) * adv_s;
        c = adv_s / (qa + E);
      } else {
        term = -log(pa + E) * adv_s;
        c = adv_s / (pa + E);
      }
      s_loss += term;
      s_kl += kl;
      m_kl = fmax(m_kl, kl);
      if (MODE == MODE_LOSS) continue;
      if (a.loss_kind == B200RL_LOSS_KL)
        cat_kl_logit_grad(p, r, dz);
      else
        cat_surr_logit_grad(c, p, xa, dz);
    } else {
      cat_dense_d<O, H>(sv + N::oW0, sv + N::ob0, x, th1);
#pragma unroll
      for (int j = 0; j < H; ++j) th1[j] *= (1.0 - h1[j] * h1[j]);
      cat_dense_d<H, H>(sp + N::oW1, sv + N::ob1, th1, th2);
#pragma unroll 2
      for (int i = 0; i < H; ++i)
#pragma unroll
        for (int j = 0; j < H; ++j) th2[j] = fma(h1[i], sv[N::oW1 + i * H + j], th2[j]);
#pragma unroll
      for (int j = 0; j < H; ++j) th2[j] *= (1.0 - h2[j] * h2[j]);
      double tz[A];
#pragma unroll
      for (int k = 0; k < A; ++k) {
        double m = sv[N::obo + k];
#pragma unroll 4
        for (int j = 0; j < H; ++j) m = fma(th2[j], sp[N::oWo + j * A + k], fma(h2[j], sv[N::oWo + j * A + k], m));
        tz[k] = m;
      }
      // M tz (q = p) and g = d kl / dz at q = p
      double r[A];
#pragma unroll
      for (int k = 0; k < A; ++k) r[k] = p[k] * p[k] / (p[k] + E);
      cat_logit_hvp(p, tz, dz);
      cat_kl_logit_grad(p, r, g);
    }
    // backward + accumulation.  FVP adds the tangent of g's backward pass:
    //   dWout += th2 (x) g;  D2 = d2(dz) + (g Vout^T)(1-h2^2) - 2 (g Wout^T) h2 th2;  dW1 += h1 (x) D2 + th1 (x) d2(g);
    //   D1 = (D2 W1^T + d2(g) V1^T)(1-h1^2) - 2 (d2(g) W1^T) h1 th1,   d2(g) = (g Wout^T)(1-h2^2)
    double d2[H], d2g[H];
#pragma unroll
    for (int j = 0; j < H; ++j) {
      double sacc = 0.0, eg = 0.0, vg = 0.0;
#pragma unroll
      for (int k = 0; k < A; ++k) {
        sacc = fma(dz[k], sp[N::oWo + j * A + k], sacc);
        double w = h2[j] * dz[k];
        if (MODE == MODE_FVP) {
          eg = fma(g[k], sp[N::oWo + j * A + k], eg);
          vg = fma(g[k], sv[N::oWo + j * A + k], vg);
          w += th2[j] * g[k];
        }
        atomicAdd(&acc[N::oWo + j * A + k], w);
      }
      const double dh = 1.0 - h2[j] * h2[j];
      d2[j] = sacc * dh;
      if (MODE == MODE_FVP) {
        d2g[j] = eg * dh;
        d2[j] += vg * dh - 2.0 * eg * h2[j] * th2[j];
      }
      atomicAdd(&acc[N::ob1 + j], d2[j]);
    }
#pragma unroll
    for (int k = 0; k < A; ++k) atomicAdd(&acc[N::obo + k], dz[k]);
#pragma unroll 1
    for (int i = 0; i < H; ++i) {
      double sacc = 0.0, sg = 0.0, vg = 0.0;
#pragma unroll
      for (int j = 0; j < H; ++j) {
        sacc = fma(d2[j], sp[N::oW1 + i * H + j], sacc);
        double w = h1[i] * d2[j];
        if (MODE == MODE_FVP) {
          sg = fma(d2g[j], sp[N::oW1 + i * H + j], sg);
          vg = fma(d2g[j], sv[N::oW1 + i * H + j], vg);
          w += th1[i] * d2g[j];
        }
        atomicAdd(&acc[N::oW1 + i * H + j], w);
      }
      double d1 = (sacc + vg) * (1.0 - h1[i] * h1[i]);
      if (MODE == MODE_FVP) d1 -= 2.0 * sg * h1[i] * th1[i];
      atomicAdd(&acc[N::ob0 + i], d1);
#pragma unroll
      for (int o = 0; o < O; ++o) atomicAdd(&acc[N::oW0 + o * H + i], x[o] * d1);
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

template <int MODE>
static int launch_cat_f64(const CatArgs64& a, int* grid_out, cudaStream_t st) {
  const size_t smem = (size_t)3 * CAT_P * sizeof(double);
  B200RL_SET_MAX_SMEM((cat_f64_kernel<MODE>), smem);
  long long grid = (long long)num_sms() * 2;
  const long long need = (a.B + 127) / 128;
  if (grid > need) grid = need;
  cat_f64_kernel<MODE><<<(unsigned)grid, 128, smem, st>>>(a);
  B200RL_LAUNCH_CHECK("cat_f64_kernel");
  *grid_out = (int)grid;
  return 0;
}

static void cat_fill_args(UpdArgs& a, const float* params, long long B, const float* obs, const float* act,
                          const float* adv, const float* old_prob, int loss_kind, const unsigned char* flags,
                          double* ws) {
  a.params = params; a.log_min_std = -INFINITY; a.B = B;
  a.obs = obs; a.act = act; a.adv = adv; a.old_mean = old_prob; a.old_log_std = nullptr;
  a.loss_kind = loss_kind; a.flags = flags; a.partial = ws;
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

long long b200rl_categorical_num_params(int obs_dim, int h1, int h2, int n_actions) {
  B200RL_REQUIRE_CAT_SHAPE(obs_dim, h1, h2, n_actions, "categorical_num_params");
  return CAT_P;
}

int b200rl_categorical_get_actions(const float* params_f32, int obs_dim, int h1, int h2, int n_actions,
                                   const float* obs, long long n, const float* u, unsigned int seed, unsigned int iter,
                                   int row, long long lane0, int* act_out, float* prob_out, void* stream) {
  B200RL_REQUIRE(params_f32 && obs && n > 0 && act_out && prob_out, "categorical_get_actions: bad arguments");
  B200RL_REQUIRE_CAT_SHAPE(obs_dim, h1, h2, n_actions, "categorical_get_actions");
  const unsigned grid = (unsigned)((n + 127) / 128);
  cat_get_actions_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(params_f32, obs, n, u, seed, iter, row, lane0,
                                                                 act_out, prob_out);
  B200RL_LAUNCH_CHECK("cat_get_actions_kernel");
  return 0;
}

int b200rl_rollout_categorical(int env_kind, const float* params_f32, int h1, int h2, int N, int T,
                               int max_path_length, const float* u, const float* reset_raw, unsigned int seed,
                               unsigned int iter, long long lane0, float* obs, float* act, float* prob, float* rew,
                               unsigned char* flags, unsigned short* tstep, void* stream) {
  const RolloutArgs a{params_f32, 0.f, N, T, max_path_length, u, reset_raw, seed, iter, lane0,
                      obs, act, prob, rew, flags, tstep, nullptr};
  if (int rc = check_rollout_args("rollout_categorical", a, false)) return rc;
  if (env_kind != B200RL_ENV_GYM_CARTPOLE) {
    set_error("rollout_categorical: env kind %d has no discrete action space compiled in (only %d, CartPole-v0)",
              env_kind, B200RL_ENV_GYM_CARTPOLE);
    return B200RL_EUNSUPPORTED;
  }
  B200RL_REQUIRE_CAT_SHAPE(GymCartPoleEnvD::O, h1, h2, EnvNumActions<GymCartPoleEnvD>::value, "rollout_categorical");
  cat_rollout_kernel<GymCartPoleEnvD><<<(N + 127) / 128, 128, 0, (cudaStream_t)stream>>>(a);
  B200RL_LAUNCH_CHECK("cat_rollout_kernel");
  return 0;
}

int b200rl_categorical_loss_kl(int loss_kind, const float* params_f32, int obs_dim, int h1, int h2, int n_actions,
                               long long B, const float* obs, const float* act, const float* adv,
                               const float* old_prob, const unsigned char* flags, double scale, const double* count,
                               double* out, double* ws, void* stream) {
  B200RL_REQUIRE(params_f32 && obs && act && adv && old_prob && out && ws && B > 0, "categorical_loss_kl: bad arguments");
  if (int rc = check_loss_kind("categorical_loss_kl", loss_kind)) return rc;
  B200RL_REQUIRE_CAT_SHAPE(obs_dim, h1, h2, n_actions, "categorical_loss_kl");
  cudaStream_t st = (cudaStream_t)stream;
  UpdArgs a{};
  cat_fill_args(a, params_f32, B, obs, act, adv, old_prob, loss_kind, flags, ws);
  const int grid = partial_grid(4, (B + 127) / 128);
  cat_loss_kernel<<<grid, 128, 0, st>>>(a);
  B200RL_LAUNCH_CHECK("cat_loss_kernel");
  return launch_finalize_update(fin_loss(ws, grid, out, scale, count), st);
}

int b200rl_categorical_grad(int loss_kind, double penalty, const float* params_f32, int obs_dim, int h1, int h2,
                            int n_actions, long long B, const float* obs, const float* act, const float* adv,
                            const float* old_prob, const unsigned char* flags, double scale, const double* count,
                            double* g_out, double* loss_out, float* h_cache_out, double* ws, void* stream) {
  B200RL_REQUIRE(params_f32 && obs && act && adv && old_prob && g_out && ws && B > 0, "categorical_grad: bad arguments");
  if (int rc = check_loss_kind("categorical_grad", loss_kind)) return rc;
  B200RL_REQUIRE(penalty >= 0.0 && penalty <= 3.0e38, "categorical_grad: penalty must be finite and >= 0");
  B200RL_REQUIRE_CAT_SHAPE(obs_dim, h1, h2, n_actions, "categorical_grad");
  cudaStream_t st = (cudaStream_t)stream;
  UpdArgs a{};
  cat_fill_args(a, params_f32, B, obs, act, adv, old_prob, loss_kind, flags, ws);
  a.h_cache = h_cache_out;
  a.penalty = (float)penalty;
  int grid = 0;
  int rc = penalty == 0.0 ? launch_cat_tile<MODE_GRAD>(a, &grid, st) : launch_cat_tile<MODE_GRAD_KL>(a, &grid, st);
  if (rc) return rc;
  // no log_std block (A = 0): the gradient's min_std mask touches no entry
  return launch_finalize_update(fin_grad(ws, grid, CAT_P, g_out, loss_out, scale, count, {CAT_P, 0, nullptr, nullptr, 0.0}),
                                st);
}

int b200rl_categorical_fvp(const float* params_f32, int obs_dim, int h1, int h2, int n_actions, long long B,
                           const float* obs, const unsigned char* flags, const double* x, double scale,
                           const double* count, double reg_coeff, double diag_scale, double* Hx_out,
                           const float* h_cache, const int* tile_list, int n_list, double* ws, void* stream) {
  B200RL_REQUIRE(params_f32 && obs && x && Hx_out && ws && B > 0, "categorical_fvp: bad arguments");
  B200RL_REQUIRE(tile_list == nullptr || n_list > 0, "categorical_fvp: empty tile list");
  B200RL_REQUIRE_CAT_SHAPE(obs_dim, h1, h2, n_actions, "categorical_fvp");
  cudaStream_t st = (cudaStream_t)stream;
  UpdArgs a{};
  cat_fill_args(a, params_f32, B, obs, nullptr, nullptr, nullptr, B200RL_LOSS_TRPO, flags, ws);
  a.xvec = x; a.h_cache = const_cast<float*>(h_cache); a.tile_list = tile_list; a.n_list = n_list;
  int grid = 0;
  int rc = launch_cat_tile<MODE_FVP>(a, &grid, st);
  if (rc) return rc;
  return launch_finalize_update(fin_fvp(ws, grid, CAT_P, Hx_out, scale, count, {CAT_P, 0, params_f32, nullptr, 0.0}, x,
                                        reg_coeff, diag_scale),   // no log_std block
                                st);
}

int b200rl_categorical_update_f64(int mode, int loss_kind, const double* params_f64, int obs_dim, int h1, int h2,
                                  int n_actions, long long B, const float* obs, const float* act, const float* adv,
                                  const float* old_prob, const unsigned char* flags, const double* x, double scale,
                                  const double* count, double reg_coeff, double diag_scale, double* vec_out,
                                  double* loss_out, double* ws, void* stream) {
  B200RL_REQUIRE(params_f64 && obs && ws && B > 0, "categorical_update_f64: bad arguments");
  if (int rc = check_f64_args("categorical_update_f64", mode, loss_kind, act && adv && old_prob, x, vec_out, loss_out))
    return rc;
  B200RL_REQUIRE_CAT_SHAPE(obs_dim, h1, h2, n_actions, "categorical_update_f64");
  cudaStream_t st = (cudaStream_t)stream;
  CatArgs64 a{};
  a.params = params_f64; a.xvec = x; a.B = B; a.obs = obs; a.act = act; a.adv = adv; a.old_prob = old_prob;
  a.loss_kind = loss_kind; a.flags = flags; a.partial = ws;
  int grid = 0;
  int rc = (mode == MODE_LOSS) ? launch_cat_f64<MODE_LOSS>(a, &grid, st)
         : (mode == MODE_GRAD) ? launch_cat_f64<MODE_GRAD>(a, &grid, st)
                               : launch_cat_f64<MODE_FVP>(a, &grid, st);
  if (rc) return rc;
  return launch_finalize_update(fin_f64(mode, ws, grid, CAT_P, vec_out, loss_out, scale, count,
                                        {CAT_P, 0, nullptr, params_f64, 0.0}, x, reg_coeff, diag_scale),
                                st);
}

int b200rl_categorical_entropy(int n_actions, long long B, const float* prob, const unsigned char* flags, double* out,
                               double* ws, void* stream) {
  B200RL_REQUIRE(prob && out && ws && B > 0, "categorical_entropy: bad arguments");
  if (n_actions != CAT_N) {
    set_error("categorical_entropy: n_actions=%d is not compiled in (only %d)", n_actions, CAT_N);
    return B200RL_EUNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = partial_grid(4, (B + 255) / 256);
  cat_entropy_kernel<<<grid, 256, 0, st>>>(B, prob, flags, ws);
  B200RL_LAUNCH_CHECK("cat_entropy_kernel");
  return launch_finalize_sum(ws, grid, 2, out, 1.0, st);
}
}
