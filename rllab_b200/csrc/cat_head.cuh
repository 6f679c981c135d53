// The softmax head shared by the categorical policies (CategoricalMLPPolicy in categorical.cu, CategoricalGRUPolicy in
// gru.cu; rllab/distributions/categorical.py, rllab/misc/special.py): softmax, the weighted_sample draw and its
// uniforms, the per-sample surrogate and KL terms, and the logit-space derivatives of both passes.
#pragma once
#include "common.cuh"

namespace b200rl {

constexpr float CAT_TINY = 1e-8f;   // TINY of rllab/distributions/categorical.py

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

}  // namespace b200rl
