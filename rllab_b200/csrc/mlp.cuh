// GaussianMLPPolicy mean network (rllab/policies/gaussian_mlp_policy.py:61-137, rllab/core/network.py:36-81):
//   h1 = tanh(x W0 + b0); h2 = tanh(h1 W1 + b1); mean = h2 Wout + bout; log_std = max(param, log(min_std)).
//
// Canonical summation order (shared by the thread-per-lane rollout and the warp-per-sample update kernels so
// that mean(theta_old) is bit-identical in both, i.e. the likelihood ratio at theta_old is exactly 1):
//   dot(in, w, n, bias): s0 = bias, s1 = 0; s0 += in[i]*w[i] for even i, s1 += in[i]*w[i] for odd i (fma, ascending
//   i); result = s0 + s1.   ffma2() computes an even/odd pair (two FFMAs on sm_90).
#pragma once
#include "common.cuh"

namespace b200rl {

template <int O_, int H1_, int H2_, int A_>
struct Net {
  static constexpr int O = O_, H1 = H1_, H2 = H2_, A = A_;
  static constexpr int oW0 = 0, ob0 = oW0 + O * H1, oW1 = ob0 + H1, ob1 = oW1 + H1 * H2, oWo = ob1 + H2,
                       obo = oWo + H2 * A, ols = obo + A, P = ols + A;
  static_assert(H1 % 32 == 0 && H2 % 32 == 0, "hidden sizes must be multiples of 32");
};

__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ >= 1000)
  return __ffma2_rn(a, b, c);
#else
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
#endif
}

// Gram products over the sample axis with packed FFMA2: four consecutive samples (one LDS.128 per row) are folded as two
// (even, odd) pairs, so acc.x / acc.y are the even- / odd-sample partial sums and the caller adds the halves at the end.
__device__ __forceinline__ void gram_fma4(const float4& u, const float4& v, float2& acc) {
  acc = ffma2(make_float2(u.x, u.y), make_float2(v.x, v.y), acc);
  acc = ffma2(make_float2(u.z, u.w), make_float2(v.z, v.w), acc);
}
__device__ __forceinline__ void gram_4x4(const float4 (&u)[4], const float4 (&v)[4], float2 (&acc)[4][4]) {
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) gram_fma4(u[r], v[c], acc[r][c]);
}

// Dense layer, thread-per-sample, weights W [NIN][NOUT] row-major + bias in shared memory (broadcast LDS.128).
// Output pairs (j, j+1) share one packed FFMA2; even and odd inputs accumulate in separate chains (canonical order).
// FENCE > 0 inserts a compiler memory barrier every FENCE input rows: it bounds how many weight loads ptxas may hoist
// ahead (each LDS.128 holds 4 registers), which keeps the big fused kernels from spilling.
template <int NIN, int NOUT, bool BIAS = true, int FENCE = 0>
__device__ __forceinline__ void dense_thread(const float* __restrict__ W, const float* __restrict__ b,
                                             const float (&in)[NIN], float (&pre)[NOUT]) {
  float2 ae[NOUT / 2], ao[NOUT / 2];
#pragma unroll
  for (int j = 0; j < NOUT; j += 4) {
    float4 bb = BIAS ? *reinterpret_cast<const float4*>(b + j) : make_float4(0.f, 0.f, 0.f, 0.f);
    ae[j / 2] = make_float2(bb.x, bb.y);
    ae[j / 2 + 1] = make_float2(bb.z, bb.w);
    ao[j / 2] = make_float2(0.f, 0.f);
    ao[j / 2 + 1] = make_float2(0.f, 0.f);
  }
#pragma unroll
  for (int i = 0; i < NIN; ++i) {
    if (FENCE > 0 && i > 0 && (i % FENCE) == 0) asm volatile("" ::: "memory");
    const float2 xin = make_float2(in[i], in[i]);
#pragma unroll
    for (int j = 0; j < NOUT; j += 4) {
      float4 w = *reinterpret_cast<const float4*>(W + i * NOUT + j);
      if ((i & 1) == 0) {
        ae[j / 2] = ffma2(xin, make_float2(w.x, w.y), ae[j / 2]);
        ae[j / 2 + 1] = ffma2(xin, make_float2(w.z, w.w), ae[j / 2 + 1]);
      } else {
        ao[j / 2] = ffma2(xin, make_float2(w.x, w.y), ao[j / 2]);
        ao[j / 2 + 1] = ffma2(xin, make_float2(w.z, w.w), ao[j / 2 + 1]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < NOUT; j += 2) {
    pre[j] = ae[j / 2].x + ao[j / 2].x;
    pre[j + 1] = ae[j / 2].y + ao[j / 2].y;
  }
}

// Same layer with the INPUT vector read from this thread's column of a shared-memory matrix (in_col[i * ld]) and a
// rolled loop over input pairs: for 64-wide layers the fully unrolled form is ~90 KB of code per layer and thrashes
// the instruction cache (ncu: "no_instructions" was the top stall of the Hopper rollout, icc hit rate 73 %).
template <int NIN, int NOUT>
__device__ __forceinline__ void dense_thread_col(const float* __restrict__ W, const float* __restrict__ b,
                                                 const float* in_col, int ld, float (&pre)[NOUT]) {
  static_assert(NIN % 2 == 0, "even number of inputs");
  float2 ae[NOUT / 2], ao[NOUT / 2];
#pragma unroll
  for (int j = 0; j < NOUT; j += 4) {
    const float4 bb = *reinterpret_cast<const float4*>(b + j);
    ae[j / 2] = make_float2(bb.x, bb.y);
    ae[j / 2 + 1] = make_float2(bb.z, bb.w);
    ao[j / 2] = make_float2(0.f, 0.f);
    ao[j / 2 + 1] = make_float2(0.f, 0.f);
  }
#pragma unroll 1
  for (int i = 0; i < NIN; i += 2) {
    const float a0 = in_col[i * ld], a1 = in_col[(i + 1) * ld];
    const float2 x0 = make_float2(a0, a0), x1 = make_float2(a1, a1);
#pragma unroll
    for (int j = 0; j < NOUT; j += 4) {
      const float4 w0 = *reinterpret_cast<const float4*>(W + i * NOUT + j);
      const float4 w1 = *reinterpret_cast<const float4*>(W + (i + 1) * NOUT + j);
      ae[j / 2] = ffma2(x0, make_float2(w0.x, w0.y), ae[j / 2]);
      ae[j / 2 + 1] = ffma2(x0, make_float2(w0.z, w0.w), ae[j / 2 + 1]);
      ao[j / 2] = ffma2(x1, make_float2(w1.x, w1.y), ao[j / 2]);
      ao[j / 2 + 1] = ffma2(x1, make_float2(w1.z, w1.w), ao[j / 2 + 1]);
    }
  }
#pragma unroll
  for (int j = 0; j < NOUT; j += 2) {
    pre[j] = ae[j / 2].x + ao[j / 2].x;
    pre[j + 1] = ae[j / 2].y + ao[j / 2].y;
  }
}

// Thread-per-sample forward, parameters in shared memory.
template <class N>
__device__ __forceinline__ void mlp_forward_thread(const float* __restrict__ sp, const float (&x)[N::O],
                                                   float (&h1)[N::H1], float (&h2)[N::H2], float (&mu)[N::A],
                                                   float* hcol = nullptr, int hld = 0) {
  dense_thread<N::O, N::H1>(sp + N::oW0, sp + N::ob0, x, h1);
#pragma unroll
  for (int j = 0; j < N::H1; ++j) h1[j] = tanh_f(h1[j]);
  if (N::H1 > 32 && hcol != nullptr) {
#pragma unroll
    for (int j = 0; j < N::H1; ++j) hcol[j * hld] = h1[j];
    dense_thread_col<N::H1, N::H2>(sp + N::oW1, sp + N::ob1, hcol, hld, h2);
  } else {
    dense_thread<N::H1, N::H2>(sp + N::oW1, sp + N::ob1, h1, h2);
  }
#pragma unroll
  for (int j = 0; j < N::H2; ++j) h2[j] = tanh_f(h2[j]);
#pragma unroll
  for (int a = 0; a < N::A; ++a) {
    float s0 = sp[N::obo + a], s1 = 0.f;
#pragma unroll
    for (int j = 0; j < N::H2; j += 2) {
      s0 = fmaf(h2[j], sp[N::oWo + j * N::A + a], s0);
      s1 = fmaf(h2[j + 1], sp[N::oWo + (j + 1) * N::A + a], s1);
    }
    mu[a] = s0 + s1;
  }
}

// log_std after the min_std clamp (gaussian_mlp_policy.py:100-101): max(param, log(min_std))
__device__ __forceinline__ float clamp_log_std(float param, float log_min_std) { return fmaxf(param, log_min_std); }

// Supported network shapes: (O, A) of the compiled env kinds x hidden (32,32) | (64,64).
#define B200RL_DISPATCH_NET_OA(O_, A_, H_, ...)                                             \
  if (obs_dim == O_ && act_dim == A_ && h1 == H_ && h2 == H_) {                              \
    using NetT = ::b200rl::Net<O_, H_, H_, A_>;                                              \
    __VA_ARGS__;                                                                             \
  } else

#define B200RL_DISPATCH_NET_H(H_, ...)                                                       \
  B200RL_DISPATCH_NET_OA(2, 2, H_, __VA_ARGS__)                                              \
  B200RL_DISPATCH_NET_OA(4, 1, H_, __VA_ARGS__)                                              \
  B200RL_DISPATCH_NET_OA(3, 1, H_, __VA_ARGS__)                                              \
  B200RL_DISPATCH_NET_OA(6, 1, H_, __VA_ARGS__)                                              \
  B200RL_DISPATCH_NET_OA(13, 2, H_, __VA_ARGS__)                                             \
  B200RL_DISPATCH_NET_OA(20, 3, H_, __VA_ARGS__)                                             \
  B200RL_DISPATCH_NET_OA(20, 6, H_, __VA_ARGS__)                                             \
  {                                                                                          \
    ::b200rl::set_error("network shape O=%d A=%d hidden=(%d,%d) is not compiled in", obs_dim, act_dim, h1, h2); \
    return B200RL_EUNSUPPORTED;                                                              \
  }

#define B200RL_DISPATCH_NET(...)                                                             \
  B200RL_DISPATCH_NET_OA(2, 2, 32, __VA_ARGS__)                                              \
  B200RL_DISPATCH_NET_OA(4, 1, 32, __VA_ARGS__)                                              \
  B200RL_DISPATCH_NET_OA(3, 1, 32, __VA_ARGS__)                                              \
  B200RL_DISPATCH_NET_OA(6, 1, 32, __VA_ARGS__)                                              \
  B200RL_DISPATCH_NET_OA(13, 2, 32, __VA_ARGS__)                                             \
  B200RL_DISPATCH_NET_OA(20, 3, 32, __VA_ARGS__)                                             \
  B200RL_DISPATCH_NET_OA(2, 2, 64, __VA_ARGS__)                                              \
  B200RL_DISPATCH_NET_OA(4, 1, 64, __VA_ARGS__)                                              \
  B200RL_DISPATCH_NET_OA(3, 1, 64, __VA_ARGS__)                                              \
  B200RL_DISPATCH_NET_OA(6, 1, 64, __VA_ARGS__)                                              \
  B200RL_DISPATCH_NET_OA(13, 2, 64, __VA_ARGS__)                                             \
  B200RL_DISPATCH_NET_OA(20, 3, 64, __VA_ARGS__)                                             \
  B200RL_DISPATCH_NET_OA(20, 6, 32, __VA_ARGS__)                                             \
  B200RL_DISPATCH_NET_OA(20, 6, 64, __VA_ARGS__)                                             \
  {                                                                                          \
    ::b200rl::set_error("network shape O=%d A=%d hidden=(%d,%d) is not compiled in", obs_dim, act_dim, h1, h2); \
    return B200RL_EUNSUPPORTED;                                                              \
  }

inline bool net_supported(int O, int h1, int h2, int A) {
  if (h1 != h2 || (h1 != 32 && h1 != 64)) return false;
  return (O == 2 && A == 2) || (O == 4 && A == 1) || (O == 3 && A == 1) || (O == 6 && A == 1) || (O == 13 && A == 2) || (O == 20 && A == 3) ||
         (O == 20 && A == 6);
}

}  // namespace b200rl
