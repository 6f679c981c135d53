// Shared device/host helpers for libb200rl (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/b200rl.h"

namespace b200rl {

// ---------------------------------------------------------------- error handling (C ABI: status + message)
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);

#define B200RL_CUDA_CHECK(expr)                                   \
  do {                                                            \
    cudaError_t _e = (expr);                                      \
    if (_e != cudaSuccess) return ::b200rl::cuda_fail(_e, #expr); \
  } while (0)

extern unsigned long long g_kernel_launches;  // every kernel launch of the library passes through LAUNCH_CHECK

#define B200RL_LAUNCH_CHECK(name)                                 \
  do {                                                            \
    ++::b200rl::g_kernel_launches;                                \
    cudaError_t _e = cudaGetLastError();                          \
    if (_e != cudaSuccess) return ::b200rl::cuda_fail(_e, name);  \
  } while (0)

#define B200RL_REQUIRE(cond, ...)       \
  do {                                  \
    if (!(cond)) {                      \
      ::b200rl::set_error(__VA_ARGS__); \
      return B200RL_EINVAL;             \
    }                                   \
  } while (0)

int num_sms();

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a per-DEVICE attribute: guard it per (kernel instantiation, device)
// so that a process that drives several GPUs sets it on each of them (one static mask per call site).
#define B200RL_SET_MAX_SMEM(kernel, bytes)                                                           \
  do {                                                                                               \
    static unsigned long long _done_mask = 0ull;                                                     \
    int _dev = 0;                                                                                    \
    B200RL_CUDA_CHECK(cudaGetDevice(&_dev));                                                         \
    if (!((_done_mask >> (_dev & 63)) & 1ull)) {                                                     \
      B200RL_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,    \
                                             (int)(bytes)));                                         \
      _done_mask |= 1ull << (_dev & 63);                                                             \
    }                                                                                                \
  } while (0)

// partial-reduction workspace geometry: every reduction kernel uses at most MAX_PARTIAL_BLOCKS blocks and
// writes [block][K] float64 partials; K <= MAX_PARTIAL_K.  (8 blocks per SM on GPUs of up to 148 SMs.)
constexpr int MAX_PARTIAL_BLOCKS = 148 * 8;
constexpr int MAX_PARTIAL_K = 8192;

// ---------------------------------------------------------------- Philox4x32-10 (Salmon et al. 2011)
struct Philox {
  static constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
  __host__ __device__ static inline void round(uint32_t c[4], uint32_t k0, uint32_t k1) {
#ifdef __CUDA_ARCH__
    uint32_t hi0 = __umulhi(M0, c[0]), hi1 = __umulhi(M1, c[2]);
#else
    uint32_t hi0 = (uint32_t)(((uint64_t)M0 * c[0]) >> 32), hi1 = (uint32_t)(((uint64_t)M1 * c[2]) >> 32);
#endif
    uint32_t lo0 = M0 * c[0], lo1 = M1 * c[2];
    uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
  }
  __host__ __device__ static inline void gen(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                             uint32_t k1, uint32_t out[4]) {
    uint32_t c[4] = {c0, c1, c2, c3};
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      round(c, k0, k1);
      k0 += W0;
      k1 += W1;
    }
    out[0] = c[0]; out[1] = c[1]; out[2] = c[2]; out[3] = c[3];
  }
};

// counter = (lane, row | stream<<28, chunk, lane>>32), key = (seed, iter).  Four floats per call.
// uniform: (x>>8) * 2^-24 in [0,1);  normal: Box-Muller on ((x>>8)+0.5)*2^-24 in (0,1).
// NPAIRS: how many of the two Box-Muller pairs are needed (action noise of a 1- or 2-dimensional action space only
// consumes the first pair: half the log / sqrt / sincospi work of the hot loop).
template <int NPAIRS = 2>
__device__ __forceinline__ void noise4(int kind, uint32_t seed, uint32_t iter, int stream_id, long long lane, int row,
                                       int chunk, float out[4]) {
  uint32_t r[4];
  Philox::gen((uint32_t)lane, (uint32_t)row | ((uint32_t)stream_id << 28), (uint32_t)chunk,
              (uint32_t)((unsigned long long)lane >> 32), seed, iter, r);
  const float s = 1.0f / 16777216.0f;
  if (kind == B200RL_NOISE_UNIFORM) {
#pragma unroll
    for (int i = 0; i < 4; ++i) out[i] = (float)(r[i] >> 8) * s;
  } else {
#pragma unroll
    for (int i = 0; i < 2 * NPAIRS; i += 2) {
      const float u1 = ((float)(r[i] >> 8) + 0.5f) * s;          // in (0, 1]: 16777215.5 rounds up to 2^24 in float32
      const float u2 = ((float)(r[i + 1] >> 8) + 0.5f) * s;
      // IEEE sqrtf on purpose: u1 == 1 gives t == 0 and t * rsqrtf(t) would be 0 * inf = NaN (one sample in 2^24 --
      // caught by tests/test_gpu_fullsize.py on the 13.1 M-sample batch)
      const float rad = sqrtf(-2.0f * logf(u1));
      float sn, cs;
      sincospif(2.0f * u2, &sn, &cs);
      out[i] = rad * cs;
      out[i + 1] = rad * sn;
    }
  }
}

// ---------------------------------------------------------------- math
// tanh used by every kernel (rollout and update MUST share it so that the likelihood ratio is exactly 1 at
// theta_old): 1 - 2 / (2^(2 log2(e) x) + 1) with MUFU.EX2 + MUFU.RCP -- 5 instructions instead of tanhf's ~14 (tanhf was
// 39 % of the rollout's instruction stream); saturates correctly (+inf -> 1, 0 -> -1); absolute error <= ~4e-7 (relative
// accuracy is lost near 0, which the activations do not need: policy mean off by 8e-7 of its scale against a test
// tolerance of 2e-5).
__device__ __forceinline__ float tanh_f(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * 2.885390081777927f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.0f));
  return fmaf(-2.0f, r, 1.0f);
}

// ---------------------------------------------------------------- reductions
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum of K per-thread doubles; result valid in thread 0..K-1? -> written to out[k] by thread 0.
// scratch: K * 32 doubles of shared memory.  Fixed order -> deterministic.
template <int K, bool IS_MAX = false>
__device__ inline void block_reduce_store(const double (&v)[K], double* scratch, double* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double s = IS_MAX ? warp_max(v[k]) : warp_sum(v[k]);
    if (lane == 0) scratch[k * 32 + warp] = s;
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      double s = lane < nwarp ? scratch[k * 32 + lane] : (IS_MAX ? -1.0e300 : 0.0);
      s = IS_MAX ? warp_max(s) : warp_sum(s);
      if (lane == 0) out[k] = s;
    }
  }
  __syncthreads();
}

// finalize: out[k] = post(sum_b partial[b][k]) in fixed block order; one thread per k.
int launch_finalize_sum(const double* partial, int nblocks, int K, double* out, double scale, cudaStream_t s);
int launch_finalize_max(const double* partial, int nblocks, int K, double* out, cudaStream_t s);

// Fused finalize of one policy-update pass (one launch instead of finalize + mask/diag + 2 x finalize + memcpy):
//   vec_out[k]  = sum_b partial[b][k] * scale / (*count)            k < K            (count == NULL -> 1)
//   tri_out[0..NT-2] = sum_b tri_partial[b][j] * scale / (*count),  tri_out[NT-1] = max_b tri_partial[b][NT-1]
//   post == FIN_GRAD : vec_out[ols + a] = 0 where the min_std clamp is active
//   post == FIN_FVP  : vec_out[p] += diag_scale * (reg * x[p] (+ M_l x_l on un-clamped log_std entries))
// The count is read from DEVICE memory (the all-reduced number of valid samples, sums[2] of b200rl_process_samples):
// with whole-path masking the divisor of every mean is only known on the device, and reading it there keeps the
// iteration free of host synchronisation.
//   peer.world > 1   : the vector and the tuple are additionally reduced over the ranks of the bound peer-memory
//                      communicator in the same launch (peer.cuh): sums (and the tuple's max) of every rank's result
constexpr int FIN_NONE = 0, FIN_GRAD = 1, FIN_FVP = 2;
constexpr int PEER_MAX_RANKS = B200RL_PEER_MAX_RANKS;
struct PeerArgs {
  unsigned char* win[PEER_MAX_RANKS];   // exchange-window base pointers, indexed by rank (entry `rank` = own window)
  int rank, world;                      // world <= 1: no exchange
  long long n_cap;                      // doubles per slot
  unsigned long long seq;               // 1-based sequence number of this collective (identical on all ranks)
};
bool peer_fused();                      // a communicator is bound and fusion into the update passes is enabled
PeerArgs peer_next();                   // arguments of the next collective (consumes one sequence number)
struct FinArgs {
  const double* partial; int nblocks; int K; double* vec_out;
  const double* tri_partial; int NT; double* tri_out;
  double scale; const double* count;
  int post, ols, A;
  const float* params32; const double* params64; double log_min_std;
  const double* x; double reg, diag_scale;
  PeerArgs peer;
};
int launch_finalize_update(const FinArgs& f, cudaStream_t s);

}  // namespace b200rl
