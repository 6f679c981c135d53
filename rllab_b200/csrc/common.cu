// Error plumbing, device queries and the fixed-order finalize kernels shared by every reduction.
#include <stdarg.h>

#include "peer.cuh"

namespace b200rl {

static thread_local char g_err[512] = "";
unsigned long long g_kernel_launches = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return B200RL_ECUDA;
}

int num_sms() {
  static int cached[64] = {0};       // per device: a process may drive several GPUs
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (cached[dev & 63] > 0) return cached[dev & 63];
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) return 132;
  cached[dev & 63] = sms;
  return sms;
}

int partial_grid(int blocks_per_sm, long long work) {
  long long g = (long long)num_sms() * blocks_per_sm;
  if (g > work) g = work;
  if (g > MAX_PARTIAL_BLOCKS) g = MAX_PARTIAL_BLOCKS;
  return (int)(g < 1 ? 1 : g);
}

// out[k] = op over blocks of partial[b][k].  32 outputs x FIN_SLICES block-slices per CTA: each slice walks every
// FIN_SLICES-th block (coalesced 256 B rows, 4 loads in flight), the slices are combined through shared memory in fixed
// order, so the result is deterministic and the dependent-add chain is nblocks/FIN_SLICES long instead of nblocks.
constexpr int FIN_SLICES = 32, FIN_THREADS = 32 * FIN_SLICES;
template <bool IS_MAX>
__global__ void __launch_bounds__(FIN_THREADS) finalize_kernel(const double* __restrict__ partial, int nblocks, int K,
                                                       double* __restrict__ out, double scale) {
  __shared__ double sm[FIN_SLICES][33];
  const int kx = threadIdx.x & 31, by = threadIdx.x >> 5;
  const int k = blockIdx.x * 32 + kx;
  double acc = IS_MAX ? -1.0e300 : 0.0;
  if (k < K) {
#pragma unroll 4
    for (int b = by; b < nblocks; b += FIN_SLICES) {
      const double v = partial[(size_t)b * K + k];
      acc = IS_MAX ? fmax(acc, v) : acc + v;
    }
  }
  sm[by][kx] = acc;
  __syncthreads();
  if (by == 0 && k < K) {
    double r = sm[0][kx];
#pragma unroll
    for (int y = 1; y < FIN_SLICES; ++y) r = IS_MAX ? fmax(r, sm[y][kx]) : r + sm[y][kx];
    out[k] = IS_MAX ? r : r * scale;
  }
}

int launch_finalize_sum(const double* partial, int nblocks, int K, double* out, double scale, cudaStream_t s) {
  finalize_kernel<false><<<(K + 31) / 32, FIN_THREADS, 0, s>>>(partial, nblocks, K, out, scale);
  B200RL_LAUNCH_CHECK("finalize_kernel<sum>");
  return 0;
}

int launch_finalize_max(const double* partial, int nblocks, int K, double* out, cudaStream_t s) {
  finalize_kernel<true><<<(K + 31) / 32, FIN_THREADS, 0, s>>>(partial, nblocks, K, out, 1.0);
  B200RL_LAUNCH_CHECK("finalize_kernel<max>");
  return 0;
}

// see common.cuh: blocks [0, ceil(K/32)) reduce the vector, one extra block reduces the loss/KL tuple.  With a peer
// communicator (f.peer.world > 1) every block pushes its outputs into slot[rank] of all exchange windows instead of
// writing them out, the last block to finish signals the peers, and every block then folds the `world` slots of the own
// window in rank order (peer.cuh) -- the reduction over blocks and the all-reduce over GPUs are one launch.
__global__ void __launch_bounds__(FIN_THREADS) finalize_update_kernel(FinArgs f) {
  __shared__ double sm[FIN_SLICES][33];
  __shared__ int sh_last, sh_ok;
  const int kx = threadIdx.x & 31, by = threadIdx.x >> 5;
  const double sc = f.scale / (f.count != nullptr ? f.count[0] : 1.0);
  const int nvb = (f.K + 31) / 32;
  const bool is_vec = (int)blockIdx.x < nvb;
  const bool peered = f.peer.world > 1;
  const int par = (int)(f.peer.seq & 1ull);
  // index of this thread's output in the exchanged message [vector | tuple], -1: none
  long long slot_i = -1;
  bool is_max = false;
  double r = 0.0;
  if (is_vec) {
    const int k = blockIdx.x * 32 + kx;
    double acc = 0.0;
    if (k < f.K) {
#pragma unroll 4
      for (int b = by; b < f.nblocks; b += FIN_SLICES) acc += f.partial[(size_t)b * f.K + k];
    }
    sm[by][kx] = acc;
    __syncthreads();
    if (by == 0 && k < f.K) {
      r = sm[0][kx];
#pragma unroll
      for (int y = 1; y < FIN_SLICES; ++y) r += sm[y][kx];
      r *= sc;
      const bool is_ls = (k >= f.ols && k < f.ols + f.A);
      if (f.post == FIN_GRAD) {
        // TT.maximum routes the gradient to the constant where the min_std clamp is active (gaussian_mlp_policy.py:100)
        if (is_ls) {
          const double par_k = f.params64 ? f.params64[k] : (double)f.params32[k];
          if (!(par_k > f.log_min_std)) r = 0.0;
        }
      } else if (f.post == FIN_FVP) {
        // the log_std slot of the sample sum is zero (the mean does not depend on log_std): reg * x and the M_l block
        double add = f.reg * f.x[k];
        if (is_ls) {
          const double par_k = f.params64 ? f.params64[k] : (double)f.params32[k];
          r = 0.0;
          if (par_k > f.log_min_std) {
            const double s = exp(2.0 * par_k), eps = 1e-8;
            add += 4.0 * s * (2.0 * s - eps) / ((2.0 * s + eps) * (2.0 * s + eps)) * f.x[k];
          }
        }
        r += f.diag_scale * add;
      }
      slot_i = k;
      if (!peered) f.vec_out[k] = r;
    }
  } else if (f.tri_out != nullptr) {
    // tuple: entries [0, NT-1) are sums, entry NT-1 is a max; thread (by, kx): kx < NT handles column kx
    double acc = (kx == f.NT - 1) ? -1.0e300 : 0.0;
    if (kx < f.NT) {
      for (int b = by; b < f.nblocks; b += FIN_SLICES) {
        const double v = f.tri_partial[(size_t)b * f.NT + kx];
        acc = (kx == f.NT - 1) ? fmax(acc, v) : acc + v;
      }
    }
    sm[by][kx] = acc;
    __syncthreads();
    if (by == 0 && kx < f.NT) {
      r = sm[0][kx];
      is_max = (kx == f.NT - 1);
#pragma unroll
      for (int y = 1; y < FIN_SLICES; ++y) r = is_max ? fmax(r, sm[y][kx]) : r + sm[y][kx];
      if (!is_max) r *= sc;
      slot_i = f.K + kx;
      if (!peered) f.tri_out[kx] = r;
    }
  }
  if (!peered) return;
  // ---- exchange over the peer windows
  if (slot_i >= 0)
    for (int w = 0; w < f.peer.world; ++w) peer_slot(f.peer, w, par, f.peer.rank)[slot_i] = r;
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    sh_ok = 1;
    unsigned int* cnt = peer_done_counter(f.peer.win[f.peer.rank]);
    const unsigned int prev = atomicAdd(cnt, 1u);
    sh_last = (prev == gridDim.x - 1) ? 1 : 0;
    if (sh_last) {
      *cnt = 0u;                 // every block has counted: ready for the next collective (next launch on this stream)
      __threadfence_system();
    }
  }
  __syncthreads();
  if (sh_last && (int)threadIdx.x < f.peer.world) peer_signal(f.peer, threadIdx.x);
  if ((int)threadIdx.x < f.peer.world && !peer_wait(f.peer, threadIdx.x)) sh_ok = 0;
  __syncthreads();
  if (slot_i >= 0) {
    double acc = peer_slot(f.peer, f.peer.rank, par, 0)[slot_i];
    for (int w = 1; w < f.peer.world; ++w) {
      const double v = peer_slot(f.peer, f.peer.rank, par, w)[slot_i];
      acc = is_max ? fmax(acc, v) : acc + v;
    }
    if (!sh_ok) acc = __longlong_as_double(0x7FF8000000000000ll);    // a peer never arrived: poison
    if (is_vec) f.vec_out[slot_i] = acc; else f.tri_out[slot_i - f.K] = acc;
  }
}

int launch_finalize_update(FinArgs f, cudaStream_t s) {
  if (peer_fused()) f.peer = peer_next();
  const int nvb = (f.K + 31) / 32;
  finalize_update_kernel<<<nvb + (f.tri_out != nullptr ? 1 : 0), FIN_THREADS, 0, s>>>(f);
  B200RL_LAUNCH_CHECK("finalize_update_kernel");
  return 0;
}

FinArgs fin_loss(const double* ws, int grid, double* tri_out, double scale, const double* count) {
  FinArgs f{};
  f.nblocks = grid;
  f.tri_partial = ws; f.NT = 3; f.tri_out = tri_out;
  f.scale = scale; f.count = count; f.post = FIN_NONE;
  return f;
}

static void set_log_std(FinArgs& f, const LogStdBlock& ls) {
  f.ols = ls.ols; f.A = ls.A;
  f.params32 = ls.params32; f.params64 = ls.params64; f.log_min_std = ls.log_min_std;
}

FinArgs fin_grad(const double* ws, int grid, int P, double* vec_out, double* tri_out, double scale, const double* count,
                 const LogStdBlock& ls) {
  FinArgs f{};
  f.partial = ws; f.nblocks = grid; f.K = P; f.vec_out = vec_out;
  f.tri_partial = ws + (size_t)grid * P; f.NT = 3; f.tri_out = tri_out;
  f.scale = scale; f.count = count; f.post = FIN_GRAD;
  set_log_std(f, ls);
  return f;
}

FinArgs fin_fvp(const double* ws, int grid, int P, double* vec_out, double scale, const double* count,
                const LogStdBlock& ls, const double* x, double reg, double diag_scale) {
  FinArgs f{};
  f.partial = ws; f.nblocks = grid; f.K = P; f.vec_out = vec_out;
  f.scale = scale; f.count = count; f.post = FIN_FVP;
  set_log_std(f, ls);
  f.x = x; f.reg = reg; f.diag_scale = diag_scale;
  return f;
}

FinArgs fin_f64(int mode, const double* ws, int grid, int P, double* vec_out, double* tri_out, double scale,
                const double* count, const LogStdBlock& ls, const double* x, double reg, double diag_scale) {
  if (mode == MODE_LOSS) return fin_loss(ws, grid, tri_out, scale, count);
  if (mode == MODE_GRAD) return fin_grad(ws, grid, P, vec_out, tri_out, scale, count, ls);
  return fin_fvp(ws, grid, P, vec_out, scale, count, ls, x, reg, diag_scale);
}

int check_loss_kind(const char* entry, int loss_kind) {
  B200RL_REQUIRE(loss_kind == B200RL_LOSS_TRPO || loss_kind == B200RL_LOSS_VPG, "%s: bad loss kind", entry);
  return 0;
}

int check_f64_args(const char* entry, int mode, int loss_kind, bool inputs_ok, const double* x, const double* vec_out,
                   const double* loss_out) {
  B200RL_REQUIRE(mode == MODE_LOSS || mode == MODE_GRAD || mode == MODE_FVP, "%s: bad mode", entry);
  B200RL_REQUIRE(mode == MODE_FVP ? (x && vec_out) : inputs_ok, "%s: null buffer", entry);
  B200RL_REQUIRE(mode != MODE_GRAD || vec_out, "%s: gradient output missing", entry);
  B200RL_REQUIRE(mode != MODE_LOSS || loss_out, "%s: loss output missing", entry);
  B200RL_REQUIRE(loss_kind == B200RL_LOSS_TRPO || loss_kind == B200RL_LOSS_VPG ||
                 (loss_kind == B200RL_LOSS_KL && mode == MODE_GRAD), "%s: bad loss kind", entry);
  return 0;
}

// FP32 issue-rate microbenchmark: 16 independent float2 FMA chains per thread (two scalar FFMAs each on sm_90, one
// packed FFMA2 where the GPU has it), no memory traffic.  bench.py times it with CUDA events to obtain the FP32 roofline
// of the GPU it runs on: the policy passes are bound by FP32 / instruction issue, not by HBM.
__global__ void __launch_bounds__(256) peak_ffma2_kernel(int iters, float seed, float* __restrict__ sink) {
  float2 acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = make_float2(seed + (float)i, seed - (float)i);
  const float2 m = make_float2(0.999f, 1.001f), c = make_float2(1e-3f, -1e-3f);
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ >= 1000)
      acc[i] = __ffma2_rn(acc[i], m, c);
#else
      acc[i] = make_float2(fmaf(acc[i].x, m.x, c.x), fmaf(acc[i].y, m.y, c.y));
#endif
    }
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) s += acc[i].x + acc[i].y;
  if (s == 12345.678f) sink[0] = s;    // never true: keeps the chains alive
}

}  // namespace b200rl

extern "C" {

int b200rl_bench_ffma2(int iters, float* sink, long long* fma_out, void* stream) {
  B200RL_REQUIRE(iters > 0 && sink, "bench_ffma2: bad arguments");
  const int blocks = b200rl::num_sms() * 8;
  b200rl::peak_ffma2_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(iters, 1.0f, sink);
  B200RL_LAUNCH_CHECK("peak_ffma2_kernel");
  if (fma_out) *fma_out = (long long)blocks * 256 * (long long)iters * 16 * 2;   // scalar FMAs (2 per packed FFMA2)
  return 0;
}

const char* b200rl_last_error(void) { return b200rl::g_err; }

int b200rl_version(void) { return B200RL_VERSION; }

int b200rl_device_sms(int* sms_out) {
  int dev = 0, sms = 0;
  B200RL_CUDA_CHECK(cudaGetDevice(&dev));
  B200RL_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (sms_out) *sms_out = sms;
  return 0;
}

unsigned long long b200rl_kernel_launches(void) { return b200rl::g_kernel_launches; }

long long b200rl_ws_doubles(void) {
  return (long long)b200rl::MAX_PARTIAL_BLOCKS * b200rl::MAX_PARTIAL_K;
}
}
