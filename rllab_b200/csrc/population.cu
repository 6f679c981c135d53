// Population kernels of the cross-entropy method: parameter sampling, a rollout in which every member of the
// population has its own policy, and the elite update.
//
// Replaces: rllab/algos/cem.py:30-59 (_worker_rollout_policy: sample params, n_evals rollouts, fitness = mean - stderr of
// the evals), rllab/sampler/utils.py:6-43 (rollout, one episode from reset to done or max_path_length),
// rllab/algos/cem.py:138-145 (argsort of the fitness, mean / std of the best rows, best_x).
//
// Population rollout, one warp per member.  The lane rollout (rollout.cu) shares one theta over the whole CTA and reads
// every weight with a broadcast LDS; here every member has its own theta, which cannot be broadcast and is far too large
// to stream per step.  So a warp owns one member at a time: thread j holds hidden unit j (j and j+32 for 64-wide nets):
// its column of W0, b0[j], its column of W1 (32-wide nets; 64-wide nets and Hopper keep W1 in the warp's shared memory)
// and b1[j].
// The activations of a layer are broadcast through a per-warp shared-memory row, the output layer (Wout, bout, also in the
// warp's shared memory) is summed redundantly by every thread from that row.  The env state, the action noise and the
// reset noise are computed redundantly by all 32 threads, so the control flow stays warp-uniform.  The warp runs the
// member's n_evals episodes one after another, then takes the next member from a global counter (persistent grid): a
// member whose episodes end early frees its warp at once.
//
// Every hidden unit keeps the canonical even/odd fmaf chains of dense_thread / dense_thread_col (mlp.cuh), and tanh_f,
// Env::step, scale_action and noise4 are the lane rollout's own, so episode (m, e) is bit-identical to the first path of
// lane e of b200rl_rollout with the float32 shadow of theta_m, N = n_evals and lane0 = lane0 + m * n_evals.
#include "envs.cuh"
#include "mlp.cuh"

namespace b200rl {

constexpr int POP_THREADS = 128;           // 4 warps = 4 members in flight per CTA
constexpr int POP_WARPS = POP_THREADS / 32;
constexpr int POP_STREAM = 2;              // Philox stream of the parameter draws (0 = action noise, 1 = reset noise)

// Register budget: the classic-control envs with 32-wide nets fit 128 registers (4 CTAs = 16 warps per SM) without
// spilling (80 registers spill 100-200 bytes); the planar envs and the 64-wide nets take what they need.
template <class Env, int H>
constexpr int pop_minblocks() { return (H == 32 && Env::S <= 4) ? 4 : 1; }

// Per-warp shared memory, in floats: activation row [H], Wout [H][A], bout [A rounded up to 4], and W1 [H][H] for
// 64-wide nets and for 20-input nets (Hopper's 23-float state and HalfCheetah's 18 leave no room for a
// register-resident W1 column).
template <class Env, int H>
struct PopLayout {
  static constexpr int oH = 0, oWo = oH + H, oBo = oWo + H * Env::A, oW1 = oBo + ((Env::A + 3) & ~3);
  static constexpr bool W1_SMEM = H > 32 || Env::O > 13;
  static constexpr int FLOATS = oW1 + (W1_SMEM ? H * H : 0);
  static_assert(oWo % 4 == 0 && oBo % 4 == 0 && oW1 % 4 == 0, "float4 alignment of the per-warp rows");
};

struct PopArgs {
  const double* theta;          // [M][P] float64 rows
  float log_min_std;
  int M, E, max_path_length;
  double discount;
  uint32_t seed, iter;
  long long lane0;
  double *ret, *undisc;         // [M][E]
  int* len;                     // [M][E]
  float *obs_first, *obs_last;  // [M][E][O] or NULL
  double* member;               // [M][3]: fitness, statistic of the undiscounted returns, mean action std
  unsigned long long* next;     // work counter (zeroed before the launch)
};

// mean - std(ddof = 1 if n > 1 else 0) / sqrt(n) of x[0..n) (cem.py:15-27 at time index 0)
__device__ __forceinline__ double stderr_lb(const double* x, int n) {
  double s = 0.0;
  for (int i = 0; i < n; ++i) s += x[i];
  const double mu = s / n;
  double v = 0.0;
  for (int i = 0; i < n; ++i) v += (x[i] - mu) * (x[i] - mu);
  const double sd = sqrt(v / (n > 1 ? n - 1 : 1));
  return mu - sd / sqrt((double)n);
}

template <class Env, int H>
__global__ void __launch_bounds__(POP_THREADS, pop_minblocks<Env, H>()) population_rollout_kernel(PopArgs a) {
  using N_ = Net<Env::O, H, H, Env::A>;
  using LY = PopLayout<Env, H>;
  constexpr int O = Env::O, A = Env::A, U = H / 32;
  extern __shared__ __align__(16) float pop_smem[];
  const int lane = threadIdx.x & 31;
  float* ws = pop_smem + (threadIdx.x >> 5) * LY::FLOATS;
  float* hrow = ws + LY::oH;
  const float4* hrow4 = reinterpret_cast<const float4*>(hrow);
  float* wo = ws + LY::oWo;
  float* bo = ws + LY::oBo;
  float* w1s = ws + LY::oW1;

  for (;;) {
    unsigned long long mm = 0;
    if (lane == 0) mm = atomicAdd(a.next, 1ull);
    mm = __shfl_sync(0xffffffffu, mm, 0);
    if (mm >= (unsigned long long)a.M) break;
    const int m = (int)mm;
    const double* th = a.theta + (size_t)m * N_::P;

    // stage the member's policy, rounded to float32 (the float32 shadow the lane rollout reads)
    float w0[U][O], b0[U], b1[U];
    float w1[LY::W1_SMEM ? 1 : U][LY::W1_SMEM ? 1 : H];
    __syncwarp();   // the previous member's last reads of the shared rows are done
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int j = lane + 32 * u;
#pragma unroll
      for (int i = 0; i < O; ++i) w0[u][i] = (float)th[N_::oW0 + i * H + j];
      b0[u] = (float)th[N_::ob0 + j];
      b1[u] = (float)th[N_::ob1 + j];
      if (!LY::W1_SMEM) {
#pragma unroll
        for (int i = 0; i < H; ++i) w1[LY::W1_SMEM ? 0 : u][LY::W1_SMEM ? 0 : i] = (float)th[N_::oW1 + i * H + j];
      }
    }
    if (LY::W1_SMEM) {
      for (int i = lane; i < H * H; i += 32) w1s[i] = (float)th[N_::oW1 + i];
    }
    for (int i = lane; i < H * A; i += 32) wo[i] = (float)th[N_::oWo + i];
    if (lane < A) bo[lane] = (float)th[N_::obo + lane];
    float std_[A];
    double std_sum = 0.0;
#pragma unroll
    for (int k = 0; k < A; ++k) {
      std_[k] = expf(clamp_log_std((float)th[N_::ols + k], a.log_min_std));
      std_sum += (double)std_[k];
    }
    __syncwarp();

    for (int e = 0; e < a.E; ++e) {
      const long long lid = a.lane0 + (long long)m * a.E + e;
      float s[Env::S], o[O], o_last[O];
      draw_reset<Env>(s, nullptr, 0, 0, 0, a.seed, a.iter, lid);
      double G = 0.0, Usum = 0.0, disc = 1.0;
      int t = 0;
      for (;;) {
        Env::obs(s, o);
#pragma unroll
        for (int k = 0; k < O; ++k) o_last[k] = o[k];
        if (t == 0 && a.obs_first != nullptr && lane == 0) {
          float* dst = a.obs_first + ((size_t)m * a.E + e) * O;
#pragma unroll
          for (int k = 0; k < O; ++k) dst[k] = o[k];
        }
        // layer 1: unit j from the observation (dense_thread order: bias + even inputs, odd inputs, then the sum)
        float h[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          float s0 = b0[u], s1 = 0.f;
#pragma unroll
          for (int i = 0; i < O; ++i) {
            if ((i & 1) == 0) s0 = fmaf(o[i], w0[u][i], s0);
            else s1 = fmaf(o[i], w0[u][i], s1);
          }
          h[u] = tanh_f(s0 + s1);
        }
        __syncwarp();
#pragma unroll
        for (int u = 0; u < U; ++u) hrow[lane + 32 * u] = h[u];
        __syncwarp();
        // layer 2: unit j from the broadcast h1 row
        float s0[U], s1[U];
#pragma unroll
        for (int u = 0; u < U; ++u) { s0[u] = b1[u]; s1[u] = 0.f; }
#pragma unroll
        for (int q = 0; q < H / 4; ++q) {
          const float4 v = hrow4[q];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            float wa, wb, wc, wd;
            if (LY::W1_SMEM) {
              const int j = lane + 32 * u;
              wa = w1s[(4 * q) * H + j]; wb = w1s[(4 * q + 1) * H + j];
              wc = w1s[(4 * q + 2) * H + j]; wd = w1s[(4 * q + 3) * H + j];
            } else {
              const int uu = LY::W1_SMEM ? 0 : u;
              wa = w1[uu][LY::W1_SMEM ? 0 : 4 * q]; wb = w1[uu][LY::W1_SMEM ? 0 : 4 * q + 1];
              wc = w1[uu][LY::W1_SMEM ? 0 : 4 * q + 2]; wd = w1[uu][LY::W1_SMEM ? 0 : 4 * q + 3];
            }
            s0[u] = fmaf(v.x, wa, s0[u]);
            s1[u] = fmaf(v.y, wb, s1[u]);
            s0[u] = fmaf(v.z, wc, s0[u]);
            s1[u] = fmaf(v.w, wd, s1[u]);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) h[u] = tanh_f(s0[u] + s1[u]);
        __syncwarp();
#pragma unroll
        for (int u = 0; u < U; ++u) hrow[lane + 32 * u] = h[u];
        __syncwarp();
        // output layer, summed by every thread in the canonical order from the broadcast h2 row
        float mu[A];
#pragma unroll
        for (int k = 0; k < A; ++k) {
          float r0 = bo[k], r1 = 0.f;
#pragma unroll
          for (int q = 0; q < H / 4; ++q) {
            const float4 v = hrow4[q];
            r0 = fmaf(v.x, wo[(4 * q) * A + k], r0);
            r1 = fmaf(v.y, wo[(4 * q + 1) * A + k], r1);
            r0 = fmaf(v.z, wo[(4 * q + 2) * A + k], r0);
            r1 = fmaf(v.w, wo[(4 * q + 3) * A + k], r1);
          }
          mu[k] = r0 + r1;
        }
        float ep[A], u_[A];
        draw_eps<A>(ep, nullptr, t, 0, 0, a.seed, a.iter, lid);
#pragma unroll
        for (int k = 0; k < A; ++k) u_[k] = scale_action(fmaf(std_[k], ep[k], mu[k]), Env::lb(k), Env::ub(k));
        float r;
        bool done;
        Env::step(s, u_, r, done);
        G += disc * (double)r;
        disc *= a.discount;
        Usum += (double)r;
        ++t;
        if (done || t >= a.max_path_length) break;
      }
      if (lane == 0) {
        const size_t me = (size_t)m * a.E + e;
        a.ret[me] = G;
        a.undisc[me] = Usum;
        a.len[me] = t;
        if (a.obs_last != nullptr) {
#pragma unroll
          for (int k = 0; k < O; ++k) a.obs_last[me * O + k] = o_last[k];
        }
      }
    }
    if (lane == 0) {
      // the same thread wrote the member's episodes above: its own writes are visible to it
      a.member[(size_t)m * 3 + 0] = stderr_lb(a.ret + (size_t)m * a.E, a.E);
      a.member[(size_t)m * 3 + 1] = stderr_lb(a.undisc + (size_t)m * a.E, a.E);
      a.member[(size_t)m * 3 + 2] = std_sum / A;
    }
  }
}

template <class Env, int H>
static int launch_population(const PopArgs& a, cudaStream_t st) {
  using LY = PopLayout<Env, H>;
  const size_t smem = (size_t)LY::FLOATS * POP_WARPS * sizeof(float);
  if (smem > 48 * 1024) B200RL_SET_MAX_SMEM((population_rollout_kernel<Env, H>), smem);
  int per_sm = 0;
  B200RL_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, population_rollout_kernel<Env, H>,
                                                                  POP_THREADS, smem));
  const long long need = ((long long)a.M + POP_WARPS - 1) / POP_WARPS;
  const long long cap = (long long)num_sms() * (per_sm > 0 ? per_sm : 1);
  const int grid = (int)(need < cap ? need : cap);
  population_rollout_kernel<Env, H><<<grid, POP_THREADS, smem, st>>>(a);
  B200RL_LAUNCH_CHECK("population_rollout_kernel");
  return 0;
}

// theta[r][k] = cur_mean[k] + sample_std[k] * eps(seed, iter, member_r, k), sample_std[k] = sqrt(cur_std[k]^2 + extra_var);
// eps from Philox stream 2 (lane = member index, row 0, chunk = k / 4).  Every float64 operation is explicitly rounded, so
// NumPy float64 arithmetic on the same eps gives the same bits.  One thread per (row, chunk of four).
__global__ void population_sample_kernel(long long P, const double* __restrict__ cur_mean,
                                         const double* __restrict__ cur_std, double extra_var, uint32_t seed,
                                         uint32_t iter, const long long* __restrict__ members, long long member0, int n,
                                         double* __restrict__ out) {
  const long long chunks = (P + 3) / 4;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= chunks * n) return;
  const int r = (int)(i / chunks);
  const int c = (int)(i % chunks);
  const long long m = members != nullptr ? members[r] : member0 + r;
  float q[4];
  noise4(B200RL_NOISE_NORMAL, seed, iter, POP_STREAM, m, 0, c, q);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long k = 4LL * c + j;
    if (k < P) {
      const double cs = cur_std[k];
      const double sd = __dsqrt_rn(__dadd_rn(__dmul_rn(cs, cs), extra_var));
      out[(size_t)r * P + k] = __dadd_rn(__dmul_rn((double)q[j], sd), cur_mean[k]);
    }
  }
}

// Orderable key of a fitness value: ascending key = descending fitness, NaN last, -0 == +0.
__device__ __forceinline__ unsigned long long fitness_key(double f) {
  if (f != f) return ~0ull;
  const unsigned long long u = (unsigned long long)__double_as_longlong(f == 0.0 ? 0.0 : f);
  const unsigned long long asc = (u >> 63) ? ~u : (u | 0x8000000000000000ull);
  return ~asc;
}

constexpr int TOPK_THREADS = 1024;

// Inclusive block scan of one int per thread (TOPK_THREADS threads); returns this thread's inclusive prefix and the total.
__device__ __forceinline__ int block_scan_incl(int v, int* scratch, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += y;
  }
  if (lane == 31) scratch[warp] = v;
  __syncthreads();
  if (warp == 0) {
    int w = scratch[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    scratch[lane] = w;
  }
  __syncthreads();
  const int res = v + (warp > 0 ? scratch[warp - 1] : 0);
  total = scratch[31];
  __syncthreads();
  return res;
}

// Top-k selection, one CTA: an 8-pass radix select finds the k-th smallest key K*, then one ordered pass keeps every key
// below K* and the lowest-index keys equal to K*, in index order.  Writes sel_key / sel_idx [k].
__global__ void __launch_bounds__(TOPK_THREADS) topk_select_kernel(const double* __restrict__ f, int M, int k,
                                                                   unsigned long long* __restrict__ sel_key,
                                                                   long long* __restrict__ sel_idx) {
  __shared__ int hist[256];
  __shared__ int scratch[32];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_krem;
  unsigned long long prefix = 0, mask = 0;
  if (threadIdx.x == 0) s_krem = k;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int b = threadIdx.x; b < 256; b += blockDim.x) hist[b] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < M; i += blockDim.x) {
      const unsigned long long key = fitness_key(f[i]);
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 0xFF], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int krem = s_krem, b = 0;
      while (b < 255 && hist[b] < krem) krem -= hist[b++];
      s_krem = krem;
      s_prefix = prefix | ((unsigned long long)b << shift);
    }
    __syncthreads();
    prefix = s_prefix;
    mask |= 0xFFull << shift;
  }
  const unsigned long long kstar = prefix;
  const int take_eq = s_krem;            // keys equal to K* to keep (the lowest indices)
  int eq_seen = 0, taken = 0;
  for (int base = 0; base < M; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const unsigned long long key = i < M ? fitness_key(f[i]) : ~0ull;
    const bool lt = i < M && key < kstar, eq = i < M && key == kstar;
    int eq_total;
    const int eq_incl = block_scan_incl(eq ? 1 : 0, scratch, eq_total);
    const bool take = lt || (eq && eq_seen + eq_incl <= take_eq);
    int take_total;
    const int pos = block_scan_incl(take ? 1 : 0, scratch, take_total) - 1 + taken;
    if (take) {
      sel_key[pos] = key;
      sel_idx[pos] = i;
    }
    eq_seen += eq_total;
    taken += take_total;
  }
}

// Rank sort of the k selected (key, index) pairs: rank = number of pairs before this one in (key, index) order.
__global__ void topk_rank_kernel(const unsigned long long* __restrict__ sel_key, const long long* __restrict__ sel_idx,
                                 int k, long long* __restrict__ idx_out) {
  __shared__ unsigned long long tk[256];
  __shared__ long long ti[256];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long key = i < k ? sel_key[i] : 0ull;
  const long long idx = i < k ? sel_idx[i] : 0;
  int rank = 0;
  for (int base = 0; base < k; base += 256) {
    if (base + (int)threadIdx.x < k) {
      tk[threadIdx.x] = sel_key[base + threadIdx.x];
      ti[threadIdx.x] = sel_idx[base + threadIdx.x];
    }
    __syncthreads();
    const int n = min(256, k - base);
    for (int j = 0; j < n; ++j) rank += (tk[j] < key) || (tk[j] == key && ti[j] < idx);
    __syncthreads();
  }
  if (i < k) idx_out[rank] = idx;
}

// Column mean and population std (ddof 0) of k rows [k][P], summed over the rows in row order with explicitly rounded
// float64 operations: NumPy's axis-0 reduction (rows added one after another, then a true division) gives the same bits.
__global__ void rows_mean_std_kernel(long long P, int k, const double* __restrict__ rows, double* __restrict__ mean_out,
                                     double* __restrict__ std_out) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  double s = 0.0;
  for (int r = 0; r < k; ++r) s = __dadd_rn(s, rows[(size_t)r * P + p]);
  const double mu = __ddiv_rn(s, (double)k);
  double v = 0.0;
  for (int r = 0; r < k; ++r) {
    const double d = __dsub_rn(rows[(size_t)r * P + p], mu);
    v = __dadd_rn(v, __dmul_rn(d, d));
  }
  mean_out[p] = mu;
  std_out[p] = __dsqrt_rn(__ddiv_rn(v, (double)k));
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_population_sample(long long P, const double* cur_mean, const double* cur_std, double extra_var,
                             unsigned int seed, unsigned int iter, const long long* members, long long member0, int n,
                             double* theta_out, void* stream) {
  B200RL_REQUIRE(P > 0 && n >= 0 && cur_mean && cur_std && theta_out, "population_sample: bad arguments");
  B200RL_REQUIRE(extra_var >= 0.0, "population_sample: extra_var must be >= 0");
  if (n == 0) return 0;
  const long long total = ((P + 3) / 4) * n;
  population_sample_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      P, cur_mean, cur_std, extra_var, seed, iter, members, member0, n, theta_out);
  B200RL_LAUNCH_CHECK("population_sample_kernel");
  return 0;
}

int b200rl_population_rollout(int env_kind, int h1, int h2, float min_std, const double* theta, int M, int n_evals,
                              int max_path_length, double discount, unsigned int seed, unsigned int iter,
                              long long lane0, double* ret_out, double* undisc_out, int* len_out, float* obs_first,
                              float* obs_last, double* member_out, double* ws, void* stream) {
  B200RL_REQUIRE(theta && ret_out && undisc_out && len_out && member_out && ws, "population_rollout: null buffer");
  B200RL_REQUIRE(M >= 0 && n_evals > 0 && max_path_length > 0, "population_rollout: bad sizes");
  B200RL_REQUIRE((obs_first == nullptr) == (obs_last == nullptr), "population_rollout: obs_first and obs_last go together");
  if (h1 != h2) {
    set_error("population_rollout: hidden sizes (%d,%d) not compiled in (32,32) or (64,64)", h1, h2);
    return B200RL_EUNSUPPORTED;
  }
  if (M == 0) return 0;
  PopArgs a;
  a.theta = theta;
  a.log_min_std = min_std > 0.f ? logf(min_std) : -INFINITY;
  a.M = M; a.E = n_evals; a.max_path_length = max_path_length;
  a.discount = discount;
  a.seed = seed; a.iter = iter; a.lane0 = lane0;
  a.ret = ret_out; a.undisc = undisc_out; a.len = len_out;
  a.obs_first = obs_first; a.obs_last = obs_last;
  a.member = member_out;
  a.next = reinterpret_cast<unsigned long long*>(ws);
  cudaStream_t st = (cudaStream_t)stream;
  B200RL_CUDA_CHECK(cudaMemsetAsync(a.next, 0, sizeof(unsigned long long), st));
  B200RL_DISPATCH_ENV(env_kind, {
    int rc;
    if (h1 == 32) {
      rc = launch_population<Env, 32>(a, st);
    } else if (h1 == 64) {
      rc = launch_population<Env, 64>(a, st);
    } else {
      set_error("hidden size %d not compiled in (32 or 64)", h1);
      rc = B200RL_EUNSUPPORTED;
    }
    if (rc) return rc;
  });
  return 0;
}

int b200rl_population_topk(const double* f, int M, int k, long long* idx_out, double* ws, void* stream) {
  B200RL_REQUIRE(f && idx_out && ws, "population_topk: null buffer");
  B200RL_REQUIRE(M > 0 && k > 0 && k <= M, "population_topk: need 0 < k <= M");
  // (key, index) scratch of 2k words; the workspace holds b200rl_ws_doubles() >= 9.6 M entries
  B200RL_REQUIRE(2LL * k <= (long long)MAX_PARTIAL_BLOCKS * MAX_PARTIAL_K, "population_topk: k too large");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* sel_key = reinterpret_cast<unsigned long long*>(ws);
  long long* sel_idx = reinterpret_cast<long long*>(ws + k);
  topk_select_kernel<<<1, TOPK_THREADS, 0, st>>>(f, M, k, sel_key, sel_idx);
  B200RL_LAUNCH_CHECK("topk_select_kernel");
  topk_rank_kernel<<<(k + 255) / 256, 256, 0, st>>>(sel_key, sel_idx, k, idx_out);
  B200RL_LAUNCH_CHECK("topk_rank_kernel");
  return 0;
}

int b200rl_rows_mean_std(long long P, int k, const double* rows, double* mean_out, double* std_out, void* stream) {
  B200RL_REQUIRE(P > 0 && k > 0 && rows && mean_out && std_out, "rows_mean_std: bad arguments");
  rows_mean_std_kernel<<<(unsigned)((P + 127) / 128), 128, 0, (cudaStream_t)stream>>>(P, k, rows, mean_out, std_out);
  B200RL_LAUNCH_CHECK("rows_mean_std_kernel");
  return 0;
}
}
