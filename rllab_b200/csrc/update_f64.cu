// float64 "parity mode" of the policy-update passes (loss/KL, surrogate gradient, Fisher-vector product).
//
// The reference's default floatX is float64 (SURVEY.md section 5); with the default cg_iters = 10 the CG recursion on
// the ill-conditioned Fisher system amplifies float32 rounding of the Hessian-vector product to O(1) differences in
// the search direction (DESIGN.md "Parity limit"), so a float32 pipeline cannot match a float64 run to 1e-5.  These
// kernels evaluate the same three passes in float64 arithmetic on the float64 master parameters, which lets the whole
// TRPO step be compared with the oracle at the reference's default settings.  They are deliberately simple -- one
// thread per sample, weights in shared memory, weight gradients accumulated with shared-memory float64 atomics -- and
// ~10x slower than the float32 kernels; the half-rate FP64 pipe of the data-centre GPUs makes that a usable
// verification mode.
//
// Same formulas and reference citations as update.cu / update_tile.cu.
#include "update_common.cuh"

namespace b200rl {

constexpr int D_THREADS = 128;

struct UpdArgs64 {
  const double* params;
  const double* xvec;
  double log_min_std;
  long long B;
  const float *obs, *act, *adv, *old_mean, *old_log_std;
  int loss_kind;
  const unsigned char* flags;
  double* partial;
};

template <int NIN, int NOUT>
__device__ __forceinline__ void dense_d(const double* W, const double* b, const double (&in)[NIN], double (&out)[NOUT]) {
#pragma unroll
  for (int j = 0; j < NOUT; ++j) out[j] = b ? b[j] : 0.0;
#pragma unroll 2
  for (int i = 0; i < NIN; ++i) {
    const double a = in[i];
#pragma unroll
    for (int j = 0; j < NOUT; ++j) out[j] = fma(a, W[i * NOUT + j], out[j]);
  }
}

template <class N, int MODE>
__global__ void __launch_bounds__(D_THREADS) update_f64_kernel(UpdArgs64 a) {
  constexpr int O = N::O, H1 = N::H1, H2 = N::H2, A = N::A, P = N::P;
  extern __shared__ __align__(16) double sd[];
  double* sp = sd;                                  // parameters
  double* acc = sd + P;                             // block accumulators (GRAD / FVP)
  double* sv = sd + 2 * P;                          // tangent (FVP)
  __shared__ double red_scratch[3 * 32];
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    sp[i] = a.params[i];
    if (MODE != MODE_LOSS) acc[i] = 0.0;
    if (MODE == MODE_FVP) sv[i] = a.xvec[i];
  }
  __syncthreads();
  double ls_new[A], sd_new[A], ls_old[A], sd_old[A];
  double sum_ls_new = 0.0, sum_ls_old = 0.0;
#pragma unroll
  for (int k = 0; k < A; ++k) {
    ls_new[k] = fmax(sp[N::ols + k], a.log_min_std);
    sd_new[k] = exp(ls_new[k]);
    ls_old[k] = (MODE == MODE_FVP) ? ls_new[k] : (double)a.old_log_std[k];
    sd_old[k] = exp(ls_old[k]);
    sum_ls_new += ls_new[k];
    sum_ls_old += ls_old[k];
  }
  const double half_log2pi_A = 0.5 * (double)A * 1.8378770664093454836;
  double s_loss = 0.0, s_kl = 0.0, m_kl = -1.0e300;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < a.B; s += stride) {
    if (a.flags != nullptr && (a.flags[s] & B200RL_FLAG_MASKED)) continue;      // sample of a dropped (cut) path
    double x[O], h1[H1], h2[H2], mu[A], dmu[A], dls[A];
#pragma unroll
    for (int o = 0; o < O; ++o) x[o] = (double)a.obs[(size_t)o * a.B + s];
    dense_d<O, H1>(sp + N::oW0, sp + N::ob0, x, h1);
#pragma unroll
    for (int j = 0; j < H1; ++j) h1[j] = tanh(h1[j]);
    dense_d<H1, H2>(sp + N::oW1, sp + N::ob1, h1, h2);
#pragma unroll
    for (int j = 0; j < H2; ++j) h2[j] = tanh(h2[j]);
    if (MODE != MODE_FVP) {
#pragma unroll
      for (int k = 0; k < A; ++k) {
        double m = sp[N::obo + k];
#pragma unroll 4
        for (int j = 0; j < H2; ++j) m = fma(h2[j], sp[N::oWo + j * A + k], m);
        mu[k] = m;
      }
      double zsq = 0.0, zsq_old = 0.0, kl = 0.0, z[A], dkl_mu[A], dkl_ls[A];
#pragma unroll
      for (int k = 0; k < A; ++k) {
        const double act = (double)a.act[(size_t)k * a.B + s], om = (double)a.old_mean[(size_t)k * a.B + s];
        z[k] = (act - mu[k]) / sd_new[k];
        zsq += z[k] * z[k];
        const double zo = (act - om) / sd_old[k];
        zsq_old += zo * zo;
        const double dm = om - mu[k];
        const double sn = sd_new[k] * sd_new[k], so = sd_old[k] * sd_old[k], den = 2.0 * sn + 1e-8;
        kl += (dm * dm + so - sn) / den + ls_new[k] - ls_old[k];
        // d kl / d mu_new and d kl / d log_std_new (diagonal_gaussian.py:14-34), used by the B200RL_LOSS_KL gradient
        dkl_mu[k] = -2.0 * dm / den;
        dkl_ls[k] = 1.0 - (2.0 * sn * den + 4.0 * sn * (dm * dm + so - sn)) / (den * den);
      }
      const double adv_s = (double)a.adv[s];
      const double logp_new = -sum_ls_new - 0.5 * zsq - half_log2pi_A;
      double w_s, term;
      if (a.loss_kind == B200RL_LOSS_TRPO) {
        const double logp_old = -sum_ls_old - 0.5 * zsq_old - half_log2pi_A;
        w_s = exp(logp_new - logp_old) * adv_s;
        term = -w_s;
      } else {
        w_s = adv_s;
        term = -logp_new * adv_s;
      }
      s_loss += term;
      s_kl += kl;
      m_kl = fmax(m_kl, kl);
      if (MODE == MODE_LOSS) continue;
#pragma unroll
      for (int k = 0; k < A; ++k) {
        if (a.loss_kind == B200RL_LOSS_KL) {          // gradient of mean KL(old || new) (FiniteDifferenceHvp)
          dmu[k] = dkl_mu[k];
          dls[k] = dkl_ls[k];
        } else {
          dmu[k] = -w_s * z[k] / sd_new[k];
          dls[k] = -w_s * (z[k] * z[k] - 1.0);
        }
      }
    } else {
      // tangent forward
      double t1[H1], t2[H2];
      dense_d<O, H1>(sv + N::oW0, sv + N::ob0, x, t1);
#pragma unroll
      for (int j = 0; j < H1; ++j) t1[j] *= (1.0 - h1[j] * h1[j]);
      dense_d<H1, H2>(sp + N::oW1, sv + N::ob1, t1, t2);
#pragma unroll 2
      for (int i = 0; i < H1; ++i) {
        const double hv = h1[i];
#pragma unroll
        for (int j = 0; j < H2; ++j) t2[j] = fma(hv, sv[N::oW1 + i * H2 + j], t2[j]);
      }
#pragma unroll
      for (int j = 0; j < H2; ++j) t2[j] *= (1.0 - h2[j] * h2[j]);
#pragma unroll
      for (int k = 0; k < A; ++k) {
        double m = sv[N::obo + k];
#pragma unroll 4
        for (int j = 0; j < H2; ++j) m = fma(t2[j], sp[N::oWo + j * A + k], fma(h2[j], sv[N::oWo + j * A + k], m));
        const double s2 = sd_new[k] * sd_new[k];
        dmu[k] = m * (2.0 / (2.0 * s2 + 1e-8));
        dls[k] = 0.0;
      }
    }
    // backward + accumulation (shared-memory float64 atomics)
    double d2[H2];
#pragma unroll
    for (int j = 0; j < H2; ++j) {
      double sacc = 0.0;
#pragma unroll
      for (int k = 0; k < A; ++k) {
        sacc = fma(dmu[k], sp[N::oWo + j * A + k], sacc);
        atomicAdd(&acc[N::oWo + j * A + k], h2[j] * dmu[k]);
      }
      d2[j] = sacc * (1.0 - h2[j] * h2[j]);
      atomicAdd(&acc[N::ob1 + j], d2[j]);
    }
#pragma unroll
    for (int k = 0; k < A; ++k) {
      atomicAdd(&acc[N::obo + k], dmu[k]);
      atomicAdd(&acc[N::ols + k], dls[k]);
    }
#pragma unroll 1
    for (int i = 0; i < H1; ++i) {
      double sacc = 0.0;
#pragma unroll
      for (int j = 0; j < H2; ++j) {
        sacc = fma(d2[j], sp[N::oW1 + i * H2 + j], sacc);
        atomicAdd(&acc[N::oW1 + i * H2 + j], h1[i] * d2[j]);
      }
      const double d1 = sacc * (1.0 - h1[i] * h1[i]);
      atomicAdd(&acc[N::ob0 + i], d1);
#pragma unroll
      for (int o = 0; o < O; ++o) atomicAdd(&acc[N::oW0 + o * H1 + i], x[o] * d1);
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

template <class N, int MODE>
static int launch_f64(const UpdArgs64& a, int* grid_out, cudaStream_t st) {
  const size_t smem = (size_t)3 * N::P * sizeof(double);
  B200RL_SET_MAX_SMEM((update_f64_kernel<N, MODE>), smem);
  long long grid = (long long)num_sms() * 2;
  const long long need = (a.B + D_THREADS - 1) / D_THREADS;
  if (grid > need) grid = need;
  update_f64_kernel<N, MODE><<<(unsigned)grid, D_THREADS, smem, st>>>(a);
  B200RL_LAUNCH_CHECK("update_f64_kernel");
  *grid_out = (int)grid;
  return 0;
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_update_f64(int mode, int loss_kind, const double* params_f64, int obs_dim, int h1, int h2, int act_dim,
                      double min_std, long long B, const float* obs, const float* act, const float* adv,
                      const float* old_mean, const float* old_log_std, const unsigned char* flags, const double* x,
                      double scale, const double* count, double reg_coeff, double diag_scale, double* vec_out,
                      double* loss_out, double* ws, void* stream) {
  B200RL_REQUIRE(params_f64 && obs && ws && B > 0, "update_f64: bad arguments");
  B200RL_REQUIRE(mode == MODE_LOSS || mode == MODE_GRAD || mode == MODE_FVP, "update_f64: bad mode");
  B200RL_REQUIRE(mode == MODE_FVP ? (x && vec_out) : (act && adv && old_mean && old_log_std), "update_f64: null buffer");
  B200RL_REQUIRE(mode != MODE_GRAD || vec_out, "update_f64: gradient output missing");
  B200RL_REQUIRE(mode != MODE_LOSS || loss_out, "update_f64: loss output missing");
  B200RL_REQUIRE(loss_kind == B200RL_LOSS_TRPO || loss_kind == B200RL_LOSS_VPG ||
                 (loss_kind == B200RL_LOSS_KL && mode == MODE_GRAD), "update_f64: bad loss kind");
  cudaStream_t st = (cudaStream_t)stream;
  UpdArgs64 a{};
  a.params = params_f64; a.xvec = x; a.log_min_std = min_std > 0.0 ? log(min_std) : -INFINITY; a.B = B;
  a.obs = obs; a.act = act; a.adv = adv; a.old_mean = old_mean; a.old_log_std = old_log_std;
  a.loss_kind = loss_kind; a.flags = flags; a.partial = ws;
  int grid = 0, P = 0, ols = 0;
  B200RL_DISPATCH_NET({
    P = NetT::P; ols = NetT::ols;
    int rc = (mode == MODE_LOSS) ? launch_f64<NetT, MODE_LOSS>(a, &grid, st)
           : (mode == MODE_GRAD) ? launch_f64<NetT, MODE_GRAD>(a, &grid, st)
                                 : launch_f64<NetT, MODE_FVP>(a, &grid, st);
    if (rc) return rc;
  });
  FinArgs f{};
  f.nblocks = grid; f.scale = scale; f.count = count; f.ols = ols; f.A = act_dim;
  f.params64 = params_f64; f.log_min_std = a.log_min_std;
  if (mode != MODE_LOSS) { f.partial = ws; f.K = P; f.vec_out = vec_out; }
  f.post = (mode == MODE_GRAD) ? FIN_GRAD : (mode == MODE_FVP ? FIN_FVP : FIN_NONE);
  if (mode == MODE_FVP) { f.x = x; f.reg = reg_coeff; f.diag_scale = diag_scale; }
  if (mode != MODE_FVP && loss_out != nullptr) {
    f.tri_partial = (mode == MODE_LOSS) ? ws : ws + (size_t)grid * P;
    f.NT = 3; f.tri_out = loss_out;
  }
  if (peer_fused()) f.peer = peer_next();
  return launch_finalize_update(f, st);
}
}
