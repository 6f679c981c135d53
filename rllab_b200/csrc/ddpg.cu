// DDPG (rllab/algos/ddpg.py) on the GPU: one CTA per independent training run.  The run's networks, Adam moments, targets
// and minibatch live in shared memory for a whole launch; only the replay pool is in global memory.  A step is the
// train() loop body (ddpg.py:216-251): policy forward on the current observation, the exploration draw, Env::step, the
// pool write and, once the pool holds min_pool_size samples, n_updates_per_sample calls of do_training (ddpg.py:331-365):
// the minibatch draw, the target forwards, critic forward / backward / Adam, actor forward / backward through Q's action
// input / Adam, and the soft target update.  Every sum runs in a fixed order on one thread or one output entry per
// thread, with no atomics, so a rerun is bit-identical and a run's result does not depend on the other runs in the grid.
//
// Also: DeterministicMLPPolicy.get_actions, ContinuousMLPQFunction.get_qval and the noise-free lane rollout that
// DDPG.evaluate samples (rllab/policies/deterministic_mlp_policy.py, rllab/q_functions/continuous_mlp_q_function.py).
#include <type_traits>

#include "envs.cuh"

namespace b200rl {

constexpr int DDPG_THREADS = 256;
constexpr int DB = B200RL_DDPG_BATCH;   // minibatch size
constexpr int DH = 32;                  // hidden width of both nets
constexpr double ADAM_B1 = 0.9, ADAM_B2 = 0.999, ADAM_EPS = 1e-8;   // lasagne.updates.adam defaults

// Flat parameter layout (b200rl.h): policy [W0 (O,H), b0, W1 (H,H), b1, W2 (H,A), b2], then qf [W0 (O,H), b0,
// W1 (H+A,H), b1, W2 (H,1), b2] at offset PP.
template <int O_, int A_>
struct DdpgNet {
  static constexpr int O = O_, A = A_, H = DH, HA = DH + A_;
  static constexpr int PW0 = 0, PB0 = O * H, PW1 = PB0 + H, PB1 = PW1 + H * H, PW2 = PB1 + H, PB2 = PW2 + H * A,
                       PP = PB2 + A;
  static constexpr int QW0 = 0, QB0 = O * H, QW1 = QB0 + H, QB1 = QW1 + HA * H, QW2 = QB1 + H, QB2 = QW2 + H,
                       QP = QB2 + 1;
  static constexpr int P = PP + QP;
  // weight entries (not biases): the ones the weight decay terms cover (get_params(regularizable=True))
  __host__ __device__ static bool is_weight(int i) {
    if (i < PP) return i < PB0 || (i >= PW1 && i < PB1) || (i >= PW2 && i < PB2);
    i -= PP;
    return i < QB0 || (i >= QW1 && i < QB1) || (i >= QW2 && i < QB2);
  }
};

__device__ __forceinline__ float fmaR(float a, float b, float c) { return fmaf(a, b, c); }
__device__ __forceinline__ double fmaR(double a, double b, double c) { return fma(a, b, c); }
__device__ __forceinline__ float tanhR(float x) { return tanhf(x); }
__device__ __forceinline__ double tanhR(double x) { return tanh(x); }

// Shared-memory layout of one run (byte offsets): float64 masters theta, m, v, target and the gradient, each [P]; the
// compute copies of theta and target (float32 shadows when Real = float, the masters themselves when Real = double);
// the minibatch and the activations / deltas of the passes in Real.
template <class D, class Real>
struct DdpgSmem {
  static constexpr bool SHADOW = std::is_same<Real, float>::value;
  static constexpr size_t al(size_t x) { return (x + 15) & ~size_t(15); }
  static constexpr size_t th = 0, m = th + al(8 * D::P), v = m + al(8 * D::P), tg = v + al(8 * D::P),
                          g = tg + al(8 * D::P), red = g + al(8 * D::P), cth = red + al(8 * 16),
                          ctg = cth + (SHADOW ? al(4 * D::P) : 0), s = ctg + (SHADOW ? al(4 * D::P) : 0),
                          a = s + al(sizeof(Real) * DB * D::O), r = a + al(sizeof(Real) * DB * D::A),
                          tm = r + al(sizeof(Real) * DB), s2 = tm + al(sizeof(Real) * DB),
                          A1 = s2 + al(sizeof(Real) * DB * D::O), A2 = A1 + al(sizeof(Real) * DB * DH),
                          X1 = A2 + al(sizeof(Real) * DB * DH), X2 = X1 + al(sizeof(Real) * DB * D::HA),
                          D1 = X2 + al(sizeof(Real) * DB * DH), D2 = D1 + al(sizeof(Real) * DB * D::HA),
                          mu = D2 + al(sizeof(Real) * DB * DH), q = mu + al(sizeof(Real) * DB * D::A),
                          y = q + al(sizeof(Real) * DB), dq = y + al(sizeof(Real) * DB),
                          idx = dq + al(sizeof(Real) * DB), bytes = idx + al(4 * DB);
};

template <class D, class Real>
struct DdpgBufs {
  double *th, *m, *v, *tg, *g, *red;
  Real *cth, *ctg, *s, *a, *r, *tm, *s2, *A1, *A2, *X1, *X2, *D1, *D2, *mu, *q, *y, *dq;
  int* idx;
  __device__ explicit DdpgBufs(unsigned char* base) {
    using L = DdpgSmem<D, Real>;
    th = (double*)(base + L::th); m = (double*)(base + L::m); v = (double*)(base + L::v); tg = (double*)(base + L::tg);
    g = (double*)(base + L::g); red = (double*)(base + L::red);
    cth = L::SHADOW ? (Real*)(base + L::cth) : (Real*)th;
    ctg = L::SHADOW ? (Real*)(base + L::ctg) : (Real*)tg;
    s = (Real*)(base + L::s); a = (Real*)(base + L::a); r = (Real*)(base + L::r); tm = (Real*)(base + L::tm);
    s2 = (Real*)(base + L::s2); A1 = (Real*)(base + L::A1); A2 = (Real*)(base + L::A2); X1 = (Real*)(base + L::X1);
    X2 = (Real*)(base + L::X2); D1 = (Real*)(base + L::D1); D2 = (Real*)(base + L::D2); mu = (Real*)(base + L::mu);
    q = (Real*)(base + L::q); y = (Real*)(base + L::y); dq = (Real*)(base + L::dq); idx = (int*)(base + L::idx);
  }
};

constexpr int ACT_NONE = 0, ACT_RELU = 1, ACT_TANH = 2;

// Block-wide dense layer: Y[b][j] = act(bias[j] + sum_k X[b][k] W[k][j]), k ascending.  W is [K][M] row-major.
template <class Real>
__device__ void dense(const Real* W, const Real* bias, const Real* X, int ldx, int K, int M, int B, Real* Y, int ldy,
                      int act) {
  for (int e = threadIdx.x; e < B * M; e += blockDim.x) {
    const int b = e / M, j = e - b * M;
    Real acc = bias[j];
    for (int k = 0; k < K; ++k) acc = fmaR(X[b * ldx + k], W[k * M + j], acc);
    Y[b * ldy + j] = act == ACT_RELU ? (acc > Real(0) ? acc : Real(0)) : act == ACT_TANH ? tanhR(acc) : acc;
  }
}

// Block-wide weight gradient of a dense layer: gW[k][j] = sum_b X[b][k] Dl[b][j], gb[j] = sum_b Dl[b][j], b ascending.
template <class Real>
__device__ void grad_w(const Real* X, int ldx, int K, const Real* Dl, int ldd, int M, double* gW, double* gb) {
  for (int e = threadIdx.x; e < (K + 1) * M; e += blockDim.x) {
    Real acc = Real(0);
    if (e < K * M) {
      const int k = e / M, j = e - k * M;
      for (int b = 0; b < DB; ++b) acc = fmaR(X[b * ldx + k], Dl[b * ldd + j], acc);
      gW[e] = (double)acc;
    } else {
      const int j = e - K * M;
      for (int b = 0; b < DB; ++b) acc += Dl[b * ldd + j];
      gb[j] = (double)acc;
    }
  }
}

// Block-wide input delta: out[b][k] = sum_j Dl[b][j] W[k][j] (j ascending), times the ReLU derivative (Xa[b][k] > 0,
// Xa the layer's input activations) for k < kmask.
template <class Real>
__device__ void back_x(const Real* Dl, int ldd, int M, const Real* W, int K, const Real* Xa, int lda, int kmask,
                       Real* out, int ldo) {
  for (int e = threadIdx.x; e < DB * K; e += blockDim.x) {
    const int b = e / K, k = e - b * K;
    Real acc = Real(0);
    for (int j = 0; j < M; ++j) acc = fmaR(Dl[b * ldd + j], W[k * M + j], acc);
    if (k < kmask && !(Xa[b * lda + k] > Real(0))) acc = Real(0);
    out[b * ldo + k] = acc;
  }
}

// Adam (lasagne.updates.adam) on entries [lo, hi) with the weight decay gradient wd * theta added on weights; the
// gradient buffer keeps the gradient Adam consumed.
template <class D, class Real>
__device__ void adam_range(const DdpgBufs<D, Real>& S, int lo, int hi, double lr, double wd, long long t) {
  const double a_t = lr * sqrt(1.0 - pow(ADAM_B2, (double)t)) / (1.0 - pow(ADAM_B1, (double)t));
  for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const double gi = S.g[i] + (D::is_weight(i) ? wd * S.th[i] : 0.0);
    S.g[i] = gi;
    const double mi = ADAM_B1 * S.m[i] + (1.0 - ADAM_B1) * gi;
    const double vi = ADAM_B2 * S.v[i] + (1.0 - ADAM_B2) * gi * gi;
    S.m[i] = mi;
    S.v[i] = vi;
    const double t_ = S.th[i] - a_t * mi / (sqrt(vi) + ADAM_EPS);
    S.th[i] = t_;
    if (DdpgSmem<D, Real>::SHADOW) S.cth[i] = (Real)t_;
  }
}

// Q forward on the minibatch: X1 = [relu(s W0 + b0) | act] (act already in X1[:, H:]), X2 = relu(X1 W1 + b1),
// q = X2 W2 + b2.  q_params: the Q block of the compute parameters.
template <class D, class Real>
__device__ void q_forward(const DdpgBufs<D, Real>& S, const Real* qp, const Real* obs) {
  dense(qp + D::QW0, qp + D::QB0, obs, D::O, D::O, DH, DB, S.X1, D::HA, ACT_RELU);
  __syncthreads();
  dense(qp + D::QW1, qp + D::QB1, S.X1, D::HA, D::HA, DH, DB, S.X2, DH, ACT_RELU);
  __syncthreads();
  dense(qp + D::QW2, qp + D::QB2, S.X2, DH, DH, 1, DB, S.q, 1, ACT_NONE);
  __syncthreads();
}

// Policy forward on the minibatch: A1, A2 hidden, tanh output into X1[:, H:] (Q's action input).
template <class D, class Real>
__device__ void pi_forward(const DdpgBufs<D, Real>& S, const Real* pp, const Real* obs) {
  dense(pp + D::PW0, pp + D::PB0, obs, D::O, D::O, DH, DB, S.A1, DH, ACT_RELU);
  __syncthreads();
  dense(pp + D::PW1, pp + D::PB1, S.A1, DH, DH, DH, DB, S.A2, DH, ACT_RELU);
  __syncthreads();
  dense(pp + D::PW2, pp + D::PB2, S.A2, DH, DH, D::A, DB, S.X1 + DH, D::HA, ACT_TANH);
  __syncthreads();
}

// Back-propagation through Q from dq: writes the Q gradient (without weight decay) at g + PP when want_qgrad, and leaves
// D1 = d(loss)/d(X1) (its action columns: the gradient with respect to Q's action input).
template <class D, class Real>
__device__ void q_backward(const DdpgBufs<D, Real>& S, const Real* qp, const Real* obs, bool want_qgrad) {
  back_x(S.dq, 1, 1, qp + D::QW2, DH, S.X2, DH, DH, S.D2, DH);
  if (want_qgrad) grad_w(S.X2, DH, DH, S.dq, 1, 1, S.g + D::PP + D::QW2, S.g + D::PP + D::QB2);
  __syncthreads();
  back_x(S.D2, DH, DH, qp + D::QW1, D::HA, S.X1, D::HA, DH, S.D1, D::HA);
  if (want_qgrad) grad_w(S.X1, D::HA, D::HA, S.D2, DH, DH, S.g + D::PP + D::QW1, S.g + D::PP + D::QB1);
  __syncthreads();
  if (want_qgrad) {
    grad_w(obs, D::O, D::O, S.D1, D::HA, DH, S.g + D::PP + D::QW0, S.g + D::PP + D::QB0);
    __syncthreads();
  }
}

// One DDPG.do_training on the minibatch staged in S.s, S.a, S.r, S.tm, S.s2 (ddpg.py:331-365 and init_opt):
//   y = r + (1 - terminal) discount Q'(s', mu'(s'))       the targets before this step's soft update
//   critic: mean((y - Q(s, a))^2) + 0.5 qf_wd |W_q|^2, one Adam step; qf_loss and q are the pre-update values
//   actor: -mean(Q(s, mu(s))) with the UPDATED critic + 0.5 pi_wd |W_pi|^2, one Adam step; policy_surr pre-step
//   target <- (1 - tau) target + tau theta over both nets
// Leaves q, y in S.q, S.y and writes (qf_loss, policy_surr) to S.red[0..1].  t: the Adam step count (>= 1).
template <class D, class Real>
__device__ void ddpg_update(const DdpgBufs<D, Real>& S, const b200rl_ddpg_hparams& hp, long long t) {
  const int tid = threadIdx.x;
  const Real* qc = S.cth + D::PP;
  // targets
  pi_forward(S, S.ctg, S.s2);
  q_forward(S, S.ctg + D::PP, S.s2);
  if (tid < DB) S.y[tid] = S.r[tid] + (Real(1) - S.tm[tid]) * (Real)hp.discount * S.q[tid];
  // critic forward at (s, a)
  for (int e = tid; e < DB * D::A; e += blockDim.x) S.X1[(e / D::A) * D::HA + DH + e % D::A] = S.a[e];
  __syncthreads();
  q_forward(S, qc, S.s);
  if (tid < DB) S.dq[tid] = Real(-2) * (S.y[tid] - S.q[tid]) / Real(DB);
  if (tid == 0) {
    double l = 0.0;
    for (int b = 0; b < DB; ++b) l += ((double)S.y[b] - (double)S.q[b]) * ((double)S.y[b] - (double)S.q[b]);
    S.red[0] = l / DB;
  }
  __syncthreads();
  q_backward(S, qc, S.s, true);
  adam_range(S, D::PP, D::P, hp.qf_learning_rate, hp.qf_weight_decay, t);
  __syncthreads();
  // the statistics behind AverageQ ... AverageAbsQYDiff, from the critic's pre-update q
  if (tid == 0) {
    double sq = 0.0, saq = 0.0, sy = 0.0, say = 0.0, sd = 0.0;
    for (int b = 0; b < DB; ++b) {
      const double qb = S.q[b], yb = S.y[b];
      sq += qb; saq += fabs(qb); sy += yb; say += fabs(yb); sd += fabs(qb - yb);
    }
    S.red[2] = sq; S.red[3] = saq; S.red[4] = sy; S.red[5] = say; S.red[6] = sd;
  }
  // actor: Q(s, mu(s)) with the updated critic, its values in dq (S.q keeps the critic's values for the caller)
  pi_forward(S, S.cth, S.s);
  dense(qc + D::QW0, qc + D::QB0, S.s, D::O, D::O, DH, DB, S.X1, D::HA, ACT_RELU);
  __syncthreads();
  dense(qc + D::QW1, qc + D::QB1, S.X1, D::HA, D::HA, DH, DB, S.X2, DH, ACT_RELU);
  __syncthreads();
  dense(qc + D::QW2, qc + D::QB2, S.X2, DH, DH, 1, DB, S.dq, 1, ACT_NONE);
  __syncthreads();
  if (tid == 0) {
    double sq = 0.0;
    for (int b = 0; b < DB; ++b) sq += (double)S.dq[b];
    S.red[1] = -sq / DB;
  }
  __syncthreads();
  if (tid < DB) S.dq[tid] = Real(-1) / Real(DB);
  __syncthreads();
  q_backward(S, qc, S.s, false);
  // through the tanh output: dz = dL/da (1 - mu^2)
  for (int e = tid; e < DB * D::A; e += blockDim.x) {
    const int b = e / D::A, k = e - b * D::A;
    const Real mu = S.X1[b * D::HA + DH + k];
    S.mu[e] = S.D1[b * D::HA + DH + k] * (Real(1) - mu * mu);
  }
  __syncthreads();
  const Real* pc = S.cth;
  grad_w(S.A2, DH, DH, S.mu, D::A, D::A, S.g + D::PW2, S.g + D::PB2);
  back_x(S.mu, D::A, D::A, pc + D::PW2, DH, S.A2, DH, DH, S.D2, DH);
  __syncthreads();
  grad_w(S.A1, DH, DH, S.D2, DH, DH, S.g + D::PW1, S.g + D::PB1);
  back_x(S.D2, DH, DH, pc + D::PW1, DH, S.A1, DH, DH, S.D1, D::HA);
  __syncthreads();
  grad_w(S.s, D::O, D::O, S.D1, D::HA, DH, S.g + D::PW0, S.g + D::PB0);
  __syncthreads();
  adam_range(S, 0, D::PP, hp.policy_learning_rate, hp.policy_weight_decay, t);
  __syncthreads();
  const double tau = hp.soft_target_tau;
  for (int i = tid; i < D::P; i += blockDim.x) {
    const double v = S.tg[i] * (1.0 - tau) + S.th[i] * tau;
    S.tg[i] = v;
    if (DdpgSmem<D, Real>::SHADOW) S.ctg[i] = (Real)v;
  }
  __syncthreads();
}

// Stage the minibatch rows idx of a pool ([rows][O], [rows][A], [rows], [rows]) into S; s' is row (idx + 1) % rows.
template <class D, class Real>
__device__ void gather(const DdpgBufs<D, Real>& S, const float* obs, const float* act, const float* rew,
                       const unsigned char* term, int rows) {
  for (int e = threadIdx.x; e < DB * D::O; e += blockDim.x) {
    const int b = e / D::O, k = e - b * D::O, i = S.idx[b];
    S.s[e] = (Real)obs[(size_t)i * D::O + k];
    S.s2[e] = (Real)obs[(size_t)((i + 1) % rows) * D::O + k];
  }
  for (int e = threadIdx.x; e < DB * D::A; e += blockDim.x) S.a[e] = (Real)act[(size_t)S.idx[e / D::A] * D::A + e % D::A];
  if (threadIdx.x < DB) {
    S.r[threadIdx.x] = (Real)rew[S.idx[threadIdx.x]];
    S.tm[threadIdx.x] = term[S.idx[threadIdx.x]] ? Real(1) : Real(0);
  }
}

// Load nets [4][P] (theta, m, v, target) into shared memory and fill the float32 shadows.
template <class D, class Real>
__device__ void load_nets(const DdpgBufs<D, Real>& S, const double* nets) {
  for (int i = threadIdx.x; i < D::P; i += blockDim.x) {
    S.th[i] = nets[i]; S.m[i] = nets[D::P + i]; S.v[i] = nets[2 * D::P + i]; S.tg[i] = nets[3 * D::P + i];
    if (DdpgSmem<D, Real>::SHADOW) { S.cth[i] = (Real)nets[i]; S.ctg[i] = (Real)nets[3 * D::P + i]; }
  }
  __syncthreads();
}

template <class D, class Real>
__device__ void store_nets(const DdpgBufs<D, Real>& S, double* nets) {
  for (int i = threadIdx.x; i < D::P; i += blockDim.x) {
    nets[i] = S.th[i]; nets[D::P + i] = S.m[i]; nets[2 * D::P + i] = S.v[i]; nets[3 * D::P + i] = S.tg[i];
  }
}

// Philox words of run `run` at step itr (layout in b200rl.h).
__device__ __forceinline__ void ddpg_words(uint32_t seed, long long itr, int run, int stream_id, uint32_t sub,
                                           uint32_t w[4]) {
  Philox::gen((uint32_t)run, (uint32_t)(itr & 0x0FFFFFFF) | ((uint32_t)stream_id << 28), sub, 0u, seed,
              (uint32_t)((unsigned long long)itr >> 28), w);
}

// SimpleReplayPool.random_batch's index draws (ddpg.py:54-70) by warp 0: candidate j is accepted unless its index is
// size - 1; the ballot keeps the accepted ones in candidate order.
__device__ void draw_indices(int* idx, uint32_t seed, long long itr, int run, int update, int bottom, int size,
                             int rows) {
  if (threadIdx.x >= 32) return;
  const int lane = threadIdx.x;
  int count = 0;
  for (int round = 0; count < DB; ++round) {
    const int c = round * 32 + lane;
    uint32_t w[4];
    ddpg_words(seed, itr, run, B200RL_DDPG_STREAM_INDEX, ((uint32_t)update << 16) | (uint32_t)(c >> 2), w);
    const uint32_t x = w[c & 3];
    const int index = (int)(((long long)bottom + (long long)__umulhi(x, (uint32_t)size)) % rows);
    const bool ok = index != size - 1;
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    const int pos = count + __popc(bal & ((1u << lane) - 1u));
    if (ok && pos < DB) idx[pos] = index;
    count += __popc(bal);
  }
}

// N(0,1) draws for the A action entries at step itr (float64 Box-Muller, b200rl.h).
template <int A>
__device__ void explore_normals(uint32_t seed, long long itr, int run, double (&n)[A]) {
#pragma unroll
  for (int c = 0; c < (A + 3) / 4; ++c) {
    uint32_t w[4];
    ddpg_words(seed, itr, run, B200RL_DDPG_STREAM_EXPLORE, (uint32_t)c, w);
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      const double u0 = ((double)w[2 * p] + 0.5) * 2.3283064365386963e-10;
      const double u1 = ((double)w[2 * p + 1] + 0.5) * 2.3283064365386963e-10;
      const double rad = sqrt(-2.0 * log(u0));
      double sn, cs;
      sincospi(2.0 * u1, &sn, &cs);
      if (c * 4 + 2 * p < A) n[c * 4 + 2 * p] = rad * cs;
      if (c * 4 + 2 * p + 1 < A) n[c * 4 + 2 * p + 1] = rad * sn;
    }
  }
}

struct DdpgTrainK {
  int n_steps, es_cap;
  uint32_t seed;
  b200rl_ddpg_hparams hp;
  b200rl_ddpg_state* state;
  double* nets;
  float *pool_obs, *pool_act, *pool_rew;
  unsigned char* pool_term;
  double *stats, *es_returns;
};

template <class Env, class Real>
__global__ void __launch_bounds__(DDPG_THREADS, 1) ddpg_train_kernel(DdpgTrainK k) {
  using D = DdpgNet<Env::O, Env::A>;
  extern __shared__ __align__(16) unsigned char ddpg_smem[];
  const DdpgBufs<D, Real> S(ddpg_smem);
  __shared__ b200rl_ddpg_state st;
  const int run = blockIdx.x, tid = threadIdx.x;
  const b200rl_ddpg_hparams& hp = k.hp;
  const int rows = hp.replay_pool_size;
  double* nets = k.nets + (size_t)run * 4 * D::P;
  const float* pobs_r = k.pool_obs + (size_t)run * rows * D::O;
  float* pobs = k.pool_obs + (size_t)run * rows * D::O;
  float* pact = k.pool_act + (size_t)run * rows * D::A;
  float* prew = k.pool_rew + (size_t)run * rows;
  unsigned char* pterm = k.pool_term + (size_t)run * rows;
  double* stats = k.stats + (size_t)run * B200RL_DDPG_NSTAT;
  double* es_ret = k.es_returns + (size_t)run * k.es_cap;
  if (tid == 0) st = k.state[run];
  load_nets(S, nets);
  for (int step = 0; step < k.n_steps; ++step) {
    if (tid == 0) {
      if (st.terminal) {   // ddpg.py:218-228: env.reset(), es.reset(), record the finished path's return
        float s[Env::S], o[Env::O];
        draw_reset<Env>(s, nullptr, (int)(st.itr & 0x0FFFFFFF), 1, 0, k.seed, (uint32_t)((unsigned long long)st.itr >> 28),
                        run);
        Env::obs(s, o);
        for (int i = 0; i < Env::S; ++i) st.env_state[i] = s[i];
        for (int i = 0; i < Env::O; ++i) st.obs[i] = o[i];
        for (int i = 0; i < Env::A; ++i) st.ou_state[i] = hp.ou_mu;
        if (st.terminal == 1) {
          const long long n = (long long)stats[8];
          if (n < k.es_cap) es_ret[n] = st.path_return;
          stats[8] = (double)(n + 1);
        }
        st.path_length = 0;
        st.path_return = 0.0;
        st.terminal = 0;
      }
    }
    __syncthreads();
    for (int i = tid; i < D::O; i += blockDim.x) S.s[i] = (Real)st.obs[i];
    __syncthreads();
    dense(S.cth + D::PW0, S.cth + D::PB0, S.s, D::O, D::O, DH, 1, S.A1, DH, ACT_RELU);
    __syncthreads();
    dense(S.cth + D::PW1, S.cth + D::PB1, S.A1, DH, DH, DH, 1, S.A2, DH, ACT_RELU);
    __syncthreads();
    dense(S.cth + D::PW2, S.cth + D::PB2, S.A2, DH, DH, D::A, 1, S.mu, D::A, ACT_TANH);
    __syncthreads();
    if (tid == 0) {
      // es.get_action (ou_strategy.py:44-53, gaussian_strategy.py:21-25): clip(mu(obs) + noise, -1, 1), the bounds of
      // the normalized env's action space
      double nz[Env::A];
      explore_normals<Env::A>(k.seed, st.itr, run, nz);
      float act[Env::A], u[Env::A];
      const double sigma = hp.gs_max_sigma - (hp.gs_max_sigma - hp.gs_min_sigma) *
                                                 fmin(1.0, (double)st.itr / hp.gs_decay_period);
      for (int i = 0; i < Env::A; ++i) {
        double x;
        if (hp.es_kind == B200RL_ES_OU) {
          const double xs = st.ou_state[i];
          st.ou_state[i] = xs + (hp.ou_theta * (hp.ou_mu - xs) + hp.ou_sigma * nz[i]);
          x = (double)S.mu[i] + st.ou_state[i];
        } else {
          x = (double)S.mu[i] + nz[i] * sigma;
        }
        act[i] = (float)fmin(fmax(x, -1.0), 1.0);
        u[i] = scale_action(act[i], Env::lb(i), Env::ub(i));
      }
      float s[Env::S], o[Env::O], r;
      bool done;
      for (int i = 0; i < Env::S; ++i) s[i] = st.env_state[i];
      Env::step(s, u, r, done);
      Env::obs(s, o);
      st.path_length += 1;
      st.path_return += (double)r;
      bool add = true, term = done;
      if (!done && st.path_length >= hp.max_path_length) {   // horizon cut (ddpg.py:237-241)
        term = true;
        add = hp.include_horizon_terminal_transitions != 0;
      }
      if (add) {
        const int top = st.top;
        for (int i = 0; i < Env::O; ++i) pobs[(size_t)top * Env::O + i] = st.obs[i];
        for (int i = 0; i < Env::A; ++i) pact[(size_t)top * Env::A + i] = act[i];
        prew[top] = (float)((double)r * hp.scale_reward);
        pterm[top] = term ? 1 : 0;
        st.top = (top + 1) % rows;
        if (st.size >= rows) st.bottom = (st.bottom + 1) % rows;
        else st.size += 1;
      }
      st.terminal = term ? 1 : 0;
      for (int i = 0; i < Env::S; ++i) st.env_state[i] = s[i];
      for (int i = 0; i < Env::O; ++i) st.obs[i] = o[i];
    }
    __syncthreads();
    if (st.size >= hp.min_pool_size) {
      for (int upd = 0; upd < hp.n_updates_per_sample; ++upd) {
        draw_indices(S.idx, k.seed, st.itr, run, upd, st.bottom, st.size, rows);
        __syncthreads();
        gather(S, pobs_r, pact, prew, pterm, rows);
        __syncthreads();
        const long long t = st.adam_t + 1;
        ddpg_update(S, hp, t);
        if (tid == 0) {
          st.adam_t = t;
          stats[0] += 1.0;
          stats[1] += S.red[0];
          stats[2] += S.red[1];
          for (int i = 0; i < 5; ++i) stats[3 + i] += S.red[2 + i];
        }
        __syncthreads();
      }
    }
    if (tid == 0) st.itr += 1;
    __syncthreads();
  }
  store_nets(S, nets);
  if (tid == 0) k.state[run] = st;
}

struct DdpgUpdK {
  b200rl_ddpg_hparams hp;
  const float *pool_obs, *pool_act, *pool_rew;
  const unsigned char* pool_term;
  int rows;
  const int* idx;
  double* nets;
  long long t;
  double *grad_out, *qval_out, *y_out, *loss_out;
};

template <class Env, class Real>
__global__ void __launch_bounds__(DDPG_THREADS, 1) ddpg_update_kernel(DdpgUpdK k) {
  using D = DdpgNet<Env::O, Env::A>;
  extern __shared__ __align__(16) unsigned char ddpg_smem[];
  const DdpgBufs<D, Real> S(ddpg_smem);
  load_nets(S, k.nets);
  if (threadIdx.x < DB) S.idx[threadIdx.x] = k.idx[threadIdx.x];
  __syncthreads();
  gather(S, k.pool_obs, k.pool_act, k.pool_rew, k.pool_term, k.rows);
  __syncthreads();
  ddpg_update(S, k.hp, k.t);
  store_nets(S, k.nets);
  for (int i = threadIdx.x; i < D::P; i += blockDim.x) k.grad_out[i] = S.g[i];
  if (threadIdx.x < DB) {
    k.qval_out[threadIdx.x] = (double)S.q[threadIdx.x];
    k.y_out[threadIdx.x] = (double)S.y[threadIdx.x];
  }
  if (threadIdx.x == 0) { k.loss_out[0] = S.red[0]; k.loss_out[1] = S.red[1]; }
}

// DeterministicMLPPolicy forward of one observation by one thread (float32, parameters in shared memory).
template <class D>
__device__ __forceinline__ void det_forward(const float* __restrict__ p, const float (&o)[D::O], float (&mu)[D::A]) {
  float h1[DH], h2[DH];
#pragma unroll
  for (int j = 0; j < DH; ++j) {
    float acc = p[D::PB0 + j];
#pragma unroll
    for (int k = 0; k < D::O; ++k) acc = fmaf(o[k], p[D::PW0 + k * DH + j], acc);
    h1[j] = fmaxf(acc, 0.0f);
  }
#pragma unroll
  for (int j = 0; j < DH; ++j) {
    float acc = p[D::PB1 + j];
#pragma unroll
    for (int k = 0; k < DH; ++k) acc = fmaf(h1[k], p[D::PW1 + k * DH + j], acc);
    h2[j] = fmaxf(acc, 0.0f);
  }
#pragma unroll
  for (int j = 0; j < D::A; ++j) {
    float acc = p[D::PB2 + j];
#pragma unroll
    for (int k = 0; k < DH; ++k) acc = fmaf(h2[k], p[D::PW2 + k * D::A + j], acc);
    mu[j] = tanhf(acc);
  }
}

template <class D>
__global__ void __launch_bounds__(128) det_get_actions_kernel(const float* __restrict__ params,
                                                              const float* __restrict__ obs, long long n_,
                                                              float* __restrict__ act_out) {
  __shared__ float sp[D::PP];
  for (int i = threadIdx.x; i < D::PP; i += blockDim.x) sp[i] = params[i];
  __syncthreads();
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_) return;
  float o[D::O], mu[D::A];
#pragma unroll
  for (int k = 0; k < D::O; ++k) o[k] = obs[(size_t)k * n_ + n];
  det_forward<D>(sp, o, mu);
#pragma unroll
  for (int k = 0; k < D::A; ++k) act_out[(size_t)k * n_ + n] = mu[k];
}

template <class D>
__global__ void __launch_bounds__(128) qf_get_qval_kernel(const float* __restrict__ params,
                                                          const float* __restrict__ obs, const float* __restrict__ act,
                                                          long long n_, float* __restrict__ q_out) {
  __shared__ float sp[D::QP];
  for (int i = threadIdx.x; i < D::QP; i += blockDim.x) sp[i] = params[i];
  __syncthreads();
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_) return;
  float x[D::HA], h2[DH];
#pragma unroll
  for (int j = 0; j < DH; ++j) {
    float acc = sp[D::QB0 + j];
#pragma unroll
    for (int k = 0; k < D::O; ++k) acc = fmaf(obs[(size_t)k * n_ + n], sp[D::QW0 + k * DH + j], acc);
    x[j] = fmaxf(acc, 0.0f);
  }
#pragma unroll
  for (int k = 0; k < D::A; ++k) x[DH + k] = act[(size_t)k * n_ + n];
#pragma unroll
  for (int j = 0; j < DH; ++j) {
    float acc = sp[D::QB1 + j];
#pragma unroll
    for (int k = 0; k < D::HA; ++k) acc = fmaf(x[k], sp[D::QW1 + k * DH + j], acc);
    h2[j] = fmaxf(acc, 0.0f);
  }
  float acc = sp[D::QB2];
#pragma unroll
  for (int k = 0; k < DH; ++k) acc = fmaf(h2[k], sp[D::QW2 + k], acc);
  q_out[n] = acc;
}

// One thread per lane (lane_rollout, envs.cuh); the head is the deterministic policy without exploration noise.
template <class Env>
__global__ void __launch_bounds__(128) det_rollout_kernel(RolloutArgs a) {
  using D = DdpgNet<Env::O, Env::A>;
  __shared__ float sp[D::PP];
  for (int i = threadIdx.x; i < D::PP; i += blockDim.x) sp[i] = a.params[i];
  __syncthreads();
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= a.N) return;
  float mu[Env::A];
  lane_rollout<Env>(
      a, n, [&](int, int, const float (&o)[Env::O]) { det_forward<D>(sp, o, mu); },
      [&](size_t idx, size_t TN, float (&u)[Env::A]) {
#pragma unroll
        for (int k = 0; k < Env::A; ++k) {
          a.act[k * TN + idx] = mu[k];
          u[k] = scale_action(mu[k], Env::lb(k), Env::ub(k));
        }
      });
}

// (obs_dim, act_dim) pairs of the classic-control Box kinds.
#define B200RL_DISPATCH_DDPG_SHAPE(O, A, entry, ...)                                                             \
  if ((O) == 2 && (A) == 2) { using D = DdpgNet<2, 2>; __VA_ARGS__; }                                             \
  else if ((O) == 3 && (A) == 1) { using D = DdpgNet<3, 1>; __VA_ARGS__; }                                        \
  else if ((O) == 4 && (A) == 1) { using D = DdpgNet<4, 1>; __VA_ARGS__; }                                        \
  else if ((O) == 6 && (A) == 1) { using D = DdpgNet<6, 1>; __VA_ARGS__; }                                        \
  else {                                                                                                          \
    set_error("%s: obs_dim %d, act_dim %d is not compiled in", entry, (int)(O), (int)(A));                        \
    return B200RL_EUNSUPPORTED;                                                                                   \
  }

// The classic-control Box kinds; the planar and discrete kinds are not compiled in.
#define B200RL_DISPATCH_DDPG_ENV(kind, entry, ...)                                                               \
  switch (kind) {                                                                                                 \
    case B200RL_ENV_POINT: { using Env = PointEnvD; __VA_ARGS__; } break;                                          \
    case B200RL_ENV_CARTPOLE: { using Env = CartPoleEnvD; __VA_ARGS__; } break;                                    \
    case B200RL_ENV_PENDULUM: { using Env = PendulumEnvD; __VA_ARGS__; } break;                                    \
    case B200RL_ENV_CARTPOLE_SWINGUP: { using Env = CartPoleSwingupEnvD; __VA_ARGS__; } break;                     \
    case B200RL_ENV_DOUBLE_PENDULUM: { using Env = DoublePendulumEnvD; __VA_ARGS__; } break;                       \
    default:                                                                                                      \
      set_error("%s: env kind %d is not supported by DDPG (classic-control Box kinds only)", entry, (int)(kind)); \
      return B200RL_EUNSUPPORTED;                                                                                 \
  }

static int check_hparams(const char* entry, const b200rl_ddpg_hparams& hp) {
  B200RL_REQUIRE(hp.replay_pool_size > DB && hp.max_path_length > 0 && hp.n_updates_per_sample >= 0 &&
                     hp.n_updates_per_sample < (1 << 16) && hp.min_pool_size > DB &&
                     (hp.es_kind == B200RL_ES_OU || hp.es_kind == B200RL_ES_GAUSSIAN),
                 "%s: bad hyperparameters (replay_pool_size and min_pool_size must exceed the batch size %d, "
                 "es_kind must be OU or Gaussian)", entry, DB);
  return 0;
}

}  // namespace b200rl

using namespace b200rl;

long long b200rl_ddpg_num_params(int obs_dim, int act_dim, int which) {
  B200RL_REQUIRE(which == 0 || which == 1, "ddpg_num_params: which must be 0 (policy) or 1 (qf)");
  B200RL_DISPATCH_DDPG_SHAPE(obs_dim, act_dim, "ddpg_num_params", return which == 0 ? D::PP : D::QP);
}

int b200rl_deterministic_get_actions(const float* params_f32, int obs_dim, int act_dim, const float* obs, long long n,
                                     float* act_out, void* stream) {
  B200RL_REQUIRE(params_f32 && obs && act_out && n > 0, "deterministic_get_actions: bad arguments");
  B200RL_DISPATCH_DDPG_SHAPE(obs_dim, act_dim, "deterministic_get_actions", {
    det_get_actions_kernel<D><<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(params_f32, obs, n,
                                                                                              act_out);
  });
  B200RL_LAUNCH_CHECK("det_get_actions_kernel");
  return 0;
}

int b200rl_qf_get_qval(const float* params_f32, int obs_dim, int act_dim, const float* obs, const float* act,
                       long long n, float* q_out, void* stream) {
  B200RL_REQUIRE(params_f32 && obs && act && q_out && n > 0, "qf_get_qval: bad arguments");
  B200RL_DISPATCH_DDPG_SHAPE(obs_dim, act_dim, "qf_get_qval", {
    qf_get_qval_kernel<D><<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(params_f32, obs, act, n,
                                                                                          q_out);
  });
  B200RL_LAUNCH_CHECK("qf_get_qval_kernel");
  return 0;
}

int b200rl_rollout_deterministic(int env_kind, const float* params_f32, int N, int T, int max_path_length,
                                 const float* reset_raw, unsigned int seed, unsigned int iter, long long lane0, float* obs,
                                 float* act, float* rew, unsigned char* flags, unsigned short* tstep, void* stream) {
  const RolloutArgs a{params_f32, 0.f, N, T, max_path_length, nullptr, reset_raw, seed, iter, lane0,
                      obs, act, act, rew, flags, tstep, nullptr};
  if (int rc = check_rollout_args("rollout_deterministic", a, false)) return rc;
  B200RL_DISPATCH_DDPG_ENV(env_kind, "rollout_deterministic", {
    det_rollout_kernel<Env><<<(N + 127) / 128, 128, 0, (cudaStream_t)stream>>>(a);
  });
  B200RL_LAUNCH_CHECK("det_rollout_kernel");
  return 0;
}

int b200rl_ddpg_update(int env_kind, int f64, const b200rl_ddpg_hparams* hp, const float* pool_obs,
                       const float* pool_act, const float* pool_rew, const unsigned char* pool_term, int pool_size,
                       const int* idx, double* nets, long long adam_t, double* grad_out, double* qval_out,
                       double* y_out, double* loss_out, void* stream) {
  B200RL_REQUIRE(hp && pool_obs && pool_act && pool_rew && pool_term && idx && nets && grad_out && qval_out && y_out &&
                     loss_out && pool_size > 1 && adam_t >= 1,
                 "ddpg_update: bad arguments");
  const DdpgUpdK k{*hp, pool_obs, pool_act, pool_rew, pool_term, pool_size, idx, nets, adam_t,
                   grad_out, qval_out, y_out, loss_out};
  B200RL_DISPATCH_DDPG_ENV(env_kind, "ddpg_update", {
    using D = DdpgNet<Env::O, Env::A>;
    if (f64) {
      constexpr size_t bytes = DdpgSmem<D, double>::bytes;
      auto* kern = ddpg_update_kernel<Env, double>;
      B200RL_SET_MAX_SMEM(kern, bytes);
      kern<<<1, DDPG_THREADS, bytes, (cudaStream_t)stream>>>(k);
    } else {
      constexpr size_t bytes = DdpgSmem<D, float>::bytes;
      auto* kern = ddpg_update_kernel<Env, float>;
      B200RL_SET_MAX_SMEM(kern, bytes);
      kern<<<1, DDPG_THREADS, bytes, (cudaStream_t)stream>>>(k);
    }
  });
  B200RL_LAUNCH_CHECK("ddpg_update_kernel");
  return 0;
}

int b200rl_ddpg_train(const b200rl_ddpg_train_args* args) {
  B200RL_REQUIRE(args != nullptr, "ddpg_train: null arguments");
  const b200rl_ddpg_train_args& a = *args;
  B200RL_REQUIRE(a.state && a.nets && a.pool_obs && a.pool_act && a.pool_rew && a.pool_term && a.stats &&
                     a.es_returns,
                 "ddpg_train: null buffer");
  B200RL_REQUIRE(a.n_runs > 0 && a.n_steps >= 0 && a.es_cap > 0, "ddpg_train: n_runs, es_cap must be positive");
  if (int rc = check_hparams("ddpg_train", a.hp)) return rc;
  if (a.n_steps == 0) return 0;
  const DdpgTrainK k{a.n_steps, a.es_cap, a.seed, a.hp, a.state, a.nets, a.pool_obs, a.pool_act, a.pool_rew,
                     a.pool_term, a.stats, a.es_returns};
  B200RL_DISPATCH_DDPG_ENV(a.env_kind, "ddpg_train", {
    using D = DdpgNet<Env::O, Env::A>;
    if (a.f64) {
      constexpr size_t bytes = DdpgSmem<D, double>::bytes;
      auto* kern = ddpg_train_kernel<Env, double>;
      B200RL_SET_MAX_SMEM(kern, bytes);
      kern<<<a.n_runs, DDPG_THREADS, bytes, (cudaStream_t)a.stream>>>(k);
    } else {
      constexpr size_t bytes = DdpgSmem<D, float>::bytes;
      auto* kern = ddpg_train_kernel<Env, float>;
      B200RL_SET_MAX_SMEM(kern, bytes);
      kern<<<a.n_runs, DDPG_THREADS, bytes, (cudaStream_t)a.stream>>>(k);
    }
  });
  B200RL_LAUNCH_CHECK("ddpg_train_kernel");
  return 0;
}
