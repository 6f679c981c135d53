// Per-lane environment dynamics (device functions, state in registers).  Each env is a struct with
//   O, A, S (state floats), K (raw reset noise count), NOISE (uniform|normal), lb()/ub()
//   reset(s, raw) ; obs(s, o) ; step(s, u, r, done)   with u = action after NormalizedEnv scaling.
// Reference classes are cited per struct; the NormalizedEnv action map lives in scale_action().
#pragma once
#include <type_traits>
#include "common.cuh"

namespace b200rl {

// NormalizedEnv.step (rllab/envs/normalized_env.py:81-83): clip(lb + (a+1)*0.5*(ub-lb), lb, ub).
// Written with explicit round-to-nearest ops (no FMA contraction) so that it is bit-identical to NumPy float32.
__device__ __forceinline__ float scale_action(float a, float lb, float ub) {
  float t = __fmul_rn(__fmul_rn(__fadd_rn(a, 1.0f), 0.5f), __fsub_rn(ub, lb));
  float s = __fadd_rn(lb, t);
  return fminf(fmaxf(s, lb), ub);
}

// ---------------------------------------------------------------- examples/point_env.py:16-27
struct PointEnvD {
  static constexpr int KIND = B200RL_ENV_POINT, O = 2, A = 2, S = 2, K = 2, NOISE = B200RL_NOISE_UNIFORM;
  __host__ __device__ static constexpr float lb(int) { return -0.1f; }
  __host__ __device__ static constexpr float ub(int) { return 0.1f; }
  __device__ static void reset(float (&s)[S], const float (&raw)[K]) {
    s[0] = __fadd_rn(-1.0f, __fmul_rn(2.0f, raw[0]));  // np.random.uniform(-1,1)
    s[1] = __fadd_rn(-1.0f, __fmul_rn(2.0f, raw[1]));
  }
  __device__ static void obs(const float (&s)[S], float (&o)[O]) { o[0] = s[0]; o[1] = s[1]; }
  __device__ static void step(float (&s)[S], const float (&u)[A], float& r, bool& done) {
    s[0] = __fadd_rn(s[0], u[0]);
    s[1] = __fadd_rn(s[1], u[1]);
    r = -__fsqrt_rn(__fadd_rn(__fmul_rn(s[0], s[0]), __fmul_rn(s[1], s[1])));
    done = (fabsf(s[0]) < 0.01f) && (fabsf(s[1]) < 0.01f);
  }
};

// ---------------------------------------------------------------- rllab/envs/box2d/cartpole_env.py:13-56
// Reduced-coordinate restatement of the Box2D model (models/cartpole.xml.mako:3-45), see oracle/envs.py.
struct CartPoleEnvD {
  static constexpr int KIND = B200RL_ENV_CARTPOLE, O = 4, A = 1, S = 4, K = 4, NOISE = B200RL_NOISE_UNIFORM;
  __host__ __device__ static constexpr float lb(int) { return -10.0f; }
  __host__ __device__ static constexpr float ub(int) { return 10.0f; }
  __device__ static void reset(float (&s)[S], const float (&raw)[K]) {
    const float b[4] = {2.4f * 0.05f, 4.0f * 0.05f, 0.2f * 0.05f, 4.0f * 0.05f};
#pragma unroll
    for (int i = 0; i < 4; ++i) s[i] = -b[i] + (2.0f * b[i]) * raw[i];
  }
  __device__ static void obs(const float (&s)[S], float (&o)[O]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = s[i];
  }
  __device__ static void step(float (&s)[S], const float (&u)[A], float& r, bool& done) {
    const float M = 1.0f, m = 0.1f, l = 0.5f, g = 10.0f, h = 0.05f;
    const float I = 0.1f * (0.1f * 0.1f + 1.0f) / 12.0f;
    float x = s[0], xd = s[1], th = s[2], thd = s[3];
    float F = fminf(fmaxf(u[0], -10.0f), 10.0f);
    float sn, cs;
    sincosf(th, &sn, &cs);
    float a11 = M + m, a12 = -m * l * cs, a22 = I + m * l * l;
    float b1 = F - m * l * sn * thd * thd;
    float b2 = m * g * l * sn;
    const float idet = 1.0f / (a11 * a22 - a12 * a12);   // one IEEE division per step instead of two
    float xdd = (a22 * b1 - a12 * b2) * idet;
    float thdd = (a11 * b2 - a12 * b1) * idet;
    xd += h * xdd;
    thd += h * thdd;
    x += h * xd;
    th += h * thd;
    s[0] = x; s[1] = xd; s[2] = th; s[3] = thd;
    done = (fabsf(x) > 2.4f) || (fabsf(th) > 0.2f);
    float notdone = done ? 0.0f : 1.0f;
    float ucost = 1e-5f * (u[0] * u[0]);
    float xcost = 1.0f - cosf(th);
    r = notdone * 10.0f - notdone * xcost - notdone * ucost;
  }
};

// ---------------------------------------------------------------- rllab/envs/box2d/cartpole_swingup_env.py:15-58
// Same Box2D model (models/cartpole.xml.mako) and therefore the same reduced-coordinate dynamics as CartPoleEnvD; what
// differs is the task: reset x, xdot, theta, thetadot ~ U([-1,-2,pi-1,-3], [1,2,pi+1,3]) (pole hanging down), done =
// |x| > 3, reward (post-step) = -100 if done, else cos(theta) (the "-1 beyond max_reward_cart_pos" branch cannot fire:
// max_reward_cart_pos == max_cart_pos == 3).
struct CartPoleSwingupEnvD {
  static constexpr int KIND = B200RL_ENV_CARTPOLE_SWINGUP, O = 4, A = 1, S = 4, K = 4, NOISE = B200RL_NOISE_UNIFORM;
  __host__ __device__ static constexpr float lb(int) { return -10.0f; }
  __host__ __device__ static constexpr float ub(int) { return 10.0f; }
  __device__ static void reset(float (&s)[S], const float (&raw)[K]) {
    const float PI = 3.14159265358979323846f;
    const float lo[4] = {-1.0f, -2.0f, PI - 1.0f, -3.0f}, hi[4] = {1.0f, 2.0f, PI + 1.0f, 3.0f};
#pragma unroll
    for (int i = 0; i < 4; ++i) s[i] = lo[i] + (hi[i] - lo[i]) * raw[i];
  }
  __device__ static void obs(const float (&s)[S], float (&o)[O]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = s[i];
  }
  __device__ static void step(float (&s)[S], const float (&u)[A], float& r, bool& done) {
    float rr;
    bool dd;
    CartPoleEnvD::step(s, u, rr, dd);          // shared dynamics; its reward / termination are replaced below
    done = fabsf(s[0]) > 3.0f;
    r = done ? -100.0f : cosf(s[2]);
  }
};

// ---------------------------------------------------------------- rllab/envs/box2d/double_pendulum_env.py:11-61
// Reduced-coordinate restatement of models/double_pendulum.xml.mako (see oracle/envs.py::DoublePendulumEnv): two rods of
// length L = 1 (width 0.1, density 5 -> m = 0.5, I_com = m (w^2 + L^2) / 12) hanging from the origin, absolute body angles
// th1, th2 (CCW, 0 = hanging down), gravity (0, -10), torque u in [-50, 50] on the joint between the links (+u on link 2,
// -u on link 1: the revolute motor of box2d_env.py:134-144), semi-implicit Euler, dt = 0.01, frame_skip = 2.
// obs = [sin th1, cos th1, w1, sin th2, cos th2, w2]; reward (post-step) = -|tip - (0, 2L)| with the reference's tip
// formula (double_pendulum_env.py:43-50: link-2 origin minus L (sin th2, cos th2)); never done.
struct DoublePendulumEnvD {
  static constexpr int KIND = B200RL_ENV_DOUBLE_PENDULUM, O = 6, A = 1, S = 4, K = 4, NOISE = B200RL_NOISE_NORMAL;
  __host__ __device__ static constexpr float lb(int) { return -50.0f; }
  __host__ __device__ static constexpr float ub(int) { return 50.0f; }
  __device__ static void reset(float (&s)[S], const float (&raw)[K]) {
    s[0] = 0.1f * raw[0]; s[1] = 0.1f * raw[1]; s[2] = 0.01f * raw[2]; s[3] = 0.01f * raw[3];   // th1, th2, w1, w2
  }
  __device__ static void obs(const float (&s)[S], float (&o)[O]) {
    float sn, cs;
    sincosf(s[0], &sn, &cs);
    o[0] = sn; o[1] = cs; o[2] = s[2];
    sincosf(s[1], &sn, &cs);
    o[3] = sn; o[4] = cs; o[5] = s[3];
  }
  __device__ static void step(float (&s)[S], const float (&u)[A], float& r, bool& done) {
    const float L = 1.0f, m = 0.5f, lc = 0.5f, g = 10.0f, h = 0.01f;
    const float I = 0.5f * (0.1f * 0.1f + 1.0f) / 12.0f;
    const float m11 = I + m * lc * lc + m * L * L, m22 = I + m * lc * lc, mlc = m * L * lc;
    float th1 = s[0], th2 = s[1], w1 = s[2], w2 = s[3];
    const float tau = fminf(fmaxf(u[0], -50.0f), 50.0f);
#pragma unroll
    for (int k = 0; k < 2; ++k) {                 // frame_skip = 2 (double_pendulum_env.py:16)
      float sd, cd, s1, c1, s2, c2;
      sincosf(th1 - th2, &sd, &cd);
      sincosf(th1, &s1, &c1);
      sincosf(th2, &s2, &c2);
      const float m12 = mlc * cd;
      const float b1 = -tau - mlc * sd * w2 * w2 - (m * lc + m * L) * g * s1;
      const float b2 = tau + mlc * sd * w1 * w1 - m * g * lc * s2;
      const float idet = 1.0f / (m11 * m22 - m12 * m12);
      const float a1 = (m22 * b1 - m12 * b2) * idet;
      const float a2 = (m11 * b2 - m12 * b1) * idet;
      w1 += h * a1;
      w2 += h * a2;
      th1 += h * w1;
      th2 += h * w2;
    }
    s[0] = th1; s[1] = th2; s[2] = w1; s[3] = w2;
    float s1, c1, s2, c2;
    sincosf(th1, &s1, &c1);
    sincosf(th2, &s2, &c2);
    const float tx = L * s1 - L * s2, ty = -L * c1 - L * c2;      // link-2 origin (L sin th1, -L cos th1) - L (sin th2, cos th2)
    const float dx = tx, dy = ty - 2.0f * L;
    r = -sqrtf(dx * dx + dy * dy);
    done = false;
  }
};

// ---------------------------------------------------------------- gym 0.7.4 Pendulum-v0 via rllab/envs/gym_env.py:58-116
struct PendulumEnvD {
  static constexpr int KIND = B200RL_ENV_PENDULUM, O = 3, A = 1, S = 2, K = 2, NOISE = B200RL_NOISE_UNIFORM;
  __host__ __device__ static constexpr float lb(int) { return -2.0f; }
  __host__ __device__ static constexpr float ub(int) { return 2.0f; }
  __device__ static void reset(float (&s)[S], const float (&raw)[K]) {
    const float PI = 3.14159265358979323846f;
    s[0] = -PI + (2.0f * PI) * raw[0];
    s[1] = -1.0f + 2.0f * raw[1];
  }
  __device__ static void obs(const float (&s)[S], float (&o)[O]) {
    float sn, cs;
    sincosf(s[0], &sn, &cs);
    o[0] = cs; o[1] = sn; o[2] = s[1];
  }
  __device__ static void step(float (&s)[S], const float (&u)[A], float& r, bool& done) {
    const float PI = 3.14159265358979323846f;
    float th = s[0], thd = s[1];
    float uu = fminf(fmaxf(u[0], -2.0f), 2.0f);
    float t = th + PI;
    float an = t - floorf(t / (2.0f * PI)) * (2.0f * PI) - PI;  // ((th+pi) mod 2pi) - pi, python-style mod
    float cost = an * an + 0.1f * thd * thd + 0.001f * (uu * uu);
    float nthd = thd + (-15.0f * sinf(th + PI) + 3.0f * uu) * 0.05f;
    float nth = th + nthd * 0.05f;
    nthd = fminf(fmaxf(nthd, -8.0f), 8.0f);
    s[0] = nth; s[1] = nthd;
    r = -cost;
    done = false;
  }
};

// ---------------------------------------------------------------- gym 0.7.4 CartPole-v0 via rllab/envs/gym_env.py
// gym/envs/classic_control/cartpole.py restated (no in-tree reference dynamics, as Pendulum-v0): explicit Euler with
// tau = 0.02, the cart moved with the OLD velocities; action index 1 pushes with +10, 0 with -10.  done when |x| > 2.4 or
// |theta| > 12 deg; reward 1 on every step, the terminal one included.  The single action float is the index
// (NACT = 2 actions): NormalizedEnv passes a Discrete action through unscaled (normalized_env.py:71-75).
struct GymCartPoleEnvD {
  static constexpr int KIND = B200RL_ENV_GYM_CARTPOLE, O = 4, A = 1, S = 4, K = 4, NOISE = B200RL_NOISE_UNIFORM,
                       NACT = 2;
  __host__ __device__ static constexpr float lb(int) { return 0.0f; }
  __host__ __device__ static constexpr float ub(int) { return (float)(NACT - 1); }
  __device__ static void reset(float (&s)[S], const float (&raw)[K]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) s[i] = -0.05f + 0.1f * raw[i];    // np_random.uniform(-0.05, 0.05, size=(4,))
  }
  __device__ static void obs(const float (&s)[S], float (&o)[O]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = s[i];
  }
  __device__ static void step(float (&s)[S], const float (&u)[A], float& r, bool& done) {
    const float g = 9.8f, mp = 0.1f, total = 1.1f, l = 0.5f, pml = 0.05f, tau = 0.02f;
    const float thr = 12.0f * 2.0f * 3.14159265358979323846f / 360.0f;
    const float x = s[0], xd = s[1], th = s[2], thd = s[3];
    const float force = ((int)u[0] == 1) ? 10.0f : -10.0f;
    float sn, cs;
    sincosf(th, &sn, &cs);
    const float temp = (force + pml * thd * thd * sn) / total;
    const float thacc = (g * sn - cs * temp) / (l * (4.0f / 3.0f - mp * cs * cs / total));
    const float xacc = temp - pml * thacc * cs / total;
    s[0] = x + tau * xd;
    s[1] = xd + tau * xacc;
    s[2] = th + tau * thd;
    s[3] = thd + tau * thacc;
    done = (s[0] < -2.4f) || (s[0] > 2.4f) || (s[2] < -thr) || (s[2] > thr);
    r = 1.0f;
  }
};

// Number of discrete actions of an env kind: Env::NACT where the struct declares it, 0 for a Box action space.
template <class Env, class = void>
struct EnvNumActions {
  static constexpr int value = 0;
};
template <class Env>
struct EnvNumActions<Env, std::void_t<decltype(Env::NACT)>> {
  static constexpr int value = Env::NACT;
};

}  // namespace b200rl

#include "planar.cuh"

namespace b200rl {

#ifdef B200RL_HAVE_PLANAR
#define B200RL_PLANAR_CASES(...)                                                              \
    case B200RL_ENV_SWIMMER: { using Env = ::b200rl::SwimmerEnvD; __VA_ARGS__; } break;       \
    case B200RL_ENV_HOPPER: { using Env = ::b200rl::HopperEnvD; __VA_ARGS__; } break;       \
    case B200RL_ENV_HALF_CHEETAH: { using Env = ::b200rl::HalfCheetahEnvD; __VA_ARGS__; } break;
#else
#define B200RL_PLANAR_CASES(...)
#endif

// Reset of one lane: raw noise from reset_raw [row][K][N] (tests) or Philox stream 1 at (lane, row).  Shared by the lane
// rollout and the population rollout, so both draw the same reset for the same lane.
template <class Env>
__device__ __forceinline__ void draw_reset(float (&s)[Env::S], const float* __restrict__ reset_raw, int row, int N,
                                           int n, uint32_t seed, uint32_t iter, long long lane) {
  float raw[Env::K];
  if (reset_raw != nullptr) {
#pragma unroll
    for (int k = 0; k < Env::K; ++k) raw[k] = reset_raw[((size_t)row * Env::K + k) * N + n];
  } else {
#pragma unroll
    for (int c = 0; c < (Env::K + 3) / 4; ++c) {
      float q[4];
      noise4(Env::NOISE, seed, iter, 1, lane, row, c, q);
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (c * 4 + i < Env::K) raw[c * 4 + i] = q[i];
    }
  }
  Env::reset(s, raw);
}

// Action noise of one lane at step `row`: eps [row][A][N] (tests) or Philox stream 0 at (lane, row).
template <int A, typename std::enable_if<(A <= 4), int>::type = 0>
__device__ __forceinline__ void draw_eps(float (&e)[A], const float* __restrict__ eps, int row, long long N,
                                         long long n, uint32_t seed, uint32_t iter, long long lane) {
  if (eps != nullptr) {
#pragma unroll
    for (int a = 0; a < A; ++a) e[a] = eps[((size_t)row * A + a) * N + n];
  } else {
    float q[4];
    noise4<(A + 1) / 2>(B200RL_NOISE_NORMAL, seed, iter, 0, lane, row, 0, q);
#pragma unroll
    for (int a = 0; a < A; ++a) e[a] = q[a];
  }
}

// A > 4: chunk c of the Philox stream holds eps[4c .. 4c+3], as in draw_reset and b200rl_fill_noise.
template <int A, typename std::enable_if<(A > 4), int>::type = 0>
__device__ __forceinline__ void draw_eps(float (&e)[A], const float* __restrict__ eps, int row, long long N,
                                         long long n, uint32_t seed, uint32_t iter, long long lane) {
  if (eps != nullptr) {
#pragma unroll
    for (int a = 0; a < A; ++a) e[a] = eps[((size_t)row * A + a) * N + n];
  } else {
#pragma unroll
    for (int c = 0; c < (A + 3) / 4; ++c) {
      float q[4];
      noise4<2>(B200RL_NOISE_NORMAL, seed, iter, 0, lane, row, c, q);   // an unused last pair is dead code
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (c * 4 + i < A) e[c * 4 + i] = q[i];
    }
  }
}

// Arguments of the fused lane rollouts (rollout_kernel, cat_rollout_kernel, gru_rollout_kernel).  eps: the action noise
// [T][A][N] (the categorical rollout's uniforms [T][N]) or NULL for Philox; mean: the mean plane (the categorical
// rollout's probabilities); log_min_std, log_std_out: the Gaussian policies' log_std only.
struct RolloutArgs {
  const float* params;
  float log_min_std;
  int N, T, max_path_length;
  const float* eps;
  const float* reset_raw;
  uint32_t seed, iter;
  long long lane0;
  float *obs, *act, *mean, *rew;
  unsigned char* flags;
  unsigned short* tstep;
  float* log_std_out;
};

// The checks the fused rollouts' entry points make first; `entry` prefixes the error text.  with_log_std: the policy
// has a log_std to report (log_std_out required).
inline int check_rollout_args(const char* entry, const RolloutArgs& a, bool with_log_std) {
  B200RL_REQUIRE(a.params && a.obs && a.act && a.mean && a.rew && a.flags && a.tstep &&
                 (a.log_std_out || !with_log_std), "%s: null buffer", entry);
  B200RL_REQUIRE(a.N > 0 && a.T > 0 && a.max_path_length > 0, "%s: N, T, max_path_length must be positive", entry);
  B200RL_REQUIRE(a.max_path_length <= 65535, "%s: max_path_length must fit uint16 tstep", entry);
  return 0;
}

// The lane loop of the fused rollouts: lane n runs all T steps in one thread with the env state in registers.  The loop
// owns the sample bookkeeping that process_samples, the whole-path masking, REPS and the GRU passes read: obs and rew
// planes, tstep (the step's index in its path, so a path starts where tstep == 0), the DONE / END / CUT flags, and the
// resets (row 0 for the first path, row t + 1 after a path ends at step t).  The policy's head runs in two calls per step:
//   act(t, plen, o)      computes the action from the observation o (plen == 0: the first step of a path);
//   record(idx, TN, u)   writes the policy's act and mean planes at [k * TN + idx] and returns the env input in u.
// The obs plane is stored between the two, after the noise loads and before the act / mean stores: the compiler may not
// reorder these possibly aliasing accesses, and any other order changes the hot rollout's generated code.
template <class Env, class Act, class Record>
__device__ __forceinline__ void lane_rollout(const RolloutArgs& a, int n, Act&& act, Record&& record) {
  const long long lane = a.lane0 + n;
  const size_t N = a.N, TN = (size_t)a.T * a.N;
  float s[Env::S];
  draw_reset<Env>(s, a.reset_raw, 0, a.N, n, a.seed, a.iter, lane);
  int plen = 0;
  for (int t = 0; t < a.T; ++t) {
    float o[Env::O], u[Env::A];
    // compiler barrier: without it the loop-invariant LDS of all P weights is hoisted out of the t loop and spilled
    asm volatile("" ::: "memory");
    Env::obs(s, o);
    act(t, plen, o);
    const size_t idx = (size_t)t * N + n;
#pragma unroll
    for (int k = 0; k < Env::O; ++k) a.obs[k * TN + idx] = o[k];
    record(idx, TN, u);
    float r;
    bool done;
    Env::step(s, u, r, done);
    a.tstep[idx] = (unsigned short)plen;
    ++plen;
    const bool whole = done || (plen >= a.max_path_length);
    const bool end = whole || (t == a.T - 1);
    a.rew[idx] = r;
    // FLAG_CUT: the path is cut by the end of the lane buffer, not by the env or max_path_length (process_samples drops
    // such paths when the caller asks for whole paths only, batch_polopt.py:30-34)
    a.flags[idx] = (unsigned char)((done ? B200RL_FLAG_DONE : 0) | (end ? B200RL_FLAG_END : 0) |
                                   ((end && !whole) ? B200RL_FLAG_CUT : 0));
    if (end) {
      draw_reset<Env>(s, a.reset_raw, t + 1, a.N, n, a.seed, a.iter, lane);
      plen = 0;
    }
  }
}

// Dispatch an env kind to its struct: F is a generic lambda / functor called as f(Env{}).
#define B200RL_DISPATCH_ENV(kind, ...)                                                        \
  switch (kind) {                                                                             \
    case B200RL_ENV_POINT: { using Env = ::b200rl::PointEnvD; __VA_ARGS__; } break;           \
    case B200RL_ENV_CARTPOLE: { using Env = ::b200rl::CartPoleEnvD; __VA_ARGS__; } break;     \
    case B200RL_ENV_PENDULUM: { using Env = ::b200rl::PendulumEnvD; __VA_ARGS__; } break;     \
    case B200RL_ENV_CARTPOLE_SWINGUP: { using Env = ::b200rl::CartPoleSwingupEnvD; __VA_ARGS__; } break; \
    case B200RL_ENV_DOUBLE_PENDULUM: { using Env = ::b200rl::DoublePendulumEnvD; __VA_ARGS__; } break; \
    B200RL_PLANAR_CASES(__VA_ARGS__)                                                          \
    default:                                                                                  \
      ::b200rl::set_error("unknown env kind %d", (int)(kind));                                \
      return B200RL_EUNSUPPORTED;                                                             \
  }

// B200RL_DISPATCH_ENV plus the discrete-action kinds (Env::A = 1 float holding the action index).  For the entry points
// that take any env (info, reset, step); the Gaussian rollout and the population rollout dispatch Box kinds only.
#define B200RL_DISPATCH_ENV_ANY(kind, ...)                                                    \
  if ((kind) == B200RL_ENV_GYM_CARTPOLE) {                                                    \
    using Env = ::b200rl::GymCartPoleEnvD;                                                    \
    __VA_ARGS__;                                                                              \
  } else                                                                                      \
    B200RL_DISPATCH_ENV(kind, __VA_ARGS__)

}  // namespace b200rl
