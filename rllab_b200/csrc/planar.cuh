// Planar articulated-body environments: rllab's MuJoCo Swimmer, Hopper and HalfCheetah restated as planar kinematic
// trees (generalised coordinates, M(q) qacc + bias = tau, semi-implicit Euler x50 / RK4 / Euler, inertia-box fluid
// forces, soft joint-limit and contact constraints solved by a fixed number of projected Gauss-Seidel sweeps).
// One thread per lane, float32, everything in registers except HalfCheetah's active constraint rows (local memory).
// The float64 statement of the same models is oracle/planar.py (serial chains) and tests/planar_tree_oracle.py (the
// tree, HalfCheetah), which document the modelling choices and cite the reference files; they must agree to float32
// tolerance (tests/test_gpu_kernels.py::test_env_step_matches_oracle, tests/test_gpu_half_cheetah.py).
//
// Reference call sites: rllab/envs/mujoco/mujoco_env.py:109-132,184-191, swimmer_env.py:25-45, hopper_env.py:38-61,
// half_cheetah_env.py:22-48, rllab/mujoco_py/mjcore.py:58-81, vendor/mujoco_models/{swimmer,hopper,half_cheetah}.xml.
// The arithmetic of the closed MuJoCo 1.31 binary is absent: PARITY UNPINNED (SURVEY.md 8c).
#pragma once
#define B200RL_HAVE_PLANAR 1
#include "common.cuh"

namespace b200rl {

constexpr int PLANAR_PGS_SWEEPS = 8;
constexpr float PLANAR_PI = 3.14159265358979323846f;

struct CapsuleC {
  float m, Ip, Ia;
};
__host__ __device__ constexpr CapsuleC capsule_c(double r, double L) {
  const double rho = 1000.0, pi = 3.14159265358979323846;
  const double mc = rho * pi * r * r * L, mh = rho * (2.0 / 3.0) * pi * r * r * r;
  return CapsuleC{(float)(mc + 2 * mh),
                  (float)(mc * (r * r / 4 + L * L / 12) + 2 * mh * (2 * r * r / 5 + L * L / 4 + 3 * L * r / 8)),
                  (float)(mc * r * r / 2 + 2 * mh * (2 * r * r / 5))};
}

// Defaults of the model terms that only HalfCheetah uses; each leaves the Swimmer / Hopper arithmetic unchanged.
struct PlanarModelDefaults {
  static constexpr float y0 = 0.f;                      // world height of the root body at rootz = 0
  static constexpr bool active_rows = false;            // PGS over the compacted active rows (else dense, in registers)
  // joint limits: solref (.02, 1), solimp (.9, .95, .001);  contacts: solref (.02, 1), solimp (.8, .8, .01)
  static constexpr float lim_tc = 0.02f, lim_d0 = 0.9f, lim_d1 = 0.95f, lim_w = 0.001f;
  static constexpr float con_tc = 0.02f, con_d0 = 0.8f, con_d1 = 0.8f, con_w = 0.01f;
  __host__ __device__ static constexpr float stiffness(int) { return 0.f; }   // spring to qpos0 = 0
  __host__ __device__ static constexpr float gear(int) { return 1.f; }
};

// Topology: body i hangs from M::parent(i) < i (body 0 is the root); M::is_ancestor(k, i): k is an ancestor of i, or i
// itself, stated in closed form so that it folds inside the unrolled Jacobian loops.  planar_topology_ok checks the two
// against each other at compile time.
template <class M>
__host__ __device__ constexpr bool planar_topology_ok() {
  for (int i = 0; i < M::n; ++i)
    for (int k = 0; k < M::n; ++k) {
      int j = i;
      while (j > k) j = M::parent(j);
      if (M::is_ancestor(k, i) != (j == k) || (i > 0 && M::parent(i) >= i)) return false;
    }
  return true;
}

// ---------------------------------------------------------------- model descriptions (compile-time accessors)
struct SwimmerModel : PlanarModelDefaults {
  static constexpr int n = 3, nv = 5, nu = 2, iX = 0, iY = 1, nlim = 2, ncon = 0;
  static constexpr bool rk4 = false, fluid = true;
  static constexpr int frame_skip = 50;
  static constexpr float dt = 0.001f, gX = 0.f, gY = 0.f, density = 4000.f, viscosity = 0.1f, ctrl_lim = 50.f;
  __host__ __device__ static constexpr int parent(int i) { return i - 1; }
  __host__ __device__ static constexpr bool is_ancestor(int k, int i) { return k <= i; }
  __host__ __device__ static constexpr float sgn(int) { return 1.f; }
  __host__ __device__ static constexpr float ax(int i) { return i == 1 ? 0.5f : (i == 2 ? -1.f : 0.f); }
  __host__ __device__ static constexpr float ay(int) { return 0.f; }
  __host__ __device__ static constexpr float cx(int i) { return i == 0 ? 1.f : -0.5f; }
  __host__ __device__ static constexpr float cy(int) { return 0.f; }
  __host__ __device__ static constexpr float box(int) { return 0.f; }
  __host__ __device__ static constexpr float boy(int) { return 0.f; }
  __host__ __device__ static constexpr CapsuleC cap(int) { return capsule_c(0.1, 1.0); }
  __host__ __device__ static constexpr float lax(int) { return 1.f; }
  __host__ __device__ static constexpr float lay(int) { return 0.f; }
  __host__ __device__ static constexpr float armature(int) { return 0.f; }
  __host__ __device__ static constexpr float damping(int) { return 0.f; }
  __host__ __device__ static constexpr int act(int j) { return j + 1; }             // actuated hinge index
  __host__ __device__ static constexpr int lim_hinge(int j) { return j + 1; }       // limited hinge index
  __host__ __device__ static constexpr float lim_lo(int) { return -100.f * PLANAR_PI / 180.f; }
  __host__ __device__ static constexpr float lim_hi(int) { return 100.f * PLANAR_PI / 180.f; }
  __host__ __device__ static constexpr float q0(int) { return 0.f; }
  // contacts unused
  __host__ __device__ static constexpr int con_body(int) { return 0; }
  __host__ __device__ static constexpr float con_ex(int) { return 0.f; }
  __host__ __device__ static constexpr float con_ey(int) { return 0.f; }
  __host__ __device__ static constexpr float con_r(int) { return 0.f; }
  static constexpr float mu = 0.f, margin = 0.f;
};

struct HopperModel : PlanarModelDefaults {
  static constexpr int n = 4, nv = 6, nu = 3, iX = 1, iY = 0, nlim = 3, ncon = 2;
  static constexpr bool rk4 = true, fluid = false;
  static constexpr int frame_skip = 1;
  static constexpr float dt = 0.02f, gX = 0.f, gY = -9.81f, density = 0.f, viscosity = 0.f, ctrl_lim = 200.f;
  __host__ __device__ static constexpr int parent(int i) { return i - 1; }
  __host__ __device__ static constexpr bool is_ancestor(int k, int i) { return k <= i; }
  __host__ __device__ static constexpr float sgn(int i) { return i == 0 ? -1.f : 1.f; }
  __host__ __device__ static constexpr float ax(int) { return 0.f; }
  __host__ __device__ static constexpr float ay(int i) { return i == 1 ? -0.2f : (i == 2 ? -0.45f : (i == 3 ? -0.5f : 0.f)); }
  __host__ __device__ static constexpr float cx(int i) { return i == 3 ? 0.065f : 0.f; }
  __host__ __device__ static constexpr float cy(int i) { return i == 1 ? -0.225f : (i == 2 ? -0.25f : 0.f); }
  __host__ __device__ static constexpr float box(int i) { return i == 3 ? 0.065f : 0.f; }
  __host__ __device__ static constexpr float boy(int i) { return i == 2 ? -0.25f : 0.f; }
  __host__ __device__ static constexpr CapsuleC cap(int i) {
    return i == 0 ? capsule_c(0.05, 0.4) : (i == 1 ? capsule_c(0.05, 0.45) : (i == 2 ? capsule_c(0.04, 0.5) : capsule_c(0.06, 0.39)));
  }
  __host__ __device__ static constexpr float lax(int i) { return i == 3 ? 1.f : 0.f; }
  __host__ __device__ static constexpr float lay(int i) { return i == 3 ? 0.f : 1.f; }
  __host__ __device__ static constexpr float armature(int k) { return k >= 3 ? 1.f : 0.f; }
  __host__ __device__ static constexpr float damping(int k) { return k >= 3 ? 1.f : 0.f; }
  __host__ __device__ static constexpr int act(int j) { return j + 1; }
  __host__ __device__ static constexpr int lim_hinge(int j) { return j + 1; }
  __host__ __device__ static constexpr float lim_lo(int j) { return j == 2 ? -45.f * PLANAR_PI / 180.f : -150.f * PLANAR_PI / 180.f; }
  __host__ __device__ static constexpr float lim_hi(int j) { return j == 2 ? 45.f * PLANAR_PI / 180.f : 0.f; }
  __host__ __device__ static constexpr float q0(int k) { return k == 0 ? 1.25f : 0.f; }
  __host__ __device__ static constexpr int con_body(int) { return 3; }
  __host__ __device__ static constexpr float con_ex(int c) { return c == 0 ? -0.13f : 0.26f; }
  __host__ __device__ static constexpr float con_ey(int) { return 0.f; }
  __host__ __device__ static constexpr float con_r(int) { return 0.06f; }
  static constexpr float mu = 2.0f, margin = 0.001f;
};

// vendor/mujoco_models/half_cheetah.xml.  Bodies: 0 torso, 1 bthigh, 2 bshin, 3 bfoot, 4 fthigh, 5 fshin, 6 ffoot;
// q = [rootx, rootz, rooty, bthigh, bshin, bfoot, fthigh, fshin, ffoot] (plane X = x, Y = z, every hinge about +y).
// Eight capsules of radius .046 (the torso body carries `torso` and `head`); body masses and inertias are summed over a
// body's capsules with the parallel-axis theorem, then scaled by settotalmass = 14 / (total geom mass).
struct CheetahGeom {
  int body;
  double hl, px, py;   // capsule half-length and centre (body frame, (x, z)); its axis lies in the plane, so Iyy = Ip
};
__host__ __device__ constexpr CheetahGeom cheetah_geom(int g) {
  return g == 0 ? CheetahGeom{0, 0.5, 0.0, 0.0} : g == 1 ? CheetahGeom{0, 0.15, 0.6, 0.1}
       : g == 2 ? CheetahGeom{1, 0.145, 0.1, -0.13} : g == 3 ? CheetahGeom{2, 0.15, -0.14, -0.07}
       : g == 4 ? CheetahGeom{3, 0.094, 0.03, -0.097} : g == 5 ? CheetahGeom{4, 0.133, -0.07, -0.12}
       : g == 6 ? CheetahGeom{5, 0.106, 0.065, -0.09} : CheetahGeom{6, 0.07, 0.045, -0.07};
}
constexpr double CHEETAH_R = 0.046;
__host__ __device__ constexpr double cheetah_geom_m(int g) {
  const double r = CHEETAH_R, L = 2 * cheetah_geom(g).hl, pi = 3.14159265358979323846;
  return 1000.0 * pi * r * r * L + 2 * 1000.0 * (2.0 / 3.0) * pi * r * r * r;
}
__host__ __device__ constexpr double cheetah_geom_Ip(int g) {
  const double r = CHEETAH_R, L = 2 * cheetah_geom(g).hl, pi = 3.14159265358979323846;
  const double mc = 1000.0 * pi * r * r * L, mh = 1000.0 * (2.0 / 3.0) * pi * r * r * r;
  return mc * (r * r / 4 + L * L / 12) + 2 * mh * (2 * r * r / 5 + L * L / 4 + 3 * L * r / 8);
}
__host__ __device__ constexpr double cheetah_mass_scale() {
  double s = 0.0;
  for (int g = 0; g < 8; ++g) s += cheetah_geom_m(g);
  return 14.0 / s;
}
// unscaled body mass, COM (axis 0: x, 1: z) and inertia about the COM
__host__ __device__ constexpr double cheetah_body_m(int b) {
  double m = 0.0;
  for (int g = 0; g < 8; ++g) m += cheetah_geom(g).body == b ? cheetah_geom_m(g) : 0.0;
  return m;
}
__host__ __device__ constexpr double cheetah_body_c(int b, int axis) {
  double s = 0.0;
  for (int g = 0; g < 8; ++g)
    s += cheetah_geom(g).body == b ? cheetah_geom_m(g) * (axis == 0 ? cheetah_geom(g).px : cheetah_geom(g).py) : 0.0;
  return s / cheetah_body_m(b);
}
__host__ __device__ constexpr double cheetah_body_I(int b) {
  double s = 0.0;
  for (int g = 0; g < 8; ++g) {
    if (cheetah_geom(g).body != b) continue;
    const double dx = cheetah_geom(g).px - cheetah_body_c(b, 0), dy = cheetah_geom(g).py - cheetah_body_c(b, 1);
    s += cheetah_geom_Ip(g) + cheetah_geom_m(g) * (dx * dx + dy * dy);
  }
  return s;
}

struct HalfCheetahModel : PlanarModelDefaults {
  static constexpr int n = 7, nv = 9, nu = 6, iX = 0, iY = 1, nlim = 6, ncon = 16;
  static constexpr bool rk4 = false, fluid = false, active_rows = true;
  static constexpr int frame_skip = 1;
  static constexpr float dt = 0.01f, gX = 0.f, gY = -9.81f, density = 0.f, viscosity = 0.f, ctrl_lim = 1.f;
  static constexpr float y0 = 0.7f;
  // limits: solreflimit (.02, 1), solimplimit (0, .8, .03);  geoms: solref (.02, 1), solimp (0, .8, .01)
  static constexpr float lim_tc = 0.02f, lim_d0 = 0.f, lim_d1 = 0.8f, lim_w = 0.03f;
  static constexpr float con_tc = 0.02f, con_d0 = 0.f, con_d1 = 0.8f, con_w = 0.01f;
  __host__ __device__ static constexpr int parent(int i) { return (i == 1 || i == 4) ? 0 : i - 1; }
  __host__ __device__ static constexpr bool is_ancestor(int k, int i) {   // torso -> back leg 1..3, front leg 4..6
    return k == i || k == 0 || (k <= i && (k >= 4) == (i >= 4));
  }
  __host__ __device__ static constexpr float sgn(int) { return -1.f; }
  __host__ __device__ static constexpr float ax(int i) {
    return i == 1 ? -0.5f : i == 2 ? 0.16f : i == 3 ? -0.28f : i == 4 ? 0.5f : i == 5 ? -0.14f : i == 6 ? 0.13f : 0.f;
  }
  __host__ __device__ static constexpr float ay(int i) {
    return i == 2 ? -0.25f : i == 3 ? -0.14f : i == 5 ? -0.24f : i == 6 ? -0.18f : 0.f;
  }
  __host__ __device__ static constexpr float cx(int i) { return (float)cheetah_body_c(i, 0); }
  __host__ __device__ static constexpr float cy(int i) { return (float)cheetah_body_c(i, 1); }
  __host__ __device__ static constexpr float box(int) { return 0.f; }   // every joint sits at its body's origin
  __host__ __device__ static constexpr float boy(int) { return 0.f; }
  __host__ __device__ static constexpr CapsuleC cap(int i) {
    return CapsuleC{(float)(cheetah_mass_scale() * cheetah_body_m(i)), (float)(cheetah_mass_scale() * cheetah_body_I(i)),
                    0.f};
  }
  __host__ __device__ static constexpr float lax(int) { return 0.f; }
  __host__ __device__ static constexpr float lay(int) { return 0.f; }
  __host__ __device__ static constexpr float armature(int k) { return k >= 3 ? 0.1f : 0.f; }
  __host__ __device__ static constexpr float damping(int k) {
    return k == 3 ? 6.f : k == 4 ? 4.5f : k == 5 ? 3.f : k == 6 ? 4.5f : k == 7 ? 3.f : k == 8 ? 1.5f : 0.f;
  }
  __host__ __device__ static constexpr float stiffness(int k) {
    return k == 3 ? 240.f : k == 4 ? 180.f : k == 5 ? 120.f : k == 6 ? 180.f : k == 7 ? 120.f : k == 8 ? 60.f : 0.f;
  }
  __host__ __device__ static constexpr float gear(int j) {
    return j == 0 ? 120.f : j == 1 ? 90.f : j == 2 ? 60.f : j == 3 ? 120.f : j == 4 ? 60.f : 30.f;
  }
  __host__ __device__ static constexpr int act(int j) { return j + 1; }
  __host__ __device__ static constexpr int lim_hinge(int j) { return j + 1; }
  __host__ __device__ static constexpr float lim_lo(int j) {
    return j == 0 ? -0.52f : j == 1 ? -0.785f : j == 2 ? -0.4f : j == 3 ? -1.f : j == 4 ? -1.2f : -0.5f;
  }
  __host__ __device__ static constexpr float lim_hi(int j) {
    return j == 0 ? 1.05f : j == 1 ? 0.785f : j == 2 ? 0.785f : j == 3 ? 0.7f : j == 4 ? 0.87f : 0.5f;
  }
  __host__ __device__ static constexpr float q0(int) { return 0.f; }
  // contact candidates: both end spheres of every capsule, centre +- hl (sin a, cos a) for axisangle (0 1 0 a), in geom
  // order (torso, head, bthigh, bshin, bfoot, fthigh, fshin, ffoot), minus end first
  __host__ __device__ static constexpr int con_body(int c) { return cheetah_geom(c / 2).body; }
  __host__ __device__ static constexpr float con_ex(int c) {
    constexpr float e[16] = {-0.5f, 0.5f, 0.48535067f, 0.7146493f, 0.011280606f, 0.18871939f, -0.005539139f,
                             -0.27446085f, 0.055072755f, 0.004927245f, -0.13608506f, -0.0039149416f, 0.1248521f,
                             0.0051478976f, 0.084524974f, 0.005475027f};
    return e[c];
  }
  __host__ __device__ static constexpr float con_ey(int c) {
    constexpr float e[16] = {0.f, 0.f, 0.003276018f, 0.19672398f, -0.015309682f, -0.24469031f, -0.0035148377f,
                             -0.13648516f, -0.18759446f, -0.0064055356f, -0.23541994f, -0.0045800493f, -0.17748557f,
                             -0.0025144247f, -0.1277735f, -0.012226507f};
    return e[c];
  }
  __host__ __device__ static constexpr float con_r(int) { return 0.046f; }
  static constexpr float mu = 0.4f, margin = 0.f;
};

static_assert(planar_topology_ok<SwimmerModel>() && planar_topology_ok<HopperModel>() &&
              planar_topology_ok<HalfCheetahModel>(), "is_ancestor must match parent");

struct PlanarKin {
  float comX, comY, comvelX;
};

// sin/cos of a body angle: two-constant Cody-Waite reduction to [-pi, pi] + MUFU.SIN/COS (abs. error ~5e-7).  The
// library sincosf carries a Payne-Hanek slow path (CALL + convergence barrier at each of the 13 call sites) that the
// bounded joint angles never need; together with the IEEE divisions it made up most of the integrator's latency.
__device__ __forceinline__ void planar_sincos(float x, float* s, float* c) {
  const float k = rintf(x * 0.15915494309189535f);
  float r = fmaf(k, -6.2831854820251465f, x);
  r = fmaf(k, 1.7484555e-7f, r);
  __sincosf(r, s, c);
}

// d(r) = d0 + (d1-d0) min(|r|/width, 1), clamped to MuJoCo's [1e-4, 0.9999] when d0 or d1 lies outside it (d0 = 0 would
// make R = (1-d)/d A infinite at r = 0).  d0, d1 are compile-time constants, so the test folds away.
__device__ __forceinline__ float planar_imp(float d0, float d1, float w, float r) {
  const float d = d0 + (d1 - d0) * fminf(fabsf(r) * (1.0f / w), 1.0f);
  return (fminf(d0, d1) < 1e-4f || fmaxf(d0, d1) > 0.9999f) ? fminf(fmaxf(d, 1e-4f), 0.9999f) : d;
}

// Body angles, angular velocities and their sin / cos down the tree: phi_i = phi_parent(i) + s_i q_hinge_i.
template <class M>
__device__ __forceinline__ void planar_angles(const float (&q)[M::nv], const float (&v)[M::nv], float (&om)[M::n],
                                              float (&cs)[M::n], float (&sn)[M::n]) {
  float ap[M::n];
#pragma unroll
  for (int i = 0; i < M::n; ++i) {
    ap[i] = (i == 0 ? 0.f : ap[M::parent(i)]) + M::sgn(i) * q[2 + i];
    om[i] = (i == 0 ? 0.f : om[M::parent(i)]) + M::sgn(i) * v[2 + i];
    planar_sincos(ap[i], &sn[i], &cs[i]);
  }
}

// Constraint solve over the active rows only (models with active_rows): HalfCheetah has 6 limit + 32 contact rows, and
// the dense (A + R) system of planar_dynamics does not fit in registers.  Active rows are compacted, in the all-rows
// order, into local-memory arrays sized for every row (nothing is dropped), and PGS runs matrix-free on them:
// sum_j A_ij f_j = J_i . w with w = M^-1 J^T f kept up to date after each row.  Inactive rows have f = 0 in the all-rows
// statement, so this is the same system and the same sweep order.
template <class M, class Solve>
__device__ __forceinline__ void planar_constraints_active(const float (&q)[M::nv], const float (&v)[M::nv],
                                                          const float (&cs)[M::n], const float (&sn)[M::n],
                                                          const float (&hx)[M::n], const float (&hy)[M::n],
                                                          const float (&tau)[M::nv], const float (&a0)[M::nv],
                                                          Solve& solve, float (&acc)[M::nv], float (&qfc)[M::nv]) {
  constexpr int nv = M::nv, NC = M::nlim + 2 * M::ncon;
  float cJ[NC][nv], cMiJ[NC][nv], crhs[NC], cR[NC], cid[NC], cf[NC];
  int cnrm[NC];   // -1: unilateral row (limit, contact normal); else the slot of the tangential row's normal
  int m = 0;
  auto push = [&](const float (&J)[nv], float aref, float d, int nrm) {
    float MiJ[nv];
    solve(J, MiJ);
    float Aii = 0.f, Ja0 = 0.f;
#pragma unroll
    for (int k = 0; k < nv; ++k) { Ja0 += J[k] * a0[k]; Aii += J[k] * MiJ[k]; }
#pragma unroll
    for (int k = 0; k < nv; ++k) { cJ[m][k] = J[k]; cMiJ[m][k] = MiJ[k]; }
    crhs[m] = aref - Ja0;
    cR[m] = (1.0f - d) / d * Aii;
    cid[m] = 1.0f / (Aii + cR[m]);
    cf[m] = 0.f;
    cnrm[m] = nrm;
    ++m;
  };
  {
    const float dmax = fmaxf(M::lim_d0, M::lim_d1), tc = M::lim_tc;
    const float bb = 2.0f / (dmax * tc), kk = 1.0f / (dmax * dmax * tc * tc);
#pragma unroll
    for (int j = 0; j < M::nlim; ++j) {
      const int hk = 2 + M::lim_hinge(j);
      const float rlo = q[hk] - M::lim_lo(j), rhi = M::lim_hi(j) - q[hk];
      const bool hi = rhi < 0.f;
      if (!(rlo < 0.f || hi)) continue;
      const float sg = hi ? -1.f : 1.f, r_ = hi ? rhi : rlo;
      float J[nv];
#pragma unroll
      for (int k = 0; k < nv; ++k) J[k] = 0.f;
      J[hk] = sg;
      const float d = planar_imp(M::lim_d0, M::lim_d1, M::lim_w, r_);
      push(J, -bb * (sg * v[hk]) - kk * d * r_, d, -1);
    }
  }
  {
    const float dmax = fmaxf(M::con_d0, M::con_d1), tc = M::con_tc;
    const float bb = 2.0f / (dmax * tc), kk = 1.0f / (dmax * dmax * tc * tc);
#pragma unroll
    for (int c = 0; c < M::ncon; ++c) {
      const int bi = M::con_body(c);
      const float ex = cs[bi] * M::con_ex(c) - sn[bi] * M::con_ey(c), ey = sn[bi] * M::con_ex(c) + cs[bi] * M::con_ey(c);
      const float sx = hx[bi] + ex, sy = hy[bi] + ey;
      const float r_ = sy - M::con_r(c) - M::margin;
      if (!(r_ < 0.f)) continue;
      const float ptx = sx, pty = sy - M::con_r(c);
      float Jn[nv], Jt[nv];
#pragma unroll
      for (int k = 0; k < nv; ++k) { Jn[k] = 0.f; Jt[k] = 0.f; }
      Jt[M::iX] = 1.f; Jn[M::iY] = 1.f;
#pragma unroll
      for (int k = 0; k <= bi; ++k) {
        if (!M::is_ancestor(k, bi)) continue;
        Jt[2 + k] = -M::sgn(k) * (pty - hy[k]);
        Jn[2 + k] = M::sgn(k) * (ptx - hx[k]);
      }
      const float d = planar_imp(M::con_d0, M::con_d1, M::con_w, r_);
      float vn = 0.f, vt = 0.f;
#pragma unroll
      for (int k = 0; k < nv; ++k) { vn += Jn[k] * v[k]; vt += Jt[k] * v[k]; }
      push(Jn, -bb * vn - kk * d * r_, d, -1);
      push(Jt, -bb * vt, d, m - 1);
    }
  }
#pragma unroll
  for (int k = 0; k < nv; ++k) qfc[k] = 0.f;
  if (m == 0) {
#pragma unroll
    for (int k = 0; k < nv; ++k) acc[k] = a0[k];
    return;
  }
  float w[nv];
#pragma unroll
  for (int k = 0; k < nv; ++k) w[k] = 0.f;
#pragma unroll 1
  for (int sweep = 0; sweep < PLANAR_PGS_SWEEPS; ++sweep) {
#pragma unroll 1
    for (int i = 0; i < m; ++i) {
      float s = crhs[i] - cR[i] * cf[i];
#pragma unroll
      for (int k = 0; k < nv; ++k) s -= cJ[i][k] * w[k];
      float fi = cf[i] + s * cid[i];
      if (cnrm[i] < 0) fi = fmaxf(fi, 0.f);
      else {
        const float lim = M::mu * cf[cnrm[i]];
        fi = fminf(fmaxf(fi, -lim), lim);
      }
      const float df = fi - cf[i];
#pragma unroll
      for (int k = 0; k < nv; ++k) w[k] = fmaf(cMiJ[i][k], df, w[k]);
      cf[i] = fi;
    }
  }
  float tot[nv];
#pragma unroll 1
  for (int i = 0; i < m; ++i) {
#pragma unroll
    for (int k = 0; k < nv; ++k) qfc[k] += cJ[i][k] * cf[i];
  }
#pragma unroll
  for (int k = 0; k < nv; ++k) tot[k] = tau[k] + qfc[k];
  solve(tot, acc);
}

// qacc, qfrc_constraint and COM quantities at (q, v, ctrl).
template <class M>
__device__ __forceinline__ void planar_dynamics(const float (&q)[M::nv], const float (&v)[M::nv], const float (&ctrl)[M::nu],
                                             float (&acc)[M::nv], float (&qfc)[M::nv], PlanarKin& kin) {
  constexpr int n = M::n, nv = M::nv;
  // ---- kinematics
  float om[n], cs[n], sn[n];
  planar_angles<M>(q, v, om, cs, sn);
  float hx[n], hy[n], hdx[n], hdy[n], hddx[n], hddy[n];
  hx[0] = q[M::iX]; hy[0] = M::y0 == 0.f ? q[M::iY] : q[M::iY] + M::y0;
  hdx[0] = v[M::iX]; hdy[0] = v[M::iY]; hddx[0] = 0.f; hddy[0] = 0.f;
#pragma unroll
  for (int i = 1; i < n; ++i) {
    const int p = M::parent(i);
    const float rax = cs[p] * M::ax(i) - sn[p] * M::ay(i), ray = sn[p] * M::ax(i) + cs[p] * M::ay(i);
    hx[i] = hx[p] + rax; hy[i] = hy[p] + ray;
    hdx[i] = hdx[p] - om[p] * ray; hdy[i] = hdy[p] + om[p] * rax;
    const float w2 = om[p] * om[p];
    hddx[i] = hddx[p] - w2 * rax; hddy[i] = hddy[p] - w2 * ray;
  }
  // ---- mass matrix (upper), generalised forces
  float Mm[nv][nv], tau[nv];
#pragma unroll
  for (int r = 0; r < nv; ++r) {
    tau[r] = 0.f;
#pragma unroll
    for (int c = 0; c < nv; ++c) Mm[r][c] = 0.f;
  }
  float mt = 0.f, comX = 0.f, comY = 0.f, cvX = 0.f;
#pragma unroll
  for (int i = 0; i < n; ++i) {
    const CapsuleC cp = M::cap(i);
    const float rcx = cs[i] * M::cx(i) - sn[i] * M::cy(i), rcy = sn[i] * M::cx(i) + cs[i] * M::cy(i);
    const float px = hx[i] + rcx, py = hy[i] + rcy;
    const float pdx = hdx[i] - om[i] * rcy, pdy = hdy[i] + om[i] * rcx;
    const float w2 = om[i] * om[i];
    const float pddx = hddx[i] - w2 * rcx, pddy = hddy[i] - w2 * rcy;
    float JX[nv], JY[nv], wv[nv];
#pragma unroll
    for (int k = 0; k < nv; ++k) { JX[k] = 0.f; JY[k] = 0.f; wv[k] = 0.f; }
    JX[M::iX] = 1.f; JY[M::iY] = 1.f;
#pragma unroll
    for (int k = 0; k <= i; ++k) {   // ancestors precede their descendants
      if (!M::is_ancestor(k, i)) continue;
      JX[2 + k] = -M::sgn(k) * (py - hy[k]);
      JY[2 + k] = M::sgn(k) * (px - hx[k]);
      wv[2 + k] = M::sgn(k);
    }
    float fX = cp.m * M::gX - cp.m * pddx, fY = cp.m * M::gY - cp.m * pddy, tq = 0.f;
    if (M::fluid) {
      const float lX = cs[i] * M::lax(i) - sn[i] * M::lay(i), lY = sn[i] * M::lax(i) + cs[i] * M::lay(i);
      const float vl = pdx * lX + pdy * lY, vp = -pdx * lY + pdy * lX;
      const float bl = sqrtf(6.0f * (2.f * cp.Ip - cp.Ia) / cp.m), bp = sqrtf(6.0f * cp.Ia / cp.m);
      const float diam = (bl + 2.f * bp) / 3.0f;
      const float Fl = -0.5f * M::density * bp * bp * fabsf(vl) * vl - 3.f * PLANAR_PI * M::viscosity * diam * vl;
      const float Fp = -0.5f * M::density * bl * bp * fabsf(vp) * vp - 3.f * PLANAR_PI * M::viscosity * diam * vp;
      fX += Fl * lX - Fp * lY;
      fY += Fl * lY + Fp * lX;
      const float bl2 = bl * bl, bp2 = bp * bp;
      tq = -M::density * bp * (bl2 * bl2 + bp2 * bp2) / 64.0f * fabsf(om[i]) * om[i] -
           PLANAR_PI * M::viscosity * diam * diam * diam * om[i];
    }
#pragma unroll
    for (int r = 0; r < nv; ++r) {
      tau[r] += JX[r] * fX + JY[r] * fY + wv[r] * tq;
#pragma unroll
      for (int c = r; c < nv; ++c) Mm[r][c] += cp.m * (JX[r] * JX[c] + JY[r] * JY[c]) + cp.Ip * wv[r] * wv[c];
    }
    mt += cp.m; comX += cp.m * px; comY += cp.m * py;
    const float rox = cs[i] * M::box(i) - sn[i] * M::boy(i);
    const float roy = sn[i] * M::box(i) + cs[i] * M::boy(i);
    (void)rox;
    cvX += cp.m * (hdx[i] - om[i] * roy);
  }
  { const float imt = 1.0f / mt; kin.comX = comX * imt; kin.comY = comY * imt; kin.comvelX = cvX * imt; }
#pragma unroll
  for (int r = 0; r < nv; ++r) {
    Mm[r][r] += M::armature(r);
    tau[r] -= M::damping(r) * v[r];
    if (M::stiffness(r) != 0.f) tau[r] -= M::stiffness(r) * q[r];
  }
#pragma unroll
  for (int j = 0; j < M::nu; ++j) tau[2 + M::act(j)] += M::gear(j) * fminf(fmaxf(ctrl[j], -M::ctrl_lim), M::ctrl_lim);
  // ---- Cholesky (lower factor stored in the lower triangle of Mm)
  float idg[nv];
#pragma unroll
  for (int r = 0; r < nv; ++r) {
#pragma unroll
    for (int c = 0; c <= r; ++c) {
      float s = Mm[c][r];  // upper entry (c <= r)
#pragma unroll
      for (int k = 0; k < c; ++k) s -= Mm[r][k] * Mm[c][k];
      // reciprocal diagonal (MUFU.RSQ) kept in idg[]: every later division by L[r][r] becomes a multiply -- an IEEE
      // float division is ~10 instructions + a slow-path CALL, and the Cholesky / triangular solves had ~40 of them per call
      if (c == r) { idg[r] = rsqrtf(s); Mm[r][r] = s * idg[r]; }
      else Mm[r][c] = s * idg[c];
    }
  }
  auto solve = [&](const float (&b)[nv], float (&x)[nv]) {
    float y[nv];
#pragma unroll
    for (int r = 0; r < nv; ++r) {
      float s = b[r];
#pragma unroll
      for (int k = 0; k < r; ++k) s -= Mm[r][k] * y[k];
      y[r] = s * idg[r];
    }
#pragma unroll
    for (int r = nv - 1; r >= 0; --r) {
      float s = y[r];
#pragma unroll
      for (int k = r + 1; k < nv; ++k) s -= Mm[k][r] * x[k];
      x[r] = s * idg[r];
    }
  };
  float a0[nv];
  solve(tau, a0);
#pragma unroll
  for (int k = 0; k < nv; ++k) qfc[k] = 0.f;

  // ---- constraints
  if constexpr (M::active_rows) {
    planar_constraints_active<M>(q, v, cs, sn, hx, hy, tau, a0, solve, acc, qfc);
    return;
  }
  constexpr int NC = M::nlim + 2 * M::ncon;
  float J[NC][nv], aref[NC], dimp[NC];
  bool active[NC];
  bool any = false;
  {
    const float dmax = fmaxf(M::lim_d0, M::lim_d1), tc = M::lim_tc;
    const float bb = 2.0f / (dmax * tc), kk = 1.0f / (dmax * dmax * tc * tc);
#pragma unroll
    for (int j = 0; j < M::nlim; ++j) {
      const int hk = 2 + M::lim_hinge(j);
      const float rlo = q[hk] - M::lim_lo(j), rhi = M::lim_hi(j) - q[hk];
      const bool lo = rlo < 0.f, hi = rhi < 0.f;
      const float sg = hi ? -1.f : 1.f;
      const float r_ = hi ? rhi : rlo;
#pragma unroll
      for (int k = 0; k < nv; ++k) J[j][k] = 0.f;
      J[j][hk] = sg;
      dimp[j] = planar_imp(M::lim_d0, M::lim_d1, M::lim_w, r_);
      aref[j] = -bb * (sg * v[hk]) - kk * dimp[j] * r_;
      active[j] = lo || hi;
      any = any || active[j];
    }
  }
  if (M::ncon > 0) {
    const float dmax = fmaxf(M::con_d0, M::con_d1), tc = M::con_tc;
    const float bb = 2.0f / (dmax * tc), kk = 1.0f / (dmax * dmax * tc * tc);
#pragma unroll
    for (int c = 0; c < M::ncon; ++c) {
      const int bi = M::con_body(c);
      const float ex = cs[bi] * M::con_ex(c) - sn[bi] * M::con_ey(c), ey = sn[bi] * M::con_ex(c) + cs[bi] * M::con_ey(c);
      const float sx = hx[bi] + ex, sy = hy[bi] + ey;
      const float dist = sy - M::con_r(c);
      const float ptx = sx, pty = sy - M::con_r(c);
      const int rn = M::nlim + 2 * c, rt = rn + 1;
#pragma unroll
      for (int k = 0; k < nv; ++k) { J[rn][k] = 0.f; J[rt][k] = 0.f; }
      J[rt][M::iX] = 1.f; J[rn][M::iY] = 1.f;
#pragma unroll
      for (int k = 0; k <= bi; ++k) {
        if (!M::is_ancestor(k, bi)) continue;
        J[rt][2 + k] = -M::sgn(k) * (pty - hy[k]);
        J[rn][2 + k] = M::sgn(k) * (ptx - hx[k]);
      }
      const float r_ = dist - M::margin;
      const float d = planar_imp(M::con_d0, M::con_d1, M::con_w, r_);
      float vn = 0.f, vt = 0.f;
#pragma unroll
      for (int k = 0; k < nv; ++k) { vn += J[rn][k] * v[k]; vt += J[rt][k] * v[k]; }
      dimp[rn] = d; dimp[rt] = d;
      aref[rn] = -bb * vn - kk * d * r_;
      aref[rt] = -bb * vt;
      active[rn] = active[rt] = (r_ < 0.f);
      any = any || active[rn];
    }
  }
  if (!any) {
#pragma unroll
    for (int k = 0; k < nv; ++k) acc[k] = a0[k];
    return;
  }
  float MiJ[NC][nv], A[NC][NC], rhs[NC], Rr[NC], f[NC], iden[NC];
#pragma unroll
  for (int i = 0; i < NC; ++i) solve(J[i], MiJ[i]);
#pragma unroll
  for (int i = 0; i < NC; ++i) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < nv; ++k) s += J[i][k] * a0[k];
    rhs[i] = aref[i] - s;
#pragma unroll
    for (int j = 0; j < NC; ++j) {
      float t = 0.f;
#pragma unroll
      for (int k = 0; k < nv; ++k) t += J[i][k] * MiJ[j][k];
      A[i][j] = t;
    }
    Rr[i] = (1.0f - dimp[i]) / dimp[i] * A[i][i];
    iden[i] = 1.0f / (A[i][i] + Rr[i]);   // hoisted out of the PGS sweeps
    f[i] = 0.f;
  }
  for (int sweep = 0; sweep < PLANAR_PGS_SWEEPS; ++sweep) {
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      float s = rhs[i] - Rr[i] * f[i];
#pragma unroll
      for (int j = 0; j < NC; ++j) s -= A[i][j] * f[j];
      float fi = f[i] + s * iden[i];
      const bool tangential = (i >= M::nlim) && (((i - M::nlim) & 1) == 1);
      if (!tangential) fi = fmaxf(fi, 0.f);
      else {
        const float lim = M::mu * f[i - 1];
        fi = fminf(fmaxf(fi, -lim), lim);
      }
      f[i] = active[i] ? fi : 0.f;
    }
  }
  float tot[nv];
#pragma unroll
  for (int k = 0; k < nv; ++k) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NC; ++i) s += J[i][k] * f[i];
    qfc[k] = s;
    tot[k] = tau[k] + s;
  }
  solve(tot, acc);
}

// Subtree COM position and the reference's body-origin "COM velocity" only (no dynamics): what obs / reward need.
template <class M>
__device__ __forceinline__ void planar_kin(const float (&q)[M::nv], const float (&v)[M::nv], PlanarKin& kin) {
  constexpr int n = M::n;
  float om[n], cs[n], sn[n];
  planar_angles<M>(q, v, om, cs, sn);
  // (hx, hy, hdx, hdy): hinge of the current body; the arrays keep every hinge for the children of a branching body
  float hx = q[M::iX], hy = M::y0 == 0.f ? q[M::iY] : q[M::iY] + M::y0, hdx = v[M::iX], hdy = v[M::iY];
  float hxs[n], hys[n], hdxs[n], hdys[n];
  float mt = 0.f, comX = 0.f, comY = 0.f, cvX = 0.f;
#pragma unroll
  for (int i = 0; i < n; ++i) {
    if (i > 0) {
      const int p = M::parent(i);
      if (p != i - 1) { hx = hxs[p]; hy = hys[p]; hdx = hdxs[p]; hdy = hdys[p]; }
      const float rax = cs[p] * M::ax(i) - sn[p] * M::ay(i), ray = sn[p] * M::ax(i) + cs[p] * M::ay(i);
      hx += rax; hy += ray;
      hdx -= om[p] * ray; hdy += om[p] * rax;
    }
    hxs[i] = hx; hys[i] = hy; hdxs[i] = hdx; hdys[i] = hdy;
    const CapsuleC cp = M::cap(i);
    const float rcx = cs[i] * M::cx(i) - sn[i] * M::cy(i), rcy = sn[i] * M::cx(i) + cs[i] * M::cy(i);
    const float roy = sn[i] * M::box(i) + cs[i] * M::boy(i);
    mt += cp.m; comX += cp.m * (hx + rcx); comY += cp.m * (hy + rcy);
    cvX += cp.m * (hdx - om[i] * roy);
  }
  { const float imt = 1.0f / mt; kin.comX = comX * imt; kin.comY = comY * imt; kin.comvelX = cvX * imt; }
}

// frame_skip x (semi-implicit Euler | RK4).  RK4 is written as a 4-stage loop so that the (inlined) dynamics has a
// single call site: y' = y + h * sum_s b_s k_s, stage state y_s = y + a_s h k_{s-1}, a = (0, 1/2, 1/2, 1), b = (1,2,2,1)/6.
template <class M>
__device__ __forceinline__ void planar_integrate(float (&q)[M::nv], float (&v)[M::nv], const float (&ctrl)[M::nu]) {
  constexpr int nv = M::nv;
  const float h = M::dt;
  float a[nv], qf[nv];
  PlanarKin kin;
  if (!M::rk4) {
#pragma unroll 1
    for (int s = 0; s < M::frame_skip; ++s) {
      planar_dynamics<M>(q, v, ctrl, a, qf, kin);
#pragma unroll
      for (int k = 0; k < nv; ++k) { v[k] += h * a[k]; q[k] += h * v[k]; }
    }
  } else {
#pragma unroll 1
    for (int s = 0; s < M::frame_skip; ++s) {
      float qs[nv], vs[nv], sq[nv], sv_[nv];
#pragma unroll
      for (int k = 0; k < nv; ++k) { qs[k] = q[k]; vs[k] = v[k]; sq[k] = 0.f; sv_[k] = 0.f; }
#pragma unroll 1
      for (int st = 0; st < 4; ++st) {
        planar_dynamics<M>(qs, vs, ctrl, a, qf, kin);
        const float b = (st == 0 || st == 3) ? (1.0f / 6.0f) : (1.0f / 3.0f);
        const float an = (st == 2) ? 1.0f : 0.5f;   // coefficient of the NEXT stage
#pragma unroll
        for (int k = 0; k < nv; ++k) {
          sq[k] += b * vs[k];
          sv_[k] += b * a[k];
          const float nq = q[k] + an * h * vs[k], nvv = v[k] + an * h * a[k];
          qs[k] = nq; vs[k] = nvv;
        }
      }
#pragma unroll
      for (int k = 0; k < nv; ++k) { q[k] += h * sq[k]; v[k] += h * sv_[k]; }
    }
  }
}

// ---------------------------------------------------------------- rllab/envs/mujoco/swimmer_env.py:10-45
struct SwimmerEnvD {
  using M = SwimmerModel;
  static constexpr int KIND = B200RL_ENV_SWIMMER, O = 13, A = 2, S = 10, K = 10, NOISE = B200RL_NOISE_NORMAL;
  __host__ __device__ static constexpr float lb(int) { return -50.0f; }
  __host__ __device__ static constexpr float ub(int) { return 50.0f; }
  __device__ static void reset(float (&s)[S], const float (&raw)[K]) {
#pragma unroll
    for (int k = 0; k < 5; ++k) { s[k] = M::q0(k) + 0.01f * raw[k]; s[5 + k] = 0.1f * raw[5 + k]; }
  }
  __device__ static void obs(const float (&s)[S], float (&o)[O]) {
    float q[5], v[5];
    PlanarKin kin;
#pragma unroll
    for (int k = 0; k < 5; ++k) { q[k] = s[k]; v[k] = s[5 + k]; }
    planar_kin<M>(q, v, kin);
#pragma unroll
    for (int k = 0; k < 10; ++k) o[k] = s[k];
    o[10] = kin.comX; o[11] = kin.comY; o[12] = 0.f;
  }
  __device__ static void step(float (&s)[S], const float (&u)[A], float& r, bool& done) {
    float q[5], v[5];
    PlanarKin kin;
#pragma unroll
    for (int k = 0; k < 5; ++k) { q[k] = s[k]; v[k] = s[5 + k]; }
    planar_integrate<M>(q, v, u);
    planar_kin<M>(q, v, kin);
    const float c0 = u[0] / 50.0f, c1 = u[1] / 50.0f;
    r = kin.comvelX - 0.5f * 1e-2f * (c0 * c0 + c1 * c1);
#pragma unroll
    for (int k = 0; k < 5; ++k) { s[k] = q[k]; s[5 + k] = v[k]; }
    done = false;
  }
};

// ---------------------------------------------------------------- rllab/envs/mujoco/hopper_env.py:19-61
// state = [qpos 6, qvel 6, ctrl 3, qfrc_constraint 6, comX, comY]: the last 8 entries cache what mj_forward leaves in
// mjData after the step (mujoco_env.py:184-191) so that get_current_obs needs no second dynamics evaluation.
struct HopperEnvD {
  using M = HopperModel;
  static constexpr int KIND = B200RL_ENV_HOPPER, O = 20, A = 3, S = 23, K = 12, NOISE = B200RL_NOISE_NORMAL;
  __host__ __device__ static constexpr float lb(int) { return -200.0f; }
  __host__ __device__ static constexpr float ub(int) { return 200.0f; }
  __device__ __noinline__ static void forward_cache(float (&s)[S]) {   // mj_forward at the current (q, v, ctrl)
    float q[6], v[6], a[6], qf[6], c[3];
    PlanarKin kin;
#pragma unroll
    for (int k = 0; k < 6; ++k) { q[k] = s[k]; v[k] = s[6 + k]; }
    c[0] = s[12]; c[1] = s[13]; c[2] = s[14];
    planar_dynamics<M>(q, v, c, a, qf, kin);
#pragma unroll
    for (int k = 0; k < 6; ++k) s[15 + k] = qf[k];
    s[21] = kin.comX; s[22] = kin.comY;
  }
  __device__ static void reset(float (&s)[S], const float (&raw)[K]) {
#pragma unroll
    for (int k = 0; k < 6; ++k) { s[k] = M::q0(k) + 0.01f * raw[k]; s[6 + k] = 0.1f * raw[6 + k]; }
    s[12] = s[13] = s[14] = 0.f;
    forward_cache(s);
  }
  __device__ static void obs(const float (&s)[S], float (&o)[O]) {
    o[0] = s[0];
#pragma unroll
    for (int k = 0; k < 4; ++k) o[1 + k] = s[2 + k];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      o[5 + k] = fminf(fmaxf(s[6 + k], -10.f), 10.f);
      o[11 + k] = fminf(fmaxf(s[15 + k], -10.f), 10.f);
    }
    o[17] = s[21]; o[18] = 0.f; o[19] = s[22];
  }
  __device__ static void step(float (&s)[S], const float (&u)[A], float& r, bool& done) {
    float q[6], v[6], a[6], qf[6];
    PlanarKin kin;
#pragma unroll
    for (int k = 0; k < 6; ++k) { q[k] = s[k]; v[k] = s[6 + k]; }
    planar_integrate<M>(q, v, u);
    planar_dynamics<M>(q, v, u, a, qf, kin);
    float cost = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) { const float c = u[k] / 200.0f; cost += c * c; }
    r = kin.comvelX + 1.0f - 0.5f * 0.01f * cost;
    bool ok = (q[0] > 0.7f) && (fabsf(q[2]) < 0.2f);
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      ok = ok && isfinite(q[k]) && isfinite(v[k]) && (fabsf(v[k]) < 100.f);
      if (k >= 3) ok = ok && (fabsf(q[k]) < 100.f);
    }
    done = !ok;
#pragma unroll
    for (int k = 0; k < 6; ++k) { s[k] = q[k]; s[6 + k] = v[k]; s[15 + k] = qf[k]; }
    s[12] = u[0]; s[13] = u[1]; s[14] = u[2];
    s[21] = kin.comX; s[22] = kin.comY;
  }
};

// ---------------------------------------------------------------- rllab/envs/mujoco/half_cheetah_env.py:14-48
// state = [qpos 9, qvel 9]; obs = [qpos[1:], qvel, torso subtree COM (x, 0, z)] (mujoco_env.py:184-191 leaves mjData at
// the post-step state, so obs needs positions only); reward = torso subtree "COM velocity" x (body-origin velocities,
// mjcore.py:58-81) - 0.05 sum clip(a, -1, 1)^2; never done.
struct HalfCheetahEnvD {
  using M = HalfCheetahModel;
  static constexpr int KIND = B200RL_ENV_HALF_CHEETAH, O = 20, A = 6, S = 18, K = 18, NOISE = B200RL_NOISE_NORMAL;
  __host__ __device__ static constexpr float lb(int) { return -1.0f; }
  __host__ __device__ static constexpr float ub(int) { return 1.0f; }
  __device__ static void reset(float (&s)[S], const float (&raw)[K]) {
#pragma unroll
    for (int k = 0; k < 9; ++k) { s[k] = M::q0(k) + 0.01f * raw[k]; s[9 + k] = 0.1f * raw[9 + k]; }
  }
  __device__ static void obs(const float (&s)[S], float (&o)[O]) {
    float q[9], v[9];
    PlanarKin kin;
#pragma unroll
    for (int k = 0; k < 9; ++k) { q[k] = s[k]; v[k] = s[9 + k]; }
    planar_kin<M>(q, v, kin);
#pragma unroll
    for (int k = 0; k < 17; ++k) o[k] = s[1 + k];
    o[17] = kin.comX; o[18] = 0.f; o[19] = kin.comY;
  }
  __device__ static void step(float (&s)[S], const float (&u)[A], float& r, bool& done) {
    float q[9], v[9];
    PlanarKin kin;
#pragma unroll
    for (int k = 0; k < 9; ++k) { q[k] = s[k]; v[k] = s[9 + k]; }
    planar_integrate<M>(q, v, u);
    planar_kin<M>(q, v, kin);
    float cost = 0.f;
#pragma unroll
    for (int k = 0; k < A; ++k) { const float c = fminf(fmaxf(u[k], -1.f), 1.f); cost += c * c; }
    r = kin.comvelX - 0.05f * cost;
#pragma unroll
    for (int k = 0; k < 9; ++k) { s[k] = q[k]; s[9 + k] = v[k]; }
    done = false;
  }
};

}  // namespace b200rl
