"""Float64 oracle of the planar kinematic tree and of rllab's HalfCheetahEnv (TEST INFRASTRUCTURE ONLY).

Restates oracle/planar.py's serial-chain statement for a tree: body i hangs from parent[i] < i, its angle is
phi_i = phi_parent + s_i q_hinge_i, and the Jacobian of a point on body b has a column for every ancestor of b.  On a
serial model (parent[i] = i - 1, no new terms) `dynamics` performs the same float64 operations as
oracle.planar.dynamics, which tests/test_half_cheetah.py checks bit for bit on Hopper.

Terms added for HalfCheetah (each defaults to the serial models' behaviour):
  * y0: world height of the root body at rootz = 0 (the torso sits at z = 0.7);
  * stiffness: a joint spring to qpos0 = 0;  gear: torque = gear * clip(ctrl, -ctrl_lim, ctrl_lim);
  * the solimp impedance is clamped to [1e-4, 0.9999], as MuJoCo does (solimp d0 = 0 would make R infinite at r = 0);
  * per-model limit and contact solref / solimp.

References: rllab/envs/mujoco/half_cheetah_env.py:14-48, mujoco_env.py:109-132,184-191 (reset: qpos + 0.01 N,
qvel + 0.1 N; step: frame_skip x mj_step, then mj_forward), mujoco_py/mjcore.py:58-81 (subtree "COM velocity" from
body-origin velocities), vendor/mujoco_models/half_cheetah.xml.  PARITY UNPINNED: the arithmetic of the closed MuJoCo
1.31 binary is absent (SURVEY 8c).
"""
import numpy as np

from oracle.envs import LaneEnv
from oracle.planar import PGS_SWEEPS, _kb, _rot, capsule, hopper_model, swimmer_model

# --------------------------------------------------------------------------- HalfCheetah model, from the XML values
CHEETAH_R = 0.046
# geom: (body, half-length, centre (x, z) in the body frame, axis angle about +y: the capsule axis is (sin a, cos a));
# the torso capsule is fromto (-.5 0 0) (.5 0 0): centre 0, half-length .5, axis +x (a = pi/2)
CHEETAH_GEOMS = [
    ("torso", 0, 0.5, (0.0, 0.0), np.pi / 2),
    ("head", 0, 0.15, (0.6, 0.1), 0.87),
    ("bthigh", 1, 0.145, (0.1, -0.13), -3.8),
    ("bshin", 2, 0.15, (-0.14, -0.07), -2.03),
    ("bfoot", 3, 0.094, (0.03, -0.097), -0.27),
    ("fthigh", 4, 0.133, (-0.07, -0.12), 0.52),
    ("fshin", 5, 0.106, (0.065, -0.09), -0.6),
    ("ffoot", 6, 0.07, (0.045, -0.07), -0.6),
]


def composite_bodies(geoms, n, r, total_mass):
    """Per-body mass, COM and inertia about the COM (perpendicular to the plane) of capsules summed with the
    parallel-axis theorem, every mass and inertia scaled so that the geoms weigh `total_mass` (settotalmass)."""
    gm = [capsule(r, 2 * hl) for _, _, hl, _, _ in geoms]
    scale = total_mass / sum(m for m, _, _ in gm)
    mass, com, inertia = [], [], []
    for b in range(n):
        idx = [k for k, g in enumerate(geoms) if g[1] == b]
        m = sum(gm[k][0] for k in idx)
        c = (sum(gm[k][0] * geoms[k][3][0] for k in idx) / m, sum(gm[k][0] * geoms[k][3][1] for k in idx) / m)
        I = sum(gm[k][1] + gm[k][0] * ((geoms[k][3][0] - c[0]) ** 2 + (geoms[k][3][1] - c[1]) ** 2) for k in idx)
        mass.append(scale * m)
        com.append(c)
        inertia.append(scale * I)
    return mass, com, inertia


def half_cheetah_model():
    m = _Model()
    m.name = "half_cheetah"
    m.n = 7                                   # torso, bthigh, bshin, bfoot, fthigh, fshin, ffoot
    m.parent = [-1, 0, 1, 2, 0, 4, 5]
    m.iX, m.iY = 0, 1                         # q = [rootx, rootz, rooty, bthigh, bshin, bfoot, fthigh, fshin, ffoot]
    m.y0 = 0.7
    m.sgn = [-1.0] * 7                        # every hinge about +y: clockwise in the (x, z) plane
    m.a = [(0.0, 0.0), (-0.5, 0.0), (0.16, -0.25), (-0.28, -0.14), (0.5, 0.0), (-0.14, -0.24), (0.13, -0.18)]
    m.mass, m.c, m.Ip = composite_bodies(CHEETAH_GEOMS, 7, CHEETAH_R, 14.0)
    m.Ia = [0.0] * 7
    m.bo = [(0.0, 0.0)] * 7                   # every joint sits at its body's origin
    m.long_axis = [(1.0, 0.0)] * 7            # unused: no fluid
    m.armature = [0.0] * 3 + [0.1] * 6
    m.damping = [0.0, 0.0, 0.0, 6.0, 4.5, 3.0, 4.5, 3.0, 1.5]
    m.stiffness = [0.0, 0.0, 0.0, 240.0, 180.0, 120.0, 180.0, 120.0, 60.0]
    m.gravity = (0.0, -9.81)
    m.density, m.viscosity = 0.0, 0.0
    m.act = [1, 2, 3, 4, 5, 6]
    m.gear = [120.0, 90.0, 60.0, 120.0, 60.0, 30.0]
    m.ctrl_lim = 1.0
    m.limits = [None, (-0.52, 1.05), (-0.785, 0.785), (-0.4, 0.785), (-1.0, 0.7), (-1.2, 0.87), (-0.5, 0.5)]
    m.lim_solref, m.lim_solimp = (0.02, 1.0), (0.0, 0.8, 0.03)
    # both end spheres of every capsule, each against the plane z = 0 (contype 1, conaffinity 0: no geom pairs)
    m.contacts = []
    for _, body, hl, (px, pz), ang in CHEETAH_GEOMS:
        ax = (np.sin(ang), np.cos(ang))
        for s in (-1.0, 1.0):
            m.contacts.append(dict(body=body, e=(px + s * hl * ax[0], pz + s * hl * ax[1]), r=CHEETAH_R))
    m.mu, m.margin = 0.4, 0.0
    m.con_solref, m.con_solimp = (0.02, 1.0), (0.0, 0.8, 0.01)
    m.dt, m.frame_skip, m.rk4 = 0.01, 1, False
    m.q0 = [0.0] * 9
    return m


class _Model(object):
    pass


def tree_model(m):
    """Fill the tree attributes of a serial oracle.planar model with their serial defaults."""
    if not hasattr(m, "parent"):
        m.parent = [i - 1 for i in range(m.n)]
    for k, v in (("y0", 0.0), ("stiffness", [0.0] * (m.n + 2)), ("gear", [1.0] * len(m.act))):
        if not hasattr(m, k):
            setattr(m, k, v)
    return m


def ancestors(m, i):
    """Ancestors of body i and i itself, in ascending order."""
    out = []
    while i >= 0:
        out.append(i)
        i = m.parent[i]
    return sorted(out)


def _impedance(solimp, r):
    d0, d1, w = solimp
    x = np.minimum(np.abs(r) / w, 1.0)
    d = d0 + (d1 - d0) * x
    return np.clip(d, 1e-4, 0.9999) if min(d0, d1) < 1e-4 or max(d0, d1) > 0.9999 else d


def kinematics(m, q, v, dt=np.float64):
    """Body angles, angular velocities, sin/cos, hinge positions / velocities / centripetal accelerations."""
    n = m.n
    z = np.zeros(q[0].shape[0], dt)
    phi, om = [], []
    for i in range(n):
        p = m.parent[i]
        phi.append((z if p < 0 else phi[p]) + dt(m.sgn[i]) * q[2 + i])
        om.append((z if p < 0 else om[p]) + dt(m.sgn[i]) * v[2 + i])
    cs = [np.cos(x) for x in phi]
    sn = [np.sin(x) for x in phi]
    hy0 = q[m.iY] if m.y0 == 0.0 else q[m.iY] + dt(m.y0)
    h, hd, hdd = [(q[m.iX], hy0)], [(v[m.iX], v[m.iY])], [(z, z)]
    for i in range(1, n):
        p = m.parent[i]
        ra = _rot(cs[p], sn[p], (dt(m.a[i][0]), dt(m.a[i][1])))
        h.append((h[p][0] + ra[0], h[p][1] + ra[1]))
        hd.append((hd[p][0] - om[p] * ra[1], hd[p][1] + om[p] * ra[0]))
        w2 = om[p] * om[p]
        hdd.append((hdd[p][0] - w2 * ra[0], hdd[p][1] - w2 * ra[1]))
    return om, cs, sn, h, hd, hdd


def subtree_com(m, q, v, dt=np.float64):
    """Whole-tree COM and the reference's body-origin "COM velocity" (mjcore.py:58-81), without dynamics."""
    m = tree_model(m)
    om, cs, sn, h, hd, _ = kinematics(m, q, v, dt)
    mt = sum(m.mass)
    comX, comY, cvX = 0.0, 0.0, 0.0
    for i in range(m.n):
        rc = _rot(cs[i], sn[i], (dt(m.c[i][0]), dt(m.c[i][1])))
        ro = _rot(cs[i], sn[i], (dt(m.bo[i][0]), dt(m.bo[i][1])))
        comX = comX + dt(m.mass[i]) * (h[i][0] + rc[0])
        comY = comY + dt(m.mass[i]) * (h[i][1] + rc[1])
        cvX = cvX + dt(m.mass[i]) * (hd[i][0] - om[i] * ro[1])
    return dict(comX=comX / dt(mt), comY=comY / dt(mt), comvelX=cvX / dt(mt))


def constraint_residuals(m, q, dt=np.float64):
    """(rows, N) constraint residuals r at positions q: both sides of every limit, then every contact candidate's
    gap minus margin.  A row is active where r < 0; lanes with some |r| within float32 rounding of 0 may take a
    different active set in float32."""
    m = tree_model(m)
    _, cs, sn, h, _, _ = kinematics(m, q, np.zeros_like(np.asarray(q)), dt)
    rows = []
    for k in range(m.n):
        if m.limits[k] is not None:
            rows += [q[2 + k] - dt(m.limits[k][0]), dt(m.limits[k][1]) - q[2 + k]]
    for cdef in m.contacts:
        bi = cdef["body"]
        e = _rot(cs[bi], sn[bi], (dt(cdef["e"][0]), dt(cdef["e"][1])))
        rows.append(h[bi][1] + e[1] - dt(cdef["r"]) - dt(m.margin))
    return np.stack(rows)


def dynamics(m, q, v, ctrl, dt=np.float64):
    """qacc (nv,N), qfrc_constraint (nv,N), kin dict.  q, v: lists/arrays (nv, N); ctrl (nu, N).  All constraint rows
    are stated (inactive ones have f = 0) and solved by PGS_SWEEPS projected Gauss-Seidel sweeps."""
    m = tree_model(m)
    n, nv = m.n, m.n + 2
    N = q[0].shape[0]
    z = np.zeros(N, dt)
    one = np.ones(N, dt)
    om, cs, sn, h, hd, hdd = kinematics(m, q, v, dt)
    p, pd, pdd = [], [], []
    for i in range(n):
        rc = _rot(cs[i], sn[i], (dt(m.c[i][0]), dt(m.c[i][1])))
        p.append((h[i][0] + rc[0], h[i][1] + rc[1]))
        pd.append((hd[i][0] - om[i] * rc[1], hd[i][1] + om[i] * rc[0]))
        w2 = om[i] * om[i]
        pdd.append((hdd[i][0] - w2 * rc[0], hdd[i][1] - w2 * rc[1]))

    def point_jac(body, pt):
        JX = [z] * nv
        JY = [z] * nv
        JX[m.iX] = one
        JY[m.iY] = one
        for k in ancestors(m, body):
            JX[2 + k] = -dt(m.sgn[k]) * (pt[1] - h[k][1])
            JY[2 + k] = dt(m.sgn[k]) * (pt[0] - h[k][0])
        return JX, JY

    M = [[z for _ in range(nv)] for _ in range(nv)]
    tau = [z for _ in range(nv)]
    for i in range(n):
        JX, JY = point_jac(i, p[i])
        mi, Ii = dt(m.mass[i]), dt(m.Ip[i])
        fX = mi * dt(m.gravity[0]) - mi * pdd[i][0]
        fY = mi * dt(m.gravity[1]) - mi * pdd[i][1]
        tq = z
        if m.density > 0 or m.viscosity > 0:
            la = _rot(cs[i], sn[i], (dt(m.long_axis[i][0]), dt(m.long_axis[i][1])))
            vl = pd[i][0] * la[0] + pd[i][1] * la[1]
            vp = -pd[i][0] * la[1] + pd[i][1] * la[0]
            bl = dt(np.sqrt(6.0 * (2 * m.Ip[i] - m.Ia[i]) / m.mass[i]))
            bp = dt(np.sqrt(6.0 * m.Ia[i] / m.mass[i]))
            diam = (bl + 2 * bp) / dt(3.0)
            rho, beta = dt(m.density), dt(m.viscosity)
            Fl = -dt(0.5) * rho * bp * bp * np.abs(vl) * vl - dt(3 * np.pi) * beta * diam * vl
            Fp = -dt(0.5) * rho * bl * bp * np.abs(vp) * vp - dt(3 * np.pi) * beta * diam * vp
            fX = fX + Fl * la[0] - Fp * la[1]
            fY = fY + Fl * la[1] + Fp * la[0]
            tq = -rho * bp * (bl ** 4 + bp ** 4) / dt(64.0) * np.abs(om[i]) * om[i] - dt(np.pi) * beta * diam ** 3 * om[i]
        wv = [z] * nv
        for k in ancestors(m, i):
            wv[2 + k] = dt(m.sgn[k]) * one
        for r in range(nv):
            tau[r] = tau[r] + JX[r] * fX + JY[r] * fY + wv[r] * tq
            for c_ in range(r, nv):
                M[r][c_] = M[r][c_] + mi * (JX[r] * JX[c_] + JY[r] * JY[c_]) + Ii * wv[r] * wv[c_]
    for r in range(nv):
        M[r][r] = M[r][r] + dt(m.armature[r])
        tau[r] = tau[r] - dt(m.damping[r]) * v[r]
        if m.stiffness[r] != 0.0:
            tau[r] = tau[r] - dt(m.stiffness[r]) * q[r]
        for c_ in range(r):
            M[r][c_] = M[c_][r]
    for j, hk in enumerate(m.act):
        u = np.clip(ctrl[j], -dt(m.ctrl_lim), dt(m.ctrl_lim))
        tau[2 + hk] = tau[2 + hk] + (u if m.gear[j] == 1.0 else dt(m.gear[j]) * u)

    Lc = [[z for _ in range(nv)] for _ in range(nv)]
    for r in range(nv):
        for c_ in range(r + 1):
            s = M[r][c_]
            for k in range(c_):
                s = s - Lc[r][k] * Lc[c_][k]
            Lc[r][c_] = np.sqrt(s) if r == c_ else s / Lc[c_][c_]

    def solve(b):
        y = [None] * nv
        for r in range(nv):
            s = b[r]
            for k in range(r):
                s = s - Lc[r][k] * y[k]
            y[r] = s / Lc[r][r]
        x = [None] * nv
        for r in range(nv - 1, -1, -1):
            s = y[r]
            for k in range(r + 1, nv):
                s = s - Lc[k][r] * x[k]
            x[r] = s / Lc[r][r]
        return x

    a0 = solve(tau)
    rows = []
    kl, bl_ = _kb(m.lim_solref, m.lim_solimp)
    for k in range(n):
        if m.limits[k] is None:
            continue
        lo, hi = m.limits[k]
        for side, sgn_ in ((lo, 1.0), (hi, -1.0)):
            r_ = dt(sgn_) * (q[2 + k] - dt(side))
            J = [z] * nv
            J[2 + k] = dt(sgn_) * one
            d = _impedance(m.lim_solimp, r_)
            aref = -dt(bl_) * (dt(sgn_) * v[2 + k]) - dt(kl) * d * r_
            rows.append(dict(J=J, aref=aref, d=d, active=(r_ < 0), normal=None))
    if m.contacts:
        kc, bc = _kb(m.con_solref, m.con_solimp)
        for cdef in m.contacts:
            bi = cdef["body"]
            e = _rot(cs[bi], sn[bi], (dt(cdef["e"][0]), dt(cdef["e"][1])))
            sc = (h[bi][0] + e[0], h[bi][1] + e[1])
            dist = sc[1] - dt(cdef["r"])
            pt = (sc[0], sc[1] - dt(cdef["r"]))
            JX, JY = point_jac(bi, pt)
            r_ = dist - dt(m.margin)
            d = _impedance(m.con_solimp, r_)
            vn = sum(JY[k] * v[k] for k in range(nv))
            vt = sum(JX[k] * v[k] for k in range(nv))
            active = r_ < 0
            rows.append(dict(J=JY, aref=-dt(bc) * vn - dt(kc) * d * r_, d=d, active=active, normal=None))
            rows.append(dict(J=JX, aref=-dt(bc) * vt, d=d, active=active, normal=len(rows) - 1))
    nc = len(rows)
    qfc = [z for _ in range(nv)]
    if nc > 0:
        MiJ = [solve(rw["J"]) for rw in rows]
        A = [[sum(rows[i]["J"][k] * MiJ[j][k] for k in range(nv)) for j in range(nc)] for i in range(nc)]
        rhs = [rows[i]["aref"] - sum(rows[i]["J"][k] * a0[k] for k in range(nv)) for i in range(nc)]
        Rr = [(dt(1.0) - rows[i]["d"]) / rows[i]["d"] * A[i][i] for i in range(nc)]
        f = [z for _ in range(nc)]
        for _ in range(PGS_SWEEPS):
            for i in range(nc):
                s = rhs[i] - Rr[i] * f[i]
                for j in range(nc):
                    s = s - A[i][j] * f[j]
                fi = f[i] + s / (A[i][i] + Rr[i])
                if rows[i]["normal"] is None:
                    fi = np.maximum(fi, 0.0)
                else:
                    lim = dt(m.mu) * f[rows[i]["normal"]]
                    fi = np.clip(fi, -lim, lim)
                f[i] = np.where(rows[i]["active"], fi, z)
        for i in range(nc):
            for k in range(nv):
                qfc[k] = qfc[k] + rows[i]["J"][k] * f[i]
    acc = solve([tau[k] + qfc[k] for k in range(nv)]) if nc > 0 else a0
    mt = sum(m.mass)
    comX = sum(dt(m.mass[i]) * p[i][0] for i in range(n)) / dt(mt)
    comY = sum(dt(m.mass[i]) * p[i][1] for i in range(n)) / dt(mt)
    cvX = z
    for i in range(n):
        ro = _rot(cs[i], sn[i], (dt(m.bo[i][0]), dt(m.bo[i][1])))
        cvX = cvX + dt(m.mass[i]) * (hd[i][0] - om[i] * ro[1])
    cvX = cvX / dt(mt)
    n_active = sum(np.asarray(rw["active"], np.int64) for rw in rows) if rows else np.zeros(N, np.int64)
    return acc, qfc, dict(comX=comX, comY=comY, comvelX=cvX, n_active=n_active)


def integrate(m, q, v, ctrl, dt=np.float64):
    """One env step of frame_skip semi-implicit Euler sub-steps (HalfCheetah: one)."""
    assert not m.rk4
    nv = m.n + 2
    h = dt(m.dt)
    q = [np.asarray(x, dt) for x in q]
    v = [np.asarray(x, dt) for x in v]
    for _ in range(m.frame_skip):
        a, _, _ = dynamics(m, q, v, ctrl, dt)
        v = [v[k] + h * a[k] for k in range(nv)]
        q = [q[k] + h * v[k] for k in range(nv)]
    return np.stack(q), np.stack(v)


class HalfCheetahEnv(LaneEnv):
    """rllab/envs/mujoco/half_cheetah_env.py:14-48.  state = [qpos(9), qvel(9)];
    obs = [qpos[1:], qvel, torso subtree COM (x, 0, z)]; reward = torso subtree COM velocity x (body-origin velocities)
    - 0.05 * sum(clip(a, -1, 1)^2); never done."""
    name, kind = "half_cheetah", 7
    O, A, S, K = 20, 6, 18, 18
    noise_kind = "normal"
    lb, ub = (-1.0,) * 6, (1.0,) * 6

    def __init__(self, dtype=np.float64):
        LaneEnv.__init__(self, dtype)
        self.m = half_cheetah_model()

    def reset(self, raw):
        dt = self.dtype
        raw = np.asarray(raw, dt)
        q = np.asarray(self.m.q0, dt).reshape(-1, 1) + dt(0.01) * raw[:9]
        v = dt(0.1) * raw[9:18]
        return np.concatenate([q, v]).astype(dt)

    def kin(self, s):
        return subtree_com(self.m, list(s[:9]), list(s[9:18]), self.dtype)

    def obs(self, s):
        kin = self.kin(s)
        return np.concatenate([s[1:18], np.stack([kin["comX"], np.zeros_like(kin["comX"]), kin["comY"]])]).astype(
            self.dtype)

    def step(self, s, u):
        dt = self.dtype
        q, v = integrate(self.m, list(s[:9]), list(s[9:18]), u, dt)
        kin = self.kin(np.concatenate([q, v]))
        a = np.clip(np.asarray(u, dt), -1.0, 1.0)
        r = kin["comvelX"] - dt(0.05) * (a * a).sum(axis=0)
        return np.concatenate([q, v]).astype(dt), r.astype(dt), np.zeros(s.shape[1], bool)


def make(name, dtype=np.float64):
    if name == "half_cheetah":
        return HalfCheetahEnv(dtype)
    raise ValueError(name)


__all__ = ["half_cheetah_model", "HalfCheetahEnv", "dynamics", "integrate", "kinematics", "tree_model", "make",
           "hopper_model", "swimmer_model", "composite_bodies", "CHEETAH_GEOMS"]
