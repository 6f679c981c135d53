"""HalfCheetah without a GPU: the oracle model against the reference XML, the tree dynamics against a torch.autograd
Lagrangian, the tree code against the serial-chain oracle on Hopper, and the host-side env surface."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import planar as SP
import planar_tree_oracle as T

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_half_cheetah_model.json")


@pytest.fixture(scope="module")
def ref():
    with open(GOLDEN) as f:
        return json.load(f)


def _joint_param(ref, j, key):
    return j[key][0] if key in j else ref["default"]["joint"][key][0]


def test_model_constants_rederived_from_the_reference_xml(ref):
    m = T.half_cheetah_model()
    bodies = ref["bodies"]
    names = [b["name"] for b in bodies]
    assert names == ["torso", "bthigh", "bshin", "bfoot", "fthigh", "fshin", "ffoot"]
    assert m.parent == [-1] + [names.index(b["parent"]) for b in bodies[1:]]
    # root height and hinge anchors: body pos (x, z) in the parent frame; joints sit at the body origin
    assert m.y0 == bodies[0]["pos"][2]
    for i, b in enumerate(bodies[1:], 1):
        assert m.a[i] == (b["pos"][0], b["pos"][2])
    for b in bodies:
        for j in b["joints"]:
            assert j["pos"] == [0.0, 0.0, 0.0]
    # geoms -> capsules: (body, half-length, centre, axis angle about +y); composite mass / COM / inertia
    geoms = []
    for i, b in enumerate(bodies):
        for g in b["geoms"]:
            assert g["type"] == "capsule"
            if "fromto" in g:
                f = g["fromto"]
                c = ((f[0] + f[3]) / 2, (f[2] + f[5]) / 2)
                dx, dz = f[3] - f[0], f[5] - f[2]
                hl, ang = 0.5 * np.hypot(dx, dz), np.arctan2(dx, dz)
            else:
                assert g["axisangle"][:3] == [0.0, 1.0, 0.0]
                c, hl, ang = (g["pos"][0], g["pos"][2]), g["size"][1], g["axisangle"][3]
            assert g["size"][0] == T.CHEETAH_R
            geoms.append((g["name"], i, hl, c, ang))
    assert len(geoms) == len(T.CHEETAH_GEOMS) == 8
    for a, b in zip(geoms, T.CHEETAH_GEOMS):
        assert a[:2] == b[:2]
        np.testing.assert_allclose([a[2], a[3][0], a[3][1], a[4]], [b[2], b[3][0], b[3][1], b[4]], rtol=0, atol=1e-15)
    assert ref["compiler"]["settotalmass"] == [14.0]
    mass, com, inertia = T.composite_bodies(geoms, 7, T.CHEETAH_R, 14.0)
    np.testing.assert_allclose(m.mass, mass, rtol=1e-15)
    np.testing.assert_allclose(np.array(m.c), np.array(com), rtol=1e-15, atol=1e-15)
    np.testing.assert_allclose(m.Ip, inertia, rtol=1e-15)
    assert abs(sum(m.mass) - 14.0) < 1e-12
    # the torso inertia is the two capsules about their joint COM, not either one alone
    m_t, ip_t, _ = SP.capsule(T.CHEETAH_R, 1.0)
    assert m.Ip[0] > 14.0 / sum(SP.capsule(T.CHEETAH_R, 2 * g[2])[0] for g in geoms) * ip_t
    # contact candidates: both end spheres of every capsule
    ends = [(g[1], (g[3][0] + s * g[2] * np.sin(g[4]), g[3][1] + s * g[2] * np.cos(g[4]))) for g in geoms
            for s in (-1.0, 1.0)]
    assert len(m.contacts) == 16
    for (bi, e), c in zip(ends, m.contacts):
        assert c["body"] == bi and c["r"] == T.CHEETAH_R
        np.testing.assert_allclose(c["e"], e, rtol=0, atol=1e-15)
    # joints: q = [rootx, rootz, rooty, 6 hinges]; limits, stiffness, damping, armature; every hinge about +y
    joints = [j for b in bodies for j in b["joints"]]
    assert [j["name"] for j in joints] == ["rootx", "rootz", "rooty", "bthigh", "bshin", "bfoot", "fthigh", "fshin",
                                           "ffoot"]
    assert joints[0]["axis"] == [1.0, 0.0, 0.0] and joints[1]["axis"] == [0.0, 0.0, 1.0]
    for j in joints[2:]:
        assert j["type"] == "hinge" and j["axis"] == [0.0, 1.0, 0.0]
    assert m.sgn == [-1.0] * 7
    for k, j in enumerate(joints):
        assert m.stiffness[k] == _joint_param(ref, j, "stiffness")
        assert m.damping[k] == _joint_param(ref, j, "damping")
        assert m.armature[k] == _joint_param(ref, j, "armature")
        limited = j.get("limited", ref["default"]["joint"]["limited"]) == "true"
        if k >= 2:
            assert (m.limits[k - 2] is not None) == limited
            if limited:
                assert list(m.limits[k - 2]) == j["range"]
    assert list(m.lim_solref) == ref["default"]["joint"]["solreflimit"]
    assert list(m.lim_solimp) == ref["default"]["joint"]["solimplimit"]
    # actuators, contacts, option
    acts = ref["actuators"]
    assert [a["joint"] for a in acts] == [j["name"] for j in joints[3:]]
    assert m.act == [1, 2, 3, 4, 5, 6]
    assert m.gear == [a["gear"][0] for a in acts]
    assert ref["default"]["motor"]["ctrlrange"] == [-m.ctrl_lim, m.ctrl_lim]
    gd = ref["default"]["geom"]
    assert m.mu == gd["friction"][0] and list(m.con_solref) == gd["solref"] and list(m.con_solimp) == gd["solimp"]
    assert gd["contype"] == "1" and gd["conaffinity"] == "0" and gd["condim"] == "3"
    assert m.dt == ref["option"]["timestep"][0] and m.gravity == (0.0, ref["option"]["gravity"][2])
    assert m.frame_skip == 1 and not m.rk4 and m.margin == 0.0


# --------------------------------------------------------------------------- dynamics against autograd
def _torch_lagrangian_acc(m, q, v, ctrl):
    """qacc of the unconstrained tree from L = T - V with torch.autograd (float64): M = d2T/dv2 + armature,
    bias = d2T/dvdq v - dT/dq + dV/dq, plus damping, stiffness and geared actuation."""
    nv = m.n + 2
    q = torch.tensor(q, dtype=torch.float64, requires_grad=True)
    v = torch.tensor(v, dtype=torch.float64, requires_grad=True)

    def energies(q, v):
        phi, om, h, hd = [], [], [], []
        for i in range(m.n):
            p = m.parent[i]
            phi.append((0.0 if p < 0 else phi[p]) + m.sgn[i] * q[2 + i])
            om.append((0.0 if p < 0 else om[p]) + m.sgn[i] * v[2 + i])
        for i in range(m.n):
            p = m.parent[i]
            if p < 0:
                h.append(torch.stack([q[m.iX], q[m.iY] + m.y0]))
            else:
                R = torch.stack([torch.stack([torch.cos(phi[p]), -torch.sin(phi[p])]),
                                 torch.stack([torch.sin(phi[p]), torch.cos(phi[p])])])
                h.append(h[p] + R @ torch.tensor(m.a[i], dtype=torch.float64))
        Tk, V = 0.0, 0.0
        for i in range(m.n):
            R = torch.stack([torch.stack([torch.cos(phi[i]), -torch.sin(phi[i])]),
                             torch.stack([torch.sin(phi[i]), torch.cos(phi[i])])])
            pc = h[i] + R @ torch.tensor(m.c[i], dtype=torch.float64)
            J = torch.autograd.functional.jacobian(lambda qq: _com_of(m, qq, i), q, create_graph=True)
            vel = J @ v
            Tk = Tk + 0.5 * m.mass[i] * (vel @ vel) + 0.5 * m.Ip[i] * om[i] ** 2
            V = V - m.mass[i] * (m.gravity[0] * pc[0] + m.gravity[1] * pc[1])
        return Tk, V

    Tk, V = energies(q, v)
    dT_dv = torch.autograd.grad(Tk, v, create_graph=True)[0]
    Mm = torch.stack([torch.autograd.grad(dT_dv[r], v, retain_graph=True)[0] for r in range(nv)])
    dT_dq = torch.autograd.grad(Tk, q, retain_graph=True)[0]
    dV_dq = torch.autograd.grad(V, q, retain_graph=True)[0]
    Cv = torch.stack([torch.autograd.grad(dT_dv[r], q, retain_graph=True)[0] @ v for r in range(nv)])
    tau = -(Cv - dT_dq) - dV_dq
    tau = tau - torch.tensor(m.damping, dtype=torch.float64) * v - torch.tensor(m.stiffness, dtype=torch.float64) * q
    for j, hk in enumerate(m.act):
        tau[2 + hk] = tau[2 + hk] + m.gear[j] * float(np.clip(ctrl[j], -m.ctrl_lim, m.ctrl_lim))
    Mm = Mm + torch.diag(torch.tensor(m.armature, dtype=torch.float64))
    return torch.linalg.solve(Mm.detach(), tau.detach()).numpy(), Mm.detach().numpy()


def _com_of(m, q, i):
    phi = []
    for k in range(m.n):
        p = m.parent[k]
        phi.append((0.0 if p < 0 else phi[p]) + m.sgn[k] * q[2 + k])
    chain = T.ancestors(m, i)
    pos = torch.stack([q[m.iX], q[m.iY] + m.y0])
    for k in chain[1:]:
        p = m.parent[k]
        R = torch.stack([torch.stack([torch.cos(phi[p]), -torch.sin(phi[p])]),
                         torch.stack([torch.sin(phi[p]), torch.cos(phi[p])])])
        pos = pos + R @ torch.tensor(m.a[k], dtype=torch.float64)
    R = torch.stack([torch.stack([torch.cos(phi[i]), -torch.sin(phi[i])]),
                     torch.stack([torch.sin(phi[i]), torch.cos(phi[i])])])
    return pos + R @ torch.tensor(m.c[i], dtype=torch.float64)


def _free_states(rng, n):
    """Airborne states with every hinge inside its limits: no constraint row is active."""
    m = T.half_cheetah_model()
    q = np.zeros((9, n))
    q[0] = rng.uniform(-1, 1, n)
    q[1] = rng.uniform(0.6, 1.0, n)                     # torso at z = 1.3 .. 1.7
    q[2] = rng.uniform(-0.3, 0.3, n)
    for k, (lo, hi) in enumerate(m.limits[1:]):
        q[3 + k] = rng.uniform(lo + 0.05, hi - 0.05, n)
    v = rng.normal(0, 1.5, (9, n))
    u = rng.uniform(-1.3, 1.3, (6, n))
    return q, v, u


def test_tree_dynamics_match_autograd_lagrangian():
    rng = np.random.RandomState(3)
    m = T.half_cheetah_model()
    q, v, u = _free_states(rng, 6)
    acc, qfc, kin = T.dynamics(m, list(q), list(v), u)
    assert (kin["n_active"] == 0).all()
    assert np.abs(np.stack(qfc)).max() == 0.0
    acc = np.stack(acc)
    for n in range(q.shape[1]):
        ref_acc, _ = _torch_lagrangian_acc(m, q[:, n], v[:, n], u[:, n])
        np.testing.assert_allclose(acc[:, n], ref_acc, rtol=1e-9, atol=1e-9 * np.abs(ref_acc).max())


def test_tree_code_reproduces_the_serial_oracle_on_hopper():
    rng = np.random.RandomState(5)
    N = 64
    hm = SP.hopper_model()
    q = np.asarray(hm.q0)[:, None] + rng.normal(0, 0.3, (6, N))
    q[0] = rng.uniform(0.9, 1.4, N)                     # some feet in contact, some limits active
    v = rng.normal(0, 2, (6, N))
    u = rng.normal(0, 150, (3, N))
    a0, f0, k0 = SP.dynamics(SP.hopper_model(), list(q), list(v), u)
    a1, f1, k1 = T.dynamics(SP.hopper_model(), list(q), list(v), u)
    assert (k1["n_active"] > 0).any()
    for x, y in zip(a0 + f0, a1 + f1):
        assert np.array_equal(x, y)
    for key in ("comX", "comY", "comvelX"):
        assert np.array_equal(k0[key], k1[key])


def test_contact_rows_engage_on_the_ground():
    m = T.half_cheetah_model()
    env = T.HalfCheetahEnv()
    s = env.reset(np.zeros((18, 3)))
    s[1] = [-0.3, -0.65, -0.8]                           # feet, legs and torso pressed into the floor
    s[2] = [0.0, 0.0, np.pi]                             # last lane upside down: torso and head on the ground
    _, _, kin = T.dynamics(m, list(s[:9]), list(s[9:]), np.zeros((6, 3)))
    assert (kin["n_active"] > 0).all()
    s2, r, d = env.step(s, np.zeros((6, 3)))
    assert np.isfinite(s2).all() and np.isfinite(r).all() and not d.any()
    assert (s2[10] > 0).all()                            # the floor pushes up


# --------------------------------------------------------------------------- ABI and host API
def test_env_info_half_cheetah():
    from rllab_b200 import _lib as L
    info = L.env_info(L.ENV_KINDS["half_cheetah"])
    assert L.ENV_HALF_CHEETAH == 7
    assert (info["obs_dim"], info["act_dim"], info["state_dim"], info["reset_dim"], info["noise_kind"]) == \
        (20, 6, 18, 18, L.NOISE_NORMAL)
    assert info["lb"] == [-1.0] * 6 and info["ub"] == [1.0] * 6


def test_half_cheetah_env_spec_and_defaults():
    from rllab_b200.envs.mujoco.half_cheetah_env import HalfCheetahEnv
    env = HalfCheetahEnv()
    assert env.observation_space.flat_dim == 20
    assert env.action_space.flat_dim == 6
    lb, ub = env.action_bounds
    assert list(lb) == [-1.0] * 6 and list(ub) == [1.0] * 6
    HalfCheetahEnv(action_noise=0.0, file_path=None, template_args=None)
    with pytest.raises(NotImplementedError):
        HalfCheetahEnv(action_noise=0.1)
    with pytest.raises(NotImplementedError):
        HalfCheetahEnv(file_path="other.xml")
    with pytest.raises(TypeError):
        HalfCheetahEnv(ctrl_cost_coeff=1.0)


def test_log_diagnostics_reads_forward_progress_from_obs_minus_3():
    from rllab_b200.envs.mujoco.half_cheetah_env import HalfCheetahEnv
    from rllab_b200.misc import logger
    env = HalfCheetahEnv()
    o = np.zeros((4, 20))
    o[:, -3] = [0.0, 1.0, 2.0, 3.5]
    recorded = {}
    orig = logger.record_tabular
    logger.record_tabular = lambda k, v: recorded.__setitem__(k, v)
    try:
        env.log_diagnostics([dict(observations=o), dict(observations=o[:2])])
    finally:
        logger.record_tabular = orig
    assert recorded["AverageForwardProgress"] == pytest.approx(2.25)
    assert recorded["MaxForwardProgress"] == 3.5 and recorded["MinForwardProgress"] == 1.0
