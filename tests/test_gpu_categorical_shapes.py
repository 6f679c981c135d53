"""GPU: the categorical path (csrc/categorical.cu) at the rollout grid's shapes and at saturated softmax probabilities,
against the float64 oracle (tests/categorical_oracle.py).

Rollout grid (env kinds of DISCRETE_ENVS, the discrete counterpart of test_gpu_rollout_shapes.py's ENVS), lane counts
1, 77, 128 x 37 and (4 n_sm + 3) x 128 - 45 (more than one resident wave of the 4-CTA/SM cat_rollout_kernel, a partial
last CTA), T = 40 (48 for the largest), max_path_length 17, theta with non-zero biases and logits large enough that
some lanes are confident.  On every sample:
  forward     prob against the oracle in float64 on the device's own obs (2e-5 rel + 2e-6 abs); prob and the action
              bit-identical to b200rl_categorical_get_actions on the same obs and u
  action      one-hot, and exactly weighted_sample(prob, u) evaluated on the device's float32 prob with float32 cumsum
  bookkeeping flags and tstep re-derived from the DONE bits: exact
  replay      obs, rew and DONE through b200rl_env_reset / b200rl_env_step with the recorded actions: bit for bit
  env oracle  one float64 CartPole-v0 step from obs[t] against obs[t+1] where the path continues (samples within 1e-5 of
              the 2.4 / 12 degree bounds excused), ENV_TOL
  philox      u = reset_raw = NULL bit-identical to fill_noise blocks, also at lane0 = 2^32 - 40 (blocks against
              oracle.philox); get_actions with u = NULL at row 3, lane0 = 2^32 - 40
  shards      [0, k) and [k, N) with lane0 = k (k not a multiple of 128) bit-identical to the N-lane run; reruns too
Edges: T = 1, max_path_length 1, = T, > T, 65 535 (accepted) and 65 536 (rejected); rejected calls write nothing.
Entropy kernel called directly, process_samples and the LinearFeatureBaseline fit on a kind-8 rollout.

Saturated buckets: theta_old = categorical_oracle.saturated_params(gap) puts every sample's logit gap within gap +- 0.25,
gap in GAPS; actions drawn by the device's get_actions, a few samples forced to the unlikely action (TRPO's
c = adv / (q + TINY) with q down to the unlikely probability).  Batch sizes 77 and the persistent-loop size, with and
without masking.  Per bucket: loss / KL, float32 gradients (TRPO, VPG; penalty 0 and 2.5) per parameter block, the
float32 Fisher-vector product (recomputed and cached) against the oracle's Gauss-Newton product J^T M J x, and the
float64 parity modes against the exact oracle; invariants of softmax's shift invariance (g[bout0] + g[bout1] = 0, the
bout rows of H x sum to zero) and of H's symmetry.  The float32 pass leaves out the O(TINY) curvature term of the exact
product (DESIGN.md section 5): above a gap of ~12 it is no longer small against J^T M J, so the float32 pass is held to
the product it computes.  Worst errors are printed at the end of the module (DESIGN.md section 5 has the figures).
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import categorical_oracle as C          # noqa: E402
from oracle import philox as PH         # noqa: E402
from oracle import sampler as S         # noqa: E402
from test_gpu_categorical import _batch_size, _f32, _rel   # noqa: E402
from test_gpu_process_shapes import REG, _assert_f32, _unpack   # noqa: E402
from test_gpu_rollout_shapes import CTA, ITER, LANE0_HIGH, SEED, _bits, _expected_bookkeeping, _geometry  # noqa: E402
from test_gpu_update_shapes import dev, n_sm  # noqa: E402,F401

DISCRETE_ENVS = ("gym_cartpole",)
DIMS = C.CatDims(4, (32, 32), 2)
CDIMS = (4, 32, 32, 2)
SIZES = ("1", "77", "exact", "large")
GAPS = (4, 8, 12, 16, 20, 30, 60)
SAT_SIZES = ("77", "large")
FIELDS = ("obs", "act", "mean", "rew", "flags", "tstep")
FWD_CHUNK = 1 << 18
NEAR = 1e-5                             # |x| or |theta| within this of the termination bound: the done bit may differ
ENV_TOL = (1e-5, 1e-6)                  # one-step CartPole-v0 (rtol, atol): ~10x the worst error an H100 measured (2.2e-7)
N_UNLIKELY = 5                          # samples per saturated batch that take the unlikely action
WORST = {}


def _ops():
    from rllab_b200 import ops
    return ops


def _L():
    from rllab_b200 import _lib
    return _lib


def _record(key, value):
    WORST[key] = max(WORST.get(key, 0.0), float(value))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst errors measured by test_gpu_categorical_shapes:")
    for k in sorted(WORST):
        print("worst %-40s %.4g" % (k, WORST[k]))


# ------------------------------------------------------------------------------------------- the rollout grid
def _rollout_theta(seed):
    """Non-zero biases everywhere; Wout x 12 and bout = (2.5, -2.5), so that part of the lanes is confident (a logit gap
    above 4 on ~13 % of the samples with the default seed, up to ~6)."""
    rng = np.random.RandomState(seed)
    ts = C.unpack(C.init_params(DIMS, rng) + 0.05 * rng.randn(DIMS.P), DIMS)
    ts[-2] *= 12.0
    ts[-1] = np.array([2.5, -2.5])
    return np.concatenate([t.reshape(-1) for t in ts])


def _noise(dev, N, T, lane0):
    """fill_noise blocks of one rollout: action uniforms u [T][1][N] (stream 0), reset noise [T+1][4][N] (stream 1)."""
    ops, L = _ops(), _L()
    u = torch.empty((T, 1, N), dtype=torch.float32, device=dev)
    ops.fill_noise(u, T, 0, 1, N, lane0, L.NOISE_UNIFORM, SEED, ITER, 0)
    rr = torch.empty((T + 1, 4, N), dtype=torch.float32, device=dev)
    ops.fill_noise(rr, T + 1, 0, 4, N, lane0, L.NOISE_UNIFORM, SEED, ITER, 1)
    return u, rr


def _poison(b):
    for k in ("obs", "act", "mean", "rew"):
        getattr(b, k).fill_(float("nan"))
    b.flags.fill_(0xFF)
    b.tstep.view(torch.int16).fill_(-1)


def _diff(b, other, sl=slice(None)):
    return [k for k in FIELDS if not torch.equal(_bits(getattr(b, k))[..., sl], _bits(getattr(other, k)))]


class CatCase(object):
    """One categorical rollout, N lanes x T steps, fed fill_noise blocks (lane0 0), and its host copy."""

    def __init__(self, dev, N, T, mpl, tag, seed=8):
        self.dev, self.N, self.T, self.mpl, self.tag = dev, N, T, mpl, tag
        self.th32 = torch.tensor(_rollout_theta(seed), dtype=torch.float32, device=dev)
        self.theta = self.th32.double().cpu().numpy()
        self.u, self.rr = _noise(dev, N, T, 0)
        self.b = self.rollout(N, self.u.view(T, N), self.rr, 0)
        self.traj = self.b.to_numpy()
        self.memo = {}
        torch.cuda.synchronize()

    def rollout(self, N, u, rr, lane0, T=None):
        ops = _ops()
        b = ops.LaneBatch(4, 2, N, T or self.T, self.dev)
        b.categorical = True
        _poison(b)
        ops.rollout(_L().ENV_GYM_CARTPOLE, self.th32, 32, 32, None, b, self.mpl, u, rr, SEED, ITER, lane0)
        return b

    def philox(self):
        if "philox" not in self.memo:
            self.memo["philox"] = self.rollout(self.N, None, None, 0)
        return self.memo["philox"]

    def release(self):
        self.b = self.u = self.rr = None
        self.memo.clear()


def _check_forward(c):
    """prob against the float64 oracle on the device's obs; returns the fraction of samples with a logit gap above 4."""
    obs = c.traj["obs"].reshape(4, -1)
    prob = c.traj["mean"].reshape(2, -1)
    worst, confident = 0.0, 0
    for i0 in range(0, obs.shape[1], FWD_CHUNK):
        sl = slice(i0, min(obs.shape[1], i0 + FWD_CHUNK))
        z, _ = C.forward(c.theta, obs[:, sl].T.astype(np.float64), DIMS)
        p = C.softmax(z)
        share = np.abs(prob[:, sl].T.astype(np.float64) - p) / (2e-6 + 2e-5 * p)
        k = np.unravel_index(np.argmax(share), share.shape)
        assert share[k] <= 1.0, "%s: prob of sample %d: device %r, oracle %r" % (c.tag, i0 + k[0], prob[k[1], i0 + k[0]],
                                                                                  p[k])
        worst = max(worst, share.max())
        confident += int((np.abs(z[:, 0] - z[:, 1]) > 4.0).sum())
    _record("rollout prob [share of tol]", worst)
    return confident / obs.shape[1]


def _sample32(prob, u):
    """weighted_sample on float32 probabilities with float32 cumsum: #{k : c_k < u} clipped to 1, c_1 = p0 + p1."""
    p = prob.astype(np.float32)
    c0, c1 = p[0], p[0] + p[1]
    return np.minimum((c0 < u).astype(np.int64) + (c1 < u), 1)


def _check_actions(c):
    act = c.traj["act"].reshape(2, -1)
    assert set(np.unique(act)) <= {0.0, 1.0} and np.all(act.sum(axis=0) == 1), c.tag
    k_ref = _sample32(c.traj["mean"].reshape(2, -1), c.u.cpu().numpy().reshape(-1))
    bad = act[1] != k_ref
    assert not bad.any(), "%s: action differs from weighted_sample on %d samples" % (c.tag, int(bad.sum()))


def _check_get_actions(c):
    ops = _ops()
    n = c.N * c.T
    act = torch.full((n,), -1, dtype=torch.int32, device=c.dev)
    prob = torch.full((2, n), float("nan"), device=c.dev)
    ops.categorical_get_actions(c.th32, CDIMS, c.b.obs.view(4, n), n, c.u.view(n), 0, 0, 0, 0, act, prob)
    assert torch.equal(_bits(prob), _bits(c.b.mean.view(2, n))), c.tag
    assert torch.equal(act.float(), c.b.act.view(2, n)[1]), c.tag


def _check_bookkeeping(c):
    L = _L()
    fl, ts = c.traj["flags"], c.traj["tstep"]
    assert not np.any(fl & ~np.uint8(L.FLAG_DONE | L.FLAG_END | L.FLAG_CUT)), c.tag
    ef, et = _expected_bookkeeping((fl & L.FLAG_DONE) != 0, c.mpl)
    assert np.array_equal(fl, ef), "%s: flags differ on %d samples" % (c.tag, int((fl != ef).sum()))
    assert np.array_equal(ts, et), "%s: tstep differs on %d samples" % (c.tag, int((ts != et).sum()))


def _check_replay(c, b=None, rr=None):
    """env_reset from reset row 0, env_step with the recorded action indices, the reset of row t+1 where a path ended."""
    ops, L = _ops(), _L()
    b = c.b if b is None else b
    rr = c.rr if rr is None else rr
    N, dev, kind = b.N, c.dev, L.ENV_GYM_CARTPOLE
    state = torch.empty((4, N), dtype=torch.float32, device=dev)
    obs = torch.empty_like(state)
    fresh_s, fresh_o = torch.empty_like(state), torch.empty_like(obs)
    rew = torch.empty((N,), dtype=torch.float32, device=dev)
    done = torch.empty((N,), dtype=torch.uint8, device=dev)
    end_dev = (b.flags & L.FLAG_END) != 0
    done_dev = (b.flags & L.FLAG_DONE) != 0
    ops.env_reset(kind, N, state, obs, rr[0])
    for t in range(b.T):
        assert torch.equal(_bits(obs), _bits(b.obs[:, t])), "%s: replayed obs differs at t=%d" % (c.tag, t)
        ops.env_step(kind, N, state, b.act[1, t].contiguous().view(1, N), obs, rew, done)
        assert torch.equal(_bits(rew), _bits(b.rew[t])), "%s: replayed rew differs at t=%d" % (c.tag, t)
        assert torch.equal(done != 0, done_dev[t]), "%s: DONE differs at t=%d" % (c.tag, t)
        ops.env_reset(kind, N, fresh_s, fresh_o, rr[t + 1])
        e = end_dev[t][None]
        state = torch.where(e, fresh_s, state).contiguous()
        obs = torch.where(e, fresh_o, obs).contiguous()


def _check_env_oracle(c):
    L = _L()
    tr = c.traj
    keep = (tr["flags"][:-1] & L.FLAG_END) == 0
    o_t = tr["obs"][:, :-1][:, keep].astype(np.float64)
    o_t1 = tr["obs"][:, 1:][:, keep].astype(np.float64)
    k = tr["act"][1, :-1][keep].astype(np.int64)
    assert np.array_equal(tr["rew"], np.ones_like(tr["rew"])), c.tag
    if o_t.shape[1] == 0:
        return 0
    ns, _, _ = C.CartPoleV0().step(o_t, k)
    near = np.any(np.abs(np.abs(ns[[0, 2]]) - [[2.4], [C.CartPoleV0.THR]]) < NEAR, axis=0)
    rtol, atol = ENV_TOL
    err = np.abs(o_t1 - ns)[:, ~near]
    share = err / (atol + rtol * np.abs(ns[:, ~near]))
    i = np.unravel_index(np.argmax(share), share.shape)
    assert share[i] <= 1.0, "%s: obs component %d: device %r, oracle %r" % (c.tag, i[0], o_t1[:, ~near][i],
                                                                            ns[:, ~near][i])
    _record("env cartpole_v0 obs [abs]", err.max())
    _record("env cartpole_v0 obs [share of tol]", share[i])
    return o_t.shape[1]


@pytest.fixture(scope="module", params=SIZES)
def case(request, dev, n_sm):
    N, T, mpl = _geometry(request.param, n_sm)
    c = CatCase(dev, N, T, mpl, "gym_cartpole-%s" % request.param)
    c.size = request.param
    yield c
    c.release()
    torch.cuda.empty_cache()


def test_forward_and_actions(case):
    conf = _check_forward(case)
    if case.N > 1:
        assert conf > 0.01, "%s: only %.3g of the samples have a logit gap above 4" % (case.tag, conf)
    _check_actions(case)
    _check_get_actions(case)


def test_bookkeeping(case):
    _check_bookkeeping(case)


def test_replay(case):
    _check_replay(case)


def test_env_one_step_oracle(case):
    assert _check_env_oracle(case) > 0


def test_philox_equals_injected(case):
    assert not _diff(case.b, case.philox()), case.tag


def test_shard_and_determinism(case):
    c = case
    assert not _diff(c.philox(), c.rollout(c.N, None, None, 0)), c.tag
    if c.N > 1:
        k = 33 if c.N < 2 * CTA else CTA * (c.N // (2 * CTA)) + 45
        lo, hi = c.rollout(k, None, None, 0), c.rollout(c.N - k, None, None, k)
        assert not _diff(c.philox(), lo, slice(0, k)), "%s: shard [0, %d)" % (c.tag, k)
        assert not _diff(c.philox(), hi, slice(k, None)), "%s: shard [%d, %d)" % (c.tag, k, c.N)


def test_philox_high_lane(dev):
    """N = 77 at lane0 = 2^32 - 40: NULL noise equals the fill_noise blocks at that lane0, the blocks equal oracle.philox
    bit for bit, and the replay holds."""
    N, T = 77, 40
    c = CatCase(dev, N, T, 17, "gym_cartpole lane0=2^32-40")
    u, rr = _noise(dev, N, T, LANE0_HIGH)
    inj = c.rollout(N, u.view(T, N), rr, LANE0_HIGH)
    kern = c.rollout(N, None, None, LANE0_HIGH)
    assert not _diff(inj, kern), c.tag
    assert _diff(c.b, kern), "lane0 does not change the noise"
    assert np.array_equal(u.cpu().numpy(), PH.uniform_from_raw(PH.raw_block(T, 0, 1, N, LANE0_HIGH, SEED, ITER, 0)))
    assert np.array_equal(rr.cpu().numpy(), PH.uniform_from_raw(PH.raw_block(T + 1, 0, 4, N, LANE0_HIGH, SEED, ITER, 1)))
    c.b, c.u, c.rr, c.traj = inj, u, rr, inj.to_numpy()
    _check_replay(c)
    _check_actions(c)
    _check_forward(c)


@pytest.mark.parametrize("lane0", [0, LANE0_HIGH])
def test_get_actions_philox(dev, lane0):
    """u = NULL at row 3 equals the fill_noise stream-0 block of row 3 at that lane0."""
    ops, L = _ops(), _L()
    n = 333
    th32 = torch.tensor(_rollout_theta(4), dtype=torch.float32, device=dev)
    obs = torch.tensor(np.random.RandomState(9).randn(4, n) * 0.5, dtype=torch.float32, device=dev)
    u = torch.empty((1, 1, n), dtype=torch.float32, device=dev)
    ops.fill_noise(u, 1, 3, 1, n, lane0, L.NOISE_UNIFORM, SEED, ITER, 0)
    out = []
    for uu in (u.view(n), None):
        act = torch.full((n,), -1, dtype=torch.int32, device=dev)
        prob = torch.full((2, n), float("nan"), device=dev)
        L.call("b200rl_categorical_get_actions", L.ptr(th32), 4, 32, 32, 2, L.ptr(obs), n, L.ptr(uu), SEED, ITER, 3,
               lane0, L.ptr(act), L.ptr(prob), ops._stream())
        out.append((act, prob))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(_bits(out[0][1]), _bits(out[1][1]))
    k_ref = _sample32(out[1][1].cpu().numpy(), u.cpu().numpy().reshape(-1))
    assert np.array_equal(out[1][0].cpu().numpy(), k_ref)
    if lane0:
        raw = PH.raw_block(1, 3, 1, n, lane0, SEED, ITER, 0)
        assert np.array_equal(u.cpu().numpy(), PH.uniform_from_raw(raw))


def test_get_actions_ties(dev):
    """u exactly at the cumulative probability: weighted_sample counts c_k < u strictly, so u = p0 takes action 0 and the
    next float32 above p0 takes action 1."""
    ops = _ops()
    n = 333
    th32 = torch.tensor(_rollout_theta(6), dtype=torch.float32, device=dev)
    obs = torch.tensor(np.random.RandomState(10).randn(4, n) * 0.5, dtype=torch.float32, device=dev)
    act = torch.empty((n,), dtype=torch.int32, device=dev)
    prob = torch.empty((2, n), dtype=torch.float32, device=dev)
    ops.categorical_get_actions(th32, CDIMS, obs, n, torch.zeros(n, device=dev), 0, 0, 0, 0, act, prob)
    p0 = prob[0].cpu().numpy()
    assert np.all(act.cpu().numpy() == 0)
    for u, want in ((p0, 0), (np.nextafter(p0, np.float32(2.0)), 1)):
        ops.categorical_get_actions(th32, CDIMS, obs, n, torch.tensor(u, device=dev), 0, 0, 0, 0, act, prob)
        got = act.cpu().numpy()
        assert np.array_equal(got, _sample32(prob.cpu().numpy(), u)) and np.all(got[p0 < 1] == want), want


EDGE_TM = [(1, 17), (40, 1), (40, 40), (40, 57), (40, 65535)]


@pytest.mark.parametrize("T,mpl", EDGE_TM, ids=["T%d-mpl%d" % p for p in EDGE_TM])
def test_edges(dev, T, mpl):
    L = _L()
    c = CatCase(dev, 333, T, mpl, "gym_cartpole T=%d mpl=%d" % (T, mpl))
    fl, ts = c.traj["flags"], c.traj["tstep"]
    end, cut, done = ((fl & f) != 0 for f in (L.FLAG_END, L.FLAG_CUT, L.FLAG_DONE))
    assert end[-1].all() and np.array_equal(cut[-1], ~done[-1] & (ts[-1] + 1 < mpl))
    if mpl == 1:
        assert end.all() and not cut.any() and not ts.any()
    if mpl >= T:
        assert not cut[:-1].any() and np.array_equal(end[:-1], done[:-1])
    _check_bookkeeping(c)
    _check_forward(c)
    _check_actions(c)
    _check_get_actions(c)
    _check_replay(c)
    if T > 1:
        _check_env_oracle(c)
    assert not _diff(c.b, c.philox()), c.tag


def test_rejected_calls_write_nothing(dev):
    """A Box env kind, hidden (64, 64) / (32, 64), N <= 0 and max_path_length 65 536 to the categorical rollout, and
    get_actions / entropy with a shape or n_actions that is not compiled in: errors, outputs untouched."""
    ops, L = _ops(), _L()
    N, T = 77, 8
    th = torch.zeros(DIMS.P + 4096, dtype=torch.float32, device=dev)
    for kind, h1, h2, n, mpl in ((L.ENV_CARTPOLE, 32, 32, N, 5), (L.ENV_GYM_CARTPOLE, 64, 64, N, 5),
                                 (L.ENV_GYM_CARTPOLE, 32, 64, N, 5), (L.ENV_GYM_CARTPOLE, 32, 32, 0, 5),
                                 (L.ENV_GYM_CARTPOLE, 32, 32, -1, 5), (L.ENV_GYM_CARTPOLE, 32, 32, N, 65536)):
        b = ops.LaneBatch(4, 2, N, T, dev)
        ref = ops.LaneBatch(4, 2, N, T, dev)
        _poison(b), _poison(ref)
        with pytest.raises(L.B200RLError):
            L.call("b200rl_rollout_categorical", kind, L.ptr(th), h1, h2, n, T, mpl, None, None, SEED, ITER, 0,
                   L.ptr(b.obs), L.ptr(b.act), L.ptr(b.mean), L.ptr(b.rew), L.ptr(b.flags), L.ptr(b.tstep),
                   ops._stream())
        torch.cuda.synchronize()
        assert not _diff(b, ref), (kind, h1, h2, n, mpl)
    obs = torch.zeros((8, N), dtype=torch.float32, device=dev)
    for O, h1, h2, A in ((5, 32, 32, 2), (4, 64, 64, 2), (4, 32, 32, 3), (4, 32, 32, 1)):
        act = torch.full((N,), -7, dtype=torch.int32, device=dev)
        prob = torch.full((3, N), float("nan"), device=dev)
        with pytest.raises(L.B200RLError):
            L.call("b200rl_categorical_get_actions", L.ptr(th), O, h1, h2, A, L.ptr(obs), N, None, SEED, ITER, 0, 0,
                   L.ptr(act), L.ptr(prob), ops._stream())
        torch.cuda.synchronize()
        assert bool((act == -7).all()) and bool(torch.isnan(prob).all()), (O, h1, h2, A)
    p = torch.full((3, N), 0.5, device=dev)
    for A in (1, 3):
        out = torch.full((2,), -3.0, dtype=torch.float64, device=dev)
        with pytest.raises(L.B200RLError):
            L.call("b200rl_categorical_entropy", A, N, L.ptr(p), None, L.ptr(out), L.ptr(ops.workspace(dev)),
                   ops._stream())
        torch.cuda.synchronize()
        assert out.tolist() == [-3.0, -3.0], A


# ------------------------------------------------------------------------------------------- entropy
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("size", SIZES)
def test_entropy_kernel(dev, n_sm, size, masked):
    """b200rl_categorical_entropy on probabilities that include exact 0, exact 1 and values around TINY: the count
    exactly, the sum within 4 float32 ulps of the float64 sum over the same float32 probabilities, relative to the sum of
    the terms' magnitudes, plus 2^-24 per sample: where p + TINY rounds to p in float32 (p near 1), log(p + TINY) is off
    by up to 2^-24 (the term -log(1 + TINY) of p = 1 is -1e-8 exactly, 0 in float32)."""
    ops, L = _ops(), _L()
    B = _batch_size(size, n_sm)
    rng = np.random.RandomState(B + masked)
    special = np.array([0.0, 1.0, 1e-8, 5e-9, 2e-8, 1e-9, 1e-12, 1e-30, 0.5, 1 - 2 ** -24], np.float32)
    p0 = np.where(rng.rand(B) < 0.3, special[rng.randint(0, len(special), B)], rng.rand(B)).astype(np.float32)
    p0[:min(B, len(special))] = special[:min(B, len(special))]
    p1 = (np.float32(1.0) - p0).astype(np.float32)
    swap = rng.rand(B) < 0.5
    prob = np.stack([np.where(swap, p1, p0), np.where(swap, p0, p1)])
    keep = np.ones(B, bool)
    b = ops.LaneBatch(4, 2, B, 1, dev)
    b.categorical = True
    b.mean.copy_(torch.tensor(prob.reshape(2, 1, B)))
    if masked:
        keep = rng.rand(B) > 0.3
        keep[0] = True
        b.flags.copy_(torch.tensor(np.where(keep, 0, L.FLAG_MASKED).astype(np.uint8).reshape(1, B)))
        b.masked = True
    out = torch.full((2,), float("nan"), dtype=torch.float64, device=dev)
    ops.categorical_entropy(b, out)
    got = out.cpu().numpy()
    pk = prob[:, keep].astype(np.float64)
    terms = -pk * np.log(pk + C.TINY)
    ref = float(np.sum(terms))
    assert got[1] == keep.sum(), (got[1], keep.sum())
    err = abs(got[0] - ref) / (np.sum(np.abs(terms)) * 2.0 ** -23 + keep.sum() * 2.0 ** -24 / 4)
    _record("entropy sum [float32 ulps rel]", err)
    assert err <= 4.0, (got[0], ref, err)


# ------------------------------------------------------------------------------------------- process_samples, fit
@pytest.mark.parametrize("drop", [False, True], ids=["cut_kept", "drop_cut"])
def test_process_samples_and_fit_on_rollout(dev, drop):
    """A 2048-lane x 200-step kind-8 rollout at max_path_length 200: process_samples with a fitted baseline against
    oracle.sampler.process_samples_lanes (1 ulp + 1e-12 of the suffix sums), and the LinearFeatureBaseline fit with
    test_gpu_process_shapes.py's FIT_ENVS tolerances (solve alone 1e-6, end to end 1e-5 of max |ret|)."""
    ops, L = _ops(), _L()
    N, T = 2048, 200
    th32 = torch.tensor(_rollout_theta(5), dtype=torch.float32, device=dev)
    b = ops.LaneBatch(4, 2, N, T, dev)
    b.categorical = True
    ops.rollout(L.ENV_GYM_CARTPOLE, th32, 32, 32, None, b, T, None, None, 11, 0)
    flags0 = b.flags.clone()
    ws = []
    for it in range(2):                     # the second pass predicts with the first pass's fit
        b.flags.copy_(flags0)
        w = None if it == 0 else ws[-1]
        ops.process_samples(b, w, 0.99, 1.0, drop_cut_paths=drop)
        gram = torch.empty((13 * 14 // 2,), dtype=torch.float64, device=dev)
        ops.lfb_gram(b, gram)
        w_out = torch.empty((12,), dtype=torch.float64, device=dev)
        fit = torch.zeros((3,), dtype=torch.float64, device=dev)
        ops.lfb_solve(4, gram, REG, w_out, fit)
        ws.append(w_out)
        assert tuple(fit.cpu().tolist()) == (REG, 0.0, 1.0)
        traj = b.to_numpy()
        keep = b.valid_mask().reshape(-1)
        F = S.lfb_features_lanes(traj["obs"], traj["tstep"]).reshape(12, -1)[:, keep]
        y = b.ret.cpu().numpy().reshape(-1)[keep].astype(np.float64)
        Gd = _unpack(gram.cpu().numpy(), 13)
        pred = w_out.cpu().numpy() @ F
        s = np.abs(y).max()
        e_solve = np.abs(pred - S.lfb_fit_normal(Gd[:-1, :-1], Gd[:-1, -1], REG) @ F).max() / s
        e_fit = np.abs(pred - S.lfb_fit_normal(F @ F.T, F @ y, REG) @ F).max() / s
        _record("lfb fit solve [of max|ret|]", e_solve)
        _record("lfb fit end to end [of max|ret|]", e_fit)
        assert e_solve <= 1e-6 and e_fit <= 1e-5, (e_solve, e_fit)
        # process_samples against the oracle on the device's own baseline
        base = b.base.cpu().numpy()
        tr = dict(rew=traj["rew"], flags=flags0.cpu().numpy(), tstep=traj["tstep"], log_std=np.zeros(1))
        ref = S.process_samples_lanes(tr, None, 0.99, 1.0, center_adv=False, drop_cut=drop, base=base)
        absr = np.abs(traj["rew"].astype(np.float64)) + 2.0 * np.abs(base.astype(np.float64))
        suf = S.process_samples_lanes(dict(tr, rew=absr), None, 1.0, 1.0, center_adv=False)["ret"]
        exp_flags = tr["flags"] | np.where(ref["valid"], 0, L.FLAG_MASKED).astype(np.uint8) if drop else tr["flags"]
        assert np.array_equal(traj["flags"], exp_flags)
        _record("process ret [ulp]", _assert_f32(b.ret.cpu().numpy(), ref["ret"], 1e-12 * suf, "ret"))
        _record("process adv [ulp]", _assert_f32(b.adv.cpu().numpy(), ref["adv_raw"], 1e-12 * suf, "adv"))
        if it == 1:
            Fw = S.lfb_features_lanes(traj["obs"], traj["tstep"])
            exact = np.tensordot(ws[0].cpu().numpy(), Fw, axes=(0, 0))
            scale = np.tensordot(np.abs(ws[0].cpu().numpy()), np.abs(Fw), axes=(0, 0))
            _record("process base [ulp]", _assert_f32(base, exact, 1e-13 * scale, "base"))


# ------------------------------------------------------------------------------------------- saturated buckets
def _blocks():
    out, k = [], 0
    for s in DIMS.shapes:
        n = int(np.prod(s))
        out.append(slice(k, k + n))
        k += n
    return out


BLOCKS = _blocks()
BOUT = BLOCKS[-1]


def _sat_case(dev, n_sm, gap, size, masked):
    """A batch of B samples (lanes N = B, T = 1) at theta_old = saturated_params(gap), actions by the device's
    get_actions, N_UNLIKELY samples switched to the unlikely action; with the oracle's view of it."""
    ops, L = _ops(), _L()
    B = _batch_size(size, n_sm)
    rng = np.random.RandomState(1000 * gap + B + (7 if masked else 0))
    theta_old = _f32(C.saturated_params(DIMS, gap, rng, 1.0 if GAPS.index(gap) % 2 == 0 else -1.0))
    obs = (rng.randn(4, B) * [[1.0], [1.5], [0.2], [1.5]]).astype(np.float32)
    b = ops.LaneBatch(4, 2, B, 1, dev)
    b.categorical = True
    b.obs.copy_(torch.tensor(obs.reshape(4, 1, B)))
    th32 = torch.tensor(theta_old, dtype=torch.float32, device=dev)
    u = torch.tensor(rng.rand(B).astype(np.float32), device=dev)
    act = torch.empty(B, dtype=torch.int32, device=dev)
    prob = torch.empty((2, B), dtype=torch.float32, device=dev)
    ops.categorical_get_actions(th32, CDIMS, b.obs.view(4, B), B, u, 0, 0, 0, 0, act, prob)
    a = act.cpu().numpy()
    pr = prob.cpu().numpy()
    unl = np.unique(np.linspace(0, B - 1, N_UNLIKELY).astype(int))
    a[unl] = np.argmin(pr[:, unl], axis=0)
    b.mean.copy_(prob.view(2, 1, B))
    b.act.copy_(torch.tensor(np.eye(2, dtype=np.float32)[a].T.reshape(2, 1, B)))
    b.adv.copy_(torch.tensor(rng.randn(1, B).astype(np.float32)))
    keep = np.ones(B, dtype=bool)
    if masked:
        keep = rng.rand(B) > 0.3
        keep[unl] = True
        b.flags.copy_(torch.tensor(np.where(keep, 0, L.FLAG_MASKED).astype(np.uint8).reshape(1, B)))
        b.count.fill_(float(keep.sum()))
        b.masked = True
    batch = dict(obs=obs.T.astype(np.float64)[keep], actions=np.eye(2)[a][keep],
                 adv=b.adv.view(B).double().cpu().numpy()[keep], old_prob=pr.T.astype(np.float64)[keep])
    z, _ = C.forward(theta_old, batch["obs"], DIMS)
    gaps = np.abs(z[:, 0] - z[:, 1])
    assert gaps.min() > gap - 0.3 and gaps.max() < gap + 0.3, (gaps.min(), gaps.max())
    return b, theta_old, batch, rng


def _check_blocks(got, ref, what, rtol=1e-3, atol_rel=2e-5):
    """Element-wise rtol, plus atol_rel x the largest |ref| of the whole vector and, separately, of each block."""
    np.testing.assert_allclose(got, ref, rtol=rtol, atol=atol_rel * np.abs(ref).max() + 1e-300, err_msg=what)
    worst = 0.0
    for i, sl in enumerate(BLOCKS):
        g, r = got[sl], ref[sl]
        share = np.abs(g - r) / (rtol * np.abs(r) + atol_rel * np.abs(r).max() + 1e-300)
        assert share.max() <= 1.0, "%s, block %d: %.3g of the tolerance at %d (device %r, oracle %r)" % (
            what, i, share.max(), int(np.argmax(share)), g[np.argmax(share)], r[np.argmax(share)])
        worst = max(worst, share.max())
    return worst


def _bout_sum(v):
    return abs(v[BOUT][0] + v[BOUT][1]) / max(abs(v[BOUT][1]), 1e-300)


SAT_CASES = [(g, s, m) for g in GAPS for s in SAT_SIZES for m in (False, True)]


@pytest.fixture(scope="module", params=SAT_CASES, ids=["gap%d-%s-%s" % (g, s, "masked" if m else "all")
                                                        for g, s, m in SAT_CASES])
def sat(request, dev, n_sm):
    gap, size, masked = request.param
    b, theta_old, batch, rng = _sat_case(dev, n_sm, gap, size, masked)
    yield dict(gap=gap, b=b, theta_old=theta_old, batch=batch, rng=rng, dims=_ops().CategoricalDims(4, 32, 32, 2),
               theta=_f32(theta_old + 0.01 * rng.randn(DIMS.P)), x=rng.randn(DIMS.P), y=rng.randn(DIMS.P))
    torch.cuda.empty_cache()


def test_saturated_loss_kl(sat, dev):
    """Ratio exactly 1, KL exactly 0 at theta_old; off it the loss and KL against the oracle (test_gpu_categorical's
    tolerances; the KL with an allowance of 4 float32 ulps of 1 per sample for log(q + TINY) - log(p + TINY), whose two
    logs of numbers near 1 float32 resolves to 6e-8)."""
    L, ops = _L(), _ops()
    b, batch, dims = sat["b"], sat["batch"], sat["dims"]
    out = torch.zeros(3, dtype=torch.float64, device=dev)
    ops.loss_kl(L.LOSS_TRPO, torch.tensor(sat["theta_old"], dtype=torch.float32, device=dev), dims, None, b, out)
    o = out.cpu().numpy()
    assert o[1] == 0.0 and o[2] == 0.0
    np.testing.assert_allclose(o[0], -np.mean(batch["adv"]), rtol=1e-12, atol=1e-15)
    theta = sat["theta"]
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    kl_allow = 4 * 2.0 ** -24
    for kind, lk in (("trpo", L.LOSS_TRPO), ("vpg", L.LOSS_VPG)):
        ops.loss_kl(lk, th32, dims, None, b, out)
        o = out.cpu().numpy()
        ref = C.surr_loss(theta, batch, DIMS, kind)
        np.testing.assert_allclose(o[0], ref, rtol=2e-5, atol=1e-7)
        mkl, xkl = C.kl_stats(theta, batch, DIMS)
        _record("sat loss [rel]", abs(o[0] - ref) / abs(ref))
        _record("sat mean kl [abs]", abs(o[1] - mkl))
        _record("sat max kl [abs]", abs(o[2] - xkl))
        np.testing.assert_allclose(o[1:], [mkl, xkl], rtol=2e-3, atol=1e-8 + kl_allow)


def test_saturated_gradients(sat, dev):
    L, ops = _L(), _ops()
    b, batch, dims, theta = sat["b"], sat["batch"], sat["dims"], sat["theta"]
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    out = torch.zeros(3, dtype=torch.float64, device=dev)
    for kind, lk in (("trpo", L.LOSS_TRPO), ("vpg", L.LOSS_VPG)):
        ops.loss_kl(lk, th32, dims, None, b, out)
        for pen in (0.0, 2.5):
            g = torch.zeros(DIMS.P, dtype=torch.float64, device=dev)
            tri = torch.zeros(3, dtype=torch.float64, device=dev)
            if pen:
                ops.grad_penalized(lk, pen, th32, dims, None, b, g, tri)
            else:
                ops.grad(lk, th32, dims, None, b, g, tri, b.hcache(32, 32))
            gd = g.cpu().numpy()
            ref = C.grad_surr(theta, batch, DIMS, kind, pen)
            w = _check_blocks(gd, ref, "gap %d %s penalty %g" % (sat["gap"], kind, pen))
            _record("sat grad [share of tol]", w)
            inv = _bout_sum(gd)
            _record("sat grad |g_bout0 + g_bout1| / |g_bout1|", inv)
            assert inv <= 1e-4, inv
            np.testing.assert_allclose(tri.cpu().numpy(), out.cpu().numpy(), rtol=1e-12, atol=1e-18)


def test_saturated_fvp(sat, dev):
    """The float32 Fisher-vector product at theta_old (recomputed and from the activation cache) against the oracle's
    J^T M J x, per block; at reg_coeff = 0: x^T H x > 0, symmetry, and bout rows summing to zero."""
    L, ops = _L(), _ops()
    b, batch, dims, x, y = sat["b"], sat["batch"], sat["dims"], sat["x"], sat["y"]
    th_old32 = torch.tensor(sat["theta_old"], dtype=torch.float32, device=dev)
    hc = b.hcache(32, 32)
    ops.grad(L.LOSS_TRPO, th_old32, dims, None, b, torch.zeros(DIMS.P, dtype=torch.float64, device=dev), None, hc)
    res = {}
    for reg in (1e-5, 0.0):
        for cache in (None, hc):
            for name, v in (("x", x), ("y", y)):
                Hv = torch.zeros(DIMS.P, dtype=torch.float64, device=dev)
                ops.fvp(th_old32, dims, None, b, torch.tensor(v, device=dev), reg, 1.0, Hv, cache)
                res[reg, cache is None, name] = Hv.cpu().numpy()
        ref = C.fvp(sat["theta_old"], batch, _f32(x), DIMS, reg, curvature=False)
        for recompute in (True, False):
            w = _check_blocks(res[reg, recompute, "x"], ref, "gap %d fvp reg %g recompute %s" % (sat["gap"], reg,
                                                                                                 recompute))
            _record("sat fvp [share of tol]", w)
    for recompute in (True, False):
        hx, hy = res[0.0, recompute, "x"], res[0.0, recompute, "y"]
        xhx, yhy = x @ hx, y @ hy
        assert xhx > 0 and yhy > 0, (xhx, yhy)
        sym = abs(x @ hy - y @ hx) / np.sqrt(xhx * yhy)
        _record("sat fvp symmetry", sym)
        assert sym <= 1e-4, sym
        inv = _bout_sum(hx)
        _record("sat fvp |Hx_bout0 + Hx_bout1| / |Hx_bout1|", inv)
        assert inv <= 1e-4, inv


def test_saturated_f64_parity(sat, dev):
    """update_f64 modes 0 / 1 / 2 (TRPO, VPG, the LOSS_KL gradient, the exact Fisher product) within 1e-10 of the oracle
    per block; g[bout0] + g[bout1] = 0, symmetry and bout rows of H x within 1e-12."""
    L, ops = _L(), _ops()
    b, batch, dims, theta, x, y = sat["b"], sat["batch"], sat["dims"], sat["theta"], sat["x"], sat["y"]
    th64 = torch.tensor(theta, dtype=torch.float64, device=dev)
    out = torch.zeros(3, dtype=torch.float64, device=dev)
    v = torch.zeros(DIMS.P, dtype=torch.float64, device=dev)
    for kind, lk in (("trpo", L.LOSS_TRPO), ("vpg", L.LOSS_VPG)):
        ops.update_f64(0, lk, th64, dims, None, b, None, 0.0, 0.0, None, out)
        o = out.cpu().numpy()
        np.testing.assert_allclose(o[0], C.surr_loss(theta, batch, DIMS, kind), rtol=1e-10, atol=1e-15)
        # both sides form log(q + TINY) - log(p + TINY) of numbers near 1: 1e-15 of absolute allowance per sample
        np.testing.assert_allclose(o[1:], C.kl_stats(theta, batch, DIMS), rtol=1e-10, atol=1e-15)
        ops.update_f64(1, lk, th64, dims, None, b, None, 0.0, 0.0, v, out)
        checks = [(kind, v.cpu().numpy(), C.grad_surr(theta, batch, DIMS, kind))]
        if lk == L.LOSS_VPG:
            ops.update_f64(1, L.LOSS_KL, th64, dims, None, b, None, 0.0, 0.0, v, None)
            checks.append(("kl", v.cpu().numpy(), C.grad_kl(theta, batch, DIMS)))
        for what, got, ref in checks:
            w = _check_blocks(got, ref, "gap %d f64 grad %s" % (sat["gap"], what), rtol=0.0, atol_rel=1e-10)
            _record("sat f64 grad [share of tol]", w)
            inv = _bout_sum(got)
            _record("sat f64 grad |g_bout0 + g_bout1| / |g_bout1|", inv)
            assert inv <= 1e-12, (what, inv)
    th_old64 = torch.tensor(sat["theta_old"], dtype=torch.float64, device=dev)
    hv = {}
    for name, vec in (("x", x), ("y", y)):
        ops.update_f64(2, L.LOSS_TRPO, th_old64, dims, None, b, torch.tensor(vec, device=dev), 0.0, 1.0, v, None)
        hv[name] = v.cpu().numpy().copy()
        ref = C.fvp(sat["theta_old"], batch, vec, DIMS, 0.0)
        w = _check_blocks(hv[name], ref, "gap %d f64 fvp" % sat["gap"], rtol=0.0, atol_rel=1e-10)
        _record("sat f64 fvp [share of tol]", w)
    # the exact product includes the TINY curvature term and is indefinite once p_small < TINY: normalise by norms
    sym = abs(x @ hv["y"] - y @ hv["x"]) / (np.linalg.norm(x) * np.linalg.norm(hv["y"]) +
                                            np.linalg.norm(y) * np.linalg.norm(hv["x"]))
    _record("sat f64 fvp symmetry", sym)
    assert sym <= 1e-12, sym
    if sat["gap"] <= 16:
        assert x @ hv["x"] > 0 and y @ hv["y"] > 0
    inv = _bout_sum(hv["x"])
    _record("sat f64 fvp |Hx_bout0 + Hx_bout1| / |Hx_bout1|", inv)
    assert inv <= 1e-12, inv


# ------------------------------------------------------------------------------------------- one TRPO step, saturated
SAT_TRPO_GAP = 12


@pytest.mark.parametrize("precision", ["f32", "f64"])
def test_trpo_step_on_saturated_rollout(dev, precision):
    """One TRPO step (4 CG iterations) from a policy whose logit gap is SAT_TRPO_GAP at every input, on a 512-lane x 50
    rollout, against categorical_oracle.trpo_step as test_gpu_categorical.py's TRPO tests check it."""
    from test_gpu_categorical import _algo, _oracle_batch
    kw = dict(cg_iters=4) if precision == "f32" else dict(cg_iters=4, precision="f64")
    algo = _algo("trpo", 512, 50, optimizer_args=kw)
    algo.policy.set_param_values(_f32(C.saturated_params(DIMS, SAT_TRPO_GAP, np.random.RandomState(3))))
    algo.start_worker()
    algo.init_opt()
    sd = algo.sampler.process_samples(0, algo.sampler.obtain_samples(0))
    batch = _oracle_batch(sd)
    z, _ = C.forward(algo.policy.get_param_values(), batch["obs"], DIMS)
    assert np.abs(z[:, 0] - z[:, 1]).min() > SAT_TRPO_GAP - 0.3
    theta0 = algo.policy.get_param_values()
    algo.optimize_policy(0, sd)
    theta_dev = algo.policy.get_param_values()
    # the float32 pass solves with the Gauss-Newton product, the f64 mode with the exact one (1 % apart at gap 12)
    theta_ref, info = C.trpo_step(theta0, batch, DIMS, 0.01, 4, curvature=precision == "f64")
    li = algo.optimizer.last_info
    assert li["n_iter"] == info["n_iter"] and li["rejected"] == info["rejected"] and not info["rejected"]
    step = _rel(theta_dev - theta0, theta_ref - theta0)
    _record("sat trpo step %s [rel]" % precision, step)
    if precision == "f32":
        assert step < 1e-3 and _rel(theta_dev, theta_ref) < 1e-5, step
        np.testing.assert_allclose(li["constraint_val"], info["constraint_val"], rtol=2e-3)
    else:
        assert _rel(theta_dev, theta_ref) < 1e-5, _rel(theta_dev, theta_ref)
        np.testing.assert_allclose(li["constraint_val"], info["constraint_val"], rtol=1e-3)
