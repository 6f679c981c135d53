"""GPU: the fused lane rollout (rollout_kernel<Env,H>), env reset / step and get_actions against the float64 oracle at
every env kind and hidden width, on the injected noise tensors and on the in-kernel Philox stream training uses.

Grid: env kind in {point, cartpole, pendulum, cartpole_swingup, double_pendulum, swimmer, hopper, half_cheetah} x hidden
{32, 64} (16 kernel instantiations, all 14 compiled nets) x lane counts derived from the SM count n_sm of the device:
  1             one lane
  77            one partial CTA
  exact         128 x 37 lanes, whole CTAs
  large         (4 n_sm + 3) x 128 - 45 lanes: more than one resident wave of the 4-CTA/SM 32-wide classic-control
                kernels, several waves of the 1-CTA/SM kernels (planar envs, 64-wide nets), a partial last CTA
T = 40 steps (large: 48), max_path_length 17.  theta has non-zero biases and a distinct log_std per component.

The fused step is checked piece by piece, so that every sample is compared without chaotic divergence:
  forward     mean against oracle.policy.forward in float64 on the device's own obs (2e-5 rel + 2e-6 abs), and mean,
              act, log_std bit-identical to b200rl_policy_get_actions on the same obs and noise
  action      act within 2 float32 ulps of mean + exp(log_std) eps (float64), ulps of |mean| + |std eps|
  bookkeeping flags and tstep re-derived from the device's DONE bits, max_path_length and T with the rollout_lanes
              recurrence: exact
  replay      the recorded actions and the same reset noise replayed through b200rl_env_reset / b200rl_env_step:
              obs, rew and the DONE bit bit-identical to the fused rollout's
  env oracle  one step of the float64 oracle env from the state rebuilt from obs[t] (atan2 for the angles) with act[t],
              against obs[t+1] and rew[t] at every sample that does not end a path (Swimmer: a fixed subsample of ~5 000
              samples that includes the last CTA; Point: the float32 oracle, bit-exact).  Hopper's obs clips qvel and
              the constraint forces, so it does not determine the state: the replay holds Hopper's fused step to the
              stand-alone env kernels, which tests/test_gpu_round2.py holds to the oracle.  HalfCheetah: the float64
              tree oracle (tests/planar_tree_oracle.py) on the same kind of subsample, rootx rebuilt from comX; a
              sample whose constraint residual lies within 1e-5 of zero may take a different active set in float32
              and is excused (under 1 % of the samples)
  philox      the rollout with eps = reset_raw = NULL bit-identical to the rollout fed b200rl_fill_noise blocks
              (stream 0 [T][A][N], stream 1 [T+1][K][N]); also at lane0 = 2^32 - 40, where the lane counter crosses
              into its high word, with the blocks against oracle.philox; env_reset and get_actions with NULL noise
  shards      lanes [0, k) and [k, N) with lane0 = k (k not a multiple of 128) bit-identical to the N-lane rollout, and
              two identical calls bit-identical
Edges on cartpole-32, hopper-64 and pendulum-32: T = 1, max_path_length 1, = T and > T; pendulum-32 with paths that
reach the uint16 tstep limit; a min_std that binds for some components (Hopper; HalfCheetah, in both Philox chunks of
its action noise); calls that must be rejected.

Measured on an H100 80GB HBM3 (132 SMs, 400 W power limit; the HalfCheetah cases at 700 W) -- see DESIGN.md section 5
for the figures per check.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import envs as E            # noqa: E402
from oracle import philox as PH         # noqa: E402
from oracle import policy as P          # noqa: E402
import planar_tree_oracle as TREE       # noqa: E402
from test_gpu_half_cheetah import _state_from_obs as cheetah_state_from_obs  # noqa: E402
from test_gpu_update_shapes import dev, n_sm  # noqa: E402,F401

# new env kinds go at the end: the per-case seeds come from ENVS.index
ENVS = ("point", "cartpole", "pendulum", "cartpole_swingup", "double_pendulum", "swimmer", "hopper", "half_cheetah")
HIDDEN = (32, 64)
SIZES = ("1", "77", "exact", "large")
CASES = [(e, h, s) for e in ENVS for h in HIDDEN for s in SIZES]
CTA = 128
SEED, ITER = 3, 5
MIN_STD = 1e-6
LANE0_HIGH = (1 << 32) - 40
FWD_CHUNK = 1 << 18                     # samples per host chunk of the float64 forward
SUBSAMPLE = 4096                        # Swimmer, HalfCheetah: samples of random lanes for the one-step planar oracle
SUBSAMPLED = ("swimmer", "half_cheetah")
NEAR = 1e-5                             # HalfCheetah: |constraint residual| below which a sample is excused
# one-step env tolerances (rtol, atol), float32 kernel against the float64 oracle: about 10x the worst error the H100
# measured, as a share of the env tests' 2e-4 / 2e-5 (classic) and 4e-3 / 1e-3 (planar): cartpole 0.011, swingup 0.012,
# pendulum 0.014, swimmer 0.0047.  DoublePendulum used 0.48 of its ceiling (6e-5 on an angular velocity after two
# sub-steps, from the atan2-recovered angles) and keeps it.  HalfCheetah stays at the 1e-3 / 1e-3 of
# tests/test_gpu_half_cheetah.py's rollout check: it used 0.22 of that (2.7e-4 absolute on obs), so 10x would be looser.
ENV_TOL = dict(cartpole=(2.5e-5, 2.5e-6), cartpole_swingup=(2.5e-5, 2.5e-6), pendulum=(3e-5, 3e-6),
               double_pendulum=(2e-4, 2e-5), swimmer=(2e-4, 5e-5), half_cheetah=(1e-3, 1e-3))
FIELDS = ("obs", "act", "mean", "rew", "flags", "tstep", "log_std")
WORST = {}                              # check -> worst measured error (printed at the end of the module)


def _ops():
    from rllab_b200 import ops
    return ops


def _L():
    from rllab_b200 import _lib
    return _lib


def _record(key, value):
    WORST[key] = max(WORST.get(key, 0.0), float(value))


@pytest.fixture(scope="session", autouse=True)
def _report():
    yield
    print("\nworst errors measured by test_gpu_rollout_shapes:")
    for k in sorted(WORST):
        print("worst %-28s %.4g" % (k, WORST[k]))


def _oracle_env(env):
    """The float64 oracle env: oracle.envs, or the planar tree oracle for the branched bodies it does not hold."""
    try:
        return E.make(env)
    except ValueError:
        return TREE.make(env)


def _geometry(size, n_sm):
    """(N, T, max_path_length) of a grid size."""
    if size == "large":
        return (4 * n_sm + 3) * CTA - 45, 48, 17
    return {"1": 1, "77": 77, "exact": CTA * 37}[size], 40, 17


def _bits(t):
    """A view whose equality is bit equality (NaN payloads included)."""
    if t.dtype == torch.float32:
        return t.view(torch.int32)
    if t.dtype == torch.uint16:
        return t.view(torch.int16)
    return t


def _poison(b):
    """Sentinels in every output buffer: a sample the kernel does not write shows up as NaN / 0xFF / 0xFFFF."""
    for k in ("obs", "act", "mean", "rew", "log_std"):
        getattr(b, k).fill_(float("nan"))
    b.flags.fill_(0xFF)
    b.tstep.view(torch.int16).fill_(-1)


def _diff(b, other, sl=slice(None)):
    """Fields of `other` that differ in any bit from lanes `sl` of `b`."""
    bad = []
    for k in FIELDS:
        x = _bits(getattr(b, k))
        if k != "log_std":
            x = x[..., sl]
        if not torch.equal(x, _bits(getattr(other, k))):
            bad.append(k)
    return bad


class Case(object):
    """One rollout of `env` at hidden H, N lanes x T steps, fed b200rl_fill_noise blocks (stream 0 action noise, stream
    1 reset noise at seed SEED, iter ITER, lane0 0), plus the host copy of its outputs.  `memo` caches further device
    runs (the in-kernel Philox rollout) for the checks that share them."""

    def __init__(self, dev, env, H, N, T, mpl, min_std=MIN_STD, log_std=None, tag=""):
        L = _L()
        self.dev, self.env, self.H, self.N, self.T, self.mpl, self.min_std = dev, env, H, N, T, mpl, min_std
        self.tag = tag or "%s-%d N=%d T=%d mpl=%d" % (env, H, N, T, mpl)
        self.kind = L.ENV_KINDS[env]
        self.env64 = _oracle_env(env)
        O, A = self.O, self.A = self.env64.O, self.env64.A
        self.dims = P.Dims(O, (H, H), A)
        rng = np.random.RandomState(100 * ENVS.index(env) + H)
        theta = P.init_params(self.dims, rng)
        theta += rng.randn(self.dims.P) * 0.05                             # non-zero biases
        theta[-A:] = -0.5 + 0.1 * np.arange(A) if log_std is None else log_std   # a distinct log_std per component
        self.th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
        self.theta = self.th32.double().cpu().numpy()
        self.eps, self.rr = _noise(dev, self.env64, N, T, 0)
        self.b = self.rollout(N, self.eps, self.rr, 0)
        self.traj = self.b.to_numpy()
        self.memo = {}
        torch.cuda.synchronize()

    def rollout(self, N, eps, rr, lane0):
        ops = _ops()
        b = ops.LaneBatch(self.O, self.A, N, self.T, self.dev)
        _poison(b)
        ops.rollout(self.kind, self.th32, self.H, self.H, self.min_std, b, self.mpl, eps, rr, SEED, ITER, lane0)
        return b

    def philox(self):
        """The same rollout with eps = reset_raw = NULL: noise drawn in the kernel, as LaneSampler runs it."""
        if "philox" not in self.memo:
            self.memo["philox"] = self.rollout(self.N, None, None, 0)
        return self.memo["philox"]

    def release(self):
        self.b = self.eps = self.rr = None
        self.memo.clear()


def _noise(dev, env64, N, T, lane0):
    """b200rl_fill_noise blocks of one rollout: action noise [T][A][N] (stream 0, normal) and reset noise [T+1][K][N]
    (stream 1, the env's kind)."""
    ops, L = _ops(), _L()
    eps = torch.empty((T, env64.A, N), dtype=torch.float32, device=dev)
    ops.fill_noise(eps, T, 0, env64.A, N, lane0, L.NOISE_NORMAL, SEED, ITER, 0)
    kind = L.NOISE_UNIFORM if env64.noise_kind == "uniform" else L.NOISE_NORMAL
    rr = torch.empty((T + 1, env64.K, N), dtype=torch.float32, device=dev)
    ops.fill_noise(rr, T + 1, 0, env64.K, N, lane0, kind, SEED, ITER, 1)
    return eps, rr


# ------------------------------------------------------------------------------------------- checks shared by the tests
def _check_log_std(c):
    """log_std_out within 1 float32 ulp of max(param, log(min_std))."""
    param = c.theta[-c.A:]
    ref = np.maximum(param, np.log(np.float64(np.float32(c.min_std))))
    got = c.traj["log_std"].astype(np.float64)
    ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    err = np.abs(got - ref) / ulp
    assert np.all(err <= 1.0), (c.tag, got, ref)
    _record("log_std [ulp]", err.max())


def _check_forward(c):
    """mean against the float64 oracle on the device's obs, every sample; returns the worst error as a share of the
    2e-5 rel + 2e-6 abs tolerance."""
    obs = c.traj["obs"].reshape(c.O, -1)
    mean = c.traj["mean"].reshape(c.A, -1)
    worst, worst_abs = 0.0, 0.0
    for i0 in range(0, obs.shape[1], FWD_CHUNK):
        sl = slice(i0, min(obs.shape[1], i0 + FWD_CHUNK))
        mu, _ = P.forward(c.theta, obs[:, sl].T, c.dims, c.min_std)
        err = np.abs(mean[:, sl].T.astype(np.float64) - mu)
        share = err / (2e-6 + 2e-5 * np.abs(mu))
        k = np.unravel_index(np.argmax(share), share.shape)
        assert share[k] <= 1.0, "%s: mean of sample %d component %d: device %r, oracle %r" % (
            c.tag, i0 + k[0], k[1], float(mean[k[1], i0 + k[0]]), mu[k])
        worst, worst_abs = max(worst, share.max()), max(worst_abs, err.max())
    _record("forward [share of tol] H%d" % c.H, worst)
    _record("forward [abs] H%d" % c.H, worst_abs)
    return worst


def _check_get_actions(c):
    """b200rl_policy_get_actions on the rollout's obs and noise: mean, act and log_std bit-identical."""
    ops = _ops()
    n = c.N * c.T
    eps = c.eps.permute(1, 0, 2).contiguous().view(c.A, n)
    act = torch.empty((c.A, n), dtype=torch.float32, device=c.dev)
    mean = torch.empty_like(act)
    ls = torch.empty((c.A,), dtype=torch.float32, device=c.dev)
    ops.policy_get_actions(c.th32, c.O, c.H, c.H, c.A, c.min_std, c.b.obs.view(c.O, n), n, eps, 0, 0, 0, 0, act, mean,
                           ls)
    for name, x, y in (("mean", mean, c.b.mean.view(c.A, n)), ("act", act, c.b.act.view(c.A, n)),
                       ("log_std", ls, c.b.log_std)):
        same = _bits(x) == _bits(y)
        assert bool(same.all()), "%s: get_actions %s differs from the rollout's on %d of %d entries (first %d)" % (
            c.tag, name, int((~same).sum()), same.numel(), int(torch.nonzero(~same.view(-1))[0]))


def _check_action(act, mean, log_std, eps, tag):
    """act within 2 float32 ulps of mean + exp(log_std) eps in float64; (A, ...) arrays, ulps of |mean| + |std eps|."""
    std = np.exp(log_std.astype(np.float64)).reshape((-1,) + (1,) * (act.ndim - 1))
    se = std * eps.astype(np.float64)
    ref = mean.astype(np.float64) + se
    ulp = np.spacing((np.abs(mean.astype(np.float64)) + np.abs(se)).astype(np.float32)).astype(np.float64)
    err = np.abs(act.astype(np.float64) - ref) / ulp
    k = np.unravel_index(np.argmax(err), err.shape)
    assert err[k] <= 2.0, "%s: act %r, mean + std eps = %r (%.2f ulp) at %s" % (tag, float(act[k]), ref[k], err[k], k)
    _record("action [ulp]", err[k])


def _expected_bookkeeping(done, mpl):
    """flags and tstep of sampler.rollout_lanes from the per-sample done bits (T, N)."""
    L = _L()
    T, N = done.shape
    flags = np.zeros((T, N), np.uint8)
    tstep = np.zeros((T, N), np.uint16)
    plen = np.zeros(N, np.int64)
    for t in range(T):
        tstep[t] = plen
        plen += 1
        whole = done[t] | (plen >= mpl)
        end = whole | (t == T - 1)
        flags[t] = np.where(done[t], L.FLAG_DONE, 0) | np.where(end, L.FLAG_END, 0) | np.where(end & ~whole, L.FLAG_CUT, 0)
        plen[end] = 0
    return flags, tstep


def _check_bookkeeping(c):
    L = _L()
    fl, ts = c.traj["flags"], c.traj["tstep"]
    assert not np.any(fl & ~np.uint8(L.FLAG_DONE | L.FLAG_END | L.FLAG_CUT)), c.tag
    ef, et = _expected_bookkeeping((fl & L.FLAG_DONE) != 0, c.mpl)
    for name, got, exp in (("flags", fl, ef), ("tstep", ts, et)):
        bad = got != exp
        if bad.any():
            t, n = np.argwhere(bad)[0]
            raise AssertionError("%s: %s differs on %d samples; first (t=%d, lane %d): device %d, expected %d" % (
                c.tag, name, int(bad.sum()), t, n, int(got[t, n]), int(exp[t, n])))


def _check_replay(c):
    """Reset every lane from reset row 0, step with the recorded actions, take the reset of row t+1 where the device
    ended a path at t: obs, rew and done must be the fused rollout's bit for bit."""
    ops, L = _ops(), _L()
    N, T, dev = c.N, c.T, c.dev
    S, O = c.env64.S, c.O
    state = torch.empty((S, N), dtype=torch.float32, device=dev)
    obs = torch.empty((O, N), dtype=torch.float32, device=dev)
    fresh_s, fresh_o = torch.empty_like(state), torch.empty_like(obs)
    rew = torch.empty((N,), dtype=torch.float32, device=dev)
    done = torch.empty((N,), dtype=torch.uint8, device=dev)
    end_dev = (c.b.flags & L.FLAG_END) != 0
    done_dev = (c.b.flags & L.FLAG_DONE) != 0
    ops.env_reset(c.kind, N, state, obs, c.rr[0])
    for t in range(T):
        ne = (_bits(obs) != _bits(c.b.obs[:, t])).any(0)
        assert not bool(ne.any()), "%s: replayed obs differs at t=%d on %d lanes (first %d)" % (
            c.tag, t, int(ne.sum()), int(torch.nonzero(ne)[0]))
        ops.env_step(c.kind, N, state, c.b.act[:, t].contiguous(), obs, rew, done)
        ne = _bits(rew) != _bits(c.b.rew[t])
        assert not bool(ne.any()), "%s: replayed rew differs at t=%d on %d lanes (first %d)" % (
            c.tag, t, int(ne.sum()), int(torch.nonzero(ne)[0]))
        ne = (done != 0) != done_dev[t]
        assert not bool(ne.any()), "%s: DONE bit differs from the replayed done at t=%d on %d lanes (first %d)" % (
            c.tag, t, int(ne.sum()), int(torch.nonzero(ne)[0]))
        ops.env_reset(c.kind, N, fresh_s, fresh_o, c.rr[t + 1])
        e = end_dev[t][None]
        state = torch.where(e, fresh_s, state).contiguous()
        obs = torch.where(e, fresh_o, obs).contiguous()


def _state_from_obs(env, o):
    """Env state (S, n) from its obs (O, n), float64."""
    if env in ("point", "cartpole", "cartpole_swingup"):
        return o
    if env == "pendulum":
        return np.stack([np.arctan2(o[1], o[0]), o[2]])
    if env == "double_pendulum":
        return np.stack([np.arctan2(o[0], o[1]), np.arctan2(o[3], o[4]), o[2], o[5]])
    if env == "swimmer":
        return o[:10]
    if env == "half_cheetah":
        return cheetah_state_from_obs(TREE.HalfCheetahEnv(), o)
    raise ValueError(env)


def _subsample_lanes(N, T):
    """Swimmer, HalfCheetah: the last 32 lanes (the tail of the last CTA) plus a fixed random set of ~SUBSAMPLE
    samples."""
    want = max(1, SUBSAMPLE // max(1, T - 1))
    rng = np.random.default_rng([N, T])
    lanes = np.concatenate([np.arange(max(0, N - 32), N), rng.choice(N, size=min(N, want), replace=False)])
    return np.unique(lanes)


def _check_env_oracle(c):
    """One oracle env step from the state in obs[t] with act[t] against obs[t+1], rew[t] where t does not end a path."""
    L = _L()
    tr = c.traj
    lanes = _subsample_lanes(c.N, c.T) if c.env in SUBSAMPLED else np.arange(c.N)
    fl = tr["flags"][:-1][:, lanes]
    keep = (fl & L.FLAG_END) == 0                                    # (T-1, n): obs[t+1] continues the path
    o_t = tr["obs"][:, :-1][:, :, lanes][:, keep]
    o_t1 = tr["obs"][:, 1:][:, :, lanes][:, keep]
    a_t = tr["act"][:, :-1][:, :, lanes][:, keep]
    r_t = tr["rew"][:-1][:, lanes][keep]
    if o_t.shape[1] == 0:
        return 0
    if c.env == "point":                                             # float32 oracle: bit-exact
        env32 = E.make("point", np.float32)
        s2, r, d = env32.step(o_t, env32.scale_action(a_t))
        assert np.array_equal(env32.obs(s2), o_t1), c.tag
        assert np.array_equal(r, r_t) and not d.any(), c.tag
        return o_t.shape[1]
    env64 = c.env64
    s = _state_from_obs(c.env, o_t.astype(np.float64))
    s2, r, _ = env64.step(s, env64.scale_action(a_t.astype(np.float64)))
    rtol, atol = ENV_TOL[c.env]
    held = np.ones(s.shape[1], bool)
    if c.env == "half_cheetah":
        # the device and the oracle step the same float32 state; only a residual within rounding of zero can make
        # their active sets differ
        near = (np.abs(TREE.constraint_residuals(env64.m, list(s[:9]))) < NEAR).any(axis=0)
        assert near.mean() < 0.01, "%s: %.3g of the samples have a residual within %g of zero" % (
            c.tag, near.mean(), NEAR)
        _record("env half_cheetah excused [share]", near.mean())
        held = ~near
    for name, got, ref in (("obs", o_t1, env64.obs(s2)), ("rew", r_t, r)):
        got, ref = got[..., held], ref[..., held]
        err = np.abs(got.astype(np.float64) - ref)
        share = err / (atol + rtol * np.abs(ref))
        k = np.unravel_index(np.argmax(share), share.shape)
        assert share[k] <= 1.0, "%s: %s: device %r, oracle %r at %s (|diff| %.3g)" % (
            c.tag, name, float(got[k]), ref[k], k, err[k])
        _record("env %s %s [abs]" % (c.env, name), err.max())
        _record("env %s %s [rel]" % (c.env, name), (err / np.maximum(np.abs(ref), 1e-30)).max())
        _record("env %s %s [share of tol]" % (c.env, name), share[k])
    return o_t.shape[1]


# ------------------------------------------------------------------------------------------- the case grid
@pytest.fixture(scope="module", params=CASES, ids=["%s-%d-%s" % p for p in CASES])
def case(request, dev, n_sm):
    env, H, size = request.param
    N, T, mpl = _geometry(size, n_sm)
    c = Case(dev, env, H, N, T, mpl, tag="%s-%d-%s" % (env, H, size))
    c.size = size
    yield c
    c.release()
    torch.cuda.empty_cache()


def test_forward(case):
    """mean against the float64 oracle on every sample, and bit-identical to get_actions (64-wide: the rollout's rolled
    dense_thread_col layer 2 against get_actions' unrolled dense_thread)."""
    _check_log_std(case)
    _check_forward(case)
    _check_get_actions(case)


def test_action(case):
    c = case
    _check_action(c.traj["act"], c.traj["mean"], c.traj["log_std"], c.eps.cpu().numpy().transpose(1, 0, 2), c.tag)


def test_bookkeeping(case):
    _check_bookkeeping(case)


def test_replay(case):
    _check_replay(case)


def test_env_one_step_oracle(case):
    if case.env == "hopper":
        pytest.skip("Hopper's obs does not determine its state (clipped qvel and constraint forces): test_replay")
    assert _check_env_oracle(case) > 0


def test_philox_equals_injected(case):
    bad = _diff(case.b, case.philox())
    assert not bad, "%s: in-kernel Philox rollout differs from the fill_noise-fed one in %s" % (case.tag, bad)


def test_shard_and_determinism(case):
    c = case
    again = c.rollout(c.N, None, None, 0)
    bad = _diff(c.philox(), again)
    assert not bad, "%s: two identical rollouts differ in %s" % (c.tag, bad)
    if c.N > 1:
        k = 33 if c.N < 2 * CTA else CTA * (c.N // (2 * CTA)) + 45          # never a multiple of 128
        lo, hi = c.rollout(k, None, None, 0), c.rollout(c.N - k, None, None, k)
        assert not _diff(c.philox(), lo, slice(0, k)), "%s: shard [0, %d) differs" % (c.tag, k)
        assert not _diff(c.philox(), hi, slice(k, None)), "%s: shard [%d, %d) with lane0 = %d differs" % (
            c.tag, k, c.N, k)


# ------------------------------------------------------------------------------------------- in-kernel Philox streams
@pytest.mark.parametrize("env,H", [(e, h) for e in ENVS for h in HIDDEN])
def test_philox_high_lane(dev, env, H):
    """N = 77 at lane0 = 2^32 - 40 (the lane counter's high word changes inside the CTA): the NULL-noise rollout equals
    the rollout fed fill_noise blocks at that lane0, and the blocks equal oracle.philox (uniform bit-exact, normal
    5e-5)."""
    N, T, mpl = 77, 40, 17
    c = Case(dev, env, H, N, T, mpl, tag="%s-%d lane0=2^32-40" % (env, H))
    eps, rr = _noise(dev, c.env64, N, T, LANE0_HIGH)
    inj = c.rollout(N, eps, rr, LANE0_HIGH)
    kern = c.rollout(N, None, None, LANE0_HIGH)
    bad = _diff(inj, kern)
    assert not bad, "%s: in-kernel Philox differs from the injected blocks in %s" % (c.tag, bad)
    assert _diff(c.b, kern), "%s: lane0 does not change the noise" % c.tag
    A2 = c.A + (c.A & 1)                                            # Box-Muller pairs
    ref_eps = PH.normal_from_raw(PH.raw_block(T, 0, A2, N, LANE0_HIGH, SEED, ITER, 0))[:, :c.A]
    np.testing.assert_allclose(eps.cpu().numpy(), ref_eps, rtol=5e-5, atol=2e-5)
    raw = PH.raw_block(T + 1, 0, c.env64.K, N, LANE0_HIGH, SEED, ITER, 1)
    if c.env64.noise_kind == "uniform":
        assert np.array_equal(rr.cpu().numpy(), PH.uniform_from_raw(raw))
    else:
        np.testing.assert_allclose(rr.cpu().numpy(), PH.normal_from_raw(raw), rtol=5e-5, atol=2e-5)
    # the replay of this rollout through the stand-alone kernels, on the injected blocks
    c.b, c.eps, c.rr, c.traj = inj, eps, rr, inj.to_numpy()
    _check_replay(c)
    _check_forward(c)
    _check_action(c.traj["act"], c.traj["mean"], c.traj["log_std"], eps.cpu().numpy().transpose(1, 0, 2), c.tag)


@pytest.mark.parametrize("env", ENVS)
def test_env_reset_philox(dev, env):
    """b200rl_env_reset with reset_raw = NULL at rows 0 and 7 equals the reset from the fill_noise stream-1 block of
    that row, at lane0 0 and 2^32 - 40."""
    ops, L = _ops(), _L()
    env64 = _oracle_env(env)
    kind = L.ENV_KINDS[env]
    nk = L.NOISE_UNIFORM if env64.noise_kind == "uniform" else L.NOISE_NORMAL
    N = 77
    for lane0 in (0, LANE0_HIGH):
        for row in (0, 7):
            blk = torch.empty((1, env64.K, N), dtype=torch.float32, device=dev)
            ops.fill_noise(blk, 1, row, env64.K, N, lane0, nk, SEED, ITER, 1)
            s1 = torch.full((env64.S, N), float("nan"), device=dev)
            o1 = torch.full((env64.O, N), float("nan"), device=dev)
            s2, o2 = s1.clone(), o1.clone()
            ops.env_reset(kind, N, s1, o1, blk.view(env64.K, N), SEED, ITER, 0, lane0)
            ops.env_reset(kind, N, s2, o2, None, SEED, ITER, row, lane0)
            assert torch.equal(_bits(s1), _bits(s2)) and torch.equal(_bits(o1), _bits(o2)), (env, lane0, row)
            assert not torch.isnan(s1).any()
            if row == 7:
                assert not torch.equal(_bits(s2), _bits(s_row0)), (env, lane0)
            else:
                s_row0 = s2


@pytest.mark.parametrize("H", HIDDEN)
@pytest.mark.parametrize("O,A", [(2, 2), (4, 1), (3, 1), (6, 1), (13, 2), (20, 3)])
def test_get_actions_philox(dev, O, A, H):
    """b200rl_policy_get_actions with eps = NULL, row 3, lane0 = 2^32 - 40 equals the call fed the fill_noise stream-0
    block of that row, and its act is mean + exp(log_std) eps within 2 ulps."""
    ops, L = _ops(), _L()
    n = 333
    dims = P.Dims(O, (H, H), A)
    rng = np.random.RandomState(7 * O + A + H)
    theta = P.init_params(dims, rng) + rng.randn(dims.P) * 0.05
    theta[-A:] = -0.5 + 0.1 * np.arange(A)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    obs = torch.tensor(rng.randn(O, n) * 2.0, dtype=torch.float32, device=dev)
    eps = torch.empty((1, A, n), dtype=torch.float32, device=dev)
    ops.fill_noise(eps, 1, 3, A, n, LANE0_HIGH, L.NOISE_NORMAL, SEED, ITER, 0)
    out = []
    for e in (eps.view(A, n), None):
        act = torch.full((A, n), float("nan"), device=dev)
        mean, ls = act.clone(), torch.full((A,), float("nan"), device=dev)
        ops.policy_get_actions(th32, O, H, H, A, MIN_STD, obs, n, e, SEED, ITER, 3, LANE0_HIGH, act, mean, ls)
        out.append((act, mean, ls))
    for x, y in zip(*out):
        assert torch.equal(_bits(x), _bits(y))
    act, mean, ls = (t.cpu().numpy() for t in out[1])
    _check_action(act, mean, ls, eps.view(A, n).cpu().numpy(), "get_actions O%dA%dH%d" % (O, A, H))
    mu, _ = P.forward(th32.double().cpu().numpy(), obs.cpu().numpy().T.astype(np.float64), dims)
    np.testing.assert_allclose(mean.T, mu, rtol=2e-5, atol=2e-6)


# ------------------------------------------------------------------------------------------- edges
EDGE_NETS = [("cartpole", 32), ("hopper", 64), ("pendulum", 32)]
EDGE_TM = [(1, 17), (40, 1), (40, 40), (40, 57)]


@pytest.mark.parametrize("T,mpl", EDGE_TM, ids=["T%d-mpl%d" % p for p in EDGE_TM])
@pytest.mark.parametrize("env,H", EDGE_NETS, ids=["%s-%d" % p for p in EDGE_NETS])
def test_edges(dev, env, H, T, mpl):
    """T = 1; max_path_length 1 (every sample ends a path, none is cut); = T; > T (a lane's last path is cut unless the
    env is done on its last step)."""
    L = _L()
    c = Case(dev, env, H, 333, T, mpl)
    fl, ts = c.traj["flags"], c.traj["tstep"]
    end = (fl & L.FLAG_END) != 0
    cut = (fl & L.FLAG_CUT) != 0
    done = (fl & L.FLAG_DONE) != 0
    assert end[-1].all() and np.array_equal(cut[-1], ~done[-1] & (ts[-1] + 1 < mpl))
    if mpl == 1:
        assert end.all() and not cut.any() and not ts.any()
    if mpl >= T:
        assert not cut[:-1].any() and np.array_equal(end[:-1], done[:-1])
    _check_bookkeeping(c)
    _check_log_std(c)
    _check_forward(c)
    _check_get_actions(c)
    _check_action(c.traj["act"], c.traj["mean"], c.traj["log_std"], c.eps.cpu().numpy().transpose(1, 0, 2), c.tag)
    _check_replay(c)
    if env != "hopper":
        _check_env_oracle(c)
    assert not _diff(c.b, c.philox()), c.tag


def test_paths_at_the_tstep_limit(dev):
    """Pendulum is never done: with max_path_length 65 535 and T = 65 537, tstep counts 0 .. 65 534, END falls at
    t = 65 534 (a whole path, no CUT), and the second path ends cut by the buffer at t = 65 536."""
    L = _L()
    N, T, mpl = 33, 65537, 65535
    c = Case(dev, "pendulum", 32, N, T, mpl)
    fl, ts = c.traj["flags"], c.traj["tstep"]
    exp_ts = np.concatenate([np.arange(65535), [0, 1]]).astype(np.uint16)
    exp_fl = np.zeros(T, np.uint8)
    exp_fl[65534] = L.FLAG_END
    exp_fl[65536] = L.FLAG_END | L.FLAG_CUT
    assert np.array_equal(ts, np.repeat(exp_ts[:, None], N, axis=1))
    assert np.array_equal(fl, np.repeat(exp_fl[:, None], N, axis=1))
    _check_bookkeeping(c)
    _check_forward(c)
    _check_get_actions(c)


CLAMP_LOG_STD = dict(hopper=(-0.5, -0.3, -0.1), half_cheetah=(-0.5, -0.3, -0.1, -0.2, -0.6, -0.1))
CLAMP_CASES = [(e, h) for e in CLAMP_LOG_STD for h in HIDDEN]
CLAMP_IDS = [str(h) if e == "hopper" else "%s-%d" % (e, h) for e, h in CLAMP_CASES]   # Hopper keeps its original ids


@pytest.mark.parametrize("env,H", CLAMP_CASES, ids=CLAMP_IDS)
def test_min_std_clamp(dev, env, H):
    """min_std = e^-0.35 with log_std CLAMP_LOG_STD[env]: the clamp binds for the components below -0.35 only (Hopper:
    the first; HalfCheetah: one in each Philox chunk of its action noise, eps[0..3] and eps[4..5]).  log_std_out, the
    forward and the action noise use the clamped std."""
    min_std = float(np.exp(-0.35))
    param = np.array(CLAMP_LOG_STD[env])
    c = Case(dev, env, H, 77, 40, 17, min_std=min_std, log_std=param)
    ls = c.traj["log_std"]
    binds = param < -0.35
    assert binds.any() and not binds.all()
    assert np.all(np.abs(ls[binds] + 0.35) < 1e-6) and np.array_equal(ls[~binds], param[~binds].astype(np.float32))
    _check_log_std(c)
    _check_forward(c)
    _check_get_actions(c)
    _check_action(c.traj["act"], c.traj["mean"], ls, c.eps.cpu().numpy().transpose(1, 0, 2), c.tag)
    _check_replay(c)


def test_rejected_calls_write_nothing(dev):
    """max_path_length 65 536 (tstep would overflow uint16), hidden (32, 64) and hidden 48 are errors, and the output
    buffers keep their contents."""
    ops, L = _ops(), _L()
    c = Case(dev, "cartpole", 32, 77, 8, 5)
    th64 = torch.zeros(P.Dims(4, (64, 64), 1).P, dtype=torch.float32, device=dev)
    th48 = torch.zeros(P.Dims(4, (48, 48), 1).P, dtype=torch.float32, device=dev)
    for th, h1, h2, mpl in ((c.th32, 32, 32, 65536), (th64, 32, 64, 5), (th48, 48, 48, 5)):
        b = ops.LaneBatch(4, 1, 77, 8, dev)
        _poison(b)
        ref = ops.LaneBatch(4, 1, 77, 8, dev)
        _poison(ref)
        with pytest.raises(L.B200RLError):
            ops.rollout(L.ENV_CARTPOLE, th, h1, h2, MIN_STD, b, mpl, None, None, SEED, ITER, 0)
        torch.cuda.synchronize()
        assert not _diff(b, ref), (h1, h2, mpl)
