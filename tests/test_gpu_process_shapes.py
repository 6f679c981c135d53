"""GPU: process_samples and the LinearFeatureBaseline fit against the float64 oracle at every compiled obs_dim, at batch
sizes that run the grid-stride loops.

Kernels: lfb_predict_kernel, gae_scan_kernel (b200rl_process_samples), center_adv_kernel (b200rl_center_advantages),
lfb_gram_reg_kernel / lfb_gram_tile_kernel (b200rl_lfb_gram) and lfb_solve_kernel (b200rl_lfb_solve).  The batches are
synthetic lane batches (random paths, observations with 5 % of entries beyond the +-10 clip, seeded baseline weights of
realistic size) for obs_dim O in {2, 3, 4, 6, 13, 20} and three modes:
  unmasked    every lane's last path ends with the buffer (no FLAG_CUT)
  drop_cut    the last paths that do not end with the buffer carry FLAG_CUT and process_samples(drop_cut_paths=True)
              drops them (FLAG_MASKED, adv = 0, left out of every statistic, of the centering and of the Gram)
  cut         the same cut paths, kept (whole_paths=False)
Geometries, N lanes x T steps, from the SM count n_sm of the device:
  1x7         one lane (scalar loops only)
  33x37       B % 4 != 0, N % 32 != 0: scalar predict and Gram loops, unstaged (register) scan
  96x41       B % 4 == 0, N % 32 == 0: 128-bit predict and Gram loops, staged (cp.async) scan
  sweep       T = 500, N = the multiple of 32 with B >= 2.5 x 16 384 n_sm.  At n_sm = 132 (H100 SXM): N = 10 816,
              B = 5 408 000 = 2.5 grid-stride sweeps of the predict kernel (16 n_sm CTAs x 256 threads x 4 samples),
              107 samples accumulated in float32 registers per thread of the register Gram (3 n_sm CTAs x 128 threads,
              13 iterations of its two-vector loop), 106-107 128-sample tiles per CTA of the tile Gram (3 n_sm CTAs).
              Modes unmasked and drop_cut.
  sweep-5     N - 5 lanes and T = 501 (B odd: 5 416 311 at n_sm = 132): the same loop counts through the scalar
              predict / Gram loops (10 sweeps of one sample per thread) and the unstaged scan.  Mode drop_cut.
Every reference is the float64 oracle (oracle/sampler.py, pinned to the reference's own process_samples by
tests/test_oracle_golden.py), evaluated in lane chunks so that the large cases fit in host memory.  One grid case (device
batch, host arrays, oracle results) is alive at a time: the `case` fixture is module scoped and parametrised, so pytest
runs all tests of a case together.

Tolerances, and what an H100 80GB HBM3 (132 SMs, 400 W power limit) measured:
  predict     within 1 float32 ulp of float32(F w) + 1e-13 sum_j |w_j phi_j| (the kernel sums in float64, rounds once);
              measured <= 1 ulp
  scan        the oracle is fed the device's float32 baseline, so both run the same float64 recurrence on identical
              inputs: ret and adv within 1 ulp + 1e-12 of the suffix sum of the recurrence's operands |r| + 2 |b|;
              the 13 sums and 4 maxima to 1e-10 of the sum of absolute terms; NumTrajs, count and FLAG_MASKED exactly
  centering   rtol 1e-6, atol 1e-6 max|adv|; masked samples exactly 0
  Gram        |dG_ij| <= 1e-5 (|F| |F|^T)_ij, element-wise (entries such as sum o_k ret cancel); measured <= 1.4e-7
              (float32 register Gram, O <= 4) and <= 5e-14 (float64 tile Gram, O >= 6)
  solve       info == (1e-5, 0, 1) and backward error <= 1e-12 (|A| |w| + |b|) at every d = 2 O + 4; measured <= 1e-16
The whole module ran in 3 3/4 minutes there.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import policy as P          # noqa: E402
from oracle import sampler as S         # noqa: E402
from test_gpu_update_shapes import dev, n_sm  # noqa: E402,F401

OBS_DIMS = (2, 3, 4, 6, 13, 20)
GEOMS = ("1x7", "33x37", "96x41", "sweep", "sweep-5")
MODES = ("unmasked", "drop_cut", "cut")
SWEEP_MODES = {"sweep": ("unmasked", "drop_cut"), "sweep-5": ("drop_cut",)}      # (host oracle time)
CASES = [(O, g, m) for O in OBS_DIMS for g in GEOMS for m in MODES if m in SWEEP_MODES.get(g, MODES)]
CENTERING = ((1, 0), (0, 1), (1, 1))                       # (center_adv, positive_adv); (1, 1) is ERWR's setting
GAMMA_LAMBDA = ((0.99, 0.95), (1.0, 1.0), (0.99, 0.0))
DISCOUNT, GAE_LAMBDA = GAMMA_LAMBDA[0]
REG = 1e-5
CHUNK = 1 << 24                                            # float64 feature entries per host chunk of lanes


def _ops():
    from rllab_b200 import ops
    return ops


def _L():
    from rllab_b200 import _lib
    return _lib


def _sweep_lanes(n_sm):
    """Lanes of the `sweep` geometry: the multiple of 32 with 500 N >= 2.5 x 16 384 n_sm."""
    need = -(-int(2.5 * 16384 * n_sm) // 500)
    return -(-need // 32) * 32


def _geometry(geom, n_sm):
    if geom == "sweep":
        return _sweep_lanes(n_sm), 500
    if geom == "sweep-5":
        return _sweep_lanes(n_sm) - 5, 501
    N, T = geom.split("x")
    return int(N), int(T)


def _weights(O, seed):
    """Baseline weights of the size a fit produces: O(1) linear terms, small quadratic ones, a time trend."""
    rng = np.random.default_rng([seed, O, 7])
    return np.concatenate([rng.standard_normal(O) * 0.5, rng.standard_normal(O) * 0.05,
                           np.array([3.0, -0.8, 0.05, 5.0]) * (1.0 + 0.1 * rng.standard_normal(4))])


class Case(object):
    """A synthetic lane batch on the device and its float32 host arrays.  Paths end with probability p_end per step;
    with mode != "unmasked" each lane's last path is cut by the end of the buffer (FLAG_END | FLAG_CUT) unless it ends
    there anyway.  In drop_cut mode lane 0 always keeps a whole path, so no batch is empty; `long_lane0` makes lane 0 one
    path over the whole buffer instead.  `memo` caches the device outputs and the oracle's results."""

    def __init__(self, dev, O, N, T, mode, seed=0, p_end=0.06, long_lane0=False):
        ops, L = _ops(), _L()
        self.O, self.N, self.T, self.mode = O, N, T, mode
        self.drop = mode == "drop_cut"
        self.memo = {}
        rng = np.random.default_rng([seed, O, N, T])
        obs = rng.standard_normal((O, T, N), dtype=np.float32)
        obs *= 3.0
        big = rng.random((O, T, N), dtype=np.float32) < 0.05
        nb = int(big.sum())
        obs[big] = (np.sign(rng.standard_normal(nb)) * rng.uniform(10.0, 30.0, nb)).astype(np.float32)
        del big
        rew = rng.random((T, N), dtype=np.float32) * np.float32(2.0) - np.float32(0.5)
        ends = rng.random((T, N)) < p_end
        if long_lane0:
            ends[:, 0] = False
        elif self.drop and T > 2:
            ends[T // 2, 0] = True
        flags = np.where(ends, L.FLAG_END, 0).astype(np.uint8)
        flags[T - 1] |= L.FLAG_END
        if mode != "unmasked":
            flags[T - 1] |= np.where(ends[T - 1], 0, L.FLAG_CUT).astype(np.uint8)
        tstep = np.zeros((T, N), np.uint16)
        for t in range(1, T):
            tstep[t] = np.where(flags[t - 1] & L.FLAG_END, 0, tstep[t - 1] + 1)
        self.obs, self.rew, self.flags, self.tstep = obs, rew, flags, tstep
        self.w = _weights(O, seed)
        b = ops.LaneBatch(O, 1, N, T, dev)
        b.obs.copy_(torch.from_numpy(obs))
        b.rew.copy_(torch.from_numpy(rew))
        b.tstep.copy_(torch.from_numpy(tstep.view(np.int16)).view(torch.uint16))
        b.log_std.zero_()
        self.flags_dev = torch.from_numpy(flags).to(dev)
        self.b = b
        torch.cuda.synchronize()

    def traj(self, rew=None):
        return dict(rew=self.rew if rew is None else rew, flags=self.flags, tstep=self.tstep, log_std=np.zeros(1))

    def valid(self):
        return S.valid_mask(dict(flags=self.flags), self.drop)

    def chunks(self, rows):
        n = max(1, CHUNK // (rows * self.T))
        for n0 in range(0, self.N, n):
            yield slice(n0, min(self.N, n0 + n))

    def out(self):
        if "out" not in self.memo:
            self.memo["out"] = _pipeline(self, DISCOUNT, GAE_LAMBDA)
        return self.memo["out"]

    def release(self):
        self.b = self.flags_dev = None
        self.memo.clear()


def _pipeline(c, discount, gae_lambda):
    """One pass of what the sampler runs per iteration: process_samples with c.w, the three centerings (each from the
    raw advantages), the Gram of the normal equations and the device solve.  Host copies of every output."""
    ops, L = _ops(), _L()
    b, dev = c.b, c.b.device
    b.flags.copy_(c.flags_dev)
    w = torch.tensor(c.w, dtype=torch.float64, device=dev)
    ops.process_samples(b, w, discount, gae_lambda, drop_cut_paths=c.drop)
    out = dict(base=b.base.cpu().numpy(), adv=b.adv.cpu().numpy(), ret=b.ret.cpu().numpy(),
               flags=b.flags.cpu().numpy(), sums=b.sums.cpu().numpy().copy(), maxs=b.maxs.cpu().numpy().copy())
    raw = b.adv.clone()
    for ce, po in CENTERING:
        b.adv.copy_(raw)
        ops.center_advantages(b, ce, po)
        out["adv%d%d" % (ce, po)] = b.adv.cpu().numpy()
    b.adv.copy_(raw)
    gram = torch.empty((b.n_gram,), dtype=torch.float64, device=dev)
    ops.lfb_gram(b, gram)
    w_out = torch.empty((2 * c.O + 4,), dtype=torch.float64, device=dev)
    info = torch.zeros((3,), dtype=torch.float64, device=dev)
    ops.lfb_solve(c.O, gram, REG, w_out, info)
    out.update(gram=gram.cpu().numpy(), w=w_out.cpu().numpy(), info=info.cpu().numpy())
    return out


def _assert_f32(got, ref64, extra, what):
    """|got - float32(ref64)| <= 1 float32 ulp + extra, element-wise; returns the worst error in ulps."""
    r32 = np.asarray(ref64, np.float64).astype(np.float32)
    ulp = np.spacing(np.abs(r32)).astype(np.float64)
    err = np.abs(np.asarray(got, np.float64) - r32.astype(np.float64))
    bad = err > ulp + extra
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, err / (ulp + extra), 0.0)), err.shape)
        raise AssertionError("%s: %d of %d samples beyond 1 ulp + allowance; worst at %s: got %r, oracle %r (ulp %.3g, "
                             "allowance %.3g)" % (what, int(bad.sum()), bad.size, i, float(np.asarray(got)[i]),
                                                  float(ref64[i]), ulp[i], np.broadcast_to(extra, err.shape)[i]))
    return float(np.max(err / ulp)) if err.size else 0.0


def _unpack(packed, d1):
    G = np.zeros((d1, d1))
    G[np.triu_indices(d1)] = packed
    return G + G.T - np.diag(np.diag(G))


# ------------------------------------------------------------------------------------------- checks shared by the tests
def _check_predict(c, base):
    """b = float32(phi(o, t) . w) against the oracle's float64 F w, lane chunk by lane chunk."""
    worst = 0.0
    for sl in c.chunks(2 * c.O + 4):
        F = S.lfb_features_lanes(c.obs[:, :, sl], c.tstep[:, sl])
        exact = np.tensordot(c.w, F, axes=(0, 0))
        scale = np.tensordot(np.abs(c.w), np.abs(F), axes=(0, 0))
        worst = max(worst, _assert_f32(base[:, sl], exact, 1e-13 * scale, "base"))
    return worst


def _scan_oracle(c, out, discount, gae_lambda):
    """The oracle's process_samples on the device's own float32 baseline, and the suffix sums of |r| + 2 |b| over each
    path (the operands of the remaining recurrence steps: r_t, discount * b_{t+1}, b_t)."""
    key = ("scan", discount, gae_lambda)
    if key not in c.memo:
        ref = S.process_samples_lanes(c.traj(), None, discount, gae_lambda, center_adv=False, drop_cut=c.drop,
                                      base=out["base"])
        absr = np.abs(c.rew.astype(np.float64)) + 2.0 * np.abs(out["base"].astype(np.float64))
        suf = S.process_samples_lanes(c.traj(absr), None, 1.0, 1.0, center_adv=False)["ret"]
        c.memo[key] = (ref, suf)
    return c.memo[key]


def _check_scan(c, out, discount, gae_lambda):
    """ret / raw adv per sample, FLAG_MASKED, and the 13 sums + 4 maxima behind the tabular statistics."""
    L = _L()
    ref, suf = _scan_oracle(c, out, discount, gae_lambda)
    valid = ref["valid"]
    exp_flags = c.flags | np.where(valid, 0, L.FLAG_MASKED).astype(np.uint8) if c.drop else c.flags
    assert np.array_equal(out["flags"], exp_flags), "FLAG_MASKED differs on %d samples" % int(
        (out["flags"] != exp_flags).sum())
    u_ret = _assert_f32(out["ret"], ref["ret"], 1e-12 * suf, "ret")
    u_adv = _assert_f32(out["adv"], ref["adv_raw"], 1e-12 * suf, "adv")
    starts = (c.tstep == 0) & valid
    a, r, e = ref["adv_raw"][valid], ref["ret"][valid], suf[valid]
    bb = out["base"].astype(np.float64)[valid]
    res = r - bb
    rs, us, es = ref["ret"][starts], ref["und"][starts], suf[starts]
    zero = np.zeros(1)
    # slot: (terms, propagated allowance per term) -- the allowance carries the float64 recurrence's operands
    terms = {0: (a, e), 1: (a * a, 2 * np.abs(a) * e), 4: (rs, es), 5: (us, es), 6: (us * us, 2 * np.abs(us) * es),
             7: (r, e), 8: (r * r, 2 * np.abs(r) * e), 9: (bb, zero), 10: (bb * bb, zero), 11: (res, e),
             12: (res * res, 2 * np.abs(res) * e)}
    s = out["sums"]
    assert s[2] == valid.sum(), (s[2], valid.sum())                     # count: exactly
    assert s[3] == starts.sum(), (s[3], starts.sum())                   # NumTrajs: exactly
    worst = 0.0
    for k, (x, ex) in terms.items():
        tol = 1e-10 * (np.sum(np.abs(x)) + np.sum(ex))
        err = abs(s[k] - np.sum(x))
        assert err <= tol, "sum %d: device %r, oracle %r, |diff| %.3g > %.3g" % (k, s[k], np.sum(x), err, tol)
        worst = max(worst, err / (1e-10 * np.sum(np.abs(x)) or 1.0))
    m = out["maxs"]
    for k, x, ex in ((0, us, es), (1, -us, es), (2, -a, e), (3, a, e)):
        tol = 1e-10 * (np.max(np.abs(x)) + np.max(ex))
        assert abs(m[k] - np.max(x)) <= tol, "max %d: device %r, oracle %r" % (k, m[k], np.max(x))
    return u_ret, u_adv, worst


def _check_gram(c, out):
    """The packed Gram of [features | ret] over the valid samples against float64 products of float64 features (the
    device's own float32 returns), |dG_ij| <= 1e-5 (|F| |F|^T)_ij."""
    d1 = 2 * c.O + 5
    valid = c.valid()
    G = np.zeros((d1, d1))
    Ga = np.zeros((d1, d1))
    for sl in c.chunks(d1):
        F = S.lfb_features_lanes(c.obs[:, :, sl], c.tstep[:, sl])
        F = np.concatenate([F, out["ret"][None, :, sl].astype(np.float64)], axis=0).reshape(d1, -1)
        F = F[:, valid[:, sl].reshape(-1)]
        G += F @ F.T
        np.abs(F, out=F)
        Ga += F @ F.T
    iu = np.triu_indices(d1)
    err = np.abs(out["gram"] - G[iu])
    rel = err / Ga[iu]
    bad = rel > 1e-5
    assert not bad.any(), "Gram: %d of %d entries beyond 1e-5 of sum |f_i f_j|; worst (%d, %d): %.3g" % (
        int(bad.sum()), bad.size, iu[0][np.argmax(rel)], iu[1][np.argmax(rel)], rel.max())
    return float(rel.max())


# ------------------------------------------------------------------------------------------- the case grid
@pytest.fixture(scope="module", params=CASES, ids=["O%d-%s-%s" % p for p in CASES])
def case(request, dev, n_sm):
    O, geom, mode = request.param
    c = Case(dev, O, *_geometry(geom, n_sm), mode)
    c.geom = geom
    if geom == "sweep":
        B = c.N * c.T
        print("sweep at n_sm=%d: N=%d B=%d, %.2f predict sweeps, %.1f samples per register-Gram thread, %.1f tiles per "
              "tile-Gram CTA" % (n_sm, c.N, B, B / (16 * n_sm * 256 * 4), B / (3 * n_sm * 128),
                                 -(-B // 128) / (3 * n_sm)))
    yield c
    c.release()
    torch.cuda.empty_cache()


def test_predict(case):
    """lfb_predict_kernel<OT> (OT 2, 3, 4, 13, 20; the runtime-O loop for 6) on the 128-bit and the scalar path."""
    c = case
    worst = _check_predict(c, c.out()["base"])
    print("O=%d %s %s B=%d: base within %.2f float32 ulp" % (c.O, c.geom, c.mode, c.N * c.T, worst))


def test_scan(case):
    c = case
    u_ret, u_adv, worst = _check_scan(c, c.out(), DISCOUNT, GAE_LAMBDA)
    print("O=%d %s %s: ret %.2f ulp, adv %.2f ulp, sums %.3g of 1e-10 x sum|terms|" % (c.O, c.geom, c.mode, u_ret,
                                                                                          u_adv, worst))


def test_center_advantages(case):
    """center_adv_kernel with (center, positive) in {(1, 0), (0, 1), (1, 1)} against the oracle's centering of the same
    advantages; masked samples stay exactly 0."""
    c = case
    out = c.out()
    for ce, po in CENTERING:
        ref = S.process_samples_lanes(c.traj(), None, DISCOUNT, GAE_LAMBDA, center_adv=bool(ce), positive_adv=bool(po),
                                      drop_cut=c.drop, base=out["base"])
        got = out["adv%d%d" % (ce, po)]
        assert np.all(got[~ref["valid"]] == 0.0), (ce, po)
        np.testing.assert_allclose(got, ref["adv"], rtol=1e-6, atol=1e-6 * np.abs(ref["adv"]).max(),
                                   err_msg="center=%d positive=%d" % (ce, po))


def test_gram(case):
    """lfb_gram_reg_kernel<O> (O <= 4; 128-bit loop if B % 4 == 0, scalar otherwise) and lfb_gram_tile_kernel<O>
    (O 6 / 13 / 20), masked samples left out."""
    c = case
    worst = _check_gram(c, c.out())
    print("O=%d %s %s B=%d: Gram within %.3g of sum |f_i f_j|" % (c.O, c.geom, c.mode, c.N * c.T, worst))


def test_pipeline_bit_identical(case):
    """A second pass over the same batch reproduces base, adv (raw and centred), ret, flags, the sums, the Gram and w
    bit for bit (fixed-order reductions everywhere)."""
    c = case
    first = c.out()
    again = _pipeline(c, DISCOUNT, GAE_LAMBDA)
    for k, v in first.items():
        assert np.array_equal(v, again[k]), k


# ------------------------------------------------------------------------------------------- the scan's parameters
@pytest.mark.parametrize("mode", ["drop_cut", "cut"])
@pytest.mark.parametrize("geom", ["33x37", "96x41"])
@pytest.mark.parametrize("discount,gae_lambda", GAMMA_LAMBDA, ids=["g%g-l%g" % gl for gl in GAMMA_LAMBDA])
def test_scan_discount_settings(dev, n_sm, discount, gae_lambda, geom, mode):
    """gamma = lambda = 1 (undiscounted returns, advantages = return-to-go - b) and lambda = 0 (one-step TD errors) on
    the staged and the unstaged scan."""
    c = Case(dev, 3, *_geometry(geom, n_sm), mode, seed=2)
    _check_scan(c, _pipeline(c, discount, gae_lambda), discount, gae_lambda)
    c.release()


_LONG = {}


def _long_case(dev, N, O):
    """T = max_path_length = 65 535 (the uint16 bound of tstep): lane 0 is one whole path, so tstep reaches 65 534 and
    (t/100)^3 ~ 2.8e8; the other lanes end a path with probability 1e-5 per step."""
    if (N, O) not in _LONG:
        for c in _LONG.values():
            c.release()
        _LONG.clear()
        _LONG[(N, O)] = Case(dev, O, N, 65535, "unmasked", seed=3, p_end=1e-5, long_lane0=True)
    return _LONG[(N, O)]


@pytest.mark.parametrize("discount,gae_lambda", GAMMA_LAMBDA, ids=["g%g-l%g" % gl for gl in GAMMA_LAMBDA])
@pytest.mark.parametrize("N,O", [(32, 4), (1, 13)], ids=["N32-O4", "N1-O13"])
def test_max_path_length_65535(dev, N, O, discount, gae_lambda):
    """Predict, scan and Gram at the longest path the uint16 step index allows."""
    c = _long_case(dev, N, O)
    assert int(c.tstep.max()) == 65534
    out = _pipeline(c, discount, gae_lambda)
    _check_predict(c, out["base"])
    _check_scan(c, out, discount, gae_lambda)
    worst = _check_gram(c, out)
    print("N=%d O=%d T=65535: Gram within %.3g of sum |f_i f_j|" % (N, O, worst))


# ------------------------------------------------------------------------------------------- the solve
def _solve(dev, O, G):
    ops = _ops()
    d1 = 2 * O + 5
    gram = torch.tensor(G[np.triu_indices(d1)], dtype=torch.float64, device=dev)
    w = torch.empty((d1 - 1,), dtype=torch.float64, device=dev)
    info = torch.zeros((3,), dtype=torch.float64, device=dev)
    ops.lfb_solve(O, gram, REG, w, info)
    return w.cpu().numpy(), tuple(float(x) for x in info.cpu().numpy())


@pytest.mark.parametrize("cond", [1e2, 1e8, 1e12])
@pytest.mark.parametrize("O", OBS_DIMS)
def test_solve_synthetic(dev, O, cond):
    """lfb_solve_kernel at d = 8, 10, 12, 16, 30, 44 (44 = LFB_DMAX) on SPD systems with eigenvalues 1 .. cond: one
    attempt, and a backward error ||(A + reg I) w - b|| <= 1e-12 (||A|| ||w|| + ||b||)."""
    d = 2 * O + 4
    rng = np.random.RandomState(100 * O + int(np.log10(cond)))
    Q, _ = np.linalg.qr(rng.randn(d, d))
    A = (Q * np.logspace(0.0, np.log10(cond), d)) @ Q.T
    A = 0.5 * (A + A.T)
    b = A @ rng.randn(d) + rng.randn(d)
    G = np.zeros((d + 1, d + 1))
    G[:d, :d], G[:d, d], G[d, :d], G[d, d] = A, b, b, 1.0
    w, info = _solve(dev, O, G)
    assert info == (REG, 0.0, 1.0)
    Ar = A + REG * np.eye(d)
    back = np.linalg.norm(Ar @ w - b) / (np.linalg.norm(Ar, 2) * np.linalg.norm(w) + np.linalg.norm(b))
    assert back <= 1e-12, back
    print("d=%d cond %.0e: backward error %.3g" % (d, cond, back))


def test_solve_retry_and_failure_at_dmax(dev):
    """d = 44: a Gram that is positive definite only from reg 1e-3 on takes the third attempt (linear_feature_baseline.py
    :30-37); a NaN in the Gram exhausts all five and leaves w exactly zero (no baseline) with ok = 0."""
    O = 20
    d1 = 2 * O + 5
    X = np.random.RandomState(3).randn(d1, 3)
    G = X @ X.T - 2e-4 * np.eye(d1)
    w, info = _solve(dev, O, G)
    assert info == (1e-3, 2.0, 1.0), info
    A = G[:-1, :-1] + info[0] * np.eye(d1 - 1)
    back = np.linalg.norm(A @ w - G[:-1, -1]) / (np.linalg.norm(A, 2) * np.linalg.norm(w) + np.linalg.norm(G[:-1, -1]))
    assert back <= 1e-12, back
    G[5, 7] = G[7, 5] = np.nan
    w, info = _solve(dev, O, G)
    assert info[1:] == (5.0, 0.0), info
    assert np.all(w == 0.0)


# (env, hidden, lanes, horizon): bench.py / examples horizons.  DoublePendulum runs 40 steps: under the random initial
# policy (torques up to +-50) its angular velocities overflow float32 after ~70 steps, and the fit needs finite inputs.
FIT_ENVS = [("point", 32, 4096, 100), ("cartpole", 32, 2048, 200), ("pendulum", 32, 2048, 200),
            ("cartpole_swingup", 32, 4096, 100), ("double_pendulum", 32, 4096, 40), ("swimmer", 32, 512, 500),
            ("hopper", 32, 512, 500), ("hopper", 64, 512, 500), ("half_cheetah", 32, 512, 500),
            ("half_cheetah", 64, 512, 500)]


@pytest.mark.parametrize("env_name,hidden,lanes,T", FIT_ENVS, ids=["%s-%d" % (e[0], e[1]) for e in FIT_ENVS])
def test_lfb_fit_on_rollout(dev, env_name, hidden, lanes, T):
    """The whole baseline fit on one device rollout at the env's training horizon (max_path_length = T, cut paths
    dropped): lfb_gram + lfb_solve.  Checks, with s = max |ret| over the valid samples:
      * one attempt, ok (a failed fit would silently zero the baseline);
      * the solve alone: F w against lfb_fit_normal (the reference's lstsq) on the device's own Gram, to 1e-6 s;
      * end to end: F w against lfb_fit_normal on float64 features of the valid samples, to 1e-5 s -- the difference
        between the two is the Gram's.
    Measured on an H100 80GB HBM3 (400 W limit), solve alone / end to end, condition number of A + reg I:
      point 4.3e-14 / 1.0e-7 (4e6), cartpole 3.9e-14 / 4.4e-7 (2e7), pendulum 1.2e-14 / 6.7e-7 (2e10),
      cartpole_swingup 8.5e-14 / 7.5e-7 (1e7), double_pendulum 9.9e-14 / 3.2e-13 (2e14), swimmer 7.0e-12 / 7.4e-12
      (6e13), hopper-32 5.9e-9 / 6.5e-9 (5e14), hopper-64 3.1e-7 / 4.8e-7 (6e14), half_cheetah-32 9.0e-12 / 2.6e-11
      (4e14), half_cheetah-64 3.2e-11 / 3.2e-11 (3e14; 700 W); one attempt everywhere.  HalfCheetah's obs holds an
      identically zero column (comY), so two feature columns are zero and A + reg I has the eigenvalue reg exactly.  The two
      solves are backward stable on the same system, so their gap follows the conditioning: 1e-8 holds below κ ~ 1e14,
      Hopper's κ ~ 6e14 takes it to 3.1e-7.  With the float32 tile Gram this module was written against, Hopper's end to
      end figure was 2.8e-4 (hopper-32) and 4.8e-2 (hopper-64), and TRPO's first Hopper-64 fit needed reg 1e-4."""
    ops, L = _ops(), _L()
    info = L.env_info(L.ENV_KINDS[env_name])
    O, A = info["obs_dim"], info["act_dim"]
    dims = P.Dims(O, (hidden, hidden), A)
    theta = P.init_params(dims, np.random.RandomState(5))
    theta[-A:] = -0.5
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    b = ops.LaneBatch(O, A, lanes, T, dev)
    ops.rollout(L.ENV_KINDS[env_name], th32, hidden, hidden, 1e-6, b, T, None, None, 11, 0)
    ops.process_samples(b, None, 0.99, 1.0, drop_cut_paths=True)
    d1 = 2 * O + 5
    gram = torch.empty((d1 * (d1 + 1) // 2,), dtype=torch.float64, device=dev)
    ops.lfb_gram(b, gram)
    w = torch.empty((d1 - 1,), dtype=torch.float64, device=dev)
    fit = torch.zeros((3,), dtype=torch.float64, device=dev)
    ops.lfb_solve(O, gram, REG, w, fit)
    traj = b.to_numpy()
    keep = b.valid_mask().reshape(-1)
    F = S.lfb_features_lanes(traj["obs"], traj["tstep"]).reshape(d1 - 1, -1)[:, keep]
    y = b.ret.cpu().numpy().reshape(-1)[keep].astype(np.float64)
    assert np.isfinite(F).all() and np.isfinite(y).all()
    Gd = _unpack(gram.cpu().numpy(), d1)
    pred = w.cpu().numpy() @ F
    s = np.abs(y).max()
    e_solve = np.abs(pred - S.lfb_fit_normal(Gd[:-1, :-1], Gd[:-1, -1], REG) @ F).max() / s
    e_fit = np.abs(pred - S.lfb_fit_normal(F @ F.T, F @ y, REG) @ F).max() / s
    print("%s-%d: %d valid samples, cond %.2g, info %s, solve %.3g, end to end %.3g of max|ret| = %.4g" % (
        env_name, hidden, keep.sum(), np.linalg.cond(Gd[:-1, :-1] + REG * np.eye(d1 - 1)), fit.cpu().tolist(),
        e_solve, e_fit, s))
    assert tuple(fit.cpu().tolist()) == (REG, 0.0, 1.0)
    assert e_solve <= 1e-6, e_solve
    assert e_fit <= 1e-5, e_fit


@pytest.mark.parametrize("env_name,hidden", [("swimmer", 32), ("hopper", 64), ("half_cheetah", 64)])
def test_fit_flag_through_trpo(dev, env_name, hidden):
    """Through the plugin API (TRPO + LinearFeatureBaseline, 512 lanes x 500 steps): every iteration's device fit
    succeeds at the first attempt."""
    from test_gpu_algos import _algo
    algo = _algo(env_name, "trpo", 512, 500, hidden, n_itr=3, step_size=0.01)
    algo.start_worker()
    algo.init_opt()
    for itr in range(3):
        algo.train_itr(itr)
        assert algo.baseline.last_fit_info() == (REG, 0.0, 1.0), (itr, algo.baseline.last_fit_info())
