"""Policy-update kernels against the float64 oracle for every compiled net shape, at batch sizes that run the persistent
tile loop.

The batches are synthetic (no environment): for each of the 12 compiled nets, (O, A) in {(2,2), (4,1), (3,1), (6,1),
(13,2), (20,3)} x hidden 32 / 64, observations and advantages are drawn from a seeded normal with a few large entries,
and actions / old means / log_std are written by `policy_get_actions` at theta_old.  Batch sizes derive from the SM count
n_sm of the device:
  1             every row of the one tile maps to sample 0, only one row may count
  77            one partial tile
  128 * 37      exact tiles, fewer tiles than CTAs
  B_L = (17 n_sm + 5) * 128 - 51
                >= 17 tiles per CTA of the 64-wide kernel (one CTA per SM: two mid-loop flushes of its float32 accumulators
                and a remainder flush), 8-9 tiles per CTA of the 32-wide kernels (2 CTAs per SM), ~4 grid-stride sweeps of
                the 64-wide loss kernel (4 CTAs of 128 threads per SM), a partial last tile and uneven tile counts per CTA.
Every reference is the oracle (oracle/policy.py) in float64 on the float32-rounded inputs the kernel saw.  Oracle results
are cached per case in module scope; the device batches are kept for the module too (a few GB at most on an 80 GB GPU).
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import policy as P          # noqa: E402

NETS = [(2, 2), (4, 1), (3, 1), (6, 1), (13, 2), (20, 3)]
SHAPES = [(O, A, H) for H in (32, 64) for (O, A) in NETS]
SIZES = ["1", "77", "exact", "large"]
TILE = 128
REG = 1e-5


def _id(shape):
    return "O%dA%dH%d" % shape


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from rllab_b200 import _lib
    _lib.load()                          # fails loudly if the extension is missing
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def n_sm(dev):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _L():
    from rllab_b200 import _lib
    return _lib


def _ops():
    from rllab_b200 import ops
    return ops


def _batch_size(size, n_sm):
    return {"1": 1, "77": 77, "exact": TILE * 37, "large": (17 * n_sm + 5) * TILE - 51}[size]


def _f32(theta):
    return theta.astype(np.float32).astype(np.float64)


class Case(object):
    """One synthetic batch on the device plus float32 host copies of what the kernels read, and a memo of oracle
    results.  `keep` marks the samples the passes count (all of them unless the case is masked)."""

    def __init__(self, dev, n_sm, O, A, H, size, masked):
        ops, L = _ops(), _L()
        self.O, self.A, self.H, self.size, self.n_sm = O, A, H, size, n_sm
        self.B = B = _batch_size(size, n_sm)
        self.dims = P.Dims(O, (H, H), A)
        self.dd = (O, H, H, A)
        self.memo = {}
        rng = np.random.RandomState(1000 * O + 100 * A + H + (7 if masked else 0))
        theta = P.init_params(self.dims, rng)
        theta += rng.randn(self.dims.P) * 0.05                         # non-zero biases
        theta[-A:] = -0.5 + 0.2 * np.arange(A)                         # a distinct log_std per component
        self.th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
        self.theta = self.th32.double().cpu().numpy()
        # observations: the policy does not clip them, so a few percent are far out (|x| 20..50)
        obs = rng.randn(O, B)
        big = rng.rand(O, B) < 0.03
        obs[big] = np.sign(rng.randn(int(big.sum()))) * rng.uniform(20.0, 50.0, int(big.sum()))
        adv = rng.randn(B)
        far = rng.rand(B) < 0.005
        adv[far] = np.sign(rng.randn(int(far.sum()))) * rng.uniform(45.0, 50.0, int(far.sum()))
        self.obs, self.adv = obs.astype(np.float32), adv.astype(np.float32)
        eps = rng.randn(A, B).astype(np.float32)
        b = ops.LaneBatch(O, A, B, 1, dev)
        b.obs.copy_(torch.tensor(self.obs).view(O, 1, B))
        b.adv.copy_(torch.tensor(self.adv).view(1, B))
        b.flags.zero_()
        ops.policy_get_actions(self.th32, O, H, H, A, 1e-6, b.obs, B, torch.tensor(eps, device=dev), 0, 0, 0, 0,
                               b.act, b.mean, b.log_std)
        self.act = b.act.view(A, B).cpu().numpy()
        self.mean = b.mean.view(A, B).cpu().numpy()
        self.log_std = b.log_std.cpu().numpy()
        # the first assertion of every case: the forward kernel against the oracle forward
        mu, lsd = P.forward(self.theta, self.obs.T.astype(np.float64), self.dims)
        np.testing.assert_allclose(self.mean.T, mu, rtol=2e-5, atol=2e-6)
        np.testing.assert_allclose(self.act.T, mu + np.exp(lsd) * eps.T.astype(np.float64), rtol=2e-5, atol=2e-6)
        np.testing.assert_allclose(self.log_std, lsd, rtol=1e-6)
        self.keep = np.ones(B, dtype=bool)
        if masked:
            ntiles = -(-B // TILE)
            masks = rng.rand(B) < 0.2
            if size == "large":
                masks[3 * TILE:6 * TILE] = True                       # three whole tiles
                masks[(ntiles - 1) * TILE:] = True                    # the partial last tile
            elif size == "77":
                masks[64:] = True                                     # the last 13 samples
            fl = np.where(masks, L.FLAG_MASKED, 0).astype(np.uint8)
            b.flags.copy_(torch.tensor(fl).view(1, B))
            b.masked = True
            self.keep = ~masks
            b.sums[2] = float(self.keep.sum())                         # the device-resident valid-sample count
        self.b = b
        torch.cuda.synchronize()

    def batch(self, sel=None):
        """Oracle batch of the counted samples (and of `sel`, a (B,) bool selection, if given)."""
        k = self.keep if sel is None else self.keep & sel
        return dict(obs=self.obs.T[k].astype(np.float64), actions=self.act.T[k].astype(np.float64),
                    adv=self.adv[k].astype(np.float64), old_mean=self.mean.T[k].astype(np.float64),
                    old_log_std=self.log_std.astype(np.float64))

    def ref(self, key, fn):
        if key not in self.memo:
            self.memo[key] = fn()
        return self.memo[key]

    def theta2(self):
        """theta + 0.02 randn: on-policy neighbourhood (float32-rounded, the kernels read float32 parameters)."""
        return _f32(self.theta + np.random.RandomState(9).randn(self.dims.P) * 0.02)

    def theta3(self):
        """Off-policy theta: the smallest of a few step sizes along a few seeded directions for which the likelihood
        ratios exp(logp_new - logp_old) of the batch span at least e^-2 .. e^2 (a single sample has one ratio: B = 1
        takes the first candidate)."""
        def pick():
            batch = self.batch()
            lp_old = P.log_likelihood(batch["actions"], batch["old_mean"], batch["old_log_std"])
            first = None
            for seed in range(10, 20):
                d = np.random.RandomState(seed).randn(self.dims.P)
                d[-self.A:] = 0.2                                  # the std moves too
                for step in (0.1, 0.15, 0.2, 0.3):
                    th = _f32(self.theta + d * step)
                    if first is None:
                        first = th
                    if self.keep.sum() < 2:
                        return th, None
                    mu, ls = P.forward(th, batch["obs"], self.dims)
                    lr = P.log_likelihood(batch["actions"], mu, ls) - lp_old
                    if lr.min() <= -2.0 and lr.max() >= 2.0:
                        return th, (lr.min(), lr.max())
            raise AssertionError("no candidate theta_3 spans the likelihood ratios e^-2 .. e^2")
        return self.ref("theta3", pick)


_CASES = {}


def _case(dev, n_sm, shape, size, masked=False):
    key = shape + (size, masked)
    if key not in _CASES:
        _CASES[key] = Case(dev, n_sm, *shape, size=size, masked=masked)
    return _CASES[key]


def _triple_ref(c, th, name, min_std=1e-6):
    batch = c.batch()
    loss = P.surr_loss_trpo(th, batch, c.dims, min_std) if name == "trpo" else P.surr_loss_vpg(th, batch, c.dims, min_std)
    return np.array((loss,) + tuple(P.kl_stats(th, batch, c.dims, min_std)))


def _assert_triple(o, ref):
    np.testing.assert_allclose(o[0], ref[0], rtol=2e-5, atol=2e-6, err_msg="loss")
    np.testing.assert_allclose(o[1], ref[1], rtol=2e-5, atol=1e-8, err_msg="mean KL")
    np.testing.assert_allclose(o[2], ref[2], rtol=1e-4, atol=1e-8, err_msg="max KL")


def _assert_grad(g, ref):
    # three-pass TF32 chain (tensor cores): 4e-7 of the scale of the summands, i.e. a few 1e-6 of the largest entry
    np.testing.assert_allclose(g, ref, rtol=2e-4, atol=5e-6 * np.abs(ref).max() + 1e-9)


def _assert_fvp(Hx, ref):
    np.testing.assert_allclose(Hx, ref, rtol=2e-4, atol=2e-6 * np.abs(ref).max())


def _assert_fvp_kernels_agree(Hx_c, Hx):
    # 5e-6 of the largest entry, plus 5e-5 of the entry itself: an entry that one sample dominates (B = 1, or the 1e6
    # Fisher weight 2 / (2 sigma^2) of a component clamped at min_std = 1e-3) carries that sample's float32 rounding of
    # both chains without averaging (measured up to 1.9e-5 relative); each kernel alone is held to 2e-4 relative
    # against the oracle, so the two may differ by up to 4e-4 relative without either being wrong
    np.testing.assert_allclose(Hx_c, Hx, rtol=5e-5, atol=5e-6 * np.abs(Hx).max())


def _assert_activations(hc, c):
    """The [H1 + H2][B] activation cache against the oracle's tanh outputs: 2e-6, or, where the inputs of a unit are
    large, the error bound of the 3xTF32 layer it came out of.  The split a b ~ a_hi b_hi + a_hi b_lo + a_lo b_hi drops
    a_lo b_lo and the tensor cores read a_lo, b_lo at TF32 precision; with |x_lo| <= 2^-10 |x| each of the three is at
    most 2^-20 |a b|, and the float32 accumulation of K products and the bias adds at most (K + 1) 2^-24 of the sum of
    their magnitudes.  So the pre-activation is off by at most eps_K S, S = sum_i |a_i w_i| + |b|, and h = tanh(pre)
    by (1 - h^2) eps_K S; the second layer adds the first layer's error carried through |W1|.  An observation of 20..50
    makes S ~ 10..20 for its first-layer units, so their bound exceeds 2e-6 (measured up to 1.2e-5).  Entries with
    ordinary inputs stay at 2e-6, and a NaN (unwritten entry) or a value of another sample always fails."""
    H, dims = c.H, c.dims
    W0, b0, W1, b1 = [np.abs(t) for t in P.unpack(c.theta, dims)[:4]]
    x = c.obs.T.astype(np.float64)
    _, _, acts = P.forward(c.theta, x, dims, keep=True)
    h1, h2 = acts[1], acts[2]
    eps1 = 3 * 2.0 ** -20 + (c.O + 1) * 2.0 ** -24
    eps2 = 3 * 2.0 ** -20 + (H + 1) * 2.0 ** -24
    d1 = (1 - h1 ** 2) * eps1 * (np.abs(x) @ W0 + b0)                   # first-layer error bound
    d2 = (1 - h2 ** 2) * (d1 @ W1 + eps2 * (np.abs(h1) @ W1 + b1))
    tol = np.maximum(2e-6, np.concatenate([d1.T, d2.T], axis=0))
    got = hc.view(2 * H, c.B).cpu().numpy().astype(np.float64)
    err = np.abs(got - np.concatenate([h1.T, h2.T], axis=0))
    bad = ~(err <= tol)                                                  # NaN counts as bad
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:5].tolist(), np.nanmax(err / tol))


def _check_loss_grad(c, dev):
    """loss / KL (loss_kl) and gradient + fused triple (grad) at theta_2 and theta_3, TRPO and VPG."""
    ops, L = _ops(), _L()
    th3, spread = c.theta3()
    if c.keep.sum() >= 2:
        assert spread is not None and spread[0] <= -2.0 and spread[1] >= 2.0, spread
    for tag, th in (("th2", c.theta2()), ("th3", th3)):
        th_d = torch.tensor(th, dtype=torch.float32, device=dev)
        for kind, name in ((L.LOSS_TRPO, "trpo"), (L.LOSS_VPG, "vpg")):
            out = torch.zeros(3, dtype=torch.float64, device=dev)
            ops.loss_kl(kind, th_d, c.dd, 1e-6, c.b, out)
            o = out.cpu().numpy()
            ref = c.ref((tag, name, "triple"), lambda: _triple_ref(c, th, name))
            _assert_triple(o, ref)
            g = torch.zeros(c.dims.P, dtype=torch.float64, device=dev)
            out_g = torch.zeros(3, dtype=torch.float64, device=dev)
            ops.grad(kind, th_d, c.dd, 1e-6, c.b, g, out_g)
            og = out_g.cpu().numpy()
            _assert_triple(og, ref)
            if c.H == 32:
                # the loss pass is the gradient pass's forward, instruction for instruction: the per-sample terms are
                # identical and only the float64 order of the per-block sums differs (the grids differ)
                np.testing.assert_allclose(og, o, rtol=1e-12, atol=0)
            else:
                # 64-wide: FFMA forward (loss) against the tensor-core forward (gradient), both float32-grade
                np.testing.assert_allclose(og, o, rtol=1e-4, atol=2e-6)
            ref_g = c.ref((tag, name, "grad"), lambda: P.grad_surr(th, c.batch(), c.dims, name))
            _assert_grad(g.cpu().numpy(), ref_g)


def _check_fvp(c, dev, hc):
    """Fisher-vector product at theta_old with the activation cache (tensor-core kernels) and without it (FP32 tile /
    tiled-GEMM kernels); `hc` must hold the activations of theta_old."""
    ops = _ops()
    x = np.random.RandomState(4).randn(c.dims.P)
    xd = torch.tensor(x, dtype=torch.float64, device=dev)
    x32 = _f32(x)                                    # the kernels round the tangent to float32
    ref = c.ref("fvp", lambda: P.fvp(c.theta, c.batch(), x32, c.dims, 0.0) + REG * x)
    Hx = torch.zeros(c.dims.P, dtype=torch.float64, device=dev)
    ops.fvp(c.th32, c.dd, 1e-6, c.b, xd, REG, 1.0, Hx)
    Hx_c = torch.zeros_like(Hx)
    ops.fvp(c.th32, c.dd, 1e-6, c.b, xd, REG, 1.0, Hx_c, hc)
    Hx, Hx_c = Hx.cpu().numpy(), Hx_c.cpu().numpy()
    _assert_fvp(Hx, ref)
    _assert_fvp(Hx_c, ref)
    _assert_fvp_kernels_agree(Hx_c, Hx)


def _grad_with_cache(c, dev):
    ops, L = _ops(), _L()
    hc = c.b.hcache(c.H, c.H)
    hc.fill_(float("nan"))                           # a row the gradient pass does not write stays NaN
    g = torch.zeros(c.dims.P, dtype=torch.float64, device=dev)
    ops.grad(L.LOSS_TRPO, c.th32, c.dd, 1e-6, c.b, g, None, hc)
    return hc


def _check_f64(c, dev):
    """float64 parity kernels: modes 0 (loss / KL), 1 (gradient), 2 (Fisher-vector product)."""
    ops, L = _ops(), _L()
    th = c.theta + np.random.RandomState(5).randn(c.dims.P) * 0.02          # NOT rounded to float32
    thd = torch.tensor(th, dtype=torch.float64, device=dev)
    out = torch.zeros(3, dtype=torch.float64, device=dev)
    g = torch.zeros(c.dims.P, dtype=torch.float64, device=dev)
    for kind, name in ((L.LOSS_TRPO, "trpo"), (L.LOSS_VPG, "vpg")):
        ops.update_f64(0, kind, thd, c.dd, 1e-6, c.b, None, 0.0, 0.0, None, out)
        ref = c.ref(("f64", name, "triple"), lambda: _triple_ref(c, th, name))
        np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-9, atol=1e-13)
        ops.update_f64(1, kind, thd, c.dd, 1e-6, c.b, None, 0.0, 0.0, g, out)
        ref_g = c.ref(("f64", name, "grad"), lambda: P.grad_surr(th, c.batch(), c.dims, name))
        np.testing.assert_allclose(g.cpu().numpy(), ref_g, rtol=1e-8, atol=1e-12 * np.abs(ref_g).max())
    x = np.random.RandomState(6).randn(c.dims.P)
    Hx = torch.zeros(c.dims.P, dtype=torch.float64, device=dev)
    th0 = torch.tensor(c.theta, dtype=torch.float64, device=dev)
    ops.update_f64(2, L.LOSS_TRPO, th0, c.dd, 1e-6, c.b, torch.tensor(x, dtype=torch.float64, device=dev), REG, 1.0,
                   Hx, None)
    ref_H = c.ref(("f64", "fvp"), lambda: P.fvp(c.theta, c.batch(), x, c.dims, REG))
    np.testing.assert_allclose(Hx.cpu().numpy(), ref_H, rtol=1e-8, atol=1e-12 * np.abs(ref_H).max())


# ------------------------------------------------------------------------------------------- batch geometry
def test_large_batch_runs_the_persistent_loop(dev, n_sm):
    """The geometry B_L is built for, from the launchers' grid sizes: 64-wide passes n_sm CTAs, 32-wide gradient / Fisher
    passes 2 n_sm, 64-wide loss pass 4 n_sm CTAs of 128 threads."""
    B = _batch_size("large", n_sm)
    ntiles = -(-B // TILE)
    assert B % TILE != 0 and ntiles % n_sm != 0
    assert ntiles // n_sm >= 17                       # 64-wide: flushes after tiles 8 and 16, then the remainder
    assert 8 <= ntiles // (2 * n_sm) and -(-ntiles // (2 * n_sm)) <= 9
    assert B / (4 * n_sm * 128) > 4
    assert TILE * 37 < TILE * n_sm                    # the exact-tiles size has fewer tiles than CTAs


# ------------------------------------------------------------------------------------------- per (shape, size)
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_loss_kl_at_theta_old(dev, n_sm, shape, size):
    """At theta_old the likelihood ratio is 1: loss = -mean(adv), KL = 0.  64-wide nets: loss_thread_kernel and
    get_actions_kernel both run mlp_forward_thread<Net> on theta in shared memory, so the mean is bit-identical and the
    result exact up to the float64 sums.  32-wide nets: the loss pass runs its forward on the tensor cores (3xTF32), the
    mean agrees to float32 rounding."""
    ops, L = _ops(), _L()
    c = _case(dev, n_sm, shape, size)
    out = torch.zeros(3, dtype=torch.float64, device=dev)
    ops.loss_kl(L.LOSS_TRPO, c.th32, c.dd, 1e-6, c.b, out)
    o = out.cpu().numpy()
    adv_mean = c.adv.astype(np.float64).mean()
    if c.H == 64:
        assert abs(o[0] + adv_mean) < 1e-9 and abs(o[1]) < 1e-12 and abs(o[2]) < 1e-12, (o, adv_mean)
    else:
        assert abs(o[0] + adv_mean) < 1e-6 and abs(o[1]) < 1e-10 and abs(o[2]) < 1e-8, (o, adv_mean)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_loss_and_gradient_off_theta_old(dev, n_sm, shape, size):
    _check_loss_grad(_case(dev, n_sm, shape, size), dev)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_activation_cache_and_fvp(dev, n_sm, shape, size):
    """The gradient pass at theta_old writes the [H1 + H2][B] activation cache: every entry equals the oracle's tanh
    output (a missing write stays NaN; a row >= B written into the next feature row overwrites a real entry).  The
    Fisher-vector products with and without the cache then match the oracle and each other."""
    c = _case(dev, n_sm, shape, size)
    hc = _grad_with_cache(c, dev)
    _assert_activations(hc, c)
    _check_fvp(c, dev, hc)


@pytest.mark.parametrize("size", ["77", "large"])
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_f64_parity_kernels(dev, n_sm, shape, size):
    _check_f64(_case(dev, n_sm, shape, size), dev)


@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_float32_passes_are_deterministic(dev, n_sm, shape):
    """Fixed-order reductions: the same inputs give bit-identical outputs (the float64 parity kernels accumulate with
    atomics and are not covered)."""
    ops, L = _ops(), _L()
    c = _case(dev, n_sm, shape, "large")
    th2 = torch.tensor(c.theta2(), dtype=torch.float32, device=dev)
    x = torch.tensor(np.random.RandomState(4).randn(c.dims.P), dtype=torch.float64, device=dev)

    def run():
        res = []
        for kind in (L.LOSS_TRPO, L.LOSS_VPG):
            out = torch.zeros(3, dtype=torch.float64, device=dev)
            ops.loss_kl(kind, th2, c.dd, 1e-6, c.b, out)
            g = torch.zeros(c.dims.P, dtype=torch.float64, device=dev)
            og = torch.zeros(3, dtype=torch.float64, device=dev)
            ops.grad(kind, th2, c.dd, 1e-6, c.b, g, og)
            res += [out, g, og]
        hc = _grad_with_cache(c, dev)
        res.append(hc.clone())
        for cache in (None, hc):
            Hx = torch.zeros(c.dims.P, dtype=torch.float64, device=dev)
            ops.fvp(c.th32, c.dd, 1e-6, c.b, x, REG, 1.0, Hx, cache)
            res.append(Hx)
        torch.cuda.synchronize()
        return res

    first, second = run(), run()
    for i, (u, v) in enumerate(zip(first, second)):
        assert torch.equal(u, v), i


# ------------------------------------------------------------------------------------------- variants
@pytest.mark.parametrize("size", ["77", "large"])
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_masked_samples(dev, n_sm, shape, size):
    """About 20 % of the samples carry FLAG_MASKED, plus whole masked tiles (B_L: tiles 3-5 and the partial last tile;
    B = 77: the last 13 samples).  Every pass divides by the device-resident valid count; the oracle runs on the kept
    samples, at the unmasked bounds."""
    c = _case(dev, n_sm, shape, size, masked=True)
    _check_loss_grad(c, dev)
    hc = _grad_with_cache(c, dev)
    _check_fvp(c, dev, hc)
    _check_f64(c, dev)


@pytest.mark.parametrize("size", ["77", "large"])
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_fvp_tile_lists(dev, n_sm, shape, size):
    """Sub-sampled Fisher-vector products (subsample_factor < 1) over unsorted tile lists without repeats that include
    the partial last tile, on a masked batch: a list shorter than every grid and one of about 6 n_sm tiles (B = 77: the
    one tile).  The divisor is the valid-sample count of the listed tiles (count_valid); the oracle runs on the selected,
    valid samples.  Both kernels of the width: tensor cores with the activation cache, FP32 without."""
    ops = _ops()
    c = _case(dev, n_sm, shape, size, masked=True)
    ntiles = -(-c.B // TILE)
    rng = np.random.RandomState(21)
    if size == "large":
        lists = []
        for n in (n_sm // 3, 6 * n_sm):
            t = np.concatenate([rng.permutation(ntiles - 1)[:n - 1], [ntiles - 1]])
            rng.shuffle(t)
            assert len(set(t.tolist())) == n and np.any(np.diff(t) < 0)
            lists.append(t)
        assert len(lists[0]) < n_sm
    else:
        lists = [np.array([0])]
    hc = _grad_with_cache(c, dev)
    x = np.random.RandomState(8).randn(c.dims.P)
    xd = torch.tensor(x, dtype=torch.float64, device=dev)
    for i, t in enumerate(lists):
        sel = np.zeros(ntiles * TILE, dtype=bool)
        for k in t:
            sel[k * TILE:(k + 1) * TILE] = True
        sel = sel[:c.B]
        tl = torch.tensor(t.astype(np.int32), device=dev)
        cnt = torch.zeros(1, dtype=torch.float64, device=dev)
        ops.count_valid(c.b, tl, cnt)
        assert float(cnt.cpu()[0]) == float((sel & c.keep).sum())
        ref = c.ref(("tiles", i), lambda: P.fvp(c.theta, c.batch(sel), _f32(x), c.dims, 0.0) + REG * x)
        res = []
        for cache in (None, hc):
            Hx = torch.zeros(c.dims.P, dtype=torch.float64, device=dev)
            ops.fvp(c.th32, c.dd, 1e-6, c.b, xd, REG, 1.0, Hx, cache, tile_list=tl, count=cnt)
            res.append(Hx.cpu().numpy())
            _assert_fvp(res[-1], ref)
        _assert_fvp_kernels_agree(res[1], res[0])


@pytest.mark.parametrize("size", ["77", "large"])
@pytest.mark.parametrize("shape", [s for s in SHAPES if s[1] > 1], ids=_id)
def test_min_std_clamp_per_component(dev, n_sm, shape, size):
    """min_std = 1e-3 with log_std[0] clearly below log(1e-3) and the other components above: the clamped component's
    gradient is exactly 0, its Fisher entry is reg * x only, and the other components keep their gradient (the log_std
    block is also compared on its own scale, since the clamped component dominates the mean gradient)."""
    ops, L = _ops(), _L()
    c = _case(dev, n_sm, shape, size)
    A, ols = c.A, c.dims.P - c.A
    th = c.theta2()
    th[ols] = np.log(1e-3) - 1.0
    th = _f32(th)
    assert np.all(th[ols + 1:] > np.log(1e-3) + 1.0)
    th_d = torch.tensor(th, dtype=torch.float32, device=dev)
    g = torch.zeros(c.dims.P, dtype=torch.float64, device=dev)
    ops.grad(L.LOSS_VPG, th_d, c.dd, 1e-3, c.b, g)
    g = g.cpu().numpy()
    ref_g = c.ref("min_std_grad", lambda: P.grad_surr(th, c.batch(), c.dims, "vpg", min_std=1e-3))
    assert g[ols] == 0.0 and ref_g[ols] == 0.0
    _assert_grad(g, ref_g)
    _assert_grad(g[ols:], ref_g[ols:])
    # Fisher-vector product at the clamped theta (the closed form reads only obs and theta)
    th0 = c.theta.copy()
    th0[ols] = np.log(1e-3) - 1.0
    th0 = _f32(th0)
    th0_d = torch.tensor(th0, dtype=torch.float32, device=dev)
    hc = c.b.hcache(c.H, c.H)
    hc.fill_(float("nan"))
    ops.grad(L.LOSS_VPG, th0_d, c.dd, 1e-3, c.b, torch.zeros(c.dims.P, dtype=torch.float64, device=dev), None, hc)
    x = np.random.RandomState(12).randn(c.dims.P)
    xd = torch.tensor(x, dtype=torch.float64, device=dev)
    ref = c.ref("min_std_fvp", lambda: P.fvp(th0, c.batch(), _f32(x), c.dims, 0.0, min_std=1e-3) + REG * x)
    res = []
    for cache in (None, hc):
        Hx = torch.zeros(c.dims.P, dtype=torch.float64, device=dev)
        ops.fvp(th0_d, c.dd, 1e-3, c.b, xd, REG, 1.0, Hx, cache)
        Hx = Hx.cpu().numpy()
        assert Hx[ols] == REG * x[ols]
        _assert_fvp(Hx, ref)
        res.append(Hx)
    _assert_fvp_kernels_agree(res[1], res[0])
