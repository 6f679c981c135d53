"""32-wide tensor-core update passes at batch sizes cut to their grid: one CTA per SM of three warpgroups (loss pass,
gradient pass of act_dim 1) or two (the other gradient passes, the Fisher pass), tiles dealt to the warpgroups
round-robin, each warpgroup's inputs requested one tile ahead into a two-slot ring.  With n_sm the SM count of the
device the batches are
  one     3 n_sm tiles, the last one partial: every warpgroup of a three-per-SM grid takes exactly one tile (one ring
          fill, no refill)
  two     3 n_sm + 1 exact tiles: one warpgroup takes a second tile (one refill of the other slot), the rest one
  many    (21 n_sm + 5) tiles, the last one partial: 7-8 tiles per warpgroup at three per SM (the ring wraps), 10-11 at
          two
The gradient, the (loss, KL) triple of both passes and the Fisher-vector product over an unsorted tile list of 3 n_sm + 2
tiles (more tiles than the pass's 2 n_sm warpgroups, not a multiple of them: some take two list entries, some one) are
compared with the float64 oracle (oracle/policy.py), and two runs must agree bit for bit.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import policy as P          # noqa: E402

NETS = [(2, 2), (4, 1), (3, 1), (6, 1), (13, 2), (20, 3)]
H = 32
TILE = 128
REG = 1e-5


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from rllab_b200 import _lib
    _lib.load()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def n_sm(dev):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _batch_size(size, n_sm):
    return {"one": 3 * n_sm * TILE - 51, "two": (3 * n_sm + 1) * TILE, "many": (21 * n_sm + 5) * TILE - 51}[size]


def _make(dev, O, A, B):
    from rllab_b200 import ops
    dims = P.Dims(O, (H, H), A)
    rng = np.random.RandomState(500 + 10 * O + A)
    theta = P.init_params(dims, rng) + rng.randn(dims.P) * 0.05
    theta[-A:] = -0.5 + 0.2 * np.arange(A)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    obs = rng.randn(O, B).astype(np.float32)
    adv = rng.randn(B).astype(np.float32)
    eps = rng.randn(A, B).astype(np.float32)
    b = ops.LaneBatch(O, A, B, 1, dev)
    b.obs.copy_(torch.tensor(obs).view(O, 1, B))
    b.adv.copy_(torch.tensor(adv).view(1, B))
    b.flags.zero_()
    ops.policy_get_actions(th32, O, H, H, A, 1e-6, b.obs, B, torch.tensor(eps, device=dev), 0, 0, 0, 0,
                           b.act, b.mean, b.log_std)
    torch.cuda.synchronize()
    batch = dict(obs=obs.T.astype(np.float64), actions=b.act.view(A, B).cpu().numpy().T.astype(np.float64),
                 adv=adv.astype(np.float64), old_mean=b.mean.view(A, B).cpu().numpy().T.astype(np.float64),
                 old_log_std=b.log_std.cpu().numpy().astype(np.float64))
    return dims, th32.double().cpu().numpy(), th32, b, batch


@pytest.mark.parametrize("size", ["one", "two", "many"])
@pytest.mark.parametrize("net", NETS, ids=lambda n: "O%dA%d" % n)
def test_grad_and_loss_on_grid_sized_batches(dev, n_sm, net, size):
    from rllab_b200 import _lib as L, ops
    O, A = net
    B = _batch_size(size, n_sm)
    dims, theta, _, b, batch = _make(dev, O, A, B)
    th = (theta + np.random.RandomState(9).randn(dims.P) * 0.02).astype(np.float32).astype(np.float64)
    th_d = torch.tensor(th, dtype=torch.float32, device=dev)
    dd = (O, H, H, A)
    for kind, name in ((L.LOSS_TRPO, "trpo"), (L.LOSS_VPG, "vpg")):
        runs = []
        for _ in range(2):
            out = torch.zeros(3, dtype=torch.float64, device=dev)
            ops.loss_kl(kind, th_d, dd, 1e-6, b, out)
            g = torch.zeros(dims.P, dtype=torch.float64, device=dev)
            og = torch.zeros(3, dtype=torch.float64, device=dev)
            ops.grad(kind, th_d, dd, 1e-6, b, g, og)
            torch.cuda.synchronize()
            runs.append([out.cpu().numpy(), g.cpu().numpy(), og.cpu().numpy()])
        for u, v in zip(*runs):
            assert np.array_equal(u, v), "two runs differ"
        o, g, og = runs[0]
        loss = P.surr_loss_trpo(th, batch, dims, 1e-6) if name == "trpo" else P.surr_loss_vpg(th, batch, dims, 1e-6)
        ref = np.array((loss,) + tuple(P.kl_stats(th, batch, dims, 1e-6)))
        np.testing.assert_allclose(o[0], ref[0], rtol=2e-5, atol=2e-6)
        np.testing.assert_allclose(o[1], ref[1], rtol=2e-5, atol=1e-8)
        np.testing.assert_allclose(o[2], ref[2], rtol=1e-4, atol=1e-8)
        np.testing.assert_allclose(og, o, rtol=1e-12, atol=0)
        ref_g = P.grad_surr(th, batch, dims, name)
        np.testing.assert_allclose(g, ref_g, rtol=2e-4, atol=5e-6 * np.abs(ref_g).max() + 1e-9)


@pytest.mark.parametrize("net", NETS, ids=lambda n: "O%dA%d" % n)
def test_fvp_tile_list_not_a_multiple_of_three(dev, n_sm, net):
    from rllab_b200 import _lib as L, ops
    O, A = net
    B = _batch_size("many", n_sm)
    dims, theta, th32, b, batch = _make(dev, O, A, B)
    dd = (O, H, H, A)
    hc = b.hcache(H, H)
    ops.grad(L.LOSS_TRPO, th32, dd, 1e-6, b, torch.zeros(dims.P, dtype=torch.float64, device=dev), None, hc)
    ntiles = -(-B // TILE)
    n = 3 * n_sm + 2
    rng = np.random.RandomState(31)
    t = np.concatenate([rng.permutation(ntiles - 1)[:n - 1], [ntiles - 1]])
    rng.shuffle(t)
    assert len(t) % 3 != 0 and np.any(np.diff(t) < 0)
    sel = np.zeros(ntiles * TILE, dtype=bool)
    for k in t:
        sel[k * TILE:(k + 1) * TILE] = True
    sel = sel[:B]
    tl = torch.tensor(t.astype(np.int32), device=dev)
    cnt = torch.zeros(1, dtype=torch.float64, device=dev)
    ops.count_valid(b, tl, cnt)
    x = np.random.RandomState(8).randn(dims.P)
    xd = torch.tensor(x, dtype=torch.float64, device=dev)
    res = []
    for _ in range(2):
        Hx = torch.zeros(dims.P, dtype=torch.float64, device=dev)
        ops.fvp(th32, dd, 1e-6, b, xd, REG, 1.0, Hx, hc, tile_list=tl, count=cnt)
        res.append(Hx.cpu().numpy())
    assert np.array_equal(res[0], res[1]), "two runs differ"
    sub = {k: (v[sel] if k != "old_log_std" else v) for k, v in batch.items()}
    ref = P.fvp(theta, sub, x.astype(np.float32).astype(np.float64), dims, 0.0) + REG * x
    np.testing.assert_allclose(res[0], ref, rtol=2e-4, atol=2e-6 * np.abs(ref).max())
