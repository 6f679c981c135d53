"""Device-side helpers shared by the DDPG GPU tests (tests/test_gpu_ddpg.py, tests/test_gpu_ddpg_grid.py): the
hyperparameters and networks they start from, one b200rl_ddpg_update call, a run's device state as an oracle state dict,
and the oracle's env callables on the device's own float32 env."""
import numpy as np
import torch

import ddpg_oracle as K
from rllab_b200 import _lib as L
from rllab_b200 import ops

DEV = torch.device("cuda:0")
BOX_KINDS = dict(point=L.ENV_POINT, cartpole=L.ENV_CARTPOLE, pendulum=L.ENV_PENDULUM,
                 cartpole_swingup=L.ENV_CARTPOLE_SWINGUP, double_pendulum=L.ENV_DOUBLE_PENDULUM)


def _hp(**kw):
    base = dict(n_updates_per_sample=1, max_path_length=30, min_pool_size=40, replay_pool_size=150,
                include_horizon_terminal_transitions=0, es_kind=L.ES_OU, discount=0.99, scale_reward=0.01,
                soft_target_tau=0.05, qf_weight_decay=0.01, qf_learning_rate=1e-3, policy_weight_decay=0.02,
                policy_learning_rate=1e-3, ou_mu=0.0, ou_theta=0.15, ou_sigma=0.3, gs_max_sigma=1.0, gs_min_sigma=0.1,
                gs_decay_period=200.0)
    base.update(kw)
    return base


def _dims(kind):
    info = L.env_info(kind)
    return K.Dims(info["obs_dim"], info["act_dim"])


def _nets(d, seed, moments=False):
    rng = np.random.RandomState(seed)
    th = np.concatenate([K.init_params(d.pshapes, rng), K.init_params(d.qshapes, rng)])
    tg = th + 0.05 * rng.randn(d.P)
    if moments:
        return np.stack([th, 1e-3 * rng.randn(d.P), 1e-6 * rng.rand(d.P), tg])
    return np.stack([th, np.zeros(d.P), np.zeros(d.P), tg])


def _pool(d, rows, seed):
    rng = np.random.RandomState(seed)
    return dict(obs=rng.randn(rows, d.O).astype(np.float32), act=rng.uniform(-1, 1, (rows, d.A)).astype(np.float32),
                rew=(0.1 * rng.randn(rows)).astype(np.float32), term=(rng.rand(rows) < 0.2).astype(np.uint8))


def _run_update(kind, f64, hp, pool, idx, nets, t):
    d = _dims(kind)
    g = lambda x, dt: torch.tensor(np.ascontiguousarray(x), dtype=dt, device=DEV)
    nets_t = g(nets, torch.float64)
    outs = [torch.empty(n, dtype=torch.float64, device=DEV) for n in (d.P, 32, 32, 2)]
    ops.ddpg_update(kind, f64, ops.ddpg_hparams(**hp), g(pool["obs"], torch.float32), g(pool["act"], torch.float32),
                    g(pool["rew"], torch.float32), g(pool["term"], torch.uint8), g(idx, torch.int32), nets_t, t, *outs)
    grad, q, y, loss = [x.cpu().numpy() for x in outs]
    return nets_t.cpu().numpy(), dict(grad=grad, q=q, y=y, qf_loss=loss[0], policy_surr=loss[1])


class _DeviceEnv(object):
    """The oracle's env callables on the device's own float32 env (b200rl_env_reset / b200rl_env_step)."""

    def __init__(self, kind, seed, run):
        self.kind, self.seed, self.run = kind, seed, run
        self.S = L.env_info(kind)["state_dim"]
        self.O = L.env_info(kind)["obs_dim"]

    def reset(self, itr):
        st = torch.empty((self.S, 1), dtype=torch.float32, device=DEV)
        o = torch.empty((self.O, 1), dtype=torch.float32, device=DEV)
        ops.env_reset(self.kind, 1, st, o, seed=self.seed, it=itr >> 28, row=itr & 0x0FFFFFFF, lane0=self.run)
        return st.cpu().numpy()[:, 0], o.cpu().numpy()[:, 0]

    def step(self, state, act):
        st = torch.tensor(np.asarray(state, np.float32).reshape(self.S, 1), device=DEV)
        o = torch.empty((self.O, 1), dtype=torch.float32, device=DEV)
        r = torch.empty(1, dtype=torch.float32, device=DEV)
        dn = torch.empty(1, dtype=torch.uint8, device=DEV)
        ops.env_step(self.kind, 1, st, torch.tensor(act.reshape(-1, 1), device=DEV), o, r, dn)
        return st.cpu().numpy()[:, 0], o.cpu().numpy()[:, 0], float(r.item()), bool(dn.item())


def _oracle_state(runs, r, d):
    s = runs.host_state()[r]
    return dict(nets=runs.nets[r].cpu().numpy().copy(), env_state=np.array(s.env_state[:8], np.float32),
                obs=np.array(s.obs[:d.O], np.float32), ou=np.array(s.ou_state[:d.A]), path_return=s.path_return,
                path_length=s.path_length, terminal=s.terminal, itr=s.itr, adam_t=s.adam_t,
                pool=dict(obs=runs.pool_obs[r].cpu().numpy().copy(), act=runs.pool_act[r].cpu().numpy().copy(),
                          rew=runs.pool_rew[r].cpu().numpy().copy(), term=runs.pool_term[r].cpu().numpy().copy()),
                top=s.top, bottom=s.bottom, size=s.size)
