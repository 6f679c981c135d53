"""GymEnv (rllab/envs/gym_env.py:58-116 over gym==0.7.4) for the two gym envs on the hot path: Pendulum-v0 and
CartPole-v0."""
from .lane_env import LaneEnv


class PendulumEnv(LaneEnv):
    ENV_NAME = "pendulum"
    HORIZON = 200      # gym TimeLimit of Pendulum-v0 [3P]; gym_env.py:104-105 exposes it as env.horizon


class CartPoleV0Env(LaneEnv):
    """gym CartPole-v0: Discrete(2) actions (0 pushes left, 1 right), reward 1 per step, done at |x| > 2.4 or
    |theta| > 12 deg; the dynamics are restated in csrc/envs.cuh (GymCartPoleEnvD)."""
    ENV_NAME = "gym_cartpole"
    HORIZON = 200      # gym TimeLimit of CartPole-v0


_GYM_ENVS = {"Pendulum-v0": PendulumEnv, "CartPole-v0": CartPoleV0Env}


def GymEnv(env_name, record_video=True, video_schedule=None, log_dir=None, record_log=True, force_reset=False):
    """Same signature as gym_env.py:59-60.  The gym Monitor (video / log recording) is outside the hot path: like the
    reference without a snapshot directory (gym_env.py:61-63), monitoring is skipped."""
    if env_name not in _GYM_ENVS:
        raise NotImplementedError("only GymEnv(%s) is on the B200 hot path (got %r)"
                                  % (" / ".join(repr(k) for k in sorted(_GYM_ENVS)), env_name))
    return _GYM_ENVS[env_name]()
