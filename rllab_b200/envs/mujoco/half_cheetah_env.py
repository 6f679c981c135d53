"""HalfCheetahEnv (rllab/envs/mujoco/half_cheetah_env.py:14-58); planar-tree restatement in csrc/planar.cuh."""
import numpy as np

from ...misc import logger
from ..lane_env import LaneEnv, require_defaults


class HalfCheetahEnv(LaneEnv):
    ENV_NAME = "half_cheetah"

    def __init__(self, *args, **kwargs):
        # half_cheetah_env.py:18-20 forwards everything to MujocoEnv.__init__(action_noise=0.0, file_path=None,
        # template_args=None)
        if args:
            raise TypeError("HalfCheetahEnv() takes keyword arguments only in this port (got %d positional)" % len(args))
        require_defaults("HalfCheetahEnv", kwargs, dict(action_noise=0.0, file_path=None, template_args=None))
        super(HalfCheetahEnv, self).__init__()

    def log_diagnostics(self, paths):
        # forward progress from obs[-3], the torso subtree COM x (half_cheetah_env.py:50-58)
        progs = [path["observations"][-1][-3] - path["observations"][0][-3] for path in paths]
        logger.record_tabular('AverageForwardProgress', np.mean(progs))
        logger.record_tabular('MaxForwardProgress', np.max(progs))
        logger.record_tabular('MinForwardProgress', np.min(progs))
        logger.record_tabular('StdForwardProgress', np.std(progs))
