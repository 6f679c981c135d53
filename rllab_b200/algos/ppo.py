"""PPO (rllab/algos/ppo.py:6-21) = NPO + PenaltyLbfgsOptimizer: the KL-penalty method of rllab (penalised L-BFGS with an
adaptive penalty), not the clipped-ratio objective of later papers."""
from ..optimizers.penalty_lbfgs_optimizer import PenaltyLbfgsOptimizer
from .npo import NPO


class PPO(NPO):
    """
    Penalized Policy Optimization.
    """

    def __init__(self, optimizer=None, optimizer_args=None, **kwargs):
        if optimizer is None:
            if optimizer_args is None:
                optimizer_args = dict()
            optimizer = PenaltyLbfgsOptimizer(**optimizer_args)
        super(PPO, self).__init__(optimizer=optimizer, **kwargs)
