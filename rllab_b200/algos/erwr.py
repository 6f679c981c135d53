"""ERWR (rllab/algos/erwr.py:6-36) = VPG + LbfgsOptimizer on positive (shifted) advantages."""
from ..optimizers.lbfgs_optimizer import LbfgsOptimizer
from .vpg import VPG


class ERWR(VPG):
    """
    Episodic Reward Weighted Regression (Kober and Peters, "Policy search for motor primitives in robotics", NIPS 2009).
    """

    def __init__(self, optimizer=None, optimizer_args=None, positive_adv=None, **kwargs):
        if optimizer is None:
            if optimizer_args is None:
                optimizer_args = dict()
            optimizer = LbfgsOptimizer(**optimizer_args)
        super(ERWR, self).__init__(optimizer=optimizer, positive_adv=True if positive_adv is None else positive_adv,
                                   **kwargs)
