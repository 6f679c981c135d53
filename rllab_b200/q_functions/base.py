"""QFunction (rllab/q_functions/base.py)."""


class QFunction(object):
    pass
