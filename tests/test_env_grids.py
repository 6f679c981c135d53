"""The GPU grids that claim to cover every env kind name exactly the kinds of rllab_b200._lib.ENV_KINDS (the discrete
grids: DISCRETE_ENV_KINDS), so that a new env kind cannot skip them unnoticed.  No GPU needed: the grids are module
constants."""
import pytest

pytest.importorskip("torch")

from rllab_b200 import _lib as L        # noqa: E402
import test_gpu_algos                   # noqa: E402
import test_gpu_categorical_shapes      # noqa: E402
import test_gpu_cem                     # noqa: E402
import test_gpu_process_shapes          # noqa: E402
import test_gpu_rollout_shapes          # noqa: E402
import test_gpu_round2                  # noqa: E402

# Kinds a grid leaves out on purpose.  Each entry says why.
EXCLUDED = {
    # full episodes against the planar oracles only; tests/test_gpu_kernels.py steps the classic-control envs
    "planar_episodes": {"point", "cartpole", "pendulum", "cartpole_swingup", "double_pendulum"},
}

GRIDS = {
    "rollout": lambda: test_gpu_rollout_shapes.ENVS,
    "population": lambda: test_gpu_cem.ENVS,
    "baseline_fit": lambda: [e for e, _, _, _ in test_gpu_process_shapes.FIT_ENVS],
    "env_protocol": lambda: test_gpu_algos.PROTOCOL_ENVS,
    "planar_episodes": lambda: [e for e, _ in test_gpu_round2.PLANAR_EPISODES],
}

# grids over the discrete-action kinds (rllab_b200._lib.DISCRETE_ENV_KINDS)
DISCRETE_GRIDS = {
    "discrete_rollout": lambda: test_gpu_categorical_shapes.DISCRETE_ENVS,
}


@pytest.mark.parametrize("grid", sorted(GRIDS))
def test_grid_covers_every_env_kind(grid):
    names = set(GRIDS[grid]())
    expected = set(L.ENV_KINDS) - EXCLUDED.get(grid, set())
    assert names == expected, "%s grid: missing %s, unknown %s" % (grid, sorted(expected - names),
                                                                   sorted(names - expected))


@pytest.mark.parametrize("grid", sorted(DISCRETE_GRIDS))
def test_grid_covers_every_discrete_env_kind(grid):
    names = set(DISCRETE_GRIDS[grid]())
    expected = set(L.DISCRETE_ENV_KINDS)
    assert names == expected, "%s grid: missing %s, unknown %s" % (grid, sorted(expected - names),
                                                                   sorted(names - expected))


def test_exclusions_name_env_kinds():
    for grid, kinds in EXCLUDED.items():
        assert grid in GRIDS and kinds <= set(L.ENV_KINDS), grid
