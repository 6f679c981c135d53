"""CPU: the CEM oracle (tests/cem_oracle.py) against the reference's own CEM.train (tests/golden/reference_cem_golden.npz,
made by tests/golden/make_cem_golden.py), the CEM signature against tests/golden/reference_api_cem.json, and the
oracle's restatement of the parameter-sampling Philox stream."""
import importlib
import inspect
import json
import os

import numpy as np
import pytest

import cem_oracle as K
from oracle import philox

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(HERE, "golden", "reference_cem_golden.npz")))


def _cases(g):
    return sorted({k.split("/")[0] for k in g})


def _episodes(g, q, E):
    """Per-episode rewards of one iteration, [members][evals] lists."""
    flat, lens = g[q + "rew_flat"], g[q + "rew_len"]
    cuts = np.concatenate([[0], np.cumsum(lens)])
    rews = [flat[cuts[i]:cuts[i + 1]] for i in range(len(lens))]
    return [rews[m * E:(m + 1) * E] for m in range(len(rews) // E)], lens.reshape(-1, E)


def test_golden_covers_the_cases(golden):
    cases = _cases(golden)
    assert len(cases) == 3
    evals = {int(golden[c + "/n_evals"]) for c in cases}
    assert {1, 3} <= evals
    nbest = {int(golden[c + "/n_best"]) for c in cases}
    assert 1 in nbest and max(nbest) > 1
    assert any(c + "/args_batch_size" in golden for c in cases)
    assert any(c + "/args_extra_decay_time" in golden and int(golden[c + "/args_extra_decay_time"]) < 3 for c in cases)


def test_fitness_and_returns_match_reference(golden):
    for c in _cases(golden):
        E, disc = int(golden[c + "/n_evals"]), float(golden[c + "/discount"])
        for it in range(int(golden[c + "/n_itr"])):
            q = "%s/%d/" % (c, it)
            eps, _ = _episodes(golden, q, E)
            fs = np.array([K.stderr_lb([K.discounted_return(r, disc) for r in ep]) for ep in eps])
            us = np.array([K.stderr_lb([np.sum(r) for r in ep]) for ep in eps])
            np.testing.assert_allclose(fs, golden[q + "fs"], rtol=1e-12, atol=1e-12)
            np.testing.assert_allclose(us, golden[q + "ustat"], rtol=1e-12, atol=1e-12)


def test_elite_update_and_table_match_reference(golden):
    for c in _cases(golden):
        E, nb = int(golden[c + "/n_evals"]), int(golden[c + "/n_best"])
        for it in range(int(golden[c + "/n_itr"])):
            q = "%s/%d/" % (c, it)
            xs, fs = golden[q + "xs"], golden[q + "fs"]
            _, mean, std, bx = K.elite_update(xs, fs, min(nb, len(fs)))
            scale = np.max(np.abs(xs))
            assert np.max(np.abs(mean - golden[q + "cur_mean"])) <= 1e-12 * scale
            assert np.max(np.abs(std - golden[q + "cur_std"])) <= 1e-12 * scale
            assert np.array_equal(bx, golden[q + "best_x"])
            _, lens = _episodes(golden, q, E)
            tab = K.tabular(it, std, golden[q + "ustat"], fs, lens)
            tab["AveragePolicyStd"] = K.average_policy_std(xs, lens, 2)
            for key, v in tab.items():
                assert v == pytest.approx(float(golden[q + "tab_" + key]), rel=1e-12, abs=1e-12), (c, it, key)


def test_batch_size_criterion_matches_reference(golden):
    c = [c for c in _cases(golden) if c + "/args_batch_size" in golden][0]
    E, bs = int(golden[c + "/n_evals"]), int(golden[c + "/args_batch_size"])
    for it in range(int(golden[c + "/n_itr"])):
        q = "%s/%d/" % (c, it)
        _, lens = _episodes(golden, q, E)
        assert K.batch_prefix(lens[:, -1], bs) == len(lens) == int(golden[q + "tab_NumTrajs"])


def test_std_schedule_explains_reference_rows(golden):
    """Members of iteration i+1 are cur_mean_i + sample_std_i * z with z standard normal: the schedule (including the
    decay of extra_std past extra_decay_time) must make z unit-variance."""
    for c in _cases(golden):
        kw = {k.split("args_")[1]: golden[k] for k in golden if k.startswith(c + "/args_")}
        extra_std, decay = float(kw.get("extra_std", 1.0)), float(kw.get("extra_decay_time", 100))
        for it in range(1, int(golden[c + "/n_itr"])):
            prev = "%s/%d/" % (c, it - 1)
            sd = K.sample_std(golden[prev + "cur_std"], it, extra_std, decay)
            z = (golden["%s/%d/xs" % (c, it)] - golden[prev + "cur_mean"]) / np.where(sd > 0, sd, 1.0)
            z = z[:, sd > 0]
            assert 0.8 < np.mean(z ** 2) < 1.25, (c, it, np.mean(z ** 2))


def test_sampling_stream_restatement():
    """The parameter rows draw from Philox stream 2 at (lane = member, row 0, chunk = k // 4): the oracle's word layout
    for single members (including indices above 2^32, whose high word goes into the fourth counter) equals the block
    layout of b200rl_fill_noise, and the transformed draws are standard normal."""
    P, seed, it = 1250, 99, 4
    members = [0, 3, 2 ** 32 - 1, 2 ** 32, 5 * 2 ** 32 + 17]
    block = philox.raw_block(1, 0, P, 3, 0, seed, it, 2)
    for m in range(3):
        assert np.array_equal(philox.raw_block(1, 0, P, 1, m, seed, it, 2)[0, :, 0], block[0, :, m])
    for m in members:
        w = philox.philox4x32_10(np.array([m & 0xFFFFFFFF]), np.array([2 << 28]), np.array([1]), np.array([m >> 32]),
                                 seed, it)
        assert [int(x[0]) for x in w] == list(philox.raw_block(1, 0, P, 1, m, seed, it, 2)[0, 4:8, 0])
    assert not np.array_equal(philox.raw_block(1, 0, 8, 1, 2 ** 32, seed, it, 2),
                              philox.raw_block(1, 0, 8, 1, 0, seed, it, 2))
    z = philox.normal_from_raw(philox.raw_block(1, 0, 4000, 50, 0, seed, it, 2))
    assert abs(z.mean()) < 0.01 and abs(z.std() - 1) < 0.01


def test_cem_signature_matches_reference():
    api = json.load(open(os.path.join(HERE, "golden", "reference_api_cem.json")))
    assert set(api) == {"CEM"}
    d = api["CEM"]
    mod, cls = d["mirror"].rsplit(".", 1)
    C = getattr(importlib.import_module(mod), cls)
    params = inspect.signature(C.__init__).parameters
    assert [p for p in params if p not in ("self", "kwargs")] == [a["name"] for a in d["init"]["args"]]
    for a in d["init"]["args"]:
        if a["default"] is not None:
            assert params[a["name"]].default == a["default"]["literal"], a["name"]
    assert any(p.kind == inspect.Parameter.VAR_KEYWORD for p in params.values()) == d["init"]["kwargs"]
    for base in d["bases"]:
        assert base in [b.__name__ for b in C.__mro__[1:]], base
    for m in d["methods"] + d["properties"]:
        assert hasattr(C, m), m


def test_cem_rejects_plot_and_pickles_constructor():
    import pickle
    from rllab_b200.algos.cem import CEM
    with pytest.raises(NotImplementedError):
        CEM(None, None, plot=True)
    algo = CEM(None, None, n_itr=4, n_samples=33, batch_size=500, seed=5)
    back = pickle.loads(pickle.dumps(algo))
    assert (back.n_itr, back.n_samples, back.batch_size, back.seed) == (4, 33, 500, 5)
