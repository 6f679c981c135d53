"""ctypes binding of libb200rl.so (the C ABI declared in include/b200rl.h).

The product path has NO fallback: if the shared library is missing or a call fails, a RuntimeError is raised.
PyTorch is used only as the device-memory / stream container: every call passes raw device pointers
(`tensor.data_ptr()`) and the current CUDA stream.
"""
import ctypes
import os
from ctypes import (POINTER, c_char_p, c_double, c_float, c_int, c_longlong, c_uint, c_void_p)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libb200rl.so")

ENV_POINT, ENV_CARTPOLE, ENV_PENDULUM, ENV_SWIMMER, ENV_HOPPER, ENV_CARTPOLE_SWINGUP, ENV_DOUBLE_PENDULUM = 0, 1, 2, 3, 4, 5, 6
ENV_HALF_CHEETAH = 7
ENV_KINDS = dict(point=ENV_POINT, cartpole=ENV_CARTPOLE, pendulum=ENV_PENDULUM, swimmer=ENV_SWIMMER, hopper=ENV_HOPPER,
                 cartpole_swingup=ENV_CARTPOLE_SWINGUP, double_pendulum=ENV_DOUBLE_PENDULUM,
                 half_cheetah=ENV_HALF_CHEETAH)
# Discrete-action env kinds (b200rl_env_num_actions > 0): driven by the categorical rollout only, so they are kept out of
# ENV_KINDS, the Box-action kinds every Gaussian test grid covers.
ENV_GYM_CARTPOLE = 8
DISCRETE_ENV_KINDS = dict(gym_cartpole=ENV_GYM_CARTPOLE)
NOISE_UNIFORM, NOISE_NORMAL = 0, 1
LOSS_TRPO, LOSS_VPG, LOSS_KL = 0, 1, 2
FLAG_DONE, FLAG_END, FLAG_CUT, FLAG_MASKED = 1, 2, 4, 8
PS_NSUM, PS_NMAX = 16, 4

_P = c_void_p
_LL = c_longlong

DDPG_BATCH, DDPG_NSTAT = 32, 9
DDPG_STREAM_EXPLORE, DDPG_STREAM_INDEX = 3, 4
ES_OU, ES_GAUSSIAN = 0, 1


class DdpgHparams(ctypes.Structure):
    """b200rl_ddpg_hparams."""
    _fields_ = [(n, c_int) for n in ("n_updates_per_sample", "max_path_length", "min_pool_size", "replay_pool_size",
                                     "include_horizon_terminal_transitions", "es_kind")] + \
               [(n, c_double) for n in ("discount", "scale_reward", "soft_target_tau", "qf_weight_decay",
                                        "qf_learning_rate", "policy_weight_decay", "policy_learning_rate", "ou_mu",
                                        "ou_theta", "ou_sigma", "gs_max_sigma", "gs_min_sigma", "gs_decay_period")]


class DdpgState(ctypes.Structure):
    """b200rl_ddpg_state: one run's train() loop state between launches."""
    _fields_ = [("env_state", c_float * 8), ("obs", c_float * 8), ("ou_state", c_double * 4), ("path_return", c_double),
                ("itr", c_longlong), ("adam_t", c_longlong), ("path_length", c_int), ("terminal", c_int),
                ("top", c_int), ("bottom", c_int), ("size", c_int), ("pad_", c_int)]


class DdpgTrainArgs(ctypes.Structure):
    """b200rl_ddpg_train_args."""
    _fields_ = [("env_kind", c_int), ("f64", c_int), ("n_runs", c_int), ("n_steps", c_int), ("es_cap", c_int),
                ("seed", c_uint), ("hp", DdpgHparams), ("state", c_void_p), ("nets", c_void_p),
                ("pool_obs", c_void_p), ("pool_act", c_void_p), ("pool_rew", c_void_p), ("pool_term", c_void_p),
                ("stats", c_void_p), ("es_returns", c_void_p), ("stream", c_void_p)]

# name -> (restype, argtypes).  Mirrors include/b200rl.h one to one (tests/test_abi.py checks the header against this).
SIGNATURES = {
    "b200rl_last_error": (c_char_p, []),
    "b200rl_version": (c_int, []),
    "b200rl_kernel_launches": (ctypes.c_ulonglong, []),
    "b200rl_device_sms": (c_int, [POINTER(c_int)]),
    "b200rl_bench_ffma2": (c_int, [c_int, _P, POINTER(_LL), _P]),
    "b200rl_env_info": (c_int, [c_int, POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_int),
                                POINTER(c_float), POINTER(c_float)]),
    "b200rl_env_num_actions": (c_int, [c_int, POINTER(c_int)]),
    "b200rl_policy_num_params": (_LL, [c_int, c_int, c_int, c_int]),
    "b200rl_fill_noise": (c_int, [_P, c_int, c_int, c_int, c_int, _LL, c_int, c_uint, c_uint, c_int, _P]),
    "b200rl_env_reset": (c_int, [c_int, c_int, _P, _P, _P, c_uint, c_uint, c_int, _LL, _P]),
    "b200rl_env_step": (c_int, [c_int, c_int, c_int, _P, _P, _P, _P, _P, _P]),
    "b200rl_policy_get_actions": (c_int, [_P, c_int, c_int, c_int, c_int, c_float, _P, _LL, _P, c_uint, c_uint, c_int,
                                          _LL, _P, _P, _P, _P]),
    "b200rl_rollout": (c_int, [c_int, _P, c_int, c_int, c_float, c_int, c_int, c_int, _P, _P, c_uint, c_uint, _LL,
                               _P, _P, _P, _P, _P, _P, _P, _P]),
    "b200rl_process_samples": (c_int, [c_int, c_int, c_int, _P, _P, _P, _P, _P, c_double, c_double, c_int, _P, _P, _P,
                                       _P, _P, _P, _P]),
    "b200rl_process_samples_base": (c_int, [c_int, c_int, c_int, _P, _P, _P, _P, _P, c_double, c_double, c_int, _P, _P,
                                            _P, _P, _P, _P]),
    "b200rl_center_advantages": (c_int, [_P, _LL, _P, _P, _P, c_int, c_int, _P]),
    "b200rl_lfb_gram": (c_int, [c_int, _LL, _P, _P, _P, _P, _P, _P, _P]),
    "b200rl_lfb_solve": (c_int, [c_int, _P, c_double, _P, _P, _P]),
    "b200rl_loss_kl": (c_int, [c_int, _P, c_int, c_int, c_int, c_int, c_float, _LL, _P, _P, _P, _P, _P, _P, c_double, _P,
                               _P, _P, _P]),
    "b200rl_grad": (c_int, [c_int, _P, c_int, c_int, c_int, c_int, c_float, _LL, _P, _P, _P, _P, _P, _P, c_double, _P,
                            _P, _P, _P, _P, _P]),
    "b200rl_grad_penalized": (c_int, [c_int, c_double, _P, c_int, c_int, c_int, c_int, c_float, _LL, _P, _P, _P, _P,
                                      _P, _P, c_double, _P, _P, _P, _P, _P]),
    "b200rl_fvp": (c_int, [_P, c_int, c_int, c_int, c_int, c_float, _LL, _P, _P, _P, c_double, _P, c_double, c_double,
                           _P, _P, _P, c_int, _P, _P]),
    "b200rl_count_valid": (c_int, [_LL, _P, _P, c_int, _P, _P, _P]),
    "b200rl_update_f64": (c_int, [c_int, c_int, _P, c_int, c_int, c_int, c_int, c_double, _LL, _P, _P, _P, _P, _P, _P,
                                  _P, c_double, _P, c_double, c_double, _P, _P, _P, _P]),
    "b200rl_ws_doubles": (_LL, []),
    "b200rl_cg_init": (c_int, [_LL, _P, _P, _P, _P, _P, c_int, _P]),
    "b200rl_cg_step": (c_int, [_LL, _P, _P, _P, _P, _P, c_double, c_int, _P]),
    "b200rl_trpo_step_size": (c_int, [_LL, _P, _P, c_double, _P, _P, _P]),
    "b200rl_axpy_params": (c_int, [_LL, _P, _P, c_double, _P, _P, _P]),
    "b200rl_adam_step": (c_int, [_LL, _P, _P, _P, _P, _P, _LL, c_double, c_double, c_double, c_double, _P]),
    "b200rl_f64_to_f32": (c_int, [_LL, _P, _P, _P]),
    "b200rl_peer_window_bytes": (_LL, [c_int, _LL]),
    "b200rl_peer_window_create": (c_int, [c_int, _LL, POINTER(c_void_p), _P]),
    "b200rl_peer_window_open": (c_int, [_P, POINTER(c_void_p)]),
    "b200rl_peer_window_close": (c_int, [_P]),
    "b200rl_peer_window_destroy": (c_int, [_P]),
    "b200rl_peer_bind": (c_int, [_P, c_int, c_int, _LL]),
    "b200rl_peer_allreduce_mixed": (c_int, [_P, _LL, _LL, _P]),
    "b200rl_peer_fuse_updates": (c_int, [c_int]),
    "b200rl_peer_timeouts": (c_int, [POINTER(c_uint)]),
    "b200rl_reduce_ranks": (c_int, [_P, c_int, _LL, _LL, _P, _P]),
    "b200rl_planes_to_rows_f64": (c_int, [c_int, _LL, _P, _P, _P]),
    "b200rl_vf_num_params": (_LL, [c_int, c_int, c_int]),
    "b200rl_vf_norm_stats": (c_int, [c_int, _LL, _P, _P, _P, c_int, _P, _P, _P, _P]),
    "b200rl_vf_forward": (c_int, [_P, c_int, c_int, c_int, _LL, _P, _P, c_int, _P, _P]),
    "b200rl_vf_loss_grad": (c_int, [_P, c_int, c_int, c_int, _LL, _P, _P, _P, _P, _P, c_float, c_double, c_int, c_double,
                                    _P, _P, _P, _P, _P]),
    "b200rl_population_sample": (c_int, [_LL, _P, _P, c_double, c_uint, c_uint, _P, _LL, c_int, _P, _P]),
    "b200rl_population_rollout": (c_int, [c_int, c_int, c_int, c_float, _P, c_int, c_int, c_int, c_double, c_uint, c_uint,
                                          _LL, _P, _P, _P, _P, _P, _P, _P, _P]),
    "b200rl_population_topk": (c_int, [_P, c_int, c_int, _P, _P, _P]),
    "b200rl_rows_mean_std": (c_int, [_LL, c_int, _P, _P, _P, _P]),
    "b200rl_reps_delta_max": (c_int, [c_int, c_int, c_int, _P, _P, _P, _P, c_int, _P, _P, _P, _P]),
    "b200rl_reps_dual_sums": (c_int, [c_int, c_int, c_int, _P, _P, _P, _P, c_int, _P, c_double, _P, _P, _P, _P, _P]),
    "b200rl_categorical_num_params": (_LL, [c_int, c_int, c_int, c_int]),
    "b200rl_categorical_get_actions": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _LL, _P, c_uint, c_uint, c_int, _LL,
                                               _P, _P, _P]),
    "b200rl_rollout_categorical": (c_int, [c_int, _P, c_int, c_int, c_int, c_int, c_int, _P, _P, c_uint, c_uint, _LL,
                                           _P, _P, _P, _P, _P, _P, _P]),
    "b200rl_categorical_loss_kl": (c_int, [c_int, _P, c_int, c_int, c_int, c_int, _LL, _P, _P, _P, _P, _P, c_double, _P,
                                           _P, _P, _P]),
    "b200rl_categorical_grad": (c_int, [c_int, c_double, _P, c_int, c_int, c_int, c_int, _LL, _P, _P, _P, _P, _P,
                                        c_double, _P, _P, _P, _P, _P, _P]),
    "b200rl_categorical_fvp": (c_int, [_P, c_int, c_int, c_int, c_int, _LL, _P, _P, _P, c_double, _P, c_double, c_double,
                                       _P, _P, _P, c_int, _P, _P]),
    "b200rl_categorical_entropy": (c_int, [c_int, _LL, _P, _P, _P, _P, _P]),
    "b200rl_categorical_update_f64": (c_int, [c_int, c_int, _P, c_int, c_int, c_int, c_int, _LL, _P, _P, _P, _P, _P,
                                              _P, c_double, _P, c_double, c_double, _P, _P, _P, _P]),
    "b200rl_gru_num_params": (_LL, [c_int, c_int, c_int, c_int]),
    "b200rl_gru_get_actions": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P, _P, _LL, _P, c_uint, c_uint, c_int, _LL,
                                       _P, _P, _P, _P, _P]),
    "b200rl_rollout_gru": (c_int, [c_int, _P, c_int, c_int, c_int, c_int, c_int, _P, _P, c_uint, c_uint, _LL, _P, _P,
                                   _P, _P, _P, _P, _P, _P]),
    "b200rl_gru_loss_kl": (c_int, [c_int, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P,
                                   c_double, _P, _P, _P, _P, _P]),
    "b200rl_gru_grad": (c_int, [c_int, c_double, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P,
                                _P, c_double, _P, _P, _P, _P, _P, _P]),
    "b200rl_gru_fvp": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, c_double, _P, c_double,
                               c_double, _P, _P, c_int, _P, _P]),
    "b200rl_gru_update_f64": (c_int, [c_int, c_int, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P,
                                      _P, _P, _P, c_double, _P, c_double, c_double, _P, _P, _P, _P, _P]),
    "b200rl_categorical_gru_num_params": (_LL, [c_int, c_int, c_int, c_int]),
    "b200rl_categorical_gru_get_actions": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P, _P, _LL, _P, c_uint, c_uint,
                                                   c_int, _LL, _P, _P, _P, _P]),
    "b200rl_rollout_categorical_gru": (c_int, [c_int, _P, c_int, c_int, c_int, c_int, c_int, _P, _P, c_uint, c_uint, _LL,
                                               _P, _P, _P, _P, _P, _P, _P]),
    "b200rl_categorical_gru_loss_kl": (c_int, [c_int, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P,
                                               _P, c_double, _P, _P, _P, _P, _P]),
    "b200rl_categorical_gru_grad": (c_int, [c_int, c_double, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, _P,
                                            _P, _P, _P, c_double, _P, _P, _P, _P, _P, _P]),
    "b200rl_categorical_gru_fvp": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, c_double,
                                           _P, c_double, c_double, _P, _P, c_int, _P, _P, _P]),
    "b200rl_categorical_gru_update_f64": (c_int, [c_int, c_int, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, _P,
                                                  _P, _P, _P, _P, c_double, _P, c_double, c_double, _P, _P, _P, _P, _P]),
    "b200rl_ddpg_num_params": (_LL, [c_int, c_int, c_int]),
    "b200rl_deterministic_get_actions": (c_int, [_P, c_int, c_int, _P, _LL, _P, _P]),
    "b200rl_qf_get_qval": (c_int, [_P, c_int, c_int, _P, _P, _LL, _P, _P]),
    "b200rl_rollout_deterministic": (c_int, [c_int, _P, c_int, c_int, c_int, _P, c_uint, c_uint, _LL, _P, _P, _P, _P,
                                             _P, _P]),
    "b200rl_ddpg_update": (c_int, [c_int, c_int, POINTER(DdpgHparams), _P, _P, _P, _P, c_int, _P, _P, _LL, _P, _P, _P,
                                   _P, _P]),
    "b200rl_ddpg_train": (c_int, [POINTER(DdpgTrainArgs)]),
}

_lib = None
launch_count = 0   # number of library calls that enqueue at least one kernel (bench.py reports it)


class B200RLError(RuntimeError):
    pass


def load():
    """Load libb200rl.so; raise loudly if it has not been built (python __graft_entry__.py / make -C rllab_b200/csrc)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200RLError(
            "libb200rl.so not found at %s: build it with `make -C rllab_b200/csrc -j8` "
            "(there is no CPU fallback for the hot path)" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if a declared symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error():
    return load().b200rl_last_error().decode("utf-8", "replace")


def check(rc, what=""):
    if rc != 0:
        raise B200RLError("%s failed (%d): %s" % (what or "libb200rl call", rc, last_error()))


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else c_void_p(t.data_ptr())


def call(name, *args):
    global launch_count
    lib = load()
    rc = getattr(lib, name)(*args)
    launch_count += 1
    check(rc, name)


def kernel_launches():
    return int(load().b200rl_kernel_launches())


def env_info(kind):
    lib = load()
    o, a, s, k, nk = c_int(), c_int(), c_int(), c_int(), c_int()
    lb = (c_float * 8)()
    ub = (c_float * 8)()
    check(lib.b200rl_env_info(kind, o, a, s, k, nk, lb, ub), "b200rl_env_info")
    return dict(obs_dim=o.value, act_dim=a.value, state_dim=s.value, reset_dim=k.value, noise_kind=nk.value,
                lb=[lb[i] for i in range(a.value)], ub=[ub[i] for i in range(a.value)])


def policy_num_params(O, h1, h2, A):
    n = load().b200rl_policy_num_params(O, h1, h2, A)
    if n < 0:
        raise B200RLError("unsupported policy network O=%d hidden=(%d,%d) A=%d: %s" % (O, h1, h2, A, last_error()))
    return int(n)


def vf_num_params(O, h1=32, h2=32):
    n = load().b200rl_vf_num_params(O, h1, h2)
    if n < 0:
        raise B200RLError("unsupported regressor network O=%d hidden=(%d,%d): %s" % (O, h1, h2, last_error()))
    return int(n)


def env_num_actions(kind):
    """Number of discrete actions of an env kind (its action space is Discrete(n)); 0 for a Box action space."""
    lib = load()
    n = c_int()
    check(lib.b200rl_env_num_actions(kind, n), "b200rl_env_num_actions")
    return n.value


def categorical_num_params(O, h1, h2, n):
    p = load().b200rl_categorical_num_params(O, h1, h2, n)
    if p < 0:
        raise B200RLError("unsupported categorical network O=%d hidden=(%d,%d) n=%d: %s" % (O, h1, h2, n, last_error()))
    return int(p)


def gru_num_params(O, H, A, include_action):
    p = load().b200rl_gru_num_params(O, H, A, int(bool(include_action)))
    if p < 0:
        raise B200RLError("unsupported GRU network O=%d hidden=%d A=%d: %s" % (O, H, A, last_error()))
    return int(p)


def categorical_gru_num_params(O, H, n, include_action):
    p = load().b200rl_categorical_gru_num_params(O, H, n, int(bool(include_action)))
    if p < 0:
        raise B200RLError("unsupported categorical GRU network O=%d hidden=%d n=%d: %s" % (O, H, n, last_error()))
    return int(p)


def ddpg_num_params(O, A):
    """(P_policy, P_qf) of the DDPG nets at (obs_dim, act_dim)."""
    lib = load()
    pp, qp = lib.b200rl_ddpg_num_params(O, A, 0), lib.b200rl_ddpg_num_params(O, A, 1)
    if pp < 0 or qp < 0:
        raise B200RLError("unsupported DDPG networks O=%d A=%d: %s" % (O, A, last_error()))
    return int(pp), int(qp)
