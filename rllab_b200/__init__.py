"""rllab_b200: H100-native (sm_90a CUDA behind a ctypes C ABI) implementation of rllab's data-parallel hot path --
lock-step lane rollout, process_samples, VPG / TRPO update -- behind rllab's own plugin API
(Env / Policy / Baseline / Sampler / BatchPolopt).  See DESIGN.md and INTEGRATION.md."""
__version__ = "0.1.0"
