"""GaussianMLPBaseline (rllab/baselines/gaussian_mlp_baseline.py:10-49): the value function as a GaussianMLPRegressor
(rllab_b200/regressors/gaussian_mlp_regressor.py) named "vf", so the fit records vf_LossBefore, vf_LossAfter, vf_dLoss
and vf_MeanKL.

Host API fit(paths) / predict(path) as the reference's.  The sampler uses the device hooks instead:
  predict_lanes(batch)     batch.base = the regressor mean on the batch's observations (b200rl_vf_forward), before
                           process_samples (b200rl_process_samples_base), with the previous fit's weights
  fit_lanes(batch, comm)   the fit on the batch's returns of the valid samples, after the advantages (base.py:163-167)
Before the first fit the normalisation constants are 0 / 1, so iteration 0 is baselined by the untrained network, as in
the reference (LinearFeatureBaseline predicts zeros there).
"""
import numpy as np

from ..regressors.gaussian_mlp_regressor import GaussianMLPRegressor


class GaussianMLPBaseline(object):

    def __init__(
            self,
            env_spec,
            subsample_factor=1.,
            num_seq_inputs=1,
            regressor_args=None,
    ):
        if num_seq_inputs != 1:
            raise NotImplementedError("num_seq_inputs != 1")
        self._env_spec = env_spec
        self._subsample_factor = subsample_factor      # stored and never used, as in the reference
        self._num_seq_inputs = num_seq_inputs
        if regressor_args is None:
            regressor_args = dict()
        self._regressor_args = dict(regressor_args)
        self._regressor = GaussianMLPRegressor(
            input_shape=(env_spec.observation_space.flat_dim * num_seq_inputs,),
            output_dim=1,
            name="vf",
            **regressor_args
        )

    @property
    def regressor(self):
        return self._regressor

    def fit(self, paths):
        observations = np.concatenate([p["observations"] for p in paths])
        returns = np.concatenate([p["returns"] for p in paths])
        self._regressor.fit(observations, returns.reshape((-1, 1)))

    def predict(self, path):
        return self._regressor.predict(path["observations"]).flatten()

    def get_param_values(self, **tags):
        return self._regressor.get_param_values(**tags)

    def set_param_values(self, flattened_params, **tags):
        self._regressor.set_param_values(flattened_params, **tags)

    def log_diagnostics(self, paths):
        pass

    # ---- device hooks (LaneSampler.process_samples)
    def predict_lanes(self, batch):
        self._regressor.predict_device(batch.obs, batch.base.view(-1))

    def fit_lanes(self, batch, comm=None):
        flags = batch.flags.view(-1) if batch.masked else None
        self._regressor.fit_device(batch.obs, batch.ret.view(-1), flags, comm)

    def __getstate__(self):
        return dict(env_spec=self._env_spec, subsample_factor=self._subsample_factor,
                    num_seq_inputs=self._num_seq_inputs, regressor=self._regressor)

    def __setstate__(self, d):
        self._env_spec = d["env_spec"]
        self._subsample_factor = d["subsample_factor"]
        self._num_seq_inputs = d["num_seq_inputs"]
        self._regressor = d["regressor"]
        self._regressor_args = dict()
