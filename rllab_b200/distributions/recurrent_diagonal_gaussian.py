"""RecurrentDiagonalGaussian (rllab/distributions/recurrent_diagonal_gaussian.py): the reference defines it as
DiagonalGaussian itself.  Its numeric API works unchanged on the padded (n_paths, max_len, dim) arrays of a recurrent
samples_data: every reduction is over the last axis."""
from .diagonal_gaussian import DiagonalGaussian

RecurrentDiagonalGaussian = DiagonalGaussian
