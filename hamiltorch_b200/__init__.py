"""hamiltorch_b200 -- an H100-native (sm_90a) batched-chain HMC engine behind the hamiltorch surface.

Exports the same names as the reference's ``hamiltorch/__init__.py:1-4`` plus the engine's native additions
(``targets``, ``sample_chains``, ``diagnostics``, ``loo``, ``predictive``: held-out accuracy, NLL, Brier score,
calibration and predictive uncertainty of Bayesian NNs; ``sbc``: simulation-based calibration of a Bayesian-NN fit;
``ppc``: posterior predictive checks and LOO-PIT of a fitted Bayesian NN; chain and model stacking in ``loo``;
``sensitivity``: power-scaling prior and likelihood sensitivity of a fitted Bayesian NN).
The CUDA library is loaded lazily by the first sampling call and that call fails loudly if libhmcx.so is missing or no GPU
is present: there is no CPU fallback.
"""
__version__ = '0.1.0'

from . import diagnostics, loo, ppc, predictive, sbc, sensitivity, targets, util
from .samplers import (sample, sample_chains, sample_model, sample_split_model, predict_model, Sampler, Integrator,
                       Metric, leapfrog, hamiltonian, gibbs, acceptance, adaptation, define_model_log_prob,
                       define_split_model_log_prob)
from .util import set_random_seed
