"""CPU: the fp64 per-iteration replay of the in-kernel-metric RMHMC kernels (tests/rmhmc_ref.py), which
tests/test_rmhmc_ref_gpu.py holds those kernels to, is itself checked here.

* It accepts the unmodified reference's chains (committed fixtures: an explicit funnel with jitter, a dense softabs
  metric with jitter at D = 48, the implicit JACOBIAN_DIAG chain at D = 24) as if they were kernel output: identical
  decisions, Hamiltonians and proposals within the fixture's own measured error (parity.tol_for of the kernel's tags for
  that fixture: 8 x the kernel-vs-fixture error, floor 1e-5).
* It consumes the jitter rows the kernels consume: 8L + 3 per explicit iteration, and 3 + L (2m + 2) per implicit
  iteration with fixed_point_threshold = 0 (checked against the fp32 oracle's own count).
"""
import os

import numpy as np
import pytest
import torch

from hamiltorch_b200 import targets as T
from oracle import cases as K, rmhmc_oracle as R
from tests import dense_ref, parity, rmhmc_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _fixture_bound(name, chains):
    return max(parity.tol_for('rmhmc/%s/default/c%d/%s' % (name, c, k), 2e-3)
               for c in chains for k in ('ham_old', 'ham_new', 'samples'))


@pytest.mark.parametrize('name', ['rmhmc_exp_funnel5', 'rmhmc_exp_softabs_full48_jitter', 'rmhmc_imp_jacdiag_diag24'])
def test_replay_accepts_the_reference_rmhmc_chains(name):
    case = K.rmhmc_cases()[name]
    f = np.load(os.path.join(GOLDEN, name + '.npz'))
    # a chain whose reference run raised LogProbError (JACOBIAN_DIAG without jitter: a vanishing gradient component) has
    # no Hamiltonian there to compare with: its seed 24 of rmhmc_imp_jacdiag_diag24 is left out
    chains = [c for c in range(len(case['seeds'])) if not f.get('diverged_%d' % c, np.zeros(1, bool)).any()]
    assert chains
    C = len(chains)
    t = lambda k: torch.from_numpy(np.stack([f['%s_%d' % (k, c)] for c in chains]))
    S, L, burn, D = case['num_samples'], case['num_steps_per_sample'], case['burn'], case['target'].dim
    explicit = case['integrator'] == 'EXPLICIT'
    uni = None
    if case['jitter'] is not None:
        uni = t('uniforms').transpose(0, 1)                                     # (S, C, J, D)
        assert uni.shape[2] == 8 * L + 3                                        # the reference made no NaN retries
    model = rmhmc_ref.InKernelMetric(case['target'], case['metric'], case['jitter'], case['softabs_const'],
                                     explicit=explicit, omega=case.get('explicit_binding_const', 100),
                                     threshold=case.get('fixed_point_threshold', 1e-5),
                                     max_iter=case.get('fixed_point_max_iterations', 1000), uniforms=uni)
    init = torch.tensor(case['init'], dtype=torch.float32).expand(C, D).contiguous()
    eps = torch.full((C,), case['step_size'], dtype=torch.float64)             # the reference's python float
    acc, samples = t('accepted'), t('samples')
    ham = torch.stack([t('ham_old'), t('ham_new')], -1)
    rep = dense_ref.replay(model, init, acc, samples, t('z').transpose(0, 1), eps, L, burn)
    flips = dense_ref.check('cpu_rmhmc_replay/' + name, rep, init, samples, acc, ham, t('logu').t(), burn,
                            ceiling=_fixture_bound(name, chains))
    assert flips == 0
    if uni is not None:
        assert bool((model.counts() == 8 * L + 3).all())


def test_replay_consumes_the_implicit_rows_of_the_fp32_oracle():
    """fixed_point_threshold = 0: every fixed point runs m iterations on both sides, so an implicit iteration takes
    exactly 3 + L (2m + 2) jitter rows; the fp64 replay takes the same rows as the fp32 oracle and agrees with it."""
    tgt, D, S, L, m, burn, jitter = T.Funnel(5), 5, 4, 2, 3, 1, 1e-3
    J = 3 + L * (2 * m + 2)
    g = torch.Generator().manual_seed(3)
    init = torch.tensor([0.3, 0.8, -0.5, 0.4, -0.9])
    z, logu, uni = torch.randn(S, D, generator=g), torch.log(torch.rand(S, generator=g)), torch.rand(S, J, D, generator=g)
    logu[2] = 1.0                                                   # a forced reject after the burn-in
    o = R.sample_rmhmc(tgt, init, num_samples=S, num_steps_per_sample=L, step_size=0.1, burn=burn, jitter=jitter,
                       softabs_const=1e6, fixed_point_threshold=0.0, fixed_point_max_iterations=m,
                       integrator=R.IMPLICIT, metric=R.SOFTABS, normals=z, log_uniforms=logu, uniforms=uni)
    assert o['jitter_draws'] == [J] * S and o['nan_retries'] == [0] * S
    model = rmhmc_ref.InKernelMetric(tgt, 'SOFTABS', jitter, 1e6, explicit=False, threshold=0.0, max_iter=m,
                                     uniforms=uni[:, None])
    assert rmhmc_ref.rows_per_iteration(False, L, m) == J
    acc = torch.tensor([o['accepted']])
    samples = torch.stack(o['samples'])[None]
    ham = torch.tensor([o['ham_old'], o['ham_new']], dtype=torch.float64).t()[None]
    rep = dense_ref.replay(model, init[None], acc, samples, z[:, None], torch.tensor([0.1], dtype=torch.float64), L, burn)
    assert dense_ref.check('cpu_rmhmc_replay/implicit_funnel5', rep, init[None], samples, acc, ham, logu[:, None], burn,
                           ceiling=1e-5) == 0
    assert bool((model.counts() == J).all())
    assert 0 < int(acc.sum()) < S
