"""CPU: the fp64 per-iteration replay of the dense paths (tests/dense_ref.py), which the wide-tile GPU tests
(tests/test_dense_tiles_gpu.py) hold the kernels to, is itself checked here.

* It accepts the unmodified reference's chains (the committed fixtures) as if they were kernel output: identical
  decisions, states and Hamiltonians within FIXTURE_BOUND (funnel11_nuts, whose LogProbError iterations go through
  check(diverged=) and dual_averaging(diverged=), within FUNNEL_NUTS_BOUND).  The element-wise fixtures' accepted rows
  also equal the fp32 replay (replay_rows32) bit for bit.
* It accepts the fp32 oracle's chains at D = 250 (a full target with a full and with a diagonal mass) within
  ORACLE_BOUND.
* It rejects the same oracle runs made with one 64-column block of the precision or of inv_mass off by a relative 1e-4
  (of the order of one missing lo term of a 3xTF32 product, an estimate): the harness catches a one-tile error.
* It accepts the fp32 oracle's funnel chains at D = 16 and rejects them when the oracle's exp(v) sum(x^2) term is
  scaled by 1 + 1e-4.
* It accepts the fp32 oracle's element-wise chains at D = 250 (GaussianDiag, diagonal mass) and rejects them when one
  inv_var element is one ulp off, or the mass factor of a 64-column block is.
"""
import copy
import os

import numpy as np
import pytest
import torch

from hamiltorch_b200 import targets as T
from oracle import cases as K, hmc_oracle as O, rmhmc_oracle as R
from tests import dense_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
# 2x the largest scaled error max|a - d| / (1 + |d|) measured on the CPU: fixtures 1.2e-6 (the explicit RMHMC states;
# funnel11_hmc states 2.0e-6), oracle at D = 250 4.9e-7.  The perturbed runs below measure 1.9e-6 (inv_mass block) and
# 5.1e-6 (precision block).
FIXTURE_BOUND = 2.5e-6
ORACLE_BOUND = 1e-6
# funnel11_nuts: 2x its measured 5.3e-5 (states; Hamiltonians 9.1e-7).  Looser than the rest because its trajectories
# are chaotic: dual averaging drives the step size up to 1.35 over L = 25 steps through the funnel's neck, where the
# fp32 round-off of one evaluation (expf, summation order) is amplified along the trajectory before it ends.
FUNNEL_NUTS_BOUND = 1.1e-4


def _load(name):
    f = np.load(os.path.join(GOLDEN, name + '.npz'))
    C = len(f['seeds'])
    t = lambda k: torch.from_numpy(np.stack([f['%s_%d' % (k, c)] for c in range(C)]))
    ham = torch.stack([t('ham_old'), t('ham_new')], -1)
    return f, C, t, ham


def _run(model, init, acc, samples, z, logu, ham, eps, L, burn, tag, bound):
    rep = dense_ref.replay(model, init, acc, samples, z, eps, L, burn)
    return dense_ref.check(tag, rep, init, samples, acc, ham, logu, burn, ceiling=bound)


# the element-wise fixtures (GaussianIso / GaussianDiag, inv_mass None or (D,)): the kernels of hmcx_hmc.cu
ELEMENTWISE = ['cfg1_gauss3', 'iso256', 'diag48_mass', 'diag16_rejects', 'nuts_iso128']


@pytest.mark.parametrize('name', ['full48_dense', 'full40_fullmass', 'iso40_fullmass_nuts', 'iso40_blockmass',
                                  'cfg1_corr_gauss3', 'diag5_fullmass', 'diag6_blockmass', 'funnel11_hmc',
                                  'funnel11_nuts'] + ELEMENTWISE)
def test_replay_accepts_the_reference_hmc_chains(name):
    case = K.plain_cases()[name]
    kw = case['kw']
    f, C, t, ham = _load(name)
    S, L, burn = kw['num_samples'], kw['num_steps_per_sample'], kw['burn']
    init = t('init')
    z, logu = t('z').transpose(0, 1), t('logu').t()
    diverged = t('diverged')
    if kw.get('nuts'):
        eps = t('step_sizes').t().float()                    # teacher-forced: the step size each iteration used
        # the dual averaging restated in fp64 proposes the reference's next step sizes (eps_bar at n = burn); a
        # LogProbError iteration adapts with alpha = 0
        prop = dense_ref.dual_averaging(ham, burn, kw['step_size'], kw['desired_accept_rate'], diverged=diverged)
        np.testing.assert_allclose(prop.numpy(), eps[1:burn + 2].t().numpy(), rtol=2e-6)
    else:
        eps = torch.full((C,), kw['step_size'])
    model = dense_ref.HMC(case['target'], kw.get('inv_mass'))
    rep = dense_ref.replay(model, init, t('accepted'), t('samples'), z, eps, L, burn)
    flips = dense_ref.check('cpu_replay/' + name, rep, init, t('samples'), t('accepted'), ham, logu, burn,
                            ceiling=FUNNEL_NUTS_BOUND if name == 'funnel11_nuts' else FIXTURE_BOUND, diverged=diverged)
    assert flips == 0
    assert bool(diverged.any()) == (name == 'funnel11_nuts')
    if name in ELEMENTWISE:                                  # and every accepted retained row, bit for bit
        n = dense_ref.replay_rows32('cpu_replay/' + name, case['target'], kw.get('inv_mass'), init, t('accepted'),
                                    t('samples'), z, eps, L, burn)
        assert n == int(t('accepted')[:, burn + 1:].sum()) > 0


@pytest.mark.parametrize('name', ['rmhmc_exp_hess_full24', 'rmhmc_imp_softabs_diag20'])
def test_replay_accepts_the_reference_constant_metric_rmhmc_chains(name):
    case = K.rmhmc_cases()[name]
    f, C, t, ham = _load(name)
    D = case['target'].dim
    init = torch.tensor(case['init'], dtype=torch.float32).expand(C, D).contiguous()
    model = dense_ref.RMHMC(case['target'], case['metric'] == 'SOFTABS', case['softabs_const'],
                            explicit=case['integrator'] == 'EXPLICIT', omega=case.get('explicit_binding_const', 100))
    eps = torch.full((C,), case['step_size'])
    flips = _run(model, init, t('accepted'), t('samples'), t('z').transpose(0, 1), t('logu').t(), ham, eps,
                 case['num_steps_per_sample'], case['burn'], 'cpu_replay/' + name, FIXTURE_BOUND)
    assert flips == 0


# ---- the fp32 oracle at D = 250, a shape of the wide-tile GPU tests ------------------------------------------------
D250, C3, S6, L5 = 250, 3, 6, 5
EPS3 = torch.tensor([0.22, 0.25, 0.28])          # one step size per chain, as in the GPU tests


def _target(D, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(D, D, generator=g, dtype=torch.float64) / D ** 0.5
    return T.GaussianFull(torch.randn(D, generator=g), cov=A @ A.t() + 0.5 * torch.eye(D, dtype=torch.float64))


def _mass(kind, D):
    g = torch.Generator().manual_seed(7)
    if kind == 'diag':
        return 0.5 + torch.rand(D, generator=g)
    A = torch.randn(D, D, generator=g, dtype=torch.float64) / D ** 0.5
    return (A @ A.t() + 0.7 * torch.eye(D, dtype=torch.float64)).float()


def _oracle(tgt, im):
    D = tgt.dim
    outs, inits, zs, lus = [], [], [], []
    for c in range(C3):
        init, z, logu, _ = O.reference_stream(300 + c, D, S6, prior=lambda: tgt.mean + 0.3 * torch.randn(D))
        outs.append(O.sample_hmc(tgt, init, num_samples=S6, num_steps_per_sample=L5, step_size=float(EPS3[c]),
                                 inv_mass=im, normals=z, log_uniforms=logu))
        inits.append(init), zs.append(z), lus.append(logu)
    acc = torch.tensor([o['accepted'] for o in outs])
    samples = torch.stack([torch.stack(o['samples']) for o in outs])
    ham = torch.tensor([[o['ham_old'], o['ham_new']] for o in outs], dtype=torch.float64).transpose(1, 2)
    return torch.stack(inits), acc, samples, torch.stack(zs, 1), torch.stack(lus, 1), ham


@pytest.mark.parametrize('mass', ['full', 'diag'])
def test_replay_accepts_the_oracle_at_d250(mass):
    tgt, im = _target(D250, 5), _mass(mass, D250)
    init, acc, samples, z, logu, ham = _oracle(tgt, im)
    assert 0 < int(acc.sum()) < acc.numel() + 1
    flips = _run(dense_ref.HMC(tgt, im), init, acc, samples, z, logu, ham, EPS3, L5, 0, 'cpu_replay/d250_' + mass,
                 ORACLE_BOUND)
    assert flips == 0


@pytest.mark.parametrize('mass,operand', [('full', 'prec'), ('full', 'inv_mass'), ('diag', 'prec')])
def test_replay_rejects_one_perturbed_64_column_block(mass, operand):
    tgt, im = _target(D250, 5), _mass(mass, D250)
    bad_tgt, bad_im = tgt, im
    if operand == 'prec':
        bad_tgt = copy.copy(tgt)                 # same log_norm: only the contraction is off
        bad_tgt.prec = tgt.prec.clone()
        bad_tgt.prec[:, 64:128] *= 1 + 1e-4
    else:
        bad_im = im.clone()
        bad_im[:, 64:128] *= 1 + 1e-4
    init, acc, samples, z, logu, ham = _oracle(bad_tgt, bad_im)
    with pytest.raises(AssertionError, match='tolerance'):
        _run(dense_ref.HMC(tgt, im), init, acc, samples, z, logu, ham, EPS3, L5, 0,
             'cpu_replay/d250_%s_bad_%s' % (mass, operand), ORACLE_BOUND)


# ---- Neal's funnel: the fp32 oracle at D = 16, and a mutated funnel ----------------------------------------------------
class _ScaledFunnel(T.Funnel):
    """targets.Funnel with its exp(v) sum(x^2) term scaled by 1 + rel."""

    def __init__(self, dim, rel):
        super().__init__(dim)
        self.rel = rel

    def __call__(self, w):
        return super().__call__(w) - 0.5 * self.rel * torch.exp(w[0]) * (w[1:] * w[1:]).sum()


def _funnel_oracle(tgt, eps):
    D = tgt.dim
    outs, inits, zs, lus = [], [], [], []
    for c in range(C3):
        init, z, logu, _ = O.reference_stream(
            400 + c, D, S6, prior=lambda: torch.cat([0.3 * torch.randn(1), 0.6 * torch.randn(D - 1)]))
        outs.append(O.sample_hmc(tgt, init, num_samples=S6, num_steps_per_sample=L5, step_size=float(eps[c]),
                                 normals=z, log_uniforms=logu))
        inits.append(init), zs.append(z), lus.append(logu)
    acc = torch.tensor([o['accepted'] for o in outs])
    samples = torch.stack([torch.stack(o['samples']) for o in outs])
    ham = torch.tensor([[o['ham_old'], o['ham_new']] for o in outs], dtype=torch.float64).transpose(1, 2)
    return torch.stack(inits), acc, samples, torch.stack(zs, 1), torch.stack(lus, 1), ham


@pytest.mark.parametrize('rel', [0.0, 1e-4])
def test_replay_checks_the_funnel(rel):
    """The unmodified oracle passes within ORACLE_BOUND; scaling its exp(v) sum(x^2) term by 1 + 1e-4 fails the replay."""
    eps = torch.tensor([0.1, 0.12, 0.14])
    tgt = T.Funnel(16)
    init, acc, samples, z, logu, ham = _funnel_oracle(_ScaledFunnel(16, rel) if rel else tgt, eps)
    assert 0 < int(acc.sum()) < acc.numel()
    args = (dense_ref.HMC(tgt), init, acc, samples, z, logu, ham, eps, L5, 0, 'cpu_replay/funnel16_%g' % rel,
            ORACLE_BOUND)
    if rel:
        with pytest.raises(AssertionError, match='tolerance'):
            _run(*args)
    else:
        assert _run(*args) == 0


# ---- element-wise chains: the fp32 oracle at D = 250, with one inv_var element or a block of the mass factor one ulp off --
def _elem_problem():
    g = torch.Generator().manual_seed(11)
    tgt = T.GaussianDiag(torch.linspace(-1, 1, D250), 0.5 + torch.rand(D250, generator=g))
    return tgt, 0.5 + torch.rand(D250, generator=g)


def _elem_oracle(tgt, im):
    outs, inits, zs, lus = [], [], [], []
    for c in range(C3):
        init, z, logu, _ = O.reference_stream(500 + c, D250, S6, prior=lambda: tgt.mean + torch.randn(D250))
        outs.append(O.sample_hmc(tgt, init, num_samples=S6, num_steps_per_sample=L5, step_size=float(EPS3[c]),
                                 burn=1, inv_mass=im, normals=z, log_uniforms=logu))
        inits.append(init), zs.append(z), lus.append(logu)
    acc = torch.tensor([o['accepted'] for o in outs])
    samples = torch.stack([torch.stack(o['samples']) for o in outs])
    ham = torch.tensor([[o['ham_old'], o['ham_new']] for o in outs], dtype=torch.float64).transpose(1, 2)
    return torch.stack(inits), acc, samples, torch.stack(zs, 1), torch.stack(lus, 1), ham


def _up_one_ulp(x):
    return torch.nextafter(x, torch.full_like(x, float('inf')))


@pytest.mark.parametrize('fault', [None, 'inv_var', 'mass_factor'])
def test_elementwise_row_replay_is_bit_exact(fault, monkeypatch):
    """replay + check + replay_rows32 accept the oracle's GaussianDiag chains with a diagonal mass; one inv_var element
    one ulp off, or the mass factor of columns 64..127 one ulp off, makes some accepted row differ bit-wise."""
    tgt, im = _elem_problem()
    run_tgt = tgt
    if fault == 'inv_var':
        run_tgt = copy.copy(tgt)
        run_tgt.inv_var = tgt.inv_var.clone()
        run_tgt.inv_var[100] = _up_one_ulp(tgt.inv_var[100])
    elif fault == 'mass_factor':
        factor = (1 / im) ** 0.5
        factor[64:128] = _up_one_ulp(factor[64:128])
        monkeypatch.setattr(O, 'momentum_from_normals', lambda z, mass, scale_tril=None: z * factor)
    init, acc, samples, z, logu, ham = _elem_oracle(run_tgt, im)
    assert 0 < int(acc[:, 2:].sum()) < acc[:, 2:].numel()
    flips = _run(dense_ref.HMC(tgt, im), init, acc, samples, z, logu, ham, EPS3, L5, 1, 'cpu_replay/elem250',
                 ORACLE_BOUND)
    assert flips == 0
    rows = lambda: dense_ref.replay_rows32('cpu_replay/elem250', tgt, im, init, acc, samples, z, EPS3, L5, 1)
    if fault:
        with pytest.raises(AssertionError, match='bit-wise'):
            rows()
    else:
        assert rows() == int(acc[:, 2:].sum())
