"""GPU: simulation-based calibration of Bayesian NNs (hamiltorch_b200.sbc, csrc/hmcx_sbc.cu).

1. simulate: theta~, the chain starts and regression y against tests/sbc_oracle.py within the Box-Muller .approx bounds;
   binary and multi-class labels identical away from class boundaries; the same bits on every call and for the first
   sims of a larger call.
2. Every fit row is, bit for bit, a one-chain sample_chains on its sim's data with its chain id as chain_offset: SIMT and
   tensor-core stacks, regression and multi-class, HMC and HMC_NUTS, and a run whose last launch is smaller.
3. ranks: parameter columns equal a count on the returned block; the log-likelihood column a count against fp64 sums of
   loo.pointwise_log_lik.
4. Calibration, with fixed seeds: the conjugate nn.Linear(3, 1) regression and an nn.Linear(2, 3) multi-class logistic
   regression pass every column; a stalled fit fails the log-likelihood column while its parameter columns pass."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn

import hamiltorch_b200 as hb
from hamiltorch_b200 import loo as LOO, sbc, targets as T
from oracle import cases
from tests import sbc_oracle as SO
from tests.test_loo_cpu import _conjugate

pytestmark = pytest.mark.gpu

NORMAL_ATOL = 5e-5              # the momentum stream's bound on a Box-Muller normal (tests/test_philox_stream_gpu.py)


def _tanh_target(loss='regression', n=50, n_out=2, tau_out=4.0):
    g = torch.Generator().manual_seed(3)
    model = nn.Sequential(nn.Linear(3, 8), nn.Tanh(), nn.Linear(8, n_out))
    x = torch.randn(n, 3, generator=g)
    y = torch.randint(0, n_out, (n,), generator=g).float() if loss == 'multi_class_linear_output' else \
        torch.zeros(n, n_out)
    tau = [torch.tensor(v) for v in (1.0, 4.0, 0.5, 2.0)]
    return T.MLPTarget.from_model(model, x, y, tau, tau_out, prior_scale=1.5, model_loss=loss)


def _tc_target():                                                  # 64-128-1: the tensor-core form (config 4's network)
    model, x, y = cases.mlp_problem(seed=8, n=300, n_in=64, hidden=128)
    # prior sd 1/8: the prior draws' outputs stay O(1), so plain HMC from one prior draw accepts on another's data
    return T.MLPTarget.from_model(model, x, y, [torch.tensor(64.)] * 4, 20., prior_scale=1.0)


def _f64(target, theta):
    """(M, N, O) fp64 network outputs of the GPU's theta~ rows."""
    th = theta.detach().cpu().double()
    x = target.x.double()
    t = copy.copy(target)
    return torch.stack([t.forward(th[m], x) for m in range(th.shape[0])]).numpy()


# ------------------------------------------------------------------------------------------------------------------
# 1. simulation
# ------------------------------------------------------------------------------------------------------------------
def test_prior_draws_and_regression_data_match_the_oracle():
    t = _tanh_target()
    sim = sbc.simulate(t, 12, chains_per_sim=3, seed=5)
    torch.cuda.synchronize()
    ref = SO.prior(5, range(12), 3, t)                            # (12, 4, D)
    sd = SO.element_sd(t)
    got = sim.block[:, :, :t.dim].cpu().double().numpy()
    assert np.all(np.abs(got - ref) <= NORMAL_ATOL * sd + 1e-6 * np.abs(ref))
    assert torch.equal(sim.theta.cpu(), sim.block[:, 0, :t.dim].cpu()) and sim.init.shape == (12, 3, t.dim)
    assert float(sim.block[:, :, t.dim:].abs().max()) == 0.0 if sim.block.shape[2] > t.dim else True
    f = _f64(t, sim.theta)
    yref = SO.simulate_regression(5, range(12), f, t.tau_out)
    assert np.all(np.abs(sim.y.cpu().double().numpy() - yref) <= NORMAL_ATOL / np.sqrt(t.tau_out) + 1e-5)
    # the same bits on a second call; the first 5 sims of 12 are a call of 5
    again = sbc.simulate(t, 12, chains_per_sim=3, seed=5)
    five = sbc.simulate(t, 5, chains_per_sim=3, seed=5)
    torch.cuda.synchronize()
    assert torch.equal(again.block, sim.block) and torch.equal(again.y, sim.y)
    assert torch.equal(five.block, sim.block[:5]) and torch.equal(five.y, sim.y[:5])
    other = sbc.simulate(t, 5, chains_per_sim=3, seed=6)
    assert not torch.equal(other.block, five.block)


# seeds and sizes whose every draw lies more than 1e-4 from its class boundary (fp64 oracle on the oracle's prior draws)
@pytest.mark.parametrize('loss, n_out, n, seed', [('binary_class_linear_output', 2, 100, 10),
                                                  ('multi_class_linear_output', 4, 400, 11)])
def test_classification_labels_match_the_oracle(loss, n_out, n, seed):
    t = _tanh_target(loss, n=n, n_out=n_out, tau_out=1.0)
    sim = sbc.simulate(t, 16, chains_per_sim=2, seed=seed)
    torch.cuda.synchronize()
    f = _f64(t, sim.theta)
    if loss == 'binary_class_linear_output':
        yref, dist = SO.simulate_binary(seed, range(16), f)
    else:
        yref, dist = SO.simulate_multiclass(seed, range(16), f)
        yref = yref[..., None]
        dist = dist[..., None]
    got = sim.y.cpu().double().numpy()
    assert got.shape == yref.shape
    near = dist < 1e-5
    assert int(near.sum()) == 0                                   # none at these sizes: every label is compared
    assert np.array_equal(got[~near], yref[~near])
    assert set(np.unique(got)) <= set(range(n_out))
    again = sbc.simulate(t, 16, chains_per_sim=2, seed=seed)
    assert torch.equal(again.y, sim.y)


# ------------------------------------------------------------------------------------------------------------------
# 2. every fit row is a plain run
# ------------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.contiguous().view(torch.int32)


def _plain(sim, t, m, r, g, kw):
    tm = copy.copy(t)
    tm.y = sim.y[m]
    a = dict(kw)
    thin = a.pop('thin', 1)
    return hb.sample_chains(tm, sim.init[m, r][None].clone(), chain_offset=g, rng='philox', thin=thin, **a)


def _assert_row(res, c, ref):
    assert torch.equal(res.accepted[c], ref.accepted[0]) and torch.equal(res.num_rejected[c], ref.num_rejected[0])
    assert torch.equal(res.step_size[c], ref.step_size[0])
    assert torch.equal(_bits(res.samples[c]), _bits(ref.samples[0]))


FITS = [('tanh', 'HMC'), ('tanh', 'NUTS'), ('tc', 'NUTS'), ('tc', 'HMC'), ('multiclass', 'HMC'),
        ('multiclass', 'NUTS')]


@pytest.mark.parametrize('shape, sampler', FITS)
def test_every_fit_row_is_a_plain_run(shape, sampler):
    t = {'tanh': _tanh_target, 'tc': _tc_target,
         'multiclass': lambda: _tanh_target('multi_class_linear_output', n=80, n_out=3, tau_out=1.0)}[shape]()
    sim = sbc.simulate(t, 9, chains_per_sim=2, seed=1)
    kw = dict(num_samples=14, num_steps_per_sample=3, step_size=1e-4 if shape == 'tc' else 0.02, burn=4, seed=17,
              sampler=hb.Sampler.HMC_NUTS if sampler == 'NUTS' else hb.Sampler.HMC, thin=2)
    sims = [2, 3, 4, 5]
    res = sbc.fit(sim, t, sims=sims, **kw)
    K, R = 4, 2
    off = sbc.chain_offset(2, K, R)
    assert off == 4 * 2                                          # K ceil(a (R + 1) / K) = 4 ceil(6 / 4)
    for k, r in ((0, 0), (1, 1), (3, 0), (2, 1)):
        c = r * K + k
        _assert_row(res, c, _plain(sim, t, sims[k], r, off + c, kw))
    assert 0.0 < float(res.accepted.float().mean())


def test_run_with_a_smaller_last_launch():
    t = _tanh_target()
    R = 2
    kw = dict(num_samples=12, num_steps_per_sample=3, step_size=0.02, burn=3, sampler=hb.Sampler.HMC_NUTS)
    out = sbc.run(t, 5, chains_per_sim=R, seed=2, sims_per_launch=2, bins=3, **kw)
    kw['seed'] = 2                                                # run's seed keys the simulation and the fits
    assert sbc.batches(5, 2) == [(0, 3), (3, 2)] and out.num_launches == 2
    sim = out.simulation
    for a, K in sbc.batches(5, 2):
        off = sbc.chain_offset(a, K, R)
        for k in range(K):
            for r in range(R):
                ref = _plain(sim, t, a + k, r, off + r * K + k, kw)
                assert torch.equal(out.step_size[a + k, r], ref.step_size[0])
                assert float(out.accept_rate[a + k, r]) == float(ref.accept_rate[0])
                if r == 0:
                    got = ref.samples[0, 1:]
                    draws = [got] + [_plain(sim, t, a + k, rr, off + rr * K + k, kw).samples[0, 1:]
                                     for rr in range(1, R)]
                    cnt = (torch.cat(draws) < sim.theta[a + k]).sum(0).to(torch.int32)
                    assert torch.equal(out.ranks[a + k, :t.dim], cnt)
    assert out.num_draws == R * 8 and out.ranks.shape == (5, t.dim + 1)
    assert int(out.hist.sum()) == 5 * (t.dim + 1)


# ------------------------------------------------------------------------------------------------------------------
# 3. ranks
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('shape', ['tanh', 'multiclass'])
def test_ranks_equal_counts_on_the_block(shape):
    t = _tanh_target() if shape == 'tanh' else _tanh_target('multi_class_linear_output', n=80, n_out=3, tau_out=1.0)
    sim = sbc.simulate(t, 6, chains_per_sim=3, seed=8)
    res = sbc.fit(sim, t, num_samples=30, num_steps_per_sample=4, step_size=0.03, burn=10, seed=2, thin=3,
                  sampler=hb.Sampler.HMC_NUTS)
    rk = sbc.ranks(res, sim, t)
    torch.cuda.synchronize()
    K, R, D = 6, 3, t.dim
    x = res.samples[:, 1:]                                        # (R K, keep - 1, D)
    for k in range(K):
        draws = x[k::K]                                           # (R, keep - 1, D)
        cnt = (draws.reshape(-1, D) < sim.theta[k]).sum(0)
        assert torch.equal(rk[k, :D].long(), cnt)
        tm = copy.copy(t)
        tm.y = sim.y[k]
        ll = LOO.pointwise_log_lik(draws.contiguous(), tm).double().sum(2)
        # theta~ as a chain of 4 identical draws (the likelihood pass reads at least 4 per chain)
        lt = LOO.pointwise_log_lik(sim.theta[k][None].repeat(4, 1), tm)[0, 0].double().sum()
        assert int(rk[k, D]) == int((ll < lt).sum())
    assert rk.dtype == torch.int32 and int(rk.max()) <= R * (x.shape[1])


# ------------------------------------------------------------------------------------------------------------------
# 4. calibration and detection
# ------------------------------------------------------------------------------------------------------------------
CONJ = dict(num_samples=500, burn=200, thin=10, num_steps_per_sample=10, step_size=0.05, sampler=hb.Sampler.HMC_NUTS)


def test_conjugate_regression_is_calibrated():
    t, _, _, _ = _conjugate(N=40, d=3, tau_out=4.0)
    out = sbc.run(t, 200, chains_per_sim=4, seed=1, **CONJ)
    assert out.ranks.shape == (200, 5) and out.num_draws == 4 * 29 and out.bins == 20 and out.num_launches == 4
    assert float(out.accept_rate.mean()) > 0.6
    assert bool((out.p_value >= 1e-3).all()), out.p_value


def test_multiclass_logistic_regression_is_calibrated():
    g = torch.Generator().manual_seed(4)
    x = torch.randn(60, 2, generator=g)
    t = T.MLPTarget.from_model(nn.Linear(2, 3), x, torch.zeros(60), None, 1.0, model_loss='multi_class_linear_output')
    out = sbc.run(t, 128, chains_per_sim=4, seed=2, **dict(CONJ, step_size=0.1))
    assert out.ranks.shape == (128, 10) and out.num_launches == 2
    assert bool((out.p_value >= 1e-3).all()), out.p_value


def test_a_stalled_fit_fails_the_log_likelihood_column():
    """Chains that never leave their independent prior starts look like prior draws to every parameter column: each chain
    contributes all or none of its draws to a rank, so with B = R + 1 bins the parameter histograms are flat.  The
    log-likelihood of the simulated data is far higher at theta~ than at any prior draw: every rank is L."""
    t, _, _, _ = _conjugate(N=40, d=3, tau_out=4.0)
    R = 4
    out = sbc.run(t, 200, chains_per_sim=R, seed=1, bins=R + 1, num_samples=40, burn=0, num_steps_per_sample=1,
                  step_size=1e-4, sampler=hb.Sampler.HMC)
    assert float(out.p_value[-1]) < 1e-10
    assert int(out.hist[-1, -1]) == 200
    assert bool((out.p_value[:-1] >= 1e-3).all()), out.p_value
