"""GPU: posterior predictive checks and LOO-PIT of Bayesian NNs (hamiltorch_b200.ppc, csrc/hmcx_ppc.cu, the LOO-PIT pass
of csrc/hmcx_loo.cu) against tests/ppc_oracle.py.

1. replicate: regression y_rep = f + z / sqrt(tau_g) within the Box-Muller .approx bound; binary and multi-class labels
   identical away from class boundaries; the same bits on every call, in any draws subset and at any slab size.
2. check: statistics and deviances against the oracle on the returned replicates, p-values exact given t_rep and t_obs,
   the same bytes at 1 draw per slab and all draws in one; SIMT and tensor-core (64-128-1) networks, every loss, a split
   list and a tau_out hyperprior run.
3. loo_pit: the oracle on the same outputs, pareto_k bitwise psis_loo's, the same bytes at every slab size.
4. Behaviour, fixed seeds: a well-specified conjugate fit passes every check; the same data fitted with tau_out 25x too
   large gives a U-shaped LOO-PIT and a small sd p-value."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn

import hamiltorch_b200 as hb
from hamiltorch_b200 import loo as LOO, ppc, predictive as PR, samplers, sbc, targets as T
from tests import ppc_oracle as PO
from tests.test_loo_cpu import _conjugate
from tests.test_loo_gpu import _data, _draws, _net

pytestmark = pytest.mark.gpu

NORMAL_ATOL = 5e-5              # the momentum stream's bound on a Box-Muller normal (tests/test_philox_stream_gpu.py)
LOSSES = ['regression', 'binary_class_linear_output', 'multi_class_linear_output', 'multi_class_log_softmax_output']


def _problem(loss, form='simt', C=2, n=40, N=150, seed=1):
    torch.manual_seed(seed)
    if form == 'tc':
        model, O_ = nn.Sequential(nn.Linear(64, 128), nn.ReLU(), nn.Linear(128, 1)), 1
    else:
        model, O_ = _net(loss, 7, 24)
    x, y = _data(loss, N, model[0].in_features, O_, seed + 1)
    tau = 2.5 if loss == 'regression' else 1.0
    tgt = T.MLPTarget.from_model(model, x, y, None, tau, model_loss=loss)
    return tgt, _draws(model, C, n, 0.3, seed + 2).cuda()


def _outputs(draws, tgt):
    """(S, N, O) fp32 outputs of every pooled draw: the values the PPC pass reads (predictive.pointwise_outputs)."""
    f = PR.pointwise_outputs(draws, tgt)
    return f.reshape(-1, f.shape[2], f.shape[3]).cpu().double().numpy()


def _y_obs(tgt):
    items = tgt if isinstance(tgt, list) else [tgt]
    return torch.cat([t.y.reshape(-1, t.y_cols) for t in items]).double().numpy()


# ------------------------------------------------------------------------------------------------------------------
# 1. replicate
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('loss', LOSSES)
def test_replicate_matches_the_oracle(loss):
    tgt, draws = _problem(loss)
    S = draws.shape[0] * draws.shape[1]
    rep = ppc.replicate(draws, tgt, seed=11).cpu().double().numpy()
    f = _outputs(draws, tgt)
    g = np.arange(S)
    if loss == 'regression':
        want = PO.replicate_regression(11, g, f, np.full(S, tgt.tau_out))
        assert rep.shape == f.shape
        assert np.all(np.abs(rep - want) <= NORMAL_ATOL / np.sqrt(tgt.tau_out) + 1e-5 * (1 + np.abs(want)))
    elif loss == 'binary_class_linear_output':
        want, dist = PO.replicate_binary(11, g, f)
        far = dist > 1e-4
        assert far.mean() > 0.99 and np.array_equal(rep[far], want[far])
    else:
        want, dist = PO.replicate_multiclass(11, g, f)
        far = dist > 1e-4
        assert rep.shape == (S, f.shape[1], 1)
        assert far.mean() > 0.99 and np.array_equal(rep[far], want[far])


@pytest.mark.parametrize('loss', ['regression', 'multi_class_linear_output'])
def test_replicate_is_keyed_by_seed_and_draw_only(loss):
    tgt, draws = _problem(loss, C=3, n=20)
    full = ppc.replicate(draws, tgt, seed=4)
    assert torch.equal(full, ppc.replicate(draws, tgt, seed=4))
    assert not torch.equal(full, ppc.replicate(draws, tgt, seed=5))
    sub = torch.tensor([41, 3, 59, 0, 17])
    try:
        for k in (1, 2, 7):
            ppc._slab_draws_override = k
            assert torch.equal(ppc.replicate(draws, tgt, seed=4), full)
            assert torch.equal(ppc.replicate(draws, tgt, draws=sub, seed=4), full[sub.cuda()])
    finally:
        ppc._slab_draws_override = None


# ------------------------------------------------------------------------------------------------------------------
# 2. check
# ------------------------------------------------------------------------------------------------------------------
def _check_against_oracle(draws, tgt, tau=None, seed=3, **kw):
    items = tgt if isinstance(tgt, list) else [tgt]
    first = items[0]
    S = draws.shape[0] * draws.shape[1]
    r = ppc.check(draws, tgt, seed=seed, **kw)
    rep = ppc.replicate(draws, tgt, seed=seed, **kw).cpu().double().numpy()
    f = _outputs(draws, tgt)
    y = _y_obs(tgt)
    tau = np.full(S, first.tau_out) if tau is None else np.asarray(tau, dtype=np.float64).reshape(-1)
    O_ = first.widths[-1]
    t_rep = r.t_rep.cpu().numpy()
    assert r.names == ppc.stat_names(tgt) and t_rep.shape == (S, len(r.names)) and r.num_nonfinite == 0
    want = np.concatenate([PO.statistics(rep, first.loss_id, O_), PO.deviance(f, rep, first.loss_id, tau)[:, None]], 1)
    assert np.all(np.abs(t_rep - want) <= 1e-9 * (1 + np.abs(want))), np.abs(t_rep - want).max()
    dev_obs = PO.deviance(f, y, first.loss_id, tau)
    assert np.all(np.abs(r.dev_obs.cpu().numpy() - dev_obs) <= 1e-9 * (1 + np.abs(dev_obs)))
    t_obs = r.t_obs.cpu().numpy()
    obs = PO.statistics(y[None], first.loss_id, O_)[0]
    assert np.all(np.abs(t_obs[:-1] - obs) <= 1e-12 * (1 + np.abs(obs)))
    if first.loss_id != 0:          # counts over N, divided as the kernel divides: a tied count compares equal
        assert np.array_equal(t_obs[:-1], obs) and np.array_equal(t_rep[:, :-1], want[:, :-1])
    assert abs(t_obs[-1] - r.dev_obs.mean().item()) <= 1e-12 * abs(t_obs[-1])
    per = np.concatenate([np.broadcast_to(t_obs[:-1], (S, len(obs))), r.dev_obs.cpu().numpy()[:, None]], 1)
    assert np.array_equal(r.p_value.cpu().numpy(), PO.p_values(t_rep, per))
    # the same bytes at 1 draw per slab and with every draw in one slab
    try:
        for k in (1, S):
            ppc._slab_draws_override = k
            o = ppc.check(draws, tgt, seed=seed, **kw)
            assert torch.equal(o.t_rep, r.t_rep) and torch.equal(o.dev_obs, r.dev_obs)
            assert torch.equal(o.p_value, r.p_value) and torch.equal(o.t_obs, r.t_obs)
    finally:
        ppc._slab_draws_override = None
    return r


@pytest.mark.parametrize('loss', LOSSES)
def test_check_matches_the_oracle(loss):
    tgt, draws = _problem(loss, C=2, n=25)
    _check_against_oracle(draws, tgt)


def test_check_on_the_tensor_core_network():
    tgt, draws = _problem('regression', form='tc', C=2, n=10, N=300)
    from hamiltorch_b200 import engine
    assert engine.native_target(tgt, 'cuda').mlp_struct.x_packed, 'the 64-128-1 stack should take the tensor cores'
    _check_against_oracle(draws, tgt)


def test_check_on_a_split_list():
    torch.manual_seed(4)
    model, O_ = _net('regression', 6, 16)
    x, y = _data('regression', 250, 6, O_, 5)
    bounds = [0, 70, 190, 250]
    parts = [T.MLPTarget.from_model(model, x[a:b], y[a:b], None, 3.0, prior_scale=3) for a, b in zip(bounds, bounds[1:])]
    draws = _draws(model, 2, 15, 0.2, 6).cuda()
    r = _check_against_oracle(draws, parts)
    whole = T.MLPTarget.from_model(model, x, y, None, 3.0, prior_scale=3)
    assert torch.equal(ppc.check(draws, whole, seed=3).t_rep, r.t_rep)


def test_check_of_a_tau_out_hyperprior_run():
    g = torch.Generator().manual_seed(8)
    x = torch.randn(60, 3, generator=g)
    y = x @ torch.tensor([[0.8], [-0.5], [0.3]]) + 0.2 + 0.3 * torch.randn(60, 1, generator=g)
    tgt = T.MLPTarget.from_model(nn.Linear(3, 1), x, y, [torch.tensor(1.0)] * 2, 1.0)
    res = samplers.sample_chains(tgt, 0.1 * torch.randn(3, 4, generator=g), num_samples=40, num_steps_per_sample=5,
                                 step_size=0.02, burn=10, tau_out_prior=(2.0, 0.2), seed=5)
    tau = res.tau_out_trace
    assert float(tau.std()) > 0
    _check_against_oracle(res.samples, tgt, tau=tau.cpu(), tau_out=tau)
    # an HMCResult brings its own trace
    a, b = ppc.check(res, tgt, seed=3), ppc.check(res.samples, tgt, seed=3, tau_out=tau)
    assert torch.equal(a.t_rep, b.t_rep) and torch.equal(a.dev_obs, b.dev_obs)
    lp = ppc.loo_pit(res, tgt)
    assert torch.equal(lp.pareto_k, LOO.psis_loo(res, tgt).pareto_k)


def test_check_flags_a_non_finite_draw():
    tgt, draws = _problem('regression', C=2, n=20)
    draws = draws.clone()
    draws[1, 4, 0] = float('nan')
    r = ppc.check(draws, tgt)
    bad = 20 + 4
    assert r.num_nonfinite == 1 and torch.isnan(r.t_rep[bad]).all() and torch.isnan(r.dev_obs[bad])
    ok = torch.ones(40, dtype=torch.bool)
    ok[bad] = False
    assert torch.isfinite(r.p_value).all() and torch.isfinite(r.t_rep[ok.cuda()]).all()


# ------------------------------------------------------------------------------------------------------------------
# 3. LOO-PIT
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('form', ['simt', 'tc'])
def test_loo_pit_matches_the_oracle(form):
    tgt, draws = _problem('regression', form=form, C=3, n=200, N=150 if form == 'simt' else 300, seed=7)
    draws = draws.clone()
    draws[1:] = draws[1:] * 0.6 + draws[:1].mean(1, keepdim=True) * 0.4      # chains that disagree: a heavier tail
    lp = ppc.loo_pit(draws, tgt, r_eff=0.8, bins=10)
    lo = LOO.psis_loo(draws, tgt, r_eff=0.8)
    assert torch.equal(lp.pareto_k, lo.pareto_k) and lp.num_bad_k == lo.num_bad_k
    ll = LOO.pointwise_log_lik(draws, tgt)
    S = ll.shape[0] * ll.shape[1]
    f = _outputs(draws, tgt)
    pit, kh = PO.loo_pit(ll.reshape(S, -1).cpu().numpy(), f, _y_obs(tgt), np.full(S, tgt.tau_out), r_eff=0.8)
    got = lp.pit.cpu().numpy()
    assert np.abs(got - pit).max() < 1e-9, np.abs(got - pit).max()
    assert np.array_equal(lp.pareto_k.cpu().numpy(), kh) or np.allclose(lp.pareto_k.cpu().numpy(), kh, rtol=1e-9)
    hist, chi2, p = PO.uniformity(got, 10)
    assert np.array_equal(lp.hist.cpu().numpy(), hist) and abs(lp.chi2 - chi2) < 1e-9 * chi2 and abs(lp.p_value - p) < 1e-9
    # the same bytes at any slab size
    try:
        for k in (1, 7, 128):
            LOO._slab_points_override = k
            o = ppc.loo_pit(draws, tgt, r_eff=0.8, bins=10)
            assert torch.equal(o.pit, lp.pit) and torch.equal(o.pareto_k, lp.pareto_k)
    finally:
        LOO._slab_points_override = None


def test_loo_pit_with_per_draw_noise_precision():
    tgt, draws = _problem('regression', C=2, n=150, N=80, seed=9)
    tau = (1.0 + torch.rand(2, 150, generator=torch.Generator().manual_seed(1)) * 3).cuda()
    lp = ppc.loo_pit(draws, tgt, tau_out=tau)
    assert torch.equal(lp.pareto_k, LOO.psis_loo(draws, tgt, tau_out=tau).pareto_k)
    ll = LOO.pointwise_log_lik(draws, tgt, tau_out=tau).reshape(300, -1).cpu().numpy()
    pit, _ = PO.loo_pit(ll, _outputs(draws, tgt), _y_obs(tgt), tau.reshape(-1).cpu().numpy())
    assert np.abs(lp.pit.cpu().numpy() - pit).max() < 1e-9


# ------------------------------------------------------------------------------------------------------------------
# 4. behaviour
# ------------------------------------------------------------------------------------------------------------------
FIT = dict(num_samples=700, burn=200, num_steps_per_sample=10, step_size=0.05, sampler=hb.Sampler.HMC_NUTS, seed=3)


def _prior_predictive_data():
    """The conjugate nn.Linear(3, 1) regression (tau_out 4) at N = 200, with y from its own prior predictive."""
    t, _, _, _ = _conjugate(N=200, d=3, tau_out=4.0)
    sim = sbc.simulate(t, 2, chains_per_sim=1, seed=21)
    t = copy.copy(t)
    t.y = sim.y[0].clone()
    return t


def _fit(t):
    """4 chains started near the exact posterior mean of the conjugate model; the posterior draws without slot 0 (the
    start, not a draw) as a (4, n, 4) block."""
    tau_w, tau_b, tau = 2.0, 0.5, float(t.tau_out)
    X1 = torch.cat([t.x.double(), torch.ones(t.x.shape[0], 1, dtype=torch.float64)], 1)
    Pm = torch.diag(torch.tensor([tau_w] * 3 + [tau_b], dtype=torch.float64)) + tau * X1.t() @ X1
    mu = torch.linalg.solve(Pm, tau * X1.t() @ t.y.double().cpu().reshape(-1))
    q0 = (mu + 0.01 * torch.randn(4, 4, generator=torch.Generator().manual_seed(0), dtype=torch.float64)).float()
    res = samplers.sample_chains(t, q0, **FIT)
    return res.samples[:, 1:]


def test_well_specified_fit_passes_every_check():
    t = _prior_predictive_data()
    res = _fit(t)
    r = ppc.check(res, t, seed=1)
    lp = ppc.loo_pit(res, t)
    print('well specified: rank R-hat max %.4f,' % float(hb.diagnostics.rank_summary(res).rhat.max()),
          'pareto_k max %.3f;' % float(lp.pareto_k.max()), end=' ')
    print('well specified: p-values', dict(zip(r.names, [round(v, 4) for v in r.p_value.tolist()])),
          'LOO-PIT chi2 p %.4g' % lp.p_value)
    assert r.num_nonfinite == 0 and lp.num_nonfinite == 0
    assert bool(((r.p_value >= 0.01) & (r.p_value <= 0.99)).all()), r
    assert lp.p_value > 1e-3, lp


def test_overconfident_noise_model_is_flagged():
    t = _prior_predictive_data()
    bad = T.MLPTarget.from_model(nn.Linear(3, 1), t.x, t.y, [torch.tensor(2.0), torch.tensor(0.5)], 100.0)
    res = _fit(bad)
    r = ppc.check(res, bad, seed=1)
    lp = ppc.loo_pit(res, bad)
    print('tau_out x25: rank R-hat max %.4f,' % float(hb.diagnostics.rank_summary(res).rhat.max()), end=' ')
    print('tau_out x25: p-values', dict(zip(r.names, [round(v, 4) for v in r.p_value.tolist()])),
          'LOO-PIT chi2 p %.4g' % lp.p_value, 'hist', lp.hist.tolist())
    assert lp.p_value < 1e-6, lp
    h = lp.hist.double()
    assert h[0] + h[-1] > 4 * h[1:-1].mean()                                 # U-shaped
    assert r.p_value[r.names.index('sd[0]')] < 0.01, r
