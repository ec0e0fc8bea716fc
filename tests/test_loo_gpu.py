"""GPU: the pointwise log-likelihood kernel (hmcx_mlp_pointwise_ll) and the PSIS / WAIC pass (hmcx_loo_pass) against the
fp64 definition of tests/loo_oracle.py."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import hamiltorch_b200 as hb
from hamiltorch_b200 import loo as LOO
from hamiltorch_b200 import targets as T
from hamiltorch_b200 import util
from tests import loo_oracle as O
from tests.test_loo_cpu import _conjugate, _posterior_draws

pytestmark = pytest.mark.gpu

LOSSES = ['regression', 'binary_class_linear_output', 'multi_class_linear_output', 'multi_class_log_softmax_output']


def _net(loss, n0, hidden, act=nn.Tanh):
    O_ = {'regression': 2, 'binary_class_linear_output': 3}.get(loss, 4)
    layers = [nn.Linear(n0, hidden), act(), nn.Linear(hidden, O_)]
    if loss == 'multi_class_log_softmax_output':
        layers.append(nn.LogSoftmax(dim=1))
    return nn.Sequential(*layers), O_


def _data(loss, N, n0, O_, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, n0, generator=g)
    if loss == 'regression':
        y = torch.randn(N, O_, generator=g)
    elif loss == 'binary_class_linear_output':
        y = (torch.rand(N, O_, generator=g) < 0.5).float()
    else:
        y = torch.randint(0, O_, (N,), generator=g).float()
    return x, y


def _draws(model, C, n, scale, seed):
    th = util.flatten(model).detach()
    g = torch.Generator().manual_seed(seed)
    return (th + scale * torch.randn(C, n, th.numel(), generator=g)).float()


def _check_ll(got, draws, target):
    want = O.pointwise_log_lik(draws.reshape(-1, draws.shape[-1]), target).reshape(got.shape)
    g = got.double().cpu().numpy()
    assert np.all(np.abs(g - want) <= 1e-5 * (1 + np.abs(want))), np.abs(g - want).max()


@pytest.mark.parametrize('loss', LOSSES)
@pytest.mark.parametrize('form', ['simt', 'tc', 'tc_off'])
def test_pointwise_log_lik_matches_the_oracle(loss, form):
    torch.manual_seed(1)
    if form == 'simt':
        model, O_ = _net(loss, 7, 24)
        N = 203
    else:
        model, O_ = _net(loss, 64, 128, nn.ReLU)
        N = 300
    x, y = _data(loss, N, model[0].in_features, O_, 2)
    tau = 2.5 if loss == 'regression' else 1.7
    tgt = T.MLPTarget.from_model(model, x, y, None, tau, model_loss=loss)
    if form == 'tc_off':
        tgt.tensor_cores = 1
    if form == 'tc':
        from hamiltorch_b200 import engine
        assert engine.native_target(tgt, 'cuda').mlp_struct.x_packed, 'the 64-128-O stack should take the tensor cores'
    draws = _draws(model, 3, 5, 0.05, 3)
    ll = LOO.pointwise_log_lik(draws.cuda(), tgt)
    torch.cuda.synchronize()
    assert ll.shape == (3, 5, N) and ll.dtype == torch.float32
    _check_ll(ll, draws, tgt)


@pytest.mark.parametrize('tc', [True, False])
def test_pointwise_log_lik_of_a_split_list(tc):
    torch.manual_seed(4)
    model, O_ = _net('regression', 64 if tc else 6, 128 if tc else 16)
    x, y = _data('regression', 250, model[0].in_features, O_, 5)
    bounds = [0, 70, 190, 250]
    parts = [T.MLPTarget.from_model(model, x[a:b], y[a:b], None, 3.0, prior_scale=3) for a, b in zip(bounds, bounds[1:])]
    draws = _draws(model, 2, 4, 0.05, 6)
    ll = LOO.pointwise_log_lik(draws.cuda(), parts)
    torch.cuda.synchronize()
    _check_ll(ll, draws, parts)


def _heavy_block(C, n, Np, seed):
    """ll = -k_i E - a_i with E ~ Exp(1): the importance ratios exp(-ll) are Pareto-tailed with shape k_i in (0.1, 1.2)."""
    rng = np.random.default_rng(seed)
    k = rng.uniform(0.1, 1.2, Np)
    ll = -rng.standard_exponential(size=(C, n, Np)) * k - rng.normal(size=Np)
    return torch.from_numpy(ll.astype(np.float32))


def _check_loo(blk, r_eff=1.0, **kw):
    lo = LOO.psis_loo(blk.cuda(), r_eff=r_eff)
    wa = LOO.waic(blk.cuda())
    ref = O.psis_loo(blk.numpy(), r_eff)
    wref = O.waic(blk.numpy())
    tol = lambda a, b: np.all((np.abs(a - b) <= 1e-9 * (1 + np.abs(b))) | (np.isnan(a) & np.isnan(b))
                              | ((a == b) & np.isinf(b)))
    assert np.array_equal(lo.tail_size.cpu().numpy(), ref['tail'])
    for got, key in ((lo.pointwise, 'elpd_loo'), (lo.p_loo_i, 'p_loo'), (lo.pareto_k, 'pareto_k'), (lo.lppd, 'lppd')):
        assert tol(got.cpu().numpy(), ref[key]), (key, np.nanmax(np.abs(got.cpu().numpy() - ref[key])))
    for got, key in ((wa.p_waic, 'p_waic'), (wa.pointwise, 'elpd_waic'), (wa.lppd, 'lppd')):
        assert tol(got.cpu().numpy(), wref[key]), key
    if ref['num_nonfinite'] == 0:
        for a, b in ((lo.elpd_loo, ref['elpd_total']), (lo.se, ref['se']), (lo.p_loo, ref['p_loo_total']),
                     (lo.looic, ref['looic']), (wa.elpd_waic, wref['elpd_total']), (wa.se, wref['se']),
                     (wa.p_waic_total, wref['p_waic_total'])):
            assert abs(a - b) <= 1e-9 * (1 + abs(b)), (a, b)
    assert lo.num_bad_k == ref['num_bad_k'] and lo.num_nonfinite == ref['num_nonfinite']
    assert lo.k_threshold == ref['k_threshold'] and wa.num_p_waic_warn == wref['num_p_waic_warn']
    return lo, ref


@pytest.mark.parametrize('shape,r_eff', [((4, 500, 37), 1.0), ((3, 333, 20), 0.7), ((1, 1200, 9), 1.0),
                                         ((8, 1300, 5), 2.0)])
def test_psis_pass_matches_the_oracle_on_heavy_tailed_blocks(shape, r_eff):
    lo, ref = _check_loo(_heavy_block(*shape, seed=sum(shape)), r_eff)
    assert np.isfinite(ref['pareto_k']).all() and (ref['tail'] > 4).all()


def test_psis_pass_flags_a_non_finite_draw():
    blk = _heavy_block(2, 400, 6, 9)
    blk[1, 7, 2] = float('-inf')
    blk[0, 0, 4] = float('nan')
    lo, ref = _check_loo(blk)
    assert lo.num_nonfinite == 2 and np.isnan(lo.pointwise.cpu().numpy()[[2, 4]]).all()


def test_psis_pass_on_a_low_acceptance_bnn_run():
    torch.manual_seed(7)
    model, O_ = _net('regression', 5, 12)
    x, y = _data('regression', 60, 5, O_, 8)
    tgt = T.MLPTarget.from_model(model, x, y, None, 20.0)
    init = util.flatten(model).detach()[None].repeat(4, 1)
    res = hb.sample_chains(tgt, init, num_samples=300, num_steps_per_sample=3, step_size=0.05,
                           integrator=hb.Integrator.IMPLICIT, rng='philox', seed=3)
    torch.cuda.synchronize()
    assert float(res.accept_rate.mean()) < 0.8
    ll = LOO.pointwise_log_lik(res, tgt)
    blk = ll.cpu()
    assert len(np.unique(blk[:, :, 0].numpy())) < blk.shape[0] * blk.shape[1]        # repeated draws
    _check_loo(blk)
    # samples + target, slab by slab, give the bits of the block
    a, b = LOO.psis_loo(res, tgt), LOO.psis_loo(ll)
    assert torch.equal(a.pointwise, b.pointwise) and torch.equal(a.pareto_k, b.pareto_k)


def test_slabs_and_repeated_calls_give_the_same_bits():
    blk = _heavy_block(4, 600, 23, 11).cuda()
    torch.manual_seed(12)
    model, O_ = _net('binary_class_linear_output', 64, 128)
    x, y = _data('binary_class_linear_output', 260, 64, O_, 13)
    tgt = T.MLPTarget.from_model(model, x, y, None, 1.0, model_loss='binary_class_linear_output')
    draws = _draws(model, 2, 300, 0.02, 14).cuda()
    base = [LOO.psis_loo(blk), LOO.psis_loo(draws, tgt), LOO.waic(draws, tgt)]
    again = [LOO.psis_loo(blk), LOO.psis_loo(draws, tgt), LOO.waic(draws, tgt)]
    try:
        forced = {}
        for k in (1, 7):
            LOO._slab_points_override = k
            forced[k] = [LOO.psis_loo(blk), LOO.psis_loo(draws, tgt), LOO.waic(draws, tgt)]
    finally:
        LOO._slab_points_override = None
    for runs in [again] + list(forced.values()):
        for r0, r1 in zip(base, runs):
            for name in ('pointwise', 'lppd') + (('pareto_k', 'p_loo_i', 'tail_size') if r0.kind == 'loo' else ('p_waic',)):
                assert torch.equal(getattr(r0, name), getattr(r1, name)), name


def test_conjugate_regression_end_to_end():
    tgt, mu, L, exact = _conjugate()
    th = _posterior_draws(mu, L, 4000).float().reshape(4, 1000, -1).cuda()
    lo = LOO.psis_loo(th, tgt)
    got = lo.pointwise.cpu().numpy()
    assert np.abs(got - exact).max() < 0.02, np.abs(got - exact).max()
    assert float(lo.pareto_k.max()) < 0.5 and lo.num_bad_k == 0
    wa = LOO.waic(th, tgt)
    other = LOO.psis_loo(th, _conjugate(tau_out=1.0)[0])          # the same draws scored by a mis-specified noise level
    c = LOO.compare(lo, other)
    assert c.elpd_diff[c.order[0]] == 0.0 and c.se_diff[c.order[0]] == 0.0 and c.elpd_diff[c.order[1]] < 0
    assert abs(wa.elpd_waic - lo.elpd_loo) < 1.0


def test_pinned_host_samples_are_refused():
    tgt, mu, L, _ = _conjugate()
    th = _posterior_draws(mu, L, 40).float().reshape(1, 40, -1).pin_memory()
    with pytest.raises(RuntimeError, match='pinned host memory'):
        LOO.psis_loo(th, tgt)
    with pytest.raises(RuntimeError, match='pinned host memory'):
        LOO.pointwise_log_lik(th, tgt)
