"""GPU: per-chain PSIS-LOO (hmcx_loo_chain_pass) bit for bit against psis_loo of each chain alone and against
tests/stacking_oracle.py; the stacking pass (hmcx_stack_eval / hmcx_stack_em) against the oracle objective and solver;
the chain-weighted held-out predictive (hmcx_pred_pass_weighted) against the weighted oracle; and chain stacking of a run
in which some chains are stuck."""
import numpy as np
import pytest
import torch
import torch.nn as nn

from hamiltorch_b200 import _native as NA
from hamiltorch_b200 import loo as LOO
from hamiltorch_b200 import predictive as P
from hamiltorch_b200 import samplers, util
from hamiltorch_b200 import targets as T
from tests import stacking_oracle as SO
from tests.test_loo_gpu import LOSSES, _data, _draws, _heavy_block, _net
from tests.test_predictive_gpu import _check_oracle, _problem, _same

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.detach().contiguous().view(torch.uint8).cpu()


def _same_bits(a, b, name=''):
    assert a.dtype == b.dtype and a.shape == b.shape, name
    assert torch.equal(_bits(a), _bits(b)), name


def _chain_pinned_to_psis_loo(blk, r_eff=1.0):
    """Every column c of psis_loo_chains is psis_loo of chain c alone, bit for bit."""
    cl = LOO.psis_loo_chains(blk, r_eff=r_eff)
    for c in range(blk.shape[0]):
        one = LOO.psis_loo(blk[c:c + 1], r_eff=r_eff)
        _same_bits(cl.pointwise[c], one.pointwise, 'elpd_loo %d' % c)
        _same_bits(cl.pareto_k[c], one.pareto_k, 'pareto_k %d' % c)
        _same_bits(cl.lppd[c], one.lppd, 'lppd %d' % c)
        assert torch.equal(cl.tail_size[c], one.tail_size)
    return cl


def _close(got, want, rtol=1e-9):
    g = got.detach().cpu().double().numpy() if torch.is_tensor(got) else np.asarray(got, np.float64)
    w = np.asarray(want, np.float64)
    ok = (np.abs(g - w) <= rtol * (1 + np.abs(w))) | (np.isnan(g) & np.isnan(w)) | ((g == w) & np.isinf(w))
    assert ok.all(), np.nanmax(np.abs(g - w))


def _check_chain_oracle(cl, blk, r_eff=1.0):
    ref = SO.psis_loo_chains(blk.detach().cpu().numpy(), r_eff)
    for k in ('elpd_loo', 'lppd', 'pareto_k'):
        _close(getattr(cl, k if k != 'elpd_loo' else 'pointwise'), ref[k])
    assert np.array_equal(cl.tail_size.cpu().numpy(), ref['tail'])
    if np.isfinite(ref['elpd_loo']).all():
        _close(cl.elpd_loo, ref['elpd_total'])
        _close(cl.se, ref['se'])
    assert cl.k_threshold == ref['k_threshold']
    assert np.array_equal(cl.num_bad_k.cpu().numpy(), ref['num_bad_k'])


# ------------------------------------------------------------------------------------------------------------------
# 1. Per-chain PSIS-LOO
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [5, 100, 1000, 8192])
def test_each_chain_is_psis_loo_of_that_chain_alone(n):
    C_, Np = (3, 9) if n < 8192 else (2, 4)
    blk = _heavy_block(C_, n, Np, seed=n).cuda()
    cl = _chain_pinned_to_psis_loo(blk, r_eff=0.8 if n == 1000 else 1.0)
    assert cl.num_chains == C_ and cl.num_draws == n and cl.num_points == Np and cl.num_nonfinite == 0
    if n <= 1000:
        _check_chain_oracle(cl, blk, r_eff=0.8 if n == 1000 else 1.0)


def test_a_non_finite_draw_poisons_its_chain_and_point_only():
    blk = _heavy_block(3, 300, 6, seed=21).cuda()
    blk[1, 7, 2] = float('-inf')
    blk[2, 0, 4] = float('nan')
    cl = _chain_pinned_to_psis_loo(blk)
    assert cl.num_nonfinite == 2
    pw = cl.pointwise.cpu().numpy()
    assert np.isnan(pw[1, 2]) and np.isnan(pw[2, 4]) and np.isfinite(np.delete(pw.ravel(), [1 * 6 + 2, 2 * 6 + 4])).all()
    _check_chain_oracle(cl, blk)


def _samples_problem(loss, form, seed):
    torch.manual_seed(seed)
    if form == 'simt':
        model, O_ = _net(loss, 7, 24)
        N_ = 203
    else:
        model, O_ = _net(loss, 64, 128, nn.ReLU)
        N_ = 300
    x, y = _data(loss, N_, model[0].in_features, O_, seed + 1)
    tau = 2.5 if loss == 'regression' else 1.0
    tgt = T.MLPTarget.from_model(model, x, y, None, tau, model_loss=loss)
    return model, tgt


@pytest.mark.parametrize('form', ['simt', 'tc'])
@pytest.mark.parametrize('loss', LOSSES)
def test_from_samples_matches_the_block_and_the_oracle(loss, form):
    model, tgt = _samples_problem(loss, form, 3)
    draws = _draws(model, 3, 40, 0.03, 4).cuda()
    ll = LOO.pointwise_log_lik(draws, tgt)
    cl = LOO.psis_loo_chains(draws, tgt)
    blk = LOO.psis_loo_chains(ll)
    for k in ('pointwise', 'lppd', 'pareto_k', 'tail_size'):
        _same_bits(getattr(cl, k), getattr(blk, k), k)
    _check_chain_oracle(cl, ll)
    try:
        for k in (1, 7, 128):
            LOO._slab_points_override = k
            for a, b in ((LOO.psis_loo_chains(draws, tgt), cl), (LOO.psis_loo_chains(ll), blk)):
                for f in ('pointwise', 'lppd', 'pareto_k', 'tail_size'):
                    _same_bits(getattr(a, f), getattr(b, f), '%s at slab %d' % (f, k))
    finally:
        LOO._slab_points_override = None


def test_split_list_and_per_draw_tau_out():
    torch.manual_seed(5)
    model, O_ = _net('regression', 6, 16)
    x, y = _data('regression', 150, 6, O_, 6)
    b = [0, 50, 150]
    parts = [T.MLPTarget.from_model(model, x[i:j], y[i:j], None, 20.0, prior_scale=2) for i, j in zip(b, b[1:])]
    draws = _draws(model, 2, 30, 0.03, 7).cuda()
    ll = LOO.pointwise_log_lik(draws, parts)
    cl = LOO.psis_loo_chains(draws, parts)
    _same_bits(cl.pointwise, LOO.psis_loo_chains(ll).pointwise)
    _check_chain_oracle(cl, ll)
    tau = torch.rand(2, 30, generator=torch.Generator().manual_seed(8)).cuda() * 20 + 5
    whole = T.MLPTarget.from_model(model, x, y, None, 20.0)
    llt = LOO.pointwise_log_lik(draws, whole, tau_out=tau)
    ct = LOO.psis_loo_chains(draws, whole, tau_out=tau)
    _same_bits(ct.pointwise, LOO.psis_loo_chains(llt).pointwise)
    _check_chain_oracle(ct, llt)
    assert not torch.equal(ct.pointwise, LOO.psis_loo_chains(draws, whole).pointwise)


# ------------------------------------------------------------------------------------------------------------------
# 2. The stacking pass
# ------------------------------------------------------------------------------------------------------------------
def _stack_eval(E, w):
    lib = NA.load_library()
    K, Np = E.shape
    obj = torch.empty(1, dtype=torch.float64, device='cuda')
    grad = torch.empty(K, dtype=torch.float64, device='cuda')
    pw = torch.empty(Np, dtype=torch.float64, device='cuda')
    nb = lib.hmcx_stack_workspace_bytes(K, Np)
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')
    rc = lib.hmcx_stack_eval(NA.ptr(E), K, Np, NA.ptr(w), NA.ptr(obj), NA.ptr(grad), NA.ptr(pw), NA.ptr(ws), nb,
                             NA.stream_ptr(E.device))
    NA.check(rc, 'hmcx_stack_eval')
    return obj, grad, pw


def test_stack_eval_matches_the_oracle_and_repeats_its_bits():
    rng = np.random.default_rng(0)
    for K, Np in ((1, 7), (5, 1000), (64, 1024), (3, 300)):
        E = rng.normal(size=(K, Np)) * 3 - 2
        w = rng.random(K)
        if K > 2:
            w[1] = 0.0
        w /= w.sum()
        Ed, wd = torch.from_numpy(E).cuda(), torch.from_numpy(w).cuda()
        obj, grad, pw = _stack_eval(Ed, wd)
        f, g, p = SO.objective(E, w)
        _close(obj, [f], 1e-12)
        _close(grad, g, 1e-12)
        _close(pw, p, 1e-12)
        again = _stack_eval(Ed, wd)
        for a, b in zip((obj, grad, pw), again):
            _same_bits(a, b)


def _fake(kind, pw):
    r = LOO.LooResult() if kind == 'loo' else LOO.WaicResult()
    r.pointwise, r.num_points = pw, pw.numel()
    return r


def test_stacking_weights_are_optimal_and_reproducible():
    from tests.test_stacking_cpu import _two_models
    E = _two_models()
    p1, p2 = np.exp(E[0]), np.exp(E[1])
    from scipy.optimize import brentq
    w_star = brentq(lambda w: ((p1 - p2) / (w * p1 + (1 - w) * p2)).sum(), 0.0, 1.0, xtol=1e-15, rtol=1e-15)
    rs = [_fake('loo', torch.from_numpy(e).cuda()) for e in E]
    st = LOO.stacking_weights(*rs, tol=1e-10)
    assert st.converged and st.kkt_gap <= 1e-10
    assert abs(float(st.weights[0]) - w_star) <= 1e-5, (float(st.weights[0]), w_star)
    rng = np.random.default_rng(4)
    Np = 500
    base = rng.normal(size=Np)
    E = np.stack([base + rng.normal(scale=s, size=Np) - s for s in (0.3, 0.6, 1.0, 1.5, 0.6)])
    E[4] = E[1]                                                    # a duplicate: the optimum is not unique
    rs = [_fake('waic', torch.from_numpy(e).cuda()) for e in E]
    st = LOO.stacking_weights(rs)
    _, f_star, _ = SO.solve_em(E)
    assert st.kkt_gap <= 1e-6 and st.converged and st.objective >= f_star - Np * 1e-6
    assert st.objective <= f_star + 1e-9 * abs(f_star)
    _close(st.pointwise, SO.objective(E, st.weights.cpu().numpy())[2], 1e-12)
    assert abs(float(st.weights.sum()) - 1.0) <= 1e-12 and bool((st.weights >= 0).all())
    again = LOO.stacking_weights(rs)
    _same_bits(st.weights, again.weights)
    assert st.iterations == again.iterations and st.objective == again.objective
    # max_iter bounds the work, and the result is still evaluated at the weights it returns
    short = LOO.stacking_weights(rs, max_iter=3)
    assert short.iterations == 3 and not short.converged
    _close(short.pointwise, SO.objective(E, short.weights.cpu().numpy())[2], 1e-12)
    bad = E.copy()
    bad[2, 5] = np.nan
    with pytest.raises(ValueError, match='1 of the 5 x 500'):
        LOO.stacking_weights([_fake('waic', torch.from_numpy(e).cuda()) for e in bad])


def test_chain_stacking_of_a_block():
    blk = _heavy_block(6, 400, 120, seed=31)
    blk[:2] -= 1.5                                                 # two chains predict worse everywhere
    blk = blk.cuda()
    st = LOO.chain_stacking(blk)
    E = st.chain_loo.pointwise.cpu().numpy()
    _, f_star, _ = SO.solve_em(E, gap=1e-12)
    assert st.kkt_gap <= 1e-6 and st.objective >= f_star - E.shape[1] * 1e-6
    assert float(st.weights[:2].sum()) < 1e-3
    _same_bits(st.weights, LOO.chain_stacking(blk).weights)


# ------------------------------------------------------------------------------------------------------------------
# 3. The weighted held-out predictive
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('form', ['simt', 'tc'])
@pytest.mark.parametrize('loss', LOSSES)
def test_weighted_evaluate_matches_the_oracle(loss, form):
    model, tgt, y, tau, draws = _problem(loss, form, False)
    w = torch.tensor([0.5, 0.0, 0.5 + 1e-7], dtype=torch.float64) if form == 'simt' else \
        torch.tensor([0.2, 0.3, 0.5], dtype=torch.float64)
    out = P.pointwise_outputs(draws, tgt)
    r = P.evaluate(draws, tgt, chain_weights=w)
    ref = SO.evaluate_weighted(out.cpu().numpy(), y.numpy(), loss, w.numpy(), tau if loss == 'regression' else None)
    assert r.num_nonfinite == 0
    _check_oracle(r, ref, loss)
    assert torch.equal(r.chain_weights, w / w.sum())
    _same(r, P.evaluate(out, tgt, chain_weights=w))
    _same(r, P.evaluate(draws, tgt, chain_weights=w))
    try:
        for k in (1, 7):
            P._slab_points_override = k
            _same(r, P.evaluate(draws, tgt, chain_weights=w))
    finally:
        P._slab_points_override = None
    pooled = P.evaluate(draws, tgt)
    assert pooled.chain_weights is None and not torch.equal(pooled.nll_i, r.nll_i)


@pytest.mark.parametrize('loss', LOSSES)
def test_one_hot_weights_are_that_chain_alone(loss):
    _, tgt, _, _, draws = _problem(loss, 'simt', False)
    for c in range(draws.shape[0]):
        hot = torch.zeros(draws.shape[0], dtype=torch.float64)
        hot[c] = 1.0
        a = P.evaluate(draws, tgt, chain_weights=hot)
        b = P.evaluate(draws[c:c + 1], tgt)
        for k in ('nll_i', 'nll_curve', 'probs', 'brier_i', 'entropy', 'expected_entropy', 'mean', 'var', 'pit',
                  'rmse_curve', 'accuracy_curve'):
            if hasattr(b, k):
                _close(getattr(a, k), getattr(b, k).cpu().numpy(), 1e-12)


def test_weighted_evaluate_with_per_draw_tau_out():
    torch.manual_seed(3)
    model, O_ = _net('regression', 6, 16)
    x, y = _data('regression', 150, 6, O_, 4)
    tgt = T.MLPTarget.from_model(model, x, y, None, 20.0)
    draws = _draws(model, 3, 20, 0.03, 5).cuda()
    tau = torch.rand(3, 20, generator=torch.Generator().manual_seed(6)).cuda() * 20 + 5
    w = torch.tensor([0.6, 0.1, 0.3], dtype=torch.float64)
    r = P.evaluate(draws, tgt, tau_out=tau, chain_weights=w)
    out = P.pointwise_outputs(draws, tgt)
    ref = SO.evaluate_weighted(out.cpu().numpy(), y.numpy(), 'regression', w.numpy(), tau.cpu().numpy())
    _check_oracle(r, ref, 'regression')


# ------------------------------------------------------------------------------------------------------------------
# 4. End to end: chains stuck at a poor start
# ------------------------------------------------------------------------------------------------------------------
def _sine(N_, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(N_, 1, generator=g) * 6 - 3
    return x, torch.sin(x) + 0.1 * torch.randn(N_, 1, generator=g)


def test_stuck_chains_get_no_weight_and_stacking_improves_the_held_out_nll():
    model = nn.Sequential(nn.Linear(1, 16), nn.Tanh(), nn.Linear(16, 1))
    torch.manual_seed(0)
    x, y = _sine(120, 1)
    xt, yt = _sine(300, 2)
    tau_list = [torch.tensor(1.0)] * 4
    tgt = T.MLPTarget.from_model(model, x, y, tau_list, 100.0)
    test = T.MLPTarget.from_model(model, xt, yt, tau_list, 100.0)
    D = util.flatten(model).numel()
    g = torch.Generator().manual_seed(3)
    good0 = util.flatten(model).detach()[None] + 0.1 * torch.randn(6, D, generator=g)
    good = samplers.sample_chains(tgt, good0, num_samples=500, num_steps_per_sample=20, step_size=0.003, burn=300,
                                  seed=5)
    stuck0 = 0.01 * torch.randn(2, D, generator=g)                 # near the zero network: a flat, poor fit
    stuck = samplers.sample_chains(tgt, stuck0, num_samples=500, num_steps_per_sample=1, step_size=1e-6, burn=300,
                                   seed=6)
    draws = torch.cat([good.samples, stuck.samples]).contiguous()
    st = LOO.chain_stacking(draws, tgt)
    w = st.weights.cpu()
    print('chain weights', w.tolist(), 'elpd per chain', st.chain_loo.elpd_loo.cpu().tolist())
    assert st.converged and st.kkt_gap <= 1e-6
    assert float(w[6:].sum()) < 0.05, w.tolist()
    stacked = P.evaluate(draws, test, chain_weights=w)
    pooled = P.evaluate(draws, test)
    print('held-out nll stacked %.4f pooled %.4f' % (stacked.nll, pooled.nll))
    assert stacked.nll <= pooled.nll, (stacked.nll, pooled.nll)


def test_chain_stacking_of_a_tempered_run():
    model = nn.Sequential(nn.Linear(1, 8), nn.Tanh(), nn.Linear(8, 1))
    x, y = _sine(64, 4)
    tgt = T.MLPTarget.from_model(model, x, y, None, 50.0)
    D = util.flatten(model).numel()
    R, betas = 4, [1.0, 0.5, 0.25]
    q0 = util.flatten(model).detach()[None] + 0.1 * torch.randn(R * len(betas), D,
                                                                generator=torch.Generator().manual_seed(7))
    res = samplers.sample_chains(tgt, q0, num_samples=120, num_steps_per_sample=5, step_size=0.005, burn=20,
                                 betas=betas, swap_every=5, seed=8)
    assert res.samples.shape[0] == R
    st = LOO.chain_stacking(res, tgt)
    assert st.weights.shape == (R,) and st.chain_loo.num_chains == R and st.kkt_gap <= 1e-6
    _same_bits(st.chain_loo.pointwise, LOO.psis_loo_chains(res.samples, tgt).pointwise)
