"""CPU: the power-scaling oracle (tests/psens_oracle.py) -- the CJS properties, its components against the target's
own closure, the Gaussian case whose power-scaled posteriors are known in closed form -- and every refusal of
hamiltorch_b200.sensitivity raised before any CUDA call."""
import math

import numpy as np
import pytest
import torch
import torch.nn as nn
from scipy import stats

from hamiltorch_b200 import _native as NA
from hamiltorch_b200 import sensitivity as SE
from hamiltorch_b200 import targets as T
from tests import loo_oracle as LO
from tests import psens_oracle as PS


def _rng(seed):
    return np.random.default_rng(seed)


# ------------------------------------------------------------------------------------------------------------------
# 1. CJS
# ------------------------------------------------------------------------------------------------------------------
def _random_weights(S, seed):
    w = _rng(seed).gamma(0.5, size=S)
    return w / w.sum()


def test_cjs_is_zero_for_equal_weights():
    x = _rng(0).normal(size=500)
    assert PS.cjs(x, np.full(500, 1.0 / 500)) == pytest.approx(0.0, abs=1e-7)


@pytest.mark.parametrize('seed', range(5))
def test_cjs_lies_in_the_unit_interval(seed):
    r = _rng(seed)
    x = r.standard_t(3, size=400)
    q = _random_weights(400, seed + 10)
    d = PS.cjs(x, q)
    assert 0.0 < d <= 1.0
    # all the weight on one draw: the distance stays below 1
    q1 = np.zeros(400)
    q1[int(np.argmax(x))] = 1.0
    assert 0.0 < PS.cjs(x, q1) <= 1.0


@pytest.mark.parametrize('a, b', [(3.0, 1.5), (-2.0, 7.0), (0.01, -4.0), (-1.0, 0.0)])
def test_cjs_is_invariant_under_affine_maps(a, b):
    x = _rng(2).normal(size=300)
    q = _random_weights(300, 3)
    assert PS.cjs(a * x + b, q) == pytest.approx(PS.cjs(x, q), rel=1e-9)


def test_cjs_of_a_constant_column_is_zero_and_ties_need_no_rule():
    q = _random_weights(200, 4)
    assert PS.cjs(np.full(200, 2.5), q) == 0.0
    x = _rng(5).integers(0, 5, size=200).astype(np.float64)          # heavy ties
    perm = _rng(6).permutation(200)
    assert PS.cjs(x[perm], q[perm]) == pytest.approx(PS.cjs(x, q), rel=1e-12)


def test_oracle_weights_are_psis_of_the_rounded_negated_log_ratios():
    r = _rng(7)
    lp, ll = r.normal(size=3000) * 30, r.normal(size=3000) * 200 - 500
    w, khat = PS.weights(lp, ll, 0.99, 1.01)
    assert w.shape == (4, 3000) and np.allclose(w.sum(1), 1.0)
    for k, (comp, a) in enumerate(((lp, 0.99), (lp, 1.01), (ll, 0.99), (ll, 1.01))):
        nr = (-((a - 1.0) * comp)).astype(np.float32).astype(np.float64)
        assert khat[k] == pytest.approx(LO.psis_point(nr)['pareto_k'], rel=1e-12)
    # prior scaled up (alpha > 1) moves weight towards draws with a larger prior term
    assert (w[1] * lp).sum() > lp.mean() > (w[0] * lp).sum()


# ------------------------------------------------------------------------------------------------------------------
# 2. Components against the closure the sampler differentiates
# ------------------------------------------------------------------------------------------------------------------
def test_normal_log_prior_matches_scipy():
    r = _rng(8)
    th = r.normal(size=(5, 11))
    sizes, taus = [6, 2, 3], [2.0, 0.0, 0.5]
    want = stats.norm.logpdf(th[:, :6], scale=2.0 ** -0.5).sum(1) + stats.norm.logpdf(th[:, 8:], scale=0.5 ** -0.5).sum(1)
    assert np.allclose(PS.normal_log_prior(th, sizes, taus), want, rtol=1e-12)


@pytest.mark.parametrize('loss', ['binary_class_linear_output', 'multi_class_linear_output',
                                  'multi_class_log_softmax_output'])
def test_classification_likelihood_is_the_closure_minus_the_prior(loss):
    O_ = 3
    layers = [nn.Linear(4, 5), nn.Tanh(), nn.Linear(5, O_)] + ([nn.LogSoftmax(dim=1)] if 'softmax' in loss else [])
    torch.manual_seed(0)
    model = nn.Sequential(*layers)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(50, 4, generator=g)
    y = (torch.rand(50, O_, generator=g) < 0.5).float() if 'binary' in loss else \
        torch.randint(0, O_, (50,), generator=g).float()
    bounds = [0, 20, 50]
    parts = [T.MLPTarget.from_model(model, x[a:b], y[a:b], None, 2.5, prior_scale=2, model_loss=loss)
             for a, b in zip(bounds, bounds[1:])]
    th = torch.randn(3, parts[0].dim, generator=g)
    ll = LO.pointwise_log_lik(th, parts)
    got = PS.log_lik_total(ll, parts[0].loss_id, 2.5, [20, 30])
    want = [sum(float(t(th[s]) - t.log_prior(th[s]) / t.prior_scale) for t in parts) for s in range(3)]
    assert np.allclose(got, want, rtol=1e-4, atol=1e-4)


# ------------------------------------------------------------------------------------------------------------------
# 3. A Gaussian posterior with exact draws: the power-scaled posteriors are Gaussian too
# ------------------------------------------------------------------------------------------------------------------
def test_gaussian_power_scaled_moments_match_the_closed_form():
    tau0, tauL, mL = 1.0, 4.0, 1.0
    prec = tau0 + tauL
    S = 40000
    th = _rng(9).normal(tauL * mL / prec, prec ** -0.5, size=S)
    lp = -0.5 * tau0 * th ** 2
    ll = -0.5 * tauL * (th - mL) ** 2
    for a in (0.8, 1.25):
        r = PS.power_scale(th[:, None], lp, ll, lo=0.8, hi=1.25)
        k = 1 if a > 1 else 0
        for comp in ('prior', 'lik'):
            p = a * tau0 + tauL if comp == 'prior' else tau0 + a * tauL
            m, s = tauL * mL * (a if comp == 'lik' else 1.0) / p, p ** -0.5
            row = 1 + k + (2 if comp == 'lik' else 0)
            mcse = s / math.sqrt(S / 2)
            assert abs(r['mean'][row, 0] - m) < 5 * mcse, (comp, a, r['mean'][row, 0], m)
            assert abs(r['sd'][row, 0] - s) < 5 * mcse, (comp, a, r['sd'][row, 0], s)
    # the likelihood is 4x as informative as the prior here
    r = PS.power_scale(th[:, None], lp, ll)
    assert r['likelihood'][0] > r['prior'][0] > 0


# ------------------------------------------------------------------------------------------------------------------
# 4. Refusals before any CUDA call
# ------------------------------------------------------------------------------------------------------------------
def _blk(C=2, n=10, D=3):
    return torch.zeros(C, n, D)


@pytest.mark.parametrize('lo, hi', [(0.0, 1.01), (-0.5, 1.01), (1.0, 1.01), (1.2, 1.5), (0.99, 1.0), (0.99, 0.5),
                                    (0.99, float('inf')), (float('nan'), 1.01)])
def test_bad_alphas_are_refused(lo, hi):
    with pytest.raises(ValueError, match='alpha'):
        SE.power_scale(_blk(), log_prior=torch.zeros(2, 10), log_lik=torch.zeros(2, 10), lower_alpha=lo,
                       upper_alpha=hi)


def test_a_kfold_result_is_refused():
    class Fold:
        folds = torch.zeros(4)
    with pytest.raises(TypeError, match='K-fold'):
        SE.power_scale(Fold(), log_prior=torch.zeros(1), log_lik=torch.zeros(1))
    with pytest.raises(TypeError, match='K-fold'):
        SE.log_components(Fold(), None)


def test_a_target_without_data_is_refused():
    t = T.MLPTarget([2, 3, 1], [T.ACT_TANH, T.ACT_NONE], None, None, [1.0] * 4)
    with pytest.raises(RuntimeError, match='no data'):
        SE.power_scale(_blk(D=t.dim), t)
    with pytest.raises(RuntimeError, match='no data'):
        SE.log_components(_blk(D=t.dim), t)


@pytest.mark.parametrize('which', ['log_prior', 'log_lik'])
def test_components_of_the_wrong_shape_are_refused(which):
    kw = dict(log_prior=torch.zeros(2, 10), log_lik=torch.zeros(2, 10))
    kw[which] = torch.zeros(2, 9)
    with pytest.raises(RuntimeError, match=which):
        SE.power_scale(_blk(), **kw)


def test_quantities_of_the_wrong_shape_are_refused():
    kw = dict(log_prior=torch.zeros(2, 10), log_lik=torch.zeros(2, 10))
    with pytest.raises(RuntimeError, match='quantities'):
        SE.power_scale(_blk(), quantities=torch.zeros(2, 11, 4), **kw)
    with pytest.raises(TypeError, match='quantities'):
        SE.power_scale(_blk(), quantities=np.zeros((2, 10, 4)), **kw)


def test_missing_or_doubled_components_are_refused():
    with pytest.raises(ValueError, match='both'):
        SE.power_scale(_blk(), log_prior=torch.zeros(2, 10))
    t = T.MLPTarget([2, 1], [T.ACT_NONE], torch.zeros(5, 2), torch.zeros(5, 1), [1.0] * 2)
    with pytest.raises(ValueError, match='not both'):
        SE.power_scale(_blk(D=t.dim), t, log_prior=torch.zeros(2, 10), log_lik=torch.zeros(2, 10))


def test_too_few_and_too_many_draws_are_refused():
    with pytest.raises(RuntimeError, match='at least 2'):
        SE.power_scale(torch.zeros(1, 1, 3), log_prior=torch.zeros(1, 1), log_lik=torch.zeros(1, 1))
    big = torch.zeros(1, 1, 1).expand(65536, 32768, 1)
    assert 65536 * 32768 > NA.RANK_MAX_DRAWS
    with pytest.raises(RuntimeError, match='exceed'):
        SE.power_scale(big, log_prior=torch.zeros(1, 1).expand(65536, 32768),
                       log_lik=torch.zeros(1, 1).expand(65536, 32768))


def test_cpu_samples_are_refused_without_a_fallback():
    with pytest.raises(RuntimeError, match='CPU fallback|cpu tensor'):
        SE.power_scale(_blk(), log_prior=torch.zeros(2, 10), log_lik=torch.zeros(2, 10))


def test_diagnosis_rule():
    d = SE.diagnose(torch.tensor([0.2, 0.2, 0.01, 0.05, float('nan')]), torch.tensor([0.1, 0.01, 0.3, 0.05, 0.2]))
    assert d == [SE.CONFLICT, SE.STRONG_PRIOR, SE.NONE, SE.CONFLICT, SE.NONE]
    assert d == PS.diagnose([0.2, 0.2, 0.01, 0.05, float('nan')], [0.1, 0.01, 0.3, 0.05, 0.2])
