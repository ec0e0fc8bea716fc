"""CPU: the stacking oracle (tests/stacking_oracle.py) against closed forms and scipy, the chain-weighted predictive
oracle against tests/predictive_oracle.py, and the argument refusals of psis_loo_chains / stacking_weights /
chain_stacking / evaluate(..., chain_weights=) that come before any CUDA work."""
import numpy as np
import pytest
import torch
from scipy.optimize import brentq

from hamiltorch_b200 import _native as NA
from hamiltorch_b200 import loo as LOO
from hamiltorch_b200 import predictive as P
from hamiltorch_b200.engine import HMCResult
from tests import predictive_oracle as PO
from tests import stacking_oracle as SO

LOSSES = ['regression', 'binary_class_linear_output', 'multi_class_linear_output', 'multi_class_log_softmax_output']


def _two_models(N=300, seed=0):
    """Log densities of two predictives, neither dominating: the optimal mixture weight is interior."""
    rng = np.random.default_rng(seed)
    y = rng.standard_t(3, size=N)
    l1 = -0.5 * y ** 2 - 0.5 * np.log(2 * np.pi)                              # N(0, 1)
    l2 = -np.log(np.pi * 2.0 * (1 + (y / 2.0) ** 2))                           # Cauchy(0, 2)
    return np.stack([l1, l2])


def test_two_model_weight_is_the_root_of_the_score_equation():
    E = _two_models()
    p1, p2 = np.exp(E[0]), np.exp(E[1])
    h = lambda w: ((p1 - p2) / (w * p1 + (1 - w) * p2)).sum()
    assert h(0.0) > 0 > h(1.0)
    w_star = brentq(h, 0.0, 1.0, xtol=1e-15, rtol=1e-15)
    w, f, _ = SO.solve_em(E)
    assert abs(w[0] - w_star) <= 1e-9 and abs(w.sum() - 1.0) <= 1e-12
    assert abs(f - SO.objective(E, [w_star, 1 - w_star])[0]) <= 1e-9


def test_em_and_slsqp_reach_the_same_objective():
    rng = np.random.default_rng(3)
    N = 400
    base = rng.normal(size=N)
    E = np.stack([base + rng.normal(scale=s, size=N) - s for s in (0.3, 0.6, 1.0, 1.5)])
    w_em, f_em, _ = SO.solve_em(E)
    w_sq, f_sq = SO.solve_slsqp(E)
    assert abs(f_em - f_sq) <= N * 1e-10, (f_em, f_sq)
    assert f_em >= f_sq - N * 1e-10
    # the objective and gradient of the oracle against finite differences
    f0, g, pw = SO.objective(E, w_em)
    assert abs(pw.sum() - f0) <= 1e-9 * abs(f0)
    d = np.zeros(4)
    d[1] = 1e-6
    assert abs((SO.objective(E, w_em + d)[0] - SO.objective(E, w_em - d)[0]) / 2e-6 - g[1]) <= 1e-4 * abs(g[1])


def test_a_dominated_row_gets_no_weight():
    E = _two_models(seed=1)
    E = np.vstack([E, E[0] - 1.0])                 # everywhere worse than row 0
    w, _, _ = SO.solve_em(E)
    assert w[2] < 1e-6, w


def test_duplicated_rows_share_their_weight():
    E = _two_models(seed=2)
    w, f, _ = SO.solve_em(E)
    w3, f3, _ = SO.solve_em(np.vstack([E, E[1]]))
    assert w3[1] == w3[2]
    assert abs(w3[1] + w3[2] - w[1]) <= 1e-8 and abs(f3 - f) <= E.shape[1] * 1e-12


def _outputs(loss, C=3, n=6, N=11, O=3, seed=0):
    rng = np.random.default_rng(seed)
    f = rng.normal(size=(C, n, N, O)).astype(np.float32) * np.arange(1, C + 1, dtype=np.float32)[:, None, None, None]
    if loss == 'regression':
        y = rng.normal(size=(N, O))
    elif loss == 'binary_class_linear_output':
        y = (rng.random((N, O)) < 0.5).astype(np.float64)
    else:
        y = rng.integers(0, O, N).astype(np.float64)
    tau = rng.uniform(0.5, 2.0, size=(C, n)).astype(np.float32)
    return f, y, tau


def _same(a, b, rtol=1e-12):
    if isinstance(a, dict):
        for k in a:
            assert abs(a[k] - b[k]) <= rtol * (1 + abs(b[k])) or (np.isnan(a[k]) and np.isnan(b[k])), k
        return
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape
    ok = (np.abs(a - b) <= rtol * (1 + np.abs(b))) | (np.isnan(a) & np.isnan(b))
    assert ok.all(), np.nanmax(np.abs(a - b))


KEYS = {'regression': ('mean', 'var', 'epistemic', 'pit', 'lppd', 'nll_i', 'rmse_curve', 'nll_curve', 'coverage'),
        'cls': ('probs', 'pred', 'nll_i', 'brier_i', 'entropy', 'expected_entropy', 'mutual_info', 'accuracy_curve',
                'nll_curve', 'reliability_sums', 'ece')}


@pytest.mark.parametrize('loss', LOSSES)
def test_weighted_oracle_reduces_to_the_unweighted_one(loss):
    f, y, tau = _outputs(loss)
    C = f.shape[0]
    keys = KEYS['regression' if loss == 'regression' else 'cls']
    tau_arg = tau if loss == 'regression' else None
    pooled = PO.evaluate(f, y, loss, tau_arg)
    uni = SO.evaluate_weighted(f, y, loss, np.full(C, 1.0 / C), tau_arg)
    for k in keys:
        _same(uni[k], pooled[k])
    for c in range(C):
        hot = np.zeros(C)
        hot[c] = 1.0
        one = SO.evaluate_weighted(f, y, loss, hot, tau_arg)
        alone = PO.evaluate(f[c:c + 1], y, loss, None if tau_arg is None else tau[c:c + 1])
        for k in keys:
            _same(one[k], alone[k])


def test_a_zero_weight_chain_is_not_read():
    f, y, tau = _outputs('multi_class_linear_output')
    g = f.copy()
    g[1, 2, 4, 0] = np.nan
    w = np.array([0.5, 0.0, 0.5])
    a = SO.evaluate_weighted(f, y, 'multi_class_linear_output', w)
    b = SO.evaluate_weighted(g, y, 'multi_class_linear_output', w)
    assert b['num_nonfinite'] == 0
    _same(a['nll_i'], b['nll_i'], 0.0)


# ------------------------------------------------------------------------------------------------------------------
# Refusals before the device
# ------------------------------------------------------------------------------------------------------------------
def _loo_like(kind, N_):
    r = LOO.LooResult() if kind == 'loo' else LOO.WaicResult()
    r.pointwise = torch.zeros(N_, dtype=torch.float64)
    r.num_points = N_
    return r


def test_stacking_weights_refusals():
    with pytest.raises(ValueError, match='at least two'):
        LOO.stacking_weights(_loo_like('loo', 5))
    with pytest.raises(TypeError, match='psis_loo results only'):
        LOO.stacking_weights(_loo_like('loo', 5), _loo_like('waic', 5))
    with pytest.raises(TypeError, match='psis_loo results only'):
        LOO.stacking_weights(torch.zeros(5), torch.zeros(5))
    with pytest.raises(RuntimeError, match='different numbers of data points'):
        LOO.stacking_weights(_loo_like('loo', 5), _loo_like('loo', 6))
    with pytest.raises(RuntimeError, match='CUDA device'):
        LOO.stacking_weights([_loo_like('loo', 5), _loo_like('loo', 5)])
    for tol in (0.0, -1.0, float('nan'), float('inf')):
        with pytest.raises(ValueError, match='tol'):
            LOO.stacking_weights(_loo_like('loo', 5), _loo_like('loo', 5), tol=tol)
    for it in (0, 2.5, True):
        with pytest.raises(ValueError, match='max_iter'):
            LOO.stacking_weights(_loo_like('loo', 5), _loo_like('loo', 5), max_iter=it)
        with pytest.raises(ValueError, match='max_iter'):
            LOO.chain_stacking(torch.zeros(2, 10, 4), max_iter=it)


def test_psis_loo_chains_refusals():
    res = HMCResult(torch.zeros(4, 10, 4), None, None, None, None, None, 3, 10)
    res.folds, res.num_folds = torch.zeros(7, dtype=torch.int64), 2
    for fn in (LOO.psis_loo_chains, LOO.chain_stacking):
        with pytest.raises(TypeError, match='K-fold'):
            fn(res)
    big = torch.zeros(2, NA.LOO_CHAIN_MAX_DRAWS + 1, 3)
    for fn in (LOO.psis_loo_chains, LOO.chain_stacking):
        with pytest.raises(RuntimeError, match='thin'):
            fn(big)
    with pytest.raises(RuntimeError, match='thin'):
        LOO.psis_loo_chains(torch.zeros(NA.LOO_CHAIN_MAX_DRAWS + 1, 3))
    with pytest.raises(ValueError, match='r_eff'):
        LOO.psis_loo_chains(torch.zeros(2, 10, 3), r_eff=0.0)
    with pytest.raises(RuntimeError, match='tau_out applies'):
        LOO.psis_loo_chains(torch.zeros(2, 10, 3), tau_out=torch.ones(2, 10))
    with pytest.raises(TypeError, match='expected an HMCResult'):
        LOO.psis_loo_chains(np.zeros((2, 10, 3)))
    # the block itself: a CPU tensor has no kernel to run on
    with pytest.raises(RuntimeError, match='CUDA device'):
        LOO.psis_loo_chains(torch.zeros(2, 10, 3))


def test_chain_weights_refusals():
    f = torch.zeros(3, 5, 4, 2)
    y = torch.zeros(4, dtype=torch.float32)
    kw = dict(y=y, model_loss='multi_class_linear_output')
    with pytest.raises(ValueError, match='holds 2 weights, the draws come from 3 chains'):
        P.evaluate(f, chain_weights=[0.5, 0.5], **kw)
    with pytest.raises(ValueError, match='non-negative'):
        P.evaluate(f, chain_weights=[1.2, -0.1, -0.1], **kw)
    with pytest.raises(ValueError, match='non-negative'):
        P.evaluate(f, chain_weights=[float('nan'), 0.5, 0.5], **kw)
    with pytest.raises(ValueError, match='sum to 1'):
        P.evaluate(f, chain_weights=[0.5, 0.5, 0.5], **kw)
    with pytest.raises(ValueError, match='vector'):
        P.evaluate(f, chain_weights=[[1.0, 0.0, 0.0]], **kw)
    # within 1e-6 of 1: normalised and accepted, then the CPU block is refused
    with pytest.raises(RuntimeError, match='CUDA device'):
        P.evaluate(f, chain_weights=[0.5, 0.25, 0.25 + 5e-7], **kw)
    with pytest.raises(ValueError, match='sum to 1'):
        P.evaluate(torch.zeros(2, 4, 3), chain_weights=[0.5, 0.6], **kw)
    w = P._chain_weights([0.5, 0.25, 0.25 + 5e-7])
    assert w.dtype == torch.float64 and abs(float(w.sum()) - 1.0) <= 1e-15
