"""CPU: the PSIS-LOO / WAIC definition of tests/loo_oracle.py (generalised-Pareto fit, an exact conjugate leave-one-out,
edge cases, the likelihood identities against the sampling closure), the host-side refusals of hamiltorch_b200.loo and
the argument checks of the ABI v12 entry points."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn as nn

from hamiltorch_b200 import loo as LOO
from hamiltorch_b200 import targets as T
from tests import loo_oracle as O


# ------------------------------------------------------------------------------------------------------------------
# the oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('xi', [0.2, 0.5, 0.9])
def test_gpd_fit_recovers_the_shape(xi):
    from scipy.stats import genpareto
    x = np.sort(genpareto.rvs(xi, scale=1.7, size=20000, random_state=np.random.default_rng(int(xi * 10))))
    khat, sigma = O.gpd_fit(x)
    assert abs(khat - xi) < 0.05, khat
    assert abs(sigma / 1.7 - 1.0) < 0.1, sigma


def _conjugate(N=40, d=3, tau_out=4.0, seed=0, outlier=False):
    """nn.Linear(d, 1) regression with Gaussian priors: the exact posterior, its exact leave-one-out predictive
    densities (rank-1 downdates of the posterior covariance) and the MLPTarget of the same model."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, d, generator=g, dtype=torch.float64)
    w_true = torch.tensor([0.8, -0.5, 0.3][:d], dtype=torch.float64)
    y = x @ w_true + 0.2 + torch.randn(N, generator=g, dtype=torch.float64) / math.sqrt(tau_out)
    if outlier:
        x[0] = torch.tensor([6.0, -6.0, 5.0][:d], dtype=torch.float64)
        y[0] = 12.0
    tau_w, tau_b = 2.0, 0.5
    X1 = torch.cat([x, torch.ones(N, 1, dtype=torch.float64)], 1)
    P = torch.diag(torch.tensor([tau_w] * d + [tau_b], dtype=torch.float64)) + tau_out * X1.t() @ X1
    Sig = torch.linalg.inv(P)
    h = tau_out * X1.t() @ y
    mu = Sig @ h
    exact = []
    for i in range(N):
        xi_ = X1[i]
        u = Sig @ xi_
        Sig_i = Sig + tau_out * torch.outer(u, u) / (1.0 - tau_out * (xi_ @ u))      # Sherman-Morrison downdate
        mu_i = Sig_i @ (h - tau_out * xi_ * y[i])
        m, v = float(xi_ @ mu_i), 1.0 / tau_out + float(xi_ @ Sig_i @ xi_)
        exact.append(-0.5 * math.log(2 * math.pi * v) - 0.5 * (float(y[i]) - m) ** 2 / v)
    model = nn.Linear(d, 1)
    tgt = T.MLPTarget.from_model(model, x.float(), y.float()[:, None], [torch.tensor(tau_w), torch.tensor(tau_b)],
                                 tau_out)
    L = torch.linalg.cholesky(Sig)
    return tgt, mu, L, np.array(exact)


def _posterior_draws(mu, L, S, seed=1):
    z = torch.randn(S, mu.numel(), generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    return mu + z @ L.t()                                   # flat layout of nn.Linear(d, 1): weight row, then bias


def test_conjugate_regression_matches_exact_leave_one_out():
    tgt, mu, L, exact = _conjugate()
    th = _posterior_draws(mu, L, 4000)
    ll = O.pointwise_log_lik(th, tgt)
    r = O.psis_loo(ll)
    assert np.abs(r['elpd_loo'] - exact).max() < 0.02, np.abs(r['elpd_loo'] - exact).max()
    assert r['pareto_k'].max() < 0.5
    assert r['num_bad_k'] == 0


def test_planted_high_leverage_outlier_gets_a_large_k_hat():
    tgt, mu, L, exact = _conjugate(outlier=True)
    ll = O.pointwise_log_lik(_posterior_draws(mu, L, 4000), tgt)
    r = O.psis_loo(ll)
    assert r['pareto_k'][0] > 0.7, r['pareto_k'][0]
    assert r['num_bad_k'] >= 1


def test_constant_log_likelihood_has_no_effective_parameters():
    ll = np.full((4, 50, 3), -1.25, dtype=np.float32)
    r, w = O.psis_loo(ll), O.waic(ll)
    assert np.all(np.abs(r['p_loo']) < 1e-12) and np.all(w['p_waic'] == 0.0)
    assert np.all(np.abs(r['elpd_loo'] + 1.25) < 1e-12)
    assert np.all(r['tail'] == 0) and np.all(np.isinf(r['pareto_k']))


def test_ties_at_the_cutoff_shrink_the_tail():
    S = 1000
    M = O.tail_cap(S)
    assert M == 95
    ll = np.concatenate([-10.0 - np.arange(50, dtype=np.float64), np.full(200, -5.0), -np.linspace(0, 4, 750)])
    p = O.psis_point(ll)
    assert p['tail'] == 50                                  # the 200 tied draws at the cutoff stay out of the tail
    assert np.isfinite(p['pareto_k'])
    ll2 = np.concatenate([np.array([-30.0, -20.0, -15.0]), np.full(300, -5.0), -np.linspace(0, 4, 697)])
    p2 = O.psis_point(ll2)
    assert p2['tail'] == 3 and p2['pareto_k'] == math.inf  # M' <= 4: nothing is smoothed


def test_non_finite_draw_makes_the_point_nan():
    ll = np.random.default_rng(0).normal(size=(2, 30, 4))
    ll[1, 3, 2] = -np.inf
    r = O.psis_loo(ll)
    assert np.isnan(r['elpd_loo'][2]) and np.isnan(r['pareto_k'][2]) and r['num_nonfinite'] == 1
    assert np.all(np.isfinite(r['elpd_loo'][[0, 1, 3]]))


# ------------------------------------------------------------------------------------------------------------------
# likelihood identities against the sampling closure (MLPTarget.__call__ minus the prior)
# ------------------------------------------------------------------------------------------------------------------
LOSSES = ['regression', 'binary_class_linear_output', 'multi_class_linear_output', 'multi_class_log_softmax_output']


def _loss_target(loss, tau_out, N=37, seed=0):
    torch.manual_seed(seed)
    O_ = {'regression': 2, 'binary_class_linear_output': 2}.get(loss, 4)
    layers = [nn.Linear(5, 8), nn.Tanh(), nn.Linear(8, O_)]
    if loss == 'multi_class_log_softmax_output':
        layers.append(nn.LogSoftmax(dim=1))
    model = nn.Sequential(*layers)
    x = torch.randn(N, 5)
    if loss == 'regression':
        y = torch.randn(N, O_)
    elif loss == 'binary_class_linear_output':
        y = (torch.rand(N, O_) < 0.5).float()
    else:
        y = torch.randint(0, O_, (N,)).float()
    from hamiltorch_b200 import util
    return T.MLPTarget.from_model(model, x, y, None, tau_out, model_loss=loss), util.flatten(model).detach()


@pytest.mark.parametrize('loss', LOSSES)
def test_pointwise_log_likelihood_identities(loss):
    tau = 1.0 if loss != 'regression' else 3.5
    tgt, th = _loss_target(loss, tau)
    ll = O.pointwise_log_lik(th[None], tgt)[0]
    ref = float((tgt(th) - tgt.log_prior(th) / tgt.prior_scale).double().sum())
    Np, O_ = tgt.x.shape[0], tgt.widths[-1]
    if loss == 'regression':
        want = ref + 0.5 * Np * O_ * math.log(tau / (2 * math.pi))
    elif loss == 'multi_class_log_softmax_output':
        want = Np * ref
    else:
        want = ref
    assert abs(ll.sum() - want) < 1e-4 * (1 + abs(want)), (ll.sum(), want)


def test_pointwise_log_likelihood_of_a_split_list_is_in_split_order():
    tgt, th = _loss_target('regression', 2.0, N=30)
    parts = [T.MLPTarget(tgt.widths, tgt.acts, tgt.x[a:b], tgt.y[a:b], tgt.tau_list, tgt.tau_out, prior_scale=3)
             for a, b in ((0, 7), (7, 20), (20, 30))]
    assert np.array_equal(O.pointwise_log_lik(th[None], parts), O.pointwise_log_lik(th[None], tgt))


# ------------------------------------------------------------------------------------------------------------------
# host-side refusals
# ------------------------------------------------------------------------------------------------------------------
def test_refusals_on_the_host():
    tgt, th = _loss_target('regression', 2.0)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        LOO.psis_loo(torch.zeros(2, 10, 5))
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        LOO.pointwise_log_lik(th.expand(2, 8, -1), tgt)
    with pytest.raises(TypeError, match='MLPTarget'):
        LOO.psis_loo(torch.zeros(2, 10, 3), T.GaussianIso(3))
    with pytest.raises(ValueError, match='r_eff'):
        LOO.psis_loo(torch.zeros(2, 10, 5), r_eff=0.0)
    with pytest.raises(ValueError, match='r_eff'):
        LOO.psis_loo(torch.zeros(2, 10, 5), r_eff=-1.0)
    with pytest.raises(RuntimeError, match='parameters per draw'):
        LOO.psis_loo(torch.zeros(2, 10, th.numel() + 1), tgt)
    nodata = T.MLPTarget(tgt.widths, tgt.acts, None, None, tgt.tau_list)
    with pytest.raises(RuntimeError, match='no data'):
        LOO.waic(torch.zeros(2, 10, th.numel()), nodata)


def _fake(kind, pointwise):
    r = LOO.LooResult() if kind == 'loo' else LOO.WaicResult()
    r.pointwise = torch.as_tensor(pointwise, dtype=torch.float64)
    r.num_points = r.pointwise.numel()
    if kind == 'loo':
        r.elpd_loo = float(r.pointwise.sum())
    else:
        r.elpd_waic = float(r.pointwise.sum())
    return r


def test_compare_differences_and_refusals():
    a, b = _fake('loo', [-1.0, -2.0, -0.5, -1.5]), _fake('loo', [-1.2, -1.9, -0.9, -1.6])
    c = LOO.compare(a, b)
    d = (b.pointwise - a.pointwise).numpy()
    assert c.order == [0, 1] and c.elpd_diff[0] == 0.0 and abs(c.elpd_diff[1] - d.sum()) < 1e-12
    assert abs(c.se_diff[1] - math.sqrt(4) * d.std(ddof=1)) < 1e-12 and c.se_diff[0] == 0.0
    with pytest.raises(RuntimeError, match='different numbers of data points'):
        LOO.compare(a, _fake('loo', [-1.0, -2.0]))
    with pytest.raises(TypeError):
        LOO.compare(a, _fake('waic', [-1.0, -2.0, -0.5, -1.5]))


# ------------------------------------------------------------------------------------------------------------------
# ABI v12
# ------------------------------------------------------------------------------------------------------------------
def test_abi_v12_entry_points_check_their_arguments(built_library):
    from hamiltorch_b200 import _native as N
    from hamiltorch_b200.engine import NativeTarget
    lib = N.load_library()
    assert lib.hmcx_abi_version() == 12
    for name in ('hmcx_mlp_pointwise_ll', 'hmcx_loo_workspace_bytes', 'hmcx_loo_pass'):
        assert hasattr(lib, name)
    tgt, _ = _loss_target('regression', 2.0)
    nt = NativeTarget(tgt, 'cpu')
    junk = C.c_void_p(16)
    args = lambda **kw: [kw.get(k, v) for k, v in (('t', nt.ref()), ('s', junk), ('cs', 8), ('ds', 64), ('C', 1),
                                                     ('n', 4), ('r0', 0), ('r1', 37), ('o', junk), ('ocs', 148),
                                                     ('ods', 37), ('st', None))]
    for bad in (dict(t=None), dict(s=None), dict(o=None), dict(C=0), dict(n=0), dict(cs=-1), dict(ods=-1),
                dict(r0=-1), dict(r1=38), dict(r0=5, r1=5)):
        assert lib.hmcx_mlp_pointwise_ll(*args(**bad)) == N.ERR_INVALID_ARG, bad
    gauss = N.TargetStruct()
    gauss.kind, gauss.dim = 0, 8
    assert lib.hmcx_mlp_pointwise_ll(*args(t=C.byref(gauss))) == N.ERR_UNSUPPORTED
    nodata = NativeTarget(T.MLPTarget(tgt.widths, tgt.acts, None, None, tgt.tau_list), 'cpu')
    assert lib.hmcx_mlp_pointwise_ll(*args(t=nodata.ref())) == N.ERR_INVALID_ARG

    assert lib.hmcx_loo_workspace_bytes(0, 10, 1) == 0 and lib.hmcx_loo_workspace_bytes(1, 1, 1) == 0
    assert lib.hmcx_loo_workspace_bytes(2, 10, 0) == 0 and lib.hmcx_loo_workspace_bytes(2, 10, N.RANK_MAX_SLAB + 1) == 0
    ws = lib.hmcx_loo_workspace_bytes(4, 100, 3)
    assert ws >= 4 * 4 * 100 * 3 and lib.hmcx_loo_workspace_bytes(4, 100, 6) > ws
    assert ws <= lib.hmcx_rank_workspace_bytes(4, 100, 3)
    largs = lambda **kw: [kw.get(k, v) for k, v in (('x', junk), ('cs', 500), ('ds', 5), ('C', 4), ('n', 100),
                                                      ('N', 5), ('i0', 1), ('k', 3), ('r', 1.0), ('pw', junk),
                                                      ('tl', junk), ('nf', junk), ('ws', junk), ('wb', ws),
                                                      ('st', None))]
    for bad in (dict(x=None), dict(pw=None), dict(tl=None), dict(nf=None), dict(ws=None), dict(cs=-1), dict(C=0),
                dict(n=0), dict(C=1, n=1), dict(N=0), dict(i0=-1), dict(i0=3), dict(k=0), dict(r=0.0), dict(r=-2.0),
                dict(r=float('inf')), dict(r=float('nan')), dict(wb=ws - 1)):
        assert lib.hmcx_loo_pass(*largs(**bad)) == N.ERR_INVALID_ARG, bad
