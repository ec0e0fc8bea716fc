"""CPU: the numpy definition of posterior predictive checks and LOO-PIT (tests/ppc_oracle.py) on its own, and every
refusal of hamiltorch_b200.ppc that is raised before the device is touched.

The conjugate nn.Linear(3, 1) regression of test_loo_cpu has closed-form leave-one-out predictives N(m_i, v_i), so
its exact LOO-PIT is Phi((y_i - m_i) / sqrt(v_i)); PSIS-weighted PIT from exact posterior draws must match it within
Monte-Carlo error."""
import math

import numpy as np
import pytest
import torch
import torch.nn as nn
from scipy import special, stats

from hamiltorch_b200 import ppc, targets as T
from tests import loo_oracle as LO
from tests import ppc_oracle as PO
from tests.test_loo_cpu import _conjugate, _posterior_draws


def _exact_loo_pit(tgt, tau_w=2.0, tau_b=0.5):
    """Phi((y_i - m_i) / sqrt(v_i)) of the conjugate model's exact leave-one-out predictive, from the target's data."""
    x, y, tau = tgt.x.double(), tgt.y.double()[:, 0], float(tgt.tau_out)
    N_, d = x.shape
    X1 = torch.cat([x, torch.ones(N_, 1, dtype=torch.float64)], 1)
    Pm = torch.diag(torch.tensor([tau_w] * d + [tau_b], dtype=torch.float64)) + tau * X1.t() @ X1
    Sig = torch.linalg.inv(Pm)
    h = tau * X1.t() @ y
    out = []
    for i in range(N_):
        xi = X1[i]
        u = Sig @ xi
        Sig_i = Sig + tau * torch.outer(u, u) / (1.0 - tau * (xi @ u))
        mu_i = Sig_i @ (h - tau * xi * y[i])
        m, v = float(xi @ mu_i), 1.0 / tau + float(xi @ Sig_i @ xi)
        out.append(0.5 * special.erfc(-(float(y[i]) - m) / math.sqrt(2.0 * v)))
    return np.array(out)


def _outputs(th, tgt):
    """(S, N, 1) fp64 outputs of nn.Linear(d, 1) draws (weight row, then bias)."""
    x = tgt.x.double().numpy()
    th = np.asarray(th, dtype=np.float64)
    return (th[:, :-1] @ x.T + th[:, -1:])[..., None]


def test_psis_weights_reproduce_loo_oracle_elpd():
    rng = np.random.default_rng(3)
    ll = -rng.standard_exponential(size=(2000, 5)) * rng.uniform(0.2, 1.0, 5)
    ref = LO.psis_loo(ll)
    for i in range(5):
        w, kh = PO.psis_weights(ll[:, i])
        assert abs(w.sum() - 1.0) < 1e-12
        assert abs(kh - ref['pareto_k'][i]) < 1e-12
        assert abs(math.log((w * np.exp(ll[:, i])).sum()) - ref['elpd_loo'][i]) < 1e-10


def test_tied_draws_take_the_stable_sort_order():
    # 30 tied log-likelihoods at the very top of r, all in the tail: ascending flat index = ascending sorted position
    ll = np.concatenate([np.full(30, -9.0), -np.linspace(0.0, 3.0, 970)])
    w, kh = PO.psis_weights(ll)
    assert math.isfinite(kh)
    tied = w[:30]
    assert np.all(np.diff(tied) <= 0) and tied[0] > tied[-1]       # lower index: smaller p, larger z, larger weight


def test_conjugate_loo_pit_matches_the_closed_form():
    tgt, mu, L, _ = _conjugate()
    th = _posterior_draws(mu, L, 4000)
    ll = LO.pointwise_log_lik(th, tgt)
    f = _outputs(th.numpy(), tgt)
    pit, kh = PO.loo_pit(ll, f, tgt.y.double().numpy(), np.full(4000, float(tgt.tau_out)))
    exact = _exact_loo_pit(tgt)
    assert np.abs(pit[:, 0] - exact).max() < 0.02, np.abs(pit[:, 0] - exact).max()
    assert kh.max() < 0.5


def test_in_sample_pit_is_less_dispersed_than_loo_pit():
    # the data used twice pulls every PIT value towards 1/2: the in-sample sd is below LOO-PIT's
    tgt, mu, L, _ = _conjugate(N=25)
    th = _posterior_draws(mu, L, 3000)
    f = _outputs(th.numpy(), tgt)
    y = tgt.y.double().numpy()
    tau = float(tgt.tau_out)
    ins = (0.5 * special.erfc(-(y[None] - f) * math.sqrt(tau) / math.sqrt(2.0))).mean(0)[:, 0]
    loo = PO.loo_pit(LO.pointwise_log_lik(th, tgt), f, y, np.full(3000, tau))[0][:, 0]
    assert np.abs(ins - 0.5).mean() < np.abs(loo - 0.5).mean()


def test_p_value_tie_convention():
    t_rep = np.array([[1.0, 0.5], [2.0, 0.5], [3.0, 0.25], [2.0, 0.75]])
    t_obs = np.array([2.0, 0.5])
    want = np.array([(1 + 0.5 * 2) / 4, (1 + 0.5 * 2) / 4])
    assert np.array_equal(PO.p_values(t_rep, t_obs), want)
    got = ppc.p_values(torch.from_numpy(t_rep), torch.from_numpy(t_obs))
    assert np.array_equal(got.numpy(), want)
    # per-draw observed values (the deviance column)
    obs = np.array([[0.0, 1.0], [3.0, 0.5], [3.0, 0.0], [2.0, 0.75]])
    assert np.array_equal(ppc.p_values(torch.from_numpy(t_rep), torch.from_numpy(obs)).numpy(), PO.p_values(t_rep, obs))


def test_statistics_and_deviance_definitions():
    rng = np.random.default_rng(1)
    y = rng.normal(size=(3, 40, 2))
    s = PO.statistics(y, 0, 2)
    assert s.shape == (3, 8)
    assert np.allclose(s[:, 1], y[:, :, 0].std(1, ddof=1)) and np.allclose(s[:, 6], y[:, :, 1].min(1))
    lab = rng.integers(0, 4, size=(3, 40, 1)).astype(np.float64)
    fr = PO.statistics(lab, 2, 4)
    assert np.allclose(fr.sum(1), 1.0)
    f = rng.normal(size=(3, 40, 4))
    ll = PO.log_lik(f, lab, 2, None)
    want = torch.log_softmax(torch.from_numpy(f), -1).gather(-1, torch.from_numpy(lab).long())[..., 0].numpy()
    assert np.allclose(ll, want)
    fb, yb = rng.normal(size=(3, 40, 2)), (rng.uniform(size=(3, 40, 2)) < 0.5).astype(np.float64)
    want = -torch.nn.functional.binary_cross_entropy_with_logits(torch.from_numpy(fb), torch.from_numpy(yb),
                                                                 reduction='none').sum(-1).numpy()
    assert np.allclose(PO.log_lik(fb, yb, 1, None), want)
    tau = np.array([1.0, 2.0, 4.0])
    d = PO.deviance(f[..., :2], y, 0, tau)
    want = -2 * stats.norm.logpdf(y, f[..., :2], 1 / np.sqrt(tau)[:, None, None]).sum((1, 2))
    assert np.allclose(d, want)


def test_uniformity_test_matches_scipy():
    u = np.random.default_rng(4).uniform(size=537)
    u[:3] = [0.0, 1.0, np.nan]
    hist, chi2, p = PO.uniformity(u, 20)
    ref = stats.chisquare(hist)
    assert hist.sum() == 536 and abs(chi2 - ref.statistic) < 1e-9 and abs(p - ref.pvalue) < 1e-12
    h2, c2, p2 = ppc.uniformity(torch.from_numpy(u), 20)
    assert np.array_equal(h2.numpy(), hist) and abs(c2 - chi2) < 1e-9 and abs(p2 - p) < 1e-12


# ------------------------------------------------------------------------------------------------------------------
# refusals before any CUDA work
# ------------------------------------------------------------------------------------------------------------------
def _cls_target(loss):
    model = nn.Linear(3, 4 if loss != 'binary_class_linear_output' else 2)
    if loss == 'multi_class_log_softmax_output':
        model = nn.Sequential(model, nn.LogSoftmax(dim=1))
    x = torch.randn(20, 3)
    y = torch.randint(0, 4, (20,)).float() if loss != 'binary_class_linear_output' else torch.zeros(20, 2)
    return T.MLPTarget.from_model(model, x, y, None, 1.0, model_loss=loss)


def test_refusals_before_the_device():
    tgt, mu, L, _ = _conjugate()
    th = _posterior_draws(mu, L, 8).float()
    gauss = T.GaussianIso(4)
    for fn in (ppc.replicate, ppc.check, ppc.loo_pit):
        with pytest.raises(TypeError, match='Bayesian-NN target'):
            fn(th, gauss)
    nodata = T.MLPTarget.from_model(nn.Linear(3, 1), None, None, None, 1.0)
    for fn in (ppc.replicate, ppc.check, ppc.loo_pit):
        with pytest.raises(RuntimeError, match='no data'):
            fn(th, nodata)
    for loss in ('binary_class_linear_output', 'multi_class_linear_output', 'multi_class_log_softmax_output'):
        with pytest.raises(NotImplementedError, match='reliability'):
            ppc.loo_pit(th, _cls_target(loss))
    for bins in (1, 2.5, True):
        with pytest.raises(ValueError, match='bins'):
            ppc.loo_pit(th, tgt, bins=bins)
    with pytest.raises(ValueError, match='r_eff'):
        ppc.loo_pit(th, tgt, r_eff=0.0)
    for draws in (torch.zeros(2, 2, dtype=torch.int64), torch.tensor([0.5]), torch.tensor([], dtype=torch.int64)):
        with pytest.raises(ValueError, match='draws'):
            ppc.replicate(th, tgt, draws=draws)
    with pytest.raises(ValueError, match='seed'):
        ppc.check(th, tgt, seed=-1)
    # the samples themselves: a CPU block has no kernel to run on
    with pytest.raises(RuntimeError, match='CUDA device'):
        ppc.check(th, tgt)


def test_stat_names():
    tgt, _, _, _ = _conjugate()
    assert ppc.stat_names(tgt) == ['mean[0]', 'sd[0]', 'min[0]', 'max[0]', 'deviance']
    assert ppc.stat_names(_cls_target('binary_class_linear_output')) == ['mean[0]', 'mean[1]', 'deviance']
    assert ppc.stat_names(_cls_target('multi_class_log_softmax_output')) == ['freq[%d]' % c for c in range(4)] + \
        ['deviance']
