"""GPU: power-scaling sensitivity (hmcx_psens.cu, hamiltorch_b200/sensitivity.py) against tests/psens_oracle.py for
the four losses, SIMT and tensor-core networks, a split list, a hyperprior run, a tempered run, thinned draws and a
quantities block; the same bits on every call and at every slab size; the power-scaled moments of a conjugate linear
regression fitted with HMC against their closed forms; and the three diagnoses on fits with fixed seeds.

Tolerance of the oracle parity: the components are compared at 2e-5 relative (the GPU's per-row log-likelihoods are
fp32 network passes, which tests/test_loo_gpu.py holds to 1e-5 per row against the fp64 oracle).  Everything after the
components is fed the GPU's own components, so both sides weigh and sort the same fp32 values and differ only in the
order of fp64 sums: k-hat, means and sds at 1e-9 relative, CJS distances and sensitivities at 1e-7 (the CJS numerator
cancels about three digits) -- loose against fp64 rounding, tight against any change of definition."""
import numpy as np
import pytest
import torch
import torch.nn as nn

from hamiltorch_b200 import diagnostics, samplers, util
from hamiltorch_b200 import sensitivity as SE
from hamiltorch_b200 import targets as T
from tests import loo_oracle as LO
from tests import psens_oracle as PS
from tests.test_loo_gpu import LOSSES, _data, _draws, _net

pytestmark = pytest.mark.gpu

_FIELDS = ('log_prior', 'log_lik', 'cjs', 'mean', 'sd', 'prior', 'likelihood', 'pareto_k', 'tail_size')


def _close(got, want, tol, name):
    g = got.detach().cpu().double().numpy() if torch.is_tensor(got) else np.asarray(got, np.float64)
    w = np.asarray(want, np.float64)
    ok = (np.abs(g - w) <= tol * (1 + np.abs(w))) | (np.isnan(g) & np.isnan(w))
    assert ok.all(), (name, np.nanmax(np.abs(g - w)))


def _bits(t):
    return t.detach().contiguous().view(torch.uint8).cpu()


def _same(a, b, what=''):
    for f in _FIELDS:
        assert torch.equal(_bits(getattr(a, f)), _bits(getattr(b, f))), (f, what)
    assert a.diagnosis == b.diagnosis, what


def _oracle_components(draws, target, tau=None, hyper=None, tau_trace=None):
    items = target if isinstance(target, list) else [target]
    first = items[0]
    th = draws.detach().cpu().double().reshape(-1, first.dim).numpy()
    K = 2 * first.num_layers
    sampled = [False] * (K + 1) if hyper is None else [ab is not None for ab in hyper]
    taus = [0.0 if sampled[k] else float(first.tau_list[k]) for k in range(K)]
    lp = PS.normal_log_prior(th, first.sizes, taus) * len(items) / float(first.prior_scale)
    for k in range(K + 1):
        if sampled[k]:
            t = (tau_trace[0][..., k] if k < K else tau_trace[1]).detach().cpu().double().reshape(-1).numpy()
            lp = lp + PS.gamma_log_pdf(t, *hyper[k])
    tv = None if tau is None else tau.detach().cpu().double().reshape(-1).numpy()
    if first.loss_id == T.LOSS_REGRESSION and tv is not None:
        ll = PS.regression_ll(th, target, tv)
    else:
        ll = LO.pointwise_log_lik(th, target)
    tau_out = tv if tv is not None else first.tau_out
    return lp, PS.log_lik_total(ll, first.loss_id, tau_out, [t.x.shape[0] for t in items])


def _check(s, draws, target, quantities=None, lo=0.99, hi=1.01, **comp):
    """s against the oracle: the components from the draws, everything else from the GPU's components."""
    C_, n = draws.shape[0], draws.shape[1]
    lp, ll = _oracle_components(draws, target, **comp)
    _close(s.log_prior.reshape(-1), lp, 2e-5, 'log_prior')
    _close(s.log_lik.reshape(-1), ll, 2e-5, 'log_lik')
    glp, gll = s.log_prior.reshape(-1).cpu().numpy(), s.log_lik.reshape(-1).cpu().numpy()
    cols = [draws.detach().cpu().double().reshape(C_ * n, -1).numpy(),
            np.stack([glp, gll], 1).astype(np.float32).astype(np.float64)]
    if quantities is not None:
        cols.append(quantities.detach().cpu().double().reshape(C_ * n, -1).numpy())
    ref = PS.power_scale(np.concatenate(cols, 1), glp, gll, lo, hi, s.r_eff, s.threshold)
    _close(s.pareto_k, ref['pareto_k'], 1e-9, 'pareto_k')
    for f, tol in (('mean', 1e-9), ('sd', 1e-9), ('cjs', 1e-7), ('prior', 1e-7), ('likelihood', 1e-7)):
        _close(getattr(s, f), ref[f], tol, f)
    near = np.abs(np.stack([ref['prior'], ref['likelihood']]) - s.threshold).min(0) < 1e-6
    assert all(a == b or nr for a, b, nr in zip(s.diagnosis, ref['diagnosis'], near))
    assert len(s.names) == len(s.diagnosis) == s.cjs.shape[1]
    return ref


def _tgt_draws(loss, form, seed, C=3, n=40):
    torch.manual_seed(seed)
    if form == 'simt':
        model, O_ = _net(loss, 7, 24)
        N_ = 203
    else:
        model, O_ = _net(loss, 64, 128, nn.ReLU)
        N_ = 300
    x, y = _data(loss, N_, model[0].in_features, O_, seed + 1)
    tgt = T.MLPTarget.from_model(model, x, y, [torch.tensor(2.0), torch.tensor(0.5)] * 2,
                                 2.5 if loss == 'regression' else 1.5, model_loss=loss)
    return tgt, _draws(model, C, n, 0.03, seed + 2).cuda()


# ------------------------------------------------------------------------------------------------------------------
# 1. Oracle parity
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('form', ['simt', 'tc'])
@pytest.mark.parametrize('loss', LOSSES)
def test_matches_the_oracle(loss, form):
    tgt, draws = _tgt_draws(loss, form, 3)
    s = SE.power_scale(draws, tgt)
    _check(s, draws, tgt)
    assert s.names[0] == 'w0[0,0]' and s.names[-2:] == ['log_prior', 'log_lik']
    assert [r['name'] for r in s.by_tensor] == ['w0', 'b0', 'w1', 'b1']
    assert sum(r['size'] for r in s.by_tensor) == tgt.dim
    # the generic path with the same components gives the same bits
    g = SE.power_scale(draws, log_prior=s.log_prior, log_lik=s.log_lik)
    for f in ('cjs', 'mean', 'sd', 'pareto_k'):
        assert torch.equal(getattr(g, f), getattr(s, f)), f


def test_a_split_list_run_with_splitting():
    torch.manual_seed(4)
    model, O_ = _net('regression', 6, 16)
    x, y = _data('regression', 250, 6, O_, 5)
    bounds = [0, 70, 190, 250]
    parts = [T.MLPTarget.from_model(model, x[a:b], y[a:b], None, 3.0, prior_scale=3) for a, b in zip(bounds, bounds[1:])]
    q0 = util.flatten(model).detach()[None].repeat(3, 1)
    res = samplers.sample_chains(parts, q0, num_samples=60, num_steps_per_sample=4, step_size=0.01, burn=10,
                                 integrator=samplers.Integrator.SPLITTING, seed=2)
    s = SE.power_scale(res, parts)
    _check(s, res.samples, parts)


def test_a_hyperprior_run():
    g = torch.Generator().manual_seed(8)
    x = torch.randn(60, 3, generator=g)
    y = x @ torch.tensor([[0.8], [-0.5], [0.3]]) + 0.2 + 0.3 * torch.randn(60, 1, generator=g)
    tgt = T.MLPTarget.from_model(nn.Linear(3, 1), x, y, [torch.tensor(1.0)] * 2, 1.0)
    res = samplers.sample_chains(tgt, 0.1 * torch.randn(3, 4, generator=g), num_samples=60, num_steps_per_sample=5,
                                 step_size=0.02, burn=10, tau_prior=[(2.0, 1.0), None], tau_out_prior=(2.0, 0.2),
                                 seed=5)
    assert res.hyper == [(2.0, 1.0), None, (2.0, 0.2)]
    s = SE.power_scale(res, tgt)
    _check(s, res.samples, tgt, tau=res.tau_out_trace, hyper=res.hyper,
           tau_trace=(res.tau_list_trace, res.tau_out_trace))
    lp, ll = SE.log_components(res, tgt)
    assert torch.equal(lp, s.log_prior) and torch.equal(ll, s.log_lik)


def test_a_tempered_run_scores_its_cold_rows():
    tgt, _ = _tgt_draws('regression', 'simt', 6)
    q0 = (0.1 * torch.randn(4, tgt.dim, generator=torch.Generator().manual_seed(0)))
    res = samplers.sample_chains(tgt, q0, num_samples=40, num_steps_per_sample=3, step_size=0.005, burn=5,
                                 betas=[1.0, 0.4], swap_every=5, seed=1)
    assert res.samples.shape[0] == 2
    _check(SE.power_scale(res, tgt), res.samples, tgt)


def test_thinned_draws_and_a_quantities_block():
    tgt, _ = _tgt_draws('binary_class_linear_output', 'simt', 7)
    q0 = 0.1 * torch.randn(3, tgt.dim, generator=torch.Generator().manual_seed(1))
    res = samplers.sample_chains(tgt, q0, num_samples=91, num_steps_per_sample=3, step_size=0.01, burn=10, thin=3,
                                 seed=3)
    C_, n = res.samples.shape[:2]
    qb = torch.randn(C_, n, 5, generator=torch.Generator().manual_seed(2)).cuda()
    s = SE.power_scale(res, tgt, quantities=qb, lower_alpha=0.9, upper_alpha=1.2)
    _check(s, res.samples, tgt, quantities=qb, lo=0.9, hi=1.2)
    assert s.names[-5:] == ['q[%d]' % j for j in range(5)]


def test_a_nan_quantity_poisons_its_column_only():
    tgt, draws = _tgt_draws('regression', 'simt', 9)
    qb = torch.randn(3, 40, 4, generator=torch.Generator().manual_seed(3)).cuda()
    qb[1, 7, 2] = float('nan')
    s = SE.power_scale(draws, tgt, quantities=qb)
    assert s.num_nonfinite == 1
    col = tgt.dim + 2 + 2
    for f in ('cjs', 'mean', 'sd'):
        v = getattr(s, f)
        assert torch.isnan(v[:, col]).all() and torch.isfinite(torch.cat([v[:, :col], v[:, col + 1:]], 1)).all()
    assert s.diagnosis[col] == SE.NONE
    _check(s, draws, tgt, quantities=qb)


# ------------------------------------------------------------------------------------------------------------------
# 2. Determinism
# ------------------------------------------------------------------------------------------------------------------
def test_same_bits_on_every_call_and_at_every_slab_size():
    tgt, draws = _tgt_draws('multi_class_log_softmax_output', 'tc', 11)
    qb = torch.randn(3, 40, 3, generator=torch.Generator().manual_seed(4)).cuda()
    a = SE.power_scale(draws, tgt, quantities=qb)
    _same(a, SE.power_scale(draws, tgt, quantities=qb), 'second call')
    try:
        for cols, rows in ((1, 128), (7, 256), (1000, None), (None, 128)):
            SE._slab_cols_override, SE._slab_rows_override = cols, rows
            _same(a, SE.power_scale(draws, tgt, quantities=qb), 'slabs %s x %s' % (cols, rows))
    finally:
        SE._slab_cols_override = SE._slab_rows_override = None


# ------------------------------------------------------------------------------------------------------------------
# 3. Conjugate truth and behaviour: one-layer linear regression, a Gaussian posterior
# ------------------------------------------------------------------------------------------------------------------
def _linear(N_, tau, w_true, b_true, tau_out, seed):
    g = torch.Generator().manual_seed(seed)
    d = len(w_true)
    x = torch.randn(N_, d, generator=g)
    y = x @ torch.tensor(w_true)[:, None] + b_true + tau_out ** -0.5 * torch.randn(N_, 1, generator=g)
    tgt = T.MLPTarget.from_model(nn.Linear(d, 1), x, y, [torch.tensor(tau)] * 2, tau_out)
    return tgt, x.double(), y.double()


def _posterior(x, y, tau_prior, tau_out):
    """Mean and covariance of the Gaussian posterior with prior precision tau_prior and noise precision tau_out."""
    X1 = torch.cat([x, torch.ones(x.shape[0], 1, dtype=torch.float64)], 1)
    P = tau_prior * torch.eye(X1.shape[1], dtype=torch.float64) + tau_out * X1.t() @ X1
    cov = torch.linalg.inv(P)
    return cov @ (tau_out * X1.t() @ y.reshape(-1)), cov


def _fit(tgt, x, y, tau, tau_out, seed, C=16, n=2000):
    """HMC draws of the Gaussian posterior, started in it.  The trajectory is about half the smallest posterior sd times
    pi (a quarter period of the harmonic motion), so neither the draws nor their squares are antithetic."""
    mu, cov = _posterior(x, y, tau, tau_out)
    sd = cov.diagonal().sqrt()
    q0 = (mu + sd * torch.randn(C, mu.numel(), generator=torch.Generator().manual_seed(seed), dtype=torch.float64))
    res = samplers.sample_chains(tgt, q0.float(), num_samples=n + 100, num_steps_per_sample=10,
                                 step_size=0.15 * float(sd.min()), burn=100, seed=seed)
    return res.samples[:, 1:]


def test_conjugate_power_scaled_moments_match_the_closed_form():
    tau, tau_out = 2.0, 4.0
    tgt, x, y = _linear(15, tau, [0.7, -0.4], 0.3, tau_out, 1)
    blk = _fit(tgt, x, y, tau, tau_out, 2)
    ess_m = diagnostics.summary(blk).ess.cpu()
    ess_v = diagnostics.summary(((blk - blk.mean((0, 1))) ** 2).contiguous()).ess.cpu()
    s = SE.power_scale(blk, tgt, lower_alpha=0.8, upper_alpha=1.25)
    base_sd = _posterior(x, y, tau, tau_out)[1].diagonal().sqrt()
    moved = 0
    for row, (comp, a) in enumerate((('prior', 0.8), ('prior', 1.25), ('lik', 0.8), ('lik', 1.25))):
        mu, cov = _posterior(x, y, a * tau, tau_out) if comp == 'prior' else _posterior(x, y, tau, a * tau_out)
        sd = cov.diagonal().sqrt()
        got_m, got_s = s.mean[row + 1, :3].cpu(), s.sd[row + 1, :3].cpu()
        # 5 MCSE, the effective sizes halved for the importance weighting
        tol_m, tol_s = 5 * sd / torch.sqrt(0.5 * ess_m), 5 * sd / torch.sqrt(0.5 * ess_v)
        assert (torch.abs(got_m - mu) < tol_m).all(), (comp, a, got_m, mu, tol_m)
        assert (torch.abs(got_s - sd) < tol_s).all(), (comp, a, got_s, sd, tol_s)
        moved += int((torch.abs(sd - base_sd) > tol_s).sum())
    assert moved > 0           # some closed-form sd differs from the base posterior's by more than its tolerance


def _diagnoses(N_, tau, w_true, b_true, tau_out, seed):
    tgt, x, y = _linear(N_, tau, w_true, b_true, tau_out, seed)
    s = SE.power_scale(_fit(tgt, x, y, tau, tau_out, seed + 1), tgt)
    return s, s.diagnosis[:tgt.dim]


def test_a_vague_prior_with_plenty_of_data_flags_no_weight():
    s, d = _diagnoses(500, 1e-4, [1.0, -1.0], 0.5, 1.0, 3)
    assert d == [SE.NONE] * 3, (d, s.prior[:3], s.likelihood[:3])
    assert s.by_tensor[0]['num_conflict'] == s.by_tensor[0]['num_strong_prior'] == 0


def test_a_tight_prior_with_few_rows_is_a_strong_prior():
    s, d = _diagnoses(5, 400.0, [0.02, -0.02], 0.0, 1.0, 5)
    assert d == [SE.STRONG_PRIOR] * 3, (d, s.prior[:3], s.likelihood[:3])


def test_a_tight_prior_far_from_the_data_is_a_conflict():
    s, d = _diagnoses(100, 25.0, [3.0, -3.0], 3.0, 1.0, 7)
    assert d == [SE.CONFLICT] * 3, (d, s.prior[:3], s.likelihood[:3])
    assert s.num_conflict >= 3
