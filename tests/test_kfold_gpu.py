"""GPU: K-fold refits of Bayesian NNs (sample_chains(folds=...), hmcx_split_run_folds), their scoring (loo.kfold) and the
exact refits of flagged PSIS-LOO points (loo.reloo).

* Every fold chain equals, bit for bit, a plain run on the MLPTarget of its fold's training rows with the same seed, the
  chain's global id as chain_offset and the same pinned cluster size: SIMT and tensor-core stacks, HMC and HMC_NUTS,
  1 / 2 / 4 CTAs per chain, regression and classification (the log-softmax loss is a mean over the training rows), the
  sink forms and the injected stream.
* kfold's pointwise values equal the fp64 logmeanexp of the likelihood block pointwise_log_lik gives for the same draws.
* On the conjugate regression of tests/test_loo_cpu.py the HMC fold runs match the exact K-fold values (K = 5) and the
  exact leave-one-out values (K = N), and reloo replaces the flagged planted outlier's PSIS value by its exact value."""
import numpy as np
import pytest
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import engine, loo as LOO, targets as T
from oracle import cases
from tests import kfold_oracle as KO
from tests.test_loo_cpu import _conjugate

pytestmark = pytest.mark.gpu

LOSS = {'regression': 'regression', 'binary': 'binary_class_linear_output',
        'logsoftmax': 'multi_class_log_softmax_output', 'multiclass': 'multi_class_linear_output'}


def _problem(shape, n=300):
    if shape == 'tc':                                            # 64-128-1: the tensor-core (wgmma) form
        model, x, y = cases.mlp_problem(seed=8, n=n, n_in=64, hidden=128)
        task, tau = 'regression', 20.
    elif shape == 'simt':                                        # 1-10-10-1, D = 141: SIMT tiles
        model, x, y = cases.mlp_problem(seed=9, n=n, n_in=1, hidden=10, depth=2)
        task, tau = 'regression', 20.
    else:                                                        # 3-8-3 classifiers
        model, x, y = cases.mlp_problem(seed=4, n=n, n_in=3, hidden=8, n_out=3 if shape != 'binary' else 1,
                                        task=shape)
        task, tau = shape, 1.
    tgt = T.MLPTarget.from_model(model, x, y, None, tau, prior_scale=1.5, model_loss=LOSS[task])
    return tgt, model


def _init(model, C_, seed=0, scale=0.05):
    D = hb.util.flatten(model).numel()
    return hb.util.flatten(model).detach()[None] + scale * torch.randn(C_, D, generator=torch.Generator().manual_seed(seed))


def _bits(t):
    return t.contiguous().view(torch.int32)


def _assert_same_chain(res, c, ref, thin=1):
    assert torch.equal(res.accepted[c], ref.accepted[0]) and torch.equal(res.diverged[c], ref.diverged[0])
    assert torch.equal(_bits(res.ham[c]), _bits(ref.ham[0]))
    assert torch.equal(res.step_size[c], ref.step_size[0]) and torch.equal(res.num_rejected[c], ref.num_rejected[0])
    assert torch.equal(_bits(res.samples[c].cpu()), _bits(ref.samples[0, ::thin].cpu()))
    assert torch.equal(res.final_state[c], ref.final_state[0])


def _check_against_plain_runs(tgt, f, init, K, kw, chain_offset=0, injected=None):
    res = hb.sample_chains(tgt, init, folds=f, chain_offset=chain_offset, **kw, **(injected or {}))
    parts = engine.fold_targets(tgt, f)
    for c in range(init.shape[0]):
        g = chain_offset + c
        one = {} if injected is None else dict(normals=injected['normals'][:, c:c + 1],
                                               log_uniforms=injected['log_uniforms'][:, c:c + 1])
        ref = hb.sample_chains(parts[g % K], init[c:c + 1], chain_offset=g, **kw, **one)
        torch.cuda.synchronize()
        _assert_same_chain(res, c, ref)
    assert res.num_folds == K and torch.equal(res.folds.cpu(), f) and res.folds.is_cuda
    return res


CASES = [('tc', 'HMC', 1), ('tc', 'NUTS', 2), ('tc', 'HMC', 4), ('simt', 'NUTS', 1), ('simt', 'HMC', 2),
         ('simt', 'NUTS', 4), ('logsoftmax', 'HMC', 1), ('logsoftmax', 'NUTS', 2), ('binary', 'HMC', 4)]


@pytest.mark.parametrize('shape, sampler, cluster', CASES)
def test_fold_chain_equals_plain_run_on_its_training_rows(shape, sampler, cluster):
    tgt, model = _problem(shape)
    tgt.cluster_size = cluster
    K, R = 3, 2
    f = LOO.kfold_split(tgt.x.shape[0], K, seed=cluster)
    kw = dict(num_samples=12, num_steps_per_sample=3, step_size=0.004 if shape in ('tc', 'simt') else 0.02, burn=3,
              rng='philox', seed=11, record_ham=True,
              sampler=hb.Sampler.HMC_NUTS if sampler == 'NUTS' else hb.Sampler.HMC)
    res = _check_against_plain_runs(tgt, f, _init(model, R * K, seed=cluster), K, kw, chain_offset=3 * K)
    assert 0.0 < float(res.accepted.float().mean())


def test_rows_left_in_every_fit_and_a_diagonal_mass():
    """reloo's layout: singleton folds, every other row at -1; with a 1-D inv_mass."""
    tgt, model = _problem('simt', n=130)
    f = torch.full((130,), -1, dtype=torch.int64)
    f[[4, 77, 129]] = torch.arange(3)
    im = 0.5 + torch.rand(tgt.dim, generator=torch.Generator().manual_seed(2))
    kw = dict(num_samples=10, num_steps_per_sample=3, step_size=0.004, burn=2, rng='philox', seed=5, record_ham=True,
              inv_mass=im)
    _check_against_plain_runs(tgt, f, _init(model, 6), 3, kw)


def test_injected_stream():
    tgt, model = _problem('simt', n=120)
    K, C_, S, D = 4, 8, 10, tgt.dim
    g = torch.Generator().manual_seed(6)
    inj = dict(normals=torch.randn(S, C_, D, generator=g), log_uniforms=torch.log(torch.rand(S, C_, generator=g)))
    kw = dict(num_samples=S, num_steps_per_sample=3, step_size=0.004, burn=2, rng='injected', record_ham=True)
    _check_against_plain_runs(tgt, LOO.kfold_split(120, K, seed=1), _init(model, C_), K, kw, injected=inj)


@pytest.mark.parametrize('shape', ['tc', 'logsoftmax'])
def test_sink_forms(shape):
    """thin / moments / keep_samples=False / store_on_GPU=False on a fold run equal the fold run without them."""
    tgt, model = _problem(shape)
    K = 3
    f = LOO.kfold_split(tgt.x.shape[0], K, seed=0)
    kw = dict(num_samples=14, num_steps_per_sample=3, step_size=0.004 if shape == 'tc' else 0.02, burn=2, rng='philox',
              seed=2, record_ham=True, folds=f)
    init = _init(model, 2 * K)
    full = hb.sample_chains(tgt, init, **kw)
    thin = hb.sample_chains(tgt, init, thin=3, moments=True, **kw)
    host = hb.sample_chains(tgt, init, store_on_GPU=False, **kw)
    none = hb.sample_chains(tgt, init, keep_samples=False, moments=True, **kw)
    torch.cuda.synchronize()
    for r in (thin, host, none):
        assert torch.equal(r.accepted, full.accepted) and torch.equal(_bits(r.ham), _bits(full.ham))
        assert torch.equal(r.final_state, full.final_state) and torch.equal(r.step_size, full.step_size)
    assert torch.equal(_bits(thin.samples.cpu()), _bits(full.samples[:, ::3].cpu()))
    assert not host.samples.is_cuda and torch.equal(_bits(host.samples), _bits(full.samples.cpu()))
    x = full.samples[:, 1:].double()
    assert torch.allclose(thin.moment_sum, x.sum(1), rtol=1e-10, atol=1e-10)
    assert torch.allclose(thin.moment_sumsq, (x * x).sum(1), rtol=1e-10, atol=1e-10)
    assert torch.equal(none.moment_sum, thin.moment_sum)


# ------------------------------------------------------------------------------------------------------------------
# scoring
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('shape', ['simt', 'tc', 'multiclass'])
def test_kfold_equals_logmeanexp_of_the_likelihood_block(shape):
    tgt, model = _problem(shape, n=200)
    K, R = 4, 3
    f = LOO.kfold_split(200, K, seed=5)
    res = hb.sample_chains(tgt, _init(model, R * K), num_samples=30, num_steps_per_sample=3,
                           step_size=0.004 if shape != 'multiclass' else 0.02, burn=5, rng='philox', seed=9, folds=f)
    kf = LOO.kfold(res, tgt)
    torch.cuda.synchronize()
    assert kf.kind == 'kfold' and kf.num_folds == K and kf.num_points == 200 and kf.num_draws == R * 25
    assert kf.pointwise.dtype == torch.float64 and kf.num_nonfinite == 0
    expect = np.empty(200)
    for k in range(K):
        ll = LOO.pointwise_log_lik(res.samples[k::K], tgt).cpu().numpy()            # (R, n, N) fp32
        rows = (f == k).numpy()
        expect[rows] = KO.logmeanexp(ll.reshape(-1, 200)[:, rows])
    pw = kf.pointwise.cpu().numpy()
    assert np.abs(pw - expect).max() <= 1e-12 * np.abs(expect).max(), np.abs(pw - expect).max()
    assert kf.elpd_kfold == pytest.approx(expect.sum(), rel=1e-12)
    assert kf.se == pytest.approx(np.sqrt(200) * expect.std(ddof=1), rel=1e-10)
    assert kf.kfoldic == -2 * kf.elpd_kfold and kf.kfoldic_se == 2 * kf.se
    again = LOO.kfold(res, tgt)
    assert torch.equal(again.pointwise, kf.pointwise)
    try:
        for slab in (1, 7):
            LOO._slab_points_override = slab
            assert torch.equal(LOO.kfold(res, tgt).pointwise, kf.pointwise), slab
    finally:
        LOO._slab_points_override = None


# ------------------------------------------------------------------------------------------------------------------
# end to end on the conjugate regression
# ------------------------------------------------------------------------------------------------------------------
# Tolerance: a held-out row's elpd is log of the posterior mean of its likelihood p_i, estimated from the fit's draws.
# Its Monte-Carlo standard error is mcse(p_i) / mean(p_i), mcse from the effective sample size of the p_i draws
# (diagnostics.summary over the chains of the fit); the test allows 4 of those, and at least 0.05.  With 8 chains x 800
# HMC draws per fit that is 0.05 for most rows and up to ~0.15 for rows far in the predictive's tail.  The runs use the
# diagonal of the full-data posterior covariance as inv_mass and a trajectory of 1.2 scaled units: a fixed trajectory
# near a multiple of half a period of the Gaussian posterior's oscillation would leave a direction's |theta| unmixed,
# a bias the ESS of the draws does not show.
_HMC = dict(num_samples=900, num_steps_per_sample=8, step_size=0.15, burn=100, rng='philox', seed=21)


def _mass(L):
    return (L * L).sum(1).float()                                # diag of the posterior covariance L L^T


def _conj_data(tgt):
    return tgt.x.double().numpy(), tgt.y.double().numpy().reshape(-1)


def _ess_tol(draws, tgt, rows):
    """max(0.05, 4 x the Monte-Carlo standard error of log mean p_i) for the data rows ``rows`` under ``draws``."""
    ll = LOO.pointwise_log_lik(draws, tgt)[..., rows].double()
    w = torch.exp(ll - ll.amax(dim=(0, 1), keepdim=True)).float().contiguous()
    d = hb.diagnostics.summary(w)
    return np.maximum(0.05, 4 * (d.mcse / d.mean).cpu().numpy())


@pytest.mark.parametrize('K', [5, 40])
def test_conjugate_fold_runs_match_the_exact_values(K):
    tgt, mu, L, exact = _conjugate()
    f = LOO.kfold_split(40, K, seed=K)
    R = 8
    init = mu.float()[None].repeat(R * K, 1) + 0.05 * torch.randn(R * K, 4, generator=torch.Generator().manual_seed(0))
    res = hb.sample_chains(tgt, init, folds=f, inv_mass=_mass(L), **_HMC)
    kf = LOO.kfold(res, tgt)
    x, y = _conj_data(tgt)
    want = KO.conjugate_kfold(x, y, f.numpy(), 4.0, 2.0, 0.5)
    if K == 40:
        assert np.abs(want - exact).max() < 1e-5                # K = N is leave-one-out
    tol = np.empty(40)
    for k in range(K):
        rows = torch.nonzero(f == k).flatten()
        tol[rows.numpy()] = _ess_tol(res.samples[k::K], tgt, rows.to(res.samples.device))
    err = np.abs(kf.pointwise.cpu().numpy() - want)
    bad = np.nonzero(err >= tol)[0]
    assert bad.size == 0, [(int(i), err[i], tol[i], want[i]) for i in bad]
    assert np.median(tol) < 0.06
    assert float(res.accepted.float().mean()) > 0.6


def test_reloo_replaces_the_flagged_outlier_with_its_exact_value():
    tgt, mu, L, exact = _conjugate(outlier=True)
    R = 8
    init = mu.float()[None].repeat(R, 1) + 0.02 * torch.randn(R, 4, generator=torch.Generator().manual_seed(1))
    kw = dict(_HMC, inv_mass=_mass(L))
    res = hb.sample_chains(tgt, init, **kw)
    lo = LOO.psis_loo(res, tgt)
    pk = lo.pareto_k.cpu()
    assert float(pk[0]) > lo.k_threshold and lo.num_bad_k >= 1
    snapshot = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in lo.__dict__.items()}
    out = LOO.reloo(lo, tgt, init, **dict(kw, seed=33))
    torch.cuda.synchronize()
    for k, v in snapshot.items():                                 # the input result is not modified
        assert torch.equal(getattr(lo, k), v) if torch.is_tensor(v) else getattr(lo, k) == v
    flagged = torch.nonzero(pk > lo.k_threshold).flatten()
    assert torch.equal(out.refit_points, flagged) and 0 in flagged.tolist()
    # the refit reloo ran, again (Philox: the same draws), for its ESS and the exact bits of its scoring
    K = flagged.numel()
    f = torch.full((40,), -1, dtype=torch.int64)
    f[flagged] = torch.arange(K)
    if K == 1:
        refit = hb.sample_chains(engine.fold_targets(tgt, f)[0], init, **dict(kw, seed=33))
    else:
        refit = hb.sample_chains(tgt, init.repeat_interleave(K, dim=0), folds=f, **dict(kw, seed=33))
    e, _, _ = LOO._fold_elpd(refit.samples, tgt, f, K)
    assert torch.equal(out.pointwise[flagged], e[flagged.to(e.device)])
    tol = np.array([_ess_tol(refit.samples[k::K], tgt, flagged[k:k + 1].to(e.device))[0] for k in range(K)])
    new, old = out.pointwise.cpu().numpy()[flagged.numpy()], lo.pointwise.cpu().numpy()[flagged.numpy()]
    ex = exact[flagged.numpy()]
    assert np.all(np.abs(new - ex) < tol), (new, ex, tol)
    assert abs(old[0] - ex[0]) > tol[0], (old[0], ex[0], tol[0])  # what PSIS could not get right
    keep = np.setdiff1d(np.arange(40), flagged.numpy())
    for name in ('pointwise', 'p_loo_i', 'pareto_k', 'lppd'):    # unflagged points: the same bits
        assert torch.equal(getattr(out, name)[keep], getattr(lo, name)[keep]), name
    assert out.num_bad_k == 0 and float(out.pareto_k[flagged].abs().max()) == 0.0
    assert torch.equal(out.p_loo_i[flagged], out.lppd[flagged] - out.pointwise[flagged])
    assert out.elpd_loo == pytest.approx(float(out.pointwise.sum()), rel=1e-12)
    assert out.kind == 'loo' and LOO.compare(out, lo).order in ([0, 1], [1, 0])
