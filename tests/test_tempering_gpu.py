"""GPU: replica exchange for Bayesian NNs (DESIGN §3.17) -- tempered ladders across the chain batch, swapped on the GPU.

betas=[1.0] against the plain sink run, bit for bit; a ladder without swaps against independent runs at beta_t * tau_out;
the kernel and the swap rounds against tests/temper_oracle.py under the injected stream; every swap decision against the
fp64 rule; Philox mode against its injected twin and against ladder sharding; the tempered Gaussian posteriors of a
conjugate linear regression; a sign-symmetric network whose modes plain chains cannot cross; the sink options and the
consumers of the result."""
import math

import numpy as np
import pytest
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import engine, samplers, targets as T
from hamiltorch_b200 import diagnostics, loo, predictive
from oracle import cases, hmc_oracle as O
from tests import philox_ref as P
from tests import temper_oracle as TO
from tests.test_philox_stream_gpu import _stream

pytestmark = pytest.mark.gpu
MLP_RTOL = 2e-4               # tests/test_mlp_gpu.py
LL_RTOL = 1e-4                # the untempered log-likelihood: fp32 loss sums against the oracle's fp64 ones
STREAM_SWAP = 5
INTEGRATORS = {'PLAIN': (samplers.Integrator.IMPLICIT, None), 'SPLITTING': (samplers.Integrator.SPLITTING, O.SPLIT_SYM),
               'SPLITTING_RAND': (samplers.Integrator.SPLITTING_RAND, O.SPLIT_RAND),
               'SPLITTING_KMID': (samplers.Integrator.SPLITTING_KMID, O.SPLIT_KMID)}


def _problem(kind):
    """(model, targets for M = 1 and M = 2)."""
    if kind.startswith('tc'):                         # 16 -> 128 -> 1: the tensor-core form
        model, x, y = cases.mlp_problem(seed=4, n=512, n_in=16, hidden=128)
        loss = 'regression'
    elif kind == 'multiclass':                        # iris-shaped: 4 features, 3 classes
        model, x, y = cases.mlp_problem(seed=6, n=96, n_in=4, hidden=8, n_out=3, task='multiclass')
        loss = 'multi_class_linear_output'
    elif kind == 'binary':
        model, x, y = cases.mlp_problem(seed=6, n=64, n_in=4, hidden=8, task='binary')
        loss = 'binary_class_linear_output'
    elif kind == 'logsoftmax':
        model, x, y = cases.mlp_problem(seed=7, n=96, n_in=4, hidden=8, n_out=3, task='logsoftmax')
        loss = 'multi_class_log_softmax_output'
    else:                                             # 4-8-1 regression
        model, x, y = cases.mlp_problem(seed=5, n=64, n_in=4, hidden=8)
        loss = 'regression'
    tau_out = 20.0 if loss == 'regression' else 1.0
    one = T.MLPTarget.from_model(model, x, y, None, tau_out, model_loss=loss)
    n = x.shape[0] // 2
    two = [T.MLPTarget.from_model(model, x[a:a + n], y[a:a + n], None, tau_out, prior_scale=2, model_loss=loss)
           for a in (0, n)]
    return model, one, two


def _pin(tgt, cs):
    for d in (tgt if isinstance(tgt, list) else [tgt]):
        d.cluster_size = cs
    return tgt


def _q0(model, C_, seed=2, scale=0.05):
    D = hb.util.flatten(model).numel()
    return hb.util.flatten(model).detach()[None] + scale * torch.randn(C_, D, generator=torch.Generator().manual_seed(seed))


def _bits(t):
    t = t.detach().cpu().contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


# ------------------------------------------------------------------------------------------------------------------
# 1. betas = [1.0] is the plain sink run
# ------------------------------------------------------------------------------------------------------------------
CASES_1 = [('reg', 'PLAIN', False, 0), ('reg', 'SPLITTING', False, 0), ('reg', 'SPLITTING_RAND', False, 0),
           ('reg', 'SPLITTING_KMID', False, 0), ('reg', 'PLAIN', True, 0), ('reg', 'SPLITTING', True, 0),
           ('reg', 'SPLITTING_RAND', True, 0), ('reg', 'SPLITTING_KMID', True, 0),
           ('tc', 'PLAIN', False, 1), ('tc', 'PLAIN', True, 2), ('tc', 'SPLITTING', False, 4)]


@pytest.mark.parametrize('kind,integ,nuts,cs', CASES_1)
def test_single_rung_is_the_plain_sink_run(kind, integ, nuts, cs):
    model, one, two = _problem(kind)
    integrator, _ = INTEGRATORS[integ]
    tgt = _pin(one if integ == 'PLAIN' else two, cs)
    q0 = _q0(model, 4)
    kw = dict(num_samples=20, num_steps_per_sample=3, step_size=0.002 if kind == 'tc' else 0.004, burn=5,
              integrator=integrator, sampler=samplers.Sampler.HMC_NUTS if nuts else samplers.Sampler.HMC, seed=31,
              moments=True)
    plain = samplers.sample_chains(tgt, q0, **kw)
    temp = samplers.sample_chains(tgt, q0, betas=[1.0], swap_every=7, **kw)
    torch.cuda.synchronize()
    assert _same(plain.samples, temp.samples) and _same(plain.accepted, temp.accepted)
    assert _same(plain.step_size, temp.step_size) and _same(plain.final_state, temp.final_state)
    assert torch.equal(plain.moment_sum, temp.moment_sum) and torch.equal(plain.moment_sumsq, temp.moment_sumsq)
    assert temp.swap_accepted.shape == (2, 4, 0) and temp.swap_ll.shape == (2, 4)


# ------------------------------------------------------------------------------------------------------------------
# 2. no swaps: row t is the run at beta_t * tau_out
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind,integ,nuts', [('reg', 'PLAIN', False), ('reg', 'SPLITTING', True),
                                             ('binary', 'SPLITTING_RAND', False), ('tc', 'PLAIN', False)])
def test_without_swaps_each_rung_is_its_own_run(kind, integ, nuts):
    model, one, two = _problem(kind)
    integrator, _ = INTEGRATORS[integ]
    tgt = one if integ == 'PLAIN' else two
    betas, R, S = [1.0, 0.5, 0.2], 2, 16
    Tn = len(betas)
    C_ = R * Tn
    q0 = _q0(model, C_)
    g = torch.Generator().manual_seed(9)
    z = torch.randn(S, C_, q0.shape[1], generator=g)
    lu = torch.log(torch.rand(S, C_, generator=g))
    M = 1 if integ == 'PLAIN' else 2
    perms = torch.stack([torch.stack([torch.randperm(M, generator=g) for _ in range(C_)]) for _ in range(S)])
    kw = dict(num_samples=S, num_steps_per_sample=3, step_size=0.002 if kind == 'tc' else 0.004, burn=4,
              integrator=integrator, sampler=samplers.Sampler.HMC_NUTS if nuts else samplers.Sampler.HMC,
              rng='injected')
    res = samplers.sample_chains(tgt, q0, normals=z, log_uniforms=lu, perms=perms, betas=betas, swap_every=S,
                                 swap_log_uniforms=torch.zeros(0, R, Tn - 1, dtype=torch.float64), **kw)
    for t, b in enumerate(betas):
        ref = samplers.sample_chains(TO.tempered(tgt, b), q0[t::Tn], normals=z[:, t::Tn], log_uniforms=lu[:, t::Tn],
                                     perms=perms[:, t::Tn], **kw)
        torch.cuda.synchronize()
        assert _same(res.accepted[t::Tn], ref.accepted) and _same(res.step_size[t::Tn], ref.step_size)
        assert _same(res.final_state[t::Tn], ref.final_state)
        if t == 0:
            assert _same(res.samples, ref.samples)


# ------------------------------------------------------------------------------------------------------------------
# 3 + 4. injected parity with swaps against the oracle; every decision is the fp64 rule
# ------------------------------------------------------------------------------------------------------------------
def _check_decisions(res, betas, lu_swap):
    acc, ll = res.swap_accepted.cpu().numpy(), res.swap_ll.cpu().numpy()
    rounds, R, P_ = acc.shape
    Tn = len(betas)
    for k in range(rounds):
        for r in range(R):
            for t in range(P_):
                if t % 2 != k % 2:
                    assert acc[k, r, t] == -1
                    continue
                a = r * Tn + t
                assert acc[k, r, t] == TO.swap_decision(betas[t], betas[t + 1], ll[k, a], ll[k, a + 1],
                                                        float(lu_swap[k, r, t])), (k, r, t)


@pytest.mark.parametrize('kind,integ', [('reg', 'PLAIN'), ('multiclass', 'PLAIN'), ('binary', 'PLAIN'),
                                        ('logsoftmax', 'SPLITTING')])
def test_oracle_parity_with_swaps(kind, integ):
    model, one, two = _problem(kind)
    integrator, osch = INTEGRATORS[integ]
    tgt = one if integ == 'PLAIN' else two
    betas, R, S, E, burn = [1.0, 0.6, 0.3, 0.1], 2, 14, 3, 3
    Tn = len(betas)
    C_ = R * Tn
    q0 = _q0(model, C_, scale=0.3)
    g = torch.Generator().manual_seed(21)
    z = torch.randn(S, C_, q0.shape[1], generator=g)
    lu = torch.log(torch.rand(S, C_, generator=g))
    rounds = engine.swap_rounds(S, E)
    lus = torch.log(torch.rand(rounds, R, Tn - 1, generator=g, dtype=torch.float64))
    eps = 0.01
    res = samplers.sample_chains(tgt, q0, num_samples=S, num_steps_per_sample=3, step_size=eps, burn=burn,
                                 integrator=integrator, rng='injected', normals=z, log_uniforms=lu, betas=betas,
                                 swap_every=E, swap_log_uniforms=lus)
    torch.cuda.synchronize()
    o = TO.sample_tempered(tgt, betas, q0, S, 3, eps, burn, E, z, lu, lus.numpy(), split_scheme=osch)
    assert res.accepted.cpu().bool().tolist() == o['accepted']
    assert np.array_equal(res.swap_accepted.cpu().numpy(), o['swap_accepted'])
    assert (res.swap_accepted == 1).any() and (res.swap_accepted == 0).any()
    np.testing.assert_allclose(res.swap_ll.cpu().numpy(), o['swap_ll'], rtol=LL_RTOL, atol=1e-3)
    np.testing.assert_allclose(res.samples.cpu().numpy(), o['samples'].numpy(), rtol=MLP_RTOL, atol=MLP_RTOL)
    np.testing.assert_allclose(res.final_state.cpu().numpy(), o['final'].numpy(), rtol=MLP_RTOL, atol=MLP_RTOL)
    _check_decisions(res, betas, lus.numpy())


def test_philox_decisions_follow_the_rule():
    model, one, _ = _problem('reg')
    betas, R, seed, off = [1.0, 0.5, 0.25, 0.1, 0.0], 3, 77, 10
    res = samplers.sample_chains(one, _q0(model, R * 5, scale=0.3), num_samples=25, num_steps_per_sample=3,
                                 step_size=0.01, burn=5, betas=betas, swap_every=4, seed=seed, chain_offset=off)
    rounds = res.swap_accepted.shape[0]
    k, r, t = np.meshgrid(np.arange(rounds), off // 5 + np.arange(R), np.arange(4), indexing='ij')
    w = P.draw(seed, r.astype(np.uint64), k.astype(np.uint64), t.astype(np.uint64), STREAM_SWAP)[..., 0]
    _check_decisions(res, betas, np.log(P.u01(w).astype(np.float64)))
    rate = (res.swap_accepted == 1).sum(dim=(0, 1)).double() / (res.swap_accepted >= 0).sum(dim=(0, 1)).double()
    assert torch.equal(res.swap_rate, rate) and res.betas.tolist() == betas


# ------------------------------------------------------------------------------------------------------------------
# 5. Philox: the injected twin, and ladder sharding
# ------------------------------------------------------------------------------------------------------------------
def _philox_swap_stream(seed, ladder0, rounds, R, Tn):
    k, r, t = np.meshgrid(np.arange(rounds), ladder0 + np.arange(R), np.arange(Tn - 1), indexing='ij')
    w = P.draw(seed, r.astype(np.uint64), k.astype(np.uint64), t.astype(np.uint64), STREAM_SWAP)[..., 0]
    return torch.from_numpy(np.log(P.u01(w).astype(np.float64)))


@pytest.mark.parametrize('integ', ['PLAIN', 'SPLITTING_RAND'])
def test_philox_equals_the_injected_twin(integ):
    model, one, two = _problem('reg')
    integrator, _ = INTEGRATORS[integ]
    tgt = one if integ == 'PLAIN' else two
    betas, R, S, E, seed, off = [1.0, 0.4, 0.1], 2, 15, 4, 123, 6
    Tn = len(betas)
    C_ = R * Tn
    q0 = _q0(model, C_, scale=0.3)
    kw = dict(num_samples=S, num_steps_per_sample=3, step_size=0.01, burn=3, integrator=integrator, betas=betas,
              swap_every=E, chain_offset=off)
    ph = samplers.sample_chains(tgt, q0, seed=seed, **kw)
    s = _stream(seed, off, C_, S, q0.shape[1], M=2 if integ != 'PLAIN' else 0)
    lus = _philox_swap_stream(seed, off // Tn, engine.swap_rounds(S, E), R, Tn)
    inj = samplers.sample_chains(tgt, q0, rng='injected', swap_log_uniforms=lus, **s, **kw)
    torch.cuda.synchronize()
    assert _same(ph.samples, inj.samples) and _same(ph.accepted, inj.accepted)
    assert torch.equal(ph.swap_accepted, inj.swap_accepted) and torch.equal(ph.swap_ll, inj.swap_ll)
    assert _same(ph.final_state, inj.final_state)
    assert (ph.swap_accepted == 1).any()


def test_results_do_not_depend_on_ladder_sharding():
    model, one, _ = _problem('reg')
    tgt = _pin(one, 1)
    betas, R = [1.0, 0.5, 0.2], 2
    Tn = len(betas)
    q0 = _q0(model, 2 * R * Tn, scale=0.3)
    kw = dict(num_samples=20, num_steps_per_sample=3, step_size=0.01, burn=4, betas=betas, swap_every=3, seed=5,
              sampler=samplers.Sampler.HMC_NUTS)
    whole = samplers.sample_chains(tgt, q0, **kw)
    parts = [samplers.sample_chains(tgt, q0[o:o + R * Tn], chain_offset=o, **kw) for o in (0, R * Tn)]
    torch.cuda.synchronize()
    assert _same(whole.samples, torch.cat([p.samples for p in parts]))
    assert _same(whole.final_state, torch.cat([p.final_state for p in parts]))
    assert torch.equal(whole.swap_accepted, torch.cat([p.swap_accepted for p in parts], dim=1))
    assert torch.equal(whole.swap_ll, torch.cat([p.swap_ll for p in parts], dim=1))


# ------------------------------------------------------------------------------------------------------------------
# 6. conjugate check: Bayesian linear regression, every rung against its closed-form tempered posterior
# ------------------------------------------------------------------------------------------------------------------
def test_rungs_sample_the_tempered_gaussian_posteriors():
    g = torch.Generator().manual_seed(8)
    n, d, tau_out = 40, 5, 4.0
    x = torch.randn(n, d, generator=g)
    y = x @ torch.randn(d, 1, generator=g) + 0.3 + 0.5 * torch.randn(n, 1, generator=g)
    model = torch.nn.Linear(d, 1)
    tgt = T.MLPTarget.from_model(model, x, y, None, tau_out)
    betas, R = [1.0, 0.3, 0.1, 0.03], 64
    Tn = len(betas)
    q0 = 0.5 * torch.randn(R * Tn, d + 1, generator=g)
    res = samplers.sample_chains(tgt, q0, num_samples=1500, num_steps_per_sample=10, step_size=0.05, burn=300,
                                 sampler=samplers.Sampler.HMC_NUTS, betas=betas, swap_every=5, seed=42, moments=True,
                                 keep_samples=False)
    torch.cuda.synchronize()
    X = torch.cat([x, torch.ones(n, 1)], 1).double()
    cnt = res.moment_count
    m = (res.moment_sum / cnt).cpu()
    v = (res.moment_sumsq / cnt).cpu() - m * m
    for t, b in enumerate(betas):
        prec = torch.eye(d + 1, dtype=torch.float64) + b * tau_out * X.T @ X
        cov = torch.linalg.inv(prec)
        mean = cov @ (b * tau_out * X.T @ y.double()).reshape(-1)
        mt, vt = m[t::Tn], v[t::Tn]
        z_mean = (mt.mean(0) - mean) / (mt.std(0) / math.sqrt(R))
        pooled_var = vt.mean(0) + mt.var(0, unbiased=False)
        z_var = (pooled_var - cov.diagonal()) / (vt.std(0) / math.sqrt(R))
        assert bool((z_mean.abs() < 4.5).all()), (t, z_mean)
        assert bool((z_var.abs() < 4.5).all()), (t, z_var)
    assert bool((res.swap_rate > 0.1).all()), res.swap_rate


# ------------------------------------------------------------------------------------------------------------------
# 7. what the feature is for: the sign-symmetric modes of a 1-1-1 tanh network
# ------------------------------------------------------------------------------------------------------------------
BIMODAL_BETAS = [1.0, 0.5, 0.25, 0.12, 0.06, 0.03, 0.015, 0.007, 0.0035, 0.0015, 0.0]


def bimodal_problem():
    """y = tanh(2x) + noise at tau_out = 100: (w1, b1, w2, b2) and (-w1, -b1, -w2, b2) fit equally, and w2 = 0 (a
    constant network) costs ~1000 nats."""
    g = torch.Generator().manual_seed(0)
    x = torch.linspace(-2, 2, 32).reshape(-1, 1)
    y = torch.tanh(2 * x) + 0.1 * torch.randn(32, 1, generator=g)
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(1, 1), torch.nn.Tanh(), torch.nn.Linear(1, 1))
    tgt = T.MLPTarget.from_model(model, x, y, None, 100.0)
    return tgt


def bimodal_runs(R=16, S=3000, burn=500, seed=3):
    tgt = bimodal_problem()
    Tn = len(BIMODAL_BETAS)
    kw = dict(num_samples=S, num_steps_per_sample=10, step_size=0.02, burn=burn, sampler=samplers.Sampler.HMC_NUTS)
    q0 = torch.randn(R * Tn, 4, generator=torch.Generator().manual_seed(seed))
    plain = samplers.sample_chains(tgt, q0[::Tn], seed=seed, **kw)
    temp = samplers.sample_chains(tgt, q0, seed=seed, betas=BIMODAL_BETAS, swap_every=2, **kw)
    torch.cuda.synchronize()
    return plain, temp


def test_tempering_crosses_the_modes_plain_chains_cannot():
    plain, temp = bimodal_runs()
    w2p = plain.samples[:, 1:, 2].cpu()
    side = (w2p > 0).double().mean(1)
    assert bool(((side >= 0.99) | (side <= 0.01)).all()), side
    w2t = temp.samples[:, 1:, 2].cpu()
    share = float((w2t > 0).double().mean())
    assert 0.35 <= share <= 0.65, share
    crossed = ((w2t[:, 1:] > 0) != (w2t[:, :-1] > 0)).any(1)
    assert bool(crossed.all()), crossed


# ------------------------------------------------------------------------------------------------------------------
# 8. sink options and consumers
# ------------------------------------------------------------------------------------------------------------------
def test_sink_options_equal_post_processing():
    model, one, _ = _problem('reg')
    betas, R = [1.0, 0.5, 0.2], 3
    Tn = len(betas)
    q0 = _q0(model, R * Tn, scale=0.3)
    kw = dict(num_samples=25, num_steps_per_sample=3, step_size=0.01, burn=4, betas=betas, swap_every=3, seed=13)
    base = samplers.sample_chains(one, q0, **kw)
    thin = samplers.sample_chains(one, q0, thin=3, **kw)
    mom = samplers.sample_chains(one, q0, moments=True, keep_samples=False, **kw)
    host = samplers.sample_chains(one, q0, store_on_GPU=False, **kw)
    ld = base.samples_padded.shape[-1]
    out = torch.zeros(R, base.samples.shape[1], ld, device='cuda')
    into = samplers.sample_chains(one, q0, out=out, **kw)
    torch.cuda.synchronize()
    assert base.samples.shape == (R, 21, q0.shape[1])
    assert _same(thin.samples, base.samples[:, ::3])
    assert not host.samples.is_cuda and _same(host.samples, base.samples)
    assert into.samples_padded.data_ptr() == out.data_ptr() and _same(into.samples, base.samples)
    cold = base.samples[:, 1:].double()
    np.testing.assert_allclose(mom.moment_sum[::Tn].cpu().numpy(), cold.sum(1).cpu().numpy(), rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(mom.moment_sumsq[::Tn].cpu().numpy(), (cold ** 2).sum(1).cpu().numpy(), rtol=1e-6,
                               atol=1e-6)
    assert mom.moment_sum.shape[0] == R * Tn and _same(mom.final_state, base.final_state)
    assert _same(mom.swap_accepted, base.swap_accepted)


def test_consumers_take_the_result():
    model, one, _ = _problem('reg')
    betas, R = [1.0, 0.5], 4
    q0 = _q0(model, R * 2, scale=0.3)
    res = samplers.sample_chains(one, q0, num_samples=40, num_steps_per_sample=3, step_size=0.01, burn=5, betas=betas,
                                 swap_every=5, seed=3)
    torch.cuda.synchronize()
    a, b = diagnostics.summary(res), diagnostics.summary(res.samples)
    assert torch.equal(a.rhat, b.rhat) and torch.equal(a.ess, b.ess)
    a, b = diagnostics.rank_summary(res), diagnostics.rank_summary(res.samples)
    assert torch.equal(a.rhat, b.rhat)
    la, lb = loo.psis_loo(res, one), loo.psis_loo(res.samples, one)
    assert la.elpd_loo == lb.elpd_loo
    wa, wb = loo.waic(res, one), loo.waic(res.samples, one)
    assert wa.elpd_waic == wb.elpd_waic
    pa, pb = predictive.evaluate(res, one), predictive.evaluate(res.samples, one)
    assert pa.rmse == pb.rmse and pa.nll == pb.nll
