"""GPU: diagonal-mass adaptation during HMC_NUTS warm-up (sample_chains(adapt_mass=True), DESIGN §3.13).

The element-wise kernel is pinned bit for bit to tests/adapt_oracle.py under the injected stream with the oracle's step
sizes teacher-forced (eps_schedule): accept decisions, samples and every window's inv_mass; the kernel's own restarted dual
averaging (eps_trace) within the NUTS tolerance.  The Bayesian-NN kernel within the Bayesian-NN tolerances.  Philox mode
against its injected twin, the reduction kernel alone against the estimator, and the statistics the feature exists for."""
import ctypes as C

import numpy as np
import pytest
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import engine, targets as T, _native as N
from oracle import cases, hmc_oracle as O
from tests import adapt_oracle as A, parity
from tests.test_philox_stream_gpu import _philox_vs_injected

pytestmark = pytest.mark.gpu
MLP_RTOL = 2e-4               # tests/test_mlp_gpu.py


def _streams(C_, D, S, seed0, prior):
    inits, zs, lus = [], [], []
    for c in range(C_):
        init, z, logu, _ = O.reference_stream(seed0 + c, D, S, prior=prior)
        inits.append(init), zs.append(z), lus.append(logu)
    return torch.stack(inits), torch.stack(zs, 1), torch.stack(lus, 1)


def _check_parity(res, o, lus, burn, exact, rtol=0.0):
    torch.cuda.synchronize()
    for c in range(res.accepted.shape[0]):
        parity.assert_chain_parity(res.samples[c].cpu().numpy(), res.accepted[c].cpu().numpy(), res.ham[c].cpu().numpy(),
                                   o['samples'][c].numpy(), o['accepted'][c], o['ham_old'][c], o['ham_new'][c],
                                   lus[:, c].numpy(), burn, exact=exact, rtol=rtol)
        # the kernel's own restarted dual averaging: the oracle's, restarted from the kernel's step size at each window end
        own = res.eps_trace[c].cpu().numpy().astype(np.float64)
        ref = A.replay_step_sizes(o['rho'][c], burn, o['step_sizes'][c][0], lambda b: float(own[b - 1]))
        tol = parity.nuts_eps_rtol(max(abs(h) for h in o['ham_old'][c]))
        np.testing.assert_allclose(own[:burn + 1], ref, rtol=tol)
        np.testing.assert_allclose(ref[:-1], np.array(o['step_sizes'][c])[1:burn + 1], rtol=tol * 4)


# D = 6 and 37: <E=4, K=1, 256> with dead pad lanes; D = 1024: a full 256-thread CTA
@pytest.mark.parametrize('D', [6, 37, 1024])
def test_elementwise_parity_with_the_oracle(D):
    C_, S, L, burn, eps0 = 3, 215, 4, 200, 0.3          # windows [75, 100), [100, 150)
    g = torch.Generator().manual_seed(D)
    sd = torch.logspace(-1, 0, D)
    tgt = T.GaussianDiag(torch.randn(D, generator=g), sd ** 2)
    init, z, lu = _streams(C_, D, S, 10 * D, lambda: tgt.mean + 0.5 * torch.randn(D))
    im0 = 0.5 + torch.rand(D, generator=g)
    o = A.sample_adapted(tgt, init, S, L, eps0, burn, inv_mass=im0, normals=z, log_uniforms=lu)
    sched = torch.tensor(o['step_sizes'], dtype=torch.float32).t()
    res = engine.hmc_run(tgt, init, S, L, eps0, burn=burn, inv_mass=im0, nuts=True, normals=z, log_uniforms=lu,
                         record_ham=True, eps_schedule=sched, record_eps=True, adapt_mass=True)
    _check_parity(res, o, lu, burn, exact=True)
    assert res.mass_windows == o['windows'] == [(75, 100), (100, 150)]
    assert np.array_equal(res.inv_mass_trace.cpu().numpy(), o['inv_mass_trace'])
    assert torch.equal(res.inv_mass, res.inv_mass_trace[-1])


@pytest.mark.parametrize('scheme', [None, 'SPLITTING'])
def test_bayesian_nn_parity_with_the_oracle(scheme):
    C_, S, L, burn, eps0 = 2, 26, 3, 20, 0.004           # one window, [3, 18)
    model, x, y = cases.mlp_problem(seed=5, n=96, n_in=5, hidden=12)
    if scheme is None:
        tgt = T.MLPTarget.from_model(model, x, y, None, 20.)
        kw, okw = dict(scheme=N.SCHEME_PLAIN), {}
    else:
        tgt = [T.MLPTarget.from_model(model, x[m * 48:(m + 1) * 48], y[m * 48:(m + 1) * 48], None, 20., prior_scale=2)
               for m in range(2)]
        kw, okw = dict(scheme=N.SCHEME_SPLIT_SYM), dict(split_scheme=O.SPLIT_SYM)
    D = hb.util.flatten(model).numel()
    init, z, lu = _streams(C_, D, S, 70, lambda: hb.util.flatten(model).detach() + 0.05 * torch.randn(D))
    o = A.sample_adapted(tgt, init, S, L, eps0, burn, normals=z, log_uniforms=lu, **okw)
    sched = torch.tensor(o['step_sizes'], dtype=torch.float32).t()
    res = engine.hmc_run(tgt, init, S, L, eps0, burn=burn, nuts=True, normals=z, log_uniforms=lu, record_ham=True,
                         eps_schedule=sched, record_eps=True, adapt_mass=True, **kw)
    _check_parity(res, o, lu, burn, exact=False, rtol=MLP_RTOL)
    np.testing.assert_allclose(res.inv_mass_trace.cpu().numpy(), o['inv_mass_trace'], rtol=1e-3, atol=1e-7)


@pytest.mark.parametrize('D,scheme', [(37, None), (1024, None), (0, 'PLAIN')])
def test_philox_equals_the_injected_twin(D, scheme):
    C_, S, L, burn = 4, 40, 4, 25                        # one window, [3, 22)
    if scheme is None:
        g = torch.Generator().manual_seed(D)
        tgt = T.GaussianDiag(torch.linspace(-1, 1, D), torch.logspace(-1, 0, D) ** 2)
        q0 = tgt.mean + 0.3 * torch.randn(C_, D, generator=g)
        kw, eps0 = {}, 0.3
    else:
        model, x, y = cases.mlp_problem(seed=3, n=64, n_in=4, hidden=8)
        tgt = T.MLPTarget.from_model(model, x, y, None, 20.)
        D = hb.util.flatten(model).numel()
        q0 = hb.util.flatten(model).detach()[None] + 0.05 * torch.randn(C_, D, generator=torch.Generator().manual_seed(1))
        kw, eps0 = dict(scheme=N.SCHEME_PLAIN), 0.004

    def run(**rng):
        return engine.hmc_run(tgt, q0, S, L, eps0, burn=burn, nuts=True, record_ham=True, record_eps=True,
                              adapt_mass=True, thin=2, moments=True, **kw, **rng)
    ph = _philox_vs_injected(run, 77, 5, C_, S, D)
    assert ph.inv_mass.shape == (D,) and bool(torch.isfinite(ph.inv_mass).all())


def _adapt_call(sums, n, eps, ld, D):
    Cn, Ce = sums[0].shape[0], eps.shape[0]
    dev = sums[0].device
    im, mf = torch.full((ld,), float('nan'), device=dev), torch.full((ld,), float('nan'), device=dev)
    # one guard entry past the C_chains restarted chains: the kernel must not write it
    mu, hb_, eb = (torch.full((Ce + 1,), float('nan'), dtype=torch.float64, device=dev) for _ in range(3))
    lib = N.load_library()
    rc = lib.hmcx_adapt_diag_mass(*(N.ptr(t) for t in sums), Cn, ld, D, n, N.ptr(eps), Ce, N.ptr(im), N.ptr(mf), N.ptr(mu),
                                  N.ptr(hb_), N.ptr(eb), N.stream_ptr(dev))
    N.check(rc, 'hmcx_adapt_diag_mass')
    torch.cuda.synchronize()
    return im, mf, mu, hb_, eb


# C_chains < C: sums gathered from every device, this device restarting its own chains (a few, or more than ld of them)
@pytest.mark.parametrize('C_,D,mean,C_chains', [(3, 5, 0.0, 3), (256, 1024, 0.0, 256), (64, 300, 1e3, 64),
                                                (7, 4093, -50.0, 7), (9, 37, 2.0, 4), (700, 6, 0.0, 350)])
def test_reduction_kernel_matches_the_estimator_bitwise(C_, D, mean, C_chains):
    """Random per-chain sums of n draws (built with the sink's compensated arithmetic), |mean| >> std included."""
    n = 40
    ld = N.padded_ld(D)
    rng = np.random.default_rng(C_ + D)
    scale = np.exp(rng.uniform(-3, 1, D))
    acc = [np.zeros((C_, ld), np.float32) for _ in range(4)]
    for c in range(C_):
        s = A.Sums(D)
        for row in (mean + scale * rng.standard_normal((n, D))).astype(np.float32):
            s.add(row)
        for a, f in zip(acc, ('s', 'q', 'c', 'cq')):
            a[c, :D] = getattr(s, f)
    sums = [torch.from_numpy(a).cuda() for a in acc]
    eps = torch.from_numpy(rng.uniform(0.01, 0.5, C_chains).astype(np.float32)).cuda()
    im, mf, mu, hb_, eb = _adapt_call(sums, n, eps, ld, D)
    assert all(bool(torch.isnan(t[-1])) for t in (mu, hb_, eb))
    mu, hb_, eb = mu[:-1], hb_[:-1], eb[:-1]
    ref_im, ref_mf = A.pooled_inv_mass(*(a[:, :D] for a in acc), n)
    assert np.array_equal(im[:D].cpu().numpy(), ref_im) and np.array_equal(mf[:D].cpu().numpy(), ref_mf)
    assert float(im[D:].abs().sum()) == 0 and float(mf[D:].abs().sum()) == 0
    assert all(float(t.abs().sum()) == 0 for t in sums)                     # zeroed for the next window
    assert mu.cpu().tolist() == [A.restart_mu(e) for e in eps.cpu().tolist()]
    assert bool((hb_ == 0).all()) and bool((eb == 1).all())
    # the factor is the one engine.NativeMass builds from the same inv_mass
    nm = engine.NativeMass(im[:D].clone(), D, 'cuda')
    assert torch.equal(nm._keep['sd'], mf[:D])
    # the estimate itself: |mean| >> std costs nothing -- the pooled variance within sampling error of scale^2
    assert np.all(np.abs(ref_im / scale ** 2 - 1) < 8 / np.sqrt(C_ * n) + 0.05 + 1e-3 / scale ** 2)


def test_pooled_branch_with_a_gather_hook_equals_the_oracle_on_the_gathered_chains():
    """engine.hmc_run(mass_pool=...) -- the multi-GPU branch: the reduction over the gathered sums (C_sums = 2C != C_chains
    = C) and the zeroing of the local accumulators after it.  The hook stands for a second device whose chains are copies
    of this one's (same start, same injected stream), so the run must equal the oracle over those 2C chains: its first C
    chains bit for bit, and its pooled mass of every window."""
    D, C_, S, L, burn, eps0 = 37, 2, 215, 4, 200, 0.3          # windows [75, 100), [100, 150)
    g = torch.Generator().manual_seed(11)
    tgt = T.GaussianDiag(torch.randn(D, generator=g), torch.logspace(-1, 0, D) ** 2)
    init, z, lu = _streams(C_, D, S, 500, lambda: tgt.mean + 0.5 * torch.randn(D))
    o = A.sample_adapted(tgt, torch.cat([init, init]), S, L, eps0, burn, normals=torch.cat([z, z], 1),
                         log_uniforms=torch.cat([lu, lu], 1))
    sched = torch.tensor(o['step_sizes'][:C_], dtype=torch.float32).t()
    res = engine.hmc_run(tgt, init, S, L, eps0, burn=burn, nuts=True, normals=z, log_uniforms=lu, record_ham=True,
                         eps_schedule=sched, record_eps=True, adapt_mass=True, mass_pool=lambda t: torch.cat([t, t]))
    _check_parity(res, {k: (v[:C_] if isinstance(v, list) and len(v) == 2 * C_ else v) for k, v in o.items()}, lu, burn,
                  exact=True)
    assert np.array_equal(res.inv_mass_trace.cpu().numpy(), o['inv_mass_trace'])


def test_adapted_mass_recovers_the_scales_and_raises_the_minimum_ess():
    """GaussianDiag with standard deviations log-spaced over 1e-2..1, D = 1024, C = 256, burn = 1000, S = 2000, L = 10."""
    D, C_, S, L, burn = 1024, 256, 2000, 10, 1000
    sd = torch.logspace(-2, 0, D)
    tgt = T.GaussianDiag(torch.zeros(D), sd ** 2)              # (mean, variance)
    q0 = 0.01 * torch.randn(C_, D, generator=torch.Generator().manual_seed(0))
    kw = dict(num_samples=S, num_steps_per_sample=L, step_size=0.01, burn=burn, sampler=hb.Sampler.HMC_NUTS,
              rng='philox', seed=3)
    plain = hb.sample_chains(tgt, q0, **kw)
    ad = hb.sample_chains(tgt, q0, adapt_mass=True, **kw)
    torch.cuda.synchronize()
    ratio = (ad.inv_mass.cpu().double() / sd.double() ** 2)
    print('inv_mass / sigma^2: min %.4f max %.4f' % (float(ratio.min()), float(ratio.max())))
    assert float((ratio - 1).abs().max()) <= 0.10
    ess_ad = hb.diagnostics.rank_summary(ad.samples[:, 1:]).ess_bulk.min()
    ess_plain = hb.diagnostics.rank_summary(plain.samples[:, 1:]).ess_bulk.min()
    print('min bulk-ESS: adapted %.1f, plain %.1f' % (float(ess_ad), float(ess_plain)))
    assert float(ess_ad) >= 5 * float(ess_plain)
