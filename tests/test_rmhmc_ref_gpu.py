"""GPU: the in-kernel-metric RMHMC kernels against the fp64 per-iteration replay of tests/rmhmc_ref.py, at every
dimension class, odd D and all three metrics.

  rmhmc2_quad_kernel       D = 2, explicit: C = 33 (a partly filled CTA of 32-chain lanes)
  rmhmc_run_kernel<DM>     one thread per chain: DM = 2 (D = 2 implicit), 6 (D = 1, 6 at capacity, C = 130: a partly
                           filled 128-thread block), 16 (D = 7, 11, 13, 16)
  rmhmc_cta_kernel         one CTA per chain, D <= 64: odd D (the round-robin's dummy player) 17, 31, 33, 47, 63; a
                           dense 64 x 64 metric (Jacobi rotations at full size); C = 300 (several waves); and, forced by
                           HMCX_RMHMC_FORCE_CTA=1, the small D of the thread kernels

Every case runs the kernel on injected streams, replays each checked chain iteration by iteration in fp64 from the
kernel's own retained rows (dense_ref.replay), and holds Hamiltonians and proposals to 2e-4 (ten times tighter than
the golden-chain ceiling RM_RTOL) under the measured tolerances of tests/golden/measured_errors.json (rmhmc_ref/...).
Burn-in is >= 1 and every fifth chain is forced to reject (log u > 0) at the burn-in iteration and after it.  Implicit
cases run fixed_point_threshold = 0 with a few fixed-point iterations, so neither side exits a fixed point early and
both consume the same 3 + L (2m + 2) jitter rows; they also give every chain its own step size.
"""
import os
import time

import pytest
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import engine, targets as T
from oracle import rmhmc_oracle as R
from tests import dense_ref, parity, rmhmc_ref

pytestmark = pytest.mark.gpu
CEIL = 2e-4
_REPLAY_SECONDS = []


@pytest.fixture(scope='module', autouse=True)
def _report_replay_time():
    yield
    print('\nrmhmc_ref: fp64 replay time %.1f s over %d runs' % (sum(_REPLAY_SECONDS), len(_REPLAY_SECONDS)))


def _full(D, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(D, D, generator=g, dtype=torch.float64) / D ** 0.5
    return T.GaussianFull(0.3 * torch.randn(D, generator=g), cov=A @ A.t() + 0.5 * torch.eye(D, dtype=torch.float64))


def _diag(D, seed):
    g = torch.Generator().manual_seed(seed)
    return T.GaussianDiag(torch.linspace(-1, 1, D), 0.25 + 1.5 * torch.rand(D, generator=g))


def _case(target, metric, jitter, alpha=None, explicit=True, C=3, S=4, L=2, burn=1, eps=0.05, m=6, replay=None,
          force_cta=False):
    return dict(target=target, metric=metric, jitter=jitter, alpha=alpha, explicit=explicit, C=C, S=S, L=L, burn=burn,
                eps=eps, m=m, replay=replay, force_cta=force_cta)


def _cases():
    F, SA, HE, JD = T.Funnel, 'SOFTABS', 'HESSIAN', 'JACOBIAN_DIAG'
    c = {
        # ---- rmhmc_run_kernel<DM>: one thread per chain
        'thread_iso1_hessian_jitter': _case(T.GaussianIso(1), HE, 1e-2, C=4, S=5, L=3, eps=0.3),
        'thread_full2_implicit_jitter': _case(_full(2, 6), SA, 1e-3, 1.0, explicit=False, S=5, L=3, eps=0.2),
        'thread_full6_softabs_jitter_c130': _case(_full(6, 1), SA, 1e-2, 1.0, C=130, L=3, eps=0.2,
                                                  replay=[0, 1, 64, 127, 128, 129]),
        'thread_funnel7_softabs_jitter': _case(F(7), SA, 1e-3, 1e6, L=3),
        'thread_full16_hessian_jitter': _case(_full(16, 2), HE, 1e-2, L=3, eps=0.2),
        'thread_funnel11_implicit_jitter': _case(F(11), SA, 1e-3, 1e6, explicit=False),
        'thread_jacdiag13_explicit': _case(F(13), JD, 1e-2, L=3, eps=0.03),
        # ---- rmhmc2_quad_kernel: BASELINE config 3's alpha, omega (= 10 below), eps, L and jitter, C = 33
        'quad_full2_c33': _case(_full(2, 7), SA, 1e-3, 1e6, C=33, L=10, eps=0.05, replay=[0, 5, 31, 32]),
        # ---- rmhmc_cta_kernel
        'cta_funnel17_softabs': _case(F(17), SA, 1e-3, 1e6, C=2, eps=0.03),
        'cta_funnel63_softabs': _case(F(63), SA, 1e-3, 1e6, C=2, S=3, eps=0.03),
        'cta_full33_softabs_jitter': _case(_full(33, 3), SA, 1e-3, 1.0, C=2, S=3, eps=0.2),
        'cta_full64_hessian_jitter': _case(_full(64, 4), HE, 1e-3, C=2, S=3, eps=0.2),
        'cta_jacdiag31_explicit': _case(F(31), JD, 1e-2, C=2, S=3, eps=0.02),
        'cta_funnel47_implicit_jitter': _case(F(47), SA, 1e-3, 1e6, explicit=False, C=2, S=3, eps=0.03),
        'cta_jacdiag40_implicit': _case(_diag(40, 5), JD, None, explicit=False, C=2, S=3, eps=0.03),
        'cta_funnel33_alpha1': _case(F(33), SA, 1e-3, 1.0, C=2, S=3, eps=0.03),
        'cta_funnel17_c300': _case(F(17), SA, 1e-3, 1e6, C=300, S=3, eps=0.03, replay=[0, 131, 132, 263, 264, 299]),
        # ---- the CTA kernel forced at the thread kernels' sizes
        'force_cta_iso1_hessian_jitter': _case(T.GaussianIso(1), HE, 1e-2, C=4, S=5, L=3, eps=0.3, force_cta=True),
        'force_cta_full2_explicit': _case(_full(2, 7), SA, 1e-3, 1e6, L=5, force_cta=True),
        'force_cta_full3_implicit_jitter': _case(_full(3, 8), SA, 1e-3, 1.0, explicit=False, eps=0.2, force_cta=True),
        'force_cta_funnel7_alpha1': _case(F(7), SA, 1e-3, 1.0, force_cta=True),
        'force_cta_full16_hessian_jitter': _case(_full(16, 2), HE, 1e-2, eps=0.2, force_cta=True),
    }
    return c


CASES = _cases()


def _init(tgt, C, g, metric='SOFTABS'):
    D = tgt.dim
    if isinstance(tgt, T.Funnel) and metric == 'JACOBIAN_DIAG':
        # G = diag(g^2) + jitter: keep every gradient component, g_0 = -v/9 + (D-1)/2 (1 - e^v) + ... included, well away
        # from 0, or G has entries of the size of the jitter and H is ill-conditioned beyond what fp32 can follow
        x = (0.8 + 0.4 * torch.rand(C, D - 1, generator=g)) * torch.sign(torch.randn(C, D - 1, generator=g))
        return torch.cat([0.5 + 0.1 * torch.randn(C, 1, generator=g), x], 1)
    if isinstance(tgt, T.Funnel):
        return torch.cat([0.3 * torch.randn(C, 1, generator=g), 0.6 * torch.randn(C, D - 1, generator=g)], 1)
    mean = getattr(tgt, 'mean', torch.zeros(D))
    if isinstance(tgt, T.GaussianDiag):                      # JACOBIAN_DIAG without jitter: keep every g_i away from 0
        return mean[None] + 1.5 + 0.2 * torch.rand(C, D, generator=g)
    return mean[None] + 0.3 * torch.randn(C, D, generator=g)


@pytest.mark.parametrize('name', sorted(CASES))
def test_in_kernel_metric_vs_fp64_replay(name, monkeypatch):
    cs = CASES[name]
    if cs['force_cta']:
        monkeypatch.setenv('HMCX_RMHMC_FORCE_CTA', '1')
    else:
        monkeypatch.delenv('HMCX_RMHMC_FORCE_CTA', raising=False)
    tgt, C, S, L, burn = cs['target'], cs['C'], cs['S'], cs['L'], cs['burn']
    D = tgt.dim
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    init = _init(tgt, C, g, cs['metric'])
    z = torch.randn(S, C, D, generator=g)
    logu = torch.log(torch.rand(S, C, generator=g))
    logu[burn::2, ::5] = 1.0                # > 0 >= rho: rejects at the burn-in iteration, burn + 2, ...
    if cs['explicit']:
        eps = torch.full((C,), cs['eps'])   # one binding rotation per launch: one step size (engine.rmhmc_run)
    else:
        eps = cs['eps'] * (0.8 + 0.4 * torch.rand(C, generator=g))
    J = rmhmc_ref.rows_per_iteration(cs['explicit'], L, cs['m'])
    uni = torch.rand(S, C, J, D, generator=g) if cs['jitter'] is not None else None
    res = engine.rmhmc_run(tgt, init.cuda(), S, L, eps.cuda(), burn=burn, jitter=cs['jitter'],
                           softabs_const=cs['alpha'], explicit_binding_const=10.0, fixed_point_threshold=0.0,
                           fixed_point_max_iterations=cs['m'], explicit=cs['explicit'], softabs=cs['metric'] == 'SOFTABS',
                           jacdiag=cs['metric'] == 'JACOBIAN_DIAG', normals=z.cuda(), log_uniforms=logu.cuda(),
                           uniforms=None if uni is None else uni.cuda(), record_ham=True)
    torch.cuda.synchronize()
    assert int(res.diverged.sum()) == 0
    idx = torch.tensor(cs['replay'] if cs['replay'] is not None else list(range(C)))
    acc, samples, ham = res.accepted.cpu()[idx], res.samples.cpu()[idx], res.ham.cpu()[idx]
    model = rmhmc_ref.InKernelMetric(tgt, cs['metric'], cs['jitter'], cs['alpha'], explicit=cs['explicit'], omega=10.0,
                                     threshold=0.0, max_iter=cs['m'], uniforms=None if uni is None else uni[:, idx])
    t0 = time.time()
    rep = dense_ref.replay(model, init[idx], acc, samples, z[:, idx], eps[idx], L, burn)
    _REPLAY_SECONDS.append(time.time() - t0)
    if uni is not None:
        assert bool((model.counts() == J).all()), 'the replay consumed other jitter rows than the kernel was given'
    dense_ref.check('rmhmc_ref/' + name, rep, init[idx], samples, acc, ham, logu[:, idx], burn, ceiling=CEIL)
    assert 0 < int(res.accepted.sum()) < C * S


# ---- stand-alone samplers.leapfrog / samplers.hamiltonian with sampler=RMHMC (the CTA kernel) -------------------------
STANDALONE = {
    'funnel17_explicit': dict(D=17, explicit=True, steps=3, eps=0.03),
    'funnel33_implicit': dict(D=33, explicit=False, steps=2, eps=0.03, m=4),
    'funnel63_explicit': dict(D=63, explicit=True, steps=2, eps=0.03),
}


@pytest.mark.parametrize('name', sorted(STANDALONE))
def test_standalone_leapfrog_and_hamiltonian_vs_fp64_oracle(name):
    s = STANDALONE[name]
    D, C, L, m = s['D'], 2, s['steps'], s.get('m', 6)
    tgt, jitter, alpha = T.Funnel(D), 1e-3, 1e6
    g = torch.Generator().manual_seed(D)
    q = _init(tgt, C, g)
    p = torch.randn(C, D, generator=g)
    J = 8 * L if s['explicit'] else L * (2 * m + 2)
    uni_h, uni_l = torch.rand(C, 1, D, generator=g), torch.rand(C, J, D, generator=g)
    integ = hb.Integrator.EXPLICIT if s['explicit'] else hb.Integrator.IMPLICIT
    kw = dict(jitter=jitter, softabs_const=alpha, sampler=hb.Sampler.RMHMC, integrator=integ, metric=hb.Metric.SOFTABS)
    H = hb.hamiltonian(q.cuda(), p.cuda(), tgt, explicit_binding_const=10.0, rng_uniforms=uni_h.cuda(), **kw)
    ret_q, ret_p = hb.leapfrog(q.cuda(), p.cuda(), tgt, steps=L, step_size=s['eps'], explicit_binding_const=10.0,
                               fixed_point_threshold=0.0, fixed_point_max_iterations=m, rng_uniforms=uni_l.cuda(), **kw)
    torch.cuda.synchronize()
    if s['explicit']:
        (qs, qc), (ps, pc) = ret_q, ret_p
    else:
        qs, ps = ret_q, ret_p
    t0 = time.time()
    want = {k: [] for k in ('H', 'q', 'p', 'q_copy', 'p_copy')}
    for c in range(C):
        q64, p64 = q[c].double(), p[c].double()
        jit = R.JitterSource(uni_h[c])
        h = float(R.rm_hamiltonian(q64, p64, tgt, jitter, alpha, R.SOFTABS, jit).detach())
        want['H'].append(2 * h if s['explicit'] else h)                     # the explicit integrator's H is doubled (:822)
        jit = R.JitterSource(uni_l[c])
        args = (tgt, jitter, alpha, R.SOFTABS, jit)
        if s['explicit']:
            cp = []
            oq, op = R.leapfrog_explicit(q64, p64, args, L, s['eps'], 10.0, copies=cp)
            want['q_copy'].append(cp[0].detach())
            want['p_copy'].append(cp[1].detach())
        else:
            oq, op = R.leapfrog_implicit(q64, p64, args, L, s['eps'], 0.0, m)
        assert jit.i == J and jit.retries == 0
        want['q'].append(torch.stack([x.detach() for x in oq]))
        want['p'].append(torch.stack([x.detach() for x in op]))
    _REPLAY_SECONDS.append(time.time() - t0)
    tag = 'rmhmc_ref/standalone_' + name
    parity.assert_close(tag + '/H', H.cpu().double().numpy(), torch.tensor(want['H']).numpy(), CEIL)
    parity.assert_close(tag + '/q', torch.stack(qs, 1).cpu().double().numpy(), torch.stack(want['q']).numpy(), CEIL)
    parity.assert_close(tag + '/p', torch.stack(ps, 1).cpu().double().numpy(), torch.stack(want['p']).numpy(), CEIL)
    if s['explicit']:
        parity.assert_close(tag + '/q_copy', qc.cpu().double().numpy(), torch.stack(want['q_copy']).numpy(), CEIL)
        parity.assert_close(tag + '/p_copy', pc.cpu().double().numpy(), torch.stack(want['p_copy']).numpy(), CEIL)
