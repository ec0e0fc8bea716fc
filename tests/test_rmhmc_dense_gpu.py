"""GPU parity of the constant-metric RMHMC path (hmcx_rmhmc_dense_run: Gaussian targets, jitter=None, every flow a
tensor-core GEMM over all chains) against the live oracle -- which differentiates rm_hamiltonian by autograd through the
Hessian, eigh and the Cholesky solve exactly like the reference (oracle/rmhmc_oracle.py).

Tolerance: the kernel applies G^-1 as a matrix (3xTF32 GEMM), the reference solves two triangular systems per call:
fp32 evaluations of the same map with different expression trees -> states to RM_RTOL, identical accept decisions."""
import numpy as np
import pytest
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import engine, targets as T
from oracle import hmc_oracle as O, rmhmc_oracle as R
from tests import parity

pytestmark = pytest.mark.gpu
RM_RTOL = 2e-3            # CEILING only: per-quantity tolerances from measured errors (tests/parity.py)


def _full_gaussian(D, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(D, D, generator=g, dtype=torch.float64) / D ** 0.5
    cov = A @ A.t() + 0.5 * torch.eye(D, dtype=torch.float64)
    return T.GaussianFull(torch.randn(D, generator=g), cov=cov)


CASES = {
    'full40_softabs_explicit': dict(D=40, target='full', metric=R.SOFTABS, integrator=R.EXPLICIT, eps=0.9, L=3),
    'full24_hessian_implicit': dict(D=24, target='full', metric=R.HESSIAN, integrator=R.IMPLICIT, eps=0.6, L=3),
    'diag24_softabs_explicit': dict(D=24, target='diag', metric=R.SOFTABS, integrator=R.EXPLICIT, eps=1.2, L=3),
    'iso20_hessian_explicit': dict(D=20, target='iso', metric=R.HESSIAN, integrator=R.EXPLICIT, eps=0.8, L=3),
    # 3 and 4 register slots per lane of the persistent small-D kernel (64 < D <= 96, 96 < D <= 128)
    'full72_hessian_explicit': dict(D=72, target='full', metric=R.HESSIAN, integrator=R.EXPLICIT, eps=0.5, L=3),
    'full100_softabs_implicit': dict(D=100, target='full', metric=R.SOFTABS, integrator=R.IMPLICIT, eps=0.5, L=2),
}


@pytest.mark.parametrize('path', ['flow', 'tcgen05'])
@pytest.mark.parametrize('name', sorted(CASES))
def test_constant_metric_rmhmc_parity_vs_live_oracle(name, path, monkeypatch):
    # D <= 128: the persistent small-D kernel (hmcx_flow.cu, exact fp32 FMAs) by default; HMCX_FLOW_SMALL=0 keeps the
    # step-synchronous tensor-core GEMM path (the default above D = 128) under the same test
    monkeypatch.setenv('HMCX_FLOW_SMALL', '1' if path == 'flow' else '0')
    cs = CASES[name]
    D, S, burn, C = cs['D'], 6, 2, 3
    if cs['target'] == 'full':
        tgt = _full_gaussian(D, 31)
    elif cs['target'] == 'diag':
        g = torch.Generator().manual_seed(32)
        tgt = T.GaussianDiag(torch.randn(D, generator=g), 0.4 + torch.rand(D, generator=g))
    else:
        tgt = T.GaussianIso(D)
    alpha, omega = 1.0, 10.0
    mean = getattr(tgt, 'mean', None)
    inits, zs, lus = [], [], []
    for seed in range(C):
        init, z, logu, _ = O.reference_stream(1200 + seed, D, S,
                                              prior=lambda: (0 if mean is None else mean) + 0.5 * torch.randn(D))
        inits.append(init), zs.append(z), lus.append(logu)
    os_ = [R.sample_rmhmc(tgt, inits[c], num_samples=S, num_steps_per_sample=cs['L'], step_size=cs['eps'], burn=burn,
                          jitter=None, softabs_const=alpha, explicit_binding_const=omega, integrator=cs['integrator'],
                          metric=cs['metric'], normals=zs[c], log_uniforms=lus[c]) for c in range(C)]
    res = engine.rmhmc_run(tgt, torch.stack(inits), S, cs['L'], cs['eps'], burn=burn, jitter=None, softabs_const=alpha,
                           explicit_binding_const=omega, explicit=cs['integrator'] == R.EXPLICIT,
                           softabs=cs['metric'] == R.SOFTABS, normals=torch.stack(zs, 1),
                           log_uniforms=torch.stack(lus, 1), record_ham=True)
    torch.cuda.synchronize()
    assert int(res.diverged.sum()) == 0
    n_acc = 0
    for c in range(C):
        o = os_[c]
        assert not any(o['diverged'])
        ham = res.ham[c].cpu().numpy().astype(np.float64)
        tag = 'rmhmc_const/%s/%s/c%d' % (name, path, c)            # tolerance = 8 x the measured error (tests/parity.py)
        parity.assert_close(tag + '/ham_old', ham[:, 0], np.array(o['ham_old']), RM_RTOL)
        parity.assert_close(tag + '/ham_new', ham[:, 1], np.array(o['ham_new']), RM_RTOL)
        m = parity.first_decision_mismatch(res.accepted[c].cpu().numpy(), o['accepted'])
        assert m is None, 'accept decision differs at iteration %d' % m
        parity.assert_close(tag + '/samples', res.samples[c].cpu().numpy(), torch.stack(o['samples']).numpy(), RM_RTOL)
        n_acc += sum(o['accepted'])
    assert n_acc > 0, 'fixture never accepts: it would not exercise the trajectory'


def test_sample_dropin_rmhmc_gaussian_full():
    """hb.sample(GaussianFull, sampler=RMHMC) is routed to the tensor-core path (one chain) and returns the reference's
    list shape."""
    D = 24
    tgt = _full_gaussian(D, 33)
    torch.manual_seed(5)
    out = hb.sample(tgt, tgt.mean.clone(), num_samples=8, num_steps_per_sample=3, step_size=0.15, burn=2,
                    sampler=hb.Sampler.RMHMC, integrator=hb.Integrator.EXPLICIT, metric=hb.Metric.HESSIAN,
                    explicit_binding_const=10, verbose=False)
    assert len(out) == 6 and out[0].shape == (D,) and torch.equal(out[0].cpu(), tgt.mean)
    assert all(torch.isfinite(t).all() for t in out)


@pytest.mark.parametrize('integrator', ['EXPLICIT', 'IMPLICIT'])
def test_flow_and_tcgen05_paths_agree_d64(integrator, monkeypatch):
    """Same Philox streams, same element-wise operation order: the two forms of the constant-metric explicit integrator give
    the same chains up to the summation order of the contractions (compared while the decisions agree)."""
    D, C, S, L = 64, 70, 6, 4
    tgt = _full_gaussian(D, 35)
    init = tgt.mean[None] + 0.5 * torch.randn(C, D, generator=torch.Generator().manual_seed(9))
    kw = dict(num_samples=S, num_steps_per_sample=L, step_size=0.2, explicit_binding_const=10, sampler=hb.Sampler.RMHMC,
              integrator=getattr(hb.Integrator, integrator), metric=hb.Metric.HESSIAN,
              rng='philox', seed=12, record_ham=True)
    monkeypatch.setenv('HMCX_FLOW_SMALL', '1')
    a = hb.sample_chains(tgt, init, **kw)
    monkeypatch.setenv('HMCX_FLOW_SMALL', '0')
    b = hb.sample_chains(tgt, init, **kw)
    torch.cuda.synchronize()
    assert torch.equal(a.accepted, b.accepted)
    assert torch.allclose(a.ham, b.ham, rtol=1e-4, atol=1e-3)
    assert torch.allclose(a.samples, b.samples, rtol=2e-4, atol=2e-4)
    assert 0 < int(a.accepted.sum())
    # chains per warp (1 / 2 / 4, picked from the batch size) never change a chain's bits
    monkeypatch.setenv('HMCX_FLOW_SMALL', '1')
    for r in ('1', '2', '4'):
        monkeypatch.setenv('HMCX_FLOW_R', r)
        c = hb.sample_chains(tgt, init, **kw)
        torch.cuda.synchronize()
        assert torch.equal(a.samples, c.samples) and torch.equal(a.ham, c.ham)


@pytest.mark.parametrize('path', ['flow', 'tcgen05'])
def test_constant_metric_rmhmc_philox_statistics_d64(path, monkeypatch):
    monkeypatch.setenv('HMCX_FLOW_SMALL', '1' if path == 'flow' else '0')
    """SURVEY 8d's 'D=64 Gaussian-Hessian variant' of config 3: 512 chains, explicit integrator, Hessian metric.  With
    G = P the dynamics are isotropic in the whitened space: high acceptance, second moment along a direction = cov."""
    D, C, S, L = 64, 512, 40, 6
    tgt = _full_gaussian(D, 34)
    cov = torch.linalg.inv(tgt.prec.double())
    Lc = torch.linalg.cholesky(cov)
    init = tgt.mean[None] + (torch.randn(C, D, dtype=torch.float64, generator=torch.Generator().manual_seed(7)) @ Lc.t()).float()
    res = hb.sample_chains(tgt, init, num_samples=S, num_steps_per_sample=L, step_size=0.2, explicit_binding_const=10,
                           sampler=hb.Sampler.RMHMC, integrator=hb.Integrator.EXPLICIT, metric=hb.Metric.HESSIAN,
                           rng='philox', seed=11, record_ham=True)
    torch.cuda.synchronize()
    assert int(res.diverged.sum()) == 0
    acc = res.accepted.float().mean().item()
    assert 0.7 < acc <= 1.0, acc
    u = torch.randn(D, dtype=torch.float64, generator=torch.Generator().manual_seed(8))
    u /= u.norm()
    proj = ((res.samples[:, S // 2:].cpu().double() - tgt.mean.double()) @ u)
    assert abs(proj.var().item() / float(u @ cov @ u) - 1.0) < 0.1
