"""GPU: the wgmma GEMM building block (3xTF32 split operands) against an fp64 reference."""
import pytest
import torch

from hamiltorch_b200 import engine

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('shape', [(128, 128, 32), (256, 384, 1024), (128, 1024, 96)])
def test_gemm_nt_tf32x3_is_fp32_accurate(shape):
    M, N, K = shape
    g = torch.Generator().manual_seed(M + N + K)
    A = torch.randn(M, K, generator=g).cuda()
    B = torch.randn(N, K, generator=g).cuda()
    D = engine.gemm_nt(A, B)
    torch.cuda.synchronize()
    ref = (A.double() @ B.double().t())
    err = (D.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    fp32 = ((A @ B.t()).double() - ref).abs().max().item()       # what a plain fp32 GEMM achieves
    # 3xTF32 (hi*hi + hi*lo + lo*hi, the lo*lo term dropped): 22 significant bits per operand -> a few times the
    # rounding error of a plain fp32 GEMM, three orders of magnitude below a single tf32 product (~1e-3 relative)
    assert err <= 2e-5 * scale, (err, fp32, scale)


def _corr_gaussian(D, seed):
    import hamiltorch_b200.targets as T
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(D, D, generator=g, dtype=torch.float64) / D ** 0.5
    cov = A @ A.t() + 0.5 * torch.eye(D, dtype=torch.float64)
    return T.GaussianFull(torch.randn(D, generator=g), cov=cov)


@pytest.mark.parametrize('D', [200, 96, 128])
@pytest.mark.parametrize('variant', ['hmc', 'diag_mass', 'nuts'])
def test_dense_gaussian_full_chain_parity_vs_live_oracle(variant, D):
    """Full-covariance Gaussian at D=200 (> 16: the tensor-core step-synchronous path, one GEMM over all chains per
    leapfrog step) against the oracle under the injected stream.  The gradient is a 3xTF32 tensor-core contraction
    (~1e-6 relative), the reference's an fp32 mv: states agree to 2e-4, decisions identical."""
    import numpy as np
    import hamiltorch_b200 as hb
    from hamiltorch_b200 import engine
    from oracle import hmc_oracle as O
    from tests import parity
    # D = 200: the tensor-core step-synchronous path; D = 96 / 128: the persistent small-D kernel (hmcx_flow.cu) with 3 / 4
    # register slots per lane
    C, S, L, burn = 5, 12, 6, 3
    tgt = _corr_gaussian(D, 1)
    im = None
    if variant == 'diag_mass':
        im = 0.5 + torch.rand(D, generator=torch.Generator().manual_seed(2))
    nuts = variant == 'nuts'
    eps0 = 0.1 if nuts else 0.25
    inits, zs, lus = [], [], []
    for seed in range(C):
        init, z, logu, _ = O.reference_stream(700 + seed, D, S, prior=lambda: tgt.mean + 0.3 * torch.randn(D))
        inits.append(init), zs.append(z), lus.append(logu)
    os_ = [O.sample_hmc(tgt, inits[c], num_samples=S, num_steps_per_sample=L, step_size=eps0, burn=burn, inv_mass=im,
                        nuts=nuts, normals=zs[c], log_uniforms=lus[c]) for c in range(C)]
    sched = torch.tensor([o['step_sizes'] for o in os_], dtype=torch.float32).t() if nuts else None
    res = engine.hmc_run(tgt, torch.stack(inits), S, L, eps0, burn=burn, inv_mass=im, nuts=nuts,
                         normals=torch.stack(zs, 1), log_uniforms=torch.stack(lus, 1), record_ham=True,
                         eps_schedule=sched, record_eps=nuts)
    torch.cuda.synchronize()
    assert int(res.diverged.sum()) == 0
    for c in range(C):
        o = os_[c]
        parity.assert_chain_parity(res.samples[c].cpu().numpy(), res.accepted[c].cpu().numpy(),
                                   res.ham[c].cpu().numpy(), torch.stack(o['samples']).numpy(), o['accepted'],
                                   o['ham_old'], o['ham_new'], lus[c].numpy(), burn, exact=False, rtol=2e-4,
                                   tag='dense_d%d/%s/c%d' % (D, variant, c))
        if nuts:
            own = res.eps_trace[c].cpu().numpy().astype(np.float64)
            np.testing.assert_allclose(own[:S - 1], np.array(o['step_sizes'])[1:], rtol=2e-3)


def test_dense_gaussian_full_philox_statistics_d1024():
    """256 chains of a D=1024 correlated Gaussian (the 'full-covariance ... becomes tensor-core work' regime of SURVEY
    8d): acceptance and energy errors of a working sampler; second moment along a random direction matches cov."""
    import hamiltorch_b200 as hb
    D, C, S, L = 1024, 256, 30, 8
    tgt = _corr_gaussian(D, 3)
    cov = torch.linalg.inv(tgt.prec.double())
    Lc = torch.linalg.cholesky(cov)
    init = tgt.mean[None] + (torch.randn(C, D, dtype=torch.float64, generator=torch.Generator().manual_seed(4)) @ Lc.t()).float()
    res = hb.sample_chains(tgt, init, num_samples=S, num_steps_per_sample=L, step_size=0.12, rng='philox', seed=5,
                           record_ham=True)
    torch.cuda.synchronize()
    assert int(res.diverged.sum()) == 0
    acc = res.accepted.float().mean().item()
    assert 0.6 < acc <= 1.0, acc
    u = torch.randn(D, dtype=torch.float64, generator=torch.Generator().manual_seed(6))
    u /= u.norm()
    proj = ((res.samples[:, S // 2:].cpu().double() - tgt.mean.double()) @ u)
    assert abs(proj.var().item() / float(u @ cov @ u) - 1.0) < 0.15


def _spd(D, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(D, D, generator=g, dtype=torch.float64) / D ** 0.5
    return (scale * (A @ A.t() + 0.7 * torch.eye(D, dtype=torch.float64))).float()


@pytest.mark.parametrize('D', [150, 96, 128])
@pytest.mark.parametrize('variant', ['full_target', 'diag_target', 'iso_target_nuts'])
def test_full_inv_mass_large_d_chain_parity_vs_live_oracle(variant, D):
    """2-D inv_mass at D > 16 (samplers.py:199 gibbs through the Cholesky factor of inverse(inv_mass), :294 drift
    q += eps*(M^-1 p), :812 kinetic): momentum refresh, every drift and both kinetic energies are tensor-core GEMMs over
    all chains (dense_lin_kernel), the gradient one more GEMM (GaussianFull) or element-wise (GaussianIso / Diag).
    3xTF32 contractions vs the reference's fp32 matmuls: states to 2e-4, identical decisions."""
    import numpy as np
    import hamiltorch_b200.targets as T
    from oracle import hmc_oracle as O
    from tests import parity
    C, S, L, burn = 4, 10, 5, 3            # D = 150: tensor-core GEMMs; D = 96 / 128: the persistent small-D kernel
    nuts = variant.endswith('nuts')
    if variant == 'full_target':
        tgt = _corr_gaussian(D, 11)
    elif variant == 'diag_target':
        g = torch.Generator().manual_seed(12)
        tgt = T.GaussianDiag(torch.randn(D, generator=g), 0.4 + torch.rand(D, generator=g))
    else:
        tgt = T.GaussianIso(D)
    im = _spd(D, 13)
    eps0 = 0.1 if nuts else 0.2
    mean = getattr(tgt, 'mean', None)
    inits, zs, lus = [], [], []
    for seed in range(C):
        init, z, logu, _ = O.reference_stream(900 + seed, D, S,
                                              prior=lambda: (0 if mean is None else mean) + 0.3 * torch.randn(D))
        inits.append(init), zs.append(z), lus.append(logu)
    os_ = [O.sample_hmc(tgt, inits[c], num_samples=S, num_steps_per_sample=L, step_size=eps0, burn=burn, inv_mass=im,
                        nuts=nuts, normals=zs[c], log_uniforms=lus[c]) for c in range(C)]
    sched = torch.tensor([o['step_sizes'] for o in os_], dtype=torch.float32).t() if nuts else None
    res = engine.hmc_run(tgt, torch.stack(inits), S, L, eps0, burn=burn, inv_mass=im, nuts=nuts,
                         normals=torch.stack(zs, 1), log_uniforms=torch.stack(lus, 1), record_ham=True,
                         eps_schedule=sched, record_eps=nuts)
    torch.cuda.synchronize()
    assert int(res.diverged.sum()) == 0
    assert 0 < int(res.accepted.sum()) and not torch.equal(res.samples[:, -1], res.samples[:, 0])
    for c in range(C):
        o = os_[c]
        parity.assert_chain_parity(res.samples[c].cpu().numpy(), res.accepted[c].cpu().numpy(),
                                   res.ham[c].cpu().numpy(), torch.stack(o['samples']).numpy(), o['accepted'],
                                   o['ham_old'], o['ham_new'], lus[c].numpy(), burn, exact=False, rtol=2e-4,
                                   tag='fullmass_d%d/%s/c%d' % (D, variant, c))
        if nuts:
            own = res.eps_trace[c].cpu().numpy().astype(np.float64)
            np.testing.assert_allclose(own[:S - 1], np.array(o['step_sizes'])[1:], rtol=2e-3)


def test_full_inv_mass_philox_statistics_d512():
    """Philox mode, 192 chains of N(0, I_512) preconditioned by a dense mass matrix: p ~ N(0, M) (kinetic energy
    p.(M^-1 p) averages D), healthy acceptance, unit marginal variance."""
    import hamiltorch_b200 as hb
    import hamiltorch_b200.targets as T
    D, C, S, L = 512, 192, 24, 6
    im = _spd(D, 21)
    init = torch.randn(C, D, generator=torch.Generator().manual_seed(22))
    res = hb.sample_chains(T.GaussianIso(D), init, num_samples=S, num_steps_per_sample=L, step_size=0.15,
                           inv_mass=im, rng='philox', seed=8, record_ham=True)
    torch.cuda.synchronize()
    assert int(res.diverged.sum()) == 0
    acc = res.accepted.float().mean().item()
    assert 0.6 < acc <= 1.0, acc
    # H_old at iteration 0 = -log p(init) + K0:  2*K0 ~ chi2_D
    lp0 = torch.stack([T.GaussianIso(D)(init[c]) for c in range(C)]).double()
    k0 = 2 * (res.ham[:, 0, 0].cpu().double() + lp0)
    assert abs(k0.mean().item() / D - 1.0) < 0.05, k0.mean().item()
    v = res.samples[:, S // 2:].cpu().double().var().item()
    assert abs(v - 1.0) < 0.1, v


@pytest.mark.parametrize('path', ['flow', 'tcgen05'])
def test_dense_paths_edge_shapes(path, monkeypatch):
    monkeypatch.setenv('HMCX_FLOW_SMALL', '1' if path == 'flow' else '0')
    """Ragged shapes on the tensor-core paths: D = 17 (the smallest dense dimension, padded to one 32-wide K chunk),
    C = 130 chains (two 128-row tiles, the second almost empty), one iteration, and D = 33 (two chunks, last nearly empty):
    chain c of the big launch equals the same chain launched alone (rows never interact), decisions equal the oracle's."""
    import hamiltorch_b200.targets as T
    from oracle import hmc_oracle as O
    for D, C in ((17, 130), (33, 3)):
        tgt = _corr_gaussian(D, 50 + D)
        im = _spd(D, 60 + D)
        S, L = 3, 4
        g = torch.Generator().manual_seed(D)
        init = tgt.mean[None] + 0.3 * torch.randn(C, D, generator=g)
        z = torch.randn(S, C, D, generator=g)
        logu = torch.log(torch.rand(S, C, generator=g))
        for mass in (None, im):
            res = engine.hmc_run(tgt, init, S, L, 0.2, inv_mass=mass, normals=z, log_uniforms=logu, record_ham=True)
            torch.cuda.synchronize()
            for c in (0, C - 1):
                one = engine.hmc_run(tgt, init[c:c + 1], S, L, 0.2, inv_mass=mass, normals=z[:, c:c + 1],
                                     log_uniforms=logu[:, c:c + 1], record_ham=True)
                torch.cuda.synchronize()
                assert torch.equal(one.samples[0], res.samples[c]) and torch.equal(one.accepted[0], res.accepted[c])
                o = O.sample_hmc(tgt, init[c], num_samples=S, num_steps_per_sample=L, step_size=0.2, inv_mass=mass,
                                 normals=z[:, c], log_uniforms=logu[:, c])
                assert res.accepted[c].cpu().bool().tolist() == o['accepted']
                assert torch.allclose(res.samples[c].cpu(), torch.stack(o['samples']), rtol=2e-4, atol=2e-4)
    # one iteration, nothing retained but params_init
    r1 = engine.hmc_run(_corr_gaussian(20, 1), torch.zeros(2, 20), 1, 3, 0.1, inv_mass=_spd(20, 2), seed=3)
    torch.cuda.synchronize()
    assert r1.samples.shape == (2, 1, 20) and torch.equal(r1.samples[:, 0].cpu(), torch.zeros(2, 20))
