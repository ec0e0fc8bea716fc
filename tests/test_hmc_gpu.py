"""GPU parity tests of the plain-HMC hot path (through the C-ABI, hamiltorch_b200/_native.py):
CUDA kernels vs the golden fixtures produced by the unmodified reference, vs the live oracle on seeded inputs,
and -- at BASELINE sizes -- size-independent properties.  Tolerances: tests/parity.py."""
import os

import numpy as np
import pytest
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import engine, targets as T
from oracle import cases, hmc_oracle as O
from tests import dense_ref, parity

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _run_case(case, d, tuning=0, teacher_forcing=True):
    """NUTS cases replay the reference's step-size schedule (``teacher_forcing``): dual averaging feeds rho -- a
    difference of two O(D) fp32 sums -- back into the step size, which amplifies the 1e-7-relative summation-order
    difference between torch.dot and the kernel's reduction tree into diverging chains within a few iterations.  The
    chain is therefore compared under the reference's schedule (bit-exact) and the kernel's own adaptation is compared
    with that schedule iteration by iteration (tests/parity.py tolerances)."""
    tgt, kw = case['target'], dict(case['kw'])
    nuts = kw.pop('nuts', False)
    nC = len(case['seeds'])
    sched = None
    if nuts and teacher_forcing:
        sched = torch.stack([torch.from_numpy(d['step_sizes_%d' % c]).float() for c in range(nC)], 1)   # (S, C)
    init = torch.stack([torch.from_numpy(d['init_%d' % c]) for c in range(nC)])
    z = torch.stack([torch.from_numpy(d['z_%d' % c]) for c in range(nC)], 1)          # (S, C, D)
    logu = torch.stack([torch.from_numpy(d['logu_%d' % c]) for c in range(nC)], 1)    # (S, C)
    res = engine.hmc_run(tgt, init, kw['num_samples'], kw['num_steps_per_sample'], kw['step_size'],
                         burn=kw['burn'], inv_mass=kw.get('inv_mass'), nuts=nuts,
                         desired_accept_rate=kw.get('desired_accept_rate', 0.8), normals=z, log_uniforms=logu,
                         record_ham=True, tuning=tuning, eps_schedule=sched, record_eps=nuts)
    torch.cuda.synchronize()
    return res, nuts


@pytest.mark.parametrize('name', sorted(cases.plain_cases()))
def test_golden_chain_parity(name):
    """Same chain as hamiltorch.sample given the reference's own random stream: identical accept sequence,
    bit-identical retained samples (HMC), Hamiltonians to summation-order tolerance."""
    case = cases.plain_cases()[name]
    d = np.load(os.path.join(GOLD, name + '.npz'))
    res, nuts = _run_case(case, d)
    exact = 'rtol' not in case          # coupled targets / full mass: matvec summation order differs from torch's
    for c in range(len(case['seeds'])):
        # LogProbError iterations (non-finite log-prob -> reject, samplers.py:1045) must be the reference's
        assert np.array_equal(res.diverged[c].cpu().numpy(), d['diverged_%d' % c])
        parity.assert_chain_parity(
            res.samples[c].cpu().numpy(), res.accepted[c].cpu().numpy(), res.ham[c].cpu().numpy(),
            d['samples_%d' % c], d['accepted_%d' % c], d['ham_old_%d' % c], d['ham_new_%d' % c],
            d['logu_%d' % c], case['kw']['burn'], exact=exact, rtol=case.get('rtol', 0.0),
            tag=None if exact else 'hmc/%s/%s/c%d' % (name, 'tcgen05' if os.environ.get('HMCX_FLOW_SMALL') == '0' else 'default', c))
        assert int(res.num_rejected[c]) == int((d['accepted_%d' % c] == 0).sum())
        if nuts:
            # the kernel's own dual averaging, fed the same history, proposes the reference's step sizes
            S, burn = case['kw']['num_samples'], case['kw']['burn']
            own = res.eps_trace[c].cpu().numpy().astype(np.float64)          # own[n] = eps for iteration n+1
            ref = d['step_sizes_%d' % c]
            rt = max(parity.NUTS_EPS_RTOL, 10 * case.get('rtol', 0.0))
            np.testing.assert_allclose(own[:S - 1], ref[1:], rtol=rt)
            np.testing.assert_allclose(own[burn], float(d['final_step_size_%d' % c]), rtol=rt)
            np.testing.assert_allclose(float(res.eps_bar[c]), float(d['final_step_size_%d' % c]), rtol=rt)
        else:
            assert float(res.step_size[c]) == np.float32(case['kw']['step_size'])


def _is_small_dense(case):
    """16 < D <= 128 with a dense precision or a 2-D / block-list inv_mass: runs on the persistent small-D kernel
    (hmcx_flow.cu) by default and on the step-synchronous tensor-core path when HMCX_FLOW_SMALL=0."""
    import hamiltorch_b200.targets as T
    tgt, im = case['target'], case['kw'].get('inv_mass')
    full_mass = isinstance(im, list) or (torch.is_tensor(im) and im.dim() == 2)
    return 16 < tgt.dim <= 128 and (isinstance(tgt, T.GaussianFull) or full_mass)


@pytest.mark.parametrize('name', sorted(n for n, c in cases.plain_cases().items() if _is_small_dense(c)))
def test_golden_chain_parity_tcgen05_path(name, monkeypatch):
    """The golden chains of the small dense cases ALSO through the tensor-core GEMM path (the default at D > 128)."""
    monkeypatch.setenv('HMCX_FLOW_SMALL', '0')
    test_golden_chain_parity(name)


@pytest.mark.parametrize('tuning', [1, 2, 4, 21, 22, 41, 42])
def test_register_geometry_variants_agree(tuning):
    """The register geometry (float2 / float4 groups, 1-4 groups per thread; 41 / 42: the chain spread over a thread-block
    cluster of 4 / 2 CTAs with the reduction through distributed shared memory) only changes the reduction tree, never
    the element-wise state -- and, in Philox mode, not the random stream either."""
    for name in ('iso256', 'diag48_mass'):
        case = cases.plain_cases()[name]
        d = np.load(os.path.join(GOLD, name + '.npz'))
        res, _ = _run_case(case, d, tuning=tuning)
        for c in range(len(case['seeds'])):
            assert np.array_equal(res.accepted[c].cpu().numpy(), d['accepted_%d' % c])
            assert np.array_equal(res.samples[c].cpu().numpy(), d['samples_%d' % c])
    tgt = T.GaussianDiag(torch.zeros(200), torch.linspace(0.5, 2, 200))
    init = 0.1 * torch.randn(3, 200, generator=torch.Generator().manual_seed(0))
    kw = dict(num_samples=21, num_steps_per_sample=5, step_size=0.3, burn=2, seed=9)
    a = engine.hmc_run(tgt, init, **kw)
    b = engine.hmc_run(tgt, init, tuning=tuning, **kw)
    assert torch.equal(a.accepted, b.accepted) and torch.equal(a.samples, b.samples)


def test_leapfrog_matches_reference_trajectory_and_reverses():
    """The reference's only hot-path test (tests/test_util.py:97-110): all 100 clones of the trajectory equal the
    reference's bit for bit (descriptor target), and the reversed trajectory returns to the start."""
    d = np.load(os.path.join(GOLD, 'ref_reversibility.npz'))
    tgt = T.GaussianDiag(torch.zeros(2), torch.tensor([.10, .10]))
    q0, p0, im = torch.tensor([1., 1.]), torch.tensor([1., 1.]), torch.tensor([1., 1.])
    qs, ps = hb.leapfrog(q0, p0, tgt, steps=100, step_size=0.1, inv_mass=im, sampler=hb.Sampler.HMC,
                         integrator=hb.Integrator.EXPLICIT)
    assert len(qs) == 100 and len(ps) == 100 and qs[0].shape == (2,) and qs[0].device == q0.device
    assert np.array_equal(torch.stack(qs).numpy(), d['fwd_q_desc'])
    assert np.array_equal(torch.stack(ps).numpy(), d['fwd_p_desc'])
    qb, pb = hb.leapfrog(qs[-1], -ps[-1].clone(), tgt, steps=100, step_size=0.1, inv_mass=im)
    assert np.array_equal(torch.stack(qb).numpy(), d['bwd_q_desc'])
    assert torch.allclose(qb[-1], q0, atol=5e-6)


def test_leapfrog_batched_vs_oracle_all_mass_kinds():
    torch.manual_seed(4)
    D, C, L = 37, 5, 7          # D not a multiple of 4: exercises the padded layout
    var = 0.2 + torch.rand(D)
    for tgt in (T.GaussianIso(D), T.GaussianDiag(torch.randn(D), var)):
        for im in (None, 0.5 + torch.rand(D)):
            q, p = torch.randn(C, D), torch.randn(C, D)
            eps = torch.tensor([0.1, 0.2, 0.05, 0.3, 0.15])
            qt, pt = engine.leapfrog(tgt, q, p, L, eps, inv_mass=im, return_trajectory=True)
            qf, pf = engine.leapfrog(tgt, q, p, L, eps, inv_mass=im)
            assert torch.equal(qf, qt[-1]) and torch.equal(pf, pt[-1])
            for c in range(C):
                oq, op = O.leapfrog_hmc(tgt, q[c], p[c], L, float(eps[c]), im)
                assert torch.equal(qt[:, c].cpu(), torch.stack(oq))
                assert torch.equal(pt[:, c].cpu(), torch.stack(op))


def test_hamiltonian_vs_oracle_and_nonfinite_flag():
    torch.manual_seed(5)
    D, C = 1000, 6
    tgt = T.GaussianDiag(torch.randn(D), 0.3 + torch.rand(D))
    im = 0.5 + torch.rand(D)
    q, p = torch.randn(C, D), torch.randn(C, D)
    for mass in (None, im):
        H, flags = engine.hamiltonian(tgt, q, p, inv_mass=mass)
        assert int(flags.sum()) == 0
        for c in range(C):
            ref = float(O.hamiltonian_hmc(tgt, q[c], p[c], mass))
            assert abs(float(H[c]) - ref) <= 50 * parity.H_TOL_REL * (abs(ref) + 1)
    # against fp64 at the widths where hamiltonian_kernel's block (ld / 4 threads, rounded up to a warp, at most 256)
    # changes: one warp at D = 1 and 3, 256 threads with one float4 each at D = 1000, several per thread at 4099, 9001
    for Dw in (1, 3, 1000, 4099, 9001):
        g = torch.Generator().manual_seed(Dw)
        for tgt_w in (T.GaussianIso(Dw), T.GaussianDiag(torch.randn(Dw, generator=g), 0.3 + torch.rand(Dw, generator=g))):
            qw, pw = torch.randn(C, Dw, generator=g), torch.randn(C, Dw, generator=g)
            for mass in (None, 0.5 + torch.rand(Dw, generator=g)):
                H, flags = engine.hamiltonian(tgt_w, qw, pw, inv_mass=mass)
                assert int(flags.sum()) == 0
                want = dense_ref.HMC(tgt_w, mass).hamiltonian(qw.double(), pw.double())
                parity.assert_close('elem_ref/hamiltonian_%s_%s_d%d' % (type(tgt_w).__name__, 'none' if mass is None
                                                                        else 'diag', Dw),
                                    H.double().cpu().numpy(), want.numpy(), 2e-4)
    h1 = hb.hamiltonian(q[0], p[0], tgt)
    assert h1.dim() == 0
    q[2, 5] = float('inf')
    H, flags = engine.hamiltonian(tgt, q, p)
    assert flags.cpu().tolist() == [0, 0, 1, 0, 0, 0]
    with pytest.raises(hb.util.LogProbError):
        hb.hamiltonian(q[2], p[2], tgt)


def test_cfg2_size_chain_parity_vs_live_oracle():
    """BASELINE config 2 dimensions (D=1024 isotropic, L=10, eps=.05), a few chains x a few iterations so the
    oracle finishes in seconds: bit-identical chains under the injected stream."""
    D, C, S, L = 1024, 4, 12, 10
    tgt = T.GaussianIso(D)
    inits, zs, lus = [], [], []
    for seed in range(C):
        init, z, logu, _ = O.reference_stream(seed, D, S, prior=lambda: 0.1 * torch.randn(D))
        inits.append(init), zs.append(z), lus.append(logu)
    res = hb.sample_chains(tgt, torch.stack(inits), num_samples=S, num_steps_per_sample=L, step_size=0.05,
                           rng='injected', normals=torch.stack(zs, 1), log_uniforms=torch.stack(lus, 1),
                           record_ham=True)
    for c in range(C):
        o = O.sample_hmc(tgt, inits[c], num_samples=S, num_steps_per_sample=L, step_size=0.05,
                         normals=zs[c], log_uniforms=lus[c])
        parity.assert_chain_parity(res.samples[c].cpu().numpy(), res.accepted[c].cpu().numpy(),
                                   res.ham[c].cpu().numpy(), torch.stack(o['samples']).numpy(), o['accepted'],
                                   o['ham_old'], o['ham_new'], lus[c].numpy(), 0, exact=True)


def test_cfg5_size_nuts_vs_live_oracle():
    """BASELINE config 5 dimensions (D=4096, HMC_NUTS, eps0=.1, L=10), 2 chains, burn 12 of 16."""
    D, C, S, L, burn = 4096, 2, 16, 10, 12
    tgt = T.GaussianIso(D)
    inits, zs, lus = [], [], []
    for seed in range(C):
        init, z, logu, _ = O.reference_stream(100 + seed, D, S, prior=lambda: 0.1 * torch.randn(D))
        inits.append(init), zs.append(z), lus.append(logu)
    os_ = [O.sample_hmc(tgt, inits[c], num_samples=S, num_steps_per_sample=L, step_size=0.1, burn=burn, nuts=True,
                        normals=zs[c], log_uniforms=lus[c]) for c in range(C)]
    sched = torch.tensor([o['step_sizes'] for o in os_], dtype=torch.float32).t()            # (S, C)
    res = engine.hmc_run(tgt, torch.stack(inits), S, L, 0.1, burn=burn, nuts=True, normals=torch.stack(zs, 1),
                         log_uniforms=torch.stack(lus, 1), record_ham=True, eps_schedule=sched, record_eps=True)
    for c in range(C):
        o = os_[c]
        parity.assert_chain_parity(res.samples[c].cpu().numpy(), res.accepted[c].cpu().numpy(),
                                   res.ham[c].cpu().numpy(), torch.stack(o['samples']).numpy(), o['accepted'],
                                   o['ham_old'], o['ham_new'], lus[c].numpy(), burn, exact=True)
        own = res.eps_trace[c].cpu().numpy().astype(np.float64)
        rtol = parity.nuts_eps_rtol(max(abs(h) for h in o['ham_old']))      # H ~ 4e3 at D=4096: fp32 ulp 2.4e-4
        np.testing.assert_allclose(own[:S - 1], np.array(o['step_sizes'])[1:], rtol=rtol)
        np.testing.assert_allclose(float(res.eps_bar[c]), o['eps_bar'], rtol=rtol)


def test_nuts_free_running_adapts_like_the_reference():
    """Without teacher forcing the adapted step size is a chaotic function of fp32 round-off, for the reference too
    (its value changes with the CPU's dot-product vectorisation).  What is reproducible: the distribution.  64 chains
    of the config-5 twin: median adapted step size within 10% of the oracle's over the same seeds, acceptance after
    burn-in close to the 0.8 target."""
    D, C, S, L, burn = 128, 64, 140, 10, 100
    tgt = T.GaussianIso(D)
    init = 0.1 * torch.randn(C, D, generator=torch.Generator().manual_seed(3))
    res = hb.sample_chains(tgt, init, num_samples=S, num_steps_per_sample=L, step_size=0.1, burn=burn,
                           sampler=hb.Sampler.HMC_NUTS, rng='philox', seed=11)
    eps = res.step_size.cpu()
    oracle_eps = []
    for c in range(12):
        torch.manual_seed(500 + c)
        o = O.sample_hmc(tgt, init[c], num_samples=S, num_steps_per_sample=L, step_size=0.1, burn=burn, nuts=True)
        oracle_eps.append(o['step_size'])
    med, omed = float(eps.median()), float(np.median(oracle_eps))
    assert abs(med - omed) / omed < 0.10, (med, omed)
    post = res.accepted[:, burn + 1:].float().mean().item()
    assert 0.65 < post < 0.95, post


def test_sample_dropin_reproduces_reference_after_set_random_seed():
    """hb.set_random_seed(123); hb.sample(...) == the reference's notebook run (BASELINE config 1,
    notebooks/hamiltorch_log_prob_examples.ipynb cells 6-9), chain and acceptance rate."""
    case = cases.plain_cases()['cfg1_gauss3']
    d = np.load(os.path.join(GOLD, 'cfg1_gauss3.npz'))
    hb.set_random_seed(123)
    samples, rate = hb.sample(log_prob_func=case['target'], params_init=torch.zeros(3), debug=2, verbose=False,
                              **case['kw'])
    assert isinstance(samples, list) and len(samples) == 400 and samples[0].shape == (3,)
    assert samples[0].device.type == 'cpu'                       # results come back on params_init.device
    assert np.array_equal(torch.stack(samples).numpy(), d['samples_0'])
    assert abs(rate - d['accepted_0'].mean()) < 1e-12


def test_multi_chain_runs_batched_and_matches_reference_chains():
    """util.multi_chain (util.py:392-405) as ONE launch: chain-by-chain equal to the reference's serial chains."""
    case = cases.plain_cases()['iso256']
    d = np.load(os.path.join(GOLD, 'iso256.npz'))
    kwargs = dict(log_prob_func=case['target'], verbose=False, **case['kw'])
    chain = hb.util.setup_chain(hb.sample, lambda: 0.1 * torch.randn(256), kwargs)
    out = hb.util.multi_chain(chain, 2, case['seeds'], parallel=False)
    assert len(out) == 3 and len(out[0]) == 30
    for c in range(3):
        assert np.array_equal(torch.stack(out[c]).numpy(), d['samples_%d' % c])
    # and the single-chain closure gives the same answer as the batched run
    one = chain(case['seeds'][1])
    assert np.array_equal(torch.stack(one).numpy(), d['samples_1'])


def test_philox_is_reproducible_and_sharding_invariant():
    """Chains keyed by (seed, global chain id): one launch of 8 == two launches of 4 with chain_offset."""
    D, C, S = 200, 8, 25
    tgt = T.GaussianDiag(torch.zeros(D), torch.linspace(0.5, 2, D))
    init = 0.1 * torch.randn(C, D, generator=torch.Generator().manual_seed(0))
    kw = dict(num_samples=S, num_steps_per_sample=6, step_size=0.3, burn=3, rng='philox', seed=42)
    a = hb.sample_chains(tgt, init, **kw)
    b = hb.sample_chains(tgt, init, **kw)
    assert torch.equal(a.samples, b.samples) and torch.equal(a.accepted, b.accepted)
    lo = hb.sample_chains(tgt, init[:4], chain_offset=0, **kw)
    hi = hb.sample_chains(tgt, init[4:], chain_offset=4, **kw)
    assert torch.equal(torch.cat([lo.samples, hi.samples]), a.samples)
    c = hb.sample_chains(tgt, init, **dict(kw, seed=43))
    assert not torch.equal(c.samples, a.samples)


def test_philox_gibbs_moments_and_mass_scaling():
    D, C = 512, 256
    p = engine.gibbs(D, C, seed=7, iteration=3)
    assert p.shape == (C, D)
    assert abs(float(p.mean())) < 0.01 and abs(float(p.var()) - 1) < 0.02
    assert abs(float((p ** 4).mean()) - 3) < 0.1                 # Gaussian kurtosis
    im = torch.linspace(0.25, 4, D)
    pm = engine.gibbs(D, C, seed=7, iteration=3, inv_mass=im)
    assert torch.equal(pm.cpu(), (p.cpu() * ((1 / im) ** 0.5)))
    p2 = engine.gibbs(D, C, seed=7, iteration=4)
    assert abs(float((p * p2).mean())) < 0.01                    # iterations are independent streams


def test_baseline_config2_full_size_properties():
    """BASELINE config 2 at full width (C=256 chains, D=1024, L=10, eps=.05), S=60: properties that do not need
    the oracle -- slot 0 is params_init; a rejected stored iteration repeats the previous slot; accepted ones
    conserve energy to integrator accuracy; acceptance ~0.99; pooled moments of N(0, I)."""
    C, D, S, L = 256, 1024, 60, 10
    tgt = T.GaussianIso(D)
    init = torch.randn(C, D, generator=torch.Generator().manual_seed(1))
    res = hb.sample_chains(tgt, init, num_samples=S, num_steps_per_sample=L, step_size=0.05, rng='philox', seed=5,
                           record_ham=True)
    s = res.samples.cpu()
    acc = res.accepted.cpu().bool()
    assert s.shape == (C, S, D)
    assert torch.equal(s[:, 0], init)
    same = (s[:, 2:] == s[:, 1:-1]).all(-1)                       # slot n vs n-1, n >= 2
    assert torch.equal(same, ~acc[:, 2:])
    assert int(res.diverged.sum()) == 0
    rate = acc.float().mean().item()
    assert 0.97 < rate <= 1.0
    dH = (res.ham[..., 1] - res.ham[..., 0]).cpu()
    assert dH.abs().max() < 1.0 and dH.abs().mean() < 0.2
    tail = s[:, S // 2:]
    assert abs(tail.mean().item()) < 0.01
    assert abs(tail.var().item() - 1.0) < 0.02
    assert torch.equal(res.num_rejected.cpu().long(), (~acc).sum(1))


@pytest.mark.parametrize('D', [4100, 9001])
def test_large_dimension_streamed_kernel_vs_live_oracle(D):
    """D > 4096: the chain state no longer fits one CTA's registers and is streamed through a caller-provided
    workspace (hmcx_hmc_workspace_bytes).  Same bit-exact chain parity, incl. diagonal mass, burn-in and rejections."""
    C, S, L, burn = 3, 10, 4, 2
    g = torch.Generator().manual_seed(D)
    var = 0.5 + torch.rand(D, generator=g)
    tgt = T.GaussianDiag(torch.randn(D, generator=g), var)
    im = var.clone()
    inits, zs, lus = [], [], []
    for seed in range(C):
        init, z, logu, _ = O.reference_stream(300 + seed, D, S, prior=lambda: tgt.mean + 0.1 * torch.randn(D))
        inits.append(init), zs.append(z), lus.append(logu)
    res = hb.sample_chains(tgt, torch.stack(inits), num_samples=S, num_steps_per_sample=L, step_size=0.9, burn=burn,
                           inv_mass=im, rng='injected', normals=torch.stack(zs, 1), log_uniforms=torch.stack(lus, 1),
                           record_ham=True)
    n_rej = 0
    for c in range(C):
        o = O.sample_hmc(tgt, inits[c], num_samples=S, num_steps_per_sample=L, step_size=0.9, burn=burn, inv_mass=im,
                         normals=zs[c], log_uniforms=lus[c])
        parity.assert_chain_parity(res.samples[c].cpu().numpy(), res.accepted[c].cpu().numpy(),
                                   res.ham[c].cpu().numpy(), torch.stack(o['samples']).numpy(), o['accepted'],
                                   o['ham_old'], o['ham_new'], lus[c].numpy(), burn, exact=True)
        n_rej += o['num_rejected']
    assert n_rej > 0, 'the case should exercise the reject / restore path'
    # and the production RNG path runs and mixes
    r = hb.sample_chains(T.GaussianIso(D), torch.randn(4, D, generator=g), num_samples=30, num_steps_per_sample=10,
                         step_size=0.04, rng='philox', seed=1)
    assert 0.8 < float(r.accept_rate.mean()) <= 1.0
    assert abs(float(r.samples[:, 15:].var()) - 1.0) < 0.1         # started in stationarity, must stay there


@pytest.mark.parametrize('D', [3, 11, 150])
def test_standalone_leapfrog_and_hamiltonian_coupled_targets_vs_oracle(D):
    """samplers.leapfrog / samplers.hamiltonian (the reference's utility entry points) for what is not element-wise:
    GaussianFull and Funnel targets, and the 2-D inv_mass of :294 / :812, at small and large D (one CTA per chain,
    hmcx_coupled.cu).  Matrix-vector sums differ from torch.mv in summation order only."""
    g = torch.Generator().manual_seed(40 + D)
    A = torch.randn(D, D, generator=g, dtype=torch.float64) / D ** 0.5
    cov = A @ A.t() + 0.5 * torch.eye(D, dtype=torch.float64)
    B = torch.randn(D, D, generator=g, dtype=torch.float64) / D ** 0.5
    im_full = (B @ B.t() + 0.7 * torch.eye(D, dtype=torch.float64)).float()
    im_diag = 0.5 + torch.rand(D, generator=g)
    targets = [T.GaussianFull(torch.randn(D, generator=g), cov=cov), T.GaussianDiag(torch.randn(D, generator=g),
                                                                                   0.3 + torch.rand(D, generator=g))]
    if D <= 11:
        targets.append(T.Funnel(D))
    C, L = 4, 6
    eps = torch.tensor([0.05, 0.1, 0.02, 0.08])
    for tgt in targets:
        for im in (None, im_diag, im_full):
            if isinstance(tgt, T.GaussianDiag) and (im is None or im.dim() == 1):
                continue                                # element-wise: covered by the bit-exact tests above
            q = 0.5 * torch.randn(C, D, generator=g)
            p = torch.randn(C, D, generator=g)
            qt, pt = engine.leapfrog(tgt, q, p, L, eps, inv_mass=im, return_trajectory=True)
            qf, pf = engine.leapfrog(tgt, q, p, L, eps, inv_mass=im)
            H, flags = engine.hamiltonian(tgt, q, p, inv_mass=im)
            torch.cuda.synchronize()
            assert torch.equal(qf, qt[-1]) and torch.equal(pf, pt[-1]) and int(flags.sum()) == 0
            for c in range(C):
                oq, op = O.leapfrog_hmc(tgt, q[c], p[c], L, float(eps[c]), im)
                np.testing.assert_allclose(qt[:, c].cpu().numpy(), torch.stack(oq).detach().numpy(), rtol=2e-4, atol=2e-5)
                np.testing.assert_allclose(pt[:, c].cpu().numpy(), torch.stack(op).detach().numpy(), rtol=2e-4, atol=2e-4)
                ref = float(O.hamiltonian_hmc(tgt, q[c], p[c], im))
                assert abs(float(H[c]) - ref) <= 1e-5 * (1 + abs(ref))
    # the drop-in wrappers: (D,) in, lists of (D,) out; reversibility (tests/test_util.py:97-110) on a coupled target
    tgt = targets[0]
    q0, p0 = torch.randn(D, generator=g), torch.randn(D, generator=g)
    qs, ps = hb.leapfrog(q0, p0, tgt, steps=8, step_size=0.05, inv_mass=im_full)
    assert len(qs) == 8 and qs[0].shape == (D,)
    qb, pb = hb.leapfrog(qs[-1], -ps[-1].clone(), tgt, steps=8, step_size=0.05, inv_mass=im_full)
    assert torch.allclose(qb[-1], q0, atol=2e-4)
    assert hb.hamiltonian(q0, p0, tgt, inv_mass=im_full).dim() == 0


def test_standalone_hamiltonian_flags_nonfinite_funnel():
    """A funnel point whose log-density overflows: samplers.hamiltonian raises LogProbError (:783-785)."""
    tgt = T.Funnel(5)
    q = torch.tensor([200., 1., 1., 1., 1.])          # exp(200) = inf
    with pytest.raises(hb.util.LogProbError):
        hb.hamiltonian(q, torch.zeros(5), tgt)
