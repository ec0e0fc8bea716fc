"""GPU: Gamma hyperpriors on tau_list / tau_out, Gibbs-updated inside the Bayesian-NN kernel (DESIGN §3.15).

The kernel against tests/hyper_oracle.py under the injected stream (accept sequences identical, samples and both traces
within the Bayesian-NN tolerance) over the four integrators, HMC_NUTS with teacher-forced step sizes, a classification
loss, and the tensor-core shape at cluster sizes 1, 2 and 4; Philox mode against its injected twin, bit for bit; the
gamma sampler against scipy; the prior-only and exact linear-regression posteriors; the sample sink's forms."""
import numpy as np
import pytest
import scipy.stats
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import engine, samplers, targets as T, _native as N
from oracle import cases, hmc_oracle as O
from tests import hyper_oracle as H
from tests.test_philox_stream_gpu import _stream

pytestmark = pytest.mark.gpu
MLP_RTOL = 2e-4               # tests/test_mlp_gpu.py
TRACE_RTOL = 2e-3             # tau = g / (b + |w|^2 / 2): the samples' fp32 noise through a fixed-order sum


def _problem(kind, cs=0):
    if kind.startswith('tc'):                         # n0 -> 128 -> 1: the tensor-core form ('tc': n0 = 16, 'tc48': 48)
        model, x, y = cases.mlp_problem(seed=4, n=512, n_in=int(kind[2:] or 16), hidden=128)
    elif kind == 'cls':
        model, x, y = cases.mlp_problem(seed=6, n=64, n_in=5, hidden=12, task='binary')
    else:
        model, x, y = cases.mlp_problem(seed=5, n=96, n_in=5, hidden=12)
    loss = 'binary_class_linear_output' if kind == 'cls' else 'regression'
    return model, x, y, loss


def test_tensor_core_shapes_take_the_tensor_cores():
    for kind in ('tc', 'tc32', 'tc48', 'tc64'):
        model, x, y, loss = _problem(kind)
        assert engine.native_target(_targets(model, x, y, loss, 1, 20.0, 0), 'cuda').mlp_struct.x_packed, kind


def _targets(model, x, y, loss, M, tau_out, cs):
    tau = [torch.tensor(t) for t in (2.0, 1.5, 3.0, 1.0)]
    if M == 1:
        tgt = T.MLPTarget.from_model(model, x, y, tau, tau_out, model_loss=loss)
        parts = [tgt]
    else:
        n = x.shape[0] // M
        parts = [T.MLPTarget.from_model(model, x[m * n:(m + 1) * n], y[m * n:(m + 1) * n], tau, tau_out, prior_scale=M,
                                        model_loss=loss) for m in range(M)]
        tgt = parts
    for d in parts:
        d.cluster_size = cs
    return tgt


SCHEMES = {'PLAIN': (N.SCHEME_PLAIN, None), 'SPLITTING': (N.SCHEME_SPLIT_SYM, O.SPLIT_SYM),
           'SPLITTING_RAND': (N.SCHEME_SPLIT_RAND, O.SPLIT_RAND), 'SPLITTING_KMID': (N.SCHEME_SPLIT_KMID, O.SPLIT_KMID)}
CASES = [('reg', 'PLAIN', False, 0), ('reg', 'SPLITTING', False, 0), ('reg', 'SPLITTING_RAND', False, 0),
         ('reg', 'SPLITTING_KMID', False, 0), ('reg', 'PLAIN', True, 0), ('reg', 'SPLITTING', True, 0),
         ('reg', 'SPLITTING_RAND', True, 0), ('reg', 'SPLITTING_KMID', True, 0), ('tc32', 'PLAIN', False, 2),
         ('tc48', 'SPLITTING', False, 1), ('tc64', 'PLAIN', True, 4),
         ('cls', 'PLAIN', False, 0), ('tc', 'PLAIN', False, 1), ('tc', 'PLAIN', False, 2), ('tc', 'PLAIN', False, 4),
         ('tc', 'SPLITTING', False, 2)]


@pytest.mark.parametrize('kind,scheme,nuts,cs', CASES)
def test_oracle_parity_injected(kind, scheme, nuts, cs):
    C_, S, L, burn = 2, 14, 3, 4
    model, x, y, loss = _problem(kind)
    M = 1 if scheme == 'PLAIN' else 2
    tgt = _targets(model, x, y, loss, M, 20.0, cs)
    hyper = [(2.0, 1.0), None, (1.5, 0.5), (3.0, 2.0), None if kind == 'cls' else (2.0, 0.05)]
    sch, osch = SCHEMES[scheme]
    D = hb.util.flatten(model).numel()
    g = torch.Generator().manual_seed(11)
    q0 = hb.util.flatten(model).detach()[None] + 0.05 * torch.randn(C_, D, generator=g)
    z = torch.randn(S, C_, D, generator=g)
    lu = torch.log(torch.rand(S, C_, generator=g))
    perms = torch.stack([torch.stack([torch.randperm(M, generator=g) for _ in range(C_)]) for _ in range(S)]) \
        if scheme == 'SPLITTING_RAND' else None
    shapes = samplers._reference_gamma_shapes(tgt, hyper).clamp_min(1.0)
    gam = torch.from_numpy(np.random.default_rng(3).gamma(shapes.numpy(), size=(S, C_, 5)))
    eps0 = 0.002 if kind.startswith('tc') else 0.004
    sched = (eps0 * (1 + 0.2 * torch.sin(torch.arange(S, dtype=torch.float32)))[:, None]).repeat(1, C_) if nuts else None
    res = engine.hmc_run(tgt, q0, S, L, eps0, burn=burn, nuts=nuts, normals=z, log_uniforms=lu, perms=perms,
                         record_ham=True, scheme=sch, hyper=hyper, gammas=gam,
                         **(dict(eps_schedule=sched) if nuts else {}))
    torch.cuda.synchronize()
    for c in range(C_):
        o = H.sample_hyper(tgt, q0[c], S, L, eps0, burn, hyper, z[:, c], lu[:, c], gam[:, c],
                           perms=None if perms is None else perms[:, c], split_scheme=osch,
                           eps_schedule=None if sched is None else sched[:, c])
        assert res.accepted[c].cpu().bool().tolist() == o['accepted']
        np.testing.assert_allclose(res.samples[c].cpu().numpy(), o['samples'].numpy(), rtol=MLP_RTOL, atol=MLP_RTOL)
        np.testing.assert_allclose(res.tau_list_trace[c].cpu().numpy(), o['tau_list'], rtol=TRACE_RTOL)
        np.testing.assert_allclose(res.tau_out_trace[c].cpu().numpy(), o['tau_out'], rtol=TRACE_RTOL)
    assert bool((res.tau_list_trace[..., 1] == 1.5).all())          # group 1 is fixed at its tau_list value


def _hyper_run(tgt, q0, S, **kw):
    return engine.hmc_run(tgt, q0, S, 3, 0.004, burn=4, record_ham=True, scheme=N.SCHEME_PLAIN,
                          hyper=[(2.0, 1.0), (1.0, 1.0), (1.5, 0.5), (0.5, 2.0), (2.0, 0.05)], **kw)


@pytest.mark.parametrize('kind', ['reg', 'tc'])
def test_philox_equals_the_injected_twin(kind):
    C_, S, seed, off = 4, 12, 91, 3
    model, x, y, loss = _problem(kind)
    tgt = _targets(model, x, y, loss, 1, 20.0, 2 if kind == 'tc' else 0)
    D = hb.util.flatten(model).numel()
    q0 = hb.util.flatten(model).detach()[None] + 0.05 * torch.randn(C_, D, generator=torch.Generator().manual_seed(2))
    ph = _hyper_run(tgt, q0, S, seed=seed, chain_offset=off)
    ph2 = _hyper_run(tgt, q0, S, seed=seed, chain_offset=off)
    s = _stream(seed, off, C_, S, D)
    shapes = samplers._reference_gamma_shapes(tgt, [(2.0, 1.0), (1.0, 1.0), (1.5, 0.5), (0.5, 2.0), (2.0, 0.05)])
    gam = engine.hyper_gamma_draws(seed, C_, 0, S, shapes.tolist(), chain_offset=off)
    inj = _hyper_run(tgt, q0, S, gammas=gam, **s)
    torch.cuda.synchronize()
    for a in (ph2, inj):
        assert torch.equal(ph.samples, a.samples) and torch.equal(ph.accepted, a.accepted)
        assert torch.equal(ph.tau_list_trace, a.tau_list_trace) and torch.equal(ph.tau_out_trace, a.tau_out_trace)
        assert torch.equal(ph.tau_list_final, a.tau_list_final)
    assert not torch.equal(ph.tau_out_trace[:, 1], ph.tau_out_trace[:, 2])


def test_results_do_not_depend_on_chain_offset_sharding():
    model, x, y, loss = _problem('reg')
    tgt = _targets(model, x, y, loss, 1, 20.0, 1)
    D = hb.util.flatten(model).numel()
    q0 = hb.util.flatten(model).detach()[None] + 0.05 * torch.randn(4, D, generator=torch.Generator().manual_seed(2))
    whole = _hyper_run(tgt, q0, 10, seed=5)
    parts = [_hyper_run(tgt, q0[o:o + 2], 10, seed=5, chain_offset=o) for o in (0, 2)]
    torch.cuda.synchronize()
    assert torch.equal(whole.samples, torch.cat([p.samples for p in parts]))
    assert torch.equal(whole.tau_list_trace, torch.cat([p.tau_list_trace for p in parts]))
    assert torch.equal(whole.tau_out_trace, torch.cat([p.tau_out_trace for p in parts]))


@pytest.mark.parametrize('shape', [0.3, 1.0, 2.5, 4000.0, 12345.6])
def test_gamma_sampler_ks(shape):
    draws = engine.hyper_gamma_draws(2024, 64, 0, 250, [shape, 1.0]).cpu().numpy()[..., 0].reshape(-1)
    assert np.all(draws > 0)
    p = scipy.stats.kstest(draws, scipy.stats.gamma(shape).cdf).pvalue
    assert p > 1e-3, (shape, p)
    other = engine.hyper_gamma_draws(2024, 64, 0, 250, [shape, 1.0]).cpu().numpy()[..., 0].reshape(-1)
    assert np.array_equal(draws, other)


def test_prior_only_precisions_are_gamma_marginally():
    model, _, _, _ = _problem('reg')
    tau = [torch.tensor(1.0)] * 4
    tgt = T.MLPTarget.from_model(model, None, None, tau, 1.0)
    a, b = 3.0, 2.0
    C_, S = 64, 600
    q0 = 0.3 * torch.randn(C_, tgt.dim, generator=torch.Generator().manual_seed(0))
    res = samplers.sample_chains(tgt, q0, num_samples=S, num_steps_per_sample=8, step_size=0.25, burn=100,
                                 tau_prior=(a, b), seed=17)
    tr = res.tau_list_trace[:, 1:].float()
    d = hb.diagnostics.summary(tr)
    mean, mcse = d.mean.cpu().numpy(), d.mcse.cpu().numpy()
    assert np.all(np.abs(mean - a / b) <= 4 * mcse), (mean, mcse)
    var = tr.double().var(dim=(0, 1)).cpu().numpy()
    assert np.all(np.abs(var - a / b ** 2) <= 0.25 * a / b ** 2), var


def test_exact_posterior_of_bayesian_linear_regression():
    g = torch.Generator().manual_seed(8)
    n, d = 60, 3
    x = torch.randn(n, d, generator=g)
    y = x @ torch.tensor([[0.8], [-0.5], [0.3]]) + 0.2 + 0.3 * torch.randn(n, 1, generator=g)
    model = torch.nn.Linear(d, 1)
    tgt = T.MLPTarget.from_model(model, x, y, [torch.tensor(1.0)] * 2, 1.0)
    pri = dict(a_w=2.0, b_w=1.0, a_b=2.0, b_b=1.0, a_o=2.0, b_o=0.2)
    C_, S, burn = 64, 900, 300
    q0 = 0.1 * torch.randn(C_, d + 1, generator=g)
    res = samplers.sample_chains(tgt, q0, num_samples=S, num_steps_per_sample=10, step_size=0.02, burn=burn,
                                 sampler=samplers.Sampler.HMC_NUTS, tau_prior=[(2.0, 1.0), (2.0, 1.0)],
                                 tau_out_prior=(2.0, 0.2), seed=123)
    torch.cuda.synchronize()
    draws = torch.cat([res.samples[:, 1:].double(), res.tau_list_trace[:, 1:].double().log(),
                       res.tau_out_trace[:, 1:, None].double().log()], dim=2)
    dg = hb.diagnostics.summary(draws.float())
    ref = H.linear_gibbs(x.numpy(), y.numpy(), num_samples=60000, seed=1, **pri)[5000:]
    ref_mean = ref.mean(0)
    ref_mcse = ref.std(0) / np.sqrt(len(ref) / 10)             # generous: Gibbs autocorrelation of the precisions
    got, mcse = dg.mean.cpu().numpy(), dg.mcse.cpu().numpy()
    z = np.abs(got - ref_mean) / np.sqrt(mcse ** 2 + ref_mcse ** 2)
    assert np.all(z <= 4), (got, ref_mean, z)
    tau_o = res.tau_out_trace[:, 1:].double().cpu().numpy().reshape(-1)
    q_ref = np.quantile(np.exp(ref[:, -1]), [0.05, 0.5, 0.95])
    np.testing.assert_allclose(np.quantile(tau_o, [0.05, 0.5, 0.95]), q_ref, rtol=0.06)


def test_sink_forms_keep_the_same_traces():
    model, x, y, loss = _problem('reg')
    tgt = _targets(model, x, y, loss, 2, 20.0, 0)
    D = hb.util.flatten(model).numel()
    q0 = hb.util.flatten(model).detach()[None] + 0.05 * torch.randn(3, D, generator=torch.Generator().manual_seed(2))
    kw = dict(num_samples=31, num_steps_per_sample=3, step_size=0.004, burn=4, integrator=samplers.Integrator.SPLITTING,
              tau_prior=(2.0, 1.0), tau_out_prior=(2.0, 0.05), seed=9)
    plain = samplers.sample_chains(tgt, q0, **kw)
    thin = samplers.sample_chains(tgt, q0, thin=3, moments=True, **kw)
    bare = samplers.sample_chains(tgt, q0, keep_samples=False, thin=3, **kw)
    host = samplers.sample_chains(tgt, q0, store_on_GPU=False, **kw)
    torch.cuda.synchronize()
    assert torch.equal(thin.samples, plain.samples[:, ::3])
    for r, step in ((thin, 3), (bare, 3), (host, 1)):
        assert r.tau_list_trace.is_cuda and r.tau_out_trace.is_cuda
        assert torch.equal(r.tau_list_trace, plain.tau_list_trace[:, ::step])
        assert torch.equal(r.tau_out_trace, plain.tau_out_trace[:, ::step])
        assert torch.equal(r.tau_list_final, plain.tau_list_final)
    assert torch.equal(host.samples, plain.samples.cpu())


def test_adapt_mass_windows_carry_the_hyper_state():
    model, x, y, loss = _problem('reg')
    tgt = _targets(model, x, y, loss, 1, 20.0, 0)
    D = hb.util.flatten(model).numel()
    q0 = hb.util.flatten(model).detach()[None] + 0.05 * torch.randn(2, D, generator=torch.Generator().manual_seed(2))
    res = samplers.sample_chains(tgt, q0, num_samples=60, num_steps_per_sample=3, step_size=0.004, burn=40,
                                 sampler=samplers.Sampler.HMC_NUTS, adapt_mass=True, tau_prior=(2.0, 1.0),
                                 tau_out_prior=(2.0, 0.05), seed=4)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(res.tau_list_trace).all()) and bool((res.tau_out_trace > 0).all())
    assert torch.equal(res.tau_list_trace[:, -1], res.tau_list_final)
    assert res.inv_mass.shape == (D,)


def test_sample_model_returns_the_hyper_traces():
    model, x, y, loss = _problem('reg')
    q0 = hb.util.flatten(model).detach()
    out = samplers.sample_model(model, x, y, q0, model_loss='regression', num_samples=12, num_steps_per_sample=3,
                                step_size=0.004, burn=2, tau_out=20., tau_prior=(2.0, 1.0), tau_out_prior=(2.0, 0.05),
                                verbose=False)
    samples, hyper = out
    assert len(samples) == 10 and hyper['tau_list'].shape == (10, 4) and hyper['tau_out'].shape == (10,)
    samples, hyper, rate = samplers.sample_model(model, x, y, q0, model_loss='regression', num_samples=12,
                                                 num_steps_per_sample=3, step_size=0.004, burn=2, tau_out=20., debug=2,
                                                 tau_prior=(2.0, 1.0), verbose=False)
    assert 0.0 <= rate <= 1.0 and float(hyper['tau_out'][3]) == 20.0


def test_two_abi_windows_equal_one_launch():
    """hmcx_split_run_hyper over [0, k) then [k, S), chaining q_cur, eps and the tau / tau_out state, equals one launch."""
    import ctypes as C
    model, x, y, loss = _problem('reg')
    tgt = _targets(model, x, y, loss, 2, 20.0, 0)
    D = hb.util.flatten(model).numel()
    C_, S, burn, L, seed = 3, 16, 4, 3, 21
    q0 = hb.util.flatten(model).detach()[None] + 0.05 * torch.randn(C_, D, generator=torch.Generator().manual_seed(2))
    hyper = [(2.0, 1.0), (1.0, 1.0), (1.5, 0.5), (0.5, 2.0), (2.0, 0.05)]
    one = engine.hmc_run(tgt, q0, S, L, 0.004, burn=burn, scheme=N.SCHEME_SPLIT_SYM, hyper=hyper, seed=seed)
    lib = N.load_library()
    nt = engine.native_target(tgt, 'cuda')
    ld = N.padded_ld(D)
    q_init = N.pad_rows(q0.cuda().contiguous(), ld)
    q_cur = q_init.clone()
    eps = torch.full((C_,), 0.004, dtype=torch.float32, device='cuda')
    keep = S - burn
    samples = torch.zeros((C_, keep, ld), dtype=torch.float32, device='cuda')
    acc = torch.zeros((C_, S), dtype=torch.uint8, device='cuda')
    div = torch.zeros_like(acc)
    rej = torch.zeros(C_, dtype=torch.int32, device='cuda')
    tau = torch.tensor([2.0, 1.5, 3.0, 1.0], device='cuda').repeat(C_, 1).contiguous()
    tau_out = torch.full((C_,), 20.0, device='cuda')
    tr, tro = torch.zeros((C_, keep, 4), device='cuda'), torch.zeros((C_, keep), device='cuda')
    rng = N.RngStruct()
    rng.mode, rng.seed = N.RNG_PHILOX, seed
    nuts = N.NutsStruct()
    nuts.step_size_init = 0.004
    h = N.HyperStruct()
    for k, (a, b) in enumerate(hyper):
        h.sampled[k], h.a[k], h.b[k] = 1, a, b
    h.tau, h.tau_out, h.tau_trace, h.tau_out_trace = tau.data_ptr(), tau_out.data_ptr(), tr.data_ptr(), tro.data_ptr()
    mass = engine.native_mass(None, D, 'cuda')
    for it0, it1 in ((0, 7), (7, S)):
        rc = lib.hmcx_split_run_hyper(nt.ref(), mass.ref(), C.byref(rng), C.byref(nuts), N.SCHEME_SPLIT_SYM,
                                      N.ptr(q_init), N.ptr(q_cur), N.ptr(eps), C_, ld, L, S, burn, it0, it1,
                                      N.ptr(samples), N.ptr(acc), N.ptr(div), None, N.ptr(rej), None, C.byref(h),
                                      N.stream_ptr(torch.device('cuda')))
        N.check(rc, 'hmcx_split_run_hyper')
    torch.cuda.synchronize()
    assert torch.equal(samples[..., :D], one.samples) and torch.equal(acc, one.accepted)
    assert torch.equal(tr, one.tau_list_trace) and torch.equal(tro, one.tau_out_trace)
    assert torch.equal(tau, one.tau_list_final) and torch.equal(tau_out, one.tau_out_final)
    assert torch.equal(q_cur[:, :D], one.final_state)


# ------------------------------------------------------------------------------------------------------------------
# PSIS-LOO / WAIC with each draw's tau_out
# ------------------------------------------------------------------------------------------------------------------
def _loo_run(form):
    kind = 'tc' if form == 'tc' else 'reg'
    model, x, y, loss = _problem(kind)
    tgt = _targets(model, x, y, loss, 1, 20.0, 0)
    D = hb.util.flatten(model).numel()
    q0 = hb.util.flatten(model).detach()[None] + 0.05 * torch.randn(2, D, generator=torch.Generator().manual_seed(2))
    res = samplers.sample_chains(tgt, q0, num_samples=30, num_steps_per_sample=3, step_size=0.002, burn=5,
                                 tau_prior=(2.0, 1.0), tau_out_prior=(2.0, 0.05), seed=8)
    torch.cuda.synchronize()
    return tgt, res


@pytest.mark.parametrize('form', ['simt', 'tc'])
def test_pointwise_log_lik_uses_each_draws_tau_out(form):
    from hamiltorch_b200 import loo as LOO
    from tests import loo_oracle as LO
    tgt, res = _loo_run(form)
    tr = res.tau_out_trace
    assert len(set(tr[:, 1:].reshape(-1).tolist())) > 10        # the precisions moved
    ll = LOO.pointwise_log_lik(res, tgt)                          # the result brings its trace
    assert torch.equal(ll, LOO.pointwise_log_lik(res.samples, tgt, tau_out=tr))
    draws = res.samples.cpu()
    want = np.stack([np.stack([LO.pointwise_log_lik(draws[c, s][None], H.rebuild(tgt, tgt.tau_list, float(tr[c, s])))[0]
                               for s in range(draws.shape[1])]) for c in range(draws.shape[0])])
    got = ll.double().cpu().numpy()
    assert np.all(np.abs(got - want) <= 1e-5 * (1 + np.abs(want))), np.abs(got - want).max()
    lo = LOO.psis_loo(res, tgt)
    ref = LO.psis_loo(ll.cpu().numpy())
    assert np.allclose(lo.pointwise.cpu().numpy(), ref['elpd_loo'], rtol=1e-9, atol=1e-9)
    wa = LOO.waic(res.samples[0], tgt, tau_out=tr[0])
    assert np.allclose(wa.pointwise.cpu().numpy(), LO.waic(ll[0].cpu().numpy())['elpd_waic'], rtol=1e-9, atol=1e-9)


def test_a_constant_tau_out_trace_gives_the_existing_bits():
    from hamiltorch_b200 import loo as LOO
    tgt, res = _loo_run('simt')
    const = torch.full_like(res.tau_out_trace, tgt.tau_out)
    a = LOO.pointwise_log_lik(res.samples, tgt)
    b = LOO.pointwise_log_lik(res.samples, tgt, tau_out=const)
    assert torch.equal(a, b)
    la, lb = LOO.psis_loo(res.samples, tgt), LOO.psis_loo(res.samples, tgt, tau_out=const)
    assert torch.equal(la.pointwise, lb.pointwise) and la.elpd_loo == lb.elpd_loo
