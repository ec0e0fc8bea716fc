"""GPU: the sample sink of the Bayesian-NN kernel (hmcx_split_run_sink): thinning, running moments, no-sample runs and
store_on_GPU=False streaming into pinned host memory.  Every sink run is checked against the plain run of the same chains
(same Philox stream): flags, Hamiltonians, step sizes and samples bit for bit, moments against fp64 sums of the samples."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.utils.data as tud

import hamiltorch_b200 as hb
from hamiltorch_b200 import engine, targets as T, _native as N
from oracle import cases

pytestmark = pytest.mark.gpu

LOSS = {'regression': 'regression', 'binary': 'binary_class_linear_output'}
INTEGRATOR = {'SPLITTING': hb.Integrator.SPLITTING, 'SPLITTING_RAND': hb.Integrator.SPLITTING_RAND,
              'SPLITTING_KMID': hb.Integrator.SPLITTING_KMID}


def _descs(model, x, y, splits, tau_out=50., task='regression'):
    b = np.linspace(0, x.shape[0], splits + 1).astype(int)
    return [T.MLPTarget.from_model(model, x[i:j], y[i:j], None, tau_out, prior_scale=splits, model_loss=LOSS[task])
            for i, j in zip(b[:-1], b[1:])]


def _init(model, C_, seed=0, scale=0.05):
    D = hb.util.flatten(model).numel()
    return hb.util.flatten(model).detach()[None] + scale * torch.randn(C_, D, generator=torch.Generator().manual_seed(seed))


def _bits(t):
    return t.contiguous().view(torch.int32)           # NaN Hamiltonians of diverged proposals compare too


def _assert_same_run(sink, full, thin):
    assert torch.equal(sink.accepted, full.accepted) and torch.equal(sink.diverged, full.diverged)
    assert torch.equal(_bits(sink.ham), _bits(full.ham))
    assert torch.equal(sink.step_size, full.step_size) and torch.equal(sink.num_rejected, full.num_rejected)
    assert sink.samples.shape[1] == 1 + (full.samples.shape[1] - 1) // thin
    assert torch.equal(_bits(sink.samples.cpu()), _bits(full.samples[:, ::thin].cpu()))
    assert torch.equal(sink.final_state, full.final_state)


def _assert_moments(res, full):
    x = full.samples[:, 1:].double()
    assert res.moment_count == x.shape[1]
    assert torch.allclose(res.moment_sum, x.sum(1), rtol=1e-10, atol=1e-10)
    assert torch.allclose(res.moment_sumsq, (x * x).sum(1), rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize('nuts', [False, True])
@pytest.mark.parametrize('scheme', ['PLAIN', 'SPLITTING', 'SPLITTING_RAND', 'SPLITTING_KMID'])
def test_thinning_and_moments_equal_the_plain_run(scheme, nuts):
    model, x, y = cases.mlp_problem(seed=5, n=96, n_in=6, hidden=16)
    if scheme == 'PLAIN':
        target, integ = T.MLPTarget.from_model(model, x, y, None, 50.), hb.Integrator.IMPLICIT
    else:
        target, integ = _descs(model, x, y, 3), INTEGRATOR[scheme]
    kw = dict(num_samples=20, num_steps_per_sample=4, step_size=0.01, burn=4, integrator=integ, rng='philox', seed=7,
              record_ham=True, sampler=hb.Sampler.HMC_NUTS if nuts else hb.Sampler.HMC)
    init = _init(model, 5)
    full = hb.sample_chains(target, init, **kw)
    thin = hb.sample_chains(target, init, thin=3, moments=True, **kw)
    none = hb.sample_chains(target, init, keep_samples=False, moments=True, **kw)
    torch.cuda.synchronize()
    _assert_same_run(thin, full, 3)
    _assert_moments(thin, full)
    assert torch.equal(none.moment_sum, thin.moment_sum) and torch.equal(none.moment_sumsq, thin.moment_sumsq)
    assert torch.equal(none.final_state, full.final_state) and torch.equal(none.accepted, full.accepted)
    with pytest.raises(RuntimeError):
        none.samples


@pytest.mark.parametrize('cluster', [1, 2, 4])
@pytest.mark.parametrize('shape', ['tc', 'simt', 'simt_binary'])
def test_pinned_cluster_sizes_and_kernel_shapes(shape, cluster):
    """Every rank of a cluster stores and accumulates its own slice of the row: sink == plain for 1, 2 and 4 CTAs per
    chain, on the tensor-core shape (16-128-1, D = 2305) and the SIMT shape 1-10-10-1 (D = 141, so the last float4 of a
    row is partly padding), with a regression and a classification likelihood."""
    task = 'binary' if shape == 'simt_binary' else 'regression'
    if shape == 'tc':
        model, x, y = cases.mlp_problem(seed=8, n=512, n_in=16, hidden=128, task=task)
    else:
        model, x, y = cases.mlp_problem(seed=9, n=512, n_in=1, hidden=10, depth=2, task=task)
    descs = _descs(model, x, y, 2, tau_out=20. if task == 'regression' else 1., task=task)
    descs[0].cluster_size = cluster
    assert descs[0].dim == (2305 if shape == 'tc' else 141)
    kw = dict(num_samples=12, num_steps_per_sample=3, step_size=0.004, burn=2, integrator=hb.Integrator.SPLITTING,
              rng='philox', seed=11, record_ham=True)
    init = _init(model, 3, seed=cluster)
    full = hb.sample_chains(descs, init, **kw)
    thin = hb.sample_chains(descs, init, thin=3, moments=True, **kw)
    torch.cuda.synchronize()
    _assert_same_run(thin, full, 3)
    _assert_moments(thin, full)


def test_store_on_gpu_false_streams_samples_to_pinned_host_memory():
    model, x, y = cases.mlp_problem(seed=9, n=512, n_in=1, hidden=10, depth=2)
    descs = _descs(model, x, y, 2, tau_out=20.)
    kw = dict(num_samples=400, num_steps_per_sample=2, step_size=0.004, burn=0, integrator=hb.Integrator.SPLITTING,
              rng='philox', seed=3)
    init = _init(model, 8)
    full = hb.sample_chains(descs, init, **kw)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    host = hb.sample_chains(descs, init, store_on_GPU=False, **kw)
    torch.cuda.synchronize()
    grown = torch.cuda.max_memory_allocated() - base
    assert not host.samples.is_cuda and host.samples_padded.is_pinned()
    assert torch.equal(host.samples_padded, full.samples_padded.cpu())
    block = host.samples_padded.numel() * 4
    assert grown < block // 4, (grown, block)          # the run keeps no device copy of the sample block

    # the reference-shaped entry points after set_random_seed: lists of CPU tensors equal to store_on_GPU=True
    model, x, y = cases.mlp_problem(seed=1, n=48)
    M, D = 3, hb.util.flatten(model).numel()
    loader = tud.DataLoader(tud.TensorDataset(x, y), batch_size=x.shape[0] // M, shuffle=False)
    p0 = hb.util.flatten(model).detach().clone()
    kw = dict(model_loss='regression', num_samples=10, num_steps_per_sample=3, step_size=0.01, burn=2, tau_out=50.,
              verbose=False)
    runs = {}
    for on_gpu in (True, False):
        hb.set_random_seed(4)
        runs['split', on_gpu] = hb.sample_split_model(model, loader, params_init=p0 + 0.05 * torch.randn(D),
                                                      num_splits=M, integrator=hb.Integrator.SPLITTING,
                                                      store_on_GPU=on_gpu, **kw)
        hb.set_random_seed(4)
        runs['model', on_gpu] = hb.sample_model(model, x, y, params_init=p0 + 0.05 * torch.randn(D), store_on_GPU=on_gpu,
                                                **kw)
    for name in ('split', 'model'):
        a, b = runs[name, True], runs[name, False]
        assert len(a) == len(b) == 8 and all(not t.is_cuda for t in b)
        assert all(torch.equal(s, t) for s, t in zip(a, b)), name


def test_sink_edge_cases():
    """burn = S-1 (nothing but params_init is retained: zero moment count), thin larger than the run."""
    model, x, y = cases.mlp_problem(seed=2, n=64, n_in=1, hidden=10, depth=2)
    descs = _descs(model, x, y, 2)
    init = _init(model, 3)
    kw = dict(num_steps_per_sample=3, step_size=0.01, integrator=hb.Integrator.SPLITTING_RAND, rng='philox', seed=2)
    r = hb.sample_chains(descs, init, num_samples=6, burn=5, moments=True, **kw)
    torch.cuda.synchronize()
    assert r.samples.shape == (3, 1, 141) and torch.equal(r.samples[:, 0].cpu(), init)
    assert r.moment_count == 0 and float(r.moment_sum.abs().sum()) == 0.0 and float(r.moment_sumsq.abs().sum()) == 0.0
    full = hb.sample_chains(descs, init, num_samples=12, burn=2, **kw)
    thin = hb.sample_chains(descs, init, num_samples=12, burn=2, thin=50, moments=True, **kw)
    torch.cuda.synchronize()
    assert thin.samples.shape == (3, 1, 141) and torch.equal(thin.samples[:, 0], full.samples[:, 0])
    assert torch.equal(thin.final_state, full.final_state)
    _assert_moments(thin, full)


def _split_run_sink(nt, q0, S, burn, L, step, thin, windows, seed, scheme):
    """hmcx_split_run_sink through ctypes, the iterations cut into `windows`; every output buffer starts as NaN / 0xFF so
    that a slot or flag no launch wrote shows up."""
    lib = N.load_library()
    dev = torch.device('cuda')
    D, ld, Cn = nt.dim, N.padded_ld(nt.dim), q0.shape[0]
    q_init = engine._as_rows(q0, ld, dev)
    q_cur = q_init.clone()
    eps = torch.full((Cn,), step, dtype=torch.float32, device=dev)
    keep = 1 + (S - burn - 1) // thin
    samples = torch.full((Cn, keep, ld), float('nan'), device=dev)
    acc = torch.full((Cn, S), 255, dtype=torch.uint8, device=dev)
    div = torch.full_like(acc, 255)
    ham = torch.full((Cn, S, 2), float('nan'), device=dev)
    nrej = torch.zeros(Cn, dtype=torch.int32, device=dev)
    mom = [torch.zeros((Cn, ld), dtype=torch.float32, device=dev) for _ in range(4)]
    sink = N.SinkStruct()
    sink.thin = thin
    sink.sum, sink.sumsq, sink.sum_lo, sink.sumsq_lo = (t.data_ptr() for t in mom)
    rng = N.RngStruct()
    rng.mode, rng.seed = N.RNG_PHILOX, seed
    nuts = N.NutsStruct()
    nuts.step_size_init = step
    mass = engine.native_mass(None, D, dev)
    for a, b in windows:
        rc = lib.hmcx_split_run_sink(nt.ref(), mass.ref(), C.byref(rng), C.byref(nuts), scheme, N.ptr(q_init),
                                     N.ptr(q_cur), N.ptr(eps), Cn, ld, L, S, burn, a, b, N.ptr(samples), N.ptr(acc),
                                     N.ptr(div), N.ptr(ham), N.ptr(nrej), C.byref(sink), N.stream_ptr(dev))
        assert rc == N.OK, rc
    torch.cuda.synchronize()
    return dict(samples=samples, acc=acc, div=div, ham=ham, nrej=nrej, eps=eps, q_cur=q_cur, mom=torch.stack(mom))


@pytest.mark.parametrize('cut', [3, 4, 9])
def test_windows_of_iterations_equal_one_launch(cut):
    """Two launches [0, cut) and [cut, S) chain through q_cur, eps, the reject counters and the in/out accumulators, and
    take their slot indices from the absolute iteration: the same bytes as one launch (cut = burn + 1 starts the second
    window on the first stored iteration, whose reject path reloads params_init)."""
    model, x, y = cases.mlp_problem(seed=3, n=192, n_in=6, hidden=16)
    nt = engine.NativeTarget(_descs(model, x, y, 3), 'cuda')
    init = _init(model, 4, scale=0.1)
    kw = dict(S=16, burn=3, L=4, step=0.02, thin=2, seed=5, scheme=N.SCHEME_SPLIT_SYM)
    one = _split_run_sink(nt, init, windows=[(0, 16)], **kw)
    two = _split_run_sink(nt, init, windows=[(0, cut), (cut, 16)], **kw)
    for k in one:
        assert torch.equal(_bits(one[k]) if one[k].is_floating_point() else one[k],
                           _bits(two[k]) if two[k].is_floating_point() else two[k]), k
