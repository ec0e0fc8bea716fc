"""CPU: Gamma hyperpriors on tau_list / tau_out (DESIGN §3.15) -- the oracle's conditional update, the refusals raised
before any CUDA work, the C-ABI argument checks and the sharded call's routing."""
import ctypes as C
import math

import numpy as np
import pytest
import scipy.stats
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import samplers, targets as T
from oracle import cases
from tests import hyper_oracle as H


def _reg(n=40, hidden=6, task='regression', tau_out=10.):
    model, x, y = cases.mlp_problem(seed=1, n=n, n_in=3, hidden=hidden, task=task)
    loss = {'regression': 'regression', 'binary': 'binary_class_linear_output'}[task]
    return T.MLPTarget.from_model(model, x, y, None, tau_out, model_loss=loss), model


def test_conditional_update_matches_scipy_gamma():
    tgt, model = _reg()
    q = hb.util.flatten(model).detach() * 1.7
    hyper = [(2.0, 0.5), None, (0.3, 1.5), (1.0, 1.0), (3.0, 4.0)]
    u = np.array([0.1, 0.5, 0.7, 0.25, 0.9])
    sizes, off, g = H.tensor_sizes(tgt), 0, np.zeros(5)
    expect = {}
    for k, n in enumerate(sizes):
        w = q[off:off + n].double().numpy()
        off += n
        if hyper[k] is not None:
            shape, rate = hyper[k][0] + n / 2, hyper[k][1] + (w @ w) / 2
            g[k] = scipy.stats.gamma(shape).ppf(u[k])
            expect[k] = scipy.stats.gamma(shape, scale=1 / rate).ppf(u[k])
    out = tgt.forward(q, tgt.x).double()
    sse = float(((out - tgt.y.double().view_as(out)) ** 2).sum())
    shape, rate = 3.0 + tgt.x.shape[0] / 2, 4.0 + sse / 2
    g[4] = scipy.stats.gamma(shape).ppf(u[4])
    tau_list, tau_out = H.gibbs_update(tgt, q, hyper, [1.0] * 4, 10.0, g)
    for k, v in expect.items():
        assert tau_list[k] == pytest.approx(v, rel=1e-6)
    assert tau_list[1] == 1.0
    assert tau_out == pytest.approx(scipy.stats.gamma(shape, scale=1 / rate).ppf(u[4]), rel=1e-6)


def test_rebuilt_target_carries_the_new_constants():
    tgt, model = _reg()
    new = H.rebuild([tgt, tgt], [2.0, 3.0, 4.0, 5.0], 7.0)
    assert len(new) == 2 and new[0].tau_out == 7.0
    ref = T.MLPTarget.from_model(model, tgt.x, tgt.y, [torch.tensor(v) for v in (2.0, 3.0, 4.0, 5.0)], 7.0)
    assert all(float(a) == float(b) for a, b in zip(new[1].log_scale, ref.log_scale))


def test_group_list_and_refusals():
    tgt, _ = _reg()
    g = samplers._hyper_groups(tgt, samplers.Sampler.HMC, (1.0, 2.0), (3.0, 4.0))
    assert g == [(1.0, 2.0)] * 4 + [(3.0, 4.0)]
    g = samplers._hyper_groups([tgt, tgt], samplers.Sampler.HMC_NUTS, [None, (1, 1), None, (2, 2)], None)
    assert g == [None, (1.0, 1.0), None, (2.0, 2.0), None]
    assert samplers._hyper_groups(tgt, samplers.Sampler.HMC, None, None) is None
    with pytest.raises(ValueError, match='one entry per parameter tensor'):
        samplers._hyper_groups(tgt, samplers.Sampler.HMC, [(1, 1)] * 3, None)
    for bad in ((0.0, 1.0), (1.0, -1.0), (math.inf, 1.0), (1.0, math.nan), (1.0,)):
        with pytest.raises(ValueError):
            samplers._hyper_groups(tgt, samplers.Sampler.HMC, bad, None)
    with pytest.raises(ValueError):
        samplers._hyper_groups(tgt, samplers.Sampler.HMC, None, (1.0, 0.0))
    cls, _ = _reg(task='binary')
    assert samplers._hyper_groups(cls, samplers.Sampler.HMC, (1.0, 1.0), None)[-1] is None
    with pytest.raises(NotImplementedError, match='regression only'):
        samplers._hyper_groups(cls, samplers.Sampler.HMC, None, (1.0, 1.0))
    with pytest.raises(NotImplementedError, match='Bayesian-NN targets only'):
        samplers._hyper_groups(T.GaussianIso(4), samplers.Sampler.HMC, (1.0, 1.0), None)
    with pytest.raises(NotImplementedError, match='HMC or HMC_NUTS'):
        samplers._hyper_groups(tgt, samplers.Sampler.RMHMC, (1.0, 1.0), None)
    prior_only = T.MLPTarget(tgt.widths, tgt.acts, None, None, tgt.tau_list)
    with pytest.raises(RuntimeError, match='needs data'):
        samplers._hyper_groups(prior_only, samplers.Sampler.HMC, None, (1.0, 1.0))


def test_public_entries_refuse_before_cuda():
    tgt, model = _reg()
    q0 = hb.util.flatten(model).detach()
    with pytest.raises(NotImplementedError, match='Bayesian-NN targets only'):
        samplers.sample_chains(T.GaussianIso(3), torch.zeros(2, 3), tau_prior=(1.0, 1.0))
    with pytest.raises(NotImplementedError):
        samplers.sample(tgt, q0, sampler=samplers.Sampler.RMHMC, tau_prior=(1.0, 1.0))
    with pytest.raises(ValueError):
        samplers.sample_chains(tgt, q0[None], tau_prior=[(1.0, 1.0)])


def test_reference_stream_draws_gammas_after_rand():
    shapes = torch.tensor([0.0, 2.5, 0.0, 7.0], dtype=torch.float64)
    torch.manual_seed(3)
    z, logu, gam = samplers._draw_reference_stream(5, 3, 'cpu', gamma_shapes=shapes)
    torch.manual_seed(3)
    for n in range(3):
        assert torch.equal(z[n], torch.randn(5))
        assert float(logu[n]) == float(torch.log(torch.rand(1))[0])
        assert torch.equal(gam[n, [1, 3]], torch._standard_gamma(shapes[[1, 3]]))
    assert bool((gam[:, [0, 2]] == 0).all())


def test_posterior_shapes_count_every_split_row():
    tgt, _ = _reg(n=40)
    a = [T.MLPTarget(tgt.widths, tgt.acts, tgt.x[:25], tgt.y[:25], tgt.tau_list, 10., 2),
         T.MLPTarget(tgt.widths, tgt.acts, tgt.x[25:], tgt.y[25:], tgt.tau_list, 10., 2)]
    sh = samplers._reference_gamma_shapes(a, [(1.0, 1.0), None, None, (2.0, 1.0), (3.0, 1.0)])
    assert sh.tolist() == [1.0 + 0.5 * tgt.sizes[0], 0.0, 0.0, 2.0 + 0.5 * tgt.sizes[3], 3.0 + 0.5 * 40]


# ------------------------------------------------------------------------------------------------------------------
# C ABI: argument checks return before any CUDA work
# ------------------------------------------------------------------------------------------------------------------
def test_abi_hyper_entries_check_their_arguments(built_library):
    from hamiltorch_b200 import _native as N
    from hamiltorch_b200.engine import NativeTarget
    lib = N.load_library()
    tgt, _ = _reg()
    cls, _ = _reg(task='binary')
    junk = C.c_void_p(16)

    def run(nt=None, hyper=None, mode=N.RNG_PHILOX):
        nt = nt or NativeTarget(tgt, 'cpu')
        rng = N.RngStruct()
        rng.mode = mode
        rng.normals = rng.log_uniforms = 16
        nuts = N.NutsStruct()
        D = nt.dim
        ld = N.padded_ld(D)
        return lib.hmcx_split_run_hyper(nt.ref(), None, C.byref(rng), C.byref(nuts), 0, junk, junk, junk, 2, ld, 3, 10, 2,
                                        0, 10, junk, junk, junk, None, junk, None, None if hyper is None else C.byref(hyper),
                                        None)

    def hyp(**kw):
        h = N.HyperStruct()
        h.tau, h.tau_out = 16, 16
        for k, (a, b) in kw.get('groups', {0: (1.0, 1.0)}).items():
            h.sampled[k], h.a[k], h.b[k] = 1, a, b
        if 'gammas' in kw:
            h.gammas = kw['gammas']
        if kw.get('no_tau'):
            h.tau = None
        return h

    for bad in (dict(groups={0: (0.0, 1.0)}), dict(groups={1: (1.0, -2.0)}), dict(groups={2: (math.inf, 1.0)}),
                dict(groups={3: (1.0, math.nan)}), dict(groups={5: (1.0, 1.0)}), dict(no_tau=True)):
        assert run(hyper=hyp(**bad)) == N.ERR_INVALID_ARG, bad
    assert run(hyper=hyp(), mode=N.RNG_INJECTED) == N.ERR_INVALID_ARG            # injected without gammas
    assert run(NativeTarget(cls, 'cpu'), hyp(groups={4: (1.0, 1.0)})) == N.ERR_UNSUPPORTED
    nodata = NativeTarget(T.MLPTarget(tgt.widths, tgt.acts, None, None, tgt.tau_list), 'cpu')
    assert run(nodata, hyp(groups={4: (1.0, 1.0)})) == N.ERR_INVALID_ARG

    sh = (C.c_double * 3)(1.0, 2.0, 0.5)
    ok = (16, 0, 4, 0, 10, 3, sh, junk, None)
    for i, v in ((2, 0), (3, -1), (4, 0), (5, 0), (5, N.HYPER_GROUPS + 1), (6, None), (7, None)):
        args = list(ok)
        args[i] = v
        assert lib.hmcx_hyper_gamma_draws(*args) == N.ERR_INVALID_ARG, (i, v)
    bad_shape = (C.c_double * 3)(1.0, 0.0, 0.5)
    assert lib.hmcx_hyper_gamma_draws(16, 0, 4, 0, 10, 3, bad_shape, junk, None) == N.ERR_INVALID_ARG


# ------------------------------------------------------------------------------------------------------------------
# multi-GPU routing (gloo, world 2): the injected gamma stream is sliced and the traces gathered with the samples
# ------------------------------------------------------------------------------------------------------------------
def _worker(rank, port, out):
    import os
    import torch.distributed as dist
    from hamiltorch_b200 import distributed as Dd
    os.environ['MASTER_ADDR'], os.environ['MASTER_PORT'] = '127.0.0.1', str(port)
    dist.init_process_group('gloo', rank=rank, world_size=2)
    seen = {}

    class Res:
        pass

    def runner(lp, q0, **kw):
        seen.update(kw)
        r = Res()
        C_ = q0.shape[0]
        r.num_rejected, r.step_size, r.dim = torch.zeros(C_, dtype=torch.int32), torch.ones(C_), 2
        r.samples_padded = q0[:, None, :].repeat(1, 3, 1)
        r.tau_list_trace = q0[:, :1, None].repeat(1, 3, 4)
        r.tau_out_trace = q0[:, :1].repeat(1, 3)
        return r
    q0 = torch.arange(8.0).reshape(4, 2)
    gam = torch.arange(5 * 4 * 5, dtype=torch.float64).reshape(5, 4, 5)
    o = Dd.sample_chains_sharded(None, q0, gather_samples=True, runner=runner, tau_prior=(1.0, 2.0), gammas=gam)
    out[rank] = (seen['tau_prior'], seen['gammas'].shape[1], float(seen['gammas'][0, 0, 0]),
                 o['tau_list_trace'][:, 0, 0].tolist(), o['tau_out_trace'][:, 0].tolist())
    dist.destroy_process_group()


def test_sharded_call_routes_the_hyper_arguments():
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    out = mp.Manager().dict()
    mp.spawn(_worker, args=(port, out), nprocs=2, join=True)
    for r in range(2):
        prior, cols, first, tl, to = out[r]
        assert prior == (1.0, 2.0) and cols == 2 and first == float(r * 2 * 5)
        assert tl == [0.0, 2.0, 4.0, 6.0] and to == [0.0, 2.0, 4.0, 6.0]


def test_loo_takes_one_tau_out_per_draw():
    from hamiltorch_b200 import loo

    class Res:
        tau_out_trace = torch.tensor([[10.0, 12.5, 9.0]])
    x = torch.zeros(1, 3, 5)
    assert torch.equal(loo._tau_block(Res(), x, None), Res.tau_out_trace)
    assert loo._tau_block(object(), x, None) is None
    assert loo._tau_block(None, x, [1.0, 2.0, 3.0]).shape == (1, 3)
    with pytest.raises(RuntimeError, match='one value per draw'):
        loo._tau_block(None, x, [1.0, 2.0])
    with pytest.raises(ValueError, match='positive'):
        loo._tau_block(None, x, [1.0, -2.0, 3.0])
    with pytest.raises(RuntimeError, match='not to a log-likelihood block'):
        loo._prepare(torch.zeros(1, 4, 3), None, tau_out=[1.0] * 4)
