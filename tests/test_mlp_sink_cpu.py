"""CPU: host-side routing of the Bayesian-NN sample sink (thin / moments / keep_samples / store_on_GPU=False reach the
engine for MLP targets and split lists; the other kernels keep refusing them) and the argument checks of
hmcx_split_run_sink, which return before any CUDA work."""
import ctypes as C

import pytest
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import engine, samplers, targets as T, _native as N
from oracle import cases


class _Routed(Exception):
    pass


@pytest.fixture
def routed(monkeypatch):
    """engine.hmc_run replaced by a stub that raises with the keyword arguments it was called with."""
    def stub(*args, **kw):
        raise _Routed(kw)
    monkeypatch.setattr(engine, 'hmc_run', stub)

    def call(fn, *args, **kw):
        with pytest.raises(_Routed) as e:
            fn(*args, **kw)
        return e.value.args[0]
    return call


def _mlp(splits):
    model, x, y = cases.mlp_problem(seed=1, n=48)
    descs = [T.MLPTarget.from_model(model, x[16 * m:16 * (m + 1)], y[16 * m:16 * (m + 1)], None, 50., prior_scale=splits)
             for m in range(splits)]
    return descs, torch.zeros(2, descs[0].dim)


def test_bnn_sink_options_reach_the_engine(routed):
    descs, init = _mlp(3)
    plain = T.MLPTarget.from_model(*cases.mlp_problem(seed=1, n=48), None, 50.)
    kw = routed(hb.sample_chains, plain, init, num_samples=9, thin=3, moments=True, keep_samples=False)
    assert kw['scheme'] == N.SCHEME_PLAIN and kw['thin'] == 3 and kw['moments'] and not kw['keep_samples']
    for integ, scheme in ((hb.Integrator.SPLITTING, N.SCHEME_SPLIT_SYM), (hb.Integrator.SPLITTING_RAND, N.SCHEME_SPLIT_RAND),
                          (hb.Integrator.SPLITTING_KMID, N.SCHEME_SPLIT_KMID)):
        kw = routed(hb.sample_chains, descs, init, num_samples=9, integrator=integ, store_on_GPU=False, thin=2,
                    sampler=hb.Sampler.HMC_NUTS, burn=2)
        assert kw['scheme'] == scheme and kw['host_samples'] and kw['thin'] == 2 and kw['nuts']
    # the one-chain drop-in: store_on_GPU=False streams into pinned host memory; store_on_GPU=True asks for no sink
    kw = routed(hb.sample, descs, init[0], integrator=hb.Integrator.SPLITTING, store_on_GPU=False, rng='philox')
    assert kw['host_samples']
    kw = routed(hb.sample, plain, init[0], store_on_GPU=False, rng='philox', inv_mass=torch.ones(init.shape[1]))
    assert kw['host_samples'] and kw['scheme'] == N.SCHEME_PLAIN
    kw = routed(hb.sample, descs, init[0], integrator=hb.Integrator.SPLITTING, rng='philox')
    assert 'host_samples' not in kw


def test_sink_predicate():
    descs, init = _mlp(2)
    D = init.shape[1]
    ok = samplers._sink_supported
    assert ok(descs, hb.Sampler.HMC, hb.Integrator.SPLITTING, None)
    assert ok(descs[0], hb.Sampler.HMC_NUTS, hb.Integrator.IMPLICIT, torch.ones(D))
    assert ok(T.GaussianDiag(torch.zeros(4), torch.ones(4)), hb.Sampler.HMC, hb.Integrator.IMPLICIT, None)
    assert not ok(descs, hb.Sampler.HMC, hb.Integrator.IMPLICIT, None)              # a list needs a SPLITTING integrator
    assert not ok(descs[0], hb.Sampler.HMC, hb.Integrator.SPLITTING, None)
    assert not ok(descs, hb.Sampler.HMC, hb.Integrator.SPLITTING, torch.eye(D))     # full mass: no BNN kernel for it
    assert not ok(descs, hb.Sampler.RMHMC, hb.Integrator.SPLITTING, None)
    assert not ok(T.GaussianFull(torch.zeros(4), cov=torch.eye(4, dtype=torch.float64)), hb.Sampler.HMC,
                  hb.Integrator.IMPLICIT, None)
    assert not ok(T.Funnel(3), hb.Sampler.HMC, hb.Integrator.IMPLICIT, None)
    with pytest.raises(NotImplementedError):
        hb.sample_chains(descs, init, num_samples=5, integrator=hb.Integrator.SPLITTING, inv_mass=torch.eye(D), thin=2)


def test_split_run_sink_argument_checks_without_cuda(built_library):
    lib = N.load_library()
    descs, _ = _mlp(2)
    nt = engine.NativeTarget(descs, 'cpu')
    ld = N.padded_ld(nt.dim)
    mass, rng, nuts = N.MassStruct(), N.RngStruct(), N.NutsStruct()
    rng.mode = N.RNG_PHILOX
    buf = (C.c_float * 16)()

    def run(target, sink, ld=ld):
        return lib.hmcx_split_run_sink(target, C.byref(mass), C.byref(rng), C.byref(nuts), N.SCHEME_SPLIT_SYM, None, None,
                                       None, 2, ld, 3, 10, 0, 0, 10, None, None, None, None, None, sink, None)

    sink = N.SinkStruct()
    sink.thin = 0
    assert run(nt.ref(), C.byref(sink)) == N.ERR_INVALID_ARG
    sink.thin = 1
    sink.sum_lo = C.addressof(buf)                                 # compensation terms without the sums
    assert run(nt.ref(), C.byref(sink)) == N.ERR_INVALID_ARG
    sink.sum_lo, sink.sumsq_lo = None, C.addressof(buf)
    assert run(nt.ref(), C.byref(sink)) == N.ERR_INVALID_ARG
    sink.sumsq_lo = None
    assert run(None, C.byref(sink)) == N.ERR_INVALID_ARG
    other = N.TargetStruct()
    other.kind, other.dim = T.GaussianIso.kind, 8
    assert run(C.byref(other), C.byref(sink)) == N.ERR_UNSUPPORTED   # the sink of element-wise targets is hmcx_hmc_run_sink
    # a well-formed sink goes on to the run's own argument checks (ld % 4 != 0, NULL state), as NULL does
    assert run(nt.ref(), C.byref(sink), ld=ld + 1) == N.ERR_INVALID_ARG
    assert run(nt.ref(), None, ld=ld + 1) == N.ERR_INVALID_ARG
