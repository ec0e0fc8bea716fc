"""CPU: replica exchange for Bayesian NNs (DESIGN §3.17) -- the refusals raised before any CUDA work, the even-odd swap
schedule, the swap stream's Philox counters, the oracle without swaps against independent runs, the ladder sharding of
the multi-GPU call and the C-ABI argument checks."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import engine, samplers, targets as T
from oracle import cases, hmc_oracle as O
from tests import philox_ref as P
from tests import temper_oracle as TO

STREAM_SWAP = 5


def _reg(n=24, hidden=4, task='regression', tau_out=10.):
    model, x, y = cases.mlp_problem(seed=1, n=n, n_in=3, hidden=hidden, task=task)
    loss = {'regression': 'regression', 'binary': 'binary_class_linear_output'}[task]
    return T.MLPTarget.from_model(model, x, y, None, tau_out, model_loss=loss), model


def _q0(model, C_):
    return hb.util.flatten(model).detach()[None].repeat(C_, 1)


def test_refusals_before_any_cuda_work():
    tgt, model = _reg()
    q0 = _q0(model, 4)
    run = lambda lp=tgt, q=q0, num_samples=10, **kw: samplers.sample_chains(lp, q, num_samples=num_samples, **kw)
    b = [1.0, 0.5]
    with pytest.raises(NotImplementedError, match='Bayesian-NN targets only'):
        run(T.GaussianIso(3), torch.zeros(4, 3), betas=b)
    with pytest.raises(NotImplementedError, match='HMC or HMC_NUTS'):
        run(sampler=samplers.Sampler.RMHMC, betas=b)
    with pytest.raises(NotImplementedError, match='inv_mass None or 1-D'):
        run(inv_mass=torch.eye(tgt.dim), betas=b)
    with pytest.raises(NotImplementedError, match='inv_mass None or 1-D'):
        run(inv_mass=[torch.eye(tgt.dim)], betas=b)
    with pytest.raises(NotImplementedError, match='adapt_mass'):
        run(sampler=samplers.Sampler.HMC_NUTS, num_samples=60, burn=30, num_steps_per_sample=2, adapt_mass=True, betas=b)
    with pytest.raises(NotImplementedError, match='hyperpriors'):
        run(tau_prior=(1.0, 1.0), betas=b)
    with pytest.raises(NotImplementedError, match='hyperpriors'):
        run(tau_out_prior=(1.0, 1.0), betas=b)
    with pytest.raises(NotImplementedError, match='reference'):
        run(rng='reference', betas=b)
    for bad in ([0.9, 0.5], [1.0, 1.0], [1.0, 0.5, 0.7], [1.0, -0.1], [1.0, math.nan], [1.0, math.inf], [],
                [1.0] + [0.5 ** k for k in range(1, 40)], 'ab'):
        with pytest.raises(ValueError):
            run(betas=bad)
    with pytest.raises(ValueError, match='multiple of T'):
        run(tgt, _q0(model, 3), betas=b)
    with pytest.raises(ValueError, match='chain_offset'):
        run(betas=b, chain_offset=3)
    for se in (0, -1, 2.5, True):
        with pytest.raises(ValueError, match='swap_every'):
            run(betas=b, swap_every=se)
    z, lu = torch.zeros(10, 4, tgt.dim), torch.zeros(10, 4)
    with pytest.raises(ValueError, match='swap_log_uniforms'):
        run(betas=b, rng='injected', normals=z, log_uniforms=lu, swap_every=3)
    with pytest.raises(ValueError, match='swap_log_uniforms'):
        run(betas=b, rng='injected', normals=z, log_uniforms=lu, swap_every=3,
            swap_log_uniforms=torch.zeros(3, 2, 2, dtype=torch.float64))


def test_accepted_arguments_build_the_temper_dict():
    tgt, model = _reg()
    t = samplers._temper_args([tgt, tgt], _q0(model, 6), 31, samplers.Sampler.HMC_NUTS, torch.ones(tgt.dim), False,
                              None, 'philox', 3, torch.tensor([1.0, 0.4, 0.0], dtype=torch.float64), 10, torch.zeros(1))
    assert t == dict(betas=[1.0, 0.4, 0.0], swap_every=10, swap_log_uniforms=None)
    assert samplers._temper_args(tgt, _q0(model, 2), 10, samplers.Sampler.HMC, None, False, None, 'philox', 0, None, 10,
                                 None) is None


@pytest.mark.parametrize('S,E,rounds', [(30, 10, 2), (31, 10, 3), (10, 10, 0), (10, 11, 0), (5, 1, 4), (1, 1, 0)])
def test_round_count(S, E, rounds):
    assert engine.swap_rounds(S, E) == rounds == TO.num_rounds(S, E)


def test_even_odd_schedule():
    assert TO.swap_pairs(0, 5) == [0, 2] and TO.swap_pairs(1, 5) == [1, 3] and TO.swap_pairs(2, 5) == [0, 2]
    assert TO.swap_pairs(0, 2) == [0] and TO.swap_pairs(1, 2) == [] and TO.swap_pairs(3, 4) == [1]
    for k in range(4):                   # the pairs of a round are disjoint; two rounds in a row cover every neighbour
        p = TO.swap_pairs(k, 7)
        rows = [t for t in p] + [t + 1 for t in p]
        assert len(rows) == len(set(rows))
        assert sorted(TO.swap_pairs(k, 7) + TO.swap_pairs(k + 1, 7)) == list(range(6))


def test_swap_stream_counters_are_distinct_from_the_other_streams():
    # counter (t, k_lo, k_hi | 5 << 24, ladder_lo): the stream byte keeps it off every (vec, n, chain) of streams 0-4
    t, k, ladder = np.meshgrid(np.arange(4), np.arange(6), np.array([0, 1, 2 ** 32 + 1]), indexing='ij')
    sw = P.counter(STREAM_SWAP, t, k, ladder).reshape(-1, 4)
    assert np.all((sw[:, 2] >> np.uint64(24)) == STREAM_SWAP)
    for s in range(5):
        other = P.counter(s, t, k, ladder).reshape(-1, 4)
        assert not set(map(tuple, sw.tolist())) & set(map(tuple, other.tolist()))
    # ladders 1 and 2^32 + 1 share the counter and differ in the key
    w = P.draw(7, np.array([1, 2 ** 32 + 1]), 0, 0, STREAM_SWAP)
    assert w[0, 0] != w[1, 0]
    logu = np.log(P.u01(P.draw(7, 3, 2, 1, STREAM_SWAP)[..., 0]).astype(np.float64))
    assert -30 < float(logu) < 0


def test_decision_rule():
    assert TO.swap_decision(1.0, 0.5, -10.0, -8.0, math.log(0.99))          # the hotter state fits better: always
    assert not TO.swap_decision(1.0, 0.5, -8.0, -28.0, math.log(0.5))       # exp(-10) < 0.5
    assert TO.swap_decision(1.0, 0.5, -8.0, -9.0, math.log(0.5))            # exp(-0.5) > 0.5
    assert not TO.swap_decision(1.0, 0.5, math.nan, -9.0, -1.0)


@pytest.mark.parametrize('scheme', [None, O.SPLIT_SYM])
def test_oracle_without_swaps_matches_independent_runs(scheme):
    tgt, model = _reg(n=24)
    if scheme is not None:
        tgt = [T.MLPTarget(tgt.widths, tgt.acts, tgt.x[a:a + 12], tgt.y[a:a + 12], tgt.tau_list, 10., 2)
               for a in (0, 12)]
    betas, R, S, L, burn, eps = [1.0, 0.3], 2, 8, 3, 2, 0.05
    Tn = len(betas)
    g = torch.Generator().manual_seed(4)
    D = hb.util.flatten(model).numel()
    q0 = hb.util.flatten(model).detach()[None] + 0.05 * torch.randn(R * Tn, D, generator=g)
    z = torch.randn(S, R * Tn, D, generator=g)
    lu = torch.log(torch.rand(S, R * Tn, generator=g))
    lu[burn + 1], lu[S - 2] = 0.0, 0.0                      # reject unless H fell: the first-stored-iteration quirk runs
    o = TO.sample_tempered(tgt, betas, q0, S, L, eps, burn, S, z, lu, np.zeros((0, R, Tn - 1)), split_scheme=scheme)
    assert o['swap_accepted'].shape == (0, R, Tn - 1)
    for c in range(R * Tn):
        ref = O.sample_hmc(TO.tempered(tgt, betas[c % Tn]), q0[c], S, L, eps, burn, split_scheme=scheme,
                           normals=z[:, c], log_uniforms=lu[:, c])
        assert o['accepted'][c] == ref['accepted']
        if c % Tn == 0:
            assert torch.equal(o['samples'][c // Tn], torch.stack(ref['samples']))
    assert any(not a for row in o['accepted'] for a in row)               # the rejection branch ran


def test_tempered_target_scales_tau_out_only():
    tgt, model = _reg(task='binary', tau_out=3.0)
    hot = TO.tempered(tgt, 0.1)
    assert hot.tau_out == 0.1 * 3.0 and hot.model_loss == tgt.model_loss
    assert all(float(a) == float(b) for a, b in zip(hot.log_scale, tgt.log_scale))
    q = hb.util.flatten(model).detach()
    ll = TO.loglik(tgt, q)
    expect = -float(np.float32(3.0)) * float(torch.nn.BCEWithLogitsLoss(reduction='sum')(
        tgt.forward(q, tgt.x).double(), tgt.y.double().view(-1, 1)))
    assert ll == pytest.approx(expect, rel=1e-12)


# ------------------------------------------------------------------------------------------------------------------
# multi-GPU routing (gloo, world 2): ladders, not chains, are partitioned
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
        seen['rows'] = q0[:, 0].tolist()
        r = Res()
        C_ = q0.shape[0]
        r.num_rejected, r.step_size, r.dim = q0[:, 0].to(torch.int32), q0[:, 0].clone(), 2
        r.samples_padded = q0[::3, None, :].repeat(1, 2, 1)           # the beta = 1 rows
        r.moment_sum, r.moment_sumsq, r.moment_count = q0.double(), q0.double() ** 2, 1
        return r
    q0 = torch.arange(18.0).reshape(9, 2)                  # R = 3 ladders of T = 3 rows
    lu = torch.arange(4 * 3 * 2, dtype=torch.float64).reshape(4, 3, 2)
    z = torch.zeros(5, 9, 2)
    o = Dd.sample_chains_sharded(None, q0, gather_samples=True, runner=runner, betas=[1.0, 0.5, 0.2],
                                 swap_log_uniforms=lu, normals=z, chain_offset=6)
    out[rank] = (seen['rows'], seen['chain_offset'], seen['swap_log_uniforms'].tolist(), seen['normals'].shape[1],
                 o['num_rejected'].tolist(), o['samples'][:, 0, 0].tolist(), o['bounds'], o['posterior_mean'].tolist())
    dist.destroy_process_group()


def test_sharded_call_partitions_ladders():
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    out = mp.Manager().dict()
    mp.spawn(_worker, args=(port, out), nprocs=2, join=True)
    lu = torch.arange(4 * 3 * 2, dtype=torch.float64).reshape(4, 3, 2)
    for r, (ladders, rows) in enumerate([((0, 1), list(range(0, 3))), ((1, 3), list(range(3, 9)))]):
        seen_rows, off, slu, ncols, rej, cold, bounds, mean = out[r]
        assert seen_rows == [2.0 * i for i in rows] and bounds == (rows[0], rows[-1] + 1)
        assert off == 6 + rows[0] and ncols == len(rows)
        assert slu == lu[:, ladders[0]:ladders[1]].tolist()
        assert rej == [2 * i for i in range(9)]
        assert cold == [0.0, 6.0, 12.0]
        assert mean == [6.0, 7.0]                              # pooled over the beta = 1 rows only


# ------------------------------------------------------------------------------------------------------------------
# C ABI: argument checks return before any CUDA work
# ------------------------------------------------------------------------------------------------------------------
def test_abi_temper_entries_check_their_arguments(built_library):
    from hamiltorch_b200 import _native as N
    from hamiltorch_b200.engine import NativeTarget
    lib = N.load_library()
    tgt, _ = _reg()
    junk = C.c_void_p(16)
    nt = NativeTarget(tgt, 'cpu')
    ld = N.padded_ld(nt.dim)

    def temper(taus, T_=None):
        t = N.TemperStruct()
        t.num_temps = len(taus) if T_ is None else T_
        for i, v in enumerate(taus):
            t.tau_out[i] = v
        return t

    def run(tp, C_=4, hyper=None):
        rng = N.RngStruct()
        rng.mode = N.RNG_PHILOX
        return lib.hmcx_split_run_temper(nt.ref(), None, C.byref(rng), C.byref(N.NutsStruct()), 0, junk, junk, junk, C_,
                                         ld, 3, 10, 2, 0, 10, junk, junk, junk, None, junk, None,
                                         None if tp is None else C.byref(tp), None)

    assert run(None) == N.ERR_INVALID_ARG
    for bad in (temper([], 0), temper([10.0], 33), temper([10.0, 5.0, 1.0]), temper([10.0, -1.0]),
                temper([10.0, math.inf]), temper([10.0, math.nan]), temper([5.0, 10.0])):
        assert run(bad) == N.ERR_INVALID_ARG
    gauss = NativeTarget(T.GaussianIso(4), 'cpu')
    rng = N.RngStruct()
    rng.mode = N.RNG_PHILOX
    assert lib.hmcx_split_run_temper(gauss.ref(), None, C.byref(rng), C.byref(N.NutsStruct()), 0, junk, junk, junk, 4, 4,
                                     3, 10, 2, 0, 10, junk, junk, junk, None, junk, None, C.byref(temper([1.0, 0.5])),
                                     None) == N.ERR_UNSUPPORTED

    betas = (C.c_double * 3)(1.0, 0.5, 0.1)

    def swap(q=C.c_void_p(256), C_=6, ld_=8, T_=3, b=betas, ll=junk, rnd=0, mode=N.RNG_PHILOX, off=0, lu=None, acc=junk):
        r = N.RngStruct()
        r.mode, r.chain_offset = mode, off
        return lib.hmcx_temper_swap(q, C_, ld_, T_, b, ll, rnd, C.byref(r), lu, acc, None)

    for kw in (dict(q=None), dict(q=C.c_void_p(260)), dict(C_=0), dict(C_=5), dict(T_=1), dict(T_=33), dict(ld_=6),
               dict(ld_=0), dict(b=None), dict(ll=None), dict(acc=None), dict(rnd=-1), dict(off=4),
               dict(mode=N.RNG_INJECTED), dict(mode=7), dict(b=(C.c_double * 3)(0.9, 0.5, 0.1)),
               dict(b=(C.c_double * 3)(1.0, 0.5, 0.5)), dict(b=(C.c_double * 3)(1.0, 0.5, -0.1)),
               dict(b=(C.c_double * 3)(1.0, math.nan, 0.1))):
        assert swap(**kw) == N.ERR_INVALID_ARG, kw
