"""CPU: diagonal-mass adaptation during HMC_NUTS warm-up (sample_chains(adapt_mass=True)) -- the window schedule, the
restarted dual-averaging table, the test-side definition in tests/adapt_oracle.py on hand-worked cases, every refusal
(raised on the host before any CUDA work), the argument checks of hmcx_adapt_diag_mass and the multi-GPU pooling over
gloo."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import hamiltorch_b200 as hb
from hamiltorch_b200 import distributed as DI, engine, targets as T, _native as N
from tests import adapt_oracle as A


@pytest.mark.parametrize('burn,windows', [
    (1000, [(75, 100), (100, 150), (150, 250), (250, 450), (450, 950)]),
    (150, [(75, 100)]),                     # 75 + 25 + 50 == burn: the default buffers still fit
    (100, [(15, 90)]),                      # buffers int(0.15 * 100) and int(0.1 * 100), one window of what remains
    (20, [(3, 18)]),
    # the next doubled window ending exactly at burn - 50 does not cross into the terminal buffer: no stretch (Stan)
    (300, [(75, 100), (100, 150), (150, 250)]),
    (500, [(75, 100), (100, 150), (150, 250), (250, 450)]),
    (900, [(75, 100), (100, 150), (150, 250), (250, 450), (450, 850)]),
    (1700, [(75, 100), (100, 150), (150, 250), (250, 450), (450, 850), (850, 1650)]),
    (400, [(75, 100), (100, 150), (150, 350)]),   # 250 + 2 * 200 crosses 350: the third window is stretched
])
def test_mass_windows_hand_worked_cases(burn, windows):
    assert engine.mass_windows(burn) == windows


def _stan_windows(burn):
    """Stan's windowed_adaptation (restart / compute_next_window / end_adaptation_window) restated with its own inclusive
    last-index bookkeeping, run over the warm-up iterations: the slow windows as [a, b) ranges."""
    init, term, base = 75, 50, 25
    if init + term + base > burn:
        init, term = int(0.15 * burn), int(0.1 * burn)
        base = burn - (init + term)
    size, nxt, start, out = base, init + base - 1, init, []
    for counter in range(burn):
        if counter == nxt and counter < burn - term:                 # end_adaptation_window()
            out.append((start, counter + 1))
            start = counter + 1
            if nxt != burn - term - 1:                               # compute_next_window()
                size *= 2
                nxt = counter + size
                if nxt != burn - term - 1 and nxt + 2 * size >= burn - term:
                    nxt = burn - term - 1
    return out


def test_mass_windows_follow_stan_for_every_burn():
    for burn in range(20, 3001):
        assert engine.mass_windows(burn) == _stan_windows(burn), burn


def test_mass_windows_refuse_burn_below_20():
    with pytest.raises(RuntimeError, match='burn >= 20'):
        engine.mass_windows(19)


def test_restarted_table_rows():
    t = engine.nuts_table_restarted(1000)
    plain = engine.nuts_table(1000)
    assert t.shape == plain.shape == (1001, 5)
    assert torch.equal(t[:100], plain[:100])                 # t = n + 1 until the first window ends
    for b, nxt in ((100, 150), (150, 250), (250, 450), (450, 950), (950, 1001)):
        assert torch.equal(t[b:nxt], plain[:nxt - b])        # row n >= b holds t = n - b + 1


def test_comp_add_restatement_on_hand_cases():
    s, c = np.float32(0), np.float32(0)
    for x in (1e8, 1.0, -1e8):                               # the 1 is lost by a plain fp32 sum
        s, c = A.comp_add(s, c, x)
    assert float(s) + float(c) == 1.0
    acc = A.Sums(1)
    for x in (3.0, 1e4, -1e4):
        acc.add([x])
    assert float(acc.s[0]) + float(acc.c[0]) == 3.0
    assert float(acc.q[0]) + float(acc.cq[0]) == 9.0 + 2e8
    # |mean| >> std: the compensated sums carry the variance that a plain fp32 sum of squares loses
    g = np.random.default_rng(0)
    x = (1000.0 + g.standard_normal((4000, 3))).astype(np.float32)
    acc = A.Sums(3)
    for row in x:
        acc.add(row)
    s1 = acc.s.astype(np.float64) + acc.c
    s2 = acc.q.astype(np.float64) + acc.cq
    x64 = x.astype(np.float64)
    np.testing.assert_allclose(s1, x64.sum(0), rtol=1e-12)
    var = (s2 - s1 * (s1 / 4000)) / 3999
    np.testing.assert_allclose(var, x64.var(0, ddof=1), rtol=1e-4)


def test_pooled_estimator_hand_case():
    # chain 0 draws 1, 2, 3 (variance 1), chain 1 draws 2, 4, 6 (variance 4): W = 2.5, N = 6
    s = np.array([[6.0], [12.0]], np.float32)
    sq = np.array([[14.0], [56.0]], np.float32)
    z = np.zeros_like(s)
    im, mf = A.pooled_inv_mass(s, sq, z, z, 3)
    expect = (6 / 11) * 2.5 + 1e-3 * (5 / 11)
    assert im.dtype == np.float32 and im[0] == np.float32(expect)
    assert mf[0] == np.sqrt(np.float32(1) / np.float32(expect))
    # the lo terms enter as hi + lo in fp64
    im2, _ = A.pooled_inv_mass(s - 1, sq, z + 1, z, 3)
    assert im2[0] == im[0]
    assert A.restart_mu(0.05) == float(np.float32(np.log(0.5)))


def _gauss(D=8):
    return T.GaussianDiag(torch.zeros(D), torch.ones(D))


@pytest.mark.parametrize('case', ['full_mass', 'block_mass', 'gauss_full', 'funnel', 'rmhmc', 'big_d', 'host_windows',
                                  'split_without_list'])
def test_unsupported_combinations_are_refused_on_the_host(case):
    D = 8
    kw = dict(num_samples=40, burn=25, sampler=hb.Sampler.HMC_NUTS, adapt_mass=True)
    tgt, q0 = _gauss(D), torch.zeros(2, D)
    if case == 'full_mass':
        kw['inv_mass'] = torch.eye(D)
    elif case == 'block_mass':
        kw['inv_mass'] = [torch.eye(4), torch.eye(4)]
    elif case == 'gauss_full':
        tgt = T.GaussianFull(torch.zeros(D), cov=torch.eye(D, dtype=torch.float64))
    elif case == 'funnel':
        tgt = T.Funnel(D)
    elif case == 'rmhmc':
        kw['sampler'] = hb.Sampler.RMHMC
    elif case == 'big_d':
        tgt, q0 = T.GaussianIso(4100), torch.zeros(2, 4100)
    elif case == 'host_windows':
        kw['host_windows'] = 4
    elif case == 'split_without_list':
        kw['integrator'] = hb.Integrator.SPLITTING
    with pytest.raises(NotImplementedError):
        hb.sample_chains(tgt, q0, **kw)


def test_adapt_mass_needs_nuts_and_burn_20():
    with pytest.raises(RuntimeError, match='HMC_NUTS'):
        hb.sample_chains(_gauss(), torch.zeros(2, 8), num_samples=40, burn=25, sampler=hb.Sampler.HMC, adapt_mass=True)
    with pytest.raises(RuntimeError, match='burn >= 20'):
        hb.sample_chains(_gauss(), torch.zeros(2, 8), num_samples=40, burn=19, sampler=hb.Sampler.HMC_NUTS,
                         adapt_mass=True)


def test_adapt_diag_mass_argument_checks(built_library):
    lib = N.load_library()
    fake = C.c_void_p(16)           # never dereferenced: every call below fails its argument checks first
    good = dict(C=2, ld=8, D=6, n=5, C_chains=2)

    def call(ptrs=(fake,) * 4, eps=fake, outs=(fake,) * 5, **over):
        a = dict(good, **over)
        return lib.hmcx_adapt_diag_mass(*ptrs, a['C'], a['ld'], a['D'], a['n'], eps, a['C_chains'], *outs, None)

    assert call(ptrs=(None, fake, fake, fake)) == N.ERR_INVALID_ARG
    assert call(ptrs=(fake, fake, fake, None)) == N.ERR_INVALID_ARG
    assert call(eps=None) == N.ERR_INVALID_ARG
    assert call(outs=(fake, fake, fake, fake, None)) == N.ERR_INVALID_ARG
    for over in (dict(C=0), dict(C_chains=0), dict(n=1), dict(D=0), dict(ld=4), dict(ld=10)):
        assert call(**over) == N.ERR_INVALID_ARG, over


def test_per_chain_mu_is_refused_by_the_non_sink_entries(built_library):
    lib = N.load_library()
    tgt = N.TargetStruct()
    tgt.kind, tgt.dim = T.GaussianIso.kind, 8
    mass, rng, nuts = N.MassStruct(), N.RngStruct(), N.NutsStruct()
    rng.mode = N.RNG_PHILOX
    nuts.enabled, nuts.mu_chain = 1, 16
    fake = C.c_void_p(16)
    rc = lib.hmcx_hmc_run(C.byref(tgt), C.byref(mass), C.byref(rng), C.byref(nuts), fake, fake, fake,
                          1, 8, 5, 10, 2, 0, 10, None, None, None, None, None, 0, None, None)
    assert rc == N.ERR_UNSUPPORTED
    rc = lib.hmcx_hmc_run_sink(C.byref(tgt), C.byref(mass), C.byref(rng), C.byref(nuts), fake, fake, fake,
                               1, 8, 5, 10, 2, 0, 10, None, None, None, None, None, 0, None, None, None)
    assert rc == N.ERR_UNSUPPORTED                            # no sink: the plain loop would ignore mu_chain
    mlp = N.MlpStruct()
    tgt.kind, tgt.mlp = T.KIND_MLP, C.pointer(mlp)
    rc = lib.hmcx_split_run(C.byref(tgt), C.byref(mass), C.byref(rng), C.byref(nuts), N.SCHEME_PLAIN, fake, fake, fake,
                            1, 8, 5, 10, 2, 0, 10, None, None, None, None, None, None)
    assert rc == N.ERR_UNSUPPORTED


# ---- multi-GPU pooling over gloo: the engine's CUDA stages are replaced by a host runner that calls the same gather hook
class _Pooled:
    pass


def _window_sums(chain_ids, D, n):
    """Per-chain window sums that depend only on the GLOBAL chain id (what Philox keying gives the real kernels)."""
    out = []
    for cid in chain_ids:
        g = np.random.default_rng(1000 + int(cid))
        x = (g.standard_normal((n, D)) * np.linspace(0.1, 3.0, D) + 50.0).astype(np.float32)
        acc = A.Sums(D)
        for row in x:
            acc.add(row)
        out.append(acc)
    return [torch.from_numpy(np.stack([getattr(a, f) for a in out])) for f in ('s', 'q', 'c', 'cq')]


def _pool_runner(log_prob_func, q0, chain_offset=0, mass_pool=None, adapt_mass=False, **kw):
    Cl, D = q0.shape
    sums = _window_sums(range(chain_offset, chain_offset + Cl), D, 30)
    pooled = [mass_pool(t) for t in sums]                  # the engine's gather, then its reduction stage (here: host)
    r = _Pooled()
    r.inv_mass = torch.from_numpy(A.pooled_inv_mass(*(t.numpy() for t in pooled), 30)[0])
    r.num_rejected, r.step_size = torch.zeros(Cl, dtype=torch.int32), torch.zeros(Cl)
    return r


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _pool_worker(rank, world, port, Cn, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        D = 5
        out = DI.sample_chains_sharded(None, torch.zeros(Cn, D), runner=_pool_runner, adapt_mass=True)
        ref = A.pooled_inv_mass(*(t.numpy() for t in _window_sums(range(Cn), D, 30)), 30)[0]
        q.put((rank, bool(np.array_equal(out['inv_mass'].numpy(), ref))))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('Cn', [8, 7])                     # even and ragged shards
def test_sharded_mass_pooling_equals_one_process_gloo_world2(Cn):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_pool_worker, args=(r, 2, port, Cn, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
    assert res == [(0, True), (1, True)]
