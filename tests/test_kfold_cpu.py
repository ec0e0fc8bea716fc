"""CPU: K-fold cross-validation and exact refits of Bayesian NNs -- the balanced fold assignment, the refusals of
sample_chains(folds=...) and of the scoring calls (all before any CUDA work), the host layout of the fold target, the fp64
oracle of the conjugate regression, the multi-GPU partition by groups of K rows (gloo, world 2) and the argument checks
of hmcx_split_run_folds."""
import ctypes as C
import math
import os
import socket

import numpy as np
import pytest
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import engine, loo as LOO, samplers, targets as T
from oracle import cases
from tests import kfold_oracle as KO
from tests.test_loo_cpu import _conjugate


def _reg(n=24, hidden=4, task='regression', tau_out=10.):
    model, x, y = cases.mlp_problem(seed=1, n=n, n_in=3, hidden=hidden, task=task)
    loss = {'regression': 'regression', 'logsoftmax': 'multi_class_log_softmax_output'}[task]
    return T.MLPTarget.from_model(model, x, y, None, tau_out, prior_scale=2.0, model_loss=loss), model


def _q0(model, C_):
    return hb.util.flatten(model).detach()[None].repeat(C_, 1)


# ------------------------------------------------------------------------------------------------------------------
# kfold_split
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('N_, K', [(40, 5), (41, 5), (10, 10), (100, 64), (7, 2)])
def test_kfold_split_is_balanced_deterministic_and_complete(N_, K):
    f = LOO.kfold_split(N_, K, seed=3)
    assert f.dtype == torch.int64 and f.shape == (N_,) and f.device.type == 'cpu'
    sizes = torch.bincount(f, minlength=K)
    assert sizes.numel() == K and int(sizes.min()) >= 1 and int(sizes.max() - sizes.min()) <= 1
    assert torch.equal(f, LOO.kfold_split(N_, K, seed=3))
    torch.manual_seed(123)
    a = LOO.kfold_split(N_, K, seed=3)
    torch.manual_seed(456)
    assert torch.equal(a, LOO.kfold_split(N_, K, seed=3))            # the global generator plays no part


def test_kfold_split_refuses_bad_k():
    for N_, K in ((10, 1), (10, 11), (100, 65)):
        with pytest.raises(ValueError, match='2 <= K'):
            LOO.kfold_split(N_, K)


# ------------------------------------------------------------------------------------------------------------------
# refusals of sample_chains(folds=...): raised before any CUDA work
# ------------------------------------------------------------------------------------------------------------------
def test_refusals_before_any_cuda_work():
    tgt, model = _reg()
    f = LOO.kfold_split(24, 3)
    q0 = _q0(model, 6)
    run = lambda lp=tgt, q=q0, folds=f, num_samples=10, **kw: samplers.sample_chains(lp, q, num_samples=num_samples,
                                                                                      folds=folds, **kw)
    with pytest.raises(NotImplementedError, match='split lists or SPLITTING integrators'):
        run([tgt, tgt], integrator=hb.Integrator.SPLITTING)
    with pytest.raises(NotImplementedError, match='split lists or SPLITTING integrators'):
        run(integrator=hb.Integrator.SPLITTING_RAND)
    with pytest.raises(NotImplementedError, match='Bayesian-NN targets only'):
        run(T.GaussianIso(3), torch.zeros(6, 3))
    with pytest.raises(NotImplementedError, match='not RMHMC'):
        run(sampler=hb.Sampler.RMHMC)
    with pytest.raises(RuntimeError, match='no data'):
        run(T.MLPTarget.from_model(model, None, None))
    with pytest.raises(NotImplementedError, match='inv_mass None or 1-D'):
        run(inv_mass=torch.eye(tgt.dim))
    with pytest.raises(NotImplementedError, match='inv_mass None or 1-D'):
        run(inv_mass=[torch.eye(tgt.dim)])
    with pytest.raises(NotImplementedError, match='replica exchange'):
        run(betas=[1.0, 0.5])
    with pytest.raises(NotImplementedError, match='hyperpriors'):
        run(tau_prior=(2.0, 1.0))
    with pytest.raises(NotImplementedError, match='hyperpriors'):
        run(tau_out_prior=(2.0, 1.0))
    with pytest.raises(NotImplementedError, match='adapt_mass'):
        run(adapt_mass=True, sampler=hb.Sampler.HMC_NUTS, burn=20, num_samples=30)
    with pytest.raises(NotImplementedError, match="rng='philox' or 'injected'"):
        run(q=q0[:1], rng='reference')
    with pytest.raises(ValueError, match='integer tensor'):
        run(folds=f.float())
    with pytest.raises(ValueError, match='integer tensor'):
        run(folds=f.tolist())
    with pytest.raises(ValueError, match='integer tensor'):
        run(folds=f > 0)
    with pytest.raises(ValueError, match=r'\(N,\) = \(24,\)'):
        run(folds=f[:-1])
    with pytest.raises(ValueError, match=r'\(N,\) = \(24,\)'):
        run(folds=f[None])
    with pytest.raises(ValueError, match='2 <= K <= 64'):
        run(folds=torch.zeros(24, dtype=torch.int64), q=q0[:1])                          # K = 1
    with pytest.raises(ValueError, match='2 <= K <= 64'):
        run(folds=torch.arange(24) * 3)                                                  # K = 70
    with pytest.raises(ValueError, match='2 <= K <= 64'):
        run(folds=f - 2)                                                                 # ids below -1
    with pytest.raises(ValueError, match=r'missing \[1\]'):
        run(folds=torch.where(f == 1, torch.zeros_like(f), f))
    with pytest.raises(ValueError, match='not a multiple of K = 3'):
        run(q=q0[:5])
    with pytest.raises(ValueError, match='chain_offset 4 is not a multiple of K = 3'):
        run(chain_offset=4)
    assert torch.equal(samplers._fold_args(tgt, q0, hb.Sampler.HMC, hb.Integrator.IMPLICIT, None, False, None, None,
                                           'philox', 6, f.to(torch.int32)), f)   # accepted: the int64 CPU assignment


# ------------------------------------------------------------------------------------------------------------------
# the fold target's host layout
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('task', ['regression', 'logsoftmax'])
def test_fold_target_layout(task):
    tgt, _ = _reg(n=30, task=task)
    f = LOO.kfold_split(30, 4, seed=1)
    f[5] = -1                                                   # a row every fit keeps
    parts = engine.fold_targets(tgt, f)
    assert len(parts) == 4
    nt = engine.NativeTarget(parts, 'cpu')
    m = nt.mlp_struct
    y = tgt.y.reshape(30, tgt.y_cols)
    begin = [0]
    for k in range(4):
        keep = torch.nonzero(f != k).flatten()                   # increasing: the original order
        assert torch.equal(parts[k].x, tgt.x[keep]) and torch.equal(parts[k].y, y[keep])
        assert bool((keep == 5).any())
        assert float(parts[k].prior_scale) == 2.0 and parts[k].tau_out == tgt.tau_out
        assert parts[k].tau_list is tgt.tau_list and parts[k].loss_id == tgt.loss_id
        begin.append(begin[-1] + keep.numel())
    assert m.num_splits == 4 and list(m.split_begin[:5]) == begin and m.num_rows == begin[-1]
    assert m.prior_scale == 2.0
    assert torch.equal(nt._keep['x'], torch.cat([p.x for p in parts]))
    assert torch.equal(nt._keep['y'], torch.cat([p.y for p in parts]))
    assert begin[-1] == 3 * 29 + 4                              # (K - 1) N scored rows + K copies of the -1 row


def test_fold_target_keeps_the_pinned_settings():
    tgt, _ = _reg()
    tgt.cluster_size, tgt.tensor_cores = 2, 1
    nt = engine.NativeTarget(engine.fold_targets(tgt, LOO.kfold_split(24, 3)), 'cpu')
    assert nt.mlp_struct.cluster_size == 2 and nt.mlp_struct.tensor_cores == 1


# ------------------------------------------------------------------------------------------------------------------
# the fp64 oracle
# ------------------------------------------------------------------------------------------------------------------
def _conj_data(tgt):
    return tgt.x.double().numpy(), tgt.y.double().numpy().reshape(-1)


def test_oracle_at_k_equals_n_is_exact_leave_one_out():
    tgt, _, _, exact = _conjugate()
    x, y = _conj_data(tgt)
    kf = KO.conjugate_kfold(x, y, np.arange(40), 4.0, 2.0, 0.5)
    assert np.abs(kf - exact).max() < 1e-5, np.abs(kf - exact).max()      # (x, y rounded to fp32 in the target)


def test_oracle_k_fold_against_monte_carlo_of_the_fold_posterior():
    """Fold k's predictive of a held-out row, as an average of the likelihood over exact posterior draws of the fit
    without that fold."""
    tgt, _, _, _ = _conjugate()
    x, y = _conj_data(tgt)
    f = LOO.kfold_split(40, 5, seed=2).numpy()
    kf = KO.conjugate_kfold(x, y, f, 4.0, 2.0, 0.5)
    rng = np.random.default_rng(0)
    X1 = np.concatenate([x, np.ones((40, 1))], 1)
    for k in range(5):
        tr, ho = f != k, np.nonzero(f == k)[0]
        P = np.diag([2.0] * 3 + [0.5]) + 4.0 * X1[tr].T @ X1[tr]
        Sig = np.linalg.inv(P)
        mu = Sig @ (4.0 * X1[tr].T @ y[tr])
        th = rng.multivariate_normal(mu, Sig, size=20000)
        ll = -0.5 * 4.0 * (X1[ho] @ th.T - y[ho][:, None]) ** 2 + 0.5 * math.log(4.0 / (2 * math.pi))
        mc = KO.logmeanexp(ll.T)
        assert np.abs(mc - kf[ho]).max() < 0.01
    assert np.all(np.isfinite(kf))
    part = KO.conjugate_kfold(x, y, np.where(f == 0, -1, f), 4.0, 2.0, 0.5)      # fold 0's rows in every fit
    assert np.isnan(part[f == 0]).all() and np.isfinite(part[f != 0]).all()


def test_oracle_k_fold_differs_from_leave_one_out_at_small_k():
    tgt, _, _, exact = _conjugate()
    x, y = _conj_data(tgt)
    kf = KO.conjugate_kfold(x, y, LOO.kfold_split(40, 2, seed=0).numpy(), 4.0, 2.0, 0.5)
    assert kf.sum() < exact.sum()                               # half the data per fit predicts worse


# ------------------------------------------------------------------------------------------------------------------
# scoring: refusals and the host-side paths that launch nothing
# ------------------------------------------------------------------------------------------------------------------
class _Res:
    pass


def test_kfold_refusals():
    tgt, _ = _reg()
    with pytest.raises(TypeError, match='folds=...'):
        LOO.kfold(_Res(), tgt)
    r = _Res()
    r.folds, r.num_folds = LOO.kfold_split(24, 3), 3
    r.folds[0] = -1
    with pytest.raises(RuntimeError, match='fold -1'):
        LOO.kfold(r, tgt)
    r.folds = LOO.kfold_split(23, 3)
    with pytest.raises(RuntimeError, match='23 rows'):
        LOO.kfold(r, tgt)
    with pytest.raises(TypeError, match='not a split list'):
        LOO.kfold(r, [tgt, tgt])
    with pytest.raises(TypeError, match='MLPTarget'):
        LOO.kfold(r, T.GaussianIso(3))


def _fake_loo(pareto_k, thr=0.7):
    r = LOO.LooResult()
    n = len(pareto_k)
    r.pointwise = -torch.arange(1, n + 1, dtype=torch.float64)
    r.lppd = r.pointwise + 0.25
    r.p_loo_i = r.lppd - r.pointwise
    r.pareto_k = torch.as_tensor(pareto_k, dtype=torch.float64)
    r.tail_size = torch.full((n,), 5, dtype=torch.int32)
    r.elpd_loo, r.se = LOO._total(r.pointwise)
    r.p_loo, r.p_loo_se = LOO._total(r.p_loo_i)
    r.looic, r.looic_se = -2 * r.elpd_loo, 2 * r.se
    r.k_threshold, r.num_bad_k = thr, int((r.pareto_k > thr).sum())
    r.num_nonfinite, r.num_points, r.num_draws, r.r_eff = 0, n, 400, 1.0
    return r


class _Launched(Exception):
    pass


def _recording_sampler(monkeypatch):
    calls = []

    def fake(lp, q0, **kw):
        calls.append((lp, q0, kw))
        raise _Launched()
    monkeypatch.setattr(samplers, 'sample_chains', fake)
    return calls


def test_reloo_without_flagged_points_copies_and_launches_nothing(monkeypatch):
    tgt, model = _reg()
    calls = _recording_sampler(monkeypatch)
    lo = _fake_loo([0.1] * 24)
    out = LOO.reloo(lo, tgt, _q0(model, 1)[0], num_samples=10)
    assert not calls
    assert out is not lo and out.kind == 'loo' and out.refit_points.numel() == 0
    for k, v in lo.__dict__.items():
        w = getattr(out, k)
        if torch.is_tensor(v):
            assert w is not v and torch.equal(w, v)
        else:
            assert w == v


def test_reloo_launches_one_fold_per_flagged_point(monkeypatch):
    tgt, model = _reg()
    calls = _recording_sampler(monkeypatch)
    q = _q0(model, 2) + torch.arange(2.0)[:, None]
    with pytest.raises(_Launched):                               # three flagged points: one K = 3 fold run
        LOO.reloo(_fake_loo([0.1, 0.9, 0.1, 0.8, 0.1, 1.5] + [0.1] * 18), tgt, q, num_samples=10, seed=4)
    lp, q0, kw = calls[-1]
    assert lp is tgt and kw['num_samples'] == 10 and kw['seed'] == 4
    assert kw['folds'].tolist() == [-1, 0, -1, 1, -1, 2] + [-1] * 18
    assert torch.equal(q0, q.repeat_interleave(3, dim=0))        # row r K + k: chain r of fold k
    with pytest.raises(_Launched):                               # one flagged point: a plain run without it
        LOO.reloo(_fake_loo([0.1] * 5 + [0.9] + [0.1] * 18), tgt, q[0], num_samples=10)
    lp, q0, kw = calls[-1]
    assert 'folds' not in kw and torch.equal(q0, q[:1])
    keep = [i for i in range(24) if i != 5]
    assert torch.equal(lp.x, tgt.x[keep]) and torch.equal(lp.y, tgt.y.reshape(24, 1)[keep])


def test_reloo_refusals_and_batches():
    tgt, model = _reg()
    with pytest.raises(TypeError, match='psis_loo'):
        LOO.reloo(_Res(), tgt, _q0(model, 1))
    with pytest.raises(RuntimeError, match='23 points'):
        LOO.reloo(_fake_loo([0.1] * 23), tgt, _q0(model, 1))
    with pytest.raises(ValueError, match='do not pass folds'):
        LOO.reloo(_fake_loo([0.1] * 24), tgt, _q0(model, 1), folds=None)
    for n, sizes in ((1, [1]), (2, [2]), (64, [64]), (65, [33, 32]), (129, [43, 43, 43]), (200, [50] * 4)):
        b = LOO._reloo_batches(list(range(n)))
        assert [len(x) for x in b] == sizes and sum(b, []) == list(range(n))


def _fake(kind, pointwise):
    r = {'loo': LOO.LooResult, 'waic': LOO.WaicResult, 'kfold': LOO.KfoldResult}[kind]()
    r.pointwise = torch.as_tensor(pointwise, dtype=torch.float64)
    r.num_points = r.pointwise.numel()
    setattr(r, LOO._ELPD[kind], float(r.pointwise.sum()))
    return r


def test_compare_takes_kfold_results_among_themselves():
    a, b = _fake('kfold', [-1.0, -2.0, -0.5, -1.5]), _fake('kfold', [-1.2, -1.9, -0.9, -1.6])
    c = LOO.compare(b, a)
    d = (b.pointwise - a.pointwise).numpy()
    assert c.order == [1, 0] and c.elpd_diff[1] == 0.0 and abs(c.elpd_diff[0] - d.sum()) < 1e-12
    assert abs(c.se_diff[0] - math.sqrt(4) * d.std(ddof=1)) < 1e-12
    for other in ('loo', 'waic'):
        with pytest.raises(TypeError, match='kfold results only'):
            LOO.compare(a, _fake(other, [-1.0, -2.0, -0.5, -1.5]))
    with pytest.raises(RuntimeError, match='different numbers of data points'):
        LOO.compare(a, _fake('kfold', [-1.0, -2.0]))
    lo = LOO.reloo(_fake_loo([0.1] * 4), T.MLPTarget.from_model(torch.nn.Linear(3, 1), torch.zeros(4, 3),
                                                                 torch.zeros(4, 1)), torch.zeros(4))
    assert LOO.compare(lo, _fake('loo', [-1.0, -2.0, -0.5, -1.5])).order == [1, 0]


# ------------------------------------------------------------------------------------------------------------------
# multi-GPU routing (gloo, world 2): groups of K rows are partitioned
# ------------------------------------------------------------------------------------------------------------------
def _worker(rank, port, out):
    import torch.distributed as dist
    from hamiltorch_b200 import distributed as Dd
    os.environ['MASTER_ADDR'], os.environ['MASTER_PORT'] = '127.0.0.1', str(port)
    dist.init_process_group('gloo', rank=rank, world_size=2)
    seen = {}

    def runner(lp, q0, num_samples=2, chain_offset=0, **kw):
        seen.update(kw)
        seen['rows'], seen['chain_offset'] = q0[:, 0].tolist(), chain_offset
        r = _Res()
        ids = torch.arange(chain_offset, chain_offset + q0.shape[0], dtype=torch.float32)
        r.num_rejected, r.step_size, r.dim = ids.to(torch.int32), ids / 7, 2
        r.samples_padded = torch.zeros(q0.shape[0], num_samples, 4)
        r.samples_padded[..., :2] = ids[:, None, None] * 100 + torch.arange(num_samples)[None, :, None]
        r.moment_sum, r.moment_sumsq, r.moment_count = q0.double(), q0.double() ** 2, 1
        return r
    q0 = torch.arange(30.0).reshape(15, 2)                      # R = 5 groups of K = 3 rows
    f = torch.tensor([0, 1, 2, 0, 1, 2, -1, 0])
    z = torch.arange(4 * 15 * 2, dtype=torch.float32).reshape(4, 15, 2)
    lu = torch.arange(4 * 15, dtype=torch.float32).reshape(4, 15)
    o = Dd.sample_chains_sharded(None, q0, gather_samples=True, runner=runner, folds=f, normals=z, log_uniforms=lu,
                                 chain_offset=6, moments=True)
    out[rank] = (seen['rows'], seen['chain_offset'], seen['normals'].tolist(), seen['log_uniforms'].tolist(),
                 seen['folds'].tolist(), o['num_rejected'].tolist(), o['samples'][:, :, 0].tolist(), o['bounds'],
                 'posterior_mean' in o)
    dist.destroy_process_group()


def test_sharded_call_partitions_groups_of_k_rows():
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    out = mp.Manager().dict()
    mp.spawn(_worker, args=(port, out), nprocs=2, join=True)
    z = torch.arange(4 * 15 * 2, dtype=torch.float32).reshape(4, 15, 2)
    lu = torch.arange(4 * 15, dtype=torch.float32).reshape(4, 15)
    for r, rows in enumerate([list(range(0, 6)), list(range(6, 15))]):        # groups [0, 2) and [2, 5)
        seen_rows, off, zs, lus, folds, rej, smp, bounds, pooled = out[r]
        assert seen_rows == [2.0 * i for i in rows] and bounds == (rows[0], rows[-1] + 1)
        assert off == 6 + rows[0] and off % 3 == 0
        assert zs == z[:, rows[0]:rows[-1] + 1].tolist() and lus == lu[:, rows[0]:rows[-1] + 1].tolist()
        assert folds == [0, 1, 2, 0, 1, 2, -1, 0]
        assert rej == list(range(6, 21))                         # every row's global id, in global order
        g = torch.tensor(smp)
        assert g.shape == (15, 2) and torch.equal(g[:, 0], torch.arange(6, 21, dtype=torch.float32) * 100)
        for k in range(3):                                       # [k::K] is fold k: global ids = k (mod K)
            assert all(int(v) // 100 % 3 == k for v in g[k::3, 0])
        assert not pooled                                        # the folds are different posteriors


# ------------------------------------------------------------------------------------------------------------------
# C ABI: argument checks return before any CUDA work
# ------------------------------------------------------------------------------------------------------------------
def test_abi_split_run_folds_checks_its_arguments(built_library):
    from hamiltorch_b200 import _native as N
    lib = N.load_library()
    assert hasattr(lib, 'hmcx_split_run_folds') and lib.hmcx_abi_version() == 12
    tgt, _ = _reg()
    junk = C.c_void_p(16)
    nt3 = engine.NativeTarget(engine.fold_targets(tgt, LOO.kfold_split(24, 3)), 'cpu')
    ld = N.padded_ld(nt3.dim)

    def run(nt=nt3, K=3, scheme=N.SCHEME_PLAIN, sink=None, C_=6):
        rng = N.RngStruct()
        rng.mode = N.RNG_PHILOX
        return lib.hmcx_split_run_folds(None if nt is None else nt.ref(), None, C.byref(rng), C.byref(N.NutsStruct()),
                                        scheme, junk, junk, junk, C_, ld, 3, 10, 2, 0, 10, junk, junk, junk, None, junk,
                                        sink, K, None)

    assert run(nt=None) == N.ERR_INVALID_ARG
    for K in (0, 1, 2, 4, 65, -3):
        assert run(K=K) == N.ERR_INVALID_ARG, K                  # out of range, or num_splits != K
    bad_sink = N.SinkStruct()
    bad_sink.thin = 0
    assert run(sink=C.byref(bad_sink)) == N.ERR_INVALID_ARG
    for scheme in (N.SCHEME_SPLIT_SYM, N.SCHEME_SPLIT_RAND, N.SCHEME_SPLIT_KMID):
        assert run(scheme=scheme) == N.ERR_UNSUPPORTED
    assert run(nt=engine.NativeTarget(T.GaussianIso(4), 'cpu')) == N.ERR_UNSUPPORTED
    nodata = T.MLPTarget.from_model(torch.nn.Linear(3, 1), None, None)
    nd = engine.NativeTarget(nodata, 'cpu')
    nd.mlp_struct.num_splits = 3                                 # a three-split target without rows
    assert run(nt=nd) == N.ERR_INVALID_ARG
