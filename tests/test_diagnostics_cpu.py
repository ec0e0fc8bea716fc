"""CPU: the fp64 definition of split-R-hat / ESS / MCSE (oracle/diagnostics_oracle.py) against processes whose answers
are known, its internals and edge cases; the host logic of hamiltorch_b200.diagnostics (Geyer scan on pooled sums, lag
blocks) against it, with the oracle's partial stages standing in for the CUDA passes; the gloo world-2 pooling; and the
argument checks of the ABI entries and of ``summary``."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from hamiltorch_b200 import diagnostics as DG
from hamiltorch_b200 import distributed as DS
from oracle import diagnostics_oracle as O


def ar1(C, n, D, phi, seed, mean=0.0, scale=1.0):
    """Stationary AR(1) chains with unit marginal variance (times scale, plus mean): (C, n, D) float32."""
    rng = np.random.default_rng(seed)
    e = rng.standard_normal((C, n, D))
    x = np.empty((C, n, D))
    x[:, 0] = e[:, 0]
    s = np.sqrt(1 - phi * phi)
    for t in range(1, n):
        x[:, t] = phi * x[:, t - 1] + s * e[:, t]
    return (mean + scale * x).astype(np.float32)


class OraclePartials:
    """The partial stages of hamiltorch_b200.diagnostics computed by the numpy oracle (in place of the CUDA passes)."""
    lag_block = 32

    def __init__(self, x):
        self.x = np.asarray(x, dtype=np.float64)
        if self.x.ndim == 2:
            self.x = self.x[None]
        self.C, self.n, self.D = self.x.shape
        self.m, self.device = self.n // 2, torch.device('cpu')

    def means(self):
        self.mu, s = O.partial_means(self.x)
        return torch.from_numpy(s), 2 * self.C

    def acov(self, mu_bar, t0):
        a, b = O.partial_acov(self.x, self.mu, None if mu_bar is None else mu_bar.numpy(), t0, self.lag_block)
        return torch.from_numpy(a), None if b is None else torch.from_numpy(b)


def assert_matches_oracle(got, ref, rtol):
    for k in ('mean', 'sd', 'mcse', 'ess', 'rhat'):
        g = getattr(got, k).cpu().numpy()
        r = ref[k]
        assert np.array_equal(np.isnan(g), np.isnan(r)), k
        assert np.array_equal(np.isinf(g), np.isinf(r)), k
        ok = np.isfinite(r)
        assert np.allclose(g[ok], r[ok], rtol=rtol, atol=0), (k, np.max(np.abs(g[ok] - r[ok]) / np.abs(r[ok]).clip(1e-300)))
    assert np.array_equal(got.max_lag.cpu().numpy(), ref['max_lag'])


# ---------------------------------------------------------------------------------------------------------------
# The oracle against known processes
# ---------------------------------------------------------------------------------------------------------------
def test_iid_normal_has_rhat_one_and_ess_near_n():
    x = ar1(4, 2000, 3, 0.0, 0)
    r = O.summary(x)
    N = 4 * 2000
    assert np.all(np.abs(r['rhat'] - 1) < 0.01)
    assert np.all(np.abs(r['ess'] / N - 1) < 0.1)
    assert np.allclose(r['mcse'], r['sd'] / np.sqrt(r['ess']))


def test_ar1_ess_matches_theory():
    phi = 0.9
    x = ar1(4, 20000, 2, phi, 1)
    r = O.summary(x)
    theory = (1 - phi) / (1 + phi)
    assert np.all(np.abs(r['ess'] / (4 * 20000) / theory - 1) < 0.2), r['ess']


def test_shifted_chains_have_large_rhat():
    x = ar1(4, 500, 2, 0.0, 2)
    x[2:] += 3.0
    assert np.all(O.summary(x)['rhat'] > 1.5)


def test_antithetic_chain_has_ess_above_n():
    x = ar1(4, 4000, 2, -0.5, 3)
    assert np.all(O.summary(x)['ess'] > 4 * 4000)


# ---------------------------------------------------------------------------------------------------------------
# Oracle internals and edge cases
# ---------------------------------------------------------------------------------------------------------------
def test_direct_lag_sums_equal_fft_autocovariance():
    x = ar1(3, 301, 4, 0.7, 4)
    y = O.split_chains(x)
    mu = y.mean(1)
    fft = O.autocov_fft(y, mu)
    scale = np.abs(fft[:, 0]).max()
    for t in range(y.shape[1]):
        assert np.allclose(O.autocov(y, mu, t), fft[:, t], rtol=0, atol=1e-12 * scale), t
    assert np.array_equal(O.autocov(y, mu, y.shape[1]), np.zeros((6, 4)))


def test_odd_n_drops_the_middle_draw():
    x = ar1(3, 201, 5, 0.5, 5)
    even = np.delete(x, 100, axis=1)
    a, b = O.summary(x), O.summary(even)
    for k in ('mean', 'sd', 'mcse', 'ess', 'rhat', 'max_lag'):
        assert np.array_equal(a[k], b[k]), k


def test_constant_and_nonfinite_dimensions():
    x = ar1(2, 40, 5, 0.3, 6)
    x[:, :, 1] = 2.5                        # all draws equal
    x[0, 7, 2] = np.nan                     # a NaN draw
    x[1, 3, 3] = np.inf                     # an infinite draw
    x[0, :, 4] = 1.0                        # every half-chain constant, chains differ: W = 0, B > 0
    x[1, :, 4] = 2.0
    r = O.summary(x)
    assert (r['ess'][1], r['rhat'][1], r['mcse'][1], r['sd'][1], r['mean'][1]) == (80, 1.0, 0.0, 0.0, 2.5)
    assert r['max_lag'][1] == 0
    for d in (2, 3):
        assert all(np.isnan(r[k][d]) for k in ('mean', 'sd', 'mcse', 'ess', 'rhat')) and r['max_lag'][d] == 0
    assert np.isinf(r['rhat'][4]) and np.isfinite(r['ess'][4]) and r['ess'][4] > 0
    assert np.isfinite(r['ess'][0]) and np.isfinite(r['rhat'][0])


def test_n_below_four_is_refused():
    with pytest.raises(ValueError):
        O.summary(np.zeros((2, 3, 1)))


# ---------------------------------------------------------------------------------------------------------------
# Host logic (pooled sums -> Geyer scan on torch ops, lag blocks on demand) against the oracle
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('C,n,D,phi', [(1, 8, 3, 0.0), (2, 9, 2, 0.5), (7, 501, 3, 0.9), (3, 1000, 2, 0.995),
                                       (4, 64, 3, -0.5), (2, 5, 4, 0.0)])
def test_host_scan_matches_oracle(C, n, D, phi):
    x = ar1(C, n, D, phi, 10 + C + n)
    got = DG.summary_from_partials(OraclePartials(x), num_chains=C, num_draws=n)
    assert_matches_oracle(got, O.summary(x), 1e-12)
    assert got.num_lag_blocks == max(1, -(-(int(got.max_lag.max()) + 1) // 32))     # a block only while a scan runs


def test_host_scan_needs_many_lag_blocks_for_a_slow_chain():
    x = ar1(2, 4000, 2, 0.995, 11)
    got = DG.summary_from_partials(OraclePartials(x))
    ref = O.summary(x)
    assert_matches_oracle(got, ref, 1e-12)
    assert got.num_lag_blocks > 4
    assert got.num_lag_blocks * 32 > ref['max_lag'].max() >= (got.num_lag_blocks - 1) * 32


def test_host_scan_edge_cases_match_oracle():
    x = ar1(2, 40, 5, 0.3, 6)
    x[:, :, 1] = 2.5
    x[0, 7, 2] = np.nan
    x[1, 3, 3] = np.inf
    x[0, :, 4], x[1, :, 4] = 1.0, 2.0
    assert_matches_oracle(DG.summary_from_partials(OraclePartials(x)), O.summary(x), 1e-12)


def test_pooled_partials_equal_one_block():
    x = ar1(5, 300, 3, 0.8, 12)
    one = DG.summary_from_partials(OraclePartials(x))
    two = DG.summary_from_partials(DG.PooledPartials([OraclePartials(x[:2]), OraclePartials(x[2:])]))
    for k in ('mean', 'sd', 'mcse', 'ess', 'rhat'):
        assert torch.allclose(getattr(one, k), getattr(two, k), rtol=1e-12, atol=0), k
    assert torch.equal(one.max_lag, two.max_lag) and two.num_chains == 5


# ---------------------------------------------------------------------------------------------------------------
# gloo world 2: pooled over ranks == the single-process oracle on all chains
# ---------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _fake_runner(log_prob_func, q0, num_samples=4, chain_offset=0, **kw):
    """Chain c (global id) = a stored AR(1) chain; the per-rank result carries a pad column like ld > D."""
    Cl, Dd = q0.shape
    full = torch.from_numpy(ar1(5, num_samples, Dd, 0.6, 99))
    blk = torch.zeros(Cl, num_samples, Dd + 1)
    blk[..., :Dd] = full[chain_offset:chain_offset + Cl]

    class R:
        pass
    r = R()
    r.samples_padded, r.dim = blk, Dd
    r.num_rejected = torch.zeros(Cl, dtype=torch.int32)
    r.step_size = torch.zeros(Cl)
    return r


def _pool_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        Ct, n, D = 5, 203, 3
        x = ar1(Ct, n, D, 0.9, 42)
        lo, hi = DS.shard_bounds(Ct, rank, world)            # ragged: 2 + 3 chains
        got = DS.pooled_diagnostics(torch.from_numpy(x[lo:hi]), partials=OraclePartials)
        ref = O.summary(x)
        ok = got.num_chains == Ct and got.num_draws == n
        try:
            assert_matches_oracle(got, ref, 1e-12)
        except AssertionError:
            ok = False
        out = DS.sample_chains_sharded(None, torch.zeros(Ct, D), runner=_fake_runner, num_samples=50, diagnostics=True,
                                       diagnostics_partials=OraclePartials)
        try:
            assert_matches_oracle(out['diagnostics'], O.summary(ar1(5, 50, D, 0.6, 99)), 1e-12)
        except AssertionError:
            ok = False
        q.put((rank, bool(ok), [float(v) for v in got.ess]))
    finally:
        dist.destroy_process_group()


def test_pooled_diagnostics_gloo_world2_ragged_shards():
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_pool_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
    assert [(r, ok) for r, ok, _ in res] == [(0, True), (1, True)]
    assert res[0][2] == res[1][2]                            # identical on every rank


# ---------------------------------------------------------------------------------------------------------------
# Argument checks that need no GPU
# ---------------------------------------------------------------------------------------------------------------
def test_abi_entries_reject_invalid_arguments(built_library):
    from hamiltorch_b200 import _native as N
    lib = N.load_library()
    buf = C.c_void_p(16)                                     # never dereferenced: validation returns first
    assert lib.hmcx_diag_means(buf, 12, 4, 1, 3, 4, buf, buf, None) == N.ERR_INVALID_ARG          # n < 4
    assert lib.hmcx_diag_means(None, 12, 4, 1, 8, 4, buf, buf, None) == N.ERR_INVALID_ARG         # null block
    assert lib.hmcx_diag_means(buf, 12, 4, 1, 8, 4, None, buf, None) == N.ERR_INVALID_ARG         # null output
    assert lib.hmcx_diag_means(buf, 12, 4, 0, 8, 4, buf, buf, None) == N.ERR_INVALID_ARG          # no chain
    assert lib.hmcx_diag_acov(buf, 12, 4, 1, 8, 4, None, None, 0, buf, None, None) == N.ERR_INVALID_ARG  # null mu
    assert lib.hmcx_diag_acov(buf, 12, 4, 1, 8, 4, buf, None, -1, buf, None, None) == N.ERR_INVALID_ARG  # lag < 0
    assert lib.hmcx_diag_acov(buf, 12, 4, 1, 8, 4, buf, buf, 0, buf, None, None) == N.ERR_INVALID_ARG    # no between_out
    assert lib.hmcx_diag_acov(buf, -1, 4, 1, 8, 4, buf, None, 0, buf, None, None) == N.ERR_INVALID_ARG   # stride < 0
    assert N.DIAG_LAG_BLOCK == 32


def test_summary_refuses_cpu_inputs_and_runs_without_samples():
    import hamiltorch_b200 as hb
    from hamiltorch_b200.engine import HMCResult
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        hb.diagnostics.summary(torch.zeros(2, 10, 3))
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        hb.diagnostics.summary([torch.zeros(3) for _ in range(10)])
    res = HMCResult(None, None, None, None, None, None, 3, 10)
    with pytest.raises(RuntimeError, match='keep_samples=False'):
        hb.diagnostics.summary(res)
    with pytest.raises(TypeError):
        hb.diagnostics.summary(3.0)
