"""GPU: the diagnostics passes (hmcx_diag_means / hmcx_diag_acov) and hamiltorch_b200.diagnostics.summary against the
fp64 oracle (oracle/diagnostics_oracle.py) on the same fp32 blocks; input forms from real runs; determinism; pooling of
partial stages; config 2 end to end."""
import numpy as np
import pytest
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import diagnostics as DG
from hamiltorch_b200 import targets as T
from oracle import diagnostics_oracle as O

pytestmark = pytest.mark.gpu

KEYS = ('mean', 'sd', 'mcse', 'ess', 'rhat')


def ar1(C, n, D, phi, seed, mean=0.0, scale=1.0):
    rng = np.random.default_rng(seed)
    e = rng.standard_normal((C, n, D))
    x = np.empty((C, n, D))
    x[:, 0] = e[:, 0]
    s = np.sqrt(1 - phi * phi)
    for t in range(1, n):
        x[:, t] = phi * x[:, t - 1] + s * e[:, t]
    return (mean + scale * x).astype(np.float32)


def padded_block(x, extra=4):
    """The (C, n, D) block as a view into a (C, n, ld) device buffer with pad columns (ld > D, ld % 4 == 0)."""
    C, n, D = x.shape
    ld = (D + 3) // 4 * 4 + extra
    buf = torch.full((C, n, ld), 7.0, dtype=torch.float32, device='cuda')
    buf[..., :D] = torch.from_numpy(x).cuda()
    return buf[..., :D]


def oracle_with_margin(x):
    """The oracle's summary of x, and the smallest |pair sum| its Geyer scan compares against 0 (over every dimension
    and every pair it reads)."""
    y = O.split_chains(x)
    K, m, D = y.shape
    mu = y.mean(1)
    yc = y - mu[:, None, :]
    g0 = O.autocov_centered(yc, 0).mean(0)
    between = ((mu - mu.mean(0)) ** 2).sum(0)
    W = m / (m - 1) * g0
    varp = (m - 1) / m * W + between / (K - 1)
    ref = O.summary(x)
    lag = int(ref['max_lag'].max())
    rho = np.stack([1.0 - (W - O.autocov_centered(yc, t).mean(0)) / varp for t in range(lag + 1)])
    rho[0] = 1.0
    margin = np.inf
    for d in range(D):
        if ref['max_lag'][d] == 0:
            continue
        pairs = rho[0:ref['max_lag'][d] + 1:2, d] + rho[1:ref['max_lag'][d] + 1:2, d]
        margin = min(margin, np.abs(pairs).min())
    return ref, margin


def assert_close(got, ref, rtol=1e-9):
    for k in KEYS:
        g = getattr(got, k).cpu().numpy()
        r = ref[k]
        assert np.array_equal(np.isnan(g), np.isnan(r)), k
        ok = np.isfinite(r)
        err = np.abs(g[ok] - r[ok]) / np.maximum(np.abs(r[ok]), 1e-300)
        assert err.size == 0 or err.max() <= rtol, (k, err.max())
    assert np.array_equal(got.max_lag.cpu().numpy(), ref['max_lag'])


CASES = [  # (C, n, D, phi, mean, scale)
    (1, 8, 1, 0.0, 0.0, 1.0),
    (2, 9, 3, 0.0, 0.0, 1.0),
    (7, 501, 130, 0.9, 0.0, 1.0),
    (256, 1000, 3, 0.0, 0.0, 1.0),
    (7, 1000, 1024, 0.9, 0.0, 1.0),
    (2, 1000, 3, 0.995, 0.0, 1.0),
    (256, 501, 130, 0.9, 0.0, 1.0),
    (1, 9, 1024, 0.0, 0.0, 1.0),
    (7, 501, 130, 0.5, 100.0, 0.01),     # offset block: mean 100, std 0.01
]


@pytest.mark.parametrize('C,n,D,phi,mean,scale', CASES)
def test_kernel_matches_oracle(C, n, D, phi, mean, scale):
    x = ar1(C, n, D, phi, 1000 + C * 7 + n + D, mean, scale)
    ref, margin = oracle_with_margin(x)
    assert margin > 1e-9                               # no Geyer decision within rounding of its threshold
    got = DG.summary(padded_block(x))
    torch.cuda.synchronize()
    assert got.num_chains == C and got.num_draws == n
    assert_close(got, ref)


def test_edge_case_dimensions_match_oracle():
    x = ar1(3, 40, 6, 0.3, 6)
    x[:, :, 1] = 2.5                                    # all draws equal
    x[0, 7, 2] = np.nan
    x[1, 3, 3] = np.inf
    x[0, :, 4], x[1, :, 4], x[2, :, 4] = 1.0, 2.0, 1.0     # W = 0, B > 0
    got = DG.summary(padded_block(x))
    ref = O.summary(x)
    assert_close(got, ref)
    assert float(got.ess[1]) == 120 and float(got.rhat[1]) == 1 and float(got.mcse[1]) == 0
    assert torch.isinf(got.rhat[4]) and torch.isnan(got.ess[2:4]).all()


def test_repeated_calls_are_bitwise_equal():
    x = padded_block(ar1(64, 700, 300, 0.95, 7))
    a, b = DG.summary(x), DG.summary(x)
    for k in KEYS + ('max_lag',):
        assert torch.equal(getattr(a, k), getattr(b, k)), k


def test_partials_of_two_chain_subsets_pool_to_the_single_call():
    x = padded_block(ar1(9, 400, 70, 0.9, 8))
    one = DG.summary(x)
    two = DG.summary_from_partials(DG.PooledPartials([DG.NativePartials(x[:4]), DG.NativePartials(x[4:])]))
    for k in KEYS:
        assert torch.allclose(getattr(one, k), getattr(two, k), rtol=1e-12, atol=0), k
    assert torch.equal(one.max_lag, two.max_lag) and two.num_chains == 9


# ---------------------------------------------------------------------------------------------------------------
# Input forms
# ---------------------------------------------------------------------------------------------------------------
def test_strided_and_thinned_blocks_of_a_real_run():
    kw = dict(num_samples=60, num_steps_per_sample=5, step_size=0.2, rng='philox', seed=3)
    init = 0.1 * torch.randn(6, 10, generator=torch.Generator().manual_seed(0))
    res = hb.sample_chains(T.GaussianIso(10), init, **kw)
    thin = hb.sample_chains(T.GaussianIso(10), init, thin=3, **kw)
    torch.cuda.synchronize()
    for blk in (res.samples[:, 1:], thin.samples, res.samples):
        assert_close(DG.summary(blk), O.summary(blk.cpu().numpy()))
    assert_close(DG.summary(res), O.summary(res.samples.cpu().numpy()))         # an HMCResult: its .samples


def test_bayesian_nn_result_with_odd_dimension():
    import torch.nn as nn
    torch.manual_seed(0)
    model = nn.Sequential(nn.Linear(5, 7), nn.Tanh(), nn.Linear(7, 1))      # D = 5*7 + 7 + 7 + 1 = 50
    xx, yy = torch.randn(40, 5), torch.randn(40, 1)
    desc = T.MLPTarget.from_model(model, xx, yy, None, 10.)
    th = hb.util.flatten(model).detach()
    assert th.numel() % 4 != 0
    init = th[None].repeat(4, 1) + 0.01 * torch.randn(4, th.numel(), generator=torch.Generator().manual_seed(1))
    res = hb.sample_chains(desc, init, num_samples=40, num_steps_per_sample=3, step_size=0.005, rng='philox', seed=2)
    torch.cuda.synchronize()
    blk = res.samples[:, 1:]
    assert_close(DG.summary(blk), O.summary(blk.cpu().numpy()))


def test_reference_shaped_list_is_one_chain():
    tgt = T.GaussianDiag(torch.zeros(5), torch.ones(5))
    out = hb.sample(tgt, torch.zeros(5, device='cuda'), num_samples=50, num_steps_per_sample=4, step_size=0.3,
                    verbose=False)
    d = DG.summary(out)
    assert d.num_chains == 1 and d.num_draws == 50
    assert_close(d, O.summary(torch.stack(out).cpu().numpy()[None]))


def test_refused_inputs():
    kw = dict(num_samples=12, num_steps_per_sample=3, step_size=0.2, rng='philox', seed=1)
    init = torch.zeros(3, 8)
    none = hb.sample_chains(T.GaussianIso(8), init, keep_samples=False, moments=True, **kw)
    with pytest.raises(RuntimeError, match='keep_samples=False'):
        DG.summary(none)
    host = hb.sample_chains(T.GaussianIso(8), init, store_on_GPU=False, **kw)
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match='pinned host memory'):
        DG.summary(host)
    with pytest.raises(RuntimeError, match='pinned host memory'):
        DG.summary(host.samples)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        DG.summary(torch.zeros(3, 12, 8))
    with pytest.raises(RuntimeError, match='4 draws'):
        DG.summary(torch.zeros(2, 3, 4, device='cuda'))
    with pytest.raises(RuntimeError, match='float32'):
        DG.summary(torch.zeros(2, 8, 4, device='cuda', dtype=torch.float64))


# ---------------------------------------------------------------------------------------------------------------
# Config 2 end to end: 256 chains x 1000 iterations x D = 1024, plain HMC under Philox
# ---------------------------------------------------------------------------------------------------------------
def test_config2_end_to_end():
    """ESS of the config-2 block equals the oracle's.  Its chains mix like an AR(1) with phi = cos(L*eps) = cos(0.5)
    (tau ~ 15), so split-R-hat of a stationary chain is ~ sqrt(1 + (tau-1)/m) ~ 1.014 at m = 499 draws per half-chain,
    and the definition itself keeps it above 1.01 here; four times the iterations from the same start bring it below."""
    C, D = 256, 1024
    init = 0.1 * torch.randn(C, D, generator=torch.Generator().manual_seed(1234))
    kw = dict(num_steps_per_sample=10, step_size=0.05, rng='philox', seed=0)
    res = hb.sample_chains(T.GaussianIso(D), init, num_samples=1000, **kw)
    blk = res.samples[:, 1:]
    d = DG.summary(blk)
    torch.cuda.synchronize()
    m, N = 499, 2 * C * 499
    stationary = torch.sqrt(1 + (N / d.ess - 1) / m)          # R-hat a converged chain of this ESS has
    assert float(d.rhat.max()) < 1.03
    assert abs(float(d.rhat.median()) - float(stationary.median())) < 0.003
    dims = torch.arange(0, D, 16)                       # the oracle is per dimension: every 16th keeps its host time low
    ref, margin = oracle_with_margin(blk[..., dims].cpu().numpy())
    assert margin > 1e-9
    assert np.allclose(d.ess[dims].cpu().numpy(), ref['ess'], rtol=1e-9, atol=0)
    assert np.array_equal(d.max_lag[dims].cpu().numpy(), ref['max_lag'])
    del res, blk
    long = hb.sample_chains(T.GaussianIso(D), init, num_samples=4000, **kw)
    assert float(DG.summary(long.samples[:, 1:]).rhat.max()) < 1.01
