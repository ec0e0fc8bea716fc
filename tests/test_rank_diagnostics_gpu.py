"""GPU: hamiltorch_b200.diagnostics.rank_summary (the rank pass of hmcx_rank.cu, then the split-R-hat / ESS passes on
its score and indicator blocks) against the numpy definition (tests/rank_oracle.py) on the same fp32 blocks: the shapes
of the split-R-hat tests, ties from real runs, edge dimensions, and invariances of the definition."""
import numpy as np
import pytest
import torch

import hamiltorch_b200 as hb
from hamiltorch_b200 import _native as N
from hamiltorch_b200 import diagnostics as DG
from hamiltorch_b200 import targets as T
from oracle import diagnostics_oracle as O
from tests import rank_oracle as R
from tests.test_diagnostics_gpu import CASES, ar1, padded_block

pytestmark = pytest.mark.gpu

KEYS = ('rhat', 'rhat_bulk', 'rhat_tail', 'ess_bulk', 'ess_tail')


def geyer_margin(x):
    """The smallest |pair sum| the oracle's Geyer scans on a block compare against 0 (as test_diagnostics_gpu)."""
    y = O.split_chains(x)
    K, m, D = y.shape
    mu = y.mean(1)
    yc = y - mu[:, None, :]
    g0 = O.autocov_centered(yc, 0).mean(0)
    W = m / (m - 1) * g0
    varp = (m - 1) / m * W + ((mu - mu.mean(0)) ** 2).sum(0) / (K - 1)
    ref = O.summary(x)
    margin = np.inf
    for d in range(D):
        lag = int(ref['max_lag'][d])
        if lag == 0:
            continue
        with np.errstate(invalid='ignore', divide='ignore'):
            rho = np.array([1.0 if t == 0 else 1.0 - (W[d] - O.autocov_centered(yc[..., d:d + 1], t).mean(0)[0])
                            / varp[d] for t in range(lag + 1)])
        margin = min(margin, np.abs(rho[0::2][:len(rho[1::2])] + rho[1::2]).min())
    return margin


def rank_blocks_on_gpu(x):
    """The bulk / folded scores, quantiles and flags of one rank pass over the whole (C, n, D) device block."""
    lib = N.load_library()
    C, n, D = x.shape
    bz = torch.empty((C, n, D), dtype=torch.float32, device=x.device)
    fz = torch.empty_like(bz)
    q = torch.empty((3, D), dtype=torch.float64, device=x.device)
    flag = torch.empty(D, dtype=torch.int32, device=x.device)
    nb = lib.hmcx_rank_workspace_bytes(C, n, D)
    ws = torch.empty(nb, dtype=torch.uint8, device=x.device)
    rc = lib.hmcx_rank_pass(N.ptr(x), x.stride(0), x.stride(1), C, n, D, 0, D, N.ptr(bz), bz.stride(0), bz.stride(1),
                            N.ptr(fz), fz.stride(0), fz.stride(1), N.ptr(q), N.ptr(flag), N.ptr(ws), nb,
                            N.stream_ptr(x.device))
    N.check(rc, 'hmcx_rank_pass')
    torch.cuda.synchronize()
    return bz.cpu().numpy(), fz.cpu().numpy(), q.cpu().numpy(), flag.cpu().numpy()


def ulp_mismatches(got, ref):
    """Elements differing, and the largest difference in fp32 ulps."""
    g = got.view(np.int32).astype(np.int64)
    r = ref.view(np.int32).astype(np.int64)
    g = np.where(g < 0, -(g & 0x7fffffff), g)
    r = np.where(r < 0, -(r & 0x7fffffff), r)
    d = np.abs(g - r)
    return int((d > 0).sum()), int(d.max()) if d.size else 0


def assert_quantiles_equal(g, r):
    """Bit-equal, except that a zero quantile is +0.0 where numpy may return -0.0 (equal as values)."""
    assert np.array_equal(g, r, equal_nan=True)
    nz = np.isfinite(r) & (r != 0)
    assert np.array_equal(g[nz].view(np.int64), r[nz].view(np.int64))
    assert not np.signbit(g[np.isfinite(g) & (g == 0)]).any()


def assert_rank_close(got, ref, rtol=1e-9):
    for k in KEYS + ('q05', 'median', 'q95'):
        g = getattr(got, k).cpu().numpy()
        r = ref[k]
        assert np.array_equal(np.isnan(g), np.isnan(r)), k
        assert np.array_equal(np.isinf(g), np.isinf(r)), k
        ok = np.isfinite(r)
        if k in ('q05', 'median', 'q95'):
            assert_quantiles_equal(g, r)
            continue
        err = np.abs(g[ok] - r[ok]) / np.maximum(np.abs(r[ok]), 1e-300)
        assert err.size == 0 or err.max() <= rtol, (k, err.max())
    assert np.array_equal(got.max_lag.cpu().numpy(), ref['max_lag'])


def oracle_on_scores(host, bz, fz, q):
    """The oracle's R-hat / ESS on given score blocks (and the indicators of the given quantiles)."""
    bulk, fold = O.summary(bz), O.summary(fz)
    s05 = O.summary((host <= q[0][None, None]).astype(np.float32))
    s95 = O.summary((host <= q[2][None, None]).astype(np.float32))
    out = {'rhat_bulk': bulk['rhat'], 'rhat_tail': fold['rhat'], 'ess_bulk': bulk['ess'],
           'ess_tail': np.minimum(s05['ess'], s95['ess']), 'q05': q[0], 'median': q[1], 'q95': q[2]}
    out['rhat'] = np.maximum(out['rhat_bulk'], out['rhat_tail'])
    bad = ref_nonfinite(host)
    out = {k: np.where(bad, np.nan, v) for k, v in out.items()}
    out['max_lag'] = np.stack([np.where(bad, 0, r['max_lag']) for r in (bulk, s05, s95)])
    return out


def check_against_oracle(blk, max_ulp_elements=8):
    """The rank pass against the oracle: quantiles bit-equal, the bulk and folded fp32 scores equal up to a handful of
    1-ulp differences (CUDA normcdfinv vs scipy ndtri), counted and returned.  rank_summary's R-hat / ESS within 1e-9
    of the oracle's on the same scores, with the same max_lag; where no score differs, that is the oracle itself."""
    host = blk.cpu().numpy()
    ref = R.rank_summary(host)
    bz, fz, q, flag = rank_blocks_on_gpu(blk)
    bad = ref_nonfinite(host)
    assert np.array_equal(flag != 0, bad)
    for k, row in (('q05', 0), ('median', 1), ('q95', 2)):
        assert_quantiles_equal(q[row], ref[k])
    counts = []
    for got, want in ((bz, ref['bulk_z']), (fz, ref['fold_z'])):
        cnt, worst = ulp_mismatches(got[..., ~bad], want[..., ~bad])
        assert worst <= 1 and cnt <= max_ulp_elements, (cnt, worst)
        counts.append(cnt)
    on_scores = oracle_on_scores(host, bz, fz, q)
    for series in (bz, fz, (host <= q[0][None, None]).astype(np.float32), (host <= q[2][None, None]).astype(np.float32)):
        if (~bad).any():
            assert geyer_margin(series[..., ~bad]) > 1e-9       # no Geyer decision within rounding of its threshold
    got = DG.rank_summary(blk)
    torch.cuda.synchronize()
    assert got.num_chains == host.shape[0] and got.num_draws == host.shape[1]
    assert_rank_close(got, on_scores)
    if sum(counts) == 0:
        assert_rank_close(got, ref)
    return counts


def ref_nonfinite(x):
    return ~np.isfinite(x.reshape(-1, x.shape[-1])).all(0)


@pytest.mark.parametrize('C,n,D,phi,mean,scale', CASES)
def test_rank_summary_matches_oracle(C, n, D, phi, mean, scale):
    x = ar1(C, n, D, phi, 2000 + C * 7 + n + D, mean, scale)
    counts = check_against_oracle(padded_block(x))
    print('1-ulp score differences (bulk, folded): %s' % counts)


# ---------------------------------------------------------------------------------------------------------------
# Ties from real runs
# ---------------------------------------------------------------------------------------------------------------
def test_low_acceptance_run_repeats_rows():
    init = torch.randn(6, 300, generator=torch.Generator().manual_seed(11))
    res = hb.sample_chains(T.GaussianIso(300), init, num_samples=120, num_steps_per_sample=10, step_size=0.5,
                           rng='philox', seed=5)
    torch.cuda.synchronize()
    blk = res.samples[:, 1:]
    host = blk.cpu().numpy()
    assert (host[:, 1:] == host[:, :-1]).all(-1).sum() > 100                    # rejections repeat rows: ties
    check_against_oracle(blk)


def test_bayesian_nn_block_with_odd_dimension():
    import torch.nn as nn
    torch.manual_seed(0)
    model = nn.Sequential(nn.Linear(5, 7), nn.Tanh(), nn.Linear(7, 1))      # D = 50
    xx, yy = torch.randn(40, 5), torch.randn(40, 1)
    desc = T.MLPTarget.from_model(model, xx, yy, None, 10.)
    th = hb.util.flatten(model).detach()
    init = th[None].repeat(4, 1) + 0.01 * torch.randn(4, th.numel(), generator=torch.Generator().manual_seed(1))
    res = hb.sample_chains(desc, init, num_samples=40, num_steps_per_sample=3, step_size=0.005, rng='philox', seed=2)
    torch.cuda.synchronize()
    check_against_oracle(res.samples[:, 1:])


def test_many_exact_duplicates():
    rng = np.random.default_rng(3)
    x = rng.integers(-3, 4, size=(6, 301, 37)).astype(np.float32) * 0.5
    x[:, ::7, 5] = -0.0                                                        # -0.0 ties with +0.0
    x[:, :, 6] = np.where(rng.random((6, 301)) < 0.5, 0.0, -0.0)
    check_against_oracle(padded_block(x))


def test_edge_case_dimensions_match_oracle():
    x = ar1(3, 40, 7, 0.3, 6)
    x[:, :, 1] = 2.5                                    # constant
    x[0, 7, 2] = np.nan
    x[1, 3, 3] = np.inf
    x[2, 5, 5] = -np.inf
    x[0, :, 4], x[1, :, 4], x[2, :, 4] = 1.0, 2.0, 1.0     # W = 0, B > 0
    blk = padded_block(x)
    got = DG.rank_summary(blk)
    ref = R.rank_summary(x)
    assert_rank_close(got, ref)
    Ns = 3 * 2 * 20
    assert float(got.ess_bulk[1]) == Ns and float(got.rhat[1]) == 1 and float(got.ess_tail[1]) == Ns
    for d in (2, 3, 5):
        assert all(torch.isnan(getattr(got, k)[d]) for k in KEYS + ('q05', 'median', 'q95'))
    assert torch.isinf(got.rhat_bulk[4])


def test_more_dimensions_than_one_slab_takes():
    """D > HMCX_RANK_MAX_SLAB at a small C*n, where the workspace budget alone would ask for a larger slab: two
    slabs, each dimension as in a block of its own, and the oracle on dimensions either side of the slab edge."""
    C, n, D = 4, 25, N.RANK_MAX_SLAB + 4465
    x = ar1(C, n, D, 0.5, 12)
    blk = torch.from_numpy(x).cuda()
    got = DG.rank_summary(blk)
    tail = DG.rank_summary(blk[..., N.RANK_MAX_SLAB - 40:])
    torch.cuda.synchronize()
    for k in KEYS + ('q05', 'median', 'q95'):
        assert torch.equal(getattr(got, k)[N.RANK_MAX_SLAB - 40:], getattr(tail, k)), k
    dims = np.r_[0:8, N.RANK_MAX_SLAB - 8:N.RANK_MAX_SLAB + 8, D - 8:D]
    ref = R.rank_summary(x[..., dims])
    for k in KEYS:
        assert np.allclose(getattr(got, k).cpu().numpy()[dims], ref[k], rtol=1e-9, atol=0), k
    for k in ('q05', 'median', 'q95'):
        assert_quantiles_equal(getattr(got, k).cpu().numpy()[dims], ref[k])


# ---------------------------------------------------------------------------------------------------------------
# Invariance
# ---------------------------------------------------------------------------------------------------------------
def _fields(d):
    return [getattr(d, k) for k in KEYS + ('q05', 'median', 'q95', 'max_lag')]


def test_repeated_calls_are_bitwise_equal():
    x = padded_block(ar1(64, 301, 90, 0.9, 7))
    for a, b in zip(_fields(DG.rank_summary(x)), _fields(DG.rank_summary(x))):
        assert torch.equal(a, b)


def test_doubling_keeps_ranks_and_folds():
    x = padded_block(ar1(16, 203, 40, 0.7, 8))
    a, b = DG.rank_summary(x), DG.rank_summary(2 * x)
    for k in KEYS:
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    assert torch.equal(2 * a.median, b.median) and torch.equal(a.max_lag, b.max_lag)


def test_slab_of_eight_dimensions_gives_the_same_bits(monkeypatch):
    x = padded_block(ar1(9, 151, 61, 0.8, 9))
    one = DG.rank_summary(x)
    monkeypatch.setattr(DG, '_slab_dims_override', 8)
    eight = DG.rank_summary(x)
    for a, b in zip(_fields(one), _fields(eight)):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------
# Config 2 end to end: 256 chains x 1000 iterations x D = 1024, plain HMC under Philox
# ---------------------------------------------------------------------------------------------------------------
def test_config2_end_to_end():
    C, D = 256, 1024
    init = 0.1 * torch.randn(C, D, generator=torch.Generator().manual_seed(1234))
    res = hb.sample_chains(T.GaussianIso(D), init, num_samples=1000, num_steps_per_sample=10, step_size=0.05,
                           rng='philox', seed=0)
    blk = res.samples[:, 1:]
    r = DG.rank_summary(blk)
    s = DG.summary(blk)
    torch.cuda.synchronize()
    assert float(r.rhat.max()) < 1.03
    assert abs(float(r.ess_bulk.median()) / float(s.ess.median()) - 1) < 0.05
    dims = torch.arange(0, D, 16)
    host = blk[..., dims].cpu().numpy()
    ref = R.rank_summary(host)
    for k in KEYS:
        g = getattr(r, k)[dims].cpu().numpy()
        assert np.allclose(g, ref[k], rtol=1e-6, atol=0), (k, np.max(np.abs(g - ref[k]) / ref[k]))
    for k in ('q05', 'median', 'q95'):
        assert np.array_equal(getattr(r, k)[dims].cpu().numpy(), ref[k]), k
    assert np.array_equal(r.max_lag[:, dims].cpu().numpy(), ref['max_lag'])
