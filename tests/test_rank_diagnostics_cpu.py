"""CPU: the numpy definition of rank-normalised R-hat, bulk / tail ESS and quantiles (tests/rank_oracle.py) against
hand-made ranks and Vehtari et al.'s motivating cases; the split-R-hat-only helper of hamiltorch_b200.diagnostics
against the full host scan; the argument checks of the ABI v10 entries and of ``rank_summary``."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy import special

from hamiltorch_b200 import diagnostics as DG
from oracle import diagnostics_oracle as O
from tests import rank_oracle as R
from tests.test_diagnostics_cpu import OraclePartials, ar1


@pytest.fixture(scope='module')
def rank_library():
    """libhmcx.so built in-tree and loaded (nvcc cross-compiles without a GPU)."""
    from hamiltorch_b200 import _native as N
    from hamiltorch_b200 import build
    build.build()
    return N.load_library()


def test_bulk_z_of_a_tie_free_block_is_argsort_of_argsort():
    x = np.random.default_rng(0).standard_normal((3, 10, 4)).astype(np.float32)
    t = R.rank_transform(x)
    ys = x.astype(np.float64).reshape(-1, 4)                    # n even: every draw is in the split set
    r = np.argsort(np.argsort(ys, axis=0), axis=0) + 1.0
    want = special.ndtri((r - 0.375) / (ys.shape[0] + 0.25)).astype(np.float32).reshape(3, 10, 4)
    assert np.array_equal(t['bulk_z'], want)


def test_ties_share_their_mean_rank():
    x = np.array([1, 2, 2, 3], dtype=np.float32)[None, :, None]
    z = R.rank_transform(x)['bulk_z'][0, :, 0]
    r = np.array([1, 2.5, 2.5, 4])
    assert np.array_equal(z, special.ndtri((r - 0.375) / 4.25).astype(np.float32))


def test_negative_zero_ties_with_positive_zero():
    x = np.array([-0.0, 0.0, 1.0, -1.0], dtype=np.float32)[None, :, None]
    z = R.rank_transform(x)['bulk_z'][0, :, 0]
    assert z[0] == z[1] and z[3] < z[0] < z[2]


def test_odd_n_middle_draw_enters_quantiles_but_not_ranks():
    x = np.array([0.0, 1.0, 100.0, 2.0, 3.0], dtype=np.float32)[None, :, None]      # n = 5: draw 2 is dropped
    t = R.rank_transform(x)
    assert t['median'][0] == 2.0                                 # np.median of all five, not of [0, 1, 2, 3]
    assert t['q95'][0] == np.quantile([0, 1, 100, 2, 3], 0.95) and t['q95'][0] > 3
    assert t['bulk_z'][0, 2, 0] == 0                             # the dropped draw holds no score
    r = np.array([1, 2, 3, 4])                                   # ranks of 0, 1, 2, 3 among the four split draws
    assert np.array_equal(t['bulk_z'][0, [0, 1, 3, 4], 0], special.ndtri((r - 0.375) / 4.25).astype(np.float32))
    # folded: |x - 2| of the split draws 0, 1, 2, 3 = 2, 1, 0, 1 -> ranks 4, 2.5, 1, 2.5
    f = np.array([4, 2.5, 1, 2.5])
    assert np.array_equal(t['fold_z'][0, [0, 1, 3, 4], 0], special.ndtri((f - 0.375) / 4.25).astype(np.float32))


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_scale_disagreement_is_caught_by_rhat_tail_only(seed):
    x = np.random.default_rng(seed).standard_normal((4, 1000, 3))
    x[3] *= 3.0
    x = x.astype(np.float32)
    assert np.all(O.summary(x)['rhat'] < 1.01)
    r = R.rank_summary(x)
    assert np.all(r['rhat_tail'] > 1.05) and np.array_equal(r['rhat'], np.maximum(r['rhat_bulk'], r['rhat_tail']))


def test_cauchy_chains_have_bulk_ess_near_ns():
    x = np.random.default_rng(0).standard_cauchy((4, 1000, 3)).astype(np.float32)
    r = R.rank_summary(x)
    assert np.all(np.abs(r['ess_bulk'] / 4000 - 1) < 0.15), r['ess_bulk']
    assert np.all(np.isfinite(r['ess_tail'])) and np.all(r['rhat'] < 1.01)


def test_rank_outputs_are_invariant_under_a_monotone_map():
    x = ar1(3, 301, 4, 0.7, 5).astype(np.float64)
    a, b = R.rank_summary(x), R.rank_summary(np.exp(x))
    for k in ('rhat_bulk', 'ess_bulk', 'ess_tail'):
        assert np.array_equal(a[k], b[k]), k
    assert np.allclose(np.exp(a['median']), b['median'], rtol=1e-12)


def test_edge_dimensions():
    x = ar1(3, 40, 5, 0.3, 6)
    x[:, :, 1] = 2.5
    x[0, 7, 2] = np.nan
    x[1, 3, 3] = -np.inf
    x[0, :, 4], x[1, :, 4], x[2, :, 4] = 1.0, 2.0, 1.0
    r = R.rank_summary(x)
    assert (r['ess_bulk'][1], r['ess_tail'][1], r['rhat'][1]) == (120, 120, 1.0)
    for d in (2, 3):
        assert all(np.isnan(r[k][d]) for k in ('rhat', 'rhat_bulk', 'rhat_tail', 'ess_bulk', 'ess_tail', 'q05',
                                               'median', 'q95'))
    assert np.isinf(r['rhat_bulk'][4])


@pytest.mark.parametrize('C,n,D,phi', [(1, 8, 3, 0.0), (2, 9, 2, 0.5), (7, 501, 3, 0.9)])
def test_rhat_helper_equals_the_full_scan(C, n, D, phi):
    x = ar1(C, n, D, phi, 30 + n)
    x[..., 0] = 1.5 if D > 2 else x[..., 0]
    full = DG.summary_from_partials(OraclePartials(x))
    assert torch.equal(DG._rhat_from_partials(OraclePartials(x)), full.rhat)


def test_abi_entries_reject_invalid_arguments(rank_library):
    from hamiltorch_b200 import _native as N
    lib = rank_library
    buf = C.c_void_p(16)                                     # never dereferenced: validation returns first
    nb = lib.hmcx_rank_workspace_bytes(2, 8, 3)
    assert nb > 0 and lib.hmcx_rank_workspace_bytes(2, 8, 6) > nb
    assert lib.hmcx_rank_workspace_bytes(2, 3, 3) == 0                                        # n < 4
    assert lib.hmcx_rank_workspace_bytes(0, 8, 3) == 0                                        # no chain
    assert lib.hmcx_rank_workspace_bytes(2, 8, 0) == 0                                        # no dimension
    assert lib.hmcx_rank_workspace_bytes(1 << 16, 1 << 15, 1) == 0                            # C*n beyond int32

    def rank_pass(x=buf, C_=2, n=8, D=4, d0=0, k=3, bz=buf, bcs=32, fz=buf, q=buf, flag=buf, ws=buf, wsb=nb, cs=32):
        return lib.hmcx_rank_pass(x, cs, 4, C_, n, D, d0, k, bz, bcs, 4, fz, 32, 4, q, flag, ws, wsb, None)
    assert rank_pass(x=None) == N.ERR_INVALID_ARG
    assert rank_pass(n=3) == N.ERR_INVALID_ARG
    assert rank_pass(C_=0) == N.ERR_INVALID_ARG
    assert rank_pass(d0=2, k=3) == N.ERR_INVALID_ARG                                          # slab past D
    assert rank_pass(d0=-1) == N.ERR_INVALID_ARG
    assert rank_pass(k=0) == N.ERR_INVALID_ARG
    assert rank_pass(bz=None) == N.ERR_INVALID_ARG
    assert rank_pass(fz=None) == N.ERR_INVALID_ARG
    assert rank_pass(q=None) == N.ERR_INVALID_ARG
    assert rank_pass(flag=None) == N.ERR_INVALID_ARG
    assert rank_pass(ws=None) == N.ERR_INVALID_ARG
    assert rank_pass(wsb=nb - 1) == N.ERR_INVALID_ARG                                         # workspace too small
    assert rank_pass(bcs=-1) == N.ERR_INVALID_ARG
    assert rank_pass(cs=-1) == N.ERR_INVALID_ARG
    assert rank_pass(C_=1 << 16, n=1 << 15) == N.ERR_INVALID_ARG
    ind = lib.hmcx_rank_indicator
    assert ind(None, 32, 4, 2, 8, 4, buf, buf, 32, 4, None) == N.ERR_INVALID_ARG
    assert ind(buf, 32, 4, 2, 8, 4, None, buf, 32, 4, None) == N.ERR_INVALID_ARG                 # no threshold
    assert ind(buf, 32, 4, 2, 8, 4, buf, None, 32, 4, None) == N.ERR_INVALID_ARG
    assert ind(buf, 32, 4, 2, 3, 4, buf, buf, 32, 4, None) == N.ERR_INVALID_ARG                  # n < 4
    assert ind(buf, 32, 4, 2, 8, 4, buf, buf, -32, 4, None) == N.ERR_INVALID_ARG
    assert N.RANK_MAX_DRAWS == (1 << 31) - (1 << 16)


def test_rank_pass_rejects_a_slab_beyond_the_grid_limit(rank_library):
    from hamiltorch_b200 import _native as N
    lib = rank_library
    buf = C.c_void_p(16)
    K = N.RANK_MAX_SLAB
    assert K == 65535 and lib.hmcx_rank_workspace_bytes(4, 25, K) > 0
    assert lib.hmcx_rank_workspace_bytes(4, 25, K + 1) == 0
    nb = lib.hmcx_rank_workspace_bytes(4, 25, K)
    args = (buf, 100 * (K + 1), K + 1, 4, 25, K + 1)
    assert lib.hmcx_rank_pass(*args, 0, K + 1, buf, 100 * (K + 1), K + 1, buf, 100 * (K + 1), K + 1, buf, buf, buf,
                              1 << 40, None) == N.ERR_INVALID_ARG


def test_slab_size_stays_within_the_grid_limit(rank_library):
    from hamiltorch_b200 import _native as N
    assert DG._slab_dims(rank_library, 4, 25, 200000) == N.RANK_MAX_SLAB      # the budget alone would allow more
    assert DG.RANK_WORKSPACE_BUDGET // rank_library.hmcx_rank_workspace_bytes(4, 25, 1) > N.RANK_MAX_SLAB
    assert DG._slab_dims(rank_library, 256, 999, 1024) < 1024


def test_rank_summary_refuses_what_summary_refuses():
    import hamiltorch_b200 as hb
    from hamiltorch_b200.engine import HMCResult
    for bad, exc, msg in ((torch.zeros(2, 10, 3), RuntimeError, 'no CPU fallback'),
                          ([torch.zeros(3) for _ in range(10)], RuntimeError, 'no CPU fallback'),
                          (HMCResult(None, None, None, None, None, None, 3, 10), RuntimeError, 'keep_samples=False'),
                          (3.0, TypeError, 'expected an HMCResult')):
        with pytest.raises(exc) as a:
            hb.diagnostics.summary(bad)
        with pytest.raises(exc) as b:
            hb.diagnostics.rank_summary(bad)
        assert str(a.value) == str(b.value) and msg in str(b.value)
