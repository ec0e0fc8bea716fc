"""CPU: simulation-based calibration (hamiltorch_b200.sbc) without a GPU.

* Philox streams 6 (prior) and 7 (data) of tests/sbc_oracle.py against a scalar Philox4x32-10 written out here (checked
  on the Random123 known-answer vectors), and their counters against those of streams 0-5.
* The oracle's histogram / chi^2 / p against scipy.stats.chisquare with the exact expected counts, and sbc.rank_histogram
  (torch) against the oracle.
* The launch batching and the chain-id rule: balanced launches of 2 .. sims_per_launch sims with disjoint chain ids.
* Every refusal, raised before any CUDA work, and the C ABI's argument checks."""
import ctypes as C
import math

import numpy as np
import pytest
import scipy.stats
import torch
import torch.nn as nn

import hamiltorch_b200 as hb
from hamiltorch_b200 import engine, sbc, targets as T
from tests import philox_ref as P
from tests import sbc_oracle as SO


# ------------------------------------------------------------------------------------------------------------------
# Philox streams 6 and 7
# ------------------------------------------------------------------------------------------------------------------
def _philox_scalar(ctr, key):
    """Philox4x32-10 on Python integers (Salmon et al. 2011)."""
    x, y, z, w = ctr
    k0, k1 = key
    for _ in range(10):
        p0, p1 = 0xD2511F53 * x, 0xCD9E8D57 * z
        x, y, z, w = ((p1 >> 32) ^ y ^ k0, p1 & 0xFFFFFFFF, (p0 >> 32) ^ w ^ k1, p0 & 0xFFFFFFFF)
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return [x, y, z, w]


def test_scalar_philox_known_answers():
    assert _philox_scalar([0, 0, 0, 0], [0, 0]) == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    assert _philox_scalar([0xffffffff] * 4, [0xffffffff] * 2) == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]


@pytest.mark.parametrize('seed', [0, 7, 0x123456789ABCDEF])
def test_prior_and_data_words_match_the_counter_layout(seed):
    sims = [0, 1, 5, 2 ** 32 + 3]                                 # a sim id above 2^32 reaches the key's high word
    words = SO.prior_words(seed, sims, 3, 10)                     # (4, 3, 3, 4)
    dwords = SO.data_words(seed, sims, 3)                         # (4, 3, 4)
    for a, m in enumerate(sims):
        key = [seed & 0xFFFFFFFF, (seed >> 32) ^ (m >> 32)]
        for j in range(3):
            for v in range(3):
                ref = _philox_scalar([v, j, 6 << 24, m & 0xFFFFFFFF], key)
                assert [int(t) for t in words[a, j, v]] == ref
        for v in range(3):
            assert [int(t) for t in dwords[a, v]] == _philox_scalar([v, 0, 7 << 24, m & 0xFFFFFFFF], key)


def test_counters_are_distinct_from_the_other_streams():
    vec = np.arange(0, 40, dtype=np.uint64)[:, None, None]
    n = np.array([0, 1, 2, 2 ** 32 + 1], dtype=np.uint64)[None, :, None]
    chain = np.array([0, 3, 2 ** 32 + 3], dtype=np.uint64)[None, None, :]
    seen = {}
    for s in range(8):
        c = P.counter(s, vec, n, chain).reshape(-1, 4)
        k = P.key(11, np.broadcast_to(chain, np.broadcast_shapes(vec.shape, n.shape, chain.shape))).reshape(-1, 2)
        for row in np.concatenate([c, k], 1):
            t = tuple(int(v) for v in row)
            assert t not in seen, (s, seen.get(t))
            seen[t] = s
    assert SO.STREAM_SBC_PRIOR == 6 and SO.STREAM_SBC_DATA == 7


def test_prior_scaling_and_normals():
    model = nn.Sequential(nn.Linear(3, 4), nn.Tanh(), nn.Linear(4, 2))
    tau = [torch.tensor(t) for t in (1.0, 4.0, 0.25, 2.0)]
    tgt = T.MLPTarget.from_model(model, torch.zeros(5, 3), torch.zeros(5, 2), tau, prior_scale=2.0)
    sd = SO.element_sd(tgt)
    assert sd.shape == (tgt.dim,)
    np.testing.assert_allclose(sd[:12], math.sqrt(2.0), rtol=1e-15)
    np.testing.assert_allclose(sd[12:16], math.sqrt(0.5), rtol=1e-15)
    np.testing.assert_allclose(sd[16:24], math.sqrt(8.0), rtol=1e-15)
    np.testing.assert_allclose(sd[24:], 1.0, rtol=1e-15)
    th = SO.prior(3, range(400), 2, tgt)                          # (400, 3, D): standardised, about N(0, 1)
    z = (th / sd).reshape(-1)
    assert abs(z.mean()) < 0.03 and abs(z.std() - 1.0) < 0.03
    # the first 5 sims of 10 are the 5 sims of a call of 5
    np.testing.assert_array_equal(SO.prior(3, range(5), 2, tgt), SO.prior(3, range(10), 2, tgt)[:5])


def test_simulators_have_the_model_distribution():
    f = np.random.default_rng(0).normal(size=(300, 40, 2))
    y = SO.simulate_regression(1, range(300), f, 4.0)
    r = (y - f).reshape(-1) * 2.0
    assert abs(r.mean()) < 0.03 and abs(r.std() - 1.0) < 0.03
    yb, dist = SO.simulate_binary(1, range(300), f)
    assert set(np.unique(yb)) <= {0.0, 1.0} and dist.shape == f.shape
    p = 1 / (1 + np.exp(-f))
    assert abs((yb - p).mean()) < 0.01
    fc = np.random.default_rng(1).normal(size=(300, 40, 3))
    lab, dist = SO.simulate_multiclass(1, range(300), fc)
    pc = np.exp(fc) / np.exp(fc).sum(-1, keepdims=True)
    for c in range(3):
        assert abs((lab == c).mean() - pc[..., c].mean()) < 0.01


# ------------------------------------------------------------------------------------------------------------------
# Histogram, chi^2, p
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('M, L, B', [(200, 156, 20), (64, 99, 12), (37, 4, 5), (128, 116, 20)])
def test_histogram_matches_scipy_chisquare(M, L, B):
    rk = np.random.default_rng(M + L).integers(0, L + 1, size=(M, 6))
    rk[:, 5] = L                                                  # a column with every rank at the top
    hist, expected, chi2, p = SO.histogram(rk, L, B)
    assert hist.sum(1).tolist() == [M] * 6 and math.isclose(expected.sum(), M, rel_tol=1e-12)
    for c in range(6):
        ref = scipy.stats.chisquare(hist[c], expected)
        assert math.isclose(chi2[c], ref.statistic, rel_tol=1e-12)
        assert math.isclose(p[c], ref.pvalue, rel_tol=1e-9, abs_tol=1e-300)
    assert p[5] < 1e-10
    h, e, c2, pv = sbc.rank_histogram(torch.tensor(rk, dtype=torch.int32), L, B)
    np.testing.assert_array_equal(h.numpy(), hist)
    np.testing.assert_allclose(e.numpy(), expected, rtol=1e-15)
    np.testing.assert_allclose(c2.numpy(), chi2, rtol=1e-12)
    np.testing.assert_allclose(pv.numpy(), p, rtol=1e-9, atol=1e-300)
    assert c2.dtype == torch.float64 and pv.dtype == torch.float64


def test_default_bins():
    assert [sbc.default_bins(m) for m in (2, 9, 10, 64, 100, 200, 1000)] == [2, 2, 2, 12, 20, 20, 20]


# ------------------------------------------------------------------------------------------------------------------
# Launch batching and chain ids
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('spl', [2, 3, 7, 32, 64])
@pytest.mark.parametrize('R', [1, 4])
def test_batches_are_balanced_with_disjoint_chain_ids(spl, R):
    for M in list(range(2, 70)) + [128, 129, 200, 1000]:
        parts = sbc.batches(M, spl)
        assert [a for a, _ in parts] == list(np.cumsum([0] + [k for _, k in parts])[:-1])
        sizes = [k for _, k in parts]
        assert sum(sizes) == M and max(sizes) - min(sizes) <= 1 and min(sizes) >= 2
        assert max(sizes) <= (spl if not (spl == 2 and M % 2) else 3)
        if spl > 2 or M % 2 == 0:
            assert len(parts) == -(-M // spl)
        ids = []
        for a, k in parts:
            off = sbc.chain_offset(a, k, R)
            assert off % k == 0 and off >= a * (R + 1)
            ids += list(range(off, off + R * k))
        assert len(set(ids)) == len(ids)


# ------------------------------------------------------------------------------------------------------------------
# Refusals: before any CUDA work
# ------------------------------------------------------------------------------------------------------------------
def _reg(n=20, loss='regression', n_out=1, tau_out=4.0):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(n, 3, generator=g)
    y = torch.randn(n, n_out, generator=g) if loss in ('regression', 'binary_class_linear_output') else \
        torch.randint(0, n_out, (n,), generator=g).float()
    model = nn.Linear(3, n_out) if loss != 'multi_class_log_softmax_output' else \
        nn.Sequential(nn.Linear(3, n_out), nn.LogSoftmax(dim=1))
    return T.MLPTarget.from_model(model, x, y, None, tau_out, model_loss=loss)


def test_refusals_of_the_likelihood_and_the_target():
    with pytest.raises(NotImplementedError, match='MEAN'):
        sbc.simulate(_reg(loss='multi_class_log_softmax_output', n_out=3, tau_out=1.0), 10)
    for loss, k in (('binary_class_linear_output', 1), ('multi_class_linear_output', 3)):
        with pytest.raises(NotImplementedError, match='tau_out'):
            sbc.simulate(_reg(loss=loss, n_out=k, tau_out=2.0), 10)
    nodata = T.MLPTarget.from_model(nn.Linear(3, 1), None, None)
    with pytest.raises(ValueError, match='no data'):
        sbc.simulate(nodata, 10)
    with pytest.raises(NotImplementedError, match='split'):
        sbc.run([_reg(), _reg()], 10)
    with pytest.raises(NotImplementedError, match='MLPTarget'):
        sbc.simulate(T.GaussianIso(3), 10)
    for fn in (lambda t, **k: sbc.simulate(t, **k), lambda t, **k: sbc.run(t, **k)):
        with pytest.raises(ValueError, match='num_sims'):
            fn(_reg(), num_sims=1)
        with pytest.raises(ValueError, match='chains_per_sim'):
            fn(_reg(), num_sims=10, chains_per_sim=0)


def test_refusals_of_the_sampling_arguments():
    t = _reg()
    cases = [(dict(integrator=hb.Integrator.SPLITTING), NotImplementedError),
             (dict(sampler=hb.Sampler.RMHMC), NotImplementedError),
             (dict(tau_prior=(2.0, 1.0)), NotImplementedError),
             (dict(tau_out_prior=(2.0, 1.0)), NotImplementedError),
             (dict(betas=[1.0, 0.5]), NotImplementedError),
             (dict(adapt_mass=True, sampler=hb.Sampler.HMC_NUTS, burn=30, num_samples=60), NotImplementedError),
             (dict(inv_mass=torch.eye(t.dim)), NotImplementedError),
             (dict(inv_mass=[torch.eye(2), torch.eye(t.dim - 2)]), NotImplementedError),
             (dict(folds=torch.zeros(20, dtype=torch.int64)), NotImplementedError),
             (dict(num_samples=5, burn=5), RuntimeError),
             (dict(sampler=hb.Sampler.HMC_NUTS, burn=0), RuntimeError),
             (dict(num_samples=5, burn=3, thin=2), ValueError),     # one retained slot: params_init only
             (dict(thin=0), ValueError),
             (dict(store_on_GPU=False), TypeError)]
    for kw, err in cases:
        with pytest.raises(err):
            sbc.fit(None, t, **kw)
        with pytest.raises(err):
            sbc.run(t, 10, **kw)
    for spl in (0, 1, 65, 2.5, True):
        with pytest.raises(ValueError, match='sims_per_launch'):
            sbc.run(t, 10, sims_per_launch=spl)
    for bins in (1, 0, 42, 3.5):                                  # L + 1 = 4 (10 - 0 - 1) + 1 = 37 with R = 4
        with pytest.raises(ValueError, match='bins'):
            sbc.run(t, 10, bins=bins)
    # the accepted values of the refused keywords pass the checks (they stop at the missing GPU, not at a refusal)
    assert sbc._fit_args(dict(adapt_mass=False, betas=None, sampler=hb.Sampler.HMC_NUTS, burn=2))['burn'] == 2


# ------------------------------------------------------------------------------------------------------------------
# C ABI: argument checks return before any CUDA work
# ------------------------------------------------------------------------------------------------------------------
def test_abi_sbc_entries_check_their_arguments(built_library):
    from hamiltorch_b200 import _native as N
    lib = N.load_library()
    junk = C.c_void_p(16)
    t = _reg()
    nt = engine.NativeTarget(t, 'cpu')
    ld = N.padded_ld(nt.dim)
    assert lib.hmcx_sbc_prior(None, 0, 0, 4, 2, ld, junk, None) == N.ERR_INVALID_ARG
    assert lib.hmcx_sbc_prior(engine.NativeTarget(T.GaussianIso(4), 'cpu').ref(), 0, 0, 4, 2, 4, junk, None) == \
        N.ERR_UNSUPPORTED
    for M, R, ldx, s0 in ((0, 2, ld, 0), (4, -1, ld, 0), (4, 2, ld - 4, 0), (4, 2, ld + 2, 0), (4, 2, ld, -1)):
        assert lib.hmcx_sbc_prior(nt.ref(), 0, s0, M, R, ldx, junk, None) == N.ERR_INVALID_ARG
    assert lib.hmcx_sbc_prior(nt.ref(), 0, 0, 4, 2, ld, None, None) == N.ERR_INVALID_ARG
    nd = engine.NativeTarget(T.MLPTarget.from_model(nn.Linear(3, 1), None, None), 'cpu')
    assert lib.hmcx_sbc_prior(nd.ref(), 0, 0, 4, 2, ld, junk, None) == N.ERR_INVALID_ARG
    assert lib.hmcx_sbc_simulate(nt.ref(), None, 0, 0, 4, junk, None) == N.ERR_INVALID_ARG
    assert lib.hmcx_sbc_simulate(nt.ref(), junk, 0, 0, 0, junk, None) == N.ERR_INVALID_ARG
    for loss, k, tau in (('multi_class_log_softmax_output', 3, 1.0), ('binary_class_linear_output', 1, 2.0),
                         ('multi_class_linear_output', 3, 0.5)):
        bad = engine.NativeTarget(_reg(loss=loss, n_out=k, tau_out=tau), 'cpu')
        assert lib.hmcx_sbc_simulate(bad.ref(), junk, 0, 0, 4, junk, None) == N.ERR_UNSUPPORTED, loss

    def rank(C_=8, keep=5, K=4, D=3, cs=40, ds=8, ts=8, x=junk):
        return lib.hmcx_sbc_rank(x, cs, ds, C_, keep, K, D, junk, ts, junk, None)

    for kw in (dict(x=None), dict(C_=0), dict(K=0), dict(C_=6), dict(keep=1), dict(D=0), dict(cs=-1), dict(ds=-1),
               dict(ts=-1)):
        assert rank(**kw) == N.ERR_INVALID_ARG, kw
