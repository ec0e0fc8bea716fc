"""Helpers shared by the parity tests.

Tolerances (stated once, used everywhere):
  * element-wise state (positions, momenta, retained samples while the accept sequences agree): the kernel uses
    the reference's fp32 operation order without FMA contraction, so these are compared BIT-EXACT against the
    oracle / golden fixtures.
  * Hamiltonians: a sum over D terms whose summation order differs from torch.dot -> |dH| <= H_TOL_REL * (|U|+|K|)
    i.e. a few fp32 ulps of the partial sums.
  * accept/reject decisions: identical, except that an iteration whose margin |rho - log u| is inside the
    Hamiltonian summation noise may legitimately flip; the comparison stops at such an iteration and the test
    requires that it is rare (never in the committed fixtures).
"""
import json
import os

import numpy as np

H_TOL_REL = 2e-6

# ---------------------------------------------------------------------------------------------------------------------
# Tolerances of the NON-bit-exact comparisons (RMHMC: closed form + Jacobi vs autograd through eigh; coupled / dense /
# Bayesian-NN contractions: summation order) are set from MEASUREMENT, not from a guess: tests/golden/measured_errors.json
# holds, per compared quantity (tag), the error max |a - d| / (1 + |d|) observed on the H100 (regenerate: run the GPU tests with
# HMCX_PARITY_REPORT=<file>.jsonl, then scripts/collect_parity.py).  A comparison passes when its error is within
# TOL_FACTOR x that measurement (floor TOL_FLOOR, so that a re-ordered reduction does not flip a test), and never above the
# test's ceiling -- the old blanket bound (2e-3 RMHMC, 2e-4 contractions).  A tag without a measurement uses the ceiling.
# ---------------------------------------------------------------------------------------------------------------------
TOL_FACTOR = 8.0
TOL_FLOOR = 1e-5
_MEASURED_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'measured_errors.json')
try:
    with open(_MEASURED_PATH) as _f:
        MEASURED = json.load(_f)
except (OSError, ValueError):
    MEASURED = {}


def tol_for(tag, ceiling):
    m = MEASURED.get(tag)
    if m is None:
        return ceiling
    return min(ceiling, max(TOL_FACTOR * m, TOL_FLOOR))


def scaled_error(actual, desired):
    """max |a - d| / (1 + |d|): the quantity np.testing.assert_allclose(rtol=T, atol=T) bounds by T."""
    a, d = np.asarray(actual, dtype=np.float64), np.asarray(desired, dtype=np.float64)
    if a.size == 0:
        return 0.0
    e = np.abs(a - d) / (1.0 + np.abs(d))
    return float(np.nanmax(e)) if np.isfinite(e).any() else float('inf')


def assert_close(tag, actual, desired, ceiling):
    a, d = np.asarray(actual), np.asarray(desired)
    assert a.shape == d.shape, (tag, a.shape, d.shape)
    assert np.array_equal(np.isfinite(a), np.isfinite(d)), tag + ': non-finite pattern differs'
    fin = np.isfinite(d)
    m = scaled_error(a[fin], d[fin])
    rep = os.environ.get('HMCX_PARITY_REPORT')
    if rep:
        with open(rep, 'a') as f:
            f.write(json.dumps({'tag': tag, 'error': m}) + '\n')
    tol = tol_for(tag, ceiling)
    assert m <= tol, '%s: error %.3g > tolerance %.3g (measured: %s, ceiling %.3g)' % (
        tag, m, tol, MEASURED.get(tag), ceiling)

# dual averaging (samplers.py:629-674): fp32 exp/log (CUDA libm vs Sleef, <= 2 ulp) and the summation-order noise of
# rho are amplified by sqrt(t)/(gamma*(t+t0)) <= ~2 into the proposed step size
NUTS_EPS_RTOL = 2e-4


def nuts_eps_rtol(h_scale):
    """Tolerance on a dual-averaging step-size proposal when the Hamiltonians are of size ``h_scale``: rho is a
    difference of two fp32 numbers of that size (ulp = 1.2e-7*h), the recursion multiplies its error by at most ~2
    and accumulates it over the burn-in -> ~1e-6*h, floored at NUTS_EPS_RTOL."""
    return max(NUTS_EPS_RTOL, 1e-6 * float(h_scale))


def first_decision_mismatch(acc_a, acc_b):
    acc_a, acc_b = np.asarray(acc_a).astype(bool), np.asarray(acc_b).astype(bool)
    bad = np.nonzero(acc_a != acc_b)[0]
    return int(bad[0]) if bad.size else None


def assert_chain_parity(samples, accepted, ham, ref_samples, ref_accepted, ref_ham_old, ref_ham_new, ref_logu,
                        burn, exact=True, rtol=0.0, tag=None):
    """samples (S-burn, D) vs reference; accepted (S,); ham (S,2) or None."""
    samples, ref_samples = np.asarray(samples), np.asarray(ref_samples)
    S = len(ref_accepted)
    m = first_decision_mismatch(accepted, ref_accepted)
    if m is not None:
        scale = abs(ref_ham_old[m]) + abs(ref_ham_new[m]) + 1.0
        margin = abs(min(0.0, ref_ham_old[m] - ref_ham_new[m]) - ref_logu[m])
        assert margin <= 20 * H_TOL_REL * scale, (
            'accept decision differs at iteration %d with margin %g (not explainable by summation order)' % (m, margin))
        raise AssertionError('decision flip inside summation noise at iteration %d -- pick another seed' % m)
    if ham is not None:
        ham = np.asarray(ham, dtype=np.float64)
        htol = max(50 * H_TOL_REL, 10 * rtol)
        for col, ref in ((0, ref_ham_old), (1, ref_ham_new)):
            ref = np.asarray(ref, dtype=np.float64)
            ok = np.isfinite(ref) & (np.abs(ref) < 1e30)
            scale = np.abs(ref[ok]) + 1.0
            assert np.all(np.abs(ham[ok, col] - ref[ok]) <= htol * scale), 'Hamiltonian mismatch'
    assert samples.shape == ref_samples.shape, (samples.shape, ref_samples.shape)
    if exact:
        assert np.array_equal(samples, ref_samples), 'samples differ (max abs %g)' % np.abs(samples - ref_samples).max()
    elif tag is not None:
        assert_close(tag + '/samples', samples, ref_samples, rtol)          # measured tolerance, `rtol` is the ceiling
    else:
        np.testing.assert_allclose(samples, ref_samples, rtol=rtol, atol=rtol)
