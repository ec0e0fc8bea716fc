"""numpy fp64 definition of power-scaling sensitivity (hamiltorch_b200/sensitivity.py, hmcx_psens.cu; Kallioinen,
Paananen, Buerkner & Vehtari 2023).  Draws are pooled as g = c n + s.

  components  log_prior: the Normal(0, tau^-1/2) log densities of the parameter tensors with a fixed tau, times M /
              prior_scale for M splits of the target, plus log Gamma(tau; a, b) of every sampled tau; log_lik: the
              per-row log-likelihoods summed (regression), tau_out times their sum (binary, multi-class) or tau_out times
              the sum over splits of the split's mean (LogSoftmax output).
  weights     per weight set (component, alpha): r = (alpha - 1) component in fp64, -r rounded to fp32, Pareto-smoothed
              as psis_loo smooths one point's ll (ppc_oracle.psis_weights: the GPU's stable-sort order).
  cjs         over the draws sorted ascending, widths d_j = x_(j+1) - x_(j) (the last x_(S) - x_(S-1)), prefix sums P_j of
              p = 1/S and Q_j of q: sqrt(sum d [P log2(2P/(P+Q)) + Q log2(2Q/(P+Q))] / sum d (P+Q)) (0 log 0 = 0, 0 when
              the denominator is 0; a negative rounding of the numerator counts as 0), then max over x and -x.
"""
import math

import numpy as np
from scipy import special

from tests import loo_oracle as LO
from tests import ppc_oracle as PO

THRESHOLD = 0.05


def normal_log_prior(theta, sizes, taus):
    """theta (S, D) -> (S,): sum over the tensors with tau > 0 of the Normal(0, tau^-1/2) log densities."""
    th = np.asarray(theta, np.float64)
    out = np.zeros(th.shape[0])
    i = 0
    for n, tau in zip(sizes, taus):
        if tau > 0:
            w = th[:, i:i + n]
            out += (-0.5 * tau * w * w + 0.5 * (math.log(tau) - math.log(2 * math.pi))).sum(1)
        i += n
    return out


def gamma_log_pdf(t, a, b):
    t = np.asarray(t, np.float64)
    return a * math.log(b) - special.gammaln(a) + (a - 1.0) * np.log(t) - b * t


def regression_ll(samples, target, tau):
    """(S, N) normalised Gaussian log-likelihoods with a per-draw noise precision tau (S,)."""
    import copy
    t1 = [copy.copy(t) for t in (target if isinstance(target, list) else [target])]
    for t in t1:
        t.tau_out = 1.0
    ll1 = LO.pointwise_log_lik(samples, t1 if isinstance(target, list) else t1[0])
    O_ = t1[0].widths[-1]
    c1 = 0.5 * O_ * math.log(1.0 / (2 * math.pi))
    tau = np.asarray(tau, np.float64)[:, None]
    return tau * (ll1 - c1) + 0.5 * O_ * np.log(tau / (2 * math.pi))


def log_lik_total(ll, loss, tau_out, split_sizes):
    """ll (S, N) per-row values -> (S,) the sampled likelihood term; tau_out a float or (S,)."""
    ll = np.asarray(ll, np.float64)
    if loss == 0:
        return ll.sum(1)
    tau = np.asarray(tau_out, np.float64)
    if loss == 3:
        b = np.cumsum([0] + list(split_sizes))
        return tau * sum(ll[:, b[t]:b[t + 1]].mean(1) for t in range(len(split_sizes)))
    return tau * ll.sum(1)


def weights(log_prior, log_lik, lo, hi, r_eff=1.0):
    """-> (w (4, S) in draw order, k-hat (4,)) of the sets (prior, lo), (prior, hi), (lik, lo), (lik, hi)."""
    out, ks = [], []
    for comp in (log_prior, log_lik):
        c = np.asarray(comp, np.float64).reshape(-1)
        for a in (lo, hi):
            nr = (-((a - 1.0) * c)).astype(np.float32).astype(np.float64)
            w, k = PO.psis_weights(nr, r_eff)
            out.append(w)
            ks.append(k)
    return np.stack(out), np.array(ks)


def cjs_plus(x, q):
    x = np.asarray(x, np.float64)
    S = x.size
    order = np.argsort(x, kind='stable')
    xs = x[order]
    P = np.cumsum(np.full(S, 1.0 / S))
    Q = np.cumsum(np.asarray(q, np.float64)[order])
    d = np.empty(S)
    d[:-1] = np.diff(xs)
    d[-1] = xs[-1] - xs[-2]
    with np.errstate(divide='ignore', invalid='ignore'):
        tq = np.where(Q > 0, Q * np.log2(2 * Q / (P + Q)), 0.0)
    num = (d * (P * np.log2(2 * P / (P + Q)) + tq)).sum()
    den = (d * (P + Q)).sum()
    return 0.0 if den == 0 else math.sqrt(max(num, 0.0) / den)


def cjs(x, q):
    return max(cjs_plus(x, q), cjs_plus(-np.asarray(x, np.float64), q))


def diagnose(prior, lik, thr=THRESHOLD):
    return ['potential prior-data conflict' if p >= thr and l >= thr else
            'potential strong prior / weak likelihood' if p >= thr else '-' for p, l in zip(prior, lik)]


def power_scale(cols, log_prior, log_lik, lo=0.99, hi=1.01, r_eff=1.0, thr=THRESHOLD):
    """cols (S, K) the column values (fp32 values, in fp64) -> dict of cjs (4, K), mean / sd (5, K), prior, likelihood,
    diagnosis, pareto_k (4,).  The components are columns too: pass them rounded to fp32 among ``cols``."""
    X = np.asarray(cols, np.float64)
    S, K = X.shape
    w, khat = weights(log_prior, log_lik, lo, hi, r_eff)
    c = np.full((4, K), np.nan)
    mean = np.full((5, K), np.nan)
    sd = np.full((5, K), np.nan)
    for j in range(K):
        x = X[:, j]
        if not np.isfinite(x).all():
            continue
        mean[0, j] = x.mean()
        sd[0, j] = x.std()
        for k in range(4):
            c[k, j] = cjs(x, w[k])
            m = (w[k] * x).sum()
            mean[k + 1, j] = m
            sd[k + 1, j] = math.sqrt((w[k] * (x - m) ** 2).sum())
    a, b = abs(math.log2(lo)), abs(math.log2(hi))
    prior = (c[0] / a + c[1] / b) / 2
    lik = (c[2] / a + c[3] / b) / 2
    return dict(cjs=c, mean=mean, sd=sd, prior=prior, likelihood=lik, diagnosis=diagnose(prior, lik, thr),
                pareto_k=khat, weights=w)
