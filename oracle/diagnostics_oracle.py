"""Convergence diagnostics of a multi-chain sample block, in numpy fp64: the definition the CUDA passes of
hamiltorch_b200/csrc/hmcx_diag.cu (and the host scan of hamiltorch_b200/diagnostics.py) are tested against.

Split-R-hat, effective sample size and Monte-Carlo standard error of the mean as defined by the Stan reference manual
and computed by ArviZ's ``rhat(method="split")``, ``ess(method="mean")`` and ``mcse(method="mean")``.  This is a
restatement, not a wrapper: autocovariances are direct lag sums (no FFT), evaluated lazily, only up to the lags the
Geyer scan reads.

Input ``x[c, s, d]``: C chains, n >= 4 draws, D dimensions.  Half-chain 2c is draws [0, m) of chain c and 2c+1 is
draws [n-m, n), m = n // 2 (an odd n drops the middle draw): K = 2C half-chains, N = K*m draws.

Per dimension:
  * a non-finite draw makes every float output NaN (``max_lag`` 0);
  * all N split draws equal: ESS = N, R-hat = 1, MCSE = 0 (``max_lag`` 0: no lag is read);
  * W = 0 with B > 0: R-hat = +inf and ESS follows the formula.
"""
import numpy as np


def split_chains(x):
    """(C, n, D) -> (K, m, D) float64 half-chains."""
    x = np.asarray(x, dtype=np.float64)
    if x.ndim == 2:
        x = x[None]
    C, n, D = x.shape
    if n < 4:
        raise ValueError('need at least 4 draws per chain, got %d' % n)
    m = n // 2
    halves = np.empty((2 * C, m, D))
    halves[0::2] = x[:, :m]
    halves[1::2] = x[:, n - m:]
    return halves


def autocov(y, mu, t):
    """gamma_j(t) = (1/m) sum_{s < m-t} (y_s - mu_j)(y_{s+t} - mu_j) for every half-chain j: (K, D)."""
    return autocov_centered(y - mu[:, None, :], t)


def autocov_centered(yc, t):
    """autocov() of half-chains already centred on their means."""
    m = yc.shape[1]
    if t >= m:
        return np.zeros((yc.shape[0], yc.shape[2]))
    return (yc[:, :m - t] * yc[:, t:]).sum(1) / m


def autocov_fft(y, mu):
    """All lags of autocov() at once through a zero-padded FFT (a cross-check of the direct sums)."""
    m = y.shape[1]
    yc = y - mu[:, None, :]
    f = np.fft.rfft(yc, n=2 * m, axis=1)
    return np.fft.irfft(f * np.conj(f), n=2 * m, axis=1)[:, :m] / m


def geyer(rho, m, N):
    """Geyer's initial positive then initial monotone sequence over rho(t) (a callable; rho(0) = 1), exactly as the
    Stan reference manual / ArviZ ``_ess``.  Returns (ESS, max_lag) where max_lag is the largest lag read."""
    r = np.zeros(m)
    r[0] = 1.0
    r[1] = rho(1)
    even, odd = 1.0, r[1]
    t = 1
    while t < m - 3 and even + odd > 0:                 # initial positive sequence
        even, odd = rho(t + 1), rho(t + 2)
        if even + odd >= 0:
            r[t + 1], r[t + 2] = even, odd
        t += 2
    max_t = t - 2
    if even > 0:
        r[max_t + 1] = even
    t = 1
    while t <= max_t - 2:                               # initial monotone sequence
        if r[t + 1] + r[t + 2] > r[t - 1] + r[t]:
            r[t + 1] = r[t + 2] = (r[t - 1] + r[t]) / 2
        t += 2
    tau = -1.0 + 2.0 * np.sum(r[0:max_t + 1]) + r[max_t + 1]
    ess = N / max(tau, 1.0 / np.log10(N))
    return ess, max(1, max_t + 2)


@np.errstate(invalid='ignore', over='ignore')
def summary(x):
    """dict of (D,) arrays: mean, sd, mcse, ess, rhat (float64) and max_lag (int64); plus num_chains, num_draws."""
    x = np.asarray(x, dtype=np.float64)
    if x.ndim == 2:
        x = x[None]
    y = split_chains(x)
    K, m, D = y.shape
    N = K * m
    mu = y.mean(1)                                      # (K, D)
    mubar = mu.mean(0)
    out = {k: np.full(D, np.nan) for k in ('mean', 'sd', 'mcse', 'ess', 'rhat')}
    out['max_lag'] = np.zeros(D, dtype=np.int64)
    out['num_chains'], out['num_draws'] = x.shape[0], x.shape[1]
    finite = np.isfinite(y).all(axis=(0, 1))
    yc = y - mu[:, None, :]
    cache = {}

    def gbar(t):                                        # mean_j gamma_j(t) for all dimensions, lazily
        if t not in cache:
            cache[t] = autocov_centered(yc, t).mean(0)
        return cache[t]

    g0 = gbar(0)
    between = ((mu - mubar) ** 2).sum(0)
    W = m / (m - 1) * g0
    Bm = between / (K - 1)
    varp = (m - 1) / m * W + Bm
    for d in range(D):
        if not finite[d]:
            continue
        out['mean'][d] = mubar[d]
        sd = np.sqrt((m * K * g0[d] + m * between[d]) / (N - 1))
        out['sd'][d] = sd
        if (y[:, :, d] == y[0, 0, d]).all():
            out['ess'][d], out['rhat'][d], out['mcse'][d] = N, 1.0, 0.0
            continue
        out['rhat'][d] = np.sqrt(varp[d] / W[d]) if W[d] > 0 else np.inf
        ess, lag = geyer(lambda t: 1.0 - (W[d] - gbar(t)[d]) / varp[d], m, N)
        out['ess'][d], out['max_lag'][d] = ess, lag
        out['mcse'][d] = sd / np.sqrt(ess)
    return out


# ---------------------------------------------------------------------------------------------------------------
# The per-rank partial stages (what hmcx_diag_means / hmcx_diag_acov compute), in fp64: the host logic that pools them
# over ranks (hamiltorch_b200.distributed.pooled_diagnostics) is tested on CPU with these in place of the kernels.
# ---------------------------------------------------------------------------------------------------------------
@np.errstate(invalid='ignore', over='ignore')
def partial_means(x):
    """(mu (K, D), sum_j mu_j (D,)) over this block's half-chains."""
    y = split_chains(x)
    mu = y.mean(1)
    return mu, mu.sum(0)


@np.errstate(invalid='ignore', over='ignore')
def partial_acov(x, mu, mu_bar, lag_begin, lag_block=32):
    """(sum_j gamma_j(t) for t in [lag_begin, lag_begin + lag_block) as (lag_block, D), and sum_j (mu_j - mu_bar)^2
    (D,) when mu_bar is given, else None)."""
    y = split_chains(x)
    acov = np.stack([autocov(y, mu, t).sum(0) for t in range(lag_begin, lag_begin + lag_block)])
    between = None if mu_bar is None else ((mu - mu_bar) ** 2).sum(0)
    return acov, between
