"""numpy fp64 restatement of posterior predictive checks (hamiltorch_b200/ppc.py, csrc/hmcx_ppc.cu) and of LOO-PIT
(hmcx_loo_pit_pass), built on tests/loo_oracle.py (log-likelihood, PSIS pieces) and tests/sbc_oracle.py (Philox words,
Box-Muller, the simulators' boundary conventions).

    stream      counter (x, y, z, w)              use
    ppc (8)     (v, 0, 8 << 24, g_lo)             draw g's replicate: regression normals / binary uniforms over the
                                                  flattened (N O) outputs (vector v = e / 4), multi-class u01(word x) of
                                                  vector = row; key (seed_lo, seed_hi ^ g_hi)

Statistics of a data set y (N, y_cols): regression mean, sd (ddof 1), min, max per output column, in column order;
binary the mean per column; multi-class the frequency per class; then the deviance -2 sum_i ll_i(y | theta).
p-values: P(T_rep > T_obs) + P(T_rep = T_obs) / 2, as (#greater + #equal / 2) / S.

LOO-PIT weights come from the smoothing of loo_oracle.psis_point applied in the order of the GPU's stable radix sort:
draws ascending in ll, ties by flat index; sorted position p has tail rank z = M' - p.
"""
import math

import numpy as np
from scipy import special

from tests import loo_oracle as LO
from tests import philox_ref as P
from tests import sbc_oracle as SO

STREAM_PPC = 8


def words(seed, draws, nvec):
    """(len(draws), nvec, 4) uint64 words of stream 8."""
    g = np.asarray(draws, dtype=np.uint64)[:, None]
    return P.draw(seed, g, 0, np.arange(nvec, dtype=np.uint64)[None, :], STREAM_PPC)


def replicate_regression(seed, draws, f, tau):
    """f (S, N, O), tau (S,) -> y_rep (S, N, O) fp64 = f + z / sqrt(tau_g)."""
    f = np.asarray(f, dtype=np.float64)
    n = f.shape[1] * f.shape[2]
    z = SO._normals(words(seed, draws, (n + 3) // 4), n).reshape(f.shape)
    return f + z / np.sqrt(np.asarray(tau, dtype=np.float64))[:, None, None]


def replicate_binary(seed, draws, f):
    """f (S, N, O) -> (y_rep 0 / 1, distance of each uniform to sigmoid(f))."""
    f = np.asarray(f, dtype=np.float64)
    S_, n = f.shape[0], f.shape[1] * f.shape[2]
    u = P.u01(words(seed, draws, (n + 3) // 4).reshape(S_, -1)[:, :n]).astype(np.float64).reshape(f.shape)
    p = 1.0 / (1.0 + np.exp(-f))
    return (u < p).astype(np.float64), np.abs(u - p)


def replicate_multiclass(seed, draws, f):
    """f (S, N, O) -> (labels (S, N, 1), distance of u to the nearest cumulative boundary (S, N)); softmax f for both
    multi-class losses."""
    f = np.asarray(f, dtype=np.float64)
    S_, N_, O_ = f.shape
    u = P.u01(words(seed, draws, N_)[..., 0]).astype(np.float64)
    e = np.exp(f - f.max(-1, keepdims=True))
    cdf = np.cumsum(e, -1) / e.sum(-1, keepdims=True)
    label = np.minimum((u[..., None] > cdf[..., :O_ - 1]).sum(-1), O_ - 1)
    dist = np.abs(u[..., None] - cdf[..., :O_ - 1]).min(-1) if O_ > 1 else np.full(u.shape, np.inf)
    return label[..., None].astype(np.float64), dist


def statistics(y, loss, O_):
    """y (S, N, y_cols) -> (S, K - 1) fp64 statistics (without the deviance)."""
    y = np.asarray(y, dtype=np.float64)
    if loss == 0:
        cols = [y.mean(1), y.std(1, ddof=1), y.min(1), y.max(1)]          # each (S, O)
        return np.stack(cols, -1).reshape(y.shape[0], -1)
    if loss == 1:
        return y.mean(1)
    lab = y[..., 0].astype(np.int64)
    return np.stack([(lab == c).mean(1) for c in range(O_)], 1)


def log_lik(f, y, loss, tau):
    """f (S, N, O) fp32 outputs, y (S, N, y_cols) or (N, y_cols), tau (S,) -> (S, N) fp64 ll of loo.pointwise_log_lik."""
    f = np.asarray(f, dtype=np.float64)
    y = np.broadcast_to(np.asarray(y, dtype=np.float64), f.shape[:2] + (np.shape(y)[-1],))
    if loss == 0:
        t = np.asarray(tau, dtype=np.float64)[:, None]
        return (-0.5 * t[..., None] * (f - y) ** 2).sum(-1) + 0.5 * f.shape[2] * np.log(t / (2 * math.pi))
    if loss == 1:
        return -(np.maximum(f, 0) - f * y + np.log1p(np.exp(-np.abs(f)))).sum(-1)
    lab = y[..., 0].astype(np.int64)[..., None]
    if loss == 3:
        return np.take_along_axis(f, lab, -1)[..., 0]
    mx = f.max(-1, keepdims=True)
    lsm = f - mx - np.log(np.exp(f - mx).sum(-1, keepdims=True))
    return np.take_along_axis(lsm, lab, -1)[..., 0]


def deviance(f, y, loss, tau):
    return -2.0 * log_lik(f, y, loss, tau).sum(1)


def p_values(t_rep, t_obs):
    """P(T_rep > T_obs) + P(T_rep = T_obs) / 2 per column; t_obs (K,) or (S, K)."""
    t_rep = np.asarray(t_rep, dtype=np.float64)
    t_obs = np.broadcast_to(np.asarray(t_obs, dtype=np.float64), t_rep.shape)
    return ((t_rep > t_obs).sum(0) + 0.5 * (t_rep == t_obs).sum(0)) / t_rep.shape[0]


def psis_weights(ll, r_eff=1.0):
    """One point's S draws (pooled order g) -> (normalised PSIS weights (S,) in draw order, k-hat), with the GPU's
    stable-sort tie order; NaN weights for a non-finite draw."""
    ll = np.asarray(ll, dtype=np.float64).reshape(-1)
    S = ll.size
    if not np.all(np.isfinite(ll)):
        return np.full(S, np.nan), float('nan')
    order = np.argsort(ll, kind='stable')                         # sorted position p -> draw; p = 0 the largest r
    r = -ll[order]
    r = r - r[0]
    M = LO.tail_cap(S, r_eff)
    c = max(r[M], math.log(LO.DBL_MIN))
    Mt = int((r[:M] > c).sum())
    lw = r.copy()
    khat = float('inf')
    if Mt > 4:
        x = np.exp(r[:Mt][::-1]) - math.exp(c)                    # ascending exceedances, z = 1 .. M'
        khat, sigma = LO.gpd_fit(x)
        if math.isfinite(khat):
            pz = (Mt - np.arange(Mt) - 0.5) / Mt                  # position p has z = M' - p
            q = -sigma * np.log1p(-pz) if khat == 0 else sigma * np.expm1(-khat * np.log1p(-pz)) / khat
            lw[:Mt] = np.log(q + math.exp(c))
    lw = np.minimum(lw, 0.0)
    lw = lw - LO._lse(lw)
    w = np.empty(S)
    w[order] = np.exp(lw)
    return w, khat


def loo_pit(ll, f, y, tau, r_eff=1.0):
    """ll (S, N), f (S, N, O), y (N, O), tau (S,) -> (pit (N, O), k-hat (N,)) fp64:
    pit[i, o] = sum_g w_ig Phi((y_io - f_gio) sqrt(tau_g))."""
    ll = np.asarray(ll, dtype=np.float64)
    f = np.asarray(f, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    sq = np.sqrt(np.asarray(tau, dtype=np.float64))
    N_, O_ = y.shape
    pit, kh = np.empty((N_, O_)), np.empty(N_)
    for i in range(N_):
        w, kh[i] = psis_weights(ll[:, i], r_eff)
        cdf = 0.5 * special.erfc(-((y[i][None, :] - f[:, i, :]) * sq[:, None]) / math.sqrt(2.0))   # (S, O)
        pit[i] = (w[:, None] * cdf).sum(0)
    return pit, kh


def uniformity(u, B):
    """(hist (B,), chi2, p): equal-width bins of [0, 1] (1 in the last), expected M / B, p = Q((B - 1) / 2, chi2 / 2)."""
    v = np.asarray(u, dtype=np.float64).reshape(-1)
    v = v[np.isfinite(v)]
    b = np.clip(np.floor(v * B).astype(np.int64), 0, B - 1)
    hist = np.bincount(b, minlength=B)
    e = v.size / B
    chi2 = float(((hist - e) ** 2 / e).sum())
    return hist, chi2, float(special.gammaincc((B - 1) / 2.0, chi2 / 2.0))
