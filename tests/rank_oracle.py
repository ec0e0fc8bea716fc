"""Rank-normalised diagnostics of a multi-chain sample block, in numpy / scipy fp64: the definition that
hamiltorch_b200.diagnostics.rank_summary (the rank pass of hamiltorch_b200/csrc/hmcx_rank.cu) is tested against.

Rank-normalised, folded split-R-hat, bulk-ESS and tail-ESS of Vehtari, Gelman, Simpson, Carpenter & Buerkner (2021),
as ArviZ's ``rhat(method="rank")`` / ``ess(method="bulk")`` / ``ess(method="tail")`` compute them, plus the 5 %, 50 %
and 95 % quantiles.  It reuses oracle/diagnostics_oracle.py's split-R-hat and ESS on the transformed blocks.

Input ``x[c, s, d]``: C chains, n >= 4 draws, m = n // 2.  The split set is draws s < m and s >= n - m of every chain
(K = 2C half-chains, Ns = K*m draws; an odd n drops the middle draw); the full set is all C*n draws.  Per dimension:
  * median, q05, q95: np.median / np.quantile(method='linear') over the full set;
  * bulk z: Phi^-1((r - 3/8) / (Ns + 1/4)) of the average rank r of each split draw among the split draws, rounded to
    fp32 (so the fp32 diagnostics passes read it unchanged); folded z: the same of |x - median|;
  * rhat_bulk / rhat_tail: split-R-hat of the bulk / folded z block, rhat = their maximum;
  * ess_bulk: ESS of the bulk z block; ess_tail: min(ESS(x <= q05), ESS(x <= q95)) of the 0/1 indicator blocks;
  * a non-finite draw makes every output NaN; a constant series gives ESS = Ns and R-hat = 1.
"""
import numpy as np
from scipy import special, stats

from oracle import diagnostics_oracle as O

QUANTILES = (0.05, 0.95)


def _split(x):
    """(C, n, D) fp64 -> (split draws (K*m, D) in (chain, draw) order, kept mask (n,))."""
    C, n, D = x.shape
    m = n // 2
    keep = np.zeros(n, dtype=bool)
    keep[:m] = True
    keep[n - m:] = True
    return x[:, keep].reshape(-1, D), keep


def z_scores(v):
    """Phi^-1((r - 3/8) / (N + 1/4)) of the average ranks of v (N,) fp64, rounded to fp32."""
    r = stats.rankdata(v, method='average')
    return special.ndtri((r - 0.375) / (v.size + 0.25)).astype(np.float32)


@np.errstate(invalid='ignore', over='ignore')
def rank_transform(x):
    """The per-dimension pieces of the definition: dict with q05, median, q95 (D,) fp64, bulk_z, fold_z (C, n, D)
    fp32 (0 at the dropped middle draw of an odd n) and nonfinite (D,) bool."""
    x = np.asarray(x, dtype=np.float64)
    if x.ndim == 2:
        x = x[None]
    C, n, D = x.shape
    if n < 4:
        raise ValueError('need at least 4 draws per chain, got %d' % n)
    ys, keep = _split(x)
    full = x.reshape(-1, D)
    out = {'nonfinite': ~np.isfinite(full).all(0)}
    out['median'] = np.median(full, axis=0)
    out['q05'], out['q95'] = (np.quantile(full, q, axis=0, method='linear') for q in QUANTILES)
    bulk = np.zeros((C, n, D), dtype=np.float32)
    fold = np.zeros((C, n, D), dtype=np.float32)
    for d in range(D):
        bulk[:, keep, d] = z_scores(ys[:, d]).reshape(C, -1)
        fold[:, keep, d] = z_scores(np.abs(ys[:, d] - out['median'][d])).reshape(C, -1)
    out['bulk_z'], out['fold_z'] = bulk, fold
    for k in ('median', 'q05', 'q95'):
        out[k] = np.where(out['nonfinite'], np.nan, out[k])
    return out


@np.errstate(invalid='ignore', over='ignore')
def rank_summary(x):
    """dict of (D,) fp64 arrays rhat, rhat_bulk, rhat_tail, ess_bulk, ess_tail, q05, median, q95; the blocks of the
    transform (bulk_z, fold_z); max_lag (3, D), the Geyer scan's largest lag on the bulk z, I05 and I95 series;
    num_chains, num_draws."""
    x = np.asarray(x, dtype=np.float64)
    if x.ndim == 2:
        x = x[None]
    t = rank_transform(x)
    bulk, fold = O.summary(t['bulk_z']), O.summary(t['fold_z'])
    i05 = (x <= t['q05'][None, None, :]).astype(np.float32)
    i95 = (x <= t['q95'][None, None, :]).astype(np.float32)
    s05, s95 = O.summary(i05), O.summary(i95)
    e05, e95 = s05['ess'], s95['ess']
    bad = t['nonfinite']
    nan = np.full(bad.shape, np.nan)
    out = {'rhat_bulk': bulk['rhat'], 'rhat_tail': fold['rhat'], 'ess_bulk': bulk['ess'],
           'ess_tail': np.minimum(e05, e95), 'q05': t['q05'], 'median': t['median'], 'q95': t['q95']}
    out['rhat'] = np.maximum(out['rhat_bulk'], out['rhat_tail'])
    out = {k: np.where(bad, nan, v) for k, v in out.items()}
    out['max_lag'] = np.stack([np.where(bad, 0, r['max_lag']) for r in (bulk, s05, s95)])
    out['bulk_z'], out['fold_z'] = t['bulk_z'], t['fold_z']
    out['num_chains'], out['num_draws'] = x.shape[0], x.shape[1]
    return out
